#!/usr/bin/env python
"""bench_snapshot.py -- kvidx_snapshot / kvidx_restore on bench.py's 10 M-block / 256-pod index (one GPU).

    python scripts/bench_snapshot.py [--batch 1048576] [--runs 5]

The index is filled through the write path exactly as bench.py fills it.  Then, --runs times each:
  snapshot  kvidx_snapshot into a pageable host buffer (pages touched beforehand) and into a pinned one, host clock around
            the synchronous call.  A pinned buffer is written by one device copy; a pageable one through two pinned
            staging chunks and a host memcpy each, so the difference between the two is the cost of that host copy;
  restore   kvidx_restore of the image into a fresh handle of the same configuration, from either buffer, host clock around
            the call;
  parity    bench.py's resident batch of 4096-token prompts re-scored on the restored handle, bit-exact against the
            generator's closed form; and a snapshot of the restored handle byte-identical to the first image;
  copy bw   pinned host <-> device copies of 512 MB (torch, CUDA events), and one thread's host memcpy of the image from
            pinned to pageable memory, in the same run; each call is also reported as a fraction of the matching direction.
The card's name and power limit are read in the same run.  Prints one JSON line; writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "llm-d-kv-cache-manager_b200"), os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (the workload generators of the benchmark, unchanged)
from bench_remove_pods import expected_dense_dev, gpu_name_and_power_limit  # noqa: E402


def pinned_copy_gbps(torch, dev, nbytes=512 << 20, reps=5):
    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out = {}
    for name, (dst, src) in (("h2d", (d, h)), ("d2h", (h, d))):
        dst.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            dst.copy_(src, non_blocking=True)
        b.record()
        b.synchronize()
        out[name] = nbytes * reps / (a.elapsed_time(b) * 1e-3) / 1e9
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1048576)
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    import torch
    import kvidx
    from kvidx import synth
    dev = torch.device("cuda", 0)
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS, bench.N_PODS, bench.BLOCK)
    cfg = dict(block_size=bench.BLOCK, capacity=wl.n_blocks + (1 << 20), max_pods=wl.P, tier_weights=bench.WEIGHTS)
    ix = kvidx.Index(**cfg)
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        assert ix.apply_events(ev, hs, tk) == (0, 0), ix.last_error()
    st = ix.stats()
    assert st["request_keys"] == wl.n_blocks, st
    size = C.c_uint64(0)
    assert ix.L.kvidx_snapshot(ix.h, None, 0, C.byref(size)) == kvidx.ENOSPC
    n = size.value
    pageable = np.empty(n, np.uint8)
    pageable.fill(0)                                          # touch every page before the timed calls
    pinned = torch.empty(n, dtype=torch.uint8, pin_memory=True).numpy()
    pinned.fill(0)
    bufs = {"pageable": pageable, "pinned": pinned}

    def snapshot_ms(ix, buf):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rc = ix.L.kvidx_snapshot(ix.h, buf.ctypes.data_as(C.c_void_p), n, C.byref(size))
        dt = time.perf_counter() - t0
        assert rc == 0 and size.value == n, ix.last_error()
        return dt * 1e3

    snap = {k: [snapshot_ms(ix, b) for _ in range(args.runs)] for k, b in bufs.items()}
    assert np.array_equal(pageable, pinned), "the pinned and the pageable snapshot differ"
    ix.close()
    out = np.zeros(2, np.uint64)

    def restore_ms(buf, keep=False):
        t = kvidx.Index(**cfg)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rc = t.L.kvidx_restore(t.h, C.cast(buf.ctypes.data, C.c_char_p), n, out.ctypes.data_as(C.POINTER(C.c_uint64)))
        dt = time.perf_counter() - t0
        assert rc == 0 and (int(out[0]), int(out[1])) == (st["request_keys"], st["engine_keys"]), t.last_error()
        if keep:
            return dt * 1e3, t
        t.close()
        return dt * 1e3

    rest = {k: [restore_ms(b) for _ in range(args.runs - 1)] for k, b in bufs.items()}
    ms, ix2 = restore_ms(pageable, keep=True)
    rest["pageable"].append(ms)
    st2 = ix2.stats()
    assert st2["request_tombs"] == 0
    Q = args.batch
    d_tok, doc, m = bench.device_queries(wl, 0, Q, dev)
    d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
    d_scores = torch.full((Q, wl.P), -7.0, dtype=torch.float64, device=dev)
    d_has = torch.empty((Q,), dtype=torch.uint8, device=dev)
    want = expected_dense_dev(wl, doc, m, bench.WEIGHTS, dev)
    assert np.array_equal(want[:4096].cpu().numpy(), wl.expected_scores(doc[:4096], m[:4096], bench.WEIGHTS)), \
        "device closed form differs from synth.expected_scores"
    torch.cuda.synchronize()
    ix2.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, d_scores.data_ptr(), d_has_keys=d_has.data_ptr())
    ix2.synchronize()
    scores_ok = bool(torch.equal(d_scores, want))
    img2 = np.empty(n, np.uint8)
    rc = ix2.L.kvidx_snapshot(ix2.h, img2.ctypes.data_as(C.c_void_p), n, C.byref(size))
    image_ok = rc == 0 and size.value == n and np.array_equal(pageable, img2)
    bw = pinned_copy_gbps(torch, dev)
    host_copy = []                                            # one thread copying the image between pinned and pageable memory
    for _ in range(3):
        t0 = time.perf_counter()
        np.copyto(img2, pinned)
        host_copy.append(n / (time.perf_counter() - t0) / 1e9)

    def spread(v):
        return {"runs_ms": [round(x, 2) for x in v], "median_ms": float(np.median(v)), "min_ms": min(v), "max_ms": max(v)}
    res = {"metric": "snapshot_restore_ms", "gpu": gpu_name_and_power_limit(), "index_blocks": wl.n_blocks, "pods": wl.P,
           "request_keys": st["request_keys"], "engine_keys": st["engine_keys"], "image_bytes": n,
           "pinned_d2h_GBps": bw["d2h"], "pinned_h2d_GBps": bw["h2d"], "host_memcpy_pinned_to_pageable_GBps": max(host_copy)}
    for k in bufs:
        res["snapshot_" + k] = spread(snap[k])
        res["restore_" + k] = spread(rest[k])
        res["snapshot_%s_frac_of_d2h" % k] = n / (np.median(snap[k]) * 1e-3) / 1e9 / bw["d2h"]
        res["restore_%s_frac_of_h2d" % k] = n / (np.median(rest[k]) * 1e-3) / 1e9 / bw["h2d"]
    res.update({"batch_prompts": Q, "restored_scores_bit_exact": scores_ok, "restored_image_identical": bool(image_ok),
                "note": "host clock around each synchronous call; every call includes allocating and freeing its device scratch; "
                        "the first snapshot call also allocates the pinned staging chunks"})
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
