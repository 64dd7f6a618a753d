#!/usr/bin/env python
"""bench_score_keys.py -- Score() from request keys (kvidx_score_keys*) against Score() from tokens (kvidx_score_batch*) on
bench.py's 10 M-block / 256-pod index (one GPU).

    python scripts/bench_score_keys.py [--batches 1048576,65536,2048,32] [--runs 5] [--block-size 16]

  hash    the prompts' keys come from kvidx_hash_keys_dev once, outside the timed region; its time is reported apart;
  device  kvidx_score_keys_dev and kvidx_score_batch_dev on the same prompts, alternating, CUDA events around each call,
          medians over --runs: ms per step, their ratio, the achieved algorithmic bytes per second of each path
          (tokens: 4 T + 32 n_probe + 8 P per prompt; keys: 8 n_probe + 32 n_probe + 8 P, SURVEY 8(d)), and whether the
          two outputs are byte-identical;
  e2e     kvidx_score_keys_sparse against kvidx_score_batch_sparse from pinned host buffers (65 536 prompts), prompts/s;
  latency one prompt per host call (both paths), host clock: p50 and p99.
--block-size 64: the same token budget on a B = 64 index, where kvidx_score_batch takes the thread-per-prompt kernel.
The card's name and power limit are read in the same run.  Prints one JSON line; writes nothing.
"""
import argparse
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
from bench_remove_pods import gpu_name_and_power_limit  # noqa: E402


def same_sparse(a, b):
    """equal sparse results: counts, has_keys, and the first cnt[i] (pod, score) pairs of every row (the rest is not written)"""
    (pa, sa, ca, ha), (pb, sb, cb, hb) = a, b
    if not (np.array_equal(ca, cb) and np.array_equal(ha, hb)):
        return False
    live = np.arange(pa.shape[1])[None, :] < ca[:, None]
    return bool(np.array_equal(pa[live], pb[live]) and sa[live].tobytes() == sb[live].tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1048576,65536,2048,32")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--block-size", type=int, default=bench.BLOCK)
    ap.add_argument("--e2e-prompts", type=int, default=65536)
    args = ap.parse_args()
    import torch
    import kvidx
    from kvidx import synth
    dev = torch.device("cuda", 0)
    B = args.block_size
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS * bench.BLOCK // B, bench.N_PODS, B)
    ix = kvidx.Index(block_size=B, max_pods=wl.P, tier_weights=bench.WEIGHTS, table_slots=1 << 26, capacity=wl.n_blocks + (1 << 20))
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        assert ix.apply_events(ev, hs, tk) == (0, 0), ix.last_error()
    out = {"gpu": gpu_name_and_power_limit(), "block_size": B, "blocks": wl.n_blocks, "tokens_per_prompt": wl.T}
    st = torch.cuda.Stream(dev)
    ix.set_stream(st.cuda_stream)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(st)
        fn()
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1)

    for Q in (int(x) for x in args.batches.split(",")):
        d_tok, doc, m = bench.device_queries(wl, 0, Q, dev)
        d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
        d_koff = torch.arange(0, (Q + 1) * wl.n, wl.n, dtype=torch.int64, device=dev)
        d_keys = torch.empty(Q * wl.n, dtype=torch.int64, device=dev)
        hash_ms = timed(lambda: ix.hash_keys_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, d_koff.data_ptr(), d_keys.data_ptr()))
        o_tok = torch.empty((Q, wl.P), dtype=torch.float64, device=dev)
        o_key = torch.empty((Q, wl.P), dtype=torch.float64, device=dev)
        h_tok = torch.empty(Q, dtype=torch.uint8, device=dev)
        h_key = torch.empty(Q, dtype=torch.uint8, device=dev)
        t_tok, t_key = [], []
        for r in range(args.runs + 1):
            a = timed(lambda: ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, o_tok.data_ptr(), d_has_keys=h_tok.data_ptr()))
            b = timed(lambda: ix.score_keys_dev(d_keys.data_ptr(), d_koff.data_ptr(), Q, o_key.data_ptr(), d_has_keys=h_key.data_ptr()))
            if r:
                t_tok.append(a)
                t_key.append(b)
        torch.cuda.synchronize()
        n_probe = np.minimum(wl.n, m + 1)
        bytes_tok = float((4 * wl.T + 32 * n_probe + 8 * wl.P).sum())
        bytes_key = float((8 * n_probe + 32 * n_probe + 8 * wl.P).sum())
        mt, mk = float(np.median(t_tok)), float(np.median(t_key))
        out["step_%d" % Q] = {"tokens_ms": mt, "keys_ms": mk, "keys_over_tokens": mk / mt,
                              "tokens_GBps": bytes_tok / mt / 1e6, "keys_GBps": bytes_key / mk / 1e6,
                              "mean_n_probe": float(n_probe.mean()), "hash_keys_ms": hash_ms,
                              "identical": bool(torch.equal(o_tok.view(torch.int64), o_key.view(torch.int64)) and torch.equal(h_tok, h_key))}
        del d_tok, d_off, d_koff, d_keys, o_tok, o_key
        torch.cuda.empty_cache()
    ix.set_stream(0)
    # e2e from pinned host buffers, sparse rows
    Q = args.e2e_prompts
    toks, doc, m = wl.queries(0, Q)
    off = np.arange(0, (Q + 1) * wl.T, wl.T, dtype=np.int64)
    p_tok = kvidx.pinned_array((Q * wl.T,), np.uint32)
    p_tok[:] = toks.reshape(-1)
    keys, koff = ix.hash_keys(p_tok, off)
    p_keys = kvidx.pinned_array(keys.shape, np.uint64)
    p_keys[:] = keys
    outs = {n: tuple(kvidx.pinned_array(s, d) for s, d in (((Q, 10), np.uint16), ((Q, 10), np.float64), ((Q,), np.uint8), ((Q,), np.uint8)))
            for n in ("tokens", "keys")}
    e2e = {"tokens": [], "keys": []}
    for r in range(args.runs + 1):
        for name in ("tokens", "keys"):
            t0 = time.perf_counter()
            if name == "tokens":
                ix.score_batch_sparse(p_tok, off, out=outs[name])
            else:
                ix.score_keys_sparse(p_keys, koff, out=outs[name])
            if r:
                e2e[name].append(time.perf_counter() - t0)
    out["e2e_pinned_sparse"] = {"prompts": Q, **{"%s_prompts_per_s" % k: Q / float(np.median(v)) for k, v in e2e.items()},
                                "identical": same_sparse(outs["tokens"], outs["keys"])}
    # latency: one prompt per host call
    one = np.array([0, wl.T], np.int64)
    kone = np.array([0, wl.n], np.int64)
    lat = {"tokens": [], "keys": []}
    for r in range(512):
        t0 = time.perf_counter()
        ix.score_batch(toks[r], one)
        lat["tokens"].append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        ix.score_keys(keys[r * wl.n:(r + 1) * wl.n], kone)
        lat["keys"].append((time.perf_counter() - t0) * 1e3)
    out["latency_batch_1"] = {k: {"p50_ms": float(np.percentile(v[32:], 50)), "p99_ms": float(np.percentile(v[32:], 99))} for k, v in lat.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
