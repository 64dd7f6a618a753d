#!/usr/bin/env python
"""bench_block_size.py -- Score() from tokens at 16-, 32-, 64- and 128-token blocks: the warp-per-prompt kernels
(coop_score_kernel<B>, score_turn_kernel<B>) against the thread-per-prompt kernel (score_kernel_v1) on the index of
bench_score_keys.py --block-size B: bench.py's token budget (10 M 16-token blocks, as 10 M x 16 / B blocks), 4096-token
prompts, 256 pods, one GPU.

    python scripts/bench_block_size.py [--sizes 16,32,64,128] [--batches 1,32,256,2048,4096,8192,16384,65536] [--runs 5]

Per block size, two handles over the same events: one created under KVIDX_SCORE_PATH=coop (so batches above coop_max
also take the warp-per-prompt kernel; below it this is the default dispatch) and one under KVIDX_SCORE_KERNEL=v1.
  device   kvidx_score_batch_dev on both, alternating, CUDA events around each call, medians over --runs: ms per call,
           v1 / coop, and whether the dense rows and has_keys are byte-identical;
  latency  one prompt per host call from pinned memory (the zero-copy path), host clock: p50 and p99 of both;
  e2e      kvidx_score_batch_sparse of 2048 prompts from pinned host buffers: prompts/s of both;
  turn     kvidx_score_turn_dev, each prompt's first half held as keys and the rest new tokens, fused (coop handle) against
           composed (v1 handle), at 32 and 2048 prompts: ms per call and whether the rows are byte-identical.
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
from bench_score_keys import same_sparse  # noqa: E402


def handle(kvidx, wl, B, env):
    old = {k: os.environ.pop(k, None) for k in ("KVIDX_SCORE_PATH", "KVIDX_SCORE_KERNEL")}
    os.environ.update(env)
    try:
        ix = kvidx.Index(block_size=B, max_pods=wl.P, tier_weights=bench.WEIGHTS, table_slots=1 << 26, capacity=wl.n_blocks + (1 << 20))
    finally:
        for k in env:
            del os.environ[k]
        os.environ.update({k: v for k, v in old.items() if v is not None})
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        assert ix.apply_events(ev, hs, tk) == (0, 0), ix.last_error()
    return ix


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,32,64,128")
    ap.add_argument("--batches", default="1,32,256,2048,4096,8192,16384,65536")
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    import torch
    import kvidx
    from kvidx import synth
    dev = torch.device("cuda", 0)
    out = {"gpu": gpu_name_and_power_limit(), "tokens_per_prompt": bench.T_TOKENS, "pods": bench.N_PODS}
    st = torch.cuda.Stream(dev)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(st)
        fn()
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1)

    for B in (int(x) for x in args.sizes.split(",")):
        wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS * bench.BLOCK // B, bench.N_PODS, B)
        hs = {"coop": handle(kvidx, wl, B, {"KVIDX_SCORE_PATH": "coop"}), "v1": handle(kvidx, wl, B, {"KVIDX_SCORE_KERNEL": "v1"})}
        for ix in hs.values():
            ix.set_stream(st.cuda_stream)
        res = {"blocks": wl.n_blocks}
        # ---- device sweep ----
        for Q in (int(x) for x in args.batches.split(",")):
            d_tok, doc, m = bench.device_queries(wl, 0, Q, dev)
            d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
            o = {k: torch.empty((Q, wl.P), dtype=torch.float64, device=dev) for k in hs}
            h = {k: torch.empty(Q, dtype=torch.uint8, device=dev) for k in hs}
            t = {k: [] for k in hs}
            for r in range(args.runs + 1):
                for k, ix in hs.items():
                    ms = timed(lambda: ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, o[k].data_ptr(), d_has_keys=h[k].data_ptr()))
                    if r:
                        t[k].append(ms)
            mc, mv = float(np.median(t["coop"])), float(np.median(t["v1"]))
            res["step_%d" % Q] = {"coop_ms": mc, "v1_ms": mv, "v1_over_coop": mv / mc,
                                  "identical": bool(torch.equal(o["coop"].view(torch.int64), o["v1"].view(torch.int64)) and torch.equal(h["coop"], h["v1"]))}
            del d_tok, d_off, o, h
            torch.cuda.empty_cache()
        # ---- turns: the first half of each prompt's blocks held as keys ----
        for Q in (32, 2048):
            d_tok, doc, m = bench.device_queries(wl, 0, Q, dev)
            d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
            d_koff = torch.arange(0, (Q + 1) * wl.n, wl.n, dtype=torch.int64, device=dev)
            d_keys = torch.empty(Q * wl.n, dtype=torch.int64, device=dev)
            hs["coop"].hash_keys_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, d_koff.data_ptr(), d_keys.data_ptr())
            nh = wl.n // 2
            held = d_keys.view(Q, wl.n)[:, :nh].contiguous()
            hoff = torch.arange(0, (Q + 1) * nh, nh, dtype=torch.int64, device=dev)
            nt = d_tok[:, nh * B:].contiguous()
            toff = torch.arange(0, (Q + 1) * nt.shape[1], nt.shape[1], dtype=torch.int64, device=dev)
            o = {k: torch.empty((Q, wl.P), dtype=torch.float64, device=dev) for k in hs}
            t = {k: [] for k in hs}
            for r in range(args.runs + 1):
                for k, ix in hs.items():
                    ms = timed(lambda: ix.score_turn_dev(held.data_ptr(), hoff.data_ptr(), nt.data_ptr(), toff.data_ptr(), Q, o[k].data_ptr()))
                    if r:
                        t[k].append(ms)
            mc, mv = float(np.median(t["coop"])), float(np.median(t["v1"]))
            res["turn_%d" % Q] = {"fused_ms": mc, "composed_ms": mv, "composed_over_fused": mv / mc,
                                  "identical": bool(torch.equal(o["coop"].view(torch.int64), o["v1"].view(torch.int64)))}
        for ix in hs.values():
            ix.set_stream(0)
        # ---- host: one prompt per call (zero-copy), and 2048 pinned sparse prompts ----
        Q = 2048
        toks, doc, m = wl.queries(0, Q)
        p_tok = kvidx.pinned_array((Q * wl.T,), np.uint32)
        p_tok[:] = toks.reshape(-1)
        one = np.array([0, wl.T], np.int64)
        lat = {k: [] for k in hs}
        for r in range(544):
            for k, ix in hs.items():
                t0 = time.perf_counter()
                ix.score_batch(p_tok[r * wl.T:(r + 1) * wl.T], one)
                lat[k].append((time.perf_counter() - t0) * 1e3)
        res["latency_batch_1"] = {k: {"p50_ms": float(np.percentile(v[32:], 50)), "p99_ms": float(np.percentile(v[32:], 99))} for k, v in lat.items()}
        off = np.arange(0, (Q + 1) * wl.T, wl.T, dtype=np.int64)
        outs = {k: tuple(kvidx.pinned_array(s, d) for s, d in (((Q, 10), np.uint16), ((Q, 10), np.float64), ((Q,), np.uint8), ((Q,), np.uint8)))
                for k in hs}
        e2e = {k: [] for k in hs}
        for r in range(args.runs + 1):
            for k, ix in hs.items():
                t0 = time.perf_counter()
                ix.score_batch_sparse(p_tok, off, out=outs[k])
                if r:
                    e2e[k].append(time.perf_counter() - t0)
        res["e2e_pinned_sparse_2048"] = {**{"%s_prompts_per_s" % k: Q / float(np.median(v)) for k, v in e2e.items()},
                                         "identical": same_sparse(outs["coop"], outs["v1"])}
        out["B%d" % B] = res
        for ix in hs.values():
            ix.close()
        del hs
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
