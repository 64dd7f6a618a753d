#!/usr/bin/env python
"""bench_clock.py -- CLOCK key cap (evict_policy="clock") on bench.py's 10 M-block / 256-pod index (one GPU).

    python scripts/bench_clock.py [--batches 1048576,65536] [--runs 5] [--churn 20]

  step    a default handle and a CLOCK handle whose capacity exceeds the contents (no eviction) score bench.py's resident
          batch of 4096-token prompts, alternating, CUDA events around each kvidx_score_batch_dev call; reports both step
          times, their ratio, and whether the two handles' outputs are byte-identical;
  churn   a CLOCK handle capped at --cap blocks (default 8 M) is filled to its cap, then takes --churn event batches of fresh
          documents (each keeps it over the cap); the same batches go to an uncapped handle.  Reports the time per batch
          (host clock around the synchronous kvidx_apply_events), the keys each batch evicted (kvidx_get_evictions), and the
          difference of the two batch times per evicted key, and how many sweeps went past a full turn of the hand
          (kvidx_get_sweeps; a sweep makes at most two turns);
  latency the batch-1 host call (kvidx_score_batch, the zero-copy path) on both handles of the step measurement,
          alternating, host clock: p50 and p99.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1048576,65536")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--cap", type=int, default=8 << 20)
    ap.add_argument("--churn", type=int, default=20)
    args = ap.parse_args()
    import torch
    import kvidx
    from kvidx import synth
    dev = torch.device("cuda", 0)
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS, bench.N_PODS, bench.BLOCK)
    base = dict(block_size=bench.BLOCK, max_pods=wl.P, tier_weights=bench.WEIGHTS, table_slots=1 << 26)
    big = wl.n_blocks + (1 << 20)

    def filled(**kw):
        ix = kvidx.Index(**base, **kw)
        for d0 in range(0, wl.D, 4096):
            ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
            assert ix.apply_events(ev, hs, tk) == (0, 0), ix.last_error()
        return ix

    out = {"gpu": gpu_name_and_power_limit()}
    a, b = filled(capacity=big), filled(capacity=big, evict_policy="clock")
    st = torch.cuda.Stream(dev)                               # both handles score on the stream the CUDA events are recorded on
    for ix in (a, b):
        ix.set_stream(st.cuda_stream)
    for Q in (int(x) for x in args.batches.split(",")):
        d_tok, doc, m = bench.device_queries(wl, 0, Q, dev)
        d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
        res = {}
        outs = {}
        for name, ix in (("default", a), ("clock", b)):
            outs[name] = torch.empty((Q, wl.P), dtype=torch.float64, device=dev)
            res[name] = []
        for r in range(args.runs + 1):
            for name, ix in (("default", a), ("clock", b)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record(st)
                ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, outs[name].data_ptr())
                e1.record(st)
                e1.synchronize()
                if r:
                    res[name].append(e0.elapsed_time(e1))
        torch.cuda.synchronize()
        med = {k: float(np.median(v)) for k, v in res.items()}
        out["step_%d" % Q] = {"default_ms": med["default"], "clock_ms": med["clock"], "ratio": med["clock"] / med["default"],
                              "identical": bool(torch.equal(outs["default"], outs["clock"])), "evictions": b.evictions()}
        del d_tok, d_off, outs
    # latency: one prompt per host call (the zero-copy cooperative kernel), default against CLOCK
    toks, doc, m = wl.queries(0, 512)
    one = np.array([0, wl.T], np.int64)
    lat = {"default": [], "clock": []}
    for r in range(512):
        for name, ix in (("default", a), ("clock", b)):
            t0 = time.perf_counter()
            ix.score_batch(toks[r], one)
            lat[name].append((time.perf_counter() - t0) * 1e3)
    out["latency_batch_1"] = {k: {"p50_ms": float(np.percentile(v[32:], 50)), "p99_ms": float(np.percentile(v[32:], 99))} for k, v in lat.items()}
    a.close()
    b.close()
    # churn: capped CLOCK handle against an uncapped one, the same fresh-document batches
    cap = args.cap
    c = kvidx.Index(**base, capacity=cap, evict_policy="clock")
    u = kvidx.Index(**base, capacity=big)
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        for ix in (c, u):
            assert ix.apply_events(ev, hs, tk) == (0, 0), ix.last_error()
    times = {"clock": [], "uncapped": []}
    ev_before, sw_before = c.evictions(), c.sweeps()
    rng = np.random.default_rng(1)
    for i in range(args.churn):
        d0 = int(rng.integers(0, wl.D - 4096))
        ev, hs, tk = wl.fill_events(d0, d0 + 4096)
        hs = hs ^ np.uint64(0x9E3779B97F4A7C15 * (i + 1) & ((1 << 64) - 1))   # fresh engine hashes: fresh mappings
        tk = tk.copy()
        tk[::bench.BLOCK] += np.uint32(i + 1)                                 # fresh tokens: fresh request keys
        for name, ix in (("clock", c), ("uncapped", u)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rc = ix.apply_events(ev, hs, tk)
            times[name].append((time.perf_counter() - t0) * 1e3)
            if name == "uncapped" and rc[0] == kvidx.ENOSPC:
                times[name].pop()
    st = c.stats()
    evs = c.evictions()
    sws = c.sweeps()
    n_ev = evs[0] - ev_before[0]
    tc, tu = float(np.median(times["clock"])), float(np.median(times["uncapped"])) if times["uncapped"] else float("nan")
    out["churn"] = {"cap": cap, "batches": args.churn, "clock_ms_per_batch": tc, "uncapped_ms_per_batch": tu,
                    "request_keys": st["request_keys"], "engine_keys": st["engine_keys"],
                    "evicted_request_keys": n_ev, "evicted_engine_keys": evs[1] - ev_before[1],
                    "sweeps": sws[0] - sw_before[0], "sweeps_past_a_full_turn": sws[1] - sw_before[1],
                    "sweep_ns_per_evicted_key": (tc - tu) * 1e6 / max(n_ev / args.churn, 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
