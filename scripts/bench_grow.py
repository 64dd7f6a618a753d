#!/usr/bin/env python
"""bench_grow.py -- growable tables (grow_tables, include/kvidx.h) against fixed ones on bench.py's 10 M-block / 256-pod
index (one GPU).

    python scripts/bench_grow.py [--batch 1048576] [--runs 5]

capacity = n_blocks + 2^20, so the ceiling C is 2^26 slots, the table the other scripts use.  Two handles are filled
through kvidx_apply_events exactly as bench.py fills its index (batches of 4096 documents):
  fixed     2^26 slots from the start;
  grown     grow_tables, from 2^20 slots.
For each fill: its total time; every call that grew the tables (slots before and after, and that call's duration, host
clock around the synchronous call); the table bytes at each stage (64 B a slot: a 32-byte request slot and a 32-byte
engine slot); and the latency of single-prompt score_batch calls that a reader thread makes back to back during the fill
(p50 / p99 / max, host clock), which shows the pause a growth imposes on readers.  Then bench.py's resident Score() step
(--batch prompts, device-resident, CUDA events) on both handles, alternated --runs times, with the outputs compared byte
for byte and against the generator's closed form.  The card's name and power limit are read in the same run.  Prints one
JSON line; writes nothing.
"""
import argparse
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "llm-d-kv-cache-manager_b200"), os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (the workload generators of the benchmark, unchanged)
from bench_remove_pods import expected_dense_dev, gpu_name_and_power_limit  # noqa: E402


def pct(v):
    v = np.asarray(v)
    return {"n": int(len(v)), "p50_ms": float(np.percentile(v, 50)), "p99_ms": float(np.percentile(v, 99)), "max_ms": float(v.max())}


def fill(kvidx, wl, cfg, toks):
    """One handle filled through the write path while a reader thread scores one prompt per call.  -> (handle, report)."""
    ix = kvidx.Index(**cfg)
    one = np.array([0, wl.T], np.int64)
    stop, lat = threading.Event(), []

    def reader():
        r = 0
        while not stop.is_set():
            t0 = time.perf_counter()
            ix.score_batch(toks[r % len(toks)], one)
            t1 = time.perf_counter()
            lat.append((t0, (t1 - t0) * 1e3))
            r += 1

    slots = ix.stats()["request_slots"]
    stages, growths, calls = [{"slots": slots, "table_bytes": slots * 64}], [], []
    th = threading.Thread(target=reader, daemon=True)
    th.start()
    t_fill = time.perf_counter()
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        t0 = time.perf_counter()
        rc = ix.apply_events(ev, hs, tk)
        t1 = time.perf_counter()
        assert rc == (0, 0), ix.last_error()
        calls.append((t1 - t0) * 1e3)
        s = ix.stats()["request_slots"]
        if s != slots:
            growths.append({"slots_before": slots, "slots_after": s, "call_ms": (t1 - t0) * 1e3, "at_doc": d0, "t0": t0, "t1": t1})
            stages.append({"slots": s, "table_bytes": s * 64})
            slots = s
    t_fill = time.perf_counter() - t_fill
    stop.set()
    th.join()
    st = ix.stats()
    assert st["request_keys"] == wl.n_blocks, st
    # reader calls that started during a growing call, and every reader call of the fill
    during = [ms for t, ms in lat if any(g["t0"] <= t < g["t1"] for g in growths)]
    for g in growths:
        del g["t0"], g["t1"]
    rep = {"fill_s": t_fill, "write_calls": len(calls), "write_call_ms": pct(calls), "growths": growths, "stages": stages,
           "rebuilds": st["rebuilds"], "reader_batch_1": pct([ms for _, ms in lat[32:]])}
    if during:
        rep["reader_batch_1_started_during_a_growth"] = pct(during)
    return ix, rep


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
    base = dict(block_size=bench.BLOCK, capacity=wl.n_blocks + (1 << 20), max_pods=wl.P, tier_weights=bench.WEIGHTS)
    toks, _, _ = wl.queries(0, 512)
    out = {"metric": "grow_tables", "gpu": gpu_name_and_power_limit(), "index_blocks": wl.n_blocks, "pods": wl.P}
    a, out["fixed"] = fill(kvidx, wl, base, toks)
    b, out["grown"] = fill(kvidx, wl, dict(base, grow_tables=True), toks)
    assert out["fixed"]["stages"][-1]["slots"] == out["grown"]["stages"][-1]["slots"] == 1 << 26
    # the resident step, alternated on one stream
    st = torch.cuda.Stream(dev)
    for ix in (a, b):
        ix.set_stream(st.cuda_stream)
    Q = args.batch
    d_tok, doc, m = bench.device_queries(wl, 0, Q, dev)
    d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
    outs = {k: torch.empty((Q, wl.P), dtype=torch.float64, device=dev) for k in ("fixed", "grown")}
    res = {k: [] for k in outs}
    for r in range(args.runs + 1):
        for name, ix in (("fixed", a), ("grown", b)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(st)
            ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, outs[name].data_ptr())
            e1.record(st)
            e1.synchronize()
            if r:
                res[name].append(e0.elapsed_time(e1))
    want = expected_dense_dev(wl, doc, m, bench.WEIGHTS, dev)
    med = {k: float(np.median(v)) for k, v in res.items()}
    out["step"] = {"batch_prompts": Q, "fixed_ms": res["fixed"], "grown_ms": res["grown"], "fixed_median_ms": med["fixed"],
                   "grown_median_ms": med["grown"], "ratio": med["grown"] / med["fixed"],
                   "identical": bool(torch.equal(outs["fixed"], outs["grown"])), "bit_exact": bool(torch.equal(outs["grown"], want))}
    out["note"] = ("host clock around each synchronous write call and each single-prompt read; the reader runs on the handle "
                   "being filled; the resident step uses CUDA events on one stream, handles alternated")
    a.close()
    b.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
