#!/usr/bin/env python
"""bench_inventory.py -- kvidx_pod_inventory on bench.py's 10 M-block / 256-pod index (one GPU).

    python scripts/bench_inventory.py [--reps 9]

The index is filled through the write path exactly as bench.py fills it.  Both forms of the call -- the request pass alone,
and with the engine pass -- are checked against the generator's closed form (synth.Workload.expected_inventory: every
entries / keys / sole / sole_engine / totals value), warmed up, and timed --reps times two ways:
  call_ms     host clock around the synchronous call (scratch clear, kernels, read-back of the histograms, copies out);
  stream_ms   CUDA events recorded on the handle's stream before and after the call: the scratch clear, the kernels and
              the read-back as the device ran them.
Medians are reported.  Bytes swept = 32 B per slot of the tables the call streams (the engine pass also issues one random
64-byte probe per resident mapping, not counted); the fraction given is of the H100 SXM data sheet's 3.35 TB/s for the WHOLE
call, not a kernel's share of peak.  `remove_pods_no_match_ms` is the nearest relative: kvidx_remove_pods sweeping both
tables without a match.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "llm-d-kv-cache-manager_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (the workload generators of the benchmark, unchanged)
from bench_remove_pods import DATASHEET_BPS, gpu_name_and_power_limit  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    args = ap.parse_args()
    assert args.reps >= 5
    import torch
    import kvidx
    from kvidx import synth
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS, bench.N_PODS, bench.BLOCK)
    ix = kvidx.Index(block_size=bench.BLOCK, capacity=wl.n_blocks + (1 << 20), max_pods=wl.P, tier_weights=bench.WEIGHTS)
    stream = torch.cuda.Stream()
    ix.set_stream(stream.cuda_stream)                       # so that the events below sit on the stream the kernels run on
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        assert ix.apply_events(ev, hs, tk) == (0, 0), ix.last_error()
    st = ix.stats()
    assert st["request_keys"] == wl.n_blocks, st
    want = wl.expected_inventory()
    legs = []
    for engine in (False, True):
        got = ix.pod_inventory(None, engine)                # warm-up, and the check
        for k in ("entries", "keys", "sole", "totals") + (("sole_engine",) if engine else ()):
            w = want[k] if engine or k != "totals" else np.append(want[k][:2], [0, 0]).astype(np.uint64)
            assert np.array_equal(got[k], w), (engine, k)
        call, kern = [], []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(stream)
            t0 = time.perf_counter()
            ix.pod_inventory(None, engine)
            call.append((time.perf_counter() - t0) * 1e3)
            e1.record(stream)
            e1.synchronize()
            kern.append(e0.elapsed_time(e1))
        swept = 32 * (st["request_slots"] + (st["engine_slots"] if engine else 0))
        c, k = statistics.median(call), statistics.median(kern)
        legs.append({"engine_pass": engine, "call_ms_median": c, "call_ms_min_max": [min(call), max(call)], "stream_ms_median": k,
                     "bytes_swept": swept, "GBps_whole_call": swept / c / 1e6, "frac_of_datasheet_whole_call": swept / (c / 1e3) / DATASHEET_BPS,
                     "GBps_stream": swept / k / 1e6, "parity": "closed form, every output"})
    for _ in range(2):                                      # the first call allocates the removal's bitmaps
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        none = ix.remove_pods(list(range(wl.P)), tier_ids=[15])
        no_match_ms = (time.perf_counter() - t0) * 1e3
        assert none == {"entries": 0, "request_keys": 0, "engine_keys": 0}, none
    print(json.dumps({"metric": "pod_inventory_call_ms", "gpu": gpu_name_and_power_limit(), "index_blocks": wl.n_blocks, "pods": wl.P,
                      "request_slots": st["request_slots"], "engine_slots": st["engine_slots"], "reps": args.reps, "legs": legs,
                      "remove_pods_no_match_ms": no_match_ms}), flush=True)


if __name__ == "__main__":
    main()
