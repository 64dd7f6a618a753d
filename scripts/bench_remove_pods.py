#!/usr/bin/env python
"""bench_remove_pods.py -- kvidx_remove_pods on bench.py's 10 M-block / 256-pod index (one GPU).

    python scripts/bench_remove_pods.py [--pods 1,16] [--batch 1048576]

The index is filled through the write path exactly as bench.py fills it and bench.py's resident batch of 4096-token prompts
is generated on the device.  Then:
  warm-up  one call with a tier mask no entry carries (tier 15): both tables are swept, nothing matches, the scratch is
           allocated -- reported as `sweep_no_match_ms`;
  legs     for each K of --pods, the next K pods are removed; the call is timed with a host clock around it (the call is
           synchronous), and the whole resident batch is re-scored and checked bit-exact against the generator's closed
           form with the removed pods' columns absent (a pod's longest-prefix score does not depend on other pods).
Bytes swept = both tables, 32 B per slot; the fraction given is of the H100 SXM data sheet's 3.35 TB/s for the WHOLE call
(bitmap clear, both sweeps, counter read-back), not a kernel's share of peak.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "llm-d-kv-cache-manager_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (the workload generators of the benchmark, unchanged)

DATASHEET_BPS = 3.35e12


def expected_dense_dev(wl, doc, m, weights, device):
    """synth.Workload.expected_scores for a whole resident batch, built on the device (a dense host copy of a 1 M-prompt
    batch would be 2 GB): the same sequential f64 sums, scattered into a (n, P) tensor."""
    import torch
    seq = np.zeros((2, wl.n + 1))
    for t in range(2):
        w, acc = max(0.0, float(weights[t])), 0.0
        for L in range(1, wl.n + 1):
            acc = acc + w if L > 1 else w
            seq[t, L] = acc
    pods = wl.doc_pods(0, wl.D)[doc]
    out = torch.full((len(doc), wl.P), -1.0, dtype=torch.float64, device=device)
    rows = np.arange(len(doc))
    for j in range(4):
        tier = (((doc * 4 + j) % 8) == 7).astype(np.int64)
        ok = (m > 0) & (pods[:, j] >= 0)
        val = seq[tier[ok], np.minimum(m, wl.depth(j))[ok]]
        out[torch.from_numpy(rows[ok]).to(device), torch.from_numpy(pods[ok, j]).to(device)] = torch.from_numpy(val).to(device)
    return out


def gpu_name_and_power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip()
    except Exception as e:      # noqa: BLE001
        return "unknown (%r)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", default="1,16", type=lambda v: [int(x) for x in v.split(",")])
    ap.add_argument("--batch", type=int, default=1048576)
    args = ap.parse_args()
    import torch
    import kvidx
    from kvidx import synth
    dev = torch.device("cuda", 0)
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS, bench.N_PODS, bench.BLOCK)
    assert sum(args.pods) <= wl.P, "more pods than the index has"
    ix = kvidx.Index(block_size=bench.BLOCK, capacity=wl.n_blocks + (1 << 20), max_pods=wl.P, tier_weights=bench.WEIGHTS)
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        assert ix.apply_events(ev, hs, tk) == (0, 0), ix.last_error()
    st = ix.stats()
    assert st["request_keys"] == wl.n_blocks, st
    swept = 32 * (st["request_slots"] + st["engine_slots"])
    Q = args.batch
    d_tok, doc, m = bench.device_queries(wl, 0, Q, dev)
    d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
    d_scores = torch.empty((Q, wl.P), dtype=torch.float64, device=dev)
    d_has = torch.empty((Q,), dtype=torch.uint8, device=dev)
    want = expected_dense_dev(wl, doc, m, bench.WEIGHTS, dev)
    assert np.array_equal(want[:4096].cpu().numpy(), wl.expected_scores(doc[:4096], m[:4096], bench.WEIGHTS)), \
        "device closed form differs from synth.expected_scores"

    def rescore_ok():
        d_scores.fill_(-7.0)
        torch.cuda.synchronize()
        ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, d_scores.data_ptr(), d_has_keys=d_has.data_ptr())
        ix.synchronize()
        return bool(torch.equal(d_scores, want))

    assert rescore_ok(), "scores differ from the closed form before any removal"
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    none = ix.remove_pods(list(range(wl.P)), tier_ids=[15])
    no_match_s = time.perf_counter() - t0
    assert none == {"entries": 0, "request_keys": 0, "engine_keys": 0}, none
    legs, first = [], 0
    for K in args.pods:
        pods = list(range(first, first + K))
        first += K
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = ix.remove_pods(pods)
        call_s = time.perf_counter() - t0
        want[:, pods] = -1.0
        ok = rescore_ok()
        assert ok, "scores after removing %d pods differ from the closed form" % K
        legs.append({"pods": K, "call_ms": call_s * 1e3, "entries": res["entries"], "request_keys": res["request_keys"],
                     "engine_keys": res["engine_keys"], "GBps_whole_call": swept / call_s / 1e9,
                     "frac_of_datasheet_whole_call": swept / call_s / DATASHEET_BPS, "parity": "whole batch, closed form"})
    print(json.dumps({"metric": "remove_pods_call_ms", "gpu": gpu_name_and_power_limit(), "index_blocks": wl.n_blocks,
                      "pods": wl.P, "batch_prompts": Q, "bytes_swept": swept, "sweep_no_match_ms": no_match_s * 1e3,
                      "legs": legs}), flush=True)


if __name__ == "__main__":
    main()
