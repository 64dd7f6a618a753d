#!/usr/bin/env python
"""bench_lookup_hits.py -- what the instrumented Lookup costs (kvcache_index_* hit metrics) on bench.py's 10 M-block / 256-pod
index (one GPU).

    python scripts/bench_lookup_hits.py [--batches 1,32,2048,65536] [--dev-batches 65536,1048576] [--runs 3] [--tree A,B,...]

  host    kvhost_get_pod_scores_batch over bench.py's prompts with enable_metrics on and off (two host mirrors over the same
          events), host clock around each call, median over --runs: ms per call and prompts/s.  With --tree, the host part
          runs once per built repository tree (e.g. this one and a checkout of the parent commit), one process each, the
          trees in turn as listed (list one twice to interleave).
  device  kvidx_lookup_hits_keys_dev and kvidx_score_keys_dev on the same keys (hashed once, untimed), CUDA events, medians
          over --runs; achieved algorithmic bytes per second of the hit count: 8 B per key + 32 B per probed key (every
          key: Lookup has no early exit) + 4 B per prompt.
The card's name and power limit are read in the same run.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TREE = os.environ.get("KVIDX_BENCH_TREE", ROOT)                # the tree whose kvidx package and library are measured
for p in (ROOT, os.path.join(ROOT, "scripts"), os.path.join(ROOT, "llm-d-kv-cache-manager_b200"), TREE,
          os.path.join(TREE, "llm-d-kv-cache-manager_b200")):      # inserted in turn at the front: TREE's package wins
    if p in sys.path:
        sys.path.remove(p)
    sys.path.insert(0, p)

import bench  # noqa: E402  (the workload generators of the benchmark, unchanged)
from bench_remove_pods import gpu_name_and_power_limit  # noqa: E402


def _fill(handle, wl):
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        assert handle.apply_events(ev, hs, tk) == (0, 0), handle.last_error()


def host_part(batches, runs):
    """{batch: {"on": ms, "off": ms}} for the library this process loaded; runs alternate on / off"""
    import kvidx
    from kvidx import host as kh
    from kvidx import synth
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS, bench.N_PODS, bench.BLOCK)
    hs = {}
    for on in (True, False):
        h = kh.HostIndexer(block_size=bench.BLOCK, capacity=wl.n_blocks + (1 << 20), max_pods=wl.P, enable_metrics=on)
        for p in range(wl.P):                                  # pod ids 0 .. P-1 carry names
            h.pod_id("pod-%d" % p)
        _fill(kvidx.Index.borrow(h.L.kvhost_index(h.h), bench.BLOCK, wl.P), wl)
        hs[on] = h
    out = {}
    for Q in batches:
        toks, _, _ = wl.queries(0, Q)
        tok = np.ascontiguousarray(toks.reshape(-1), np.uint32)
        off = np.arange(0, (Q + 1) * wl.T, wl.T, dtype=np.int64)
        t = {True: [], False: []}
        for r in range(runs + 1):
            for on in (True, False):
                t0 = time.perf_counter()
                hs[on].get_pod_scores_batch(tok, off, "m")
                if r:
                    t[on].append((time.perf_counter() - t0) * 1e3)
        out[Q] = {"on_ms": float(np.median(t[True])), "off_ms": float(np.median(t[False]))}
        out[Q]["on_prompts_per_s"] = Q / out[Q]["on_ms"] * 1e3
    return out


def device_part(batches, runs):
    import torch
    import kvidx
    from kvidx import synth
    dev = torch.device("cuda", 0)
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS, bench.N_PODS, bench.BLOCK)
    ix = kvidx.Index(max_pods=wl.P, tier_weights=bench.WEIGHTS, table_slots=1 << 26, capacity=wl.n_blocks + (1 << 20))
    _fill(ix, wl)
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

    out = {}
    for Q in batches:
        d_tok, _, _ = bench.device_queries(wl, 0, Q, dev)
        d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
        d_koff = torch.arange(0, (Q + 1) * wl.n, wl.n, dtype=torch.int64, device=dev)
        d_keys = torch.empty(Q * wl.n, dtype=torch.int64, device=dev)
        ix.hash_keys_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, d_koff.data_ptr(), d_keys.data_ptr())
        del d_tok
        d_hits = torch.empty(Q, dtype=torch.int32, device=dev)
        d_rows = torch.empty((Q, wl.P), dtype=torch.float64, device=dev)
        th, ts = [], []
        for r in range(runs + 1):
            a = timed(lambda: ix.lookup_hits_keys_dev(d_keys.data_ptr(), d_koff.data_ptr(), Q, d_hits.data_ptr()))
            b = timed(lambda: ix.score_keys_dev(d_keys.data_ptr(), d_koff.data_ptr(), Q, d_rows.data_ptr()))
            if r:
                th.append(a); ts.append(b)
        nk = Q * wl.n
        ms = float(np.median(th))
        out[Q] = {"keys": nk, "lookup_hits_ms": ms, "score_keys_ms": float(np.median(ts)),
                  "lookup_hits_GBps": (8 * nk + 32 * nk + 4 * Q) / ms / 1e6,
                  "max_hits": int(d_hits.max().item())}
        del d_keys, d_rows, d_hits
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,32,2048,65536")
    ap.add_argument("--dev-batches", default="65536,1048576")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--tree", default="", help="comma-separated built repository trees: the host part runs once per tree")
    ap.add_argument("--host-only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    batches = [int(x) for x in args.batches.split(",") if x]
    if args.host_only:
        print(json.dumps(host_part(batches, args.runs)))
        return
    res = {"gpu": gpu_name_and_power_limit(), "blocks": bench.N_BLOCKS, "tokens_per_prompt": bench.T_TOKENS}
    trees = [x for x in args.tree.split(",") if x]
    if trees:
        res["host"] = []
        for tree in trees:                                     # one process per tree (each loads its own package and library)
            env = dict(os.environ, KVIDX_BENCH_TREE=os.path.abspath(tree))
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--host-only", "--batches", args.batches,
                                "--runs", str(args.runs)], env=env, capture_output=True, text=True)
            if r.returncode:
                sys.exit("host part in %s failed:\n%s" % (tree, r.stderr[-3000:]))
            res["host"].append({"tree": tree, "calls": json.loads(r.stdout.strip().splitlines()[-1])})
    else:
        res["host"] = host_part(batches, args.runs)
    res["device"] = device_part([int(x) for x in args.dev_batches.split(",") if x], args.runs)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
