#!/usr/bin/env python
"""Small-batch Score() latency (host call -> host result) per dispatch path.  Usage: python scripts/lat.py [blocks]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "llm-d-kv-cache-manager_b200")]


def run(path):
    os.environ["KVIDX_SCORE_PATH"] = path
    import kvidx
    from kvidx import synth
    nblocks = int(sys.argv[2]) if len(sys.argv) > 2 else 1 << 20
    wl = synth.Workload(6, 4096, nblocks, 256)
    ix = kvidx.Index(capacity=wl.n_blocks + (1 << 16), max_pods=256)
    for d0 in range(0, wl.D, 2048):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 2048))
        assert ix.apply_events(ev, hs, tk) == (0, 0)
    nq = 4096
    toks, doc, m = wl.queries(0, nq)
    h_tok = kvidx.pinned_array((nq * wl.T,), np.uint32)
    h_tok[:] = toks.reshape(-1)
    h_off = np.arange(0, (nq + 1) * wl.T, wl.T, dtype=np.int64)
    h_sc = kvidx.pinned_array((nq, 256), np.float64)
    exp = wl.expected_scores(doc, m)
    out = {"path": path, "m_first": int(m[0])}
    for n in (1, 8, 64, 256, 1024, 4096):
        ts = []
        for it in range(40):
            t0 = time.perf_counter()
            ix.score_batch(h_tok[: n * wl.T], h_off[: n + 1], out=h_sc[:n])
            ts.append(time.perf_counter() - t0)
        assert np.array_equal(h_sc[:n], exp[:n]), (path, n)
        ts = np.array(ts[8:]) * 1e3
        out["n%d" % n] = {"p50_ms": round(float(np.percentile(ts, 50)), 4), "p99_ms": round(float(np.percentile(ts, 99)), 4),
                          "prompts_per_s": round(n / (float(np.percentile(ts, 50)) / 1e3))}
    # full-depth single prompt (all 256 blocks hit): the worst-case chain
    td, dd, md = wl.queries(0, 1, full_depth=True)
    h_tok[: wl.T] = td.reshape(-1)
    ts = []
    for it in range(40):
        t0 = time.perf_counter()
        ix.score_batch(h_tok[: wl.T], h_off[:2], out=h_sc[:1])
        ts.append(time.perf_counter() - t0)
    assert np.array_equal(h_sc[:1], wl.expected_scores(dd, md))
    out["n1_full_depth_p50_ms"] = round(float(np.percentile(np.array(ts[8:]) * 1e3, 50)), 4)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] != "all":
        run(sys.argv[1])
    else:
        for p in ("coop", "auto"):
            subprocess.check_call([sys.executable, os.path.abspath(__file__), p] + sys.argv[2:])
