#!/usr/bin/env python
"""Kernel timeline of live Score() steps (CUPTI through torch.profiler -- there is no nsys in the image): which kernels run
beside which, how long the device idles between them, and what lies on the critical path.  Timings under the profiler carry
its per-launch overhead; read shares and overlaps, not absolutes.
usage: python scripts/timeline.py [blocks] [prompts] [out.json]"""
import collections
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "llm-d-kv-cache-manager_b200")]
import torch          # noqa: E402
from torch.profiler import profile, ProfilerActivity   # noqa: E402
import kvidx          # noqa: E402
from kvidx import synth   # noqa: E402
from bench import device_queries   # noqa: E402

nblocks = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
nq = int(sys.argv[2]) if len(sys.argv) > 2 else 1 << 20
out = sys.argv[3] if len(sys.argv) > 3 else os.path.join(ROOT, "gpurun_out", "timeline_%d.json" % nq)

wl = synth.Workload(6, 4096, nblocks, 256)
ix = kvidx.Index(capacity=wl.n_blocks + (1 << 18), max_pods=256, device=0)
for d0 in range(0, wl.D, 2048):
    ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 2048))
    assert ix.apply_events(ev, hs, tk) == (0, 0)
dev = torch.device("cuda", 0)
torch.cuda.set_device(0)
d_tok, doc, m = device_queries(wl, 0, nq, dev)
d_off = torch.arange(0, (nq + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
d_sc = torch.empty((nq, 256), dtype=torch.float64, device=dev)
torch.cuda.synchronize()


def step():
    ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), nq, d_sc.data_ptr())
    ix.synchronize()


for _ in range(3):
    step()
t0 = time.perf_counter()
for _ in range(5):
    step()
plain_ms = (time.perf_counter() - t0) / 5 * 1e3
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    step()
prof.export_chrome_trace(out.replace('.json', '_trace.json'))
ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > e.time_range.start]
ev.sort(key=lambda e: e.time_range.start)
# the second step: everything after the largest gap in the middle
starts = [e.time_range.start for e in ev]
half = len(ev) // 2
ev = ev[half:]
t_begin = min(e.time_range.start for e in ev)
t_end = max(e.time_range.end for e in ev)
span = t_end - t_begin


def short(n):
    return re.sub(r"\(.*", "", n).replace("void ", "").replace("kvx::", "")[:40]


agg = collections.defaultdict(lambda: [0, 0.0])
for e in ev:
    a = agg[short(e.name)]
    a[0] += 1
    a[1] += e.time_range.end - e.time_range.start
# sweep: time with k kernels in flight, and -- per kernel name -- the time during which it is the ONLY thing running
pts = []
for i, e in enumerate(ev):
    pts.append((e.time_range.start, 1, i))
    pts.append((e.time_range.end, -1, i))
pts.sort()
conc = collections.Counter()
alone = collections.Counter()
mix = collections.Counter()
live = set()
last = t_begin
for t, d, i in pts:
    if t > last:
        conc[len(live)] += t - last
        names = sorted({short(ev[j].name) for j in live})
        if len(live) and len(names) == 1:
            alone[names[0]] += t - last
        mix["+".join(names)] += t - last
        last = t
    if d > 0:
        live.add(i)
    else:
        live.discard(i)


def part_streams(trace_path):
    """Class pipeline, second step of the trace: per part (its kernel-G stream and its short-kernel stream, paired by launch
    order), the time within the part's own span when neither stream runs a kernel, in all and per round."""
    kern = [e for e in json.load(open(trace_path))["traceEvents"] if e.get("cat") == "kernel"]
    kern.sort(key=lambda e: e["args"]["correlation"])
    kern = kern[len(kern) // 2:]
    pair, out = {}, {}
    for a, b in zip(kern, kern[1:]):
        if "group_round" in a["name"] and "group_lists" in b["name"]:
            pair.setdefault(a["args"]["stream"], b["args"]["stream"])
    for q, (sg, ss) in enumerate(pair.items()):
        iv = sorted((e["ts"], e["ts"] + e["dur"]) for e in kern if e["args"]["stream"] in (sg, ss))
        rounds = sum(1 for e in kern if e["args"]["stream"] == sg and "group_round" in e["name"])
        busy, end = 0.0, iv[0][0]
        for s, e in iv:
            if e > end:
                busy += e - max(s, end)
                end = e
        span = iv[-1][1] - iv[0][0]
        out["part%d" % q] = {"span_ms": round(span / 1e3, 3), "idle_ms": round((span - busy) / 1e3, 3), "rounds": rounds,
                             "idle_us_per_round": round((span - busy) / max(rounds, 1), 1)}
    return out


res = {
    "what": "second of two profiled Score() steps, %d prompts, %d-block index (CUPTI via torch.profiler)" % (nq, wl.n_blocks),
    "unprofiled_step_ms": round(plain_ms, 3), "profiled_span_ms": round(span / 1e3, 3), "launches": len(ev),
    "kernels": {k: {"launches": v[0], "busy_ms": round(v[1] / 1e3, 3), "only_kind_running_ms": round(alone[k] / 1e3, 3)}
                for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1])},
    "ms_with_k_kernels_in_flight": {str(k): round(v / 1e3, 3) for k, v in sorted(conc.items())},
    "top_mixes_ms": {k or "idle": round(v / 1e3, 3) for k, v in mix.most_common(14)},
    "part_streams_idle": part_streams(out.replace('.json', '_trace.json')),
}
exp = wl.expected_scores(doc[:2048], m[:2048])
assert np.array_equal(d_sc[:2048].cpu().numpy(), exp)
os.makedirs(os.path.dirname(out), exist_ok=True)
json.dump(res, open(out, "w"), indent=1)
print(json.dumps({k: res[k] for k in ('unprofiled_step_ms', 'profiled_span_ms', 'launches', 'ms_with_k_kernels_in_flight')}))
