#!/usr/bin/env python
"""Token work of the prefix-class pipeline, round by round, on bench.py's resident batch: one Score() with
KVIDX_ROUNDS_TRACE=1, its per-part trace lines summed per round.  Columns: live prompts, representatives, followers,
partial followers, chunks kernel G streams, election losers that read two chunks again in G, chunk compares in G2,
blocks kernel H hashes.  usage: python scripts/trace_rounds.py [blocks] [prompts]"""
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "llm-d-kv-cache-manager_b200")]
import torch          # noqa: E402
import kvidx          # noqa: E402
from kvidx import synth   # noqa: E402
from bench import device_queries   # noqa: E402

LINE = re.compile(r"round (\d+) part (\d+): live (\d+) -> representatives (\d+), followers (\d+), partial (\d+) .*?; "
                  r"G streamed (\d+) chunks, (\d+) losers re-read, G2 compared (\d+), H hashed (\d+) blocks")
COLS = ("live", "reps", "followers", "partial", "G chunks", "G losers", "G2 compares", "H blocks")

nblocks = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
nq = int(sys.argv[2]) if len(sys.argv) > 2 else 1 << 20
os.environ["KVIDX_ROUNDS_TRACE"] = "1"          # read at kvidx_create
wl = synth.Workload(6, 4096, nblocks, 256)
dev = torch.device("cuda", 0)
torch.cuda.set_device(0)
d_tok, doc, m = device_queries(wl, 0, nq, dev)
d_off = torch.arange(0, (nq + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
d_sc = torch.empty((nq, 256), dtype=torch.float64, device=dev)
ix = kvidx.Index(capacity=wl.n_blocks + (1 << 18), max_pods=256, device=0)
for d0 in range(0, wl.D, 2048):
    assert ix.apply_events(*wl.fill_events(d0, min(wl.D, d0 + 2048))) == (0, 0)
with tempfile.TemporaryFile(mode="w+") as f:      # the library writes the trace to file descriptor 2
    sys.stderr.flush()
    saved = os.dup(2)
    os.dup2(f.fileno(), 2)
    try:
        launches0 = ix.stats()["kernel_launches"]
        ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), nq, d_sc.data_ptr())
        torch.cuda.synchronize()
        launches = ix.stats()["kernel_launches"] - launches0
    finally:
        os.dup2(saved, 2)
        os.close(saved)
    f.seek(0)
    text = f.read()
per_round = {}
for mt in LINE.finditer(text):
    v = [int(x) for x in mt.groups()]
    row = per_round.setdefault(v[0], np.zeros(len(COLS), np.int64))
    row += np.array(v[2:], np.int64)
if not per_round:
    sys.exit("no trace lines (is this batch on the class pipeline?):\n" + text[-2000:])
print("%d prompts, %d-block index, %d kernel launches in the Score() call" % (nq, wl.n_blocks, launches))
print("round " + " ".join("%12s" % c for c in COLS) + "   (losers + G2) / G chunks")
tot = np.zeros(len(COLS), np.int64)
for r in sorted(per_round):
    v = per_round[r]
    tot += v
    print("%5d " % r + " ".join("%12d" % x for x in v) + "   %.3f" % ((v[5] + v[6]) / max(v[4], 1)))
print("  all " + " ".join("%12d" % x for x in tot) + "   %.3f" % ((tot[5] + tot[6]) / max(tot[4], 1)))
exp = wl.expected_scores(doc[:4096], m[:4096])
print("parity of the first 4096 prompts with the closed form:", np.array_equal(d_sc[:4096].cpu().numpy(), exp))
