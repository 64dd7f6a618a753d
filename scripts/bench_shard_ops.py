#!/usr/bin/env python
"""bench_shard_ops.py -- pod removal, snapshot and restore on a hash-range sharded index: bench.py's 10 M-block / 256-pod fill
sharded over N ranks.

    torchrun --nproc-per-node N scripts/bench_shard_ops.py [--pods 1,16] [--batch 1048576]     one shard per rank and GPU
    python scripts/bench_shard_ops.py --same-gpu S [...]                                          S shards in one process, GPU 0

The index is filled through the write path as bench.py fills it, each pod's events through one rank (kvidx.dist's ingest
rule).  Then, each step timed with a host clock around calls that end synchronised, on every rank (the number given is the
slowest rank's; in the one-process layout the shards' calls run one after the other and the sum is given):
  remove      the collective removal of 1 pod, then of 16 more (phase 0 on every shard, then phase 1 on every shard);
  snapshot    every shard's snapshot of the keys it owns, and the host-side merge of the parts into one image;
  restore     the merged image into empty shards, and the same image restored and re-taken on one unsharded handle (a 1 -> N
              resharding source), restored into empty shards again.
After each step the whole resident batch of 4096-token prompts is re-scored through rank 0 (one process) or in slices
through every rank (torchrun) and checked bit-exact against the generator's closed form, with the removed pods' columns
absent, as scripts/bench_remove_pods.py does.  Prints one JSON line (rank 0) with the card's name and power limit read in
the same run; writes nothing.
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
from bench_remove_pods import expected_dense_dev, gpu_name_and_power_limit  # noqa: E402


class OneProcess:
    """S shards of one index in this process, all on GPU 0 (kvidx_shard_attach)."""

    def __init__(self, S, cfg):
        self.S, self.cfg, self.rank = S, cfg, 0
        self.shards = self.make()

    def make(self):
        import kvidx
        sh = [kvidx.Index(**self.cfg, device=0, shard_rank=r, shard_count=self.S) for r in range(self.S)]
        for r in range(self.S):
            for q in range(self.S):
                if q != r:
                    sh[r].shard_attach(q, sh[q])
        return sh

    def fill(self, ev, hs, tk):
        from kvidx import dist as kd
        for r, s in enumerate(self.shards):
            assert s.apply_events(kd.events_for_rank(ev, r, self.S), hs, tk)[0] == 0, s.last_error()

    def keys(self):
        return sum(s.stats()["request_keys"] for s in self.shards)

    def remove(self, pods):
        r0 = [s.shard_remove_pods(pods, phase=0) for s in self.shards]
        r1 = [s.shard_remove_pods(pods, phase=1) for s in self.shards]
        return {"entries": sum(r["entries"] for r in r0), "request_keys": sum(r["request_keys"] for r in r0),
                "engine_keys": sum(r["engine_keys"] for r in r1)}

    def snapshot_parts(self):
        return [s.shard_snapshot() for s in self.shards]

    def fresh_restore(self, image, timed):
        for s in self.shards:
            s.close()
        self.shards = self.make()
        t0 = time.perf_counter()
        got = [s.shard_restore(image) for s in self.shards]
        timed.append(time.perf_counter() - t0)
        return sum(g["request_keys"] for g in got)

    def rescore_ok(self, d_tok, d_off, Q, want, dev):
        import torch
        ix = self.shards[0]
        d_scores = torch.full((Q, want.shape[1]), -7.0, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, d_scores.data_ptr())
        ix.synchronize()
        return bool(torch.equal(d_scores, want))

    def slowest(self, v):
        return v


class Torchrun(OneProcess):
    """One shard per rank (torchrun), CUDA IPC between them, kvidx.dist for the collectives."""

    def __init__(self, cfg):
        import torch
        import torch.distributed as dist
        self.world, self.rank = int(os.environ["WORLD_SIZE"]), int(os.environ["RANK"])
        n = torch.cuda.device_count()
        self.dev_id = int(os.environ.get("LOCAL_RANK", self.rank)) % n
        torch.cuda.set_device(self.dev_id)
        dist.init_process_group("nccl" if n >= self.world else "gloo")
        self.tdev = torch.device("cuda", self.dev_id) if dist.get_backend() == "nccl" else None
        self.cfg = cfg
        self.shards = self.make()

    def make(self):
        import kvidx
        from kvidx import dist as kd
        ix = kvidx.Index(**self.cfg, device=self.dev_id, shard_rank=self.rank, shard_count=self.world)
        kd.connect_shards(ix, self.tdev)
        return [ix]

    def fill(self, ev, hs, tk):
        from kvidx import dist as kd
        assert self.shards[0].apply_events(kd.events_for_rank(ev, self.rank, self.world), hs, tk)[0] == 0

    def keys(self):
        from kvidx import dist as kd
        return kd._sum_over_ranks([self.shards[0].stats()["request_keys"]], self.tdev)[0]

    def remove(self, pods):
        from kvidx import dist as kd
        return kd.remove_pods_shards(self.shards[0], pods, device=self.tdev)

    def merged(self, timed):
        from kvidx import dist as kd
        t0 = time.perf_counter()
        img = kd.snapshot_shards(self.shards[0], dst=0, device=self.tdev)
        timed.append(time.perf_counter() - t0)
        return img

    def fresh_restore(self, image, timed):
        from kvidx import dist as kd
        self.shards[0].close()
        self.shards = self.make()
        t0 = time.perf_counter()
        got = kd.restore_shards(self.shards[0], image, src=0, device=self.tdev)
        timed.append(time.perf_counter() - t0)
        return got["request_keys"]

    def rescore_ok(self, d_tok, d_off, Q, want, dev):
        import torch
        from kvidx import dist as kd
        lo, hi = kd.shard_range(Q, self.rank, self.world)
        T = int(d_off[1].item())
        off = torch.arange(0, (hi - lo + 1) * T, T, dtype=torch.int64, device=dev)
        d_scores = torch.full((hi - lo, want.shape[1]), -7.0, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        self.shards[0].score_batch_dev(d_tok[lo:].data_ptr(), off.data_ptr(), hi - lo, d_scores.data_ptr())
        self.shards[0].synchronize()
        return kd._all_ok(bool(torch.equal(d_scores, want[lo:hi])), self.tdev)

    def slowest(self, v):
        from kvidx import dist as kd
        return kd.max_over_ranks(v, self.tdev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--same-gpu", type=int, default=0, help="S shards in one process on GPU 0 (else: torchrun, one shard per rank)")
    ap.add_argument("--pods", default="1,16", type=lambda v: [int(x) for x in v.split(",")])
    ap.add_argument("--batch", type=int, default=1048576)
    args = ap.parse_args()
    import torch
    import kvidx
    from kvidx import synth
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS, bench.N_PODS, bench.BLOCK)
    cfg = dict(block_size=bench.BLOCK, capacity=wl.n_blocks + (1 << 20), max_pods=wl.P, tier_weights=bench.WEIGHTS)
    ops = OneProcess(args.same_gpu, cfg) if args.same_gpu else Torchrun(cfg)
    layout = ("same-gpu", args.same_gpu) if args.same_gpu else ("torchrun", ops.world)
    dev = torch.device("cuda", 0 if args.same_gpu else ops.dev_id)
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        ops.fill(ev, hs, tk)
    assert ops.keys() == wl.n_blocks
    Q = args.batch
    d_tok, doc, m = bench.device_queries(wl, 0, Q, dev)
    d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)
    want = expected_dense_dev(wl, doc, m, bench.WEIGHTS, dev)
    assert ops.rescore_ok(d_tok, d_off, Q, want, dev), "scores differ from the closed form before any step"
    out = {"metric": "shard_ops_ms", "layout": "%s x%d" % layout, "gpu": gpu_name_and_power_limit(), "index_blocks": wl.n_blocks,
           "pods": wl.P, "batch_prompts": Q, "parity": "whole batch, closed form, after every step"}
    # removal
    legs, first = [], 0
    for K in args.pods:
        pods = list(range(first, first + K))
        first += K
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = ops.remove(pods)
        call_s = ops.slowest(time.perf_counter() - t0)
        want[:, pods] = -1.0
        assert ops.rescore_ok(d_tok, d_off, Q, want, dev), "scores after removing %d pods differ from the closed form" % K
        legs.append({"pods": K, "call_ms": call_s * 1e3, **res})
    out["remove"] = legs
    # snapshot + merge
    if args.same_gpu:
        t0 = time.perf_counter()
        parts = ops.snapshot_parts()
        t1 = time.perf_counter()
        img = kvidx.snapshot_merge(parts)
        t2 = time.perf_counter()
        out["snapshot"] = {"shard_snapshots_ms": (t1 - t0) * 1e3, "merge_ms": (t2 - t1) * 1e3, "image_bytes": len(img)}
    else:
        tm = []
        img = ops.merged(tm)
        out["snapshot"] = {"snapshot_shards_ms": ops.slowest(tm[0]) * 1e3, "image_bytes": len(img) if img is not None else None}
    # restore from the merged image, then from the image an unsharded handle gives back (1 -> N)
    tm = []
    n = ops.fresh_restore(img, tm)
    assert ops.rescore_ok(d_tok, d_off, Q, want, dev), "scores after the restore differ"
    out["restore_merged_ms"] = ops.slowest(tm[0]) * 1e3
    if ops.rank == 0:
        one = kvidx.Index(**cfg)
        one.restore(img)
        flat = one.snapshot()
        assert flat == img, "the unsharded handle's image differs from the merged one"
        one.close()
        del one
    else:
        flat = None
    tm = []
    n2 = ops.fresh_restore(flat, tm)
    assert n == n2 and ops.rescore_ok(d_tok, d_off, Q, want, dev), "scores after the 1 -> N restore differ"
    out["restore_from_unsharded_ms"] = ops.slowest(tm[0]) * 1e3
    out["restored_request_keys"] = n
    if ops.rank == 0:
        print(json.dumps(out), flush=True)
    if not args.same_gpu:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
