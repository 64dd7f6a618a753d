#!/usr/bin/env python
"""Upper bound on what a live-list-ordered layout of the class pipeline's per-prompt state can gain.

Every per-prompt array of the class pipeline (kernels_rounds.cuh) is indexed by the prompt id, while the live list is in
the order of the round-0 radix sort by first-block fingerprint: each kernel reaches a live slot's state through
p = act[i] and gathers from scattered addresses.  This script builds bench.py's resident batch (1 048 576 prompts of 4096
tokens against the 10 M-block index) twice: as bench.py has it, and with its rows permuted into the order the library's
sort will produce (rounds_init_kernel's fingerprint, stably sorted by its top 32 bits).  The sort then returns the
identity, act[i] == i, and every gather by prompt id is monotone in list order.  Both orders are timed alternately with
CUDA events, and the scores of the permuted batch must equal the original ones row for row.

What the gap contains besides the state gathers: in the permuted batch the token rows of list neighbours are also
neighbours in memory, so the token chunks kernels G and H read are sequential too.  The gap is therefore an upper bound.

usage: python scripts/ablate_list_order.py [--blocks N] [--prompts Q] [--reps 4] [--steps 10] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "llm-d-kv-cache-manager_b200")]
import torch          # noqa: E402
import kvidx          # noqa: E402
from kvidx import synth   # noqa: E402
from bench import device_queries, _i64, BLOCK, CONFIG_ID, N_PODS, WEIGHTS   # noqa: E402

M64 = (1 << 64) - 1


def _lsr(x, k):
    return (x >> k) & ((1 << (64 - k)) - 1)


def t_mix64(x):
    """fnv_cbor.cuh mix64 on int64 tensors (uint64 arithmetic, wrapping)."""
    x = x ^ _lsr(x, 33)
    x = x * _i64(0xff51afd7ed558ccd)
    x = x ^ _lsr(x, 33)
    x = x * _i64(0xc4ceb9fe1a85ec53)
    return x ^ _lsr(x, 33)


def first_block_fingerprint(tok, block=16):
    """rounds_init_kernel's fingerprint of each row's first block (every row here has a full block), bit 63 cleared."""
    t = tok[:, :block].to(torch.int64) & 0xffffffff
    g = torch.zeros(tok.shape[0], dtype=torch.int64, device=tok.device)
    for j in range(0, block - 1, 2):
        g ^= t_mix64(((t[:, j + 1] << 32) | t[:, j]) + _i64(0xC2B2AE3D27D4EB4F * (j + 1)))
    f = t_mix64(g ^ _i64(0x9E3779B97F4A7C15))
    return f & _i64((1 << 63) - 1)


def np_fingerprint(row, block=16):
    """The same fingerprint in Python integers, to check the tensor version."""
    def mix(x):
        x &= M64
        x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & M64
        x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & M64
        return x ^ (x >> 33)
    g = 0
    for j in range(0, block - 1, 2):
        g ^= mix(((int(row[j + 1]) << 32 | int(row[j])) + 0xC2B2AE3D27D4EB4F * (j + 1)) & M64)
    return mix(0x9E3779B97F4A7C15 ^ g) & ((1 << 63) - 1)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip()
    except Exception as e:      # noqa: BLE001
        return repr(e)[:100]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=10_000_000)
    ap.add_argument("--prompts", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the result line to this JSON file")
    args = ap.parse_args()
    Q = args.prompts
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    wl = synth.Workload(CONFIG_ID, 4096, args.blocks, N_PODS, BLOCK)
    ix = kvidx.Index(block_size=BLOCK, capacity=wl.n_blocks + (1 << 20), max_pods=wl.P, tier_weights=WEIGHTS, device=0)
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        assert ix.apply_events(ev, hs, tk) == (0, 0)
    d_tok, doc, m = device_queries(wl, 0, Q, dev)
    d_off = torch.arange(0, (Q + 1) * wl.T, wl.T, dtype=torch.int64, device=dev)

    fp = first_block_fingerprint(d_tok, BLOCK)
    for r in (0, 1, Q // 2, Q - 1):
        assert np_fingerprint(d_tok[r, :BLOCK].cpu().numpy()) == int(fp[r].item()) & M64, r
    perm = torch.sort(fp >> 32, stable=True).indices
    d_tok_s = d_tok[perm].contiguous()
    moved = int((perm != torch.arange(Q, device=dev)).sum().item())
    del fp

    sc = {k: torch.empty((Q, wl.P), dtype=torch.float64, device=dev) for k in ("batch", "sorted")}
    toks = {"batch": d_tok, "sorted": d_tok_s}
    st = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(st)
    ix.set_stream(st.cuda_stream)

    def step(k):
        ix.score_batch_dev(toks[k].data_ptr(), d_off.data_ptr(), Q, sc[k].data_ptr())

    for k in ("batch", "sorted"):
        for _ in range(3):
            step(k)
    st.synchronize()
    ms = {"batch": [], "sorted": []}
    for _ in range(args.reps):
        for k in ("batch", "sorted"):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(args.steps):
                step(k)
            e1.record(st)
            e1.synchronize()
            ms[k].append(e0.elapsed_time(e1) / args.steps)
    torch.cuda.synchronize()
    exp = wl.expected_scores(doc[:4096], m[:4096], WEIGHTS)
    parity_batch = bool(np.array_equal(sc["batch"][:4096].cpu().numpy(), exp))
    same = bool(torch.equal(sc["sorted"], sc["batch"][perm]))
    mb, msr = float(np.mean(ms["batch"])), float(np.mean(ms["sorted"]))
    res = {"gpu": gpu_info(), "prompts": Q, "index_blocks": wl.n_blocks, "rows_moved_by_presort": moved,
           "step_ms_batch_order": [round(x, 4) for x in ms["batch"]], "step_ms_presorted": [round(x, 4) for x in ms["sorted"]],
           "mean_ms_batch_order": round(mb, 4), "mean_ms_presorted": round(msr, 4), "presorted_faster_pct": round(100 * (mb / msr - 1), 2),
           "closed_form_first_4096": parity_batch, "presorted_scores_equal_after_unpermuting": same}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)
    print(json.dumps(res))
    ix.set_stream(0)
    assert parity_batch and same


if __name__ == "__main__":
    main()
