#!/usr/bin/env python
"""bench_score_turn.py -- Score() for a conversation turn (kvidx_score_turn*) against the two ways a caller had before, on
bench.py's 10 M-block / 256-pod index (one GPU).  Each prompt of bench.py's query mix is split into held keys for its first
3/4 of blocks and tokens for the rest, and the same turn is scored three ways:

  turn      kvidx_score_turn_dev: held keys + new tokens, new keys returned (one call);
  two_call  kvidx_hash_keys_dev(new tokens, parent = last held key), the held and new keys concatenated on the device,
            then kvidx_score_keys_dev (what a caller holding its keys did before);
  tokens    kvidx_score_batch_dev on the prompts' full tokens.

    python scripts/bench_score_turn.py [--batches 32,2048,65536,1048576] [--runs 5]

  device  the three ways alternated, CUDA events around each (the two-call time includes its concatenation), medians
          over --runs, and whether every output is byte-identical: rows and has_keys of all three, new keys of the first two;
  e2e     the three from pinned host buffers at --e2e-prompts prompts (two_call: kvidx_hash_keys, a host concatenation,
          kvidx_score_keys), prompts/s;
  latency one prompt per host call, host clock: p50 and p99 of each way.
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
from bench_score_keys import same_sparse  # noqa: E402


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32,2048,65536,1048576")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--e2e-prompts", type=int, default=65536)
    args = ap.parse_args()
    import torch
    import kvidx
    from kvidx import synth
    dev = torch.device("cuda", 0)
    B = bench.BLOCK
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS, bench.N_PODS, B)
    ix = kvidx.Index(block_size=B, max_pods=wl.P, tier_weights=bench.WEIGHTS, table_slots=1 << 26, capacity=wl.n_blocks + (1 << 20))
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        assert ix.apply_events(ev, hs, tk) == (0, 0), ix.last_error()
    n, T = wl.n, wl.T
    h = 3 * n // 4                                          # held blocks per prompt
    nn = n - h                                              # new blocks per prompt
    out = {"gpu": gpu_name_and_power_limit(), "blocks": wl.n_blocks, "tokens_per_prompt": T, "held_blocks": h, "new_blocks": nn}
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

    for Q in (int(x) for x in args.batches.split(",")):
        d_tok, doc, m = bench.device_queries(wl, 0, Q, dev)
        d_off = torch.arange(0, (Q + 1) * T, T, dtype=torch.int64, device=dev)
        d_koff = torch.arange(0, (Q + 1) * n, n, dtype=torch.int64, device=dev)
        d_keys = torch.empty(Q * n, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()                            # the inputs above come from torch's stream, the hash runs on st
        ix.hash_keys_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, d_koff.data_ptr(), d_keys.data_ptr())
        torch.cuda.synchronize()
        held = d_keys.view(Q, n)[:, :h].contiguous()
        new_tok = d_tok.view(Q, T)[:, h * B:].contiguous()
        d_hoff = torch.arange(0, (Q + 1) * h, h, dtype=torch.int64, device=dev)
        d_toff = torch.arange(0, (Q + 1) * nn * B, nn * B, dtype=torch.int64, device=dev)
        d_noff = torch.arange(0, (Q + 1) * nn, nn, dtype=torch.int64, device=dev)
        parent = held[:, h - 1].contiguous()
        o = {k: torch.empty((Q, wl.P), dtype=torch.float64, device=dev) for k in ("turn", "two_call", "tokens")}
        hk = {k: torch.empty(Q, dtype=torch.uint8, device=dev) for k in o}
        nk_turn = torch.empty((Q, nn), dtype=torch.int64, device=dev)
        nk_two = torch.empty((Q, nn), dtype=torch.int64, device=dev)

        def turn():
            ix.score_turn_dev(held.data_ptr(), d_hoff.data_ptr(), new_tok.data_ptr(), d_toff.data_ptr(), Q, o["turn"].data_ptr(),
                              d_has_keys=hk["turn"].data_ptr(), d_new_key_off=d_noff.data_ptr(), d_new_keys=nk_turn.data_ptr())

        def two_call():
            ix.hash_keys_dev(new_tok.data_ptr(), d_toff.data_ptr(), Q, d_noff.data_ptr(), nk_two.data_ptr(), d_parent=parent.data_ptr())
            with torch.cuda.stream(st):
                cat = torch.cat([held, nk_two], dim=1)
            ix.score_keys_dev(cat.data_ptr(), d_koff.data_ptr(), Q, o["two_call"].data_ptr(), d_has_keys=hk["two_call"].data_ptr())
            cat.record_stream(st)

        def tokens():
            ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), Q, o["tokens"].data_ptr(), d_has_keys=hk["tokens"].data_ptr())

        ways = {"turn": turn, "two_call": two_call, "tokens": tokens}
        t = {k: [] for k in ways}
        for r in range(args.runs + 1):
            for k, fn in ways.items():
                if not r:
                    log("device step: %d prompts, %s" % (Q, k))
                ms = timed(fn)
                if r:
                    t[k].append(ms)
        torch.cuda.synchronize()
        med = {k: float(np.median(v)) for k, v in t.items()}
        same = all(torch.equal(o[k].view(torch.int64), o["tokens"].view(torch.int64)) and torch.equal(hk[k], hk["tokens"]) for k in o)
        same = same and torch.equal(nk_turn, nk_two) and torch.equal(nk_turn, d_keys.view(Q, n)[:, h:])
        out["step_%d" % Q] = {**{"%s_ms" % k: v for k, v in med.items()},
                              "turn_over_two_call": med["turn"] / med["two_call"], "turn_over_tokens": med["turn"] / med["tokens"],
                              "mean_blocks_walked": float(np.minimum(n, m + 1).mean()), "identical": bool(same)}
        del d_tok, d_off, d_koff, d_keys, held, new_tok, o, hk, nk_turn, nk_two
        torch.cuda.empty_cache()
    ix.set_stream(0)
    # e2e from pinned host buffers, sparse rows
    Q = args.e2e_prompts
    toks, doc, m = wl.queries(0, Q)
    toks = toks.reshape(Q, T)
    off = np.arange(0, (Q + 1) * T, T, dtype=np.int64)
    keys, koff = ix.hash_keys(toks.reshape(-1), off)
    keys = keys.reshape(Q, n)

    def pinned(a):
        p = kvidx.pinned_array(a.shape, a.dtype)
        p[:] = a
        return p
    p_tok, p_held, p_new = pinned(toks.reshape(-1)), pinned(keys[:, :h].reshape(-1)), pinned(toks[:, h * B:].reshape(-1))
    hoff = np.arange(0, (Q + 1) * h, h, dtype=np.int64)
    toff = np.arange(0, (Q + 1) * nn * B, nn * B, dtype=np.int64)
    parent = pinned(keys[:, h - 1].copy())
    outs = {k: tuple(kvidx.pinned_array(s, d) for s, d in (((Q, 10), np.uint16), ((Q, 10), np.float64), ((Q,), np.uint8), ((Q,), np.uint8)))
            for k in ("turn", "two_call", "tokens")}
    new_keys = {}

    def e2e_turn():
        new_keys["turn"] = ix.score_turn_sparse(p_held, hoff, p_new, toff, out=outs["turn"])[4]

    def e2e_two_call():
        nk, _ = ix.hash_keys(p_new, toff, parent=parent)
        new_keys["two_call"] = nk
        cat = np.concatenate([keys[:, :h], nk.reshape(Q, nn)], axis=1).reshape(-1)
        ix.score_keys_sparse(cat, koff, out=outs["two_call"])

    def e2e_tokens():
        ix.score_batch_sparse(p_tok, off, out=outs["tokens"])
    e2e_ways = {"turn": e2e_turn, "two_call": e2e_two_call, "tokens": e2e_tokens}
    e2e = {k: [] for k in e2e_ways}
    for r in range(args.runs + 1):
        for k, fn in e2e_ways.items():
            if not r:
                log("e2e: %d prompts, %s" % (Q, k))
            t0 = time.perf_counter()
            fn()
            if r:
                e2e[k].append(time.perf_counter() - t0)
    out["e2e_pinned_sparse"] = {"prompts": Q, **{"%s_prompts_per_s" % k: Q / float(np.median(v)) for k, v in e2e.items()},
                                "identical": bool(same_sparse(outs["turn"], outs["tokens"]) and same_sparse(outs["two_call"], outs["tokens"])
                                                  and new_keys["turn"].tobytes() == new_keys["two_call"].tobytes() == keys[:, h:].tobytes())}
    # latency: one prompt per host call, pinned inputs
    one, hone, tone = np.array([0, T], np.int64), np.array([0, h], np.int64), np.array([0, nn * B], np.int64)
    lat = {k: [] for k in e2e_ways}
    same1 = True
    log("latency")
    for r in range(512):
        ht, nt, ft = p_held[r * h:(r + 1) * h], p_new[r * nn * B:(r + 1) * nn * B], p_tok[r * T:(r + 1) * T]
        t0 = time.perf_counter()
        a = ix.score_turn(ht, hone, nt, tone)
        lat["turn"].append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        nk, _ = ix.hash_keys(nt, tone, parent=parent[r:r + 1])
        b = ix.score_keys(np.concatenate([ht, nk]), one // B)
        lat["two_call"].append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        c = ix.score_batch(ft, one)
        lat["tokens"].append((time.perf_counter() - t0) * 1e3)
        same1 = same1 and a[0].tobytes() == b[0].tobytes() == c[0].tobytes() and a[2].tobytes() == nk.tobytes()
    out["latency_batch_1"] = {k: {"p50_ms": float(np.percentile(v[32:], 50)), "p99_ms": float(np.percentile(v[32:], 99))} for k, v in lat.items()}
    out["latency_batch_1"]["identical"] = bool(same1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
