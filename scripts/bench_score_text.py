#!/usr/bin/env python
"""bench_score_text.py -- Score() from prompt text (kvidx_score_text) on bench.py's 10 M-block / 256-pod index (one GPU),
for 4096-token prompts whose text is all cached in the prefix store.  A prompt's text is its token ids' 16 384 bytes (four
bytes per token), so the store's 256-byte blocks hold 64 tokens each and the contained tokens are the prompt's tokens.

  device   kvidx_score_text from pinned text: find on the device, then the Score() dispatch (one call);
  host     the host prefix store's finds in one thread (kvhost_prefix_store_find per prompt, into pinned tokens), then
           kvidx_score_batch from the pinned tokens -- what a caller with the host store does;
  tokens   kvidx_score_batch from pinned tokens alone: the ceiling.

    python scripts/bench_score_text.py [--batches 1,32,2048,65536] [--runs 3]

Prompts/s of each way (median over --runs, host clock around synchronous calls), the time of kvidx_text_store_add for the
batch, and whether the rows and has_keys of all three are byte-identical.  The card's name and power limit are read in the
same run.  Prints one JSON line; writes nothing.
"""
import argparse
import ctypes as C
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


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,32,2048,65536")
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    import kvidx
    from kvidx import synth
    from kvidx.host import PrefixStore
    B = bench.BLOCK
    batches = [int(x) for x in args.batches.split(",")]
    wl = synth.Workload(bench.CONFIG_ID, bench.T_TOKENS, bench.N_BLOCKS, bench.N_PODS, B)
    ix = kvidx.Index(block_size=B, max_pods=wl.P, tier_weights=bench.WEIGHTS, table_slots=1 << 26, capacity=wl.n_blocks + (1 << 20))
    for d0 in range(0, wl.D, 4096):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 4096))
        assert ix.apply_events(ev, hs, tk) == (0, 0), ix.last_error()
    T, BB = wl.T, 256
    cache = max(batches) * (4 * T // BB) + 1024                     # every block of the largest batch stays resident
    ix.text_store_init(cache, BB)
    store = PrefixStore(cache_size=cache, block_size=BB)
    out = {"gpu": gpu_name_and_power_limit(), "blocks": wl.n_blocks, "tokens_per_prompt": T, "text_bytes_per_prompt": 4 * T,
           "block_bytes": BB, "batches": {}}
    spans = np.stack([np.arange(T) * 4, np.arange(T) * 4 + 4], 1).astype(np.uint64)
    for Q in batches:
        toks, _, _ = wl.queries(0, Q)
        tok = kvidx.pinned_array(Q * T, np.uint32)
        tok[:] = toks.reshape(-1)
        text = kvidx.pinned_array(Q * T * 4, np.uint8)
        text[:] = tok.view(np.uint8)
        off = np.arange(0, (Q + 1) * T * 4, T * 4, dtype=np.int64)
        toff = np.arange(0, (Q + 1) * T, T, dtype=np.int64)
        add_s, step = 0.0, 8192                                       # adds of up to 8192 prompts (512 MB of token spans each)
        for q0 in range(0, Q, step):
            q1 = min(Q, q0 + step)
            t0 = time.perf_counter()
            ix.text_store_add(text[off[q0]:off[q1]], off[q0:q1 + 1] - off[q0], tok[toff[q0]:toff[q1]], np.tile(spans, (q1 - q0, 1)),
                              toff[q0:q1 + 1] - toff[q0])
            add_s += time.perf_counter() - t0
        for i in range(Q):
            store.add_tokenization(bytes(text[off[i]:off[i + 1]]), tok[toff[i]:toff[i + 1]], spans)
        htok = kvidx.pinned_array(Q * T, np.uint32)
        ratio = C.c_double(0.0)
        find = store.L.kvhost_prefix_store_find
        base = text.ctypes.data

        def device():
            return ix.score_text(text, off, min_ratio=0.8)

        def host():
            at = 0
            for i in range(Q):
                at += find(store.h, C.c_char_p(base + int(off[i])), T * 4, C.c_void_p(htok.ctypes.data + 4 * at), Q * T - at, C.byref(ratio))
            assert at == Q * T
            return ix.score_batch(kvidx._native._Raw(htok.ctypes.data), toff)

        def tokens():
            return ix.score_batch(kvidx._native._Raw(tok.ctypes.data), toff)

        ways = {"device": device, "host": host, "tokens": tokens}
        res = {k: f() for k, f in ways.items()}                      # warm-up, and the outputs compared
        same = all(res[k][0].tobytes() == res["tokens"][0].tobytes() and res[k][1].tobytes() == res["tokens"][1].tobytes() for k in res)
        same = same and bool(res["device"][2].sum() == 0) and np.array_equal(htok, tok)
        times = {k: [] for k in ways}
        for _ in range(args.runs):
            for k, f in ways.items():
                t0 = time.perf_counter()
                f()
                times[k].append(time.perf_counter() - t0)
        row = {k + "_prompts_per_s": Q / float(np.median(v)) for k, v in times.items()}
        row.update({"text_store_add_ms": add_s * 1e3, "outputs_identical": bool(same)})
        out["batches"][str(Q)] = row
        log(Q, row)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
