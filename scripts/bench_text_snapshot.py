#!/usr/bin/env python
"""bench_text_snapshot.py -- kvidx_text_store_snapshot / _restore on a full prefix store at the reference's defaults
(500 000 blocks of 256 bytes) on one GPU.

    python scripts/bench_text_snapshot.py [--tokens-per-block 60] [--runs 5]

The store is filled with seeded random text (prompts of 100 blocks) and seeded tokens, about --tokens-per-block ending
in each block.  Then, --runs times each:
  snapshot  into a pageable host buffer (pages touched beforehand) and into a pinned one, host clock around the
            synchronous call;
  restore   into a fresh store of the same shape, from either buffer, host clock around the synchronous call;
  parity    the restored store's image byte-identical to the first one.
Seconds are the median run; GB/s is image bytes over that.  The card's name and power limit are read in the same run.
Prints one JSON line; writes nothing.
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

from bench_remove_pods import gpu_name_and_power_limit  # noqa: E402

CACHE_BLOCKS, BLOCK_BYTES, BLOCKS_PER_PROMPT = 500000, 256, 100


def fill(ix, rng, per):
    """Adds 1000 prompts per call until the store holds CACHE_BLOCKS blocks."""
    from kvidx import pack_text
    nb, m = BLOCKS_PER_PROMPT, 1000
    for _ in range(CACHE_BLOCKS // (nb * m)):
        prompts = [rng.integers(0, 256, nb * BLOCK_BYTES, dtype=np.uint8).tobytes() for _ in range(m)]
        ends = np.sort(rng.integers(1, nb * BLOCK_BYTES + 1, nb * per)).astype(np.uint64)
        spans = np.tile(np.stack([ends - 1, ends], 1), (m, 1))
        tok = rng.integers(0, 1 << 32, m * nb * per, dtype=np.uint64).astype(np.uint32)
        text, off = pack_text(prompts)
        ix.text_store_add(text, off, tok, spans, np.arange(m + 1, dtype=np.int64) * nb * per)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens-per-block", type=int, default=60)
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    import kvidx

    def store():
        ix = kvidx.Index(capacity=4096, max_pods=16)
        ix.text_store_init(CACHE_BLOCKS, BLOCK_BYTES)
        return ix

    src = store()
    fill(src, np.random.default_rng(1), args.tokens_per_block)
    assert src.text_store_len() == CACHE_BLOCKS
    image = src.text_store_snapshot()
    size = len(image)
    bufs = {"pageable": np.ones(size, np.uint8), "pinned": kvidx.pinned_array((size,), np.uint8)}
    bufs["pinned"][:] = 1
    res = {"gpu": gpu_name_and_power_limit(), "blocks": CACHE_BLOCKS, "block_bytes": BLOCK_BYTES,
           "tokens": int(np.frombuffer(image, np.uint64, 1, 32)[0]), "image_bytes": size}
    got, n = C.c_uint64(0), C.c_int64(0)
    for kind, buf in bufs.items():
        ptr = buf.ctypes.data_as(C.c_void_p)
        snap, rest = [], []
        for _ in range(args.runs):
            t0 = time.perf_counter()
            rc = src.L.kvidx_text_store_snapshot(src.h, ptr, size, C.byref(got))
            snap.append(time.perf_counter() - t0)
            assert rc == 0 and got.value == size
            dst = store()
            t0 = time.perf_counter()
            rc = dst.L.kvidx_text_store_restore(dst.h, C.cast(ptr, C.c_char_p), size, C.byref(n))
            rest.append(time.perf_counter() - t0)
            assert rc == 0 and n.value == CACHE_BLOCKS
        assert buf.tobytes() == image and dst.text_store_snapshot() == image, kind
        del dst
        for name, ts in (("snapshot", snap), ("restore", rest)):
            s = float(np.median(ts))
            res["%s_%s_s" % (name, kind)] = round(s, 4)
            res["%s_%s_GBps" % (name, kind)] = round(size / s / 1e9, 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
