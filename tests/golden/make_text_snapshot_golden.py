#!/usr/bin/env python
"""Generates tests/golden/text_snapshot_v1.json: the v1 prefix store image (include/kvidx.h) of a small fixed store built
with the Python oracle (oracle/kvoracle.py::LRUTokenStore) and written by the spec encoder (tests/text_snapshot_oracle.py).
No kvidx import: the fixture pins the format's bytes independently of the library.

    python tests/golden/make_text_snapshot_golden.py

The store: 8-byte blocks, room for 6 blocks.  It holds a block without tokens (a token spans it), a block whose tokens
were rewritten by a later add, a block refreshed by a find, and has evicted the oldest blocks of the first prompt.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from oracle import kvoracle as ko  # noqa: E402
import text_snapshot_oracle as tso  # noqa: E402

CACHE_BLOCKS, BLOCK_BYTES = 6, 8


def build():
    st = ko.LRUTokenStore(CACHE_BLOCKS, BLOCK_BYTES)
    st.add_tokenization(b"The capital of France is Paris.", [10, 11, 12, 13, 14, 15, 16],
                        [(0, 3), (4, 11), (12, 14), (15, 21), (22, 24), (25, 30), (30, 31)])
    st.add_tokenization(b"A token spanning a whole block", [20, 21, 22], [(0, 1), (2, 20), (21, 30)])      # block 1 gets none
    st.add_tokenization(b"The capital of Spain is Madrid", [30, 31, 32, 33, 34, 35],
                        [(0, 3), (4, 11), (12, 14), (15, 20), (21, 23), (24, 30)])                        # rewrites block 0
    st.find_longest_contained_tokens(b"A token spanning")                                                  # refreshes 2 blocks
    return st


def main():
    st = build()
    image = tso.encode(st)
    recs = tso.decode(image, BLOCK_BYTES)
    assert len(recs) == CACHE_BLOCKS and any(not t for _, t in recs)
    doc = {"about": "v1 prefix store image (include/kvidx.h) of the oracle store built by tests/golden/make_text_snapshot_golden.py",
           "cache_blocks": CACHE_BLOCKS, "block_bytes": BLOCK_BYTES,
           "records": [{"key": k, "tokens": t} for k, t in recs], "image_hex": image.hex()}
    with open(os.path.join(HERE, "text_snapshot_v1.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
