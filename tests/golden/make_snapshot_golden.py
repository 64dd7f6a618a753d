#!/usr/bin/env python
"""Generates tests/golden/snapshot_v1.json: the v1 index image (include/kvidx.h) of a small fixed index built with the
Python oracle (oracle/kvoracle.py) and written by the spec encoder (tests/snapshot_oracle.py).  No kvidx import: the
fixture pins the format's bytes independently of the library.

    python tests/golden/make_snapshot_golden.py

The index: two models, three pods on two tiers, keys with 1..10 entries (one at the pod-cache cap, so its oldest entry
was dropped), a key whose entries were all evicted, and a stale engine mapping (its request key is gone, the mapping
stays: in_memory.go:225-230 cleans it up only on a later Evict).
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from oracle import kvoracle as ko  # noqa: E402
import snapshot_oracle as so  # noqa: E402

MODELS = ["llama", "qwen"]
PODS = ["pod-a", "pod-b", "pod-c"] + ["pod-%d" % i for i in range(3, 12)]
TIERS = ["gpu", "cpu"]
BLOCK_SIZE, PODS_PER_KEY = 16, 10
INIT_HASH = ko.fnv64a(b"golden")


def build():
    ix = ko.InMemoryIndex(1000, PODS_PER_KEY)

    def add(model, pairs, entries):
        ix.add([ko.Key(model, e) for e, _ in pairs], [ko.Key(model, r) for _, r in pairs],
               [ko.PodEntry(p, t) for p, t in entries])

    add("llama", [(0x1001, 0xA001), (0x1002, 0xA002), (0x1003, 0xA003)], [("pod-a", "gpu")])
    add("llama", [(0x1002, 0xA002)], [("pod-b", "cpu"), ("pod-a", "gpu")])            # pod-a refreshed to newest
    add("qwen", [(0x1001, 0xA001), (0x2002, 0xB002)], [("pod-c", "gpu"), ("pod-c", "cpu")])
    add("qwen", [(0x2003, 0xFFFFFFFFFFFFFFF0)], [(p, "gpu") for p in PODS[:11]])       # 11 pods into a 10-entry cache
    add("llama", [(0x1004, 0xA004), (0x1005, 0xA004)], [("pod-b", "gpu")])              # two engine keys -> one request key
    ix.evict(ko.Key("llama", 0x1004), [ko.PodEntry("pod-b", "gpu")])                   # A004 emptied: 0x1005 -> A004 is stale
    add("llama", [(0x0FFF, 0x0001)], [("pod-c", "cpu")])
    return ix


def main():
    ix = build()
    assert ko.Key("llama", 0xA004) not in ix.data.d and ix.engine_to_request.d[ko.Key("llama", 0x1005)] == ko.Key("llama", 0xA004)
    ids = ({m: i for i, m in enumerate(MODELS)}, {p: i for i, p in enumerate(PODS)}, {t: i for i, t in enumerate(TIERS)})
    image = so.encode(ix, *ids, BLOCK_SIZE, INIT_HASH, PODS_PER_KEY)
    doc = {"about": "v1 index image (include/kvidx.h) of the oracle index built by tests/golden/make_snapshot_golden.py",
           "models": MODELS, "pods": PODS, "tiers": TIERS, "block_size": BLOCK_SIZE, "pods_per_key": PODS_PER_KEY,
           "init_hash": INIT_HASH, "request_keys": len(ix.data), "engine_keys": len(ix.engine_to_request), "image_hex": image.hex()}
    with open(os.path.join(HERE, "snapshot_v1.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
