"""CPU: the C++ oracle's index image (ko_snapshot) equals the spec encoder's image of the Python oracle fed the same
events, on generated write streams of both families at every block size; it equals the golden image; and the stream
generator (tests/write_stream.py) really produces the shapes the GPU write-path tests rely on."""
import numpy as np
import pytest

from helpers import golden
from oracle import kvoracle as ko
from oracle.kvoracle_c import COracle
import snapshot_oracle as so
import write_stream as ws

BLOCK_SIZES = [1, 4, 16, 23, 24, 256]


def _py_feed(pool, B, e):
    pod, model, medium = "p%d" % e.pod, "m%d" % e.model, "T%d" % e.tier
    hs = [int(h) for h in e.hashes]
    if e.op == ws.STORED:
        pool.digest_events(pod, model, [ko.BlockStored(hs, e.parent, [int(t) for t in e.tokens], B, None, medium)])
    else:
        pool.digest_events(pod, model, [ko.BlockRemoved(hs, medium)])


def _py_image(py, B, ppk, recency, pods, models, tiers):
    return so.encode(py.index, {"m%d" % m: m for m in range(models)}, {"p%d" % p: p for p in pods},
                     {"t%d" % t: t for t in range(tiers)}, B, py.tokens_processor.init_hash(), ppk, recency=recency)


@pytest.mark.parametrize("B", BLOCK_SIZES)
@pytest.mark.parametrize("family", ["a", "a1", "b"])
def test_oracle_image_equals_python_oracle(B, family):
    rng = np.random.default_rng(B * 7 + len(family))
    pods = (0, 3, 17)
    kw = dict(max_blocks=70 if B <= 24 else 40, docs_per_pod=3 if B <= 24 else 1)
    s = ws.WriteStream(rng, B, family=family[0], pods=pods, single_queue=family == "a1", **kw)
    size, ppk = (150 if family != "b" else 10 ** 6), 6          # family "a": the key-LRU cap is reached too
    py = ko.Indexer(block_size=B, hash_seed="w", size=size, pod_cache_size=ppk)
    pool = ko.EventsPool(py.index, py.tokens_processor)
    co = COracle(block_size=B, init_hash=ko.fnv64a(b"w"), size=size, pod_cache_size=ppk, max_pods=64)
    n_ev = 40 if B <= 24 else 12
    for _ in range(3):
        batch = s.batch(n_ev)
        ev, hs, tk = ws.pack(batch)
        rc, _ = co.apply_events(ev, hs, tk)
        assert rc == 0
        for e in batch:
            _py_feed(pool, B, e)
        for rec in (False, True):
            assert co.snapshot(recency=rec) == _py_image(py, B, ppk, rec, pods, 2, 2)
    assert co.len_request() > 0 and co.len_engine() > 0


def test_oracle_image_equals_golden():
    """tests/golden/snapshot_v1.json's index (tests/golden/make_snapshot_golden.py), built through the C++ oracle."""
    d = golden("snapshot_v1.json")
    M, P, T = ({n: i for i, n in enumerate(d[k])} for k in ("models", "pods", "tiers"))
    co = COracle(block_size=d["block_size"], init_hash=d["init_hash"], size=1000, pod_cache_size=d["pods_per_key"])

    def pt(p, t):
        return (P[p] << 4) | T[t]

    def add(model, pairs, entries):
        e, r = zip(*pairs)
        assert co.add(M[model], e, r, [pt(*x) for x in entries]) == 0
    add("llama", [(0x1001, 0xA001), (0x1002, 0xA002), (0x1003, 0xA003)], [("pod-a", "gpu")])
    add("llama", [(0x1002, 0xA002)], [("pod-b", "cpu"), ("pod-a", "gpu")])
    add("qwen", [(0x1001, 0xA001), (0x2002, 0xB002)], [("pod-c", "gpu"), ("pod-c", "cpu")])
    add("qwen", [(0x2003, 0xFFFFFFFFFFFFFFF0)], [(p, "gpu") for p in d["pods"][:11]])
    add("llama", [(0x1004, 0xA004), (0x1005, 0xA004)], [("pod-b", "gpu")])
    assert co.evict(M["llama"], 0x1004, [pt("pod-b", "gpu")]) == 0
    add("llama", [(0x0FFF, 0x0001)], [("pod-c", "cpu")])
    assert co.snapshot() == bytes.fromhex(d["image_hex"])


def test_empty_oracle_image():
    co = COracle(block_size=23, init_hash=1, pod_cache_size=4)
    assert co.snapshot() == so.encode(ko.InMemoryIndex(10, 4), {}, {}, {}, 23, 1, 4)
    assert co.snapshot(recency=True) == so.encode(ko.InMemoryIndex(10, 4), {}, {}, {}, 23, 1, 4, recency=True)


def _shapes(batch, co, B):
    """What a batch holds, read from its packed arrays and the oracle state before it."""
    ev, hs, tk = ws.pack(batch)
    got = set()
    hashable = [e.hashable(B) for e in batch]
    for i, e in enumerate(batch):
        n, t = len(e.hashes), len(e.tokens)
        if e.op == ws.STORED:
            if hashable[i]:
                got.add("aligned" if ev[i]["tok_off"] % 4 == 0 else "misaligned")
                if t % B:
                    got.add("partial_tail")
                if n >= 33:
                    got.add("blocks>32")
                if n >= 65:
                    got.add("blocks>64")
                if len(set(e.hashes[:32].tolist())) < min(n, 32):
                    got.add("dup_same_pass")
                if n > 32 and set(e.hashes[32:].tolist()) & set(e.hashes[:32].tolist()):
                    got.add("dup_across_passes")
                if set(e.tokens.tolist()) & {0, 23, 24, 255, 256, 65535, 65536, 2 ** 32 - 1}:
                    got.add("edge_tokens")
            elif n == 0:
                got.add("zero_hashes_with_parent" if e.parent is not None else "zero_hashes")
            elif t < B:
                got.add("drop_short")
            elif t // B > n:
                got.add("drop_more")
            else:
                got.add("drop_less")
            if not hashable[i] or e.parent is None:
                continue
            prods = [j for j in range(i) if batch[j].op == ws.STORED and batch[j].pod == e.pod and batch[j].model == e.model
                     and e.parent in set(batch[j].hashes.tolist())]
            live = [j for j in prods if hashable[j]]
            if live:
                b = np.nonzero(batch[live[-1]].hashes == e.parent)[0][-1]
                got.add("parent_last" if b == len(batch[live[-1]].hashes) - 1 else "parent_middle")
                if len(live) >= 2:
                    got.add("parent_stored_twice")
                if any(batch[j].op == ws.REMOVED and e.parent in set(batch[j].hashes.tolist()) for j in range(live[-1] + 1, i)):
                    got.add("parent_removed_in_batch")
            elif prods:
                got.add("parent_from_dropped_event")
            elif co.peek_request_key(e.model, e.parent) is not None:
                got.add("parent_before_batch")
            else:
                got.add("parent_unknown")
        else:
            got.add("remove")
            if len(set(e.hashes.tolist())) < n:
                got.add("remove_dups")
    if len({e.model for e in batch}) > 1:
        got.add("models")
    by_hash = {}
    for e in batch:
        if e.op == ws.STORED:
            for h in e.hashes.tolist():
                by_hash.setdefault(h, set()).add(e.model)
    if any(len(m) > 1 for m in by_hash.values()):
        got.add("hash_under_two_models")
    return got


def test_generator_covers_the_grammar():
    """Family "a" at B = 16 over a few batches: every shape the write-path tests count on occurs, phase 1 mispredicts
    some events, and taking the earliest in-batch producer instead of the latest would change some predictions."""
    rng = np.random.default_rng(5)
    s = ws.WriteStream(rng, 16, family="a", pods=(0, 1, 2, 5))
    co = COracle(block_size=16, size=10 ** 6, max_pods=64)
    got, rehashed, earliest_differs = set(), 0, 0
    for _ in range(4):
        batch = s.batch(300)
        got |= _shapes(batch, co, 16)
        late = ws.phase1_predictions(co, batch, 16, 0xCBF29CE484222325)
        early = ws.phase1_predictions(co, batch, 16, 0xCBF29CE484222325, earliest=True)
        earliest_differs += sum(late[i] != early[i] for i in late)
        rehashed += ws.expect_batch(co, batch, 16, 0xCBF29CE484222325, True)[1]
    want = {"aligned", "misaligned", "partial_tail", "blocks>32", "blocks>64", "dup_same_pass", "dup_across_passes",
            "edge_tokens", "zero_hashes_with_parent", "drop_short", "drop_more", "drop_less", "parent_last", "parent_middle",
            "parent_stored_twice", "parent_removed_in_batch", "parent_from_dropped_event", "parent_before_batch",
            "parent_unknown", "remove", "remove_dups", "models", "hash_under_two_models"}
    assert want <= got, want - got
    assert rehashed > 0 and earliest_differs > 0


@pytest.mark.parametrize("B", BLOCK_SIZES)
def test_family_b_keeps_true_keys(B):
    """Family "b": every engine hash maps to its document's true request key, so phase 1 never mispredicts, and the pod
    entries of a key stay within pods_per_key."""
    rng = np.random.default_rng(B)
    pods = (0, 1, 4)
    s = ws.WriteStream(rng, B, family="b", pods=pods, max_blocks=70 if B <= 24 else 20, docs_per_pod=3 if B <= 24 else 1)
    co = COracle(block_size=B, size=10 ** 6, max_pods=64)
    ih = 0xCBF29CE484222325
    for _ in range(3):
        batch = s.batch(40)
        assert ws.expect_batch(co, batch, B, ih, True)[1] == 0
    for d in s.docs:
        keys, _ = co.hash_keys(d.blocks.reshape(-1), np.array([0, d.blocks.size], np.int64))
        for m in range(2):
            for h, k in zip(d.eh.tolist(), keys.tolist()):
                got = co.peek_request_key(m, h)
                assert got in (None, k)
    assert co.len_engine() > 0
