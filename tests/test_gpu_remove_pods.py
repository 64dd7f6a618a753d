"""GPU (-m gpu): kvidx_remove_pods / kvhost_remove_pod -- removing departed pods -- bit-exact against the Python oracle
with the removal spec of tests/remove_oracle.py, beside concurrent readers, under churn, and through the host mirror and ZMQ ingest."""
import threading
import time

import msgpack
import numpy as np
import pytest

from helpers import EVENT_DTYPE, SEED_ORDER_SIZES, csr
import kvidx
from kvidx.host import HostIndexer
from oracle import kvoracle as ko
from remove_oracle import ClearingEventsPool, remove_pods
from test_gpu_parity import _random_stream, _select_path

pytestmark = pytest.mark.gpu
MODEL = "m"
TIERS = ("gpu", "cpu", "t2")
W = (1.0, 0.8, 0.3)


def PT(p, t=0):
    return (p << 4) | t


def _pair(P=16, capacity=1 << 16, lru_exact=0, BS=16):
    ix = kvidx.Index(block_size=BS, hash_seed="abc", capacity=capacity, pods_per_key=4, tier_weights=W, max_pods=P, lru_exact=lru_exact)
    ox = ko.Indexer(block_size=BS, hash_seed="abc", size=capacity if lru_exact else 10 ** 8, pod_cache_size=4, weights=dict(zip(TIERS, W)))
    return ix, ox, ko.EventsPool(ox.index, ox.tokens_processor)


def _oracle_apply(pool, r, hs, tk):
    pod, med = "p%d" % (int(r["podtier"]) >> 4), TIERS[int(r["podtier"]) & 15]
    h = [int(x) for x in hs[r["hash_off"]: r["hash_off"] + r["n_hashes"]]]
    if r["op"] == 0:
        toks = [int(x) for x in tk[r["tok_off"]: r["tok_off"] + r["n_tokens"]]]
        ev = ko.BlockStored(h, int(r["parent_hash"]) if r["has_parent"] else None, toks, medium=med)
    else:
        ev = ko.BlockRemoved(h, medium=med)
    pool.digest_events(pod, MODEL, [ev])


def _remove_both(ix, ox, rng, P, NT):
    pods = sorted(rng.choice(P, size=int(rng.integers(1, 4)), replace=False).tolist())
    tiers = None if rng.random() < 0.5 else sorted(rng.choice(NT, size=int(rng.integers(1, NT + 1)), replace=False).tolist())
    got = ix.remove_pods(pods, tiers)
    want = remove_pods(ox.index, {"p%d" % p for p in pods}, None if tiers is None else {TIERS[t] for t in tiers})
    assert (got["entries"], got["request_keys"], got["engine_keys"]) == want, (pods, tiers)
    return want


def _dense(scores, P):
    row = np.full(P, -1.0)
    for pod, s in (scores or {}).items():
        row[int(pod[1:])] = s
    return row


def _check_state(ix, ox, seen, engine_keys):
    st = ix.stats()
    assert st["request_keys"] == len(ox.index.data) and st["engine_keys"] == len(ox.index.engine_to_request)
    keys = sorted(seen)
    rc, pt, cnt = ix.lookup(0, np.array(keys, np.uint64))
    want = ox.index.lookup([ko.Key(MODEL, k) for k in keys])
    assert rc == 0
    for i, k in enumerate(keys):
        got = [(int(e) >> 4, int(e) & 15) for e in pt[i, :cnt[i]]]
        assert got == [(int(e.pod[1:]), TIERS.index(e.tier)) for e in want.get(ko.Key(MODEL, k), [])], k
    for e in engine_keys:
        rc, r = ix.get_request_key(0, e)
        try:
            exp = ox.index.get_request_key(ko.Key(MODEL, e)).chunk_hash
        except ko.IndexError_:
            exp = None
        assert (rc, r) == (0, exp) if exp is not None else rc == kvidx.ENOENT, e


def _oracle_scores(ox, keys):
    """Indexer.get_pod_scores after the prompt's keys are computed (computed once per prompt: the hash is not under test)."""
    return ox.scorer.score(keys, ox.index.lookup(keys, set())) if keys else None


def _prompts(rng, docs, n, BS):
    out = []
    for _ in range(n):
        d = docs[int(rng.integers(0, len(docs)))]
        out.append(d[:BS * int(rng.integers(0, len(d) // BS + 1))] + rng.integers(0, 128256, size=int(rng.integers(0, 20))).tolist())
    return out


# batch sizes on both sides of the dispatch thresholds: 2048 / 2049 prompts straddle the cooperative kernel's limit and the
# round pipeline's start; "auto" lowers the class pipeline's start to 64 prompts (tests/test_gpu_parity.py _select_path)
PATH_SIZES = {"v1": (1, 32), "coop": (1, 32), "rounds": (1, 32), "classes": (1, 32), "default": (2048, 2049),
              "auto": (63, 64)}


@pytest.mark.parametrize("path", list(PATH_SIZES))
def test_random_stream_with_removals_vs_oracle(path, monkeypatch):
    """Random BlockStored / BlockRemoved streams (one event per call: the oracle's linearisation) interleaved with removals
    of random pod sets and tier masks.  After every removal: the removed counts, Lookup of every key ever added,
    GetRequestKey of every engine key, the key counts and Score() on the path are bit-exact against the oracle."""
    if path != "default":
        _select_path(monkeypatch, path)
    rng = np.random.default_rng(SEED_ORDER_SIZES.index(path) + 70)
    BS, P, NT = 16, 12, 3
    ix, ox, pool = _pair(P=16)
    docs = [rng.integers(0, 128256, size=BS * int(rng.integers(1, 30))).tolist() for _ in range(24)]
    for i in range(8, 24):
        docs[i] = docs[i % 8][:BS * int(rng.integers(1, 6))] + docs[i]
    ev, hs, tk = _random_stream(rng, 400, BS, P, NT, docs)
    prompts = _prompts(rng, docs, 32, BS)
    pkeys = [ox.tokens_processor.tokens_to_kv_block_keys(None, p, MODEL) for p in prompts]
    tok_off = {n: csr([prompts[i % len(prompts)] for i in range(n)]) for n in PATH_SIZES[path]}
    seen, engine_keys = set(), sorted({int(x) for x in hs})
    removed = np.zeros(3, np.int64)
    for step in range(25):
        for i in range(16 * step, 16 * (step + 1)):
            assert ix.apply_events(ev[i:i + 1], hs, tk)[0] == 0
            _oracle_apply(pool, ev[i], hs, tk)
            seen |= {k.chunk_hash for k in ox.index.data.d}
        removed += _remove_both(ix, ox, rng, P, NT)
        _check_state(ix, ox, seen, engine_keys)
        want = np.stack([_dense(_oracle_scores(ox, k), 16) for k in pkeys])
        for n, (tok, off) in tok_off.items():
            s, has = ix.score_batch(tok, off)
            assert np.array_equal(s, want[np.arange(n) % len(prompts)]), (step, n, np.argwhere(s != want[np.arange(n) % len(prompts)])[:4])
    assert (removed > 0).all(), removed                   # entries, whole keys and engine mappings were all removed


def test_exact_lru_stream_with_removals_vs_capped_oracle():
    """Size-capped index (exact-LRU mode) under single-block events, Score() / Lookup calls (which refresh recency) and
    removals (which refresh nothing): later cap evictions must pick the oracle's victims."""
    rng = np.random.default_rng(43)
    BS, P, NT, CAP = 16, 10, 2, 40
    ix, ox, pool = _pair(P=16, capacity=CAP, lru_exact=1)
    docs = [rng.integers(0, 128256, size=BS * int(rng.integers(2, 9))).tolist() for _ in range(14)]
    seen, engine_keys = set(), sorted({d * 1000 + b for d in range(len(docs)) for b in range(len(docs[d]) // BS)})
    n_removed = 0
    for step in range(600):
        d = int(rng.integers(0, len(docs))); b = int(rng.integers(0, len(docs[d]) // BS))
        r = np.zeros(1, EVENT_DTYPE)
        r["podtier"] = PT(int(rng.integers(0, P)), int(rng.integers(0, NT)))
        hs = np.array([d * 1000 + b], np.uint64)
        if rng.random() < 0.75:
            r["op"] = 0; r["has_parent"] = b > 0; r["parent_hash"] = d * 1000 + b - 1 if b > 0 else 0
            r["n_hashes"] = 1; r["n_tokens"] = BS
            tk = np.array(docs[d][b * BS:(b + 1) * BS], np.uint32)
        else:
            r["op"] = 1; r["n_hashes"] = 1
            tk = np.zeros(0, np.uint32)
        assert ix.apply_events(r, hs, tk)[0] == 0
        _oracle_apply(pool, r[0], hs, tk)
        seen |= {k.chunk_hash for k in ox.index.data.d}
        if step % 5 == 4:
            q = _prompts(rng, docs, 1, BS)[0]
            s, _ = ix.score_batch(*csr([q]))
            assert np.array_equal(s[0], _dense(ox.get_pod_scores(q, MODEL), 16)), step
        if step % 20 == 19:
            n_removed += _remove_both(ix, ox, rng, P, NT)[1]
            _check_state(ix, ox, seen, engine_keys)
        st = ix.stats()
        assert st["request_keys"] == len(ox.index.data) and st["engine_keys"] == len(ox.index.engine_to_request), step
    assert n_removed > 0 and ix.stats()["request_keys"] <= CAP


def test_churn_of_short_lived_pods_never_fills_the_table():
    """Pods join with 256 blocks each and go away, 3000 times over, on a 4096-slot table: with removal the table never
    reports ENOSPC and is empty after every removal; without removal it fills up within a few dozen pods."""
    rng = np.random.default_rng(8)
    ix = kvidx.Index(capacity=1024, table_slots=4096, max_pods=256)
    for cycle in range(3000):
        pod = cycle % 256
        eng = rng.integers(1, 1 << 62, 256, dtype=np.uint64)
        req = rng.integers(1, 1 << 62, 256, dtype=np.uint64)
        assert ix.add(0, eng, req, [PT(pod), PT(pod, 1)]) == 0, (cycle, ix.last_error())
        assert ix.remove_pods([pod]) == {"entries": 512, "request_keys": 256, "engine_keys": 256}
        st = ix.stats()
        assert st["request_keys"] == 0 and st["engine_keys"] == 0, cycle
    assert ix.stats()["rebuilds"] > 0
    keep = kvidx.Index(capacity=1024, table_slots=4096, max_pods=256)
    rcs = [keep.add(0, rng.integers(1, 1 << 62, 256, dtype=np.uint64), rng.integers(1, 1 << 62, 256, dtype=np.uint64), [PT(c)])
           for c in range(40)]
    assert kvidx.ENOSPC in rcs


def test_readers_see_before_or_after_images_while_pods_are_removed():
    """A writer keeps adding two pods to every block of a prompt and removing them again, and adding / removing a pod that
    alone owns a second group of keys (removal tombstones them, the re-add claims new slots).  Readers must see every slot
    either before or after each update: pod 1 always, pods 2 and 3 together or not at all, the second group empty or whole;
    a Score() beside them is consistent with some per-key before / after choice."""
    BS = 16
    rng = np.random.default_rng(9)
    ix = kvidx.Index(capacity=1 << 12, max_pods=64)
    toks = rng.integers(0, 128256, size=BS * 8).astype(np.uint32)
    keys, _ = ix.hash_keys(toks, [0, len(toks)])
    eng = (keys ^ np.uint64(0x99)).astype(np.uint64)
    keys2 = rng.integers(1, 1 << 62, 16, dtype=np.uint64)
    eng2 = (keys2 ^ np.uint64(0x77)).astype(np.uint64)
    assert ix.add(0, eng, keys, [PT(1)]) == 0
    stop = threading.Event()
    errs = []
    n_removals = [0]

    def writer():
        try:
            while not stop.is_set():
                assert ix.add(0, eng, keys, [PT(2), PT(3), PT(1)]) == 0
                assert ix.add(0, eng2, keys2, [PT(4, 1)]) == 0
                assert ix.remove_pods([2, 3, 4]) == {"entries": 2 * 8 + 16, "request_keys": 16, "engine_keys": 16}
                n_removals[0] += 1
        except Exception as ex:                                       # noqa: BLE001
            errs.append(ex)

    def reader():
        try:
            while not stop.is_set():
                rc, pt, cnt = ix.lookup(0, keys)
                assert rc == 0
                for j in range(len(keys)):
                    assert pt[j, :cnt[j]].tolist() in ([PT(1)], [PT(2), PT(3), PT(1)]), pt[j, :cnt[j]]
                rc, pt, cnt = ix.lookup(0, keys2)
                for j in range(len(keys2)):
                    assert pt[j, :cnt[j]].tolist() in ([], [PT(4, 1)])
                rc, r = ix.get_request_key(0, int(eng2[0]))
                assert rc == kvidx.ENOENT or r == int(keys2[0])
                s, has = ix.score_batch(toks, [0, len(toks)])
                assert has[0] == 1 and s[0, 1] == 8.0 and s[0, 2] == s[0, 3] and s[0, 2] in [-1.0] + [float(k) for k in range(1, 9)], s[0][:4]
        except Exception as ex:                                       # noqa: BLE001
            errs.append(ex)

    ths = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
    for t in ths:
        t.start()
    time.sleep(3.0)
    stop.set()
    for t in ths:
        t.join()
    assert not errs, errs[:2]
    assert n_removals[0] > 10


def test_remove_pods_argument_errors_and_sharded_handle():
    ix = kvidx.Index(capacity=1024, max_pods=64)
    assert ix.add(0, [1], [2], [PT(5)]) == 0
    zero = np.zeros(ix.filter_words, np.uint64)
    import ctypes as C
    assert ix.L.kvidx_remove_pods(ix.h, zero.ctypes.data_as(C.POINTER(C.c_uint64)), 0xFFFF, None) == kvidx.EINVAL
    with pytest.raises(kvidx.KvidxError) as ei:
        ix.remove_pods([5], tier_ids=[])
    assert ei.value.code == kvidx.EINVAL
    with pytest.raises(kvidx.KvidxError) as ei:
        ix.remove_pods([64])
    assert ei.value.code == kvidx.ERANGE
    assert ix.remove_pods([5], [1]) == {"entries": 0, "request_keys": 0, "engine_keys": 0}
    assert ix.remove_pods([5], [0]) == {"entries": 1, "request_keys": 1, "engine_keys": 1}
    sh = kvidx.Index(capacity=1024, max_pods=64, shard_rank=0, shard_count=2)
    with pytest.raises(kvidx.KvidxError) as ei:
        sh.remove_pods([5])
    assert ei.value.code == kvidx.EINVAL and "sharded" in str(ei.value)


# ---- host mirror ----------------------------------------------------------------------------------------------------
def test_host_remove_pod_frees_the_name_and_scores_follow_reused_ids():
    BS = 16
    h = HostIndexer(block_size=BS, capacity=4096, max_pods=4)
    ox = ko.Indexer(block_size=BS, size=10 ** 6, weights={"gpu": 1.0, "cpu": 0.8})
    toks = list(range(1000, 1000 + BS * 6))
    keys = [k.chunk_hash for k in ox.tokens_processor.tokens_to_kv_block_keys(None, toks, MODEL)]
    eng = [k ^ 0x55 for k in keys]

    def add(pod, tier, n):
        assert h.add(MODEL, eng[:n], keys[:n], [(pod, tier)]) == 0, h.err()
        ox.index.add([ko.Key(MODEL, e) for e in eng[:n]], [ko.Key(MODEL, k) for k in keys[:n]], [ko.PodEntry(pod, tier)])

    def same():
        assert h.get_pod_scores(toks, MODEL) == ox.get_pod_scores(toks, MODEL)
        want = {k.chunk_hash: [(e.pod, e.tier) for e in v] for k, v in ox.index.lookup([ko.Key(MODEL, k) for k in keys]).items()}
        assert h.lookup(MODEL, keys) == (0, want)

    add("a", "gpu", 6); add("b", "cpu", 3); add("c", "gpu", 2); add("d", "gpu", 1)
    same()
    assert h.add(MODEL, eng[:1], keys[:1], [("e", "gpu")]) == kvidx.ERANGE            # four ids, all taken
    assert h.remove_pod("a") == 0
    remove_pods(ox.index, {"a"})
    same()
    assert "a" not in h.get_pod_scores(toks, MODEL)
    add("e", "gpu", 4)                                                                # takes a's id (0)
    assert h.pod_id("e") == 0
    same()
    assert h.get_pod_scores(toks, MODEL)["e"] == 4.0
    assert h.remove_pod("b", ["cpu"]) == 0                                            # one tier: b keeps its id
    remove_pods(ox.index, {"b"}, {"cpu"})
    same()
    assert h.pod_id("b") == 1


def test_zmq_all_blocks_cleared_option_matches_the_oracle():
    """vLLM publishers -> ZmqSubscriber -> host mirror with clear_on_all_blocks_cleared: an AllBlocksCleared in the middle of
    one pod's events removes that pod's gpu-tier entries stored before it (its cpu ones stay) and nothing stored after it;
    other pods are untouched.  Same wire payloads through the oracle's EventsPool with the same option."""
    import zmq
    from kvidx import service
    BS = 4
    rng = np.random.default_rng(10)
    host = HostIndexer(block_size=BS, capacity=1 << 14, max_pods=64, clear_on_all_blocks_cleared=True)
    ox = ko.Indexer(block_size=BS, hash_seed="", size=10 ** 6, pod_cache_size=10, weights={"gpu": 1.0, "cpu": 0.8})
    opool = ClearingEventsPool(ox.index, ox.tokens_processor)
    sub = service.ZmqSubscriber(host, "tcp://127.0.0.1:*").start()
    pub = zmq.Context.instance().socket(zmq.PUB)
    pub.connect(sub.bound_endpoint)
    t0 = time.time()
    while sub.malformed < 1 and time.time() - t0 < 20:           # slow joiner: probe until the subscription has arrived
        pub.send_multipart([b"kv@probe", (0).to_bytes(8, "big"), b"x"])
        time.sleep(0.05)
    assert sub.malformed >= 1
    docs = {("pod-%d" % p): rng.integers(0, 30000, size=BS * 18).tolist() for p in range(4)}

    def H(pod, b):
        return hash((pod, b)) & (2 ** 63 - 1)

    def stored(pod, b0, b1, medium):
        return ["BlockStored", [H(pod, b) for b in range(b0, b1)], H(pod, b0 - 1) if b0 else None, docs[pod][b0 * BS:b1 * BS], BS, None, medium]
    msgs = []
    for pod in docs:
        msgs.append((pod, [stored(pod, 0, 6, None)]))
        msgs.append((pod, [stored(pod, 6, 12, "CPU")] + ([["AllBlocksCleared"], stored(pod, 12, 18, None)] if pod == "pod-0" else [])))
        if pod != "pod-0":
            msgs.append((pod, [stored(pod, 12, 18, None)]))
    for seq, (pod, body) in enumerate(msgs):
        payload = msgpack.packb([time.time(), body, 0])
        pub.send_multipart([("kv@%s@%s" % (pod, MODEL)).encode(), seq.to_bytes(8, "big"), payload])
        opool.process_event(pod, MODEL, payload)
    t0 = time.time()
    while sub.messages < len(msgs) and time.time() - t0 < 20:
        time.sleep(0.01)
    assert sub.messages == len(msgs) and sub.flush()
    for pod, d in docs.items():
        keys = [k.chunk_hash for k in ox.tokens_processor.tokens_to_kv_block_keys(None, d, MODEL)]
        want = {k.chunk_hash: [(e.pod, e.tier) for e in v] for k, v in ox.index.lookup([ko.Key(MODEL, k) for k in keys]).items()}
        assert host.lookup(MODEL, keys) == (0, want), pod
        for cut in (len(d), BS * 7, BS * 2):
            assert host.get_pod_scores(d[:cut], MODEL) == ox.get_pod_scores(d[:cut], MODEL), (pod, cut)
        if pod == "pod-0":                                      # before the clear: gpu gone, cpu kept
            assert all(k not in want for k in keys[:6]) and all(want[k] == [(pod, "cpu")] for k in keys[6:12])
        else:
            assert all(want[k] == [(pod, "gpu" if i < 6 or i >= 12 else "cpu")] for i, k in enumerate(keys))
    # after the clear: pod-0's last blocks are present (their parent's cpu mapping survived, so the chain continues)
    assert host.get_pod_scores(docs["pod-0"], MODEL) is not None
    k0 = [k.chunk_hash for k in ox.tokens_processor.tokens_to_kv_block_keys(None, docs["pod-0"], MODEL)]
    assert host.lookup(MODEL, k0[12:])[1] == {k: [("pod-0", "gpu")] for k in k0[12:]}
    sub.stop(); pub.close(0)
