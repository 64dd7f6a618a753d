"""GPU (-m gpu): kvidx_snapshot / kvidx_restore and the host mirror's snapshot / restore -- byte-exact against the image
spec (tests/snapshot_oracle.py) and bit-exact against the Python oracle after a restore and while the stream continues."""
import copy
import struct
import ctypes as C
import threading

import msgpack
import numpy as np
import pytest

from helpers import EVENT_DTYPE, SEED_ORDER_SIZES, csr
import kvidx
from kvidx.host import HostIndexer
from oracle import kvoracle as ko
import snapshot_oracle as so
from test_gpu_parity import _random_stream, _select_path
from test_gpu_remove_pods import (MODEL, PATH_SIZES, PT, TIERS, W, _check_state, _dense, _oracle_apply, _oracle_scores, _pair,
                                  _prompts, _remove_both)
from test_snapshot_cpu import golden, malformed, recency_image

pytestmark = pytest.mark.gpu
SEED_HASH = ko.fnv64a(b"abc")            # _pair's hash_seed


def _encode(ox, P=16, lru=False):
    return so.encode(ox.index, {MODEL: 0}, {"p%d" % p: p for p in range(P)}, {t: i for i, t in enumerate(TIERS)}, 16, SEED_HASH, 4,
                     recency=lru)


def _fresh(P=16, capacity=1 << 16, table_slots=0, lru_exact=0):
    return kvidx.Index(block_size=16, hash_seed="abc", capacity=capacity, pods_per_key=4, tier_weights=W, max_pods=P,
                       table_slots=table_slots, lru_exact=lru_exact)


def _empty(ix):
    st = ix.stats()
    return (st["request_keys"], st["engine_keys"], st["request_tombs"], st["engine_tombs"]) == (0, 0, 0, 0)


@pytest.mark.parametrize("path", list(PATH_SIZES))
def test_random_stream_snapshot_restore_continue_vs_oracle(path, monkeypatch):
    """Random BlockStored / BlockRemoved streams with pod removals (so tombstones and stale mappings exist).  At two points
    the handle's image must equal the spec's encoding of the oracle; after the first, the stream moves to a handle of
    another table size restored from it: Lookup, GetRequestKey, stats (no tombstones) and Score() on the path stay
    bit-exact against the oracle, also as the stream continues (parents resolve through restored engine mappings)."""
    if path != "default":
        _select_path(monkeypatch, path)
    rng = np.random.default_rng(SEED_ORDER_SIZES.index(path) + 170)
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
    stale = 0
    for step in range(25):
        for i in range(16 * step, 16 * (step + 1)):
            assert ix.apply_events(ev[i:i + 1], hs, tk)[0] == 0
            _oracle_apply(pool, ev[i], hs, tk)
            seen |= {k.chunk_hash for k in ox.index.data.d}
        _remove_both(ix, ox, rng, P, NT)
        if step in (3, 15):                                 # two engine keys -> one request key, evicted through the first:
            e1, e2, rk = 0xDEAD0000 + step, 0xDEAD1000 + step, 0xBEEF0000 + step       # the second mapping is left stale
            assert ix.add(0, [e1, e2], [rk, rk], [PT(15)]) == 0 and ix.evict(0, e1, [PT(15)]) == 0
            ox.index.add([ko.Key(MODEL, e1), ko.Key(MODEL, e2)], [ko.Key(MODEL, rk)] * 2, [ko.PodEntry("p15", "gpu")])
            ox.index.evict(ko.Key(MODEL, e1), [ko.PodEntry("p15", "gpu")])
            engine_keys += [e1, e2]
        if step in (10, 24):
            img = ix.snapshot()
            assert img == _encode(ox), step
            stale = max(stale, sum(rk not in ox.index.data.d for rk in ox.index.engine_to_request.d.values()))
        if step == 10:
            assert ix.stats()["request_tombs"] > 0
            ix = _fresh(table_slots=1 << 13)
            assert ix.restore(img) == {"request_keys": len(ox.index.data), "engine_keys": len(ox.index.engine_to_request)}
            st = ix.stats()
            assert st["request_tombs"] == 0 and st["engine_tombs"] == 0 and st["request_slots"] == 1 << 13
        if step >= 10:
            _check_state(ix, ox, seen, engine_keys)
            want = np.stack([_dense(_oracle_scores(ox, k), 16) for k in pkeys])
            for n, (tok, off) in tok_off.items():
                s, has = ix.score_batch(tok, off)
                assert np.array_equal(s, want[np.arange(n) % len(prompts)]), (step, n)
    assert stale > 0                                        # the images carried stale engine mappings


def test_equal_contents_give_identical_images():
    """Same contents, different table sizes and histories (one handle rebuilt after churn): the same bytes."""
    rng = np.random.default_rng(5)
    eng = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
    req = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
    a, b, c = _fresh(), _fresh(table_slots=1 << 16), _fresh(capacity=1024, table_slots=4096)
    for cycle in range(40):                                 # churn on c until it has rebuilt its tables
        e2 = rng.integers(1, 1 << 62, 256, dtype=np.uint64)
        assert c.add(0, e2, rng.integers(1, 1 << 62, 256, dtype=np.uint64), [PT(9)]) == 0
        c.remove_pods([9])
    assert c.stats()["rebuilds"] > 0
    for ix in (a, b, c):
        for j in range(0, 300, 50):
            assert ix.add(j % 3, eng[j:j + 50], req[j:j + 50], [PT(j % 7, 1), PT(3)]) == 0
        assert ix.evict(1, int(eng[60]), [PT(3)]) == 0
    img = a.snapshot()
    assert b.snapshot() == img and c.snapshot() == img
    assert struct_counts(img) == (a.stats()["request_keys"], a.stats()["engine_keys"])


def struct_counts(img):
    return tuple(int(v) for v in np.frombuffer(img[32:48], np.uint64))


def test_golden_image_restores_and_snapshots_back():
    d, img = golden()
    ix = kvidx.Index(block_size=d["block_size"], init_hash=d["init_hash"], pods_per_key=d["pods_per_key"], max_pods=16, capacity=1024)
    assert ix.restore(img) == {"request_keys": d["request_keys"], "engine_keys": d["engine_keys"]}
    assert ix.snapshot() == img
    assert ix.get_request_key(0, 0x1005) == (0, 0xA004)     # the stale mapping
    rc, pt, cnt = ix.lookup(0, np.array([0xA004, 0xA002], np.uint64))
    assert rc == 0 and cnt[0] == 0 and pt[1, :cnt[1]].tolist() == [PT(1, 1), PT(0, 0)]


def test_restore_error_paths_leave_the_target_empty():
    d, img = golden()
    cfg = dict(block_size=d["block_size"], init_hash=d["init_hash"], pods_per_key=d["pods_per_key"], max_pods=16, capacity=1024)
    rimg, _ = recency_image()                                # exact-LRU cases: stamps >= 2^63, repeated stamps, bad engine record
    rcfg = dict(block_size=16, init_hash=7, pods_per_key=4, max_pods=16, capacity=1024, lru_exact=1)
    kvidx.Index(**rcfg).restore(rimg)                        # the unbroken image is accepted
    for c, image in ((cfg, img), (rcfg, rimg)):
        for case, (bad, _, why) in malformed(image).items():
            ix = kvidx.Index(**c)
            with pytest.raises(kvidx.KvidxError) as ei:
                ix.restore(bad)
            assert ei.value.code == kvidx.EINVAL and why in str(ei.value), (case, str(ei.value))
            assert _empty(ix), case
    for kw, code in (({"block_size": 32}, kvidx.EINVAL), ({"init_hash": 5}, kvidx.EINVAL), ({"pods_per_key": 4}, kvidx.EINVAL),
                     ({"max_pods": 8}, kvidx.ERANGE), ({"lru_exact": 1}, kvidx.EINVAL)):
        ix = kvidx.Index(**{**cfg, **kw})
        with pytest.raises(kvidx.KvidxError) as ei:
            ix.restore(img)
        assert ei.value.code == code, kw
        assert _empty(ix), kw
    ix = kvidx.Index(**cfg)                                  # live keys in the target
    assert ix.add(0, [1], [2], [PT(1)]) == 0
    with pytest.raises(kvidx.KvidxError) as ei:
        ix.restore(img)
    assert ei.value.code == kvidx.EINVAL and ix.stats()["request_keys"] == 1
    assert ix.evict(0, 1, [PT(1)]) == 0                      # only a tombstone left: restore drops it
    assert ix.stats()["request_tombs"] == 1
    ix.restore(img)
    assert ix.snapshot() == img and ix.stats()["request_tombs"] == 0
    big = kvidx.Index(**cfg)                                 # more keys than the target's table admits
    rng = np.random.default_rng(3)
    assert big.add(0, rng.integers(1, 1 << 62, 1000, dtype=np.uint64), rng.integers(1, 1 << 62, 1000, dtype=np.uint64), [PT(2)]) == 0
    small = kvidx.Index(**{**cfg, "table_slots": 1024})
    with pytest.raises(kvidx.KvidxError) as ei:
        small.restore(big.snapshot())
    assert ei.value.code == kvidx.ENOSPC and _empty(small)
    sh = kvidx.Index(**{**cfg, "shard_rank": 0, "shard_count": 2})
    for call in (sh.snapshot, lambda: sh.restore(img)):
        with pytest.raises(kvidx.KvidxError) as ei:
            call()
        assert ei.value.code == kvidx.EINVAL and "sharded" in str(ei.value)
    ix = kvidx.Index(**cfg)                                  # a too-small buffer: ENOSPC, the size, nothing written
    ix.restore(img)
    buf, size = C.create_string_buffer(b"\x5a" * 100, 100), C.c_uint64(0)
    assert ix.L.kvidx_snapshot(ix.h, buf, 100, C.byref(size)) == kvidx.ENOSPC and size.value == len(img)
    assert buf.raw == b"\x5a" * 100
    assert ix.L.kvidx_snapshot(ix.h, None, 0, C.byref(size)) == kvidx.ENOSPC and size.value == len(img)


def _exact_stream(ix, ox, pool, rng, docs, steps, seen, check_every=20):
    BS, P, NT = 16, 10, 2
    for step in range(steps):
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
        st = ix.stats()
        assert st["request_keys"] == len(ox.index.data) and st["engine_keys"] == len(ox.index.engine_to_request), step
        if step % check_every == check_every - 1:
            _check_state(ix, ox, seen, [d * 1000 + b for d in range(len(docs)) for b in range(len(docs[d]) // BS)])


def test_exact_lru_snapshot_midway_and_continue_vs_capped_oracle():
    """A capped exact-LRU stream is snapshotted midway and restored into a fresh exact handle; the stream continues on it
    and on a deep copy of the oracle, and its key evictions match.  snapshot(restore(s)) == s; a restore into a smaller
    capacity keeps the most recent keys of each map, as the oracle's LRU does."""
    rng = np.random.default_rng(44)
    CAP = 40
    ix, ox, pool = _pair(P=16, capacity=CAP, lru_exact=1)
    docs = [rng.integers(0, 128256, size=16 * int(rng.integers(2, 9))).tolist() for _ in range(14)]
    seen = set()
    _exact_stream(ix, ox, pool, rng, docs, 300, seen)
    s = ix.snapshot()
    R, E = len(ox.index.data), len(ox.index.engine_to_request)
    assert struct_counts(s) == (R, E) and R > CAP // 2 and len(s) == 64 + 32 * R + 24 * E + 8 * (R + E)
    inv = ({0: MODEL}, {p: "p%d" % p for p in range(16)}, dict(enumerate(TIERS)))
    back, hd = so.decode(s, *inv, pods_per_key=4, size=CAP)          # the image's recency order is the oracle's LRU order
    assert hd["flags"] == so.FLAG_RECENCY
    assert list(back.data.d) == list(ox.index.data.d) and list(back.engine_to_request.d) == list(ox.index.engine_to_request.d)
    ix3 = _fresh(capacity=CAP, lru_exact=1)
    ix3.restore(s)
    assert ix3.snapshot() == s
    small = _fresh(capacity=CAP // 2, lru_exact=1)
    assert small.restore(s) == {"request_keys": min(R, CAP // 2), "engine_keys": min(E, CAP // 2)}
    want, _ = so.decode(s, *inv, pods_per_key=4, size=CAP // 2)
    rc, pt, cnt = small.lookup(0, np.array(sorted(seen), np.uint64))
    got = {k for k, c in zip(sorted(seen), cnt) if c}
    assert rc == 0 and got == {k.chunk_hash for k in want.data.d}
    for ek, rk in want.engine_to_request.d.items():
        assert small.get_request_key(0, ek.chunk_hash) == (0, rk.chunk_hash)
    plain = _fresh(capacity=CAP)                             # a default handle drops the recency section
    plain.restore(s)
    assert plain.snapshot() == _encode(ox)
    ix2 = _fresh(capacity=CAP, lru_exact=1)
    ix2.restore(s)
    ox2 = copy.deepcopy(ox)
    pool2 = ko.EventsPool(ox2.index, ox2.tokens_processor)
    _exact_stream(ix2, ox2, pool2, rng, docs, 300, seen)


def test_snapshot_beside_a_writer_and_a_reader_is_a_prefix_of_the_stream():
    """One thread applies single-event calls, another scores; snapshots taken meanwhile each equal the spec's encoding of
    the oracle after some prefix of the events, and the reader sees no error."""
    rng = np.random.default_rng(12)
    BS, P, NT = 16, 12, 3
    ix, ox, pool = _pair(P=16)
    docs = [rng.integers(0, 128256, size=BS * int(rng.integers(1, 20))).tolist() for _ in range(16)]
    ev, hs, tk = _random_stream(rng, 300, BS, P, NT, docs)
    prefixes = {_encode(ox): 0}
    for i in range(len(ev)):
        _oracle_apply(pool, ev[i], hs, tk)
        prefixes.setdefault(_encode(ox), i + 1)
    tok, off = csr(_prompts(rng, docs, 64, BS))
    done, errs = threading.Event(), []

    def writer():
        try:
            for i in range(len(ev)):
                assert ix.apply_events(ev[i:i + 1], hs, tk)[0] == 0
        except Exception as ex:                              # noqa: BLE001
            errs.append(ex)
        finally:
            done.set()

    def reader():
        try:
            while not done.is_set():
                s, has = ix.score_batch(tok, off)
                assert s.shape == (64, 16)
        except Exception as ex:                              # noqa: BLE001
            errs.append(ex)

    ths = [threading.Thread(target=writer), threading.Thread(target=reader)]
    for t in ths:
        t.start()
    seen_at = []
    while not done.is_set():
        img = ix.snapshot()
        assert img in prefixes
        seen_at.append(prefixes[img])
    for t in ths:
        t.join()
    assert not errs, errs[:2]
    assert ix.snapshot() == _encode(ox) and len(seen_at) >= 1


def test_host_mirror_snapshot_restore_with_named_pods():
    """Fill a HostIndexer through add_task / process with named pods, remove one, snapshot, restore into a fresh one: scores
    by name, pod ids and the reuse of the freed id are the same on both."""
    BS = 16
    rng = np.random.default_rng(21)
    a = HostIndexer(block_size=BS, capacity=1 << 14, max_pods=8)
    docs = {("pod-%d" % p): rng.integers(0, 30000, size=BS * 12).tolist() for p in range(5)}
    shared = rng.integers(0, 30000, size=BS * 4).tolist()

    def H(pod, b):
        return (hash((pod, b)) & (2 ** 62 - 1)) | (1 << 62)        # msgpack uint64: a hash type getHashAsUint64 accepts
    for pod, d in docs.items():
        toks = shared + d
        body = [["BlockStored", [H(pod, b) for b in range(8)], None, toks[:8 * BS], BS, None, None],
                ["BlockStored", [H(pod, b) for b in range(8, 16)], H(pod, 7), toks[8 * BS:16 * BS], BS, None, "CPU"]]
        assert a.add_task(pod, "llama", msgpack.packb([0.0, body, 0])) == 0
    n, dropped = a.process()
    assert n == 10 and dropped == 0
    a.remove_pod("pod-2")
    img = a.snapshot()
    b = HostIndexer(block_size=BS, capacity=1 << 14, max_pods=8)
    b.restore(img)
    assert b.snapshot() == img
    prompts = [shared + d[:BS * k] for d in docs.values() for k in (0, 3, 12)]
    for p in prompts:
        assert a.get_pod_scores(p, "llama") == b.get_pod_scores(p, "llama")
    assert a.get_pod_scores(prompts[2], "llama")               # something is scored
    for pod in docs:
        if pod != "pod-2":
            assert a.pod_id(pod) == b.pod_id(pod)
    assert a.pod_id("newcomer") == b.pod_id("newcomer") == 2  # the freed id, on both


def _host_image(models, tiers, pods, index_image):
    """A host mirror image (include/kvidx_host.h) around an index image; None in `pods` marks a freed id."""
    def table(names):
        out = struct.pack("<I", len(names))
        for n in names:
            out += struct.pack("<I", 0xFFFFFFFF) if n is None else struct.pack("<I", len(n)) + n.encode()
        return out
    return (b"KVHOSTSN" + struct.pack("<II", 1, 0) + table(models) + table(tiers) + table(pods) + struct.pack("<Q", len(index_image))
            + index_image)


def test_host_restore_refuses_entries_of_unnamed_pods():
    """Every pod id that owns entries in the index section must be named: a freed id or one past the pod table is refused
    and the target stays fresh; the consistent image restores and snapshots back to itself."""
    d, img = golden()

    def target():
        return HostIndexer(block_size=d["block_size"], hash_seed="golden", pods_per_key=d["pods_per_key"], max_pods=16, capacity=1024)
    for pods in ([None if i == 1 else p for i, p in enumerate(d["pods"])], d["pods"][:5]):
        h = target()
        with pytest.raises(kvidx.KvidxError) as ei:
            h.restore(_host_image(d["models"], d["tiers"], pods, img))
        assert ei.value.code == kvidx.EINVAL and "no name" in str(ei.value)
        assert h.pod_id("zz") == 0 and h.get_pod_scores(list(range(64)), "llama") == {}
    good = _host_image(d["models"], d["tiers"], d["pods"], img)
    h = target()
    h.restore(good)
    assert h.snapshot() == good and h.pod_id("pod-b") == 1
