"""GPU: CLOCK key cap (evict_policy="clock", include/kvidx.h).  Reference bits set by the write path, Lookup,
GetRequestKey and every Score() path; the sweep after each write call; rebuild, restore and the host mirror."""
import ctypes as C
import struct

import msgpack
import numpy as np
import pytest

import kvidx
import snapshot_oracle as so
from clock_oracle import referenced_keys
from helpers import EVENT_DTYPE, PATHS, SEED_ORDER, _select_path, csr
from kvidx.host import HostIndexer
from oracle import kvoracle as ko

pytestmark = pytest.mark.gpu

BS, P = 16, 8
MODELS = ["m0", "m1"]
PODS = ["p%d" % i for i in range(P)]
TIERS = ["gpu", "cpu"]
W = (1.0, 0.8)


def PT(p, t=0):
    return (p << 4) | t


def resident(ix):
    """(request hashes, engine hashes) of the handle's snapshot, as (model, hash) pairs."""
    img = ix.snapshot()
    R, E = struct.unpack_from("<QQ", img, 32)
    req = {(struct.unpack_from("<H", img, 64 + 32 * i + 8)[0], struct.unpack_from("<Q", img, 64 + 32 * i)[0]) for i in range(R)}
    base = 64 + 32 * R
    eng = {(struct.unpack_from("<H", img, base + 24 * i + 16)[0], struct.unpack_from("<Q", img, base + 24 * i)[0]) for i in range(E)}
    return req, eng, img


def oracle_of(img):
    return so.decode(img, MODELS, PODS, TIERS, max_pods=P)[0]


def oracle_rows(oix, prompts, filters):
    sc = ko.LongestPrefixScorer(dict(zip(TIERS, W)))
    tp = ko.ChunkedTokenDatabase(BS)
    rows = np.full((len(prompts), P), -1.0)
    for i, (t, m) in enumerate(prompts):
        keys = tp.tokens_to_kv_block_keys(None, list(t), m)
        if not keys:
            continue
        got = sc.score(keys, oix.lookup(keys, filters[i] if filters else ()))
        for p, s in got.items():
            rows[i, PODS.index(p)] = s
    return rows


def score(ix, prompts, filters):
    tok, off = csr([t for t, _ in prompts])
    model = np.array([MODELS.index(m) for _, m in prompts], np.uint32)
    fm = None
    if filters:
        fm = np.zeros((len(prompts), ix.filter_words), np.uint64)
        for i, f in enumerate(filters):
            for p in f or ():
                fm[i, PODS.index(p) // 64] |= np.uint64(1) << np.uint64(PODS.index(p) % 64)
    return ix.score_batch(tok, off, model=model, filter_mask=fm)[0]


def keys_of(ix, tokens):
    k, _ = ix.hash_keys(np.asarray(tokens, np.uint32), np.array([0, len(tokens)], np.int64))
    return [int(x) for x in k]


class Fill:
    """C = 64 documents x 16 blocks, model m0 for even documents and m1 for odd ones.  Blocks 0..7 hold pods {0, 1}; blocks
    8..15 hold {1} on documents whose index is 0 mod 4, else {0, 1}.  So a prompt filtered to pod 0 ends its walk at block 8
    of those documents and blocks 9..15 stay present but unprobed."""
    D, NB = 64, 16

    def __init__(self, ix, rng):
        self.docs = [rng.integers(0, 128256, size=BS * self.NB).tolist() for _ in range(self.D)]
        self.keys = [keys_of(ix, d) for d in self.docs]
        groups = {}
        for d in range(self.D):
            m = d % 2
            for b in range(self.NB):
                ents = (PT(1),) if (b >= 8 and d % 4 == 0) else (PT(0), PT(1))
                groups.setdefault((m, ents), []).append(self.keys[d][b])
        for (m, ents), ks in sorted(groups.items()):
            eng = [k ^ 0x5A5A5A5A5A5A5A5A for k in ks]
            assert ix.add(m, eng, ks, list(ents)) == 0
        self.C = self.D * self.NB

    def queries(self, rng, n, with_filters=True, docs=24):
        """n prompts over the first `docs` documents (the others stay unreferenced)."""
        prompts, filters = [], []
        for _ in range(n):
            d = int(rng.integers(0, docs))
            kind = int(rng.integers(0, 5))
            m = MODELS[d % 2]
            t = list(self.docs[d])
            f = None
            if kind == 1:                                    # gap: the doc's prefix, then foreign blocks
                cut = int(rng.integers(0, self.NB))
                t = t[:BS * cut] + rng.integers(0, 128256, size=BS * 3).tolist()
            elif kind == 2 and with_filters:                 # filtered to pod 0: ends at block 8 on every 4th doc
                f = ["p0"]
            elif kind == 3 and with_filters:                 # filtered to a pod no block holds: ends at block 0
                f = ["p5"]
            elif kind == 4:                                  # a prefix of the doc
                t = t[:BS * int(rng.integers(1, self.NB + 1))] + [7] * int(rng.integers(0, BS))
            prompts.append((t, m))
            filters.append(f)
        return prompts, (filters if with_filters else None)


def clock_index(capacity, **kw):
    return kvidx.Index(block_size=kw.pop("block_size", BS), capacity=capacity, table_slots=4 * capacity, pods_per_key=4, tier_weights=W,
                       max_pods=P, evict_policy="clock", **kw)


def _new_keys(rng, k):
    ks = [int(x) for x in rng.integers(1, 2 ** 63, size=k, dtype=np.int64)]
    return ks, [x ^ 0x1234 for x in ks]


# ---- 1. config ------------------------------------------------------------------------------------------------------
def test_config_validation():
    assert C.sizeof(kvidx.Config) == 208
    for kw in ({"evict_policy": 2}, {"evict_policy": "clock", "lru_exact": 1}, {"evict_policy": "clock", "shard_count": 2}):
        with pytest.raises(kvidx.KvidxError) as ei:
            kvidx.Index(capacity=1024, **kw)
        assert ei.value.code == kvidx.EINVAL
    ix = kvidx.Index(capacity=1024)                              # zeroed reserved == NONE: no cap
    assert ix.add(0, list(range(1, 2001)), list(range(1, 2001)), [PT(0)]) == 0
    assert ix.stats()["request_keys"] == 2000 and ix.evictions() == (0, 0)


# ---- 2. below capacity nothing differs -----------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["v1", "coop", "rounds", "classes"])
def test_below_capacity_same_as_default(path, monkeypatch):
    _select_path(monkeypatch, path)
    rng = np.random.default_rng(1)
    a = kvidx.Index(capacity=4096, table_slots=16384, pods_per_key=4, tier_weights=W, max_pods=P)
    b = clock_index(4096)
    fa, fb = Fill(a, np.random.default_rng(5)), Fill(b, np.random.default_rng(5))
    for d in range(0, 64, 3):                                     # evictions of some entries, some keys
        for ix, f in ((a, fa), (b, fb)):
            assert ix.evict(d % 2, f.keys[d][5] ^ 0x5A5A5A5A5A5A5A5A, [PT(0)]) == 0
    prompts, filters = fa.queries(rng, 300)
    assert np.array_equal(score(a, prompts, filters), score(b, prompts, filters))
    assert a.snapshot() == b.snapshot()
    assert b.evictions() == (0, 0)


# ---- 4. second chance, exactly ---------------------------------------------------------------------------------------
def _second_chance(ix, rng, n_queries, k_less, with_filters=True):
    f = Fill(ix, rng)
    C_ = f.C
    ka, ea = _new_keys(rng, 1)
    assert ix.add(0, ea, ka, [PT(2)]) == 0                      # full turn: every resident key unreferenced
    req0, _, img0 = resident(ix)
    assert len(req0) == C_ and ix.evictions()[0] == 1
    assert ix.sweeps() == (2, 2)                                  # one sweep per map, each past a full turn
    oix = oracle_of(img0)
    prompts, filters = f.queries(rng, n_queries, with_filters)
    rows = score(ix, prompts, filters)
    assert np.array_equal(rows, oracle_rows(oix, prompts, filters))
    R = {(MODELS.index(k.model), k.chunk_hash) for k in referenced_keys(oix, prompts, filters, block_size=BS)}
    assert R and len(R) < C_
    k = C_ - len(R) - k_less
    kn, en = _new_keys(rng, k)
    assert ix.add(0, en, kn, [PT(3)]) == 0
    req1, _, _ = resident(ix)
    new = {(0, x) for x in kn}
    assert len(req1) == C_ and ix.evictions()[0] == 1 + k
    assert R | new <= req1
    assert ix.sweeps() == (4, 2)                                  # two more sweeps, each a partial turn
    if k_less == 0:
        assert req1 == R | new
    else:
        assert len(req0 - R - req1) == k
    return f, R


@pytest.mark.parametrize("path", PATHS)
def test_second_chance_on_every_path(path, monkeypatch):
    _select_path(monkeypatch, path)
    rng = np.random.default_rng(SEED_ORDER.index(path) + 100)
    _second_chance(clock_index(1024), rng, 300, 0)
    _second_chance(clock_index(1024), rng, 300, 17)


@pytest.mark.parametrize("n", [2048, 4096, 131072])
def test_second_chance_by_batch_size(n):
    """The default dispatch: the cooperative kernel, the per-prompt rounds and the prefix-class pipeline (prompts share
    prefixes: they are the 64 documents' prefixes)."""
    _second_chance(clock_index(1024), np.random.default_rng(n), n, 0)


def test_second_chance_block_size_4():
    ix = clock_index(1024, block_size=4)
    rng = np.random.default_rng(3)
    docs = [rng.integers(0, 1000, size=4 * 16).tolist() for _ in range(64)]
    keys = [[int(x) for x in ix.hash_keys(np.asarray(d, np.uint32), np.array([0, len(d)], np.int64))[0]] for d in docs]
    flat = [k for ks in keys for k in ks]
    assert ix.add(0, [k ^ 9 for k in flat], flat, [PT(0)]) == 0
    assert ix.add(0, [1], [2], [PT(1)]) == 0
    req0, _, img = resident(ix)
    q = [d[:4 * (1 + i % 16)] for i, d in enumerate(docs[:32])]
    tok, off = csr(q)
    ix.score_batch(tok, off)
    R = {(0, k.chunk_hash) for k in referenced_keys(oracle_of(img), [(t, "m0") for t in q], None, block_size=4)}
    kn, en = _new_keys(rng, 1024 - len(R))
    assert ix.add(0, en, kn, [PT(2)]) == 0
    assert resident(ix)[0] == R | {(0, x) for x in kn}


def test_second_chance_engine_map_and_lookup():
    rng = np.random.default_rng(11)
    ix = clock_index(1024)
    f = Fill(ix, rng)
    assert ix.add(0, [77], [78], [PT(2)]) == 0                   # full turn in both maps
    req0, eng0, _ = resident(ix)
    # GetRequestKey marks engine mappings
    picks = [(d % 2, f.keys[d][b] ^ 0x5A5A5A5A5A5A5A5A) for d in range(0, 64, 2) for b in range(0, 16, 3)]
    got = {(m, e) for m, e in picks if ix.get_request_key(m, e)[0] == 0}
    assert got and got <= eng0
    # Lookup marks request keys
    look = [f.keys[d][b] for d in range(1, 64, 8) for b in range(16)]
    rc, _, cnt = ix.lookup(1, np.array(look, np.uint64))
    assert rc == 0
    R = {(1, k) for k in look} & req0
    kn, en = _new_keys(rng, 1024 - len(got))
    assert ix.add(0, en, kn, [PT(3)]) == 0
    _, eng1, _ = resident(ix)
    assert eng1 == got | {(0, x) for x in en}
    # request side: the engine-map fill above also added len(got) ... request keys; R and the new ones survive
    req1, _, _ = resident(ix)
    assert {(0, x) for x in kn} <= req1
    kn2, en2 = _new_keys(rng, len(req1 - R - {(0, x) for x in kn}))
    assert ix.add(0, en2, kn2, [PT(3)]) == 0
    req2, _, _ = resident(ix)
    assert req2 == R | {(0, x) for x in kn} | {(0, x) for x in kn2}


# ---- 5. a rebuild keeps the bits -------------------------------------------------------------------------------------
def test_rebuild_keeps_reference_bits():
    rng = np.random.default_rng(12)
    ix = clock_index(1024)
    f = Fill(ix, rng)
    assert ix.add(0, [77], [78], [PT(2)]) == 0
    req0, eng0, img0 = resident(ix)
    oix = oracle_of(img0)
    prompts, filters = f.queries(rng, 300)
    score(ix, prompts, filters)
    R = {(MODELS.index(k.model), k.chunk_hash) for k in referenced_keys(oix, prompts, filters, block_size=BS)}
    # tombstones: drop some unreferenced keys through Evict, then compact
    gone = set()
    for d in range(64):
        for b in (2, 12):
            key = (d % 2, f.keys[d][b])
            if key in req0 and key not in R and (d % 2, f.keys[d][b] ^ 0x5A5A5A5A5A5A5A5A) in eng0:   # Evict goes through the mapping
                assert ix.evict(d % 2, f.keys[d][b] ^ 0x5A5A5A5A5A5A5A5A, [PT(0), PT(1)]) == 0
                gone.add(key)
    assert gone and ix.stats()["request_tombs"] >= len(gone)
    ix.shard_compact()
    assert ix.stats()["request_tombs"] == 0
    req1, _, _ = resident(ix)
    assert req1 == req0 - gone
    kn, en = _new_keys(rng, 1024 - len(R))                    # fills the room Evict left, then evicts the rest
    assert ix.add(0, en, kn, [PT(3)]) == 0
    assert resident(ix)[0] == R | {(0, x) for x in kn}


# ---- 6. restore ------------------------------------------------------------------------------------------------------
def test_restore_cuts_to_capacity():
    rng = np.random.default_rng(13)
    src = kvidx.Index(capacity=4096, table_slots=16384, pods_per_key=4, tier_weights=W, max_pods=P)
    f = Fill(src, rng)
    img = src.snapshot()
    small = clock_index(4096)
    assert small.restore(img) == {"request_keys": 1024, "engine_keys": 1024}
    assert small.snapshot() == img and small.evictions() == (0, 0)
    ix = clock_index(700)
    out = ix.restore(img)
    assert out == {"request_keys": 700, "engine_keys": 700}
    req, eng, own = resident(ix)
    src_req, src_eng, _ = resident(src)
    assert req <= src_req and eng <= src_eng and ix.evictions() == (324, 324)
    prompts, filters = f.queries(rng, 300)
    assert np.array_equal(score(ix, prompts, filters), oracle_rows(oracle_of(own), prompts, filters))


# ---- 3. bound under random streams ------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["v1", "coop", "rounds", "rounds-lane", "classes", "classes8-nodedup"])
def test_random_stream_stays_bounded(path, monkeypatch):
    _select_path(monkeypatch, path)
    rng = np.random.default_rng(SEED_ORDER.index(path) + 300)
    CAP = 1024
    ix = clock_index(CAP)
    docs = [rng.integers(0, 128256, size=BS * int(rng.integers(2, 24))).tolist() for _ in range(400)]
    for step in range(60):
        req0, eng0, _ = resident(ix)
        ev0 = ix.evictions()
        op = step % 3
        if op == 0:                                               # add: one document's keys
            d = docs[int(rng.integers(0, len(docs)))]
            ks = keys_of(ix, d)
            es = [k ^ 0x77 for k in ks]
            assert ix.add(0, es, ks, [PT(int(rng.integers(0, P)))]) == 0
            new_r, new_e = {(0, k) for k in ks}, {(0, e) for e in es}
        elif op == 1:                                             # a batch of BlockStored events without parents
            sel = [docs[int(x)] for x in rng.integers(0, len(docs), size=8)]
            ev = np.zeros(len(sel), EVENT_DTYPE)
            hashes, toks, new_r, new_e = [], [], set(), set()
            for i, d in enumerate(sel):
                ks = keys_of(ix, d)
                es = [int(x) for x in rng.integers(1, 2 ** 63, size=len(ks), dtype=np.int64)]
                ev[i] = (0, 0, PT(i % P), 0, 0, len(hashes), len(toks), len(ks), len(d))
                hashes += es
                toks += d
                new_r |= {(0, k) for k in ks}
                new_e |= {(0, e) for e in es}
            rc, dropped = ix.apply_events(ev, np.array(hashes, np.uint64), np.array(toks, np.uint32))
            assert rc == 0 and dropped == 0
        else:                                                     # evict a few resident mappings
            for m, e in list(eng0)[:5]:
                assert ix.evict(m, e, [PT(p) for p in range(P)]) == 0
            st = ix.stats()
            assert ix.evictions() == ev0
            continue
        st = ix.stats()
        assert st["request_keys"] <= CAP and st["engine_keys"] <= CAP
        req1, eng1, img = resident(ix)
        ev1 = ix.evictions()
        assert len(req0 | new_r) - len(req1) == ev1[0] - ev0[0]
        assert len(eng0 | new_e) - len(eng1) == ev1[1] - ev0[1]
    assert ix.evictions()[0] > 0
    _, _, img = resident(ix)                                      # the contents after the last call
    prompts = [(d[:BS * int(rng.integers(1, len(d) // BS + 1))], "m0") for d in docs[:300]]
    assert np.array_equal(score(ix, prompts, None), oracle_rows(oracle_of(img), prompts, None))


# ---- 7. concurrency ------------------------------------------------------------------------------------------------
def test_readers_beside_evicting_writer():
    """Every document's blocks all hold pod 0 with tier 0, so a prompt's row is a pure function of how many of its blocks
    are still consecutively present: Score() beside evicting batches must give 1.0 * j for some j <= blocks."""
    import threading
    import torch
    rng = np.random.default_rng(14)
    ix = clock_index(1024)
    docs = [rng.integers(0, 128256, size=BS * 12).tolist() for _ in range(600)]
    stop = threading.Event()
    errors = []

    def reader():
        r = np.random.default_rng(threading.get_ident() % 1000)
        while not stop.is_set():
            sel = [docs[int(x)] for x in r.integers(0, len(docs), size=64)]
            tok, off = csr(sel)
            rows = ix.score_batch(tok, off)[0]
            ok = np.isin(rows[:, 0], [-1.0] + [float(j) for j in range(1, 13)]) & np.all(rows[:, 1:] == -1.0, axis=1)
            if not ok.all():
                errors.append(rows[~ok][:2])

    threads = [threading.Thread(target=reader) for _ in range(3)]
    for t in threads:
        t.start()
    try:
        dev = torch.device("cuda")
        for i in range(40):
            sel = [docs[int(x)] for x in rng.integers(0, len(docs), size=16)]
            ev = np.zeros(len(sel), EVENT_DTYPE)
            hashes, toks = [], []
            for j, d in enumerate(sel):
                ev[j] = (0, 0, PT(0), 0, 0, len(hashes), len(toks), 12, len(d))
                hashes += [int(x) for x in rng.integers(1, 2 ** 63, size=12, dtype=np.int64)]
                toks += d
            if i % 2:
                rc, _ = ix.apply_events(ev, np.array(hashes, np.uint64), np.array(toks, np.uint32))
                assert rc == 0
            else:
                d_ev = torch.from_numpy(ev.view(np.uint8).copy()).to(dev)
                d_q = torch.tensor([0, len(sel)], dtype=torch.int64, device=dev)
                d_h = torch.tensor(np.array(hashes, np.uint64).view(np.int64), device=dev)
                d_t = torch.tensor(np.array(toks, np.uint32).view(np.int32), device=dev)
                torch.cuda.synchronize()
                ix.apply_events_dev(d_ev.data_ptr(), d_q.data_ptr(), 1, len(sel), d_h.data_ptr(), len(hashes), d_t.data_ptr())
                ix.synchronize()
            st = ix.stats()
            assert st["request_keys"] <= 1024 and st["engine_keys"] <= 1024
    finally:
        stop.set()
        for t in threads:
            t.join()
    assert not errors, errors[:2]
    assert ix.evictions()[0] > 0


# ---- 8. host mirror --------------------------------------------------------------------------------------------------
def test_host_mirror_bounded_and_counted():
    rng = np.random.default_rng(15)
    h = HostIndexer(block_size=BS, capacity=1024, max_pods=P, enable_metrics=True, evict_policy="clock")
    for i in range(200):
        toks = rng.integers(0, 128256, size=BS * 10).tolist()
        hs = [int(x) for x in rng.integers(1, 2 ** 62, size=10)]
        payload = msgpack.packb([1700000000.0 + i, [["BlockStored", hs, None, toks, BS, None, "gpu"]], 0])
        assert h.add_task("pod%d" % (i % 4), "m", payload) == 0
        h.process()
    L, hix = kvidx._native.load(), C.c_void_p(h.L.kvhost_index(h.h))
    st, ev = kvidx._native.Stats(), np.zeros(2, np.uint64)
    assert L.kvidx_get_stats(hix, C.byref(st)) == 0
    assert L.kvidx_get_evictions(hix, ev.ctypes.data_as(C.POINTER(C.c_uint64))) == 0
    assert st.request_keys <= 1024 and st.engine_keys <= 1024 and ev[0] >= 2000 - 1024
    text = h.metrics_text()
    assert "kvcache_index_capacity_evictions_total %d\n" % ev[0] in text
    assert text.rstrip().split("\n")[-1].startswith("kvcache_index_lookup_latency_seconds")


# ---- tombstones of the sweep under asynchronous ingest ---------------------------------------------------------------
def test_async_ingest_compacts_sweep_tombstones():
    """Only kvidx_apply_events_dev writes, far past 0.8 x slots of evictions: the room check sees the sweep's tombstones
    and compacts them, so no batch is refused, every insert lands and both maps stay at capacity."""
    import torch
    rng = np.random.default_rng(16)
    CAP = 1024
    ix = clock_index(CAP)                                         # 4096 slots
    dev = torch.device("cuda")
    slots = ix.stats()["request_slots"]
    n_docs, nb = 32, 8
    batches = 0
    keep = []                    # the call is asynchronous on the handle's write stream: inputs live until synchronize()
    while ix.evictions()[0] < 2 * slots:
        ev = np.zeros(n_docs, EVENT_DTYPE)
        hashes, toks = [], []
        for j in range(n_docs):
            d = rng.integers(0, 128256, size=BS * nb).tolist()
            ev[j] = (0, 0, PT(0), 0, 0, len(hashes), len(toks), nb, len(d))
            hashes += [int(x) for x in rng.integers(1, 2 ** 63, size=nb, dtype=np.int64)]
            toks += d
        d_ev = torch.from_numpy(ev.view(np.uint8).copy()).to(dev)
        d_q = torch.tensor([0, n_docs], dtype=torch.int64, device=dev)
        d_h = torch.tensor(np.array(hashes, np.uint64).view(np.int64), device=dev)
        d_t = torch.tensor(np.array(toks, np.uint32).view(np.int32), device=dev)
        torch.cuda.synchronize()                                  # the inputs have landed (the write stream does not wait for torch's)
        ix.apply_events_dev(d_ev.data_ptr(), d_q.data_ptr(), 1, n_docs, d_h.data_ptr(), len(hashes), d_t.data_ptr())
        keep.append((d_ev, d_q, d_h, d_t))
        batches += 1
        assert batches < 200
    ix.synchronize()
    st = ix.stats()
    assert st["request_keys"] == CAP and st["engine_keys"] == CAP
    assert st["rebuilds"] > 0 and st["request_tombs"] + CAP <= 0.9 * slots
    # every insert landed: the keys that entered equal the keys resident plus the keys evicted
    assert ix.evictions() == (batches * n_docs * nb - CAP, batches * n_docs * nb - CAP)
