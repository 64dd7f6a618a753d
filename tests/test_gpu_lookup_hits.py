"""GPU (-m gpu): Lookup hit counts (kvidx_lookup_hits*, include/kvidx.h): per prompt, recordHitMetrics(Lookup(K_i, F_i)) --
the count the instrumented index adds to kvcache_index_max_pod_hit_count_total and kvcache_index_lookup_hits_total
(instrumented_index.go:71-92).  Checked against the oracle's InstrumentedIndex over random contents (filters, tiers, gaps,
repeated keys with and without a filter, short prompts, offsets, block sizes), at batch sizes up to 1 M prompts against
kvidx_lookup and the map rules in numpy, across the tokens / keys / host / device / pinned forms, for the touches an
exact-LRU or CLOCK handle records, on sharded handles, and through the host mirror's metrics."""
import numpy as np
import pytest

from helpers import decode_snapshot, filter_mask
import kvidx
from kvidx import host as kh
from kvidx._native import _Raw, host_alloc, host_free, pack_text
from oracle import kvoracle as ko

pytestmark = pytest.mark.gpu
W16 = tuple(1.0 - 0.05 * t for t in range(16))


def PT(p, t=0):
    return (p << 4) | t


def key_csr(lists, base=0):
    off = np.zeros(len(lists) + 1, np.int64)
    off[1:] = np.cumsum([len(k) for k in lists])
    body = np.concatenate([np.asarray(k, np.uint64) for k in lists]) if off[-1] else np.zeros(0, np.uint64)
    pad = np.arange(base, dtype=np.uint64) ^ np.uint64(0xBADBAD)            # elements before the first prompt's
    return np.concatenate([pad, body]), off + base


class Pair:
    """A handle and the oracle's InstrumentedIndex over the same Add calls."""

    def __init__(self, P, **kw):
        self.ix = kvidx.Index(max_pods=P, tier_weights=W16, **kw)
        self.oi = ko.InstrumentedIndex(ko.InMemoryIndex(10 ** 8, kw.get("pods_per_key", 10)))

    def add(self, model, request, pts):
        eng = [int(k) ^ 0x5EED for k in request]
        assert self.ix.add(model, eng, request, pts) == 0
        self.oi.add([ko.Key(str(model), e) for e in eng], [ko.Key(str(model), int(k)) for k in request],
                    [ko.PodEntry(str(p >> 4), str(p & 15)) for p in pts])

    def hits(self, lists, models, fm):
        """the oracle's max for each prompt (0 for a prompt without keys: Lookup errors before counting)"""
        out = []
        for i, ks in enumerate(lists):
            if not len(ks):
                out.append(0)
                continue
            row = None if fm is None else fm[i]
            pods = () if row is None or not row.any() else {str(p) for p in range(len(row) * 64) if (int(row[p >> 6]) >> (p & 63)) & 1}
            before = self.oi.metrics.max_pod_hit_count_total
            self.oi.lookup([ko.Key(str(int(models[i])), int(k)) for k in ks], pods)
            out.append(self.oi.metrics.max_pod_hit_count_total - before)
        return np.array(out, np.uint32)


def _contents(rng, pair, P, n_keys=400, models=(0, 3)):
    """random keys of several models, one to twelve entries each (pods of the whole row, all sixteen tiers, one pod on two
    tiers of a key), and keys of one model present only under another"""
    present = {m: [] for m in models}
    for m in models:
        ks = rng.integers(1, 2 ** 63, n_keys, dtype=np.uint64)
        for k in ks:
            pts = list({PT(int(rng.integers(0, P)), int(rng.integers(0, 16))) for _ in range(int(rng.integers(1, 13)))})
            if rng.random() < 0.3:
                p = int(rng.integers(0, P))
                pts += [PT(p, 0), PT(p, 1)]
            pair.add(m, [int(k)], pts)
        present[m] = ks
    return present


def _prompts(rng, present, n=64, models=(0, 3)):
    lists, mids = [], []
    for i in range(n):
        m = models[i % len(models)]
        other = present[models[(i + 1) % len(models)]]
        L = int(rng.integers(0, 60)) if i % 7 else 0                   # empty prompts too
        ks = []
        for _ in range(L):
            r = rng.random()
            ks.append(int(rng.choice(present[m])) if r < 0.6 else int(rng.choice(other)) if r < 0.75 else
                      int(rng.integers(1, 2 ** 63)) if r < 0.85 else (ks[-1] if ks else 5))        # absent keys, repeats
        if ks and i % 3 == 0:
            ks += ks[: len(ks) // 2]                                  # repeats far apart
        lists.append(ks)
        mids.append(m)
    return lists, np.array(mids, np.uint32)


def _filters(rng, n, P, kind):
    FW = (P + 63) // 64
    if kind == "none":
        return None
    if kind == "zero":
        return np.zeros((n, FW), np.uint64)
    if kind == "absent":                                              # pods no entry holds
        return np.stack([filter_mask([P - 1], FW) for _ in range(n)])
    return np.stack([filter_mask(sorted(set(rng.integers(0, P, int(rng.integers(1, 20))).tolist())), FW) if i % 4 else
                     np.zeros(FW, np.uint64) for i in range(n)])


@pytest.mark.parametrize("P", [64, 257, 4096])
@pytest.mark.parametrize("kind", ["none", "zero", "absent", "random"])
def test_against_the_oracle(P, kind):
    rng = np.random.default_rng(P + len(kind))
    pair = Pair(P)
    present = _contents(rng, pair, P - 1 if kind == "absent" else P)
    lists, mids = _prompts(rng, present)
    fm = _filters(rng, len(lists), P, kind)
    want = pair.hits(lists, mids, fm)
    assert kind == "absent" or want.max() > 1
    for base in (0, 5):
        keys, off = key_csr(lists, base)
        got = pair.ix.lookup_hits_keys(keys, off, model=mids, filter_mask=fm)
        assert np.array_equal(got, want), np.nonzero(got != want)
    if kind == "absent":
        assert not want.any()


@pytest.mark.parametrize("filtered", [False, True])
def test_long_prompt_with_repeats(filtered):
    """a prompt of 48 000 keys (past the shared-memory set of one chunk) whose keys repeat within and across chunks"""
    rng = np.random.default_rng(7 + filtered)
    P = 64
    pair = Pair(P)
    present = _contents(rng, pair, P, n_keys=3000, models=(0,))
    ks = rng.choice(present[0], 40000).tolist() + rng.integers(1, 2 ** 63, 4000, dtype=np.uint64).tolist()
    ks += ks[:4000]
    rng.shuffle(ks)
    lists = [ks, ks[:1500], ks[:3], []]
    mids = np.zeros(len(lists), np.uint32)
    fm = np.stack([filter_mask(list(range(0, P, 2)), 1)] * len(lists)) if filtered else None
    want = pair.hits(lists, mids, fm)
    keys, off = key_csr(lists)
    assert np.array_equal(pair.ix.lookup_hits_keys(keys, off, model=mids, filter_mask=fm), want)


@pytest.mark.parametrize("bs", [4, 16, 64, 256])
def test_tokens_form(bs):
    """tokens == hash_keys + the keys form == the oracle; prompts shorter than a block; off[0] != 0; the _dev form"""
    import torch
    rng = np.random.default_rng(bs)
    P = 64
    pair = Pair(P, block_size=bs)
    docs = [rng.integers(0, 1000, bs * int(rng.integers(1, 20)), dtype=np.uint32) for _ in range(24)]
    for d, doc in enumerate(docs):
        k, _ = pair.ix.hash_keys(doc, [0, len(doc)])
        depth = max(1, len(k) - d % 4)
        for j in range(depth):
            pair.add(0, [int(k[j])], [PT((d + j) % P, j % 16), PT((d * 7) % P, 1)])
    prompts = [doc[: len(doc) - int(rng.integers(0, bs))] for doc in docs] + [docs[0][: bs - 1], docs[1][:0]]
    prompts.append(np.concatenate([docs[2], docs[2]]))                # the second copy chains on: other keys
    tok = np.concatenate([np.arange(3, dtype=np.uint32)] + prompts)
    off = 3 + np.concatenate([[0], np.cumsum([len(p) for p in prompts])]).astype(np.int64)
    for fm in (None, np.stack([filter_mask([q for q in range(P) if q % 3], 1)] * len(prompts))):
        keys, koff = pair.ix.hash_keys(tok, off)
        want = pair.hits([keys[koff[i]:koff[i + 1]].tolist() for i in range(len(prompts))], np.zeros(len(prompts)), fm)
        got = pair.ix.lookup_hits(tok, off, filter_mask=fm)
        assert np.array_equal(got, want)
        assert np.array_equal(pair.ix.lookup_hits_keys(keys, koff, filter_mask=fm), want)
        dev = torch.device("cuda", 0)
        d_t = torch.from_numpy(tok.view(np.int32)).to(dev)
        d_o = torch.from_numpy(off).to(dev)
        d_h = torch.zeros(len(prompts), dtype=torch.int32, device=dev)
        d_f = None if fm is None else torch.from_numpy(fm.view(np.int64)).to(dev)
        torch.cuda.synchronize(dev)
        pair.ix.lookup_hits_dev(d_t.data_ptr(), d_o.data_ptr(), len(prompts), d_h.data_ptr(), d_filter=0 if d_f is None else d_f.data_ptr())
        pair.ix.synchronize()
        assert d_h.cpu().numpy().view(np.uint32).tobytes() == got.tobytes()


def _numpy_hits(ix, keys, off, model0, fm, P):
    """the reference at scale: ONE kvidx_lookup over the concatenated keys (no filter), then each prompt's filter and the
    map rules (unfiltered: a repeated key once; filtered: every occurrence) in numpy"""
    n = len(off) - 1
    rc, pt, cnt = ix.lookup(model0, keys)
    assert rc == 0
    pid = np.repeat(np.arange(n), np.diff(off))
    rows = fm if fm is not None else np.zeros((n, (P + 63) // 64), np.uint64)
    unf = ~rows.any(axis=1)
    first = np.zeros(len(keys), bool)
    _, idx = np.unique(np.stack([pid, keys.view(np.int64)], 1), axis=0, return_index=True)
    first[idx] = True
    keep_key = np.where(unf[pid], first, True)
    j = np.arange(10)[None, :] < cnt[:, None]
    kk, jj = np.nonzero(j & keep_key[:, None])
    pods = (pt[kk, jj] >> 4).astype(np.int64)
    pr = pid[kk]
    inrow = (rows[pr, pods >> 6] >> (pods & 63).astype(np.uint64)) & np.uint64(1)
    ok = unf[pr] | (inrow == 1)
    u, c = np.unique(pr[ok] * P + pods[ok], return_counts=True)
    out = np.zeros(n, np.uint32)
    np.maximum.at(out, u // P, c.astype(np.uint32))
    return out


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4096, 65536, 1 << 20])
def test_at_scale(n):
    rng = np.random.default_rng(n)
    P = 257
    ix = kvidx.Index(max_pods=P, capacity=1 << 21)
    pool = rng.integers(1, 2 ** 63, 200000, dtype=np.uint64)
    for s in range(0, len(pool), 20000):
        ks = pool[s:s + 20000]
        assert ix.add(0, ks ^ np.uint64(0x5EED), ks, [PT(int(rng.integers(0, P)), t) for t in range(3)] + [PT(s // 20000, 5)]) == 0
    lens = rng.integers(0, 9, n)
    keys = rng.choice(np.concatenate([pool, rng.integers(1, 2 ** 63, 50000, dtype=np.uint64)]), int(lens.sum()))
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    dup = rng.random(len(keys)) < 0.1                                  # repeats inside a prompt
    keys[1:][dup[1:]] = keys[:-1][dup[1:]]
    fm = np.zeros((n, 5), np.uint64)                                   # 40 random pods per row; every third row all pods
    for c in range(40):
        q = rng.integers(0, P, n)
        fm[np.arange(n), q >> 6] |= np.uint64(1) << (q & 63).astype(np.uint64)
    fm[::3] = 0
    ref = kvidx.Index(max_pods=P, capacity=1 << 21)
    ref.restore(ix.snapshot())
    want = _numpy_hits(ref, keys, off, 0, fm, P)
    got = ix.lookup_hits_keys(keys, off, filter_mask=fm)
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:5]
    assert np.array_equal(ix.lookup_hits_keys(keys, off), _numpy_hits(ref, keys, off, 0, None, P))
    # host == _dev, byte for byte; pinned == pageable
    import torch
    dev = torch.device("cuda", 0)
    d_k, d_o = torch.from_numpy(keys.view(np.int64)).to(dev), torch.from_numpy(off).to(dev)
    d_f, d_h = torch.from_numpy(fm.view(np.int64)).to(dev), torch.zeros(n, dtype=torch.int32, device=dev)
    torch.cuda.synchronize(dev)
    ix.lookup_hits_keys_dev(d_k.data_ptr(), d_o.data_ptr(), n, d_h.data_ptr(), d_filter=d_f.data_ptr())
    ix.synchronize()
    assert d_h.cpu().numpy().view(np.uint32).tobytes() == got.tobytes()
    p = host_alloc(max(keys.nbytes, 8))
    try:
        np.ctypeslib.as_array((np.ctypeslib.ctypes.c_uint64 * len(keys)).from_address(p))[:] = keys
        assert ix.lookup_hits_keys(_Raw(p), off, filter_mask=fm).tobytes() == got.tobytes()
    finally:
        host_free(p)


def _ranks(img):
    req, _ = decode_snapshot(img)
    R = len(req)
    rec = np.frombuffer(bytes(img), "<u8", R, 64 + 32 * R + 24 * len(_))
    return dict(zip(zip(req["model"].tolist(), req["hash"].tolist()), np.argsort(np.argsort(rec)).tolist()))


def test_exact_lru_touches_equal_one_lookup_per_prompt():
    rng = np.random.default_rng(11)
    P = 64
    a = kvidx.Index(max_pods=P, lru_exact=1, capacity=4096)
    ks = rng.integers(1, 2 ** 63, 600, dtype=np.uint64)
    for i in range(0, 600, 50):
        assert a.add(0, ks[i:i + 50] ^ np.uint64(1), ks[i:i + 50], [PT(i % P), PT(3, 2)]) == 0
    b = kvidx.Index(max_pods=P, lru_exact=1, capacity=4096)
    b.restore(a.snapshot())
    lists = [rng.choice(ks, int(rng.integers(1, 40))).tolist() + [int(x) for x in rng.integers(1, 2 ** 63, 2, dtype=np.uint64)] for _ in range(50)]
    lists[3] = lists[3] + lists[3][:5]                                # a key repeated: ranks as of its last occurrence
    keys, off = key_csr(lists)
    a.lookup_hits_keys(keys, off)
    for l in lists:
        assert b.lookup(0, l)[0] == 0
    assert _ranks(a.snapshot()) == _ranks(b.snapshot())


def _ranks_any(ix):
    req, _ = decode_snapshot(ix.snapshot())
    return [(int(h), int(m)) for h, m in zip(req["hash"], req["model"])]


def test_clock_touches_equal_one_lookup_per_prompt():
    rng = np.random.default_rng(12)
    P = 64
    mk = lambda: kvidx.Index(max_pods=P, evict_policy="clock", capacity=512)
    a, b = mk(), mk()
    ks = rng.integers(1, 2 ** 63, 512, dtype=np.uint64)
    pre = rng.integers(1, 2 ** 63, 64, dtype=np.uint64)
    for ix in (a, b):
        assert ix.add(0, ks ^ np.uint64(1), ks, [PT(2)]) == 0
        assert ix.add(0, pre ^ np.uint64(1), pre, [PT(3)]) == 0            # past capacity: the sweep clears bits as it goes
    ks = np.array([k for k, _ in _ranks_any(a)], np.uint64)
    lists = [rng.choice(ks, 8).tolist() for _ in range(20)]
    keys, off = key_csr(lists)
    a.lookup_hits_keys(keys, off)
    for l in lists:
        assert b.lookup(0, l)[0] == 0
    new = rng.integers(1, 2 ** 63, 200, dtype=np.uint64)
    for ix in (a, b):
        assert ix.add(0, new ^ np.uint64(1), new, [PT(4)]) == 0
    assert a.snapshot() == b.snapshot()


@pytest.mark.parametrize("shards", [2, 8])
def test_sharded_equals_unsharded(shards):
    from test_gpu_shard_ops import _shards
    rng = np.random.default_rng(shards)
    P = 64
    sh = _shards(shards, "same-gpu", hash_seed="", pods_per_key=10, max_pods=P, tier_weights=W16)
    ix = kvidx.Index(max_pods=P, tier_weights=W16)
    ks = rng.integers(1, 2 ** 63, 2000, dtype=np.uint64)
    for i in range(0, 2000, 100):
        pts = [PT(int(rng.integers(0, P)), int(rng.integers(0, 16))) for _ in range(5)]
        for t in (ix, sh[i // 100 % shards]):
            assert t.add(0, ks[i:i + 100] ^ np.uint64(1), ks[i:i + 100], pts) == 0
    lists = [rng.choice(ks, int(rng.integers(0, 70))).tolist() for _ in range(300)]
    keys, off = key_csr(lists)
    fm = _filters(rng, len(lists), P, "random")
    for f in (None, fm):
        want = ix.lookup_hits_keys(keys, off, filter_mask=f)
        for s in sh:
            assert np.array_equal(s.lookup_hits_keys(keys, off, filter_mask=f), want)


def test_host_mirror_metrics_and_launches():
    """the host mirror's hit counters against the oracle for every entry point, repeated keys included; and a metrics-on
    batch adds a constant number of kernel launches, not two per prompt"""
    rng = np.random.default_rng(5)
    model = "m"
    h = kh.HostIndexer(block_size=16, capacity=1 << 16, max_pods=64, enable_metrics=True)
    oi = ko.Indexer(block_size=16, size=10 ** 6)
    oi.index = ko.InstrumentedIndex(oi.index)
    docs = [rng.integers(0, 5000, 16 * 12, dtype=np.uint32) for _ in range(16)]
    for d, doc in enumerate(docs):
        keys = [k.chunk_hash for k in oi.tokens_processor.tokens_to_kv_block_keys(None, doc.tolist(), model)]
        for j, k in enumerate(keys[: 12 - d % 5]):
            ents = [("p%d" % ((d + j) % 5), "gpu"), ("p%d" % (d % 3), "cpu")]
            assert h.add(model, [k ^ 1], [k], ents) == 0
            oi.index.add([ko.Key(model, k ^ 1)], [ko.Key(model, k)], [ko.PodEntry(p, t) for p, t in ents])
    for d, doc in enumerate(docs[:6]):
        flt = () if d % 2 else ("p1", "p2")
        assert h.get_pod_scores(doc, model, flt) == oi.get_pod_scores(doc.tolist(), model, flt)
        keys = [k.chunk_hash for k in oi.tokens_processor.tokens_to_kv_block_keys(None, doc.tolist(), model)]
        rep = keys + keys[:4] + keys[2:3]                              # repeated keys
        h.get_pod_scores_keys(rep, model, flt)
        oi.index.lookup([ko.Key(model, k) for k in rep], set(flt))
        h.lookup(model, rep, flt)
        oi.index.lookup([ko.Key(model, k) for k in rep], set(flt))
        held, _ = keys[:5], None
        h.get_pod_scores_turn(held, doc[16 * 5:], model, flt)
        oi.index.lookup([ko.Key(model, k) for k in keys], set(flt))
    off = np.concatenate([[0], np.cumsum([len(d) for d in docs])]).astype(np.int64)
    h.get_pod_scores_batch(np.concatenate(docs), off, model)
    for doc in docs:
        oi.get_pod_scores(doc.tolist(), model)
    # text: three cached prompts of 64 four-byte tokens each, and one the store has never seen (left to the tokenizer)
    ix = kvidx.Index.borrow(h.L.kvhost_index(h.h), max_pods=64)
    ix.text_store_init(1000, 64)
    texts = [bytes(rng.integers(97, 123, 256, dtype=np.uint8)) for _ in range(4)]
    tx, toff = pack_text(texts[:3])
    span = np.array([(4 * t, 4 * t + 4) for t in range(64)] * 3, np.uint64)
    ix.text_store_add(tx, toff, np.concatenate([d[:64] for d in docs[:3]]), span, np.arange(0, 256, 64, dtype=np.int64))
    tx, toff = pack_text(texts)
    rows, tz = h.get_pod_scores_text(tx, toff, model)
    assert tz.tolist() == [0, 0, 0, 1] and rows[3] is None
    for doc in docs[:3]:
        oi.get_pod_scores(doc[:64].tolist(), model)
    got, want = h.metrics(), oi.index.metrics
    assert want.max_pod_hit_count_total > 0
    for name in ("lookup_requests_total", "max_pod_hit_count_total", "lookup_hits_total", "lookup_latency_count"):
        assert got[name] == getattr(want, name), (name, got[name], getattr(want, name))
    # launches: one batch of 4096 prompts with metrics on and off
    big = np.tile(np.concatenate(docs), 256)
    boff = np.arange(0, 4097 * 192, 192, dtype=np.int64)
    plain = kh.HostIndexer(block_size=16, capacity=1 << 16, max_pods=64)
    for hh in (h, plain):
        pix = kvidx.Index.borrow(hh.L.kvhost_index(hh.h), max_pods=64)
        hh.get_pod_scores_batch(big, boff, model)
        l0 = pix.stats()["kernel_launches"]
        hh.get_pod_scores_batch(big, boff, model)
        hh.delta = pix.stats()["kernel_launches"] - l0
    assert h.delta - plain.delta <= 4, (h.delta, plain.delta)


def test_errors():
    ix = kvidx.Index(max_pods=64)
    L, hd = ix.L, ix.h
    k = np.arange(4, dtype=np.uint64)
    off = np.array([0, 2, 4], np.int64)
    bad = np.array([0, 3, 2], np.int64)
    hits = np.zeros(2, np.uint32)
    from kvidx._native import _p, _u64p, _i64p, _u32p, EINVAL
    assert L.kvidx_lookup_hits_keys(None, _p(k, _u64p), _p(off, _i64p), 2, None, 0, None, _p(hits, _u32p)) == EINVAL
    assert L.kvidx_lookup_hits_keys(hd, _p(k, _u64p), _p(off, _i64p), -1, None, 0, None, _p(hits, _u32p)) == EINVAL
    assert L.kvidx_lookup_hits_keys(hd, _p(k, _u64p), None, 2, None, 0, None, _p(hits, _u32p)) == EINVAL
    assert L.kvidx_lookup_hits_keys(hd, _p(k, _u64p), _p(bad, _i64p), 2, None, 0, None, _p(hits, _u32p)) == EINVAL
    assert L.kvidx_lookup_hits_keys(hd, None, _p(off, _i64p), 2, None, 0, None, _p(hits, _u32p)) == EINVAL
    assert L.kvidx_lookup_hits_keys(hd, _p(k, _u64p), _p(off, _i64p), 2, None, 0, None, None) == EINVAL
    assert L.kvidx_lookup_hits(hd, None, _p(off, _i64p), 2, None, 0, None, _p(hits, _u32p)) == EINVAL
    assert L.kvidx_lookup_hits_keys_dev(hd, None, None, 2, None, 0, None, None) == EINVAL
    assert L.kvidx_lookup_hits_dev(hd, None, None, 2, None, 0, None, None) == EINVAL
    hits[:] = 7
    assert L.kvidx_lookup_hits_keys(hd, None, _p(off, _i64p), 0, None, 0, None, _p(hits, _u32p)) == 0
    assert (hits == 7).all()                                           # n_prompts == 0: nothing written
    assert L.kvidx_lookup_hits_keys(hd, None, np.zeros(3, np.int64).ctypes.data_as(_i64p), 2, None, 0, None, _p(hits, _u32p)) == 0
    assert (hits == 0).all()                                           # no key: 0
