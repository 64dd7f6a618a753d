"""GPU (-m gpu): Score() at 32-, 64- and 128-token blocks on the warp-per-prompt kernels (coop_score_kernel<B>,
score_turn_kernel<B>).  Every row is checked byte for byte against a handle forced onto the thread-per-prompt kernel
(KVIDX_SCORE_KERNEL=v1) and against the C++ oracle: batch sizes on both sides of the dispatch edges, CBOR width and
payload extremes, parents below 2^32, chunk edges, misses at every block of a chunk, filters, models, displaced probe
chains, CLOCK reference bits, shards, host buffers, conversation turns, and which kernel each call launches."""
import threading

import numpy as np
import pytest

from helpers import _index_pair, csr, filter_mask, keys_homed_at
from test_gpu_score_keys import same_sparse
from test_gpu_score_turn import split_turn
import kvidx
from oracle.kvoracle_c import COracle

pytestmark = pytest.mark.gpu
SIZES = [32, 64, 128]
CHUNK = 512                                   # tokens per staged chunk of the cooperative kernels
EDGE = np.array([0, 23, 24, 255, 256, 65535, 65536, 2 ** 32 - 1], np.uint32)


def PT(p, t=0):
    return (p << 4) | t


def _pair(monkeypatch, B, init_hash=None, **kw):
    """(default handle, v1 handle, oracle) over one configuration; init_hash: the chain's first parent (else the hash of
    the empty seed)"""
    kw = dict(dict(capacity=1 << 15, max_pods=64), block_size=B, **kw)
    ix, co = _index_pair(**kw)
    monkeypatch.setenv("KVIDX_SCORE_KERNEL", "v1")
    iv, _ = _index_pair(**kw)
    monkeypatch.delenv("KVIDX_SCORE_KERNEL")
    if init_hash is not None:
        w = kw.pop("tier_weights", (1.0, 0.8))
        ix = kvidx.Index(init_hash=init_hash, tier_weights=w, **kw)
        monkeypatch.setenv("KVIDX_SCORE_KERNEL", "v1")
        iv = kvidx.Index(init_hash=init_hash, tier_weights=w, **kw)
        monkeypatch.delenv("KVIDX_SCORE_KERNEL")
        co = COracle(block_size=B, init_hash=init_hash, size=kw["capacity"], tier_weights=w, max_pods=kw["max_pods"])
    return ix, iv, co


def _store(handles, model, keys, pts, tag=0x77):
    keys = np.asarray(keys, np.uint64)
    for h in handles:
        assert h.add(model, keys ^ np.uint64(tag), keys, pts) == 0


def _docs(rng, B, n, nblk, share=3):
    docs = [rng.integers(0, 50000, B * int(nblk[i % len(nblk)]), dtype=np.uint32) for i in range(n)]
    for d in range(4, n):
        s = min(share, len(docs[d]) // B, len(docs[d % 4]) // B)
        docs[d][:B * s] = docs[d % 4][:B * s]
    return docs


def _fill_docs(rng, handles, co, docs, P, models=(0,)):
    for d, doc in enumerate(docs):
        k = co.hash_keys(doc, [0, len(doc)])[0]
        depth = len(k) - int(rng.integers(0, len(k) // 2 + 1))
        pts = [PT(int(p), int(rng.integers(0, 2))) for p in rng.choice(P, size=int(rng.integers(1, 4)), replace=False)]
        _store(list(handles) + [co], models[d % len(models)], k[:depth], pts)


def check(ix, iv, co, tok, off, **kw):
    """dense and sparse rows of the default handle == the v1 handle's == the oracle's"""
    s, h = ix.score_batch(tok, off, **kw)
    sv, hv = iv.score_batch(tok, off, **kw)
    assert s.tobytes() == sv.tobytes(), np.argwhere(s != sv)[:5]
    assert np.array_equal(h, hv)
    assert same_sparse(ix.score_batch_sparse(tok, off, **kw), iv.score_batch_sparse(tok, off, **kw))
    okw = {k: v for k, v in kw.items() if k in ("model", "model0", "filter_mask")}
    want = co.score_batch(tok, off, n_threads=8, **okw)[0]
    assert s.tobytes() == want.tobytes(), np.argwhere(s != want)[:5]
    return s, h


# ---- 1. batch sizes on both sides of every edge ------------------------------------------------------------------------
@pytest.mark.parametrize("B", SIZES)
def test_batch_sizes(B, monkeypatch):
    rng = np.random.default_rng(B)
    P = 64
    ix, iv, co = _pair(monkeypatch, B)
    monkeypatch.setenv("KVIDX_SCORE_PATH", "coop")                   # batches above the threshold forced onto coop<B>
    ic = kvidx.Index(capacity=1 << 15, max_pods=P, block_size=B)
    monkeypatch.delenv("KVIDX_SCORE_PATH")
    docs = _docs(rng, B, 24, [2, 5, 9, 17])
    _fill_docs(rng, (ix, iv, ic), co, docs, P)
    for n in (1, 31, 32, 33, 2048, 2049):
        prompts = [docs[int(rng.integers(0, len(docs)))][:int(rng.integers(0, 20 * B))] for _ in range(n)]
        tok, off = csr(prompts)
        s, _ = check(ix, iv, co, tok, off)
        if n >= 32:
            assert (s.max(axis=1) > 1).any()
    prompts = [docs[i % len(docs)][:int(rng.integers(0, 20 * B))] for i in range(5000)]
    tok, off = csr(prompts)
    assert ic.score_batch(tok, off)[0].tobytes() == iv.score_batch(tok, off)[0].tobytes()


# ---- 2. payload extremes and 3. prompt shapes ---------------------------------------------------------------------------
@pytest.mark.parametrize("init", [None, 12345])
@pytest.mark.parametrize("B", SIZES)
def test_payloads_and_shapes(B, init, monkeypatch):
    """shortest and longest payloads, every CBOR width edge; fewer than B tokens, exactly B, partial tails, one chunk, one
    chunk and a block, 16 K tokens; a first miss at every block of a chunk; an init_hash above 2^32 and one below it (block
    0 then takes the plain chain on every lane)"""
    rng = np.random.default_rng(B + (init or 0))
    ix, iv, co = _pair(monkeypatch, B, init_hash=init)
    kinds = [
        lambda L: rng.integers(0, 24, L, dtype=np.uint32),                                     # shortest payload
        lambda L: rng.integers(65536, 2 ** 32, L, dtype=np.uint64).astype(np.uint32),          # longest: 5 B + 13 bytes
        lambda L: EDGE[rng.integers(0, len(EDGE), L)],
        lambda L: rng.integers(0, 50000, L, dtype=np.uint32),
    ]
    lens = [B - 1, B, B + 7, CHUNK, CHUNK + B, CHUNK * 2 - 1, 16384, 3 * CHUNK + B // 2]
    docs = [kinds[i % 4](lens[i % len(lens)]) for i in range(32)]
    for d, doc in enumerate(docs):                                   # every block stored: walks run to the end
        k = co.hash_keys(doc, [0, len(doc)])[0]
        if len(k):
            _store((ix, iv, co), 0, k, [PT(d % 5), PT(9, 1)])
    prompts = list(docs)
    # a first miss at every block position inside a chunk (and the one after it)
    base = docs[4] if len(docs[4]) >= CHUNK + B else docs[12]
    for j in range(CHUNK // B + 1):
        p = base[:CHUNK + B].copy()
        p[j * B] ^= 1
        prompts.append(p)
    tok, off = csr(prompts)
    check(ix, iv, co, tok, off)
    check(ix, iv, co, tok, off, filter_mask=np.array([filter_mask([d % 5], 1) for d in range(len(prompts))]))
    # tokens at an odd 4-byte offset: the LDG staging branch
    buf = np.concatenate([np.zeros(1, np.uint32), tok])
    a = ix.score_batch(buf, off + 1)[0]
    assert a.tobytes() == iv.score_batch(tok, off)[0].tobytes()


@pytest.mark.parametrize("B", SIZES)
def test_short_parent(B, monkeypatch):
    """turns whose last held key is below 2^32: the new tokens' first block takes the plain chain on every lane"""
    rng = np.random.default_rng(B + 100)
    ix, iv, co = _pair(monkeypatch, B)
    lists = [np.array([x], np.uint64) for x in (1, 2, 0xFFFFFFFF, 1 << 20)] * 8
    toks = [EDGE[rng.integers(0, len(EDGE), B * (1 + i % 12) + i % 5)] for i in range(len(lists))]
    held = np.concatenate(lists)
    hoff = np.arange(len(lists) + 1, dtype=np.int64)
    tok, toff = csr(toks)
    nk, nko = co.hash_keys(tok, toff, parent=held, parent_valid=np.ones(len(lists), np.uint8))
    for i in range(len(lists)):
        _store((ix, iv, co), 0, np.concatenate([lists[i], nk[nko[i]:nko[i + 1] - i % 3]]), [PT(i % 7)])
    a = ix.score_turn(held, hoff, tok, toff)
    b = iv.score_turn(held, hoff, tok, toff)
    assert a[0].tobytes() == b[0].tobytes() and a[2].tobytes() == b[2].tobytes() == nk.tobytes()
    assert (a[0].max(axis=1) > 1).any()


# ---- 3. filters, models, displaced chains, wide pod rows ---------------------------------------------------------------
@pytest.mark.parametrize("P", [257, 4096])
@pytest.mark.parametrize("B", SIZES)
def test_filters_models_displaced(B, P, monkeypatch):
    rng = np.random.default_rng(B * P)
    W = [1.0 - 0.05 * t for t in range(16)]
    ix, iv, co = _pair(monkeypatch, B, max_pods=P, tier_weights=W, capacity=1 << 14)
    docs = _docs(rng, B, 16, [3, 9, 20])
    pods = sorted({0, 1, 5, 63, 64, 127, 200, 256, P - 1})
    for d, doc in enumerate(docs):
        k = co.hash_keys(doc, [0, len(doc)])[0]
        m = d % 3
        for j in range(len(k)):
            pts = [PT(pods[(d + j + q) % len(pods)], (j + q) % 16) for q in range(1 + (d + j) % 3)]
            if d % 4 == 1 and j >= 2:
                pts = [PT(pods[-1], j % 16)]                 # the pods of block 0 leave: the walk's active set empties mid-chunk
            _store((ix, iv, co), m, k[j:j + 1], pts)
    # displaced and wrapped probe chains: keys homed on the pairs of the table's last slots and of slot 0
    S = 1 << 15
    ks = keys_homed_at(np.array([S - 2] * 6 + [0] * 4, np.int64), 0, S, rng)
    _store((ix, iv, co), 0, ks, [PT(3, 2)], tag=0x99)
    prompts, model = [], []
    for i in range(600):
        d = i % len(docs)
        prompts.append(docs[d][:int(rng.integers(0, len(docs[d]) + 1))] if i % 3 else docs[d])
        model.append(d % 3 if i % 7 else (d + 1) % 3)
    tok, off = csr(prompts)
    model = np.array(model, np.uint32)
    FW = (P + 63) // 64
    fm = np.zeros((len(prompts), FW), np.uint64)
    for i in range(len(prompts)):
        if i % 4 == 1:
            fm[i] = filter_mask([pods[i % len(pods)]], FW)
        elif i % 4 == 2:
            fm[i] = filter_mask(rng.choice(pods, size=int(rng.integers(1, len(pods) + 1)), replace=False).tolist(), FW)
    for kw in ({"model": model}, {"model": model, "filter_mask": fm}):
        check(ix, iv, co, tok, off, **kw)


# ---- 4. CLOCK ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", SIZES)
def test_clock_marks(B):
    from clock_oracle import referenced_keys
    from test_gpu_clock import MODELS, PODS, _new_keys, clock_index, oracle_of, resident
    rng = np.random.default_rng(B + 5)
    C = 256
    ix = clock_index(C, block_size=B)
    docs = [rng.integers(0, 128256, size=B * 8).tolist() for _ in range(32)]
    for d, doc in enumerate(docs):
        k, _ = ix.hash_keys(np.asarray(doc, np.uint32), np.array([0, len(doc)], np.int64))
        for b in range(len(k)):
            ents = [PT(1)] if (b >= 4 and d % 4 == 0) else [PT(0), PT(1)]
            assert ix.add(d % 2, [int(k[b]) ^ 0x5A5A], [int(k[b])], ents) == 0
    ka, ea = _new_keys(rng, 1)
    assert ix.add(0, ea, ka, [PT(2)]) == 0                            # a full turn: every key unreferenced
    img = resident(ix)[2]
    prompts, filters = [], []
    for i in range(300):
        d = int(rng.integers(0, 12))
        t = list(docs[d])
        kind = i % 4
        if kind == 1:
            t = t[:B * int(rng.integers(0, 8))] + rng.integers(0, 128256, B * 2).tolist()
        elif kind == 2:
            t = t[:int(rng.integers(0, len(t)))]
        prompts.append((t, MODELS[d % 2]))
        filters.append(["p0"] if kind == 3 else None)
    R = {(MODELS.index(k.model), k.chunk_hash) for k in referenced_keys(oracle_of(img), prompts, filters, block_size=B)}
    tok, off = csr([t for t, _ in prompts])
    model = np.array([MODELS.index(m) for _, m in prompts], np.uint32)
    fm = np.zeros((len(prompts), ix.filter_words), np.uint64)
    for i, f in enumerate(filters):
        if f:
            fm[i] = filter_mask([PODS.index(p) for p in f], ix.filter_words)
    ix.score_batch(tok, off, model=model, filter_mask=fm)
    kn, en = _new_keys(rng, C - len(R))
    assert ix.add(0, en, kn, [PT(3)]) == 0
    assert resident(ix)[0] == R | {(0, x) for x in kn}


# ---- 5. sharded ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shards", [2, 8])
@pytest.mark.parametrize("B", SIZES)
def test_sharded(B, shards, monkeypatch):
    from test_gpu_shard_ops import _shards
    rng = np.random.default_rng(B + shards)
    P = 64
    cfg = dict(block_size=B, hash_seed="abc", capacity=1 << 15, pods_per_key=4, tier_weights=(1.0, 0.8), max_pods=P)
    ix = kvidx.Index(**cfg)
    co = COracle(block_size=B, init_hash=kvidx.fnv64a(b"abc"), size=1 << 15)
    docs = _docs(rng, B, 16, [3, 11])
    sh = _shards(shards, "same-gpu", **cfg)
    for d, doc in enumerate(docs):
        k = co.hash_keys(doc, [0, len(doc)])[0]
        _store([ix, sh[0]], 0, k[:len(k) - d % 3], [PT(d % 9), PT(20, 1)])
    tok, off = csr([docs[i % 16][:int(rng.integers(0, len(docs[i % 16]) + 1))] for i in range(300)])
    a = ix.score_batch(tok, off)[0]
    b = sh[0].score_batch(tok, off)[0]
    assert a.tobytes() == b.tobytes() and (a > 1).any()


# ---- 6. host buffers -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", SIZES)
def test_host_buffers(B, monkeypatch):
    rng = np.random.default_rng(B + 9)
    P = 64
    monkeypatch.setenv("KVIDX_HOST_CHUNK_TOKENS", str(8 * B * 50))     # several chunks per 600-prompt call
    ix, iv, co = _pair(monkeypatch, B)
    docs = _docs(rng, B, 16, [2, 6, 12])
    _fill_docs(rng, (ix, iv), co, docs, P)
    prompts = [docs[i % 16][:int(rng.integers(0, len(docs[i % 16]) + 1))] for i in range(600)]
    tok, off = csr(prompts)
    want = co.score_batch(tok, off, n_threads=8)[0]
    ptok = kvidx.pinned_array(tok.shape, np.uint32)
    ptok[:] = tok
    for n in (1, 32, 600):                                           # zero-copy, zero-copy edge, chunked
        for src in (tok, ptok):
            o = off[:n + 1]
            assert ix.score_batch(src, o)[0].tobytes() == want[:n].tobytes()
            out = kvidx.pinned_array((n, P), np.float64)
            ix.score_batch(src, o, out=out)
            assert out.tobytes() == want[:n].tobytes()
            assert same_sparse(ix.score_batch_sparse(src, o), iv.score_batch_sparse(tok, o))
    # 16 threads, one prompt each, at once: the coalesced launch hands every caller its own row
    errs = []

    def one(t):
        try:
            for r in range(20):
                i = (t * 37 + r) % len(prompts)
                got = ix.score_batch(prompts[i], np.array([0, len(prompts[i])], np.int64))[0]
                if got.tobytes() != want[i:i + 1].tobytes():
                    errs.append((t, i))
        except Exception as e:                                       # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=one, args=(t,)) for t in range(16)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs[:3]


def test_host_indexer_b64(monkeypatch):
    from kvidx.host import HostIndexer
    rng = np.random.default_rng(64)
    B = 64
    hs = []
    for kernel in (None, "v1"):
        if kernel:
            monkeypatch.setenv("KVIDX_SCORE_KERNEL", kernel)
        hs.append(HostIndexer(block_size=B, capacity=4096, max_pods=64))
    monkeypatch.delenv("KVIDX_SCORE_KERNEL")
    docs = _docs(rng, B, 8, [3, 7])
    from oracle import kvoracle as ko
    for d, doc in enumerate(docs):
        k = [x.chunk_hash for x in ko.ChunkedTokenDatabase(B).tokens_to_kv_block_keys(None, doc.tolist(), "m")]
        for h in hs:
            assert h.add("m", [x ^ 0x33 for x in k[:len(k) - d % 2]], k[:len(k) - d % 2], [("pod-%d" % (d % 3), "gpu"), ("pod-9", "cpu")]) == 0
    seen = 0
    for i in range(40):
        p = docs[i % 8][:int(rng.integers(0, len(docs[i % 8]) + 1))].tolist()
        a, b = hs[0].get_pod_scores(p, "m"), hs[1].get_pod_scores(p, "m")
        assert a == b
        seen += bool(a)
    assert seen > 10


# ---- 7. turns ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("clock", [False, True])
@pytest.mark.parametrize("B", SIZES)
def test_turns(B, clock, monkeypatch):
    rng = np.random.default_rng(B + clock)
    P = 64
    kw = {"evict_policy": "clock", "table_slots": 1 << 17} if clock else {}
    ix, iv, co = _pair(monkeypatch, B, **kw)
    docs = _docs(rng, B, 16, [2, 9, 17, 40])
    _fill_docs(rng, (ix, iv), co, docs, P)
    prompts = [docs[i % 16][:int(rng.integers(0, len(docs[i % 16]) + 1))] if i % 3 else docs[i % 16] for i in range(400)]
    tok, off = csr(prompts)
    keys, koff = co.hash_keys(tok, off)
    want, wh = ix.score_batch(tok, off)
    assert want.tobytes() == iv.score_batch(tok, off)[0].tobytes()
    nblk = (np.diff(off) // B).max()
    for split in list(range(0, 10)) + [CHUNK // B - 1, CHUNK // B, CHUNK // B + 1, int(nblk)]:   # every block-boundary split
        held, hoff, nt, toff, nk, nko = split_turn(tok, off, keys, koff, np.full(len(prompts), split), bs=B)
        for h in (ix, iv):
            s, hh, k2, o2 = h.score_turn(held, hoff, nt, toff)
            assert s.tobytes() == want.tobytes() and np.array_equal(hh, wh)
            assert k2.tobytes() == nk.tobytes() and np.array_equal(o2, nko)
        s3, _, k3, _ = ix.score_turn(held, hoff, nt, toff, want_keys=False)
        assert k3 is None and s3.tobytes() == want.tobytes()
        assert same_sparse(ix.score_turn_sparse(held, hoff, nt, toff)[:4], iv.score_turn_sparse(held, hoff, nt, toff)[:4])


# ---- 8. dispatch ---------------------------------------------------------------------------------------------------------
def _kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize("B", SIZES)
def test_dispatch(B):
    import torch
    torch.cuda.init()
    rng = np.random.default_rng(B)
    ix = kvidx.Index(capacity=1 << 12, max_pods=16, block_size=B)
    doc = rng.integers(0, 50000, 4 * B, dtype=np.uint32)

    def names(n, turn=False):
        tok = np.tile(doc, n)
        off = np.arange(n + 1, dtype=np.int64) * len(doc)
        if turn:
            return _kernels(lambda: ix.score_turn(np.zeros(0, np.uint64), np.zeros(n + 1, np.int64), tok, off))
        return _kernels(lambda: ix.score_batch(tok, off))
    coop, v1 = "coop_score_kernel<%d>" % B, "score_kernel_v1"
    for n in (1, 2048):
        ks = names(n)
        assert any(coop in k for k in ks) and not any(v1 in k for k in ks), (n, ks)
    ks = names(2049)
    assert any(v1 in k for k in ks) and not any("coop_score_kernel" in k for k in ks), ks
    ks = names(3, turn=True)
    assert any("score_turn_kernel<%d>" % B in k for k in ks), ks
    i256 = kvidx.Index(capacity=1 << 12, max_pods=16, block_size=256)
    doc = rng.integers(0, 50000, 512, dtype=np.uint32)
    ks = _kernels(lambda: i256.score_batch(doc, np.array([0, 512], np.int64)))
    assert any(v1 in k for k in ks) and not any("coop_score_kernel" in k for k in ks), ks
