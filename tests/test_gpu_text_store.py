"""GPU (-m gpu): the device prefix store (kvidx_text_store_*) and Score() from text (kvidx_score_text*).

The store is checked call by call against the host store (kvhost_prefix_store_*, host.PrefixStore) replaying the same
prompts one at a time in array order -- every find's tokens, offsets and ratios bit for bit and the resident count after
every call -- and, on small cases, against the oracle's restatement (oracle/kvoracle.py::LRUTokenStore).  Score() from text
is checked against the host store's find followed by score_batch of the contained tokens of the prompts that pass the
overlap ratio, at batch sizes on both sides of every Score() dispatch threshold."""
import numpy as np
import pytest

import kvidx
from kvidx import pack_text
from kvidx.host import PrefixStore, xxhash64
from oracle import kvoracle as ko

pytestmark = pytest.mark.gpu
BS = 16                                   # index block size (tokens)
CHARS = np.array(list("aäöüß€漢字 xyz\n"))


def host_chain(prompt: bytes, bb: int):
    keys, prev = [], 0
    for s in range(0, len(prompt) - bb + 1, bb):
        prev = xxhash64(prev.to_bytes(8, "little") + prompt[s:s + bb])
        keys.append(prev)
    return keys


def rand_text(rng, n):
    if rng.random() < 0.3:                                       # non-ASCII UTF-8 text
        return "".join(rng.choice(CHARS, n)).encode("utf-8")[:n]
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def tokenize(rng, text: bytes):
    """Random tokens over the text with the spans tokenizers really report: mostly monotone ends, zero-width tokens,
    tokens across block edges and in the tail; special tokens reported as (0, 0) after later tokens, ends that decrease,
    ends past the end of the text, and runs of tokens that end on one byte."""
    ids, spans, pos = [], [], 0
    while pos < len(text):
        w = int(rng.choice([0, 1, 2, 3, 5, 9, 17]))
        w = min(w, len(text) - pos)
        ids.append(int(rng.integers(0, 1 << 32, dtype=np.uint64)))
        spans.append((pos, pos + w))
        r = rng.random()
        if r < 0.04:
            spans.append((0, 0))                                                # a special token after later tokens
        elif r < 0.07:
            e = max(pos + w - int(rng.integers(1, 24)), 0)                      # an end below the previous one
            spans.append((e, e))
        elif r < 0.08:
            spans.append((pos, len(text) + int(rng.integers(1, 40))))           # past the end of the text
        elif r < 0.12:
            spans.extend([(pos, pos + w)] * int(rng.integers(1, 6)))            # more tokens ending on the same byte
        ids.extend(int(x) for x in rng.integers(0, 1 << 32, len(spans) - len(ids), dtype=np.uint64))
        pos += w if w else (1 if rng.random() < 0.5 else 0)
    return ids, spans


def pack_tokens(toks):
    off = np.zeros(len(toks) + 1, np.int64)
    off[1:] = np.cumsum([len(t[0]) for t in toks])
    ids = np.array([i for t in toks for i in t[0]], np.uint32)
    spans = np.array([s for t in toks for s in t[1]], np.uint64).reshape(-1, 2)
    return ids, spans, off


def host_find(store, prompts):
    toks, ratios = [], []
    for p in prompts:
        t, r = store.find_longest_contained_tokens(p)
        toks.append(np.asarray(t, np.uint32)); ratios.append(r)
    off = np.zeros(len(prompts) + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in toks])
    return (np.concatenate(toks) if toks else np.zeros(0, np.uint32)), off, np.array(ratios, np.float64)


def dev_store(cache_blocks, bb, **kw):
    ix = kvidx.Index(capacity=4096, max_pods=64, **kw)
    ix.text_store_init(cache_blocks, bb)
    return ix


# ---- hash chains -----------------------------------------------------------------------------------------------------
_XP = [np.uint64(x) for x in (0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5)]


def _rotl(x, r):
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def _xround(acc, w):
    return _rotl(acc + w * _XP[1], 31) * _XP[0]


def xxh64_rows(msg):
    """XXH64 (seed 0) of every row of msg (m, M) uint8, in numpy: the spec's stripes of four 8-byte lanes, then the 8-,
    4- and 1-byte tails, then the avalanche."""
    m, M = msg.shape
    P1, P2, P3, P4, P5 = _XP
    w8 = np.ascontiguousarray(msg[:, :M // 8 * 8]).view("<u8")
    k = 0
    if M >= 32:
        v = [np.full(m, P1 + P2), np.full(m, P2), np.zeros(m, np.uint64), np.full(m, np.uint64(0) - P1)]
        while k + 32 <= M:
            for j in range(4):
                v[j] = _xround(v[j], w8[:, k // 8 + j])
            k += 32
        h = _rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)
        for j in range(4):
            h = (h ^ _xround(np.uint64(0), v[j])) * P1 + P4
    else:
        h = np.full(m, P5)
    h = h + np.uint64(M)
    while k + 8 <= M:
        h = _rotl(h ^ _xround(np.uint64(0), w8[:, k // 8]), 27) * P1 + P4
        k += 8
    if k + 4 <= M:
        h = _rotl(h ^ (np.ascontiguousarray(msg[:, k:k + 4]).view("<u4")[:, 0].astype(np.uint64) * P1), 23) * P2 + P3
        k += 4
    while k < M:
        h = _rotl(h ^ (msg[:, k].astype(np.uint64) * P5), 11) * P1
        k += 1
    h ^= h >> np.uint64(33)
    h *= P2
    h ^= h >> np.uint64(29)
    h *= P3
    h ^= h >> np.uint64(32)
    return h


def chains(text, off, bb):
    """Every prompt's chain of bb-byte block keys (numpy, block b of every prompt at once) -> (keys, key offsets)"""
    nb = (off[1:] - off[:-1]) // bb
    koff = np.zeros(len(nb) + 1, np.int64)
    koff[1:] = np.cumsum(nb)
    keys = np.zeros(int(koff[-1]), np.uint64)
    prev = np.zeros(len(nb), np.uint64)
    for b in range(int(nb.max()) if len(nb) else 0):
        act = np.flatnonzero(nb > b)
        at = (off[act] + b * bb)[:, None] + np.arange(bb)
        msg = np.concatenate([prev[act].view(np.uint8).reshape(-1, 8), text[at]], axis=1)
        prev[act] = xxh64_rows(msg)
        keys[koff[act] + b] = prev[act]
    return keys, koff


@pytest.fixture(scope="module")
def hash_ix():
    return dev_store(10, 4)


@pytest.mark.parametrize("bb", list(range(1, 73)) + [255, 256, 257, 1000, 1024, 4096])      # every XXH64 tail layout
@pytest.mark.parametrize("n", [1, 37, 16383, 16384, 20000])      # 4 lanes per prompt below 16384 prompts, 1 lane above
def test_hash_chains_match_the_host_store(bb, n, hash_ix):
    """Every prompt's chain against a numpy XXH64 of the same messages, which in turn matches the host store's
    xxhash64 on the first prompts.  Large batches keep most texts short; a few hundred prompts still run to 3 blocks."""
    np.seterr(over="ignore")
    rng = np.random.default_rng(bb * 7 + n)
    top = 3 * bb + 40
    long_ = rng.random(n) < (1.0 if n < 1000 else min(1.0, 600.0 / top))
    lens = np.where(long_, rng.integers(0, top, n), rng.integers(0, min(top, 2 * bb + 9), n) % max(1, min(top, 80)))
    prompts = [rand_text(rng, int(m)) for m in lens]
    text, off = pack_text(prompts)
    keys, koff = hash_ix.text_hash_keys(text, off, bb)
    want, wkoff = chains(text, off, bb)
    assert np.array_equal(koff, wkoff)
    bad = np.flatnonzero(keys != want)
    assert not len(bad), (bb, n, "first wrong key of prompt", int(np.searchsorted(koff, bad[0], side="right") - 1))
    for i in range(min(n, 40)):
        assert list(want[wkoff[i]:wkoff[i + 1]]) == host_chain(prompts[i], bb), (bb, i, len(prompts[i]))


# ---- call streams against the host store -----------------------------------------------------------------------------
def _stream(rng, cache_blocks, bb, calls, oracle=False, dup_rate=0.3):
    ix = dev_store(cache_blocks, bb)
    hs = PrefixStore(cache_size=cache_blocks, block_size=bb)
    os_ = ko.LRUTokenStore(cache_blocks, bb) if oracle else None
    pool = [rand_text(rng, int(rng.integers(0, 12 * bb))) for _ in range(12)]
    for c in range(calls):
        m = int(rng.integers(1, 9))
        prompts = []
        for _ in range(m):
            r = rng.random()
            if r < dup_rate and prompts:
                prompts.append(prompts[int(rng.integers(0, len(prompts)))])           # duplicate inside the call
            elif r < 0.75:
                base = pool[int(rng.integers(0, len(pool)))]                            # shared prefix
                prompts.append(base[:int(rng.integers(0, len(base) + 1))] + rand_text(rng, int(rng.integers(0, 2 * bb))))
            else:
                prompts.append(rand_text(rng, int(rng.integers(0, 30 * bb))))          # long: more blocks than capacity
        text, off = pack_text(prompts)
        if rng.random() < 0.5:
            toks = []
            for p in prompts:
                t = tokenize(rng, p) if rng.random() < 0.85 else ([], [])               # empty token lists too
                toks.append(t)
            ids, spans, toff = pack_tokens(toks)
            ix.text_store_add(text, off, ids, spans, toff)
            for p, (ti, ts) in zip(prompts, toks):
                hs.add_tokenization(p, ti, ts)
                if os_:
                    os_.add_tokenization(p, ti, ts)
        else:
            got = ix.text_store_find(text, off)
            want = host_find(hs, prompts)
            for g, w in zip(got, want):
                assert np.array_equal(g, w), (c, prompts)
            assert got[2].tobytes() == want[2].tobytes()
            if os_:
                for i, p in enumerate(prompts):
                    t, r = os_.find_longest_contained_tokens(p)
                    assert list(got[0][got[1][i]:got[1][i + 1]]) == list(t) and got[2][i] == r
        assert ix.text_store_len() == len(hs), c
        if os_:
            assert len(os_.cache.d) == len(hs)
    return ix, hs


@pytest.mark.parametrize("cache_blocks", [1, 2, 7, 1000, 500000])
@pytest.mark.parametrize("bb", [4, 16])
def test_random_call_streams_equal_the_host_store(cache_blocks, bb):
    _stream(np.random.default_rng(cache_blocks * 31 + bb), cache_blocks, bb, calls=60)


@pytest.mark.parametrize("cache_blocks", [1, 3, 7, 50])
def test_small_streams_equal_the_oracle(cache_blocks):
    _stream(np.random.default_rng(cache_blocks), cache_blocks, 3, calls=25, oracle=True)


def test_rewrites_until_the_arena_compacts():
    """The same keys rewritten call after call: records pile up in the arena (64 Ki tokens at first) until it compacts."""
    rng = np.random.default_rng(5)
    ix = dev_store(64, 8)
    hs = PrefixStore(cache_size=64, block_size=8)
    prompts = [rand_text(rng, 200) for _ in range(6)]
    text, off = pack_text(prompts)
    for c in range(80):
        toks = [(list(rng.integers(0, 1 << 31, 2 * len(p))), [(min(j // 2, len(p)), min(j // 2, len(p))) for j in range(2 * len(p))]) for p in prompts]
        ids, spans, toff = pack_tokens(toks)
        ix.text_store_add(text, off, ids, spans, toff)
        for p, (ti, ts) in zip(prompts, toks):
            hs.add_tokenization(p, ti, ts)
        if c % 10 == 9:
            got, want = ix.text_store_find(text, off), host_find(hs, prompts)
            assert all(np.array_equal(g, w) for g, w in zip(got, want)), c
    assert ix.text_store_len() == len(hs)


def test_enospc_find_changes_nothing():
    """A find whose tokens do not fit refreshes nothing: later adds evict exactly what the host store, which never saw
    that find, evicts."""
    rng = np.random.default_rng(9)
    ix = dev_store(8, 4)
    hs = PrefixStore(cache_size=8, block_size=4)
    prompts = [rand_text(rng, 16) for _ in range(3)]
    text, off = pack_text(prompts)
    toks = [([int(j) for j in range(16)], [(j, j + 1) for j in range(16)]) for _ in prompts]
    ids, spans, toff = pack_tokens(toks)
    ix.text_store_add(text, off, ids, spans, toff)
    for p, (ti, ts) in zip(prompts, toks):
        hs.add_tokenization(p, ti, ts)
    t1, o1 = pack_text(prompts[1:2])                             # the oldest resident prompt: a real find would keep it
    toff_out = np.zeros(2, np.int64)
    assert ix.text_store_find_into(t1, o1, np.zeros(3, np.uint32), toff_out) == kvidx.ENOSPC
    assert ix.text_store_find_into(t1, o1, None, toff_out) == kvidx.ENOSPC
    assert toff_out.tolist() == [0, 16]
    more = [rand_text(rng, 16)]
    mt, mo = pack_text(more)
    mtoks = [tokenize(rng, p) for p in more]
    ids, spans, toff = pack_tokens(mtoks)
    ix.text_store_add(mt, mo, ids, spans, toff)
    for p, (ti, ts) in zip(more, mtoks):
        hs.add_tokenization(p, ti, ts)
    allp = prompts + more
    at, ao = pack_text(allp)
    got, want = ix.text_store_find(at, ao), host_find(hs, allp)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    assert ix.text_store_len() == len(hs)


def test_csr_slices_with_nonzero_first_offsets():
    """text_off[0] and tok_off[0] may be non-zero (a slice of a larger buffer): add, find and score_text read from there."""
    rng = np.random.default_rng(21)
    ix = kvidx.Index(block_size=4, capacity=4096, max_pods=64)
    ix.text_store_init(1000, 8)
    hs = PrefixStore(cache_size=1000, block_size=8)
    prompts = [rand_text(rng, int(m)) for m in rng.integers(0, 120, 20)]
    toks = [tokenize(rng, p) for p in prompts]
    text, off = pack_text([b"junk" * 9] + prompts)
    ids, spans, toff = pack_tokens([([7, 7, 7], [(0, 1), (1, 2), (2, 36)])] + toks)
    assert off[1] > 0 and toff[1] > 0
    ix.text_store_add(text, off[1:], ids, spans, toff[1:])
    for p, (ti, ts) in zip(prompts, toks):
        hs.add_tokenization(p, ti, ts)
    queries = prompts[::2] + [p + b"tail" for p in prompts[1::3]]
    qt, qo = pack_text([b"x" * 13] + queries)
    got, want = ix.text_store_find(qt, qo[1:]), host_find(hs, queries)
    assert all(np.array_equal(g, w) for g, w in zip(got, want)) and got[2].tobytes() == want[2].tobytes()
    assert ix.text_store_len() == len(hs)
    tok, tof, ratio = want
    keys, _ = ix.hash_keys(tok, np.array([0, len(tok)], np.int64))
    assert ix.add(0, keys ^ np.uint64(3), keys, [(5 << 4)]) == 0
    passing = ratio >= 0.8
    lens = np.where(passing, tof[1:] - tof[:-1], 0)
    soff = np.zeros(len(queries) + 1, np.int64); soff[1:] = np.cumsum(lens)
    exp, exp_has = ix.score_batch(tok[np.repeat(passing, tof[1:] - tof[:-1])], soff)
    sc, has, tz, r = ix.score_text(qt, qo[1:], min_ratio=0.8)
    assert sc.tobytes() == exp.tobytes() and np.array_equal(has, exp_has) and r.tobytes() == ratio.tobytes()
    assert np.array_equal(tz, (~passing).astype(np.uint8)) and has.any()


def test_errors():
    ix = kvidx.Index(capacity=1024, max_pods=8)
    text, off = pack_text([b"abcdefgh"])
    with pytest.raises(kvidx.KvidxError) as e:
        ix.text_store_find(text, off)
    assert e.value.code == kvidx.EINVAL
    for cb, bb in ((0, 4), (4, 0), (-1, 4)):
        with pytest.raises(kvidx.KvidxError) as e:
            ix.text_store_init(cb, bb)
        assert e.value.code == kvidx.EINVAL
    ix.text_store_init(4, 4)
    with pytest.raises(kvidx.KvidxError) as e:
        ix.text_store_init(4, 4)
    assert e.value.code == kvidx.EINVAL
    with pytest.raises(kvidx.KvidxError) as e:
        ix.text_store_find(text, np.array([0, 8, 4], np.int64))
    assert e.value.code == kvidx.EINVAL
    with pytest.raises(kvidx.KvidxError) as e:
        ix.score_text(text, off, min_ratio=-1.0)
    assert e.value.code == kvidx.EINVAL
    assert ix.text_store_find(text, np.zeros(1, np.int64))[1].tolist() == [0]


# ---- Score() from text -----------------------------------------------------------------------------------------------
MODES = {"default": {}, "clock": {"evict_policy": "clock"}, "lru": {"lru_exact": 1}}


def _text_case(n, seed, mode):
    """An index holding blocks of some token prompts, a device and a host store holding the text of some of them, and n
    query texts: stored ones, stored ones extended or cut, and unknown ones (ratios 0 .. 1)."""
    rng = np.random.default_rng(seed)
    P = 64
    ix = kvidx.Index(block_size=BS, capacity=1 << 16, max_pods=P, **MODES[mode])
    ix.text_store_init(500000, 64)
    hs = PrefixStore(500000, 64)
    docs = []
    for d in range(48):
        nt = int(rng.integers(8, 160))
        ids = rng.integers(0, 50000, nt).astype(np.uint32)
        txt = rng.integers(0, 256, 4 * nt, dtype=np.uint8).tobytes() + rand_text(rng, int(rng.integers(0, 9)))
        spans = np.array([(4 * j, 4 * j + 4) for j in range(nt)], np.uint64)
        docs.append((ids, txt, spans))
    for d, (ids, txt, spans) in enumerate(docs[:40]):
        k, _ = ix.hash_keys(ids, np.array([0, len(ids)], np.int64))
        cut = int(rng.integers(0, len(k) + 1))
        if cut:
            assert ix.add(d % 3, k[:cut] ^ np.uint64(0x5a5a), k[:cut], [(int(rng.integers(0, P)) << 4) | int(rng.integers(0, 2))]) == 0
    stored = docs[:32]
    st, so = pack_text([t for _, t, _ in stored])
    sid, ssp, stoff = pack_tokens([(list(i), [tuple(x) for x in s]) for i, _, s in stored])
    ix.text_store_add(st, so, sid, ssp, stoff)
    for ids, txt, spans in stored:
        hs.add_tokenization(txt, ids, spans)
    q = []
    for i in range(n):
        ids, txt, _ = docs[int(rng.integers(0, len(docs)))]
        r = rng.random()
        q.append(txt if r < 0.5 else txt + rand_text(rng, int(rng.integers(1, 200))) if r < 0.8 else txt[:int(rng.integers(0, len(txt) + 1))])
    model = rng.integers(0, 3, n).astype(np.uint32) if rng.random() < 0.5 else None
    filt = None
    if rng.random() < 0.5:
        filt = np.zeros((n, 1), np.uint64)
        filt[:, 0] = rng.integers(0, 1 << 63, n, dtype=np.uint64) & rng.integers(0, 1 << 63, n, dtype=np.uint64)
    return ix, hs, q, model, filt


@pytest.mark.parametrize("n", [1, 32, 2048, 4096, 131072])
@pytest.mark.parametrize("mode", ["default", "clock", "lru"])
def test_score_text_equals_find_then_score_batch(n, mode):
    if mode == "lru" and n == 131072:
        n = 16384                                                  # thread per prompt either way; keeps the run short
    import torch
    ix, hs, q, model, filt = _text_case(n, n + len(mode), mode)
    text, off = pack_text(q)
    tok, toff, ratio = host_find(hs, q)
    for min_ratio in (0.0, 0.8, 1.0):
        passing = ratio >= min_ratio
        lens = np.where(passing, toff[1:] - toff[:-1], 0)
        keep = np.repeat(passing, toff[1:] - toff[:-1])
        soff = np.zeros(n + 1, np.int64); soff[1:] = np.cumsum(lens)
        want, want_has = ix.score_batch(tok[keep], soff, model=model, filter_mask=filt)
        wp, ws, wc, wh = ix.score_batch_sparse(tok[keep], soff, model=model, filter_mask=filt)
        got, has, tokz, r = ix.score_text(text, off, model=model, filter_mask=filt, min_ratio=min_ratio)
        assert got.tobytes() == want.tobytes() and np.array_equal(has, want_has), (n, mode, min_ratio)
        assert np.array_equal(tokz, (~passing).astype(np.uint8)) and r.tobytes() == ratio.tobytes()
        gp, gs, gc, gh, tz2, r2 = ix.score_text_sparse(text, off, model=model, filter_mask=filt, min_ratio=min_ratio)
        assert np.array_equal(gc, wc) and np.array_equal(gh, wh) and np.array_equal(tz2, tokz)
        for i in np.flatnonzero(gc):
            assert gp[i, :gc[i]].tolist() == wp[i, :wc[i]].tolist() and gs[i, :gc[i]].tobytes() == ws[i, :wc[i]].tobytes()
        if min_ratio != 0.8:
            continue
        dev = torch.device("cuda")
        d_text, d_off = torch.from_numpy(text.copy()).to(dev), torch.from_numpy(off).to(dev)
        d_model = torch.from_numpy(model).to(dev) if model is not None else None
        d_filt = torch.from_numpy(filt.view(np.int64)).to(dev) if filt is not None else None
        d_sc = torch.empty((n, ix.max_pods), dtype=torch.float64, device=dev)
        d_has, d_tz = torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.uint8, device=dev)
        d_r = torch.empty(n, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        ix.score_text_dev(d_text.data_ptr() if len(text) else 0, d_off.data_ptr(), n, d_sc.data_ptr(),
                          d_model=d_model.data_ptr() if d_model is not None else 0, d_filter=d_filt.data_ptr() if d_filt is not None else 0,
                          min_ratio=min_ratio, d_has_keys=d_has.data_ptr(), d_tokenize=d_tz.data_ptr(), d_ratio=d_r.data_ptr())
        ix.synchronize()
        assert d_sc.cpu().numpy().tobytes() == want.tobytes() and np.array_equal(d_has.cpu().numpy(), want_has)
        assert np.array_equal(d_tz.cpu().numpy(), tokz) and d_r.cpu().numpy().tobytes() == ratio.tobytes()
        d_p = torch.zeros((n, 10), dtype=torch.int16, device=dev); d_s = torch.zeros((n, 10), dtype=torch.float64, device=dev)
        d_c = torch.zeros(n, dtype=torch.uint8, device=dev)
        ix.score_text_sparse_dev(d_text.data_ptr() if len(text) else 0, d_off.data_ptr(), n, d_p.data_ptr(), d_s.data_ptr(), d_c.data_ptr(),
                                 d_model=d_model.data_ptr() if d_model is not None else 0,
                                 d_filter=d_filt.data_ptr() if d_filt is not None else 0, min_ratio=min_ratio, d_has_keys=d_has.data_ptr())
        ix.synchronize()
        assert np.array_equal(d_c.cpu().numpy(), wc)
        dp, ds = d_p.cpu().numpy().view(np.uint16), d_s.cpu().numpy()
        for i in np.flatnonzero(wc):
            assert dp[i, :wc[i]].tolist() == wp[i, :wc[i]].tolist() and ds[i, :wc[i]].tobytes() == ws[i, :wc[i]].tobytes()


# ---- the service's batch path ----------------------------------------------------------------------------------------
def test_get_pod_scores_batch_equals_per_prompt_get_pod_scores():
    from test_service import MODEL, POD1, FixtureTokenizer, _text
    from kvidx import service
    from kvidx.host import HostIndexer
    names = ["short", "mid", "full", "miss", "fox2", "fox100", "fox500"]
    prompts = [_text(nm) for nm in names]
    stacks = []
    for _ in range(2):
        host = HostIndexer(block_size=4, capacity=1 << 14, max_pods=64, enable_metrics=True)
        stacks.append((host, service.Indexer(host, service.TokenizationPool(tokenizer=FixtureTokenizer()))))
    tk = FixtureTokenizer()
    for host, _ in stacks:
        for nm in ("mid", "fox100"):
            ids = tk.encode(_text(nm)).ids
            tok = np.asarray(ids, np.uint32)
            ix = kvidx.Index.borrow(host.L.kvhost_index(host.h), 4, 64)
            req, _ = ix.hash_keys(tok, np.array([0, len(tok)], np.int64))
            assert host.add(MODEL, req ^ np.uint64(1), req, [(POD1, "gpu")]) == 0
    (h1, per), (h2, batch) = stacks
    for rnd in range(2):                                          # first pass: all tokenized; second: all served from the store
        for pods in ([POD1], [], ["10.9.9.9"]):
            want = [per.get_pod_scores(p, MODEL, pods) for p in prompts]
            got = batch.get_pod_scores_batch(prompts, MODEL, pods)
            assert got == want, (rnd, pods)
    assert batch.tok.encodes == per.tok.encodes
    m1, m2 = h1.metrics(), h2.metrics()                           # one instrumented Lookup per scored prompt on both paths
    for k in ("lookup_requests_total", "lookup_hits_total", "max_pod_hit_count_total"):
        assert m1[k] == m2[k] > 0, k
