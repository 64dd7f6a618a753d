"""GPU (-m gpu): exact-LRU recency when one call touches a key more than once, against the C++ oracle.

An exact-LRU handle (lru_exact=1) must leave every key's recency where the reference's golang-lru leaves it.  Inside one
call the reference touches keys in a fixed order, and when a call touches a key twice the later touch decides:
  kvidx_lookup                   keys in array order (in_memory.go:117-118)
  Score() (tokens, keys, turns)  prompt after prompt; within a prompt every present key in block order, also past the end
                                 of the walk (the oracle's score_batch on one thread; oracle_rows for key lists)
  kvidx_add                      pairs in order: the engine mapping, then the request key (in_memory.go:159-203)
  apply_events                   each pod's events in array order, pods in ascending id (the batch stably sorted by pod)
The tests touch keys shared by prompts, pairs and pods whose threads run in different CTAs, on a handle that holds fewer
keys than its capacity (nothing is evicted inside the call, so exact per call is exact).  Each one then checks
  * the recency section of the handle's image, rank by rank, against the oracle's LRU order, with no stamp repeated,
  * after one capped add of fresh keys on both sides, the whole image again: the same keys were evicted.
Two more cases touch more keys in one prompt or one event than a fixed-width stamp range per prompt or event would hold.
Score() from text must leave exactly the recency score_batch of the tokens it finds leaves.
"""
import struct

import numpy as np
import pytest

from helpers import csr
import kvidx
from oracle.kvoracle_c import COracle
from test_gpu_score_keys import oracle_rows
from test_gpu_score_turn import split_turn
from test_gpu_write_path import _dev_batch
import write_stream as ws

pytestmark = pytest.mark.gpu
P = 16
W = [1.0, 0.8] + [1.0] * 14


def PT(p, t=0):
    return (p << 4) | t


def _pair(cap, B=16, ppk=10, **kw):
    ix = kvidx.Index(block_size=B, capacity=cap, pods_per_key=ppk, max_pods=P, lru_exact=1, **kw)
    co = COracle(block_size=B, size=cap, pod_cache_size=ppk, max_pods=P)
    return ix, co


def _stamps(image):
    """-> (request stamps, engine stamps) of an image with recency"""
    R, E = struct.unpack_from("<QQ", image, 32)
    st = np.frombuffer(image, "<u8", R + E, 64 + 32 * R + 24 * E)
    return st[:R], st[R:]


def _same(got, want, what):
    """bytes equality without a byte-by-byte diff of a multi-megabyte image on failure"""
    if got != want:
        a, b = np.frombuffer(got, np.uint8), np.frombuffer(want, np.uint8)
        n = min(len(a), len(b))
        diff = np.nonzero(a[:n] != b[:n])[0]
        raise AssertionError("%s: %d / %d bytes, first difference at byte %s" % (what, len(a), len(b), diff[:1]))


def check_recency(ix, co, sort_entries=False):
    """the handle's recency ranks equal the oracle's LRU positions and no stamp repeats within a section.  sort_entries:
    compare entry lists as sets (their order inside a record depends on how pods' queues interleave).  -> the image"""
    img = ix.snapshot()
    for name, sec in zip(("request", "engine"), _stamps(img)):
        assert len(np.unique(sec)) == len(sec), "%s stamps repeat: %d of %d distinct" % (name, len(np.unique(sec)), len(sec))
    got, want = ws.recency_ranks(img), co.snapshot(recency=True)
    if sort_entries:
        got, want = ws.sorted_entries(got), ws.sorted_entries(want)
    _same(got, want, "recency ranks")
    return img


def capped_add(ix, co, rng, k, sort_entries=False):
    """k fresh keys on both sides: each map drops its oldest keys down to the capacity -- the same ones on both sides"""
    assert ix.evictions() == (0, 0)                  # the touching calls ran below the capacity
    new = rng.integers(1, 1 << 63, k, dtype=np.uint64)
    for t in (ix, co):
        assert t.add(0, new ^ np.uint64(0x3C3C), new, [PT(13)]) == 0
    assert ix.evictions()[0] > 0 and ix.evictions()[1] > 0
    check_recency(ix, co, sort_entries)


# ---- Score(): prompts that share a prefix ------------------------------------------------------------------------------
def _score_setup(B, rng, n_docs=48):
    """Documents on two 6-block system prompts.  The second one's first block is never stored (its prompts miss at block 0
    and every later block is still present); documents d % 8 == 3 miss their block 8 (a miss in the middle).  Stored on
    both sides document by document.  -> (ix, co, docs)"""
    sys_a, sys_b = (rng.integers(0, 50000, 6 * B) for _ in range(2))
    docs = [np.concatenate([sys_b if d % 8 == 7 else sys_a, rng.integers(0, 50000, B * int(rng.integers(4, 16)))]).astype(np.uint32)
            for d in range(n_docs)]
    co0 = COracle(block_size=B)
    seen, adds = set(), []
    for d, doc in enumerate(docs):
        ks, _ = co0.hash_keys(doc, [0, len(doc)])
        skip = {0} if d % 8 == 7 else {8} if d % 8 == 3 else set()
        new = [int(k) for j, k in enumerate(ks) if j not in skip and int(k) not in seen]
        seen.update(new)
        adds.append((np.array(new, np.uint64), [PT(d % 7), PT(9, 1)]))
    ix, co = _pair(len(seen), B)
    for ks, pts in adds:
        for t in (ix, co):
            assert t.add(0, ks ^ np.uint64(0x55), ks, pts) == 0
    return ix, co, docs


def _prompts(B, rng, docs, n):
    """n prompts of at least 4 blocks of a document, some running up to 2 blocks past it, most with a partial last block"""
    out = []
    for _ in range(n):
        doc = docs[int(rng.integers(0, len(docs)))]
        nb = len(doc) // B
        k = int(rng.integers(4, nb + 3))
        out.append(np.concatenate([doc[:min(k, nb) * B], rng.integers(0, 50000, max(k - nb, 0) * B + int(rng.integers(0, B)))]))
    return csr(out)


def _dev(*arrays):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _score(ix, co, mode, tok, off, B, rng):
    """One Score() call of the given form on ix; -> the oracle's dense rows for it (same touches, same order)"""
    import torch
    n = len(off) - 1
    want = co.score_batch(tok, off, n_threads=1)[0] if not mode.startswith("keys") else None
    if mode in ("dense", "chunked"):
        got = ix.score_batch(tok, off)[0]
    elif mode == "sparse":
        ix.score_batch_sparse(tok, off)
        got = None
    elif mode in ("dev", "sparse_dev"):
        d_tok, d_off = _dev(tok.view(np.int32), off)
        d_s = torch.zeros((n, P), dtype=torch.float64, device="cuda")
        if mode == "dev":
            ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), n, d_s.data_ptr())
        else:
            d_p, d_c = torch.zeros((n, 10), dtype=torch.int16, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda")
            ix.score_batch_sparse_dev(d_tok.data_ptr(), d_off.data_ptr(), n, d_p.data_ptr(), d_s.data_ptr(), d_c.data_ptr())
        ix.synchronize()
        got = d_s.cpu().numpy() if mode == "dev" else None
    elif mode.startswith("keys"):
        # held-key lists: the prompts' keys, with keys repeated inside a prompt (later copies refresh again) and absent keys
        keys, koff = co.hash_keys(tok, off)
        absent = rng.integers(1, 1 << 63, n, dtype=np.uint64)
        lists = []
        for i in range(n):
            ks = keys[koff[i]:koff[i + 1]]
            if i % 5 == 1:
                ks = np.concatenate([ks[:3], absent[i:i + 1], ks[3:], ks[::2]])
            elif i % 5 == 2:
                ks = np.concatenate([ks, ks[:4]])
            lists.append(ks)
        koff = np.zeros(n + 1, np.int64)
        koff[1:] = np.cumsum([len(k) for k in lists])
        keys = np.concatenate(lists)
        want = oracle_rows(co, W, P, keys, koff)
        if mode == "keys":
            got = ix.score_keys(keys, koff)[0]
        elif mode == "keys_sparse":
            ix.score_keys_sparse(keys, koff)
            got = None
        else:
            d_k, d_o = _dev(keys.view(np.int64), koff)
            d_s = torch.zeros((n, P), dtype=torch.float64, device="cuda")
            ix.score_keys_dev(d_k.data_ptr(), d_o.data_ptr(), n, d_s.data_ptr())
            ix.synchronize()
            got = d_s.cpu().numpy()
    else:
        # a turn: the first 0..5 blocks held as keys (the system prompt's keys are shared by every prompt), the rest tokens
        keys, koff = co.hash_keys(tok, off)
        held, hoff, nt, toff, _, _ = split_turn(tok, off, keys, koff, np.arange(n) % 6, bs=B)
        if mode == "turn":
            got = ix.score_turn(held, hoff, nt, toff)[0]
        else:
            d_h, d_ho, d_t, d_to = _dev(held.view(np.int64), hoff, nt.view(np.int32), toff)
            d_s = torch.zeros((n, P), dtype=torch.float64, device="cuda")
            ix.score_turn_dev(d_h.data_ptr(), d_ho.data_ptr(), d_t.data_ptr(), d_to.data_ptr(), n, d_s.data_ptr())
            ix.synchronize()
            got = d_s.cpu().numpy()
    if got is not None:
        assert got.tobytes() == want.tobytes(), np.argwhere(got != want)[:5]


SCORE_CASES = [(16, m) for m in ("dense", "sparse", "chunked", "dev", "sparse_dev", "keys", "keys_sparse", "keys_dev", "turn", "turn_dev")] + \
              [(B, m) for B in (4, 64) for m in ("dense", "chunked", "dev", "keys", "turn")]


@pytest.mark.parametrize("B,mode", SCORE_CASES)
def test_score_shared_prefixes(B, mode, monkeypatch):
    """4096 prompts (32 CTAs of the thread-per-prompt kernel) on one system prompt: its keys are touched by every prompt,
    each document's by the prompts on it.  "chunked": the host call split into chunks of 64 Ki tokens."""
    if mode == "chunked":
        monkeypatch.setenv("KVIDX_HOST_CHUNK_TOKENS", str(1 << 16))
    rng = np.random.default_rng(100 + B)
    ix, co, docs = _score_setup(B, rng)
    tok, off = _prompts(B, rng, docs, 4096)
    if mode == "chunked":
        assert len(tok) > 2 * (1 << 16)                      # three chunks or more
    _score(ix, co, mode, tok, off, B, rng)
    check_recency(ix, co)
    capped_add(ix, co, rng, ix.stats()["request_keys"] // 3)


# ---- Lookup and Add ----------------------------------------------------------------------------------------------------
def test_lookup_repeated_keys():
    """2048 keys: 64 keys 8 times each at scattered positions (so in every CTA), 1200 other present keys, absent keys"""
    rng = np.random.default_rng(7)
    allk = rng.integers(1, 1 << 63, 1500, dtype=np.uint64)
    ix, co = _pair(len(allk))
    for i in range(0, len(allk), 100):
        for t in (ix, co):
            assert t.add(0, allk[i:i + 100] ^ np.uint64(0x55), allk[i:i + 100], [PT(i // 100 % 16), PT(3, 1)]) == 0
    seq = np.concatenate([np.repeat(allk[:64], 8), allk[64:1264], rng.integers(1, 1 << 63, 2048 - 512 - 1200, dtype=np.uint64)])
    seq = seq[rng.permutation(len(seq))]
    r1, r2 = ix.lookup(0, seq), co.lookup(0, seq)
    assert r1[0] == r2[0] == 0 and np.array_equal(r1[2], r2[2])
    assert all(np.array_equal(r1[1][i, :c], r2[1][i, :c]) for i, c in enumerate(r2[2]))
    check_recency(ix, co)
    capped_add(ix, co, rng, 500)


@pytest.mark.parametrize("engine_repeats", [False, True])
def test_add_repeated_keys(engine_repeats):
    """1000 pairs in one add: 100 request keys 4 times each at scattered positions, half of them stored before; with
    engine_repeats, 150 engine keys also repeat, mapped to different request keys (the last pair's mapping wins)"""
    rng = np.random.default_rng(11 + engine_repeats)
    old = rng.integers(1, 1 << 63, 400, dtype=np.uint64)
    rep = np.concatenate([old[:50], rng.integers(1, 1 << 63, 50, dtype=np.uint64)])
    req = np.concatenate([np.repeat(rep, 4), old[50:250], rng.integers(1, 1 << 63, 400, dtype=np.uint64)])
    req = req[rng.permutation(len(req))]
    eng = rng.integers(1, 1 << 63, len(req), dtype=np.uint64)
    if engine_repeats:
        pool = rng.integers(1, 1 << 63, 150, dtype=np.uint64)
        at = rng.random(len(req)) < 0.4
        eng[at] = pool[rng.integers(0, len(pool), int(at.sum()))]
    dry = COracle(size=10 ** 6, pod_cache_size=10, max_pods=P)        # sizes the capacity: nothing evicted before the last add
    assert dry.add(0, old ^ np.uint64(0x55), old, [PT(1)]) == 0 and dry.add(0, eng, req, [PT(2), PT(5, 1)]) == 0
    R, E = dry.len_request(), dry.len_engine()
    ix, co = _pair(max(R, E))
    for t in (ix, co):
        for i in range(0, len(old), 100):
            assert t.add(0, old[i:i + 100] ^ np.uint64(0x55), old[i:i + 100], [PT(1)]) == 0
        assert t.add(0, eng, req, [PT(2), PT(5, 1)]) == 0
    check_recency(ix, co)
    capped_add(ix, co, rng, abs(R - E) + 200)                    # past the capacity in both maps


# ---- event batches: pods that store the same documents ------------------------------------------------------------------
def _event_docs(rng, B):
    docs = []
    for d in range(24):
        if d % 3 == 2:                                         # a prefix of an earlier document: the same engine hashes
            base = docs[int(rng.integers(0, d))]
            k = int(rng.integers(1, len(base) + 1))
            blocks = np.concatenate([base.blocks[:k], rng.integers(0, 50000, (int(rng.integers(1, 12)), B), dtype=np.uint64).astype(np.uint32)])
        else:
            blocks = rng.integers(0, 50000, (int(rng.integers(4, 30)), B), dtype=np.uint64).astype(np.uint32)
        docs.append(ws.Doc(None, blocks))
    return docs


def _shared_batch(rng, docs, B, n):
    """Pods 0..5 store slices of the documents pods 0 and 1 hold whole, each from its resident parent (so every pod's
    chain resolves the same parent mappings, whatever the schedule), plus dropped stores with parents, stores without
    hashes, and removals of shared blocks by pods 2..5 (pods 0 and 1 keep every key alive)."""
    out = []
    while len(out) < n:
        p, doc = int(rng.integers(0, 6)), docs[int(rng.integers(0, len(docs)))]
        b0 = int(rng.integers(0, len(doc)))
        b1 = int(rng.integers(b0 + 1, len(doc) + 1))
        par = int(doc.eh[b0 - 1]) if b0 > 0 else None
        r = rng.random()
        toks = doc.blocks[b0:b1].reshape(-1)
        if r < 0.5:
            out.append(ws.Ev(ws.STORED, p, 0, 0, par, doc.eh[b0:b1], toks, "store"))
        elif r < 0.62:
            cut = toks[:len(toks) - B] if rng.random() < 0.5 else np.concatenate([toks, toks[:B]])
            out.append(ws.Ev(ws.STORED, p, 0, 0, int(doc.eh[max(b0 - 1, 0)]), doc.eh[b0:b1], cut, "drop"))
        elif r < 0.7:
            out.append(ws.Ev(ws.STORED, p, 0, 0, int(doc.eh[max(b0 - 1, 0)]), [], toks, "zero_hashes"))
        elif p >= 2:
            hs = doc.eh[b0:b1]
            out.append(ws.Ev(ws.REMOVED, p, 0, 0, None, np.concatenate([hs, hs[:2]]), [], "remove"))
    return out


def _sorted_by_pod(batch):
    return sorted(batch, key=lambda e: e.pod)                  # stable: each pod's events keep their order


@pytest.mark.parametrize("phase1", [0, 1])
@pytest.mark.parametrize("api", ["host", "dev"])
def test_events_shared_documents(phase1, api, monkeypatch):
    import torch
    monkeypatch.setenv("KVIDX_WRITE_PHASE1", str(phase1))
    B = 4
    rng = np.random.default_rng(31 + phase1 + 2 * (api == "dev"))
    docs = _event_docs(rng, B)
    warm = [ws.Ev(ws.STORED, p, 0, 0, None, d.eh, d.blocks.reshape(-1), "store") for d in docs for p in (0, 1)]
    batches = [_shared_batch(rng, docs, B, 400) for _ in range(2)]
    dry = COracle(block_size=B, size=10 ** 6, pod_cache_size=10, max_pods=P)
    for b in [warm] + batches:
        assert dry.apply_events(*ws.pack(_sorted_by_pod(b)))[0] == 0
    # the _dev room check counts every hash of a batch as a new key: a table with room for that
    ix, co = _pair(max(dry.len_request(), dry.len_engine()), B, table_slots=1 << 14)
    keep = [torch.zeros(1, dtype=torch.int64, device="cuda:0")]
    for b in [warm] + batches:
        if api == "host":
            assert ix.apply_events(*ws.pack(b))[0] == 0
        else:
            _dev_batch(ix, b, keep)
            ix.synchronize()
        assert co.apply_events(*ws.pack(_sorted_by_pod(b)))[0] == 0
        check_recency(ix, co, sort_entries=True)
    capped_add(ix, co, rng, ix.stats()["request_keys"] // 3, sort_entries=True)


# ---- stamp ranges: more touches in one prompt or one event than a fixed-width range per prompt or event holds ----------
def _restores(img, B, cap):
    ix2 = kvidx.Index(block_size=B, capacity=cap, pods_per_key=10, max_pods=P, lru_exact=1)
    ix2.restore(img)
    _same(ix2.snapshot(), img, "snapshot of the restored handle")


def test_score_keys_prompt_past_2_20_keys():
    """one prompt of 2^20 + 2 present keys, then a one-key prompt, then a lookup call"""
    n = (1 << 20) + 2
    rng = np.random.default_rng(5)
    allk = rng.integers(1, 1 << 63, n + 2, dtype=np.uint64)
    cap = n + 8
    ix, co = _pair(cap)
    for t in (ix, co):
        assert t.add(0, allk ^ np.uint64(0x55), allk, [PT(2)]) == 0
    keys, koff = np.concatenate([allk[:n], allk[n:n + 1]]), np.array([0, n, n + 1], np.int64)
    got = ix.score_keys(keys, koff)[0]
    assert got.tobytes() == oracle_rows(co, W, P, keys, koff).tobytes()
    q = np.array([allk[n + 1], allk[3]], np.uint64)
    r1, r2 = ix.lookup(0, q), co.lookup(0, q)
    assert np.array_equal(r1[2], r2[2])
    img = check_recency(ix, co)
    _restores(img, 16, cap)


def test_event_past_2_19_blocks():
    """a BlockStored of 2^19 + 1 blocks at block size 1, then another event of the same pod in the same batch"""
    B, nb = 1, (1 << 19) + 1
    rng = np.random.default_rng(6)
    big = ws.Ev(ws.STORED, 3, 0, 0, None, rng.integers(1, 1 << 63, nb, dtype=np.uint64),
                rng.integers(0, 50000, nb, dtype=np.uint64).astype(np.uint32), "store")
    small = ws.Ev(ws.STORED, 3, 1, 0, None, rng.integers(1, 1 << 63, 3, dtype=np.uint64),
                  rng.integers(0, 50000, 3, dtype=np.uint64).astype(np.uint32), "store")
    cap = 1 << 20
    ix, co = _pair(cap, B)
    ev, hs, tk = ws.pack([big, small])
    for t in (ix, co):
        assert t.apply_events(ev, hs, tk) == (0, 0)
    img = check_recency(ix, co)
    _restores(img, B, cap)


# ---- Score() from text: the same touches as score_batch of the tokens it finds ------------------------------------------
def test_score_text_leaves_score_batch_recency():
    """Twin exact-LRU handles on the shared-prefix documents, the prompts' text in a device prefix store on one of them:
    Score() from text there, score_batch of the same token CSR (the host store's find, gated at 0.8) on the twin and on
    the oracle.  The images, which carry recency, are byte-equal right after the call and again after a capped add."""
    from kvidx import pack_text
    from kvidx.host import PrefixStore
    from test_gpu_text_store_scale import _text_of, _want
    B = 16
    twins = [_score_setup(B, np.random.default_rng(140)) for _ in range(2)]
    (a, co, docs), (b, _, _) = twins
    rng = np.random.default_rng(141)
    tok, off = _prompts(B, rng, docs, 4096)
    a.text_store_init(500000, 64)
    hs = PrefixStore(500000, 64)
    texts = [_text_of(d) for d in docs]
    dtext, doff = pack_text(texts)
    spans = np.concatenate([np.stack([np.arange(len(d)) * 4, np.arange(len(d)) * 4 + 4], axis=1) for d in docs]).astype(np.uint64)
    a.text_store_add(dtext, doff, np.concatenate(docs), spans, np.concatenate([[0], np.cumsum([len(d) for d in docs])]))
    for t, d in zip(texts, docs):
        hs.add_tokenization(t, d, np.stack([np.arange(len(d)) * 4, np.arange(len(d)) * 4 + 4], axis=1))
    q = [_text_of(tok[off[i]:off[i + 1]]) for i in range(len(off) - 1)]
    tq, soff, passing, _ = _want(hs, q, 0.8)
    assert passing.any() and not passing.all()
    got = a.score_text(*pack_text(q), min_ratio=0.8)[0]
    want_b = b.score_batch(tq, soff)[0]
    want_o = co.score_batch(tq, soff, n_threads=1)[0]
    assert got.tobytes() == want_b.tobytes() == want_o.tobytes()
    check_recency(a, co)
    _same(a.snapshot(), b.snapshot(), "images after score_text and score_batch")
    assert a.evictions() == (0, 0)
    new = rng.integers(1, 1 << 63, a.stats()["request_keys"] // 3, dtype=np.uint64)
    for t in (a, b, co):
        assert t.add(0, new ^ np.uint64(0x3C3C), new, [PT(13)]) == 0
    assert a.evictions()[0] > 0
    check_recency(a, co)
    _same(a.snapshot(), b.snapshot(), "images after the capped add")
