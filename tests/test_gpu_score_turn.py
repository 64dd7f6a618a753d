"""GPU (-m gpu): Score() for a conversation turn (kvidx_score_turn*): the request keys a caller holds, then the new turn's
tokens, with the new turn's keys handed back.  Checked byte for byte against the two identities of the contract (a prompt
split at any block scores as score_batch on its tokens and returns the rest of hash_keys; no new tokens scores as
score_keys) at every dispatch size, and against the oracle composition Score(K, Lookup(K)) with K = held ++
TokensToKVBlockKeys(parent = last held key, new tokens) for held lists no token prompt produces."""
import threading

import numpy as np
import pytest

from helpers import _index_pair, csr, filter_mask
from test_gpu_score_keys import (W16, _fill, _filters, _key_case, _key_index, _key_prompts, _load_case, _prefix_docs,
                                 _ragged_prompts, key_csr, oracle_rows, same_sparse)
import kvidx
from kvidx import synth
from oracle.kvoracle_c import COracle

pytestmark = pytest.mark.gpu
BS = 16
SPLITS = (0, 1, 31, 32, 33, 64, 1 << 30)          # held blocks per prompt (clipped to the prompt's full blocks)


def PT(p, t=0):
    return (p << 4) | t


def _gather(starts, lens):
    """indices of the runs [starts[i], starts[i] + lens[i]) back to back"""
    o = np.zeros(len(lens) + 1, np.int64)
    o[1:] = np.cumsum(lens)
    return np.repeat(starts - o[:-1], lens) + np.arange(o[-1]), o


def split_turn(tok, off, keys, koff, m, bs=BS):
    """Prompt i held as its first m[i] block keys plus the tokens from block m[i] on.  -> (held keys, their offsets, new
    tokens, their offsets, the new keys the contract returns, their offsets)."""
    nblk = (off[1:] - off[:-1]) // bs
    m = np.minimum(np.asarray(m, np.int64), nblk)
    hi, hoff = _gather(koff[:-1], m)
    ti, toff = _gather(off[:-1] + bs * m, off[1:] - off[:-1] - bs * m)
    ni, noff = _gather(koff[:-1] + m, nblk - m)
    return keys[hi], hoff, tok[ti], toff, keys[ni], noff


def check_turn(ix, held, hoff, tok, toff, want_rows, want_has, want_keys, want_koff, **kw):
    """every output of score_turn / score_turn_sparse, with the new keys given and not, equals the expected bytes"""
    s, h, nk, no = ix.score_turn(held, hoff, tok, toff, **kw)
    assert s.tobytes() == want_rows.tobytes(), np.argwhere(s != want_rows)[:5]
    assert np.array_equal(h, want_has)
    assert nk.tobytes() == np.asarray(want_keys, np.uint64).tobytes() and np.array_equal(no, want_koff)
    s2, h2, nk2, no2 = ix.score_turn(held, hoff, tok, toff, want_keys=False, **kw)
    assert nk2 is None and s2.tobytes() == want_rows.tobytes() and np.array_equal(h2, want_has) and np.array_equal(no2, want_koff)
    sp = ix.score_turn_sparse(held, hoff, tok, toff, **kw)
    assert sp[4].tobytes() == nk.tobytes()
    spn = ix.score_turn_sparse(held, hoff, tok, toff, want_keys=False, **kw)
    assert same_sparse(sp[:4], spn[:4])
    return sp[:4]


# ---- the two identities, at every dispatch size --------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 32, 2048, 4096, 65536, 131072])
def test_identities(n):
    rng = np.random.default_rng(n + 1)
    P = 64
    ix = kvidx.Index(capacity=1 << 16, max_pods=P)
    docs = _prefix_docs(rng, max_blocks=80)
    _fill(ix, COracle(size=1 << 16, max_pods=P), docs, rng, P)
    tok, off = csr(_ragged_prompts(rng, docs, n))
    keys, koff = ix.hash_keys(tok, off)
    want, wh = ix.score_batch(tok, off)
    want_sp = ix.score_batch_sparse(tok, off)
    m = np.array([SPLITS[(i * 7 + n) % len(SPLITS)] for i in range(n)], np.int64)
    held, hoff, nt, toff, nk, nkoff = split_turn(tok, off, keys, koff, m)
    sp = check_turn(ix, held, hoff, nt, toff, want, wh, nk, nkoff)
    assert same_sparse(sp, want_sp)
    if n >= 32:
        assert (want.max(axis=1) > 1).any() and (want.max(axis=1) < 0).any()
    # every prompt split at the same block
    for mm in (0, 33, 1 << 30):
        held, hoff, nt, toff, nk, nkoff = split_turn(tok, off, keys, koff, np.full(n, mm))
        s, h, k2, _ = ix.score_turn(held, hoff, nt, toff)
        assert s.tobytes() == want.tobytes() and np.array_equal(h, wh) and k2.tobytes() == nk.tobytes()
    # no new tokens: score_keys
    sk, hk = ix.score_keys(keys, koff)
    s, h, k3, o3 = ix.score_turn(keys, koff, np.zeros(0, np.uint32), np.zeros(n + 1, np.int64))
    assert s.tobytes() == sk.tobytes() and np.array_equal(h, hk) and len(k3) == 0 and not o3.any()
    # filters and models
    fm = np.zeros((n, 1), np.uint64)
    fm[::3, 0] = rng.integers(0, 1 << 63, len(fm[::3]), dtype=np.uint64)
    held, hoff, nt, toff, nk, nkoff = split_turn(tok, off, keys, koff, m)
    model = (np.arange(n) % 2).astype(np.uint32)
    for kw in ({"filter_mask": fm}, {"model": model}):
        w, wh2 = ix.score_batch(tok, off, **kw)
        check_turn(ix, held, hoff, nt, toff, w, wh2, nk, nkoff, **kw)
    # non-zero first offsets: the arrays hold other elements in front of the batch's
    s, _, k4, _ = ix.score_turn(np.concatenate([rng.integers(0, 1 << 63, 5, dtype=np.uint64), held]), hoff + 5,
                                np.concatenate([rng.integers(0, 50000, 3, dtype=np.uint32), nt]), toff + 3)
    assert s.tobytes() == want.tobytes() and k4.tobytes() == nk.tobytes()


# ---- arbitrary held lists against the oracle ----------------------------------------------------------------------------
def _turn_case(rng, ix, co, case, n=400):
    """held key lists of the score_keys cases, each followed by new tokens; where the held list is a stored chain, the new
    turn's keys (chained from its last key) are stored too, on the chain's pods, so that walks run on into the tokens and end
    inside them on the chunk edges.  -> (held, hoff, tok, toff, model, K, Koff, new keys, their offsets)."""
    lists, models = _key_prompts(rng, case, n)
    chains = case[0]
    stored = {k: pts for _, _, k, pts in chains}
    toks = []
    for i, ks in enumerate(lists):
        L = BS * [0, 1, 31, 32, 33, 40, 64, 70][i % 8] + (i % 3) * 5          # ragged tails
        toks.append(rng.integers(0, 50000, L, dtype=np.uint32))
    held, hoff = key_csr(lists)
    tok, toff = csr(toks)
    parent = np.array([int(ks[-1]) if len(ks) else 0 for ks in lists], np.uint64)
    pv = np.array([len(ks) > 0 for ks in lists], np.uint8)
    nk, nko = co.hash_keys(tok, toff, parent=parent, parent_valid=pv)
    for i, ks in enumerate(lists):
        if len(ks) and int(ks[-1]) in stored and i % 4:
            pts = stored[int(ks[-1])]
            new = nk[nko[i]:nko[i + 1]]
            cut = len(new) - [0, 1, 8, 33][i % 4]                              # the chain's pods stop at some block
            for j in range(max(cut, 0)):
                for t in (ix, co):
                    assert t.add(int(models[i]), [int(new[j]) ^ 0xD0D0], [int(new[j])], pts[: 1 + (j + i) % len(pts)]) == 0
    K, Koff = key_csr([np.concatenate([ks, nk[nko[i]:nko[i + 1]]]) for i, ks in enumerate(lists)])
    return held, hoff, tok, toff, models, K, Koff, nk, nko


@pytest.mark.parametrize("P", [257, 4096])
def test_arbitrary_held_lists_vs_oracle(P):
    rng = np.random.default_rng(P + 7)
    case = _key_case(rng, P)
    ix, co = _key_index(P)
    _load_case(ix, co, case)
    held, hoff, tok, toff, models, K, Koff, nk, nko = _turn_case(rng, ix, co, case)
    weights = list(W16) + [1.0] * (16 - len(W16))
    has = (np.diff(Koff) > 0).astype(np.uint8)
    for kw in ({"model": models}, {"model": models, "filter_mask": _filters(rng, len(hoff) - 1, P)}, {"model0": 0}):
        want = oracle_rows(co, weights, P, K, Koff, kw.get("model"), 0, kw.get("filter_mask"))
        sp = check_turn(ix, held, hoff, tok, toff, want, has, nk, nko, **kw)
        pods, sc, cnt, _ = sp
        for i in range(len(hoff) - 1):
            assert {int(pods[i, j]): float(sc[i, j]) for j in range(cnt[i])} == {int(q): float(want[i, q]) for q in np.nonzero(want[i] >= 0)[0]}, i
        if "filter_mask" not in kw and "model" in kw:
            # walks that run on past the held keys into the tokens (their rows differ from the held keys' alone), and
            # walks that end inside the held keys (a miss among them) while new keys are still returned
            sk, _ = ix.score_keys(held, hoff, **kw)
            assert (want != sk).any(axis=1).sum() >= 10
            assert ((np.arange(len(hoff) - 1) % 12 == 2) & (np.diff(nko) > 0) & (np.diff(hoff) > 0)).any()


def test_forced_v1_equals_fused(monkeypatch):
    P = 257
    handles = []
    for kernel in (None, "v1"):                             # the same index twice: the fused kernel and the composed path
        if kernel:
            monkeypatch.setenv("KVIDX_SCORE_KERNEL", kernel)
        rng = np.random.default_rng(5)
        case = _key_case(rng, P)
        ix, co = _key_index(P)
        _load_case(ix, co, case)
        handles.append((ix, co, _turn_case(rng, ix, co, case, 300)))
    (ix, co, (held, hoff, tok, toff, models, K, Koff, nk, nko)), (iv, _, _) = handles
    fm = _filters(rng, len(hoff) - 1, P)
    for kw in ({"model": models}, {"model": models, "filter_mask": fm}):
        a = ix.score_turn(held, hoff, tok, toff, **kw)
        b = iv.score_turn(held, hoff, tok, toff, **kw)
        assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1]) and a[2].tobytes() == b[2].tobytes() == nk.tobytes()
        assert same_sparse(ix.score_turn_sparse(held, hoff, tok, toff, **kw)[:4], iv.score_turn_sparse(held, hoff, tok, toff, **kw)[:4])
        want = oracle_rows(co, list(W16) + [1.0] * 8, P, K, Koff, models, 0, kw.get("filter_mask"))
        assert b[0].tobytes() == want.tobytes()


# ---- chain edges ----------------------------------------------------------------------------------------------------------
def test_chain_edges():
    """a last held key below 2^32 (the plain-chain branch), CBOR width edges in the token values, fewer than 16 new tokens,
    partial tails, token pointers that are not 16-byte aligned"""
    rng = np.random.default_rng(3)
    P = 16
    ix, co = _index_pair(capacity=1 << 14, max_pods=P)
    edge = np.array([0, 23, 24, 255, 256, 65535, 65536, 2 ** 32 - 1], np.uint32)
    prompts = []
    for i in range(300):
        L = [BS * 70, BS * 33 + 7, BS * 2, BS - 1, 5, BS * 40 + 15][i % 6]
        prompts.append(edge[rng.integers(0, len(edge), L)] if i % 2 else rng.integers(0, 1 << 32, L, dtype=np.uint64).astype(np.uint32))
    tok, off = csr(prompts)
    small = np.array([1, 2, 0xFFFFFFFF, 1 << 20], np.uint64)              # parents below 2^32
    lists = [small[i % 4: i % 4 + 1] if i % 3 else small[:0] for i in range(len(prompts))]
    held, hoff = key_csr(lists)
    parent = np.array([int(l[-1]) if len(l) else 0 for l in lists], np.uint64)
    pv = np.array([len(l) > 0 for l in lists], np.uint8)
    nk, nko = co.hash_keys(tok, off, parent=parent, parent_valid=pv)
    K, Koff = key_csr([np.concatenate([lists[i], nk[nko[i]:nko[i + 1]]]) for i in range(len(prompts))])
    for k in K[::2]:
        for t in (ix, co):
            assert t.add(0, [int(k) ^ 0x1234], [int(k)], [PT(int(k) % 5), PT(7, 1)]) == 0
    want = oracle_rows(co, [1.0, 0.8] + [1.0] * 14, P, K, Koff)
    has = (np.diff(Koff) > 0).astype(np.uint8)
    check_turn(ix, held, hoff, tok, off, want, has, nk, nko)
    # tokens at an odd 4-byte offset: the LDG fallback
    buf = np.zeros(len(tok) + 1, np.uint32)
    buf[1:] = tok
    s, h, k2, _ = ix.score_turn(held, hoff, buf, off + 1)
    assert s.tobytes() == want.tobytes() and k2.tobytes() == nk.tobytes()
    # the e2e suite's small held key (ChunkHash: 1) followed by a turn
    s, h, k3, _ = ix.score_turn(np.array([1], np.uint64), np.array([0, 1], np.int64), tok[:BS * 3], np.array([0, BS * 3], np.int64))
    assert k3.tobytes() == co.hash_keys(tok[:BS * 3], [0, BS * 3], parent=[1])[0].tobytes()


# ---- composed path ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [4, 64, 256])
def test_other_block_sizes(B):
    rng = np.random.default_rng(B)
    P = 32
    ix, co = _index_pair(capacity=1 << 15, max_pods=P, block_size=B)
    docs = [rng.integers(0, 50000, B * int(rng.integers(2, 80)), dtype=np.uint32) for _ in range(20)]
    for d in range(4, 20):
        docs[d][:B * 2] = docs[d % 4][:B * 2]
    _fill(ix, co, docs, rng, P)
    prompts = [docs[i % 20][:int(rng.integers(0, len(docs[i % 20]) + 1))] if i % 3 else docs[i % 20] for i in range(500)]
    tok, off = csr(prompts)
    keys, koff = ix.hash_keys(tok, off)
    want, wh = ix.score_batch(tok, off)
    assert want.tobytes() == co.score_batch(tok, off, n_threads=4)[0].tobytes()
    m = np.array([SPLITS[i % len(SPLITS)] for i in range(500)], np.int64)
    held, hoff, nt, toff, nk, nko = split_turn(tok, off, keys, koff, m, bs=B)
    check_turn(ix, held, hoff, nt, toff, want, wh, nk, nko)


def test_exact_lru_stamps_as_score_batch():
    """an exact-LRU handle scored by a turn call and an equal one scored by score_batch on the full tokens evict the same
    keys afterwards: the turn stamped every present key in the same order"""
    rng = np.random.default_rng(21)
    CAP, P = 300, 16
    a = kvidx.Index(capacity=CAP, pods_per_key=3, max_pods=P, lru_exact=1)
    b = kvidx.Index(capacity=CAP, pods_per_key=3, max_pods=P, lru_exact=1)
    docs = [rng.integers(0, 50000, BS * 20, dtype=np.uint32) for _ in range(15)]
    allk = []
    for d, doc in enumerate(docs):
        k, _ = a.hash_keys(doc, [0, len(doc)])
        allk.append(k)
        for ix in (a, b):
            assert ix.add(0, k ^ np.uint64(0x55), k, [PT(d % 7), PT(9, 1)]) == 0
    prompts = [docs[i][:BS * (5 + i)] for i in range(12)]
    prompts[3] = np.concatenate([rng.integers(0, 50000, BS, dtype=np.uint32), docs[3][BS:]])   # a miss at block 0
    tok, off = csr(prompts)
    keys, koff = a.hash_keys(tok, off)
    held, hoff, nt, toff, nk, nko = split_turn(tok, off, keys, koff, np.arange(12) % 4)
    sa, ha, ka, _ = a.score_turn(held, hoff, nt, toff)
    sb, hb = b.score_batch(tok, off)
    assert sa.tobytes() == sb.tobytes() and ka.tobytes() == nk.tobytes()
    new = rng.integers(1, 1 << 63, 100, dtype=np.uint64)
    for ix in (a, b):
        assert ix.add(0, new ^ np.uint64(0x55), new, [PT(1)]) == 0
    flat = np.concatenate(allk)
    assert np.array_equal(a.lookup(0, flat)[2], b.lookup(0, flat)[2])


# ---- CLOCK -------------------------------------------------------------------------------------------------------------
def test_clock_marks_what_the_token_path_marks():
    """as test_gpu_score_keys' test of that name: a CLOCK handle scored by turn calls keeps, after a capped write, exactly
    the referenced set of an equal handle scored by score_batch on the full tokens"""
    from clock_oracle import referenced_keys
    from test_gpu_clock import MODELS, Fill, _new_keys, clock_index, oracle_of, resident, score
    for n in (300, 4096):
        rng = np.random.default_rng(n)
        a, b = clock_index(1024), clock_index(1024)
        fa, fb = Fill(a, np.random.default_rng(9)), Fill(b, np.random.default_rng(9))
        ka, ea = _new_keys(rng, 1)
        for ix in (a, b):
            assert ix.add(0, ea, ka, [PT(2)]) == 0
        img = resident(a)[2]
        assert img == resident(b)[2]
        prompts, filters = fa.queries(rng, n)
        R = {(MODELS.index(k.model), k.chunk_hash) for k in referenced_keys(oracle_of(img), prompts, filters, block_size=BS)}
        score(a, prompts, filters)
        tok, off = csr([t for t, _ in prompts])
        model = np.array([0 if m == "m0" else 1 for _, m in prompts], np.uint32)
        fm = np.zeros((len(prompts), b.filter_words), np.uint64)
        for i, f in enumerate(filters):
            if f:
                fm[i] = filter_mask([int(p[1:]) for p in f], b.filter_words)
        keys, koff = b.hash_keys(tok, off)
        held, hoff, nt, toff, _, _ = split_turn(tok, off, keys, koff, np.array([SPLITS[i % 7] for i in range(len(prompts))]))
        b.score_turn(held, hoff, nt, toff, model=model, filter_mask=fm, want_keys=False)
        kn, en = _new_keys(rng, fa.C - len(R))
        for ix in (a, b):
            assert ix.add(0, en, kn, [PT(3)]) == 0
        want = R | {(0, x) for x in kn}
        assert resident(a)[0] == want == resident(b)[0] and a.evictions() == b.evictions()


# ---- sharded handles ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("peer_pair", [0, 1])
@pytest.mark.parametrize("layout", [("same-gpu", 2), ("same-gpu", 8), ("multi-gpu", 2)])
def test_sharded_equals_unsharded(layout, peer_pair, monkeypatch):
    from test_gpu_shard_ops import _shards
    monkeypatch.setenv("KVIDX_PEER_PAIR", str(peer_pair))
    rng = np.random.default_rng(peer_pair + 3)
    P = 64
    sh = _shards(layout[1], layout[0], hash_seed="", pods_per_key=10, max_pods=P, tier_weights=W16)
    ix, co = _key_index(P)
    case = _key_case(rng, P)
    _load_case(ix, co, case)
    held, hoff, tok, toff, models, K, Koff, nk, nko = _turn_case(rng, ix, co, case, 300)
    chains, foreign, absent, om = case
    for d, j, k, pts in chains:
        assert sh[0].add(0, [k ^ 0xE0E0], [k], pts) == 0
    for i, k in enumerate(foreign):
        assert sh[-1].add(om, [int(k) ^ 0xF0F0], [int(k)], [PT(3, i % 16), PT(4, 2)]) == 0
        assert sh[-1].add(0 if i % 2 else om, [int(k) ^ 0xF1F1], [int(k) ^ 1], [PT(7, 1)]) == 0
    # the turn keys _turn_case stored in ix: copy them to the shards from the unsharded handle's Lookup
    for mdl in sorted(set(models.tolist())):
        rc, pt, cnt = ix.lookup(mdl, nk)
        for j in np.nonzero(cnt)[0]:
            assert sh[j % len(sh)].add(mdl, [int(nk[j]) ^ 0xD0D0], [int(nk[j])], pt[j, :cnt[j]].tolist()) == 0
    fm = _filters(rng, len(hoff) - 1, P)
    want, wh, wk, _ = ix.score_turn(held, hoff, tok, toff, filter_mask=fm)
    for s in sh:
        got, gh, gk, _ = s.score_turn(held, hoff, tok, toff, filter_mask=fm)
        assert got.tobytes() == want.tobytes() and np.array_equal(gh, wh) and gk.tobytes() == wk.tobytes()


# ---- stream order, readers beside writers -------------------------------------------------------------------------------
def _dev(a, dev):
    import torch
    a = np.ascontiguousarray(a)
    v = {8: np.int64, 4: np.int32, 2: np.int16, 1: np.uint8}[a.dtype.itemsize]
    return torch.from_numpy(a.view(v).copy()).to(dev)


def test_dev_after_apply_events_dev_sees_the_batch():
    import torch
    wl = synth.Workload(4, 1024, 1 << 13, 32)
    ix = kvidx.Index(capacity=1 << 14, max_pods=32)
    ev, hs, tk = wl.fill_events(0, wl.D)
    order = np.argsort(ev["podtier"] >> 4, kind="stable")
    evs = ev[order]
    pods = (evs["podtier"] >> 4).astype(np.int64)
    qoff = np.concatenate([[0], np.nonzero(np.diff(pods))[0] + 1, [len(evs)]]).astype(np.int64)
    dev = torch.device("cuda", 0)
    d_ev, d_q, d_hs, d_tk = _dev(evs.view(np.uint8).reshape(-1), dev), _dev(qoff, dev), _dev(hs, dev), _dev(tk, dev)
    n = 300
    toks, doc, m = wl.queries(0, n)
    off = np.arange(0, (n + 1) * wl.T, wl.T, dtype=np.int64)
    co = COracle(size=1 << 14, max_pods=32)
    keys, koff = co.hash_keys(toks.reshape(-1), off)
    held, hoff, nt, toff, nk, nko = split_turn(toks.reshape(-1), off, keys, koff, np.array([SPLITS[i % 7] for i in range(n)]))
    d_pods = torch.zeros((n, 10), dtype=torch.int16, device=dev)
    d_sc = torch.zeros((n, 10), dtype=torch.float64, device=dev)
    d_cnt = torch.zeros(n, dtype=torch.uint8, device=dev)
    d_has = torch.zeros(n, dtype=torch.uint8, device=dev)
    d_nk = torch.zeros(max(len(nk), 1), dtype=torch.int64, device=dev)
    ins = [_dev(x, dev) for x in (held, hoff, nt, toff, nko)]
    torch.cuda.synchronize()
    ix.apply_events_dev(d_ev.data_ptr(), d_q.data_ptr(), len(qoff) - 1, len(evs), d_hs.data_ptr(), len(hs), d_tk.data_ptr())
    ix.score_turn_sparse_dev(ins[0].data_ptr(), ins[1].data_ptr(), ins[2].data_ptr(), ins[3].data_ptr(), n, d_pods.data_ptr(),
                             d_sc.data_ptr(), d_cnt.data_ptr(), d_has_keys=d_has.data_ptr(), d_new_key_off=ins[4].data_ptr(),
                             d_new_keys=d_nk.data_ptr())
    ix.synchronize()
    exp = wl.expected_scores(doc, m)
    cnt, pods_h, sc_h = d_cnt.cpu().numpy(), d_pods.cpu().numpy().view(np.uint16), d_sc.cpu().numpy()
    assert (d_has.cpu().numpy() == 1).all()
    assert d_nk.cpu().numpy().view(np.uint64)[:len(nk)].tobytes() == nk.tobytes()
    for i in range(n):
        got = {int(pods_h[i, j]): float(sc_h[i, j]) for j in range(cnt[i])}
        assert got == {int(p): float(exp[i, p]) for p in np.nonzero(exp[i] >= 0)[0]}, i


def test_reader_beside_writer_on_disjoint_documents():
    wl = synth.Workload(5, 1024, 1 << 14, 32)
    ix = kvidx.Index(capacity=1 << 16, max_pods=32)
    ev, hs, tk = wl.fill_events(0, wl.D)
    assert ix.apply_events(ev, hs, tk) == (0, 0)
    toks, doc, m = wl.queries(0, 3000)
    off = np.arange(0, (len(toks) + 1) * wl.T, wl.T, dtype=np.int64)
    keys, koff = ix.hash_keys(toks.reshape(-1), off)
    held, hoff, nt, toff, nk, nko = split_turn(toks.reshape(-1), off, keys, koff, np.array([SPLITS[i % 7] for i in range(3000)]))
    want = wl.expected_scores(doc, m)
    churn = []
    for s_i in range(12):
        e, h, t = wl.fill_events(wl.D + 8 * s_i, wl.D + 8 * (s_i + 1))
        r = e.copy(); r["op"] = 1; r["has_parent"] = 0; r["n_tokens"] = 0
        churn.append((e, r, h, t))
    errs = []

    def writer():
        try:
            for e, r, h, t in churn:
                assert ix.apply_events(e, h, t) == (0, 0)
                assert ix.apply_events(r, h, t)[0] == 0
        except Exception as ex:                             # noqa: BLE001
            errs.append(ex)

    th = threading.Thread(target=writer)
    th.start()
    for _ in range(6):
        s1, _, k1, _ = ix.score_turn(held, hoff, nt, toff)
        if not np.array_equal(s1, want) or k1.tobytes() != nk.tobytes():
            errs.append(AssertionError("scores changed while events were applied"))
    th.join()
    assert not errs, errs[:1]


# ---- host buffers against the device-resident call -------------------------------------------------------------------------
def _dev_turn(ix, held, hoff, tok, toff, sparse, want_keys):
    import torch
    dev = torch.device("cuda", 0)
    n = len(hoff) - 1
    nko = np.zeros(n + 1, np.int64)
    nko[1:] = np.cumsum(np.diff(toff) // ix.block_size)
    ins = [_dev(x, dev) for x in (held if len(held) else np.zeros(1, np.uint64), hoff, tok if len(tok) else np.zeros(1, np.uint32), toff, nko)]
    d_nk = torch.zeros(max(int(nko[-1]), 1), dtype=torch.int64, device=dev)
    d_has = torch.zeros(n, dtype=torch.uint8, device=dev)
    kw = dict(d_has_keys=d_has.data_ptr(), d_new_key_off=ins[4].data_ptr() if want_keys else 0, d_new_keys=d_nk.data_ptr() if want_keys else 0)
    if sparse:
        d_p = torch.zeros((n, 10), dtype=torch.int16, device=dev)
        d_s = torch.zeros((n, 10), dtype=torch.float64, device=dev)
        d_c = torch.zeros(n, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()
        ix.score_turn_sparse_dev(ins[0].data_ptr(), ins[1].data_ptr(), ins[2].data_ptr(), ins[3].data_ptr(), n, d_p.data_ptr(), d_s.data_ptr(),
                                 d_c.data_ptr(), **kw)
        ix.synchronize()
        rows = (d_p.cpu().numpy().view(np.uint16), d_s.cpu().numpy(), d_c.cpu().numpy(), d_has.cpu().numpy())
    else:
        d_s = torch.zeros((n, ix.max_pods), dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        ix.score_turn_dev(ins[0].data_ptr(), ins[1].data_ptr(), ins[2].data_ptr(), ins[3].data_ptr(), n, d_s.data_ptr(), **kw)
        ix.synchronize()
        rows = (d_s.cpu().numpy(), d_has.cpu().numpy())
    return rows, d_nk.cpu().numpy().view(np.uint64)[:int(nko[-1])], nko


@pytest.mark.parametrize("chunk", [None, 65536])
def test_host_buffers_vs_dev(chunk, monkeypatch):
    if chunk:
        monkeypatch.setenv("KVIDX_HOST_CHUNK_TOKENS", str(chunk))
    rng = np.random.default_rng(31)
    P = 64
    ix = kvidx.Index(capacity=1 << 16, max_pods=P)
    docs = _prefix_docs(rng, max_blocks=40)
    _fill(ix, None, docs, rng, P)
    tok, off = csr(_ragged_prompts(rng, docs, 12000))
    keys, koff = ix.hash_keys(tok, off)
    held, hoff, nt, toff, nk, nko = split_turn(tok, off, keys, koff, np.array([SPLITS[i % 7] for i in range(12000)]))
    if chunk:                                               # keys and tokens share the chunk budget: several chunks
        assert len(held) * 8 + len(nt) * 4 > 3 * chunk * 4
    pk = kvidx.pinned_array(held.shape, np.uint64); pk[:] = held
    pt = kvidx.pinned_array(nt.shape, np.uint32); pt[:] = nt
    for n in (1, 7, 32, 33, 2048, 12000):                   # zero-copy sizes, just above, and the pipeline
        ho, to = hoff[:n + 1], toff[:n + 1]
        for sparse in (False, True):
            for want_keys in (True, False):
                rows, dk, dko = _dev_turn(ix, held[:ho[-1]], ho, nt[:to[-1]], to, sparse, want_keys)
                for kk, tt in ((held, nt), (pk, pt), (held, pt), (pk, nt)):     # pageable, pinned, mixed
                    if sparse:
                        r = ix.score_turn_sparse(kk, ho, tt, to, want_keys=want_keys)
                        assert same_sparse(r[:4], rows)
                        k, ko = r[4], r[5]
                    else:
                        s, h, k, ko = ix.score_turn(kk, ho, tt, to, want_keys=want_keys)
                        assert s.tobytes() == rows[0].tobytes() and np.array_equal(h, rows[1])
                    assert np.array_equal(ko, dko)
                    if want_keys:
                        assert k.tobytes() == dk.tobytes() == nk[:nko[n]].tobytes()
    # pinned outputs: dense rows written in place
    out = kvidx.pinned_array((12000, P), np.float64)
    want, _ = ix.score_batch(tok, off)
    ix.score_turn(kvidx._native._Raw(pk.ctypes.data), hoff, kvidx._native._Raw(pt.ctypes.data), toff, out=out)
    assert out.tobytes() == want.tobytes()


def test_pinned_new_keys_buffer():
    """a pinned new-keys buffer is written in place, by the zero-copy kernel and by the pipeline"""
    import ctypes as C
    rng = np.random.default_rng(8)
    P = 32
    ix = kvidx.Index(capacity=1 << 16, max_pods=P)
    docs = _prefix_docs(rng, max_blocks=40)
    _fill(ix, None, docs, rng, P)
    tok, off = csr(_ragged_prompts(rng, docs, 3000))
    keys, koff = ix.hash_keys(tok, off)
    held, hoff, nt, toff, nk, nko = split_turn(tok, off, keys, koff, np.array([SPLITS[i % 7] for i in range(3000)]))
    for n in (5, 3000):
        pnk = kvidx.pinned_array((max(int(nko[n]), 1),), np.uint64)
        no = np.zeros(n + 1, np.int64)
        sc = np.zeros((n, P)); has = np.zeros(n, np.uint8)
        u64, i64, u32 = C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.POINTER(C.c_uint32)
        ho, to = np.ascontiguousarray(hoff[:n + 1]), np.ascontiguousarray(toff[:n + 1])
        rc = ix.L.kvidx_score_turn(ix.h, held.ctypes.data_as(u64), ho.ctypes.data_as(i64), nt.ctypes.data_as(u32), to.ctypes.data_as(i64), n,
                                   None, 0, None, sc.ctypes.data_as(C.POINTER(C.c_double)), has.ctypes.data_as(C.POINTER(C.c_uint8)),
                                   pnk.ctypes.data_as(u64), no.ctypes.data_as(i64))
        assert rc == 0 and np.array_equal(no, nko[:n + 1]) and pnk[:nko[n]].tobytes() == nk[:nko[n]].tobytes()
        assert sc.tobytes() == ix.score_batch(tok, off[:n + 1])[0].tobytes()


# ---- errors ---------------------------------------------------------------------------------------------------------------
def test_errors_and_empty_batch():
    import ctypes as C
    ix = kvidx.Index(capacity=1024, max_pods=8)
    L, u64, i64, u32 = ix.L, C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.POINTER(C.c_uint32)
    f64, u8, u16 = C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_uint16)
    keys = np.arange(1, 9, dtype=np.uint64)
    tok = np.arange(64, dtype=np.uint32)
    sc = np.full((4, 8), 7.0)
    has = np.full(4, 9, np.uint8)
    nk = np.zeros(8, np.uint64)
    nko = np.full(5, 99, np.int64)
    pods, ssc, cnt = np.zeros((4, 10), np.uint16), np.zeros((4, 10)), np.zeros(4, np.uint8)
    P = lambda a, t: None if a is None else a.ctypes.data_as(t)                    # noqa: E731

    def dense(k, ko, t, to, n, nkeys=nk, nkoff=nko):
        return L.kvidx_score_turn(ix.h, P(k, u64), P(ko, i64), P(t, u32), P(to, i64), n, None, 0, None, sc.ctypes.data_as(f64),
                                  has.ctypes.data_as(u8), P(nkeys, u64), P(nkoff, i64))

    def sparse(k, ko, t, to, n, nkeys=nk, nkoff=nko):
        return L.kvidx_score_turn_sparse(ix.h, P(k, u64), P(ko, i64), P(t, u32), P(to, i64), n, None, 0, None, pods.ctypes.data_as(u16),
                                         ssc.ctypes.data_as(f64), cnt.ctypes.data_as(u8), has.ctypes.data_as(u8), P(nkeys, u64), P(nkoff, i64))
    ko = np.array([0, 2, 4], np.int64)
    to = np.array([0, 32, 48], np.int64)
    for fn in (dense, sparse):
        assert fn(keys, ko, tok, to, -1) == kvidx.EINVAL
        assert fn(keys, None, tok, to, 2) == kvidx.EINVAL
        assert fn(keys, ko, tok, None, 2) == kvidx.EINVAL
        assert fn(keys, np.array([0, 3, 2], np.int64), tok, to, 2) == kvidx.EINVAL and "not monotone" in ix.last_error()
        assert fn(keys, ko, tok, np.array([0, 40, 30], np.int64), 2) == kvidx.EINVAL and "not monotone" in ix.last_error()
        assert fn(None, ko, tok, to, 2) == kvidx.EINVAL
        assert fn(keys, ko, None, to, 2) == kvidx.EINVAL
        assert fn(keys, ko, tok, to, 2, nkoff=None) == kvidx.EINVAL                  # new keys without their offsets
        assert fn(None, np.array([3, 3, 3], np.int64), None, np.array([5, 5, 5], np.int64), 2) == 0   # nothing at all: NULL is fine
        assert fn(keys, ko, tok, to, 2, nkeys=None) == 0 and np.array_equal(nko[:3], [0, 2, 3])      # offsets without keys
    args = [None] * 4
    assert L.kvidx_score_turn_dev(ix.h, *args, 1, None, 0, None, None, None, None, None) == kvidx.EINVAL
    assert L.kvidx_score_turn_dev(ix.h, None, 1, None, 1, -1, None, 0, None, 1, None, None, None) == kvidx.EINVAL
    assert L.kvidx_score_turn_dev(ix.h, None, 1, None, 1, 1, None, 0, None, 1, None, None, 1) == kvidx.EINVAL   # keys without offsets
    assert L.kvidx_score_turn_dev(ix.h, None, 1, None, 1, 0, None, 0, None, 1, None, None, None) == 0          # n == 0
    sc[:] = 7.0; has[:] = 9; nko[:] = 99
    assert dense(keys, ko, tok, to, 0) == 0 and (sc == 7.0).all() and (has == 9).all() and (nko == 99).all()   # n == 0: nothing written
    assert dense(None, np.array([3, 3, 3], np.int64), tok, np.array([0, 15, 15], np.int64), 2) == 0      # < 16 new tokens, no key
    assert (sc[:2] == -1.0).all() and (has[:2] == 0).all() and np.array_equal(nko[:3], [0, 0, 0])


# ---- host mirror ----------------------------------------------------------------------------------------------------------
def test_host_mirror_get_pod_scores_turn():
    from kvidx.host import HostIndexer
    rng = np.random.default_rng(41)
    h = HostIndexer(capacity=1 << 14, max_pods=16, enable_metrics=True)
    docs = [rng.integers(0, 50000, BS * int(rng.integers(2, 12))).tolist() for _ in range(10)]
    keys = []
    hx = kvidx.Index(capacity=1024)                       # the mirror's defaults: block 16, seed ""
    for d, doc in enumerate(docs):
        k, _ = hx.hash_keys(np.array(doc, np.uint32), np.array([0, len(doc)], np.int64))
        keys.append(k)
        ents = [("pod-%d" % (d % 4), "gpu"), ("pod-%d" % ((d + 1) % 4), "cpu")]
        assert h.add("m", k ^ np.uint64(0x99), k, ents) == 0
    for d, doc in enumerate(docs):
        for L in (len(doc), BS * 2 + 3, BS - 1):
            t = doc[:L]
            for m in sorted({0, min(1, L // BS), L // BS}):
                held, new = keys[d][:m], t[BS * m:]
                a = h.get_pod_scores(t, "m")
                b, nk = h.get_pod_scores_turn(held, new, "m")
                assert a == b and nk.tobytes() == keys[d][m:L // BS].tobytes(), d
                for pods in (["pod-%d" % (d % 4)], ["pod-9"], ["pod-1", "pod-2"]):
                    b2, nk2 = h.get_pod_scores_turn(held, new, "m", pods)
                    assert h.get_pod_scores(t, "m", pods) == b2 and nk2.tobytes() == nk.tobytes()
    r, nk = h.get_pod_scores_turn([], [1, 2, 3], "m")
    assert r is None and len(nk) == 0
    m0 = h.metrics()
    _, nk = h.get_pod_scores_turn(keys[3][:2], docs[3][2 * BS:], "m")
    m1 = h.metrics()
    assert m1["lookup_requests_total"] == m0["lookup_requests_total"] + 1
    assert m1["lookup_hits_total"] - m0["lookup_hits_total"] == len(keys[3])
    h.get_pod_scores_turn([], [], "m")                                         # no keys: no Lookup
    assert h.metrics()["lookup_requests_total"] == m1["lookup_requests_total"]
