"""GPU (-m gpu): Score() from request keys (kvidx_score_keys*, GetPodScores steps 3-4).  Checked bit-exact against the
token path on the same prompts (every dispatch size), and against the oracle composition
LongestPrefixScorer.Score(keys, Index.Lookup(keys, pods)) for key lists no token prompt produces: misses anywhere,
repeated keys, other models' keys, wide filters, all sixteen tiers, walks ending on every chunk edge."""
import threading

import numpy as np
import pytest

from helpers import _index_pair, csr, filter_mask, keys_homed_at
import kvidx
from kvidx import synth
from oracle.kvoracle_c import COracle

pytestmark = pytest.mark.gpu
BS = 16


def PT(p, t=0):
    return (p << 4) | t


def key_csr(lists):
    off = np.zeros(len(lists) + 1, np.int64)
    off[1:] = np.cumsum([len(k) for k in lists])
    keys = np.concatenate([np.asarray(k, np.uint64) for k in lists]) if off[-1] else np.zeros(0, np.uint64)
    return keys, off


def oracle_rows(co, weights, P, keys, off, model=None, model0=0, fm=None):
    """LongestPrefixScorer.Score(keys, Lookup(keys, pods)) per prompt (kvblock_scorer.go:108-151) over the C++ oracle's
    Lookup, as an in-order Python fold: the same f64 additions in the same order."""
    n = len(off) - 1
    rows = np.full((n, P), -1.0)
    for i in range(n):
        ks = keys[off[i]:off[i + 1]]
        if not len(ks):
            continue
        m = int(model[i]) if model is not None else model0
        frow = None if fm is None or not fm[i].any() else fm[i]
        rc, pt, cnt = co.lookup(m, ks, frow)
        assert rc == 0
        ents = [pt[j, :cnt[j]].tolist() for j in range(len(ks))]

        def mx(es, p):
            w = 0.0
            for e in es:
                if e >> 4 == p and weights[e & 15] > w:
                    w = weights[e & 15]
            return w
        score = {p: mx(ents[0], p) for p in {e >> 4 for e in ents[0]}}
        active = set(score)
        for es in ents[1:]:
            if not active:
                break
            active &= {e >> 4 for e in es}
            for p in active:
                score[p] += mx(es, p)
        for p, s in score.items():
            if p < P:
                rows[i, p] = s
    return rows


def same_sparse(a, b):
    """equal sparse results: counts, has_keys, and the first cnt[i] (pod, score) pairs of each row (the rest of a row is
    not written)"""
    (pa, sa, ca, ha), (pb, sb, cb, hb) = a, b
    live = np.arange(pa.shape[1])[None, :] < ca[:, None]
    return (np.array_equal(ca, cb) and np.array_equal(ha, hb) and np.array_equal(pa[live], pb[live])
            and sa[live].tobytes() == sb[live].tobytes())


def check_keys_vs_tokens(ix, tok, off, keys, koff, model=None, model0=0, fm=None):
    """score_keys on the prompts' keys == score_batch on their tokens: dense, sparse and has_keys"""
    s1, h1 = ix.score_batch(tok, off, model=model, model0=model0, filter_mask=fm)
    s2, h2 = ix.score_keys(keys, koff, model=model, model0=model0, filter_mask=fm)
    assert np.array_equal(h1, h2)
    assert s1.tobytes() == s2.tobytes(), np.argwhere(s1 != s2)[:5]
    assert same_sparse(ix.score_batch_sparse(tok, off, model=model, model0=model0, filter_mask=fm),
                       ix.score_keys_sparse(keys, koff, model=model, model0=model0, filter_mask=fm))
    return s1


def check_vs_oracle(ix, co, weights, keys, koff, model=None, model0=0, fm=None):
    want = oracle_rows(co, weights, ix.max_pods, keys, koff, model, model0, fm)
    got, has = ix.score_keys(keys, koff, model=model, model0=model0, filter_mask=fm)
    assert np.array_equal(has, (np.diff(koff) > 0).astype(np.uint8))
    assert got.tobytes() == want.tobytes(), np.argwhere(got != want)[:5]
    pods, sc, cnt, has2 = ix.score_keys_sparse(keys, koff, model=model, model0=model0, filter_mask=fm)
    assert np.array_equal(has, has2)
    for i in range(len(koff) - 1):
        assert {int(pods[i, j]): float(sc[i, j]) for j in range(cnt[i])} == {int(q): float(want[i, q]) for q in np.nonzero(want[i] >= 0)[0]}, i
    return want


# ---- the same bits as the token path ----------------------------------------------------------------------------------
def _prefix_docs(rng, n_docs=64, max_blocks=12):
    docs = [rng.integers(0, 50000, BS * int(rng.integers(2, max_blocks + 1)), dtype=np.uint32) for _ in range(n_docs)]
    for d in range(8, n_docs):
        share = min(int(rng.integers(1, 4)), len(docs[d]) // BS, len(docs[d % 8]) // BS)
        docs[d][:BS * share] = docs[d % 8][:BS * share]
    return docs


def _fill(ix, co, docs, rng, P):
    for d, doc in enumerate(docs):
        k = (co or ix).hash_keys(doc, [0, len(doc)])[0]
        for g in range(1 + d % 3):
            depth = len(k) - int(rng.integers(0, len(k) // 2 + 1))
            pts = [PT(int(p), int(rng.integers(0, 2))) for p in rng.choice(P, size=int(rng.integers(1, 4)), replace=False)]
            ek = k[:depth] ^ np.uint64(0x77 + g)
            assert ix.add(0, ek, k[:depth], pts) == 0
            if co is not None:
                assert co.add(0, ek, k[:depth], pts) == 0


def _ragged_prompts(rng, docs, n):
    prompts = []
    for i in range(n):
        doc = docs[int(rng.integers(0, len(docs)))]
        kind = i % 5
        if kind == 0:
            prompts.append(doc)
        elif kind == 1:
            prompts.append(doc[:int(rng.integers(0, len(doc) + 1))])                 # ragged, sometimes < 1 block
        elif kind == 2:
            prompts.append(np.concatenate([doc[:BS * int(rng.integers(0, len(doc) // BS + 1))], rng.integers(0, 50000, 37, dtype=np.uint32)]))
        elif kind == 3:
            prompts.append(rng.integers(0, 50000, int(rng.integers(0, 3 * BS)), dtype=np.uint32))
        else:
            prompts.append(doc[:BS * int(rng.integers(1, len(doc) // BS + 1))])
    return prompts


@pytest.mark.parametrize("n", [1, 32, 2048, 4096, 65536, 131072])
def test_same_bits_as_score_batch(n):
    rng = np.random.default_rng(n)
    P = 64
    ix = kvidx.Index(capacity=1 << 16, max_pods=P)
    docs = _prefix_docs(rng)
    _fill(ix, COracle(size=1 << 16, max_pods=P), docs, rng, P)
    prompts = _ragged_prompts(rng, docs, n)
    tok, off = csr(prompts)
    keys, koff = ix.hash_keys(tok, off)
    s = check_keys_vs_tokens(ix, tok, off, keys, koff)
    if n >= 32:
        assert (s.max(axis=1) > 1).any() and (s.max(axis=1) < 0).any()
    fm = np.zeros((n, 1), np.uint64)
    fm[::3, 0] = rng.integers(0, 1 << 63, len(fm[::3]), dtype=np.uint64)
    check_keys_vs_tokens(ix, tok, off, keys, koff, fm=fm)
    if n <= 2048:
        model = (np.arange(n) % 2).astype(np.uint32)
        check_keys_vs_tokens(ix, tok, off, keys, koff, model=model)
    # a non-zero key_off[0]: the keys array holds other keys in front of the batch's
    pad = 5
    s2, h2 = ix.score_keys(np.concatenate([rng.integers(0, 1 << 63, pad, dtype=np.uint64), keys]), koff + pad)
    assert s2.tobytes() == s.tobytes()


# ---- arbitrary key lists against the oracle composition ---------------------------------------------------------------
W16 = (1.0, 0.8, 0.3, 0.0, -0.5, 1 / 3, 5e-324, 2.5)             # ids 8..15: unknown, 1.0


def _key_case(rng, P, n_chain=70, other_model=9):
    """A chain of 70 stored keys per document (8 documents) whose entries change along the chain, and keys stored only
    under another model.  Returns (chains, foreign keys, absent keys)."""
    chains, P_ = [], min(P, 4096)
    pods_all = sorted({0, 1, 5, 63, 64, 127, 200, 256, P_ - 1} & set(range(P_)))
    for d in range(8):
        ks = rng.integers(1, 1 << 63, n_chain, dtype=np.uint64)
        base = [int(x) for x in rng.choice(pods_all, size=min(4, len(pods_all)), replace=False)]
        for j, k in enumerate(ks):
            # the block-0 pods drop out one by one at blocks 31, 32, 33, 64 (walks end on the chunk edges)
            keep = [p for q, p in enumerate(base) if j < (31, 32, 33, 64)[q % 4] + d % 2]
            pts = [PT(p, (j * 3 + q + d) % 16) for q, p in enumerate(keep)] + [PT(pods_all[(j + d) % len(pods_all)], j % 16)]
            chains.append((d, j, int(k), list(dict.fromkeys(pts))[:10]))
    foreign = rng.integers(1, 1 << 63, 40, dtype=np.uint64)
    absent = rng.integers(1, 1 << 63, 40, dtype=np.uint64)
    return chains, foreign, absent, other_model


def _key_index(P, tier_weights=W16, **kw):
    ix, co = _index_pair(capacity=1 << 15, max_pods=P, tier_weights=tier_weights, **kw)
    return ix, co


def _load_case(ix, co, case):
    chains, foreign, absent, om = case
    for d, j, k, pts in chains:
        for t in (ix, co):
            assert t.add(0, [k ^ 0xE0E0], [k], pts) == 0
    for i, k in enumerate(foreign):
        for t in (ix, co):
            assert t.add(om, [int(k) ^ 0xF0F0], [int(k)], [PT(3, i % 16), PT(4, 2)]) == 0
            assert t.add(0 if i % 2 else om, [int(k) ^ 0xF1F1], [int(k) ^ 1], [PT(7, 1)]) == 0


def _key_prompts(rng, case, n=400):
    chains, foreign, absent, om = case
    by_doc = {}
    for d, j, k, _ in chains:
        by_doc.setdefault(d, []).append(k)
    lists, models = [], []
    for i in range(n):
        d = int(rng.integers(0, 8))
        ch = np.array(by_doc[d], np.uint64)
        kind = i % 12
        L = [31, 32, 33, 64, 65, 70][i % 6]
        ks = ch[:L].copy()
        m = 0
        if kind == 1:                                   # a miss at block 0
            ks[0] = absent[i % len(absent)]
        elif kind == 2:                                 # a miss mid-prompt
            ks[int(rng.integers(1, L - 1))] = absent[i % len(absent)]
        elif kind == 3:                                 # a miss at the last key
            ks[-1] = absent[i % len(absent)]
        elif kind == 4:                                 # repeated keys
            ks = np.concatenate([ks[:5], ks[:5], ks[3:9], np.repeat(ks[9:10], 30)])
        elif kind == 5:                                 # another model's keys inside the chain
            ks[int(rng.integers(0, L))] = foreign[i % len(foreign)]
        elif kind == 6:                                 # the foreign keys as a prompt under their model
            ks = foreign[: int(rng.integers(1, 40))]
            m = om
        elif kind == 7:                                 # the same prompt under the other model (everything absent)
            m = om
        elif kind == 8:
            ks = ks[:0]                                 # no key
        elif kind == 9:                                 # keys of two documents back to back
            ks = np.concatenate([ks[:10], np.array(by_doc[(d + 1) % 8][:20], np.uint64)])
        lists.append(ks)
        models.append(m)
    return lists, np.array(models, np.uint32)


def _filters(rng, n, P):
    FW = (P + 63) // 64
    fm = np.zeros((n, FW), np.uint64)
    pods = sorted({0, 1, 5, 63, 64, 127, 200, 256, P - 1} & set(range(P)))
    for i in range(n):
        kind = i % 4
        if kind == 1:                                   # exclusive: one pod
            fm[i] = filter_mask([pods[i % len(pods)]], FW)
        elif kind == 2:                                 # wide: several words
            fm[i] = filter_mask(rng.choice(pods, size=int(rng.integers(1, len(pods) + 1)), replace=False).tolist(), FW)
        elif kind == 3 and P % 64:                      # bits only at or above max_pods: selects nothing
            fm[i, -1] = ~np.uint64(0) << np.uint64(P % 64)
    return fm


@pytest.mark.parametrize("P", [257, 4096])
def test_arbitrary_key_lists_vs_oracle(P):
    rng = np.random.default_rng(P)
    case = _key_case(rng, P)
    ix, co = _key_index(P)
    _load_case(ix, co, case)
    lists, models = _key_prompts(rng, case)
    keys, koff = key_csr(lists)
    weights = list(W16) + [1.0] * (16 - len(W16))
    s = check_vs_oracle(ix, co, weights, keys, koff, model=models)
    assert (s.max(axis=1) > 30).any() and (s.max(axis=1) == -1).any()
    check_vs_oracle(ix, co, weights, keys, koff, model=models, fm=_filters(rng, len(lists), P))
    check_vs_oracle(ix, co, weights, keys, koff, model0=0)
    # walks that end on each chunk edge: the number of blocks scored for pod base[0..3] of the unfiltered full chains
    assert len({float(x) for x in s[(np.diff(koff) == 70) & (models == 0)].ravel() if x > 0}) > 8


def test_forced_v1_equals_warp_kernel(monkeypatch):
    rng = np.random.default_rng(5)
    P = 257
    case = _key_case(rng, P)
    ix, co = _key_index(P)
    _load_case(ix, co, case)
    monkeypatch.setenv("KVIDX_SCORE_KERNEL", "v1")
    iv, cv = _key_index(P)
    _load_case(iv, cv, case)
    lists, models = _key_prompts(rng, case)
    keys, koff = key_csr(lists)
    fm = _filters(rng, len(lists), P)
    for kw in ({"model": models}, {"model": models, "filter_mask": fm}):
        a, ha = ix.score_keys(keys, koff, **kw)
        b, hb = iv.score_keys(keys, koff, **kw)
        assert a.tobytes() == b.tobytes() and np.array_equal(ha, hb)
        assert same_sparse(ix.score_keys_sparse(keys, koff, **kw), iv.score_keys_sparse(keys, koff, **kw))


# ---- probe chains ---------------------------------------------------------------------------------------------------
def test_displaced_and_wrapped_chains():
    """The chain and crowded-table plans of test_gpu_score_edges (displaced and wrapped chains, tombstones inside them)."""
    from test_gpu_score_edges import _chain_filters, _plans
    (plan, docs, keys, flat, other, prompts, models), (plan2, flat2, prompts2) = _plans()
    P = 64
    ix, co = _index_pair(capacity=1 << 16, table_slots=plan.S, max_pods=P, tier_weights=(1.0, 0.8, 0.3))
    plan.replay(ix, co)
    tok, off = csr(prompts)
    k, ko = ix.hash_keys(tok, off)
    for fm in (None, _chain_filters(len(prompts))):
        s = check_keys_vs_tokens(ix, tok, off, k, ko, model=models, fm=fm)
        want, _, _, _ = co.score_batch(tok, off, model=models, filter_mask=fm, n_threads=4)
        assert s.tobytes() == want.tobytes()
    ix2, co2 = _index_pair(capacity=1 << 16, table_slots=plan2.S, max_pods=P, tier_weights=(1.0, 0.8, 0.3))
    plan2.replay(ix2, co2)
    tok, off = csr(prompts2)
    k, ko = ix2.hash_keys(tok, off)
    s = check_keys_vs_tokens(ix2, tok, off, k, ko)
    assert s.tobytes() == co2.score_batch(tok, off, n_threads=4)[0].tobytes()


def test_keys_homed_on_one_pair_and_wrapped():
    """Keys placed with helpers.keys_homed_at: 12 keys on one home pair (a chain of six pairs), others on the last pair
    (chains wrap to slot 0), then some of them evicted (tombstones inside the chains)."""
    S, P = 1024, 16
    rng = np.random.default_rng(11)
    ix, co = _index_pair(capacity=1 << 12, table_slots=S, max_pods=P)
    crowd = keys_homed_at([100] * 12, 0, S, rng)
    wrap = keys_homed_at([S - 2] * 6, 0, S, rng)
    rest = keys_homed_at(rng.choice(np.arange(200, 900, 2), 40, replace=False), 0, S, rng)
    allk = np.concatenate([crowd, wrap, rest])
    for i, k in enumerate(allk):
        for t in (ix, co):
            assert t.add(0, [int(k) ^ 0xABC], [int(k)], [PT(i % 3), PT(5, 1)]) == 0
    for k in crowd[1:10:3]:
        for t in (ix, co):
            assert t.evict(0, int(k) ^ 0xABC, [PT(int(np.nonzero(allk == k)[0][0]) % 3), PT(5, 1)]) == 0
    assert ix.stats()["request_tombs"] >= 3
    lists = []
    for i in range(200):
        ks = rng.choice(allk, int(rng.integers(1, 50)))
        lists.append(np.concatenate([crowd[::-1][: i % 12], wrap, ks]))
    keys, koff = key_csr(lists)
    s = check_vs_oracle(ix, co, [1.0, 0.8] + [1.0] * 14, keys, koff)
    assert (s[:, 5] > 5).any()


# ---- other block sizes ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [4, 64, 256])
def test_other_block_sizes(B):
    rng = np.random.default_rng(B)
    P = 32
    ix, co = _index_pair(capacity=1 << 15, max_pods=P, block_size=B)
    docs = [rng.integers(0, 50000, B * int(rng.integers(2, 40)), dtype=np.uint32) for _ in range(20)]
    for d in range(4, 20):
        docs[d][:B * 2] = docs[d % 4][:B * 2]
    _fill(ix, co, docs, rng, P)
    prompts = []
    for i in range(500):
        doc = docs[i % 20]
        prompts.append(doc[:int(rng.integers(0, len(doc) + 1))] if i % 3 else doc)
    tok, off = csr(prompts)
    keys, koff = ix.hash_keys(tok, off)
    s = check_keys_vs_tokens(ix, tok, off, keys, koff)
    assert s.tobytes() == co.score_batch(tok, off, n_threads=4)[0].tobytes()
    assert s.tobytes() == oracle_rows(co, [1.0, 0.8] + [1.0] * 14, P, keys, koff).tobytes()


# ---- exact-LRU and CLOCK ----------------------------------------------------------------------------------------------
def test_exact_lru_stamps_every_present_key():
    """After score_keys, a capped write evicts exactly what the reference evicts: Lookup refreshed every present key of
    every prompt (no early exit), prompt after prompt, so a key held by several prompts ranks by the last of them."""
    rng = np.random.default_rng(21)
    CAP, P = 200, 16
    ix = kvidx.Index(capacity=CAP, pods_per_key=3, max_pods=P, lru_exact=1)
    co = COracle(size=CAP, pod_cache_size=3, max_pods=P)
    allk = rng.integers(1, 1 << 63, CAP, dtype=np.uint64)
    for i in range(0, CAP, 10):
        for t in (ix, co):
            assert t.add(0, allk[i:i + 10] ^ np.uint64(0x55), allk[i:i + 10], [PT(i % 7), PT(9, 1)]) == 0
    absent = rng.integers(1, 1 << 63, 20, dtype=np.uint64)
    lists = []
    perm = rng.permutation(allk[:120])
    for i in range(12):
        ks = perm[10 * i:10 * (i + 1)]
        ks = np.concatenate([ks, ks[:: 1 + i % 4]])               # repeats: the later one refreshes again
        if i % 4 == 3:
            ks = np.concatenate([ks, perm[:5 * i:7]])             # keys of earlier prompts: they rank as of this one
        if i % 3 == 0:
            ks = np.concatenate([absent[i:i + 1], ks])            # the walk ends at block 0; Lookup still touches the rest
        elif i % 3 == 1:
            ks = np.concatenate([ks[:2], absent[i:i + 1], ks[2:]])
        lists.append(ks)
    keys, koff = key_csr(lists)
    got, _ = ix.score_keys(keys, koff)
    want = oracle_rows(co, [1.0, 0.8] + [1.0] * 14, P, keys, koff)      # Lookup per prompt, in order: the same refreshes
    assert got.tobytes() == want.tobytes()
    # 80 new keys evict the 80 keys no prompt holds (keys a walk stopped short of were stamped too); 30 more evict the
    # first 30 keys stamped by the call, in prompt and key order
    for k_new in (80, 30):
        new = rng.integers(1, 1 << 63, k_new, dtype=np.uint64)
        for t in (ix, co):
            assert t.add(0, new ^ np.uint64(0x55), new, [PT(1)]) == 0
        assert ix.stats()["request_keys"] == co.len_request() == CAP
    r1, r2 = ix.lookup(0, allk), co.lookup(0, allk)
    assert np.array_equal(r1[2], r2[2]) and (r1[2][120:] == 0).all() and (r1[2][:120] == 0).sum() == 30


def test_clock_marks_what_the_token_path_marks():
    """Two identical CLOCK handles, one scored from tokens and one from the same prompts' keys, then the same capped
    write that evicts every unreferenced key: both keep exactly the oracle's referenced set R (clock_oracle) and the new
    keys, so both paths marked the same set.  (Which unreferenced keys a smaller write evicts depends on where the parallel
    inserts placed them, which may differ between two handles.)"""
    from clock_oracle import referenced_keys
    from test_gpu_clock import MODELS, Fill, _new_keys, clock_index, oracle_of, resident, score
    for n in (300, 4096):
        rng = np.random.default_rng(n)
        a, b = clock_index(1024), clock_index(1024)
        fa, fb = Fill(a, np.random.default_rng(9)), Fill(b, np.random.default_rng(9))
        ka, ea = _new_keys(rng, 1)
        for ix in (a, b):
            assert ix.add(0, ea, ka, [PT(2)]) == 0                    # a full turn: every key unreferenced
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
        b.score_keys(keys, koff, model=model, filter_mask=fm)
        kn, en = _new_keys(rng, fa.C - len(R))
        for ix in (a, b):
            assert ix.add(0, en, kn, [PT(3)]) == 0
        want = R | {(0, x) for x in kn}
        assert resident(a)[0] == want == resident(b)[0] and a.evictions() == b.evictions()


# ---- sharded handles ------------------------------------------------------------------------------------------------
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
    chains, foreign, absent, om = case
    for d, j, k, pts in chains:
        assert sh[0].add(0, [k ^ 0xE0E0], [k], pts) == 0
    for i, k in enumerate(foreign):
        assert sh[-1].add(om, [int(k) ^ 0xF0F0], [int(k)], [PT(3, i % 16), PT(4, 2)]) == 0
        assert sh[-1].add(0 if i % 2 else om, [int(k) ^ 0xF1F1], [int(k) ^ 1], [PT(7, 1)]) == 0
    lists, models = _key_prompts(rng, case)
    keys, koff = key_csr(lists)
    fm = _filters(rng, len(lists), P)
    want, wh = ix.score_keys(keys, koff, model=models, filter_mask=fm)
    for s in sh:
        got, gh = s.score_keys(keys, koff, model=models, filter_mask=fm)
        assert got.tobytes() == want.tobytes() and np.array_equal(gh, wh)
    # device-resident form through rank 0 (device 0 in every layout)
    import torch
    dev = torch.device("cuda", 0)
    d_k = torch.from_numpy(keys.view(np.int64)).to(dev)
    d_o = torch.from_numpy(koff).to(dev)
    d_s = torch.zeros((len(lists), P), dtype=torch.float64, device=dev)
    torch.cuda.synchronize(dev)
    sh[0].score_keys_dev(d_k.data_ptr(), d_o.data_ptr(), len(lists), d_s.data_ptr())
    sh[0].synchronize()
    no_f, _ = ix.score_keys(keys, koff)
    assert d_s.cpu().numpy().tobytes() == no_f.tobytes()


# ---- stream order, readers beside writers -----------------------------------------------------------------------------
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
    d_ev = torch.from_numpy(evs.view(np.uint8).reshape(-1).copy()).to(dev)
    d_q = torch.from_numpy(qoff).to(dev)
    d_hs = torch.from_numpy(hs.view(np.int64).copy()).to(dev)
    d_tk = torch.from_numpy(tk.view(np.int32).copy()).to(dev)
    toks, doc, m = wl.queries(0, 300)
    co = COracle(size=1 << 14, max_pods=32)
    keys, koff = co.hash_keys(toks.reshape(-1), np.arange(0, 301 * wl.T, wl.T, dtype=np.int64))
    d_k = torch.from_numpy(keys.view(np.int64).copy()).to(dev)
    d_o = torch.from_numpy(koff.astype(np.int64)).to(dev)
    d_pods = torch.zeros((300, 10), dtype=torch.int16, device=dev)
    d_sc = torch.zeros((300, 10), dtype=torch.float64, device=dev)
    d_cnt = torch.zeros(300, dtype=torch.uint8, device=dev)
    d_has = torch.zeros(300, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    ix.apply_events_dev(d_ev.data_ptr(), d_q.data_ptr(), len(qoff) - 1, len(evs), d_hs.data_ptr(), len(hs), d_tk.data_ptr())
    ix.score_keys_sparse_dev(d_k.data_ptr(), d_o.data_ptr(), 300, d_pods.data_ptr(), d_sc.data_ptr(), d_cnt.data_ptr(), d_has_keys=d_has.data_ptr())
    ix.synchronize()
    exp = wl.expected_scores(doc, m)
    cnt, pods_h, sc_h = d_cnt.cpu().numpy(), d_pods.cpu().numpy().view(np.uint16), d_sc.cpu().numpy()
    assert (d_has.cpu().numpy() == 1).all()
    for i in range(300):
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
        s1, _ = ix.score_keys(keys, koff)
        if not np.array_equal(s1, want):
            errs.append(AssertionError("scores changed while events were applied"))
    th.join()
    assert not errs, errs[:1]


# ---- host buffers ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [None, 65536])
def test_host_buffers_pageable_pinned_chunked_zero_copy(chunk, monkeypatch):
    if chunk:
        monkeypatch.setenv("KVIDX_HOST_CHUNK_TOKENS", str(chunk))
    rng = np.random.default_rng(31)
    P = 64
    ix = kvidx.Index(capacity=1 << 16, max_pods=P)
    docs = _prefix_docs(rng, max_blocks=40)
    _fill(ix, None, docs, rng, P)
    prompts = _ragged_prompts(rng, docs, 12000)
    tok, off = csr(prompts)
    keys, koff = ix.hash_keys(tok, off)
    if chunk:                                               # a chunk holds as many key bytes as `chunk` tokens: >= 3 chunks
        assert len(keys) > 2 * (chunk // 2)
    want, wh = ix.score_batch(tok, off)
    got, gh = ix.score_keys(keys, koff)
    assert got.tobytes() == want.tobytes() and np.array_equal(gh, wh)
    pk = kvidx.pinned_array(keys.shape, np.uint64)
    pk[:] = keys
    out = kvidx.pinned_array(want.shape, np.float64)
    got2, _ = ix.score_keys(kvidx._native._Raw(pk.ctypes.data), koff, out=out)
    assert out.tobytes() == want.tobytes()
    assert same_sparse(ix.score_keys_sparse(pk, koff), ix.score_batch_sparse(tok, off))
    for n in (1, 7, 32, 33):                                 # the zero-copy size and just above it, pageable and pinned
        o = koff[:n + 1]
        w, _ = ix.score_batch(tok, off[:n + 1])
        assert ix.score_keys(keys, o)[0].tobytes() == w.tobytes()
        assert ix.score_keys(pk, o)[0].tobytes() == w.tobytes()
        assert ix.score_keys(keys, koff[10:10 + n + 1])[0].tobytes() == ix.score_batch(tok, off[10:10 + n + 1])[0].tobytes()


# ---- errors ---------------------------------------------------------------------------------------------------------
def test_errors_and_empty_batch():
    import ctypes as C
    ix = kvidx.Index(capacity=1024, max_pods=8)
    L, u64, i64 = ix.L, C.POINTER(C.c_uint64), C.POINTER(C.c_int64)
    f64, u8, u16 = C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_uint16)
    keys = np.arange(1, 9, dtype=np.uint64)
    sc = np.full((4, 8), 7.0)
    has = np.full(4, 9, np.uint8)
    pods, ssc, cnt = np.zeros((4, 10), np.uint16), np.zeros((4, 10)), np.zeros(4, np.uint8)

    def dense(k, off, n):
        return L.kvidx_score_keys(ix.h, None if k is None else k.ctypes.data_as(u64), None if off is None else off.ctypes.data_as(i64), n,
                                  None, 0, None, sc.ctypes.data_as(f64), has.ctypes.data_as(u8))

    def sparse(k, off, n):
        return L.kvidx_score_keys_sparse(ix.h, None if k is None else k.ctypes.data_as(u64), None if off is None else off.ctypes.data_as(i64), n,
                                         None, 0, None, pods.ctypes.data_as(u16), ssc.ctypes.data_as(f64), cnt.ctypes.data_as(u8), has.ctypes.data_as(u8))
    good = np.array([0, 2, 4], np.int64)
    for fn in (dense, sparse):
        assert fn(keys, good, -1) == kvidx.EINVAL
        assert fn(keys, None, 2) == kvidx.EINVAL
        assert fn(keys, np.array([0, 3, 2], np.int64), 2) == kvidx.EINVAL and "not monotone" in ix.last_error()
        assert fn(None, good, 2) == kvidx.EINVAL
        assert fn(None, np.array([3, 3, 3], np.int64), 2) == 0               # no key at all: NULL keys is fine
        assert fn(keys, good, 0) == 0
    assert L.kvidx_score_keys_dev(ix.h, None, None, 1, None, 0, None, None, None) == kvidx.EINVAL
    assert L.kvidx_score_keys_dev(ix.h, None, None, -1, None, 0, None, 1, None) == kvidx.EINVAL
    sc[:] = 7.0; has[:] = 9
    assert dense(keys, good, 0) == 0 and (sc == 7.0).all() and (has == 9).all()   # n == 0: nothing written
    assert dense(None, np.array([3, 3, 3], np.int64), 2) == 0
    assert (sc[:2] == -1.0).all() and (has[:2] == 0).all()


# ---- host mirror ----------------------------------------------------------------------------------------------------
def test_host_mirror_get_pod_scores_keys():
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
    before = h.metrics()["lookup_requests_total"]
    for d, doc in enumerate(docs):
        for L in (len(doc), BS * 2 + 3, BS - 1):
            t = doc[:L]
            k = keys[d][:L // BS]
            a, b = h.get_pod_scores(t, "m"), h.get_pod_scores_keys(k, "m")
            assert a == b, d
            for pods in (["pod-%d" % (d % 4)], ["pod-9"], ["pod-1", "pod-2"]):
                assert h.get_pod_scores(t, "m", pods) == h.get_pod_scores_keys(k, "m", pods)
    assert h.get_pod_scores_keys([], "m") is None
    got = h.get_pod_scores_keys(keys[0], "m", ["pod-0"])
    assert got and set(got) == {"pod-0"}
    m0 = h.metrics()
    h.get_pod_scores_keys(keys[3], "m")
    m1 = h.metrics()
    assert m1["lookup_requests_total"] == m0["lookup_requests_total"] + 1 > before
    assert m1["lookup_hits_total"] - m0["lookup_hits_total"] == len(keys[3])
    h.get_pod_scores_keys([], "m")                                          # no keys: no Lookup
    assert h.metrics()["lookup_requests_total"] == m1["lookup_requests_total"]

