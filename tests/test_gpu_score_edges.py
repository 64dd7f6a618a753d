"""GPU (-m gpu): Score() on every dispatch path at the edges its walks implement separately -- keys displaced past their
home pair (behind full pairs, tombstones and equal tags of other models, wrapped past the table's end), several models
sharing hashes and tokens, pod rows of odd width and filters wider than one word, and all sixteen tier ids with unusual
weights.  Every result is compared bit-exact with the C++ oracle."""
import threading

import numpy as np
import pytest

from helpers import EVENT_DTYPE, PATHS, ROUND_PATHS, _home_of, _index_pair, _select_path, _slot_home, csr, filter_mask
import kvidx
from oracle.kvoracle_c import COracle

pytestmark = pytest.mark.gpu
BS = 16
FNV_OFFSET = 0xCBF29CE484222325


def PT(p, t=0):
    return (p << 4) | t


def _check_scores(ix, co, tok, off, model=None, model0=0, fm=None):
    s1, h1 = ix.score_batch(tok, off, model=model, model0=model0, filter_mask=fm)
    s2, h2, _, _ = co.score_batch(tok, off, model=model, model0=model0, filter_mask=fm, n_threads=4)
    assert np.array_equal(h1, h2)
    assert np.array_equal(s1, s2), np.argwhere(s1 != s2)[:5]
    return s2


def _check_sparse(ix, co, tok, off, model=None, fm=None):
    s2, _, _, _ = co.score_batch(tok, off, model=model, filter_mask=fm, n_threads=4)
    pods, sc, cnt, _ = ix.score_batch_sparse(tok, off, model=model, filter_mask=fm)
    for i in range(len(off) - 1):
        got = {int(pods[i, j]): float(sc[i, j]) for j in range(cnt[i])}
        assert got == {int(q): float(s2[i, q]) for q in np.nonzero(s2[i] >= 0)[0]}, i


def _check_lookup(ix, co, model, keys):
    r1, p1, c1 = ix.lookup(model, keys)
    r2, p2, c2 = co.lookup(model, keys)
    assert r1 == r2 == 0 and np.array_equal(c1, c2)
    for i in range(len(keys)):
        assert np.array_equal(p1[i, :c1[i]], p2[i, :c2[i]]), i


def test_home_slot_replica_matches_library():
    """The replica the chain tests place keys with: its shard bits (the top three of the mixed key) equal what an 8-shard
    handle computes, for random keys under random models and under one model0."""
    import torch
    rng = np.random.default_rng(1)
    n = 4096
    keys = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    models = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    models[:64] = np.arange(64)
    ix = kvidx.Index(capacity=1 << 12, shard_rank=0, shard_count=8)
    d_keys = torch.from_numpy(keys.view(np.int64)).cuda()
    d_model = torch.from_numpy(models.view(np.int32)).cuda()
    own = torch.zeros(n, dtype=torch.uint8, device="cuda")
    ix.key_owners_dev(d_keys.data_ptr(), n, own.data_ptr(), d_model=d_model.data_ptr())
    ix.synchronize()
    want = (_home_of(keys, models.astype(np.uint64)) >> np.uint64(61)).astype(np.uint8)
    assert np.array_equal(own.cpu().numpy(), want)
    ix.key_owners_dev(d_keys.data_ptr(), n, own.data_ptr(), model0=40000)
    ix.synchronize()
    assert np.array_equal(own.cpu().numpy(), (_home_of(keys, 40000) >> np.uint64(61)).astype(np.uint8))


# ---- displaced and wrapped probe chains ---------------------------------------------------------------------------------
class _Plan:
    """A replayable sequence of add / evict calls and a replica of where each request key lands.  Writers probe slot by
    slot from the even home slot and never reuse a tombstone, so a key lands at or after the end of the run of occupied
    slots that starts at its home when its call begins -- a lower bound that does not depend on the order of the keys
    inside one call."""

    def __init__(self, S):
        self.S, self.ops = S, []
        self.occ = np.zeros(S, np.int8)                 # 0 empty, 1 full, 2 tombstone
        self.pos, self.run = {}, {}

    def add(self, model, eng, req, pts):
        eng, req = np.atleast_1d(np.asarray(eng, np.uint64)), np.atleast_1d(np.asarray(req, np.uint64))
        self.ops.append(("add", model, eng, req, np.asarray(pts, np.uint16)))
        homes = _slot_home(req, model, self.S)
        new = [(int(r), int(h)) for r, h in zip(req, homes) if (model, int(r)) not in self.pos]
        for r, h in new:
            n = 0
            while self.occ[(h + n) % self.S]:
                n += 1
            self.run[(model, r)] = (h, n)
        for r, h in new:
            s = h
            while self.occ[s]:
                s = (s + 1) % self.S
            self.occ[s] = 1
            self.pos[(model, r)] = s

    def evict(self, model, eng, req, pts):
        """evict the engine key's only entries: its request slot becomes a tombstone"""
        self.ops.append(("evict", model, int(eng), np.asarray(pts, np.uint16)))
        self.occ[self.pos[(model, int(req))]] = 2

    def pairs_from_home(self, model, key):
        h, n = self.run[(model, int(key))]
        return n // 2, h + n >= self.S

    def tomb_before(self, model, key):
        h, s = self.run[(model, int(key))][0], self.pos[(model, int(key))]
        return any(self.occ[(h + d) % self.S] == 2 for d in range((s - h) % self.S))

    def replay(self, *targets):
        for op in self.ops:
            for t in targets:
                if op[0] == "add":
                    assert t.add(op[1], op[2], op[3], op[4]) == 0
                else:
                    assert t.evict(op[1], op[2], op[3]) == 0


class _Fillers:
    """Random request keys grouped by home pair (model 0), handed out without repetition."""

    def __init__(self, rng, S, n=1 << 21):
        keys = rng.integers(1, 1 << 63, n, dtype=np.uint64)
        pair = _slot_home(keys, 0, S) // 2
        o = np.argsort(pair, kind="stable")
        self.keys, self.pair = keys[o], pair[o]
        self.next = np.searchsorted(self.pair, np.arange(S // 2))
        self.eng = 0xF1000000

    def take(self, pair, n):
        i = self.next[pair]
        assert n == 0 or self.pair[i + n - 1] == pair
        self.next[pair] += n
        return self.keys[i:i + n]

    def engine(self):
        self.eng += 1
        return self.eng


def _block_homing_at(co, rng, parent, S, slot):
    """16 tokens whose block key under `parent` has its home at `slot` (brute force over random blocks)."""
    n = 1 << 15
    cand = rng.integers(0, 50000, (n, BS), dtype=np.uint32)
    keys, _ = co.hash_keys(cand.reshape(-1), np.arange(0, (n + 1) * BS, BS, dtype=np.int64), np.full(n, parent, np.uint64))
    hit = np.nonzero(_slot_home(keys, 0, S) == slot)[0]
    assert len(hit), "no block found"
    return cand[hit[0]]


def _other_model(key, S):
    """a model id != 0 under which `key` has the same home pair as under model 0"""
    m = np.arange(1, 1 << 16, dtype=np.uint64)
    hit = np.nonzero(_slot_home(np.full(len(m), key, np.uint64), m, S) == _slot_home(key, 0, S)[0])[0]
    assert len(hit)
    return int(m[hit[0]])


def _chain_plan(S=2048, P=64):
    """Phase one: clusters of fillers placed on purpose in front of the blocks of 14 documents.
      docs 0-2  (d)  every block behind 1-3 full pairs of fillers (consecutive retries; the tuned kernel's key ring fills);
      docs 3-5  (a)  every block behind 4 fillers that are evicted afterwards: tombstones inside the chains;
      docs 6-7  (b)  every block behind a slot with the SAME hash under another model (other pods), sometimes + fillers;
      docs 8-9  (c)  blocks whose home is the last pair of the table, behind fillers there: their chains wrap to slot 0
                     (doc 9 also has a cluster behind every other block);
      docs 10-13     no clusters."""
    rng = np.random.default_rng(7)
    co = COracle(size=10 ** 6, max_pods=P)
    plan, fill = _Plan(S), _Fillers(rng, S)
    docs = [rng.integers(0, 50000, BS * int(rng.integers(6, 12)), dtype=np.uint32) for _ in range(14)]
    docs[12][:BS * 3] = docs[10][:BS * 3]                   # shared prefixes
    docs[4][:BS * 2] = docs[0][:BS * 2]
    last = S - 2
    for d, blocks in ((8, (0, 3)), (9, (1,))):
        for j in blocks:
            parent = FNV_OFFSET if j == 0 else int(co.hash_keys(docs[d][:BS * j], [0, BS * j])[0][-1])
            docs[d][BS * j:BS * (j + 1)] = _block_homing_at(co, rng, parent, S, last)
    keys = [co.hash_keys(doc, [0, len(doc)])[0] for doc in docs]
    other, evict_later = {}, []
    for d in range(14):
        for j, k in enumerate(keys[d]):
            home_pair = int(_slot_home(k, 0, S)[0]) // 2
            if d <= 2 or (d == 9 and j % 2 == 0):
                for f in fill.take(home_pair, 2 * (1 + j % 3)):
                    plan.add(0, fill.engine(), f, [PT(int(rng.integers(0, P)), 1)])
            elif d <= 5:
                for f in fill.take(home_pair, 4):
                    e = fill.engine()
                    plan.add(0, e, f, [PT(5)])
                    evict_later.append((e, f))
            elif d <= 7:
                m = _other_model(k, S)
                other[(d, j)] = m
                plan.add(m, fill.engine(), k, [PT(60 - j, 2), PT(61, 0)])
                for f in fill.take(home_pair, j % 3):
                    plan.add(0, fill.engine(), f, [PT(5)])
            elif d <= 9 and home_pair == last // 2:
                for f in fill.take(home_pair, 2 + d % 2):
                    plan.add(0, fill.engine(), f, [PT(6)])
    for d in range(14):
        for g in range(1 + d % 3):
            pts = [PT(int(p), int(rng.integers(0, 3))) for p in rng.choice(P, size=int(rng.integers(1, 4)), replace=False)]
            if g == 0:
                pts.append(PT(0))                           # pod 0 holds every document from its first block on
            plan.add(0, keys[d] ^ np.uint64(0x5EED + g), keys[d], pts)
    for e, f in evict_later:
        plan.evict(0, e, f, [PT(5)])
    # coverage, from the replica: the chains this phase exists for are there
    dist = {(d, j): plan.pairs_from_home(0, k) for d in range(14) for j, k in enumerate(keys[d])}
    assert sum(p >= 2 for p, _ in dist.values()) >= 20
    assert all(dist[(d, j)][0] >= 1 for d in range(3) for j in range(len(keys[d])))
    assert sum(w for _, w in dist.values()) >= 2
    assert sum(plan.tomb_before(0, keys[d][j]) for d in range(3, 6) for j in range(len(keys[d]))) >= 15
    assert len(other) >= 10
    # prompts: whole documents, prefixes, divergent tails, one token changed; each three times in a row; the documents of
    # (b) also under the model of their first block's twin
    prompts, models = [], []
    for d, doc in enumerate(docs):
        nb = len(doc) // BS
        var = [doc, doc[:BS * int(rng.integers(1, nb))], np.concatenate([doc[:BS * int(rng.integers(1, nb))], rng.integers(0, 50000, 40, dtype=np.uint32)])]
        v = doc.copy(); v[BS * int(rng.integers(1, nb)) + 3] ^= 1; var.append(v)
        for pr in var:
            for m in ([0] if d not in (6, 7) else [0, other[(d, 0)]]):
                prompts += [pr] * 3
                models += [m] * 3
    flat = np.concatenate(keys)
    return plan, docs, keys, flat, other, prompts, np.array(models, np.uint32)


def _natural_plan(S=4096, P=64, fill=0.88):
    """Phase two: documents stored until about 88 % of the slots are full (no tombstones while filling, so no rebuild),
    then a few documents' tails evicted -- tombstones in a crowded table."""
    rng = np.random.default_rng(8)
    co = COracle(size=10 ** 6, max_pods=P)
    plan = _Plan(S)
    docs, keys, n = [], [], 0
    while n + 18 <= int(S * fill):
        doc = rng.integers(0, 50000, BS * 18, dtype=np.uint32)
        if docs and rng.random() < 0.3:
            doc[:BS * 4] = docs[-1][:BS * 4]
        k = co.hash_keys(doc, [0, len(doc)])[0]
        new = len(set(k.tolist()) - set(x for ks in keys for x in ks.tolist()))
        docs.append(doc); keys.append(k); n += new
        pts = [PT(int(p), int(rng.integers(0, 3))) for p in rng.choice(P, size=int(rng.integers(1, 4)), replace=False)]
        plan.add(0, k ^ np.uint64(0xABC), k, pts + [PT(0)])
    for d in range(0, len(docs), 9):
        for j in range(12, 18):
            plan.evict(0, int(keys[d][j] ^ np.uint64(0xABC)), keys[d][j], [PT(0)] + [int(x) for x in plan.ops[d][4][:-1]])
    assert (plan.occ != 0).sum() >= int(S * 0.87) and (plan.occ == 2).sum() >= 100
    dist = [plan.pairs_from_home(0, k) for ks in keys for k in ks]
    assert sum(p >= 2 for p, _ in dist) >= 300 and sum(p >= 8 for p, _ in dist) >= 20 and any(w for _, w in dist)
    prompts = []
    for i in range(600):
        doc = docs[int(rng.integers(0, len(docs)))]
        prompts.append(doc[:BS * int(rng.integers(1, 19))] if i % 3 else doc)
    return plan, np.concatenate(keys), prompts


_PLANS = {}


def _plans():
    if not _PLANS:
        _PLANS["chain"] = _chain_plan()
        _PLANS["natural"] = _natural_plan()
    return _PLANS["chain"], _PLANS["natural"]


def _chain_filters(n, P=64):
    fm = np.zeros((n, (P + 63) // 64), np.uint64)
    for i in range(0, n, 5):
        fm[i] = filter_mask([0, 60 - i % 7, 61] if i % 2 else [(i * 7) % P, 0], fm.shape[1])
    return fm


@pytest.mark.parametrize("kernel", PATHS)
def test_displaced_and_wrapped_chains(kernel, monkeypatch):
    _select_path(monkeypatch, kernel)
    (plan, docs, keys, flat, other, prompts, models), (plan2, flat2, prompts2) = _plans()
    P = 64
    ix, co = _index_pair(capacity=1 << 16, table_slots=plan.S, max_pods=P, tier_weights=(1.0, 0.8, 0.3))
    plan.replay(ix, co)
    st = ix.stats()
    assert st["rebuilds"] == 0 and st["request_keys"] == co.len_request() and st["engine_keys"] == co.len_engine()
    assert st["request_tombs"] >= 40
    tok, off = csr(prompts)
    _check_scores(ix, co, tok, off, model=models)
    s = _check_scores(ix, co, tok, off, model=models, fm=_chain_filters(len(prompts)))
    assert (s[models == 0, 0] >= 6).any() and (s[models != 0] >= 0).any()
    _check_sparse(ix, co, tok, off, model=models)
    _check_lookup(ix, co, 0, np.unique(flat))
    for (d, j), m in other.items():
        _check_lookup(ix, co, m, keys[d][j:j + 1])
    # phase two: a crowded table
    ix2, co2 = _index_pair(capacity=1 << 16, table_slots=plan2.S, max_pods=P, tier_weights=(1.0, 0.8, 0.3))
    plan2.replay(ix2, co2)
    st = ix2.stats()
    assert st["rebuilds"] == 0 and st["request_keys"] == co2.len_request() and st["request_tombs"] > 0
    tok, off = csr(prompts2)
    s = _check_scores(ix2, co2, tok, off)
    assert (s.max(axis=1) >= 10).sum() > 100
    _check_lookup(ix2, co2, 0, np.unique(flat2))


@pytest.mark.parametrize("peer_pair", [0, 1])
@pytest.mark.parametrize("kernel", ROUND_PATHS)
def test_displaced_chains_on_two_shards(kernel, peer_pair, monkeypatch):
    """The same chains on a 2-shard index on one GPU (a key's slot inside its shard is the same as unsharded), written
    through rank 0 and read through both ranks, with the peer's slot pair fetched at once or home slot first."""
    from test_gpu_shard_ops import _shards
    _select_path(monkeypatch, kernel)
    monkeypatch.setenv("KVIDX_PEER_PAIR", str(peer_pair))
    (plan, docs, keys, flat, other, prompts, models), _ = _plans()
    P = 64
    sh = _shards(2, hash_seed="", capacity=1 << 16, table_slots=plan.S, pods_per_key=10, max_pods=P, tier_weights=(1.0, 0.8, 0.3))
    co = COracle(size=1 << 16, max_pods=P, tier_weights=(1.0, 0.8, 0.3))
    plan.replay(sh[0], co)
    assert sum(s.stats()["request_keys"] for s in sh) == co.len_request()
    owners = _home_of(flat, 0) >> np.uint64(63)
    assert 0 < owners.sum() < len(flat)
    tok, off = csr(prompts)
    fm = _chain_filters(len(prompts))
    for s in sh:
        _check_scores(s, co, tok, off, model=models, fm=fm)
    _check_lookup(sh[1], co, 0, np.unique(flat))


# ---- several models ----------------------------------------------------------------------------------------------------
MODELS = (0, 7, 65535)


def _model_events(rng, P=24):
    """One event stream stored under three models: the same engine hashes and tokens, other pods per model; one event per
    call.  Then one batch on one pod in which parents stored earlier IN THE SAME BATCH under another model must not be
    found."""
    from test_gpu_parity import _random_stream
    docs = [rng.integers(0, 50000, BS * int(rng.integers(2, 12))).tolist() for _ in range(16)]
    for i in range(8, 16):
        docs[i] = docs[i - 8][:BS * int(rng.integers(1, 4))] + docs[i]
    ev, hs, tk = _random_stream(rng, 220, BS, P, 3, docs)
    calls = []
    for e in ev:
        for mi, m in enumerate(MODELS):
            r = e.copy()
            r["model"] = m
            r["podtier"] = (((int(e["podtier"]) >> 4) + 5 * mi) % P << 4) | (int(e["podtier"]) & 15)
            calls.append(np.array([r], EVENT_DTYPE))
    # the batch: T_c under model 0 and T_a under model 7 are both stored as engine hash H1; children of H1 under model 7, 0 and
    # 65535 (which never stored H1) hash from different parents
    H1, H2, H3, H5 = 9000001, 9000002, 9000003, 9000005
    blk = [rng.integers(0, 50000, BS).tolist() for _ in range(5)]
    spec = [(0, H1, None, blk[0]), (7, H1, None, blk[1]), (65535, H2, H1, blk[2]), (7, H3, H1, blk[3]), (0, H5, H1, blk[4])]
    b_ev, b_hs, b_tk = [], list(hs), list(tk)
    for m, h, par, t in spec:
        r = np.zeros((), EVENT_DTYPE)
        r["op"] = 0; r["podtier"] = PT(3, 1); r["model"] = m; r["hash_off"] = len(b_hs); r["n_hashes"] = 1
        r["has_parent"] = par is not None; r["parent_hash"] = par or 0; r["tok_off"] = len(b_tk); r["n_tokens"] = BS
        b_hs.append(h); b_tk.extend(t)
        b_ev.append(r)
    hs, tk = np.array(b_hs, np.uint64), np.array(b_tk, np.uint64).astype(np.uint32)
    batch = np.array(b_ev, EVENT_DTYPE)
    prompts = []
    for i in range(160):
        d = docs[int(rng.integers(0, len(docs)))]
        prompts.append(d[:BS * int(rng.integers(1, len(d) // BS + 1))] if i % 4 else d)
    prompts += [blk[1] + blk[3], blk[0] + blk[4], blk[2], blk[0] + blk[3]]
    return calls, batch, hs, tk, docs, prompts


@pytest.fixture(scope="module")
def model_data():
    return _model_events(np.random.default_rng(33))


def _model_pair(model_data, P=24):
    calls, batch, hs, tk, _, _ = model_data
    ix, co = _index_pair(capacity=1 << 15, max_pods=P, pods_per_key=6, tier_weights=(1.0, 0.8, 0.3))
    for c in calls:
        assert ix.apply_events(c, hs, tk)[0] == 0 and co.apply_events(c, hs, tk)[0] == 0
    assert ix.apply_events(batch, hs, tk)[0] == 0
    for i in range(len(batch)):
        assert co.apply_events(batch[i:i + 1], hs, tk)[0] == 0
    return ix, co


@pytest.mark.parametrize("kernel", PATHS)
def test_several_models(kernel, model_data, monkeypatch):
    _select_path(monkeypatch, kernel)
    calls, batch, hs, tk, docs, prompts = model_data
    ix, co = _model_pair(model_data)
    st = ix.stats()
    assert st["request_keys"] == co.len_request() and st["engine_keys"] == co.len_engine()
    if kernel == "v1":                                        # the write path and Lookup do not depend on the Score() path
        uh = np.unique(hs)
        for m in MODELS + (3,):
            assert [ix.get_request_key(m, h) for h in uh] == [co.get_request_key(m, h) for h in uh], m
        keys = np.unique(co.hash_keys(*csr(prompts))[0])
        for m in MODELS + (3,):
            _check_lookup(ix, co, m, keys)
    # identical prompts under different models next to each other (and twice, so that classes form)
    tok, off = csr([p for p in prompts for _ in range(8)])
    model = np.array([(0, 7, 65535, 3)[j % 4] for _ in prompts for j in range(8)], np.uint32)
    s = _check_scores(ix, co, tok, off, model=model)
    rows = s.reshape(len(prompts), 8, -1)
    assert sum(len({rows[i, j].tobytes() for j in range(3)}) == 3 for i in range(len(prompts))) >= 20
    assert (rows[:, 3] == -1).all()
    _check_sparse(ix, co, tok, off, model=model)
    tok, off = csr(prompts)
    for m0 in (7, 65535):
        _check_scores(ix, co, tok, off, model0=m0)
    # model ids above 16 bits never match: every row absent, has_keys set for every prompt with a block
    nb = np.diff(off) // BS
    for mdl, m0 in ((None, 70000), (None, 65536), (np.array([65536, 65536 + 7, 1 << 31, 0xFFFFFFFF] * 41, np.uint32)[:len(prompts)], 0)):
        s1, h1 = ix.score_batch(tok, off, model=mdl, model0=m0)
        assert (s1 == -1).all() and np.array_equal(h1, (nb > 0).astype(np.uint8))
        _check_scores(ix, co, tok, off, model=mdl, model0=m0)


def test_coalesced_callers_that_differ_only_in_model():
    """64 threads whose one-prompt calls differ only in model0 (1 K-token prompts, stored under three models on other
    pods): a coalesced batch carries a per-prompt model array, and every caller gets the rows of its own model."""
    rng = np.random.default_rng(34)
    P = 32
    ix, co = _index_pair(capacity=1 << 15, max_pods=P)
    docs = rng.integers(0, 50000, (40, 1024), dtype=np.uint32)
    for d in range(len(docs)):
        k = co.hash_keys(docs[d], [0, 1024])[0]
        for mi, m in enumerate(MODELS):
            n = len(k) - (d + 7 * mi) % 9                            # cached to a depth that differs per model
            pts = [PT((d + 11 * mi) % P, mi % 2)]
            assert ix.add(m, k[:n] ^ np.uint64(m + 1), k[:n], pts) == 0 and co.add(m, k[:n] ^ np.uint64(m + 1), k[:n], pts) == 0
    calls = [csr([docs[d]]) for d in range(len(docs))]
    want = {m: co.score_batch(*csr(list(docs)), model0=m)[0] for m in MODELS}
    assert all(not np.array_equal(want[0][d], want[7][d]) for d in range(len(docs)))
    errs = []
    go = threading.Barrier(64)

    def caller(c):
        try:
            go.wait()
            m = MODELS[c % 3]
            for it in range(20):
                q = (c + it) % len(docs)
                s, _ = ix.score_batch(*calls[q], model0=m)
                assert np.array_equal(s[0], want[m][q]), (c, it)
        except Exception as ex:                                       # noqa: BLE001
            errs.append(ex)

    ths = [threading.Thread(target=caller, args=(c,)) for c in range(64)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errs, errs[:2]
    assert ix.stats()["coalesced_calls"] > 0


# ---- pod rows and filters ----------------------------------------------------------------------------------------------
def _pod_case(P, rng, n_prompts):
    pods = sorted({0, 63, 64, 127, P - 1} & set(range(P)))
    FW = (P + 63) // 64
    docs = [rng.integers(0, 50000, BS * int(rng.integers(2, 9)), dtype=np.uint32) for _ in range(10)]
    adds = []
    for d, doc in enumerate(docs):
        mine = {pods[d % len(pods)]} | set(rng.choice(pods, size=int(rng.integers(1, len(pods) + 1)), replace=False).tolist())
        adds.append((doc, [PT(p, int(rng.integers(0, 2))) for p in sorted(mine)]))
    prompts, fm = [], np.zeros((n_prompts, FW), np.uint64)
    kinds = []
    for i in range(n_prompts):
        doc = docs[i % len(docs)] if i % 2 == 0 else prompts[-1]
        prompts.append(doc if i % 2 or i % 6 else doc[:BS * int(rng.integers(1, len(doc) // BS + 1))])
        kind = (i // 2) % 6
        if kind == 1:                                         # bits only in words >= 1
            if FW > 1:
                fm[i] = filter_mask([p for p in pods if p >= 64] + [int(rng.integers(64, P))], FW)
        elif kind == 2:                                       # bits at or above max_pods (in the last word), with or without a pod
            if P % 64:
                fm[i, -1] = ~np.uint64(0) << np.uint64(P % 64)
                if i % 4 == 0:
                    fm[i] |= filter_mask([pods[-1]], FW)
        elif kind >= 3:                                       # some valid pod set
            fm[i] = filter_mask(rng.choice(pods, size=int(rng.integers(1, len(pods) + 1)), replace=False).tolist(), FW)
        if i % 2:                                             # the same prompt, the filter differing only in its last word
            fm[i] = fm[i - 1]
            fm[i, -1] ^= np.uint64(1) << np.uint64((P - 1) % 64)
        kinds.append(kind)
    return adds, prompts, fm


def _pod_index(P, adds):
    ix, co = _index_pair(capacity=1 << 14, max_pods=P, tier_weights=(1.0, 0.8))
    for d, (doc, pts) in enumerate(adds):
        k = co.hash_keys(doc, [0, len(doc)])[0]
        assert ix.add(0, k ^ np.uint64(d + 1), k, pts) == 0 and co.add(0, k ^ np.uint64(d + 1), k, pts) == 0
    return ix, co


def _check_dev_offset(ix, co, tok, off, fm):
    """score_batch_dev into a torch buffer whose base is 8 bytes past an allocation: no row is 16-byte aligned"""
    import torch
    n, P = len(off) - 1, ix.max_pods
    d_tok = torch.from_numpy(tok.view(np.int32).copy()).cuda()
    d_off = torch.from_numpy(off.copy()).cuda()
    d_fm = torch.from_numpy(fm.view(np.int64).copy()).cuda()
    buf = torch.full((n * P + 1,), 7.0, dtype=torch.float64, device="cuda")
    has = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()                                  # the handle's stream does not wait for torch's
    ix.score_batch_dev(d_tok.data_ptr(), d_off.data_ptr(), n, buf.data_ptr() + 8, d_filter=d_fm.data_ptr(), d_has_keys=has.data_ptr())
    ix.synchronize()
    got = buf.cpu().numpy()
    s2, h2, _, _ = co.score_batch(tok, off, filter_mask=fm, n_threads=4)
    assert got[0] == 7.0 and np.array_equal(got[1:].reshape(n, P), s2) and np.array_equal(has.cpu().numpy(), h2)


@pytest.mark.parametrize("kernel", PATHS)
def test_pod_rows_and_wide_filters(kernel, monkeypatch):
    _select_path(monkeypatch, kernel)
    for P in (1, 3, 65, 127, 4096):
        rng = np.random.default_rng(P)
        adds, prompts, fm = _pod_case(P, rng, 240)
        ix, co = _pod_index(P, adds)
        tok, off = csr(prompts)
        s = _check_scores(ix, co, tok, off)
        assert all((s[:, p] >= 0).any() for p in {0, 63, 64, 127, P - 1} if p < P), P
        s = _check_scores(ix, co, tok, off, fm=fm)
        assert sum(not np.array_equal(s[i], s[i + 1]) for i in range(0, len(s), 2)) >= 15, P
        _check_sparse(ix, co, tok, off, fm=fm)
        small = slice(0, 21)                                  # a small host batch: the zero-copy path where it applies
        t2, o2 = csr(prompts[small])
        _check_scores(ix, co, t2, o2, fm=fm[small])
        _check_dev_offset(ix, co, tok, off, fm)
        if P == 4096 and kernel in ("auto", "coop", "classes8"):
            # 32 KB rows: a batch of more than 4096 prompts goes through the host pipeline in several chunks
            big = [prompts[i % len(prompts)][:BS * (1 + i % 3)] for i in range(4200)]
            tb, ob = csr(big)
            fb = fm[np.arange(4200) % len(fm)]
            _check_scores(ix, co, tb, ob, fm=fb)


# ---- tiers and weights -------------------------------------------------------------------------------------------------
W5 = (0.1, 1 / 3, 0.0, -0.25, 5e-324)                   # ids 5..15: the default 1.0


def _fold(co, weights, prompt):
    """LongestPrefixScorer.Score as an in-order Python fold: {pod: (score, addends)}"""
    keys, _ = co.hash_keys(np.asarray(prompt, np.uint32), [0, len(prompt)])
    if not len(keys):
        return {}
    _, pt, cnt = co.lookup(0, keys)
    ents = [pt[i, :cnt[i]].tolist() for i in range(len(keys))]

    def mx(es, p):
        m = 0.0
        for e in es:
            if e >> 4 == p and weights[e & 15] > m:
                m = weights[e & 15]
        return m
    out = {p: (mx(ents[0], p), [mx(ents[0], p)]) for p in {e >> 4 for e in ents[0]}}
    active = set(out)
    for es in ents[1:]:
        active &= {e >> 4 for e in es}
        if not active:
            break
        for p in active:
            a = mx(es, p)
            out[p] = (out[p][0] + a, out[p][1] + [a])
    return out


def _tier_case(rng, P=32):
    docs, adds = [], []
    for d in range(12):
        nb = 14 if d < 6 else int(rng.integers(2, 10))
        docs.append(rng.integers(0, 50000, BS * nb, dtype=np.uint32))
    for d, doc in enumerate(docs):
        nb = len(doc) // BS
        for j in range(nb):
            if d == 0:                                # ten distinct pods on every tier id: entries 8 and 9 in the fifth word
                pts = [PT(p, (p + j) % 16) for p in range(10)]
            elif d == 1:                              # one pod on three tiers whose maximum moves from block to block
                pts = [PT(12, j % 16), PT(12, (j + 5) % 16), PT(12, (j * 7 + 11) % 16), PT(13, 3), PT(13, 2), PT(14, 15 - j % 16)]
            elif d == 2:                              # 0.1 and 1/3, fourteen times
                pts = [PT(20, 0), PT(21, 1), PT(22, 4)]
            elif d == 3:                              # block 0 weighs <= 0 only: score 0.0, still alive
                pts = [PT(23, 3 if j == 0 else 1), PT(24, 2), PT(25, 3)]
            elif d < 6:                               # full slots of the same pattern block after block
                pts = [PT(p, (p * 3 + d) % 16) for p in range(10, 20)]
            else:
                pts = [PT(int(p), int(rng.integers(0, 16))) for p in rng.choice(P, size=int(rng.integers(1, 11)), replace=False)]
            adds.append((doc[:BS * (j + 1)], pts))
    prompts = []
    for d, doc in enumerate(docs):
        nb = len(doc) // BS
        for L in range(1, nb + 1):
            prompts += [doc[:BS * L]] * 2
        prompts.append(np.concatenate([doc, rng.integers(0, 50000, 20, dtype=np.uint32)]))
    return adds, prompts


@pytest.mark.parametrize("kernel", PATHS)
def test_all_sixteen_tiers_and_odd_weights(kernel, monkeypatch):
    _select_path(monkeypatch, kernel)
    P = 32
    adds, prompts = _tier_case(np.random.default_rng(16), P)
    ix, co = _index_pair(capacity=1 << 14, max_pods=P, pods_per_key=10, tier_weights=W5)
    for i, (pre, pts) in enumerate(adds):
        k = co.hash_keys(pre, [0, len(pre)])[0][-1:]
        assert ix.add(0, [1000 + i], k, pts) == 0 and co.add(0, [1000 + i], k, pts) == 0
    _, _, cnt = co.lookup(0, co.hash_keys(adds[0][0], [0, BS])[0])
    assert cnt[0] == 10
    tok, off = csr(prompts)
    weights = list(W5) + [1.0] * 11
    for step in range(2):
        s = _check_scores(ix, co, tok, off)
        _check_sparse(ix, co, tok, off)
        assert ((s == 0.0).sum(axis=1) > 0).any()               # a pod scored 0.0 is present, not absent
        # a few rows against the in-order fold; at least one run of equal addends sums to something other than n * w
        reassoc = 0
        for i in range(0, len(prompts), 7):
            f = _fold(co, weights, prompts[i])
            row = np.full(P, -1.0)
            for p, (v, adds_) in f.items():
                row[p] = v
                if len(adds_) > 2 and len(set(adds_)) == 1 and v != len(adds_) * adds_[0]:
                    reassoc += 1
            assert np.array_equal(s[i], row), i
        assert reassoc > 0
        if step == 0:                                           # weights change between two calls on the same handle
            for t, w in ((0, 0.7), (5, -0.0), (6, 1 / 3), (8, 0.1), (15, 2.5), (4, 1 / 3), (2, 5e-324)):
                ix.set_tier_weight(t, w)
                co.L.ko_set_tier_weight(co.h, t, w)
                weights[t] = w
