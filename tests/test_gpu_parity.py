"""GPU (-m gpu): the CUDA path through the C ABI vs the oracle / golden fixtures, bit-exact."""
import numpy as np
import pytest

from helpers import (EVENT_DTYPE, PATHS, ROUND_PATHS, Interner, _index_pair, _select_path, csr, dense_from_map, filter_mask, golden,
                     scenario_events)
import kvidx
from kvidx import synth
from oracle import kvoracle as ko
from oracle.kvoracle_c import COracle

pytestmark = pytest.mark.gpu
KATS = golden("hash_kats.json")


@pytest.mark.parametrize("case", KATS["cases"], ids=[c["name"] for c in KATS["cases"]])
def test_hash_keys_kats(case):
    ix = kvidx.Index(block_size=case["block_size"], hash_seed=case["seed"], capacity=1024)
    tok, off = csr([case["tokens"]])
    par = None if case["parent"] is None else np.array([case["parent"]], np.uint64)
    keys, koff = ix.hash_keys(tok, off, par)
    assert [int(k) for k in keys] == case["keys"] and koff[-1] == len(case["keys"])


def test_hash_keys_ragged_batch_vs_oracle():
    rng = np.random.default_rng(5)
    lens = [0, 1, 15, 16, 17, 31, 32, 33, 4096, 100, 0, 257] + rng.integers(0, 600, 200).tolist()
    prompts = [rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32) if i % 3 == 0
               else rng.integers(0, 128256, n).astype(np.uint32) for i, n in enumerate(lens)]
    tok, off = csr(prompts)
    parent = rng.integers(0, 1 << 63, len(lens), dtype=np.uint64)
    parent[::5] = [0, 23, 24, 255, 256, 65535, 65536, 2 ** 32 - 1, 2 ** 32][0] if False else parent[::5]
    pv = (rng.random(len(lens)) < 0.5).astype(np.uint8)
    ix = kvidx.Index(capacity=1024)
    co = COracle()
    for par, val in ((None, None), (parent, None), (parent, pv)):
        k1, o1 = ix.hash_keys(tok, off, par, val)
        k2, o2 = co.hash_keys(tok, off, par, val)
        assert np.array_equal(o1, o2) and np.array_equal(k1, k2)


def PT(p, t=0):
    return (p << 4) | t


def test_reference_index_suite_on_gpu():
    """pkg/kvcache/kvblock/index_test.go:66-211 + in_memory_test.go:85-116 through the C ABI."""
    ix = kvidx.Index(capacity=1024)
    # BasicAddAndLookup
    assert ix.add(0, [55269488], [10633516], [PT(1), PT(2)]) == 0
    rc, pt, cnt = ix.lookup(0, [10633516])
    assert rc == 0 and cnt[0] == 2 and sorted(pt[0, :2].tolist()) == [PT(1), PT(2)]
    # DuplicatePodHandling: same pod on two tiers is two entries; order oldest -> newest
    assert ix.add(0, [91642125], [61519471], [PT(1), PT(2)]) == 0
    assert ix.add(0, [91642125], [61519471], [PT(1), PT(2, 1), PT(3)]) == 0
    rc, pt, cnt = ix.lookup(0, [61519471])
    assert pt[0, :cnt[0]].tolist() == [PT(2), PT(1), PT(2, 1), PT(3)]
    # FilteredLookup
    assert ix.add(0, [93788608], [55204205], [PT(1), PT(2), PT(3)]) == 0
    rc, pt, cnt = ix.lookup(0, [55204205], filter_mask([1], ix.filter_words))
    assert pt[0, :cnt[0]].tolist() == [PT(1)]
    rc, pt, cnt = ix.lookup(0, [55204205], filter_mask([1, 3], ix.filter_words))
    assert pt[0, :cnt[0]].tolist() == [PT(1), PT(3)]
    rc, pt, cnt = ix.lookup(0, [55204205], filter_mask([99], ix.filter_words))
    assert cnt[0] == 0
    # EvictBasic: exact (pod,tier) pairs only
    assert ix.add(0, [17434655], [59244875], [PT(1), PT(2), PT(3)]) == 0
    assert ix.evict(0, 17434655, [PT(1), PT(3, 1)]) == 0
    rc, pt, cnt = ix.lookup(0, [59244875])
    assert pt[0, :cnt[0]].tolist() == [PT(2), PT(3)]
    # model name is part of the key identity (index.go:138-141)
    rc, pt, cnt = ix.lookup(7, [59244875])
    assert cnt[0] == 0
    # a missing key does not cut the lookup (in_memory.go:137-139)
    rc, pt, cnt = ix.lookup(0, [424242, 59244875, 10633516])
    assert cnt.tolist() == [0, 2, 2]
    # errors
    assert ix.lookup(0, [])[0] == kvidx.EINVAL
    assert ix.add(0, [], [], [PT(1)]) == kvidx.EINVAL and ix.add(0, [1, 2], [3], [PT(1)]) == kvidx.EINVAL
    assert ix.add(0, [1], [2], []) == kvidx.EINVAL and ix.evict(0, 1, []) == kvidx.EINVAL
    assert ix.evict(0, 40404, [PT(1)]) == 0                       # unknown engine key: silent no-op
    assert ix.get_request_key(0, 40404)[0] == kvidx.ENOENT and "engine key not found" in ix.last_error()
    assert ix.get_request_key(0, 17434655) == (0, 59244875)
    # evicting the last entry removes the request key and the engine mapping
    assert ix.evict(0, 17434655, [PT(2), PT(3)]) == 0
    assert ix.lookup(0, [59244875])[2][0] == 0 and ix.get_request_key(0, 17434655)[0] == kvidx.ENOENT
    # PodCacheSize cap
    ix2 = kvidx.Index(capacity=64, pods_per_key=2)
    assert ix2.add(0, [28409753], [51374550], [PT(1), PT(2), PT(3, 1)]) == 0
    rc, pt, cnt = ix2.lookup(0, [51374550])
    assert pt[0, :cnt[0]].tolist() == [PT(2), PT(3, 1)]


def test_scorer_known_answers_on_gpu():
    """kvblock_scorer_test.go:34-99 through the fused score call (block size 4, weights gpu 1.0 cpu 0.5)."""
    for third, expect in (([PT(0), PT(0, 1)], 3.0), ([PT(0, 1)], 2.5)):
        ix = kvidx.Index(block_size=4, capacity=1024, tier_weights=(1.0, 0.5), max_pods=8)
        toks = np.arange(24, dtype=np.uint32) + 100
        keys, _ = ix.hash_keys(toks, [0, 24])
        ents = [[PT(0)], [PT(0)], third, [PT(1, 1)], [PT(1, 1)], [PT(0)]]
        for i, e in enumerate(ents):
            assert ix.add(0, [9000 + i], [keys[i]], e) == 0
        scores, has = ix.score_batch(toks, [0, 24])
        assert has[0] == 1 and scores[0].tolist() == [expect] + [-1.0] * 7
        pods, sc, cnt, _ = ix.score_batch_sparse(toks, [0, 24])
        assert cnt[0] == 1 and pods[0, 0] == 0 and sc[0, 0] == expect


def _check_scenario(ix, sc, pods, tiers, P):
    tok, off = csr([p["tokens"] for p in sc["prompts"]])
    fm = np.stack([filter_mask([pods.ids[x] for x in p["filter"]], ix.filter_words) for p in sc["prompts"]])
    keys, koff = ix.hash_keys(tok, off)
    scores, has = ix.score_batch(tok, off, filter_mask=fm)
    sp_p, sp_s, sp_c, _ = ix.score_batch_sparse(tok, off, filter_mask=fm)
    for i, p in enumerate(sc["prompts"]):
        assert [int(k) for k in keys[koff[i]:koff[i + 1]]] == p["keys"]
        assert bool(has[i]) == bool(p["keys"])
        exp = dense_from_map(p["scores"], pods, P)
        assert np.array_equal(scores[i], exp), (i, p["scores"], scores[i][scores[i] >= 0])
        got = {int(sp_p[i, j]): float(sp_s[i, j]) for j in range(sp_c[i])}
        assert got == {pods.ids[k]: v for k, v in (p["scores"] or {}).items()}
        if p["keys"]:
            rc, pt, cnt = ix.lookup(0, np.array(p["keys"], np.uint64), fm[i] if p["filter"] else None)
            assert rc == 0
            for j, ents in enumerate(p["lookup"]):
                assert [(int(e) >> 4, int(e) & 15) for e in pt[j, :cnt[j]]] == [(pods.ids[a], tiers.ids[b]) for a, b in ents]


@pytest.mark.parametrize("one_by_one", [True, False])
def test_scenario_small_vs_golden(one_by_one):
    """Event stream -> index -> keys / lookups / scores, bit-exact against the Python-oracle fixture.
    one_by_one replays events in arrival order (one call each); the batched run submits everything in
    one kvidx_apply_events call, which only promises per-pod order (kvevents/pool.go:129-144)."""
    sc = golden("scenario_small.json")
    pods, tiers = Interner(sc["pods"]), Interner(sc["tiers"])
    P = 64
    w = [sc["weights"].get(t, 1.0) for t in sc["tiers"]]
    ix = kvidx.Index(block_size=sc["block_size"], hash_seed=sc["hash_seed"], capacity=4096,
                     pods_per_key=sc["pod_cache_size"], tier_weights=w, max_pods=P)
    ev, hs, tk = scenario_events(sc, pods, tiers)
    dropped = 0
    if one_by_one:
        for i in range(len(ev)):
            rc, d = ix.apply_events(ev[i:i + 1], hs, tk)
            assert rc == 0
            dropped += d
        st = ix.stats()
        assert st["request_keys"] == sc["final_request_keys"] and st["engine_keys"] == sc["final_engine_keys"]
        _check_scenario(ix, sc, pods, tiers, P)
    else:
        rc, dropped = ix.apply_events(ev, hs, tk)
        assert rc == 0
        # One call only promises per-pod order; the scenario's pods share documents and parents, so the final index depends
        # on how the pods' queues interleave (the reference's workers race the same way).  What every schedule agrees on must
        # hold exactly: replay many random merges of the per-pod queues through the oracle and keep, per prompt, the set of
        # outcomes; a prompt with ONE outcome across all of them is schedule-independent and the GPU must reproduce it.
        podid = ev["podtier"] >> 4
        queues = {int(p): np.nonzero(podid == p)[0].tolist() for p in np.unique(podid)}
        tok, off = csr([p["tokens"] for p in sc["prompts"]])
        fm = np.stack([filter_mask([pods.ids[x] for x in p["filter"]], ix.filter_words) for p in sc["prompts"]])
        rng = np.random.default_rng(0)
        outcomes = [set() for _ in sc["prompts"]]
        for it in range(120):
            q = {p: list(v) for p, v in queues.items()}
            order = []
            if it == 0:
                order = np.argsort(podid, kind="stable").tolist()            # pod after pod
            elif it == 1:
                order = list(range(len(ev)))                                   # arrival order
            else:
                while q:
                    p = int(rng.choice(list(q.keys())))
                    order.append(q[p].pop(0))
                    if not q[p]:
                        del q[p]
            co = COracle(block_size=sc["block_size"], init_hash=ko.fnv64a(sc["hash_seed"].encode()), size=10 ** 6,
                         pod_cache_size=sc["pod_cache_size"], tier_weights=w, max_pods=P)
            d_or = 0
            for i in order:
                d_or += co.apply_events(ev[i:i + 1], hs, tk)[1]
            assert d_or == dropped                                             # drops do not depend on the schedule
            s_or, _, _, _ = co.score_batch(tok, off, filter_mask=fm)
            for i in range(len(s_or)):
                outcomes[i].add(s_or[i].tobytes())
        got, has = ix.score_batch(tok, off, filter_mask=fm)
        stable = [i for i, o in enumerate(outcomes) if len(o) == 1]
        assert len(stable) >= 15
        for i in stable:
            assert got[i].tobytes() in outcomes[i], (i, got[i][got[i] >= 0])
        for i, p in enumerate(sc["prompts"]):
            assert bool(has[i]) == bool(p["keys"])
        keys, koff = ix.hash_keys(tok, off)
        for i, p in enumerate(sc["prompts"]):
            assert [int(k) for k in keys[koff[i]:koff[i + 1]]] == p["keys"]
    assert dropped > 0


def _random_stream(rng, n_steps, BS, P, NT, docs, model=0):
    ev, hs, tk = [], [], []
    for _ in range(n_steps):
        pod = int(rng.integers(0, P)); tier = int(rng.integers(0, NT))
        d = int(rng.integers(0, len(docs))); nb = len(docs[d]) // BS
        r = np.zeros((), EVENT_DTYPE)
        r["podtier"] = (pod << 4) | tier; r["model"] = model; r["hash_off"] = len(hs)
        if rng.random() < 0.7:
            b0 = int(rng.integers(0, nb)); b1 = int(rng.integers(b0 + 1, nb + 1))
            hashes = [d * 1000 + b for b in range(b0, b1)]
            toks = docs[d][b0 * BS:b1 * BS]
            r["op"] = 0; r["has_parent"] = b0 > 0; r["parent_hash"] = d * 1000 + b0 - 1 if b0 > 0 else 0
            r["tok_off"] = len(tk); r["n_tokens"] = len(toks); r["n_hashes"] = len(hashes)
            tk.extend(toks)
        else:
            hashes = [d * 1000 + int(rng.integers(0, nb)) for _ in range(int(rng.integers(1, 4)))]
            r["op"] = 1; r["n_hashes"] = len(hashes)
        hs.extend(hashes)
        ev.append(r)
    return np.array(ev, EVENT_DTYPE), np.array(hs, np.uint64), np.array(tk, np.uint64).astype(np.uint32)


@pytest.mark.parametrize("seed,BS,path", [(11, 16, "v1"), (12, 16, "rounds"), (13, 4, "v1"), (14, 16, "classes"), (15, 16, "coop")])
def test_random_event_stream_and_queries_vs_cpp_oracle(seed, BS, path, monkeypatch):
    """Differential test on a few thousand events (sequential replay => identical linearisation)."""
    _select_path(monkeypatch, path)
    rng = np.random.default_rng(seed)
    P, NT = 40, 3
    w = (1.0, 0.8, 0.3)
    ix, co = _index_pair(block_size=BS, hash_seed="abc", capacity=1 << 16, pods_per_key=4, tier_weights=w, max_pods=64)
    docs = [rng.integers(0, 128256, size=BS * int(rng.integers(1, 40))).tolist() for _ in range(30)]
    for i in range(10, 30):
        cut = BS * int(rng.integers(1, 6))
        docs[i] = docs[i % 10][:cut] + docs[i]
    ev, hs, tk = _random_stream(rng, 1500, BS, P, NT, docs)
    # apply in chunks of single-pod-ordered batches: chunk = 1 event keeps the global order identical
    for i in range(0, len(ev), 1):
        assert ix.apply_events(ev[i:i + 1], hs, tk)[0] == 0
    assert co.apply_events(ev, hs, tk)[0] == 0
    st = ix.stats()
    assert st["request_keys"] == co.len_request() and st["engine_keys"] == co.len_engine()
    prompts = []
    for q in range(400):
        d = docs[int(rng.integers(0, len(docs)))]
        cut = int(rng.integers(0, len(d) + 1))
        prompts.append(d[:cut] + rng.integers(0, 128256, size=int(rng.integers(0, 40))).tolist())
    tok, off = csr(prompts)
    fm = np.zeros((len(prompts), ix.filter_words), np.uint64)
    for i in range(0, len(prompts), 3):
        fm[i] = filter_mask(rng.choice(P, size=int(rng.integers(1, 8)), replace=False).tolist(), ix.filter_words)
    for f in (None, fm):
        s1, h1 = ix.score_batch(tok, off, filter_mask=f)
        s2, h2, _, _ = co.score_batch(tok, off, filter_mask=f)
        assert np.array_equal(h1, h2)
        assert np.array_equal(s1, s2), np.argwhere(s1 != s2)[:5]
    k1, _ = ix.hash_keys(tok, off)
    k2, _ = co.hash_keys(tok, off)
    assert np.array_equal(k1, k2)
    uk = np.unique(k1)[:500]          # Lookup results are positional; repeated keys are a map quirk in Go (see INTEGRATION.md)
    rc1, pt1, c1 = ix.lookup(0, uk)
    rc2, pt2, c2 = co.lookup(0, uk)
    assert rc1 == rc2 == 0 and np.array_equal(c1, c2)
    for i in range(len(c1)):
        assert np.array_equal(pt1[i, :c1[i]], pt2[i, :c2[i]])


def test_batched_events_per_pod_order_vs_oracle():
    """One big kvidx_apply_events call.  Documents are disjoint per pod group so that every schedule
    the reference allows gives the same final state; result must equal the oracle's."""
    rng = np.random.default_rng(21)
    BS, P = 16, 64
    ix, co = _index_pair(block_size=BS, capacity=1 << 16, max_pods=64)
    docs = [rng.integers(0, 128256, size=BS * int(rng.integers(2, 30))).tolist() for _ in range(64)]
    evs, hss, tks = [], [], []
    ho = to = 0
    for pod in range(P):                       # pod p only touches document p: no cross-pod races
        e, h, t = _random_stream(rng, 60, BS, 1, 2, [docs[pod]])
        e["podtier"] = (pod << 4) | (e["podtier"] & 15)
        e["hash_off"] += ho; e["tok_off"] += to
        e["parent_hash"] += np.uint64(pod) * np.uint64(1 << 32); h = h + np.uint64(pod) * np.uint64(1 << 32)
        ho += len(h); to += len(t)
        evs.append(e); hss.append(h); tks.append(t)
    # interleave pods round-robin to scramble arrival order across pods (per-pod order kept)
    ev = np.stack(evs, axis=1).reshape(-1)
    hs, tk = np.concatenate(hss), np.concatenate(tks)
    rc, d1 = ix.apply_events(ev, hs, tk)
    rc2, d2 = co.apply_events(ev, hs, tk)
    assert rc == rc2 == 0 and d1 == d2
    st = ix.stats()
    assert st["request_keys"] == co.len_request() and st["engine_keys"] == co.len_engine()
    tok, off = csr([d[:BS * int(rng.integers(0, len(d) // BS + 1))] for d in docs])
    s1, _ = ix.score_batch(tok, off)
    s2, _, _, _ = co.score_batch(tok, off)
    assert np.array_equal(s1, s2)


@pytest.mark.parametrize("kernel", PATHS)
def test_synth_config2_shape_vs_oracle_and_closed_form(kernel, monkeypatch):
    """BASELINE config #2 shape at reduced size (2K-token prompts, 64 pods): fill through the write path,
    then scores bit-exact vs the C++ oracle and vs the generator's closed form."""
    _select_path(monkeypatch, kernel)
    wl = synth.Workload(2, 2048, 1 << 15, 64)
    ix, co = _index_pair(capacity=1 << 16, max_pods=64)
    ev, hs, tk = wl.fill_events(0, wl.D)
    rc, d = ix.apply_events(ev, hs, tk)
    assert rc == 0 and d == 0
    assert co.apply_events(ev, hs, tk) == (0, 0)
    st = ix.stats()
    assert st["request_keys"] == wl.n_blocks == co.len_request()
    toks, doc, m = wl.queries(0, 1000)
    off = np.arange(0, (len(toks) + 1) * wl.T, wl.T, dtype=np.int64)
    s1, h1 = ix.score_batch(toks.reshape(-1), off)
    s2, h2, _, _ = co.score_batch(toks.reshape(-1), off, n_threads=4)
    assert np.array_equal(s1, s2) and h1.all()
    assert np.array_equal(s1, wl.expected_scores(doc, m))


def test_config2_at_its_stated_size():
    """BASELINE config #2 as stated: 1 K prompts x 2 K tokens against a 1 M-block / 64-pod index, bit-exact vs the C++ oracle
    (and vs the generator's closed form).  The default dispatch takes it (1000 prompts: the cooperative kernel)."""
    wl = synth.Workload(2, 2048, 1 << 20, 64)
    ix, co = _index_pair(capacity=(1 << 20) + 4096, max_pods=64)
    for d0 in range(0, wl.D, 2048):
        ev, hs, tk = wl.fill_events(d0, min(wl.D, d0 + 2048))
        assert ix.apply_events(ev, hs, tk) == (0, 0) and co.apply_events(ev, hs, tk) == (0, 0)
    assert ix.stats()["request_keys"] == wl.n_blocks == co.len_request() == 1 << 20
    toks, doc, m = wl.queries(0, 1000)
    off = np.arange(0, (len(toks) + 1) * wl.T, wl.T, dtype=np.int64)
    s1, h1 = ix.score_batch(toks.reshape(-1), off)
    s2, h2, _, _ = co.score_batch(toks.reshape(-1), off, n_threads=4)
    assert np.array_equal(s1, s2) and h1.all() and np.array_equal(s1, wl.expected_scores(doc, m))
    k1, _ = ix.hash_keys(toks[:50].reshape(-1), off[:51])
    k2, _ = co.hash_keys(toks[:50].reshape(-1), off[:51])
    assert np.array_equal(k1, k2)


@pytest.mark.parametrize("kernel", ["coop", "rounds2", "classes", "classes8"])
def test_synth_config3_shape_long_prompts(kernel, monkeypatch):
    """BASELINE config #3 shape at reduced N: 8192-token prompts (512 blocks = 16 rounds), 256 pods."""
    _select_path(monkeypatch, kernel)
    wl = synth.Workload(3, 8192, 1 << 16, 256)
    ix, co = _index_pair(capacity=1 << 17, max_pods=256)
    ev, hs, tk = wl.fill_events(0, wl.D)
    assert ix.apply_events(ev, hs, tk) == (0, 0) and co.apply_events(ev, hs, tk) == (0, 0)
    toks, doc, m = wl.queries(0, 700)
    off = np.arange(0, (len(toks) + 1) * wl.T, wl.T, dtype=np.int64)
    s1, h1 = ix.score_batch(toks.reshape(-1), off)
    s2, h2, _, _ = co.score_batch(toks.reshape(-1), off, n_threads=4)
    assert np.array_equal(s1, s2) and h1.all()
    assert np.array_equal(s1, wl.expected_scores(doc, m))
    assert m.max() > 480                                   # some walks go through (nearly) all 16 rounds


@pytest.mark.parametrize("kernel", ["v1", "coop"] + ROUND_PATHS)
def test_ragged_misaligned_and_many_prompts(kernel, monkeypatch):
    """Round lists, unaligned prompt starts (per-lane staging fallback), empty and sub-block
    prompts, pod filters, against the oracle."""
    _select_path(monkeypatch, kernel)
    rng = np.random.default_rng(31)
    wl = synth.Workload(9, 512, 1 << 13, 32)
    ix, co = _index_pair(capacity=1 << 14, max_pods=32)
    ev, hs, tk = wl.fill_events(0, wl.D)
    assert ix.apply_events(ev, hs, tk)[0] == 0 and co.apply_events(ev, hs, tk)[0] == 0
    toks, doc, m = wl.queries(0, 6000)
    prompts = []
    for i in range(len(toks)):
        L = int(rng.integers(0, wl.T + 1)) if i % 2 else wl.T
        if i % 7 == 0:
            L = int(rng.integers(0, 20))
        prompts.append(toks[i, :L])
    tok, off = csr(prompts)
    s_t, h_t = ix.score_batch(tok, off)
    s_o, h_o, _, _ = co.score_batch(tok, off, n_threads=4)
    assert np.array_equal(h_t, h_o) and np.array_equal(s_t, s_o), np.argwhere(s_t != s_o)[:5]
    assert (np.diff(off) % 4 != 0).any()        # some prompt starts are not 16-byte aligned
    fm = np.zeros((len(prompts), ix.filter_words), np.uint64)
    for i in range(0, len(prompts), 2):
        fm[i] = filter_mask(rng.choice(32, size=int(rng.integers(1, 6)), replace=False).tolist(), ix.filter_words)
    s_t, _ = ix.score_batch(tok, off, filter_mask=fm)
    s_o, _, _, _ = co.score_batch(tok, off, filter_mask=fm, n_threads=4)
    assert np.array_equal(s_t, s_o), np.argwhere(s_t != s_o)[:5]
    sp_p, sp_s, sp_c, _ = ix.score_batch_sparse(tok, off, filter_mask=fm)
    for i in range(0, len(prompts), 97):
        got = {int(sp_p[i, j]): float(sp_s[i, j]) for j in range(sp_c[i])}
        assert got == {int(q): float(s_o[i, q]) for q in np.nonzero(s_o[i] >= 0)[0]}


@pytest.mark.parametrize("kernel", ["coop"] + ROUND_PATHS)
def test_rounds_prefix_sharing_heavy_overlap(kernel, monkeypatch):
    """The round pipeline lets a prompt reuse another prompt's keys when chain state and the next 32-block chunk are
    identical.  Few documents, thousands of prompts: exact duplicates, prefixes of every length (so the shared chunk is
    shorter than the leader's), divergence at every position inside a chunk, unaligned starts, per-prompt models and
    filters.  Everything bit-exact against the oracle."""
    _select_path(monkeypatch, kernel)
    rng = np.random.default_rng(77)
    BS, T, ND = 16, 2048 + 160, 6                       # 138 blocks: four full rounds and a 10-block one
    docs = rng.integers(0, 50000, size=(ND, T), dtype=np.uint32)
    # documents 3..5 start like document 0 (37, 70 and 5 blocks) and then go their own -- indexed -- way: prompts on them
    # leave the popular prefix in the middle of a chunk and keep hitting
    for d, nshare in ((3, 37), (4, 70), (5, 5)):
        docs[d, : nshare * BS] = docs[0, : nshare * BS]
    ix, co = _index_pair(capacity=1 << 12, max_pods=16)
    for d in range(ND):
        keys = ix.hash_keys(docs[d], np.array([0, T], np.int64))[0]
        nb = len(keys) if d % 2 == 0 else int(rng.integers(20, len(keys)))      # some documents only partly cached
        for pod in rng.choice(16, size=3, replace=False):
            pt = [(int(pod) << 4) | int(rng.integers(0, 2))]
            eng = (keys[:nb] ^ np.uint64(0x5555)).astype(np.uint64)
            assert ix.add(0, eng, keys[:nb], pt) == 0
            co.add(0, eng, keys[:nb], pt)
    prompts = []
    for i in range(4000):
        d = docs[int(rng.integers(0, ND)) if i % 3 else 0]          # document 0 is the popular one
        kind = i % 5
        if kind == 0:
            pr = d.copy()                                                        # exact duplicate of a document
        elif kind == 1:
            pr = d[: int(rng.integers(0, T + 1))].copy()                         # a prefix, any length
        elif kind == 2:
            pr = d.copy(); pr[int(rng.integers(0, T)):] = rng.integers(0, 50000)  # diverges somewhere
        elif kind == 3:
            pr = d.copy(); pr[int(rng.integers(0, T))] ^= np.uint32(1)            # single-token difference
        else:
            pr = np.concatenate([d[: BS * int(rng.integers(0, T // BS))], rng.integers(0, 50000, size=int(rng.integers(0, 700)), dtype=np.uint32)])
        prompts.append(pr.astype(np.uint32))
    tok, off = csr(prompts)
    assert (off[:-1] % 4 != 0).any()
    s_t, h_t = ix.score_batch(tok, off)
    s_o, h_o, _, _ = co.score_batch(tok, off, n_threads=4)
    assert np.array_equal(h_t, h_o) and np.array_equal(s_t, s_o), np.argwhere(s_t != s_o)[:5]
    assert (s_o.max(axis=1) >= 128).any()               # some walks go through every round
    fm = np.zeros((len(prompts), ix.filter_words), np.uint64)
    for i in range(0, len(prompts), 3):
        fm[i] = filter_mask(rng.choice(16, size=int(rng.integers(1, 4)), replace=False).tolist(), ix.filter_words)
    s_t, _ = ix.score_batch(tok, off, filter_mask=fm)
    s_o, _, _, _ = co.score_batch(tok, off, filter_mask=fm, n_threads=4)
    assert np.array_equal(s_t, s_o), np.argwhere(s_t != s_o)[:5]


@pytest.mark.parametrize("kernel", ["rounds2", "classes", "classes8", "classes-whole", "classes4-nosort"])
def test_prefix_tree_workload(kernel, monkeypatch):
    """Prompts drawn from a random prefix TREE (conversations forking off shared history at arbitrary token positions,
    several levels deep), every branch cached on its own pods up to a random depth.  Prompts leave popular prefixes in
    the middle of a chunk and keep hitting along less popular -- or private -- branches, which drives the class pipeline
    through partial followers, capped solo walks, unaligned chunk starts and class re-formation.  Bit-exact vs the oracle."""
    _select_path(monkeypatch, kernel)
    rng = np.random.default_rng(2024)
    BS, P = 16, 48
    ix, co = _index_pair(capacity=1 << 15, max_pods=P)
    paths = [rng.integers(0, 60000, size=3000, dtype=np.uint32)]
    for level in range(4):
        for _ in range(12):
            parent = paths[int(rng.integers(0, len(paths)))]
            cut = int(rng.integers(1, len(parent)))                      # any token position, not block aligned
            paths.append(np.concatenate([parent[:cut], rng.integers(0, 60000, size=int(rng.integers(200, 2500)), dtype=np.uint32)]))
    for pth in paths:
        keys = ix.hash_keys(pth, np.array([0, len(pth)], np.int64))[0]
        if len(keys) == 0:
            continue
        for pod in rng.choice(P, size=int(rng.integers(1, 4)), replace=False):
            nb = int(rng.integers(1, len(keys) + 1))                     # cached up to a random depth on this pod
            pt = [(int(pod) << 4) | int(rng.integers(0, 2))]
            eng = (keys[:nb] ^ np.uint64(0xABCD)).astype(np.uint64)
            assert ix.add(0, eng, keys[:nb], pt) == 0
            co.add(0, eng, keys[:nb], pt)
    prompts = []
    for i in range(9000):
        pth = paths[int(rng.integers(0, len(paths))) if i % 4 else 0]
        cut = int(rng.integers(0, len(pth) + 1))
        tail = rng.integers(0, 60000, size=int(rng.integers(0, 300)), dtype=np.uint32) if i % 3 else np.zeros(0, np.uint32)
        prompts.append(np.concatenate([pth[:cut], tail]).astype(np.uint32))
    tok, off = csr(prompts)
    s_t, h_t = ix.score_batch(tok, off)
    s_o, h_o, _, _ = co.score_batch(tok, off, n_threads=4)
    assert np.array_equal(h_t, h_o) and np.array_equal(s_t, s_o), np.argwhere(s_t != s_o)[:5]
    assert (s_o.max(axis=1) > 100).sum() > 100
    sp_p, sp_s, sp_c, _ = ix.score_batch_sparse(tok, off)
    for i in range(0, len(prompts), 211):
        got = {int(sp_p[i, j]): float(sp_s[i, j]) for j in range(sp_c[i])}
        assert got == {int(q): float(s_o[i, q]) for q in np.nonzero(s_o[i] >= 0)[0]}


@pytest.mark.parametrize("kernel", ["classes", "classes8", "rounds2", "coop"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_tiny_alphabet_fuzz(kernel, seed, monkeypatch):
    """Prompts over a two-letter alphabet: every pair of prompts shares a prefix of some random length, chunks coincide in
    all sorts of partial ways, lengths are ragged, duplicates abound -- and about half of all short chains are cached.
    Plus the degenerate batch sizes (1, 5, 33 prompts).  Bit-exact vs the oracle."""
    _select_path(monkeypatch, kernel)
    rng = np.random.default_rng(900 + seed)
    BS, P = 16, 24
    ix, co = _index_pair(capacity=1 << 15, max_pods=P)
    base = [rng.integers(0, 2, size=int(rng.integers(BS, 1400)), dtype=np.uint32) * 7 for _ in range(40)]
    # long runs of equal blocks make distinct prompts agree for a while and then part ways
    for b in base:
        b[: BS * int(rng.integers(0, 30))] = 0
    for b in base[:25]:
        keys = ix.hash_keys(b, np.array([0, len(b)], np.int64))[0]
        if len(keys) == 0:
            continue
        nb = int(rng.integers(1, len(keys) + 1))
        pt = [(int(rng.integers(0, P)) << 4) | int(rng.integers(0, 2)) for _ in range(int(rng.integers(1, 4)))]
        eng = (keys[:nb] ^ np.uint64(0x77)).astype(np.uint64)
        assert ix.add(0, eng, keys[:nb], pt) == 0
        co.add(0, eng, keys[:nb], pt)
    prompts = []
    for i in range(5000):
        b = base[int(rng.integers(0, len(base)))]
        pr = b[: int(rng.integers(0, len(b) + 1))].copy()
        if i % 4 == 0 and len(pr):
            pr[int(rng.integers(0, len(pr))):] = 7                      # a different tail from some position on
        prompts.append(pr)
    for n in (len(prompts), 1, 5, 33):
        tok, off = csr(prompts[:n])
        s_t, h_t = ix.score_batch(tok, off)
        s_o, h_o, _, _ = co.score_batch(tok, off, n_threads=4)
        assert np.array_equal(h_t, h_o) and np.array_equal(s_t, s_o), (n, np.argwhere(s_t != s_o)[:5])
    same = [base[0]] * 3000                                             # one prompt, three thousand times
    tok, off = csr(same)
    s_t, _ = ix.score_batch(tok, off)
    s_o, _, _, _ = co.score_batch(tok, off, n_threads=4)
    assert np.array_equal(s_t, s_o) and (s_t == s_t[0]).all()


def test_automatic_fallback_by_sharing(monkeypatch, capfd):
    """A large batch goes to the class pipeline only if it repeats itself: the sorted first-block fingerprints are counted
    first.  Unique prompts: per-prompt rounds.  The same prompts repeated 16 times: classes.  Results identical either way."""
    _select_path(monkeypatch, "auto")
    monkeypatch.setenv("KVIDX_ROUNDS_TRACE", "2")
    wl = synth.Workload(9, 512, 1 << 13, 32)
    ix, co = _index_pair(capacity=1 << 14, max_pods=32)
    ev, hs, tk = wl.fill_events(0, wl.D)
    assert ix.apply_events(ev, hs, tk)[0] == 0 and co.apply_events(ev, hs, tk)[0] == 0
    rng = np.random.default_rng(3)
    uniq = [rng.integers(0, 50000, size=512, dtype=np.uint32) for _ in range(600)]
    for batch, fell_back in ((uniq, True), (uniq[:40] * 16, False)):
        tok, off = csr(batch)
        capfd.readouterr()
        s_t, _ = ix.score_batch(tok, off)
        err = capfd.readouterr().err
        assert ("per-prompt rounds instead" in err) == fell_back, err
        s_o, _, _, _ = co.score_batch(tok, off, n_threads=4)
        assert np.array_equal(s_t, s_o)


def test_round_scratch_grows_and_shrinks_through_both_pipelines(monkeypatch, capfd):
    """One handle scores batches that grow and shrink while they alternate between the class pipeline and the per-prompt
    rounds (directly, or handed over by the class pipeline after its setup), so both pipelines carve their scratch from
    the same arena as it grows and is reused at smaller sizes.  Bit-exact vs the oracle every time."""
    _select_path(monkeypatch, "auto")
    monkeypatch.setenv("KVIDX_ROUNDS_TRACE", "2")
    wl = synth.Workload(10, 512, 1 << 17, 32)                # 4096 documents of 32 blocks
    ix, co = _index_pair(capacity=1 << 18, max_pods=32)
    ev, hs, tk = wl.fill_events(0, wl.D)
    assert ix.apply_events(ev, hs, tk)[0] == 0 and co.apply_events(ev, hs, tk)[0] == 0
    toks, doc, _ = wl.queries(0, 20000)
    few = np.concatenate([toks[doc < 16]] * 80)              # prompts on 16 documents: the class pipeline keeps them
    many = toks                                              # on all 4096: too few share their first block, handed over
    for batch, handed_over in ((few[:300], False), (many[:3000], True), (few[:5000], False), (many[:40], False),
                               (few[:700], False), (many[:1500], True)):
        off = np.arange(0, (len(batch) + 1) * wl.T, wl.T, dtype=np.int64)
        capfd.readouterr()
        s_t, h_t = ix.score_batch(batch.reshape(-1), off)
        err = capfd.readouterr().err
        assert ("per-prompt rounds instead" in err) == handed_over, (len(batch), err)
        s_o, h_o, _, _ = co.score_batch(batch.reshape(-1), off, n_threads=4)
        assert np.array_equal(h_t, h_o) and np.array_equal(s_t, s_o), (len(batch), np.argwhere(s_t != s_o)[:5])
        assert (s_o.max(axis=1) > 0).any()


def test_config5_scores_while_the_write_path_runs():
    """BASELINE config #5 in miniature: one thread keeps storing and removing documents through apply_events while another
    scores prompts of documents the writer never touches.  Reads and writes on one handle do not serialise (they take
    different host locks and run on different streams): a Score() may run while an event batch is being applied.  The
    untouched documents' scores must be exact in every call, and the final index must equal the oracle's after the same
    event sequence.  Reads of keys the writer changes are checked in tests/test_gpu_reads_beside_writes.py."""
    import threading
    wl = synth.Workload(5, 1024, 1 << 14, 32)
    ix, co = _index_pair(capacity=1 << 16, max_pods=32)
    ev, hs, tk = wl.fill_events(0, wl.D)
    assert ix.apply_events(ev, hs, tk) == (0, 0) and co.apply_events(ev, hs, tk) == (0, 0)
    toks, doc, m = wl.queries(0, 3000)
    off = np.arange(0, (len(toks) + 1) * wl.T, wl.T, dtype=np.int64)
    want = wl.expected_scores(doc, m)
    churn = []
    for s_i in range(12):
        e, h, t = wl.fill_events(wl.D + 8 * s_i, wl.D + 8 * (s_i + 1))
        r = e.copy(); r["op"] = 1; r["has_parent"] = 0; r["n_tokens"] = 0
        churn.append((e, r, h, t))
    errs = []

    def writer():
        try:
            for i, (e, r, h, t) in enumerate(churn):
                assert ix.apply_events(e, h, t) == (0, 0)
                if i % 3 != 2:                              # every third batch stays
                    assert ix.apply_events(r, h, t)[0] == 0
        except Exception as ex:                             # noqa: BLE001
            errs.append(ex)

    th = threading.Thread(target=writer)
    th.start()
    for _ in range(6):
        s1, _ = ix.score_batch(toks.reshape(-1), off)
        if not np.array_equal(s1, want):
            errs.append(AssertionError("scores changed while events were applied"))
    th.join()
    assert not errs, errs[:1]
    for i, (e, r, h, t) in enumerate(churn):
        co.apply_events(e, h, t)
        if i % 3 != 2:
            co.apply_events(r, h, t)
    assert ix.stats()["request_keys"] == co.len_request()
    q2, d2, m2 = wl.queries(5000, 5400)
    kept = np.concatenate([wl.doc_tokens(wl.D + 8 * i, wl.D + 8 * (i + 1)) for i in range(12) if i % 3 == 2])
    tok2 = np.concatenate([q2.reshape(-1), kept.reshape(-1)])
    off2 = np.arange(0, (len(q2) + len(kept) + 1) * wl.T, wl.T, dtype=np.int64)
    a, _ = ix.score_batch(tok2, off2)
    b, _, _, _ = co.score_batch(tok2, off2, n_threads=4)
    assert np.array_equal(a, b) and (b[len(q2):].max(axis=1) > 0).all()


def test_rebuild_after_tombstones():
    ix = kvidx.Index(capacity=2048, table_slots=4096)
    co = COracle(size=10 ** 6)
    rng = np.random.default_rng(3)
    live = {}
    for rnd in range(12):
        eng = rng.integers(1, 1 << 62, 600, dtype=np.uint64)
        req = rng.integers(1, 1 << 62, 600, dtype=np.uint64)
        assert ix.add(0, eng, req, [PT(1)]) == 0 and co.add(0, eng, req, [PT(1)]) == 0
        for e in eng[:550]:
            assert ix.evict(0, int(e), [PT(1)]) == 0 and co.evict(0, int(e), [PT(1)]) == 0
        for e, r in zip(eng[550:], req[550:]):
            live[int(e)] = int(r)
    st = ix.stats()
    assert st["rebuilds"] >= 1 and st["request_keys"] == len(live) == co.len_request()
    keys = np.array(list(live.values()), np.uint64)
    rc, pt, cnt = ix.lookup(0, keys)
    assert rc == 0 and (cnt == 1).all() and (pt[:, 0] == PT(1)).all()
    for e, r in list(live.items())[:50]:
        assert ix.get_request_key(0, e) == (0, r)


# ---- exact key-LRU mode (InMemoryIndexConfig.Size) --------------------------------------------------------------
def test_index_size_cap_exact_lru():
    """pkg/kvcache/kvblock/in_memory_test.go:44-83: Size=2, the third Add evicts the first key; the lookup still returns
    the other two (a missing first key does not cut)."""
    ix = kvidx.Index(capacity=2, pods_per_key=1, lru_exact=1)
    assert ix.add(0, [72735753], [79215516], [PT(1)]) == 0
    assert ix.add(0, [41341092], [12871930], [PT(2)]) == 0
    assert ix.add(0, [34012886], [69914638], [PT(3, 1)]) == 0
    rc, pt, cnt = ix.lookup(0, [79215516, 12871930, 69914638])
    assert rc == 0 and cnt.tolist() == [0, 1, 1] and pt[1, 0] == PT(2) and pt[2, 0] == PT(3, 1)
    assert ix.stats()["request_keys"] == 2 and ix.stats()["engine_keys"] == 2
    # Lookup refreshes recency (in_memory.go:118): touch key2, add a fourth key -> key3 is now the oldest and goes
    assert ix.lookup(0, [12871930])[0] == 0
    assert ix.add(0, [555], [777], [PT(4)]) == 0
    rc, pt, cnt = ix.lookup(0, [12871930, 69914638, 777])
    assert cnt.tolist() == [1, 0, 1]


def test_exact_lru_random_stream_vs_oracle():
    """Size-capped index under a random single-block event stream with lookups and Score() calls in between (both refresh
    recency in the reference).  Score() calls of several prompts that share documents, and lookups that repeat keys: the
    last touch of a key in the call's order (prompt after prompt, key after key) decides its recency."""
    rng = np.random.default_rng(41)
    BS, P, CAP = 16, 12, 40
    ix = kvidx.Index(block_size=BS, capacity=CAP, pods_per_key=3, max_pods=16, lru_exact=1)
    co = COracle(block_size=BS, size=CAP, pod_cache_size=3, max_pods=16)
    docs = [rng.integers(0, 128256, size=BS * int(rng.integers(2, 9))).tolist() for _ in range(14)]
    for step in range(700):
        pod = int(rng.integers(0, P)); tier = int(rng.integers(0, 2))
        d = int(rng.integers(0, len(docs))); nb = len(docs[d]) // BS
        b = int(rng.integers(0, nb))
        r = np.zeros(1, EVENT_DTYPE)
        r["podtier"] = (pod << 4) | tier
        if rng.random() < 0.7:
            r["op"] = 0; r["has_parent"] = b > 0; r["parent_hash"] = d * 1000 + b - 1 if b > 0 else 0
            r["n_hashes"] = 1; r["n_tokens"] = BS
            hs = np.array([d * 1000 + b], np.uint64); tk = np.array(docs[d][b * BS:(b + 1) * BS], np.uint32)
        else:
            r["op"] = 1; r["n_hashes"] = 1
            hs = np.array([d * 1000 + b], np.uint64); tk = np.zeros(0, np.uint32)
        assert ix.apply_events(r, hs, tk)[0] == 0 and co.apply_events(r, hs, tk)[0] == 0
        if step % 5 == 4:
            qs = []
            for _ in range(int(rng.integers(1, 5))):
                q = docs[int(rng.integers(0, 4))]                 # a few documents: the prompts of one call overlap
                qs.append(q[:BS * int(rng.integers(0, len(q) // BS + 1))] + rng.integers(0, 128256, size=int(rng.integers(0, 20))).tolist())
            tok, off = csr(qs)
            s1, h1 = ix.score_batch(tok, off)
            s2, h2, _, _ = co.score_batch(tok, off)
            assert np.array_equal(s1, s2) and np.array_equal(h1, h2), step
        if step % 7 == 6:
            d2 = docs[int(rng.integers(0, len(docs)))]
            keys, _ = co.hash_keys(np.array(d2, np.uint32), [0, len(d2)])
            uk = np.concatenate([keys, keys[::-2], keys[:1]])      # repeated keys: the last position touches last
            r1 = ix.lookup(0, uk); r2 = co.lookup(0, uk)
            assert np.array_equal(r1[2], r2[2]), step
            for i in range(len(uk)):
                assert np.array_equal(r1[1][i, :r1[2][i]], r2[1][i, :r2[2][i]])
        st = ix.stats()
        assert st["request_keys"] == co.len_request() and st["engine_keys"] == co.len_engine(), step
    assert ix.stats()["request_keys"] <= CAP
