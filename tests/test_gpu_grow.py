"""GPU (-m gpu): growable tables (kvidx_config_t.grow_tables, include/kvidx.h).  A growable handle starts small; before a
write batch with S slots, L live keys (the larger map's) and I incoming, it rehashes both tables in one step into
min(C, pow2ceil(4 (L + I))) slots when S < C and 4 (L + I) > S, where C = pow2ceil(max(4 capacity, 1024)) is what a fixed
handle with table_slots 0 allocates.

  1. create: initial sizes, ceilings, the refused configurations, and a handle that starts at C and never grows;
  2. the rule: slot counts after kvidx_add calls of chosen sizes, one rebuild for a call that spans several doublings,
     none under add / evict churn;
  3. default mode: a handle grown from 1024 slots and a fixed handle of C slots, fed one seeded stream of every write call
     (add, evict, apply_events, apply_events_dev, apply_event_payloads, remove_pods, restore into fresh handles) through
     at least six growths, give byte-equal images and read results on every forced Score() path after every call;
  4. exact LRU with a capacity below the stream's keys: images with their recency section and eviction counts equal;
  5. CLOCK: victim by victim against the sequential hand model, with the growth step added;
  6. restore: one step to the rule's size, the fixed handle's state, KVIDX_ENOSPC beyond 90 % of C at the initial size,
     and the exact-LRU cut of an image above capacity;
  7. readers beside a writer whose handles grow under them, on every Score() path;
  8. the host mirror, growable against fixed, filled through kvhost_pool_process.

A growth whose allocation fails (the call then goes on in the old tables under the fixed-size rules) is not exercised
here: it would take exhausting the device's memory."""
import numpy as np
import pytest

import kvidx
import snapshot_oracle as so
import write_stream as ws
from clock_hand_oracle import ClockHandle, ClockMap
from helpers import _select_path, free_pairs, keys_homed_at
from history_oracle import Checker, Window
from oracle import kvoracle as ko
from oracle.kvoracle_c import COracle
from test_gpu_clock_hand import Rig
from test_gpu_event_payloads import encode_batch
from test_gpu_reads_beside_writes import (FILLER, GROUPS, KINDS, Reads, Until, Work, Writer, _check_scores, _evidence_ok,
                                          _handle, _quiescent, _race, _score_reader)
from test_gpu_text_store_scale import _text_of

pytestmark = pytest.mark.gpu

BS, P = 16, 16
W = (1.0, 0.8)
NAMES = ["gpu", "cpu"]
EMIX = np.uint64(0x5BD1E9955BD1E995)       # engine hash = request key ^ EMIX


def PT(p, t=0):
    return (p << 4) | t


def pow2ceil(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def ceiling(capacity):
    """C: the slot count a fixed handle with table_slots 0 allocates, and the most a growable one grows to."""
    return pow2ceil(max(4 * capacity, 1024))


def grown(S, C, live, incoming):
    """The growth rule: the slot count a write call's room check leaves."""
    if S >= C or 4 * (live + incoming) <= S:
        return S
    return min(C, pow2ceil(4 * (live + incoming)))


def slots(ix):
    st = ix.stats()
    assert st["request_slots"] == st["engine_slots"]
    return st["request_slots"]


def live(ix):
    st = ix.stats()
    return max(st["request_keys"], st["engine_keys"])


def header_counts(img):
    R, E = np.frombuffer(img, "<u8", 2, 32)
    return int(R), int(E)


def new_keys(rng, n):
    return np.unique(rng.integers(1, 1 << 64, n + 16, dtype=np.uint64))[:n]


# ---- 1. create -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("capacity", [1, 200, 1000, 5000, 100_000, 1 << 18, 600_000])
def test_initial_size_and_ceiling(capacity):
    C = ceiling(capacity)
    assert slots(kvidx.Index(capacity=capacity)) == C                        # fixed: unchanged
    assert slots(kvidx.Index(capacity=capacity, grow_tables=True)) == min(C, 1 << 20)
    for ts in sorted(t for t in {1, 1000, 1024, 1025, max(C // 2, 1), C} if t <= C):
        assert slots(kvidx.Index(capacity=capacity, table_slots=ts, grow_tables=True)) == max(1024, pow2ceil(ts))


def test_refused_configurations():
    C = ceiling(5000)
    for kw in (dict(table_slots=C + 1), dict(shard_count=2), dict(grow_tables=2), dict(grow_tables=0xFFFFFFFF)):
        cfg = dict(capacity=5000, grow_tables=True)
        cfg.update(kw)
        with pytest.raises(kvidx.KvidxError) as e:
            kvidx.Index(**cfg)
        assert e.value.code == kvidx.EINVAL, kw
    assert slots(kvidx.Index(capacity=5000, table_slots=C + 1)) == 2 * C    # a fixed handle still takes any table_slots


def test_a_handle_that_starts_at_its_ceiling_never_grows():
    """table_slots == C: every call runs under the fixed handle's rules, up to the same KVIDX_ENOSPC."""
    C = ceiling(5000)
    g, f = kvidx.Index(capacity=5000, table_slots=C, grow_tables=True), kvidx.Index(capacity=5000)
    rng = np.random.default_rng(1)
    for n in (1000, 3000, 7000, 12000):
        k = new_keys(rng, n)
        for ix in (g, f):
            assert ix.add(0, k ^ EMIX, k, [PT(1)]) == 0
    k = new_keys(rng, 7000)                                                  # 23 000 + 7 000 > 90 % of 32 768
    for ix in (g, f):
        assert ix.add(0, k ^ EMIX, k, [PT(1)]) == kvidx.ENOSPC
        assert "growing" not in ix.last_error()
    assert g.snapshot() == f.snapshot()
    assert slots(g) == C and g.stats()["rebuilds"] == 0


# ---- 2. the rule -----------------------------------------------------------------------------------------------------
def test_growth_rule_after_every_add():
    cap = 100_000
    C = ceiling(cap)
    ix = kvidx.Index(capacity=cap, table_slots=1024, grow_tables=True)
    rng = np.random.default_rng(2)
    S, n_live, rb = 1024, 0, 0
    for n in (10, 200, 46, 1, 300, 700, 1000, 50, 5000, 20000, 1, 30000, 40000, 15000):
        k = new_keys(rng, n)
        assert ix.add(0, k ^ EMIX, k, [PT(1)]) == 0
        want = grown(S, C, n_live, n)
        rb += want != S
        S, n_live = want, n_live + n
        st = ix.stats()
        assert (st["request_slots"], st["engine_slots"], st["rebuilds"], st["request_keys"], st["engine_keys"]) == (S, S, rb, n_live, n_live)
    assert S == C


def test_one_call_spanning_several_doublings_grows_once():
    ix = kvidx.Index(capacity=100_000, table_slots=1024, grow_tables=True)
    k = new_keys(np.random.default_rng(3), 20000)
    assert ix.add(0, k ^ EMIX, k, [PT(1)]) == 0
    st = ix.stats()
    assert st["request_slots"] == 131072 and st["rebuilds"] == 1               # 1024 -> 131 072: seven doublings, one rehash


def test_churn_never_grows_the_tables():
    """100 rounds of add / evict of the same 200 keys: tombstones pile up and are compacted at the same size."""
    ix = kvidx.Index(capacity=100_000, table_slots=1024, grow_tables=True)
    k = new_keys(np.random.default_rng(4), 200)
    for _ in range(100):
        assert ix.add(0, k ^ EMIX, k, [PT(1), PT(2, 1)]) == 0
        assert slots(ix) == 1024
        for x in k[:4]:
            assert ix.evict(0, int(x ^ EMIX), [PT(1), PT(2, 1)]) == 0
        ix.remove_pods([1, 2])
        st = ix.stats()
        assert st["request_keys"] == 0 and st["request_slots"] == 1024
    assert ix.stats()["rebuilds"] > 0                                        # compactions, not growths


# ---- 3. / 4. a growable handle against the fixed one, one stream ------------------------------------------------------
class Corpus:
    """Documents of two models: tokens, request keys (engine hash = key ^ EMIX) and text (4 bytes a token)."""

    def __init__(self, seed, n_docs=800, max_blocks=120):
        rng = np.random.default_rng(seed)
        self.docs = [rng.integers(0, 1 << 31, BS * int(rng.integers(8, max_blocks + 1))).astype(np.uint32) for _ in range(n_docs)]
        self.model = [d % 2 for d in range(n_docs)]
        off = np.zeros(n_docs + 1, np.int64)
        off[1:] = np.cumsum([len(t) for t in self.docs])
        keys, koff = COracle(block_size=BS).hash_keys(np.concatenate(self.docs), off)
        self.keys = [keys[koff[i]:koff[i + 1]] for i in range(n_docs)]
        self.text = [_text_of(t) for t in self.docs]
        spans = [np.stack([np.arange(len(t)) * 4, np.arange(len(t)) * 4 + 4], axis=1).astype(np.uint64) for t in self.docs]
        t, o = kvidx.pack_text(self.text)
        self.store = (t, o, np.concatenate(self.docs), np.concatenate(spans), off)


class Queries:
    """One fixed set of reads: prompts (tokens, keys, a conversation split, text), Lookup keys and engine keys."""

    def __init__(self, cp, seed, n=256):
        rng = np.random.default_rng(seed)
        d = rng.integers(0, len(cp.docs), n)
        nb = np.array([int(rng.integers(1, len(cp.keys[i]) + 1)) for i in d])
        tail = rng.integers(0, BS, n)
        held = np.array([int(rng.integers(0, b + 1)) for b in nb])
        self.model = np.array([cp.model[i] for i in d], np.uint32)
        self.fm = np.zeros((n, 1), np.uint64)
        for i in range(n):
            if rng.random() < 0.25:
                self.fm[i, 0] = np.uint64(int(rng.integers(1, 1 << P)))
        toks = [cp.docs[i][:BS * b + t] for i, b, t in zip(d, nb, tail)]
        self.tok, self.off = np.concatenate(toks), np.concatenate([[0], np.cumsum([len(t) for t in toks])]).astype(np.int64)
        ks = [cp.keys[i][:b] for i, b in zip(d, nb)]
        self.keys, self.koff = np.concatenate(ks), np.concatenate([[0], np.cumsum([len(k) for k in ks])]).astype(np.int64)
        hk = [cp.keys[i][:h] for i, h in zip(d, held)]
        nt = [cp.docs[i][BS * h:BS * b + t] for i, h, b, t in zip(d, held, nb, tail)]
        self.turn = (np.concatenate(hk), np.concatenate([[0], np.cumsum([len(k) for k in hk])]).astype(np.int64),
                     np.concatenate(nt), np.concatenate([[0], np.cumsum([len(t) for t in nt])]).astype(np.int64))
        self.text, self.toff = kvidx.pack_text([cp.text[i][:4 * (BS * b + t)] for i, b, t in zip(d, nb, tail)])
        self.lookups = []
        for m in (0, 1):
            docs = [i for i in rng.integers(0, len(cp.docs), 40) if cp.model[i] == m]
            self.lookups.append((m, np.concatenate([cp.keys[i] for i in docs])[:1500]))
        # engine keys under their own model and under the other one (absent), some of them never stored
        self.engines = [(cp.model[i] ^ other, int(x ^ EMIX)) for i in rng.integers(0, len(cp.docs), 24) for x in cp.keys[i][:4]
                        for other in (0, 1)] + [(0, int(x)) for x in rng.integers(1, 1 << 63, 8)]


class Pair:
    """A growable handle from 1024 slots and a fixed handle of C slots, made alike (the Score() path knobs and the prefix
    store included), so that every read can be compared between the two."""

    def __init__(self, monkeypatch, path, capacity, cp=None, **kw):
        self.mp, self.path, self.capacity, self.cp, self.kw = monkeypatch, path, capacity, cp, kw
        self.C = ceiling(capacity)
        self.g, self.f = self.make(True), self.make(False)

    def make(self, grow):
        cfg = dict(block_size=BS, capacity=self.capacity, max_pods=P, tier_weights=W, **self.kw)
        if grow:
            cfg.update(table_slots=1024, grow_tables=True)
        with self.mp.context() as mp:
            if self.path:
                _select_path(mp, self.path)
            ix = kvidx.Index(**cfg)
        if self.cp is not None:
            ix.text_store_init(1 << 20, 64)
            ix.text_store_add(*self.cp.store)
        return ix

    def both(self):
        return (self.g, self.f)


def _rows_equal(a, b):
    return all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(a, b))


def _pairs_equal(a, b):
    """Rows of (pairs (n, 10), ..., counts (n,), ...) as sparse Score() and Lookup return them: positions past a row's count
    are not part of the result."""
    (pa, sa, ca), (pb, sb, cb) = a, b
    keep = np.arange(pa.shape[1])[None, :] < ca[:, None]
    return ca.tobytes() == cb.tobytes() and pa[keep].tobytes() == pb[keep].tobytes() and (sa is None or sa[keep].tobytes() == sb[keep].tobytes())


def check_pairs(pairs, q, lru=False):
    """After a call: every handle's image is the same bytes; every pair's Score() rows are; the full pair's other reads are."""
    img = pairs[0].g.snapshot()
    for p in pairs:
        for ix in p.both():
            assert ix.snapshot() == img
        if lru:
            assert p.g.evictions() == p.f.evictions()
        g, f = (ix.score_batch(q.tok, q.off, model=q.model, filter_mask=q.fm) for ix in p.both())
        assert _rows_equal(g, f), "dense rows differ on path %s" % p.path
        g, f = (ix.score_batch_sparse(q.tok, q.off, model=q.model, filter_mask=q.fm) for ix in p.both())
        assert _pairs_equal(g[:3], f[:3]) and _rows_equal(g[3:], f[3:]), "sparse rows differ on path %s" % p.path
        if p.cp is None:
            continue
        g, f = (ix.score_keys(q.keys, q.koff, model=q.model, filter_mask=q.fm) for ix in p.both())
        assert _rows_equal(g, f)
        g, f = (ix.score_turn(*q.turn, model=q.model, filter_mask=q.fm) for ix in p.both())
        assert _rows_equal(g, f)
        g, f = (ix.score_text(q.text, q.toff, model=q.model, filter_mask=q.fm, min_ratio=0.0) for ix in p.both())
        assert _rows_equal(g, f)
        for m, keys in q.lookups:
            g, f = (ix.lookup(m, keys) for ix in p.both())
            assert g[0] == f[0] == 0 and _pairs_equal((g[1], None, g[2]), (f[1], None, f[2]))
        g, f = (ix.lookup_hits(q.tok, q.off, model=q.model, filter_mask=q.fm) for ix in p.both())
        assert _rows_equal([g], [f])
        for m, e in q.engines:
            assert p.g.get_request_key(m, e) == p.f.get_request_key(m, e)
        g, f = (ix.pod_inventory(engine=True) for ix in p.both())
        assert all(np.array_equal(g[k], f[k]) for k in g)


class Stream:
    """A seeded stream of write calls over a corpus, sized from the keys the handles hold: each batch adds about 30-70 %
    more, so that the growable handle passes every doubling on its way to C."""

    OPS = ["add", "events", "evict", "events_dev", "add", "payloads", "remove_pods", "add", "events_dev", "payloads"]

    def __init__(self, cp, seed):
        self.cp, self.rng = cp, np.random.default_rng(seed)
        self.keep = []

    def _runs(self, n, model=None):
        """Runs [a, b) of distinct documents (of one model, if given) holding about n blocks in all: [(doc, a, b)].  In an
        event batch each document then belongs to one pod, so no key's entry order depends on how the per-pod queues
        interleave, and both handles must agree byte for byte."""
        out, got = [], 0
        for d in self.rng.permutation(len(self.cp.docs)):
            d = int(d)
            if got >= n:
                break
            if model is not None and self.cp.model[d] != model:
                continue
            k = len(self.cp.keys[d])
            a = 0 if self.rng.random() < 0.5 else int(self.rng.integers(0, k))
            b = min(k, a + n - got)
            out.append((d, a, b))
            got += b - a
        return out

    def _pts(self):
        return [PT(int(p), int(self.rng.integers(0, 2))) for p in self.rng.choice(np.arange(1, P), int(self.rng.integers(1, 3)), replace=False)]

    def _events(self, n):
        """BlockStored runs under their parents (pods 1..P-1, both tiers), a few of their blocks removed after them."""
        evs = []
        for d, a, b in self._runs(n):
            pod, tier, m = int(self.rng.integers(1, P)), int(self.rng.integers(0, 2)), self.cp.model[d]
            k = self.cp.keys[d]
            parent = int(k[a - 1] ^ EMIX) if a > 0 else None
            evs.append(ws.Ev(ws.STORED, pod, tier, m, parent, k[a:b] ^ EMIX, self.cp.docs[d][BS * a:BS * b], "store"))
            if self.rng.random() < 0.3:
                rm = self.rng.choice(k[a:b], min(3, b - a), replace=False) ^ EMIX
                evs.append(ws.Ev(ws.REMOVED, pod, tier, m, None, rm, [], "remove"))
        return evs

    def next_call(self, i, n_live):
        """-> (kind, fn(ix) applying the call to a handle)."""
        kind = self.OPS[i % len(self.OPS)]
        n = max(64, int(n_live * self.rng.uniform(0.3, 0.7)))
        if kind == "add":
            m = int(self.rng.integers(0, 2))
            k = np.concatenate([self.cp.keys[d][a:b] for d, a, b in self._runs(n, m)])
            pts = self._pts()
            return kind, lambda ix: ix.add(m, k ^ EMIX, k, pts) == 0
        if kind == "evict":
            calls = [(self.cp.model[d], int(self.cp.keys[d][a] ^ EMIX), self._pts()) for d, a, _ in self._runs(24)]
            return kind, lambda ix: all(ix.evict(*c) == 0 for c in calls)
        if kind == "remove_pods":
            pods = [int(p) for p in self.rng.choice(np.arange(1, P), 2, replace=False)]
            return kind, lambda ix: ix.remove_pods(pods) is not None
        evs = self._events(n)
        if kind == "events":
            ev, hs, tk = ws.pack(evs)
            return kind, lambda ix: ix.apply_events(ev, hs, tk) == (0, 0)
        if kind == "payloads":
            msgs = encode_batch(evs, NAMES, self.rng)
            raw, pods, models = [m[0] for m in msgs], [m[1] for m in msgs], [m[2] for m in msgs]
            return kind, lambda ix: ix.apply_event_payloads(raw, pods, models, NAMES, 0)[:2] == (0, 0)
        ev, hs, tk = ws.pack(evs)                                 # events_dev: sorted by pod, one queue per pod
        order = np.argsort(ev["podtier"] >> 4, kind="stable")
        ev = ev[order]
        _, cnt = np.unique(ev["podtier"] >> 4, return_counts=True)
        qoff = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        return kind, lambda ix: self._dev(ix, ev, qoff, hs, tk)

    def _dev(self, ix, ev, qoff, hs, tk):
        import torch
        dev = torch.device("cuda", 0)
        b = [torch.from_numpy(ev.view(np.uint8).copy()).to(dev), torch.from_numpy(qoff).to(dev),
             torch.from_numpy(hs.view(np.int64).copy()).to(dev), torch.from_numpy(np.concatenate([tk, np.zeros(1, np.uint32)]).view(np.int32)).to(dev)]
        torch.cuda.synchronize()
        ix.apply_events_dev(b[0].data_ptr(), b[1].data_ptr(), len(qoff) - 1, len(ev), b[2].data_ptr(), len(hs), b[3].data_ptr())
        ix.synchronize()
        return True


def run_stream(pairs, cp, seed, min_growths, restore_at, lru=False, min_calls=0):
    """Feed one stream to every handle of `pairs`, comparing after every call, with a restore into fresh handles at
    call `restore_at`, until the first growable handle has grown `min_growths` times and reached C (and for at least
    `min_calls` calls).  -> (growths, the
    reads)."""
    q = Queries(cp, seed + 1)
    st = Stream(cp, seed)
    growths, i = 0, 0
    while growths < min_growths or slots(pairs[0].g) < pairs[0].C or i <= max(restore_at, min_calls):
        assert i < 200, "the stream did not grow the tables %d times up to C (%d, %d slots)" % (min_growths, growths, slots(pairs[0].g))
        if i == restore_at:
            img = pairs[0].g.snapshot()
            R, E = header_counts(img)
            for p in pairs:
                g, f = p.make(True), p.make(False)
                assert g.restore(img) == f.restore(img)
                assert slots(g) == grown(1024, p.C, 0, max(R, E)) and g.stats()["rebuilds"] == (slots(g) > 1024)
                p.g, p.f = g, f
            check_pairs(pairs, q, lru)
        kind, fn = st.next_call(i, live(pairs[0].g))
        s0 = slots(pairs[0].g)
        for p in pairs:
            for ix in p.both():
                assert fn(ix), (kind, ix.last_error())
        growths += slots(pairs[0].g) > s0
        for p in pairs:
            assert slots(p.f) == p.C and slots(p.g) == slots(pairs[0].g)
        check_pairs(pairs, q, lru)
        i += 1
    return growths, q


def test_default_mode_grown_equals_fixed(monkeypatch):
    cp = Corpus(5)
    pairs = [Pair(monkeypatch, None, 32768, cp)] + [Pair(monkeypatch, path, 32768) for path in ("v1", "coop", "rounds", "classes")]
    growths, q = run_stream(pairs, cp, 50, min_growths=6, restore_at=12)
    assert growths >= 6 and slots(pairs[0].g) == ceiling(32768)
    # the oracle, directly: the grown handle's rows are the reference scorer's over its own image
    g = pairs[0].g
    oix = so.decode(g.snapshot(), [0, 1], list(range(P)), list(range(16)), max_pods=P)[0]
    sc = ko.LongestPrefixScorer(dict(enumerate(W)))
    rows, has = g.score_batch(q.tok, q.off, model=q.model, filter_mask=q.fm)
    for i in range(len(q.off) - 1):
        want = np.full(P, -1.0)
        filt = [p for p in range(P) if int(q.fm[i, 0]) >> p & 1]
        keys = [ko.Key(int(q.model[i]), int(k)) for k in q.keys[q.koff[i]:q.koff[i + 1]]]
        for p, v in sc.score(keys, oix.lookup(keys, filt)).items():
            want[p] = v
        assert np.array_equal(rows[i], want), i


def test_exact_lru_grown_equals_fixed(monkeypatch):
    """capacity 6000 below the stream's keys: every write call evicts the least recent keys while the tables grow."""
    cp = Corpus(6, n_docs=300)
    pair = Pair(monkeypatch, None, 6000, cp, lru_exact=1)
    growths, _ = run_stream([pair], cp, 60, min_growths=4, restore_at=9, lru=True, min_calls=40)
    assert growths >= 4 and slots(pair.g) == ceiling(6000)
    assert pair.g.evictions()[0] > 0


# ---- 5. CLOCK ---------------------------------------------------------------------------------------------------------
class GrowClockHandle(ClockHandle):
    """The hand model with the growth step: before a call's room check, both maps are re-homed into the rule's size
    (tombstones dropped, every key's bit kept, both hands at slot 0)."""

    def __init__(self, S, C, capacity, pods_per_key=10):
        super().__init__(S, capacity, pods_per_key)
        self.C = C

    def room(self, incoming):
        S = grown(self.req.S, self.C, max(self.req.live, self.eng.live), incoming)
        if S != self.req.S:
            self.grow(S)
        super().room(incoming)

    def grow(self, S):
        for name in ("req", "eng"):
            old, new = getattr(self, name), ClockMap(S)
            for i in sorted(old.where.values()):
                new.ref[new.insert(old.at[i][0])] = bool(old.ref[i])
            setattr(self, name, new)
        self.rebuilds += 1


class GrowRig(Rig):
    """test_gpu_clock_hand's rig on a growable CLOCK handle from 1024 slots.  New keys are drawn on fully EMPTY home
    pairs of the layout their call inserts them into (the model runs the call's room check first), so no two live keys
    share a home pair in that layout or in any larger one."""

    def __init__(self, capacity, seed):
        self.rng = np.random.default_rng(seed)
        self.ix = kvidx.Index(block_size=BS, capacity=capacity, table_slots=1024, pods_per_key=4, max_pods=8,
                              evict_policy="clock", grow_tables=True)
        self.m = GrowClockHandle(1024, ceiling(capacity), capacity, pods_per_key=4)

    @property
    def S(self):
        return self.m.req.S

    def new_pairs(self, n):
        self.m.room(n)
        self.roomy(n)
        rs = self.rng.choice(free_pairs(self.m.req.state), n, replace=False)
        es = self.rng.choice(free_pairs(self.m.eng.state), n, replace=False)
        return keys_homed_at(es, 0, self.S, self.rng), keys_homed_at(rs, 0, self.S, self.rng)

    def add_new(self, n):
        e, r = self.new_pairs(n)
        self.add(e, r, (PT(int(self.rng.integers(0, 8))),))
        assert slots(self.ix) == self.S
        return e, r


def test_clock_victims_through_growths():
    """capacity 1500 (C = 8192): the sweeps evict while the tables grow 1024 -> 2048 -> 4096 -> 8192, with Lookup,
    GetRequestKey and Evict marking keys between the calls."""
    rig = GrowRig(1500, 7)
    sizes, engines = [rig.S], []
    for step in range(40):
        n = int(rig.rng.integers(20, 400))
        e, r = rig.add_new(n)
        engines.extend(int(x) for x in e[:4])
        if rig.S != sizes[-1]:
            sizes.append(rig.S)
        live_req = [k[1] for k in rig.m.req.where]
        rig.lookup(live_req[i] for i in rig.rng.choice(len(live_req), min(len(live_req), 200), replace=False))
        rig.get_request_key(engines[-8:])
        if step % 5 == 4:
            for x in engines[-3:]:
                rig.evict(x, [PT(int(rig.rng.integers(0, 8)))])
    assert len(sizes) >= 3 and sizes[0] == 1024 and sizes[-1] == 8192, sizes
    assert rig.ix.evictions()[0] > 0 and rig.ix.sweeps()[0] > 0


# ---- 6. restore -------------------------------------------------------------------------------------------------------
def _filled(capacity, n, seed, **kw):
    ix = kvidx.Index(block_size=BS, capacity=capacity, max_pods=P, **kw)
    rng = np.random.default_rng(seed)
    for part in np.array_split(new_keys(rng, n), 8):
        assert ix.add(int(rng.integers(0, 2)), part ^ EMIX, part, [PT(int(rng.integers(0, P)), int(rng.integers(0, 2)))]) == 0
    return ix


def test_restore_grows_once_to_the_rule():
    img = _filled(1 << 16, 5000, 8).snapshot()
    C = ceiling(32768)
    g = kvidx.Index(block_size=BS, capacity=32768, max_pods=P, table_slots=1024, grow_tables=True)
    f = kvidx.Index(block_size=BS, capacity=32768, max_pods=P)
    assert g.restore(img) == f.restore(img) == {"request_keys": 5000, "engine_keys": 5000}
    st = g.stats()
    assert st["request_slots"] == grown(1024, C, 0, 5000) == 32768 and st["rebuilds"] == 1
    assert g.snapshot() == f.snapshot() == img
    q = Queries(Corpus(9, n_docs=40), 9, n=64)
    keys, hits = np.frombuffer(img, "<u8", 5000, 64)[::4].copy(), 0
    for k0 in (0, 1):
        (rg, pg, cg), (rf, pf, cf) = g.lookup(k0, keys), f.lookup(k0, keys)
        assert rg == rf == 0 and _pairs_equal((pg, None, cg), (pf, None, cf))
        hits += int((cg > 0).sum())
    assert hits == len(keys)
    assert _rows_equal(g.score_batch(q.tok, q.off, model=q.model), f.score_batch(q.tok, q.off, model=q.model))


def test_restore_beyond_the_ceiling_is_refused_at_the_initial_size():
    img = _filled(1 << 14, 4000, 10).snapshot()                            # 4000 > 90 % of C = 4096
    g = kvidx.Index(block_size=BS, capacity=1000, max_pods=P, table_slots=1024, grow_tables=True)
    f = kvidx.Index(block_size=BS, capacity=1000, max_pods=P)
    for ix in (g, f):
        with pytest.raises(kvidx.KvidxError) as e:
            ix.restore(img)
        assert e.value.code == kvidx.ENOSPC
    st = g.stats()
    assert (st["request_keys"], st["engine_keys"], st["request_slots"], st["rebuilds"]) == (0, 0, 1024, 0)
    bad = bytearray(_filled(1 << 14, 900, 11).snapshot())                 # fits, but malformed: refused at the old size too
    bad[64 + 11] = 1                                                       # request record 0's padding byte
    with pytest.raises(kvidx.KvidxError) as e:
        g.restore(bytes(bad))
    assert e.value.code == kvidx.EINVAL and slots(g) == 1024 and g.stats()["rebuilds"] == 0


def test_restore_exact_lru_image_above_capacity():
    img = _filled(8000, 8000, 12, lru_exact=1).snapshot()
    g = kvidx.Index(block_size=BS, capacity=3000, max_pods=P, table_slots=1024, grow_tables=True, lru_exact=1)
    f = kvidx.Index(block_size=BS, capacity=3000, max_pods=P, lru_exact=1)
    assert g.restore(img) == f.restore(img) == {"request_keys": 3000, "engine_keys": 3000}
    assert g.snapshot() == f.snapshot()
    assert g.evictions() == f.evictions()
    assert slots(g) == grown(1024, ceiling(3000), 0, 8000) == 16384


# ---- 7. readers beside a growing writer ----------------------------------------------------------------------------------
class GrowWriter(Writer):
    """The reads-beside-writes writer with the filler op changed: it adds keys of the filler pod in batches that double,
    `first` x 1, 2, 4, 8, 16, and nothing removes them, so each of those grows the handles' tables; later filler ops add
    64 keys.  grew[h]: the op indices (positions in ops[h]) of the ops that grew handle h; overlapped[h]: those a read of
    the handle overlapped (filled in by the readers' UntilGrown)."""

    def __init__(self, *a, first=16000, **kw):
        super().__init__(*a, **kw)
        self.first, self.n_fill = first, 0
        self.grew = [set() for _ in self.handles]
        self.overlapped = [set() for _ in self.handles]

    def next_op(self):
        kind, args = super().next_op()
        if kind == "filler":
            ks = self.rng.integers(1, 1 << 63, self.first << self.n_fill if self.n_fill < 5 else 64, dtype=np.uint64)
            self.n_fill += 1
            args = (int(self.rng.integers(0, 2)), ks ^ EMIX, ks, [PT(FILLER)])
        return kind, args

    def _apply(self, h, ix, kind, args):
        s0 = slots(ix)
        super()._apply(h, ix, kind, args)
        if slots(ix) > s0:
            self.grew[h].add(len(self.ops[h]))


class UntilGrown(Until):
    """Until, and on until reads of handle h (this reader's or another's) have overlapped `growths` growths."""

    def __init__(self, writer, h, calls, kinds, growths=3, cap=2000):
        super().__init__(writer, h, calls, kinds, rebuild=True, cap=cap)
        self.growths = growths

    def more(self):
        return self.k < self.cap and (super().more() or len(self.writer.overlapped[self.h]) < self.growths)

    def saw(self, s, e):
        super().saw(s, e)
        ops = self.writer.ops[self.h]
        for i in list(self.writer.grew[self.h]):
            if i < len(ops) and ops[i][0] < e and ops[i][1] > s:
                self.writer.overlapped[self.h].add(i)


GROW_KINDS = ["add", "evict", "apply_events", "add", "apply_events_dev", "evict", "remove_pods", "add", "hot", "filler"]


def _grown_under_reads(writer, reads, n_handles, at_least=3):
    for h in range(n_handles):
        seen = set()
        for _, hh, s, e, _ in reads.calls:
            if hh == h:
                seen |= set(Window(writer.op_times(h), s, e).overlapped()) & writer.grew[h]
        assert len(seen) >= at_least, "handle %d: reads overlapped %d growths (%d in all)" % (h, len(seen), len(writer.grew[h]))


def _growable(work, monkeypatch=None, path=None):
    ix = _handle(work, monkeypatch, path, capacity=1 << 19, table_slots=1024, grow_tables=True)
    assert slots(ix) > 1024                                                # the fill grew it already
    return ix


@pytest.mark.parametrize("group", range(4))
def test_every_score_path_beside_a_growing_writer(group, monkeypatch):
    paths = GROUPS[group]
    work = Work(81 + group)
    handles = [_growable(work, monkeypatch, p) for p in paths]
    writer = GrowWriter(work, handles, np.random.default_rng(group + 40), GROW_KINDS)
    reads = Reads()
    readers = [_score_reader(work, ix, h, reads, np.random.default_rng(200 + h), 4096, UntilGrown(writer, h, 3, KINDS))
               for h, ix in enumerate(handles)]
    _race(work, writer, readers, 60)
    hist = writer.history(work)
    evidence = {}
    _check_scores(work, writer, hist, reads, Checker(hist, (1.0, 0.8, 1 / 3, 0.1)), evidence)
    _evidence_ok(evidence, len(handles), KINDS)
    _grown_under_reads(writer, reads, len(handles))
    _quiescent(work, hist, handles)


# ---- 8. the host mirror ----------------------------------------------------------------------------------------------
def test_host_mirror_grown_equals_fixed():
    from kvidx.host import HostIndexer
    cap = 1 << 15
    g = HostIndexer(block_size=BS, capacity=cap, grow_tables=True, table_slots=1024, enable_metrics=True)
    f = HostIndexer(block_size=BS, capacity=cap, enable_metrics=True)
    gi = kvidx.Index.borrow(g.L.kvhost_index(g.h), block_size=BS)
    stream = ws.WriteStream(np.random.default_rng(21), BS, pods=tuple(range(6)), models=2, tiers=2, max_blocks=120, docs_per_pod=12)
    rng = np.random.default_rng(22)
    sizes = [slots(gi)]
    for n_events in (8, 16, 40, 60, 120, 200, 400, 900, 1800):
        msgs = encode_batch(stream.batch(n_events), NAMES, rng)
        for h in (g, f):
            for payload, pod, model in msgs:
                assert h.add_task("pod%d" % pod, "m%d" % model, payload) >= 0
            assert h.process()[0] >= 0
        if slots(gi) != sizes[-1]:
            sizes.append(slots(gi))
    assert len(sizes) >= 4, sizes
    docs = [d for d in stream.docs if len(d)][:300]
    tok = np.concatenate([d.blocks.reshape(-1) for d in docs])
    off = np.concatenate([[0], np.cumsum([d.blocks.size for d in docs])]).astype(np.int64)
    for model in ("m0", "m1"):
        assert g.get_pod_scores_batch(tok, off, model) == f.get_pod_scores_batch(tok, off, model)
    mg, mf = g.metrics(), f.metrics()
    for k in ("lookup_latency_bucket", "lookup_latency_count", "lookup_latency_sum"):
        mg.pop(k), mf.pop(k)
    assert mg == mf
    img = f.snapshot()
    assert g.snapshot() == img
    r = HostIndexer(block_size=BS, capacity=cap, grow_tables=True, table_slots=1024)
    r.restore(img)
    assert r.snapshot() == img
    assert slots(kvidx.Index.borrow(r.L.kvhost_index(r.h), block_size=BS)) > 1024
