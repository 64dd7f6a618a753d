"""CPU: the history oracle of tests/history_oracle.py, which checks reads that run beside writes
(tests/test_gpu_reads_beside_writes.py).  It must accept every row that some interleaving of the writer's operations
produces, and reject the wrong rows a broken read path would return: a torn slot, a state that ended before the call,
a state that began after it, a score summed in another order, a duplicated entry, a pod that no block-0 state holds.
Without these, the GPU test could pass whatever the readers return."""
import numpy as np
import pytest

from helpers import EVENT_DTYPE, SNAP_REQ_DTYPE
from history_oracle import Checker, History, Window
from oracle import kvoracle as ko
from oracle.kvoracle_c import COracle

B = 4
W = (1.0, 0.8, 1 / 3, 0.1)
ANCHOR = 0 << 4


def PT(p, t=0):
    return (p << 4) | t


def _image_states(co):
    """{(model, hash): entry tuple} of a C++ oracle's image (an independent replay of the same op log)."""
    img = co.snapshot()
    R = int(np.frombuffer(img, "<u8", 1, 32)[0])
    req = np.frombuffer(img, SNAP_REQ_DTYPE, R, 64)
    return {(int(r["model"]), int(r["hash"])): tuple(int(x) for x in r["ent"][:r["count"]]) for r in req}


class _Log:
    """A random writer log over a few documents, replayed on the History and on a C++ oracle whose image is kept after
    every op (the instants between ops).  Op i has the fake interval [10 i + 1, 10 i + 9]."""

    def __init__(self, seed, n_ops=60):
        rng = np.random.default_rng(seed)
        self.co = COracle(block_size=B, tier_weights=W, max_pods=16)
        self.hist = History(COracle(block_size=B, tier_weights=W, max_pods=16))
        self.docs = [rng.integers(0, 1000, B * int(rng.integers(3, 9))).astype(np.uint32) for _ in range(6)]
        self.docs[3][:2 * B] = self.docs[0][:2 * B]                          # a shared prefix
        self.keys = [self.co.hash_keys(d, [0, len(d)])[0] for d in self.docs]
        self.model = [d % 2 for d in range(len(self.docs))]
        self.images = []

        def run(op, *a):
            getattr(self.hist, op)(*a)
            getattr(self.co, op)(*a)
            self.images.append(_image_states(self.co))

        self.images.append(_image_states(self.co))
        for d, k in enumerate(self.keys):                                    # the anchor on every block
            run("add", self.model[d], k ^ np.uint64(0x77), k, [ANCHOR])
        for _ in range(n_ops):
            d = int(rng.integers(0, len(self.docs)))
            k, m = self.keys[d], self.model[d]
            a = int(rng.integers(0, len(k)))
            b = int(rng.integers(a + 1, len(k) + 1))
            pod = int(rng.integers(1, 6))
            kind = int(rng.integers(0, 4))
            if kind == 0:
                run("add", m, k[a:b] ^ np.uint64(0x77), k[a:b], [PT(pod, pod % 4)] + ([PT(1, 3)] if pod == 1 else []))
            elif kind == 1:
                run("evict", m, int(k[a] ^ np.uint64(0x77)), [PT(pod, pod % 4)])
            elif kind == 2:                                                  # one pod's batch: store a run, remove a block
                ev = np.zeros(2, EVENT_DTYPE)
                ev["podtier"] = PT(pod, pod % 4)
                ev["model"] = m
                ev[0]["op"], ev[0]["n_hashes"], ev[0]["n_tokens"] = 0, b - a, B * (b - a)
                ev[0]["has_parent"], ev[0]["parent_hash"] = a > 0, int(k[a - 1] ^ np.uint64(0x77)) if a > 0 else 0
                ev[0]["tok_off"] = B * a
                ev[1]["op"], ev[1]["n_hashes"], ev[1]["hash_off"] = 1, 1, b - a
                hs = np.concatenate([k[a:b] ^ np.uint64(0x77), [k[b - 1] ^ np.uint64(0x77) if rng.random() < 0.5 else k[a] ^ np.uint64(0x77)]]).astype(np.uint64)
                self.hist.apply_events(ev, hs, self.docs[d])
                assert self.co.apply_events(ev, hs, self.docs[d]) == (0, 0)
                self.images.append(_image_states(self.co))
            else:
                run("remove_pods", [pod]) if hasattr(self.co, "remove_pods") else self._remove(pod)
        self.times = np.array([[10 * i + 1, 10 * i + 9] for i in range(self.hist.n_ops)], np.int64)

    def _remove(self, pod):
        """The C++ oracle has no removal: its twin is rebuilt from the image with the pod's entries dropped."""
        self.hist.remove_pods([pod])
        st = {key: tuple(e for e in ents if e >> 4 != pod) for key, ents in _image_states(self.co).items()}
        # replay the survivors into a fresh C++ oracle (entry order and engine mappings as before)
        fresh = COracle(block_size=B, tier_weights=W, max_pods=16)
        for d, k in enumerate(self.keys):
            for j, rk in enumerate(k):
                ents = st.get((self.model[d], int(rk)), ())
                if ents:
                    assert fresh.add(self.model[d], [int(rk ^ np.uint64(0x77))], [int(rk)], list(ents)) == 0
        self.co = fresh
        self.images.append(_image_states(self.co))

    def window(self, a, b):
        """A read that starts inside op a and ends inside op b (a <= b)."""
        return Window(self.times, 10 * a + 5, 10 * b + 5)

    def row_at(self, d, nb, instants, filt=None):
        """The row the reference scorer gives prompt (doc d, first nb blocks) when block j is read at the instant after
        instants[j] ops (the oracle's own states, one instant per block)."""
        keys = self.keys[d][:nb]
        kp = {}
        for j, k in enumerate(keys):
            ents = self.images[instants[j]].get((self.model[d], int(k)), ())
            ents = [e for e in ents if filt is None or e >> 4 in filt]
            if ents:
                kp[ko.Key(self.model[d], int(k))] = [ko.PodEntry(e >> 4, e & 15) for e in ents]
        got = ko.LongestPrefixScorer(dict(enumerate(W))).score([ko.Key(self.model[d], int(k)) for k in keys], kp)
        row = np.full(16, -1.0)
        for p, s in got.items():
            row[p] = s
        return row, int(nb > 0)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_accepts_rows_of_every_interleaving(seed):
    """Rows scored from the oracle's own states, each block read at its own random instant inside the call, and lookup
    rows at random instants, are all admissible."""
    lg = _Log(seed)
    ck = Checker(lg.hist, W)
    rng = np.random.default_rng(seed + 100)
    n = lg.hist.n_ops
    contested = 0
    for _ in range(300):
        a = int(rng.integers(0, n))
        b = int(rng.integers(a, min(n, a + 6)))
        w = lg.window(a, b)
        d = int(rng.integers(0, len(lg.docs)))
        nb = int(rng.integers(0, len(lg.keys[d]) + 1))
        filt = None if rng.random() < 0.7 else {0, 1, 2}
        # block j read after `inst` ops: anywhere from the state current at s (a ops done) to b + 1 ops done
        inst = rng.integers(a, b + 2, size=max(nb, 1))
        row, has = lg.row_at(d, nb, inst, filt)
        sets = ck.score_sets(lg.model[d], lg.keys[d][:nb], w, filt)
        assert ck.row_ok(row, has, sets) is None, (ck.row_ok(row, has, sets), a, b, d, nb)
        i = int(rng.integers(a, b + 2))
        keys = lg.keys[d]
        pt = np.zeros((len(keys), 10), np.uint16)
        cnt = np.zeros(len(keys), np.uint8)
        for j, k in enumerate(keys):
            ents = lg.images[i].get((lg.model[d], int(k)), ())
            pt[j, :len(ents)], cnt[j] = ents, len(ents)
            contested += len(lg.hist.req_states((lg.model[d], int(k)), w)) > 1
        assert ck.lookup_ok(lg.model[d], keys, pt, cnt, w) is None
    assert contested > 0


def _contested(lg, rng):
    """(window, doc, block, admissible states) of a key with at least two admissible states."""
    n = lg.hist.n_ops
    for _ in range(10000):
        a = int(rng.integers(len(lg.docs), n - 1))
        w = lg.window(a, a)
        d = int(rng.integers(0, len(lg.docs)))
        j = int(rng.integers(0, len(lg.keys[d])))
        st = lg.hist.req_states((lg.model[d], int(lg.keys[d][j])), w)
        if len(st) >= 2 and all(s is not None and len(s) >= 2 for s in st):
            return w, d, j, sorted(st)
    raise AssertionError("no contested key")


def _lookup_row(lg, d, j, ents):
    pt = np.zeros((1, 10), np.uint16)
    pt[0, :len(ents)] = ents
    return [lg.keys[d][j]], pt, np.array([len(ents)], np.uint8)


def test_rejects_a_torn_slot():
    lg = _Log(5)
    ck = Checker(lg.hist, W)
    rng = np.random.default_rng(1)
    rejected = 0
    for _ in range(40):
        w, d, j, st = _contested(lg, rng)
        s0, s1 = st[0], st[1]
        for cut in range(1, max(len(s0), len(s1))):
            torn = s0[:cut] + s1[cut:]                       # half of one image, half of the other
            if torn in st or not torn:
                continue
            assert ck.lookup_ok(lg.model[d], *_lookup_row(lg, d, j, torn), w) is not None, (st, torn)
            rejected += 1
    assert rejected > 0


def test_rejects_states_from_outside_the_call():
    """A state that ended before s (replaced by an op that finished before the call) and one that began after e (produced
    by an op that started after the call returned) are both rejected in lookup rows, and in score rows where they change
    what some pod can score."""
    lg = _Log(6, n_ops=80)
    ck = Checker(lg.hist, W)
    n = lg.hist.n_ops
    looked, scored = {"stale": 0, "future": 0}, {"stale": 0, "future": 0}
    for a in range(len(lg.docs) + 2, n - 2):
        w = lg.window(a, a)                                     # the call overlaps op a only
        for d in range(len(lg.docs)):
            sets = ck.score_sets(lg.model[d], lg.keys[d], w)
            for j, k in enumerate(lg.keys[d]):
                key = (lg.model[d], int(k))
                adm = lg.hist.req_states(key, w)
                for st, kind in ((lg.images[a - 1].get(key), "stale"), (lg.images[a + 2].get(key), "future")):
                    if st is None or st in adm:
                        continue
                    assert ck.lookup_ok(lg.model[d], *_lookup_row(lg, d, j, st), w) is not None
                    looked[kind] += 1
                    # that state at block j of the document's prompt, every other block read after op a
                    img = dict(lg.images[a + 1])
                    img[key] = st
                    lg.images.append(img)
                    inst = np.full(len(lg.keys[d]), a + 1)
                    inst[j] = len(lg.images) - 1
                    row, has = lg.row_at(d, len(lg.keys[d]), inst)
                    lg.images.pop()
                    scored[kind] += ck.row_ok(row, has, sets) is not None
    assert min(looked.values()) > 0 and min(scored.values()) > 0, (looked, scored)


def test_rejects_a_score_summed_in_another_order():
    """One pod on 1/3, 0.1, 0.1, ... tiers over the blocks: the in-order f64 sum is admissible, the same addends summed
    in another order (which changes the last bit) are not."""
    co = COracle(block_size=B, tier_weights=W, max_pods=16)
    h = History(co)
    rng = np.random.default_rng(3)
    toks = rng.integers(0, 1000, B * 12).astype(np.uint32)
    keys, _ = co.hash_keys(toks, [0, len(toks)])
    tiers = [2, 3, 3, 2, 3, 3, 3, 2, 3, 2, 3, 3]
    for k, t in zip(keys, tiers):
        h.add(0, [int(k) ^ 5], [int(k)], [PT(4, t)])
    ck = Checker(h, W)
    w = Window(np.array([[i, i] for i in range(h.n_ops)]), 10 ** 6, 10 ** 6 + 1)
    sets = ck.score_sets(0, keys, w)
    addends = [W[t] for t in tiers]
    fwd = 0.0
    for x in addends:
        fwd += x
    alt = [0.0, sum(reversed(addends)), float(np.sum(np.array(addends))), (sum(addends[:6]) + sum(addends[6:]))]
    alt = [x for x in alt if x != fwd]
    assert alt, "every order gives the same f64 sum"
    row = np.full(16, -1.0)
    row[4] = fwd
    assert ck.row_ok(row, 1, sets) is None
    for x in alt:
        row[4] = x
        assert ck.row_ok(row, 1, sets) is not None, x


def test_rejects_a_duplicated_entry_and_a_pod_never_in_block_0():
    lg = _Log(7)
    ck = Checker(lg.hist, W)
    rng = np.random.default_rng(2)
    n = lg.hist.n_ops
    for _ in range(50):
        a = int(rng.integers(len(lg.docs), n))
        w = lg.window(a, a)
        d = int(rng.integers(0, len(lg.docs)))
        j = int(rng.integers(0, len(lg.keys[d])))
        st = sorted(lg.hist.req_states((lg.model[d], int(lg.keys[d][j])), w), key=str)
        s = st[0]
        if s is None or len(s) >= 10:
            continue
        assert ck.lookup_ok(lg.model[d], *_lookup_row(lg, d, j, s), w) is None
        assert ck.lookup_ok(lg.model[d], *_lookup_row(lg, d, j, s + (s[-1],)), w) is not None
        assert ck.lookup_ok(lg.model[d], *_lookup_row(lg, d, j, (s[0],) + s), w) is not None
        # score row: a pod that no admissible block-0 state holds (pod 9 is never written)
        row, has = lg.row_at(d, len(lg.keys[d]), np.full(len(lg.keys[d]), a + 1))
        sets = ck.score_sets(lg.model[d], lg.keys[d], w)
        assert ck.row_ok(row, has, sets) is None
        bad = row.copy()
        bad[9] = 1.0
        assert ck.row_ok(bad, has, sets) is not None
        bad = row.copy()
        bad[0] = -1.0                                        # the anchor missing: never admissible
        assert ck.row_ok(bad, has, sets) is not None
        assert ck.row_ok(row, 1 - has, sets) is not None


def test_clock_suffixes_and_engine_mappings():
    """On a CLOCK handle any suffix of an admissible state (oldest entries dropped, the key absent) is admissible, and
    nothing else; get_request_key answers one admissible mapping."""
    co = COracle(block_size=B, tier_weights=W, max_pods=16)
    h = History(co, clock=True)
    h.add(0, [11], [101], [PT(0), PT(1), PT(2)])
    h.add(0, [12], [102], [PT(3)])
    h.remove_pods([3])
    ck = Checker(h, W)
    times = np.array([[10, 20], [30, 40], [50, 60]])
    w = Window(times, 25, 28)
    for s in [(PT(0), PT(1), PT(2)), (PT(1), PT(2)), (PT(2),), ()]:
        assert ck.lookup_ok(0, *_row1(101, s), w) is None, s
    for s in [(PT(0), PT(2)), (PT(0),), (PT(2), PT(1))]:
        assert ck.lookup_ok(0, *_row1(101, s), w) is not None, s
    assert ck.request_key_ok(0, 11, 0, 101, w) is None
    assert ck.request_key_ok(0, 12, -2, 0, w) is None                  # not yet added
    assert ck.request_key_ok(0, 12, 0, 102, w) is not None
    w = Window(times, 45, 55)                                           # during the removal
    assert ck.request_key_ok(0, 12, 0, 102, w) is None and ck.request_key_ok(0, 12, -2, 0, w) is None
    w = Window(times, 61, 70)
    assert ck.request_key_ok(0, 12, 0, 102, w) is not None


def _row1(k, ents):
    pt = np.zeros((1, 10), np.uint16)
    pt[0, :len(ents)] = ents
    return [k], pt, np.array([len(ents)], np.uint8)
