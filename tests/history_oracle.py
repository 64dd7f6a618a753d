"""A history oracle for reads that run beside writes: which rows a read call may return when a writer changes the index
while the call runs.

DESIGN §4 promises that a reader sees each key as it was just before or just after each single Add / Evict / event /
removal, never a half-written slot and never a state older than the call.  `History` replays a writer's operation log on
the reference oracle (oracle/kvoracle.py, removals by tests/remove_oracle.py) and keeps, for every key it touches, the
sequence of entry lists the key held and the operation that produced each (intermediate states of one operation
included, so that no legitimate interleaving is rejected).

A writer's operations run one after another; each has a host-clock interval [t0, t1] (time.monotonic_ns() before the
call and after it returns; an asynchronous batch's interval ends where it is ordered before later reads: at its return
for a read issued afterwards on the same handle, which waits for it).  For a read call with interval [s, e], a key's
admissible states are the state current at s -- the last state of the last operation that ended by s -- and every
state produced by an operation that started before e and ended after s.  The same op log serves several handles:
`Window(times, s, e)` takes one handle's operation intervals.

Rows are checked with a relaxation that is sound (never rejects a legitimate interleaving): each block may take any
admissible state of its key independently, and each pod is checked on its own by a DP over the prompt's blocks that
carries the pod's reachable (alive, score) pairs, adding the pod's max tier weight with an in-order IEEE f64 add as the
scorer does (kvblock_scorer.go:108-151).  On a CLOCK handle a key may lose its oldest entries to the sweep and be
re-added later, so every suffix of an admissible state (the empty one: the key is absent) is admissible too.
"""
import bisect

import numpy as np

from oracle import kvoracle as ko
from remove_oracle import remove_pods as _remove_pods

STORED, REMOVED = 0, 1


def _state(pc):
    """An oracle pod cache -> its entries (pod << 4 | tier) oldest -> newest, or None for an absent key."""
    if pc is None or len(pc) == 0:
        return None
    return tuple((e.pod << 4) | e.tier for e in pc.keys())


class History:
    """Per-key state histories of one writer's operation log, at id level: models, pods and tiers are ints, a request key
    is (model, hash), an entry is pod << 4 | tier.  `co` (oracle.kvoracle_c.COracle of the same block size and seed)
    hashes the block chains of BlockStored events."""

    def __init__(self, co, pods_per_key=10, clock=False):
        self.ix = ko.InMemoryIndex(1 << 40, pods_per_key)
        self.co = co
        self.clock = clock
        self.n_ops = 0
        self.kinds = []                     # op index -> kind name
        self.req = {}                       # (model, hash) -> ([op index], [state])
        self.eng = {}                       # (model, engine hash) -> ([op index], [request hash or None])

    # ---- recording ---------------------------------------------------------------------------------------------------
    def _rec(self, table, key, val):
        ops, vals = table.setdefault(key, ([-1], [None]))
        if vals[-1] != val:
            ops.append(self.n_ops)
            vals.append(val)

    def _rec_req(self, rk):
        self._rec(self.req, (rk.model, rk.chunk_hash), _state(self.ix.data.d.get(rk)))

    def _rec_eng(self, ek):
        rk = self.ix.engine_to_request.d.get(ek)
        self._rec(self.eng, (ek.model, ek.chunk_hash), None if rk is None else rk.chunk_hash)

    def _begin(self, kind):
        self.kinds.append(kind)

    def _end(self):
        self.n_ops += 1

    def _add_pair(self, model, ek, rk, pts):
        """Index.Add of one (engine, request) pair, one entry at a time, recording every state the key passes through."""
        ek, rk = ko.Key(model, int(ek)), ko.Key(model, int(rk))
        for pt in pts:
            self.ix.add([ek], [rk], [ko.PodEntry(int(pt) >> 4, int(pt) & 15)])
            self._rec_req(rk)
        self._rec_eng(ek)

    def _evict(self, model, ek, pts):
        ek = ko.Key(model, int(ek))
        rk = self.ix.engine_to_request.d.get(ek)
        for pt in pts:
            self.ix.evict(ek, [ko.PodEntry(int(pt) >> 4, int(pt) & 15)])
            if rk is not None:
                self._rec_req(rk)
        self._rec_eng(ek)

    # ---- the writer's operations, in the order the writer ran them ---------------------------------------------------
    def add(self, model, engine, request, podtiers):
        self._begin("add")
        for ek, rk in zip(engine, request):
            self._add_pair(model, ek, rk, podtiers)
        self._end()

    def fill(self, calls):
        """One op made of several Add calls (model, engine keys, request keys, podtiers): a handle's fill."""
        self._begin("fill")
        for model, engine, request, podtiers in calls:
            for ek, rk in zip(engine, request):
                self._add_pair(model, ek, rk, podtiers)
        self._end()

    def skip(self, kind):
        """An op that changes no key this history follows (a writer's keys that no read looks at)."""
        self._begin(kind)
        self._end()

    def evict(self, model, engine, podtiers):
        self._begin("evict")
        self._evict(model, engine, podtiers)
        self._end()

    def apply_events(self, events, hashes, tokens, kind="apply_events"):
        """kvidx_apply_events / _dev: digestEvents (pool.go:246-338) event by event in array order.  The batch must hold
        one pod's events (or pods on disjoint keys), so that every schedule of the library's per-pod queues gives this
        order."""
        self._begin(kind)
        B = self.co.block_size
        for ev in events:
            model, pt = int(ev["model"]), int(ev["podtier"])
            hs = hashes[int(ev["hash_off"]):int(ev["hash_off"]) + int(ev["n_hashes"])]
            if int(ev["op"]) == STORED:
                tk = tokens[int(ev["tok_off"]):int(ev["tok_off"]) + int(ev["n_tokens"])]
                parent = None
                if ev["has_parent"]:
                    rk = self.ix.engine_to_request.d.get(ko.Key(model, int(ev["parent_hash"])))
                    parent = None if rk is None else rk.chunk_hash
                nk = len(tk) // B
                if nk != len(hs) or nk == 0:
                    continue                                     # key-count mismatch: the event is dropped
                off = np.array([0, nk * B], np.int64)
                if parent is None:
                    rks, _ = self.co.hash_keys(tk[:nk * B], off)
                else:
                    rks, _ = self.co.hash_keys(tk[:nk * B], off, np.array([parent], np.uint64), np.ones(1, np.uint8))
                for ek, rk in zip(hs, rks):
                    self._add_pair(model, ek, rk, [pt])
            else:
                for h in hs:
                    self._evict(model, h, [pt])
        self._end()

    def remove_pods(self, pods, tiers=None):
        """kvidx_remove_pods (tests/remove_oracle.py).  A key may pass through every intermediate state of dropping the
        removed entries one by one."""
        self._begin("remove_pods")
        pods_s, tiers_s = set(pods), None if tiers is None else set(tiers)
        before, emptied = {}, set()
        for rk, pc in self.ix.data.d.items():
            drop = [e for e in pc.d if e.pod in pods_s and (tiers_s is None or e.tier in tiers_s)]
            if drop:
                before[rk] = list(pc.d)
                if len(drop) == len(pc.d):
                    emptied.add(rk)
        eng_before = [ek for ek, rk in self.ix.engine_to_request.d.items() if rk in emptied] if emptied else []
        _remove_pods(self.ix, pods_s, tiers_s)
        for rk, ents in before.items():
            cur = list(ents)
            for e in ents:
                if e.pod in pods_s and (tiers_s is None or e.tier in tiers_s):
                    cur.remove(e)
                    self._rec(self.req, (rk.model, rk.chunk_hash), tuple((x.pod << 4) | x.tier for x in cur) or None)
            self._rec_req(rk)
        for ek in eng_before:
            self._rec_eng(ek)
        self._end()

    # ---- admissible states -------------------------------------------------------------------------------------------
    def req_states(self, key, w):
        return self._states(self.req, key, w, self.clock)

    def eng_states(self, key, w):
        return self._states(self.eng, key, w, False)

    def _states(self, table, key, w, suffixes):
        h = table.get(key)
        if h is None:
            out = {None}
        else:
            ops, vals = h
            i = bisect.bisect_right(ops, w.done) - 1        # the state current at s
            j = bisect.bisect_left(ops, w.begun, i + 1)     # states of the ops that overlap the call
            out = set(vals[i:j])
        if suffixes:
            out = {s[k:] or None for s in out if s is not None for k in range(len(s) + 1)} | {None}
        return out

    def state_at(self, key, op):
        """The state of a request key after the first `op` operations (op = 0: before any)."""
        h = self.req.get(key)
        if h is None:
            return None
        ops, vals = h
        return vals[bisect.bisect_left(ops, op) - 1]


class Window:
    """One read call against one handle's operation intervals.  times: (n_ops, 2) int64 of [t0, t1] per op (the same
    op order as the History); [s, e]: the read's interval.  done = the last op that ended by s; the ops in
    (done, begun) started before e and ended after s."""

    def __init__(self, times, s, e):
        times = np.asarray(times, np.int64).reshape(-1, 2)
        self.s, self.e = s, e
        self.done = int(np.searchsorted(times[:, 1], s, side="right")) - 1
        self.begun = int(np.searchsorted(times[:, 0], e, side="left"))
        self.begun = max(self.begun, self.done + 1)

    def overlapped(self):
        """Indices of the ops whose interval overlaps the call."""
        return range(self.done + 1, self.begun)


class Checker:
    """Row checks of read calls against a History.  weights: tier -> weight (16 entries)."""

    def __init__(self, hist, weights):
        self.h = hist
        self.w = [float(x) for x in weights] + [1.0] * (16 - len(weights))

    def _maxw(self, state, pod):
        m = 0.0
        for pt in state:
            if pt >> 4 == pod and self.w[pt & 15] > m:
                m = self.w[pt & 15]
        return m

    def score_sets(self, model, keys, w, filt=None, memo=None):
        """-> (per-pod admissible values {pod: set of float, -1.0 for "absent"}, max block-0 pod count, has_keys) of a
        prompt with these block keys under `model`; filt: None or a set of pod ids."""
        if memo is not None:
            mk = (model, tuple(keys), None if filt is None else frozenset(filt))
            if mk in memo:
                return memo[mk]
        if len(keys) == 0:
            res = ({}, 0, 0)
        else:
            A = []
            for k in keys:
                st = self.h.req_states((model, int(k)), w)
                if filt is not None:
                    st = {tuple(pt for pt in s if pt >> 4 in filt) or None if s is not None else None for s in st}
                A.append(st)
            pods0, nmax, absent0 = set(), 0, False
            for s in A[0]:
                ps = set() if s is None else {pt >> 4 for pt in s}
                pods0 |= ps
                nmax = max(nmax, len(ps))
            sets = {}
            for p in pods0:
                pairs = set()
                for s in A[0]:
                    if s is not None and any(pt >> 4 == p for pt in s):
                        pairs.add((True, self._maxw(s, p)))
                    else:
                        pairs.add((False, -1.0))
                for st in A[1:]:
                    if not any(a for a, _ in pairs):
                        break
                    nxt = set()
                    for alive, sc in pairs:
                        if not alive:
                            nxt.add((False, sc))
                            continue
                        for s in st:
                            if s is not None and any(pt >> 4 == p for pt in s):
                                nxt.add((True, sc + self._maxw(s, p)))
                            else:
                                nxt.add((False, sc))
                    pairs = nxt
                sets[p] = {sc for _, sc in pairs}
            res = (sets, nmax, 1)
        if memo is not None:
            memo[mk] = res
        return res

    @staticmethod
    def row_ok(row, has, sets_nmax_has):
        """A dense row (max_pods f64, -1 = absent) and has_keys against score_sets()' answer -> None, or why it is not
        admissible."""
        sets, nmax, want_has = sets_nmax_has
        if int(has) != want_has:
            return "has_keys %d, want %d" % (int(has), want_has)
        row = np.asarray(row, np.float64)
        present = np.flatnonzero(row != -1.0)
        if len(present) > nmax:
            return "%d pods, at most %d admissible at block 0" % (len(present), nmax)
        for p in present:
            if int(p) not in sets:
                return "pod %d is in no admissible block-0 state" % p
        for p, vals in sets.items():
            v = float(row[p]) if p < len(row) else -1.0
            if v not in vals:
                return "pod %d scored %r, admissible %s" % (p, v, sorted(vals)[:8])
        return None

    def lookup_ok(self, model, keys, pt, cnt, w, filt=None):
        """Lookup rows: each key's entries, in order, equal one admissible state exactly (filtered).  -> None or why not."""
        memo = {}
        for i, k in enumerate(keys):
            got = tuple(int(x) for x in pt[i, :cnt[i]]) or None
            st = memo.get(int(k))
            if st is None:
                st = self.h.req_states((model, int(k)), w)
                if filt is not None:
                    st = {tuple(x for x in s if x >> 4 in filt) or None if s is not None else None for s in st}
                memo[int(k)] = st
            if got not in st:
                return "key %d (%#x): entries %s, admissible %s" % (i, int(k), got, sorted(st, key=str)[:6])
        return None

    def request_key_ok(self, model, engine, rc, value, w):
        """get_request_key: (rc, value) equals one admissible state of the engine mapping (a miss is rc != 0)."""
        got = value if rc == 0 else None
        st = self.h.eng_states((model, int(engine)), w)
        return None if got in st else "engine %#x -> %s, admissible %s" % (int(engine), got, st)
