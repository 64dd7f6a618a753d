"""Slot-level model of one CLOCK handle (evict_policy="clock", include/kvidx.h): which slot each key occupies, one
reference bit per slot, and the hand of each map.  Written from the contract at the top of csrc/kernels_clock.cuh, not
from its kernels:

  * insert: probe from the even home slot to the first EMPTY slot; tombstones are passed, never reused;
  * sweep after a write call, e = live - capacity > 0: starting at the hand and wrapping around, a FULL slot with its bit
    set has the bit cleared, a FULL slot with its bit clear is evicted (a tombstone), every other slot is passed, and the
    hand stops just after the e-th eviction -- a second turn when fewer than e keys were unreferenced;
  * rebuild: tombstones dropped, every key keeps its bit, both hands back to slot 0.

Slot positions are the library's as long as no two keys of one call (or of a rebuild) probe for the same slot: the
tests insert new keys only on home pairs that are fully EMPTY (helpers.keep_free).

Reference bits are set where the write path sets them: Add marks the mapping and the request key of every pair (new or
refreshed), Evict the mapping and the request key it finds (also when they then become tombstones), GetRequestKey the
mapping, Lookup every present request key.  Restore marks nothing.  Score() marks what clock_oracle.referenced_keys names.
"""
import numpy as np

from helpers import _slot_home

EMPTY, FULL, TOMB = 0, 1, 2


class ClockMap:
    """One table of S slots: slot states, the key of every non-EMPTY slot, the reference bits and the hand."""

    def __init__(self, S):
        assert S >= 2 and S & (S - 1) == 0
        self.S, self.mask = S, S - 1
        self.state = np.zeros(S, np.int8)
        self.ref = np.zeros(S, bool)
        self.at = {}           # slot -> (key, home) of a FULL or TOMB slot; key = (model, hash)
        self.where = {}        # live key -> its slot
        self.hand = 0
        self.tombs = 0

    @property
    def live(self):
        return len(self.where)

    def home(self, key):
        return int(_slot_home(key[1], key[0], self.S)[0])

    def insert(self, key, home=None):
        assert key not in self.where
        home = self.home(key) if home is None else home
        i = home
        while self.state[i] != EMPTY:
            i = (i + 1) & self.mask
        self.state[i] = FULL
        self.at[i] = (key, home)
        self.where[key] = i
        return i

    def mark(self, key):
        self.ref[self.where[key]] = True

    def kill(self, key):
        i = self.where.pop(key)
        self.state[i] = TOMB
        self.tombs += 1

    def rebuild(self):
        live = sorted((i, self.at[i]) for i in self.where.values())
        bits = {key: bool(self.ref[i]) for i, (key, _) in live}
        self.state[:] = EMPTY
        self.ref[:] = False
        self.at, self.where, self.tombs, self.hand = {}, {}, 0, 0
        for _, (key, home) in live:
            self.ref[self.insert(key, home)] = bits[key]

    def hand_order(self):
        """Live slots in the order the hand meets them."""
        return sorted(self.where.values(), key=lambda i: (i - self.hand) & self.mask)

    def sweep(self, capacity):
        """The sequential hand.  -> (evicted keys in eviction order, whether it went past a full turn)."""
        e = self.live - capacity
        if e <= 0:
            return [], False
        order = self.hand_order()
        out = []
        for turn in (1, 2):
            for i in order:
                if self.state[i] != FULL:
                    continue
                if self.ref[i]:
                    self.ref[i] = False
                    continue
                key = self.at[i][0]
                self.kill(key)
                out.append(key)
                if len(out) == e:
                    self.hand = (i + 1) & self.mask
                    return out, turn == 2
        raise AssertionError("unreachable: a second turn evicts every key")

    def rank(self, slot):
        """(unreferenced, referenced) live keys the hand meets up to and including `slot`, in hand order."""
        u = v = 0
        for i in self.hand_order():
            if self.ref[i]:
                v += 1
            else:
                u += 1
            if i == slot:
                return u, v
        raise KeyError(slot)

    def counts(self):
        """(unreferenced, referenced) live keys."""
        v = sum(1 for i in self.where.values() if self.ref[i])
        return self.live - v, v


class ClockHandle:
    """Both maps of one unsharded CLOCK handle, the pod entries of every request key and the target of every mapping,
    and the counters the library reports: kvidx_get_evictions, kvidx_get_sweeps and the rebuild count."""

    def __init__(self, S, capacity, pods_per_key=10):
        self.req, self.eng = ClockMap(S), ClockMap(S)
        self.capacity, self.pods_per_key = capacity, pods_per_key
        self.pods = {}         # live request key -> pod entries, oldest first
        self.target = {}       # live mapping -> request hash
        self.evictions, self.sweeps, self.rebuilds = [0, 0], [0, 0], 0
        self.victims = ([], [])  # keys evicted by the last call's sweeps, per map

    # ---- the steps of a write call ----
    def room(self, incoming):
        """The room check before a call's inserts: compact when keys + tombstones + incoming pass 80 % of a table."""
        over = lambda m: (m.live + m.tombs + incoming) * 10 > m.S * 8
        if (over(self.req) or over(self.eng)) and (self.req.tombs or self.eng.tombs):
            self.rebuild()
        for m in (self.req, self.eng):
            assert (m.live + incoming) * 10 <= m.S * 9, "the library refuses this call (KVIDX_ENOSPC)"

    def rebuild(self):
        self.req.rebuild()
        self.eng.rebuild()
        self.rebuilds += 1

    def cap(self):
        self.victims = ([], [])
        for k, (m, payload) in enumerate(((self.req, self.pods), (self.eng, self.target))):
            out, two = m.sweep(self.capacity)
            for key in out:
                del payload[key]
            self.victims[k].extend(out)
            self.evictions[k] += len(out)
            self.sweeps[0] += 1 if out else 0
            self.sweeps[1] += 1 if two else 0

    def put(self, model, engine, request, pts):
        """One pair of Add (or one block of BlockStored): upsert and mark the mapping, upsert the request key, add the
        entries and mark it."""
        ek, rk = (model, int(engine)), (model, int(request))
        if ek not in self.eng.where:
            self.eng.insert(ek)
        self.target[ek] = int(request)
        self.eng.mark(ek)
        if rk not in self.req.where:
            self.req.insert(rk)
            self.pods[rk] = []
        ents = self.pods[rk]
        for pt in pts:
            if pt in ents:
                ents.remove(pt)
            elif len(ents) >= self.pods_per_key:
                ents.pop(0)
            ents.append(pt)
        self.req.mark(rk)

    # ---- calls ----
    def add(self, model, engines, requests, pts):
        assert len(engines) == len(requests) and len(set(map(int, engines))) == len(engines)
        self.room(len(engines))
        for e, r in zip(engines, requests):
            self.put(model, e, r, pts)
        self.cap()

    def store(self, blocks, pts):
        """One batch of BlockStored events without parents: blocks = [(model, engine hash, request key), ...]."""
        self.room(len(blocks))
        for model, e, r in blocks:
            self.put(model, e, r, pts)
        self.cap()

    def evict(self, model, engine, pts):
        ek = (model, int(engine))
        if ek in self.eng.where:
            self.eng.mark(ek)
            rk = (model, self.target[ek])
            drop = True
            if rk in self.req.where:
                self.req.mark(rk)
                self.pods[rk] = [p for p in self.pods[rk] if p not in pts]
                if self.pods[rk]:
                    drop = False
                else:
                    del self.pods[rk]
                    self.req.kill(rk)
            if drop:
                del self.target[ek]
                self.eng.kill(ek)
        self.cap()

    def get_request_key(self, model, engine):
        ek = (model, int(engine))
        if ek not in self.eng.where:
            return None
        self.eng.mark(ek)
        return self.target[ek]

    def lookup(self, model, keys):
        hit = []
        for k in keys:
            rk = (model, int(k))
            hit.append(rk in self.req.where)
            if hit[-1]:
                self.req.mark(rk)
        return hit

    def restore(self, requests, mappings):
        """Into a handle holding no live key: requests = [(model, hash, [pod entries])], mappings = [(model, engine hash,
        request hash)].  Tombstones go, nothing is marked, the hands stay where they are."""
        assert not self.req.live and not self.eng.live
        for m in (self.req, self.eng):
            m.state[:] = EMPTY
            m.ref[:] = False
            m.at, m.tombs = {}, 0
        for model, h, ents in requests:
            self.req.insert((model, int(h)))
            self.pods[(model, int(h))] = list(ents)
        for model, e, r in mappings:
            self.eng.insert((model, int(e)))
            self.target[(model, int(e))] = int(r)
        self.cap()

    # ---- what the library reports ----
    def records(self):
        """(request keys, mappings) as sorted arrays: (model, hash) and (model, engine hash, request hash)."""
        rq = np.array(sorted(self.req.where), np.uint64).reshape(-1, 2)
        eg = np.array(sorted((m, e, self.target[(m, e)]) for m, e in self.eng.where), np.uint64).reshape(-1, 3)
        return rq, eg
