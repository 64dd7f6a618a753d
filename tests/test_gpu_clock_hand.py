"""GPU (-m gpu): the CLOCK sweep (csrc/kernels_clock.cuh) victim by victim against the sequential hand of
tests/clock_hand_oracle.py, from one tile of 1024 slots to 8192 tiles (eight per thread of the cut kernel).

Every key is inserted on a home pair that is fully EMPTY, so its slot is known.  After every call the resident request
keys and mappings (from the snapshot), kvidx_get_evictions, kvidx_get_sweeps, the key and tombstone counts and the
rebuild count must equal the model's exactly -- so a sweep that takes one wrong victim, stops one slot off, forgets to
clear a bit it passed or keeps a hand across a rebuild fails the call that does it."""
import numpy as np
import pytest

import kvidx
from clock_hand_oracle import ClockHandle
from helpers import (EVENT_DTYPE, SNAP_ENG_DTYPE, SNAP_REQ_DTYPE, decode_snapshot, draw_free, free_pairs, keep_free,
                     keys_homed_at)

pytestmark = pytest.mark.gpu
BS, P, TILE, CUT_THREADS = 16, 8, 1024, 1024


def PT(p, t=0):
    return (p << 4) | t


def image(requests, mappings):
    """A v1 image (include/kvidx.h) of model-0 keys with one entry each: requests = [(hash, podtier)], mappings =
    [(engine hash, request hash)]."""
    req = np.zeros(len(requests), SNAP_REQ_DTYPE)
    req["hash"] = [h for h, _ in requests]
    req["count"] = 1
    req["ent"][:, 0] = [pt for _, pt in requests]
    req.sort(order="hash")
    eng = np.zeros(len(mappings), SNAP_ENG_DTYPE)
    eng["hash"] = [e for e, _ in mappings]
    eng["request"] = [r for _, r in mappings]
    eng.sort(order="hash")
    hdr = bytearray(64)
    hdr[:8] = b"KVIDXSNP"
    hdr[8:24] = np.array([1, 0, BS, 4], "<u4").tobytes()
    hdr[24:48] = np.array([kvidx.fnv64a(b""), len(req), len(eng)], "<u8").tobytes()
    hdr[48:56] = np.array([1 + max((pt >> 4 for _, pt in requests), default=-1), 1 if len(req) or len(eng) else 0], "<u4").tobytes()
    return bytes(hdr) + req.tobytes() + eng.tobytes()


class Rig:
    """A CLOCK handle of S slots per table and its model, compared after every call."""

    def __init__(self, S, capacity, seed):
        self.S, self.T = S, S // TILE
        self.per = -(-self.T // CUT_THREADS)                 # tiles per thread of the cut kernel
        self.rng = np.random.default_rng(seed)
        self.ix = kvidx.Index(block_size=BS, capacity=capacity, table_slots=S, pods_per_key=4, max_pods=P, evict_policy="clock")
        self.m = ClockHandle(S, capacity, pods_per_key=4)
        assert self.ix.stats()["request_slots"] == S

    # ---- the comparison ----
    def check(self):
        m, st = self.m, self.ix.stats()
        assert st["rebuilds"] == m.rebuilds
        assert self.ix.evictions() == tuple(m.evictions)
        assert self.ix.sweeps() == tuple(m.sweeps)
        assert (st["request_keys"], st["engine_keys"]) == (m.req.live, m.eng.live)
        assert (st["request_tombs"], st["engine_tombs"]) == (m.req.tombs, m.eng.tombs)
        req, eng = decode_snapshot(self.ix.snapshot())
        want_r, want_e = m.records()
        got_r = np.stack([req["model"].astype(np.uint64), req["hash"]], 1)
        got_e = np.stack([eng["model"].astype(np.uint64), eng["hash"], eng["request"]], 1)
        for name, got, want, mp in (("request", got_r, want_r, m.req), ("engine", got_e, want_e, m.eng)):
            if not np.array_equal(got, want):
                g, w = {tuple(map(int, r[:2])) for r in got}, {tuple(map(int, r[:2])) for r in want}
                kept = sorted((mp.where[k] for k in w - g))
                raise AssertionError("%s map: the library evicted the keys on slots %s (model: hand %d) and kept %d others"
                                     % (name, kept[:8], mp.hand, len(g - w)))

    def _slot_keys(self, mp):
        return {i: k for k, i in mp.where.items()}

    # ---- calls, each made on both and checked ----
    def add(self, eng, req, pts=(PT(0),)):
        assert self.ix.add(0, np.asarray(eng, np.uint64), np.asarray(req, np.uint64), list(pts)) == 0
        self.m.add(0, [int(x) for x in eng], [int(x) for x in req], list(pts))
        self.check()

    def new_pairs(self, n):
        """n (engine, request) pairs of new keys, each on a random fully EMPTY home pair of its map."""
        rs = self.rng.choice(free_pairs(self.m.req.state), n, replace=False)
        es = self.rng.choice(free_pairs(self.m.eng.state), n, replace=False)
        return keys_homed_at(es, 0, self.S, self.rng), keys_homed_at(rs, 0, self.S, self.rng)

    def add_new(self, n):
        self.roomy(n)
        e, r = self.new_pairs(n)
        self.add(e, r, (PT(int(self.rng.integers(0, P))),))
        return e, r

    def lookup(self, keys):
        keys = np.asarray(list(keys), np.uint64)
        rc, _, cnt = self.ix.lookup(0, keys)
        assert rc == 0
        assert list(cnt > 0) == self.m.lookup(0, keys)

    def get_request_key(self, engines):
        for e in engines:
            rc, r = self.ix.get_request_key(0, int(e))
            want = self.m.get_request_key(0, e)
            assert (rc == 0, r if rc == 0 else None) == (want is not None, want)

    def evict(self, engine, pts):
        assert self.ix.evict(0, int(engine), list(pts)) == 0
        self.m.evict(0, engine, list(pts))
        self.check()

    def compact(self):
        self.ix.shard_compact()
        self.m.rebuild()
        self.check()

    def roomy(self, n):
        """Compact first if n new keys would make the next call's room check compact (which would move the hand to 0
        under a case that placed its cut relative to the hand), or would not find n fully EMPTY home pairs."""
        if any((mp.live + mp.tombs + n) * 10 > self.S * 8 or len(free_pairs(mp.state)) < n for mp in (self.m.req, self.m.eng)):
            self.compact()

    # ---- placing the request map's cut ----
    def rot(self, slot, mp=None):
        mp = mp or self.m.req
        return (slot - mp.hand) & (self.S - 1)

    def only_unreferenced(self, keep):
        """Lookup every live request key but those on the slots in `keep`: they are the map's only unreferenced keys."""
        sk = self._slot_keys(self.m.req)
        keep = set(keep)
        self.lookup(k[1] for i, k in sk.items() if i not in keep)
        assert set(self.m.req.where[k] for k in self.m.req.where if not self.m.req.ref[self.m.req.where[k]]) == keep

    def cut_on(self, slot, frac=0.5):
        """Make the next request-map sweep stop on `slot`, an unreferenced key.  Of the keys the hand passes before it,
        Lookup marks every anchor and a random `frac` of the others (the sweep clears their bits); the unreferenced
        rest go before it.  Keys beyond it are left alone.  Then Add as many new pairs as the cut needs (referenced, so
        they do not move it)."""
        mp = self.m.req
        self.roomy(sum(1 for i in mp.where.values() if self.rot(i) < self.rot(slot)) + 1)
        assert slot in mp.where.values() and not mp.ref[slot]
        sk = self._slot_keys(mp)
        mark = [i for i in mp.where.values() if self.rot(i) < self.rot(slot) and (i % (TILE // 2) == 0 or self.rng.random() < frac)]
        if mark:
            self.lookup(sk[i][1] for i in mark)
        u, _ = mp.rank(slot)
        hand0, key = mp.hand, sk[slot]
        self.add_new(u + mp.live - self.m.capacity)
        assert self.m.victims[0][-1] == key and mp.hand == (slot + 1) & (self.S - 1), (hand0, slot)
        return hand0


SIZES = [1024, 8192, 1 << 20, 1 << 21, 1 << 23]     # 1 tile; 8; one per cut-kernel thread; two per thread; eight


def anchors(S):
    """Slots 1024 t and 1024 t + 512 of every tile t."""
    return np.sort(np.concatenate([np.arange(0, S, TILE), np.arange(TILE // 2, S, TILE)]))


def _layout(S, fill, rng):
    """Model-0 keys on every anchor slot of both maps plus `fill` more on random free pairs (pair j on the same slot in
    both maps): (requests, mappings) for image()."""
    a = anchors(S)
    taken = np.zeros(S, np.int8)
    taken[a] = 1
    more = rng.choice(free_pairs(taken), fill, replace=False)
    slots = np.concatenate([a, more])
    req = keys_homed_at(slots, 0, S, rng)
    eng = keys_homed_at(slots, 0, S, rng)
    pts = rng.integers(0, P, len(slots))
    requests = [(int(r), PT(int(p))) for r, p in zip(req, pts)]
    mappings = [(int(e), int(r)) for e, r in zip(eng, req)]
    return requests, mappings


def _restore(rig, requests, mappings):
    got = rig.ix.restore(image(requests, mappings))
    rig.m.restore([(0, r, [pt]) for r, pt in requests], [(0, e, r) for e, r in mappings])
    assert got == {"request_keys": rig.m.req.live, "engine_keys": rig.m.eng.live}
    rig.check()


@pytest.mark.parametrize("S", SIZES)
def test_restore_above_capacity_cuts_from_slot_0(S):
    requests, mappings = _layout(S, 150, np.random.default_rng(S))
    rig = Rig(S, len(requests) - 37, S)
    _restore(rig, requests, mappings)
    lowest = sorted(rig.m.req.at)[:37]
    assert [rig.m.req.at[i][0] for i in lowest] == rig.m.victims[0]
    assert rig.m.req.hand == lowest[-1] + 1 and rig.ix.sweeps() == (2, 0)


@pytest.mark.parametrize("S", [1024, 8192])
def test_restore_into_an_emptied_handle_keeps_the_hand(S):
    """Restore drops the tombstones but leaves the hands just past the last sweep's victim.  The image fills that
    victim's slot again, so its key is the last one the next sweep reaches (a hand left on the victim's slot would
    take it first)."""
    requests, mappings = _layout(S, 40, np.random.default_rng(S + 2))
    rig = Rig(S, len(requests) - 9, S + 2)
    _restore(rig, requests, mappings)
    mp = rig.m.req
    c = mp.hand - 1                                              # the last victim's slot
    assert mp.at[c][0] == rig.m.victims[0][-1]
    for k in list(rig.m.eng.where):                              # Evict every pair: no live key is left
        rig.evict(k[1], rig.m.pods[(0, rig.m.target[k])])
    assert mp.live == 0 and rig.m.eng.live == 0 and mp.tombs == len(requests)
    _restore(rig, requests, mappings)
    assert rig.m.victims[0] == [mp.at[i][0] for i in sorted(mp.at) if i > c][:9] and mp.at[c][0] in mp.where


@pytest.mark.parametrize("S", SIZES)
def test_directed_cuts(S):
    requests, mappings = _layout(S, 200, np.random.default_rng(S + 1))
    rig = Rig(S, len(requests), S + 1)
    _restore(rig, requests, mappings)                            # at capacity: no sweep, the hands at 0
    T, per, mp = rig.T, rig.per, rig.m.req
    assert rig.m.sweeps == [0, 0] and mp.hand == 0

    # 1. on the first slot of a tile: the first tile of the cut kernel's thread 1 (thread 0's first slot with one tile)
    q = per if T > 1 else 0
    rig.cut_on(q * TILE)
    assert rig.rot(q * TILE, mp) == S - 1                       # (the hand is now just past it)

    # 2. on the last slot of a tile, after the rotated range has wrapped past S - 1; inside a thread's range when per > 1
    if T > 1:
        t = max(t for t in range(T - 1) if per == 1 or t % per == per // 2)
        target = (mp.hand + t * TILE + TILE - 1) & (S - 1)
        assert target < mp.hand and target in mp.where.values()
        rig.cut_on(target)

    # 3. mid-tile, on the first tile of a thread's range (thread 1, or tile 0 with fewer than two tiles)
    t = per if T > per else 0
    target = (mp.hand + t * TILE + TILE // 2 - 1) & (S - 1)
    assert target in mp.where.values()
    rig.cut_on(target)

    # 4. a rebuild between sweeps: the hands go back to slot 0, every key keeps its bit; then a cut on the highest
    # unreferenced key (in the last tile: the cut kernel's last thread)
    rig.compact()
    assert mp.hand == 0 and rig.m.eng.hand == 0
    rig.cut_on(max(i for i in mp.where.values() if not mp.ref[i]))

    # 5. e == U: the cut on the last unreferenced key; the next sweep takes the keys whose bits that pass cleared
    rig.roomy(24)
    unref = sorted(i for i in mp.where.values() if not mp.ref[i])
    keep = set(rig.rng.choice(unref, min(24, len(unref)), replace=False).tolist())
    rig.only_unreferenced(keep)
    last = max(keep, key=rig.rot)
    rig.add_new(len(keep) + mp.live - rig.m.capacity)
    assert set(rig.m.victims[0]) == {mp.at[i][0] for i in keep} and mp.hand == (last + 1) & (S - 1)
    assert rig.m.sweeps[1] == 0
    cleared = {k for k, i in mp.where.items() if not mp.ref[i]}  # every key between the old hand and the cut
    assert cleared
    rig.add_new(min(8, len(cleared)))                            # past the keys the pass did not reach, onto those
    assert set(rig.m.victims[0]) <= cleared and rig.m.sweeps[1] == 0

    # 6. e == U + 1: a second turn that takes the first key in hand order after the first turn
    rig.roomy(11)
    unref = sorted(i for i in mp.where.values() if not mp.ref[i])
    keep = set(rig.rng.choice(unref, min(10, len(unref)), replace=False).tolist())
    rig.only_unreferenced(keep)
    t2 = rig.m.sweeps[1]
    rig.add_new(len(keep) + 1 + mp.live - rig.m.capacity)
    assert set(rig.m.victims[0][:-1]) == {mp.at[i][0] for i in keep} and rig.m.sweeps[1] >= t2 + 1

    # 7. a second turn that ends mid-table: e == U + half the referenced keys
    rig.roomy(mp.live)
    unref = sorted(i for i in mp.where.values() if not mp.ref[i])
    keep = set(rig.rng.choice(unref, min(6, len(unref)), replace=False).tolist())
    rig.only_unreferenced(keep)
    hand0, t2 = mp.hand, rig.m.sweeps[1]
    rig.add_new(len(keep) + (mp.live - len(keep)) // 2 + mp.live - rig.m.capacity)
    assert rig.m.sweeps[1] >= t2 + 1 and mp.hand != hand0

    # 8. request and engine excesses that differ in one call: new mappings onto resident request keys, with some
    # mappings marked by GetRequestKey
    rig.get_request_key(rig.rng.choice([k[1] for k in rig.m.eng.where], 16, replace=False))
    rig.roomy(40)
    e_new, r_new = rig.new_pairs(40)
    old = [k[1] for k in list(mp.where)[:30]]
    rig.add(e_new, list(r_new[:10]) + old)
    assert len(rig.m.victims[0]) == 10 and len(rig.m.victims[1]) == 40

    # 9. Evict: marks the mapping and the request key (an entry the key does not hold); its last entries gone, both
    # become tombstones; then the room Evict left is filled again
    for j, k in enumerate(list(rig.m.eng.where)[:6]):
        pods = rig.m.pods.get((0, rig.m.target[k]))
        rig.evict(k[1], pods if pods and j % 2 else [PT(0, 3)])
    rig.add_new(12)

    # 10. one asynchronous batch of BlockStored events
    _stored_batch(rig)


def _stored_batch(rig):
    """BlockStored events without parents, one block each, through kvidx_apply_events_dev: the first batch's blocks are
    new keys; after a full turn clears every request key's bit, the second batch stores half of them again (marking their request keys
    and mappings) and as many new ones as puts a long cut through the table."""
    import torch
    dev = torch.device("cuda")
    keep = []

    def send(blocks, toks, pt):
        n = len(blocks)
        ev = np.zeros(n, EVENT_DTYPE)
        ev["podtier"] = pt
        ev["hash_off"] = np.arange(n)
        ev["tok_off"] = np.arange(n) * BS
        ev["n_hashes"] = 1
        ev["n_tokens"] = BS
        hashes = np.array([e for e, _ in blocks], np.uint64)
        d = [torch.from_numpy(ev.view(np.uint8).copy()).to(dev), torch.tensor([0, n], dtype=torch.int64, device=dev),
             torch.from_numpy(hashes.view(np.int64).copy()).to(dev), torch.from_numpy(toks.reshape(-1).astype(np.int32)).to(dev)]
        torch.cuda.synchronize()
        rig.ix.apply_events_dev(d[0].data_ptr(), d[1].data_ptr(), 1, n, d[2].data_ptr(), n, d[3].data_ptr())
        keep.append(d)
        rig.ix.synchronize()
        rig.m.store([(0, e, r) for e, r in blocks], [pt])
        rig.check()

    def fresh(n):
        """n one-block token rows whose request keys (hash_keys) sit on free pairs, and engine hashes on free pairs."""
        for more in range(1, 9):
            rows = rig.rng.integers(0, 128256, size=(16 * more * n + 64, BS), dtype=np.uint32)
            keys, _ = rig.ix.hash_keys(rows.reshape(-1), np.arange(len(rows) + 1, dtype=np.int64) * BS)
            idx = np.flatnonzero(np.isin(keys, keep_free(keys, 0, rig.m.req.state)))
            _, first = np.unique(keys[idx], return_index=True)
            idx = np.sort(idx[first])[:n]
            if len(idx) == n:
                break
        assert len(idx) == n
        eng = draw_free(rig.m.eng.state, n, 0, rig.rng)
        return [(int(e), int(keys[i])) for e, i in zip(eng, idx)], rows[idx]

    mp = rig.m.req
    n1 = min(64, rig.m.capacity // 4)
    rig.compact()                                                # free pairs for the blocks on a small table
    b1, t1 = fresh(n1)
    send(b1, t1, PT(1))
    # a full turn clears every bit of the request map
    rig.lookup(k[1] for k in mp.where)
    rig.add_new(1)
    assert not mp.ref[list(mp.where.values())].any()
    # again half of the first batch, and new blocks enough to pass nearly every key
    half = [i for i in range(n1) if i % 2 == 0 and (0, b1[i][1]) in mp.where and (0, b1[i][0]) in rig.m.eng.where]
    n2 = min(mp.live - len(half) - 1, 4096)
    rig.roomy(n2 + len(half))
    b2, t2 = fresh(n2)
    again = [b1[i] for i in half]
    send(again + b2, np.concatenate([t1[half], t2]), PT(2))
    survivors = set(mp.where)
    assert {(0, r) for _, r in again} <= survivors


# ---- random differential --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,seed", [(1024, 1), (1024, 2), (4096, 3), (4096, 4), (65536, 5), (65536, 6)])
def test_random_calls_against_model(S, seed):
    """About 150 mixed calls: new keys, refreshes, Lookup and GetRequestKey subsets, Evict and compaction."""
    cap = min(S // 8, 1024)
    rig = Rig(S, cap, seed)
    rng = rig.rng
    for step in range(150):
        op = int(rng.integers(0, 10))
        mp, me = rig.m.req, rig.m.eng
        if op <= 2 or mp.live < 8:                                   # new keys
            rig.add_new(int(rng.integers(1, cap // 2)))
        elif op == 3:                                                # refreshes of resident pairs: no insert
            pairs = [(k[1], t) for k, t in rig.m.target.items() if (0, t) in mp.where]
            sel = rng.choice(len(pairs), min(len(pairs), int(rng.integers(1, 40))), replace=False)
            rig.roomy(len(sel))                                      # (a compaction keeps every key)
            rig.add([pairs[i][0] for i in sel], [pairs[i][1] for i in sel], (PT(int(rng.integers(0, P))),))
        elif op in (4, 5):                                           # Lookup a subset, and three absent keys
            ks = [k[1] for k in mp.where]
            sel = rng.choice(len(ks), int(rng.integers(1, len(ks) + 1)), replace=False)
            rig.lookup([ks[i] for i in sel] + [int(x) for x in rng.integers(1, 1 << 63, 3)])
        elif op == 6:                                                # GetRequestKey a subset, and one absent key
            ks = [k[1] for k in me.where]
            sel = rng.choice(len(ks), min(len(ks), int(rng.integers(1, 24))), replace=False)
            rig.get_request_key([ks[i] for i in sel] + [12345])
        elif op in (7, 8):                                           # Evict: every entry the key holds, or one it lacks
            ks = list(me.where)
            for i in rng.choice(len(ks), min(len(ks), int(rng.integers(1, 6))), replace=False):
                ents = rig.m.pods.get((0, rig.m.target[ks[i]]))
                rig.evict(ks[i][1], ents if ents and rng.integers(0, 2) else [PT(int(rng.integers(0, P)), 1)])
        else:
            rig.compact()
        rig.check()
    assert rig.m.evictions[0] > 0 and rig.m.rebuilds > 0
