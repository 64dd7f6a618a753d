"""The referenced-key spec of CLOCK mode (tests/clock_oracle.py) and the slot-level hand model
(tests/clock_hand_oracle.py) on hand-made cases."""
import numpy as np
import pytest

from oracle import kvoracle as ko
from clock_hand_oracle import EMPTY, FULL, TOMB, ClockHandle, ClockMap
from clock_oracle import referenced_keys, walk_keys
from helpers import _slot_home, decode_snapshot, draw_free, keep_free, keys_homed_at

B = 4
TP = ko.ChunkedTokenDatabase(B)


def prompt(n_blocks, salt=0):
    return [1000 * salt + j for j in range(n_blocks * B)]


def keys_of(tokens, model="m"):
    return TP.tokens_to_kv_block_keys(None, tokens, model)


def index_with(keys_pods, model="m"):
    """keys_pods: [(Key, [pod, ...]), ...] -> InMemoryIndex holding them (engine key = request key)."""
    ix = ko.InMemoryIndex(1 << 20, 10)
    for k, pods in keys_pods:
        ix.add([k], [k], [ko.PodEntry(p, "gpu") for p in pods])
    return ix


def test_gap_at_block_i():
    t = prompt(6)
    ks = keys_of(t)
    ix = index_with([(k, ["a"]) for j, k in enumerate(ks) if j != 3])
    assert referenced_keys(ix, [(t, "m")], block_size=B) == set(ks[:3])


def test_filter_empties_active_set_early():
    t = prompt(5)
    ks = keys_of(t)
    ix = index_with([(ks[0], ["a", "b"]), (ks[1], ["a", "b"]), (ks[2], ["b"]), (ks[3], ["a"]), (ks[4], ["a"])])
    # unfiltered: block 2 keeps b, block 3 drops it -> blocks 0..3
    assert referenced_keys(ix, [(t, "m")], block_size=B) == set(ks[:4])
    # filter {a}: block 2 holds only b -> the walk ends at block 2
    assert referenced_keys(ix, [(t, "m")], [["a"]], block_size=B) == set(ks[:3])


def test_key0_absent():
    t = prompt(4)
    ks = keys_of(t)
    ix = index_with([(k, ["a"]) for k in ks[1:]])
    assert referenced_keys(ix, [(t, "m")], block_size=B) == set()


def test_present_but_filtered_out_counts_as_probed():
    t = prompt(3)
    ks = keys_of(t)
    ix = index_with([(k, ["a"]) for k in ks])
    assert referenced_keys(ix, [(t, "m")], [["b"]], block_size=B) == {ks[0]}
    # the same at block 1: block 1 is probed (and marked), block 2 is not
    ix2 = index_with([(ks[0], ["a", "b"]), (ks[1], ["a"]), (ks[2], ["a", "b"])])
    assert referenced_keys(ix2, [(t, "m")], [["b"]], block_size=B) == {ks[0], ks[1]}


def test_several_models():
    t = prompt(3)
    ka, kb = keys_of(t, "A"), keys_of(t, "B")
    ix = index_with([(k, ["p"]) for k in ka] + [(kb[0], ["p"])])
    got = referenced_keys(ix, [(t, "A"), (t, "B")], block_size=B)
    assert got == set(ka) | {kb[0]}
    assert referenced_keys(ix, [(t, "B")], block_size=B) == {kb[0]}


def test_walk_does_not_refresh_recency():
    t = prompt(3)
    ks = keys_of(t)
    ix = index_with([(k, ["a"]) for k in ks])
    before = list(ix.data.d)
    assert walk_keys(ix, ks) == ks
    assert list(ix.data.d) == before


# ---- the sequential hand -----------------------------------------------------------------------------------------------
def K(s):
    """The key the hand-made tables put on slot s (its home)."""
    return (0, 1000 + s)


def table(S, hand, bits):
    """bits: {slot: referenced} -> a map with one key on each of those slots."""
    m = ClockMap(S)
    for s in sorted(bits):
        m.insert(K(s), home=s)
        m.ref[s] = bits[s]
    m.hand = hand
    return m


def bits_of(m):
    return {s: bool(m.ref[s]) for s in sorted(m.where.values())}


def test_partial_turn_wraps_past_the_last_slot():
    m = table(16, 12, {13: True, 14: False, 2: False, 4: True, 8: False})
    assert m.sweep(3) == ([K(14), K(2)], False)
    assert m.hand == 3 and m.tombs == 2
    assert bits_of(m) == {4: True, 8: False, 13: False}          # 13 was passed, 4 was not
    assert m.sweep(2) == ([K(8)], False) and m.hand == 9           # 4 is passed (cleared) on the way
    assert bits_of(m) == {4: False, 13: False}


def test_e_equal_to_unreferenced_then_the_cleared_keys_go():
    m = table(16, 0, {1: True, 3: False, 5: True, 7: False, 9: True})
    assert m.sweep(3) == ([K(3), K(7)], False)                     # ends exactly at the last unreferenced key
    assert m.hand == 8 and bits_of(m) == {1: False, 5: False, 9: True}
    assert m.sweep(1) == ([K(1), K(5)], False)                     # 9 keeps its key, the pass's cleared keys go
    assert m.hand == 6 and bits_of(m) == {9: False}


def test_e_one_past_unreferenced_takes_a_second_turn():
    m = table(16, 0, {1: True, 3: False, 5: True, 7: False, 9: True})
    assert m.sweep(2) == ([K(3), K(7), K(1)], True)
    assert m.hand == 2 and bits_of(m) == {5: False, 9: False}


def test_second_turn_stops_mid_table():
    bits = {s: True for s in (22, 26, 30, 2, 6, 10)}
    bits.update({24: False, 4: False})
    m = table(32, 20, bits)
    assert m.sweep(2) == ([K(24), K(4), K(22), K(26), K(30), K(2)], True)
    assert m.hand == 3 and bits_of(m) == {6: False, 10: False}


def test_hand_continues_across_sweeps():
    m = table(16, 0, {s: False for s in range(0, 16, 2)})
    assert m.sweep(6) == ([K(0), K(2)], False) and m.hand == 3
    m.mark(K(4))
    assert m.sweep(5) == ([K(6)], False) and m.hand == 7
    assert m.sweep(4) == ([K(8)], False) and m.hand == 9
    m.mark(K(4))
    assert m.sweep(2) == ([K(10), K(12)], False) and m.hand == 13
    assert m.sweep(1) == ([K(14)], False) and m.hand == 15 and bits_of(m) == {4: True}
    assert m.sweep(0) == ([K(4)], True) and m.hand == 5           # alone and referenced: a second turn


def test_below_capacity_nothing_moves():
    m = table(16, 5, {2: False, 6: True})
    assert m.sweep(2) == ([], False) and m.hand == 5 and bits_of(m) == {2: False, 6: True}


def test_rebuild_drops_tombstones_keeps_bits_and_resets_the_hand():
    m = ClockMap(16)
    m.insert((0, 1), home=4)
    m.insert((0, 2), home=4)                                       # displaced past its home: slot 5
    m.insert((0, 3), home=10)
    assert m.where == {(0, 1): 4, (0, 2): 5, (0, 3): 10}
    m.mark((0, 2))
    m.hand = 7
    assert m.sweep(2) == ([(0, 3)], False) and m.hand == 11
    m.kill((0, 1))
    m.insert((0, 4), home=4)                                       # tombstones are never reused: slot 6
    assert m.where[(0, 4)] == 6 and m.tombs == 2
    m.rebuild()
    assert m.hand == 0 and m.tombs == 0 and not (m.state == TOMB).any()
    assert m.where == {(0, 2): 4, (0, 4): 5}
    assert bits_of(m) == {4: True, 5: False}
    assert m.sweep(1) == ([(0, 4)], False) and m.hand == 6         # from slot 0: 4 cleared, 5 evicted


def test_two_maps_with_different_excesses():
    S = 64
    h = ClockHandle(S, capacity=3)
    rng = np.random.default_rng(1)
    slots = np.arange(0, 16, 2)
    req = [int(k) for k in keys_homed_at(slots, 0, S, rng)]
    eng = [int(k) for k in keys_homed_at(slots, 0, S, rng)]
    h.add(0, eng[:3], req[:3], [1])
    assert h.sweeps == [0, 0] and h.req.where == {(0, req[i]): 2 * i for i in range(3)}
    # three new mappings onto existing request keys, one new request key: engine excess 4, request excess 1
    h.add(0, eng[3:7], req[:3] + [req[3]], [1])
    assert h.victims == ([(0, req[0])], [(0, e) for e in eng[:4]])
    assert h.sweeps == [2, 2]                                      # every key was referenced: two full turns
    assert h.req.hand == 1 and h.eng.hand == 7
    assert h.evictions == [1, 4] and h.req.live == h.eng.live == 3
    assert all(not h.req.ref[i] for i in h.req.where.values())


def test_write_path_marks():
    S = 64
    rng = np.random.default_rng(2)
    h = ClockHandle(S, capacity=8, pods_per_key=2)
    req = [int(k) for k in keys_homed_at(np.arange(0, 20, 2), 0, S, rng)]
    eng = [int(k) for k in keys_homed_at(np.arange(0, 20, 2), 0, S, rng)]
    h.add(0, eng[:8], req[:8], [16])
    h.add(0, eng[8:9], req[8:9], [16])                            # a full turn clears every bit
    assert h.sweeps == [2, 2] and not h.req.ref.any() and not h.eng.ref.any()
    assert h.lookup(0, [req[1], req[0], 5]) == [True, False, False]
    assert h.get_request_key(0, eng[2]) == req[2] and h.get_request_key(0, 99) is None
    h.evict(0, eng[3], [32])                                       # not an entry of the key: both stay, both marked
    h.evict(0, eng[4], [16])                                       # its last entry: both become tombstones
    assert h.req.tombs == 2 and h.eng.tombs == 2                   # (the full turn's victim and eng[4]'s pair)
    assert {k[1] for k in h.req.where if h.req.ref[h.req.where[k]]} == {req[1], req[3]}
    assert {k[1] for k in h.eng.where if h.eng.ref[h.eng.where[k]]} == {eng[2], eng[3]}
    h.add(0, eng[3:4], req[3:4], [48, 64])                         # a refresh marks; entries capped at pods_per_key
    assert h.pods[(0, req[3])] == [48, 64]


def test_room_check_compacts_before_the_inserts():
    S = 64
    rng = np.random.default_rng(3)
    h = ClockHandle(S, capacity=20)
    homes = np.arange(52) * 2 % S                                  # more keys than pairs: later ones probe past their home
    req = [int(k) for k in keys_homed_at(homes, 0, S, rng)]
    eng = [int(k) for k in keys_homed_at(homes, 0, S, rng)]
    h.add(0, eng[:30], req[:30], [1])                              # 20 keys and 10 tombstones
    assert h.rebuilds == 0 and h.req.tombs == 10 and h.req.hand == 19
    h.room(21)                                                     # 20 + 10 + 21 = 51 <= 0.8 x 64: no rebuild
    assert h.rebuilds == 0
    h.add(0, eng[30:52], req[30:52], [1])                          # 20 + 10 + 22 > 0.8 x 64: a rebuild before the inserts
    assert h.rebuilds == 1 and h.req.tombs == 22
    assert h.req.where[(0, req[34])] == 4 and h.req.where[(0, req[42])] == 21   # home 4 free again; 20 was taken
    # from slot 0: the 20 old (cleared) keys, then a second turn over the new ones at slots 0 and 2
    assert h.victims[0] == [(0, r) for r in req[10:30]] + [(0, req[32]), (0, req[33])]
    assert h.req.hand == 3 and h.eng.hand == 3 and h.sweeps == [4, 4]
    with pytest.raises(AssertionError):
        h.room(40)                                                 # 20 + 40 > 0.9 x 64 even without tombstones: refused


def test_restore_marks_nothing_and_cuts_from_the_hand():
    S = 64
    rng = np.random.default_rng(4)
    h = ClockHandle(S, capacity=3)
    req = [int(k) for k in keys_homed_at([40, 8, 20, 2, 60], 0, S, rng)]
    h.restore([(0, r, [1]) for r in req], [(0, r ^ 1, r) for r in req])
    assert [k[1] for k in h.victims[0]] == [req[3], req[1]]        # slot order from slot 0
    assert h.req.hand == 9 and h.sweeps == [2, 0]


# ---- the home-slot replica and the snapshot decoder --------------------------------------------------------------------
def test_keys_homed_at_and_free_filter():
    rng = np.random.default_rng(5)
    for S in (1024, 1 << 21):
        slots = rng.integers(0, S // 2, 500) * 2
        for model in (0, 7, 65535):
            k = keys_homed_at(slots, model, S, rng)
            assert np.array_equal(_slot_home(k, model, S), slots)
    state = np.zeros(1024, np.int8)
    state[[10, 13, 500]] = (FULL, TOMB, FULL)
    k = keys_homed_at(np.array([10, 12, 12, 500, 502, 20]), 3, 1024, rng)
    assert list(keep_free(k, 3, state)) == [k[4], k[5]]            # 10, 12 (13 is a tombstone), 500 taken; one per pair
    got = draw_free(state, 300, 3, rng)
    homes = _slot_home(got, 3, 1024)
    assert len(set(homes.tolist())) == 300 and not np.isin(homes, [10, 12, 500]).any()
    assert (state[homes] == EMPTY).all() and (state[homes + 1] == EMPTY).all()


def test_decode_snapshot():
    hdr = np.zeros(8, "<u8")
    img = bytearray(hdr.tobytes())
    img[:8] = b"KVIDXSNP"
    img[32:48] = np.array([2, 1], "<u8").tobytes()
    img += np.array([(5, 1, 1, 0, [16] + [0] * 9), (9, 2, 1, 0, [32] + [0] * 9)],
                    [("hash", "<u8"), ("model", "<u2"), ("count", "u1"), ("zero", "u1"), ("ent", "<u2", (10,))]).tobytes()
    img += np.array([(7, 5, 1, b"")], [("hash", "<u8"), ("request", "<u8"), ("model", "<u2"), ("zero", "V6")]).tobytes()
    req, eng = decode_snapshot(bytes(img))
    assert req["hash"].tolist() == [5, 9] and req["model"].tolist() == [1, 2] and req["ent"][1, 0] == 32
    assert eng["hash"].tolist() == [7] and eng["request"].tolist() == [5] and eng["model"].tolist() == [1]
