"""CPU: removing departed pods -- the removal spec (tests/remove_oracle.py), the opt-in AllBlocksCleared
marker of the host decoder, and pod-id reuse in the host mirror (host-only instance, no GPU)."""
import msgpack
import numpy as np
import pytest

from kvidx.host import EV_ALL_BLOCKS_CLEARED, HostIndexer
from oracle import kvoracle as ko
from remove_oracle import ClearingEventsPool, remove_pods

M = "m"


def K(h):
    return ko.Key(M, h)


def E(pod, tier="gpu"):
    return ko.PodEntry(pod, tier)


def test_remove_pods_keeps_survivor_order():
    ix = ko.InMemoryIndex()
    ix.add([K(1)], [K(100)], [E("a"), E("b"), E("c"), E("b", "cpu"), E("d")])
    assert remove_pods(ix, {"b"}) == (2, 0, 0)
    assert ix.lookup([K(100)]) == {K(100): [E("a"), E("c"), E("d")]}
    assert ix.get_request_key(K(1)) == K(100)


def test_remove_pods_drops_emptied_keys_and_their_engine_mappings():
    ix = ko.InMemoryIndex()
    ix.add([K(1), K(2)], [K(100), K(200)], [E("a")])
    ix.add([K(3)], [K(100)], [E("b")])                    # two engine keys map to request key 100
    ix.add([K(2)], [K(200)], [E("b")])
    assert remove_pods(ix, {"a", "b"}) == (4, 2, 3)
    assert ix.lookup([K(100), K(200)]) == {}
    for e in (1, 2, 3):
        with pytest.raises(ko.IndexError_):
            ix.get_request_key(K(e))
    assert len(ix.data) == 0 and len(ix.engine_to_request) == 0


def test_remove_pods_leaves_stale_mappings_of_already_absent_keys():
    ix = ko.InMemoryIndex(size=2)
    ix.add([K(1)], [K(100)], [E("a")])
    ix.add([K(2)], [K(200)], [E("b")])
    ix.add([K(3)], [K(300)], [E("c")])                    # capped: request key 100 and engine key 1 go
    ix.evict(K(9), [E("a")])                              # no-op
    ix.engine_to_request.add(K(4), K(100))               # a stale mapping (its request key is gone)
    assert remove_pods(ix, {"a"}) == (0, 0, 0)
    assert ix.get_request_key(K(4)) == K(100)            # stale: kept, Evict cleans it up lazily
    ix.add([K(5)], [K(500)], [E("x")])
    ix.engine_to_request.add(K(6), K(999))
    assert remove_pods(ix, {"x"}) == (1, 1, 1)
    assert ix.get_request_key(K(6)) == K(999)


def test_remove_pods_tier_mask_selects_entries():
    ix = ko.InMemoryIndex()
    ix.add([K(1)], [K(100)], [E("a"), E("a", "cpu"), E("b", "cpu")])
    ix.add([K(2)], [K(200)], [E("a", "gpu")])
    assert remove_pods(ix, {"a"}, {"gpu"}) == (2, 1, 1)
    assert ix.lookup([K(100)]) == {K(100): [E("a", "cpu"), E("b", "cpu")]}
    assert remove_pods(ix, {"a", "b"}, {"disk"}) == (0, 0, 0)
    assert remove_pods(ix, {"a", "b"}, {"cpu", "gpu"}) == (2, 1, 1)
    assert len(ix.data) == 0 and len(ix.engine_to_request) == 0


def test_remove_pods_changes_no_recency_in_a_capped_index():
    """Size=2: after a removal the next adds evict the same key they would evict had the removed keys never been there."""
    def run(with_removed):
        ix = ko.InMemoryIndex(size=2)
        ix.add([K(1)], [K(100)], [E("a")] + ([E("gone")] if with_removed else []))
        ix.add([K(2)], [K(200)], [E("b")])
        if with_removed:
            assert remove_pods(ix, {"gone"}) == (1, 0, 0)  # a refresh of key 100 here would make the next add evict 200
        ix.add([K(3)], [K(300)], [E("c")])                # evicts the least recent key: 100
        return ix.data.keys(), ix.engine_to_request.keys()
    assert run(True) == run(False) == ([K(200), K(300)], [K(2), K(3)])


def test_events_pool_all_blocks_cleared_option():
    tp = ko.ChunkedTokenDatabase(4)
    toks = list(range(100, 116))
    ev = [ko.BlockStored([1, 2], None, toks[:8]), ko.BlockStored([3], 2, toks[8:12], medium="CPU"), ko.AllBlocksCleared(),
          ko.BlockStored([4], 2, toks[8:12])]                # after a clear its parent is gone: the chain restarts
    for opt in (False, True):
        ix = ko.InMemoryIndex()
        pool = (ClearingEventsPool if opt else ko.EventsPool)(ix, tp)
        pool.digest_events("p", M, ev[:2])
        pool.digest_events("q", M, [ko.BlockStored([1], None, toks[:4])])
        pool.digest_events("p", M, ev[2:])
        k = tp.tokens_to_kv_block_keys(None, toks, M)
        restart = tp.tokens_to_kv_block_keys(None, toks[8:12], M)[0]
        got = ix.lookup(k[:3] + [restart])
        if not opt:
            assert got == {k[0]: [E("p"), E("q")], k[1]: [E("p")], k[2]: [E("p", "cpu"), E("p")]}
        else:                                             # the gpu entries of p before the clear are gone, cpu ones stay
            assert got == {k[0]: [E("q")], k[2]: [E("p", "cpu")], restart: [E("p")]}
            with pytest.raises(ko.IndexError_):
                ix.get_request_key(K(2))


# ---- host decoder: AllBlocksCleared marker -------------------------------------------------------------------------
def _payload(events):
    return msgpack.packb([1700000000.0, events, 0])


def test_decoder_marks_all_blocks_cleared_at_its_position():
    events = [["BlockStored", [11, 12], None, list(range(32)), 16, None, None], ["AllBlocksCleared"],
              ["BlockRemoved", [11], "CPU"], ["AllBlocksCleared", 7], ["BlockStored", [13], None, list(range(16)), 16, None, "gpu"]]
    plain = HostIndexer(no_device=True)
    opt = HostIndexer(no_device=True, clear_on_all_blocks_cleared=True)
    e0, h0, t0 = plain.decode("pod-x", "m", _payload(events))
    e1, h1, t1 = opt.decode("pod-x", "m", _payload(events))
    assert e0["op"].tolist() == [0, 1, 0]
    assert e1["op"].tolist() == [0, EV_ALL_BLOCKS_CLEARED, 1, EV_ALL_BLOCKS_CLEARED, 0]
    assert np.array_equal(e1[e1["op"] != EV_ALL_BLOCKS_CLEARED], e0) and np.array_equal(h0, h1) and np.array_equal(t0, t1)
    mk = e1[e1["op"] == EV_ALL_BLOCKS_CLEARED]
    assert (mk["podtier"] >> 4 == opt.pod_id("pod-x")).all() and (mk["n_hashes"] == 0).all() and (mk["n_tokens"] == 0).all()
    assert mk["model"].tolist() == [e1["model"][0]] * 2


# ---- host mirror: pod ids are freed and reused ----------------------------------------------------------------------
def test_pod_ids_are_reused_lowest_first():
    h = HostIndexer(no_device=True)
    assert [h.pod_id("p%d" % i) for i in range(5)] == [0, 1, 2, 3, 4]
    assert h.remove_pod("p3") == 0 and h.remove_pod("p1") == 0
    assert h.remove_pod("never-seen") == 0
    assert h.pod_id("new-a") == 1 and h.pod_id("new-b") == 3 and h.pod_id("new-c") == 5
    assert h.pod_id("p1") == 6                            # the old name is a new interning
    assert h.pod_id("p0") == 0 and h.pod_id("p4") == 4
    assert h.remove_pod("p0", tiers=["gpu"]) == 0         # some tiers only: the id stays
    assert h.pod_id("p0") == 0


def test_thousand_pods_churn_through_256_ids():
    h = HostIndexer(no_device=True, max_pods=256)
    alive = []
    for i in range(1000):
        name = "vllm-%d-%08x" % (i, (i * 2654435761) & 0xFFFFFFFF)
        assert h.add_task(name, "m", _payload([["BlockStored", [i + 1], None, list(range(16)), 16, None, None]])) == 0, h.err()
        alive.append(name)
        if len(alive) == 256:
            for n in alive[:128]:
                assert h.remove_pod(n) == 1                # its one queued message goes with it
            alive = alive[128:]
    assert max(h.pod_id(n) for n in alive) < 256


def test_queued_messages_of_a_removed_pod_are_dropped():
    h = HostIndexer(no_device=True, concurrency=1)
    msg = _payload([["BlockStored", [1], None, list(range(16)), 16, None, None]])
    for pod in ("a", "b", "a", "c", "a"):
        assert h.add_task(pod, "m", msg) == 0
    assert h.remove_pod("a") == 3
    assert h.remove_pod("a") == 0
    assert h.remove_pod("b", tiers=["cpu"]) == 1           # queued messages go whatever the tiers
    assert h.pod_id("b") == 1 and h.pod_id("c") == 2
