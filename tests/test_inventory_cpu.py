"""CPU: the pod inventory's spec (tests/inventory_oracle.py) against the removal spec (tests/remove_oracle.py) -- an
inventory says in advance what removing a pod drops --, the workload generator's closed form against the spec, and the
host mirror's inventory on a host-only instance (no GPU)."""
import copy
import ctypes as C

import numpy as np
import pytest

from inventory_oracle import dense, pod_inventory
from kvidx import _native, host, synth
from oracle import kvoracle as ko
from remove_oracle import remove_pods

MODELS = ("m0", "m1", "m2")
TIERS = tuple("t%d" % t for t in range(16))


def _random_index(rng, size, n_ops=600, P=12):
    """Random Add / Evict calls over three models, all sixteen tiers and few enough hashes that keys collect many pods, the
    same pod on several tiers, and stale engine mappings (a key under two engine keys emptied through one of them; with
    a small `size` also the two LRUs evicting independently)."""
    ix = ko.InMemoryIndex(size=size, pod_cache_size=10)
    for _ in range(n_ops):
        m = MODELS[int(rng.integers(0, 3))]
        req = [int(x) for x in rng.integers(0, 60, int(rng.integers(1, 4)))]
        eng = [r + 1000 * int(rng.integers(0, 2)) for r in req]          # two engine keys may map to one request key
        ents = [ko.PodEntry("p%d" % int(rng.integers(0, P)), TIERS[int(rng.integers(0, 16)) if rng.random() < 0.5 else 0])
                for _ in range(int(rng.integers(1, 4)))]
        u = rng.random()
        if u < 0.7:
            ix.add([ko.Key(m, e) for e in eng], [ko.Key(m, r) for r in req], ents)
        elif u < 0.8 and ko.Key(m, req[0]) in ix.data.d:
            ix.evict(ko.Key(m, eng[0]), ix.data.d[ko.Key(m, req[0])].keys())     # empties the key, whoever else maps to it
        else:
            ix.evict(ko.Key(m, eng[0]), ents)
    return ix


@pytest.mark.parametrize("seed,size", [(1, 10 ** 6), (2, 10 ** 6), (3, 40), (4, 25)])
def test_inventory_is_the_dry_run_of_removing_one_pod(seed, size):
    rng = np.random.default_rng(seed)
    ix = _random_index(rng, size)
    inv = pod_inventory(ix, None, engine=True)
    assert inv["totals"][0] == len(ix.data) and inv["totals"][2] == len(ix.engine_to_request)
    assert inv["totals"][1] == sum(inv["entries"].values()) == sum(len(pc) for pc in ix.data.d.values())
    assert inv["totals"][3] > 0 or size < 100
    assert any(c > 0 for c in inv["sole_engine"].values()) and max(len(pc) for pc in ix.data.d.values()) >= 6
    order = (ix.data.keys(), ix.engine_to_request.keys())
    for p in sorted(inv["keys"]):
        trial = copy.deepcopy(ix)
        want = (sum(c for (q, _), c in inv["entries"].items() if q == p), inv["sole"][p], inv["sole_engine"][p])
        assert remove_pods(trial, {p}) == want, p
        after = pod_inventory(trial, None, engine=True)
        assert after["keys"][p] == 0 and after["totals"][3] == inv["totals"][3]      # stale mappings stay
        assert all(after["keys"][q] == inv["keys"][q] for q in inv["keys"] if q != p)
    assert (ix.data.keys(), ix.engine_to_request.keys()) == order        # the spec itself refreshes no recency


def test_inventory_of_one_model_and_of_none():
    rng = np.random.default_rng(5)
    ix = _random_index(rng, 10 ** 6)
    parts = [pod_inventory(ix, m, engine=True) for m in MODELS]
    whole = pod_inventory(ix, None, engine=True)
    for name in ("entries", "keys", "sole", "sole_engine"):
        assert sum((p[name] for p in parts), type(whole[name])()) == whole[name]
    assert [sum(p["totals"][i] for p in parts) for i in range(4)] == whole["totals"]
    assert pod_inventory(ix, "unknown", engine=True)["totals"] == [0, 0, 0, 0]
    quick = pod_inventory(ix, None)
    assert quick["sole_engine"] is None and quick["totals"] == whole["totals"][:2] + [0, 0] and quick["sole"] == whole["sole"]
    empty = pod_inventory(ko.InMemoryIndex(), None, engine=True)
    assert empty["totals"] == [0, 0, 0, 0] and not empty["keys"]


def test_same_pod_on_two_tiers_counts_one_key_and_a_stale_mapping_is_counted():
    ix = ko.InMemoryIndex()
    K, E = (lambda h: ko.Key("m0", h)), ko.PodEntry
    ix.add([K(1), K(2)], [K(100), K(100)], [E("a", "t0"), E("a", "t1")])          # one request key under two engine keys
    ix.add([K(3)], [K(300)], [E("a", "t0"), E("b", "t0")])
    inv = pod_inventory(ix, None, engine=True)
    assert inv["entries"] == {("a", "t0"): 2, ("a", "t1"): 1, ("b", "t0"): 1}
    assert inv["keys"] == {"a": 2, "b": 1} and inv["sole"] == {"a": 1} and inv["sole_engine"] == {"a": 2}
    assert inv["totals"] == [2, 4, 3, 0]
    ix.evict(K(1), [E("a", "t0"), E("a", "t1")])                                   # evicted through one: the other goes stale
    assert pod_inventory(ix, None, engine=True)["totals"] == [1, 2, 2, 1]


@pytest.mark.parametrize("P", [1, 2, 3, 4, 16])
def test_generator_closed_form_matches_the_spec(P):
    wl = synth.Workload(1, 128, 64, P)
    ox = ko.Indexer(block_size=16, size=10 ** 6)
    pool = ko.EventsPool(ox.index, ox.tokens_processor)
    ev, hs, tk = wl.fill_events(0, wl.D)
    for r in ev:
        h = [int(x) for x in hs[r["hash_off"]: r["hash_off"] + r["n_hashes"]]]
        toks = [int(x) for x in tk[r["tok_off"]: r["tok_off"] + r["n_tokens"]]]
        pool.digest_events("p%d" % (int(r["podtier"]) >> 4), "m", [ko.BlockStored(h, int(r["parent_hash"]) if r["has_parent"] else None, toks,
                                                                                  medium=("gpu", "cpu")[int(r["podtier"]) & 15])])
    want = dense(pod_inventory(ox.index, None, engine=True), lambda s: int(s[1:]), ("gpu", "cpu").index, P)
    got = wl.expected_inventory()
    assert all(np.array_equal(want[k], got[k]) for k in want)


def test_host_only_instance_answers_zeros_with_the_right_names():
    h = host.HostIndexer(no_device=True, tiers=(("gpu", 1.0), ("cpu", 0.8)))
    assert h.pod_inventory() == {}
    for name in ("pod-a", "pod-b", "pod-c"):
        h.pod_id(name)
    assert h.remove_pod("pod-b") == 0                                      # frees id 1: skipped below
    zero = {"keys": 0, "sole_keys": 0, "sole_engine_keys": None, "entries": {}}
    assert h.pod_inventory() == {"pod-a": dict(zero, id=0), "pod-c": dict(zero, id=2)}
    pods, totals = h.pod_inventory(model="never-seen", engine=True, totals=True)
    assert pods == {"pod-a": dict(zero, id=0, sole_engine_keys=0), "pod-c": dict(zero, id=2, sole_engine_keys=0)} and totals == [0, 0, 0, 0]
    assert h.L.kvhost_model_id(h.h, b"never-seen") == 0                    # ... which the inventory did not intern
    h.pod_id('d"q')
    text = h.inventory_text()
    assert "# TYPE kvcache_index_pod_entries gauge\n# HELP kvcache_index_pod_keys" in text           # no entries: no samples
    assert 'kvcache_index_pod_keys{pod="pod-a"} 0\n' in text and 'kvcache_index_pod_sole_keys{pod="d\\"q"} 0\n' in text
    assert "pod-b" not in text and text.endswith("# TYPE kvcache_index_stale_engine_keys gauge\nkvcache_index_stale_engine_keys 0\n")
    assert "pod_keys" not in h.metrics_text()                              # the reference's metric set stays as it is
    rows = (host.PodRow * 1)()
    assert h.L.kvhost_pod_inventory(h.h, None, 0, rows, 1, None, None) == 3 and rows[0].pod == b"pod-a"   # more pods than room
    assert h.L.kvhost_pod_inventory(h.h, None, 0, None, 1, None, None) == _native.EINVAL


def test_inventory_signatures_load():
    L = _native.load()
    assert _native.SYMBOLS["kvidx_pod_inventory"][1][1:3] == [C.c_uint32, C.c_uint32] and L.kvidx_pod_inventory.restype is C.c_int
    assert (_native.ANY_MODEL, _native.INVENTORY_ENGINE) == (0xFFFFFFFF, 1)
    assert C.sizeof(host.PodRow) == 8 + 8 + 3 * 8 + 16 * 8
    assert L.kvidx_pod_inventory(None, 0, 0, None, None, None, None, None) == _native.EINVAL
