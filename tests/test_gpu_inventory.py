"""GPU (-m gpu): kvidx_pod_inventory / kvhost_pod_inventory -- what each pod holds -- against the spec of
tests/inventory_oracle.py applied to the same Add / Evict / event stream run through the Python oracle: every output array,
every capacity mode, sharded handles, beside a writer, and as the dry run of kvidx_remove_pods."""
import os
import socket
import threading
import time

import numpy as np
import pytest

import kvidx
from helpers import EVENT_DTYPE
from inventory_oracle import dense, pod_inventory
from kvidx import synth
from kvidx.host import HostIndexer
from oracle import kvoracle as ko
from remove_oracle import remove_pods
from test_gpu_parity import _random_stream

pytestmark = pytest.mark.gpu
ARRAYS = ("entries", "keys", "sole", "sole_engine", "totals")


def PT(p, t=0):
    return (p << 4) | t


def _ents(pts):
    return [ko.PodEntry("p%d" % (int(e) >> 4), "t%d" % (int(e) & 15)) for e in pts]


def _same(got, want, what=None):
    for k in ARRAYS:
        assert (got[k] is None and want[k] is None) or np.array_equal(got[k], want[k]), (what, k, got[k], want[k])


class Twin:
    """A handle and the oracle's index fed the same calls; models are ids here and "m<id>" there, pods "p<id>", tiers "t<id>"."""

    def __init__(self, P=64, pods_per_key=10, capacity=1 << 14, lru_exact=0, **kw):
        self.P = P
        self.ix = kvidx.Index(hash_seed="abc", capacity=capacity, pods_per_key=pods_per_key, max_pods=P, lru_exact=lru_exact, **kw)
        self.ox = ko.Indexer(block_size=16, hash_seed="abc", size=capacity if lru_exact else 10 ** 8, pod_cache_size=pods_per_key)
        self.pool = ko.EventsPool(self.ox.index, self.ox.tokens_processor)
        self.also = []                   # callables giving further handles that get every Add / Evict (sharded tests)

    def handles(self):
        return [self.ix] + [f() for f in self.also]

    def add(self, model, eng, req, pts):
        for ix in self.handles():
            assert ix.add(model, eng, req, pts) == 0, ix.last_error()
        m = "m%d" % model
        self.ox.index.add([ko.Key(m, int(e)) for e in eng], [ko.Key(m, int(r)) for r in req], _ents(pts))

    def evict(self, model, eng, pts):
        for ix in self.handles():
            assert ix.evict(model, int(eng), pts) == 0, ix.last_error()
        self.ox.index.evict(ko.Key("m%d" % model, int(eng)), _ents(pts))

    def event(self, r, hs, tk):
        assert self.ix.apply_events(np.array([r], EVENT_DTYPE), hs, tk)[0] == 0, self.ix.last_error()
        h = [int(x) for x in hs[r["hash_off"]: r["hash_off"] + r["n_hashes"]]]
        if r["op"] == 0:
            toks = [int(x) for x in tk[r["tok_off"]: r["tok_off"] + r["n_tokens"]]]
            ev = ko.BlockStored(h, int(r["parent_hash"]) if r["has_parent"] else None, toks, medium="t%d" % (int(r["podtier"]) & 15))
        else:
            ev = ko.BlockRemoved(h, medium="t%d" % (int(r["podtier"]) & 15))
        self.pool.digest_events("p%d" % (int(r["podtier"]) >> 4), "m%d" % int(r["model"]), [ev])

    def want(self, model=None, engine=False):
        inv = pod_inventory(self.ox.index, None if model is None else "m%d" % model, engine)
        return dense(inv, lambda s: int(s[1:]), lambda s: int(s[1:]), self.P)

    def check(self, models=(0, 1, 2), ix=None):
        """Every output, with and without the engine pass, for each model and for all; quiescent totals are the stats'."""
        ix = ix or self.ix
        for model in (None,) + tuple(models):
            for engine in (False, True):
                _same(ix.pod_inventory(model, engine), self.want(model, engine), (model, engine))
        st, tot = ix.stats(), ix.pod_inventory(None, True)["totals"]
        assert (st["request_keys"], st["engine_keys"]) == (int(tot[0]), int(tot[2]))
        return self.want(None, True)

    def random_ops(self, rng, n, pods, n_hash=80, models=3, evict_all=0.08):
        """Random Add / Evict calls: few hashes (keys collect up to ten pods), two engine keys per request key (emptying a key
        through one leaves the other mapping stale), every tier, the same pod on several tiers."""
        pods = np.asarray(pods)
        for _ in range(n):
            m = int(rng.integers(0, models))
            req = rng.integers(1, n_hash + 1, int(rng.integers(1, 4))).astype(np.uint64)
            eng = req + np.uint64(1000 * int(rng.integers(0, 2)))
            pts = [PT(int(pods[int(rng.integers(0, len(pods)))]), int(rng.integers(0, 16)) if rng.random() < 0.5 else 0)
                   for _ in range(int(rng.integers(1, 5)))]
            u, k0 = rng.random(), ko.Key("m%d" % m, int(req[0]))
            if u < 0.7:
                self.add(m, eng, req, pts)
            elif u < 0.7 + evict_all and k0 in self.ox.index.data.d:
                self.evict(m, eng[0], [PT(int(e.pod[1:]), int(e.tier[1:])) for e in self.ox.index.data.d[k0].keys()])
            else:
                self.evict(m, eng[0], pts)


# ---- 1. event streams: several models, sixteen tiers, pod-cache overflow ---------------------------------------------------
@pytest.mark.parametrize("pods_per_key", [4, 10])
def test_event_streams_over_models_and_tiers_vs_spec(pods_per_key):
    rng = np.random.default_rng(100 + pods_per_key)
    BS, P, NT = 16, 40, 16
    tw = Twin(P=64, pods_per_key=pods_per_key)
    docs = [rng.integers(0, 128256, size=BS * int(rng.integers(1, 24))).tolist() for _ in range(12)]
    streams = [_random_stream(rng, 350, BS, P, NT, docs, model=m) for m in range(3)]
    for i in range(350):
        for ev, hs, tk in streams:
            tw.event(ev[i], hs, tk)
        if i % 70 == 69:
            tw.check()
    inv = tw.check()
    counts = [len(pc) for pc in tw.ox.index.data.d.values()]
    assert max(counts) >= min(pods_per_key, 6) and (inv["entries"].sum(0) > 0).all() and inv["sole"].sum() > 0   # crowded keys, all tiers


def test_ten_entries_and_one_pod_on_two_tiers_of_a_key():
    tw = Twin(P=16)
    tw.add(0, [1, 2], [100, 200], [PT(p, p % 3) for p in range(12)])          # twelve entries into ten places: pods 0, 1 drop out
    tw.add(1, [3], [100], [PT(5, 0), PT(5, 7), PT(5, 15)])                      # one pod, three tiers: one key, sole
    tw.add(1, [4], [100], [PT(5, 0)])                                           # a second engine key of it
    inv = tw.check(models=(0, 1))
    assert inv["keys"][5] == 3 and inv["entries"][5].tolist() == [1, 0, 2] + [0] * 4 + [1] + [0] * 7 + [1]
    assert inv["sole"].tolist() == [0] * 5 + [1] + [0] * 10 and inv["sole_engine"][5] == 2 and inv["keys"][:2].tolist() == [0, 0]
    assert inv["totals"].tolist() == [3, 23, 4, 0]


# ---- 2. the width of the histograms: shared memory up to 512 pods, global atomics beyond ---------------------------------
@pytest.mark.parametrize("P", [1, 64, 257, 512, 513, 4096])
def test_every_max_pods_counts_its_highest_pod_and_tier_15(P):
    rng = np.random.default_rng(P)
    tw = Twin(P=P)
    pods = sorted({0, P - 1, P // 2} | set(rng.integers(0, P, 12).tolist()))
    tw.add(2, [7, 8, 9], [70, 80, 90], [PT(P - 1, 15)])
    tw.random_ops(rng, 300, pods)
    tw.add(0, np.arange(5000, 5600, dtype=np.uint64), np.arange(7000, 7600, dtype=np.uint64), [PT(P - 1, 15), PT(0, 15)][:min(P, 2)])
    inv = tw.check()
    assert inv["entries"][P - 1, 15] >= 600 and inv["keys"][P - 1] >= 600 and (P > 1 or inv["sole"][0] == inv["totals"][0])


# ---- 3. the dry run of kvidx_remove_pods ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("lru_exact", [0, 1])
def test_inventory_says_what_removing_each_pod_drops(lru_exact):
    rng = np.random.default_rng(31 + lru_exact)
    tw = Twin(P=64, lru_exact=lru_exact)
    tw.random_ops(rng, 900, np.arange(14), n_hash=120)
    removed = np.zeros(3, np.int64)
    for p in rng.permutation(14)[:12].tolist():
        inv = tw.ix.pod_inventory(None, True)
        want = (int(inv["entries"][p].sum()), int(inv["sole"][p]), int(inv["sole_engine"][p]))
        got = tw.ix.remove_pods([p])
        assert (got["entries"], got["request_keys"], got["engine_keys"]) == want, p
        assert remove_pods(tw.ox.index, {"p%d" % p}) == want
        after = tw.check()
        assert after["entries"][p].sum() == 0 and after["keys"][p] == 0 and after["sole"][p] == 0 and after["sole_engine"][p] == 0
        removed += want
        tw.random_ops(rng, 40, np.setdiff1d(np.arange(14), [p]), n_hash=120)
    assert (removed > 0).all(), removed


# ---- 4. stale engine mappings -----------------------------------------------------------------------------------------------
def test_a_key_evicted_through_one_of_two_engine_keys_leaves_one_stale_mapping():
    tw = Twin(P=8)
    tw.add(0, [1, 2], [100, 100], [PT(3)])
    assert tw.check(models=(0,))["totals"].tolist() == [1, 1, 2, 0]
    tw.evict(0, 1, [PT(3)])
    assert tw.check(models=(0,))["totals"].tolist() == [0, 0, 1, 1]
    assert tw.ix.pod_inventory()["totals"].tolist() == [0, 0, 0, 0]            # without the engine pass the engine side is not counted


def test_capped_exact_lru_stream_grows_stale_mappings_by_itself():
    """Both maps capped at 48 keys, three engine keys per request key, Lookups that refresh request keys only: keys emptied
    through one engine key leave the others' mappings stale until the engine LRU drops them.  Inventories are taken all
    along; had one of them refreshed anything, later evictions would pick other victims than the oracle's."""
    rng = np.random.default_rng(44)
    CAP = 48
    tw = Twin(P=16, capacity=CAP, lru_exact=1, pods_per_key=4)
    stale = 0
    for step in range(700):
        m, k = int(rng.integers(0, 2)), int(rng.integers(1, 90))
        u = rng.random()
        if u < 0.6:
            tw.add(m, [k + 1000 * int(rng.integers(0, 3))], [k], [PT(int(rng.integers(0, 9)), int(rng.integers(0, 2)))])
        elif u < 0.75:
            pc = tw.ox.index.data.d.get(ko.Key("m%d" % m, k))
            pts = [PT(int(e.pod[1:]), int(e.tier[1:])) for e in pc.keys()] if pc is not None and rng.random() < 0.6 else [PT(int(rng.integers(0, 9)))]
            tw.evict(m, k + 1000 * int(rng.integers(0, 3)), pts)
        else:
            keys = rng.integers(1, 90, 3).astype(np.uint64)
            rc, pt, cnt = tw.ix.lookup(m, keys)
            got = {int(keys[i]): [int(e) for e in pt[i, :cnt[i]]] for i in range(3) if cnt[i]}
            want = tw.ox.index.lookup([ko.Key("m%d" % m, int(x)) for x in keys])
            assert rc == 0 and got == {k_.chunk_hash: [PT(int(e.pod[1:]), int(e.tier[1:])) for e in v] for k_, v in want.items()}, step
        if step % 25 == 24:
            stale = max(stale, int(tw.check(models=(0, 1))["totals"][3]))
    assert stale > 0 and tw.ix.stats()["request_keys"] == CAP


# ---- 5. the shape of the table does not matter ---------------------------------------------------------------------------
def test_high_load_tombstones_rebuild_restore_and_an_empty_handle():
    rng = np.random.default_rng(5)
    tw = Twin(P=16, capacity=1024, table_slots=4096)
    assert tw.check()["totals"].tolist() == [0, 0, 0, 0]                        # a handle with no key at all
    eng = rng.integers(1, 1 << 62, 3000, dtype=np.uint64)
    req = rng.integers(1, 1 << 62, 3000, dtype=np.uint64)

    def pts_of(i):
        return [PT(i // 500), PT(15, 15), PT((i // 500 + 1) % 6, 1)][:1 + i // 1000]
    for i in range(0, 3000, 500):                                               # load 0.73: long displaced probe chains
        tw.add(i // 1500, eng[i:i + 500], req[i:i + 500], pts_of(i))
    tw.check()
    for i in range(0, 2000, 2):                                                 # tombstones in the middle of the chains
        tw.evict(i // 1500, eng[i], pts_of(i))
    st = tw.ix.stats()
    assert st["request_tombs"] >= 900 and st["rebuilds"] == 0
    tw.check()
    while tw.ix.stats()["rebuilds"] == 0:                                       # churn until the write path compacts
        e = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
        tw.add(2, e, e, [PT(7, 3)])
        for x in e[:280]:
            tw.evict(2, x, [PT(7, 3)])
    inv = tw.check()
    fresh = kvidx.Index(hash_seed="abc", capacity=1 << 14, pods_per_key=10, max_pods=16)
    fresh.restore(tw.ix.snapshot())
    tw.check(ix=fresh)
    assert inv["totals"][0] > 2000 and inv["sole"].sum() > 0


# ---- 6. it only reads ---------------------------------------------------------------------------------------------------
def test_exact_lru_snapshot_with_recency_is_byte_identical_around_an_inventory():
    rng = np.random.default_rng(6)
    tw = Twin(P=16, capacity=1 << 12, lru_exact=1)                              # recency is tracked; nothing is evicted
    tw.random_ops(rng, 400, np.arange(12), n_hash=150)
    before = tw.ix.snapshot()
    for model in (None, 0, 1):
        tw.ix.pod_inventory(model, True)
    assert tw.ix.snapshot() == before and len(before) > 64 + 40 * 100
    tw.check()


def test_clock_twins_evict_the_same_keys_whether_or_not_one_takes_inventories():
    """CLOCK at capacity: the next sweep's victims depend on the reference bits.  Two handles get the same calls, one of them
    also takes inventories; they must end with the same contents and the same eviction counts."""
    rng = np.random.default_rng(61)
    a, b = (kvidx.Index(capacity=64, table_slots=1024, max_pods=16, evict_policy="clock") for _ in range(2))
    for step in range(500):
        k = int(rng.integers(1, 400))
        for ix in (a, b):
            if step % 3 == 2:
                ix.get_request_key(0, k)                                         # sets the mapping's reference bit when present
                ix.lookup(0, np.array([k + 5000], np.uint64))                    # ... and the request key's
            else:
                assert ix.add(0, [k], [k + 5000], [PT(k % 16, k % 2)]) == 0
        if step % 5 == 0:
            inv = b.pod_inventory(None, True)
            assert inv["totals"][0] <= 64 and inv["totals"][2] <= 64
    assert a.snapshot() == b.snapshot() and a.evictions() == b.evictions() and a.evictions()[0] > 100
    assert a.sweeps() == b.sweeps()


# ---- 7. sharded handles ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 8])
def test_shard_inventories_sum_to_the_unsharded_answer(world):
    rng = np.random.default_rng(70 + world)
    P = 32
    shards = [kvidx.Index(hash_seed="abc", capacity=1 << 14, max_pods=P, shard_rank=r, shard_count=world) for r in range(world)]
    with pytest.raises(kvidx.KvidxError):                                       # not connected yet
        shards[0].pod_inventory()
    for r in range(world):
        for q in range(world):
            if q != r:
                shards[r].shard_attach(q, shards[q])
    tw = Twin(P=P)                                                              # the unsharded twin and the oracle ...
    turn = iter(range(10 ** 9))
    tw.also = [lambda: shards[next(turn) % world]]                              # ... and every call also through some rank
    tw.random_ops(rng, 700, np.arange(20), n_hash=300)
    plain = tw.ix
    whole = tw.check()
    assert whole["totals"][3] > 0 and whole["sole_engine"].sum() > 0
    for model in (None, 1):
        for engine in (False, True):
            parts = [s.pod_inventory(model, engine) for s in shards]
            total = {k: None if parts[0][k] is None else sum(p[k] for p in parts) for k in ARRAYS}
            _same(total, plain.pod_inventory(model, engine), (model, engine))
    parts = [s.pod_inventory(None, True) for s in shards]
    for s, p in zip(shards, parts):                                             # a rank reports what it owns
        st = s.stats()
        assert (st["request_keys"], st["engine_keys"]) == (int(p["totals"][0]), int(p["totals"][2]))
    assert sum(1 for p in parts if p["totals"][0] > 0) == world


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker_inventory(rank, world, port, q):
    """One process per rank (gloo for the collectives, CUDA IPC for the shards): every rank gets the fleet-wide inventory."""
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import torch
        from kvidx import dist as kd
        wl = synth.Workload(3, 512, 1 << 12, 16)
        ix = kvidx.Index(capacity=1 << 13, max_pods=16, device=rank % torch.cuda.device_count(), shard_rank=rank, shard_count=world)
        kd.connect_shards(ix)
        ev, hs, tk = wl.fill_events(0, wl.D)
        assert ix.apply_events(kd.events_for_rank(ev, rank, world), hs, tk) == (0, 0)
        dist.barrier()
        mine = ix.pod_inventory(None, True)
        assert 0 < mine["totals"][0] < wl.n_blocks
        _same(kd.pod_inventory_shards(ix, None, True), wl.expected_inventory())
        quick = kd.pod_inventory_shards(ix)
        assert quick["sole_engine"] is None and np.array_equal(quick["keys"], wl.expected_inventory()["keys"])
        q.put((rank, True))
    except Exception:      # noqa: BLE001
        import traceback
        q.put((rank, traceback.format_exc()[-900:]))
    finally:
        dist.destroy_process_group()


def test_pod_inventory_shards_two_ranks_cuda_ipc():
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker_inventory, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert all(r[1] is True for r in res), res


# ---- 9. beside a writer ---------------------------------------------------------------------------------------------------
def test_inventories_beside_a_writer_count_every_key_before_or_after_each_update():
    """500 keys of pod 1 stay; a writer adds 64 keys of pod 2 (two entries each) and evicts them one by one, over and over.
    Every inventory taken meanwhile returns, and sees between 500 and 564 keys, pod 1 whole, and of each churned key both
    entries or none."""
    rng = np.random.default_rng(9)
    ix = kvidx.Index(capacity=1 << 12, max_pods=64)
    base = rng.integers(1, 1 << 62, 500, dtype=np.uint64)
    assert ix.add(0, base, base, [PT(1)]) == 0
    stop, errs, rounds, seen = threading.Event(), [], [0], []

    def writer():
        try:
            while not stop.is_set():
                k = rng.integers(1, 1 << 62, 64, dtype=np.uint64)
                assert ix.add(0, k, k, [PT(2), PT(2, 1)]) == 0
                for x in k:
                    assert ix.evict(0, int(x), [PT(2), PT(2, 1)]) == 0
                rounds[0] += 1
        except Exception as ex:                                       # noqa: BLE001
            errs.append(ex)

    def reader():
        try:
            while not stop.is_set():
                inv = ix.pod_inventory(None, True)
                n = int(inv["totals"][0])
                assert 500 <= n <= 564 and inv["keys"][1] == 500 and inv["entries"][1, 0] == 500, inv["totals"]
                assert inv["keys"][2] == n - 500 == inv["entries"][2, 0] == inv["entries"][2, 1] == inv["sole"][2], (n, inv["entries"][2, :2])
                assert inv["totals"][1] == 500 + 2 * (n - 500) and 500 <= inv["totals"][2] <= 564 and inv["totals"][3] <= 64
                seen.append(n)
        except Exception as ex:                                       # noqa: BLE001
            errs.append(ex)

    ths = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(2)]
    for t in ths:
        t.start()
    time.sleep(2.0)
    stop.set()
    for t in ths:
        t.join()
    assert not errs, errs[:2]
    assert rounds[0] > 3 and len(seen) > 20 and len(set(seen)) > 1
    assert ix.pod_inventory(None, True)["totals"].tolist() == [500, 500, 500, 0]


# ---- 10. the host mirror ----------------------------------------------------------------------------------------------------
def test_host_inventory_names_freed_ids_tiers_and_models():
    h = HostIndexer(capacity=4096, max_pods=4, tiers=(("gpu", 1.0), ("cpu", 0.8)))
    K = list(range(100, 110))
    E = [k ^ 0x55 for k in K]

    def add(model, pod, tier, n, off=0):
        assert h.add(model, E[off:off + n], K[off:off + n], [(pod, tier)]) == 0, h.err()

    add("m", "a", "gpu", 6); add("m", "b", "cpu", 3); add("m", "a", "CPU", 2); add("n", "c", "disk", 4); add("m", "c", "gpu", 2, off=8)
    pods, totals = h.pod_inventory(engine=True, totals=True)
    assert pods == {"a": {"id": 0, "keys": 6, "sole_keys": 3, "sole_engine_keys": 3, "entries": {"gpu": 6, "cpu": 2}},
                    "b": {"id": 1, "keys": 3, "sole_keys": 0, "sole_engine_keys": 0, "entries": {"cpu": 3}},
                    "c": {"id": 2, "keys": 6, "sole_keys": 6, "sole_engine_keys": 6, "entries": {"disk": 4, "gpu": 2}}}
    assert totals == [12, 17, 12, 0]
    assert h.pod_inventory(model="n") == {"a": {"id": 0, "keys": 0, "sole_keys": 0, "sole_engine_keys": None, "entries": {}},
                                          "b": {"id": 1, "keys": 0, "sole_keys": 0, "sole_engine_keys": None, "entries": {}},
                                          "c": {"id": 2, "keys": 4, "sole_keys": 4, "sole_engine_keys": None, "entries": {"disk": 4}}}
    assert h.pod_inventory(model="never-seen", engine=True, totals=True)[1] == [0, 0, 0, 0]
    text = h.inventory_text()
    for line in ('kvcache_index_pod_entries{pod="a",tier="cpu"} 2', 'kvcache_index_pod_entries{pod="c",tier="disk"} 4', 'kvcache_index_pod_keys{pod="b"} 3',
                 'kvcache_index_pod_sole_keys{pod="a"} 3', 'kvcache_index_pod_sole_engine_keys{pod="c"} 6', "kvcache_index_stale_engine_keys 0"):
        assert line + "\n" in text, line
    assert h.remove_pod("a") == 0                                               # a's id is freed: no row, nothing counted for it
    pods = h.pod_inventory(engine=True)
    assert sorted(pods) == ["b", "c"] and pods["b"]["sole_keys"] == 3 and h.pod_inventory(engine=True, totals=True)[1] == [9, 9, 9, 0]
    add("m", "e", "gpu", 5)                                                     # takes id 0
    pods = h.pod_inventory(engine=True)
    assert pods["e"] == {"id": 0, "keys": 5, "sole_keys": 2, "sole_engine_keys": 2, "entries": {"gpu": 5}} and pods["b"]["sole_keys"] == 0
    assert h.evict("m", E[9], [("c", "gpu")]) == 0 and h.add("m", [777], [K[8]], [("c", "gpu")]) == 0
    assert h.evict("m", E[8], [("c", "gpu")]) == 0                              # key 108 emptied through one engine key: 777 goes stale
    assert h.pod_inventory(engine=True, totals=True)[1][3] == 1 and "kvcache_index_stale_engine_keys 1\n" in h.inventory_text()


# ---- 11. argument errors ----------------------------------------------------------------------------------------------------
def test_inventory_argument_errors():
    import ctypes as C
    ix = kvidx.Index(capacity=1024, max_pods=8)
    assert ix.add(0, [1], [2], [PT(7, 15)]) == 0
    u64p = C.POINTER(C.c_uint64)
    tot = np.zeros(4, np.uint64)
    call = ix.L.kvidx_pod_inventory
    assert call(ix.h, 0, 0, None, None, None, None, None) == kvidx.EINVAL and "NULL" in ix.last_error()
    assert call(ix.h, 0x10000, 0, None, None, None, None, tot.ctypes.data_as(u64p)) == kvidx.ERANGE
    assert call(ix.h, 0, 2, None, None, None, None, tot.ctypes.data_as(u64p)) == kvidx.EINVAL
    assert call(None, 0, 0, None, None, None, None, tot.ctypes.data_as(u64p)) == kvidx.EINVAL
    assert call(ix.h, 0xFFFFFFFF, 1, None, None, None, None, tot.ctypes.data_as(u64p)) == 0 and tot.tolist() == [1, 1, 1, 0]
    keys = np.zeros(8, np.uint64)
    assert call(ix.h, 0xFFFF, 0, None, keys.ctypes.data_as(u64p), None, None, None) == 0 and not keys.any()      # another model: nothing
    with pytest.raises(kvidx.KvidxError) as ei:
        ix.pod_inventory(model=1 << 20)
    assert ei.value.code == kvidx.ERANGE
    inv = ix.pod_inventory(0)
    assert inv["entries"][7, 15] == 1 and inv["sole_engine"] is None and inv["totals"].tolist() == [1, 1, 0, 0]
