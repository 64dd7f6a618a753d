"""GPU: hash-range sharded index.  Several handles in one process (kvidx_shard_attach) -- the same peer-memory mechanism
the one-process-per-GPU deployment gets through CUDA IPC (kvidx_shard_export / _import; tests/test_dist_gloo.py drives
that one with two processes).  "same-gpu" puts every shard on device 0, so the whole sharded code path (owner selection,
mapped tables, system-scope slot ownership, per-owner room checks, compaction) also runs on a one-GPU box; "multi-gpu"
spreads the shards over the devices there are and needs at least two."""
import numpy as np
import pytest

import kvidx
from kvidx import dist as kd
from kvidx import synth
from oracle.kvoracle_c import COracle

pytestmark = pytest.mark.gpu


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _devices(layout, world):
    if layout == "same-gpu":
        return [0] * world
    n = _n_gpus()
    if n < 2:
        pytest.skip("needs two GPUs")
    return [r % n for r in range(world)]


@pytest.mark.parametrize("layout,world", [("same-gpu", 2), ("same-gpu", 8), ("multi-gpu", 2), ("multi-gpu", 4)])
@pytest.mark.parametrize("path", ["coop", "rounds", "classes"])
def test_shards_one_process(path, layout, world, monkeypatch):
    monkeypatch.setenv("KVIDX_SCORE_PATH", path)   # coop | rounds | classes
    wl = synth.Workload(5, 1024, 1 << 14, 32)
    devs = _devices(layout, world)
    shards = [kvidx.Index(capacity=1 << 15, max_pods=32, device=devs[r], shard_rank=r, shard_count=world) for r in range(world)]
    with pytest.raises(kvidx.KvidxError):                      # not connected yet
        shards[0].score_batch(np.zeros(16, np.uint32), [0, 16])
    for r in range(world):
        for q in range(world):
            if q != r:
                shards[r].shard_attach(q, shards[q])
    co = COracle(size=10 ** 6, max_pods=32)
    ev, hs, tk = wl.fill_events(0, wl.D)
    assert co.apply_events(ev, hs, tk) == (0, 0)
    for r in range(world):                                     # each rank ingests its pods' events
        mine = kd.events_for_rank(ev, r, world)
        assert len(mine) > 0
        rc, dropped = shards[r].apply_events(mine, hs, tk)
        assert (rc, dropped) == (0, 0)
    st = [s.stats() for s in shards]
    assert sum(s["request_keys"] for s in st) == wl.n_blocks == co.len_request()
    assert all(s["request_keys"] > wl.n_blocks // (2 * world) for s in st)          # every shard holds a real share
    toks, doc, m = wl.queries(0, 3000)
    off = np.arange(0, (len(toks) + 1) * wl.T, wl.T, dtype=np.int64)
    exp, _, _, _ = co.score_batch(toks.reshape(-1), off, n_threads=4)
    for r in range(world):                                     # any rank can score any prompt
        lo, hi = kd.shard_range(len(toks), r, world)
        got, has = shards[r].score_batch(toks[lo:hi].reshape(-1), off[: hi - lo + 1])
        assert np.array_equal(got, exp[lo:hi]) and has.all()
    # Index API across shards: lookup / evict / get_request_key reach the owning shard from either rank
    k0, _ = shards[0].hash_keys(toks[0], [0, wl.T])
    rc, pt, cnt = shards[world - 1].lookup(0, k0[:8])
    rc2, pt2, cnt2 = co.lookup(0, k0[:8])
    # (entry ORDER inside a slot depends on how the two ranks' pods interleaved -- unspecified in the reference too)
    assert rc == rc2 == 0 and np.array_equal(cnt, cnt2) and all(sorted(pt[i, :cnt[i]]) == sorted(pt2[i, :cnt2[i]]) for i in range(8))
    e0 = int(wl.engine_hashes(int(doc[0]), int(doc[0]) + 1)[0, 0])
    assert shards[world - 1].get_request_key(0, e0) == co.get_request_key(0, e0)


@pytest.mark.parametrize("layout", ["same-gpu", "multi-gpu"])
def test_sharded_churn_compaction_and_full_owner(layout):
    """Steady BlockStored / BlockRemoved churn leaves tombstones on every owner.  A write batch first reads every owner's
    fill level through the mapped memory and answers KVIDX_ENOSPC instead of spinning on a full shard; kvidx_shard_compact
    (every rank, tables quiesced) drops the tombstones in place -- peers keep their mappings -- and the churn goes on.
    Index contents stay equal to the oracle's throughout."""
    world = 2
    devs = _devices(layout, world)
    shards = [kvidx.Index(capacity=2048, table_slots=4096, max_pods=16, device=devs[r], shard_rank=r, shard_count=world) for r in range(world)]
    for r in range(world):
        for q in range(world):
            if q != r:
                shards[r].shard_attach(q, shards[q])
    co = COracle(size=10 ** 6, max_pods=16)
    rng = np.random.default_rng(9)
    PTS = [(1 << 4), (2 << 4) | 1]
    live = {}
    saw_nospc = compactions = 0
    for rnd in range(40):
        eng = rng.integers(1, 1 << 62, 500, dtype=np.uint64)
        req = rng.integers(1, 1 << 62, 500, dtype=np.uint64)
        w = shards[rnd % world]
        rc = w.add(0, eng, req, PTS)
        if rc == kvidx.ENOSPC:
            saw_nospc += 1
            assert "tombstones" in w.last_error()
            for s in shards:                                   # the collective: every rank compacts its own shard
                s.shard_compact()
            compactions += 1
            rc = w.add(0, eng, req, PTS)
        assert rc == 0, w.last_error()
        assert co.add(0, eng, req, PTS) == 0
        for e in eng[:470]:
            assert shards[(rnd + 1) % world].evict(0, int(e), PTS) == 0 and co.evict(0, int(e), PTS) == 0
        for e, r in zip(eng[470:], req[470:]):
            live[int(e)] = int(r)
        st = [s.stats() for s in shards]
        assert sum(x["request_keys"] for x in st) == len(live) == co.len_request()
    assert saw_nospc >= 1 and compactions >= 1
    keys = np.array(list(live.values()), np.uint64)
    for s in shards:
        rc, pt, cnt = s.lookup(0, keys)
        assert rc == 0 and (cnt == 2).all()
    for e, r in list(live.items())[:40]:
        assert shards[0].get_request_key(0, e) == (0, r) and shards[1].get_request_key(0, e) == (0, r)
    # a shard that really is full (no tombstones to drop) keeps answering ENOSPC, and nothing hangs
    small = [kvidx.Index(capacity=256, table_slots=1024, max_pods=16, device=devs[r], shard_rank=r, shard_count=world) for r in range(world)]
    for r in range(world):
        small[r].shard_attach(1 - r, small[1 - r])
    big = rng.integers(1, 1 << 62, 4000, dtype=np.uint64)
    assert small[0].add(0, big, big, PTS) == kvidx.ENOSPC
