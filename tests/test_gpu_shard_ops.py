"""GPU (-m gpu): pod removal, snapshot and restore on a hash-range sharded index (kvidx_shard_remove_pods,
kvidx_shard_snapshot + kvidx_snapshot_merge, kvidx_shard_restore) -- bit-exact against the Python oracle with the removal
spec of tests/remove_oracle.py, byte-exact against the unsharded snapshot, through resharding 1 -> 2 -> 8 -> 1.
Several handles in one process (kvidx_shard_attach): "same-gpu" puts every shard on device 0 and always runs, "multi-gpu"
needs two GPUs.  The two-process form (CUDA IPC, gloo, kvidx.dist) is the last test."""
import os
import socket
import threading

import numpy as np
import pytest

from helpers import csr
import kvidx
from oracle import kvoracle as ko
from remove_oracle import remove_pods
from test_gpu_parity import _random_stream
from test_gpu_remove_pods import MODEL, PT, TIERS, W, _check_state, _dense, _oracle_apply, _oracle_scores, _pair, _prompts
from test_gpu_sharded import _devices
from test_gpu_snapshot import _encode, _fresh

pytestmark = pytest.mark.gpu
LAYOUTS = [("same-gpu", 2), ("same-gpu", 8), ("multi-gpu", 2)]


def _shards(world, layout="same-gpu", connect=True, **kw):
    devs = _devices(layout, world)
    cfg = dict(block_size=16, hash_seed="abc", capacity=1 << 16, pods_per_key=4, tier_weights=W, max_pods=16)
    cfg.update(kw)
    sh = [kvidx.Index(**cfg, device=devs[r], shard_rank=r, shard_count=world) for r in range(world)]
    if connect:
        for r in range(world):
            for q in range(world):
                if q != r:
                    sh[r].shard_attach(q, sh[q])
    return sh


class _Whole:
    """The sharded set seen as one index: key counts summed over shards, reads through one rank."""

    def __init__(self, shards, via=0):
        self.shards, self.via = shards, via

    def stats(self):
        st = [s.stats() for s in self.shards]
        return {k: sum(x[k] for x in st) for k in ("request_keys", "engine_keys", "request_tombs", "engine_tombs")}

    def lookup(self, *a):
        return self.shards[self.via].lookup(*a)

    def get_request_key(self, *a):
        return self.shards[self.via].get_request_key(*a)


def _remove_collective(shards, pods, tiers=None):
    r0 = [s.shard_remove_pods(pods, tiers, phase=0) for s in shards]
    r1 = [s.shard_remove_pods(pods, tiers, phase=1) for s in shards]
    assert all(r["engine_keys"] == 0 for r in r0) and all(r["entries"] == r["request_keys"] == 0 for r in r1)
    return sum(r["entries"] for r in r0), sum(r["request_keys"] for r in r0), sum(r["engine_keys"] for r in r1)


def _merged(shards):
    return kvidx.snapshot_merge([s.shard_snapshot() for s in shards])


def _restore_all(shards, image):
    got = [s.shard_restore(image) for s in shards]
    return sum(g["request_keys"] for g in got), sum(g["engine_keys"] for g in got)


def _docs(rng, BS=16):
    docs = [rng.integers(0, 128256, size=BS * int(rng.integers(1, 30))).tolist() for _ in range(24)]
    for i in range(8, 24):
        docs[i] = docs[i % 8][:BS * int(rng.integers(1, 6))] + docs[i]
    return docs


def _add_stale(ixs, ox, step, engine_keys):
    """Two engine keys -> one request key, evicted through the first: the second mapping is left stale."""
    e1, e2, rk = 0xDEAD0000 + step, 0xDEAD1000 + step, 0xBEEF0000 + step
    for ix in ixs:
        assert ix.add(0, [e1, e2], [rk, rk], [PT(15)]) == 0 and ix.evict(0, e1, [PT(15)]) == 0
    ox.index.add([ko.Key(MODEL, e1), ko.Key(MODEL, e2)], [ko.Key(MODEL, rk)] * 2, [ko.PodEntry("p15", "gpu")])
    ox.index.evict(ko.Key(MODEL, e1), [ko.PodEntry("p15", "gpu")])
    engine_keys += [e1, e2]


@pytest.mark.parametrize("layout,world", LAYOUTS)
def test_collective_removal_and_canonical_images_vs_oracle(layout, world):
    """One random BlockStored / BlockRemoved stream (one event per call, all through rank 0, so the entry order inside
    each slot is the oracle's) goes into an unsharded handle, a sharded set and the oracle, with stale mappings and a
    removal of a random pod set -- on all tiers or a random tier set -- after every 16 events.  The collective removal's
    summed counters equal kvidx_remove_pods' and the oracle's; state and Score() through every rank stay bit-exact; the
    merged shard snapshots are byte-identical to the unsharded snapshot and to the spec's encoding."""
    rng = np.random.default_rng(world * 10 + (layout == "multi-gpu"))
    BS, P, NT = 16, 12, 3
    ix, ox, pool = _pair(P=16)
    shards = _shards(world, layout)
    docs = _docs(rng)
    ev, hs, tk = _random_stream(rng, 400, BS, P, NT, docs)
    prompts = _prompts(rng, docs, 32, BS)
    pkeys = [ox.tokens_processor.tokens_to_kv_block_keys(None, p, MODEL) for p in prompts]
    tok, off = csr(prompts)
    seen, engine_keys = set(), sorted({int(x) for x in hs})
    removed, stale = np.zeros(3, np.int64), 0
    for step in range(25):
        for i in range(16 * step, 16 * (step + 1)):
            assert ix.apply_events(ev[i:i + 1], hs, tk)[0] == 0
            assert shards[0].apply_events(ev[i:i + 1], hs, tk)[0] == 0
            _oracle_apply(pool, ev[i], hs, tk)
            seen |= {k.chunk_hash for k in ox.index.data.d}
        if step in (3, 15):
            _add_stale((ix, shards[0]), ox, step, engine_keys)
        pods = sorted(rng.choice(P, size=int(rng.integers(1, 4)), replace=False).tolist())
        tiers = None if rng.random() < 0.5 else sorted(rng.choice(NT, size=int(rng.integers(1, NT + 1)), replace=False).tolist())
        want = remove_pods(ox.index, {"p%d" % p for p in pods}, None if tiers is None else {TIERS[t] for t in tiers})
        got = ix.remove_pods(pods, tiers)
        assert (got["entries"], got["request_keys"], got["engine_keys"]) == want
        assert _remove_collective(shards, pods, tiers) == want, (step, pods, tiers)
        removed += want
        _check_state(_Whole(shards, step % world), ox, seen, engine_keys)
        exp = np.stack([_dense(_oracle_scores(ox, k), 16) for k in pkeys])
        s, _ = shards[(step + 1) % world].score_batch(tok, off)
        assert np.array_equal(s, exp), step
        if step in (10, 24):
            img = ix.snapshot()
            assert _merged(shards) == img == _encode(ox), step
            stale = max(stale, sum(rk not in ox.index.data.d for rk in ox.index.engine_to_request.d.values()))
    assert (removed > 0).all() and stale > 0


def _scores_ok(ix, ox, pkeys, tok_off):
    exp = np.stack([_dense(_oracle_scores(ox, k), 16) for k in pkeys])
    for n, (tok, off) in tok_off.items():
        s, _ = ix.score_batch(tok, off)
        assert np.array_equal(s, exp[np.arange(n) % len(pkeys)]), n


@pytest.mark.parametrize("chain", [("same-gpu", (2, 8)), ("multi-gpu", (2,))])
@pytest.mark.parametrize("path", ["coop", "rounds", "classes"])
def test_resharding_round_trips(path, chain, monkeypatch):
    """An unsharded image restored into 2 shards, their merged image into 8, and theirs into one unsharded handle again:
    after each restore, Lookup / GetRequestKey / key counts and Score() on the path through every rank are bit-exact
    against the oracle, and the snapshot taken back is byte-identical to the image restored.  A single part restores
    to exactly that part's keys."""
    monkeypatch.setenv("KVIDX_SCORE_PATH", path)
    layout, worlds = chain
    rng = np.random.default_rng(77)
    BS, P, NT = 16, 12, 3
    ix, ox, pool = _pair(P=16)
    docs = _docs(rng)
    ev, hs, tk = _random_stream(rng, 300, BS, P, NT, docs)
    seen, engine_keys = set(), sorted({int(x) for x in hs})
    for i in range(len(ev)):
        assert ix.apply_events(ev[i:i + 1], hs, tk)[0] == 0
        _oracle_apply(pool, ev[i], hs, tk)
        seen |= {k.chunk_hash for k in ox.index.data.d}
        if i in (100, 200):
            pods = [int(rng.integers(0, P))]
            ix.remove_pods(pods)
            remove_pods(ox.index, {"p%d" % pods[0]})
    _add_stale((ix,), ox, 1, engine_keys)
    prompts = _prompts(rng, docs, 32, BS)
    pkeys = [ox.tokens_processor.tokens_to_kv_block_keys(None, p, MODEL) for p in prompts]
    tok_off = {n: csr([prompts[i % len(prompts)] for i in range(n)]) for n in (1, 32)}
    img = ix.snapshot()
    assert img == _encode(ox)
    counts = (len(ox.index.data), len(ox.index.engine_to_request))
    for world in worlds:
        shards = _shards(world, layout)
        assert _restore_all(shards, img) == counts
        for r in range(world):
            _check_state(_Whole(shards, r), ox, seen, engine_keys)
            _scores_ok(shards[r], ox, pkeys, tok_off)
        parts = [s.shard_snapshot() for s in shards]
        assert kvidx.snapshot_merge(parts) == img
        one = _shards(world, layout)                        # a single part: exactly its keys, canonical again
        _restore_all(one, parts[0])
        assert _merged(one) == parts[0]
        del one
        img = kvidx.snapshot_merge(parts)
    back = _fresh(table_slots=1 << 14)
    assert back.restore(img) == dict(zip(("request_keys", "engine_keys"), counts))
    assert back.snapshot() == img
    _check_state(back, ox, seen, engine_keys)
    _scores_ok(back, ox, pkeys, tok_off)


def test_unsharded_handle_takes_the_collective_calls_as_the_single_process_ones():
    rng = np.random.default_rng(8)
    a, b = _fresh(), _fresh()
    eng = rng.integers(1, 1 << 62, 400, dtype=np.uint64)
    for ix in (a, b):
        assert ix.add(0, eng, eng ^ np.uint64(5), [PT(1), PT(2, 1)]) == 0
        assert ix.add(1, eng[:100] + np.uint64(1), eng[:100], [PT(3)]) == 0
    r0 = a.shard_remove_pods([1, 3], phase=0)
    r1 = a.shard_remove_pods([1, 3], phase=1)
    want = b.remove_pods([1, 3])
    assert (r0["entries"], r0["request_keys"], r1["engine_keys"]) == (want["entries"], want["request_keys"], want["engine_keys"])
    img = b.snapshot()
    assert a.shard_snapshot() == img
    c = _fresh()
    assert c.shard_restore(img) == {"request_keys": b.stats()["request_keys"], "engine_keys": b.stats()["engine_keys"]}
    assert c.snapshot() == img


@pytest.mark.parametrize("layout", ["same-gpu", "multi-gpu"])
def test_churn_with_collective_removal_never_fills_up(layout):
    """A pod that keeps storing blocks and keeps being removed: with the collective removal and kvidx_shard_compact after
    each cycle the small shards never answer ENOSPC; the same churn without removal does within a few cycles."""
    rng = np.random.default_rng(21)
    shards = _shards(2, layout, capacity=2048, table_slots=4096)
    for cycle in range(40):
        e = rng.integers(1, 1 << 62, 500, dtype=np.uint64)
        assert shards[cycle % 2].add(0, e, rng.integers(1, 1 << 62, 500, dtype=np.uint64), [PT(9), PT(4, 1)]) == 0, cycle
        ent, rk, ek = _remove_collective(shards, [9, 4])
        assert (ent, rk, ek) == (1000, 500, 500)
        for s in shards:
            s.shard_compact()
        assert _Whole(shards).stats() == {"request_keys": 0, "engine_keys": 0, "request_tombs": 0, "engine_tombs": 0}
    shards = _shards(2, layout, capacity=2048, table_slots=4096)
    rcs = [shards[c % 2].add(0, rng.integers(1, 1 << 62, 500, dtype=np.uint64), rng.integers(1, 1 << 62, 500, dtype=np.uint64),
                             [PT(9)]) for c in range(40)]
    assert kvidx.ENOSPC in rcs


def _attempt(call, *a):
    """A write call that may succeed or be refused: either way it ends the removal that phase 0 began."""
    try:
        call(*a)
    except kvidx.KvidxError:
        pass


def test_guards():
    sh = _shards(2)
    assert sh[0].add(0, [1, 2], [3, 4], [PT(1)]) == 0

    def einval(call, why):
        with pytest.raises(kvidx.KvidxError) as ei:
            call()
        assert ei.value.code == kvidx.EINVAL and why in str(ei.value), str(ei.value)
    einval(lambda: sh[0].shard_remove_pods([1], phase=1), "without a preceding phase 0")
    sh[0].shard_remove_pods([1], phase=0)
    einval(lambda: sh[0].shard_remove_pods([2], phase=1), "other pod / tier masks")
    einval(lambda: sh[0].shard_remove_pods([1], [0], phase=1), "other pod / tier masks")
    sh[0].shard_remove_pods([1], phase=1)                        # the matching phase 1 still runs
    einval(lambda: sh[0].shard_remove_pods([1], phase=1), "without a preceding phase 0")
    writes = [lambda s: s.add(0, [7], [8], [PT(2)]), lambda s: s.evict(0, 7, [PT(2)]),
              lambda s: s.apply_events(np.zeros(1, kvidx.EVENT_DTYPE), np.array([9], np.uint64), np.zeros(16, np.uint32)),
              lambda s: s.shard_compact(), lambda s: _attempt(s.shard_restore, s.shard_snapshot())]
    for w in writes:
        for s in sh:
            s.shard_remove_pods([2], phase=0)
        w(sh[1])
        sh[0].shard_remove_pods([2], phase=1)                    # untouched rank: fine
        einval(lambda: sh[1].shard_remove_pods([2], phase=1), "a write call came between")
    einval(lambda: sh[0].shard_remove_pods([], phase=0), "empty pod mask")
    einval(lambda: sh[0].shard_remove_pods([1], [], phase=0), "empty tier mask")
    einval(lambda: sh[0].shard_remove_pods([1], phase=2), "phases 0 and 1")
    lone = _shards(2, connect=False)
    einval(lambda: lone[0].shard_remove_pods([1], phase=0), "not connected")
    for s in sh:                                                 # the single-process calls still refuse a sharded handle
        for call in (lambda: s.remove_pods([1]), s.snapshot, lambda: s.restore(_fresh().snapshot())):
            einval(call, "sharded")


def _owners(shard, keys):
    import torch
    d = torch.from_numpy(np.asarray(keys, np.uint64).view(np.int64)).cuda()
    o = torch.empty(len(keys), dtype=torch.uint8, device="cuda")
    shard.key_owners_dev(d.data_ptr(), len(keys), o.data_ptr())
    return o.cpu().numpy()


def test_restore_is_all_or_nothing():
    """An image that fits the shards in total but holds more keys of one owner than a shard admits, and a malformed image:
    every rank refuses before any inserts, and every shard stays empty."""
    sh = _shards(2, table_slots=1024)
    rng = np.random.default_rng(5)
    cand = rng.integers(1, 1 << 62, 6000, dtype=np.uint64)
    mine = cand[_owners(sh[0], cand) == 0][:1000]                # > 90 % of 1024 slots, all owned by shard 0
    assert len(mine) == 1000
    src = _fresh()
    assert src.add(0, mine + np.uint64(1), mine, [PT(3)]) == 0
    big = src.snapshot()
    for s in sh:
        with pytest.raises(kvidx.KvidxError) as ei:
            s.shard_restore(big)
        assert ei.value.code == kvidx.ENOSPC and "shard 0 full" in str(ei.value)
    small = _fresh()
    assert small.add(0, mine[:20] + np.uint64(1), mine[:20], [PT(3)]) == 0
    img = small.snapshot()
    bad = img[:64] + img[96:128] + img[64:96] + img[128:]
    for s in sh:
        with pytest.raises(kvidx.KvidxError) as ei:
            s.shard_restore(bad)
        assert ei.value.code == kvidx.EINVAL and "not in strictly ascending" in str(ei.value)
    assert _Whole(sh).stats() == {"request_keys": 0, "engine_keys": 0, "request_tombs": 0, "engine_tombs": 0}
    assert _restore_all(sh, img) == (20, 20)


def test_reader_beside_the_collective_removal():
    """A thread keeps looking up and scoring through rank 1 while the ranks run a collective removal: every key shows
    its entry set from before or from after the removal, never anything else, and the result afterwards is exact."""
    rng = np.random.default_rng(12)
    BS, P, NT = 16, 12, 2
    ix, ox, pool = _pair(P=16)
    sh = _shards(2)
    docs = _docs(rng)
    ev, hs, tk = _random_stream(rng, 300, BS, P, NT, docs)
    for i in range(len(ev)):
        assert sh[0].apply_events(ev[i:i + 1], hs, tk)[0] == 0
        _oracle_apply(pool, ev[i], hs, tk)
    keys = np.array(sorted(k.chunk_hash for k in ox.index.data.d), np.uint64)
    prompts = _prompts(rng, docs, 64, BS)
    pkeys = [ox.tokens_processor.tokens_to_kv_block_keys(None, p, MODEL) for p in prompts]
    tok, off = csr(prompts)
    before = sh[1].lookup(0, keys)
    s_before, _ = sh[1].score_batch(tok, off)
    remove_pods(ox.index, {"p%d" % p for p in range(0, P, 2)})
    after_sets = [[(e.pod, e.tier) for e in ox.index.lookup([ko.Key(MODEL, int(k))]).get(ko.Key(MODEL, int(k)), [])] for k in keys]
    stop, bad = threading.Event(), []

    def reader():
        while not stop.is_set():
            rc, pt, cnt = sh[1].lookup(0, keys)
            for i in range(len(keys)):
                got = pt[i, :cnt[i]].tolist()
                was = before[1][i, :before[2][i]].tolist()
                now = [PT(int(p[1:]), TIERS.index(t)) for p, t in after_sets[i]]
                if got != was and got != now:
                    bad.append((int(keys[i]), got, was, now))
            sh[1].score_batch(tok, off)
    th = threading.Thread(target=reader)
    th.start()
    try:
        _remove_collective(sh, list(range(0, P, 2)))
    finally:
        stop.set()
        th.join()
    assert not bad, bad[:3]
    s, _ = sh[1].score_batch(tok, off)
    assert np.array_equal(s, np.stack([_dense(_oracle_scores(ox, k), 16) for k in pkeys])) and not np.array_equal(s, s_before)


# ---- two processes, CUDA IPC, kvidx.dist ------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import torch
        from kvidx import dist as kd
        from kvidx import synth
        dev = rank % torch.cuda.device_count()
        wl = synth.Workload(3, 512, 1 << 12, 16)
        cfg = dict(capacity=1 << 13, max_pods=16, device=dev)
        ix = kvidx.Index(**cfg, shard_rank=rank, shard_count=world)
        kd.connect_shards(ix)
        ref = kvidx.Index(**cfg)                                # unsharded twin, fed the same events in the same order
        ev, hs, tk = wl.fill_events(0, wl.D)
        for i in range(len(ev)):                                # one event per call, one ingesting rank: the entry order
            assert ref.apply_events(ev[i:i + 1], hs, tk) == (0, 0)      # inside each slot is the twin's
            if rank == 0:
                assert ix.apply_events(ev[i:i + 1], hs, tk) == (0, 0)
        dist.barrier()
        toks, doc, m = wl.queries(0, 256)
        off = np.arange(0, 257 * wl.T, wl.T, dtype=np.int64)
        # removal: the counters and the state equal the unsharded removal's; the image is the unsharded image
        got = kd.remove_pods_shards(ix, [1, 5, 9], tier_ids=[0])
        assert got == ref.remove_pods([1, 5, 9], tier_ids=[0]) and got["entries"] > 0, got
        got = kd.remove_pods_shards(ix, [2, 3])
        assert got == ref.remove_pods([2, 3]) and got["engine_keys"] > 0, got
        exp, _ = ref.score_batch(toks.reshape(-1), off)
        assert np.array_equal(ix.score_batch(toks.reshape(-1), off)[0], exp)
        img = kd.snapshot_shards(ix, dst=0)
        want = ref.snapshot()
        assert (img == want) if rank == 0 else img is None
        # restore into a fresh sharded set: from the merged image on rank 0 (broadcast), and from an image every rank has
        for src_img in (img, want):
            fresh = kvidx.Index(**cfg, shard_rank=rank, shard_count=world)
            kd.connect_shards(fresh)
            n = kd.restore_shards(fresh, src_img, src=0)
            st = ref.stats()
            assert n == {"request_keys": st["request_keys"], "engine_keys": st["engine_keys"]}, n
            assert np.array_equal(fresh.score_batch(toks.reshape(-1), off)[0], exp)
            assert kd.snapshot_shards(fresh, dst=1) == (want if rank == 1 else None)
            with_keys = True
            try:                                                # a second restore: the shards are not empty, every rank refuses
                kd.restore_shards(fresh, want)
                with_keys = False
            except RuntimeError as e:
                assert "empty" in str(e)
            assert with_keys
            dist.barrier()
            del fresh
        q.put((rank, True))
    except Exception:      # noqa: BLE001
        import sys
        import traceback
        tb = traceback.format_exc()
        print("rank %d failed:\n%s" % (rank, tb), file=sys.stderr, flush=True)
        q.put((rank, tb[-900:]))
    finally:
        dist.destroy_process_group()


def test_two_processes_cuda_ipc_through_dist():
    """One process per rank with gloo for the collectives and CUDA IPC for the shards (both ranks may share device 0):
    remove, snapshot + merge and restore through kvidx.dist, with the peer's tables and removal bitmaps read over IPC."""
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert all(r[1] is True for r in res), res
