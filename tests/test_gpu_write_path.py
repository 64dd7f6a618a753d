"""GPU (-m gpu): the event write path (kvidx_apply_events / _dev: want_parents_kernel, offer_blocks_kernel,
hash_events_kernel, apply_events_kernel) against the C++ oracle, compared as whole index images.

Streams come from tests/write_stream.py: trailing partial blocks (misaligned token slices at B = 16), events longer than
32 and 64 blocks, CBOR width edges in the tokens, every kind of dropped event, parents stored earlier in the batch (at a
producer's last block, in its middle, twice), before the batch, nowhere, by a dropped event, or removed / re-mapped in
between, repeated engine hashes, several models and tiers.  Every batch checks
  * the image: kvidx_snapshot equals the oracle's ko_snapshot byte for byte,
  * the dropped count the call returns,
  * rehashed_events against the plain model of phase 1's prediction (write_stream.phase1_predictions), when phase 1 ran.
"""
import numpy as np
import pytest

from helpers import _slot_home, csr, keys_homed_at
import kvidx
from kvidx import dist as kd
from oracle.kvoracle_c import COracle
import write_stream as ws

pytestmark = pytest.mark.gpu
SEED_HASH = kvidx.fnv64a(b"")
BLOCK_SIZES = [1, 4, 16, 23, 24, 256]
P = 64


def _phase1_env(monkeypatch, mode):
    """mode 1 / 0: phase 1 always / never; None: by batch size (from 1024 engine hashes).  Read when a handle is created."""
    if mode is None:
        monkeypatch.delenv("KVIDX_WRITE_PHASE1", raising=False)
    else:
        monkeypatch.setenv("KVIDX_WRITE_PHASE1", str(mode))


def _pair(B=16, ih=SEED_HASH, ppk=10, capacity=1 << 16, oracle_size=10 ** 8, **kw):
    ix = kvidx.Index(block_size=B, init_hash=ih, capacity=capacity, pods_per_key=ppk, max_pods=P, **kw)
    co = COracle(block_size=B, init_hash=ih, size=oracle_size, pod_cache_size=ppk, max_pods=P)
    return ix, co


def _phase1_runs(mode, n_hashes):
    return n_hashes > 0 and (mode == 1 or (mode is None and n_hashes >= 1024))


def _apply(ix, co, batch, B, ih, mode):
    """One kvidx_apply_events call, checked against the oracle's dropped count and the model's rehashed count."""
    ev, hs, tk = ws.pack(batch)
    exp_drop, exp_rh = ws.expect_batch(co, batch, B, ih, _phase1_runs(mode, len(hs)))
    before = ix.stats()["rehashed_events"]
    rc, nd = ix.apply_events(ev, hs, tk)
    assert rc == 0, ix.last_error()
    assert nd == exp_drop
    assert ix.stats()["rehashed_events"] - before == exp_rh
    return exp_rh


def _stream(B, family, seed, pods=(0, 5, 9, 63)):
    rng = np.random.default_rng(seed)
    big = B > 24
    return ws.WriteStream(rng, B, family=family[0], pods=pods, single_queue=family == "a1",
                          max_blocks=40 if big else 80, docs_per_pod=2 if big else 5)


def _check_image(ix, co, family="a"):
    got, want = ix.snapshot(), co.snapshot()
    if family == "b":
        got, want = ws.sorted_entries(got), ws.sorted_entries(want)
    assert got == want


@pytest.mark.parametrize("B", BLOCK_SIZES)
@pytest.mark.parametrize("family", ["a", "a1", "b"])
def test_stream_vs_oracle_phase1_on(B, family, monkeypatch):
    """Phase 1 on every batch, at every block size; family "a" on pods with their own documents, "a1" one queue per
    batch over shared documents, "b" shared documents without removals (entries compared as sets)."""
    _phase1_env(monkeypatch, 1)
    s = _stream(B, family, B * 3 + len(family), pods=(1, 2, 3) if family == "b" else (0, 5, 9, 63))
    ix, co = _pair(B)
    rehashed = 0
    for _ in range(4):
        rehashed += _apply(ix, co, s.batch(120 if B <= 24 else 40), B, SEED_HASH, 1)
        _check_image(ix, co, family)
    if family == "a":
        assert rehashed > 0                    # the stream makes phase 1 mispredict; each one was counted exactly


@pytest.mark.parametrize("mode", [0, None])
@pytest.mark.parametrize("family", ["a", "b"])
def test_stream_vs_oracle_phase1_off_and_auto(mode, family, monkeypatch):
    _phase1_env(monkeypatch, mode)
    s = _stream(16, family, 11 if mode is None else 12, pods=(1, 2, 3) if family == "b" else (0, 5, 9, 63))
    ix, co = _pair(16)
    sizes = set()
    for n in (20, 300, 40, 300):
        batch = s.batch(n)
        sizes.add(len(ws.pack(batch)[1]) >= 1024)
        _apply(ix, co, batch, 16, SEED_HASH, mode)
        _check_image(ix, co, family)
    assert sizes == {False, True}              # the automatic rule took both sides


@pytest.mark.parametrize("n_hashes", [1023, 1024])
def test_automatic_rule_at_its_threshold(n_hashes, monkeypatch):
    """A batch whose one consumer's parent is removed between its producer and it: phase 1 mispredicts it.  Padded with
    unknown removals to exactly 1023 / 1024 engine hashes: only the second runs phase 1, so only it counts a re-hash."""
    _phase1_env(monkeypatch, None)
    rng = np.random.default_rng(3)
    B = 16
    doc = ws.Doc(0, rng.integers(0, 2 ** 32, (12, B), dtype=np.uint64).astype(np.uint32))
    ix, co = _pair(B)
    e_prod = ws.Ev(ws.STORED, 2, 0, 0, None, doc.eh[:6], doc.blocks[:6].reshape(-1), "store")
    e_rm = ws.Ev(ws.REMOVED, 2, 0, 0, None, doc.eh[5:6], [], "remove")
    e_cons = ws.Ev(ws.STORED, 2, 1, 0, int(doc.eh[5]), doc.eh[6:12], doc.blocks[6:12].reshape(-1), "consumer")
    pad = ws.Ev(ws.REMOVED, 2, 0, 0, None, rng.integers(1, 2 ** 63, n_hashes - 13, dtype=np.uint64), [], "remove")
    batch = [e_prod, e_rm, pad, e_cons]
    assert len(ws.pack(batch)[1]) == n_hashes
    assert _apply(ix, co, batch, B, SEED_HASH, None) == (1 if n_hashes == 1024 else 0)
    _check_image(ix, co)


@pytest.mark.parametrize("ih,B", [(1, 16), (23, 24), (2 ** 32 - 1, 16), (2 ** 32, 4)])
def test_init_hashes(ih, B, monkeypatch):
    """Chains seeded from init hashes on both sides of the CBOR head widths, set directly on both handles."""
    _phase1_env(monkeypatch, 1)
    s = _stream(B, "a", ih % 1000 + B)
    ix, co = _pair(B, ih=ih)
    for _ in range(3):
        _apply(ix, co, s.batch(100), B, ih, 1)
        _check_image(ix, co)


def _dev_batch(ix, batch, keep):
    """kvidx_apply_events_dev: the test sorts the events by pod (stably) and builds the queue offsets."""
    import torch
    ev, hs, tk = ws.pack(batch)
    order = np.argsort(ev["podtier"] >> 4, kind="stable")
    evs = ev[order]
    pods = (evs["podtier"] >> 4).astype(np.int64)
    qoff = np.concatenate([[0], np.nonzero(np.diff(pods))[0] + 1, [len(evs)]]).astype(np.int64)
    dev = torch.device("cuda", 0)
    d = (torch.from_numpy(evs.view(np.uint8).reshape(-1).copy()).to(dev), torch.from_numpy(qoff).to(dev),
         torch.from_numpy(np.concatenate([hs, np.zeros(1, np.uint64)]).view(np.int64)).to(dev),
         torch.from_numpy(np.concatenate([tk, np.zeros(1, np.uint32)]).view(np.int32)).to(dev))
    keep.append(d)
    ix.apply_events_dev(d[0].data_ptr(), d[1].data_ptr(), len(qoff) - 1, len(evs), d[2].data_ptr(), len(hs), d[3].data_ptr(),
                        keep[0].data_ptr())


def test_batch_splits_give_one_image(monkeypatch):
    """One family-"a" stream applied as whole batches, event by event, in random splits, and through apply_events_dev:
    byte-identical images, equal to the oracle's; apply_events_dev's dropped count is cumulative."""
    import torch
    _phase1_env(monkeypatch, 1)
    B = 16
    s = _stream(B, "a", 21)
    batches = [s.batch(n) for n in (150, 60, 200)]
    events = [e for b in batches for e in b]
    rng = np.random.default_rng(22)
    cuts = np.sort(rng.choice(np.arange(1, len(events)), 12, replace=False))
    splits = {"whole": batches, "single": [[e] for e in events],
              "random": [events[a:b] for a, b in zip([0, *cuts], [*cuts, len(events)])]}
    images = []
    for name, parts in splits.items():
        ix, co = _pair(B)
        for part in parts:
            _apply(ix, co, part, B, SEED_HASH, 1)
        _check_image(ix, co)
        images.append(ix.snapshot())
    ix, co = _pair(B)
    keep = [torch.zeros(1, dtype=torch.int64, device="cuda:0")]
    dropped = 0
    for part in splits["random"]:
        exp_drop, exp_rh = ws.expect_batch(co, part, B, SEED_HASH, True)
        dropped += exp_drop
        before = ix.stats()["rehashed_events"]
        _dev_batch(ix, part, keep)
        ix.synchronize()
        assert int(keep[0].item()) == dropped
        assert ix.stats()["rehashed_events"] - before == exp_rh
    assert dropped > 0
    _check_image(ix, co)
    images.append(ix.snapshot())
    assert all(im == images[0] for im in images)


def _block_homing_at(co, rng, parent, S, slot, B=16):
    """B tokens whose block key under `parent` has its home at `slot` (brute force over random blocks)."""
    n = 1 << 15
    cand = rng.integers(0, 2 ** 32, (n, B), dtype=np.uint64).astype(np.uint32)
    keys, _ = co.hash_keys(cand.reshape(-1), np.arange(0, (n + 1) * B, B, dtype=np.int64), np.full(n, parent, np.uint64))
    hit = np.nonzero(_slot_home(keys, 0, S) == slot)[0]
    assert len(hit), "no block found"
    return cand[hit[0]]


def test_crowded_small_table_with_rebuild(monkeypatch):
    """A 1024-slot table: documents whose engine hashes and request keys all home on the last pairs, so the write path's
    inserts, finds and tombstone steps run on displaced chains that wrap past slot S - 1; removals in between, until the
    room check's compaction has rebuilt the table mid-stream.  Image checked after every batch."""
    _phase1_env(monkeypatch, 1)
    B, S = 16, 1024
    rng = np.random.default_rng(31)
    ix, co = _pair(B, capacity=1 << 10, table_slots=S)
    assert ix.stats()["request_slots"] == S and ix.stats()["engine_slots"] == S
    s = ws.WriteStream(rng, B, family="a", pods=(0, 1), models=1, tiers=1, max_blocks=12, docs_per_pod=4)
    for d in s.docs:                                           # crowd them onto the last four pairs
        slots = S - 2 - 2 * rng.integers(0, 4, len(d))
        d.eh = keys_homed_at(slots, 0, S, rng)
        parent = SEED_HASH
        for j in range(len(d)):
            d.blocks[j] = _block_homing_at(co, rng, parent, S, int(slots[j]))
            parent = int(co.hash_keys(d.blocks[j], np.array([0, B], np.int64), parent=np.array([parent], np.uint64))[0][0])
    crowd = ws.Ev(ws.STORED, 7, 0, 0, None, keys_homed_at(np.full(6, S - 2), 0, S, rng),
                  rng.integers(0, 2 ** 32, 6 * B, dtype=np.uint64).astype(np.uint32), "store")
    _apply(ix, co, [crowd], B, SEED_HASH, 1)                   # some slots of the last pair taken before the stream
    filler = ws.WriteStream(np.random.default_rng(32), B, family="a", pods=(2, 3), models=1, tiers=1, max_blocks=60,
                            docs_per_pod=8)
    rounds = 0
    while ix.stats()["rebuilds"] < 1 or rounds < 3:
        rounds += 1
        assert rounds < 30, ix.stats()
        _apply(ix, co, s.batch(60) + filler.batch(20), B, SEED_HASH, 1)
        _check_image(ix, co)
        wipe = [ws.Ev(ws.REMOVED, p, 0, 0, None, d.eh, [], "remove") for p, d in
                [(p, d) for p in (2, 3) for d in filler._docs_of(p)]]
        _apply(ix, co, wipe, B, SEED_HASH, 1)                  # tombstones: the filler's keys come and go
        _check_image(ix, co)


@pytest.mark.parametrize("capped", [False, True])
def test_exact_lru_recency_ranks(capped, monkeypatch):
    """Exact-LRU handles: recency ranks of every request key and engine mapping equal the oracle's.  Capacity above the
    contents: whole batches of four pods, replayed on the oracle in the order their stamps give (each pod's events in
    order, pods in ascending id).  Capped: one event per call, so that eviction after each call is eviction in order."""
    _phase1_env(monkeypatch, None)
    B = 4
    cap = 150 if capped else 1 << 14
    s = _stream(B, "a1" if capped else "a", 41 + capped)
    ix, co = _pair(B, capacity=cap, oracle_size=cap, lru_exact=1)
    for r in range(3):
        if capped:
            for e in s.batch(80):
                _apply(ix, co, [e], B, SEED_HASH, None)
        else:
            batch = s.batch(80)
            exp_drop, _ = ws.expect_batch(co, sorted(batch, key=lambda e: e.pod), B, SEED_HASH, False)
            assert ix.apply_events(*ws.pack(batch)) == (0, exp_drop)
            assert len({e.pod for e in batch}) > 1
        got = ix.snapshot()
        assert ws.recency_ranks(got) == co.snapshot(recency=True)
    if capped:
        assert co.len_request() == cap and sum(ix.evictions()) > 0


def test_clock_handle_below_capacity(monkeypatch):
    """A CLOCK handle whose capacity is never reached writes exactly what the default handle writes."""
    _phase1_env(monkeypatch, 1)
    s = _stream(16, "a", 51)
    ix, co = _pair(16, evict_policy="clock")
    ix2 = kvidx.Index(block_size=16, init_hash=SEED_HASH, capacity=1 << 16, max_pods=P)
    for _ in range(3):
        batch = s.batch(150)
        _apply(ix, co, batch, 16, SEED_HASH, 1)
        ev, hs, tk = ws.pack(batch)
        assert ix2.apply_events(ev, hs, tk)[0] == 0
        _check_image(ix, co)
        assert ix.snapshot() == ix2.snapshot()
    assert ix.evictions() == (0, 0)


def test_two_shards_merge_to_the_oracle_image(monkeypatch):
    """Two same-GPU shards, each fed its pods' events (kvidx.dist.events_for_rank); the merged shard images equal the
    oracle's image."""
    _phase1_env(monkeypatch, 1)
    B = 16
    s = _stream(B, "a", 61, pods=(0, 1, 2, 7))
    sh = [kvidx.Index(block_size=B, init_hash=SEED_HASH, capacity=1 << 16, max_pods=P, shard_rank=r, shard_count=2)
          for r in range(2)]
    sh[0].shard_attach(1, sh[1])
    sh[1].shard_attach(0, sh[0])
    co = COracle(block_size=B, init_hash=SEED_HASH, max_pods=P)
    for _ in range(3):
        batch = s.batch(150)
        for r in range(2):
            part = [e for e in batch if e.pod % 2 == r]
            ev, hs, tk = ws.pack(part)
            assert np.array_equal(kd.events_for_rank(ws.pack(batch)[0], r, 2)["podtier"], ev["podtier"])
            exp_drop, exp_rh = ws.expect_batch(co, part, B, SEED_HASH, len(hs) > 0)
            before = sum(x.stats()["rehashed_events"] for x in sh)
            rc, nd = sh[r].apply_events(ev, hs, tk)
            assert rc == 0 and nd == exp_drop
            assert sum(x.stats()["rehashed_events"] for x in sh) - before == exp_rh
        assert kvidx.snapshot_merge([x.shard_snapshot() for x in sh]) == co.snapshot()


def test_score_after_the_stream(monkeypatch):
    """End to end: one score_batch over prefixes of the stream's documents, on the default path, equals the oracle's."""
    _phase1_env(monkeypatch, None)
    s = _stream(16, "a", 71)
    ix, co = _pair(16)
    for n in (300, 300, 100):
        _apply(ix, co, s.batch(n), 16, SEED_HASH, None)
    _check_image(ix, co)
    rng = np.random.default_rng(72)
    prompts = [d.blocks.reshape(-1)[:16 * int(rng.integers(0, len(d) + 1)) + int(rng.integers(0, 16))] for d in s.docs]
    tok, off = csr(prompts)
    for m in range(2):
        s1, h1 = ix.score_batch(tok, off, model0=m)
        s2, h2, _, _ = co.score_batch(tok, off, model0=m)
        assert np.array_equal(h1, h2) and np.array_equal(s1, s2)
        assert (s2 >= 0).any()
