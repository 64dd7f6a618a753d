"""GPU (-m gpu): snapshot and restore of the device prefix store (kvidx_text_store_snapshot / _restore).

The device image is checked byte for byte against the host store's (kvhost_prefix_store_snapshot) after the same call
streams; the host store is itself checked against the spec on the CPU (test_text_snapshot_cpu.py).  A restored store
must then answer finds, adds and Score() from text as its source does, and leave the same image."""
import ctypes as C

import numpy as np
import pytest

import kvidx
from kvidx import pack_text
from kvidx.host import PrefixStore
from oracle import kvoracle as ko
import text_snapshot_oracle as tso
from test_gpu_text_store import MODES, _stream, _text_case, dev_store, host_find, pack_tokens, rand_text, tokenize
from test_text_snapshot_cpu import _bad_images, valid_image

pytestmark = pytest.mark.gpu


def add_both(stores, prompts, toks):
    """One device add of the batch into each kvidx.Index, and the prompts one by one into each host.PrefixStore."""
    text, off = pack_text(prompts)
    ids, spans, toff = pack_tokens(toks)
    for st in stores:
        if isinstance(st, kvidx.Index):
            st.text_store_add(text, off, ids, spans, toff)
        else:
            for p, (ti, ts) in zip(prompts, toks):
                st.add_tokenization(p, ti, ts)


def image_of(st):
    return st.text_store_snapshot() if isinstance(st, kvidx.Index) else st.snapshot()


def _batch(rng, n, bb, pool):
    prompts = []
    for _ in range(n):
        base = pool[int(rng.integers(0, len(pool)))]
        prompts.append(base[:int(rng.integers(0, len(base) + 1))] + rand_text(rng, int(rng.integers(0, 2 * bb))))
    return prompts, [tok_fast(rng, p) if rng.random() < 0.8 else tokenize(rng, p) if rng.random() < 0.9 else ([], []) for p in prompts]


def tok_fast(rng, p):
    """About one token per three bytes, ends drawn at random (several may end on one byte, none may end in a block)."""
    ends = np.sort(rng.integers(0, len(p) + 1, len(p) // 3)).astype(np.uint64)
    return rng.integers(0, 1 << 32, len(ends), dtype=np.uint64).astype(np.uint32), np.stack([np.zeros_like(ends), ends], 1)


@pytest.mark.parametrize("cache_blocks", [1, 7, 1000, 500000])
@pytest.mark.parametrize("bb", [4, 16, 256])
def test_device_image_equals_the_host_store(cache_blocks, bb):
    """Random streams (table growth, compaction, cuts, adds larger than the cache), then a batch above kTextLaneMax."""
    rng = np.random.default_rng(cache_blocks * 3 + bb)
    ix, hs = _stream(rng, cache_blocks, bb, calls=40)
    assert ix.text_store_snapshot() == hs.snapshot()
    pool = [rand_text(rng, int(rng.integers(bb, 4 * bb))) for _ in range(64)]
    for n in (20000, 300):                                          # one lane per prompt, then four
        prompts, toks = _batch(rng, n, bb, pool)
        add_both([ix, hs], prompts, toks)
        img = ix.text_store_snapshot()
        assert img == hs.snapshot(), n
        assert ix.text_store_snapshot() == img
        got, want = ix.text_store_find(*pack_text(prompts[::3])), host_find(hs, prompts[::3])
        assert all(np.array_equal(g, w) for g, w in zip(got, want))
        assert ix.text_store_snapshot() == hs.snapshot(), n
    assert ix.text_store_len() == len(hs) == len(tso.decode(img, bb))


def test_round_trips_between_device_and_host_stores():
    rng = np.random.default_rng(7)
    ix, hs = _stream(rng, 1000, 16, calls=60)
    img = ix.text_store_snapshot()
    assert img == hs.snapshot() and len(tso.decode(img, 16)) > 100
    a = dev_store(1000, 16)
    assert a.text_store_restore(img) == ix.text_store_len()
    assert a.text_store_snapshot() == img
    b = dev_store(1000, 16)                                          # host image -> device -> host
    b.text_store_restore(hs.snapshot())
    h2 = PrefixStore(1000, 16)
    h2.restore(b.text_store_snapshot())
    assert h2.snapshot() == img
    pool = [rand_text(rng, int(rng.integers(16, 200))) for _ in range(12)]
    for c in range(30):                                              # the same continuation on source and copies
        prompts, toks = _batch(rng, int(rng.integers(1, 40)), 16, pool)
        if c % 2:
            add_both([ix, a, b, hs, h2], prompts, toks)
        else:
            text, off = pack_text(prompts)
            want = host_find(hs, prompts)
            assert host_find(h2, prompts)[0].tobytes() == want[0].tobytes()
            for st in (ix, a, b):
                got = st.text_store_find(text, off)
                assert all(np.array_equal(g, w) for g, w in zip(got, want)), c
        assert len({image_of(st) for st in (ix, a, b, hs, h2)}) == 1, c


@pytest.mark.parametrize("cap", [1, 37, 999, 1000, 5000])
def test_restore_into_a_smaller_store_keeps_the_newest_records(cap):
    rng = np.random.default_rng(cap)
    ix, _ = _stream(rng, 1000, 8, calls=60)
    img = ix.text_store_snapshot()
    recs = tso.decode(img, 8)
    small = dev_store(cap, 8)
    assert small.text_store_restore(img) == min(cap, len(recs))
    got = small.text_store_snapshot()
    assert tso.decode(got, 8) == recs[max(len(recs) - cap, 0):]
    hs = PrefixStore(cap, 8)
    hs.restore(img)
    assert got == hs.snapshot() == tso.encode(tso.restore(ko.LRUTokenStore(cap, 8), img))


def _twin(ix, mode):
    """A second handle with ix's index contents and an empty store of the same shape."""
    tw = kvidx.Index(block_size=16, capacity=1 << 16, max_pods=64, **MODES[mode])
    tw.restore(ix.snapshot())
    tw.text_store_init(500000, 64)
    return tw


@pytest.mark.parametrize("n", [1, 4096, 131072])
@pytest.mark.parametrize("mode", ["default", "clock", "lru"])
def test_restored_store_scores_text_as_its_source(n, mode):
    ix, hs, q, model, filt = _text_case(n, n + 7 * len(mode), mode)
    tw = _twin(ix, mode)
    assert tw.text_store_restore(ix.text_store_snapshot()) == ix.text_store_len()
    rng = np.random.default_rng(n)
    text, off = pack_text(q)
    for rnd in range(2):
        outs = [st.score_text(text, off, model=model, filter_mask=filt, min_ratio=0.8) for st in (ix, tw)]
        for g, w in zip(*outs):
            assert g.tobytes() == w.tobytes(), (rnd, n, mode)
        sp = [st.score_text_sparse(text, off, model=model, filter_mask=filt, min_ratio=0.8) for st in (ix, tw)]
        for g, w in zip(*sp):
            assert g.tobytes() == w.tobytes(), (rnd, n, mode)
        redo = [q[i] for i in np.flatnonzero(outs[0][2])[:2000]] + [rand_text(rng, 300)]
        add_both([ix, tw], redo, [tokenize(rng, p) for p in redo])  # the tokenizer's answers go into both stores
        assert ix.text_store_snapshot() == tw.text_store_snapshot(), (rnd, n, mode)


def test_snapshot_after_an_unsynchronised_score_text_dev_holds_its_refreshes():
    import torch
    ix, hs, q, model, filt = _text_case(4096, 11, "default")
    text, off = pack_text(q)
    dev = torch.device("cuda")
    d_text, d_off = torch.from_numpy(text.copy()).to(dev), torch.from_numpy(off).to(dev)
    d_sc = torch.empty((len(q), ix.max_pods), dtype=torch.float64, device=dev)
    torch.cuda.synchronize()
    before = ix.text_store_snapshot()
    ix.score_text_dev(d_text.data_ptr(), d_off.data_ptr(), len(q), d_sc.data_ptr(), min_ratio=0.8)
    img = ix.text_store_snapshot()                                   # no synchronise in between
    host_find(hs, q)                                                 # the score's find, on the host
    assert img == hs.snapshot() and img != before
    ix.synchronize()


def test_snapshots_change_no_find_and_no_eviction():
    rng = np.random.default_rng(12)
    stores = [dev_store(64, 8), dev_store(64, 8)]                    # the first takes snapshots, the second does not
    hs = PrefixStore(64, 8)
    pool = [rand_text(rng, int(rng.integers(8, 120))) for _ in range(10)]
    for c in range(40):
        prompts, toks = _batch(rng, int(rng.integers(1, 12)), 8, pool)
        a = stores[0].text_store_snapshot()
        assert stores[0].text_store_snapshot() == a == hs.snapshot()
        if c % 3 == 0:
            add_both(stores + [hs], prompts, toks)                   # evicts: 64 blocks only
        else:
            text, off = pack_text(prompts)
            got = [st.text_store_find(text, off) for st in stores]
            want = host_find(hs, prompts)
            for g in got:
                assert all(np.array_equal(x, y) for x, y in zip(g, want)), c
    assert stores[0].text_store_snapshot() == stores[1].text_store_snapshot() == hs.snapshot()


def test_malformed_images_are_refused_on_the_device():
    img = valid_image(4, 5000)
    n = len(tso.decode(img, 4))
    ix = dev_store(5000, 4)
    for what, bad in _bad_images(img, 4):
        with pytest.raises(kvidx.KvidxError) as e:
            ix.text_store_restore(bad)
        assert e.value.code == kvidx.EINVAL, what
        assert ix.text_store_len() == 0 and len(ix.text_store_snapshot()) == 64, what
    assert ix.text_store_restore(img) == n
    assert ix.text_store_snapshot() == img
    with pytest.raises(kvidx.KvidxError) as e:                       # a store that holds keys
        ix.text_store_restore(img)
    assert e.value.code == kvidx.EINVAL and ix.text_store_snapshot() == img
    other = dev_store(5000, 8)                                       # another block size
    with pytest.raises(kvidx.KvidxError) as e:
        other.text_store_restore(img)
    assert e.value.code == kvidx.EINVAL and other.text_store_len() == 0
    bare = kvidx.Index(capacity=1024, max_pods=8)                    # no store
    for call in (bare.text_store_snapshot, lambda: bare.text_store_restore(img)):
        with pytest.raises(kvidx.KvidxError) as e:
            call()
        assert e.value.code == kvidx.EINVAL


def test_duplicate_key_far_apart_in_a_large_image():
    R = 300000
    keys = np.random.default_rng(5).permutation(np.arange(1, R + 1, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
    rec = np.zeros((R, 2), np.uint64)
    rec[:, 0] = keys
    rec[:, 1] = 1                                                    # one token each, padding 0
    head = bytearray(64)
    head[:8] = b"KVIDXTXT"; head[8:12] = (1).to_bytes(4, "little"); head[16:20] = (16).to_bytes(4, "little")
    head[24:32] = R.to_bytes(8, "little"); head[32:40] = R.to_bytes(8, "little")
    good = bytes(head) + rec.tobytes() + np.arange(R, dtype=np.uint32).tobytes()
    rec[R - 1, 0] = keys[1]
    bad = bytes(head) + rec.tobytes() + np.arange(R, dtype=np.uint32).tobytes()
    ix = dev_store(R, 16)
    with pytest.raises(kvidx.KvidxError) as e:
        ix.text_store_restore(bad)
    assert e.value.code == kvidx.EINVAL and ix.text_store_len() == 0
    assert ix.text_store_restore(good) == R
    assert ix.text_store_snapshot() == good


def test_empty_store_image_round_trips():
    ix = dev_store(10, 4)
    img = ix.text_store_snapshot()
    assert len(img) == 64 and img == PrefixStore(10, 4).snapshot()
    cp = dev_store(10, 4)
    assert cp.text_store_restore(img) == 0 and cp.text_store_snapshot() == img


def test_full_size_store_round_trips_through_pageable_and_pinned_buffers():
    """500 000 blocks of 256 bytes with about 60 tokens each: a 128 MB image."""
    rng = np.random.default_rng(8)
    bb, per, cap = 256, 60, 500000
    ix, hs = dev_store(cap, bb), PrefixStore(cap, bb)
    nb = 100                                                         # blocks per prompt
    for call in range(cap // nb // 1000 + 1):
        m = 1000 if call < cap // nb // 1000 else 100
        prompts = [rng.integers(0, 256, nb * bb, dtype=np.uint8).tobytes() for _ in range(m)]
        ends = np.sort(rng.integers(1, nb * bb + 1, nb * per)).astype(np.uint64)
        spans = np.stack([ends - 1, ends], 1)
        toks = [(rng.integers(0, 1 << 32, nb * per, dtype=np.uint64).astype(np.uint32), spans) for _ in prompts]
        text, off = pack_text(prompts)
        toff = np.arange(m + 1, dtype=np.int64) * nb * per
        ix.text_store_add(text, off, np.concatenate([t for t, _ in toks]), np.concatenate([s for _, s in toks]), toff)
        for p, (t, s) in zip(prompts, toks):
            hs.add_tokenization(p, t, s)
    assert ix.text_store_len() == len(hs) == cap
    img = ix.text_store_snapshot()                                   # pageable
    assert img == hs.snapshot()
    buf = kvidx.pinned_array((len(img),), np.uint8)                  # pinned
    got = C.c_uint64(0)
    assert ix.L.kvidx_text_store_snapshot(ix.h, buf.ctypes.data_as(C.c_void_p), len(img), C.byref(got)) == 0
    assert got.value == len(img) and buf.tobytes() == img
    assert len(img) == 64 + 16 * cap + 4 * int(np.frombuffer(img, np.uint64, 1, 32)[0])
    a, b = dev_store(cap, bb), dev_store(cap, bb)
    n = C.c_int64(0)
    assert a.L.kvidx_text_store_restore(a.h, C.cast(buf.ctypes.data_as(C.c_void_p), C.c_char_p), len(img), C.byref(n)) == 0
    assert n.value == cap and b.text_store_restore(img) == cap
    assert a.text_store_snapshot() == b.text_store_snapshot() == img


def test_each_shard_keeps_its_own_store():
    sh = [kvidx.Index(block_size=16, capacity=1 << 16, max_pods=16, shard_rank=r, shard_count=2) for r in range(2)]
    sh[0].shard_attach(1, sh[1]); sh[1].shard_attach(0, sh[0])
    rng = np.random.default_rng(2)
    hosts = [PrefixStore(300, 8), PrefixStore(500, 8)]
    for r in range(2):
        sh[r].text_store_init(300 + 200 * r, 8)
        prompts = [rand_text(rng, int(rng.integers(0, 300))) for _ in range(60)]
        add_both([sh[r], hosts[r]], prompts, [tokenize(rng, p) for p in prompts])
    imgs = [s.text_store_snapshot() for s in sh]
    assert imgs[0] != imgs[1] and imgs == [h.snapshot() for h in hosts]
    cp = [kvidx.Index(block_size=16, capacity=1 << 16, max_pods=16, shard_rank=r, shard_count=2) for r in range(2)]
    cp[0].shard_attach(1, cp[1]); cp[1].shard_attach(0, cp[0])
    for r in range(2):
        cp[r].text_store_init(300 + 200 * r, 8)
        assert cp[r].text_store_restore(imgs[r]) == len(hosts[r])
    assert [c.text_store_snapshot() for c in cp] == imgs


def test_indexer_warm_start_sends_nothing_to_the_tokenizer():
    """service.Indexer: a restarted indexer restored from the old one's store image serves the same batch from it."""
    from test_service import MODEL, POD1, FixtureTokenizer, _text
    from kvidx import service
    from kvidx.host import HostIndexer
    prompts = [_text(nm) for nm in ("short", "mid", "full", "fox2", "fox100", "fox500")]
    old, new = [service.Indexer(HostIndexer(block_size=4, capacity=1 << 14, max_pods=64),
                                service.TokenizationPool(tokenizer=FixtureTokenizer()), text_cache_blocks=4096, text_block_bytes=64)
                for _ in range(2)]
    first = old.get_pod_scores_batch(prompts, MODEL, [POD1])
    assert old.tok.encodes > 0
    image = old.text_store_snapshot()
    assert new.text_store_restore(image) == len(tso.decode(image, 64)) > 0
    before = old.tok.encodes
    second = old.get_pod_scores_batch(prompts, MODEL, [POD1])      # the old indexer's next batch, from its warm store
    assert new.get_pod_scores_batch(prompts, MODEL, [POD1]) == second == first
    assert new.tok.encodes == old.tok.encodes - before < before
    assert new.text_store_snapshot() == old.text_store_snapshot()
