"""The prefix store image on the CPU: the host store's snapshot and restore (kvhost_prefix_store_*, host.PrefixStore)
against the spec (tests/text_snapshot_oracle.py) over the oracle's store (oracle/kvoracle.py::LRUTokenStore), and the
golden fixture that pins the format."""
import struct

import numpy as np
import pytest

import kvidx
from helpers import golden
from kvidx.host import PrefixStore
from oracle import kvoracle as ko
from test_gpu_text_store import rand_text, tokenize
import text_snapshot_oracle as tso


def _calls(rng, bb, n_calls):
    """A random stream of ("add", prompt, ids, spans) and ("find", prompt): shared prefixes (rewrites of the same blocks
    with new tokens), prompts without tokens, tokens spanning whole blocks (blocks without tokens), and long prompts."""
    pool = [rand_text(rng, int(rng.integers(bb, 10 * bb))) for _ in range(6)]
    out = []
    for _ in range(n_calls):
        r = rng.random()
        if r < 0.6:
            p = pool[int(rng.integers(0, len(pool)))]
            p = p[:int(rng.integers(0, len(p) + 1))] + rand_text(rng, int(rng.integers(0, 3 * bb)))
        else:
            p = rand_text(rng, int(rng.integers(0, 20 * bb)))
        if rng.random() < 0.55:
            if rng.random() < 0.1:
                ids, spans = [], []
            elif rng.random() < 0.2:                                              # one token over many blocks
                ids, spans = [int(rng.integers(0, 1 << 32))], [(0, len(p))]
            else:
                ids, spans = tokenize(rng, p)
            out.append(("add", p, ids, spans))
        else:
            out.append(("find", p))
    return out


def _apply(stores, calls):
    finds = []
    for c in calls:
        got = []
        for st in stores:
            if c[0] == "add":
                st.add_tokenization(c[1], c[2], c[3])
            else:
                got.append(st.find_longest_contained_tokens(c[1]))
        if got:
            assert all(g == got[0] for g in got), c
            finds.append(got[0])
    return finds


@pytest.mark.parametrize("cache_blocks", [1, 3, 7, 1000])
@pytest.mark.parametrize("bb", [4, 16])
def test_host_image_equals_the_spec(cache_blocks, bb):
    rng = np.random.default_rng(cache_blocks * 17 + bb)
    hs, os_ = PrefixStore(cache_blocks, bb), ko.LRUTokenStore(cache_blocks, bb)
    empty_blocks = 0
    for step in range(12):
        _apply([hs, os_], _calls(rng, bb, 20))
        img = hs.snapshot()
        assert img == tso.encode(os_), step
        assert len(img) == 64 + 16 * len(hs) + 4 * sum(len(t) for t in os_.cache.d.values())
        assert hs.snapshot() == img                                           # a snapshot refreshes nothing
        empty_blocks += sum(not t for _, t in tso.decode(img, bb))
    if cache_blocks >= 7:
        assert empty_blocks, "no image held a block without tokens"


@pytest.mark.parametrize("cache_blocks", [1, 3, 7, 1000])
@pytest.mark.parametrize("bb", [4, 16])
def test_restore_equals_the_replay_and_continues_alike(cache_blocks, bb):
    rng = np.random.default_rng(cache_blocks * 5 + bb)
    src = PrefixStore(cache_blocks, bb)
    _apply([src], _calls(rng, bb, 150))
    img = src.snapshot()
    n = len(src)
    for cap in sorted({cache_blocks, 1, max(1, n // 2), 5000}):
        cp = PrefixStore(cap, bb)
        cp.restore(img)
        want = tso.restore(ko.LRUTokenStore(cap, bb), img)
        assert cp.snapshot() == tso.encode(want), cap
        assert len(cp) == min(cap, n)
        assert tso.decode(cp.snapshot(), bb) == tso.decode(img, bb)[max(n - cap, 0):]     # exactly the newest cap records
    cp = PrefixStore(cache_blocks, bb)
    cp.restore(img)
    assert cp.snapshot() == img                                               # snapshot, restore, snapshot: same bytes
    more = _calls(rng, bb, 120)
    assert _apply([src], more) == _apply([cp], more)
    assert src.snapshot() == cp.snapshot()


def test_golden_fixture_round_trips():
    g = golden("text_snapshot_v1.json")
    img = bytes.fromhex(g["image_hex"])
    recs = tso.decode(img, g["block_bytes"])
    assert [(r["key"], r["tokens"]) for r in g["records"]] == recs
    assert any(not t for _, t in recs)
    st = tso.restore(ko.LRUTokenStore(g["cache_blocks"], g["block_bytes"]), img)
    assert tso.encode(st) == img
    hs = PrefixStore(g["cache_blocks"], g["block_bytes"])
    hs.restore(img)
    assert hs.snapshot() == img


def test_empty_store_image():
    hs = PrefixStore(10, 4)
    img = hs.snapshot()
    assert img == tso.encode(ko.LRUTokenStore(10, 4)) and len(img) == 64
    cp = PrefixStore(10, 4)
    cp.restore(img)
    assert len(cp) == 0 and cp.snapshot() == img


def _bad_images(img, bb):
    """Every malformed form of a valid image `img` (at least 3 records, at least 2 tokens in the first record)."""
    R, T = struct.unpack_from("<QQ", img, 24)
    def put(at, fmt, v):
        b = bytearray(img); struct.pack_into(fmt, b, at, v); return bytes(b)
    rec = lambda i: 64 + 16 * i
    yield "magic", b"KVIDXSNP" + img[8:]
    yield "version", put(8, "<I", 2)
    yield "flags", put(12, "<I", 1)
    yield "reserved u32", put(20, "<I", 1)
    for at in (40, 47, 63):
        yield "reserved byte %d" % at, put(at, "<B", 1)
    yield "block_bytes", put(16, "<I", bb + 1)
    yield "short", img[:-4]
    yield "long", img + bytes(4)
    yield "truncated header", img[:63]
    yield "records too many", put(24, "<Q", R + 1)
    yield "records huge", put(24, "<Q", 1 << 62)
    yield "tokens huge", put(32, "<Q", (1 << 64) - 1)
    yield "padding", put(rec(1) + 12, "<I", 1)
    yield "sum above", put(rec(0) + 8, "<I", struct.unpack_from("<I", img, rec(0) + 8)[0] + 1)
    yield "sum below", put(rec(0) + 8, "<I", struct.unpack_from("<I", img, rec(0) + 8)[0] - 1)
    yield "duplicate key", put(rec(R - 1), "<Q", struct.unpack_from("<Q", img, rec(0))[0])
    yield "duplicate neighbours", put(rec(1), "<Q", struct.unpack_from("<Q", img, rec(2))[0])
    yield "tokens without records", struct.pack("<8sIIIIQQ24s", b"KVIDXTXT", 1, 0, bb, 0, 0, 1, bytes(24)) + bytes(4)


def valid_image(bb=4, cache_blocks=50, seed=3):
    rng = np.random.default_rng(seed)
    st = PrefixStore(cache_blocks, bb)
    while True:
        p = rand_text(rng, 12 * bb)
        st.add_tokenization(p, list(range(1, 12 * bb + 1)), [(j, j + 1) for j in range(12 * bb)])
        img = st.snapshot()
        if struct.unpack_from("<I", img, 64 + 8)[0] >= 2 and len(st) >= 3:
            return img


def test_every_malformed_image_is_refused_and_changes_nothing():
    bb = 4
    img = valid_image(bb)
    for what, bad in _bad_images(img, bb):
        with pytest.raises(tso.TextSnapshotError):
            tso.decode(bad, bb)
        st = PrefixStore(50, bb)
        with pytest.raises(kvidx.KvidxError) as e:
            st.restore(bad)
        assert e.value.code == kvidx.EINVAL, what
        assert len(st) == 0 and len(st.snapshot()) == 64, what
        st.restore(img)                                                          # the store is still usable
        assert st.snapshot() == img, what
    full = PrefixStore(50, bb)                                                   # a store that holds keys
    full.restore(img)
    with pytest.raises(kvidx.KvidxError) as e:
        full.restore(img)
    assert e.value.code == kvidx.EINVAL and full.snapshot() == img
