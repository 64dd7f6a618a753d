"""CPU: the index image spec (tests/snapshot_oracle.py) round-trips and rejects every malformed class; the golden image
(tests/golden/snapshot_v1.json) decodes and re-encodes to itself; the host mirror's snapshot / restore on host-only
instances keeps names, freed pod ids and extra tiers, and refuses targets that are not fresh or configured otherwise."""
import json
import os
import struct

import numpy as np
import pytest

import kvidx
from kvidx.host import HostIndexer
from oracle import kvoracle as ko
from remove_oracle import remove_pods
import snapshot_oracle as so

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "snapshot_v1.json")


def golden():
    with open(GOLDEN) as f:
        d = json.load(f)
    return d, bytes.fromhex(d["image_hex"])


def malformed(image):
    """One broken image per class kvidx_restore must refuse with KVIDX_EINVAL: name -> (image, what the spec decoder says,
    what the library says).  Needs >= 2 request records, one with >= 2 entries and one with fewer than 10, and >= 2
    engine records.  An image with recency also gets the recency classes."""
    R, E = struct.unpack_from("<QQ", image, 32)
    flags = struct.unpack_from("<I", image, 12)[0]
    counts = [image[64 + 32 * i + 10] for i in range(R)]
    multi = next(i for i, c in enumerate(counts) if c >= 2)          # StopIteration: no record to repeat an entry in
    short = next(i for i, c in enumerate(counts) if c < 10)
    assert R >= 2 and E >= 2 and counts[multi] >= 2 and counts[short] < 10

    def at(off, fmt, *v):
        b = bytearray(image)
        struct.pack_into(fmt, b, off, *v)
        return bytes(b)
    r0, r1 = image[64:96], image[96:128]
    e0 = 64 + 32 * R
    m = 64 + 32 * multi
    cases = {
        "truncated": (image[:-1], "length does not match", "do not hold"),
        "longer": (image + b"\0" * 8, "length does not match", "do not hold"),
        "magic": (b"X" + image[1:], "bad magic", "bad magic"),
        "version": (at(8, "<I", 2), "bad magic or version", "unsupported snapshot version"),
        "flags": (at(12, "<I", flags | 2), "unknown flags", "unknown flags"),
        "header_padding": (at(56, "<Q", 1), "non-zero header padding", "non-zero header padding"),
        "unsorted": (image[:64] + r1 + r0 + image[128:], "request records not strictly ascending", "request record 1: not in strictly ascending"),
        "duplicate": (image[:64] + r0 + r0 + image[128:], "request records not strictly ascending", "request record 1: not in strictly ascending"),
        "engine_unsorted": (image[:e0] + image[e0 + 24:e0 + 48] + image[e0:e0 + 24] + image[e0 + 48:], "engine records not strictly ascending",
                            "engine record 1: not in strictly ascending"),
        "count0": (at(64 + 10, "<B", 0), "count outside", "entry count outside"),
        "count_above_pods_per_key": (at(64 + 10, "<B", 11), "count outside", "entry count outside"),
        "duplicate_entry": (at(m + 14, "<H", struct.unpack_from("<H", image, m + 12)[0]), "repeated entry", "repeated entry"),
        "entry_past_count": (at(64 + 32 * short + 12 + 2 * counts[short], "<H", 0x11), "non-zero padding", "non-zero padding"),
        "record_padding": (at(64 + 11, "<B", 1), "non-zero padding", "non-zero padding"),
        "engine_padding": (at(e0 + 20, "<B", 1), "non-zero padding", "non-zero padding"),
        "pod_span": (at(48, "<I", struct.unpack_from("<I", image, 48)[0] - 1), "spans disagree", "header pod_span"),
        "model_span": (at(52, "<I", struct.unpack_from("<I", image, 52)[0] + 1), "spans disagree", "header pod_span"),
    }
    if flags & so.FLAG_RECENCY:
        s0 = e0 + 24 * E                                             # request stamps, then engine stamps
        stamp = lambda i: struct.unpack_from("<Q", image, s0 + 8 * i)[0]      # noqa: E731
        cases.update({
            "stamp_high": (at(s0, "<Q", 1 << 63), "2\\^63", ">= 2^63"),
            "engine_stamp_high": (at(s0 + 8 * R, "<Q", 1 << 63), "2\\^63", ">= 2^63"),
            "stamp_repeats": (at(s0 + 8, "<Q", stamp(0)), "repeats", "recency value repeats"),
            "engine_stamp_repeats": (at(s0 + 8 * (R + 1), "<Q", stamp(R)), "repeats", "recency value repeats"),
            "engine_padding_with_recency": (at(e0 + 24 + 21, "<B", 1), "non-zero padding", "engine record 1: non-zero padding"),
        })
    return cases


def recency_image():
    """A small image with recency (exact-LRU), written by the spec encoder."""
    ix, mid, pid, tid = _random_oracle(np.random.default_rng(2), True)
    return so.encode(ix, mid, pid, tid, 16, 7, 4, recency=True), (mid, pid, tid)


def _random_oracle(rng, lru, n_ops=400):
    """A random Add / Evict / remove-pods history on the oracle (two models, 6 pods, 3 tiers, pod caches of 4)."""
    cap = 60 if lru else ko.DEFAULT_INDEX_SIZE
    ix = ko.InMemoryIndex(cap, 4)
    models, pods, tiers = ["m0", "m1"], ["p%d" % i for i in range(6)], ["gpu", "cpu", "t2"]
    for _ in range(n_ops):
        m = models[int(rng.integers(0, 2))]
        e = [ko.PodEntry(pods[int(rng.integers(0, 6))], tiers[int(rng.integers(0, 3))]) for _ in range(int(rng.integers(1, 3)))]
        r = rng.random()
        if r < 0.6:
            n = int(rng.integers(1, 5))
            eng = [ko.Key(m, int(rng.integers(0, 200))) for _ in range(n)]
            req = [ko.Key(m, int(rng.integers(0, 1 << 64, dtype=np.uint64))) if rng.random() < 0.5 else ko.Key(m, int(rng.integers(0, 120)))
                   for _ in range(n)]
            ix.add(eng, req, e)
        elif r < 0.9:
            ix.evict(ko.Key(m, int(rng.integers(0, 200))), e)
        elif r < 0.95:
            remove_pods(ix, {pods[int(rng.integers(0, 6))]})
        elif len(ix.data):
            ix.lookup([ko.Key(m, int(rng.integers(0, 120))) for _ in range(3)])      # refreshes recency
    return ix, {m: i for i, m in enumerate(models)}, {p: i for i, p in enumerate(pods)}, {t: i for i, t in enumerate(tiers)}


@pytest.mark.parametrize("lru", [False, True])
@pytest.mark.parametrize("seed", range(4))
def test_spec_round_trips(lru, seed):
    rng = np.random.default_rng(seed)
    ix, mid, pid, tid = _random_oracle(rng, lru)
    assert len(ix.data) and len(ix.engine_to_request)
    img = so.encode(ix, mid, pid, tid, 16, 7, 4, recency=lru)
    inv = ({v: k for k, v in mid.items()}, {v: k for k, v in pid.items()}, {v: k for k, v in tid.items()})
    back, hd = so.decode(img, *inv, block_size=16, init_hash=7, pods_per_key=4, size=ix.data.size)
    assert hd["n_request"] == len(ix.data) and hd["n_engine"] == len(ix.engine_to_request)
    assert so.encode(back, mid, pid, tid, 16, 7, 4, recency=lru) == img
    assert {k: v.keys() for k, v in back.data.d.items()} == {k: v.keys() for k, v in ix.data.d.items()}
    assert dict(back.engine_to_request.d) == dict(ix.engine_to_request.d)
    if lru:                                         # recency order survives: the LRU lists are equal in order
        assert list(back.data.d) == list(ix.data.d) and list(back.engine_to_request.d) == list(ix.engine_to_request.d)


def test_spec_decode_into_smaller_lru_keeps_the_most_recent():
    rng = np.random.default_rng(11)
    ix, mid, pid, tid = _random_oracle(rng, True)
    img = so.encode(ix, mid, pid, tid, 16, 7, 4, recency=True)
    inv = ({v: k for k, v in mid.items()}, {v: k for k, v in pid.items()}, {v: k for k, v in tid.items()})
    small, _ = so.decode(img, *inv, size=10)
    assert list(small.data.d) == list(ix.data.d)[-10:] and list(small.engine_to_request.d) == list(ix.engine_to_request.d)[-10:]


def test_golden_image_decodes_and_reencodes_to_itself():
    d, img = golden()
    ix, hd = so.decode(img, d["models"], d["pods"], d["tiers"], block_size=d["block_size"], init_hash=d["init_hash"],
                       pods_per_key=d["pods_per_key"])
    assert (hd["n_request"], hd["n_engine"]) == (d["request_keys"], d["engine_keys"]) and hd["flags"] == 0
    ids = [{n: i for i, n in enumerate(d[k])} for k in ("models", "pods", "tiers")]
    assert so.encode(ix, *ids, d["block_size"], d["init_hash"], d["pods_per_key"]) == img
    # the fixture has a stale mapping, a key at the pod-cache cap, and both models
    stale = [ek for ek, rk in ix.engine_to_request.d.items() if rk not in ix.data.d]
    assert stale and max(len(pc) for pc in ix.data.d.values()) == 10 and hd["model_span"] == 2


def test_golden_image_matches_its_generator():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_snapshot_golden", os.path.join(os.path.dirname(GOLDEN), "make_snapshot_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    d, img = golden()
    ids = ({m: i for i, m in enumerate(mod.MODELS)}, {p: i for i, p in enumerate(mod.PODS)}, {t: i for i, t in enumerate(mod.TIERS)})
    assert so.encode(mod.build(), *ids, mod.BLOCK_SIZE, mod.INIT_HASH, mod.PODS_PER_KEY) == img


@pytest.mark.parametrize("case", sorted(malformed(golden()[1])))
def test_spec_rejects_malformed_images(case):
    d, img = golden()
    bad, reason, _ = malformed(img)[case]
    with pytest.raises(so.SnapshotError, match=reason):
        so.decode(bad, d["models"], d["pods"], d["tiers"], pods_per_key=d["pods_per_key"])


@pytest.mark.parametrize("case", sorted(malformed(recency_image()[0])))
def test_spec_rejects_malformed_recency_images(case):
    img, ids = recency_image()
    inv = [{v: k for k, v in m.items()} for m in ids]
    so.decode(img, *inv, pods_per_key=4)
    bad, reason, _ = malformed(img)[case]
    with pytest.raises(so.SnapshotError, match=reason):
        so.decode(bad, *inv, pods_per_key=4)


def test_spec_rejects_other_configuration_and_pod_range():
    d, img = golden()
    args = (d["models"], d["pods"], d["tiers"])
    for kw in ({"block_size": 32}, {"init_hash": 1}, {"pods_per_key": 4}, {"max_pods": 4}):
        with pytest.raises(so.SnapshotError):
            so.decode(img, *args, **kw)
    so.decode(img, *args, max_pods=len(d["pods"]))


# ---- host mirror on host-only instances -----------------------------------------------------------------------------
def _model_id(h, name):
    return h.L.kvhost_model_id(h.h, name.encode())


def test_host_snapshot_keeps_names_freed_ids_and_extra_tiers():
    a = HostIndexer(no_device=True, max_pods=8)
    for p in ("a", "b", "c", "d"):
        assert a.pod_id(p) >= 0
    assert _model_id(a, "llama") == 0 and _model_id(a, "qwen") == 1
    assert a.tier_id("t2") == 2 and a.tier_id("NVME") == 3
    assert a.remove_pod("b") == 0 and a.remove_pod("d") == 0                  # ids 1 and 3 freed
    img = a.snapshot()
    assert img[:8] == b"KVHOSTSN" and img.endswith(struct.pack("<Q", 0))    # host-only: no index section
    b = HostIndexer(no_device=True, max_pods=8)
    b.restore(img)
    assert b.snapshot() == img
    for h in (a, b):
        assert (h.pod_id("a"), h.pod_id("c")) == (0, 2)
        assert (_model_id(h, "llama"), _model_id(h, "qwen")) == (0, 1)
        assert (h.tier_id("gpu"), h.tier_id("cpu"), h.tier_id("t2"), h.tier_id("nvme")) == (0, 1, 2, 3)
    for h in (a, b):                                                        # the next new names take the freed ids, lowest first
        assert (h.pod_id("e"), h.pod_id("f"), h.pod_id("g")) == (1, 3, 4)


def test_host_restore_refuses_a_target_that_is_not_fresh_or_configured_otherwise():
    a = HostIndexer(no_device=True)
    a.pod_id("a")
    img = a.snapshot()
    for dirty in (lambda h: h.pod_id("x"), lambda h: _model_id(h, "m"), lambda h: h.tier_id("t9"),
                  lambda h: h.add_task("a", "m", b"\x90")):
        h = HostIndexer(no_device=True)
        dirty(h)
        before = h.snapshot()
        with pytest.raises(kvidx.KvidxError) as ei:
            h.restore(img)
        assert ei.value.code == kvidx.EINVAL
        assert h.snapshot() == before
    for tiers in ((("gpu", 1.0), ("ssd", 0.5)), (("cpu", 0.8), ("gpu", 1.0)), (("gpu", 1.0), ("cpu", 0.8), ("ssd", 0.1))):
        h = HostIndexer(no_device=True, tiers=tiers)
        with pytest.raises(kvidx.KvidxError) as ei:
            h.restore(img)
        assert ei.value.code == kvidx.EINVAL
        assert h.pod_id("zz") == 0                                          # nothing was installed
    h = HostIndexer(no_device=True, tiers=(("GPU", 2.0), ("cpu", 0.1)))     # names compare lower-cased; weights are the target's
    h.restore(img)
    assert h.pod_id("a") == 0


def test_host_restore_rejects_malformed_images():
    a = HostIndexer(no_device=True)
    a.pod_id("a"); a.pod_id("b")
    a.remove_pod("a")
    img = a.snapshot()
    with_index = img[:-8] + struct.pack("<Q", 64) + b"\0" * 64               # an index section: refused by a host-only target
    bad = [img[:-1], b"X" + img[1:], img[:8] + struct.pack("<I", 2) + img[12:], img + b"\0", with_index]
    for b in bad:
        h = HostIndexer(no_device=True)
        with pytest.raises(kvidx.KvidxError) as ei:
            h.restore(b)
        assert ei.value.code == kvidx.EINVAL
        assert h.pod_id("q") == 0
