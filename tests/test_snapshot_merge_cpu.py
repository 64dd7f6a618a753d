"""CPU: kvidx_snapshot_merge (host only, through the library) -- shard images of disjoint parts of an index merge back into
the one canonical image of the whole, and every kind of bad input is refused for its own reason."""
import ctypes as C
import struct

import numpy as np
import pytest

import kvidx
import snapshot_oracle as so
from test_snapshot_cpu import _random_oracle, golden


def _records(image):
    """-> (header fields, request records, engine records) of a v1 image without recency."""
    hd = list(so.HEADER.unpack_from(image, 0))
    R, E = hd[6], hd[7]
    reqs = [image[64 + 32 * i: 96 + 32 * i] for i in range(R)]
    base = 64 + 32 * R
    engs = [image[base + 24 * i: base + 24 * (i + 1)] for i in range(E)]
    return hd, reqs, engs


def _image(hd, reqs, engs):
    """A v1 image of these records, with the header's counts and spans made to fit them (each part is valid on its own)."""
    hd = list(hd)
    pod_span = 0
    for r in reqs:
        cnt = r[10]
        ents = struct.unpack_from("<10H", r, 12)[:cnt]
        pod_span = max([pod_span] + [(e >> 4) + 1 for e in ents])
    models = [struct.unpack_from("<H", r, 8)[0] for r in reqs] + [struct.unpack_from("<H", e, 16)[0] for e in engs]
    hd[6], hd[7], hd[8], hd[9] = len(reqs), len(engs), pod_span, max([m + 1 for m in models], default=0)
    return so.HEADER.pack(*hd) + b"".join(reqs) + b"".join(engs)


def split(image, k, rng):
    """Split an image into k parts by an arbitrary partition of its records (some parts may be empty)."""
    hd, reqs, engs = _records(image)
    ra = rng.integers(0, k, len(reqs))
    ea = rng.integers(0, k, len(engs))
    return [_image(hd, [r for r, a in zip(reqs, ra) if a == p], [e for e, a in zip(engs, ea) if a == p]) for p in range(k)]


def _source(seed):
    ix, mid, pid, tid = _random_oracle(np.random.default_rng(seed), False)
    return so.encode(ix, mid, pid, tid, 16, 7, 4)


def _merge_raw(parts, cap=None, out=True):
    L = kvidx.load()
    ptrs = (C.c_char_p * max(len(parts), 1))(*parts)
    lens = (C.c_uint64 * max(len(parts), 1))(*[len(p) for p in parts])
    size = C.c_uint64(0)
    buf = C.create_string_buffer(b"\x5a" * (cap or 1), cap or 1) if out else None
    rc = L.kvidx_snapshot_merge(ptrs, C.cast(lens, C.POINTER(C.c_uint64)), len(parts), buf, cap or 0, C.byref(size))
    return rc, size.value, (buf.raw if out else None), L.kvidx_last_error(None).decode()


@pytest.mark.parametrize("k", [1, 2, 3, 8])
@pytest.mark.parametrize("seed", range(3))
def test_parts_merge_back_to_the_original(k, seed):
    img = _source(seed)
    rng = np.random.default_rng(100 + seed)
    for _ in range(3):
        parts = split(img, k, rng)
        assert sum(so.HEADER.unpack_from(p, 0)[6] for p in parts) == so.HEADER.unpack_from(img, 0)[6]
        for p in parts:                                     # every part is a valid image on its own
            so.decode(p, ["m0", "m1"], ["p%d" % i for i in range(6)], ["gpu", "cpu", "t2"], pods_per_key=4)
        assert kvidx.snapshot_merge(parts) == img
        assert kvidx.snapshot_merge(parts[::-1]) == img


def test_golden_image_split_and_merged():
    _, img = golden()
    rng = np.random.default_rng(4)
    for k in (1, 2, 3, 8):
        parts = split(img, k, rng)
        assert kvidx.snapshot_merge(parts) == img and kvidx.snapshot_merge(parts[::-1]) == img


def _refused(parts, why):
    with pytest.raises(kvidx.KvidxError) as ei:
        kvidx.snapshot_merge(parts)
    assert ei.value.code == kvidx.EINVAL and why in str(ei.value), str(ei.value)


def test_refusals_each_for_its_own_reason():
    img = _source(7)
    a, b = split(img, 2, np.random.default_rng(1))
    hd_b, reqs_b, engs_b = _records(b)
    assert len(reqs_b) >= 2 and len(engs_b) >= 2
    _refused([], "no parts")
    # a header or length kvidx_restore refuses
    _refused([a, b[:-1]], "part 1: malformed snapshot image")
    _refused([a, b + b"\0" * 8], "do not hold")
    _refused([a, b"X" + b[1:]], "bad magic")
    _refused([a, b[:8] + struct.pack("<I", 2) + b[12:]], "unsupported snapshot version")
    _refused([a, b[:56] + struct.pack("<Q", 1) + b[64:]], "non-zero header padding")
    _refused([a, b[:52] + struct.pack("<I", 65537) + b[56:]], "model_span")
    # parts of another configuration
    for off, fmt, v in ((16, "<I", 32), (24, "<Q", 8), (20, "<I", 5)):
        bad = bytearray(b)
        struct.pack_into(fmt, bad, off, v)
        _refused([a, bytes(bad)], "another configuration")
    # a part with recency
    ix, mid, pid, tid = _random_oracle(np.random.default_rng(2), True)
    _refused([a, so.encode(ix, mid, pid, tid, 16, 7, 4, recency=True)], "recency")
    # records out of order inside a part: request section, engine section
    _refused([a, _image(hd_b, [reqs_b[1], reqs_b[0]] + reqs_b[2:], engs_b)], "part 1 request record 1: not in strictly ascending")
    _refused([a, _image(hd_b, reqs_b, [engs_b[1], engs_b[0]] + engs_b[2:])], "part 1 engine record 1: not in strictly ascending")
    _refused([_image(hd_b, reqs_b[:1] * 2, [])], "part 0 request record 1: not in strictly ascending")
    # a key in two parts
    _refused([a, b, _image(hd_b, reqs_b[:1], [])], "request key")
    _refused([a, b, _image(hd_b, [], engs_b[-1:])], "engine key")
    _refused([b, b], "in parts 0 and 1")


def test_small_buffer_gets_enospc_and_the_size():
    img = _source(3)
    parts = split(img, 3, np.random.default_rng(2))
    rc, size, _, err = _merge_raw(parts, out=False)
    assert rc == kvidx.ENOSPC and size == len(img) and "needs" in err
    rc, size, buf, _ = _merge_raw(parts, cap=100)
    assert rc == kvidx.ENOSPC and size == len(img) and buf == b"\x5a" * 100      # nothing written
    rc, size, buf, _ = _merge_raw(parts, cap=len(img))
    assert rc == 0 and size == len(img) and buf == img
    bad = [parts[0], parts[0]] if so.HEADER.unpack_from(parts[0], 0)[6] else [parts[1], parts[1]]
    rc, size, buf, _ = _merge_raw(bad, cap=2 * len(img))                   # a refused merge writes nothing either
    assert rc == kvidx.EINVAL and buf == b"\x5a" * (2 * len(img))
