"""Spec of the prefix store image (kvidx_text_store_snapshot / _restore and kvhost_prefix_store_snapshot / _restore,
format v1 in include/kvidx.h), on top of the reference oracle's store (oracle/kvoracle.py::LRUTokenStore).

An extension with no reference counterpart: the reference's prefix store cannot be saved or loaded.  encode() writes the
image of an oracle store (cache.keys(), least recent first, with their token lists); decode() checks an image the way
both stores' restore does; restore() replays its records into a store as adds, oldest first.
"""
import struct

from oracle import kvoracle as ko

MAGIC = b"KVIDXTXT"
VERSION = 1
HEADER = struct.Struct("<8sIIII QQ 24s")           # 64 bytes
RECORD = struct.Struct("<QII")                     # 16 bytes
assert HEADER.size == 64 and RECORD.size == 16


class TextSnapshotError(ValueError):
    """A malformed image: restore answers KVIDX_EINVAL."""


def encode(store: ko.LRUTokenStore) -> bytes:
    """The v1 image of `store`: its keys in Keys() order (least recent first) with their tokens."""
    items = [(k, list(store.cache.d[k])) for k in store.cache.keys()]
    n_tok = sum(len(t) for _, t in items)
    out = [HEADER.pack(MAGIC, VERSION, 0, store.block_size, 0, len(items), n_tok, bytes(24))]
    out += [RECORD.pack(k, len(t), 0) for k, t in items]
    out += [struct.pack("<%dI" % len(t), *t) for _, t in items]
    return b"".join(out)


def decode(image: bytes, block_bytes=None):
    """Check `image` as restore does -> [(key, [tokens])] in record order (least recent first).  block_bytes, when given,
    must match the header.  Raises TextSnapshotError on a malformed image."""
    if len(image) < HEADER.size:
        raise TextSnapshotError("truncated header")
    magic, ver, flags, bb, zero, R, T, rest = HEADER.unpack_from(image, 0)
    if magic != MAGIC:
        raise TextSnapshotError("bad magic")
    if ver != VERSION or flags != 0:
        raise TextSnapshotError("bad version or flags")
    if zero != 0 or rest != bytes(24):
        raise TextSnapshotError("non-zero reserved bytes")
    if block_bytes is not None and bb != block_bytes:
        raise TextSnapshotError("block_bytes %d, expected %d" % (bb, block_bytes))
    if len(image) != HEADER.size + RECORD.size * R + 4 * T:
        raise TextSnapshotError("length does not match the header")
    recs, seen = [], set()
    for i in range(R):
        k, n, pad = RECORD.unpack_from(image, HEADER.size + RECORD.size * i)
        if pad:
            raise TextSnapshotError("non-zero record padding")
        if k in seen:
            raise TextSnapshotError("key %#x appears twice" % k)
        seen.add(k)
        recs.append((k, n))
    if sum(n for _, n in recs) != T:
        raise TextSnapshotError("record token counts do not add up to the header's")
    at = HEADER.size + RECORD.size * R
    out = []
    for k, n in recs:
        out.append((k, list(struct.unpack_from("<%dI" % n, image, at))))
        at += 4 * n
    return out


def block_bytes_of(image: bytes) -> int:
    return HEADER.unpack_from(image, 0)[3]


def restore(store: ko.LRUTokenStore, image: bytes) -> ko.LRUTokenStore:
    """Load `image` into the empty `store` (same block size): each record added as "insert this key with these tokens",
    oldest first, so a store smaller than the image keeps its newest records.  Returns the store."""
    if len(store.cache):
        raise TextSnapshotError("restore needs an empty store")
    for k, toks in decode(image, store.block_size):
        store.cache.add(k, toks)
    return store
