"""Spec of the index image (kvidx_snapshot / kvidx_restore, format v1 in include/kvidx.h), on top of the reference oracle
(oracle/kvoracle.py).

An extension with no reference counterpart: the reference's in-memory index cannot be saved or loaded.  encode() writes the
v1 image of an oracle InMemoryIndex; decode() checks an image the way kvidx_restore does and rebuilds an InMemoryIndex.
The library is the only other implementation of the format; no product code parses it in Python.
"""
import struct

from oracle import kvoracle as ko

MAGIC = b"KVIDXSNP"
VERSION = 1
FLAG_RECENCY = 1
HEADER = struct.Struct("<8sIIIIQQQIIQ")          # 64 bytes
REQ = struct.Struct("<QHBB10H")                  # 32 bytes
ENG = struct.Struct("<QQH6s")                    # 24 bytes
assert HEADER.size == 64 and REQ.size == 32 and ENG.size == 24


class SnapshotError(ValueError):
    """A malformed image: kvidx_restore answers KVIDX_EINVAL."""


def encode(index: ko.InMemoryIndex, model_ids, pod_ids, tier_ids, block_size, init_hash, pods_per_key, recency=False) -> bytes:
    """The v1 image of `index`.  model_ids / pod_ids / tier_ids map names to the interned ids.  Entries are written in
    PodCache.keys() order (oldest -> newest).  With recency, a record's value is its 1-based position in its LRU
    (oldest = 1): only the order carries meaning."""
    reqs = []
    for pos, (rk, pc) in enumerate(index.data.d.items()):
        ents = [(pod_ids[e.pod] << 4) | tier_ids[e.tier] for e in pc.keys()]
        reqs.append((model_ids[rk.model], rk.chunk_hash, ents, pos + 1))
    engs = []
    for pos, (ek, rk) in enumerate(index.engine_to_request.d.items()):
        assert rk.model == ek.model
        engs.append((model_ids[ek.model], ek.chunk_hash, rk.chunk_hash, pos + 1))
    reqs.sort(key=lambda r: (r[0], r[1]))
    engs.sort(key=lambda r: (r[0], r[1]))
    pod_span = max((max(e >> 4 for e in r[2]) + 1 for r in reqs if r[2]), default=0)
    model_span = max([r[0] + 1 for r in reqs] + [r[0] + 1 for r in engs], default=0)
    out = [HEADER.pack(MAGIC, VERSION, FLAG_RECENCY if recency else 0, block_size, pods_per_key, init_hash, len(reqs), len(engs),
                       pod_span, model_span, 0)]
    for model, h, ents, _ in reqs:
        out.append(REQ.pack(h, model, len(ents), 0, *(ents + [0] * (10 - len(ents)))))
    for model, eh, rh, _ in engs:
        out.append(ENG.pack(eh, rh, model, bytes(6)))
    if recency:
        out.append(struct.pack("<%dQ" % (len(reqs) + len(engs)), *([r[3] for r in reqs] + [e[3] for e in engs])))
    return b"".join(out)


def decode(image: bytes, models, pods, tiers, block_size=None, init_hash=None, pods_per_key=None, max_pods=4096,
           size=ko.DEFAULT_INDEX_SIZE):
    """Check `image` as kvidx_restore does and rebuild it: -> (InMemoryIndex, header dict).  models / pods / tiers map ids
    back to names (sequences or dicts).  Keys enter each LRU in recency order when the image carries recency (its values
    are distinct within a section), else in record order; an LRU of `size` keeps the most recent ones.  block_size / init_hash /
    pods_per_key, when given, must match the header.  Raises SnapshotError on a malformed image."""
    if len(image) < HEADER.size:
        raise SnapshotError("truncated header")
    magic, ver, flags, bs, ppk, ih, R, E, pod_span, model_span, zero = HEADER.unpack_from(image, 0)
    if magic != MAGIC or ver != VERSION:
        raise SnapshotError("bad magic or version")
    if flags & ~FLAG_RECENCY or zero:
        raise SnapshotError("unknown flags or non-zero header padding")
    rec = bool(flags & FLAG_RECENCY)
    if len(image) != 64 + 32 * R + 24 * E + (8 * (R + E) if rec else 0):
        raise SnapshotError("length does not match the header")
    for name, want, got in (("block_size", block_size, bs), ("init_hash", init_hash, ih), ("pods_per_key", pods_per_key, ppk)):
        if want is not None and want != got:
            raise SnapshotError("%s differs" % name)
    if pod_span > max_pods:
        raise SnapshotError("pod_span above max_pods")
    reqs, engs, prev = [], [], None
    for i in range(R):
        h, model, cnt, pad, *ent = REQ.unpack_from(image, 64 + 32 * i)
        if prev is not None and not prev < (model, h):
            raise SnapshotError("request records not strictly ascending")
        prev = (model, h)
        if not 1 <= cnt <= ppk:
            raise SnapshotError("count outside 1..pods_per_key")
        live = ent[:cnt]
        if len(set(live)) != cnt or any(e >> 4 >= max_pods for e in live):
            raise SnapshotError("repeated entry or pod id >= max_pods")
        if pad or any(ent[cnt:]):
            raise SnapshotError("non-zero padding")
        reqs.append((model, h, live))
    prev = None
    base = 64 + 32 * R
    for i in range(E):
        eh, rh, model, pad = ENG.unpack_from(image, base + 24 * i)
        if prev is not None and not prev < (model, eh):
            raise SnapshotError("engine records not strictly ascending")
        prev = (model, eh)
        if any(pad):
            raise SnapshotError("non-zero padding")
        engs.append((model, eh, rh))
    got_pod = max((max(e >> 4 for e in r[2]) + 1 for r in reqs), default=0)
    got_model = max([r[0] + 1 for r in reqs] + [e[0] + 1 for e in engs], default=0)
    if (got_pod, got_model) != (pod_span, model_span):
        raise SnapshotError("header spans disagree with the records")
    order_r, order_e = list(range(R)), list(range(E))
    if rec:
        stamps = struct.unpack_from("<%dQ" % (R + E), image, base + 24 * E)
        if any(s >> 63 for s in stamps):
            raise SnapshotError("recency value >= 2^63")
        if len(set(stamps[:R])) != R or len(set(stamps[R:])) != E:
            raise SnapshotError("a recency value repeats within a section")
        order_r.sort(key=lambda i: stamps[i])
        order_e.sort(key=lambda i: stamps[R + i])
    ix = ko.InMemoryIndex(size, ppk)
    for i in order_r:
        model, h, live = reqs[i]
        pc = ko.LRU(ppk)
        for e in live:
            pc.add(ko.PodEntry(pods[e >> 4], tiers[e & 15]), None)
        ix.data.add(ko.Key(models[model], h), pc)
    for i in order_e:
        model, eh, rh = engs[i]
        ix.engine_to_request.add(ko.Key(models[model], eh), ko.Key(models[model], rh))
    return ix, {"flags": flags, "block_size": bs, "pods_per_key": ppk, "init_hash": ih, "n_request": R, "n_engine": E,
                "pod_span": pod_span, "model_span": model_span}
