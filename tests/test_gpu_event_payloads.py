"""GPU (-m gpu): raw KVEvents msgpack messages decoded on the device (kvidx_decode_event_payloads_dev) and applied in one
call (kvidx_apply_event_payloads), against the host mirror's decoder (kvhost_decode_event_batch, itself pinned to the
Python oracle by test_host_decode.py) and the C++ oracle's index images.

  * decode equality: the device's records, queue offsets, hashes and tokens equal the host decoder's records stably
    sorted by pod, byte for byte: well-formed batches, every hash-width rule, malformed envelopes and events, the seeded
    3000-mutation fuzz, nesting 64 / 65 deep, truncated containers declaring huge counts, drains of 1 to 65 536 messages
    and messages of thousands of events;
  * the unknown-Medium protocol and tier interning, and AllBlocksCleared with and without KVIDX_PAYLOAD_STOP_AT_CLEARED;
  * index state: write_stream.py streams sent as msgpack messages leave the oracle's image on default, CLOCK, exact-LRU
    and 2- / 8-shard handles, with the oracle's dropped counts;
  * the host mirror's device path (drains above its byte threshold) against its host path;
  * Score() readers beside payload batches stay bit-exact.
Not covered: a drain of more than 2^32 token bytes (about 1 G tokens): encoding it in Python takes too long for the suite.
"""
import ctypes as C
import random
import struct
import threading

import msgpack
import numpy as np
import pytest

import kvidx
from kvidx import host as khost
from oracle import kvoracle as ko
from oracle.kvoracle_c import COracle
import write_stream as ws

pytestmark = pytest.mark.gpu

H64 = 2 ** 63 + 12345
SEED_HASH = kvidx.fnv64a(b"")
SKIP, STOP = kvidx.PAYLOAD_SKIP_UNKNOWN_TIER, kvidx.PAYLOAD_STOP_AT_CLEARED
EV = kvidx.EVENT_DTYPE
DEVICE_MIN_BYTES = 1 << 20          # kvhost.cpp kDeviceDecodeMinBytes


# ---- msgpack encoding of id-level events -------------------------------------------------------------------------------
def _arr(n):
    return bytes([0x90 | n]) if n < 16 else (b"\xdc" + struct.pack(">H", n) if n < 65536 else b"\xdd" + struct.pack(">I", n))


def _h(v):
    return b"\xcf" + struct.pack(">Q", int(v))


def _medium(tier, names, rng):
    """Tier 0 ("gpu") is sent as no Medium, nil or an upper-case name; others by name, in mixed case."""
    name = names[tier]
    r = rng.random()
    if tier == 0 and r < 0.3:
        return None
    if tier == 0 and r < 0.5:
        return b"\xc0"
    return msgpack.packb(name.upper() if r < 0.7 else name)


def encode_event(e, names, rng):
    med = _medium(e.tier, names, rng)
    hs = _arr(len(e.hashes)) + b"".join(_h(h) for h in e.hashes)
    if e.op == ws.STORED:
        f = [msgpack.packb("BlockStored"), hs, b"\xc0" if e.parent is None else _h(e.parent),
             msgpack.packb([int(t) for t in e.tokens]), msgpack.packb(16), b"\xc0"]
    else:
        f = [msgpack.packb("BlockRemoved"), hs]
    if med is not None:
        f.append(med)
    elif e.op == ws.STORED and rng.random() < 0.5:
        f = f[:4]                                            # trailing fields left out: Medium "gpu"
    return _arr(len(f)) + b"".join(f)


def encode_batch(events, names, rng, per_msg=4):
    """Id-level events -> [(payload, pod, model)]: consecutive events of one pod and model, up to per_msg a message."""
    msgs, i = [], 0
    while i < len(events):
        j = i + 1
        while j < len(events) and j - i < per_msg and (events[j].pod, events[j].model) == (events[i].pod, events[i].model):
            j += 1
        body = b"".join(encode_event(e, names, rng) for e in events[i:j])
        msgs.append((b"\x93" + msgpack.packb(1723.5) + _arr(j - i) + body + b"\x00", events[i].pod, events[i].model))
        i = j
    return msgs


# ---- the host decoder as the reference -----------------------------------------------------------------------------------
class HostDecoder:
    """kvhost_decode_event_batch over messages of interned pods, with reusable buffers; interning happens in its indexer."""

    def __init__(self, hi):
        self.hi, self.L = hi, hi.L
        self.ev = np.zeros(1 << 16, EV)
        self.hs = np.zeros(1 << 20, np.uint64)
        self.tk = np.zeros(1 << 22, np.uint32)

    def decode(self, pod_name, payload):
        nh, nt = C.c_size_t(0), C.c_size_t(0)
        n = self.L.kvhost_decode_event_batch(self.hi.h, pod_name.encode(), b"m", payload, len(payload), self.ev.ctypes.data_as(C.c_void_p),
                                             len(self.ev), self.hs.ctypes.data_as(C.POINTER(C.c_uint64)), len(self.hs), C.byref(nh),
                                             self.tk.ctypes.data_as(C.POINTER(C.c_uint32)), len(self.tk), C.byref(nt))
        assert n >= 0, self.hi.err()
        return self.ev[:n].copy(), self.hs[:nh.value].copy(), self.tk[:nt.value].copy()

    def tier_names(self):
        rows, tiers, tot = (khost.PodRow * 1)(), (C.c_char_p * 16)(), (C.c_uint64 * 4)()
        assert self.L.kvhost_pod_inventory(self.hi.h, None, 0, rows, 1, tiers, tot) >= 0
        return [t for t in tiers if t is not None]


def host_reference(dec, msgs):
    """Messages [(payload, pod id, model id)] decoded by the host one by one, concatenated, events stably sorted by pod:
    what kvidx_decode_event_payloads_dev must return."""
    evs, hss, tks, h0, t0 = [], [], [], 0, 0
    for payload, pod, model in msgs:
        ev, hs, tk = dec.decode("p%d" % pod, payload)
        ev["podtier"] = (pod << 4) | (ev["podtier"] & 15)
        ev["model"] = model
        ev["hash_off"] += h0
        ev["tok_off"] += t0
        evs.append(ev); hss.append(hs); tks.append(tk)
        h0 += len(hs); t0 += len(tk)
    ev = np.concatenate(evs + [np.zeros(0, EV)])
    ev = ev[np.argsort(ev["podtier"] >> 4, kind="stable")]
    pods = (ev["podtier"] >> 4).astype(np.int64)
    qoff = np.concatenate([[0], np.nonzero(np.diff(pods))[0] + 1, [len(ev)]]).astype(np.int64) if len(ev) else np.zeros(1, np.int64)
    return ev, np.concatenate(hss + [np.zeros(0, np.uint64)]), np.concatenate(tks + [np.zeros(0, np.uint32)]), qoff


def device_decode(ix, msgs, names, gpu_tier, flags=0, caps=None):
    import torch
    dev = torch.device("cuda", 0)
    data, off = kvidx.pack_text([m[0] for m in msgs])
    pods = np.array([m[1] for m in msgs], np.uint32)
    models = np.array([m[2] for m in msgs], np.uint32)
    t = lambda a: torch.from_numpy(np.concatenate([a.view(np.uint8), np.zeros(8, np.uint8)])).to(dev)
    d_bytes, d_off, d_pod, d_model = t(data), t(off), t(pods), t(models)
    torch.cuda.synchronize()                                 # the library's streams do not wait for torch's
    rc, cnt = ix.decode_event_payloads_dev(d_bytes.data_ptr(), d_off.data_ptr(), len(msgs), d_pod.data_ptr(), d_model.data_ptr(),
                                           names, gpu_tier, 0, 0, 0, 0, 0, 0, 0, 0, flags=flags)
    if rc != kvidx.ENOSPC:                                   # a first call without outputs: ENOSPC, unless the batch is refused
        return rc, cnt, None
    ne, nq, nh, nt = cnt["events"], cnt["queues"] + 1, cnt["hashes"], cnt["tokens"]
    if caps:
        ne, nq, nh, nt = [max(c + d, 0) for c, d in zip((ne, nq, nh, nt), caps)]
    d_ev = torch.zeros(max(ne, 1) * EV.itemsize, dtype=torch.uint8, device=dev)
    d_q = torch.full((max(nq, 1),), -1, dtype=torch.int64, device=dev)
    d_h = torch.zeros(max(nh, 1), dtype=torch.int64, device=dev)
    d_t = torch.zeros(max(nt, 1), dtype=torch.int32, device=dev)
    d_f = torch.full((len(msgs) + 1,), 0xEE, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    rc, cnt2 = ix.decode_event_payloads_dev(d_bytes.data_ptr(), d_off.data_ptr(), len(msgs), d_pod.data_ptr(), d_model.data_ptr(),
                                            names, gpu_tier, d_ev.data_ptr(), ne, d_q.data_ptr(), nq, d_h.data_ptr(), nh,
                                            d_t.data_ptr(), nt, flags=flags, d_msg_flags=d_f.data_ptr())
    assert cnt2 == cnt
    ix.synchronize()
    out = (d_ev.cpu().numpy()[:cnt["events"] * EV.itemsize].view(EV), d_h.cpu().numpy().view(np.uint64)[:cnt["hashes"]],
           d_t.cpu().numpy().view(np.uint32)[:cnt["tokens"]], d_q.cpu().numpy()[:cnt["queues"] + 1], d_f.cpu().numpy())
    return rc, cnt, out


def check_equal(ix, dec, msgs, flags=SKIP):
    """Host decodes first (interning every name), then the device decodes with the host's tier table."""
    want = host_reference(dec, msgs)
    names = dec.tier_names()
    rc, cnt, got = device_decode(ix, msgs, names, names.index(b"gpu") if b"gpu" in names else -1, flags)
    assert rc == 0, (rc, ix.last_error())
    ev, hs, tk, qoff, fl = got
    assert ev.tobytes() == want[0].tobytes()
    assert np.array_equal(hs, want[1]) and np.array_equal(tk, want[2])
    assert np.array_equal(qoff, want[3])
    assert fl[len(msgs)] == 0xEE                             # nothing past the flags array
    assert cnt["events"] == len(want[0]) and cnt["queues"] == len(want[3]) - 1
    return cnt, fl[:len(msgs)]


@pytest.fixture(scope="module")
def env():
    ix = kvidx.Index(max_pods=256)
    hi = khost.HostIndexer(max_pods=256, capacity=1 << 12)
    return ix, HostDecoder(hi)


def _pods(dec, n):
    return [dec.hi.pod_id("p%d" % p) for p in range(n)]


# ---- 1. decode equality ----------------------------------------------------------------------------------------------
def test_host_decode_cases(env):
    ix, dec = env
    _pods(dec, 4)
    p = msgpack.packb([1723.5, [["BlockStored", [H64, H64 + 1], None, list(range(32)), 16, None, "GPU"],
                                ["BlockStored", [H64 + 2], H64 + 1, [70000 + i for i in range(16)], 16],
                                ["BlockRemoved", [H64], "cpu"], ["AllBlocksCleared"],
                                ["BlockStored", [b"\x01" * 32, b"\xff\xee"], b"\x00" * 7 + b"\x09" * 3, [5] * 16, 16, 3, "Disk"]], 0])
    items = [b"\x05", b"\xcc\xc8", b"\xcd\xea\x60", b"\xce" + struct.pack(">I", 4000000000), _h(H64), b"\xd0\xfb", b"\xd1\xfe\x0c",
             b"\xd2" + struct.pack(">i", -70000), b"\xd3" + struct.pack(">q", -7), b"\xa3abc", b"\xc4\x00", b"\xc4\x03\x01\x02\x03",
             b"\xc0", b"\xcb" + struct.pack(">d", 1.5), b"\x92\x01\x02"]
    hashes = b"\xdc" + struct.pack(">H", len(items)) + b"".join(items)
    ev1 = b"\x95" + msgpack.packb("BlockStored") + hashes + b"\xc0" + msgpack.packb(list(range(16))) + b"\x10"
    ev2 = b"\x95" + msgpack.packb("BlockStored") + msgpack.packb([H64]) + b"\x07" + msgpack.packb(list(range(16))) + b"\x10"
    good = ["BlockStored", [H64], None, list(range(16)), 16]
    bad = [b"", b"\xc1", msgpack.packb({"a": 1}), msgpack.packb("str"), msgpack.packb([1.0]), msgpack.packb([1.0, None]),
           msgpack.packb([1.0, "notarray"]), msgpack.packb(["ts", [good]]), msgpack.packb([1, [good], "rank"]),
           msgpack.packb([1.0, [good, 5, [], [5], ["BlockStored"], ["BlockStored", "x"], ["BlockStored", [H64], None, "toks"],
                                ["BlockStored", [H64], None, [1.5]], ["BlockRemoved"], ["BlockRemoved", [H64], 7], ["Other", 1]]]),
           msgpack.packb([1.0, [good]])[:-3], msgpack.packb([1.0, [good], 0, "extra", [1, 2]])]
    payloads = [p, b"\x92" + msgpack.packb(1.0) + b"\x91" + ev1, b"\x92" + msgpack.packb(1.0) + b"\x91" + ev2] + bad
    msgs = [(q, i % 4, i % 3) for i, q in enumerate(payloads)]
    cnt, fl = check_equal(ix, dec, msgs)
    assert cnt["markers"] == 1 and fl[0] == 1 | 4 and fl[3] == 0 and fl[len(fl) - 1] == 1
    for q in payloads:                                       # and each message alone
        check_equal(ix, dec, [(q, 1, 7)])
    # the oracle agrees with the host on these (test_host_decode.py holds this for every case)
    got = [e for e in ko.decode_event_batch(p) if isinstance(e, (ko.BlockStored, ko.BlockRemoved))]
    assert len(got) == len(host_reference(dec, [(p, 0, 0)])[0])


def test_fuzz_differential():
    """The seeded 3000-mutation fuzz of test_host_decode.py, 16 mutants a drain (a fresh host indexer every 8 mutants, as
    there: mutated Medium names intern as new tiers)."""
    ix = kvidx.Index(max_pods=256)
    rnd = random.Random(7)
    base = msgpack.packb([1723.5, [["BlockStored", [H64, b"\x07" * 9], H64 - 1, list(range(100, 132)), 16, None, "GPU"],
                                   ["BlockRemoved", [H64, H64 + 5], "CPU"], ["BlockStored", [H64 + 9], None, [2 ** 31 + i for i in range(16)], 16]], 1])
    drain, dec = [], None
    for it in range(3000):
        if it % 8 == 0:
            if drain:
                check_equal(ix, dec, drain)
            dec, drain = HostDecoder(khost.HostIndexer(max_pods=256, capacity=1 << 10)), []
            _pods(dec, 3)
        b = bytearray(base)
        for _ in range(rnd.randrange(1, 4)):
            r = rnd.random()
            pos = rnd.randrange(len(b))
            if r < 0.6:
                b[pos] = rnd.randrange(256)
            elif r < 0.8:
                del b[pos]
            else:
                b.insert(pos, rnd.randrange(256))
        if any(isinstance(e, (ko.BlockStored, ko.BlockRemoved)) and e.medium is not None and "\x00" in e.medium
               for e in ko.decode_event_batch(bytes(b))):
            continue               # a NUL inside a Medium name does not survive the host's C-string tier names
        drain.append((bytes(b), it % 3, 0))
    check_equal(ix, dec, drain)


def _nested(k):
    """One BlockStored whose seventh field nests k arrays: the event is element depth 0 of its skip, so k = 64 fits and
    k = 65 drops the message."""
    ev = b"\x98" + msgpack.packb("BlockStored") + msgpack.packb([H64]) + b"\xc0" + msgpack.packb(list(range(16))) + b"\x10\xc0" \
         + msgpack.packb("gpu") + b"\x91" * (k - 1) + b"\xc0"
    return b"\x92" + msgpack.packb(1.0) + b"\x91" + ev


def test_nesting_depth_and_huge_counts(env):
    ix, dec = env
    _pods(dec, 2)
    msgs = [(_nested(k), k % 2, 0) for k in range(58, 70)]
    # containers that declare far more elements than the message holds, at every level
    good = msgpack.packb(["BlockStored", [H64], None, list(range(16)), 16])
    for head in (b"\xdd\xff\xff\xff\xff", b"\xdf\xff\xff\xff\xff", b"\xdc\xff\xff", b"\xc6\xff\xff\xff\xff", b"\xdb\x7f\xff\xff\xff"):
        msgs += [(head + good, 0, 0), (b"\x92\x00" + head + good, 1, 0), (b"\x92\x00\x91" + head, 0, 0),
                 (b"\x92\x00\x91\x95\xabBlockStored" + head, 1, 0), (b"\x92\x00\x91\x95\xabBlockStored\x91" + head, 0, 0),
                 (b"\x92\x00\x92" + good + head, 1, 0)]
    for cut in range(1, len(good) + 4):
        full = b"\x92\x00\x91" + good
        msgs.append((full[:cut], cut % 2, 0))
    cnt, fl = check_equal(ix, dec, msgs)
    depth = {k: fl[i] for i, k in enumerate(range(58, 70))}
    assert depth[64] & 1 and not depth[65] & 1


@pytest.mark.parametrize("n_msgs", [1, 16, 256, 4096, 65536])
def test_drain_sizes(env, n_msgs):
    ix, dec = env
    rng = np.random.default_rng(n_msgs)
    _pods(dec, 256)
    s = ws.WriteStream(rng, 16, family="a", pods=tuple(range(0, 256, 3)), models=3, tiers=2, max_blocks=24, docs_per_pod=2)
    msgs = []
    while len(msgs) < n_msgs:
        msgs += encode_batch(s.batch(min(4 * (n_msgs - len(msgs)), 4096)), ["gpu", "cpu"], rng, per_msg=int(rng.integers(1, 6)))
    check_equal(ix, dec, msgs[:n_msgs])


def test_long_messages(env):
    """Messages of thousands of events, beside one-event ones: one thread decodes each message."""
    ix, dec = env
    rng = np.random.default_rng(5)
    _pods(dec, 8)
    s = ws.WriteStream(rng, 16, family="a", pods=(1, 2, 3), models=1, tiers=2, max_blocks=16, docs_per_pod=40)
    big = encode_batch([e for e in s.batch(6000) if e.pod == 1], ["gpu", "cpu"], rng, per_msg=5000)
    small = encode_batch(s.batch(300), ["gpu", "cpu"], rng, per_msg=1)
    msgs = big[:1] + small + big[1:]
    cnt, _ = check_equal(ix, dec, msgs)
    assert max(len(m[0]) for m in msgs) > 100_000


def test_outputs_too_small_and_errors(env):
    ix, dec = env
    rng = np.random.default_rng(9)
    _pods(dec, 8)
    s = ws.WriteStream(rng, 16, family="a", pods=(0, 1, 2), models=1, tiers=2, max_blocks=8, docs_per_pod=4)
    msgs = encode_batch(s.batch(50), ["gpu", "cpu"], rng)
    for caps in ((-1, 0, 0, 0), (0, -1, 0, 0), (0, 0, -1, 0), (0, 0, 0, -1)):
        rc, cnt, out = device_decode(ix, msgs, [b"gpu", b"cpu"], 0, SKIP, caps=caps)
        assert rc == kvidx.ENOSPC and cnt["events"] > 0
        assert (out[3] == -1).all()                          # no output written
    raw = [m[0] for m in msgs]
    pods, models = [m[1] for m in msgs], [m[2] for m in msgs]
    assert ix.apply_event_payloads(raw, pods, models, [], 0)[0] == kvidx.EINVAL
    assert ix.apply_event_payloads(raw, pods, models, ["gpu"], 1)[0] == kvidx.EINVAL
    assert ix.apply_event_payloads(raw, pods, models, ["gpu"], 0, flags=4)[0] == kvidx.EINVAL
    assert ix.apply_event_payloads(raw, [256] + pods[1:], models, ["gpu", "cpu"], 0)[0] == kvidx.ERANGE
    assert ix.apply_event_payloads(raw, pods, [65536] + models[1:], ["gpu", "cpu"], 0)[0] == kvidx.ERANGE
    assert ix.apply_event_payloads([], [], [], ["gpu"], 0)[:3] == (0, 0, dict.fromkeys(kvidx.PAYLOAD_COUNTS, 0))


# ---- 2. tiers and markers ------------------------------------------------------------------------------------------
def _tier_drain(names):
    """Single-pod messages that introduce Medium names mid-batch (mixed case), some twice.  msgpack codes H64 + i (>= 2^63)
    as uint64 (0xcf): hashes."""
    msgs = []
    for i, nm in enumerate(names):
        ev = [["BlockStored", [H64 + 2 * i], None, list(range(16)), 16, None, nm], ["BlockRemoved", [H64 + 2 * i + 1], nm.lower()],
              ["BlockStored", [H64 + 2 * i + 1], None, list(range(16)), 16]]
        msgs.append(msgpack.packb([1.0, ev, 0]))
    return msgs


def test_unknown_medium_protocol_and_tier_interning():
    names = ["GPU", "cpu", "Disk", "nvme", "DISK"] + ["tier%d" % i for i in range(20)]
    raw = _tier_drain(names)
    ix = kvidx.Index(max_pods=16)
    dec = HostDecoder(khost.HostIndexer(max_pods=16, capacity=1 << 10))
    pod = dec.hi.pod_id("p0")
    ref = HostDecoder(khost.HostIndexer(max_pods=16, capacity=1 << 10))
    ref.hi.pod_id("p0")
    want = host_reference(ref, [(q, pod, 0) for q in raw])
    # the protocol: decode with the table as it is, intern the flagged messages' names on the host in order, retry skipping
    table = dec.tier_names()
    rc, n_dropped, cnt, fl = ix.apply_event_payloads(raw, [pod] * len(raw), [0] * len(raw), table, table.index(b"gpu"))
    assert rc == kvidx.ENOENT and fl[2] & 2 and not fl[0] & 2 and ix.stats()["request_keys"] == 0
    for i, q in enumerate(raw):
        if fl[i] & 2:
            dec.decode("p0", q)
    table = dec.tier_names()
    assert table == ref.tier_names() and len(table) == 16
    got = device_decode(ix, [(q, pod, 0) for q in raw], table, table.index(b"gpu"), SKIP)[2]
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1])
    rc2, _, _ = device_decode(ix, [(q, pod, 0) for q in raw], table, table.index(b"gpu"), 0)[:3]
    assert rc2 == kvidx.ENOENT                               # names past the 16th stay unknown: skipped only on request
    rc, n_dropped, cnt, fl = ix.apply_event_payloads(raw, [pod] * len(raw), [0] * len(raw), table, table.index(b"gpu"), SKIP)
    assert rc == 0 and cnt["events"] == len(want[0])
    # no "gpu" in the table yet: a Medium-less event is unknown too
    rc, _, cnt, fl = ix.apply_event_payloads(raw[:1], [pod], [0], [b"cpu"], -1)
    assert rc == kvidx.ENOENT and fl[0] & 2


def test_all_blocks_cleared_markers():
    ix = kvidx.Index(max_pods=16)
    raw = [msgpack.packb([1.0, [["BlockStored", [H64], None, list(range(16)), 16], ["AllBlocksCleared"]]]),
           msgpack.packb([1.0, [["AllBlocksCleared"], ["AllBlocksCleared", 5]]])]
    rc, _, cnt, fl = ix.apply_event_payloads(raw, [1, 2], [0, 0], ["gpu"], 0, STOP)
    assert rc == kvidx.ENOENT and cnt["markers"] == 3 and list(fl) == [5, 5] and ix.stats()["request_keys"] == 0
    rc, _, cnt, fl = ix.apply_event_payloads(raw, [1, 2], [0, 0], ["gpu"], 0)
    assert rc == 0 and cnt["events"] == 1 and ix.stats()["request_keys"] == 1


# ---- 3. index state --------------------------------------------------------------------------------------------------
NAMES = ["gpu", "cpu"]


def _apply_payloads(ix, batch, rng, per_msg=None):
    msgs = encode_batch(batch, NAMES, rng, per_msg=per_msg or int(rng.integers(1, 8)))
    rc, nd, cnt, fl = ix.apply_event_payloads([m[0] for m in msgs], [m[1] for m in msgs], [m[2] for m in msgs], NAMES, 0)
    assert rc == 0, ix.last_error()
    assert cnt["events"] == len(batch) and (fl == 1).all()
    return nd


@pytest.mark.parametrize("family", ["a", "a1", "b"])
@pytest.mark.parametrize("B", [4, 16, 24])
def test_stream_images_vs_oracle(B, family):
    rng = np.random.default_rng(B * 7 + len(family))
    s = ws.WriteStream(rng, B, family=family[0], pods=(1, 2, 3) if family == "b" else (0, 5, 9, 63), single_queue=family == "a1",
                       max_blocks=60, docs_per_pod=4)
    ix = kvidx.Index(block_size=B, init_hash=SEED_HASH, capacity=1 << 16, max_pods=64)
    co = COracle(block_size=B, init_hash=SEED_HASH, size=10 ** 8, max_pods=64)
    for _ in range(4):
        batch = s.batch(150)
        exp_drop, _ = ws.expect_batch(co, batch, B, SEED_HASH, len(ws.pack(batch)[1]) >= 1024)
        assert _apply_payloads(ix, batch, rng) == exp_drop
        got, want = ix.snapshot(), co.snapshot()
        if family == "b":
            got, want = ws.sorted_entries(got), ws.sorted_entries(want)
        assert got == want


@pytest.mark.parametrize("mode", ["clock", "lru"])
def test_capped_handles_match_decoded_batches(mode):
    """CLOCK and exact-LRU handles below their contents: payloads leave the image (recency included) that the host
    decoder's records applied by kvidx_apply_events leave, call for call."""
    rng = np.random.default_rng(3)
    B = 4
    kw = dict(evict_policy="clock") if mode == "clock" else dict(lru_exact=1)
    a, b = (kvidx.Index(block_size=B, init_hash=SEED_HASH, capacity=300, max_pods=64, **kw) for _ in range(2))
    s = ws.WriteStream(rng, B, family="a", pods=(0, 5, 9, 63), max_blocks=40, docs_per_pod=4)
    for _ in range(5):
        batch = s.batch(120)
        nd = _apply_payloads(a, batch, rng)
        rc, nd2 = b.apply_events(*ws.pack(batch))
        assert rc == 0 and nd == nd2
        assert a.snapshot() == b.snapshot()
    assert sum(a.evictions()) > 0


def test_exact_lru_recency_vs_oracle():
    rng = np.random.default_rng(41)
    B = 4
    s = ws.WriteStream(rng, B, family="a", pods=(0, 5, 9, 63), max_blocks=40, docs_per_pod=4)
    ix = kvidx.Index(block_size=B, init_hash=SEED_HASH, capacity=1 << 14, max_pods=64, lru_exact=1)
    co = COracle(block_size=B, init_hash=SEED_HASH, size=1 << 14, max_pods=64)
    for _ in range(3):
        batch = s.batch(80)
        exp_drop, _ = ws.expect_batch(co, sorted(batch, key=lambda e: e.pod), B, SEED_HASH, False)
        assert _apply_payloads(ix, batch, rng) == exp_drop
        assert ws.recency_ranks(ix.snapshot()) == co.snapshot(recency=True)


@pytest.mark.parametrize("n_shards", [2, 8])
def test_sharded_handles(n_shards):
    rng = np.random.default_rng(60 + n_shards)
    B = 16
    s = ws.WriteStream(rng, B, family="a", pods=(0, 1, 2, 7, 12, 13), max_blocks=40, docs_per_pod=4)
    sh = [kvidx.Index(block_size=B, init_hash=SEED_HASH, capacity=1 << 16, max_pods=64, shard_rank=r, shard_count=n_shards)
          for r in range(n_shards)]
    for r in range(n_shards):
        for q in range(n_shards):
            if q != r:
                sh[r].shard_attach(q, sh[q])
    co = COracle(block_size=B, init_hash=SEED_HASH, max_pods=64)
    for _ in range(3):
        batch = s.batch(150)
        for r in range(n_shards):
            part = [e for e in batch if e.pod % n_shards == r]
            if not part:
                continue
            exp_drop, _ = ws.expect_batch(co, part, B, SEED_HASH, len(ws.pack(part)[1]) > 0)
            assert _apply_payloads(sh[r], part, rng) == exp_drop
        assert kvidx.snapshot_merge([x.shard_snapshot() for x in sh]) == co.snapshot()


def test_decode_then_apply_events_dev():
    """The device-resident composition: decode_dev's outputs handed to apply_events_dev leave apply_events' image."""
    import torch
    rng = np.random.default_rng(77)
    s = ws.WriteStream(rng, 16, family="a", pods=(0, 5, 9, 63), max_blocks=40, docs_per_pod=4)
    a = kvidx.Index(capacity=1 << 16, max_pods=64)
    b = kvidx.Index(capacity=1 << 16, max_pods=64)
    drop = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    total = 0
    for _ in range(3):
        batch = s.batch(150)
        msgs = encode_batch(batch, NAMES, rng)
        rc, cnt, out = device_decode(a, msgs, [b"gpu", b"cpu"], 0)
        assert rc == 0
        ev, hs, tk, qoff, _ = out
        dev = torch.device("cuda", 0)
        d = [torch.from_numpy(np.concatenate([x.view(np.uint8), np.zeros(8, np.uint8)])).to(dev) for x in (ev, qoff, hs, tk)]
        torch.cuda.synchronize()
        a.apply_events_dev(d[0].data_ptr(), d[1].data_ptr(), len(qoff) - 1, len(ev), d[2].data_ptr(), len(hs), d[3].data_ptr(), drop.data_ptr())
        a.synchronize()
        rc, nd = b.apply_events(*ws.pack(batch))
        total += nd
        assert rc == 0 and int(drop.item()) == total
        assert a.snapshot() == b.snapshot()


# ---- 4. the host mirror ----------------------------------------------------------------------------------------------
def _mirror_messages(rng, n_docs, pods, B=16, tiers=("gpu", "cpu", "Disk", "NVMe")):
    """Documents stored (then partly removed) by named pods, as raw payloads, with Medium names that are new to the mirror."""
    out, docs = [], []
    for d in range(n_docs):
        pod = pods[d % len(pods)]
        toks = rng.integers(0, 2 ** 31, int(rng.integers(2, 40)) * B).tolist()
        eh = [int(x) | (1 << 63) for x in rng.integers(0, 2 ** 62, len(toks) // B)]
        tier = tiers[d % len(tiers)]
        evs = [["BlockStored", eh, None, toks, B, None, tier]]
        if d % 5 == 0:
            evs.append(["BlockRemoved", eh[-2:], tier])
        if d % 7 == 0:
            evs.append(["Unknown", 1, 2])
        out.append((pod, msgpack.packb([1.0 + d, evs, 0])))
        docs.append((toks, pod))
    return out, docs


@pytest.mark.parametrize("clear", [False, True])
def test_host_mirror_both_sides_of_the_threshold(clear):
    """One drain above the byte threshold (device decode) against the same messages drained in small pieces (host decode):
    scores, metrics and tier ids equal.  With clear_on_all_blocks_cleared a drain holding a marker takes the host path."""
    rng = np.random.default_rng(11)
    pods = ["10.0.0.%d" % i for i in range(6)]
    msgs, docs = _mirror_messages(rng, 2500, pods)
    if clear:
        msgs.insert(700, (pods[2], msgpack.packb([1.0, [["AllBlocksCleared"]]])))
    assert sum(len(m) for _, m in msgs) > 2 * DEVICE_MIN_BYTES
    kw = dict(max_pods=16, capacity=1 << 20, enable_metrics=True, clear_on_all_blocks_cleared=clear)
    big, small = khost.HostIndexer(**kw), khost.HostIndexer(**kw)
    for h in (big, small):
        for p in pods:                                       # same pod ids on both
            h.pod_id(p)
    for p, m in msgs:
        assert big.add_task(p, "model", m) == 0
    n_big, d_big = big.process()
    n_small = d_small = 0
    for i in range(0, len(msgs), 20):
        for p, m in msgs[i:i + 20]:
            assert small.add_task(p, "model", m) == 0
        n, d = small.process()
        assert n >= 0
        n_small += n; d_small += d
    assert n_big == n_small and d_big == d_small
    mb, ms = big.metrics(), small.metrics()
    assert mb["admissions_total"] == ms["admissions_total"] > 0 and mb["evictions_total"] == ms["evictions_total"] > 0
    assert [big.tier_id(t) for t in ("gpu", "cpu", "disk", "nvme")] == [small.tier_id(t) for t in ("gpu", "cpu", "disk", "nvme")]
    for toks, _ in docs[::37]:
        assert big.get_pod_scores(toks, "model") == small.get_pod_scores(toks, "model")
    assert kvidx.Index.borrow(big.L.kvhost_index(big.h), max_pods=16).snapshot() == \
        kvidx.Index.borrow(small.L.kvhost_index(small.h), max_pods=16).snapshot()


# ---- 5. readers beside payload batches ---------------------------------------------------------------------------------
def test_readers_beside_payload_batches():
    """Score() of a resident document set, called over and over while payload batches of other documents are applied:
    every row equals the row before the writer started."""
    rng = np.random.default_rng(21)
    B = 16
    ix = kvidx.Index(capacity=1 << 18, max_pods=64)
    fixed = ws.WriteStream(rng, B, family="a", pods=(1, 2, 3), max_blocks=40, docs_per_pod=20)
    _apply_payloads(ix, [e for e in fixed.batch(400) if e.op == ws.STORED], rng)
    toks = [d.blocks.reshape(-1) for d in fixed.docs]
    off = np.zeros(len(toks) + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in toks])
    flat = np.concatenate(toks)
    want, _ = ix.score_batch(flat, off)
    churn = ws.WriteStream(np.random.default_rng(22), B, family="a", pods=(10, 11, 12, 13), max_blocks=40, docs_per_pod=8)
    batches = [churn.batch(200) for _ in range(30)]
    stop, errors, calls = threading.Event(), [], [0]

    def reader():
        while not stop.is_set():
            got, _ = ix.score_batch(flat, off)
            calls[0] += 1
            if not np.array_equal(got, want):
                errors.append(calls[0])

    th = [threading.Thread(target=reader) for _ in range(2)]
    for t in th:
        t.start()
    for bt in batches:
        _apply_payloads(ix, bt, rng)
    stop.set()
    for t in th:
        t.join()
    assert not errors and calls[0] > 0
    assert ix.stats()["request_keys"] > 0
