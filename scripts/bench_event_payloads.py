"""KVEvents ingest: host msgpack decode + kvidx_apply_events against kvidx_apply_event_payloads (decode on the device).

Workload: BASELINE config #5's event shape (16 blocks per event, BlockStored / BlockRemoved 50 / 50, 256 pods) into the
10 M-block synthetic index, sent as raw msgpack EventBatch messages of 4 events of one pod.  Drains of 1, 16, 256, 4096
and 65 536 messages; each drain stores documents and removes them again, so every run starts from the same contents.

  host    kvhost_decode_event_batch per message (one ctypes call each, into one preallocated output), then one
          kvidx_apply_events -- what kvhost_pool_process does below its threshold
  device  kvidx_apply_event_payloads over the packed drain

Both legs run alternately on two indexes built identically; the host clock is read around the synchronous calls; the
medians of --runs runs are reported, as events/s and payload MB/s, together with the host decode alone and the cost of an
empty ctypes call (the floor the per-message loop pays in Python).  After every leg the two indexes' snapshots must be
byte-identical once each key's entries are put in one order (several pods store the same documents in one batch).
The card's name and power limit are read in the same run.

    python scripts/bench_event_payloads.py [--blocks 10000000] [--runs 5] [--out results.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "llm-d-kv-cache-manager_b200"))

import kvidx                          # noqa: E402
from kvidx import host as khost        # noqa: E402
from kvidx import synth                # noqa: E402

EV = kvidx.EVENT_DTYPE
PER_MSG = 4


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:    # noqa: BLE001
        return "unknown (%r)" % e


def encode_event(e, hs, tk):
    """One event as msgpack: hashes as uint64 (0xcf), tokens as uint32 (0xce), Medium by name."""
    h = hs[e["hash_off"]: e["hash_off"] + e["n_hashes"]]
    hb = np.zeros((len(h), 9), np.uint8)
    hb[:, 0] = 0xCF
    hb[:, 1:] = h.astype(">u8").view(np.uint8).reshape(-1, 8)
    arr16 = lambda n: b"\xdc" + int(n).to_bytes(2, "big")
    medium = b"\xa3cpu" if e["podtier"] & 15 else b"\xa3GPU"
    if e["op"] == 0:
        t = tk[e["tok_off"]: e["tok_off"] + e["n_tokens"]]
        tb = np.zeros((len(t), 5), np.uint8)
        tb[:, 0] = 0xCE
        tb[:, 1:] = t.astype(">u4").view(np.uint8).reshape(-1, 4)
        parent = (b"\xcf" + int(e["parent_hash"]).to_bytes(8, "big")) if e["has_parent"] else b"\xc0"
        return b"\x97\xabBlockStored" + arr16(len(h)) + hb.tobytes() + parent + arr16(len(t)) + tb.tobytes() + b"\x10\xc0" + medium
    return b"\x93\xacBlockRemoved" + arr16(len(h)) + hb.tobytes() + medium


def make_drain(wl, d0, n_msgs):
    """About n_msgs messages: 2 n_msgs stored events of documents from d0 on and their removals, per pod in that order.
    Event hash_off values index the drain's own hash array (documents d0.. at n blocks each)."""
    need = 2 * n_msgs
    docs = max(1, -(-need // 16))
    ev, hs, tk = wl.fill_events(d0, d0 + docs)
    # one pod per document (its deepest holder, 16 events): pods sharing a document in one batch would race their stores
    # and removals of the same keys, and the two indexes could legitimately end up different
    ev = ev[(ev["podtier"] >> 4) == wl.doc_pods(d0, d0 + docs)[(ev["hash_off"] // wl.n).astype(np.int64), 3]]
    st = ev[:need].copy()
    rm = st.copy(); rm["op"] = 1; rm["has_parent"] = 0; rm["n_tokens"] = 0
    allev = np.concatenate([st, rm])
    allev = allev[np.argsort(allev["podtier"] >> 4, kind="stable")]
    msgs, i = [], 0
    while i < len(allev):
        pod = allev[i]["podtier"] >> 4
        j = i
        while j < len(allev) and j - i < PER_MSG and allev[j]["podtier"] >> 4 == pod:
            j += 1
        body = b"".join(encode_event(e, hs, tk) for e in allev[i:j])
        msgs.append((b"\x93\xcb" + np.float64(1723.5).astype(">f8").tobytes() + bytes([0x90 | (j - i)]) + body + b"\x00", int(pod)))
        i = j
    return msgs, docs, len(allev)


SNAP_REQ = np.dtype([("hash", "<u8"), ("model", "<u2"), ("count", "u1"), ("pad", "u1"), ("ent", "<u2", (10,))])


def sorted_entries(image):
    """The image with each request record's entries sorted (kvidx.h image v1)."""
    img = bytearray(image)
    R = struct.unpack_from("<Q", img, 32)[0]
    req = np.frombuffer(img, SNAP_REQ, R, 64).copy()
    past = np.arange(10)[None, :] >= req["count"][:, None]
    ent = req["ent"].astype(np.int32)
    ent[past] = 1 << 20
    ent.sort(axis=1)
    ent[past] = 0
    req["ent"] = ent
    img[64:64 + 32 * R] = req.tobytes()
    return bytes(img)


def same(idx):
    """The two indexes hold the same keys, entries and engine mappings.  A key that several pods store in one batch gets
    their entries in the order the per-pod queues ran, so entries are compared as sets."""
    return sorted_entries(idx[0].snapshot()) == sorted_entries(idx[1].snapshot())


class HostPath:
    """kvhost_decode_event_batch per message into one output, then kvidx_apply_events."""

    def __init__(self, ix, hi, max_events, max_hashes, max_tokens):
        self.ix, self.hi, self.L = ix, hi, hi.L
        self.ev = np.zeros(max_events, EV)
        self.hs = np.zeros(max_hashes, np.uint64)
        self.tk = np.zeros(max_tokens, np.uint32)
        self.nh, self.nt = C.c_size_t(0), C.c_size_t(0)

    def decode(self, msgs, names):
        L, h = self.L, self.hi.h
        ne = nh = nt = 0
        per = []
        evp, hsp, tkp = self.ev.ctypes.data, self.hs.ctypes.data, self.tk.ctypes.data
        for (payload, pod), name in zip(msgs, names):
            n = L.kvhost_decode_event_batch(h, name, b"m", payload, len(payload), C.c_void_p(evp + ne * 40), len(self.ev) - ne,
                                            C.cast(hsp + nh * 8, C.POINTER(C.c_uint64)), len(self.hs) - nh, C.byref(self.nh),
                                            C.cast(tkp + nt * 4, C.POINTER(C.c_uint32)), len(self.tk) - nt, C.byref(self.nt))
            assert n >= 0
            per.append((n, nh, nt))
            ne += n; nh += self.nh.value; nt += self.nt.value
        counts = np.array([p[0] for p in per], np.int64)
        ev = self.ev[:ne]
        ev["hash_off"] += np.repeat(np.array([p[1] for p in per], np.uint64), counts)
        ev["tok_off"] += np.repeat(np.array([p[2] for p in per], np.uint64), counts)
        return ev, self.hs[:nh], self.tk[:nt]

    def floor(self, msgs, names):
        L, h = self.L, self.hi.h
        evp, hsp, tkp = self.ev.ctypes.data, self.hs.ctypes.data, self.tk.ctypes.data
        for (payload, pod), name in zip(msgs, names):
            L.kvhost_decode_event_batch(h, name, b"m", b"", 0, C.c_void_p(evp), 1, C.cast(hsp, C.POINTER(C.c_uint64)), 1, C.byref(self.nh),
                                        C.cast(tkp, C.POINTER(C.c_uint32)), 1, C.byref(self.nt))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=10_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--drains", default="1,16,256,4096,65536")
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    wl = synth.Workload(5, 4096, a.blocks, 256, 16, blocks_per_event=16)
    t0 = time.perf_counter()
    idx = []
    for _ in range(2):
        ix = kvidx.Index(block_size=16, capacity=wl.n_blocks + (1 << 22), max_pods=256)
        for d0 in range(0, wl.D, 4096):
            rc, nd = ix.apply_events(*wl.fill_events(d0, min(wl.D, d0 + 4096)))
            assert rc == 0 and nd == 0, ix.last_error()
        idx.append(ix)
    fill_s = time.perf_counter() - t0
    hi = khost.HostIndexer(no_device=True, max_pods=256)
    for p in range(256):
        assert hi.pod_id("p%d" % p) == p
    names = ["gpu", "cpu"]
    assert hi.tier_id("gpu") == 0 and hi.tier_id("cpu") == 1
    sizes = [int(x) for x in a.drains.split(",")]
    drains = {}
    d0 = wl.D
    for n in sizes:
        msgs, docs, n_ev = make_drain(wl, d0, n)
        d0 += docs
        drains[n] = msgs
    big = max(sum(len(m[0]) for m in v) for v in drains.values())
    hp = HostPath(idx[0], hi, 1 << 20, 1 << 24, 1 << 26)
    rows = []
    for n, msgs in drains.items():
        pods = [m[1] for m in msgs]
        pnames = [b"p%d" % p for p in pods]
        nbytes = sum(len(m[0]) for m in msgs)
        raw = [m[0] for m in msgs]

        def host_leg():
            ta = time.perf_counter()
            ev, hs, tk = hp.decode(msgs, pnames)
            tb = time.perf_counter()
            rc, nd = idx[0].apply_events(ev, hs, tk)
            tc = time.perf_counter()
            assert rc == 0, idx[0].last_error()
            return tc - ta, tb - ta, len(ev)

        def dev_leg():
            ta = time.perf_counter()
            rc, nd, cnt, fl = idx[1].apply_event_payloads(raw, pods, [0] * len(raw), names, 0)
            tb = time.perf_counter()
            assert rc == 0, idx[1].last_error()
            return tb - ta, cnt["events"]

        def floor_leg():
            ta = time.perf_counter()
            hp.floor(msgs, pnames)
            return time.perf_counter() - ta

        host_leg(); dev_leg()                                 # warm-up of every shape
        assert same(idx)
        th, td, tdec, tfl = [], [], [], []
        for r in range(a.runs):
            h, dec, ne = host_leg()
            d, ne2 = dev_leg()
            assert ne == ne2
            th.append(h); tdec.append(dec); td.append(d); tfl.append(floor_leg())
            assert same(idx), "snapshots differ after run %d of the %d-message drain" % (r, n)
        med = statistics.median
        row = {"messages": len(msgs), "events": ne, "payload_bytes": nbytes,
               "host_ms": med(th) * 1e3, "host_decode_ms": med(tdec) * 1e3, "ctypes_floor_ms": med(tfl) * 1e3,
               "device_ms": med(td) * 1e3,
               "host_events_per_s": ne / med(th), "device_events_per_s": ne / med(td),
               "host_MBps": nbytes / med(th) / 1e6, "device_MBps": nbytes / med(td) / 1e6,
               "host_decode_events_per_s": ne / med(tdec), "speedup": med(th) / med(td)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    res = {"card": card(), "torch_device": __import__("torch").cuda.get_device_name(0), "index_blocks": wl.n_blocks, "fill_s": fill_s,
           "events_per_message": PER_MSG, "blocks_per_event": 16, "runs": a.runs, "largest_drain_bytes": big, "rows": rows,
           "snapshots_identical_up_to_entry_order": True}
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "rows"}))


if __name__ == "__main__":
    main()
