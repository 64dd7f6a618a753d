"""Shared test plumbing: golden loading, string interning, scenario replay on id-level backends."""
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
M64 = (1 << 64) - 1
EVENT_DTYPE = np.dtype([("op", "u1"), ("has_parent", "u1"), ("podtier", "<u2"), ("model", "<u4"),
                        ("parent_hash", "<u8"), ("hash_off", "<u8"), ("tok_off", "<u8"),
                        ("n_hashes", "<u4"), ("n_tokens", "<u4")])


SNAP_REQ_DTYPE = np.dtype([("hash", "<u8"), ("model", "<u2"), ("count", "u1"), ("zero", "u1"), ("ent", "<u2", (10,))])
SNAP_ENG_DTYPE = np.dtype([("hash", "<u8"), ("request", "<u8"), ("model", "<u2"), ("zero", "V6")])
assert SNAP_REQ_DTYPE.itemsize == 32 and SNAP_ENG_DTYPE.itemsize == 24


def golden(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


def csr(prompts):
    """list of token lists -> (tok uint32, off int64)."""
    off = np.zeros(len(prompts) + 1, np.int64)
    for i, p in enumerate(prompts):
        off[i + 1] = off[i] + len(p)
    tok = np.zeros(max(int(off[-1]), 1), np.uint32)
    for i, p in enumerate(prompts):
        tok[off[i]:off[i + 1]] = np.asarray(p, np.uint64).astype(np.uint32)
    return tok[:int(off[-1])] if off[-1] else tok[:0], off


class Interner:
    def __init__(self, names=()):
        self.ids = {}
        for n in names:
            self.id(n)

    def id(self, name):
        if name not in self.ids:
            self.ids[name] = len(self.ids)
        return self.ids[name]


def filter_mask(pod_ids, words):
    m = np.zeros(words, np.uint64)
    for p in pod_ids:
        m[p // 64] |= np.uint64(1) << np.uint64(p % 64)
    return m


def scenario_events(sc, pods: Interner, tiers: Interner, model_id=0):
    """scenario_small.json events -> (kvidx_event_t array, hashes, tokens) in arrival order."""
    ev, hashes, tokens = [], [], []
    for e in sc["events"]:
        if e["type"] == "AllBlocksCleared":
            continue                         # no-op in the reference (kvevents/pool.go:332-333); dropped on the host
        med = e.get("medium")
        tier = tiers.id(med.lower() if med is not None else "gpu")
        r = np.zeros((), EVENT_DTYPE)
        r["op"] = 0 if e["type"] == "BlockStored" else 1
        r["podtier"] = (pods.id(e["pod"]) << 4) | tier
        r["model"] = model_id
        r["hash_off"] = len(hashes)
        r["n_hashes"] = len(e["hashes"])
        hashes.extend(e["hashes"])
        if e["type"] == "BlockStored":
            r["has_parent"] = 0 if e["parent"] is None else 1
            r["parent_hash"] = e["parent"] or 0
            r["tok_off"] = len(tokens)
            r["n_tokens"] = len(e["tokens"])
            tokens.extend(e["tokens"])
        ev.append(r)
    return (np.array(ev, EVENT_DTYPE), np.array(hashes, np.uint64), np.array(tokens, np.uint64).astype(np.uint32))


def decode_snapshot(img):
    """A v1 image (include/kvidx.h) -> (request records, engine records) as structured arrays, in image order."""
    img = bytes(img)
    assert img[:8] == b"KVIDXSNP"
    R, E = np.frombuffer(img, "<u8", 2, 32)
    req = np.frombuffer(img, SNAP_REQ_DTYPE, int(R), 64)
    eng = np.frombuffer(img, SNAP_ENG_DTYPE, int(E), 64 + 32 * int(R))
    return req, eng


# ---- numpy replica of the table's home slot (csrc/fnv_cbor.cuh home_of, csrc/table.cuh slot_home) ---------------------
_GOLDEN = np.uint64(0x9E3779B97F4A7C15)
_MIX = (0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53)
_UNMIX = tuple(pow(c, -1, 1 << 64) for c in reversed(_MIX))


def _home_of(keys, model):
    x = np.asarray(keys, np.uint64) ^ (np.asarray(model, np.uint64) * _GOLDEN)
    x = np.atleast_1d(x).copy()
    x ^= x >> np.uint64(33)
    x *= np.uint64(_MIX[0])
    x ^= x >> np.uint64(33)
    x *= np.uint64(_MIX[1])
    x ^= x >> np.uint64(33)
    return x


def _slot_home(keys, model, S):
    return (_home_of(keys, model) & np.uint64((S - 1) & ~1)).astype(np.int64)


def keys_homed_at(slots, model, S, rng):
    """One key per entry of `slots` (even slots of an S-slot table) whose home slot under `model` is that slot.  The mix
    of _home_of is a bijection (xor-shifts by 33 and odd multipliers), so a random mixed value with the wanted low bits
    is unmixed into its key."""
    slots = np.asarray(slots, np.int64)
    assert not (slots & 1).any()
    x = rng.integers(0, 1 << 64, len(slots), dtype=np.uint64)
    x = (x & ~np.uint64((S - 1) & ~1)) | slots.astype(np.uint64)
    x ^= x >> np.uint64(33)
    x *= np.uint64(_UNMIX[0])
    x ^= x >> np.uint64(33)
    x *= np.uint64(_UNMIX[1])
    x ^= x >> np.uint64(33)
    return x ^ np.uint64(int(model) * int(_GOLDEN) & M64)


def free_pairs(state):
    """Even slots s of a table's state array (0 = EMPTY) whose pair s, s + 1 is fully EMPTY."""
    return np.flatnonzero((state[0::2] == 0) & (state[1::2] == 0)) * 2


def keep_free(cands, model, state):
    """Of the candidate keys (in order), the first one for each home pair that is fully EMPTY in `state`: inserted in one
    call, each of them lands on its even home slot, wherever the call's inserts run."""
    cands = np.asarray(cands, np.uint64)
    home = _slot_home(cands, model, len(state))
    ok = (state[home] == 0) & (state[home + 1] == 0)
    _, first = np.unique(home, return_index=True)
    keep = np.zeros(len(cands), bool)
    keep[first] = True
    return cands[ok & keep]


def draw_free(state, n, model, rng):
    """n random keys (no two with one home pair) that keep_free keeps."""
    out = np.zeros(0, np.uint64)
    while len(out) < n:
        c = keep_free(rng.integers(1, 1 << 64, 4 * n + 64, dtype=np.uint64), model, state)
        c = c[~np.isin(_slot_home(c, model, len(state)), _slot_home(out, model, len(state)))]
        out = np.concatenate([out, c])
    return out[:n]


def dense_from_map(scores, pods: Interner, P):
    row = np.full(P, -1.0)
    if scores:
        for p, s in scores.items():
            row[pods.ids[p]] = s
    return row


# ---- GPU Score() paths: a handle reads these variables when it is created, so every path needs its own handle ----------
def _index_pair(**kw):
    import kvidx
    from oracle.kvoracle_c import COracle
    w = kw.pop("tier_weights", (1.0, 0.8))
    ix = kvidx.Index(tier_weights=w, **kw)
    co = COracle(block_size=kw.get("block_size", 16), init_hash=kvidx.fnv64a(kw.get("hash_seed", "").encode()),
                 size=kw.get("capacity", 1 << 20), pod_cache_size=kw.get("pods_per_key", 10), tier_weights=w,
                 max_pods=kw.get("max_pods", 256))
    return ix, co


def _select_path(monkeypatch, path):
    """v1: thread-per-prompt kernel; rounds*: hash / walk rounds, every prompt on
    its own (one stream / two halves on two streams / without the prefix sort); classes*: the round pipeline that hashes
    and walks one representative per distinct prefix (one part / 2 / 8 / 16 parts / unsorted / sharing switched off /
    whole chunks only, no partial followers; the variants also with the batch split into parts)."""
    if path == "v1":
        monkeypatch.setenv("KVIDX_SCORE_KERNEL", "v1")
        return
    if path == "auto":                       # the library chooses: here every batch is "large", so it is the class pipeline
        monkeypatch.setenv("KVIDX_COOP_MAX", "0")          # or the per-prompt rounds, by how much the batch repeats itself
                                                           # (small batches would otherwise take the warp-per-prompt kernel)
        monkeypatch.setenv("KVIDX_CLASSES_MIN", "64")
        monkeypatch.setenv("KVIDX_ROUNDS_OVERLAP_MIN", "64")
        return
    base, _, var = path.partition("-")
    parts = base.lstrip("abcdefghijklmnopqrstuvwxyz")
    base = base[: len(base) - len(parts)]
    monkeypatch.setenv("KVIDX_SCORE_PATH", base)
    if parts:
        monkeypatch.setenv("KVIDX_ROUNDS_OVERLAP_MIN", "64")
        monkeypatch.setenv("KVIDX_ROUNDS_PARTS", parts)
    else:                                    # no batch is large enough to be split
        monkeypatch.setenv("KVIDX_ROUNDS_OVERLAP_MIN", str(1 << 62))
    if var == "nosort":
        monkeypatch.setenv("KVIDX_SORT_PREFIX", "0")
    elif var == "nodedup":
        monkeypatch.setenv("KVIDX_ROUNDS_DEDUP", "0")
    elif var == "whole":
        monkeypatch.setenv("KVIDX_ROUNDS_DEDUP", "1")
    elif var == "lane":                      # per-prompt rounds with the lane-per-prompt kernel P (what batches above 131 072 take)
        monkeypatch.setenv("KVIDX_ROUNDS_WARP_MAX", "0")


ROUND_PATHS = ["rounds", "rounds2", "rounds-nosort", "rounds2-nosort", "rounds-lane", "rounds2-lane", "classes", "classes2", "classes8",
               "classes16", "classes-nosort", "classes2-nosort", "classes8-nosort", "classes-nodedup", "classes2-nodedup",
               "classes8-nodedup", "classes-whole", "classes2-whole", "classes4-whole", "classes8-whole", "auto"]
PATHS = ["v1", "coop"] + ROUND_PATHS
# Tests seed a path's random inputs from its position in one of these lists.  Both keep "fused", a Score() kernel since
# retired, so that every remaining path keeps the inputs it has always been checked on: SEED_ORDER for PATHS,
# SEED_ORDER_SIZES for the sorted names of test_gpu_remove_pods.PATH_SIZES.
SEED_ORDER = ["v1", "fused", "coop"] + ROUND_PATHS
SEED_ORDER_SIZES = ["auto", "classes", "coop", "default", "fused", "rounds", "v1"]
