"""ctypes binding of libkvidx.so (include/kvidx.h).

This is the only way Python reaches the product: there is NO Python or CPU
implementation of the path behind it.  If the library is missing or no CUDA
device is present, loading / ``Index()`` raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.environ.get("KVIDX_LIB") or os.path.join(_PKG, "lib", "libkvidx.so")   # KVIDX_LIB: experiment builds only

E = 10            # KVIDX_MAX_PODS_PER_KEY
MAX_TIERS = 16
SCORE_ABSENT = -1.0
OK, ENOENT, ECUDA, ENOMEM, EINVAL, ENOSPC, ERANGE = 0, -2, -5, -12, -22, -28, -34
EV_BLOCK_STORED, EV_BLOCK_REMOVED = 0, 1
PAYLOAD_SKIP_UNKNOWN_TIER, PAYLOAD_STOP_AT_CLEARED = 1, 2
PAYLOAD_MSG_DECODED, PAYLOAD_MSG_UNKNOWN_TIER, PAYLOAD_MSG_CLEARED = 1, 2, 4
PAYLOAD_COUNTS = ("messages", "events", "hashes", "tokens", "queues", "admitted", "removed", "markers")
EVICT_NONE, EVICT_CLOCK = 0, 1
ANY_MODEL, INVENTORY_ENGINE = 0xFFFFFFFF, 1
_EVICT_POLICIES = {"none": EVICT_NONE, "clock": EVICT_CLOCK}


class Config(C.Structure):
    """kvidx_config_t."""
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("block_size", C.c_uint32),
                ("pods_per_key", C.c_uint32), ("init_hash", C.c_uint64), ("capacity", C.c_uint64),
                ("table_slots", C.c_uint64), ("max_pods", C.c_uint32), ("n_tier_weights", C.c_uint32),
                ("tier_weight", C.c_double * MAX_TIERS), ("lru_exact", C.c_uint32), ("shard_rank", C.c_uint32),
                ("shard_count", C.c_uint32), ("evict_policy", C.c_uint32), ("grow_tables", C.c_uint32),
                ("reserved", C.c_uint32 * 3)]


class Stats(C.Structure):
    """kvidx_stats_t."""
    _fields_ = [(n, C.c_uint64) for n in ("request_keys", "engine_keys", "request_tombs", "engine_tombs",
                                          "request_slots", "engine_slots", "rebuilds", "kernel_launches",
                                          "rehashed_events", "coalesced_calls")]


EVENT_DTYPE = np.dtype([("op", "u1"), ("has_parent", "u1"), ("podtier", "<u2"), ("model", "<u4"),
                        ("parent_hash", "<u8"), ("hash_off", "<u8"), ("tok_off", "<u8"),
                        ("n_hashes", "<u4"), ("n_tokens", "<u4")])
assert EVENT_DTYPE.itemsize == 40

_u32p, _u64p, _i64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_int64)
_u16p, _u8p, _f64p = C.POINTER(C.c_uint16), C.POINTER(C.c_uint8), C.POINTER(C.c_double)

# every symbol include/kvidx.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "kvidx_abi_version": (C.c_int, []),
    "kvidx_config_default": (None, [C.POINTER(Config)]),
    "kvidx_create": (C.c_int, [C.POINTER(Config), C.POINTER(C.c_void_p)]),
    "kvidx_destroy": (None, [C.c_void_p]),
    "kvidx_last_error": (C.c_char_p, [C.c_void_p]),
    "kvidx_fnv64a": (C.c_uint64, [C.c_char_p, C.c_size_t]),
    "kvidx_fnv32a": (C.c_uint32, [C.c_char_p, C.c_size_t]),
    "kvidx_queue_index": (C.c_uint32, [C.c_char_p, C.c_size_t, C.c_uint32]),
    "kvidx_set_tier_weight": (C.c_int, [C.c_void_p, C.c_uint32, C.c_double]),
    "kvidx_host_alloc": (C.c_void_p, [C.c_size_t]),
    "kvidx_host_free": (None, [C.c_void_p]),
    "kvidx_hash_keys": (C.c_int, [C.c_void_p, _u32p, _i64p, C.c_int64, _u64p, _u8p, _u64p, _i64p]),
    "kvidx_lookup": (C.c_int, [C.c_void_p, C.c_uint32, _u64p, C.c_int64, _u64p, _u16p, _u8p]),
    "kvidx_score_batch": (C.c_int, [C.c_void_p, _u32p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, _f64p, _u8p]),
    "kvidx_score_batch_sparse": (C.c_int, [C.c_void_p, _u32p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, _u16p, _f64p, _u8p, _u8p]),
    "kvidx_lookup_hits": (C.c_int, [C.c_void_p, _u32p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, _u32p]),
    "kvidx_lookup_hits_keys": (C.c_int, [C.c_void_p, _u64p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, _u32p]),
    "kvidx_lookup_hits_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
    "kvidx_lookup_hits_keys_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
    "kvidx_score_keys": (C.c_int,[C.c_void_p, _u64p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, _f64p, _u8p]),
    "kvidx_score_keys_sparse": (C.c_int, [C.c_void_p, _u64p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, _u16p, _f64p, _u8p, _u8p]),
    "kvidx_score_keys_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kvidx_score_keys_sparse_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kvidx_score_turn": (C.c_int, [C.c_void_p, _u64p, _i64p, _u32p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, _f64p, _u8p, _u64p, _i64p]),
    "kvidx_score_turn_sparse": (C.c_int, [C.c_void_p, _u64p, _i64p, _u32p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, _u16p, _f64p, _u8p, _u8p,
                                          _u64p, _i64p]),
    "kvidx_score_turn_dev": (C.c_int, [C.c_void_p] + [C.c_void_p] * 4 + [C.c_int64, C.c_void_p, C.c_uint32] + [C.c_void_p] * 5),
    "kvidx_score_turn_sparse_dev": (C.c_int, [C.c_void_p] + [C.c_void_p] * 4 + [C.c_int64, C.c_void_p, C.c_uint32] + [C.c_void_p] * 7),
    "kvidx_add": (C.c_int, [C.c_void_p, C.c_uint32, _u64p, _u64p, C.c_int64, _u16p, C.c_int32]),
    "kvidx_evict": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint64, _u16p, C.c_int32]),
    "kvidx_get_request_key": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint64, _u64p]),
    "kvidx_apply_events": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, _u64p, C.c_int64, _u32p, C.c_int64, _i64p]),
    "kvidx_remove_pods": (C.c_int, [C.c_void_p, _u64p, C.c_uint32, _u64p]),
    "kvidx_snapshot": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "kvidx_restore": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64, _u64p]),
    "kvidx_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "kvidx_synchronize": (C.c_int, [C.c_void_p]),
    "kvidx_score_batch_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kvidx_hash_keys_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kvidx_apply_events_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "kvidx_decode_event_payloads_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, _u8p, _i64p,
                                                  C.c_uint32, C.c_int32, C.c_uint32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                                  C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, _i64p]),
    "kvidx_apply_event_payloads": (C.c_int, [C.c_void_p, _u8p, _i64p, C.c_int64, _u32p, _u32p, _u8p, _i64p, C.c_uint32, C.c_int32,
                                             C.c_uint32, _u8p, _i64p, _i64p]),
    "kvidx_score_batch_sparse_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kvidx_shard_compact": (C.c_int, [C.c_void_p]),
    "kvidx_key_owners_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p]),
    "kvidx_probe_slots_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p]),
    "kvidx_score_slots_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kvidx_get_stats": (C.c_int, [C.c_void_p, C.POINTER(Stats)]),
    "kvidx_get_evictions": (C.c_int, [C.c_void_p, _u64p]),
    "kvidx_get_sweeps": (C.c_int, [C.c_void_p, _u64p]),
    "kvidx_pod_inventory": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, _u64p, _u64p, _u64p, _u64p, _u64p]),
    "kvidx_shard_export": (C.c_int, [C.c_void_p, C.c_char_p]),
    "kvidx_shard_import": (C.c_int, [C.c_void_p, C.c_uint32, C.c_char_p]),
    "kvidx_shard_attach": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "kvidx_shard_remove_pods": (C.c_int, [C.c_void_p, _u64p, C.c_uint32, C.c_uint32, _u64p]),
    "kvidx_shard_snapshot": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "kvidx_snapshot_merge": (C.c_int, [C.POINTER(C.c_char_p), _u64p, C.c_uint32, C.c_void_p, C.c_uint64, _u64p]),
    "kvidx_shard_restore": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64, _u64p]),
    "kvidx_text_store_init": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32]),
    "kvidx_text_store_add": (C.c_int, [C.c_void_p, _u8p, _i64p, C.c_int64, _u32p, _u64p, _i64p]),
    "kvidx_text_store_find": (C.c_int, [C.c_void_p, _u8p, _i64p, C.c_int64, _u32p, C.c_int64, _i64p, _f64p]),
    "kvidx_text_store_len": (C.c_int, [C.c_void_p, _i64p]),
    "kvidx_text_store_snapshot": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "kvidx_text_store_restore": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64, _i64p]),
    "kvidx_text_hash_keys": (C.c_int, [C.c_void_p, _u8p, _i64p, C.c_int64, C.c_int32, _u64p, _i64p]),
    "kvidx_score_text": (C.c_int, [C.c_void_p, _u8p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, C.c_double, _f64p, _u8p, _u8p, _f64p]),
    "kvidx_score_text_sparse": (C.c_int, [C.c_void_p, _u8p, _i64p, C.c_int64, _u32p, C.c_uint32, _u64p, C.c_double, _u16p, _f64p, _u8p, _u8p,
                                          _u8p, _f64p]),
    "kvidx_score_text_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_double]
                             + [C.c_void_p] * 4),
    "kvidx_score_text_sparse_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_double]
                                    + [C.c_void_p] * 6),
}

_lib = None


def load():
    """dlopen libkvidx.so and type every exported symbol.  Raises if the library is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise OSError("libkvidx.so not built (%s): run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "or ./build.sh -- there is no CPU fallback" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            f = getattr(L, name)      # AttributeError if the header and the library disagree
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


class KvidxError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("kvidx error %d: %s" % (code, msg))
        self.code = code


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _u8(text):
    return np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text, np.uint8)


def pack_text(prompts):
    """Prompts (str or bytes; str as UTF-8) -> (text bytes as uint8, offsets (n+1)): the CSR the text calls take."""
    raw = [p.encode("utf-8") if isinstance(p, str) else bytes(p) for p in prompts]
    off = np.zeros(len(raw) + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in raw])
    return np.frombuffer(b"".join(raw), np.uint8) if raw else np.zeros(0, np.uint8), off


def fnv64a(data: bytes) -> int:
    return load().kvidx_fnv64a(data, len(data))


def podtier(pod: int, tier: int) -> int:
    return ((pod << 4) | (tier & 15)) & 0xFFFF


class Index:
    """One libkvidx handle (== kvblock.Index + TokenProcessor + scorer of the reference, ids not strings)."""

    def __init__(self, block_size=16, init_hash=None, hash_seed="", capacity=1 << 20, pods_per_key=10,
                 tier_weights=(1.0, 0.8), max_pods=256, table_slots=0, device=0, lru_exact=0, shard_rank=0, shard_count=0,
                 evict_policy="none", grow_tables=False):
        """evict_policy: "none" (capacity only sizes the table) or "clock" (each map held to `capacity` keys by a CLOCK
        sweep after every write call, include/kvidx.h); an int is passed to the C ABI as it is.
        grow_tables: the tables start small and grow on demand up to the size a fixed handle allocates for `capacity`
        (include/kvidx.h); an int is passed to the C ABI as it is."""
        self.L = load()
        cfg = Config()
        self.L.kvidx_config_default(C.byref(cfg))
        cfg.device = device
        cfg.block_size = block_size
        cfg.pods_per_key = pods_per_key
        cfg.init_hash = fnv64a(hash_seed.encode()) if init_hash is None else init_hash
        cfg.capacity = capacity
        cfg.table_slots = table_slots
        cfg.max_pods = max_pods
        cfg.n_tier_weights = len(tier_weights)
        for i, w in enumerate(tier_weights):
            cfg.tier_weight[i] = float(w)
        cfg.lru_exact = lru_exact
        cfg.shard_rank, cfg.shard_count = shard_rank, shard_count
        cfg.evict_policy = _EVICT_POLICIES[evict_policy] if isinstance(evict_policy, str) else int(evict_policy)
        cfg.grow_tables = int(grow_tables)
        h = C.c_void_p()
        rc = self.L.kvidx_create(C.byref(cfg), C.byref(h))
        if rc:
            raise KvidxError(rc, self.L.kvidx_last_error(None).decode())
        self.h = h
        self.block_size, self.max_pods = block_size, max_pods
        self.filter_words = (max_pods + 63) // 64
        self.lru_exact = bool(lru_exact)

    @classmethod
    def borrow(cls, handle: int, block_size=16, max_pods=256) -> "Index":
        """An Index over a handle that another owner created and destroys (kvhost_index of a HostIndexer)."""
        self = cls.__new__(cls)
        self.L, self.h, self._borrowed = load(), C.c_void_p(handle), True
        self.block_size, self.max_pods = block_size, max_pods
        self.filter_words = (max_pods + 63) // 64
        self.lru_exact = False
        return self

    # -- plumbing --
    def close(self):
        if getattr(self, "_borrowed", False):
            self.h = None
        if getattr(self, "h", None):
            self.L.kvidx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc:
            raise KvidxError(rc, self.L.kvidx_last_error(self.h).decode())

    def last_error(self) -> str:
        return self.L.kvidx_last_error(self.h).decode()

    def set_stream(self, cuda_stream: int):
        self._ck(self.L.kvidx_set_stream(self.h, C.c_void_p(cuda_stream)))

    def synchronize(self):
        self._ck(self.L.kvidx_synchronize(self.h))

    def set_tier_weight(self, tier, w):
        self._ck(self.L.kvidx_set_tier_weight(self.h, tier, float(w)))

    def stats(self) -> dict:
        s = Stats()
        self._ck(self.L.kvidx_get_stats(self.h, C.byref(s)))
        return {n: getattr(s, n) for n, _ in Stats._fields_}

    def evictions(self) -> tuple:
        """(request keys, engine mappings) dropped by the capacity bound since the handle was created."""
        out = np.zeros(2, np.uint64)
        self._ck(self.L.kvidx_get_evictions(self.h, _p(out, _u64p)))
        return int(out[0]), int(out[1])

    def sweeps(self) -> tuple:
        """CLOCK mode: (sweeps that evicted, those that went past a full turn of the hand), both maps together."""
        out = np.zeros(2, np.uint64)
        self._ck(self.L.kvidx_get_sweeps(self.h, _p(out, _u64p)))
        return int(out[0]), int(out[1])

    def pod_inventory(self, model=None, engine=False) -> dict:
        """kvidx_pod_inventory: what each pod holds, counted on the device without touching recency.  model None = all models.
        -> {"entries" (max_pods, 16), "keys", "sole" (max_pods,), "sole_engine" (max_pods,) or None without `engine`,
        "totals" [request keys, entries, engine mappings, stale engine mappings] (the last two only with `engine`)}, uint64.
        remove_pods([p]) right after an all-model inventory removes entries[p].sum() entries, sole[p] request keys and
        sole_engine[p] engine keys.  On a sharded handle: this rank's share (kvidx.dist.pod_inventory_shards sums them)."""
        ent = np.zeros((self.max_pods, MAX_TIERS), np.uint64)
        keys, sole, totals = np.zeros(self.max_pods, np.uint64), np.zeros(self.max_pods, np.uint64), np.zeros(4, np.uint64)
        sole_eng = np.zeros(self.max_pods, np.uint64) if engine else None
        self._ck(self.L.kvidx_pod_inventory(self.h, ANY_MODEL if model is None else int(model), INVENTORY_ENGINE if engine else 0,
                                            _p(ent, _u64p), _p(keys, _u64p), _p(sole, _u64p), _p(sole_eng, _u64p), _p(totals, _u64p)))
        return {"entries": ent, "keys": keys, "sole": sole, "sole_engine": sole_eng, "totals": totals}

    # -- hash-range sharding (one handle per GPU) --
    SHARD_HANDLE_BYTES = 192

    def shard_export(self) -> bytes:
        buf = C.create_string_buffer(self.SHARD_HANDLE_BYTES)
        self._ck(self.L.kvidx_shard_export(self.h, buf))
        return buf.raw

    def shard_import(self, rank: int, handle: bytes):
        self._ck(self.L.kvidx_shard_import(self.h, rank, handle))

    def shard_attach(self, rank: int, other: "Index"):
        self._ck(self.L.kvidx_shard_attach(self.h, rank, other.h))

    def shard_compact(self):
        """Drop this shard's tombstones.  Collective by contract (see kvidx.dist.compact_shards)."""
        self._ck(self.L.kvidx_shard_compact(self.h))

    # -- read path --
    def hash_keys(self, tok, tok_off, parent=None, parent_valid=None):
        tok = np.ascontiguousarray(tok, np.uint32)
        tok_off = np.ascontiguousarray(tok_off, np.int64)
        n = len(tok_off) - 1
        nk = int(((tok_off[1:] - tok_off[:-1]) // self.block_size).sum())
        keys = np.zeros(max(nk, 1), np.uint64)
        koff = np.zeros(n + 1, np.int64)
        parent = None if parent is None else np.ascontiguousarray(parent, np.uint64)
        parent_valid = None if parent_valid is None else np.ascontiguousarray(parent_valid, np.uint8)
        self._ck(self.L.kvidx_hash_keys(self.h, _p(tok, _u32p), _p(tok_off, _i64p), n, _p(parent, _u64p),
                                        _p(parent_valid, _u8p), _p(keys, _u64p), _p(koff, _i64p)))
        return keys[:nk], koff

    def lookup(self, model, keys, filter_mask=None):
        keys = np.ascontiguousarray(keys, np.uint64)
        n = len(keys)
        pt = np.zeros((max(n, 1), E), np.uint16)
        cnt = np.zeros(max(n, 1), np.uint8)
        filter_mask = None if filter_mask is None else np.ascontiguousarray(filter_mask, np.uint64)
        rc = self.L.kvidx_lookup(self.h, model, _p(keys, _u64p), n, _p(filter_mask, _u64p), _p(pt, _u16p), _p(cnt, _u8p))
        return rc, pt[:n], cnt[:n]

    def score_batch(self, tok, tok_off, model=None, model0=0, filter_mask=None, out=None):
        tok = np.ascontiguousarray(tok, np.uint32) if not isinstance(tok, _Raw) else tok
        tok_off = np.ascontiguousarray(tok_off, np.int64)
        n = len(tok_off) - 1
        scores = np.empty((n, self.max_pods), np.float64) if out is None else out
        has = np.zeros(n, np.uint8)
        model = None if model is None else np.ascontiguousarray(model, np.uint32)
        filter_mask = None if filter_mask is None else np.ascontiguousarray(filter_mask, np.uint64)
        tp = C.cast(tok.ptr, _u32p) if isinstance(tok, _Raw) else _p(tok, _u32p)
        self._ck(self.L.kvidx_score_batch(self.h, tp, _p(tok_off, _i64p), n, _p(model, _u32p), model0,
                                          _p(filter_mask, _u64p), _p(scores, _f64p), _p(has, _u8p)))
        return scores, has

    def score_batch_sparse(self, tok, tok_off, model=None, model0=0, filter_mask=None, out=None):
        """out: optional preallocated (pods (n,10) uint16, scores (n,10) float64, cnt (n,) uint8, has (n,) uint8)."""
        tok = np.ascontiguousarray(tok, np.uint32)
        tok_off = np.ascontiguousarray(tok_off, np.int64)
        n = len(tok_off) - 1
        if out is None:
            pods = np.zeros((n, E), np.uint16)
            scores = np.zeros((n, E), np.float64)
            cnt = np.zeros(n, np.uint8)
            has = np.zeros(n, np.uint8)
        else:
            pods, scores, cnt, has = out
        model = None if model is None else np.ascontiguousarray(model, np.uint32)
        filter_mask = None if filter_mask is None else np.ascontiguousarray(filter_mask, np.uint64)
        self._ck(self.L.kvidx_score_batch_sparse(self.h, _p(tok, _u32p), _p(tok_off, _i64p), n, _p(model, _u32p), model0,
                                                 _p(filter_mask, _u64p), _p(pods, _u16p), _p(scores, _f64p), _p(cnt, _u8p),
                                                 _p(has, _u8p)))
        return pods, scores, cnt, has

    def score_batch_dev(self, d_tok, d_tok_off, n, d_scores, d_model=0, model0=0, d_filter=0, d_has_keys=0):
        """All pointers are device addresses (ints).  Asynchronous on the handle's stream."""
        self._ck(self.L.kvidx_score_batch_dev(self.h, d_tok, d_tok_off, n, d_model or None, model0, d_filter or None,
                                              d_scores, d_has_keys or None))

    def score_batch_sparse_dev(self, d_tok, d_tok_off, n, d_pods, d_scores, d_cnt, d_model=0, model0=0, d_filter=0, d_has_keys=0):
        """Sparse result rows (<= 10 (pod, score) pairs per prompt) on the device; pointers are device addresses."""
        self._ck(self.L.kvidx_score_batch_sparse_dev(self.h, d_tok, d_tok_off, n, d_model or None, model0, d_filter or None,
                                                     d_pods, d_scores, d_cnt, d_has_keys or None))

    # -- Score() from request keys (GetPodScores steps 3-4): prompt i owns keys[key_off[i] .. key_off[i+1]) --
    def score_keys(self, keys, key_off, model=None, model0=0, filter_mask=None, out=None):
        """Dense rows (n, max_pods) and has_keys, as score_batch; `keys` may be a numpy array or a _Raw pinned pointer."""
        keys = np.ascontiguousarray(keys, np.uint64) if not isinstance(keys, _Raw) else keys
        key_off = np.ascontiguousarray(key_off, np.int64)
        n = len(key_off) - 1
        scores = np.empty((n, self.max_pods), np.float64) if out is None else out
        has = np.zeros(n, np.uint8)
        model = None if model is None else np.ascontiguousarray(model, np.uint32)
        filter_mask = None if filter_mask is None else np.ascontiguousarray(filter_mask, np.uint64)
        kp = C.cast(keys.ptr, _u64p) if isinstance(keys, _Raw) else _p(keys, _u64p)
        self._ck(self.L.kvidx_score_keys(self.h, kp, _p(key_off, _i64p), n, _p(model, _u32p), model0,
                                         _p(filter_mask, _u64p), _p(scores, _f64p), _p(has, _u8p)))
        return scores, has

    def score_keys_sparse(self, keys, key_off, model=None, model0=0, filter_mask=None, out=None):
        """Sparse rows as score_batch_sparse; out: optional preallocated (pods, scores, cnt, has)."""
        keys = np.ascontiguousarray(keys, np.uint64)
        key_off = np.ascontiguousarray(key_off, np.int64)
        n = len(key_off) - 1
        if out is None:
            pods = np.zeros((n, E), np.uint16)
            scores = np.zeros((n, E), np.float64)
            cnt = np.zeros(n, np.uint8)
            has = np.zeros(n, np.uint8)
        else:
            pods, scores, cnt, has = out
        model = None if model is None else np.ascontiguousarray(model, np.uint32)
        filter_mask = None if filter_mask is None else np.ascontiguousarray(filter_mask, np.uint64)
        self._ck(self.L.kvidx_score_keys_sparse(self.h, _p(keys, _u64p), _p(key_off, _i64p), n, _p(model, _u32p), model0,
                                                _p(filter_mask, _u64p), _p(pods, _u16p), _p(scores, _f64p), _p(cnt, _u8p),
                                                _p(has, _u8p)))
        return pods, scores, cnt, has

    def score_keys_dev(self, d_keys, d_key_off, n, d_scores, d_model=0, model0=0, d_filter=0, d_has_keys=0):
        """All pointers are device addresses (ints).  Asynchronous on the handle's stream."""
        self._ck(self.L.kvidx_score_keys_dev(self.h, d_keys or None, d_key_off, n, d_model or None, model0, d_filter or None,
                                             d_scores, d_has_keys or None))

    def score_keys_sparse_dev(self, d_keys, d_key_off, n, d_pods, d_scores, d_cnt, d_model=0, model0=0, d_filter=0, d_has_keys=0):
        self._ck(self.L.kvidx_score_keys_sparse_dev(self.h, d_keys or None, d_key_off, n, d_model or None, model0, d_filter or None,
                                                    d_pods, d_scores, d_cnt, d_has_keys or None))

    # -- Lookup hit counts: recordHitMetrics(Lookup(K_i, F_i)) per prompt, the full-depth count the instrumented index adds --
    def lookup_hits(self, tok, tok_off, model=None, model0=0, filter_mask=None):
        """Hit count of every prompt given as tokens (uint32 (n,)); `tok` may be a numpy array or a _Raw pinned pointer."""
        tok = np.ascontiguousarray(tok, np.uint32) if not isinstance(tok, _Raw) else tok
        tok_off = np.ascontiguousarray(tok_off, np.int64)
        n = len(tok_off) - 1
        hits = np.zeros(max(n, 0), np.uint32)
        model = None if model is None else np.ascontiguousarray(model, np.uint32)
        filter_mask = None if filter_mask is None else np.ascontiguousarray(filter_mask, np.uint64)
        tp = C.cast(tok.ptr, _u32p) if isinstance(tok, _Raw) else _p(tok, _u32p)
        self._ck(self.L.kvidx_lookup_hits(self.h, tp, _p(tok_off, _i64p), n, _p(model, _u32p), model0,
                                          _p(filter_mask, _u64p), _p(hits, _u32p)))
        return hits

    def lookup_hits_keys(self, keys, key_off, model=None, model0=0, filter_mask=None):
        """Hit count of every prompt given as request keys; `keys` may be a numpy array or a _Raw pinned pointer."""
        keys = np.ascontiguousarray(keys, np.uint64) if not isinstance(keys, _Raw) else keys
        key_off = np.ascontiguousarray(key_off, np.int64)
        n = len(key_off) - 1
        hits = np.zeros(max(n, 0), np.uint32)
        model = None if model is None else np.ascontiguousarray(model, np.uint32)
        filter_mask = None if filter_mask is None else np.ascontiguousarray(filter_mask, np.uint64)
        kp = C.cast(keys.ptr, _u64p) if isinstance(keys, _Raw) else _p(keys, _u64p)
        self._ck(self.L.kvidx_lookup_hits_keys(self.h, kp, _p(key_off, _i64p), n, _p(model, _u32p), model0,
                                               _p(filter_mask, _u64p), _p(hits, _u32p)))
        return hits

    def lookup_hits_dev(self, d_tok, d_tok_off, n, d_hits, d_model=0, model0=0, d_filter=0):
        """All pointers are device addresses (ints); d_hits: n uint32.  Reads the first and last offsets back, then asynchronous."""
        self._ck(self.L.kvidx_lookup_hits_dev(self.h, d_tok or None, d_tok_off, n, d_model or None, model0, d_filter or None, d_hits))

    def lookup_hits_keys_dev(self, d_keys, d_key_off, n, d_hits, d_model=0, model0=0, d_filter=0):
        """All pointers are device addresses (ints); d_hits: n uint32.  Asynchronous on the handle's stream."""
        self._ck(self.L.kvidx_lookup_hits_keys_dev(self.h, d_keys or None, d_key_off, n, d_model or None, model0, d_filter or None,
                                                   d_hits))

    # -- Score() for a conversation turn: prompt i is keys[key_off[i] .. key_off[i+1]) then tok[tok_off[i] .. tok_off[i+1]) --
    def _turn_args(self, keys, key_off, tok, tok_off, model, filter_mask, want_keys):
        keys = np.ascontiguousarray(keys, np.uint64) if not isinstance(keys, _Raw) else keys
        tok = np.ascontiguousarray(tok, np.uint32) if not isinstance(tok, _Raw) else tok
        key_off = np.ascontiguousarray(key_off, np.int64)
        tok_off = np.ascontiguousarray(tok_off, np.int64)
        n = len(key_off) - 1
        nk = int(((tok_off[1:] - tok_off[:-1]) // self.block_size).sum()) if n > 0 else 0
        new_keys = np.zeros(max(nk, 1), np.uint64) if want_keys else None
        new_off = np.zeros(n + 1, np.int64)
        model = None if model is None else np.ascontiguousarray(model, np.uint32)
        filter_mask = None if filter_mask is None else np.ascontiguousarray(filter_mask, np.uint64)
        kp = C.cast(keys.ptr, _u64p) if isinstance(keys, _Raw) else _p(keys, _u64p)
        tp = C.cast(tok.ptr, _u32p) if isinstance(tok, _Raw) else _p(tok, _u32p)
        return n, nk, kp, tp, key_off, tok_off, model, filter_mask, new_keys, new_off

    def score_turn(self, keys, key_off, tok, tok_off, model=None, model0=0, filter_mask=None, want_keys=True, out=None):
        """One conversation turn per prompt: held request keys, then new tokens.  -> (dense rows (n, max_pods), has_keys,
        new keys (None when want_keys is False), their offsets).  keys / tok may be numpy arrays or _Raw pinned pointers."""
        n, nk, kp, tp, key_off, tok_off, model, filter_mask, new_keys, new_off = self._turn_args(keys, key_off, tok, tok_off, model, filter_mask, want_keys)
        scores = np.empty((n, self.max_pods), np.float64) if out is None else out
        has = np.zeros(n, np.uint8)
        self._ck(self.L.kvidx_score_turn(self.h, kp, _p(key_off, _i64p), tp, _p(tok_off, _i64p), n, _p(model, _u32p), model0,
                                         _p(filter_mask, _u64p), _p(scores, _f64p), _p(has, _u8p), _p(new_keys, _u64p), _p(new_off, _i64p)))
        return scores, has, None if new_keys is None else new_keys[:nk], new_off

    def score_turn_sparse(self, keys, key_off, tok, tok_off, model=None, model0=0, filter_mask=None, want_keys=True, out=None):
        """Sparse rows as score_keys_sparse -> (pods, scores, cnt, has, new keys, their offsets); out: optional preallocated
        (pods, scores, cnt, has)."""
        n, nk, kp, tp, key_off, tok_off, model, filter_mask, new_keys, new_off = self._turn_args(keys, key_off, tok, tok_off, model, filter_mask, want_keys)
        if out is None:
            pods, scores = np.zeros((n, E), np.uint16), np.zeros((n, E), np.float64)
            cnt, has = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        else:
            pods, scores, cnt, has = out
        self._ck(self.L.kvidx_score_turn_sparse(self.h, kp, _p(key_off, _i64p), tp, _p(tok_off, _i64p), n, _p(model, _u32p), model0,
                                                _p(filter_mask, _u64p), _p(pods, _u16p), _p(scores, _f64p), _p(cnt, _u8p), _p(has, _u8p),
                                                _p(new_keys, _u64p), _p(new_off, _i64p)))
        return pods, scores, cnt, has, None if new_keys is None else new_keys[:nk], new_off

    def score_turn_dev(self, d_keys, d_key_off, d_tok, d_tok_off, n, d_scores, d_model=0, model0=0, d_filter=0, d_has_keys=0,
                       d_new_key_off=0, d_new_keys=0):
        """All pointers are device addresses (ints); d_new_keys 0: the new keys are not wanted.  Asynchronous on the handle's stream."""
        self._ck(self.L.kvidx_score_turn_dev(self.h, d_keys or None, d_key_off, d_tok or None, d_tok_off, n, d_model or None, model0,
                                             d_filter or None, d_scores, d_has_keys or None, d_new_key_off or None, d_new_keys or None))

    def score_turn_sparse_dev(self, d_keys, d_key_off, d_tok, d_tok_off, n, d_pods, d_scores, d_cnt, d_model=0, model0=0, d_filter=0,
                              d_has_keys=0, d_new_key_off=0, d_new_keys=0):
        self._ck(self.L.kvidx_score_turn_sparse_dev(self.h, d_keys or None, d_key_off, d_tok or None, d_tok_off, n, d_model or None, model0,
                                                    d_filter or None, d_pods, d_scores, d_cnt, d_has_keys or None, d_new_key_off or None,
                                                    d_new_keys or None))

    def hash_keys_dev(self, d_tok, d_tok_off, n, d_key_off, d_keys, d_parent=0, d_parent_valid=0):
        self._ck(self.L.kvidx_hash_keys_dev(self.h, d_tok, d_tok_off, n, d_parent or None, d_parent_valid or None, d_key_off, d_keys))

    def key_owners_dev(self, d_keys, n, d_owner, model0=0, d_model=0):
        self._ck(self.L.kvidx_key_owners_dev(self.h, d_keys, d_model or None, model0, n, d_owner))

    def probe_slots_dev(self, d_keys, n, d_slots, model0=0, d_model=0):
        self._ck(self.L.kvidx_probe_slots_dev(self.h, d_keys, d_model or None, model0, n, d_slots))

    def score_slots_dev(self, d_slots, d_key_off, n_prompts, d_scores, d_filter=0, d_has_keys=0):
        self._ck(self.L.kvidx_score_slots_dev(self.h, d_slots, d_key_off, n_prompts, d_filter or None, d_scores, d_has_keys or None))

    def apply_events_dev(self, d_ev_sorted, d_queue_off, n_queues, n_events, d_hashes, n_hashes, d_tokens, d_n_dropped=0):
        """Device-resident, pod-sorted event batch; asynchronous on the handle's write stream."""
        self._ck(self.L.kvidx_apply_events_dev(self.h, d_ev_sorted, d_queue_off, n_queues, n_events, d_hashes, n_hashes, d_tokens,
                                               d_n_dropped or None))

    # -- the device prefix store and Score() from text: prompt i is text[text_off[i] .. text_off[i+1]) (pack_text) --
    def text_store_init(self, cache_blocks=500000, block_bytes=256):
        """NewLRUTokenStore on this handle (once)."""
        self._ck(self.L.kvidx_text_store_init(self.h, cache_blocks, block_bytes))

    def text_store_add(self, text, text_off, tok, tok_span, tok_off):
        """AddTokenization of every prompt, in order.  tok / tok_off: the prompts' token CSR; tok_span (n_tok, 2): each
        token's [low, high) byte offsets in its prompt."""
        text, text_off = _u8(text), np.ascontiguousarray(text_off, np.int64)
        tok, tok_off = np.ascontiguousarray(tok, np.uint32), np.ascontiguousarray(tok_off, np.int64)
        span = np.ascontiguousarray(tok_span, np.uint64).reshape(-1)
        self._ck(self.L.kvidx_text_store_add(self.h, _p(text, _u8p), _p(text_off, _i64p), len(text_off) - 1, _p(tok, _u32p),
                                             _p(span, _u64p), _p(tok_off, _i64p)))

    def text_store_find_into(self, text, text_off, tok_out, tok_off_out, ratio_out=None) -> int:
        """One kvidx_text_store_find into caller arrays; returns the code (ENOSPC: tok_out too small, nothing refreshed)."""
        text, text_off = _u8(text), np.ascontiguousarray(text_off, np.int64)
        return self.L.kvidx_text_store_find(self.h, _p(text, _u8p), _p(text_off, _i64p), len(text_off) - 1, _p(tok_out, _u32p),
                                            0 if tok_out is None else len(tok_out), _p(tok_off_out, _i64p), _p(ratio_out, _f64p))

    def text_store_find(self, text, text_off):
        """FindLongestContainedTokens of every prompt -> (tokens, their offsets (n+1), ratios)."""
        n = len(text_off) - 1
        off, ratio = np.zeros(n + 1, np.int64), np.zeros(max(n, 0), np.float64)
        tok = np.zeros(0, np.uint32)
        while True:                           # ENOSPC refreshes nothing: size the buffer from the offsets and find again
            rc = self.text_store_find_into(text, text_off, tok if len(tok) else None, off, ratio)
            if rc != ENOSPC:
                break
            tok = np.zeros(int(off[-1]), np.uint32)
        self._ck(rc)
        return tok[:int(off[-1])], off, ratio

    def text_store_len(self) -> int:
        out = C.c_int64(0)
        self._ck(self.L.kvidx_text_store_len(self.h, C.byref(out)))
        return out.value

    def text_store_snapshot(self) -> bytes:
        """kvidx_text_store_snapshot: the store's image (format v1 in include/kvidx.h), least recent block first."""
        size = C.c_uint64(0)
        rc = self.L.kvidx_text_store_snapshot(self.h, None, 0, C.byref(size))
        while rc == ENOSPC:                   # sized by a first call; a store call in between can grow it: size again
            cap = size.value
            buf = bytearray(cap)
            rc = self.L.kvidx_text_store_snapshot(self.h, (C.c_char * cap).from_buffer(buf), cap, C.byref(size))
        self._ck(rc)
        return bytes(memoryview(buf)[:size.value])

    def text_store_restore(self, image) -> int:
        """kvidx_text_store_restore: load an image into this handle's empty store.  -> blocks resident afterwards."""
        image = image if isinstance(image, bytes) else bytes(image)
        out = C.c_int64(0)
        self._ck(self.L.kvidx_text_store_restore(self.h, image, len(image), C.byref(out)))
        return out.value

    def text_hash_keys(self, text, text_off, block_bytes):
        """The store's block keys of every prompt at block_bytes -> (keys, their offsets)."""
        text, text_off = _u8(text), np.ascontiguousarray(text_off, np.int64)
        n = len(text_off) - 1
        nk = int(((text_off[1:] - text_off[:-1]) // block_bytes).sum()) if n > 0 else 0
        keys, koff = np.zeros(max(nk, 1), np.uint64), np.zeros(n + 1, np.int64)
        self._ck(self.L.kvidx_text_hash_keys(self.h, _p(text, _u8p), _p(text_off, _i64p), n, block_bytes, _p(keys, _u64p), _p(koff, _i64p)))
        return keys[:nk], koff

    def _text_args(self, text, text_off, model, filter_mask):
        text, text_off = _u8(text), np.ascontiguousarray(text_off, np.int64)
        model = None if model is None else np.ascontiguousarray(model, np.uint32)
        filter_mask = None if filter_mask is None else np.ascontiguousarray(filter_mask, np.uint64)
        n = len(text_off) - 1
        return n, text, text_off, model, filter_mask, np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.float64)

    def score_text(self, text, text_off, model=None, model0=0, filter_mask=None, min_ratio=0.8):
        """Score() from text -> (dense rows (n, max_pods), has_keys, tokenize flags, ratios).  A prompt whose cached prefix
        covers less than min_ratio of its text gets an all-absent row and tokenize 1."""
        n, text, text_off, model, filter_mask, has, tokz, ratio = self._text_args(text, text_off, model, filter_mask)
        scores = np.empty((n, self.max_pods), np.float64)
        self._ck(self.L.kvidx_score_text(self.h, _p(text, _u8p), _p(text_off, _i64p), n, _p(model, _u32p), model0, _p(filter_mask, _u64p),
                                         float(min_ratio), _p(scores, _f64p), _p(has, _u8p), _p(tokz, _u8p), _p(ratio, _f64p)))
        return scores, has, tokz, ratio

    def score_text_sparse(self, text, text_off, model=None, model0=0, filter_mask=None, min_ratio=0.8):
        """Sparse rows as score_batch_sparse -> (pods, scores, cnt, has, tokenize flags, ratios)."""
        n, text, text_off, model, filter_mask, has, tokz, ratio = self._text_args(text, text_off, model, filter_mask)
        pods, scores, cnt = np.zeros((n, E), np.uint16), np.zeros((n, E), np.float64), np.zeros(n, np.uint8)
        self._ck(self.L.kvidx_score_text_sparse(self.h, _p(text, _u8p), _p(text_off, _i64p), n, _p(model, _u32p), model0,
                                                _p(filter_mask, _u64p), float(min_ratio), _p(pods, _u16p), _p(scores, _f64p),
                                                _p(cnt, _u8p), _p(has, _u8p), _p(tokz, _u8p), _p(ratio, _f64p)))
        return pods, scores, cnt, has, tokz, ratio

    def score_text_dev(self, d_text, d_text_off, n, d_scores, d_model=0, model0=0, d_filter=0, min_ratio=0.8, d_has_keys=0,
                       d_tokenize=0, d_ratio=0):
        """All pointers are device addresses (ints).  On the handle's stream."""
        self._ck(self.L.kvidx_score_text_dev(self.h, d_text or None, d_text_off, n, d_model or None, model0, d_filter or None,
                                             float(min_ratio), d_scores, d_has_keys or None, d_tokenize or None, d_ratio or None))

    def score_text_sparse_dev(self, d_text, d_text_off, n, d_pods, d_scores, d_cnt, d_model=0, model0=0, d_filter=0, min_ratio=0.8,
                              d_has_keys=0, d_tokenize=0, d_ratio=0):
        self._ck(self.L.kvidx_score_text_sparse_dev(self.h, d_text or None, d_text_off, n, d_model or None, model0, d_filter or None,
                                                    float(min_ratio), d_pods, d_scores, d_cnt, d_has_keys or None, d_tokenize or None,
                                                    d_ratio or None))

    # -- write path --
    def add(self, model, engine, request, podtiers):
        engine = np.ascontiguousarray(engine, np.uint64)
        request = np.ascontiguousarray(request, np.uint64)
        pt = np.ascontiguousarray(podtiers, np.uint16)
        if len(engine) != len(request):
            return EINVAL           # in_memory.go:153-155 (the C ABI takes one n for both arrays)
        return self.L.kvidx_add(self.h, model, _p(engine, _u64p), _p(request, _u64p), len(engine), _p(pt, _u16p), len(pt))

    def evict(self, model, engine, podtiers):
        pt = np.ascontiguousarray(podtiers, np.uint16)
        return self.L.kvidx_evict(self.h, model, int(engine), _p(pt, _u16p), len(pt))

    def get_request_key(self, model, engine):
        out = C.c_uint64(0)
        rc = self.L.kvidx_get_request_key(self.h, model, int(engine), C.byref(out))
        return rc, out.value

    def apply_events(self, events, hashes, tokens):
        events = np.ascontiguousarray(events, EVENT_DTYPE)
        hashes = np.ascontiguousarray(hashes, np.uint64)
        tokens = np.ascontiguousarray(tokens, np.uint32)
        nd = C.c_int64(0)
        rc = self.L.kvidx_apply_events(self.h, events.ctypes.data_as(C.c_void_p), len(events), _p(hashes, _u64p), len(hashes),
                                       _p(tokens, _u32p), len(tokens), C.byref(nd))
        return rc, nd.value

    # -- KVEvents wire payloads decoded on the device: message i is a raw msgpack EventBatch of pod pods[i], model models[i] --
    def decode_event_payloads_dev(self, d_bytes, d_msg_off, n_msgs, d_pods, d_models, tier_names, gpu_tier, d_ev, ev_cap, d_queue_off,
                                  queue_cap, d_hashes, hash_cap, d_tokens, tok_cap, flags=0, d_msg_flags=0):
        """kvidx_decode_event_payloads_dev -> (rc, counts dict).  tier_names: the table, by tier id (lower-case)."""
        tb, toff = pack_text(tier_names)
        counts = np.zeros(len(PAYLOAD_COUNTS), np.int64)
        rc = self.L.kvidx_decode_event_payloads_dev(self.h, d_bytes, d_msg_off, n_msgs, d_pods, d_models, _p(tb, _u8p), _p(toff, _i64p),
                                                    len(tier_names), gpu_tier, flags, d_ev or None, ev_cap, d_queue_off or None,
                                                    queue_cap, d_hashes or None, hash_cap, d_tokens or None, tok_cap,
                                                    d_msg_flags or None, _p(counts, _i64p))
        return rc, dict(zip(PAYLOAD_COUNTS, (int(c) for c in counts)))

    def apply_event_payloads(self, payloads, pods, models, tier_names, gpu_tier, flags=0):
        """kvidx_apply_event_payloads over a list of raw messages (bytes) -> (rc, n_dropped, counts dict, per-message flags)."""
        data, off = pack_text(payloads)
        pods = np.ascontiguousarray(pods, np.uint32)
        models = np.ascontiguousarray(models, np.uint32)
        assert len(pods) == len(models) == len(payloads)
        tb, toff = pack_text(tier_names)
        counts = np.zeros(len(PAYLOAD_COUNTS), np.int64)
        mflags = np.zeros(len(payloads), np.uint8)
        nd = C.c_int64(0)
        rc = self.L.kvidx_apply_event_payloads(self.h, _p(data, _u8p), _p(off, _i64p), len(payloads), _p(pods, _u32p), _p(models, _u32p),
                                               _p(tb, _u8p), _p(toff, _i64p), len(tier_names), gpu_tier, flags, _p(mflags, _u8p),
                                               _p(counts, _i64p), C.byref(nd))
        return rc, nd.value, dict(zip(PAYLOAD_COUNTS, (int(c) for c in counts))), mflags

    def removal_masks(self, pod_ids, tier_ids=None):
        """(pod mask words, tier mask) of a removal: tier_ids None = all tiers."""
        mask = np.zeros(self.filter_words, np.uint64)
        for p in pod_ids:
            p = int(p)
            if not 0 <= p < self.max_pods:
                raise KvidxError(ERANGE, "pod id %d outside 0..max_pods-1" % p)
            mask[p >> 6] |= np.uint64(1) << np.uint64(p & 63)
        tier_mask = 0xFFFF if tier_ids is None else sum(1 << (int(t) & 15) for t in set(tier_ids))
        return mask, tier_mask

    def remove_pods(self, pod_ids, tier_ids=None) -> dict:
        """kvidx_remove_pods: drop every entry of these pods (on these tiers; None = all).  No reference counterpart.
        -> {"entries", "request_keys", "engine_keys"} removed; raises KvidxError on failure."""
        mask, tier_mask = self.removal_masks(pod_ids, tier_ids)
        out = np.zeros(3, np.uint64)
        self._ck(self.L.kvidx_remove_pods(self.h, _p(mask, _u64p), tier_mask, _p(out, _u64p)))
        return {"entries": int(out[0]), "request_keys": int(out[1]), "engine_keys": int(out[2])}

    def shard_remove_pods(self, pod_ids, tier_ids=None, *, phase: int) -> dict:
        """kvidx_shard_remove_pods: one phase (0, then 1 once every rank has run 0) of the collective removal on a sharded
        index (kvidx.dist.remove_pods_shards runs both with the barriers).  -> this rank's counters of the phase."""
        mask, tier_mask = self.removal_masks(pod_ids, tier_ids)
        out = np.zeros(3, np.uint64)
        self._ck(self.L.kvidx_shard_remove_pods(self.h, _p(mask, _u64p), tier_mask, phase, _p(out, _u64p)))
        return {"entries": int(out[0]), "request_keys": int(out[1]), "engine_keys": int(out[2])}

    # -- snapshot / restore (no reference counterpart; format v1 in include/kvidx.h) --
    def snapshot(self) -> bytes:
        """kvidx_snapshot: the index's contents as a canonical image.  Raises KvidxError on failure."""
        st = self.stats()
        R, E = st["request_keys"], st["engine_keys"]
        size = 64 + 32 * R + 24 * E + (8 * (R + E) if self.lru_exact else 0)
        while True:
            buf = bytearray(size)
            got = C.c_uint64(0)
            rc = self.L.kvidx_snapshot(self.h, (C.c_char * size).from_buffer(buf), size, C.byref(got))
            if rc == ENOSPC and got.value > size:          # keys were added since stats(): size again
                size = got.value
                continue
            self._ck(rc)
            return bytes(memoryview(buf)[:got.value])

    def restore(self, image) -> dict:
        """kvidx_restore: load an image into this (empty) handle.  -> {"request_keys", "engine_keys"} resident afterwards."""
        image = image if isinstance(image, bytes) else bytes(image)
        out = np.zeros(2, np.uint64)
        self._ck(self.L.kvidx_restore(self.h, image, len(image), _p(out, _u64p)))
        return {"request_keys": int(out[0]), "engine_keys": int(out[1])}

    def shard_snapshot(self) -> bytes:
        """kvidx_shard_snapshot: the image of the keys and mappings this shard owns (a part for snapshot_merge)."""
        while True:
            st = self.stats()
            size = 64 + 32 * st["request_keys"] + 24 * st["engine_keys"]
            buf = bytearray(size)
            got = C.c_uint64(0)
            rc = self.L.kvidx_shard_snapshot(self.h, (C.c_char * size).from_buffer(buf), size, C.byref(got))
            if rc == ENOSPC and got.value > size:          # a peer added keys to this shard since stats(): size again
                continue
            self._ck(rc)
            return bytes(memoryview(buf)[:got.value])

    def shard_restore(self, image) -> dict:
        """kvidx_shard_restore: insert the records of any v1 image that this shard owns (the handle must hold no live key).
        -> {"request_keys", "engine_keys"} resident in this shard afterwards."""
        image = image if isinstance(image, bytes) else bytes(image)
        out = np.zeros(2, np.uint64)
        self._ck(self.L.kvidx_shard_restore(self.h, image, len(image), _p(out, _u64p)))
        return {"request_keys": int(out[0]), "engine_keys": int(out[1])}


def snapshot_merge(parts) -> bytes:
    """kvidx_snapshot_merge: the canonical image of the union of shard images (disjoint shards).  Host only."""
    L = load()
    parts = [p if isinstance(p, bytes) else bytes(p) for p in parts]
    ptrs = (C.c_char_p * max(len(parts), 1))(*parts)
    lens = np.array([len(p) for p in parts] or [0], np.uint64)
    size = C.c_uint64(0)
    rc = L.kvidx_snapshot_merge(ptrs, _p(lens, _u64p), len(parts), None, 0, C.byref(size))
    if rc != ENOSPC:
        raise KvidxError(rc, L.kvidx_last_error(None).decode())
    buf = bytearray(size.value)
    rc = L.kvidx_snapshot_merge(ptrs, _p(lens, _u64p), len(parts), (C.c_char * len(buf)).from_buffer(buf), len(buf), C.byref(size))
    if rc:
        raise KvidxError(rc, L.kvidx_last_error(None).decode())
    return bytes(buf)


class _Raw:
    """A raw host pointer (e.g. pinned memory from kvidx_host_alloc) passed through untouched."""

    def __init__(self, ptr: int):
        self.ptr = ptr


def host_alloc(nbytes: int) -> int:
    p = load().kvidx_host_alloc(nbytes)
    if not p:
        raise MemoryError("kvidx_host_alloc(%d) failed" % nbytes)
    return p


def host_free(p: int):
    load().kvidx_host_free(C.c_void_p(p))


def pinned_array(shape, dtype):
    """numpy array backed by pinned host memory (freed when the array's base is collected)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    p = host_alloc(max(n, 1))
    buf = (C.c_char * max(n, 1)).from_address(p)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
    _PINNED[arr.ctypes.data] = (p, buf)
    return arr


_PINNED = {}
