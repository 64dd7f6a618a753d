"""ctypes binding of the host mirror (include/kvidx_host.h): string-level Indexer / Index / Pool over libkvidx."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native
from ._native import Config, EVENT_DTYPE

MAX_TIERS = 16
NO_KEYS = -1000


class HostConfig(C.Structure):
    _fields_ = [("index", Config), ("concurrency", C.c_uint32), ("n_tiers", C.c_uint32), ("tier_names", C.c_char_p * MAX_TIERS),
                ("tier_weights", C.c_double * MAX_TIERS), ("no_device", C.c_int32), ("enable_metrics", C.c_int32),
                ("clear_on_all_blocks_cleared", C.c_int32)]


LATENCY_BUCKETS = 11
EV_ALL_BLOCKS_CLEARED = 2          # KVHOST_EV_ALL_BLOCKS_CLEARED: decoder marker record (clear_on_all_blocks_cleared)


class HostMetrics(C.Structure):
    _fields_ = [("admissions_total", C.c_uint64), ("evictions_total", C.c_uint64), ("lookup_requests_total", C.c_uint64),
                ("max_pod_hit_count_total", C.c_uint64), ("lookup_hits_total", C.c_uint64), ("lookup_latency_bucket", C.c_uint64 * LATENCY_BUCKETS),
                ("lookup_latency_count", C.c_uint64), ("lookup_latency_sum", C.c_double)]


class PodRow(C.Structure):
    """kvhost_pod_row_t."""
    _fields_ = [("pod", C.c_char_p), ("pod_id", C.c_uint32), ("reserved", C.c_uint32), ("keys", C.c_uint64), ("sole_keys", C.c_uint64),
                ("sole_engine_keys", C.c_uint64), ("entries", C.c_uint64 * MAX_TIERS)]


_cpp = C.POINTER(C.c_char_p)
_i64p = C.POINTER(C.c_int64)
_u64p, _u32p, _u8p, _f64p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8), C.POINTER(C.c_double)
SYMBOLS = {
    "kvhost_config_default": (None, [C.POINTER(HostConfig)]),
    "kvhost_create": (C.c_int, [C.POINTER(HostConfig), C.c_char_p, C.POINTER(C.c_void_p)]),
    "kvhost_destroy": (None, [C.c_void_p]),
    "kvhost_prefix_store_create": (C.c_int, [C.c_int64, C.c_int32, C.POINTER(C.c_void_p)]),
    "kvhost_prefix_store_destroy": (None, [C.c_void_p]),
    "kvhost_prefix_store_add": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t]),
    "kvhost_prefix_store_find": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_double)]),
    "kvhost_prefix_store_len": (C.c_int64, [C.c_void_p]),
    "kvhost_prefix_store_snapshot": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "kvhost_prefix_store_restore": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64]),
    "kvhost_xxhash64": (C.c_uint64, [C.c_char_p, C.c_size_t, C.c_uint64]),
    "kvhost_get_metrics": (C.c_int, [C.c_void_p, C.POINTER(HostMetrics)]),
    "kvhost_metrics_text": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "kvhost_last_error": (C.c_char_p, []),
    "kvhost_index": (C.c_void_p, [C.c_void_p]),
    "kvhost_get_pod_scores": (C.c_int, [C.c_void_p, _u32p, C.c_size_t, C.c_char_p, _cpp, C.c_size_t, _cpp, _f64p]),
    "kvhost_get_pod_scores_keys": (C.c_int, [C.c_void_p, _u64p, C.c_size_t, C.c_char_p, _cpp, C.c_size_t, _cpp, _f64p]),
    "kvhost_get_pod_scores_turn": (C.c_int, [C.c_void_p, _u64p, C.c_size_t, _u32p, C.c_size_t, C.c_char_p, _cpp, C.c_size_t, _cpp, _f64p, _u64p]),
    "kvhost_index_add":(C.c_int, [C.c_void_p, C.c_char_p, _u64p, C.c_size_t, _u64p, C.c_size_t, _cpp, _cpp, C.c_size_t]),
    "kvhost_index_evict": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64, _cpp, _cpp, C.c_size_t]),
    "kvhost_index_get_request_key": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64, _u64p]),
    "kvhost_index_lookup": (C.c_int, [C.c_void_p, C.c_char_p, _u64p, C.c_size_t, _cpp, C.c_size_t, _cpp, _cpp, _u8p]),
    "kvhost_pool_add_task": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]),
    "kvhost_pool_queue_index": (C.c_int, [C.c_void_p, C.c_char_p]),
    "kvhost_pool_process": (C.c_int64, [C.c_void_p, C.POINTER(C.c_int64)]),
    "kvhost_remove_pod": (C.c_int, [C.c_void_p, C.c_char_p, _cpp, C.c_size_t]),
    "kvhost_snapshot": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "kvhost_restore": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64]),
    "kvhost_pod_inventory": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_int32, C.POINTER(PodRow), C.c_size_t, _cpp, _u64p]),
    "kvhost_inventory_text": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "kvhost_decode_event_batch": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, _u64p, C.c_size_t,
                                              C.POINTER(C.c_size_t), _u32p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "kvhost_pod_id": (C.c_int, [C.c_void_p, C.c_char_p]),
    "kvhost_tier_id": (C.c_int, [C.c_void_p, C.c_char_p]),
    "kvhost_model_id": (C.c_int, [C.c_void_p, C.c_char_p]),
    "kvhost_get_pod_scores_text": (C.c_int, [C.c_void_p, _u8p, _i64p, C.c_size_t, C.c_char_p, _cpp, C.c_size_t, C.c_double, _cpp,
                                             C.POINTER(C.c_double), C.POINTER(C.c_int32), _u8p]),
    "kvhost_get_pod_scores_batch": (C.c_int, [C.c_void_p, _u32p, _i64p, C.c_size_t, C.c_char_p, _cpp, C.c_size_t, _cpp,
                                              C.POINTER(C.c_double), C.POINTER(C.c_int32)]),
}
_bound = False


def _lib():
    global _bound
    L = _native.load()
    if not _bound:
        for name, (res, args) in SYMBOLS.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _bound = True
    return L


def _strs(items):
    arr = (C.c_char_p * max(len(items), 1))()
    for i, s in enumerate(items):
        arr[i] = s.encode() if isinstance(s, str) else s
    return arr


class HostIndexer:
    """kvcache.Indexer + kvblock.Index + kvevents.Pool with strings (pods, tiers, models are names)."""

    def __init__(self, block_size=16, hash_seed="", capacity=1 << 20, pods_per_key=10, tiers=(("gpu", 1.0), ("cpu", 0.8)), max_pods=256,
                 concurrency=4, device=0, no_device=False, lru_exact=0, enable_metrics=False, clear_on_all_blocks_cleared=False,
                 evict_policy="none", grow_tables=False, table_slots=0):
        self.L = _lib()
        self.block_size, self.max_pods = block_size, max_pods
        cfg = HostConfig()
        self.L.kvhost_config_default(C.byref(cfg))
        cfg.index.block_size, cfg.index.capacity, cfg.index.pods_per_key = block_size, capacity, pods_per_key
        cfg.index.max_pods, cfg.index.device, cfg.index.lru_exact = max_pods, device, lru_exact
        cfg.index.evict_policy = _native._EVICT_POLICIES[evict_policy] if isinstance(evict_policy, str) else int(evict_policy)
        cfg.index.grow_tables, cfg.index.table_slots = int(grow_tables), table_slots
        cfg.concurrency, cfg.n_tiers, cfg.no_device = concurrency, len(tiers), 1 if no_device else 0
        cfg.enable_metrics = 1 if enable_metrics else 0
        cfg.clear_on_all_blocks_cleared = 1 if clear_on_all_blocks_cleared else 0
        self._tier_names = [t[0].encode() for t in tiers]
        for i, (n, w) in enumerate(tiers):
            cfg.tier_names[i] = self._tier_names[i]
            cfg.tier_weights[i] = float(w)
        h = C.c_void_p()
        rc = self.L.kvhost_create(C.byref(cfg), hash_seed.encode(), C.byref(h))
        if rc:
            raise _native.KvidxError(rc, self.L.kvhost_last_error().decode())
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.kvhost_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def err(self):
        return self.L.kvhost_last_error().decode()

    def get_pod_scores(self, tokens, model, pods=()):
        """-> dict pod -> score, or None for the reference's (nil, nil)."""
        tok = np.ascontiguousarray(tokens, np.uint32)
        po = (C.c_char_p * 10)(); so = (C.c_double * 10)()
        n = self.L.kvhost_get_pod_scores(self.h, tok.ctypes.data_as(_u32p), len(tok), model.encode(), _strs(list(pods)), len(pods), po, so)
        if n == NO_KEYS:
            return None
        if n < 0:
            raise _native.KvidxError(n, self.err())
        return {po[i].decode(): so[i] for i in range(n)}

    def _batch_rows(self, n, rc, po, so, cnt):
        if rc:
            raise _native.KvidxError(rc, self.err())
        return [None if cnt[i] < 0 else {po[i * 10 + j].decode(): so[i * 10 + j] for j in range(cnt[i])} for i in range(n)]

    def get_pod_scores_text(self, text, text_off, model, pods=(), min_ratio=0.8):
        """GetPodScores for a batch of prompt texts through the device prefix store (kvhost_get_pod_scores_text).
        -> (per prompt a dict pod -> score, or None; tokenize flags: the prompts whose cached prefix was too short)."""
        text = np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text, np.uint8)
        off = np.ascontiguousarray(text_off, np.int64)
        n = len(off) - 1
        po = (C.c_char_p * (10 * max(n, 1)))(); so = (C.c_double * (10 * max(n, 1)))(); cnt = (C.c_int32 * max(n, 1))()
        tz = np.zeros(max(n, 1), np.uint8)
        rc = self.L.kvhost_get_pod_scores_text(self.h, text.ctypes.data_as(_u8p), off.ctypes.data_as(_i64p), n, model.encode(),
                                               _strs(list(pods)), len(pods), float(min_ratio), po, so, cnt, tz.ctypes.data_as(_u8p))
        return self._batch_rows(n, rc, po, so, cnt), tz[:n]

    def get_pod_scores_batch(self, tokens, tok_off, model, pods=()):
        """GetPodScores for a batch of token prompts (CSR) -> per prompt a dict pod -> score, or None."""
        tok = np.ascontiguousarray(tokens, np.uint32)
        off = np.ascontiguousarray(tok_off, np.int64)
        n = len(off) - 1
        po = (C.c_char_p * (10 * max(n, 1)))(); so = (C.c_double * (10 * max(n, 1)))(); cnt = (C.c_int32 * max(n, 1))()
        rc = self.L.kvhost_get_pod_scores_batch(self.h, tok.ctypes.data_as(_u32p), off.ctypes.data_as(_i64p), n, model.encode(),
                                                _strs(list(pods)), len(pods), po, so, cnt)
        return self._batch_rows(n, rc, po, so, cnt)

    def get_pod_scores_keys(self, keys, model, pods=()):
        """GetPodScores from the prompt's request keys (block order) -> dict pod -> score, or None when there are no keys."""
        k = np.ascontiguousarray(keys, np.uint64)
        po = (C.c_char_p * 10)(); so = (C.c_double * 10)()
        n = self.L.kvhost_get_pod_scores_keys(self.h, k.ctypes.data_as(_u64p), len(k), model.encode(), _strs(list(pods)), len(pods), po, so)
        if n == NO_KEYS:
            return None
        if n < 0:
            raise _native.KvidxError(n, self.err())
        return {po[i].decode(): so[i] for i in range(n)}

    def get_pod_scores_turn(self, keys, tokens, model, pods=()):
        """GetPodScores for a conversation turn: the request keys held from earlier turns, then the new turn's tokens.
        -> (dict pod -> score, or None when there are no keys at all; the new turn's keys, to hold for the next turn)."""
        k = np.ascontiguousarray(keys, np.uint64)
        tok = np.ascontiguousarray(tokens, np.uint32)
        nk = np.zeros(max(len(tok) // self.block_size, 1), np.uint64)
        po = (C.c_char_p * 10)(); so = (C.c_double * 10)()
        n = self.L.kvhost_get_pod_scores_turn(self.h, k.ctypes.data_as(_u64p), len(k), tok.ctypes.data_as(_u32p), len(tok), model.encode(),
                                              _strs(list(pods)), len(pods), po, so, nk.ctypes.data_as(_u64p))
        new_keys = nk[:len(tok) // self.block_size]
        if n == NO_KEYS:
            return None, new_keys
        if n < 0:
            raise _native.KvidxError(n, self.err())
        return {po[i].decode(): so[i] for i in range(n)}, new_keys

    def add(self, model, engine, request, entries):
        e = np.ascontiguousarray(engine, np.uint64); r = np.ascontiguousarray(request, np.uint64)
        return self.L.kvhost_index_add(self.h, model.encode(), e.ctypes.data_as(_u64p), len(e), r.ctypes.data_as(_u64p), len(r),
                                       _strs([p for p, _ in entries]), _strs([t for _, t in entries]), len(entries))

    def evict(self, model, engine, entries):
        return self.L.kvhost_index_evict(self.h, model.encode(), int(engine), _strs([p for p, _ in entries]), _strs([t for _, t in entries]), len(entries))

    def get_request_key(self, model, engine):
        out = C.c_uint64(0)
        rc = self.L.kvhost_index_get_request_key(self.h, model.encode(), int(engine), C.byref(out))
        return rc, out.value

    def lookup(self, model, keys, pods=()):
        k = np.ascontiguousarray(keys, np.uint64)
        n = len(k)
        po = (C.c_char_p * (10 * max(n, 1)))(); to = (C.c_char_p * (10 * max(n, 1)))(); cnt = np.zeros(max(n, 1), np.uint8)
        rc = self.L.kvhost_index_lookup(self.h, model.encode(), k.ctypes.data_as(_u64p), n, _strs(list(pods)), len(pods), po, to, cnt.ctypes.data_as(_u8p))
        if rc:
            return rc, {}
        return 0, {int(k[i]): [(po[i * 10 + j].decode(), to[i * 10 + j].decode()) for j in range(cnt[i])] for i in range(n) if cnt[i]}

    def metrics(self):
        """kvcache_index_* counters as a dict (all zero unless enable_metrics)."""
        m = HostMetrics()
        rc = self.L.kvhost_get_metrics(self.h, C.byref(m))
        if rc:
            raise _native.KvidxError(rc, self.err())
        d = {k: getattr(m, k) for k, _ in HostMetrics._fields_ if k != "lookup_latency_bucket"}
        d["lookup_latency_bucket"] = list(m.lookup_latency_bucket)
        return d

    def metrics_text(self):
        n = self.L.kvhost_metrics_text(self.h, None, 0)
        buf = C.create_string_buffer(int(n) + 1)
        self.L.kvhost_metrics_text(self.h, buf, len(buf))
        return buf.value.decode()

    def add_task(self, pod, model, payload: bytes):
        return self.L.kvhost_pool_add_task(self.h, pod.encode(), model.encode(), payload, len(payload))

    def queue_index(self, pod):
        return self.L.kvhost_pool_queue_index(self.h, pod.encode())

    def process(self):
        nd = C.c_int64(0)
        n = self.L.kvhost_pool_process(self.h, C.byref(nd))
        return n, nd.value

    def remove_pod(self, name, tiers=()):
        """kvhost_remove_pod: drop the pod's queued messages and its entries on `tiers` (empty: all tiers, which also frees
        its id for reuse).  No reference counterpart.  -> number of queued messages dropped."""
        n = self.L.kvhost_remove_pod(self.h, name.encode(), _strs(list(tiers)), len(tiers))
        if n < 0:
            raise _native.KvidxError(n, self.err())
        return n

    def snapshot(self) -> bytes:
        """kvhost_snapshot: names (models, tiers, pods with freed ids) + the index image.  Queued messages are not included."""
        size = C.c_uint64(0)
        rc = self.L.kvhost_snapshot(self.h, None, 0, C.byref(size))
        while True:
            if rc != _native.ENOSPC:
                raise _native.KvidxError(rc, self.err())
            cap = size.value
            buf = bytearray(cap)
            rc = self.L.kvhost_snapshot(self.h, (C.c_char * cap).from_buffer(buf), cap, C.byref(size))
            if rc == 0:
                return bytes(memoryview(buf)[:size.value])

    def restore(self, image):
        """kvhost_restore: load a kvhost_snapshot image into this fresh indexer."""
        image = image if isinstance(image, bytes) else bytes(image)
        rc = self.L.kvhost_restore(self.h, image, len(image))
        if rc:
            raise _native.KvidxError(rc, self.err())

    def pod_inventory(self, model=None, engine=False, totals=False):
        """kvhost_pod_inventory: {pod name: {"id", "keys", "sole_keys", "sole_engine_keys" (None without `engine`), "entries":
        {tier name: count, non-zero tiers only}}} for every interned pod; model None = all models.  With `totals`, a pair of
        that and [request keys, entries, engine mappings, stale engine mappings] (the last two only with `engine`)."""
        cap = 256
        while True:
            rows, tiers, tot = (PodRow * cap)(), (C.c_char_p * MAX_TIERS)(), (C.c_uint64 * 4)()
            n = self.L.kvhost_pod_inventory(self.h, None if model is None else model.encode(), 1 if engine else 0, rows, cap, tiers, tot)
            if n < 0:
                raise _native.KvidxError(int(n), self.err())
            if n <= cap:
                break
            cap = int(n)
        pods = {r.pod.decode(): {"id": r.pod_id, "keys": r.keys, "sole_keys": r.sole_keys, "sole_engine_keys": r.sole_engine_keys if engine else None,
                                 "entries": {(tiers[t].decode() if tiers[t] is not None else str(t)): r.entries[t]
                                             for t in range(MAX_TIERS) if r.entries[t]}} for r in rows[:n]}
        return (pods, [int(v) for v in tot]) if totals else pods

    def inventory_text(self) -> str:
        """kvhost_inventory_text: the all-model inventory as Prometheus gauges (kvcache_index_pod_* and stale_engine_keys)."""
        n = self.L.kvhost_inventory_text(self.h, None, 0)
        if n < 0:
            raise _native.KvidxError(int(n), self.err())
        buf = C.create_string_buffer(int(n) + 4096)          # pods may join between the two calls
        self.L.kvhost_inventory_text(self.h, buf, len(buf))
        return buf.value.decode()

    def decode(self, pod, model, payload: bytes, cap=4096):
        ev = np.zeros(cap, EVENT_DTYPE); hs = np.zeros(cap * 64, np.uint64); tk = np.zeros(cap * 1024, np.uint32)
        nh, nt = C.c_size_t(0), C.c_size_t(0)
        n = self.L.kvhost_decode_event_batch(self.h, pod.encode(), model.encode(), payload, len(payload), ev.ctypes.data_as(C.c_void_p), cap,
                                             hs.ctypes.data_as(_u64p), len(hs), C.byref(nh), tk.ctypes.data_as(_u32p), len(tk), C.byref(nt))
        if n < 0:
            raise _native.KvidxError(int(n), self.err())
        return ev[:n], hs[:nh.value], tk[:nt.value]

    def pod_id(self, s):
        return self.L.kvhost_pod_id(self.h, s.encode())

    def tier_id(self, s):
        return self.L.kvhost_tier_id(self.h, s.encode("utf-8", "surrogateescape"))


def xxhash64(data: bytes, seed: int = 0) -> int:
    return int(_lib().kvhost_xxhash64(data, len(data), seed))


class PrefixStore:
    """prefixstore.LRUTokenStore (the cache in front of the tokenizer): text blocks -> the tokens that end inside them."""

    def __init__(self, cache_size=500000, block_size=256):
        self.L = _lib()
        self.cache_size, self.block_size = cache_size, block_size
        h = C.c_void_p()
        rc = self.L.kvhost_prefix_store_create(cache_size, block_size, C.byref(h))
        if rc:
            raise _native.KvidxError(rc, self.L.kvhost_last_error().decode())
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.kvhost_prefix_store_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return int(self.L.kvhost_prefix_store_len(self.h))

    def add_tokenization(self, prompt: bytes, tokens, offsets):
        tok = np.ascontiguousarray(tokens, np.uint32)
        off = np.ascontiguousarray(offsets, np.uint64).reshape(-1, 2) if len(tok) else np.zeros((0, 2), np.uint64)
        assert len(off) == len(tok)
        rc = self.L.kvhost_prefix_store_add(self.h, prompt, len(prompt), tok.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), len(tok))
        if rc:
            raise _native.KvidxError(rc, self.L.kvhost_last_error().decode())

    def find_longest_contained_tokens(self, prompt: bytes):
        ratio = C.c_double(0.0)
        n = self.L.kvhost_prefix_store_find(self.h, prompt, len(prompt), None, 0, C.byref(ratio))      # count only (and refresh)
        out = np.zeros(max(int(n), 1), np.uint32)
        n = self.L.kvhost_prefix_store_find(self.h, prompt, len(prompt), out.ctypes.data_as(C.c_void_p), len(out), C.byref(ratio))
        return out[: int(n)].tolist(), ratio.value

    def snapshot(self) -> bytes:
        """kvhost_prefix_store_snapshot: the store's image (format v1 of kvidx_text_store_snapshot), least recent first."""
        size = C.c_uint64(0)
        rc = self.L.kvhost_prefix_store_snapshot(self.h, None, 0, C.byref(size))
        while rc == _native.ENOSPC:
            cap = size.value
            buf = bytearray(cap)
            rc = self.L.kvhost_prefix_store_snapshot(self.h, (C.c_char * cap).from_buffer(buf), cap, C.byref(size))
        if rc:
            raise _native.KvidxError(rc, self.L.kvhost_last_error().decode())
        return bytes(memoryview(buf)[:size.value])

    def restore(self, image):
        """kvhost_prefix_store_restore: load an image into this empty store (it keeps its own cache_size)."""
        image = image if isinstance(image, bytes) else bytes(image)
        rc = self.L.kvhost_prefix_store_restore(self.h, image, len(image))
        if rc:
            raise _native.KvidxError(rc, self.L.kvhost_last_error().decode())
