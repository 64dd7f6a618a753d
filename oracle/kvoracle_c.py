"""ctypes loader for oracle/libkvoracle.so (the fast C++ CPU oracle).

TEST INFRASTRUCTURE ONLY -- see kvoracle.cpp.  Used by tests/, smoke() and the
cpu_baseline / --impl reference legs of bench.py.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libkvoracle.so")
E = 10  # KVIDX_MAX_PODS_PER_KEY


class Event(C.Structure):
    """kvidx_event_t (include/kvidx.h)."""
    _fields_ = [("op", C.c_uint8), ("has_parent", C.c_uint8), ("podtier", C.c_uint16), ("model", C.c_uint32),
                ("parent_hash", C.c_uint64), ("hash_off", C.c_uint64), ("tok_off", C.c_uint64),
                ("n_hashes", C.c_uint32), ("n_tokens", C.c_uint32)]


EVENT_DTYPE = np.dtype([("op", "u1"), ("has_parent", "u1"), ("podtier", "<u2"), ("model", "<u4"),
                        ("parent_hash", "<u8"), ("hash_off", "<u8"), ("tok_off", "<u8"),
                        ("n_hashes", "<u4"), ("n_tokens", "<u4")])
assert EVENT_DTYPE.itemsize == C.sizeof(Event) == 40


def build(force: bool = False) -> str:
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(os.path.join(_HERE, "kvoracle.cpp")):
        subprocess.check_call(["make", "-C", _HERE, "-B" if force else "-s", "libkvoracle.so"])
    return _LIB


def _ptr(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        L.ko_create.restype = C.c_void_p
        L.ko_create.argtypes = [C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32]
        L.ko_destroy.argtypes = [C.c_void_p]
        L.ko_set_tier_weight.argtypes = [C.c_void_p, C.c_uint32, C.c_double]
        L.ko_fnv64a.restype = C.c_uint64
        L.ko_fnv64a.argtypes = [C.c_char_p, C.c_size_t]
        L.ko_block_hash.restype = C.c_uint64
        L.ko_block_hash.argtypes = [C.c_uint64, C.POINTER(C.c_uint32), C.c_uint32]
        L.ko_hash_keys.restype = C.c_int64
        L.ko_hash_keys.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_int64), C.c_int64,
                                   C.POINTER(C.c_uint64), C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]
        L.ko_add.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_int64, C.c_int64,
                             C.POINTER(C.c_uint16), C.c_int]
        L.ko_evict.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint16), C.c_int]
        L.ko_get_request_key.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint64)]
        L.ko_len_request.restype = C.c_uint64
        L.ko_len_request.argtypes = [C.c_void_p]
        L.ko_len_engine.restype = C.c_uint64
        L.ko_len_engine.argtypes = [C.c_void_p]
        L.ko_lookup.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.c_int64, C.POINTER(C.c_uint64), C.c_uint32,
                                C.POINTER(C.c_uint16), C.POINTER(C.c_uint8)]
        L.ko_score_batch.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_int64), C.c_int64, C.POINTER(C.c_uint32),
                                     C.c_uint32, C.POINTER(C.c_uint64), C.c_uint32, C.c_uint32, C.c_int,
                                     C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_double), C.POINTER(C.c_int64)]
        L.ko_apply_events.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32),
                                      C.POINTER(C.c_int64)]
        L.ko_peek_request_key.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint64)]
        L.ko_snapshot.restype = C.c_int64
        L.ko_snapshot.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64]
        _lib = L
    return _lib


class COracle:
    """Thin object wrapper with the same call shapes as the kvidx ctypes binding."""

    def __init__(self, block_size=16, init_hash=0xCBF29CE484222325, size=10 ** 8, pod_cache_size=10,
                 tier_weights=(1.0, 0.8), max_pods=256):
        self.L = lib()
        self.h = self.L.ko_create(block_size, init_hash, size, pod_cache_size)
        if not self.h:
            raise ValueError("must provide a positive size")
        self.block_size, self.max_pods = block_size, max_pods
        self.filter_words = (max_pods + 63) // 64
        for i, w in enumerate(tier_weights):
            self.L.ko_set_tier_weight(self.h, i, float(w))

    def close(self):
        if self.h:
            self.L.ko_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def hash_keys(self, tok, tok_off, parent=None, parent_valid=None):
        tok = np.ascontiguousarray(tok, np.uint32)
        tok_off = np.ascontiguousarray(tok_off, np.int64)
        n = len(tok_off) - 1
        nk = int(((tok_off[1:] - tok_off[:-1]) // self.block_size).sum())
        keys = np.zeros(max(nk, 1), np.uint64)
        koff = np.zeros(n + 1, np.int64)
        if parent is not None:
            parent = np.ascontiguousarray(parent, np.uint64)
        if parent_valid is not None:
            parent_valid = np.ascontiguousarray(parent_valid, np.uint8)
        w = self.L.ko_hash_keys(self.h, _ptr(tok, C.c_uint32), _ptr(tok_off, C.c_int64), n, _ptr(parent, C.c_uint64),
                                _ptr(parent_valid, C.c_uint8), _ptr(keys, C.c_uint64), _ptr(koff, C.c_int64))
        assert w == nk
        return keys[:nk], koff

    def add(self, model, engine, request, podtier):
        engine = np.ascontiguousarray(engine, np.uint64)
        request = np.ascontiguousarray(request, np.uint64)
        pt = np.ascontiguousarray(podtier, np.uint16)
        return self.L.ko_add(self.h, model, _ptr(engine, C.c_uint64), _ptr(request, C.c_uint64), len(engine), len(request),
                             _ptr(pt, C.c_uint16), len(pt))

    def evict(self, model, engine, podtier):
        pt = np.ascontiguousarray(podtier, np.uint16)
        return self.L.ko_evict(self.h, model, int(engine), _ptr(pt, C.c_uint16), len(pt))

    def get_request_key(self, model, engine):
        out = C.c_uint64(0)
        rc = self.L.ko_get_request_key(self.h, model, int(engine), C.byref(out))
        return rc, out.value

    def peek_request_key(self, model, engine):
        """get_request_key without refreshing the mapping's recency: -> request key, or None on a miss."""
        out = C.c_uint64(0)
        rc = self.L.ko_peek_request_key(self.h, model, int(engine), C.byref(out))
        return out.value if rc == 0 else None

    def lookup(self, model, keys, filter_mask=None):
        keys = np.ascontiguousarray(keys, np.uint64)
        n = len(keys)
        pt = np.zeros((max(n, 1), E), np.uint16)
        cnt = np.zeros(max(n, 1), np.uint8)
        if filter_mask is not None:
            filter_mask = np.ascontiguousarray(filter_mask, np.uint64)
        rc = self.L.ko_lookup(self.h, model, _ptr(keys, C.c_uint64), n, _ptr(filter_mask, C.c_uint64), self.filter_words,
                              _ptr(pt, C.c_uint16), _ptr(cnt, C.c_uint8))
        return rc, pt[:n], cnt[:n]

    def score_batch(self, tok, tok_off, model=None, model0=0, filter_mask=None, n_threads=1, want_scores=True,
                    want_latency=False):
        tok = np.ascontiguousarray(tok, np.uint32)
        tok_off = np.ascontiguousarray(tok_off, np.int64)
        n = len(tok_off) - 1
        scores = np.empty((n, self.max_pods), np.float64) if want_scores else None
        has = np.zeros(n, np.uint8)
        lat = np.zeros(n, np.int64) if want_latency else None
        el = C.c_double(0)
        if model is not None:
            model = np.ascontiguousarray(model, np.uint32)
        if filter_mask is not None:
            filter_mask = np.ascontiguousarray(filter_mask, np.uint64)
        rc = self.L.ko_score_batch(self.h, _ptr(tok, C.c_uint32), _ptr(tok_off, C.c_int64), n, _ptr(model, C.c_uint32), model0,
                                   _ptr(filter_mask, C.c_uint64), self.filter_words, self.max_pods, n_threads,
                                   _ptr(scores, C.c_double), _ptr(has, C.c_uint8), C.byref(el), _ptr(lat, C.c_int64))
        if rc:
            raise RuntimeError("ko_score_batch rc=%d" % rc)
        return scores, has, el.value, lat

    def apply_events(self, events, hashes, tokens):
        events = np.ascontiguousarray(events, EVENT_DTYPE)
        hashes = np.ascontiguousarray(hashes, np.uint64)
        tokens = np.ascontiguousarray(tokens, np.uint32)
        nd = C.c_int64(0)
        rc = self.L.ko_apply_events(self.h, events.ctypes.data_as(C.c_void_p), len(events), _ptr(hashes, C.c_uint64),
                                    _ptr(tokens, C.c_uint32), C.byref(nd))
        return rc, nd.value

    def snapshot(self, recency=False) -> bytes:
        """The v1 index image (include/kvidx.h) of the oracle's contents, as kvidx_snapshot writes it.  With recency, each
        record's value is its 1-based position in its LRU (oldest = 1): compare a library image's by rank."""
        size = self.L.ko_snapshot(self.h, int(recency), None, 0)
        buf = (C.c_uint8 * size)()
        assert self.L.ko_snapshot(self.h, int(recency), buf, size) == size
        return bytes(buf)

    def len_request(self):
        return self.L.ko_len_request(self.h)

    def len_engine(self):
        return self.L.ko_len_engine(self.h)
