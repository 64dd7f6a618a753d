"""GPU (-m gpu): calls that move a caller's host buffers through the pinned stager -- snapshot, restore, the prefix store's
add and find, text block keys and Score() from text, dense and sparse -- return from pinned caller buffers (one direct
copy) byte for byte what they return from pageable numpy buffers (copies through two alternating pinned chunks).  One
call moves more than two 16 MB chunks each way through pageable buffers."""
import ctypes as C

import numpy as np
import pytest

import kvidx
from kvidx import pack_text
from kvidx._native import E
from test_gpu_text_store import pack_tokens, rand_text, tokenize

pytestmark = pytest.mark.gpu
P = 16
u8p, u16p, u32p, u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint16), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
i64p, f64p = C.POINTER(C.c_int64), C.POINTER(C.c_double)


def pinned(a):
    p = kvidx.pinned_array(a.shape, a.dtype)
    p[...] = a
    return p


def ptr(a, t):
    return a.ctypes.data_as(t)


def _filled(rng, n_keys=60000):
    ix = kvidx.Index(capacity=1 << 17, max_pods=P)
    for lo in range(0, n_keys, 20000):
        req = rng.integers(1, 1 << 63, 20000, dtype=np.uint64)
        assert ix.add(0, req ^ np.uint64(0x5a5a), req, [(p % P) << 4 for p in range(lo // 20000, lo // 20000 + 3)]) == 0
    return ix


def test_snapshot_and_restore():
    ix = _filled(np.random.default_rng(1))
    image = ix.snapshot()                                            # pageable buffer
    buf = kvidx.pinned_array((len(image),), np.uint8)
    got = C.c_uint64(0)
    assert ix.L.kvidx_snapshot(ix.h, buf.ctypes.data_as(C.c_void_p), len(image), C.byref(got)) == 0
    assert got.value == len(image) and buf.tobytes() == image
    a, b = kvidx.Index(capacity=1 << 17, max_pods=P), kvidx.Index(capacity=1 << 17, max_pods=P)
    out = np.zeros(2, np.uint64)
    assert a.L.kvidx_restore(a.h, C.cast(buf.ctypes.data_as(C.c_void_p), C.c_char_p), len(image), ptr(out, u64p)) == 0
    assert b.restore(image) == {"request_keys": int(out[0]), "engine_keys": int(out[1])}
    assert a.snapshot() == b.snapshot() == image


def _prompts(rng, n):
    prompts = [rand_text(rng, int(rng.integers(0, 3000))) for _ in range(n)]
    return prompts, pack_tokens([tokenize(rng, p) for p in prompts])


def test_text_store_and_score_text():
    rng = np.random.default_rng(2)
    prompts, (ids, spans, toff) = _prompts(rng, 300)
    text, text_off = pack_text(prompts)
    pa, pb = kvidx.Index(capacity=1 << 16, max_pods=P), kvidx.Index(capacity=1 << 16, max_pods=P)
    for ix in (pa, pb):
        ix.text_store_init(100000, 64)
        keys, _ = ix.hash_keys(ids, toff)                            # the index holds the prompts' token blocks
        assert ix.add(0, keys ^ np.uint64(1), keys, [(3 << 4), (5 << 4) | 1]) == 0
    pb.text_store_add(text, text_off, ids, spans, toff)
    pa.text_store_add(pinned(text), pinned(text_off), pinned(ids), pinned(spans.reshape(-1)), pinned(toff))
    assert pa.text_store_len() == pb.text_store_len()
    # find
    find, _ = _prompts(rng, 200)
    q, q_off = pack_text(prompts[:100] + find)
    tok_b, off_b, ratio_b = pb.text_store_find(q, q_off)
    n = len(q_off) - 1
    tok_a, off_a, ratio_a = (kvidx.pinned_array((max(len(tok_b), 1),), np.uint32), kvidx.pinned_array((n + 1,), np.int64),
                             kvidx.pinned_array((n,), np.float64))
    qa, qa_off = pinned(q), pinned(q_off)
    assert pa.L.kvidx_text_store_find(pa.h, ptr(qa, u8p), ptr(qa_off, i64p), n, ptr(tok_a, u32p), len(tok_a), ptr(off_a, i64p),
                                      ptr(ratio_a, f64p)) == 0
    assert off_a.tobytes() == off_b.tobytes() and ratio_a.tobytes() == ratio_b.tobytes()
    assert tok_a[:len(tok_b)].tobytes() == tok_b.tobytes()
    # Score() from text with model ids and filter rows, dense then sparse
    model = pinned(np.zeros(n, np.uint32))
    filt = pinned(np.full(n, 0xffff, np.uint64))
    sc, has, tokz, ratio = (kvidx.pinned_array((n, P), np.float64), kvidx.pinned_array((n,), np.uint8),
                            kvidx.pinned_array((n,), np.uint8), kvidx.pinned_array((n,), np.float64))
    assert pa.L.kvidx_score_text(pa.h, ptr(qa, u8p), ptr(qa_off, i64p), n, ptr(model, u32p), 0, ptr(filt, u64p), 0.5,
                                 ptr(sc, f64p), ptr(has, u8p), ptr(tokz, u8p), ptr(ratio, f64p)) == 0
    want = pb.score_text(q, q_off, model=np.zeros(n, np.uint32), filter_mask=np.full(n, 0xffff, np.uint64), min_ratio=0.5)
    assert [x.tobytes() for x in (sc, has, tokz, ratio)] == [x.tobytes() for x in want]
    assert want[0].any() and want[2].any() and not want[2].all()
    pods, ssc, cnt = (kvidx.pinned_array((n, E), np.uint16), kvidx.pinned_array((n, E), np.float64), kvidx.pinned_array((n,), np.uint8))
    assert pa.L.kvidx_score_text_sparse(pa.h, ptr(qa, u8p), ptr(qa_off, i64p), n, None, 0, None, 0.5, ptr(pods, u16p), ptr(ssc, f64p),
                                        ptr(cnt, u8p), ptr(has, u8p), ptr(tokz, u8p), ptr(ratio, f64p)) == 0
    want = pb.score_text_sparse(q, q_off, min_ratio=0.5)
    assert [x.tobytes() for x in (pods, ssc, cnt, has, tokz, ratio)] == [x.tobytes() for x in want]
    assert pa.text_store_len() == pb.text_store_len()


def test_text_hash_keys_past_two_chunks():
    """36 MB of text in and 72 MB of keys out: more than two staging chunks each way from pageable buffers"""
    rng = np.random.default_rng(3)
    ix = kvidx.Index(capacity=4096, max_pods=P)
    ix.text_store_init(1000, 64)
    text = rng.integers(0, 256, 36 << 20, dtype=np.uint8)
    text_off = np.linspace(0, len(text), 9, dtype=np.int64)
    keys, koff = ix.text_hash_keys(text, text_off, 4)
    assert len(keys) * 8 > 2 * (16 << 20) and len(text) > 2 * (16 << 20)
    pk, pko = kvidx.pinned_array((len(keys),), np.uint64), kvidx.pinned_array((len(koff),), np.int64)
    pt, pto = pinned(text), pinned(text_off)
    assert ix.L.kvidx_text_hash_keys(ix.h, ptr(pt, u8p), ptr(pto, i64p), 8, 4, ptr(pk, u64p), ptr(pko, i64p)) == 0
    assert pk.tobytes() == keys.tobytes() and pko.tobytes() == koff.tobytes()
