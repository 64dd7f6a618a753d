"""GPU (-m gpu): host-buffer Score() (kvidx_score_batch*, kvidx_score_keys*) against the device-resident call on the same
prompts (kvidx_score_batch_dev / kvidx_score_keys_dev and their sparse forms), byte for byte.  The host calls run the
zero-copy path, the chunked pipeline and the submission queue's coalesced batches; the device-resident calls run none of
them, so every host-side layout of inputs and result rows is checked against an independent reference: tokens and keys,
dense and sparse rows, has_keys given and NULL, pageable and pinned inputs and outputs, several chunks and a prompt
larger than the chunk budget, per-prompt model ids and filter rows, and prompt ranges that do not start at offset 0."""
import ctypes as C
import threading

import numpy as np
import pytest

from helpers import csr
import kvidx

pytestmark = pytest.mark.gpu
E = 10                                   # entries of a sparse row
u32, u64, i64 = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_int64)
f64, u8, u16 = C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_uint16)


def _ptr(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _index(P=64, **kw):
    """A two-model index: documents sharing prefixes, stored under model 0 and (with other pods) model 1."""
    rng = np.random.default_rng(7)
    ix = kvidx.Index(capacity=1 << 16, max_pods=P, tier_weights=(1.0, 0.8), **kw)
    bs = ix.block_size
    docs = [rng.integers(0, 50000, bs * int(rng.integers(2, 40)), dtype=np.uint32) for _ in range(48)]
    for d in range(8, len(docs)):
        share = min(int(rng.integers(1, 4)), len(docs[d]) // bs, len(docs[d % 8]) // bs)
        docs[d][:bs * share] = docs[d % 8][:bs * share]
    for d, doc in enumerate(docs):
        k = ix.hash_keys(doc, [0, len(doc)])[0]
        for m in (0, 1):
            for g in range(1 + (d + m) % 3):
                depth = len(k) - int(rng.integers(0, len(k) // 2 + 1))
                pts = [(int(p) << 4) | int(rng.integers(0, 2)) for p in rng.choice(P, size=int(rng.integers(1, 4)), replace=False)]
                assert ix.add(m, k[:depth] ^ np.uint64(0x77 + g + 8 * m), k[:depth], pts) == 0
    return ix, docs


def _prompts(rng, docs, n, bs, big=None):
    out = []
    for i in range(n):
        doc = docs[int(rng.integers(0, len(docs)))]
        kind = i % 4
        if kind == 0:
            out.append(doc)
        elif kind == 1:
            out.append(doc[:int(rng.integers(0, len(doc) + 1))])                   # ragged, sometimes < 1 block
        elif kind == 2:
            out.append(np.concatenate([doc[:bs * int(rng.integers(0, len(doc) // bs + 1))], rng.integers(0, 50000, 37, dtype=np.uint32)]))
        else:
            out.append(rng.integers(0, 50000, int(rng.integers(0, 3 * bs)), dtype=np.uint32))
    if big is not None:                  # one prompt larger than a chunk's budget: a stored prefix, then a long tail
        out[n // 2] = np.concatenate([docs[3], rng.integers(0, 50000, big, dtype=np.uint32)])
    return out


def _dev_rows(ix, keys, src, off, n, sparse, model, model0, fm):
    """The device-resident call on prompts off[0] .. off[n] of src (torch CUDA tensors in, rows back on the host)."""
    import torch
    dev = torch.device("cuda", 0)
    d_src = torch.from_numpy(src.view(np.int64 if keys else np.int32)).to(dev)
    d_off = torch.from_numpy(off).to(dev)
    d_m = torch.from_numpy(model.view(np.int32)).to(dev) if model is not None else None
    d_f = torch.from_numpy(fm.view(np.int64)).to(dev) if fm is not None else None
    d_has = torch.full((n,), 7, dtype=torch.uint8, device=dev)
    mp, fp = (d_m.data_ptr() if d_m is not None else 0), (d_f.data_ptr() if d_f is not None else 0)
    torch.cuda.synchronize(dev)
    if sparse:
        d_p = torch.zeros((n, E), dtype=torch.int16, device=dev)
        d_s = torch.zeros((n, E), dtype=torch.float64, device=dev)
        d_c = torch.zeros(n, dtype=torch.uint8, device=dev)
        fn = ix.score_keys_sparse_dev if keys else ix.score_batch_sparse_dev
        fn(d_src.data_ptr(), d_off.data_ptr(), n, d_p.data_ptr(), d_s.data_ptr(), d_c.data_ptr(), d_model=mp, model0=model0,
           d_filter=fp, d_has_keys=d_has.data_ptr())
        ix.synchronize()
        return d_p.cpu().numpy().view(np.uint16), d_s.cpu().numpy(), d_c.cpu().numpy(), d_has.cpu().numpy()
    d_s = torch.full((n, ix.max_pods), 3.0, dtype=torch.float64, device=dev)
    fn = ix.score_keys_dev if keys else ix.score_batch_dev
    fn(d_src.data_ptr(), d_off.data_ptr(), n, d_s.data_ptr(), d_model=mp, model0=model0, d_filter=fp, d_has_keys=d_has.data_ptr())
    ix.synchronize()
    return d_s.cpu().numpy(), d_has.cpu().numpy()


def _out_bufs(n, P, sparse, pinned, cache):
    """Result buffers filled with 5s; pinned ones are allocated once per shape and reused."""
    new = kvidx.pinned_array if pinned else np.empty
    key = (n, sparse, pinned)
    bufs = cache.get(key) if pinned else None
    if bufs is None:
        bufs = (new((n, E), np.uint16), new((n, E), np.float64), new(n, np.uint8), new(n, np.uint8)) if sparse else \
               (new((n, P), np.float64), new(n, np.uint8))
        cache[key] = bufs
    for b in bufs:
        b.fill(5)
    return bufs


def _host_call(ix, keys, src, off, n, sparse, model, model0, fm, bufs, want_has):
    """One raw host-buffer call (has_keys NULL unless want_has); returns the rows it wrote."""
    L, sp = ix.L, _ptr(src, u64 if keys else u32)
    args = (ix.h, sp, _ptr(off, i64), n, _ptr(model, u32), model0, _ptr(fm, u64))
    if sparse:
        p, s, c, h = bufs
        fn = L.kvidx_score_keys_sparse if keys else L.kvidx_score_batch_sparse
        rc = fn(*args, _ptr(p, u16), _ptr(s, f64), _ptr(c, u8), _ptr(h, u8) if want_has else None)
    else:
        s, h = bufs
        fn = L.kvidx_score_keys if keys else L.kvidx_score_batch
        rc = fn(*args, _ptr(s, f64), _ptr(h, u8) if want_has else None)
    assert rc == 0, ix.last_error()
    return bufs


def _same(got, want, sparse, want_has):
    if sparse:
        (pg, sg, cg, hg), (pw, sw, cw, hw) = got, want
        live = np.arange(E)[None, :] < cw[:, None]
        assert np.array_equal(cg, cw)
        assert np.array_equal(pg[live], pw[live]) and sg[live].tobytes() == sw[live].tobytes()
    else:
        (sg, hg), (sw, hw) = got, want
        assert sg.tobytes() == sw.tobytes(), np.argwhere(sg != sw)[:5]
    if want_has:
        assert np.array_equal(hg, hw)
    else:
        assert (hg == 5).all()                                   # NULL has_keys: the caller's bytes are left alone


def _check_matrix(ix, tok, off, sizes, starts, model=None, model0=0, fm=None):
    """Every host-buffer form of the call against the device-resident one, for prompts [s, s + n) of the batch."""
    keys, koff = ix.hash_keys(tok, off)
    pinned_src = {False: kvidx.pinned_array(tok.shape, np.uint32), True: kvidx.pinned_array(keys.shape, np.uint64)}
    pinned_src[False][:] = tok
    pinned_src[True][:] = keys
    cache = {}
    for n in sizes:
        for s in starts:
            m = None if model is None else np.ascontiguousarray(model[s:s + n])
            f = None if fm is None else np.ascontiguousarray(fm[s:s + n])
            for is_keys, src, o in ((False, tok, off[s:s + n + 1]), (True, keys, koff[s:s + n + 1])):
                for sparse in (False, True):
                    want = _dev_rows(ix, is_keys, src, o, n, sparse, m, model0, f)
                    for in_pinned in (False, True):
                        for out_pinned in (False, True):
                            for want_has in (True, False):
                                bufs = _out_bufs(n, ix.max_pods, sparse, out_pinned, cache)
                                got = _host_call(ix, is_keys, pinned_src[is_keys] if in_pinned else src, o, n, sparse, m, model0,
                                                 f, bufs, want_has)
                                try:
                                    _same(got, want, sparse, want_has)
                                except AssertionError as ex:
                                    raise AssertionError(f"n={n} start={s} keys={is_keys} sparse={sparse} in_pinned={in_pinned} "
                                                         f"out_pinned={out_pinned} has={want_has}") from ex


@pytest.mark.parametrize("rows", ["plain", "model_filter"])
@pytest.mark.parametrize("chunk", [None, 65536])
def test_host_calls_equal_device_calls(chunk, rows, monkeypatch):
    if chunk:
        monkeypatch.setenv("KVIDX_HOST_CHUNK_TOKENS", str(chunk))
    ix, docs = _index()
    rng = np.random.default_rng(11)
    N = 3000
    tok, off = csr(_prompts(rng, docs, N, ix.block_size, big=600000 if chunk else None))
    if chunk:                            # a chunk holds `chunk` tokens or as many bytes of keys: one prompt is over both
        assert off[-1] > 3 * chunk and (np.diff(off) // ix.block_size > chunk // 2).any()
    model, fm, model0 = None, None, 1
    if rows == "model_filter":
        model = (np.arange(N) % 3 == 0).astype(np.uint32)
        fm = np.zeros((N, 1), np.uint64)
        fm[::2, 0] = rng.integers(0, 1 << 63, len(fm[::2]), dtype=np.uint64)
        model0 = 0
    s, _ = ix.score_batch(tok, off, model=model, model0=model0, filter_mask=fm)
    assert (s.max(axis=1) > 1).any() and (s.max(axis=1) < 0).any()
    _check_matrix(ix, tok, off, (1, 32, 33, N - 7), (0, 7), model, model0, fm)


def test_exact_lru_block_size_4():
    """Exact-LRU handles and block sizes other than 16 take the thread-per-prompt kernel, and never zero-copy."""
    ix, docs = _index(block_size=4, lru_exact=1)
    rng = np.random.default_rng(12)
    tok, off = csr(_prompts(rng, docs, 400, ix.block_size))
    _check_matrix(ix, tok, off, (1, 33, 393), (0, 7))


def test_coalesced_callers_equal_device_calls():
    """Concurrent dense and sparse callers, with and without model ids and filter rows, served as coalesced batches."""
    ix, docs = _index(P=32)
    rng = np.random.default_rng(13)
    C_, IT = 48, 12
    calls = []
    for c in range(C_):
        for it in range(IT):
            n = 1 + (c + it) % 3
            tok, off = csr(_prompts(rng, docs, n, ix.block_size))
            model = (np.arange(n) % 2).astype(np.uint32) if c % 3 == 1 else None
            fm = rng.integers(0, 1 << 32, (n, 1), dtype=np.uint64) if c % 4 == 2 else None
            sparse = c % 2 == 1
            want = _dev_rows(ix, False, tok, off, n, sparse, model, 1 if c % 5 == 0 else 0, fm)
            calls.append((tok, off, n, sparse, model, 1 if c % 5 == 0 else 0, fm, want, it % 2 == 0))
    errs = []
    go = threading.Barrier(C_)

    def caller(c):
        try:
            go.wait()
            for it in range(IT):
                tok, off, n, sparse, model, model0, fm, want, want_has = calls[c * IT + it]
                bufs = _out_bufs(n, ix.max_pods, sparse, False, {})
                _same(_host_call(ix, False, tok, off, n, sparse, model, model0, fm, bufs, want_has), want, sparse, want_has)
        except Exception as ex:                                       # noqa: BLE001
            errs.append(ex)

    ths = [threading.Thread(target=caller, args=(c,)) for c in range(C_)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errs, errs[:2]
    assert ix.stats()["coalesced_calls"] > 0
