"""GPU: Score() at the batch sizes it runs at, through the library's default dispatch, every row against the workload's
closed form (tests/scale_workload.py).

The rest of the suite reaches the round pipelines by lowering the dispatch thresholds on batches of at most 20 000
prompts.  Here nothing is lowered: an index filled with the metric workload (config 6, 4096-token prompts, 10 M blocks,
256 pods, a second workload under model 1) scores

  - batch A: 2^20 + 2^16 resident 4096-token prompts of the metric workload's query stream (17 GiB of tokens).  The first
    2^20 are the benchmark's step and the rest its host-buffer batch; prompts from 2^20 on start at token 2^32 or later.
    Windows of it take every default path, several of them across the 2^32 mark;
  - batch B: 1.5 M ragged prompts, mostly short, with zero-length and sub-block prompts, 32 K+ token tails, the second
    model, prompts scored under the other model and per-prompt filter rows; and a low-sharing variant that the class
    pipeline hands over to the per-prompt rounds with the lane walk.

Each call's path is asserted from its kernel-launch count, so that a moved threshold fails here instead of quietly testing
another path.  The launch counts are those of launch_score* in csrc/kvidx.cu: R = max(1, ceil(max_blocks / 32)) rounds,
h halves, p parts:
  cooperative kernel 1;  per-prompt rounds 6 + 2 h R;  class pipeline 8 + 6 p (R + 1);  hand-over 13 + 2 h R.
"""
import os
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import kvidx
import scale_workload as sw

pytestmark = pytest.mark.gpu

B, P, W = 16, sw.P_PROD, sw.WEIGHTS_PROD
Q = 1 << 20                          # the benchmark's resident batch
QA = Q + (1 << 16)                   # ... and its host-buffer batch after it
MIB, GIB = 1 << 20, 1 << 30
NEED_BYTES = 48 * GIB                # device memory the module needs (measured peak plus room)
CHECK_ROWS = 1 << 17                 # rows of expected scores built at a time
DISPATCH_VARS = ("KVIDX_SCORE_KERNEL", "KVIDX_SCORE_PATH", "KVIDX_COOP_MAX", "KVIDX_ZEROCOPY_MAX", "KVIDX_CLASSES_MIN",
                 "KVIDX_CLASSES_SHARING", "KVIDX_SORT_PREFIX", "KVIDX_HOST_CHUNK_TOKENS", "KVIDX_ROUNDS_PARTS",
                 "KVIDX_ROUNDS_WARP_MAX", "KVIDX_ROUNDS_DEDUP", "KVIDX_ROUNDS_OVERLAP_MIN")

# (start, prompts, path) windows of batch A.  Below 131 072 prompts the size alone decides; from there the class pipeline
# hands a batch over when more than 15 % of its first blocks are distinct (the third window: about 29 %).
WINDOWS = [
    (0, Q, "classes"),                             # the benchmark's step: 8 parts, kernel G's warps take a second tile
    (QA - (1 << 19), 1 << 19, "classes"),          # across 2^32
    (QA - 131072, 131072, "handover"),             # to the per-prompt rounds, warp walk (at most 131 072 prompts)
    (QA - 131071, 131071, "rounds"),               # two halves
    (Q - 32768, 65536, "rounds"),                  # two halves, across 2^32
    (Q + 1, 65535, "rounds"),                      # one half
    (QA - 2049, 2049, "rounds"),
    (Q - 1024, 2048, "coop"),                      # across 2^32
    (QA - 1, 1, "coop"),
]
SPARSE_WINDOWS = WINDOWS[:2]


def launches(path, n, max_blocks):
    R = max(1, -(-max_blocks // 32))
    h = 2 if n >= 65536 else 1
    return {"coop": 1, "rounds": 6 + 2 * h * R, "classes": 8 + 6 * 8 * (R + 1), "handover": 13 + 2 * h * R}[path]


_mem = {"peak": 0}


def _sample():
    free, total = torch.cuda.mem_get_info()
    _mem["peak"] = max(_mem["peak"], total - free)


def _free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _index(wls, weights=W, **kw):
    return kvidx.Index(block_size=B, capacity=sum(w.n_blocks for w in wls) + (1 << 20), max_pods=P, tier_weights=weights, **kw)


@pytest.fixture(scope="module")
def idx():
    set_vars = [v for v in DISPATCH_VARS if v in os.environ]
    assert not set_vars, "this module tests the default dispatch; unset %s" % set_vars
    free, total = torch.cuda.mem_get_info()
    if total < NEED_BYTES:
        pytest.skip("the device has %.0f GiB; production-size batches need %.0f GiB" % (total / GIB, NEED_BYTES / GIB))
    t0 = time.time()
    _mem["base"] = total - free
    wls = sw.production_workloads()
    ix = _index(wls)
    for w in wls:
        for d0 in range(0, w.D, 4096):
            rc, dropped = ix.apply_events(*w.fill_events(d0, min(w.D, d0 + 4096)))
            assert rc == 0 and dropped == 0, ix.last_error()
    assert ix.stats()["request_keys"] == sum(w.n_blocks for w in wls)
    ns = SimpleNamespace(wls=wls, ix=ix, image=None)
    yield ns
    ix.close()
    del ns.ix, ns.image
    _free()
    print("\n[scale] %s: peak device memory in use %.1f GiB (%.1f GiB before the module), module wall time %.0f s"
          % (torch.cuda.get_device_name(), _mem["peak"] / GIB, _mem["base"] / GIB, time.time() - t0))


def _image(idx):
    if idx.image is None:
        idx.image = idx.ix.snapshot()
    return idx.image


def _check(what, got, has, exp_rows, n):
    """got (n, P) f64 and has (n,) u8 on the device against exp_rows(r0, r1) -> (scores, has), chunk by chunk."""
    for c0 in range(0, n, CHECK_ROWS):
        c1 = min(n, c0 + CHECK_ROWS)
        exp, exp_has = exp_rows(c0, c1)
        bad = sw.first_mismatch(got[c0:c1], exp)
        assert bad is None, "%s: row %d differs: got %s, expected %s" % (
            what, c0 + bad, _present(got[c0 + bad]), _present(exp[bad]))
        bad = sw.first_mismatch(has[c0:c1], exp_has)
        assert bad is None, "%s: has_keys of row %d is %d, expected %d" % (what, c0 + bad, int(has[c0 + bad]), int(exp_has[bad]))


def _present(row):
    r = row.cpu().numpy()
    return {int(p): float(r[p]) for p in np.flatnonzero(r != -1.0)}


# ---- batch A ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="class")
def A(idx):
    wl = idx.wls[0]
    dev = torch.device("cuda")
    tok = torch.empty((QA, wl.T), dtype=torch.int32, device=dev)
    _, doc, m = sw.query_tokens(wl, 0, QA, dev, out=tok)
    a = SimpleNamespace(
        tok=tok, off=torch.arange(0, (QA + 1) * wl.T, wl.T, dtype=torch.int64, device=dev),
        doc=torch.from_numpy(doc).to(dev), m=torch.from_numpy(m).to(dev), doc_np=doc, m_np=m,
        sc=torch.empty((Q, P), dtype=torch.float64, device=dev), has=torch.empty(Q, dtype=torch.uint8, device=dev),
        sp_pods=torch.empty((Q, 10), dtype=torch.int16, device=dev), sp_sc=torch.empty((Q, 10), dtype=torch.float64, device=dev),
        sp_cnt=torch.empty(Q, dtype=torch.uint8, device=dev))
    a.nblk = torch.full((QA,), wl.n, dtype=torch.int64, device=dev)
    a.cf = {W: sw.ClosedForm(idx.wls, W, P, dev)}
    _free()                              # the generator's temporaries
    _sample()
    yield a
    a.__dict__.clear()
    _free()


class TestBatchA:
    def _rows(self, A, start, weights=W):
        if weights not in A.cf:
            A.cf[weights] = sw.ClosedForm(A.cf[W].wls, weights, P, A.doc.device)
        cf = A.cf[weights]
        return lambda r0, r1: cf.rows(A.doc[start + r0:start + r1], A.m[start + r0:start + r1], A.nblk[start + r0:start + r1])

    def _score(self, A, ix, start, n, path, weights=W):
        """Score prompts start .. start+n-1 into sentinel-filled outputs, assert the path, check every row."""
        A.sc[:n].fill_(-7.0)
        A.has[:n].fill_(0xAB)
        torch.cuda.synchronize()
        l0 = ix.stats()["kernel_launches"]
        ix.score_batch_dev(A.tok.data_ptr(), A.off[start:].data_ptr(), n, A.sc.data_ptr(), d_has_keys=A.has.data_ptr())
        ix.synchronize()
        _sample()
        got = ix.stats()["kernel_launches"] - l0
        assert got == launches(path, n, 256), "window (%d, %d): %d launches, %s takes %d" % (start, n, got, path, launches(path, n, 256))
        _check("window (%d, %d)" % (start, n), A.sc[:n], A.has[:n], self._rows(A, start, weights), n)

    @pytest.mark.parametrize("start,n,path", WINDOWS, ids=["%s-%d-%d" % (p, s, n) for s, n, p in WINDOWS])
    def test_window_every_row(self, idx, A, start, n, path):
        m, doc = A.m_np[start:start + n], A.doc_np[start:start + n]
        if n >= 131072:                  # the side of the class pipeline's sharing threshold this window is on
            distinct = len(np.unique(doc[m > 0])) + int((m == 0).sum())
            assert (distinct > 0.15 * n) == (path == "handover"), (distinct, n)
        self._score(A, idx.ix, start, n, path)

    @pytest.mark.parametrize("start,n,path", SPARSE_WINDOWS, ids=["%d-%d" % (s, n) for s, n, _ in SPARSE_WINDOWS])
    def test_sparse_window_every_row(self, idx, A, start, n, path):
        A.sp_pods[:n].fill_(-1)
        A.sp_sc[:n].fill_(-7.0)
        A.sp_cnt[:n].fill_(0xEE)
        A.has[:n].fill_(0xAB)
        torch.cuda.synchronize()
        l0 = idx.ix.stats()["kernel_launches"]
        idx.ix.score_batch_sparse_dev(A.tok.data_ptr(), A.off[start:].data_ptr(), n, A.sp_pods.data_ptr(), A.sp_sc.data_ptr(),
                                      A.sp_cnt.data_ptr(), d_has_keys=A.has.data_ptr())
        idx.ix.synchronize()
        assert idx.ix.stats()["kernel_launches"] - l0 == launches(path, n, 256)
        rows = self._rows(A, start)
        for c0 in range(0, n, CHECK_ROWS):
            c1 = min(n, c0 + CHECK_ROWS)
            exp, exp_has = rows(c0, c1)
            cnt = A.sp_cnt[c0:c1]
            assert torch.equal(cnt.to(torch.int64), (exp != -1.0).sum(1)), "sparse window (%d, %d): entry counts" % (start, n)
            dense = sw.sparse_to_dense(A.sp_pods[c0:c1], A.sp_sc[c0:c1], cnt, P)
            bad = sw.first_mismatch(dense, exp)
            assert bad is None, "sparse window (%d, %d): row %d: got %s, expected %s" % (start, n, c0 + bad, _present(dense[bad]), _present(exp[bad]))
            assert torch.equal(A.has[c0:c1], exp_has)

    def test_round_arena_regrows_at_production_sizes(self, idx, A):
        """One handle, batches that grow, shrink and grow again: the round-scratch arena is re-carved between calls."""
        for start, n, path in [(0, Q, "classes"), (QA - 2049, 2049, "rounds"), (QA - (1 << 19), 1 << 19, "classes"),
                               (QA - 131072, 131072, "handover"), (0, Q, "classes")]:
            self._score(A, idx.ix, start, n, path)

    def test_other_tier_weights(self, idx, A):
        w = (0.1, 0.3)
        ix = _index(idx.wls, weights=w)
        try:
            ix.restore(_image(idx))
            self._score(A, ix, 0, Q, "classes", weights=w)
        finally:
            ix.close()
            _free()

    def test_two_shards_on_one_device(self, idx, A):
        sh = [_index(idx.wls, shard_rank=r, shard_count=2) for r in range(2)]
        try:
            sh[0].shard_attach(1, sh[1])
            sh[1].shard_attach(0, sh[0])
            got = [s.shard_restore(_image(idx)) for s in sh]
            assert sum(g["request_keys"] for g in got) == sum(w.n_blocks for w in idx.wls)
            for s, (start, n) in zip(sh, [(QA - (1 << 19), 1 << 19), (Q - 1024, 2048)]):
                A.sc[:n].fill_(-7.0)
                A.has[:n].fill_(0xAB)
                torch.cuda.synchronize()
                s.score_batch_dev(A.tok.data_ptr(), A.off[start:].data_ptr(), n, A.sc.data_ptr(), d_has_keys=A.has.data_ptr())
                s.synchronize()
                _sample()
                _check("shard window (%d, %d)" % (start, n), A.sc[:n], A.has[:n], self._rows(A, start), n)
        finally:
            for s in sh:
                s.close()
            _free()

    def test_host_pipeline_default_chunking(self, idx, A):
        """The benchmark's host-buffer batch: 65 536 prompts in pinned memory, 32 Mi-token chunks (8 of them, alternating
        slots, each with its own token base), dense and sparse rows."""
        ix, wl = idx.ix, idx.wls[0]
        n = QA - Q
        h_tok = kvidx.pinned_array((n * wl.T,), np.uint32)
        torch.from_numpy(h_tok.view(np.int32)).copy_(A.tok[Q:].reshape(-1))
        h_off = np.arange(0, (n + 1) * wl.T, wl.T, dtype=np.int64)
        h_sc = kvidx.pinned_array((n, P), np.float64)
        h_sc.fill(-7.0)
        exp, exp_has = self._rows(A, Q)(0, n)
        exp, exp_has = exp.cpu(), exp_has.cpu()
        per_chunk = launches("rounds", 8192, 256)
        l0 = ix.stats()["kernel_launches"]
        _, has = ix.score_batch(h_tok, h_off, out=h_sc)
        assert ix.stats()["kernel_launches"] - l0 == 8 * per_chunk
        bad = sw.first_mismatch(torch.from_numpy(h_sc), exp)
        assert bad is None, "host rows: row %d" % bad
        assert np.array_equal(has, exp_has.numpy())
        pods, scs, cnt, has = ix.score_batch_sparse(h_tok, h_off)
        assert np.array_equal(cnt.astype(np.int64), (exp != -1.0).sum(1).numpy())
        dense = sw.sparse_to_dense(torch.from_numpy(pods.view(np.int16)), torch.from_numpy(scs), torch.from_numpy(cnt), P)
        bad = sw.first_mismatch(dense, exp)
        assert bad is None, "sparse host rows: row %d" % bad
        assert np.array_equal(has, exp_has.numpy())
        del h_tok, h_sc


# ---- batch B ---------------------------------------------------------------------------------------------------------
def _ragged(idx, spec, profile):
    dev = torch.device("cuda")
    b = sw.ragged_batch(idx.wls, spec["n"], spec["seed"], P, profile)
    t = SimpleNamespace(b=b, n=spec["n"], tok=sw.ragged_tokens(idx.wls, b, spec["tok_seed"], dev),
                        off=torch.from_numpy(b["off"]).to(dev), model=torch.from_numpy(b["model"].astype(np.int32)).to(dev),
                        filt=torch.from_numpy(b["filter"].view(np.int64)).to(dev),
                        maxb=int((b["length"] // B).max()))
    cf = sw.ClosedForm(idx.wls, W, P, dev)
    t.rows = lambda r0, r1: cf.rows(
        *(torch.from_numpy(b[k][r0:r1]).to(dev) for k in ("doc", "m")), torch.from_numpy(b["length"][r0:r1] // B).to(dev),
        kind=torch.from_numpy(b["kind"][r0:r1]).to(dev), model=t.model[r0:r1].to(torch.int64), filt=t.filt[r0:r1])
    return t


def _score_ragged(ix, t, path, halves_or_parts_note):
    dev = t.tok.device
    sc = torch.full((t.n, P), -7.0, dtype=torch.float64, device=dev)
    has = torch.full((t.n,), 0xAB, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    l0 = ix.stats()["kernel_launches"]
    ix.score_batch_dev(t.tok.data_ptr(), t.off.data_ptr(), t.n, sc.data_ptr(), d_model=t.model.data_ptr(), d_filter=t.filt.data_ptr(),
                       d_has_keys=has.data_ptr())
    ix.synchronize()
    _sample()
    got = ix.stats()["kernel_launches"] - l0
    assert got == launches(path, t.n, t.maxb), "%d launches; %s (%s) takes %d" % (got, path, halves_or_parts_note, launches(path, t.n, t.maxb))
    _check("ragged batch of %d" % t.n, sc, has, t.rows, t.n)


def test_ragged_batch_class_pipeline(idx):
    t = _ragged(idx, sw.BATCH_B, sw.MIXED)
    try:
        _score_ragged(idx.ix, t, "classes", "8 parts")
    finally:
        del t
        _free()


def test_ragged_low_sharing_hand_over_lane_walk(idx):
    t = _ragged(idx, sw.BATCH_B_LOW, sw.LOW_SHARING)
    try:
        _score_ragged(idx.ix, t, "handover", "two halves, lane walk")
    finally:
        del t
        _free()
