"""Production-size Score() batches of synth.Workload and their exact expected rows, in plain torch on any device.

Two kinds of batch:
  - fixed   : prompts q0 .. q0+n-1 of a workload's query stream (synth.Workload.queries, T tokens each), generated in
              chunks straight into a device tensor, the way a resident benchmark batch is built.
  - ragged  : prompts that start with the first m blocks of a document of one of several workloads (each stored under its
              own model id) and go on with random tokens to any length m*B + r: zero-length and sub-block prompts, partial
              last blocks, unaligned starts, tails of 32 K+ tokens, prompts scored under another model than their
              document's, and per-prompt pod filter rows.

The expected rows are the closed form of synth.Workload.expected_scores extended to those prompts: pod j of the
prompt's document scores the sequential f64 sum of min(m, depth_j) copies of its tier weight, when m > 0, the prompt is
scored under the model its document is stored under, and the pod passes the filter (a non-empty row keeps only its pods;
the filter applies to block 0, so a pod outside it never scores).  Everything else is -1.  has_keys is 1 when the prompt
has a full block.  Documents are random, so no block of a tail and no block past m is in the index.
"""
from __future__ import annotations

import numpy as np
import torch

from kvidx import synth

_GAMMA = -0x61C8864680B583EB          # 0x9E3779B97F4A7C15 as int64
_M1 = -0x40A7B892E31B1A47             # 0xBF58476D1CE4E5B9
_M2 = -0x6B2FB644ECCEEE15             # 0x94D049BB133111EB


def _i64(v: int) -> int:
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >= (1 << 63) else v


def _lsr(x, k):
    return (x >> k) & ((1 << (64 - k)) - 1)


def mix(z):
    """SplitMix64's finaliser on int64 tensors (wrapping arithmetic, logical shifts)."""
    z = (z ^ _lsr(z, 30)) * _M1
    z = (z ^ _lsr(z, 27)) * _M2
    return z ^ _lsr(z, 31)


def umod(z, m: int):
    """z as uint64, mod m."""
    r = torch.remainder(z, m)
    return torch.where(z < 0, torch.remainder(r + ((1 << 64) % m), m), r)


def stream(seed: int, start: int, count: int, device):
    """Outputs start .. start+count-1 of SplitMix64(seed), as synth.stream."""
    idx = torch.arange(start + 1, start + count + 1, dtype=torch.int64, device=device)
    return mix(idx * _GAMMA + _i64(seed))


def query_tokens(wl, q0: int, nq: int, device, out=None, chunk: int = 8192):
    """Prompts q0 .. q0+nq-1 of wl's query stream: tokens (nq, T) int32 (into `out` if given) and doc, m as int64 numpy
    arrays.  Row i equals wl.queries(q0 + i, q0 + i + 1) token for token."""
    r = synth.stream(wl.s_q, q0 * 2, nq * 2).reshape(nq, 2)
    doc = (r[:, 0] % np.uint64(wl.D)).astype(np.int64)
    m = (r[:, 1] % np.uint64(wl.n + 1)).astype(np.int64)
    out = torch.empty((nq, wl.T), dtype=torch.int32, device=device) if out is None else out
    assert out.shape == (nq, wl.T) and out.dtype == torch.int32
    col = torch.arange(wl.T, dtype=torch.int64, device=device)[None, :]
    for c0 in range(0, nq, chunk):
        c1 = min(nq, c0 + chunk)
        tail = umod(stream(wl.s_tail, (q0 + c0) * wl.T, (c1 - c0) * wl.T, device), wl.vocab).view(c1 - c0, wl.T)
        d = torch.from_numpy(doc[c0:c1]).to(device)[:, None]
        dtok = umod(mix((d * wl.T + col + 1) * _GAMMA + _i64(wl.s_doc)), wl.vocab)
        mm = torch.from_numpy(m[c0:c1]).to(device)[:, None] * wl.B
        out[c0:c1] = torch.where(col < mm, dtok, tail).to(torch.int32)
        del tail, d, dtok, mm
    return out, doc, m


# ---- ragged batches --------------------------------------------------------------------------------------------------
# Shares of the prompts: "short" (no full block), "m0" (full blocks, none of them a document's), "deep" (m anywhere in
# 1 .. n), the rest m in 1 .. m_max; "kind1" start with a document of the second workload, "cross" are scored under the
# other model; "long" prompts (a count) get a random tail of 32 K+ tokens.  Filter rows: "f_none" empty, "f_super" the
# document's pods and more, "f_some" some of the document's pods (and others), the rest none of them.
MIXED = dict(short=0.03, m0=0.05, deep=0.05, m_max=96, kind1=0.10, cross=0.12, long=6, f_none=0.5, f_super=0.15, f_some=0.2)
LOW_SHARING = dict(MIXED, m0=0.40, long=2)


def ragged_batch(wls, n: int, seed: int, P: int, profile=MIXED):
    """A ragged batch of n prompts over the workloads `wls` (wls[k] stored under model wls[k].model): a dict of numpy
    arrays kind, doc, m, length, model (n,), filter (n, ceil(P/64)) uint64, the CSR offsets off (n+1,), and the block size B."""
    rng = np.random.default_rng(seed)
    B = wls[0].B
    assert all(w.B == B and w.vocab == wls[0].vocab for w in wls)
    pods = [w.doc_pods(0, w.D) for w in wls]
    kind = (rng.random(n) < profile["kind1"]).astype(np.int64) if len(wls) > 1 else np.zeros(n, np.int64)
    D = np.array([w.D for w in wls])[kind]
    nk = np.array([w.n for w in wls])[kind]
    doc = (rng.random(n) * D).astype(np.int64)
    u = rng.random(n)
    short = u < profile["short"]
    m0 = (u >= profile["short"]) & (u < profile["short"] + profile["m0"])
    deep = (u >= profile["short"] + profile["m0"]) & (u < profile["short"] + profile["m0"] + profile["deep"])
    m = 1 + (rng.random(n) * np.minimum(nk, profile["m_max"])).astype(np.int64)
    m[deep] = 1 + (rng.random(int(deep.sum())) * nk[deep]).astype(np.int64)
    m[short | m0] = 0
    r = rng.integers(0, 4 * B, n)                          # a tail: partial last block, or a few random blocks
    r[m0] = rng.integers(B, 64 * B, int(m0.sum()))
    r[short] = np.where(rng.random(int(short.sum())) < 0.5, 0, rng.integers(1, B, int(short.sum())))
    longs = rng.choice(np.flatnonzero(~short), size=min(profile["long"], int((~short).sum())), replace=False)
    r[longs] = rng.integers(32768, 40000, len(longs))
    length = m * B + r
    model = np.array([w.model for w in wls])[kind]
    if len(wls) > 1:
        cross = rng.random(n) < profile["cross"]
        model[cross] = np.array([w.model for w in wls])[1 - kind[cross]]
    # filter rows
    W = (P + 63) // 64
    filt = np.zeros((n, W), np.uint64)
    dp = np.zeros((n, 4), np.int64)                       # the prompt's document's pods
    for k in range(len(wls)):
        dp[kind == k] = pods[k][doc[kind == k]]
    v = rng.random(n)
    f_super = (v >= profile["f_none"]) & (v < profile["f_none"] + profile["f_super"])
    f_some = (v >= profile["f_none"] + profile["f_super"]) & (v < profile["f_none"] + profile["f_super"] + profile["f_some"])
    f_out = v >= profile["f_none"] + profile["f_super"] + profile["f_some"]
    keep = np.zeros((n, 4), bool)
    keep[f_super] = True
    ks = rng.random((n, 4)) < 0.5
    ks[np.arange(n), rng.integers(0, 4, n)] = False        # "some": not all of the document's pods ...
    ks[np.arange(n), rng.integers(0, 4, n)] = True         # ... but at least one (or all, when both lines pick one pod)
    keep[f_some] = ks[f_some]
    rows, cols = np.nonzero(keep & (dp >= 0))
    np.bitwise_or.at(filt, (rows, dp[rows, cols] >> 6), np.uint64(1) << (dp[rows, cols] & 63).astype(np.uint64))
    # other pods, none of the document's: 1 .. 3 for f_out (so that its row is not empty), 0 .. 2 for f_super / f_some
    extra_n = np.where(f_out, rng.integers(1, 4, n), np.where(f_super | f_some, rng.integers(0, 3, n), 0))
    for e in range(3):
        at = np.flatnonzero(e < extra_n)
        x = _not_in(dp[at], P, rng)
        np.bitwise_or.at(filt, (at, x >> 6), np.uint64(1) << (x & 63).astype(np.uint64))
    off = np.zeros(n + 1, np.int64)
    np.cumsum(length, out=off[1:])
    return dict(kind=kind, doc=doc, m=m, length=length, model=model.astype(np.int64), filter=filt, off=off, B=B)


def _not_in(dp, P, rng):
    """One pod per row of dp (k, 4) that is none of the row's pods."""
    x = rng.integers(0, P, len(dp))
    while True:
        clash = (x[:, None] == dp).any(1)
        if not clash.any():
            return x
        x[clash] = rng.integers(0, P, int(clash.sum()))


def ragged_tokens(wls, b, seed: int, device, chunk_tokens: int = 1 << 25):
    """The batch's tokens as one int32 tensor: prompt i's first m*B tokens are its document's, the rest come from a
    SplitMix64 stream of `seed` indexed by position in the batch."""
    off = b["off"]
    total = int(off[-1])
    out = torch.empty(total, dtype=torch.int32, device=device)
    s_doc = torch.tensor([_i64(w.s_doc) for w in wls], dtype=torch.int64, device=device)
    T = torch.tensor([w.T for w in wls], dtype=torch.int64, device=device)
    vocab, B = wls[0].vocab, wls[0].B
    n = len(off) - 1
    start, kind, doc = (torch.from_numpy(b[k]).to(device) for k in ("off", "kind", "doc"))
    mb = torch.from_numpy(b["m"]).to(device) * B
    i0 = 0
    while i0 < n:
        i1 = min(n, max(i0 + 1, int(np.searchsorted(off, off[i0] + chunk_tokens, side="right")) - 1))
        p0, p1 = int(off[i0]), int(off[i1])
        if p1 > p0:
            lens = torch.from_numpy(b["length"][i0:i1]).to(device)
            pid = torch.repeat_interleave(torch.arange(i0, i1, device=device), lens)
            j = torch.arange(p0, p1, dtype=torch.int64, device=device) - start[pid]
            k = kind[pid]
            dtok = umod(mix((doc[pid] * T[k] + j + 1) * _GAMMA + s_doc[k]), vocab)
            tail = umod(stream(seed, p0, p1 - p0, device), vocab)
            out[p0:p1] = torch.where(j < mb[pid], dtok, tail).to(torch.int32)
            del lens, pid, j, k, dtok, tail
        i0 = i1
    return out


# ---- the closed form -------------------------------------------------------------------------------------------------
class ClosedForm:
    """Expected Score() rows of prompts over the workloads `wls` (each filled into the index under its own model), for
    one pair of tier weights, computed on `device` from each workload's D x 4 pod table and a [2, n + 1] table of
    sequential f64 sums."""

    def __init__(self, wls, weights, P: int, device):
        self.wls, self.P, self.device = list(wls), P, device
        self.pods = [torch.from_numpy(w.doc_pods(0, w.D)).to(device) for w in wls]
        nmax = max(w.n for w in wls)
        seq = np.zeros((2, nmax + 1))
        for t in range(2):
            w, acc = max(0.0, float(weights[t])), 0.0
            for L in range(1, nmax + 1):
                acc = acc + w if L > 1 else w
                seq[t, L] = acc
        self.seq = torch.from_numpy(seq).to(device)

    def rows(self, doc, m, n_blocks, kind=None, model=None, filt=None):
        """doc, m, n_blocks (full blocks of each prompt), kind (workload index), model (scored under), filt (n, W) int64
        filter rows: tensors on the device, None = workload 0 / its model / no filter.  -> (scores (n, P) f64, has (n,) u8)."""
        n = len(doc)
        dev = self.device
        kind = torch.zeros(n, dtype=torch.int64, device=dev) if kind is None else kind
        model = torch.zeros(n, dtype=torch.int64, device=dev) if model is None else model
        out = torch.full((n, self.P), -1.0, dtype=torch.float64, device=dev)
        for k, w in enumerate(self.wls):
            live = (kind == k) & (m > 0) & (model == w.model)
            idx = torch.nonzero(live).squeeze(1)
            if len(idx) == 0:
                continue
            d, mi = doc[idx], m[idx]
            empty = (filt[idx] == 0).all(1) if filt is not None else None
            for j in range(4):
                pod = self.pods[k][d, j]
                tier = (((d * 4 + j) % 8) == 7).to(torch.int64)
                L = torch.clamp(mi, max=w.depth(j))
                ok = pod >= 0
                if filt is not None:
                    pc = pod.clamp(min=0)
                    bit = (filt[idx, pc >> 6] >> (pc & 63)) & 1
                    ok &= empty | (bit == 1)
                out[idx[ok], pod[ok]] = self.seq[tier[ok], L[ok]]
        return out, (n_blocks > 0).to(torch.uint8)


def first_mismatch(got, exp):
    """None if got equals exp bit for bit (f64 compared as int64 views), else the first differing row."""
    g = got.contiguous().view(torch.int64) if got.dtype == torch.float64 else got
    e = exp.contiguous().view(torch.int64) if exp.dtype == torch.float64 else exp
    if torch.equal(g, e):
        return None
    bad = (g != e)
    if bad.dim() > 1:
        bad = bad.any(1)
    return int(torch.nonzero(bad)[0, 0])


def sparse_to_dense(pods, scores, cnt, P: int):
    """Sparse result rows ((n, 10) pods, (n, 10) scores, (n,) counts) as dense (n, P) rows, -1 = absent.  A pod listed twice
    leaves another slot of the row at -1, so a dense comparison plus the counts compares the rows as sets."""
    n, E = pods.shape
    out = torch.full((n, P), -1.0, dtype=torch.float64, device=pods.device)
    used = torch.arange(E, device=pods.device)[None, :] < cnt.to(torch.int64)[:, None]
    r = torch.arange(n, device=pods.device)[:, None].expand(n, E)
    p = pods.to(torch.int64) & 0xFFFF
    out[r[used], p[used]] = scores[used]
    return out


def distinct_first_blocks(b) -> int:
    """How many distinct first blocks a ragged batch has: one per document that prompts start with (m > 0), one per prompt
    whose full first block is random (m = 0), and one shared by every prompt without a full block."""
    has = b["length"] >= b["B"]
    docs = np.unique(b["kind"][b["m"] > 0] * (1 << 40) + b["doc"][b["m"] > 0])
    return len(docs) + int((has & (b["m"] == 0)).sum()) + int((~has).any())


# ---- the production-size batches of the GPU module (tests/test_gpu_scale.py), described here so that the CPU suite can
# check what they hold -------------------------------------------------------------------------------------------------
P_PROD = 256
WEIGHTS_PROD = (1.0, 0.8)
BATCH_B = dict(n=1_500_000, seed=0xB0B, tok_seed=0x5CA1E)
BATCH_B_LOW = dict(n=600_000, seed=0xB0C, tok_seed=0x5CA1F)


def production_workloads():
    """The metric workload (config 6: 4096-token prompts, 10 M blocks, 256 pods) under model 0 and a smaller second one
    (1024-token documents, 1 M blocks) under model 1."""
    return (synth.Workload(6, 4096, 10_000_000, P_PROD, 16),
            synth.Workload(7, 1024, 1 << 20, P_PROD, 16, model=1))
