"""CPU: the reference of the production-size Score() module (tests/scale_workload.py).  Its torch query stream against
synth.Workload.queries, its extended closed form against the C++ oracle filled through the write path, and what its
batches hold."""
import numpy as np
import pytest
import torch

import scale_workload as sw
from kvidx import synth
from oracle.kvoracle_c import COracle

P = 64


def _small():
    return synth.Workload(3, 512, 1 << 13, P), synth.Workload(4, 256, 1 << 12, P, model=1)


@pytest.mark.parametrize("cfg,q0,nq", [((6, 256, 1 << 12, P), 0, 37), ((6, 256, 1 << 12, P), 1000, 100),
                                        ((6, 4096, 10_000_000, 256), (1 << 20) - 3, 6)])
def test_query_tokens_equal_synth_queries(cfg, q0, nq):
    """The last case is the metric workload around prompt 2^20, whose tokens start at 2^32 in the stream."""
    wl = synth.Workload(*cfg)
    tok, doc, m = sw.query_tokens(wl, q0, nq, "cpu", chunk=16)
    want, doc2, m2 = wl.queries(q0, q0 + nq)
    assert np.array_equal(tok.numpy().view(np.uint32), want)
    assert np.array_equal(doc, doc2) and np.array_equal(m, m2)


@pytest.mark.parametrize("profile", ["MIXED", "LOW_SHARING"])
def test_ragged_tokens_start_with_their_document(profile):
    wls = _small()
    b = sw.ragged_batch(wls, 600, 7, P, getattr(sw, profile))
    tok = sw.ragged_tokens(wls, b, 11, "cpu", chunk_tokens=1 << 12).numpy().view(np.uint32)
    assert len(tok) == b["off"][-1]
    for i in range(len(b["m"])):
        k, d, mb = b["kind"][i], b["doc"][i], b["m"][i] * wls[0].B
        assert np.array_equal(tok[b["off"][i]:b["off"][i] + mb], wls[k].doc_tokens(d, d + 1)[0, :mb])
        if b["length"][i] > mb + wls[0].B:           # a random tail, not the document's next block
            assert not np.array_equal(tok[b["off"][i] + mb:b["off"][i] + mb + wls[0].B], wls[k].doc_tokens(d, d + 1)[0, mb:mb + wls[0].B])


def _oracle(wls, weights):
    co = COracle(size=10 ** 6, max_pods=P, tier_weights=weights)
    for w in wls:
        ev, hs, tk = w.fill_events(0, w.D)
        assert co.apply_events(ev, hs, tk) == (0, 0)
    assert co.len_request() == sum(w.n_blocks for w in wls)
    return co


@pytest.mark.parametrize("weights", [(1.0, 0.8), (0.1, 0.3), (0.3, 1.7)])
@pytest.mark.parametrize("profile,seed", [("MIXED", 1), ("LOW_SHARING", 2)])
def test_closed_form_equals_the_oracle(weights, profile, seed):
    wls = _small()
    co = _oracle(wls, weights)
    b = sw.ragged_batch(wls, 3000, seed, P, getattr(sw, profile))
    tok = sw.ragged_tokens(wls, b, seed + 100, "cpu").numpy().view(np.uint32)
    got, has, _, _ = co.score_batch(tok, b["off"], model=b["model"].astype(np.uint32), filter_mask=b["filter"], n_threads=4)
    t = {k: torch.from_numpy(b[k]) for k in ("kind", "doc", "m", "model")}
    exp, exp_has = sw.ClosedForm(wls, weights, P, "cpu").rows(t["doc"], t["m"], torch.from_numpy(b["length"] // wls[0].B),
                                                              kind=t["kind"], model=t["model"],
                                                              filt=torch.from_numpy(b["filter"].view(np.int64)))
    bad = sw.first_mismatch(torch.from_numpy(got), exp)
    assert bad is None, "row %d: %s" % (bad, {k: b[k][bad] for k in ("kind", "doc", "m", "length", "model", "filter")})
    assert np.array_equal(has, exp_has.numpy())
    assert (got >= 0).any() and (got == -1).any()


def test_closed_form_of_fixed_prompts_equals_expected_scores():
    wl = synth.Workload(6, 256, 1 << 12, P)
    _, doc, m = sw.query_tokens(wl, 0, 500, "cpu")
    for w in [(1.0, 0.8), (0.1, 0.3)]:
        exp, has = sw.ClosedForm([wl], w, P, "cpu").rows(torch.from_numpy(doc), torch.from_numpy(m), torch.full((500,), wl.n))
        assert np.array_equal(exp.numpy().view(np.int64), wl.expected_scores(doc, m, w).view(np.int64)) and bool(has.all())


def _kinds(b, wls):
    """Which kinds of prompt a ragged batch holds."""
    B = b["B"]
    L, m, kind, model, off = b["length"], b["m"], b["kind"], b["model"], b["off"]
    fl = b["filter"]
    dp = np.zeros((len(m), 4), np.int64)
    for k, w in enumerate(wls):
        dp[kind == k] = w.doc_pods(0, w.D)[b["doc"][kind == k]]
    inside = ((fl[np.arange(len(m))[:, None], dp >> 6] >> (dp & 63).astype(np.uint64)) & np.uint64(1)).astype(bool)
    empty = ~fl.any(1)
    scored = (m > 0) & (model == np.array([w.model for w in wls])[kind])
    depth_hit = np.zeros(len(m), bool)
    for j in range(4):
        depth_hit |= m == np.array([w.depth(j) for w in wls])[kind]
    # a class: prompts that start with the same document; some must differ in model and in filter row
    key = kind * (1 << 40) + b["doc"]
    cls = m > 0
    order = np.argsort(key[cls], kind="stable")
    ks, mods = key[cls][order], model[cls][order]
    frow = fl[cls][order].view(np.int64) @ np.array([1, 3, 7, 11][:fl.shape[1]], np.int64)
    same = ks[1:] == ks[:-1]
    return {
        "zero-length": (L == 0).any(), "sub-block": ((L > 0) & (L < B)).any(), "m=0 with keys": ((m == 0) & (L >= B)).any(),
        "partial last block": ((m > 0) & (L % B != 0)).any(), "unaligned start": ((m > 0) & (off[:-1] % 4 != 0)).any(),
        "long tail": (L >= 32768).any(), "m = a pod's depth": (depth_hit & (m > 0)).any(),
        "m = n": (m == np.array([w.n for w in wls])[kind]).any(),
        "second model": (scored & (kind == 1)).any(), "model 0 prompt under model 1": ((kind == 0) & (model == 1) & (m > 0)).any(),
        "model 1 prompt under model 0": ((kind == 1) & (model == 0) & (m > 0)).any(),
        "empty filter": (scored & empty).any(), "filter keeps all of the document's pods": (scored & ~empty & inside.all(1)).any(),
        "filter keeps some": (scored & ~empty & inside.any(1) & ~inside.all(1)).any(),
        "filter excludes every pod": (scored & ~empty & ~inside.any(1)).any(),
        "class-mates differ in model": (same & (mods[1:] != mods[:-1])).any(),
        "class-mates differ in filter": (same & (frow[1:] != frow[:-1])).any(),
    }


def test_small_batches_hold_every_kind_of_prompt():
    wls = _small()
    for profile, seed in (("MIXED", 1), ("LOW_SHARING", 2)):
        got = _kinds(sw.ragged_batch(wls, 3000, seed, P, getattr(sw, profile)), wls)
        assert all(got.values()), (profile, [k for k, v in got.items() if not v])


def test_production_batches_hold_every_kind_and_take_their_paths():
    """Batch B shares its first blocks enough for the class pipeline (at most 15 % distinct), its low-sharing variant does
    not: that one is handed over to the per-prompt rounds, with the lane walk (above 131 072 prompts)."""
    wls = sw.production_workloads()
    b = sw.ragged_batch(wls, sw.BATCH_B["n"], sw.BATCH_B["seed"], sw.P_PROD, sw.MIXED)
    got = _kinds(b, wls)
    assert all(got.values()), [k for k, v in got.items() if not v]
    assert sw.distinct_first_blocks(b) <= 0.15 * len(b["m"])
    assert (b["m"] <= 96).mean() > 0.9 and b["off"][-1] < (2 << 30)
    lo = sw.ragged_batch(wls, sw.BATCH_B_LOW["n"], sw.BATCH_B_LOW["seed"], sw.P_PROD, sw.LOW_SHARING)
    assert sw.distinct_first_blocks(lo) > 0.15 * len(lo["m"]) and len(lo["m"]) > 131072
    assert 0.35 < (lo["m"] == 0).mean() < 0.45
