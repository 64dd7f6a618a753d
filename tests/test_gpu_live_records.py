"""GPU (-m gpu): the class pipeline's per-prompt state travels with the live list.

What a live prompt carries from round to round (its position, chain state and where its walk state is) is kept per live
slot of the list and moved along when the list is compacted; the walk states are stored by the slot of the round that
wrote them.  These batches exercise that bookkeeping where it can go wrong: rows in random order relative to the prefix
sort (so the live slots are a permutation of the prompt ids), several models and filter rows, and prompts of unequal
length that leave the list in every round.  Each runs through the class pipeline as one part, 8 and 16 parts, and must
give byte-identical score rows and has_keys to the per-prompt round pipeline.

The KVIDX_ROUNDS_TRACE=1 totals (chunks kernel G streams, election losers, G2 chunk compares, blocks kernel H hashes) are
checked against two runs of the layout that kept this state by prompt id (tests/golden/class_trace_counts.json): where
the state lives must not change how classes form.  On batches like these the totals are not exactly reproducible from
run to run: which prompt wins an election bucket, and which class a prompt that leaves its class attaches to, depend on
thread timing, and so does how far a partial follower gets alone.  (Both runs of the old layout differ from each other by
up to 8 %.)  So the check is the recorded range with a margin: 1 % for the chunks streamed, 15 % for the others.  A
layout error that broke class formation would multiply them."""
import json
import os
import re
import tempfile

import numpy as np
import pytest

from helpers import GOLDEN, _select_path, csr, filter_mask

pytestmark = pytest.mark.gpu
BS, P = 16, 64
TRACE = re.compile(r"round (\d+) part (\d+): .*? G streamed (\d+) chunks, (\d+) losers re-read, G2 compared (\d+), H hashed (\d+) blocks")
PARTS = [1, 8, 16]
BATCHES = ["shuffled", "models_filter", "ragged"]


def _docs(rng):
    """Documents, some forking off others at arbitrary token positions."""
    docs = [rng.integers(0, 60000, size=int(rng.integers(20, 260)) * BS + int(rng.integers(0, BS)), dtype=np.uint32) for _ in range(24)]
    for _ in range(24):
        parent = docs[int(rng.integers(0, len(docs)))]
        cut = int(rng.integers(1, len(parent)))
        docs.append(np.concatenate([parent[:cut], rng.integers(0, 60000, size=int(rng.integers(100, 3000)), dtype=np.uint32)]))
    return docs


def _batch(name):
    """(documents, models the index caches them under, prompts, per-prompt model or None, filter rows or None)"""
    rng = np.random.default_rng(BATCHES.index(name) + 70)
    docs = _docs(rng)
    models, model, fm = [0], None, None
    prompts = []
    if name == "shuffled":                 # prefixes of the documents, rows in random order
        for i in range(6000):
            d = docs[int(rng.integers(0, len(docs)))]
            cut = int(rng.integers(BS, len(d) + 1))
            tail = rng.integers(0, 60000, size=int(rng.integers(0, 200)), dtype=np.uint32) if i % 4 == 0 else np.zeros(0, np.uint32)
            prompts.append(np.concatenate([d[:cut], tail]))
    elif name == "models_filter":          # three models, a filter row on some prompts (an empty row: every pod)
        models = [0, 1, 2]
        for i in range(4000):
            d = docs[int(rng.integers(0, len(docs)))]
            prompts.append(d[:int(rng.integers(BS, len(d) + 1))])
        model = rng.integers(0, 3, size=len(prompts)).astype(np.uint32)
        fm = np.zeros((len(prompts), 1), np.uint64)
        for i in range(0, len(prompts), 3):
            fm[i] = filter_mask(sorted({int(x) for x in rng.integers(0, P, size=int(rng.integers(1, 12)))}), 1)
    else:                                  # unequal lengths: every round, some prompts run out of tokens
        for i in range(5000):
            d = docs[int(rng.integers(0, len(docs)))]
            nblk = int(rng.integers(0, len(d) // BS + 1))
            extra = int(rng.integers(0, BS))
            prompts.append(d[:min(len(d), nblk * BS + extra)])
        prompts[::97] = [np.zeros(0, np.uint32)] * len(prompts[::97])
    return docs, models, prompts, model, fm


def _index(docs, models):
    import kvidx
    ix = kvidx.Index(capacity=1 << 16, max_pods=P, tier_weights=(1.0, 0.8))
    rng = np.random.default_rng(5)
    for mdl in models:
        for d in docs:
            keys = ix.hash_keys(d, np.array([0, len(d)], np.int64))[0]
            for pod in rng.choice(P, size=int(rng.integers(1, 5)), replace=False):
                nb = int(rng.integers(1, len(keys) + 1))             # cached up to a random depth on this pod
                assert ix.add(mdl, (keys[:nb] ^ np.uint64(0x5EED + mdl)).astype(np.uint64), keys[:nb], [(int(pod) << 4) | int(rng.integers(0, 2))]) == 0
    return ix


def _score(path, name, monkeypatch, trace=False):
    """score rows, has_keys and (with trace) the summed trace counts of one batch on one path"""
    _select_path(monkeypatch, path)
    if trace:
        monkeypatch.setenv("KVIDX_ROUNDS_TRACE", "1")
    docs, models, prompts, model, fm = _batch(name)
    ix = _index(docs, models)
    tok, off = csr(prompts)
    if not trace:
        s, h = ix.score_batch(tok, off, model=model, filter_mask=fm)
        return s, h, None
    with tempfile.TemporaryFile(mode="w+") as f:       # the trace lines go to the library's stderr
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            s, h = ix.score_batch(tok, off, model=model, filter_mask=fm)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        err = f.read()
    rows = [tuple(int(v) for v in m.groups()) for m in TRACE.finditer(err)]
    assert rows, err
    return s, h, [sum(r[k] for r in rows) for k in range(2, 6)]


def trace_counts_and_scores(name, parts, monkeypatch):
    return _score("classes%s" % (parts if parts > 1 else ""), name, monkeypatch, trace=True)


@pytest.mark.parametrize("parts", PARTS)
@pytest.mark.parametrize("name", BATCHES)
def test_class_pipeline_matches_per_prompt_rounds(name, parts, monkeypatch):
    with monkeypatch.context() as m:
        s_r, h_r, _ = _score("rounds", name, m)
    with monkeypatch.context() as m:
        s_c, h_c, counts = trace_counts_and_scores(name, parts, m)
    assert s_c.tobytes() == s_r.tobytes(), np.argwhere(s_c != s_r)[:5]
    assert h_c.tobytes() == h_r.tobytes()
    assert (s_r.max(axis=1) > 0).sum() > len(s_r) // 10          # the batch does hit the index
    with open(os.path.join(GOLDEN, "class_trace_counts.json")) as f:
        runs = json.load(f)["runs"]["%s/%d" % (name, parts)]
    for k, (what, tol) in enumerate([("streamed", 0.01), ("losers", 0.15), ("compares", 0.15), ("hashed", 0.15)]):
        lo, hi = min(r[k] for r in runs), max(r[k] for r in runs)
        assert lo * (1 - tol) <= counts[k] <= hi * (1 + tol), (what, counts, runs)
