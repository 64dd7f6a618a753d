#!/usr/bin/env python
"""Randomised soak of the Score() paths against the C++ oracle (run on a GPU box):
   python scripts/soak.py [iterations] [first_seed]
Every iteration builds a random prefix tree of documents (forks at arbitrary token positions, optional tiny alphabet so
that unrelated prompts agree for a while), caches random prefixes of them on random pods / tiers / models, and scores a
random batch (duplicates, truncations, random tails, per-prompt models and filters) through a randomly chosen path
configuration.  Any mismatch prints the seed and exits non-zero."""
import os, sys
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "llm-d-kv-cache-manager_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import numpy as np

def one(seed):
    rng = np.random.default_rng(seed)
    cfg = [("classes", "1"), ("classes", "2"), ("classes", "8"), ("rounds", "2"), ("classes", "4"), ("coop", "1"), ("coop", "1")][int(rng.integers(0, 7))]
    os.environ["KVIDX_ROUNDS_WARP_MAX"] = ("0", "131072")[int(rng.integers(0, 2))]   # per-prompt rounds: lane- / warp-per-prompt walk kernel
    os.environ["KVIDX_ZEROCOPY_MAX"] = str(int(rng.choice([0, 32])))
    os.environ["KVIDX_SCORE_PATH"] = cfg[0]
    os.environ["KVIDX_ROUNDS_OVERLAP_MIN"] = "64"
    os.environ["KVIDX_ROUNDS_PARTS"] = cfg[1]
    os.environ["KVIDX_ROUNDS_DEDUP"] = str(int(rng.integers(1, 3))) if rng.random() < 0.3 else "2"
    os.environ["KVIDX_SORT_PREFIX"] = "0" if rng.random() < 0.2 else "1"
    import kvidx
    from oracle.kvoracle_c import COracle
    from helpers import csr, filter_mask
    BS, P, NM = 16, int(rng.choice([8, 24, 64])), int(rng.integers(1, 3))
    w = (1.0, 0.8, 0.3)
    ix = kvidx.Index(capacity=1 << 15, max_pods=P, tier_weights=w)
    co = COracle(block_size=BS, init_hash=kvidx.fnv64a(b""), size=1 << 15, pod_cache_size=10, tier_weights=w, max_pods=P)
    vocab = int(rng.choice([2, 3, 50000]))
    paths = [rng.integers(0, vocab, size=int(rng.integers(100, 4000)), dtype=np.uint32)]
    for _ in range(int(rng.integers(5, 40))):
        par = paths[int(rng.integers(0, len(paths)))]
        cut = int(rng.integers(1, len(par)))
        paths.append(np.concatenate([par[:cut], rng.integers(0, vocab, size=int(rng.integers(16, 2000)), dtype=np.uint32)]))
    for pth in paths:
        keys = ix.hash_keys(pth, np.array([0, len(pth)], np.int64))[0]
        if len(keys) == 0 or rng.random() < 0.2:
            continue
        for _ in range(int(rng.integers(1, 4))):
            nb = int(rng.integers(1, len(keys) + 1))
            mdl = int(rng.integers(0, NM))
            pt = [(int(rng.integers(0, P)) << 4) | int(rng.integers(0, 3)) for _ in range(int(rng.integers(1, 4)))]
            eng = (keys[:nb] ^ np.uint64(0x1234 + mdl)).astype(np.uint64)
            assert ix.add(mdl, eng, keys[:nb], pt) == 0
            co.add(mdl, eng, keys[:nb], pt)
    n = int(rng.choice([1, 40, 700, 5000]))
    prompts, models = [], np.zeros(n, np.uint32)
    for i in range(n):
        pth = paths[int(rng.integers(0, len(paths))) if rng.random() < 0.7 else 0]
        pr = pth[: int(rng.integers(0, len(pth) + 1))]
        if rng.random() < 0.4:
            pr = np.concatenate([pr, rng.integers(0, vocab, size=int(rng.integers(0, 200)), dtype=np.uint32)])
        prompts.append(pr.astype(np.uint32)); models[i] = int(rng.integers(0, NM))
    tok, off = csr(prompts)
    fm = None
    if rng.random() < 0.5:
        fm = np.zeros((n, ix.filter_words), np.uint64)
        for i in range(0, n, int(rng.integers(1, 4))):
            fm[i] = filter_mask(rng.choice(P, size=int(rng.integers(1, 4)), replace=False).tolist(), ix.filter_words)
    kw = dict(filter_mask=fm) if fm is not None else {}
    s_t, h_t = ix.score_batch(tok, off, model=models, **kw)
    s_o, h_o, _, _ = co.score_batch(tok, off, model=models, n_threads=4, **kw)
    ok = np.array_equal(h_t, h_o) and np.array_equal(s_t, s_o)
    if not ok:
        print("MISMATCH seed", seed, cfg, dict((k, os.environ[k]) for k in os.environ if k.startswith("KVIDX_")), np.argwhere(s_t != s_o)[:5])
    del ix
    return ok

if __name__ == "__main__":
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    s0 = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    bad = 0
    for s in range(s0, s0 + iters):
        bad += 0 if one(s) else 1
    print("soak: %d iterations from seed %d, %d mismatches" % (iters, s0, bad))
    sys.exit(1 if bad else 0)
