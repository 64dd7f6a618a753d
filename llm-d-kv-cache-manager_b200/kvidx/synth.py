"""Deterministic synthetic workload of SURVEY.md section 8(d) (numpy only; no oracle, no GPU).

PRNG: SplitMix64 used as a counter-based generator -- element i of a stream with
seed s is mix(s + (i+1)*GAMMA), which is exactly the i-th output of the sequential
generator, so streams can be produced vectorised / in slices.

  index fill : D documents of T tokens; document d is stored on 4 distinct pods; pod j
               of a document holds the first ceil((j+1)/4 * n) blocks; every 8th (doc,pod)
               pair is on tier "cpu" (id 1), the rest on "gpu" (id 0).  Delivered as
               BlockStored events (chunks of `blocks_per_event` blocks chained through
               parent_block_hash) so the write path builds the index.
  queries    : first m blocks of a uniformly chosen document (m uniform in [0, n]) followed by
               fresh random tokens up to T; empty pod filter.
Engine hashes are mix64 of (doc, block) -- content-identified like vLLM's, independent of the
request hash (SURVEY suggested ~request_hash; that would need the hash under test to build its
own input).
"""
from __future__ import annotations

import numpy as np

GAMMA = np.uint64(0x9E3779B97F4A7C15)
VOCAB = 128256
EVENT_DTYPE = np.dtype([("op", "u1"), ("has_parent", "u1"), ("podtier", "<u2"), ("model", "<u4"),
                        ("parent_hash", "<u8"), ("hash_off", "<u8"), ("tok_off", "<u8"),
                        ("n_hashes", "<u4"), ("n_tokens", "<u4")])


def mix(z: np.ndarray) -> np.ndarray:
    z = z.astype(np.uint64, copy=True)
    z ^= z >> np.uint64(30); z *= np.uint64(0xBF58476D1CE4E5B9)
    z ^= z >> np.uint64(27); z *= np.uint64(0x94D049BB133111EB)
    z ^= z >> np.uint64(31)
    return z


def stream(seed: int, start: int, count: int) -> np.ndarray:
    """Outputs start .. start+count-1 of SplitMix64(seed)."""
    with np.errstate(over="ignore"):
        idx = np.arange(start + 1, start + count + 1, dtype=np.uint64)
        return mix(np.uint64(seed) + idx * GAMMA)


class Workload:
    def __init__(self, config_id: int, T: int, n_blocks: int, n_pods: int, block_size: int = 16, model: int = 0,
                 blocks_per_event: int = 64, vocab: int = VOCAB):
        self.seed = 0x5EED0000 + config_id
        self.T, self.B, self.P, self.model = T, block_size, n_pods, model
        self.n = T // block_size
        self.D = max(1, n_blocks // self.n)
        self.n_blocks = self.D * self.n
        self.bpe = blocks_per_event
        self.vocab = vocab
        # independent sub-streams
        self.s_doc, self.s_pod, self.s_q, self.s_tail = (self.seed * 4 + i for i in range(4))

    # ---- documents ----
    def doc_tokens(self, d0: int, d1: int) -> np.ndarray:
        """tokens of documents d0..d1-1, shape (d1-d0, T) uint32."""
        x = stream(self.s_doc, d0 * self.T, (d1 - d0) * self.T)
        return (x % np.uint64(self.vocab)).astype(np.uint32).reshape(d1 - d0, self.T)

    def doc_pods(self, d0: int, d1: int) -> np.ndarray:
        """4 distinct pods per document (uniform, without replacement), shape (d1-d0, 4); -1 pads if P < 4."""
        r = stream(self.s_pod, d0 * 4, (d1 - d0) * 4).reshape(d1 - d0, 4)
        P, k = self.P, min(4, self.P)
        res = np.full((d1 - d0, 4), -1, np.int64)
        for j in range(k):
            cand = (r[:, j] % np.uint64(P - j)).astype(np.int64)     # index among the P-j pods not yet taken
            prev = np.sort(res[:, :j], axis=1)
            for q in range(j):
                cand += (cand >= prev[:, q]).astype(np.int64)
            res[:, j] = cand
        return res

    def depth(self, j: int) -> int:
        return -(-(j + 1) * self.n // 4)      # ceil((j+1)/4 * n)

    def engine_hashes(self, d0: int, d1: int) -> np.ndarray:
        """engine hash of (doc, block), shape (d1-d0, n) uint64."""
        with np.errstate(over="ignore"):
            d = np.arange(d0, d1, dtype=np.uint64)[:, None]
            b = np.arange(self.n, dtype=np.uint64)[None, :]
            return mix((d << np.uint64(20)) + b + np.uint64(0xE1E1E1E1) * np.uint64(self.seed))

    def fill_events(self, d0: int, d1: int):
        """BlockStored events that store documents d0..d1-1.  Returns (events, hashes, tokens).
        Events of one pod appear in chain order (chunk c before chunk c+1)."""
        toks = self.doc_tokens(d0, d1)
        pods = self.doc_pods(d0, d1)
        eh = self.engine_hashes(d0, d1)
        nd = d1 - d0
        ev = []
        # the token / hash arrays are the documents themselves; events point into them
        hashes = eh.reshape(-1)
        tokens = toks.reshape(-1)
        recs = []
        for j in range(4):
            dj = self.depth(j)
            nchunk = -(-dj // self.bpe)
            for c in range(nchunk):
                b0, b1 = c * self.bpe, min(dj, (c + 1) * self.bpe)
                docs = np.arange(nd, dtype=np.int64)
                valid = pods[:, j] >= 0
                docs = docs[valid]
                m = len(docs)
                if m == 0:
                    continue
                r = np.zeros(m, EVENT_DTYPE)
                pair = (docs + d0) * 4 + j
                tier = (pair % 8 == 7).astype(np.uint16)
                r["op"] = 0
                r["has_parent"] = 1 if c > 0 else 0
                r["podtier"] = (pods[valid, j].astype(np.uint16) << 4) | tier
                r["model"] = self.model
                r["parent_hash"] = eh[docs, b0 - 1] if c > 0 else 0
                r["hash_off"] = docs * self.n + b0
                r["tok_off"] = docs * self.T + b0 * self.B
                r["n_hashes"] = b1 - b0
                r["n_tokens"] = (b1 - b0) * self.B
                recs.append((c, r))
        # order: all chunk-0 events, then chunk-1, ... keeps every (doc,pod) chain in order
        recs.sort(key=lambda x: x[0])
        ev = np.concatenate([r for _, r in recs]) if recs else np.zeros(0, EVENT_DTYPE)
        return ev, hashes, tokens

    # ---- queries ----
    def queries(self, q0: int, q1: int, full_depth: bool = False):
        """prompts q0..q1-1 as (tokens (nq,T) uint32, doc (nq,), m (nq,))."""
        nq = q1 - q0
        r = stream(self.s_q, q0 * 2, nq * 2).reshape(nq, 2)
        doc = (r[:, 0] % np.uint64(self.D)).astype(np.int64)
        m = (r[:, 1] % np.uint64(self.n + 1)).astype(np.int64)
        if full_depth:
            m[:] = self.n
        out = (stream(self.s_tail, q0 * self.T, nq * self.T) % np.uint64(self.vocab)).astype(np.uint32).reshape(nq, self.T)
        # overwrite the matched prefix with the document's tokens (documents regenerated in sorted batches)
        order = np.argsort(doc, kind="stable")
        i = 0
        while i < nq:
            d = doc[order[i]]
            j = i
            while j < nq and doc[order[j]] == d:
                j += 1
            dt = self.doc_tokens(int(d), int(d) + 1)[0]
            for q in order[i:j]:
                out[q, : m[q] * self.B] = dt[: m[q] * self.B]
            i = j
        return out, doc, m

    def expected_scores(self, doc: np.ndarray, m: np.ndarray, weights=(1.0, 0.8)) -> np.ndarray:
        """Closed-form expectation for the fill above (a size-independent property check that needs no
        oracle): pod j of the document scores the sequential f64 sum of min(m, depth_j) copies of its
        tier weight; pods not holding block 0 are absent (-1)."""
        nq = len(doc)
        out = np.full((nq, self.P), -1.0)
        seq = np.zeros((2, self.n + 1))
        for t in range(2):
            w = max(0.0, float(weights[t]))
            acc = 0.0
            for L in range(1, self.n + 1):
                acc = acc + w if L > 1 else w
                seq[t, L] = acc
        ud, inv = np.unique(doc, return_inverse=True)
        pods_u = np.stack([self.doc_pods(int(d), int(d) + 1)[0] for d in ud]) if len(ud) else np.zeros((0, 4), np.int64)
        pods = pods_u[inv]
        rows = np.arange(nq)
        for j in range(4):
            tier = (((doc * 4 + j) % 8) == 7).astype(np.int64)
            L = np.minimum(m, self.depth(j))
            ok = (m > 0) & (pods[:, j] >= 0)
            out[rows[ok], pods[ok, j]] = seq[tier[ok], L[ok]]
        return out

    def expected_inventory(self):
        """Closed form of the pod inventory (kvidx_pod_inventory, all models, engine pass) of the fill above: block b of a
        document is held by its pods j with depth_j > b, so pod j adds depth_j keys and entries (on its pair's tier), the
        deepest pod alone holds the blocks past the second deepest's depth, and every block has one engine mapping and
        none is stale.  Documents are random, so no two blocks share a key.  Same arrays as kvidx.Index.pod_inventory."""
        pods = self.doc_pods(0, self.D)
        k = min(4, self.P)
        ent = np.zeros((self.P, 16), np.uint64)
        keys, sole = np.zeros(self.P, np.uint64), np.zeros(self.P, np.uint64)
        docs = np.arange(self.D, dtype=np.int64)
        for j in range(k):
            tier = ((docs * 4 + j) % 8 == 7).astype(np.int64)
            np.add.at(ent, (pods[:, j], tier), np.uint64(self.depth(j)))
            np.add.at(keys, pods[:, j], np.uint64(self.depth(j)))
        np.add.at(sole, pods[:, k - 1], np.uint64(self.depth(k - 1) - (self.depth(k - 2) if k > 1 else 0)))
        stored = self.D * self.depth(k - 1)
        return {"entries": ent, "keys": keys, "sole": sole, "sole_engine": sole.copy(),
                "totals": np.array([stored, int(keys.sum()), stored, 0], np.uint64)}
