"""Event streams that speak the whole write-path grammar, and a plain model of phase 1's parent prediction.

Importable without a GPU: everything here runs on numpy and the C++ oracle (oracle/kvoracle_c.py).

Documents are token sequences cut into blocks of B tokens.  Engine hashes are content-addressed, as vLLM's are: block k
of a document gets H(engine hash of block k - 1, its tokens), so the same block under the same parent has the same engine
hash on every pod and under every model.  A stream is a list of batches; a batch is a list of `Ev`.

Two families keep the final contents independent of the order in which the library's per-pod queues run:
  "a"  each pod stores and removes only its own documents (or a batch holds one pod's events only: `single_queue`).
       Everything is allowed: removals, restarts at the seed, unknown parents, re-mapped and removed parents.
  "b"  pods share documents and nothing is removed; every parent is resident before the batch or stored earlier in the
       consumer's own queue, so every engine hash maps to its one true request key whatever the schedule.  Entry order
       inside a request record still depends on the schedule: compare images with `sorted_entries`.

`expect_batch` applies a batch to the oracle event by event and returns the dropped count and the number of events phase
1 mispredicts (kvidx stats' rehashed_events), from `phase1_predictions`, a restatement of want_parents_kernel /
offer_blocks_kernel / hash_events_kernel's rule: the latest earlier block of the same pod and model in the batch that
carries the parent hash, else the index as it was before the batch, else the seed.
"""
import hashlib
import struct

import numpy as np

from helpers import EVENT_DTYPE, SNAP_REQ_DTYPE

STORED, REMOVED = 0, 1
EDGE_TOKENS = (0, 23, 24, 255, 256, 65535, 65536, 2 ** 32 - 1)
DROP_KINDS = ("drop_more", "drop_less", "drop_short")


class Ev:
    """One decoded event at id level.  kind names what the generator meant it to be (the self-test checks the shapes
    from the packed arrays, not from this label)."""
    __slots__ = ("op", "pod", "tier", "model", "parent", "hashes", "tokens", "kind")

    def __init__(self, op, pod, tier, model, parent, hashes, tokens, kind):
        self.op, self.pod, self.tier, self.model, self.parent, self.kind = op, pod, tier, model, parent, kind
        self.hashes = np.asarray(hashes, np.uint64)
        self.tokens = np.asarray(tokens, np.uint32)

    def hashable(self, B):
        """The events phase 1 hashes (event_hashable): BlockStored with hashes and as many full token blocks."""
        return self.op == STORED and len(self.hashes) > 0 and len(self.tokens) // B == len(self.hashes)


def pack(events):
    """-> (kvidx_event_t array, hashes, tokens), slices laid out back to back in event order (a trailing partial block
    leaves the next event's tokens misaligned)."""
    ev = np.zeros(len(events), EVENT_DTYPE)
    hs, tk, ho, to = [], [], 0, 0
    for i, e in enumerate(events):
        ev[i]["op"] = e.op
        ev[i]["has_parent"] = e.parent is not None
        ev[i]["parent_hash"] = 0 if e.parent is None else e.parent
        ev[i]["podtier"] = (e.pod << 4) | e.tier
        ev[i]["model"] = e.model
        ev[i]["hash_off"], ev[i]["tok_off"] = ho, to
        ev[i]["n_hashes"], ev[i]["n_tokens"] = len(e.hashes), len(e.tokens)
        hs.append(e.hashes)
        tk.append(e.tokens)
        ho += len(e.hashes)
        to += len(e.tokens)
    return ev, np.concatenate(hs + [np.zeros(0, np.uint64)]), np.concatenate(tk + [np.zeros(0, np.uint32)])


def _ehash(parent, block):
    d = hashlib.blake2b(struct.pack("<Q", parent) + block.tobytes(), digest_size=8).digest()
    return int.from_bytes(d, "little") | 1


class Doc:
    def __init__(self, owner, blocks):
        self.owner = owner
        self.blocks = blocks                                   # (n, B) uint32
        self.eh = []
        h = 0
        for b in blocks:
            h = _ehash(h, b)
            self.eh.append(h)
        self.eh = np.array(self.eh, np.uint64)
        self.alias = []                                        # other engine hashes stored for these blocks

    def __len__(self):
        return len(self.blocks)


class WriteStream:
    """A random stream of one family.  pods: the pod ids; models / tiers: how many ids of each; edge_tokens: how often a
    token is one of the CBOR width edges; removals: family "a" only."""

    def __init__(self, rng, B, family="a", pods=(0, 1, 2), models=2, tiers=2, single_queue=False, edge_tokens=0.1,
                 max_blocks=80, docs_per_pod=6):
        assert family in ("a", "b")
        self.rng, self.B, self.family = rng, B, family
        self.pods, self.models, self.tiers = list(pods), models, tiers
        self.single_queue = single_queue
        self.edge, self.max_blocks = edge_tokens, max_blocks
        self.docs = []
        owners = [None] if (family == "b" or single_queue) else self.pods
        for o in owners:
            for _ in range(docs_per_pod * (len(self.pods) if o is None else 1)):
                self._new_doc(o)
        self.resident = set()          # family "b": (model, engine hash) stored in an earlier batch

    # ---- documents ----
    def _tokens(self, n):
        t = self.rng.integers(0, 2 ** 32, (n, self.B), dtype=np.uint64)
        edge = self.rng.random((n, self.B)) < self.edge
        if not self.single_queue and self.family == "a":
            edge[:, 0] = False         # keep first tokens random so that pods' documents never share a request key
        t[edge] = self.rng.choice(np.array(EDGE_TOKENS, np.uint64), int(edge.sum()))
        return t.astype(np.uint32)

    def _new_doc(self, owner):
        n = int(self.rng.integers(1, self.max_blocks + 1))
        mine = [d for d in self.docs if d.owner == owner]
        if mine and self.rng.random() < 0.4:                  # share a prefix with an existing document
            base = mine[int(self.rng.integers(0, len(mine)))]
            k = int(self.rng.integers(1, len(base) + 1))
            blocks = np.concatenate([base.blocks[:k], self._tokens(max(n - k, 1))])
        else:
            blocks = self._tokens(n)
        self.docs.append(Doc(owner, blocks))

    def _docs_of(self, pod):
        return [d for d in self.docs if d.owner in (None, pod)]

    # ---- events ----
    def _store(self, pod, tier, model, doc, b0, b1, parent="true", tail=None, kind="store"):
        B = self.B
        toks = doc.blocks[b0:b1].reshape(-1)
        if tail is None:
            tail = int(self.rng.integers(1, B)) if B > 1 and self.rng.random() < 0.3 else 0
        if tail:
            nxt = doc.blocks[b1] if b1 < len(doc) else self._tokens(1)[0]
            toks = np.concatenate([toks, nxt[:tail]])
        if parent == "true":
            par = int(doc.eh[b0 - 1]) if b0 > 0 else None
        elif parent == "none":
            par = None
        else:                                                  # an engine hash nobody stored
            par = int(self.rng.integers(1, 2 ** 63)) * 2
        return Ev(STORED, pod, tier, model, par, doc.eh[b0:b1].copy(), toks, kind)

    def _slice(self, doc, long=False):
        n = len(doc)
        if long and n >= 34:
            ln = int(self.rng.integers(33, n + 1))
        else:
            ln = int(self.rng.integers(1, min(n, 12) + 1))
        b0 = int(self.rng.integers(0, n - ln + 1))
        return b0, b0 + ln

    def _drop(self, pod, tier, model, doc, kind):
        B = self.B
        b0, b1 = self._slice(doc)
        e = self._store(pod, tier, model, doc, b0, b1, tail=0, kind=kind)
        if kind == "drop_more":                                # n_tokens / B above n_hashes
            e.tokens = np.concatenate([e.tokens, self._tokens(1)[0]])
        elif kind == "drop_less":                              # below (a block fewer; at one hash: no full block)
            e.tokens = e.tokens[:len(e.tokens) - B]
        else:                                                  # fewer than B tokens, with hashes
            e.tokens = e.tokens[:int(self.rng.integers(0, B))]
        return e

    def _remove(self, pod, tier, model, doc):
        pool = np.concatenate([doc.eh, np.array(doc.alias, np.uint64)])
        k = int(self.rng.integers(1, min(len(pool), 40) + 1))
        hs = list(self.rng.choice(pool, k, replace=False))
        if self.rng.random() < 0.5:
            hs += list(self.rng.choice(hs, int(self.rng.integers(1, 4))))        # duplicates
        if self.rng.random() < 0.5:
            hs.append(int(self.rng.integers(1, 2 ** 63)) * 2)                     # unknown
        self.rng.shuffle(hs)
        return Ev(REMOVED, pod, tier, model, None, np.array(hs, np.uint64), [], "remove")

    def batch(self, n_events, pod=None):
        """One batch of about n_events events (family "a" with single_queue: all of pod `pod`, or a random pod)."""
        if self.family == "b":
            return self._batch_b(n_events)
        rng = self.rng
        if self.single_queue:
            pods = [pod if pod is not None else self.pods[int(rng.integers(0, len(self.pods)))]]
        else:
            pods = self.pods
        out, recent = [], {p: [] for p in pods}
        while len(out) < n_events:
            p = pods[int(rng.integers(0, len(pods)))]
            tier, model = int(rng.integers(0, self.tiers)), int(rng.integers(0, self.models))
            docs = self._docs_of(p)
            doc = docs[int(rng.integers(0, len(docs)))]
            r = rng.random()
            if r < 0.3 and recent[p]:
                # consumer of a block stored earlier in this batch: at the producer's last block or inside it
                src = recent[p][int(rng.integers(max(0, len(recent[p]) - 4), len(recent[p])))]
                sdoc, s0, s1, smodel = src
                k = s1 - 1 if rng.random() < 0.5 else int(rng.integers(s0, s1))
                if k + 1 < len(sdoc):
                    b1 = int(rng.integers(k + 2, min(len(sdoc), k + 40) + 1))
                    e = self._store(p, tier, smodel if rng.random() < 0.8 else model, sdoc, k + 1, b1, kind="consumer")
                    if rng.random() < 0.15:                    # its parent removed or re-mapped first
                        if rng.random() < 0.5:
                            out.append(Ev(REMOVED, p, int(rng.integers(0, self.tiers)), e.model, None, [sdoc.eh[k]], [], "remove"))
                        else:
                            kk = max(k - int(rng.integers(0, 3)), 0)
                            out.append(self._store(p, tier, e.model, sdoc, kk, k + 1, parent="none", kind="remap"))
                    out.append(e)
                    recent[p].append((sdoc, k + 1, b1, e.model))
                    continue
            if r < 0.5:
                b0, b1 = self._slice(doc, long=rng.random() < 0.3)
                mode = "true" if rng.random() < 0.7 else ("none" if rng.random() < 0.5 else "unknown")
                e = self._store(p, tier, model, doc, b0, b1, parent=mode)
                n = len(e.hashes)
                if n >= 3 and rng.random() < (0.5 if n > 32 else 0.15):   # a repeated engine hash inside the event
                    if n > 32 and rng.random() < 0.5:                     # in another 32-block pass
                        i = int(rng.integers(0, n - 32))
                        j = int(rng.integers(i + 32, n))
                    else:
                        i, j = rng.choice(n, 2, replace=False)
                    e.hashes[j] = e.hashes[i]
                    e.kind = "dup"
                elif rng.random() < 0.1:                       # the same blocks under other engine hashes: two mappings
                    e.hashes = rng.integers(1, 2 ** 63, n, dtype=np.uint64) * np.uint64(2)    # to one request key
                    doc.alias.extend(e.hashes.tolist())
                    e.kind = "alias"
                out.append(e)
                recent[p].append((doc, b0, b1, model))
            elif r < 0.62:
                kind = DROP_KINDS[int(rng.integers(0, 3))]
                e = self._drop(p, tier, model, doc, kind)
                out.append(e)
                if len(e.hashes) and rng.random() < 0.6:        # a consumer of the dropped event's block
                    i = int(np.nonzero(doc.eh == e.hashes[-1])[0][0])
                    if i + 1 < len(doc):
                        out.append(self._store(p, tier, model, doc, i + 1, min(len(doc), i + 1 + int(rng.integers(1, 9))),
                                               kind="after_drop"))
            elif r < 0.67:
                b0, b1 = self._slice(doc)
                e = self._store(p, tier, model, doc, b0, b1)
                e.hashes = e.hashes[:0]                        # n_hashes = 0: skipped, parent lookup still refreshes
                e.kind = "zero_hashes"
                out.append(e)
            else:
                out.append(self._remove(p, tier, model, doc))
        return out

    def _batch_b(self, n_events):
        rng = self.rng
        out, own = [], {p: set() for p in self.pods}
        tries = 0
        while len(out) < n_events and tries < 50 * n_events:
            tries += 1
            p = self.pods[int(rng.integers(0, len(self.pods)))]
            tier, model = int(rng.integers(0, self.tiers)), int(rng.integers(0, self.models))
            doc = self.docs[int(rng.integers(0, len(self.docs)))]
            r = rng.random()
            if r < 0.1:
                out.append(self._drop(p, tier, model, doc, DROP_KINDS[int(rng.integers(0, 3))]))
                continue
            b0, b1 = self._slice(doc, long=rng.random() < 0.3)
            if b0 > 0:
                ph = (model, int(doc.eh[b0 - 1]))
                if ph not in self.resident and ph not in own[p]:
                    continue                                   # its parent would be another queue's in-batch block
            e = self._store(p, tier, model, doc, b0, b1)
            if r < 0.15:
                e.hashes = e.hashes[:0]
                e.kind = "zero_hashes"
            else:
                own[p].update((model, int(h)) for h in e.hashes)
            out.append(e)
        for p in self.pods:
            self.resident |= own[p]
        return out


# ---- expectations ------------------------------------------------------------------------------------------------
def phase1_predictions(co, events, B, init_hash, earliest=False):
    """{event index: the request key phase 1 starts its chain from} for the batch's hashable events, with `co` holding
    the index as it is before the batch.  A producer's keys are computed from its own prediction.  earliest: take the
    first producer instead of the last (a wrong rule, for the self-test)."""
    keys, pred, last = {}, {}, {}
    for i, e in enumerate(events):
        if not e.hashable(B):
            continue
        h = init_hash
        if e.parent is not None:
            src = last.get((e.pod, e.model, e.parent))
            if src is not None:
                h = int(keys[src[0]][src[1]])
            else:
                r = co.peek_request_key(e.model, e.parent)
                h = init_hash if r is None else r
        pred[i] = h
        keys[i], _ = co.hash_keys(e.tokens, np.array([0, len(e.tokens)], np.int64), parent=np.array([h], np.uint64))
        for b, x in enumerate(e.hashes):
            if not earliest or (e.pod, e.model, int(x)) not in last:
                last[(e.pod, e.model, int(x))] = (i, b)
    return pred


def expect_batch(co, events, B, init_hash, phase1):
    """Applies the batch to the oracle in array order (a valid schedule of the per-pod queues) and returns (events
    dropped, events phase 1 mispredicts -- 0 when phase 1 does not run)."""
    pred = phase1_predictions(co, events, B, init_hash) if phase1 else {}
    ev, hs, tk = pack(events)
    dropped = rehashed = 0
    for i, e in enumerate(events):
        if i in pred:
            actual = init_hash
            if e.parent is not None:
                r = co.peek_request_key(e.model, e.parent)
                actual = init_hash if r is None else r
            rehashed += actual != pred[i]
        rc, nd = co.apply_events(ev[i:i + 1], hs, tk)
        assert rc == 0
        dropped += nd
    return dropped, rehashed


def sorted_entries(image):
    """The image with each request record's entries sorted (family "b": their order depends on the schedule)."""
    img = bytearray(image)
    R = struct.unpack_from("<Q", img, 32)[0]
    req = np.frombuffer(img, SNAP_REQ_DTYPE, R, 64).copy()
    for r in req:
        c = int(r["count"])
        r["ent"][:c] = np.sort(r["ent"][:c])
    img[64:64 + 32 * R] = req.tobytes()
    return bytes(img)


def recency_ranks(image):
    """An image whose recency section holds values of any scale -> the same image with each section's values replaced
    by their ranks (1 = oldest), so that a library image (stamps) compares with the oracle's (positions)."""
    R, E = struct.unpack_from("<QQ", image, 32)
    off = 64 + 32 * R + 24 * E
    assert struct.unpack_from("<I", image, 12)[0] & 1 and len(image) == off + 8 * (R + E)
    st = np.frombuffer(image, "<u8", R + E, off)
    ranks = np.zeros(R + E, np.uint64)
    for lo, hi in ((0, R), (R, R + E)):
        ranks[lo + np.argsort(st[lo:hi], kind="stable")] = np.arange(1, hi - lo + 1, dtype=np.uint64)
    return bytes(image[:off]) + ranks.tobytes()
