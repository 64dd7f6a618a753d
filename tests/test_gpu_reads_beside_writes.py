"""GPU (-m gpu): every read path against a writer in flight.  DESIGN §4: a reader sees each key as it was just before or
just after each single Add / Evict / event / removal, never a half-written slot and never a state older than the call.

Reader threads call one read path over and over on handles that one writer thread keeps changing (Add, Evict, event
batches through both write phases and on the device, pod removals, and filler keys whose removal leaves the tombstones
that make the handle rebuild its tables).  Every call records its host-clock interval and its rows; after the threads
stop, the writer's log is replayed on the oracle (tests/history_oracle.py) and every row must be one that some
interleaving of the writer's operations with the call produces.  Each case asserts that the race happened: a read
overlapped every kind of write, the tables were rebuilt under the readers, and keys were contested inside calls.  Then,
with the writer stopped, every handle's rows equal the oracle of its own snapshot, and that snapshot the replayed log.

The workload: 200 documents of 20-100 blocks (walks cross the 32-block round and the 2 KB chunk), most behind one of 8
shared system prompts (prefix classes with followers and partial followers), on two models; an anchor pod on tier 0 of
every block that no writer touches; churn pods 1..8 on tiers weighted 1.0, 0.8, 1/3 and 0.1 (at most 9 churn entries a
key, so the 10-entry pod LRU never drops the anchor); a pod filter on a quarter of the prompts; and a hot document, outside
the prompt pool, whose first 8 blocks one event batch stores and removes 32 times while Lookup reads each of their slots
256 times a call.

Score() from text reads the same documents through a device prefix store that holds their text (4 bytes a token)."""
import threading
import time

import numpy as np
import pytest

import kvidx
import snapshot_oracle as so
from helpers import EVENT_DTYPE, PATHS, SEED_ORDER, SNAP_REQ_DTYPE, _select_path
from history_oracle import Checker, History, Window
from oracle import kvoracle as ko
from oracle.kvoracle_c import COracle
from test_gpu_shard_ops import _shards

pytestmark = pytest.mark.gpu

W = (1.0, 0.8, 1 / 3, 0.1)
P = 16
ANCHOR, FILLER = 0, 9
CHURN = [(p << 4) | (p % 4) for p in range(1, 9)] + [(1 << 4) | 3]      # pod 1 on two tiers: 9 churn entries a key
EMIX = np.uint64(0x5BD1E9955BD1E995)                                     # engine key = request key ^ EMIX


def PT(p, t=0):
    return (p << 4) | t


class Work:
    """Documents, their keys and a pool of prompt specs (doc, blocks, tail tokens, filter)."""

    def __init__(self, seed, BS=16, n_docs=200, n_specs=160, max_blocks=100):
        rng = np.random.default_rng(seed)
        self.BS = BS
        self.co = COracle(block_size=BS, tier_weights=W, max_pods=P)
        sys_p = [rng.integers(0, 128256, BS * int(rng.integers(4, 41))) for _ in range(8)]
        self.docs, self.model = [], []
        for d in range(n_docs):
            n = int(rng.integers(20, max_blocks + 1))
            t = rng.integers(0, 128256, BS * n)
            if d < n_docs * 4 // 5:
                s = sys_p[d % 8][:BS * (n - 2)]
                t[:len(s)] = s
            self.docs.append(t.astype(np.uint32))
            self.model.append((d // 8) % 2)
        self.keys = [self.co.hash_keys(t, [0, len(t)])[0] for t in self.docs]
        self.specs = []
        for _ in range(n_specs):
            d = int(rng.integers(0, n_docs))
            nb = int(rng.integers(1, len(self.keys[d]) + 1)) if rng.random() < 0.6 else len(self.keys[d])
            tail = int(rng.integers(0, BS))
            filt = None
            if rng.random() < 0.25:
                filt = set(int(p) for p in rng.choice(10, size=int(rng.integers(1, 5)), replace=False))
            self.specs.append((d, nb, tail, filt))
        self.fw = (P + 63) // 64
        pool = {d for d, *_ in self.specs}
        self.hot = next(d for d in range(n_docs) if d not in pool)    # a document no prompt and no churn run touches

    def fill_calls(self):
        """The anchor on every block: one Add per model."""
        out = []
        for m in (0, 1):
            ks = np.unique(np.concatenate([k for k, mm in zip(self.keys, self.model) if mm == m]))
            out.append((m, ks ^ EMIX, ks, [PT(ANCHOR)]))
        return out

    def fill(self, ix):
        for call in self.fill_calls():
            assert ix.add(*call) == 0

    def batch(self, rng, n, max_blocks=None):
        """n prompts drawn from the pool -> (spec index per prompt, tokens, offsets, models, filter rows)."""
        idx = rng.integers(0, len(self.specs), n)
        toks, lens = [], np.zeros(n, np.int64)
        for i, s in enumerate(idx):
            d, nb, tail, _ = self.specs[s]
            if max_blocks is not None:
                nb = min(nb, max_blocks)
            t = self.docs[d][:self.BS * nb + tail]
            toks.append(t)
            lens[i] = len(t)
        off = np.zeros(n + 1, np.int64)
        off[1:] = np.cumsum(lens)
        model = np.array([self.model[self.specs[s][0]] for s in idx], np.uint32)
        fm = np.zeros((n, self.fw), np.uint64)
        for i, s in enumerate(idx):
            for p in self.specs[s][3] or ():
                fm[i, p // 64] |= np.uint64(1) << np.uint64(p % 64)
        return idx, np.concatenate(toks), off, model, fm

    def spec_keys(self, s, max_blocks=None):
        d, nb, _, filt = self.specs[s]
        if max_blocks is not None:
            nb = min(nb, max_blocks)
        return self.model[d], self.keys[d][:nb], filt


class Writer:
    """One writer thread applying every op to each of its handles in turn; ops[h][i] is op i's interval on handle h."""

    def __init__(self, work, handles, rng, kinds, remove=None, dev_read=None):
        self.w, self.handles, self.rng, self.kinds = work, handles, rng, kinds
        self.log = []
        self.ops = [[(0, 0, "fill", False)] for _ in handles]     # per handle: (t0, t1, kind, rebuilt); op 0 is the fill
        self.remove = remove or (lambda ix, pods: ix.remove_pods(pods))
        self.keep = []                                    # device buffers of asynchronous batches
        self.dev_read = dev_read                          # (h, writer) -> None: a _dev read queued right behind a _dev batch
        self.errs = []

    def _churn_run(self):
        """A run of blocks [a, b) of a document of the prompt pool; half of them start at block 0, where a pod's score
        starts."""
        d = self.w.specs[int(self.rng.integers(0, len(self.w.specs)))][0]
        k = self.w.keys[d]
        a = 0 if self.rng.random() < 0.5 else int(self.rng.integers(0, len(k)))
        b = int(self.rng.integers(a + 1, min(len(k), a + 40) + 1))
        return d, a, b

    def _events(self, n_runs):
        """One pod's batch: per run, its blocks stored under their parent (tokens and parent hash), then up to 3 of them
        removed (a removal inside a run that starts at block 0 cuts the pod's score)."""
        pt = CHURN[int(self.rng.integers(0, len(CHURN)))]
        BS = self.w.BS
        evs, hs, tks = [], [], []
        ho = to = 0
        for _ in range(n_runs):
            d, a, b = self._churn_run()
            k, m = self.w.keys[d], self.w.model[d]
            rm = self.rng.choice(np.arange(a, b), size=min(3, b - a), replace=False)
            ev = np.zeros(2, EVENT_DTYPE)
            ev["podtier"], ev["model"] = pt, m
            ev[0]["op"], ev[0]["n_hashes"], ev[0]["n_tokens"], ev[0]["hash_off"], ev[0]["tok_off"] = 0, b - a, BS * (b - a), ho, to
            ev[0]["has_parent"], ev[0]["parent_hash"] = a > 0, int(k[a - 1] ^ EMIX) if a > 0 else 0
            ev[1]["op"], ev[1]["n_hashes"], ev[1]["hash_off"] = 1, len(rm), ho + b - a
            evs.append(ev)
            hs.append(np.concatenate([k[a:b] ^ EMIX, k[rm] ^ EMIX]).astype(np.uint64))
            tks.append(self.w.docs[d][BS * a:BS * b])
            ho += len(hs[-1])
            to += len(tks[-1])
        return np.concatenate(evs), np.concatenate(hs), np.concatenate(tks)

    def _hot(self):
        """64 events of one pod that store and remove the first 8 blocks of the hot document in turn: its slots are
        republished back to back for the whole batch, and each removal shifts the count of an image whose entries 0..3
        change with it (a reader that kept half of one image and half of the next would see it)."""
        pt = CHURN[int(self.rng.integers(0, len(CHURN)))]
        d, BS = self.w.hot, self.w.BS
        k, m = self.w.keys[d][:8], self.w.model[d]
        ev = np.zeros(64, EVENT_DTYPE)
        ev["podtier"], ev["model"], ev["n_hashes"] = pt, m, 8
        ev["op"][1::2] = 1
        ev["n_tokens"][0::2] = 8 * BS
        return ev, (k ^ EMIX).astype(np.uint64), self.w.docs[d][:8 * BS]

    def next_op(self):
        kind = self.kinds[len(self.log) % len(self.kinds)]
        rng = self.rng
        if kind == "add":
            d, a, b = self._churn_run()
            pts = [CHURN[int(i)] for i in rng.choice(len(CHURN), size=int(rng.integers(1, 3)), replace=False)]
            return kind, (self.w.model[d], self.w.keys[d][a:b] ^ EMIX, self.w.keys[d][a:b], pts)
        if kind == "evict":
            d, a, _ = self._churn_run()
            return kind, (self.w.model[d], int(self.w.keys[d][a] ^ EMIX), [CHURN[int(rng.integers(0, len(CHURN)))]])
        if kind == "apply_events":
            return kind, self._events(2)
        if kind == "apply_events_dev":
            return kind, self._events(16)
        if kind == "hot":
            return kind, self._hot()
        if kind == "remove_pods":
            return kind, ([int(rng.integers(1, 9))],)
        if kind == "filler":                              # keys of the filler pod only: their removal leaves tombstones
            ks = rng.integers(1, 1 << 63, 9000, dtype=np.uint64)
            return kind, (int(rng.integers(0, 2)), ks ^ EMIX, ks, [PT(FILLER)])
        if kind == "remove_filler":
            return kind, ([FILLER],)
        raise AssertionError(kind)

    def _apply(self, h, ix, kind, args):
        if kind in ("add", "filler"):
            assert ix.add(*args) == 0, ix.last_error()
        elif kind == "evict":
            assert ix.evict(*args) == 0
        elif kind in ("apply_events", "hot"):
            assert ix.apply_events(*args) == (0, 0)
        elif kind == "apply_events_dev":
            import torch
            ev, hs, tk = args
            dev = torch.device("cuda", 0)
            bufs = [torch.from_numpy(ev.view(np.uint8).copy()).to(dev), torch.tensor([0, len(ev)], dtype=torch.int64, device=dev),
                    torch.from_numpy(hs.view(np.int64).copy()).to(dev), torch.from_numpy(tk.view(np.int32).copy()).to(dev)]
            torch.cuda.synchronize()
            self.keep.append(bufs)
            ix.apply_events_dev(bufs[0].data_ptr(), bufs[1].data_ptr(), 1, len(ev), bufs[2].data_ptr(), len(hs), bufs[3].data_ptr())
        elif kind in ("remove_pods", "remove_filler"):
            self.remove(ix, *args)

    def run(self, stop):
        try:
            while not stop.is_set():
                kind, args = self.next_op()
                for h, ix in enumerate(self.handles):
                    r0 = ix.stats()["rebuilds"]
                    t0 = time.monotonic_ns()
                    self._apply(h, ix, kind, args)
                    t1 = time.monotonic_ns()
                    if kind == "apply_events_dev" and self.dev_read is not None:
                        self.dev_read(h, self)                # before anything waits for the batch
                    self.ops[h].append((t0, t1, kind, ix.stats()["rebuilds"] > r0))
                self.log.append((kind, args))
        except Exception as ex:                           # noqa: BLE001
            self.errs.append(ex)
            stop.set()

    def history(self, work, clock=False):
        h = History(COracle(block_size=work.BS, tier_weights=W, max_pods=P), clock=clock)
        h.fill(work.fill_calls())
        for kind, args in self.log:
            if kind in ("filler", "remove_filler"):       # filler keys: no read looks at them
                h.skip(kind)
            elif kind == "add":
                h.add(*args)
            elif kind == "evict":
                h.evict(*args)
            elif kind in ("apply_events", "apply_events_dev", "hot"):
                h.apply_events(*args, kind=kind)
            else:
                h.remove_pods(*args)
            h.kinds[-1] = kind
        return h

    def op_times(self, h):
        return np.array([o[:2] for o in self.ops[h][:len(self.log) + 1]], np.int64).reshape(-1, 2)

    def seen(self, h, s, e, ev):
        """While the race runs: add to ev the kinds (and rebuilds) of the ops on handle h that overlapped [s, e] and have
        returned.  Evidence only -- the check after the race is the authority."""
        ops = self.ops[h]
        for i in range(len(ops) - 1, 0, -1):
            t0, t1, kind, rebuilt = ops[i]
            if t1 <= s:
                break
            if t0 < e:
                ev["kinds"].add(kind)
                ev["rebuild"] |= rebuilt


def _race(work, writer, readers, budget_s):
    """Run the writer and the readers for budget_s at most (readers stop on their own when they have what they need).
    readers: callables (stop) -> None.  Joins everything with a timeout that fails the test."""
    stop = threading.Event()
    wt = threading.Thread(target=writer.run, args=(stop,), daemon=True)
    errs = []

    def guard(fn):
        try:
            fn(stop)
        except Exception as ex:                           # noqa: BLE001
            errs.append(ex)
            stop.set()

    rts = [threading.Thread(target=guard, args=(r,), daemon=True) for r in readers]
    wt.start()
    time.sleep(0.05)
    for t in rts:
        t.start()
    deadline = time.monotonic() + budget_s
    for t in rts:
        t.join(max(0.0, deadline - time.monotonic()) + 30.0)
        assert not t.is_alive(), "a reader did not finish within %.0f s" % (budget_s + 30)
    stop.set()
    wt.join(60.0)
    assert not wt.is_alive(), "the writer did not stop within 60 s"
    assert not writer.errs, writer.errs[:1]
    assert not errs, errs[:2]
    for ix in writer.handles:
        ix.synchronize()


class Reads:
    """Recorded read calls: (kind, handle, s, e, payload)."""

    def __init__(self):
        self.calls = []
        self.lock = threading.Lock()

    def add(self, *rec):
        with self.lock:
            self.calls.append(rec)


class Until:
    """When a reader of handle h may stop: after `calls` calls, once the calls it made overlapped every op kind in `kinds`
    (and a rebuild, with `rebuild`), or after `cap` calls."""

    def __init__(self, writer, h, calls, kinds, rebuild=False, cap=40):
        self.writer, self.h, self.calls, self.cap = writer, h, calls, cap
        self.kinds, self.rebuild = set(kinds), rebuild
        self.ev = {"kinds": set(), "rebuild": False}
        self.k = 0

    def more(self):
        if self.k >= self.cap:
            return False
        return self.k < self.calls or not self.kinds <= self.ev["kinds"] or (self.rebuild and not self.ev["rebuild"])

    def saw(self, s, e):
        self.k += 1
        self.writer.seen(self.h, s, e, self.ev)


def _score_reader(work, ix, h, reads, rng, n, until, how="dense", max_blocks=None):
    """A reader that scores batches of n prompts from the pool on handle ix (how: dense / sparse / pinned1 / pageable1)
    as long as `until` asks for more."""
    pinned = kvidx.pinned_array((work.BS * 128,), np.uint32) if how == "pinned1" else None
    batches = [work.batch(rng, n, max_blocks) for _ in range(4 if n > 1 else 64)]     # made before the race

    def run(stop):
        while until.more() and not stop.is_set():
            idx, tok, off, model, fm = batches[until.k % len(batches)]
            if how == "pinned1":
                pinned[:len(tok)] = tok
                tok = pinned[:len(tok)]
            s = time.monotonic_ns()
            if how == "sparse":
                pods, sc, cnt, has = ix.score_batch_sparse(tok, off, model=model, filter_mask=fm)
                e = time.monotonic_ns()
                rows = np.full((n, P), -1.0)
                for i in range(n):
                    rows[i, pods[i, :cnt[i]]] = sc[i, :cnt[i]]
                    assert len(set(pods[i, :cnt[i]].tolist())) == cnt[i], "a sparse row repeats a pod"
            else:
                rows, has = ix.score_batch(tok, off, model=model, filter_mask=fm)
                e = time.monotonic_ns()
            reads.add("score", h, s, e, (idx, rows, has, max_blocks))
            until.saw(s, e)
    return run


def _check_scores(work, writer, hist, reads, ck, evidence):
    """Every recorded score row admissible; fills evidence (per handle: op kinds overlapped, contested keys)."""
    for kind, h, s, e, payload in reads.calls:
        w = Window(writer.op_times(h), s, e)
        ev = evidence.setdefault(h, {"kinds": set(), "contested": 0, "rebuild": False, "calls": 0})
        ev["calls"] += 1
        ev["kinds"] |= {hist.kinds[i] for i in w.overlapped()}
        ev["rebuild"] |= any(writer.ops[h][i][3] for i in w.overlapped())
        if kind != "score":
            continue
        idx, rows, has, mb = payload
        memo = {}
        for spec in np.unique(idx):
            model, keys, filt = work.spec_keys(int(spec), mb)
            sets = ck.score_sets(model, keys, w, filt, memo)
            if filt is None or ANCHOR in filt:
                assert sets[0][0] == {float(len(keys))}, "the anchor must score exactly"
            sel = np.flatnonzero(idx == spec)
            for r in np.unique(np.concatenate([rows[sel], has[sel, None].astype(np.float64)], axis=1), axis=0):
                why = ck.row_ok(r[:P], int(r[P]), sets)
                assert why is None, "handle %d, call [%d, %d], spec %d (doc %d, %d blocks): %s" % (
                    h, s, e, spec, work.specs[spec][0], len(keys), why)
            if ev["contested"] < 1:
                ev["contested"] += sum(len(hist.req_states((model, int(k)), w)) > 1 for k in keys)


def _quiescent(work, hist, handles, clock=False, snapshot=True):
    """Writer stopped: each handle's snapshot equals the replayed log (not on CLOCK handles, whose sweep the log does not
    model), and every handle scores every pool prompt exactly as the oracle of its own snapshot (snapshot False: as the
    replayed log, for the ranks of a sharded index)."""
    idx = np.arange(len(work.specs))
    toks = [work.docs[d][:work.BS * nb + t] for d, nb, t, _ in work.specs]
    off = np.zeros(len(toks) + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in toks])
    tok = np.concatenate(toks)
    model = np.array([work.model[d] for d, *_ in work.specs], np.uint32)
    fm = np.zeros((len(toks), work.fw), np.uint64)
    for i, (_, _, _, filt) in enumerate(work.specs):
        for p in filt or ():
            fm[i, p // 64] |= np.uint64(1) << np.uint64(p % 64)
    sc = ko.LongestPrefixScorer(dict(enumerate(W)))
    for ix in handles:
        oix = hist.ix
        if snapshot:
            img = ix.snapshot()
            oix = so.decode(img, [0, 1], list(range(P)), list(range(16)), max_pods=P)[0]
        if snapshot and not clock:
            R = int(np.frombuffer(img, "<u8", 1, 32)[0])
            req = np.frombuffer(img, SNAP_REQ_DTYPE, R, 64)
            got = {(int(r["model"]), int(r["hash"])): tuple(int(x) for x in r["ent"][:r["count"]]) for r in req
                   if any(x >> 4 != FILLER for x in r["ent"][:r["count"]])}
            for key in hist.req:
                want = hist.state_at(key, hist.n_ops)
                assert got.pop(key, None) == want, key
            assert not got, "keys the writer never wrote: %d" % len(got)
        want = np.full((len(toks), P), -1.0)
        for i in idx:
            m, keys, filt = work.spec_keys(int(i))
            keys = [ko.Key(m, int(k)) for k in keys]
            for p, v in sc.score(keys, oix.lookup(keys, filt or ())).items():
                want[i, p] = v
        rows, has = ix.score_batch(tok, off, model=model, filter_mask=fm)
        assert np.array_equal(rows, want) and has.all()


def _handle(work, monkeypatch=None, path=None, **kw):
    cfg = dict(block_size=work.BS, capacity=8192, table_slots=1 << 15, tier_weights=W, max_pods=P)
    cfg.update(kw)
    if path is None:
        ix = kvidx.Index(**cfg)
    else:
        with monkeypatch.context() as mp:
            _select_path(mp, path)
            ix = kvidx.Index(**cfg)
    work.fill(ix)
    return ix


KINDS = ["add", "evict", "apply_events", "apply_events_dev", "remove_pods"]
ALL_KINDS = ["add", "evict", "apply_events", "filler", "add", "apply_events_dev", "evict", "remove_pods", "add",
             "remove_filler", "hot"]


def _evidence_ok(evidence, n_handles, kinds, rebuilds=True):
    for h in range(n_handles):
        ev = evidence.get(h)
        assert ev is not None, "handle %d was never read" % h
        assert set(kinds) <= ev["kinds"], "handle %d: no read overlapped %s" % (h, sorted(set(kinds) - ev["kinds"]))
        assert ev["contested"] > 0, "handle %d: no key had two admissible states inside a call" % h
        if rebuilds:
            assert ev["rebuild"], "handle %d: no read overlapped a rebuild (%s)" % (h, ev)


# the groups as they were cut from helpers.SEED_ORDER, so that each path keeps its group and the group's seeds
GROUPS = [[p for p in SEED_ORDER[i::4] if p in PATHS] for i in range(4)]


@pytest.mark.parametrize("group", range(4))
def test_every_score_path_beside_the_writer(group, monkeypatch):
    """Each Score() path of the library (helpers.PATHS, a handle each) scores 4096-prompt batches while the writer runs
    every kind of write on all of them."""
    paths = GROUPS[group]
    work = Work(11 + group)
    handles = [_handle(work, monkeypatch, p) for p in paths]
    rb0 = [ix.stats()["rebuilds"] for ix in handles]
    writer = Writer(work, handles, np.random.default_rng(group), ALL_KINDS)
    reads = Reads()
    rng = [np.random.default_rng(100 + h) for h in range(len(handles))]
    # a fast path makes dozens of calls before the writer's cycle has reached every kind on its handle: it reads on until then
    readers = [_score_reader(work, ix, h, reads, rng[h], 4096, Until(writer, h, 3, KINDS, rebuild=True, cap=400))
               for h, ix in enumerate(handles)]
    _race(work, writer, readers, 40)
    hist = writer.history(work)
    evidence = {}
    _check_scores(work, writer, hist, reads, Checker(hist, W), evidence)
    _evidence_ok(evidence, len(handles), KINDS)
    assert all(ix.stats()["rebuilds"] > r for ix, r in zip(handles, rb0))
    _quiescent(work, hist, handles)


@pytest.mark.parametrize("phase1", ["1", "0"])
def test_host_buffers_dev_calls_and_lookups_beside_the_writer(phase1, monkeypatch):
    """One handle per write phase: dense and sparse rows, batch-1 calls from pinned (zero-copy) and pageable memory, _dev
    calls queued several at a time before one synchronize (across rebuilds, and right behind the writer's own _dev
    batches), Lookup of 2048 keys and GetRequestKey."""
    import torch
    monkeypatch.setenv("KVIDX_WRITE_PHASE1", phase1)
    work = Work(21)
    ix = _handle(work)
    monkeypatch.delenv("KVIDX_WRITE_PHASE1")
    rb0 = ix.stats()["rebuilds"]
    reads = Reads()
    dev = torch.device("cuda", 0)
    state = {"across": False, "behind": 0}

    # device-resident inputs made before the race (no copy or synchronisation of the device while it runs); each call
    # gets fresh result buffers, which every call writes in full
    def dev_inputs(rng, n):
        idx, tok, off, model, fm = work.batch(rng, n)
        return idx, n, [torch.from_numpy(x).to(dev) for x in (tok.view(np.int32), off, model.view(np.int32), fm.view(np.int64))]

    inputs = {n: [dev_inputs(np.random.default_rng(n + i), n) for i in range(4)] for n in (1024, 2048)}
    torch.cuda.synchronize()

    def dev_batch(rng, n):
        idx, n, b = inputs[n][int(rng.integers(0, 4))]
        return idx, b + [torch.empty((n, P), dtype=torch.float64, device=dev), torch.empty(n, dtype=torch.uint8, device=dev)]

    def queue(b, n):
        ix.score_batch_dev(b[0].data_ptr(), b[1].data_ptr(), n, b[4].data_ptr(), d_model=b[2].data_ptr(),
                           d_filter=b[3].data_ptr(), d_has_keys=b[5].data_ptr())

    def behind(h, wr):
        """Queued by the writer right after its _dev batch returned: ordered after the batch (ev_write)."""
        if state["behind"] >= 6:
            return
        idx, b = dev_batch(wr.rng, 1024)
        s = time.monotonic_ns()
        queue(b, 1024)
        ix.synchronize()
        e = time.monotonic_ns()
        reads.add("score", h, s, e, (idx, b[4].cpu().numpy(), b[5].cpu().numpy(), None))
        state["behind"] += 1

    writer = Writer(work, [ix], np.random.default_rng(5), ALL_KINDS, dev_read=behind)

    def dev_reader(stop):
        rng = np.random.default_rng(7)
        k = 0
        while (k < 6 or not state["across"]) and k < 40 and not stop.is_set():
            batches = [dev_batch(rng, 2048) for _ in range(3)]
            r0 = ix.stats()["rebuilds"]
            s = time.monotonic_ns()
            for _, b in batches:
                queue(b, 2048)
            time.sleep(0.02)
            ix.synchronize()
            e = time.monotonic_ns()
            state["across"] |= ix.stats()["rebuilds"] > r0
            for idx, b in batches:
                reads.add("score", 0, s, e, (idx, b[4].cpu().numpy(), b[5].cpu().numpy(), None))
            k += 1

    def lookup_reader(stop):
        """Lookup of 2048 keys: of random documents, or the hot document's 8 keys 256 times each (every call then reads
        each of those slots while the writer may be republishing it); GetRequestKey of a few engine keys."""
        rng = np.random.default_rng(8)
        until = Until(writer, 0, 16, ["hot"], cap=400)
        hot = np.tile(work.keys[work.hot][:8], 256)
        while until.more() and not stop.is_set():
            if until.k % 4 == 0:
                m = int(rng.integers(0, 2))
                d = [i for i in rng.integers(0, len(work.docs), 64) if work.model[i] == m]
                keys = np.concatenate([work.keys[i] for i in d])[:2048]
            else:
                m, keys = work.model[work.hot], hot
            filt = None if rng.random() < 0.75 else {0, 1, 2, 3, 9}
            fm = None if filt is None else np.array([sum(1 << p for p in filt)], np.uint64)
            s = time.monotonic_ns()
            rc, pt, cnt = ix.lookup(m, keys, fm)
            e = time.monotonic_ns()
            assert rc == 0
            reads.add("lookup", 0, s, e, (m, keys, pt, cnt, filt))
            until.saw(s, e)
            for x in keys[rng.integers(0, len(keys), 2)] ^ EMIX:
                s = time.monotonic_ns()
                rc, v = ix.get_request_key(m, int(x))
                e = time.monotonic_ns()
                reads.add("reqkey", 0, s, e, (m, int(x), rc, v))

    readers = [_score_reader(work, ix, 0, reads, np.random.default_rng(1), 4096, Until(writer, 0, 3, KINDS, rebuild=True)),
               _score_reader(work, ix, 0, reads, np.random.default_rng(2), 4096, Until(writer, 0, 3, KINDS), how="sparse"),
               _score_reader(work, ix, 0, reads, np.random.default_rng(3), 1, Until(writer, 0, 50, KINDS, cap=400), how="pinned1"),
               _score_reader(work, ix, 0, reads, np.random.default_rng(4), 1, Until(writer, 0, 50, KINDS, cap=400), how="pageable1"),
               dev_reader, lookup_reader]
    _race(work, writer, readers, 40)
    hist = writer.history(work)
    ck = Checker(hist, W)
    evidence = {}
    _check_scores(work, writer, hist, reads, ck, evidence)
    for kind, h, s, e, payload in reads.calls:
        w = Window(writer.op_times(0), s, e)
        if kind == "lookup":
            m, keys, pt, cnt, filt = payload
            why = ck.lookup_ok(m, keys, pt, cnt, w, filt)
            assert why is None, "lookup [%d, %d]: %s" % (s, e, why)
        elif kind == "reqkey":
            m, x, rc, v = payload
            why = ck.request_key_ok(m, x, rc, v, w)
            assert why is None, why
    _evidence_ok(evidence, 1, KINDS)
    assert state["across"], "no group of queued _dev calls spanned a rebuild"
    assert state["behind"] > 0
    assert ix.stats()["rebuilds"] > rb0
    _quiescent(work, hist, [ix])


def test_default_dispatch_at_131072_prompts_beside_the_writer():
    """The library's own choice (no knob) at 131 072 prompts -- the class pipeline -- while the writer runs."""
    work = Work(31)
    ix = _handle(work)
    writer = Writer(work, [ix], np.random.default_rng(9), ALL_KINDS)
    reads = Reads()
    until = Until(writer, 0, 2, ["add"], cap=3)
    _race(work, writer, [_score_reader(work, ix, 0, reads, np.random.default_rng(10), 131072, until, max_blocks=40)], 40)
    hist = writer.history(work)
    evidence = {}
    _check_scores(work, writer, hist, reads, Checker(hist, W), evidence)
    _evidence_ok(evidence, 1, [], rebuilds=False)
    assert len(evidence[0]["kinds"]) >= 2, evidence[0]["kinds"]
    _quiescent(work, hist, [ix])


@pytest.mark.parametrize("bs", [16, 64])
def test_score_keys_and_score_turn_beside_the_writer(bs):
    """Score() from request keys and for a conversation turn (held keys, then the new turn's tokens) at 16- and 64-token
    blocks while the writer runs; the new turn's keys are the document's."""
    work = Work(41, BS=bs, max_blocks=60 if bs == 64 else 100)
    ix = _handle(work)
    writer = Writer(work, [ix], np.random.default_rng(12), ALL_KINDS)
    reads = Reads()

    def keys_reader(turn, seed):
        until = Until(writer, 0, 3, ["add", "evict", "apply_events", "remove_pods"])

        def run(stop):
            rng = np.random.default_rng(seed)
            while until.more() and not stop.is_set():
                idx = rng.integers(0, len(work.specs), 4096)
                model = np.array([work.spec_keys(int(s))[0] for s in idx], np.uint32)
                fm = np.zeros((len(idx), work.fw), np.uint64)
                for i, s in enumerate(idx):
                    for p in work.spec_keys(int(s))[2] or ():
                        fm[i, 0] |= np.uint64(1) << np.uint64(p)
                ks = [work.spec_keys(int(s))[1] for s in idx]
                held = [len(k) // 2 if turn else len(k) for k in ks]
                koff = np.zeros(len(idx) + 1, np.int64)
                koff[1:] = np.cumsum(held)
                keys = np.concatenate([k[:h] for k, h in zip(ks, held)])
                if turn:
                    toks = [work.docs[work.specs[s][0]][bs * h:bs * len(k)] for s, k, h in zip(idx, ks, held)]
                    toff = np.zeros(len(idx) + 1, np.int64)
                    toff[1:] = np.cumsum([len(t) for t in toks])
                    s0 = time.monotonic_ns()
                    rows, has, nk, noff = ix.score_turn(keys, koff, np.concatenate(toks), toff, model=model, filter_mask=fm)
                    e0 = time.monotonic_ns()
                    assert np.array_equal(nk, np.concatenate([k[h:] for k, h in zip(ks, held)])), "new-turn keys"
                else:
                    s0 = time.monotonic_ns()
                    rows, has = ix.score_keys(keys, koff, model=model, filter_mask=fm)
                    e0 = time.monotonic_ns()
                reads.add("score", 0, s0, e0, (idx, rows, has, None))
                until.saw(s0, e0)
        return run

    _race(work, writer, [keys_reader(False, 1), keys_reader(True, 2)], 40)
    hist = writer.history(work)
    evidence = {}
    _check_scores(work, writer, hist, reads, Checker(hist, W), evidence)
    _evidence_ok(evidence, 1, ["add", "evict", "apply_events", "remove_pods"], rebuilds=False)
    _quiescent(work, hist, [ix])


@pytest.mark.parametrize("peer_pair", [0, 1])
def test_two_shards_beside_the_writer(peer_pair, monkeypatch):
    """A two-shard index on one GPU: readers on both ranks probe the peer's shard while the writer stores, evicts and
    removes (collectively) through rank 0.  A sharded index compacts only collectively with no reader in flight, so
    there are no filler keys here."""
    monkeypatch.setenv("KVIDX_PEER_PAIR", str(peer_pair))
    work = Work(51 + peer_pair)
    sh = _shards(2, block_size=16, hash_seed="", capacity=1 << 15, pods_per_key=10, tier_weights=W, max_pods=P)
    work.fill(sh[0])

    def remove(ix, pods):
        for phase in (0, 1):
            for s in sh:
                s.shard_remove_pods(pods, phase=phase)

    writer = Writer(work, [sh[0]], np.random.default_rng(13), ["add", "evict", "apply_events", "add", "remove_pods"],
                    remove=remove)
    reads = Reads()
    kinds = ["add", "evict", "apply_events", "remove_pods"]
    readers = [_score_reader(work, sh[r], 0, reads, np.random.default_rng(20 + r), 4096, Until(writer, 0, 3, kinds)) for r in (0, 1)]
    _race(work, writer, readers, 40)
    hist = writer.history(work)
    evidence = {}
    _check_scores(work, writer, hist, reads, Checker(hist, W), evidence)
    _evidence_ok(evidence, 1, ["add", "evict", "apply_events", "remove_pods"], rebuilds=False)
    _quiescent(work, hist, sh, snapshot=False)


def test_clock_handle_below_its_contents_beside_the_writer():
    """CLOCK key cap below the documents' keys: the sweep drops keys under the readers (a key may be absent, or re-added
    with its newest entries only), so every suffix of an admissible state is admissible and the anchor is not exact."""
    work = Work(61)
    ix = kvidx.Index(block_size=16, capacity=4096, table_slots=1 << 15, tier_weights=W, max_pods=P, evict_policy="clock")
    work.fill(ix)
    sw0 = ix.sweeps()[0]
    writer = Writer(work, [ix], np.random.default_rng(14), ["add", "add", "remove_pods"])
    reads = Reads()
    readers = [_score_reader(work, ix, 0, reads, np.random.default_rng(30 + r), 4096, Until(writer, 0, 3, ["add", "remove_pods"]))
               for r in (0, 1)]
    _race(work, writer, readers, 40)
    assert ix.sweeps()[0] > sw0, "the CLOCK sweep never ran"
    hist = writer.history(work, clock=True)
    ck = Checker(hist, W)
    times = writer.op_times(0)
    evidence = {"kinds": set(), "contested": 0}
    for kind, h, s, e, (idx, rows, has, mb) in reads.calls:
        w = Window(times, s, e)
        evidence["kinds"] |= {hist.kinds[i] for i in w.overlapped()}
        memo = {}
        for spec in np.unique(idx):
            model, keys, filt = work.spec_keys(int(spec))
            sets = ck.score_sets(model, keys, w, filt, memo)
            for i in np.flatnonzero(idx == spec)[:4]:
                why = ck.row_ok(rows[i], has[i], sets)
                assert why is None, "spec %d: %s" % (spec, why)
    assert {"add", "remove_pods"} <= evidence["kinds"]
    _quiescent(work, hist, [ix], clock=True)


def test_score_text_beside_the_writer():
    """Score() from text -- dense, sparse and _dev at 4096 prompts, dense at 131 072 -- while the writer runs, and a store
    thread adds and finds text disjoint from the queried prompts (its calls serialise with the readers' on the store's
    lock).  Every document's text is in the store before the race (4 bytes a token, 64-byte blocks: one store block per
    index block) and the cache evicts nothing, so each prompt's find is exactly its whole index blocks: the history
    oracle checks the rows as it checks score_batch rows."""
    import torch
    from kvidx import pack_text
    from kvidx.host import PrefixStore
    from test_gpu_text_store import host_find
    from test_gpu_text_store_scale import _text_of
    work = Work(71)
    ix = _handle(work)
    ix.text_store_init(1 << 22, 64)
    hs = PrefixStore(1 << 22, 64)
    dtext = [_text_of(d) for d in work.docs]
    spans = [np.stack([np.arange(len(d)) * 4, np.arange(len(d)) * 4 + 4], axis=1).astype(np.uint64) for d in work.docs]
    t, o = pack_text(dtext)
    ix.text_store_add(t, o, np.concatenate(work.docs), np.concatenate(spans), np.concatenate([[0], np.cumsum([len(d) for d in work.docs])]))
    for x, d, sp in zip(dtext, work.docs, spans):
        hs.add_tokenization(x, d, sp)
    reads = Reads()
    writer = Writer(work, [ix], np.random.default_rng(15), ALL_KINDS)
    dev = torch.device("cuda", 0)
    readers_left = [4]
    lock = threading.Lock()

    def prompt_text(s, mb):
        d, nb, tail, _ = work.specs[s]
        nb = nb if mb is None else min(nb, mb)
        return dtext[d][:4 * (work.BS * nb + tail)], nb

    def text_reader(how, n, until, seed, max_blocks=None):
        rng = np.random.default_rng(seed)
        batches = []
        for _ in range(2 if n > 4096 else 4):
            idx, _, _, model, fm = work.batch(rng, n, max_blocks)
            q, nb = zip(*[prompt_text(int(s), max_blocks) for s in idx])
            text, off = pack_text(q)
            ratio = (np.array(nb, np.int64) * 64).astype(np.float64) / (off[1:] - off[:-1]).astype(np.float64)
            if n <= 4096:                                       # the host store's find: the prompt's whole index blocks
                ftok, foff, fr = host_find(hs, q)
                assert np.array_equal(foff[1:] - foff[:-1], np.array(nb) * work.BS) and fr.tobytes() == ratio.tobytes()
            d_in = [torch.from_numpy(x).to(dev) for x in (text.copy(), off, model.view(np.int32), fm.view(np.int64))] if how == "dev" else None
            batches.append((idx, text, off, model, fm, ratio, d_in))
        torch.cuda.synchronize()

        def run(stop):
            try:
                while until.more() and not stop.is_set():
                    idx, text, off, model, fm, ratio, d_in = batches[until.k % len(batches)]
                    s = time.monotonic_ns()
                    if how == "dense":
                        rows, has, tz, r = ix.score_text(text, off, model=model, filter_mask=fm, min_ratio=0.0)
                        e = time.monotonic_ns()
                    elif how == "sparse":
                        pods, sc, cnt, has, tz, r = ix.score_text_sparse(text, off, model=model, filter_mask=fm, min_ratio=0.0)
                        e = time.monotonic_ns()
                        rows = np.full((n, P), -1.0)
                        for i in range(n):
                            rows[i, pods[i, :cnt[i]]] = sc[i, :cnt[i]]
                    else:
                        out = [torch.empty((n, P), dtype=torch.float64, device=dev), torch.empty(n, dtype=torch.uint8, device=dev),
                               torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.float64, device=dev)]
                        ix.score_text_dev(d_in[0].data_ptr(), d_in[1].data_ptr(), n, out[0].data_ptr(), d_model=d_in[2].data_ptr(),
                                          d_filter=d_in[3].data_ptr(), min_ratio=0.0, d_has_keys=out[1].data_ptr(),
                                          d_tokenize=out[2].data_ptr(), d_ratio=out[3].data_ptr())
                        ix.synchronize()
                        e = time.monotonic_ns()
                        rows, has, tz, r = (x.cpu().numpy() for x in out)
                    assert not tz.any() and r.tobytes() == ratio.tobytes(), "a queried prompt's find changed"
                    reads.add("score", 0, s, e, (idx, rows, has, max_blocks))
                    until.saw(s, e)
            finally:
                with lock:
                    readers_left[0] -= 1
        return run

    store_calls = []

    def store_thread(stop):
        """adds and finds of random text (no block of it is a document's) until the text readers are done, two calls at least"""
        rng = np.random.default_rng(16)
        k = 0
        while (readers_left[0] > 0 or k < 2) and not stop.is_set():
            ps = [rng.bytes(int(rng.integers(0, 900))) for _ in range(512)]
            text, off = pack_text(ps)
            s = time.monotonic_ns()
            if k % 2 == 0:
                toks = [(rng.integers(0, 1 << 31, len(p) // 8 + 1), [(min(8 * j, len(p)), min(8 * j + 8, len(p))) for j in range(len(p) // 8 + 1)]) for p in ps]
                toff = np.concatenate([[0], np.cumsum([len(x[0]) for x in toks])])
                ix.text_store_add(text, off, np.concatenate([x[0] for x in toks]), np.array([sp for x in toks for sp in x[1]], np.uint64), toff)
                for p, (ti, ts) in zip(ps, toks):
                    hs.add_tokenization(p, ti, ts)
            else:
                got, want = ix.text_store_find(text, off), host_find(hs, ps)
                assert all(np.array_equal(g, w) for g, w in zip(got, want)) and got[2].tobytes() == want[2].tobytes()
            store_calls.append((s, time.monotonic_ns()))
            k += 1

    readers = [text_reader("dense", 4096, Until(writer, 0, 3, KINDS, rebuild=True), 1),
               text_reader("sparse", 4096, Until(writer, 0, 3, KINDS), 2),
               text_reader("dev", 4096, Until(writer, 0, 3, KINDS), 3),
               text_reader("dense", 131072, Until(writer, 0, 2, ["add"], cap=3), 4, max_blocks=40),
               store_thread]
    _race(work, writer, readers, 60)
    hist = writer.history(work)
    evidence = {}
    _check_scores(work, writer, hist, reads, Checker(hist, W), evidence)
    _evidence_ok(evidence, 1, KINDS)
    spans_r = [(s, e) for _, _, s, e, _ in reads.calls]
    assert len(store_calls) >= 2 and any(s < e1 and s1 < e for s, e in store_calls for s1, e1 in spans_r), "no store call ran during a read"
    assert ix.text_store_len() == len(hs)
    q = [prompt_text(s, None)[0] for s in range(len(work.specs))]
    got, want = ix.text_store_find(*pack_text(q)), host_find(hs, q)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    _quiescent(work, hist, [ix])
