"""GPU (-m gpu): the device prefix store (kvidx_text_store_*) and Score() from text (kvidx_score_text*) at the sizes they
serve, against the host store (host.PrefixStore, the reference's LRUTokenStore) and score_batch of its finds' tokens.

  * Call streams of adds and finds of 1 to 131 072 prompts (both sides of the 16 384-prompt switch from 4 hash lanes per
    prompt to one), at 16-, 64- and 256-byte blocks and cache_blocks 7 to 500 000, some calls carrying more distinct
    blocks than the cache holds.  Prompts share a system prompt (one key touched by most prompts of a call), repeat inside
    a call, share family prefixes, and include unrelated, short, empty and non-ASCII text; tokenizations carry the spans
    real tokenizers report.  After every call the resident count and every find are compared bit for bit, and now and
    then a find over every prompt seen so far -- finds refresh recency on both sides, so this also pins down each cut.
  * The arena growing in one add, compacting under rewrites at 65 536 prompts a call, and one large add cut down to a
    small cache.
  * Score() from text on every Score() path, at index block sizes 24 to 128, on sharded handles, and its side effects on
    CLOCK handles; and store calls queued behind a Score() from text that still reads the store's scratch.
  * service.Indexer.get_pod_scores_batch against per-prompt get_pod_scores at 4096 prompts."""
import numpy as np
import pytest

import kvidx
from kvidx import pack_text
from kvidx.host import PrefixStore
from helpers import PATHS, SEED_ORDER, _index_pair, _select_path
from oracle.kvoracle_c import COracle
from test_gpu_text_store import host_find

pytestmark = pytest.mark.gpu
LANE_MAX = 16384                                 # kTextLaneMax: batches this large hash with a thread per prompt
UTF8 = "Grüße aus Köln, 漢字とかな, naïve café — ".encode("utf-8")


# ---- prompts and tokenizations ---------------------------------------------------------------------------------------
class Gen:
    """Prompt text for a store of bb-byte blocks: a system prompt of several blocks (non-ASCII UTF-8) in most prompts,
    families that share a prefix, duplicates inside a call, unrelated random bytes, text shorter than one block and empty
    text.  tail: the longest unique tail, in blocks (the distinct blocks a prompt brings)."""

    def __init__(self, rng, bb, tail=4, fam_blocks=6):
        self.rng, self.bb, self.tail = rng, bb, tail
        self.sys = (UTF8 * (4 * bb // len(UTF8) + 1))[:3 * bb + bb // 2]
        self.fam = [rng.bytes(int(rng.integers(bb, fam_blocks * bb + 1))) for _ in range(64)]
        self.fam_max = max(len(f) for f in self.fam)
        self.seen = []

    def prompts(self, n, reuse=0.3):
        rng, bb = self.rng, self.bb
        r = rng.random(n)
        old = rng.random(n) < reuse
        cut = rng.integers(0, self.fam_max + 1, n)
        tl = rng.integers(0, self.tail * bb + 1, n)
        fam = rng.integers(0, len(self.fam), n)
        blob = rng.bytes(int(tl.sum()) + 1)
        at = np.concatenate([[0], np.cumsum(tl)])
        out = []
        for i in range(n):
            tail = blob[at[i]:at[i + 1]]
            if old[i] and self.seen:
                p = self.seen[int(rng.integers(0, len(self.seen)))]            # seen in an earlier call
            elif r[i] < 0.08 and out:
                p = out[int(rng.integers(0, len(out)))]                        # a duplicate inside the call
            elif r[i] < 0.11:
                p = b""
            elif r[i] < 0.16:
                p = tail[:int(rng.integers(0, bb))]                            # shorter than one block
            elif r[i] < 0.26:
                p = tail + tail[:bb]                                           # unrelated text
            else:
                f = self.fam[fam[i]]
                p = (self.sys if r[i] < 0.9 else b"") + f[:min(cut[i], len(f))] + tail
            out.append(p)
        self.seen.extend(out[:: max(1, n // 2048)])
        return out


def tokenize_call(rng, text, off, bb):
    """Tokenizations of a whole call at once -> (ids, spans (n_tok, 2), tok_off).  Token ends fall every bb/6 bytes on
    average and at every prompt's end; then some tokens are reported as (0, 0) after later ones (special tokens), some
    ends decrease, some lie past the end of the text, some bytes end runs of several tokens, and a few prompts with text
    have no tokens at all."""
    n, T = len(off) - 1, len(text)
    lens = np.diff(off)
    ends = np.cumsum(rng.geometric(min(1.0, 6.0 / bb), int(T * 6.0 / bb * 1.2) + 64))
    ends = ends[ends <= T]
    ends = np.unique(np.concatenate([ends, off[1:][lens > 0]]))
    pid = np.searchsorted(off, ends, side="left") - 1
    rel = (ends - off[pid]).astype(np.int64)
    rep = np.where(rng.random(len(rel)) < 0.04, rng.integers(2, 7, len(rel)), 1)   # several tokens ending on one byte
    pid, rel = np.repeat(pid, rep), np.repeat(rel, rep)
    low = np.maximum(rel - rng.integers(0, 5, len(rel)), 0)
    u = rng.random(len(rel))
    z = u < 0.01                                                                  # (0, 0) after later tokens
    low[z], rel[z] = 0, 0
    d = (u >= 0.01) & (u < 0.02)                                                  # an end below the previous one
    rel[d] = np.maximum(rel[d] - rng.integers(1, 2 * bb, int(d.sum())), 0)
    low[d] = np.minimum(low[d], rel[d])
    p = (u >= 0.02) & (u < 0.024)                                                 # past the end of the text
    rel[p] = lens[pid[p]] + rng.integers(1, 3 * bb, int(p.sum()))
    keep = ~(rng.random(n) < 0.03)[pid]                                           # prompts without tokens
    pid, rel, low = pid[keep], rel[keep], low[keep]
    tok_off = np.zeros(n + 1, np.int64)
    tok_off[1:] = np.cumsum(np.bincount(pid, minlength=n))
    ids = rng.integers(0, 1 << 32, len(pid), dtype=np.uint64).astype(np.uint32)
    return ids, np.stack([low, rel], axis=1).astype(np.uint64), tok_off


def store_add(ix, hs, prompts, rng, bb, text=None, off=None):
    if text is None:
        text, off = pack_text(prompts)
    ids, spans, toff = tokenize_call(rng, text, off, bb)
    ix.text_store_add(text, off, ids, spans, toff)
    for i, p in enumerate(prompts):
        hs.add_tokenization(p, ids[toff[i]:toff[i + 1]], spans[toff[i]:toff[i + 1]])
    return ids, spans, toff


def same_find(ix, hs, prompts, what):
    text, off = pack_text(prompts)
    got, want = ix.text_store_find(text, off), host_find(hs, prompts)
    assert np.array_equal(got[1], want[1]), "%s: token offsets differ from prompt %d" % (what, np.flatnonzero(got[1] != want[1])[0] - 1)
    assert np.array_equal(got[0], want[0]), "%s: tokens differ" % what
    assert got[2].tobytes() == want[2].tobytes(), "%s: ratios differ" % what
    return want


# ---- call streams against the host store -----------------------------------------------------------------------------
SIZES = [1, 31, 4096, 16383, 16384, 65536, 131072]
STREAMS = {                                       # (block bytes, cache blocks, longest tail in blocks, largest call)
    "16-500000": (16, 500000, 10, 131072),        # one 131 072-prompt add carries ~1 M distinct blocks
    "16-7": (16, 7, 4, 131072),
    "64-4096": (64, 4096, 4, 131072),
    "64-100000": (64, 100000, 6, 131072),
    "256-100000": (256, 100000, 2, 65536),
    "256-500000": (256, 500000, 2, 65536),
}


@pytest.mark.parametrize("case", list(STREAMS))
def test_call_streams_at_batch_sizes_equal_the_host_store(case):
    bb, cap, tail, top = STREAMS[case]
    rng = np.random.default_rng(sum(map(ord, case)))
    ix = kvidx.Index(capacity=4096, max_pods=64)
    ix.text_store_init(cap, bb)
    hs = PrefixStore(cache_size=cap, block_size=bb)
    gen = Gen(rng, bb, tail=tail, fam_blocks=6 if bb < 256 else 3)
    sizes = [s for s in SIZES if s <= top]
    calls = [(op, s) for s in sizes for op in ("add", "find")] + [(op, s) for s in sizes[::-1][1:] for op in ("find", "add")]
    big = 0
    for c, (op, n) in enumerate(calls):
        prompts = gen.prompts(n)
        what = "%s call %d (%s of %d)" % (case, c, op, n)
        if op == "add":
            text, off = pack_text(prompts)
            store_add(ix, hs, prompts, rng, bb, text, off)
            big = max(big, len(text) // bb)
        else:
            same_find(ix, hs, prompts, what)
        assert ix.text_store_len() == len(hs), what
        if c in (len(calls) // 2, len(calls) - 1):
            same_find(ix, hs, gen.seen, what + ", then every prompt seen")
    if cap <= 100000:
        assert big > cap, "no add carried more blocks than the cache holds"


def test_one_add_grows_the_arena_past_64_ki_tokens():
    """A fresh store (64 Ki tokens of arena) takes one add of 16 384 prompts holding several times that, then one of
    65 536 prompts; every find and the resident count follow the host store."""
    rng = np.random.default_rng(3)
    ix = kvidx.Index(capacity=4096, max_pods=64)
    ix.text_store_init(500000, 16)
    hs = PrefixStore(cache_size=500000, block_size=16)
    gen = Gen(rng, 16, tail=8)
    first = gen.prompts(LANE_MAX, reuse=0)
    ids, _, _ = store_add(ix, hs, first, rng, 16)
    assert len(ids) > 3 * (1 << 16)
    assert ix.text_store_len() == len(hs)
    same_find(ix, hs, first, "after the first add")
    more = gen.prompts(65536)
    store_add(ix, hs, more, rng, 16)
    assert ix.text_store_len() == len(hs)
    same_find(ix, hs, first + more, "after the second add")


def test_rewrites_compact_the_arena_at_65536_prompts():
    """The same 65 536 prompts, most of them rewritten call after call with new tokens: every add leaves the previous
    records dead, and the arena compacts again and again."""
    rng = np.random.default_rng(4)
    ix = kvidx.Index(capacity=4096, max_pods=64)
    ix.text_store_init(500000, 16)
    hs = PrefixStore(cache_size=500000, block_size=16)
    gen = Gen(rng, 16, tail=4)
    prompts = gen.prompts(65536, reuse=0)
    text, off = pack_text(prompts)
    for c in range(8):
        store_add(ix, hs, prompts, rng, 16, text, off)
        assert ix.text_store_len() == len(hs), c
        if c % 2 == 1:
            same_find(ix, hs, prompts, "rewrite %d" % c)


@pytest.mark.parametrize("cap", [7, 4096])
def test_large_add_then_cut_to_a_small_cache(cap):
    """A warm store, then one add of 131 072 prompts (~1 M blocks) cut down to cap keys: the next finds see exactly the
    keys the host store kept."""
    rng = np.random.default_rng(cap)
    ix = kvidx.Index(capacity=4096, max_pods=64)
    ix.text_store_init(cap, 64)
    hs = PrefixStore(cache_size=cap, block_size=64)
    gen = Gen(rng, 64, tail=8)
    warm = gen.prompts(4096)
    store_add(ix, hs, warm, rng, 64)
    big = gen.prompts(131072, reuse=0.05)
    text, off = pack_text(big)
    assert len(text) // 64 > 8 * 10 ** 5
    store_add(ix, hs, big, rng, 64, text, off)
    assert ix.text_store_len() == len(hs) == cap
    same_find(ix, hs, big[-512:] + warm[:512] + big[:512], "after the cut")
    same_find(ix, hs, big, "every prompt of the large add")
    store_add(ix, hs, gen.prompts(31), rng, 64)
    same_find(ix, hs, big[-2048:], "after one more add")
    assert ix.text_store_len() == len(hs)


# ---- Score() from text -----------------------------------------------------------------------------------------------
P = 64


def _docs(rng, BS, n_docs=56, max_blocks=10):
    """Token documents and their text: 4 bytes a token (spans (4j, 4j + 4)); most documents open with one of two shared
    prefixes of 3 index blocks, so their text shares blocks too."""
    heads = [rng.integers(0, 50000, 3 * BS) for _ in range(2)]
    docs = []
    for d in range(n_docs):
        nt = int(rng.integers(BS // 2, max_blocks * BS + BS))
        ids = rng.integers(0, 50000, nt)
        if d % 4 != 3:
            h = heads[d % 2][:nt]
            ids[:len(h)] = h
        docs.append(ids.astype(np.uint32))
    return docs


def _text_of(ids):
    return (ids.astype("<u4") * np.uint32(2654435761)).tobytes()        # a token's 4 bytes depend on its id only


def _fill(rng, targets, docs, BS):
    """Keys of document prefixes, on every target (handles and the oracle), each prefix with 1 or 2 pods"""
    k0 = COracle(block_size=BS)
    for d, ids in enumerate(docs[:48]):
        k, _ = k0.hash_keys(ids, [0, len(ids)])
        cut = int(rng.integers(0, len(k) + 1))
        if not cut:
            continue
        pts = [(int(rng.integers(0, P)) << 4) | int(rng.integers(0, 2)) for _ in range(int(rng.integers(1, 3)))]
        for t in targets:
            assert t.add(d % 3, k[:cut] ^ np.uint64(0x5A5A), k[:cut], pts) == 0


def _store(stores, hs, docs, bb):
    """The text of documents 0..39 with their tokens, and one text whose tokens all end past its first blocks (a
    prefix of it passes the gate with no contained token)"""
    prompts = [_text_of(ids) for ids in docs[:40]]
    spans = [np.stack([np.arange(len(i)) * 4, np.arange(len(i)) * 4 + 4], axis=1) for i in docs[:40]]
    ids = [ids for ids in docs[:40]]
    lone = _text_of(np.concatenate(docs[48:56]))
    prompts.append(lone); ids.append(np.array([7], np.uint32)); spans.append(np.array([[0, len(lone)]]))
    text, off = pack_text(prompts)
    toff = np.zeros(len(prompts) + 1, np.int64)
    toff[1:] = np.cumsum([len(i) for i in ids])
    for s in stores:
        s.text_store_add(text, off, np.concatenate(ids), np.concatenate(spans).astype(np.uint64), toff)
    for p, i, sp in zip(prompts, ids, spans):
        hs.add_tokenization(p, i, sp)
    return lone


def _queries(rng, docs, lone, n, bb):
    """n query texts: stored documents whole, extended and cut; exactly 3 of 4 whole blocks stored (ratio 0.75); a
    prefix of the tokenless text (passes with no tokens); unknown documents (ratio 0)."""
    q = []
    for _ in range(n):
        r = rng.random()
        t = _text_of(docs[int(rng.integers(0, 48))])
        if r < 0.3:
            q.append(t)
        elif r < 0.5:
            q.append(t + rng.bytes(int(rng.integers(1, 2 * bb))))
        elif r < 0.65:
            q.append(t[:int(rng.integers(0, len(t) + 1))])
        elif r < 0.8:
            k = int(rng.integers(0, 40))
            t = _text_of(docs[k])
            if len(t) >= 3 * bb:
                q.append(t[:3 * bb] + bytes(x ^ 0xFF for x in t[3 * bb:4 * bb]) if len(t) >= 4 * bb else t[:3 * bb] + rng.bytes(bb))
            else:
                q.append(t)
        elif r < 0.85:
            q.append(lone[:bb * int(rng.integers(1, max(2, len(lone) // bb)))])
        else:
            q.append(t)
    return q


def _want(hs, q, min_ratio):
    """-> (tokens and offsets score_batch takes, passing, ratios) from the host store's find and the gate"""
    tok, toff, ratio = host_find(hs, q)
    passing = ratio >= min_ratio
    lens = np.where(passing, toff[1:] - toff[:-1], 0)
    soff = np.zeros(len(q) + 1, np.int64)
    soff[1:] = np.cumsum(lens)
    return tok[np.repeat(passing, toff[1:] - toff[:-1])], soff, passing, ratio


def _dev_text(q):
    import torch
    text, off = pack_text(q)
    return torch.from_numpy(text.copy()).cuda(), torch.from_numpy(off).cuda()


def _score_text_dev(ix, q, min_ratio, model=None, filt=None):
    """score_text_dev and score_text_sparse_dev -> (dense rows, has, tokenize, ratio, (pods, scores, cnt))"""
    import torch
    n = len(q)
    d_text, d_off = _dev_text(q)
    d_model = torch.from_numpy(model.view(np.int32)).cuda() if model is not None else None
    d_filt = torch.from_numpy(filt.view(np.int64)).cuda() if filt is not None else None
    d_sc = torch.empty((n, ix.max_pods), dtype=torch.float64, device="cuda")
    d_has, d_tz = torch.empty(n, dtype=torch.uint8, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda")
    d_r = torch.empty(n, dtype=torch.float64, device="cuda")
    d_p, d_s = torch.zeros((n, 10), dtype=torch.int16, device="cuda"), torch.zeros((n, 10), dtype=torch.float64, device="cuda")
    d_c = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    mp, fp = (d_model.data_ptr() if d_model is not None else 0), (d_filt.data_ptr() if d_filt is not None else 0)
    ix.score_text_dev(d_text.data_ptr(), d_off.data_ptr(), n, d_sc.data_ptr(), d_model=mp, d_filter=fp, min_ratio=min_ratio,
                      d_has_keys=d_has.data_ptr(), d_tokenize=d_tz.data_ptr(), d_ratio=d_r.data_ptr())
    ix.score_text_sparse_dev(d_text.data_ptr(), d_off.data_ptr(), n, d_p.data_ptr(), d_s.data_ptr(), d_c.data_ptr(), d_model=mp,
                             d_filter=fp, min_ratio=min_ratio)
    ix.synchronize()
    return (d_sc.cpu().numpy(), d_has.cpu().numpy(), d_tz.cpu().numpy(), d_r.cpu().numpy(),
            (d_p.cpu().numpy().view(np.uint16), d_s.cpu().numpy(), d_c.cpu().numpy()))


def _same_sparse(got, want):
    gp, gs, gc = got
    wp, ws, wc = want
    assert np.array_equal(gc, wc)
    for i in np.flatnonzero(wc):
        assert gp[i, :wc[i]].tolist() == wp[i, :wc[i]].tolist() and gs[i, :wc[i]].tobytes() == ws[i, :wc[i]].tobytes(), i


def _check_text(ix, co, hs, q, min_ratio, api, model=None, filt=None):
    """Score() from text on ix (api host / dev) against score_batch of the host find's gated tokens on ix and the
    oracle's rows.  -> (passing, ratio)"""
    tok, soff, passing, ratio = _want(hs, q, min_ratio)
    want, want_has = ix.score_batch(tok, soff, model=model, filter_mask=filt)
    wp, ws, wc, _ = ix.score_batch_sparse(tok, soff, model=model, filter_mask=filt)
    if co is not None:
        orows, ohas, _, _ = co.score_batch(tok, soff, model=model, filter_mask=filt)
        assert np.array_equal(want, orows) and np.array_equal(want_has, ohas)
    if api == "host":
        text, off = pack_text(q)
        got, has, tz, r = ix.score_text(text, off, model=model, filter_mask=filt, min_ratio=min_ratio)
        gp, gs, gc, gh, tz2, r2 = ix.score_text_sparse(text, off, model=model, filter_mask=filt, min_ratio=min_ratio)
        assert np.array_equal(tz2, tz) and r2.tobytes() == r.tobytes() and np.array_equal(gh, has)
        sparse = (gp, gs, gc)
    else:
        got, has, tz, r, sparse = _score_text_dev(ix, q, min_ratio, model, filt)
    assert got.tobytes() == want.tobytes(), np.argwhere(got != want)[:4]
    assert np.array_equal(has, want_has)
    assert np.array_equal(tz, (~passing).astype(np.uint8)) and r.tobytes() == ratio.tobytes()
    _same_sparse(sparse, (wp, ws, wc))
    return passing, ratio


def _gate_edges(hs, q, min_ratio=0.75):
    """the case has prompts exactly at the gate and prompts that pass it with no contained token"""
    tok, toff, ratio = host_find(hs, q)
    passing = ratio >= min_ratio
    assert (ratio == min_ratio).any(), "no prompt at exactly min_ratio"
    assert (passing & (toff[1:] == toff[:-1]) & (ratio > 0)).any(), "no prompt passes with zero tokens"
    assert (~passing).any()


def _model_filter(rng, n):
    model = rng.integers(0, 3, n).astype(np.uint32)
    filt = np.zeros((n, 1), np.uint64)
    filt[:, 0] = rng.integers(0, 1 << 63, n, dtype=np.uint64) | rng.integers(0, 1 << 63, n, dtype=np.uint64)
    filt[rng.random(n) < 0.5] = np.uint64((1 << 64) - 1)
    return model, filt


@pytest.mark.parametrize("path", PATHS)
def test_score_text_on_every_score_path(path, monkeypatch):
    """Each Score() path (a handle each) scores 4096 prompts from text, dense and sparse, host and _dev, with prompts
    exactly at min_ratio 0.75 and prompts that pass it with no contained token."""
    rng = np.random.default_rng(SEED_ORDER.index(path) + 500)
    with monkeypatch.context() as mp:
        _select_path(mp, path)
        ix, co = _index_pair(block_size=16, capacity=1 << 16, max_pods=P)
    docs = _docs(rng, 16)
    _fill(rng, [ix, co], docs, 16)
    ix.text_store_init(500000, 64)
    hs = PrefixStore(500000, 64)
    lone = _store([ix], hs, docs, 64)
    q = _queries(rng, docs, lone, 4096, 64)
    _gate_edges(hs, q)
    model, filt = _model_filter(rng, len(q))
    for min_ratio, api in ((0.75, "host"), (0.75, "dev"), (0.0, "host")):
        _check_text(ix, co, hs, q, min_ratio, api, model, filt)


@pytest.mark.parametrize("api", ["host", "dev"])
@pytest.mark.parametrize("n", [1, 32, 2048, 16384])
@pytest.mark.parametrize("BS", [24, 32, 64, 128])
def test_score_text_at_index_block_sizes(BS, n, api):
    """24-, 32-, 64- and 128-token index blocks with 256-byte store blocks: 32 to 128 run the warp-per-prompt kernel up
    to coop_max prompts and v1 above it, 24 runs v1."""
    rng = np.random.default_rng(BS * 100 + n)
    ix, co = _index_pair(block_size=BS, capacity=1 << 16, max_pods=P)
    docs = _docs(rng, BS, max_blocks=8)
    _fill(rng, [ix, co], docs, BS)
    ix.text_store_init(500000, 256)
    hs = PrefixStore(500000, 256)
    lone = _store([ix], hs, docs, 256)
    q = _queries(rng, docs, lone, n, 256)
    if n >= 2048:
        _gate_edges(hs, q)
    model, filt = _model_filter(rng, n)
    for min_ratio in (0.75, 0.8):
        _check_text(ix, co, hs, q, min_ratio, api, model, filt)


@pytest.mark.parametrize("peer_pair", [0, 1])
@pytest.mark.parametrize("shards", [2, 8])
def test_score_text_on_sharded_handles(shards, peer_pair, monkeypatch):
    """The store on one rank's handle of a 2- or 8-shard index on one GPU: its rows equal its unsharded twin's and the
    oracle's."""
    from test_gpu_shard_ops import _shards
    monkeypatch.setenv("KVIDX_PEER_PAIR", str(peer_pair))
    rng = np.random.default_rng(shards * 10 + peer_pair)
    cfg = dict(block_size=16, hash_seed="", capacity=1 << 16, pods_per_key=10, tier_weights=(1.0, 0.8), max_pods=P)
    sh = _shards(shards, **cfg)
    twin, co = _index_pair(block_size=16, capacity=1 << 16, pods_per_key=10, max_pods=P)
    docs = _docs(rng, 16)
    _fill(rng, [sh[0], twin, co], docs, 16)
    via = sh[shards - 1]
    via.text_store_init(500000, 64)
    twin.text_store_init(500000, 64)
    hs = PrefixStore(500000, 64)
    lone = _store([via, twin], hs, docs, 64)
    q = _queries(rng, docs, lone, 4096, 64)
    model, filt = _model_filter(rng, len(q))
    for api in ("host", "dev"):
        _check_text(via, co, hs, q, 0.8, api, model, filt)
    a = twin.score_text(*pack_text(q), model=model, filter_mask=filt, min_ratio=0.8)
    b = via.score_text(*pack_text(q), model=model, filter_mask=filt, min_ratio=0.8)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_score_text_leaves_the_clock_bits_score_batch_leaves():
    """Twin CLOCK handles capped below their contents: score_text on one, score_batch of the same token CSR on the other,
    then the same capped adds that sweep on both.  Their images are byte-equal after each step.  Every add stores one
    key, so both handles place every key in the same slot and their hands meet the keys in the same order: any
    difference is one of reference bits."""
    rng = np.random.default_rng(77)
    twins = [kvidx.Index(block_size=16, capacity=40, table_slots=1 << 14, max_pods=P, evict_policy="clock") for _ in range(2)]
    docs = _docs(rng, 16, n_docs=56, max_blocks=10)
    k0 = COracle(block_size=16)
    for d, ids in enumerate(docs[:48]):
        k, _ = k0.hash_keys(ids, [0, len(ids)])
        pts = [(int(rng.integers(0, P)) << 4) | int(rng.integers(0, 2))]
        for x in k[:int(rng.integers(0, len(k) + 1))]:
            for t in twins:
                assert t.add(d % 3, [x ^ np.uint64(0x5A5A)], [x], pts) == 0
    a, b = twins
    assert a.sweeps()[0] > 0 and a.snapshot() == b.snapshot()
    a.text_store_init(500000, 64)
    hs = PrefixStore(500000, 64)
    lone = _store([a], hs, docs, 64)
    q = _queries(rng, docs, lone, 4096, 64)
    model = rng.integers(0, 3, len(q)).astype(np.uint32)
    tok, soff, passing, ratio = _want(hs, q, 0.8)
    got = a.score_text(*pack_text(q), model=model, min_ratio=0.8)
    want = b.score_batch(tok, soff, model=model)
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1]) and want[1].any()
    assert a.snapshot() == b.snapshot()
    s0 = a.sweeps()[0]
    for x in rng.integers(1, 1 << 63, 24, dtype=np.uint64):
        for t in twins:
            assert t.add(1, [x ^ np.uint64(0x77)], [x], [(5 << 4)]) == 0
        assert a.snapshot() == b.snapshot(), "a sweep after score_text evicted other keys than after score_batch"
    assert a.sweeps()[0] > s0 and a.stats()["rebuilds"] == b.stats()["rebuilds"]


# ---- store calls queued behind a Score() from text -------------------------------------------------------------------
def test_store_calls_queued_behind_score_text_dev():
    """score_text_dev of 65 536 prompts is queued, not synchronised; straight after it an add that forces the eviction
    cut, a table rebuild and an arena compaction, then a find of other prompts, reuse the store's scratch.  After one
    synchronise the queued call's rows, flags and ratios are the ones expected before those calls, and the store calls
    return what the host store returns."""
    import torch
    rng = np.random.default_rng(99)
    ix, co = _index_pair(block_size=16, capacity=1 << 16, max_pods=P)
    docs = _docs(rng, 16)
    _fill(rng, [ix, co], docs, 16)
    cap = 60000
    ix.text_store_init(cap, 64)
    hs = PrefixStore(cap, 64)
    lone = _store([ix], hs, docs, 64)
    gen = Gen(rng, 64, tail=4)
    warm = gen.prompts(16384, reuse=0)
    wids, _, _ = store_add(ix, hs, warm, rng, 64)
    assert ix.text_store_len() == len(hs)
    n = 65536
    q = _queries(rng, docs, lone, n - 4096, 64) + warm[:4096]
    tok, soff, passing, ratio = _want(hs, q, 0.8)
    want, want_has = ix.score_batch(tok, soff)
    big = gen.prompts(65536, reuse=0)
    other = warm[4096:8192] + big[-4096:]
    d_text, d_off = _dev_text(q)
    d_sc = torch.empty((n, P), dtype=torch.float64, device="cuda")
    d_has, d_tz = torch.empty(n, dtype=torch.uint8, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda")
    d_r = torch.empty(n, dtype=torch.float64, device="cuda")
    btext, boff = pack_text(big)
    bids, bspans, btoff = tokenize_call(rng, btext, boff, 64)
    # the arena holds at most twice the tokens added so far: this add compacts it; its blocks alone exceed the cache
    assert len(bids) > 2 * (len(wids) + 10 ** 5) and len(btext) // 64 > cap
    otext, ooff = pack_text(other)
    torch.cuda.synchronize()
    ix.score_text_dev(d_text.data_ptr(), d_off.data_ptr(), n, d_sc.data_ptr(), min_ratio=0.8, d_has_keys=d_has.data_ptr(),
                      d_tokenize=d_tz.data_ptr(), d_ratio=d_r.data_ptr())
    ix.text_store_add(btext, boff, bids, bspans, btoff)
    got_find = ix.text_store_find(otext, ooff)
    ix.synchronize()
    assert d_sc.cpu().numpy().tobytes() == want.tobytes() and np.array_equal(d_has.cpu().numpy(), want_has)
    assert np.array_equal(d_tz.cpu().numpy(), (~passing).astype(np.uint8)) and d_r.cpu().numpy().tobytes() == ratio.tobytes()
    for i, p in enumerate(big):
        hs.add_tokenization(p, bids[btoff[i]:btoff[i + 1]], bspans[btoff[i]:btoff[i + 1]])
    wf = host_find(hs, other)
    assert all(np.array_equal(g, w) for g, w in zip(got_find, wf)) and got_find[2].tobytes() == wf[2].tobytes()
    assert ix.text_store_len() == len(hs) == cap


# ---- the service's batch path at 4096 prompts ------------------------------------------------------------------------
def test_get_pod_scores_batch_at_4096_prompts():
    """A local WordLevel tokenizer (whitespace pre-tokenisation, non-ASCII words).  Pass one: prompts that pairwise share
    less than 80 % of their bytes, so both paths tokenize every prompt; pass two: the same prompts, served from both
    stores.  Both passes equal per-prompt get_pod_scores, with equal lookup metrics and the expected encode counts."""
    from tokenizers import Tokenizer, models, pre_tokenizers
    from kvidx import service
    from kvidx.host import HostIndexer
    rng = np.random.default_rng(2026)
    words = ["[UNK]"] + ["w%d" % i for i in range(3000)] + ["grüße", "köln", "zürich", "漢字", "naïve", "café", "straße"]
    vocab = {w: i for i, w in enumerate(words)}

    def tk():
        t = Tokenizer(models.WordLevel(vocab, unk_token="[UNK]"))
        t.pre_tokenizer = pre_tokenizers.Whitespace()
        return t

    heads = [" ".join(rng.choice(words[1:], 120)) for _ in range(16)]
    prompts = []
    for i in range(4096):
        body = " ".join(rng.choice(words[1:], int(rng.integers(300, 420))))
        prompts.append((heads[i % 16] + " " + body) if i % 3 else body)      # a shared head is well under 80 % of a prompt
    model, pod_names = "m", ["10.0.0.%d" % p for p in range(8)]
    stacks = []
    for _ in range(2):
        host = HostIndexer(block_size=16, capacity=1 << 18, max_pods=64, enable_metrics=True)
        stacks.append((host, service.Indexer(host, service.TokenizationPool(tokenizer=tk()))))
    enc = tk()
    for host, _ in stacks:
        ix = kvidx.Index.borrow(host.L.kvhost_index(host.h), 16, 64)
        for j, p in enumerate(prompts[:1024]):
            ids = np.asarray(enc.encode(p, add_special_tokens=False).ids, np.uint32)
            req, _ = ix.hash_keys(ids, np.array([0, len(ids)], np.int64))
            cut = len(req) * (j % 5) // 4
            if cut:
                assert host.add(model, req[:cut] ^ np.uint64(1), req[:cut], [(pod_names[j % 8], "gpu")]) == 0
    (h1, per), (h2, batch) = stacks
    for rnd in range(2):
        want = [per.get_pod_scores(p, model, pod_names[:6]) for p in prompts]
        got = batch.get_pod_scores_batch(prompts, model, pod_names[:6])
        assert got == want, rnd
        assert sum(w is not None and len(w) > 0 for w in want) > 300
        assert per.tok.encodes == batch.tok.encodes == 4096, (rnd, per.tok.encodes, batch.tok.encodes)
    m1, m2 = h1.metrics(), h2.metrics()
    for k in ("lookup_requests_total", "lookup_hits_total", "max_pod_hit_count_total"):
        assert m1[k] == m2[k] > 0, k
