"""One-process-per-GPU plumbing for the replica mode (torch.distributed; NCCL on GPUs, gloo in the CPU tests).

The Score() path shards by prompt: every rank holds a full replica of the index (10 M blocks = 1 GB of slots),
scores its own contiguous slice of the batch, and no data-path collective is needed.  What has to be replicated is
the write path: every rank must apply the same KV events, in the same per-pod order.  `broadcast_event_batch` does
that from the ingesting rank; `shard_range` splits a batch; `max_over_ranks` is the timing reduction bench.py uses.
The hash-range sharded mode has its own helpers: `connect_shards`, and the collective maintenance calls
`compact_shards`, `remove_pods_shards`, `snapshot_shards` and `restore_shards`, which put the barriers around them,
and `pod_inventory_shards`, a read that needs none.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

EVENT_DTYPE = np.dtype([("op", "u1"), ("has_parent", "u1"), ("podtier", "<u2"), ("model", "<u4"),
                        ("parent_hash", "<u8"), ("hash_off", "<u8"), ("tok_off", "<u8"),
                        ("n_hashes", "<u4"), ("n_tokens", "<u4")])


def shard_range(n: int, rank: int, world: int):
    """Contiguous, balanced split of n prompts: ranks [0, n % world) get one extra."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def max_over_ranks(value: float, device=None) -> float:
    """Device-timed milliseconds -> max over ranks (the number a multi-GPU step is judged by)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def broadcast_event_batch(events, hashes, tokens, src: int = 0, device=None):
    """Replicate one decoded event batch (kvidx_event_t array + flat hash / token arrays) from `src` to all ranks.
    Returns numpy arrays on every rank.  Sizes go first, then the three payloads as byte tensors."""
    rank = dist.get_rank()
    if rank == src:
        ev = np.ascontiguousarray(events, EVENT_DTYPE)
        hs = np.ascontiguousarray(hashes, np.uint64)
        tk = np.ascontiguousarray(tokens, np.uint32)
        sizes = torch.tensor([len(ev), len(hs), len(tk)], dtype=torch.int64, device=device)
    else:
        sizes = torch.zeros(3, dtype=torch.int64, device=device)
    dist.broadcast(sizes, src)
    n_ev, n_hs, n_tk = (int(v) for v in sizes.tolist())
    out = []
    for arr, n, dt in ((events, n_ev, EVENT_DTYPE), (hashes, n_hs, np.dtype(np.uint64)), (tokens, n_tk, np.dtype(np.uint32))):
        nbytes = n * dt.itemsize
        if rank == src:
            buf = torch.from_numpy(np.ascontiguousarray(arr, dt).view(np.uint8).reshape(-1).copy())
        else:
            buf = torch.empty(nbytes, dtype=torch.uint8)
        if device is not None:
            buf = buf.to(device)
        if nbytes:
            dist.broadcast(buf, src)
        out.append(buf.cpu().numpy().view(dt) if nbytes else np.zeros(0, dt))
    return tuple(out)


def gather_scores(local_scores: np.ndarray, n_total: int, device=None):
    """Collect the per-rank score slices (shard_range order) on every rank (all_gather of padded rows)."""
    world, rank = dist.get_world_size(), dist.get_rank()
    P = local_scores.shape[1]
    cap = -(-n_total // world)
    pad = np.full((cap, P), -1.0)
    pad[: len(local_scores)] = local_scores
    t = torch.from_numpy(pad)
    if device is not None:
        t = t.to(device)
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t)
    out = np.empty((n_total, P))
    for r in range(world):
        lo, hi = shard_range(n_total, r, world)
        out[lo:hi] = parts[r].cpu().numpy()[: hi - lo]
    return out


def connect_shards(ix, device=None):
    """Hash-range sharded mode: exchange the CUDA-IPC handle blobs of every rank's shard (one all_gather of 192 bytes
    per rank -- the only collective this mode needs) and map them.  After this call every kernel of `ix` can probe /
    lock slots of any shard through NVLink peer memory."""
    world, rank = dist.get_world_size(), dist.get_rank()
    mine = torch.frombuffer(bytearray(ix.shard_export()), dtype=torch.uint8)
    if device is not None:
        mine = mine.to(device)
    parts = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(parts, mine)
    for r in range(world):
        if r != rank:
            ix.shard_import(r, bytes(parts[r].cpu().numpy().tobytes()))
    dist.barrier()


def compact_shards(ix):
    """Drop the tombstones of every rank's shard (kvidx_shard_compact).  Collective: a barrier either side keeps every
    rank off the index while the shards are rewritten in place (peers keep their mappings)."""
    dist.barrier()
    ix.shard_compact()
    dist.barrier()


def events_for_rank(events, rank: int, world: int):
    """Ingest rule of the sharded mode: all events of one pod go through one rank (pod id modulo world), which keeps
    the reference's per-pod ordering (kvevents/pool.go:129-144) without any cross-GPU coordination."""
    pods = events["podtier"] >> 4
    return events[(pods % world) == rank]


def _a2a(out, inp, out_split=None, in_split=None):
    """all_to_all_single on whatever backend the group has (gloo has no CUDA all-to-all: stage through the host there)."""
    if dist.get_backend() == "gloo" and inp.is_cuda:
        o = torch.empty(out.shape, dtype=out.dtype)
        dist.all_to_all_single(o, inp.cpu(), out_split, in_split)
        out.copy_(o)
    else:
        dist.all_to_all_single(out, inp, out_split, in_split)


def score_alltoall(ix, d_tok, d_off, n, d_scores, block_size=16, model0=0, d_has=None):
    """The ROUTED form of a sharded Score() (SURVEY 8(e)): every key of every prompt is hashed at the origin, sent to the rank
    that owns its hash range (NCCL all-to-all), looked up there, and its 32-byte slot image sent back (second all-to-all); the
    origin then walks and scores.  No early exit, no prefix sharing: all n_blocks keys travel.  Tensors are torch CUDA
    tensors; `ix` is a sharded handle whose stream is the CURRENT torch stream, which must be a real (non-default) stream
    -- ix.set_stream(stream.cuda_stream); handle 0 would mean the library's own stream.  Returns a dict of volumes."""
    world = dist.get_world_size()
    dev = d_tok.device
    lens = torch.div(d_off[1:n + 1] - d_off[:n], block_size, rounding_mode="floor")
    koff = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    torch.cumsum(lens, 0, out=koff[1:])
    nk = int(koff[-1].item())
    keys = torch.empty(max(nk, 1), dtype=torch.int64, device=dev)
    ix.hash_keys_dev(d_tok.data_ptr(), d_off.data_ptr(), n, koff.data_ptr(), keys.data_ptr())
    keys = keys[:nk]
    owners = torch.empty(max(nk, 1), dtype=torch.uint8, device=dev)
    ix.key_owners_dev(keys.data_ptr(), nk, owners.data_ptr(), model0)
    owners = owners[:nk]
    order = torch.argsort(owners, stable=True)
    counts = torch.bincount(owners, minlength=world).to(torch.int64)
    send = keys[order].contiguous()
    recv_counts = torch.empty_like(counts)
    _a2a(recv_counts, counts)
    in_split, out_split = counts.tolist(), recv_counts.tolist()
    recv = torch.empty(sum(out_split), dtype=torch.int64, device=dev)
    _a2a(recv, send, out_split, in_split)
    slots = torch.empty((max(len(recv), 1), 4), dtype=torch.int64, device=dev)
    ix.probe_slots_dev(recv.data_ptr(), len(recv), slots.data_ptr(), model0)
    slots = slots[: len(recv)]
    back = torch.empty((nk, 4), dtype=torch.int64, device=dev)
    _a2a(back, slots.contiguous(), in_split, out_split)
    slots_pm = torch.empty_like(back)
    slots_pm[order] = back
    ix.score_slots_dev(slots_pm.data_ptr(), koff.data_ptr(), n, d_scores.data_ptr(), d_has_keys=(d_has.data_ptr() if d_has is not None else 0))
    return {"keys": nk, "bytes_out": 8 * (nk - in_split[dist.get_rank()]), "bytes_back": 32 * (nk - in_split[dist.get_rank()])}


# ---- maintenance of a sharded index: pod removal, snapshot, restore (collective; every rank calls them) ---------------

def _all_ok(ok: bool, device=None) -> bool:
    """True on every rank iff `ok` on every rank.  The all-reduce also keeps every rank here until all have arrived."""
    t = torch.tensor([1 if ok else 0], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    return bool(t.item())


def _sum_over_ranks(values, device=None):
    t = torch.tensor([int(v) for v in values], dtype=torch.int64, device=device)
    dist.all_reduce(t)
    return [int(v) for v in t.tolist()]


def _collective_step(fn, what: str, device=None):
    """Run this rank's part of a collective call; raise on every rank if it failed on any (this rank's own error first)."""
    res, err = None, None
    try:
        res = fn()
    except Exception as e:      # noqa: BLE001  (re-raised below, after the other ranks have heard of it)
        err = e
    if not _all_ok(err is None, device):
        if err is not None:
            raise err
        raise RuntimeError("%s failed on another rank" % what)
    return res


def remove_pods_shards(ix, pod_ids, tier_ids=None, device=None) -> dict:
    """kvidx_remove_pods over a hash-range sharded index: every rank removes the entries of its request shard (phase 0),
    then, once all have, the engine mappings of its engine shard whose request key phase 0 removed on any rank (phase 1).
    Every rank must pass the same pods and tiers; that is checked first (an all-gather of the masks).  No rank may write
    to the index during the call; readers may run.  -> the summed {"entries", "request_keys", "engine_keys"}."""
    mask, tier_mask = ix.removal_masks(pod_ids, tier_ids)
    mine = torch.from_numpy(np.append(mask, np.uint64(tier_mask)).view(np.int64).copy())
    if device is not None:
        mine = mine.to(device)
    parts = [torch.empty_like(mine) for _ in range(dist.get_world_size())]
    dist.all_gather(parts, mine)
    if any(not torch.equal(p, parts[0]) for p in parts):
        raise ValueError("remove_pods_shards: the ranks were given different pod / tier sets")
    dist.barrier()
    r0 = _collective_step(lambda: ix.shard_remove_pods(pod_ids, tier_ids, phase=0), "phase 0 of the removal", device)
    r1 = _collective_step(lambda: ix.shard_remove_pods(pod_ids, tier_ids, phase=1), "phase 1 of the removal", device)
    tot = _sum_over_ranks([r0["entries"], r0["request_keys"], r1["engine_keys"]], device)
    return {"entries": tot[0], "request_keys": tot[1], "engine_keys": tot[2]}


def snapshot_shards(ix, dst: int = 0, device=None):
    """The canonical image of the whole sharded index (what kvidx_snapshot gives on an unsharded index with the same
    contents): every rank exports the keys it owns, the parts are gathered to `dst` and merged there.  No rank may write
    to the index during the call.  -> the image on `dst`, None elsewhere."""
    dist.barrier()
    part = _collective_step(ix.shard_snapshot, "the shard snapshot", device)
    world = dist.get_world_size()
    sizes = [torch.zeros(1, dtype=torch.int64, device=device) for _ in range(world)]
    dist.all_gather(sizes, torch.tensor([len(part)], dtype=torch.int64, device=device))
    sizes = [int(s.item()) for s in sizes]
    buf = torch.zeros(max(sizes), dtype=torch.uint8)
    buf[: len(part)] = torch.frombuffer(bytearray(part), dtype=torch.uint8)
    if device is not None:
        buf = buf.to(device)
    gathered = [torch.empty_like(buf) for _ in range(world)] if dist.get_rank() == dst else None
    dist.gather(buf, gathered, dst=dst)
    if dist.get_rank() != dst:
        return None
    from . import _native
    return _native.snapshot_merge([g.cpu().numpy().tobytes()[:n] for g, n in zip(gathered, sizes)])


def restore_shards(ix, image=None, src: int = 0, device=None) -> dict:
    """Load a v1 image (unsharded, merged or a single part) into an empty sharded index: each rank inserts the records it
    owns, so this also reshards (1 -> N, N -> M).  The image is broadcast from `src` unless every rank has it.  Raises on
    every rank unless every shard is empty, and on every rank if any rank's restore fails (a malformed image or one too
    large for an owner is refused by all before any inserts).  -> the summed {"request_keys", "engine_keys"} restored."""
    have = _all_ok(image is not None, device)
    if not have:
        if dist.get_rank() == src:
            if image is None:
                raise ValueError("restore_shards: rank %d holds no image" % src)
            payload = torch.frombuffer(bytearray(image), dtype=torch.uint8)
            n = torch.tensor([len(image)], dtype=torch.int64, device=device)
        else:
            n = torch.zeros(1, dtype=torch.int64, device=device)
        dist.broadcast(n, src)
        if dist.get_rank() != src:
            payload = torch.empty(int(n.item()), dtype=torch.uint8)
        if device is not None:
            payload = payload.to(device)
        dist.broadcast(payload, src)
        image = payload.cpu().numpy().tobytes()
    st = ix.stats()
    live = _sum_over_ranks([st["request_keys"], st["engine_keys"]], device)
    if any(live):
        raise RuntimeError("restore_shards needs an empty index: the shards hold %d request and %d engine keys" % tuple(live))
    dist.barrier()
    got = _collective_step(lambda: ix.shard_restore(image), "the shard restore", device)
    tot = _sum_over_ranks([got["request_keys"], got["engine_keys"]], device)
    return {"request_keys": tot[0], "engine_keys": tot[1]}


def pod_inventory_shards(ix, model=None, engine=False, device=None) -> dict:
    """kvidx_pod_inventory over a hash-range sharded index: every rank counts the request keys and engine mappings it owns
    and the arrays are summed with one all-reduce, so every rank gets the answer an unsharded index with the same contents
    gives.  A read: writers may run, and nothing but the all-reduce keeps the ranks together."""
    inv = ix.pod_inventory(model, engine)
    names = [k for k in ("entries", "keys", "sole", "sole_engine", "totals") if inv[k] is not None]
    flat = torch.from_numpy(np.concatenate([inv[k].reshape(-1) for k in names]).view(np.int64).copy())
    if device is not None:
        flat = flat.to(device)
    dist.all_reduce(flat)
    flat, out, at = flat.cpu().numpy().view(np.uint64), dict(inv), 0
    for k in names:
        out[k] = flat[at:at + inv[k].size].reshape(inv[k].shape).copy()
        at += inv[k].size
    return out
