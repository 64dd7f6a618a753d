"""Spec of the keys a Score() call marks as referenced on a CLOCK handle (evict_policy="clock", include/kvidx.h), on top
of the reference oracle (oracle/kvoracle.py).

The reference's Lookup refreshes every present key of a prompt; the library keeps Score()'s early exit and marks the
present keys among the blocks its walk probes: block 0, then blocks 1, 2, ... up to and including the block whose probe
empties the active pod set (the prompt's pod filter applies), or the last full block.  A missing key is a gap: its block
empties the active set and it has nothing to mark.
"""
from oracle import kvoracle as ko


def walk_keys(index: ko.InMemoryIndex, keys, pod_filter=None):
    """The present keys among the blocks a Score() walk over `keys` probes.  Reads the index without refreshing it."""
    filt = set(pod_filter or ())
    out, active = [], None
    for i, k in enumerate(keys):
        pc = index.data.d.get(k)
        if pc is None:
            break
        out.append(k)
        pods = {e.pod for e in pc.keys() if not filt or e.pod in filt}
        active = pods if i == 0 else active & pods
        if not active:
            break
    return out


def referenced_keys(index: ko.InMemoryIndex, prompts, filters=None, block_size=16, hash_seed=""):
    """prompts: (tokens, model name) pairs; filters: None or one pod-name collection (or None) per prompt.
    -> the set of request Keys the batch marks."""
    tp = ko.ChunkedTokenDatabase(block_size, hash_seed)
    ref = set()
    for i, (tokens, model) in enumerate(prompts):
        keys = tp.tokens_to_kv_block_keys(None, list(tokens), model)
        ref.update(walk_keys(index, keys, None if filters is None else filters[i]))
    return ref
