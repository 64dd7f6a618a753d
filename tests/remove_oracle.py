"""Spec of pod removal (kvidx_remove_pods / kvhost_remove_pod), on top of the reference oracle (oracle/kvoracle.py).

An extension with no reference counterpart: the reference's index has no operation that drops the blocks of a pod that
went away without sending BlockRemoved events, and its digestEvents ignores AllBlocksCleared (pool.go:332-333).
"""
from oracle import kvoracle as ko


def remove_pods(index: ko.InMemoryIndex, pods, tiers=None):
    """Drop every entry of `pods` on `tiers` (None = all tiers) from the oracle's InMemoryIndex.

    Survivors keep their order and no key's recency changes, in the key LRU, the engine LRU or a pod cache.  A request key
    left without entries is removed, and so is every engine mapping that points at a key removed by THIS call; a mapping
    whose key was already absent stays (a stale mapping, which Evict cleans up, in_memory.go:225-230).
    Returns (entries, request keys, engine keys) removed."""
    pods, tiers = set(pods), None if tiers is None else set(tiers)
    n_ent, removed = 0, set()
    for rk, pc in list(index.data.d.items()):
        drop = [e for e in pc.keys() if e.pod in pods and (tiers is None or e.tier in tiers)]
        for e in drop:
            pc.remove(e)
        n_ent += len(drop)
        if drop and len(pc) == 0:
            index.data.remove(rk)
            removed.add(rk)
    gone = [ek for ek, rk in index.engine_to_request.d.items() if rk in removed]
    for ek in gone:
        index.engine_to_request.remove(ek)
    return n_ent, len(removed), len(gone)


class ClearingEventsPool(ko.EventsPool):
    """EventsPool with the host mirror's opt-in clear_on_all_blocks_cleared: an AllBlocksCleared from pod P removes P's
    entries on the tier of a Medium-less event ("gpu", pool.go:258-261) at its position in P's event order (vLLM sends it
    when the GPU prefix cache is reset; blocks offloaded to other media survive).  Every other event is digested as the
    reference does."""

    def digest_events(self, pod, model, events):
        for ev in events:
            if isinstance(ev, ko.AllBlocksCleared):
                remove_pods(self.index, {pod}, {ko.medium_tier(None)})
            else:
                super().digest_events(pod, model, [ev])
