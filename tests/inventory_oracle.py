"""Spec of the pod inventory (kvidx_pod_inventory / kvhost_pod_inventory), on top of the reference oracle (oracle/kvoracle.py).

An extension with no reference counterpart: the reference's index answers questions about a prompt, none about a pod.
Nothing here refreshes recency: the LRUs are read through their dictionaries, never through get().
"""
from collections import Counter

from oracle import kvoracle as ko


def pod_inventory(index: ko.InMemoryIndex, model=None, engine=False):
    """Over the resident request keys k (of `model`, None = every model), with E(k) the key's (pod, tier) entries:
      entries[(p, t)]  keys with (p, t) in E(k)
      keys[p]          keys with an entry of pod p on any tier
      sole[p]          keys all of whose entries belong to pod p -- the request keys remove_pods({p}) removes
      sole_engine[p]   engine mappings (of `model`) whose request key is resident and counted in sole[p] -- the engine keys
                       remove_pods({p}) removes; None without `engine`
      totals           [request keys, entries, engine mappings, stale engine mappings]; a mapping is stale when its request
                       key is not resident.  The last two are 0 without `engine`.
    Counters are keyed by names; absent means 0."""
    entries, keys, sole, sole_key = Counter(), Counter(), Counter(), {}
    totals = [0, 0, 0, 0]
    for rk, pc in index.data.d.items():
        if model is not None and rk.model != model:
            continue
        ents = pc.keys()
        totals[0] += 1
        totals[1] += len(ents)
        for e in ents:
            entries[(e.pod, e.tier)] += 1
        pods = {e.pod for e in ents}
        for p in pods:
            keys[p] += 1
        if len(pods) == 1:
            (p,) = pods
            sole[p] += 1
            sole_key[rk] = p
    sole_engine = None
    if engine:
        sole_engine = Counter()
        for ek, rk in index.engine_to_request.d.items():
            if model is not None and ek.model != model:
                continue
            totals[2] += 1
            if rk not in index.data.d:
                totals[3] += 1
            elif rk in sole_key:
                sole_engine[sole_key[rk]] += 1
    return {"entries": entries, "keys": keys, "sole": sole, "sole_engine": sole_engine, "totals": totals}


def dense(inv, pod_id, tier_id, max_pods):
    """The spec's counters as the arrays kvidx.Index.pod_inventory returns; pod_id / tier_id map names to ids."""
    import numpy as np
    out = {"entries": np.zeros((max_pods, 16), np.uint64), "keys": np.zeros(max_pods, np.uint64), "sole": np.zeros(max_pods, np.uint64),
           "sole_engine": None if inv["sole_engine"] is None else np.zeros(max_pods, np.uint64), "totals": np.array(inv["totals"], np.uint64)}
    for (p, t), c in inv["entries"].items():
        out["entries"][pod_id(p), tier_id(t)] = c
    for name in ("keys", "sole", "sole_engine"):
        for p, c in (inv[name] or {}).items():
            out[name][pod_id(p)] = c
    return out
