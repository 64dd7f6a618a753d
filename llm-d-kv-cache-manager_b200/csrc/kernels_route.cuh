// kernels_route.cuh -- the pieces of the ROUTED form of the sharded Score() (SURVEY 8(e) as first drafted): hash everything at
// the origin, send each key to the rank that owns its hash range (all-to-all #1), let the owner read the slot, send the 32-byte
// slot image back (all-to-all #2), walk and score at the origin.  The exchange itself is NCCL (torch.distributed
// all_to_all_single in kvidx/dist.py::score_alltoall); these kernels are what runs before, between and after.
//
// It exists to be MEASURED against the path the library actually takes on a sharded handle -- probing the owner's shard
// straight from the walk over NVLink peer memory (table.cuh: req_peer[]), which moves only the slots the walk really needs
// (it stops at the first miss and shares prefixes between prompts) instead of every key of every prompt.
//
// Same reference semantics as everywhere: Lookup (in_memory.go:105-146), LongestPrefixScorer.Score (kvblock_scorer.go:108-151).
#pragma once
#include "kernels_v1.cuh"

namespace kvx {

// owner shard of every key (the top bits of the mixed key: table.cuh shard_of)
__global__ void key_owners_kernel(TableView t, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ model, uint32_t model0,
                                  int64_t n, uint8_t* __restrict__ owner) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) owner[i] = (uint8_t)shard_of(home_of(keys[i], model ? model[i] : model0), t.shard_bits);
}

// owner side: the slot image of every key (all zero: the key is not in the index)
__global__ void probe_slots_kernel(TableView t, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ model, uint32_t model0,
                                   int64_t n, uint4* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    SlotWords w;
    const bool hit = req_find(t, model ? model[i] : model0, keys[i], w);
    out[2 * i] = hit ? w.a : make_uint4(0, 0, 0, 0);
    out[2 * i + 1] = hit ? w.b : make_uint4(0, 0, 0, 0);
}

// origin side: the consecutive-prefix walk over the returned images, thread per prompt
__global__ void score_slots_kernel(TableView t, const uint4* __restrict__ slots, const int64_t* __restrict__ key_off, int64_t n_prompts,
                                   const uint64_t* __restrict__ filter, double* __restrict__ dense_out, uint8_t* __restrict__ has_keys) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_prompts) return;
    const int64_t k0 = key_off[i], k1 = key_off[i + 1];
    const uint64_t* frow = filter_row(filter, i, t.filter_words);
    ScoreState s; s.k = 0; s.alive = 0;
    for (int64_t k = k0; k < k1; ++k) {
        SlotWords w; w.a = slots[2 * k]; w.b = slots[2 * k + 1];
        if (meta_state(w.b.w) != kStateFull) break;
        if (k == k0) s.first(t, w, frow); else s.next(t, w);
        if (!s.alive) break;
    }
    s.write_row(t, i, k1 > k0, dense_out, nullptr, nullptr, nullptr, has_keys);
}

}  // namespace kvx
