// kernels_v1.cuh -- first-correct kernels: one thread per prompt / key / queue, tokens read
// straight from global memory.  Kept as the in-library cross-check for the warp-per-prompt
// and round-pipeline kernels (KVIDX_SCORE_KERNEL=v1) and used for the small, latency-insensitive entry points.
#pragma once
#include "score_common.cuh"

namespace kvx {

// ChunkedTokenDatabase.prefixHashes step (token_processor.go:115-123) for one block.
__device__ __forceinline__ uint64_t hash_block_global(uint64_t parent, const uint32_t* __restrict__ tok, uint32_t bs) {
    Fnv f;
    f.begin_block(parent, bs);
    for (uint32_t j = 0; j < bs; ++j) f.uint32(__ldg(tok + j));
    return f.end_block();
}

// TokensToKVBlockKeys (token_processor.go:141-162) for a CSR batch: thread per prompt.
__global__ void hash_keys_kernel_v1(TableView t, const uint32_t* __restrict__ tok, const int64_t* __restrict__ tok_off,
                                    int64_t tok_base, int64_t n_prompts, const uint64_t* __restrict__ parent,
                                    const uint8_t* __restrict__ parent_valid, const int64_t* __restrict__ key_off,
                                    int64_t key_base, uint64_t* __restrict__ keys_out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_prompts) return;
    const int64_t b = tok_off[i] - tok_base, e = tok_off[i + 1] - tok_base;
    const int64_t nblk = (e - b) / t.block_size;
    uint64_t h = t.init_hash;
    if (parent && (!parent_valid || parent_valid[i])) h = parent[i];
    uint64_t* out = keys_out + (key_off[i] - key_base);
    for (int64_t k = 0; k < nblk; ++k) {
        h = hash_block_global(h, tok + b + k * t.block_size, t.block_size);
        out[k] = h;
    }
}

// Index.Lookup (in_memory.go:105-146): thread per key.  (A FULL slot always holds >= 1 entry --
// Evict tombstones a slot the moment it empties -- so the present-but-empty cut of
// in_memory.go:119-122 cannot trigger; it is still honoured via cut_out for completeness.)
__global__ void lookup_kernel_v1(TableView t, uint32_t model, const uint64_t* __restrict__ keys, int64_t n,
                                 const uint64_t* __restrict__ filter, uint16_t* __restrict__ podtier_out,
                                 uint8_t* __restrict__ cnt_out, int* __restrict__ cut_out, unsigned long long stamp_base) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t* frow = filter_row(filter, 0, t.filter_words);
    SlotWords w;
    uint32_t c = 0;
    uint64_t slot = 0;
    if (req_find(t, model, keys[i], w, &slot)) {
        if (t.req_stamp) stamp_touch(t.req_stamp + slot, stamp_base + (unsigned long long)i);   // data.Get refreshes recency (in_memory.go:118)
        if (t.req_ref) ref_touch(t.req_ref, slot);
        const uint32_t cnt = meta_count(w.b.w);
        if (cnt == 0) atomicMin(cut_out, (int)min(i, (int64_t)0x7fffffff));
        for (uint32_t j = 0; j < cnt; ++j) {
            const uint32_t pt = slot_ent(w, j);
            if (frow && !filter_has(frow, pt >> 4)) continue;
            podtier_out[i * kMaxEnt + c++] = (uint16_t)pt;
        }
    }
    cnt_out[i] = (uint8_t)c;
}

// Indexer.GetPodScores steps 2-4 (indexer.go:141-163): thread per prompt.  Src is the prompt's source of block keys:
// uint32_t -- tokens, chained into keys as they are read (steps 2-4); uint64_t -- the request keys themselves (steps 3-4).
// src_off / src_base: the CSR of that source.  Exact-LRU mode: block k of prompt i is stamped
// stamp_base + (src_off[i] - src_off[0]) + k -- unique within the call and in prompt-then-block order, since k is below the
// prompt's element count -- so the call reserves src_off[n] - src_off[0] stamps.
template <class Src>
__global__ void score_kernel_v1(TableView t, const Src* __restrict__ src, const int64_t* __restrict__ src_off,
                                int64_t src_base, int64_t n_prompts, const uint32_t* __restrict__ model, uint32_t model0,
                                const uint64_t* __restrict__ filter, double* __restrict__ dense_out,
                                uint16_t* __restrict__ sp_pods, double* __restrict__ sp_scores, uint8_t* __restrict__ sp_cnt,
                                uint8_t* __restrict__ has_keys, unsigned long long stamp_base = 0) {
    constexpr bool kKeys = sizeof(Src) == 8;
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_prompts) return;
    const int64_t b = src_off[i] - src_base, e = src_off[i + 1] - src_base;
    const int64_t nblk = kKeys ? e - b : (e - b) / t.block_size;
    const uint32_t mdl = model ? model[i] : model0;
    const uint64_t* frow = filter_row(filter, i, t.filter_words);
    ScoreState s; s.k = 0; s.alive = 0;
    uint64_t h = t.init_hash;
    bool walking = true;
    for (int64_t k = 0; k < nblk; ++k) {
        if constexpr (kKeys) h = src[b + k];
        else h = hash_block_global(h, src + b + k * t.block_size, t.block_size);
        SlotWords w;
        uint64_t slot = 0;
        const bool hit = req_find(t, mdl, h, w, &slot);
        // exact-LRU mode: the reference's Lookup touches EVERY key of the prompt that is present, also past the end of
        // the consecutive prefix (in_memory.go:117-139), so the probe loop runs to the last block and stamps them.
        if (hit && t.req_stamp) stamp_touch(t.req_stamp + slot, stamp_base + (unsigned long long)(b + src_base - src_off[0] + k));
        if (walking) {
            if (!hit) walking = false;
            else {
                if (t.req_ref) ref_touch(t.req_ref, slot);                                // CLOCK: a block the walk looks at
                if (k == 0) s.first(t, w, frow); else s.next(t, w);
                if (!s.alive) walking = false;
            }
        }
        if (!walking && !t.req_stamp) break;
    }
    s.write_row(t, i, nblk > 0, dense_out, sp_pods, sp_scores, sp_cnt, has_keys);
}

}  // namespace kvx
