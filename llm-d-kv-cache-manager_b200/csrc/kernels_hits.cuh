// kernels_hits.cuh -- the hit count of a full-depth Lookup, for a batch of prompts: recordHitMetrics(Lookup(K_i, F_i))
// (kvblock/instrumented_index.go:71-92 over in_memory.go:105-146).  For every pod, its entries in the result map; the
// largest of those counts is the prompt's hit count.  The Score() kernels stop at the end of the consecutive prefix, so
// they cannot give it: this kernel probes every key of every prompt.
//
// One CTA per prompt (grid-stride).  Threads take the prompt's keys coalesced and probe them independently (the probes have
// no order between them, so all of them are in flight at once), touch what they find as kvidx_lookup does, and count the
// entries into per-pod shared-memory counters.  The map decides what counts:
//   * with a filter row, Lookup appends per occurrence (in_memory.go:130-135): every occurrence of a key counts;
//   * without one, it assigns podsPerKey[key] (:126-128): a key repeated in the prompt counts once.  The prompt's keys are
//     taken in chunks of kHitsChunk; each chunk's keys go into an open-addressed set in shared memory, and the one
//     occurrence that claims the key's set slot counts -- unless the key also occurs in an earlier chunk, which a scan of
//     the earlier keys against the set finds.  Prompts of at most kHitsChunk keys (all but the longest) need no scan.
// The present-but-empty cut of in_memory.go:119-122 cannot trigger: a FULL slot always holds at least one entry (Evict
// tombstones a slot the moment it empties, kernels_v1.cuh), so no code stands for it.
// Counters are cleared after each prompt only where it touched them: the first increment of a pod's counter appends the
// pod to a list, and the list is walked at the end of the prompt.
#pragma once
#include "score_common.cuh"

namespace kvx {

constexpr int kHitsThreads = 128;
constexpr int kHitsChunk = 1024;                 // keys per chunk of an unfiltered prompt (8 per thread)
constexpr int kHitsSet = 2 * kHitsChunk;         // slots of the chunk's key set: load <= 1/2
constexpr int kHitsCtasPerSm = 8;
static_assert(kHitsChunk / kHitsThreads <= 32, "a thread's chunk positions fit one mask word");

struct HitsSmem {
    uint32_t set[kHitsSet];                      // 1 + the chunk position that claimed the slot; 0 = empty
    uint8_t dup[kHitsChunk];                     // the key at this chunk position also occurs in an earlier chunk
    uint32_t wmax[kHitsThreads / 32];
    uint32_t ntouched[2];                        // pods in the touched list, by prompt parity
};
// dynamic shared memory: uint32_t cnt[max_pods], then uint16_t touched[max_pods]
inline size_t hits_dyn_smem(uint32_t max_pods) { return (size_t)max_pods * (sizeof(uint32_t) + sizeof(uint16_t)); }

__device__ __forceinline__ uint32_t hits_set_home(uint64_t key) { return (uint32_t)home_of(key, 0) & (kHitsSet - 1); }

// Claims a set slot for ck[j] unless an earlier claim holds the same key: true when this position claimed it.
__device__ __forceinline__ bool hits_set_claim(uint32_t* set, const uint64_t* __restrict__ ck, uint64_t key, uint32_t j) {
    for (uint32_t s = hits_set_home(key);; s = (s + 1) & (kHitsSet - 1)) {
        const uint32_t old = atomicCAS(set + s, 0u, j + 1);
        if (old == 0) return true;
        if (ck[old - 1] == key) return false;
    }
}
// The chunk position holding `key` in the (complete) set, or -1.
__device__ __forceinline__ int hits_set_find(const uint32_t* set, const uint64_t* __restrict__ ck, uint64_t key) {
    for (uint32_t s = hits_set_home(key);; s = (s + 1) & (kHitsSet - 1)) {
        const uint32_t e = set[s];
        if (e == 0) return -1;
        if (ck[e - 1] == key) return (int)e - 1;
    }
}

// keys / key_off / key_base: CSR, prompt i owns keys[key_off[i] - key_base .. key_off[i + 1] - key_base).  Exact-LRU: key k of
// prompt i is stamped stamp_base + (key_off[i] - key_off[0]) + k, the layout of every Score() path.
__global__ void __launch_bounds__(kHitsThreads)
lookup_hits_kernel(TableView t, const uint64_t* __restrict__ keys, const int64_t* __restrict__ key_off, int64_t key_base, int64_t n,
                   const uint32_t* __restrict__ model, uint32_t model0, const uint64_t* __restrict__ filter,
                   uint32_t* __restrict__ hits_out, unsigned long long stamp_base) {
    __shared__ HitsSmem sm;
    extern __shared__ uint32_t hits_dyn[];
    uint32_t* cnt = hits_dyn;
    uint16_t* touched = reinterpret_cast<uint16_t*>(hits_dyn + t.max_pods);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (uint32_t p = tid; p < t.max_pods; p += kHitsThreads) cnt[p] = 0;
    for (int s = tid; s < kHitsSet; s += kHitsThreads) sm.set[s] = 0;
    for (int s = tid; s < kHitsChunk; s += kHitsThreads) sm.dup[s] = 0;
    if (tid < 2) sm.ntouched[tid] = 0;
    __syncthreads();
    const int64_t off0 = key_off[0];
    uint32_t par = 0;
    for (int64_t i = blockIdx.x; i < n; i += gridDim.x, par ^= 1u) {
        const int64_t b = key_off[i] - key_base, nk = key_off[i + 1] - key_off[i];
        const uint32_t mdl = model ? model[i] : model0;
        const uint64_t* frow = filter_row(filter, i, t.filter_words);
        const unsigned long long sb = stamp_base + (unsigned long long)(key_off[i] - off0);
        uint32_t mx = 0;
        // key k of the prompt: probe and touch it; add its (filtered) entries to the pod counters when it counts
        auto probe = [&](int64_t k, bool counts) {
            SlotWords w;
            uint64_t slot = 0;
            if (!req_find(t, mdl, keys[b + k], w, &slot)) return;
            if (t.req_stamp) stamp_touch(t.req_stamp + slot, sb + (unsigned long long)k);    // data.Get (in_memory.go:118)
            if (t.req_ref) ref_touch(t.req_ref, slot);
            if (!counts) return;
            const uint32_t c = meta_count(w.b.w);
            for (uint32_t j = 0; j < c; ++j) {
                const uint32_t p = slot_ent(w, j) >> 4;
                if (p >= t.max_pods || (frow && !filter_has(frow, p))) continue;
                const uint32_t old = atomicAdd(cnt + p, 1u);
                if (old == 0) touched[atomicAdd(&sm.ntouched[par], 1u)] = (uint16_t)p;
                mx = max(mx, old + 1);
            }
        };
        if (frow) {
            for (int64_t k = tid; k < nk; k += kHitsThreads) probe(k, true);
        } else {
            for (int64_t c0 = 0; c0 < nk; c0 += kHitsChunk) {
                const int cn = (int)min((int64_t)kHitsChunk, nk - c0);
                const uint64_t* ck = keys + b + c0;
                if (c0 == 0) {                    // no earlier chunk: a claim decides at once
                    for (int j = tid; j < cn; j += kHitsThreads) probe(j, hits_set_claim(sm.set, ck, ck[j], (uint32_t)j));
                    continue;
                }
                __syncthreads();                  // the previous chunk is done with the set
                for (int s = tid; s < kHitsSet; s += kHitsThreads) sm.set[s] = 0;
                __syncthreads();
                uint32_t claimed = 0;             // bit q: position tid + q * kHitsThreads claimed its key
                for (int j = tid, q = 0; j < cn; j += kHitsThreads, ++q)
                    if (hits_set_claim(sm.set, ck, ck[j], (uint32_t)j)) claimed |= 1u << q;
                __syncthreads();
                for (int64_t e = tid; e < c0; e += kHitsThreads) {
                    const int f = hits_set_find(sm.set, ck, keys[b + e]);
                    if (f >= 0) sm.dup[f] = 1;
                }
                __syncthreads();
                for (int j = tid, q = 0; j < cn; j += kHitsThreads, ++q) probe(c0 + j, ((claimed >> q) & 1u) && !sm.dup[j]);
                __syncthreads();                  // dup is read; clear it for the next chunk
                for (int s = tid; s < kHitsChunk; s += kHitsThreads) sm.dup[s] = 0;
            }
        }
        mx = __reduce_max_sync(0xffffffffu, mx);
        if (lane == 0) sm.wmax[warp] = mx;
        __syncthreads();
        // the prompt's counters, set and (multi-chunk) flags back to zero; the other parity's list length too (its last
        // readers finished before the previous prompt's final barrier)
        const uint32_t nt = sm.ntouched[par];
        for (uint32_t k = tid; k < nt; k += kHitsThreads) cnt[touched[k]] = 0;
        if (!frow && nk > 0) for (int s = tid; s < kHitsSet; s += kHitsThreads) sm.set[s] = 0;
        if (tid == 0) {
            uint32_t m = 0;
            for (int q = 0; q < kHitsThreads / 32; ++q) m = max(m, sm.wmax[q]);
            hits_out[i] = m;
            sm.ntouched[par ^ 1u] = 0;
        }
        __syncthreads();
    }
}

// The block counts of a token CSR, the input of the in-place scan that lays out its keys: koff[0] = 0,
// koff[i + 1] = floor(len_i / bs).
__global__ void block_counts_kernel(const int64_t* __restrict__ tok_off, int64_t n, uint32_t bs, int64_t* __restrict__ koff) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i == 0) koff[0] = 0;
    if (i < n) koff[i + 1] = (tok_off[i + 1] - tok_off[i]) / bs;
}

}  // namespace kvx
