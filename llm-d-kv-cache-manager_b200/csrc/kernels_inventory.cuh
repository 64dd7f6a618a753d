// kernels_inventory.cuh -- kvidx_pod_inventory: what each pod holds, counted on the device.
//
// An extension with no reference counterpart (the reference can answer no question about a pod).  Spec:
// tests/inventory_oracle.py.  Over the resident request keys k (of one model, or of all), with E(k) the key's entries:
//   entries[p][t]  keys with (p, t) in E(k)
//   keys[p]        keys with an entry of pod p on any tier (a pod on two tiers of one key counts once)
//   sole[p]        keys all of whose entries belong to pod p: the request keys kvidx_remove_pods({p}) removes
//   sole_engine[p] engine mappings whose request key is resident and counted in sole[p]: the engine keys it removes
//   totals         {request keys, entries, engine mappings, stale engine mappings (no resident request key)}
//
// Both kernels are READERS (table.cuh): one consistent image per FULL slot through the sequence-lock read, no slot, recency
// stamp or CLOCK reference bit is written, so an inventory never changes what a later sweep evicts, and it runs beside the
// write path on the read stream.  Beside a writer every key is counted before or after each individual Add / Evict of it.
//
//   inventory_req_kernel  streams the request slots.  Per-CTA histograms in shared memory, flushed once per CTA with 64-bit
//       atomics into the call's zeroed scratch.  keys[] and sole[] (2 x 4 B x max_pods, 32 KB at 4096 pods) always live in
//       shared memory.  The (pod, tier) histogram is 64 B per pod: up to kInvSharedPods pods (32 KB) it lives there too;
//       above that it would not fit an SM (256 KB at 4096 pods), so each entry goes to the global histogram directly, one
//       atomic per distinct bin of a warp (__match_any_sync) -- with thousands of pods the bins are many and cold.
//       A 32-bit shared bin cannot overflow: a slot adds at most 1 to a bin (the entries of a key are distinct, pods are
//       de-duplicated in registers), and a table that fits an 80 GB device has fewer than 2^32 slots.
//   inventory_eng_kernel  (only when asked for) streams the engine slots; each FULL mapping probes the request table of its
//       key's owner from the key's home (req_find: req_peer[] on a sharded handle, as remove_eng_kernel reaches it), is stale
//       if the probe ends without a FULL slot of the key, and counts into sole_engine[p] if that slot's entries all belong
//       to pod p.
// A sharded handle sweeps the slots this rank owns, so the per-rank results sum to the unsharded answer.
#pragma once
#include "table.cuh"
#include "kernels_remove.cuh"   // warp_add
#include "../../include/kvidx.h"

namespace kvx {

constexpr int kInvThreads = 256;
constexpr uint32_t kInvSharedPods = 512;    // (pod, tier) bins in shared memory up to this max_pods: 32 KB + 4 KB of keys / sole

struct InvArgs {
    uint32_t model;                     // KVIDX_ANY_MODEL: every model
    unsigned long long* entries;        // [max_pods * 16], pod * 16 + tier -- the packed entry itself
    unsigned long long* keys;           // [max_pods]
    unsigned long long* sole;           // [max_pods]
    unsigned long long* sole_engine;    // [max_pods]
    unsigned long long* totals;         // [4]
};

__host__ __device__ __forceinline__ size_t inv_req_smem(uint32_t max_pods) {
    return (size_t)max_pods * 4 * (2 + (max_pods <= kInvSharedPods ? KVIDX_MAX_TIERS : 0));
}

// the pod that owns every one of the `cnt` entries, or 0xffffffff
__device__ __forceinline__ uint32_t sole_pod(const EntList& L, uint32_t cnt) {
    const uint32_t p0 = L.e[0] >> KVIDX_TIER_BITS;
    bool one = cnt > 0;
#pragma unroll
    for (int j = 1; j < kMaxEnt; ++j) if ((uint32_t)j < cnt && (L.e[j] >> KVIDX_TIER_BITS) != p0) one = false;
    return one ? p0 : 0xffffffffu;
}

__device__ __forceinline__ void flush_bins(const uint32_t* bins, uint32_t n, unsigned long long* dst) {
    for (uint32_t b = threadIdx.x; b < n; b += blockDim.x) if (bins[b]) atomicAdd(dst + b, (unsigned long long)bins[b]);
}

__global__ void __launch_bounds__(kInvThreads) inventory_req_kernel(TableView t, InvArgs r) {
    extern __shared__ uint32_t inv_sh[];
    const uint32_t P = t.max_pods;
    const bool ent_shared = P <= kInvSharedPods;
    uint32_t* h_keys = inv_sh;
    uint32_t* h_sole = inv_sh + P;
    uint32_t* h_ent = inv_sh + 2 * P;
    for (uint32_t b = threadIdx.x; b < inv_req_smem(P) / 4; b += blockDim.x) inv_sh[b] = 0;
    __syncthreads();
    unsigned long long n_key = 0, n_ent = 0;
    const bool sys = t.shard_bits != 0;
    const uint64_t slots = t.req_mask + 1, stride = (uint64_t)gridDim.x * blockDim.x;
    const uint32_t lane = threadIdx.x & 31;
    // the warp walks 32 consecutive slots together (every lane makes every trip: the global path votes across the warp)
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x + (threadIdx.x & ~31u); base < slots; base += stride) {
        const uint64_t i = base + lane;
        uint32_t cnt = 0;
        EntList L{};
        if (i < slots) {
            uint4 a, b;
            ld_slot(t.req + i, sys, a, b);
            if (meta_state(b.w) == kStateFull && (r.model == KVIDX_ANY_MODEL || meta_model(b.w) == r.model)) {
                cnt = meta_count(b.w);
                L.unpack(a, b);
                ++n_key;
                n_ent += cnt;
                const uint32_t sp = sole_pod(L, cnt);
                if (sp < P) atomicAdd(&h_sole[sp], 1u);
            }
        }
#pragma unroll
        for (int j = 0; j < kMaxEnt; ++j) {
            const uint32_t e = L.e[j], p = e >> KVIDX_TIER_BITS;
            const bool live = (uint32_t)j < cnt && p < P;       // Add refuses pod >= max_pods; the index is bounded anyway
            if (live) {
                bool first = true;                               // first entry of this pod in the slot
#pragma unroll
                for (int q = 0; q < j; ++q) if ((L.e[q] >> KVIDX_TIER_BITS) == p) first = false;
                if (first) atomicAdd(&h_keys[p], 1u);
                if (ent_shared) atomicAdd(&h_ent[e], 1u);
            }
            if (!ent_shared && __any_sync(0xffffffffu, live)) {
                const uint32_t same = __match_any_sync(0xffffffffu, live ? e : 0xffffffffu);
                if (live && lane == (uint32_t)__ffs(same) - 1) atomicAdd(r.entries + e, (unsigned long long)__popc(same));
            }
        }
    }
    __syncthreads();
    flush_bins(h_keys, P, r.keys);
    flush_bins(h_sole, P, r.sole);
    if (ent_shared) flush_bins(h_ent, P * KVIDX_MAX_TIERS, r.entries);
    warp_add(&r.totals[0], n_key);
    warp_add(&r.totals[1], n_ent);
}

__global__ void __launch_bounds__(kInvThreads) inventory_eng_kernel(TableView t, InvArgs r) {
    extern __shared__ uint32_t inv_sh[];                         // sole_engine bins, max_pods of them
    const uint32_t P = t.max_pods;
    for (uint32_t b = threadIdx.x; b < P; b += blockDim.x) inv_sh[b] = 0;
    __syncthreads();
    unsigned long long n_eng = 0, n_stale = 0;
    const bool sys = t.shard_bits != 0;
    const uint64_t slots = t.eng_mask + 1, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < slots; i += stride) {
        uint4 a, b;
        ld_slot_t<0>(t.eng + i, sys, a, b);
        if (meta_state(b.x) != kStateFull) continue;
        const uint32_t model = meta_model(b.x);
        if (r.model != KVIDX_ANY_MODEL && model != r.model) continue;
        ++n_eng;
        SlotWords w;
        if (!req_find(t, model, ((uint64_t)a.w << 32) | a.z, w)) { ++n_stale; continue; }
        EntList L; L.unpack(w.a, w.b);
        const uint32_t sp = sole_pod(L, meta_count(w.b.w));
        if (sp < P) atomicAdd(&inv_sh[sp], 1u);
    }
    __syncthreads();
    flush_bins(inv_sh, P, r.sole_engine);
    warp_add(&r.totals[2], n_eng);
    warp_add(&r.totals[3], n_stale);
}

}  // namespace kvx
