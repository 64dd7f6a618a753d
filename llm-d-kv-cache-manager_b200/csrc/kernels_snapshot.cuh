// kernels_snapshot.cuh -- kvidx_snapshot / kvidx_restore: the index as a canonical image (format v1, include/kvidx.h).
//
// An extension with no reference counterpart: vLLM sends BlockStored once, when a block is first cached, so an indexer
// that starts empty cannot relearn the blocks already cached in the fleet.  An image taken from a running handle and
// restored into a fresh one (after a restart, an upgrade, on another GPU, or into a larger table) carries them over.
// Spec: tests/snapshot_oracle.py.
//
// Export (the caller holds mu_w: no writer runs, readers may):
//   snap_compact_kernel   grid-stride sweep of one table; every FULL slot appends (tag, slot index) with one atomic per
//                         warp (ballot + popc).  The largest model id + 1 is reduced on the side.
//   cub::DeviceRadixSort  by tag (64 bits), then -- only when more than one model is present -- stably by model (as many
//                         bits as the largest model id needs): (model, hash) order, the canonical one.
//   snap_*_records_kernel thread per record: the sorted slots become records (and recency stamps in exact-LRU mode).
// Import (the caller holds mu_w; the target has no live key):
//   snap_check_*_kernel   every record before anything is inserted: strict (model, hash) order (so no duplicates),
//                         1 <= count <= pods_per_key, distinct entries with pod < max_pods, zero entries past count,
//                         zero padding, stamps below 2^63.  The largest pod id + 1, model id + 1 and stamp are reduced so
//                         that the host can hold them against the header and advance the recency clock.
//   cub::DeviceRadixSort  images with recency: each section's stamps, sorted; snap_check_ties_kernel refuses a repeated
//                         value, and the sorted stamps give the exact-LRU cut to `capacity` as one threshold per table.
//   restore_*_kernel      thread per record at or above its table's threshold: claims a slot from the key's home with the compare-and-swap EMPTY -> BUSY and
//                         publishes the image with the two-half protocol of table.cuh, as rebuild_*_kernel does, so a
//                         concurrent reader sees each key either absent or whole.
// Sharded import (kvidx_shard_restore): every rank reads the WHOLE image and inserts only the records it owns.
//   snap_owner_hist_kernel records per owning shard in each section, so that every rank can hold every owner's share
//                         against the room of a shard before any rank inserts (the verdict depends only on the image
//                         and the common geometry, so all ranks reach the same one).
//   restore_*_kernel      skip a record whose key another shard owns (unsharded: shard 0 owns every key).
#pragma once
#include "table.cuh"
#include "../../include/kvidx.h"

namespace kvx {

constexpr int kSnapThreads = 256;

// flags of SnapCheck::bad
constexpr unsigned int kSnapBadOrder = 1u, kSnapBadCount = 2u, kSnapBadEntry = 4u, kSnapBadPad = 8u, kSnapBadStamp = 16u, kSnapBadTie = 32u;

struct SnapCheck {
    unsigned int bad;                 // kSnapBad* of every failed record, OR-ed
    unsigned int pod_span;            // 1 + largest pod id in any entry (0: none)
    unsigned int model_span;          // 1 + largest model id in any record (0: none)
    unsigned int pad;
    unsigned long long first_bad;     // smallest failing record index (per table: request records, then engine records)
    unsigned long long stamp_max;
};

struct SnapMisc {                     // export side
    unsigned long long n;             // records appended by the sweep
    unsigned int model_span, pod_span;
};

// All lanes of a warp must call these (the loops below give every lane the same trip count).
__device__ __forceinline__ unsigned long long warp_append(bool take, unsigned long long* n) {
    const uint32_t m = __ballot_sync(0xffffffffu, take);
    const uint32_t lane = threadIdx.x & 31;
    unsigned long long base = 0;
    if (lane == 0 && m) base = atomicAdd(n, (unsigned long long)__popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    return base + (unsigned long long)__popc(m & ((1u << lane) - 1u));
}
__device__ __forceinline__ void warp_max_u32(unsigned int* dst, unsigned int v) {
    v = __reduce_max_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && v) atomicMax(dst, v);
}

// kMeta: index of the meta word in half b (3: request table, 0: engine table).  slots is a power of two >= 1024, so every
// lane of a warp runs the same number of iterations.
template <int kMeta>
__global__ void __launch_bounds__(kSnapThreads) snap_compact_kernel(const uint4* __restrict__ tab, uint64_t slots, uint64_t cap,
                                                                    uint64_t* __restrict__ key, uint32_t* __restrict__ idx, SnapMisc* misc) {
    unsigned int mspan = 0;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < slots; i += stride) {
        const uint4 b = tab[2 * i + 1];
        const uint32_t m = kMeta == 3 ? b.w : b.x;
        const bool full = meta_state(m) == kStateFull;
        uint64_t tag = 0;
        if (full) {
            const uint4 a = tab[2 * i];
            tag = ((uint64_t)a.y << 32) | a.x;
            mspan = max(mspan, meta_model(m) + 1u);
        }
        const unsigned long long pos = warp_append(full, &misc->n);
        if (full && pos < cap) { key[pos] = tag; idx[pos] = (uint32_t)i; }
    }
    warp_max_u32(&misc->model_span, mspan);
}

// model id of each sorted slot: the key of the second (stable) sort pass
template <int kMeta>
__global__ void snap_models_kernel(const uint4* __restrict__ tab, const uint32_t* __restrict__ idx, uint64_t n, uint16_t* __restrict__ model) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4 b = tab[2 * (uint64_t)idx[i] + 1];
    model[i] = (uint16_t)meta_model(kMeta == 3 ? b.w : b.x);
}

// request record (32 B): {hash.lo, hash.hi, model | count << 16, ent0 | ent1 << 16} {ent2|3, ent4|5, ent6|7, ent8|9}
__global__ void __launch_bounds__(kSnapThreads) snap_req_records_kernel(const ReqSlot* __restrict__ tab, const uint32_t* __restrict__ idx, uint64_t n,
                                                                        uint4* __restrict__ rec, const unsigned long long* __restrict__ req_stamp,
                                                                        unsigned long long* __restrict__ stamp_out, SnapMisc* misc) {
    unsigned int pspan = 0;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += stride) {
        const uint64_t i = base + threadIdx.x;
        if (i < n) {
            const uint64_t s = idx[i];
            const uint4* p = reinterpret_cast<const uint4*>(tab + s);
            const uint4 a = p[0], b = p[1];
            const uint32_t cnt = meta_count(b.w);
            EntList L; L.unpack(a, b);
#pragma unroll
            for (int j = 0; j < kMaxEnt; ++j) {
                if ((uint32_t)j >= cnt) L.e[j] = 0;                 // canonical: nothing past count
                else pspan = max(pspan, (L.e[j] >> KVIDX_TIER_BITS) + 1u);
            }
            rec[2 * i] = make_uint4(a.x, a.y, meta_model(b.w) | (cnt << 16), L.e[0] | (L.e[1] << 16));
            rec[2 * i + 1] = make_uint4(L.e[2] | (L.e[3] << 16), L.e[4] | (L.e[5] << 16), L.e[6] | (L.e[7] << 16), L.e[8] | (L.e[9] << 16));
            if (stamp_out) stamp_out[i] = req_stamp[s];
        }
    }
    warp_max_u32(&misc->pod_span, pspan);
}

// engine record (24 B): {engine hash, request hash, model (u16) + 6 zero bytes}
__global__ void snap_eng_records_kernel(const EngSlot* __restrict__ tab, const uint32_t* __restrict__ idx, uint64_t n,
                                        unsigned long long* __restrict__ rec, unsigned long long* __restrict__ stamp_out) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4* p = reinterpret_cast<const uint4*>(tab + idx[i]);
    const uint4 a = p[0], b = p[1];
    rec[3 * i] = ((unsigned long long)a.y << 32) | a.x;
    rec[3 * i + 1] = ((unsigned long long)a.w << 32) | a.z;
    rec[3 * i + 2] = meta_model(b.x);
    if (stamp_out) stamp_out[i] = ((unsigned long long)b.w << 32) | b.z;
}

// ---- import --------------------------------------------------------------------------------------------------------

__device__ __forceinline__ void check_reduce(SnapCheck* c, unsigned int bad, unsigned long long first, unsigned int pspan,
                                             unsigned int mspan, unsigned long long smax) {
    bad = __reduce_or_sync(0xffffffffu, bad);
    pspan = __reduce_max_sync(0xffffffffu, pspan);
    mspan = __reduce_max_sync(0xffffffffu, mspan);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
        smax = max(smax, __shfl_xor_sync(0xffffffffu, smax, o));
    }
    if ((threadIdx.x & 31) == 0) {
        if (bad) { atomicOr(&c->bad, bad); atomicMin(&c->first_bad, first); }
        if (pspan) atomicMax(&c->pod_span, pspan);
        if (mspan) atomicMax(&c->model_span, mspan);
        if (smax) atomicMax(&c->stamp_max, smax);
    }
}

__global__ void __launch_bounds__(kSnapThreads) snap_check_req_kernel(const uint4* __restrict__ rec, uint64_t n, const unsigned long long* __restrict__ stamp,
                                                                      uint32_t pods_per_key, uint32_t max_pods, SnapCheck* c) {
    unsigned int bad = 0, pspan = 0, mspan = 0;
    unsigned long long first = ~0ull, smax = 0;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += stride) {
        const uint64_t i = base + threadIdx.x;
        if (i >= n) continue;
        const uint4 a = rec[2 * i], b = rec[2 * i + 1];
        const uint64_t hash = ((uint64_t)a.y << 32) | a.x;
        const uint32_t model = a.z & 0xffffu, cnt = (a.z >> 16) & 0xffu;
        unsigned int f = 0;
        if (a.z >> 24) f |= kSnapBadPad;
        if (i > 0) {
            const uint4 q = rec[2 * (i - 1)];
            const uint64_t ph = ((uint64_t)q.y << 32) | q.x;
            const uint32_t pm = q.z & 0xffffu;
            if (!(pm < model || (pm == model && ph < hash))) f |= kSnapBadOrder;
        }
        if (cnt < 1 || cnt > pods_per_key) f |= kSnapBadCount;
        uint32_t e[kMaxEnt] = {a.w & 0xffffu, a.w >> 16, b.x & 0xffffu, b.x >> 16, b.y & 0xffffu, b.y >> 16,
                               b.z & 0xffffu, b.z >> 16, b.w & 0xffffu, b.w >> 16};
#pragma unroll
        for (int j = 0; j < kMaxEnt; ++j) {
            if ((uint32_t)j < cnt) {
                const uint32_t pod = e[j] >> KVIDX_TIER_BITS;
                if (pod >= max_pods) f |= kSnapBadEntry;
                pspan = max(pspan, pod + 1u);
#pragma unroll
                for (int k = j + 1; k < kMaxEnt; ++k)
                    if ((uint32_t)k < cnt && e[k] == e[j]) f |= kSnapBadEntry;
            } else if (e[j]) {
                f |= kSnapBadPad;
            }
        }
        mspan = max(mspan, model + 1u);
        if (stamp) {
            const unsigned long long s = stamp[i];
            if (s >> 63) f |= kSnapBadStamp;
            smax = max(smax, s);
        }
        if (f) { bad |= f; first = min(first, (unsigned long long)i); }
    }
    check_reduce(c, bad, first, pspan, mspan, smax);
}

__global__ void __launch_bounds__(kSnapThreads) snap_check_eng_kernel(const unsigned long long* __restrict__ rec, uint64_t n,
                                                                      const unsigned long long* __restrict__ stamp, SnapCheck* c) {
    unsigned int bad = 0, mspan = 0;
    unsigned long long first = ~0ull, smax = 0;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += stride) {
        const uint64_t i = base + threadIdx.x;
        if (i >= n) continue;
        const unsigned long long eh = rec[3 * i], w = rec[3 * i + 2];
        const uint32_t model = (uint32_t)(w & 0xffffu);
        unsigned int f = 0;
        if (w >> 16) f |= kSnapBadPad;
        if (i > 0) {
            const unsigned long long peh = rec[3 * (i - 1)];
            const uint32_t pm = (uint32_t)(rec[3 * (i - 1) + 2] & 0xffffu);
            if (!(pm < model || (pm == model && peh < eh))) f |= kSnapBadOrder;
        }
        mspan = max(mspan, model + 1u);
        if (stamp) {
            const unsigned long long s = stamp[i];
            if (s >> 63) f |= kSnapBadStamp;
            smax = max(smax, s);
        }
        if (f) { bad |= f; first = min(first, (unsigned long long)i); }
    }
    check_reduce(c, bad, first, 0u, mspan, smax);
}

// recency values of one section, sorted: a repeated value would make the LRU cut drop every tied key at once
__global__ void __launch_bounds__(kSnapThreads) snap_check_ties_kernel(const unsigned long long* __restrict__ sorted, uint64_t n, SnapCheck* c) {
    unsigned int bad = 0;
    unsigned long long first = ~0ull;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += stride) {
        const uint64_t i = base + threadIdx.x;
        if (i == 0 || i >= n) continue;
        if (sorted[i] == sorted[i - 1]) { bad = kSnapBadTie; first = min(first, (unsigned long long)i); }
    }
    check_reduce(c, bad, first, 0u, 0u, 0ull);
}

// sum over the warp, one atomic per warp
__device__ __forceinline__ void warp_sum_add(unsigned long long* dst, unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(dst, v);
}

// counts[o]: request records owned by shard o, counts[8 + o]: engine records (shard = top shard_bits of the mixed key)
__global__ void __launch_bounds__(kSnapThreads) snap_owner_hist_kernel(const uint4* __restrict__ req_rec, uint64_t R,
                                                                       const unsigned long long* __restrict__ eng_rec, uint64_t E,
                                                                       uint32_t shard_bits, unsigned long long* counts) {
    __shared__ unsigned long long h[16];
    if (threadIdx.x < 16) h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < R + E; i += stride) {
        uint64_t hash; uint32_t model, sect;
        if (i < R) {
            const uint4 a = req_rec[2 * i];
            hash = ((uint64_t)a.y << 32) | a.x; model = a.z & 0xffffu; sect = 0;
        } else {
            const uint64_t k = i - R;
            hash = eng_rec[3 * k]; model = (uint32_t)(eng_rec[3 * k + 2] & 0xffffu); sect = 8;
        }
        atomicAdd(&h[sect + shard_of(home_of(hash, model), shard_bits)], 1ull);
    }
    __syncthreads();
    if (threadIdx.x < 16 && h[threadIdx.x]) atomicAdd(&counts[threadIdx.x], h[threadIdx.x]);
}

// stamp: the record's recency stamp, or nullptr (default mode, or an image without recency)
// keep_from: records whose stamp is below it are not inserted (the exact-LRU cut to `capacity`, done before inserting)
__global__ void __launch_bounds__(kSnapThreads) restore_req_kernel(TableView t, const uint4* __restrict__ rec, uint64_t n,
                                                                   const unsigned long long* __restrict__ stamp, unsigned long long keep_from) {
    unsigned long long placed = 0, refused = 0;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += stride) {
        const uint64_t i = base + threadIdx.x;
        if (i >= n) continue;
        if (stamp && stamp[i] < keep_from) continue;
        const uint4 r0 = rec[2 * i], r1 = rec[2 * i + 1];
        const uint64_t hash = ((uint64_t)r0.y << 32) | r0.x;
        const uint32_t model = r0.z & 0xffffu, cnt = (r0.z >> 16) & 0xffu;
        if (shard_of(home_of(hash, model), t.shard_bits) != t.shard_rank) continue;      // another shard's key
        const uint4 a = make_uint4(r0.x, r0.y, r0.w, r1.x);
        const uint32_t busy = make_meta(kStateBusy, 0, model);
        uint4 b = make_uint4(r1.y, r1.z, r1.w, published_meta(busy, make_meta(kStateFull, cnt, model)));
        uint64_t j = slot_home(hash, model, t.req_mask);
        bool ok = false;
        for (uint64_t step = 0; step <= t.req_mask; ++step, j = (j + 1) & t.req_mask) {
            if (atomicCAS_system(&t.req[j].meta, 0u, busy) != 0u) continue;   // the target's slots are EMPTY or restored here
            if (stamp) t.req_stamp[j] = stamp[i];
            st_slot(t.req + j, a, b);
            ok = true;
            break;
        }
        if (ok) ++placed; else ++refused;
    }
    warp_sum_add(&t.cnt->req_full, placed);
    warp_sum_add(&t.cnt->nospc, refused);
}

__global__ void __launch_bounds__(kSnapThreads) restore_eng_kernel(TableView t, const unsigned long long* __restrict__ rec, uint64_t n,
                                                                   const unsigned long long* __restrict__ stamp, unsigned long long keep_from) {
    unsigned long long placed = 0, refused = 0;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += stride) {
        const uint64_t i = base + threadIdx.x;
        if (i >= n) continue;
        const unsigned long long eh = rec[3 * i], rh = rec[3 * i + 1];
        const uint32_t model = (uint32_t)(rec[3 * i + 2] & 0xffffu);
        if (shard_of(home_of(eh, model), t.shard_bits) != t.shard_rank) continue;
        const unsigned long long s = stamp ? stamp[i] : 0ull;
        if (s < keep_from) continue;
        const uint4 a = make_uint4((uint32_t)eh, (uint32_t)(eh >> 32), (uint32_t)rh, (uint32_t)(rh >> 32));
        const uint32_t busy = make_meta(kStateBusy, 0, model);
        uint4 b = make_uint4(published_meta(busy, make_meta(kStateFull, 0, model)), 0u, (uint32_t)s, (uint32_t)(s >> 32));
        uint64_t j = slot_home(eh, model, t.eng_mask);
        bool ok = false;
        for (uint64_t step = 0; step <= t.eng_mask; ++step, j = (j + 1) & t.eng_mask) {
            if (atomicCAS_system(&t.eng[j].meta, 0u, busy) != 0u) continue;
            st_slot(t.eng + j, a, b);
            ok = true;
            break;
        }
        if (ok) ++placed; else ++refused;
    }
    warp_sum_add(&t.cnt->eng_full, placed);
    warp_sum_add(&t.cnt->nospc, refused);
}

}  // namespace kvx
