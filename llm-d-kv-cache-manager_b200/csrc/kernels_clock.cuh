// kernels_clock.cuh -- CLOCK (second chance) key cap: InMemoryIndexConfig.Size (in_memory.go:59,64) approximated with one
// reference bit per slot instead of a recency list.
//
// Bits are set wherever golang-lru refreshes recency (kernels_write.cuh, lookup_kernel_v1) and, for Score(), inside every
// score kernel's fold (score_common.cuh: mark_hit, HomeProbe::hit_slot, WarpWalk::mark_walked) on the present keys among the
// blocks the walk looks at -- block 0, then each next block up to and including the one whose probe empties the active
// pod set, or the last full block -- so the referenced set of a batch is the same on every path.
//
// After every write call each table is swept back to `capacity` live keys.  The outcome is that of a sequential hand:
// starting at slot `hand` and wrapping around, a FULL slot with its bit set has the bit cleared, a FULL slot with its bit
// clear is evicted, every other slot is passed, and the hand stops just after the e-th eviction (e = live - capacity).
// In parallel that is four kernels on the write stream, all reading e from the counters on the device (no host
// readback) and doing nothing when e == 0:
//   sweep_snap_kernel   copies the bitmap: the sweep decides on that image, so readers that set bits meanwhile cannot
//                       make the count and the evictions disagree (such a touch may or may not protect its key);
//   sweep_count_kernel  per tile of 1024 slots in hand order: FULL slots with the bit clear (U) and set (V);
//   sweep_cut_kernel    one CTA: if the table holds at least e unreferenced keys, the cut is the e-th of them in hand
//                       order (one partial turn); else every unreferenced key goes, every bit is cleared (a full turn)
//                       and the cut is the (e - U)-th referenced key, where the second turn stops.  Moves the hand and
//                       counts the sweep (Counters::sweeps, and turns2 if it needed the second turn);
//   sweep_apply_kernel  clears the bits and evicts up to the cut: ownership by compare-and-swap and a two-half tombstone
//                       publish, as remove_req_kernel does, so a reader sees each key before or after its eviction.
// Evicting a request key leaves the engine map alone (a stale mapping, cleaned up by Evict, in_memory.go:225-230), and
// evicting an engine mapping leaves its request key.
#pragma once
#include <cub/block/block_scan.cuh>
#include "kernels_v1.cuh"

namespace kvx {

constexpr int kSweepThreads = 256, kSweepPer = 4, kSweepTile = kSweepThreads * kSweepPer;
constexpr int kCutThreads = 1024;                  // the cut kernel's last step: thread x examines slot x of one tile
static_assert(kCutThreads == kSweepTile, "the cut kernel takes one slot of the tile per thread");

struct SweepCtl {
    unsigned long long e;          // evictions of this sweep (0: nothing to do)
    unsigned long long hand;       // hand at the start: rotated index r is slot (hand + r) & mask
    unsigned long long cut;        // rotated index of the last slot the sweep processes
    unsigned int two_turns;        // fewer unreferenced keys than e: a full turn, then the first (e - U) referenced keys
    unsigned int pad;
};

__device__ __forceinline__ unsigned long long sweep_excess(const unsigned long long* full, uint64_t cap) {
    const unsigned long long f = *(const volatile unsigned long long*)full;
    return f > cap ? f - cap : 0ull;
}
template <class Slot> __device__ __forceinline__ uint32_t slot_meta(const Slot* s);
template <> __device__ __forceinline__ uint32_t slot_meta<ReqSlot>(const ReqSlot* s) { return ld_word_relaxed(&s->meta, false); }
template <> __device__ __forceinline__ uint32_t slot_meta<EngSlot>(const EngSlot* s) { return ld_word_relaxed(&s->meta, false); }

__global__ void sweep_snap_kernel(const uint32_t* __restrict__ ref, uint32_t* __restrict__ snap, uint64_t words,
                                  const unsigned long long* full, uint64_t cap) {
    if (!sweep_excess(full, cap)) return;
    for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < words; w += (uint64_t)gridDim.x * blockDim.x)
        snap[w] = ld_word_relaxed(ref + w, false);
}

// tile_cnt[2 t] = U, tile_cnt[2 t + 1] = V of tile t (rotated indices [t * kSweepTile, (t + 1) * kSweepTile))
template <class Slot>
__global__ void __launch_bounds__(kSweepThreads) sweep_count_kernel(const Slot* __restrict__ tab, uint64_t mask, const uint32_t* __restrict__ snap,
                                                                    const unsigned long long* full, uint64_t cap, const unsigned long long* hand,
                                                                    unsigned long long* tile_cnt) {
    if (!sweep_excess(full, cap)) return;
    const uint64_t slots = mask + 1, h = *hand & mask;
    const uint64_t tiles = (slots + kSweepTile - 1) / kSweepTile;
    __shared__ unsigned int su, sv;
    for (uint64_t tl = blockIdx.x; tl < tiles; tl += gridDim.x) {
        if (threadIdx.x == 0) { su = 0; sv = 0; }
        __syncthreads();
        unsigned int u = 0, v = 0;
#pragma unroll
        for (int k = 0; k < kSweepPer; ++k) {
            const uint64_t r = tl * kSweepTile + (uint64_t)k * kSweepThreads + threadIdx.x;
            if (r >= slots) continue;
            const uint64_t s = (h + r) & mask;
            if (meta_state(slot_meta(tab + s)) != kStateFull) continue;
            if ((snap[s >> 5] >> (s & 31)) & 1u) ++v; else ++u;
        }
        if (u) atomicAdd(&su, u);
        if (v) atomicAdd(&sv, v);
        __syncthreads();
        if (threadIdx.x == 0) { tile_cnt[2 * tl] = su; tile_cnt[2 * tl + 1] = sv; }
        __syncthreads();
    }
}

// One CTA: find the cut, move the hand.
template <class Slot>
__global__ void __launch_bounds__(kCutThreads) sweep_cut_kernel(const Slot* __restrict__ tab, uint64_t mask, const uint32_t* __restrict__ snap,
                                                                const unsigned long long* full, uint64_t cap, unsigned long long* hand,
                                                                const unsigned long long* __restrict__ tile_cnt, SweepCtl* ctl,
                                                                unsigned long long* sweeps, unsigned long long* turns2) {
    using Scan = cub::BlockScan<unsigned long long, kCutThreads>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ unsigned long long s_tot, s_base;
    __shared__ long long s_tile;
    const unsigned long long e = sweep_excess(full, cap);
    if (!e) { if (threadIdx.x == 0) ctl->e = 0; return; }
    if (threadIdx.x == 0) atomicAdd(sweeps, 1ull);           // sweeps that evict; turns2: those that needed a second turn
    const uint64_t slots = mask + 1, h = *hand & mask;
    const uint64_t tiles = (slots + kSweepTile - 1) / kSweepTile;
    const uint64_t per = (tiles + kCutThreads - 1) / kCutThreads;
    const uint64_t t0 = min(tiles, threadIdx.x * per), t1 = min(tiles, t0 + per);
    // U over the whole table
    unsigned long long mine = 0;
    for (uint64_t tl = t0; tl < t1; ++tl) mine += tile_cnt[2 * tl];
    unsigned long long excl;
    Scan(tmp).ExclusiveSum(mine, excl);
    if (threadIdx.x == kCutThreads - 1) s_tot = excl + mine;
    __syncthreads();
    const unsigned long long U = s_tot;
    const bool two = U < e;
    const int col = two ? 1 : 0;                                 // which count the cut is taken on
    const unsigned long long want = two ? e - U : e;             // 1-based rank of the slot the hand stops after
    // the tile holding it
    mine = 0;
    for (uint64_t tl = t0; tl < t1; ++tl) mine += tile_cnt[2 * tl + col];
    __syncthreads();
    Scan(tmp).ExclusiveSum(mine, excl);
    if (threadIdx.x == 0) s_tile = -1;
    __syncthreads();
    if (excl < want && want <= excl + mine) {
        unsigned long long acc = excl;
        for (uint64_t tl = t0; tl < t1; ++tl) {
            const unsigned long long c = tile_cnt[2 * tl + col];
            if (want <= acc + c) { s_tile = (long long)tl; s_base = acc; break; }
            acc += c;
        }
    }
    __syncthreads();
    if (s_tile < 0) { if (threadIdx.x == 0) ctl->e = 0; return; }   // counts changed under the sweep: cannot happen with mu_w held
    // the slot inside that tile
    const uint64_t tl = (uint64_t)s_tile;
    const unsigned long long need = want - s_base;
    const uint64_t r = tl * kSweepTile + threadIdx.x;
    unsigned long long flag = 0;
    if (r < slots) {
        const uint64_t s = (h + r) & mask;
        if (meta_state(slot_meta(tab + s)) == kStateFull && (((snap[s >> 5] >> (s & 31)) & 1u) == (unsigned)col)) flag = 1;
    }
    __syncthreads();
    Scan(tmp).ExclusiveSum(flag, excl);
    if (flag && excl + 1 == need) {
        ctl->e = e; ctl->hand = h; ctl->cut = r; ctl->two_turns = two ? 1u : 0u;
        *hand = (h + r + 1) & mask;
        if (two) atomicAdd(turns2, 1ull);
    }
}

__device__ __forceinline__ void clock_evict(ReqSlot* s) {
    for (;;) {
        uint4 a, b;
        ld_slot_fresh(s, a, b);                  // no other writer runs during the sweep: this image is the slot's
        const uint32_t m = b.w;
        if (meta_state(m) != kStateFull) return;
        if (m & kLockBit) { spin_pause(); continue; }
        if (atomicCAS_system(&s->meta, m, m | kLockBit) != m) continue;
        a.z = 0u; a.w = 0u; b.x = 0u; b.y = 0u; b.z = 0u;   // a tombstone keeps tag and model, its entries zeroed
        req_publish(s, a, b, make_meta(kStateTomb, 0, meta_model(m)));
        return;
    }
}
__device__ __forceinline__ void clock_evict(EngSlot* s) {
    for (;;) {
        uint4 a, b;
        ld_slot_fresh(s, a, b);
        const uint32_t m = b.x;
        if (meta_state(m) != kStateFull) return;
        if (m & kLockBit) { spin_pause(); continue; }
        if (atomicCAS_system(&s->meta, m, m | kLockBit) != m) continue;
        eng_publish(s, a, b, make_meta(kStateTomb, 0, meta_model(m)));
        return;
    }
}

// full / tomb / evicted: the table's counters (req_full, req_tomb, cap_evicted[0] or the engine ones)
template <class Slot>
__global__ void __launch_bounds__(kSweepThreads) sweep_apply_kernel(Slot* tab, uint64_t mask, uint32_t* ref, const uint32_t* __restrict__ snap,
                                                                    const SweepCtl* __restrict__ ctl, unsigned long long* full,
                                                                    unsigned long long* tomb, unsigned long long* evicted) {
    const SweepCtl c = *ctl;
    if (!c.e) return;
    const uint64_t slots = mask + 1, end = c.two_turns ? slots : c.cut + 1;
    __shared__ unsigned long long s_n;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    unsigned long long n = 0;
    for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < end; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t s = (c.hand + r) & mask;
        if (meta_state(slot_meta(tab + s)) != kStateFull) continue;
        const bool referenced = (snap[s >> 5] >> (s & 31)) & 1u;
        atomicAnd(ref + (s >> 5), ~(1u << (s & 31)));
        if (!referenced || (c.two_turns && r <= c.cut)) { clock_evict(tab + s); ++n; }
    }
    if (n) atomicAdd(&s_n, n);
    __syncthreads();
    if (threadIdx.x == 0 && s_n) { atomicAdd(full, ~s_n + 1ull); atomicAdd(tomb, s_n); atomicAdd(evicted, s_n); }
}

}  // namespace kvx
