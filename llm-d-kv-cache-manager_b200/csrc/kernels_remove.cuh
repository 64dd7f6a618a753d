// kernels_remove.cuh -- kvidx_remove_pods: drop every entry of a set of pods (and tiers) from the index.
//
// An extension with no reference counterpart: vLLM pods that crash, are rescheduled or scaled down send no BlockRemoved
// events, so without it their entries would stay in the index for good.  The semantics are those of a sequence of
// Evict calls, one per affected key (spec: tests/remove_oracle.py remove_pods):
//   * every request key loses the matching entries, the survivors keep their order; a key left without entries is
//     removed, and so is every engine mapping that points at a key removed BY THIS CALL (an engine mapping whose key was
//     already gone is a stale mapping, which Evict cleans up lazily, in_memory.go:225-230, so it stays);
//   * no recency changes (no stamp is written).
//
// Two streaming passes over the tables, both on the write stream.  The caller holds mu_w for the whole call, so no other
// writer runs and no rebuild happens between them; readers run beside them and see each slot before or after its update
// (the usual ownership compare-and-swap and two-half publish of table.cuh).
//   pass 1  remove_req_kernel  every request slot: a FULL slot with a matching entry is owned, compacted (vacated
//           positions zeroed, so equal live sets stay bitwise equal) and published; an emptied one becomes a tombstone that
//           keeps its tag and model, as Evict leaves it.  Each slot tombstoned here sets its bit in `removed_slot`, and the
//           bit of its key's home pair in `removed_home` (both bitmaps: slots/8 + slots/16 bytes of scratch).
//   pass 2  remove_eng_kernel  every FULL engine slot whose request key's home pair has its bit set probes the request
//           table from that home: the mapping goes if the probe reaches a tombstone of the key with its removed_slot bit
//           set; a FULL slot of the key or an EMPTY slot keeps it.  (The key has at most one slot tombstoned by this call:
//           a re-added key never reuses its old tombstone, and older tombstones of the key have no bit.)
//
// Sharded index (kvidx_shard_remove_pods): an engine mapping lives with its engine hash's owner, its request key with
// the owner of the request hash.  Every rank runs pass 1 over its own request shard (phase 0), then, once all ranks have,
// pass 2 over its own engine shard (phase 1).  Pass 2 therefore reads the request table AND the two bitmaps of the key's
// owner: the bitmaps of a sharded handle sit right behind its request slots, in the same allocation, so the mapping every
// peer already holds (CUDA IPC / kvidx_shard_attach) covers them.  Unsharded, owner 0 is the handle itself.
#pragma once
#include "table.cuh"
#include "../../include/kvidx.h"

namespace kvx {

constexpr int kRemoveThreads = 256;

struct RemoveArgs {
    const uint64_t* pod_mask;           // filter_words words, bit p = pod p
    uint32_t tier_mask;                 // bit t = tier t
    uint32_t* removed_slot;             // bit per request slot: tombstoned by this call
    uint32_t* removed_home;             // bit per home pair (home slot / 2) of a key tombstoned by this call
    unsigned long long* out;            // {entries, request keys, engine keys} removed
    const uint32_t* owner_slot[8];      // pass 2: removed_slot / removed_home of request shard r (t.req_peer[r]); entry 0
    const uint32_t* owner_home[8];      //         only on an unsharded handle
};

// system scope: a peer's bitmaps were written by a kernel of another process (or device) before the embedding program's barrier
__device__ __forceinline__ bool test_bit(const uint32_t* bits, uint64_t i) { return (ld_word_relaxed(bits + (i >> 5), true) >> (i & 31)) & 1u; }

// sum over the warp, one atomic per warp (the grid-stride loops below give every lane of a warp the same trip count)
__device__ __forceinline__ void warp_add(unsigned long long* dst, unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(dst, v);
}

__global__ void __launch_bounds__(kRemoveThreads) remove_req_kernel(TableView t, RemoveArgs r) {
    __shared__ uint64_t pm[KVIDX_MAX_PODS / 64];
    for (uint32_t w = threadIdx.x; w < t.filter_words; w += blockDim.x) pm[w] = r.pod_mask[w];
    __syncthreads();
    const uint32_t P = t.max_pods, tiers = r.tier_mask;
    auto hit = [&](uint32_t e) {
        const uint32_t p = e >> KVIDX_TIER_BITS;
        return p < P && ((pm[p >> 6] >> (p & 63)) & 1ull) && ((tiers >> (e & (KVIDX_MAX_TIERS - 1))) & 1u);
    };
    unsigned long long n_ent = 0, n_key = 0;
    const uint64_t slots = t.req_mask + 1, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < slots; i += stride) {
        ReqSlot* s = t.req + i;
        for (;;) {
            uint4 a, b;
            ld_slot_fresh(s, a, b);                  // no other writer runs during the call: this image is the slot's
            const uint32_t m = b.w;
            if (meta_state(m) != kStateFull) break;
            const uint32_t cnt = meta_count(m);
            EntList L; L.unpack(a, b);
            uint32_t count = cnt;
#pragma unroll
            for (int j = kMaxEnt - 1; j >= 0; --j)   // top down: a removal moves only the entries above it
                if ((uint32_t)j < cnt && hit(L.e[j])) { L.remove_at((uint32_t)j); --count; }
            if (count == cnt) break;                 // nothing to remove: the slot is never written
            if (m & kLockBit) { spin_pause(); continue; }
            if (atomicCAS_system(&s->meta, m, m | kLockBit) != m) continue;
            L.pack(a, b);
            const uint32_t model = meta_model(m);
            n_ent += cnt - count;
            if (count == 0) {
                req_publish(s, a, b, make_meta(kStateTomb, 0, model));
                const uint64_t tag = ((uint64_t)a.y << 32) | a.x;
                atomicOr(&r.removed_slot[i >> 5], 1u << (i & 31));
                const uint64_t hp = slot_home(tag, model, t.req_mask) >> 1;
                atomicOr(&r.removed_home[hp >> 5], 1u << (hp & 31));
                ++n_key;
            } else {
                req_publish(s, a, b, make_meta(kStateFull, count, model));
            }
            break;
        }
    }
    warp_add(&r.out[0], n_ent);
    warp_add(&r.out[1], n_key);
    warp_add(&t.cnt->req_full, 0ull - n_key);
    warp_add(&t.cnt->req_tomb, n_key);
}

__global__ void __launch_bounds__(kRemoveThreads) remove_eng_kernel(TableView t, RemoveArgs r) {
    unsigned long long n_eng = 0;
    const uint64_t slots = t.eng_mask + 1, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < slots; i += stride) {
        EngSlot* s = t.eng + i;
        for (;;) {
            uint4 a, b;
            ld_slot_fresh(s, a, b);
            const uint32_t m = b.x;
            if (meta_state(m) != kStateFull) break;
            const uint32_t model = meta_model(m);
            const uint64_t rhash = ((uint64_t)a.w << 32) | a.z;
            const uint64_t mixed = home_of(rhash, model);
            const uint32_t owner = shard_of(mixed, t.shard_bits);
            const uint64_t home = mixed & t.req_mask & ~1ull;          // slot_home
            if (!test_bit(r.owner_home[owner], home >> 1)) break;
            const ReqSlot* req = t.req_peer[owner];
            bool drop = false;
            for (uint64_t j = home, step = 0; step <= t.req_mask; ++step, j = (j + 1) & t.req_mask) {
                uint4 ra, rb;
                ld_slot_fresh(req + j, ra, rb);
                const uint32_t st = meta_state(rb.w);
                if (st == kStateEmpty) break;
                if (ra.x == (uint32_t)rhash && ra.y == (uint32_t)(rhash >> 32) && meta_model(rb.w) == model) {
                    if (st == kStateFull) break;
                    if (st == kStateTomb && test_bit(r.owner_slot[owner], j)) { drop = true; break; }
                }
            }
            if (!drop) break;
            if (m & kLockBit) { spin_pause(); continue; }
            if (atomicCAS_system(&s->meta, m, m | kLockBit) != m) continue;
            eng_publish(s, a, b, make_meta(kStateTomb, 0, model));
            ++n_eng;
            break;
        }
    }
    warp_add(&r.out[2], n_eng);
    warp_add(&t.cnt->eng_full, 0ull - n_eng);
    warp_add(&t.cnt->eng_tomb, n_eng);
}

}  // namespace kvx
