// kernels_write.cuh -- the kvevents.Pool -> Index.Add / Index.Evict write path on the device.
//
// Reference: Pool.digestEvents (pkg/kvcache/kvevents/pool.go:246-338) -> TokensToKVBlockKeys
// (kvblock/token_processor.go:141-162) -> InMemoryIndex.Add / Evict (kvblock/in_memory.go:149-260).
//
// A batch of decoded events is applied in two phases:
//
//   phase 1  hash_events_kernel   the request keys of EVERY BlockStored event of the batch, all events at once.  The
//            chain inside an event is serial, events are independent except for their starting point: the request key
//            of the parent block, which the reference looks up when the event is applied (pool.go:279-294).  Phase 1
//            PREDICTS it -- the block of an earlier event of the same pod in this batch (found through a small
//            device-side map of the wanted parent hashes), else the index as it is before the batch, else the seed --
//            and an event whose parent is produced inside the batch simply waits for that block's key (lanes are
//            persistent workers that fetch events in queue order, so a producer is always already running).
//   phase 2  apply_events_kernel  one warp per pod queue walks its events in order: the reference's per-pod FIFO
//            (pool.go:129-144).  It does the real parent lookup; if that resolves to the predicted key -- always,
//            unless another pod's worker changed the parent in between -- the keys of phase 1 are used as they are,
//            otherwise the event is re-hashed on the spot (Counters::rehashed).  The lanes of the warp then take the
//            event's blocks in parallel: engine-map upsert and pod-entry add, each one compare-and-swap to own the
//            slot and one 256-bit store to publish it (table.cuh).
//
// So the serial FNV chains of a batch run on thousands of lanes instead of one warp per pod, and the ordered part of
// the work is only the slot updates.
#pragma once
#include "kernels_v1.cuh"
#include "../../include/kvidx.h"

namespace kvx {

// One (engineKey, requestKey) pair of Index.Add (in_memory.go:159-206).  do_engine / do_request let a caller that has
// found duplicates inside one call keep only the update that wins in the reference's sequential order.
__device__ __forceinline__ void do_add(const TableView& t, uint32_t model, uint64_t ehash, uint64_t rhash,
                                       const uint16_t* __restrict__ pts, int m, unsigned long long stamp = 0,
                                       bool do_engine = true, bool do_request = true) {
    bool created, full;
    uint4 a, b;
    if (do_engine) {                                  // 1. engineToRequestKeys.Add(engineKey, requestKey)   (in_memory.go:163)
        EngSlot* es = eng_acquire(t, model, ehash, false, &created, a, b, &full);
        if (!es) atomicAdd(&t.cnt->nospc, 1ull);
        else {
            a.z = (uint32_t)rhash; a.w = (uint32_t)(rhash >> 32);
            if (t.eng_ref) ref_touch(t.eng_ref, es - t.eng);
            if (created) atomicAdd_system(&cnt_of(t, ehash, model)->eng_full, 1ull);
            if (t.req_stamp) {                         // lru Add: insert or refresh (an EMPTY slot's stamp word is 0)
                eng_stamp_touch(es, stamp);
                eng_publish_lru(es, a, b, make_meta(kStateFull, 0, model));
            } else {
                eng_publish(es, a, b, make_meta(kStateFull, 0, model));
            }
        }
    }
    if (do_request) {                                 // 2. get-or-create the PodCache and add the entries    (in_memory.go:170-203)
        ReqSlot* rs = req_acquire(t, model, rhash, false, &created, a, b, &full);
        if (!rs) { atomicAdd(&t.cnt->nospc, 1ull); return; }
        uint32_t count = created ? 0u : meta_count(b.w);
        EntList L; L.unpack(a, b);
        for (int j = 0; j < m; ++j) count = L.add(count, pts[j], t.pods_per_key);
        L.pack(a, b);
        if (t.req_stamp) stamp_touch(t.req_stamp + (rs - t.req), stamp + 1);              // data.Get refresh / ContainsOrAdd insert
        if (t.req_ref) ref_touch(t.req_ref, rs - t.req);
        if (created) atomicAdd_system(&cnt_of(t, rhash, model)->req_full, 1ull);
        req_publish(rs, a, b, make_meta(kStateFull, count, model));
    }
}

// Index.Evict (in_memory.go:212-260).
__device__ __forceinline__ void do_evict(const TableView& t, uint32_t model, uint64_t ehash,
                                         const uint16_t* __restrict__ pts, int m, unsigned long long stamp = 0) {
    uint64_t rhash;
    if (!eng_find(t, model, ehash, &rhash, nullptr, stamp, true)) return;   // :219-223 silent no-op (a hit refreshes recency)
    bool created;
    uint4 a, b;
    ReqSlot* rs = req_acquire(t, model, rhash, true, &created, a, b);
    bool drop_engine = false;
    if (!rs) {
        drop_engine = true;                                              // :225-230 stale engine mapping
    } else {
        uint32_t count = meta_count(b.w);
        if (t.req_stamp) stamp_touch(t.req_stamp + (rs - t.req), stamp + 1);          // data.Get (:225)
        if (t.req_ref) ref_touch(t.req_ref, rs - t.req);
        EntList L; L.unpack(a, b);
        for (int j = 0; j < m; ++j) count = L.remove(count, pts[j]);
        L.pack(a, b);
        if (count == 0) {                                                // :243-256 last entry gone
            Counters* c = cnt_of(t, rhash, model);
            atomicAdd_system(&c->req_tomb, 1ull);
            atomicAdd_system(&c->req_full, ~0ull);
            req_publish(rs, a, b, make_meta(kStateTomb, 0, model));
            drop_engine = true;
        } else {
            req_publish(rs, a, b, make_meta(kStateFull, count, model));
        }
    }
    if (drop_engine) {
        EngSlot* e2 = eng_acquire(t, model, ehash, true, &created, a, b);
        if (e2) {
            Counters* c = cnt_of(t, ehash, model);
            atomicAdd_system(&c->eng_tomb, 1ull);
            atomicAdd_system(&c->eng_full, ~0ull);
            eng_publish(e2, a, b, make_meta(kStateTomb, 0, model));
        }
    }
}

// Index.Add for one call: lane per key pair.  skip_engine[i] != 0 marks a pair whose engine key appears again later in
// the call (the host finds those): the reference adds the pairs in order, so the last mapping of an engine key wins
// (in_memory.go:159-163); the pod entries are added for every pair (adding an entry twice only refreshes it).
__global__ void add_kernel(TableView t, uint32_t model, const uint64_t* __restrict__ engine,
                           const uint64_t* __restrict__ request, int64_t n, const uint16_t* __restrict__ pts, int m,
                           const uint8_t* __restrict__ skip_engine, unsigned long long stamp_base) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) do_add(t, model, engine[i], request[i], pts, m, stamp_base + 2ull * (unsigned long long)i, !skip_engine || !skip_engine[i], true);
}

__global__ void evict_kernel(TableView t, uint32_t model, uint64_t engine, const uint16_t* __restrict__ pts, int m,
                             unsigned long long stamp_base) {
    if (blockIdx.x == 0 && threadIdx.x == 0) do_evict(t, model, engine, pts, m, stamp_base);
}

__global__ void get_request_key_kernel(TableView t, uint32_t model, uint64_t engine, uint64_t* out, int* found, unsigned long long stamp) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        uint64_t r = 0;
        const bool ok = eng_find(t, model, engine, &r, nullptr, stamp, true);
        *out = r; *found = ok ? 1 : 0;
    }
}

// ---- phase 1: request keys of a whole event batch ------------------------------------------------------------

// Parents wanted by the batch: fingerprint(parent engine hash, pod, model) -> the list of events that want it (their
// consumers), chained through next[]; every block of the batch that carries a wanted hash offers itself to the consumers that
// come AFTER it in the pod's queue, and each consumer keeps the latest such block: best[e] = (producer event + 1) << 32 | block.
// That is the block whose Add is the last one before event e that touches the parent's engine key -- what GetRequestKey will
// find when e is applied, unless a removal or another pod's worker gets in between (then phase 2 re-hashes the event).
struct WantEnt { unsigned long long fp; unsigned int head; unsigned int pad; };

__device__ __forceinline__ unsigned long long want_fp(uint64_t ehash, uint32_t podtier, uint32_t model) {
    const unsigned long long f = mix64(ehash ^ ((uint64_t)(podtier >> KVIDX_TIER_BITS) * 0xD6E8FEB86659FD93ull) ^ ((uint64_t)model << 48));
    return f ? f : 1ull;
}
__device__ __forceinline__ bool event_hashable(const kvidx_event_t& e, uint32_t B) {
    // the events whose keys phase 2 will ask for: BlockStored with hashes, and as many full token blocks as hashes
    return e.op == KVIDX_EV_BLOCK_STORED && e.n_hashes != 0 && e.n_tokens / B == e.n_hashes;
}

__global__ void want_parents_kernel(const kvidx_event_t* __restrict__ ev, int64_t n_ev, uint32_t B, WantEnt* map, uint32_t map_mask,
                                    unsigned int* next) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= n_ev) return;
    const kvidx_event_t evt = ev[e];
    if (!event_hashable(evt, B) || !evt.has_parent) return;
    const unsigned long long fp = want_fp(evt.parent_hash, evt.podtier, evt.model);
    for (uint32_t i = (uint32_t)fp & map_mask;; i = (i + 1) & map_mask) {
        const unsigned long long old = atomicCAS(&map[i].fp, 0ull, fp);
        if (old == 0ull || old == fp) { next[e] = atomicExch(&map[i].head, (unsigned int)e + 1u); return; }      // push front (0 = end of list)
    }
}
// lane per (event, 32-block group): offers its blocks to the later events that want them as a parent
__global__ void offer_blocks_kernel(const kvidx_event_t* __restrict__ ev, int64_t n_ev, uint32_t B, const uint64_t* __restrict__ hashes,
                                    const WantEnt* __restrict__ map, uint32_t map_mask, const unsigned int* __restrict__ next,
                                    unsigned long long* best) {
    const int64_t e = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (e >= n_ev) return;
    const kvidx_event_t evt = ev[e];
    if (!event_hashable(evt, B)) return;
    for (uint32_t b = lane; b < evt.n_hashes; b += 32) {
        const unsigned long long fp = want_fp(hashes[evt.hash_off + b], evt.podtier, evt.model);
        for (uint32_t i = (uint32_t)fp & map_mask;; i = (i + 1) & map_mask) {
            const unsigned long long cur = map[i].fp;
            if (cur == 0ull) break;                                       // nobody wants this block as a parent
            if (cur == fp) {
                for (unsigned int c = map[i].head; c != 0u; c = next[c - 1u])
                    if ((long long)(c - 1u) > e) atomicMax(&best[c - 1u], ((unsigned long long)(e + 1) << 32) | b);
                break;
            }
        }
    }
}

__device__ __forceinline__ uint64_t hash_block_any(uint64_t parent, const uint32_t* __restrict__ tk, uint32_t B) {
    if (B == 16u && (reinterpret_cast<uintptr_t>(tk) & 15u) == 0) {
        Fnv f;
        f.begin_block(parent, 16);
        const uint4* t4 = reinterpret_cast<const uint4*>(tk);
#pragma unroll
        for (int c = 0; c < 4; ++c) { const uint4 v = __ldg(t4 + c); f.token(v.x); f.token(v.y); f.token(v.z); f.token(v.w); }
        return f.end_block();
    }
    return hash_block_global(parent, tk, B);
}

constexpr int kHashEvThreads = 128;
// Persistent lanes; every lane is a worker that owns one event at a time and hashes one block per iteration of the
// warp's lock-step loop.  Events are fetched in queue order from a global counter, so the producer of a wanted parent
// (an EARLIER event of the same pod) is always held by a running lane: waiting for it cannot deadlock.
//   ready[e]  0 not yet, 1 keys of event e are in keys[hash_off ..], 2 event has no keys
__global__ void __launch_bounds__(kHashEvThreads)
hash_events_kernel(const TableView t, const kvidx_event_t* __restrict__ ev, int64_t n_ev, const uint64_t* __restrict__ hashes,
                   const uint32_t* __restrict__ tokens, const unsigned long long* __restrict__ best,
                   uint64_t* keys, uint64_t* pred, unsigned int* ready, unsigned long long* next) {
    const int lane = threadIdx.x & 31;
    const uint32_t B = t.block_size;
    long long e = -1;                  // event owned by this lane
    bool exhausted = false;
    int stage = 0;                     // 0 idle, 1 waiting for the producer of its parent, 2 hashing
    long long pe = 0; uint32_t pb = 0; // producer event / block
    uint64_t h = 0, hoff = 0;
    uint32_t nblk = 0, b = 0, model = 0; uint64_t parent = 0;
    const uint32_t* tk = nullptr;
    for (;;) {
        // ---- hand events to idle lanes ----
        const bool want = (e < 0) && !exhausted;
        const uint32_t wm = __ballot_sync(0xffffffffu, want);
        if (wm) {
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(next, (unsigned long long)__popc(wm));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (want) {
                const long long idx = (long long)base + __popc(wm & ((1u << lane) - 1u));
                if (idx >= n_ev) exhausted = true;
                else {
                    const kvidx_event_t evt = ev[idx];
                    if (!event_hashable(evt, B)) { *(volatile unsigned int*)&ready[idx] = 2u; }
                    else {
                        e = idx; hoff = evt.hash_off; nblk = evt.n_hashes; b = 0; model = evt.model; parent = evt.parent_hash;
                        tk = tokens + evt.tok_off;
                        h = t.init_hash; stage = 2;
                        if (evt.has_parent) {
                            const unsigned long long v = best[idx];                // latest earlier block of the batch carrying the parent hash
                            if (v != 0ull) { pe = (long long)(v >> 32) - 1; pb = (uint32_t)v; stage = 1; }
                            else stage = 3;                                        // 3: resolve against the index as it is now
                        }
                    }
                }
            }
        }
        // ---- parents ----
        if (stage == 1) {
            const unsigned int r = *(const volatile unsigned int*)&ready[pe];
            if (r == 1u) { __threadfence(); h = *(const volatile uint64_t*)&keys[ev[pe].hash_off + pb]; stage = 2; }
            else if (r == 2u) stage = 3;
        }
        if (stage == 3) { uint64_t r; h = eng_find(t, model, parent, &r) ? r : t.init_hash; stage = 2; }
        if (stage == 2 && b == 0) pred[e] = h;
        // ---- one block per lane ----
        if (stage == 2) {
            h = hash_block_any(h, tk + (size_t)b * B, B);
            keys[hoff + b] = h;
            if (++b == nblk) { __threadfence(); *(volatile unsigned int*)&ready[e] = 1u; e = -1; stage = 0; }
        }
        if (!__any_sync(0xffffffffu, e >= 0 || !exhausted)) break;
    }
}

// ---- phase 2: Pool.digestEvents (kvevents/pool.go:246-338), one warp per pod queue --------------------------------
//   ev        events stably sorted by pod; queue q owns ev[queue_off[q] .. queue_off[q+1])
//   keys/pred phase 1's request keys (indexed like `hashes`) and the parent key each event's chain was started from;
//             nullptr: hash here (small batches skip phase 1)
//   stamp_*   exact-LRU mode: event e owns the stamps [stamp_base + e * stamp_stride, + stamp_stride), the parent lookup
//             first, then two per block, so stamp_stride = 2 + 2 x the batch's largest n_hashes; the pod-sorted order of
//             the batch is the order its stamps give
__global__ void apply_events_kernel(TableView t, const kvidx_event_t* __restrict__ ev, const int64_t* __restrict__ queue_off,
                                    int64_t n_queues, const uint64_t* __restrict__ hashes, const uint32_t* __restrict__ tokens,
                                    const uint64_t* __restrict__ keys, const uint64_t* __restrict__ pred,
                                    unsigned long long stamp_base, unsigned long long stamp_stride) {
    const int lane = threadIdx.x & 31;
    const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (q >= n_queues) return;
    const uint32_t B = t.block_size;
    for (int64_t e = queue_off[q]; e < queue_off[q + 1]; ++e) {
        const kvidx_event_t evt = ev[e];
        const uint16_t pt = evt.podtier;
        const unsigned long long sb = stamp_base + (unsigned long long)e * stamp_stride;     // exact-LRU: this event's stamps
        if (evt.op == KVIDX_EV_BLOCK_STORED) {
            // parent request key: GetRequestKey(parent engine key); a miss restarts at the seed (pool.go:279-294)
            uint64_t h = t.init_hash;
            if (evt.has_parent) { uint64_t r; if (eng_find(t, evt.model, evt.parent_hash, &r, nullptr, lane == 0 ? sb + 1 : 0, lane == 0)) h = r; }
            if (evt.n_hashes == 0) continue;                                 // pool.go:299 `if len(engineKeys) > 0`
            const uint32_t nblk = evt.n_tokens / B;
            if (nblk == 0 || nblk != evt.n_hashes) {                         // in_memory.go:150-155 -> event dropped
                if (lane == 0) atomicAdd(&t.cnt->dropped_events, 1ull);
                continue;
            }
            const uint32_t* tk = tokens + evt.tok_off;
            const uint64_t* eh = hashes + evt.hash_off;
            const bool predicted = keys != nullptr && pred[e] == h;         // phase 1 started this event's chain from the same key
            if (keys != nullptr && !predicted && lane == 0) atomicAdd(&t.cnt->rehashed, 1ull);
            for (uint32_t base = 0; base < nblk; base += 32) {
                uint64_t mine = 0;
                const uint32_t lim = min(32u, nblk - base);
                if (predicted) { if ((uint32_t)lane < lim) mine = keys[evt.hash_off + base + lane]; }
                else {
                    for (uint32_t j = 0; j < lim; ++j) {                     // every lane walks the chain
                        h = hash_block_any(h, tk + (size_t)(base + j) * B, B);
                        if ((uint32_t)lane == j) mine = h;
                    }
                }
                const bool act = (uint32_t)lane < lim;
                const uint32_t am = __ballot_sync(0xffffffffu, act);
                if (act) {
                    // the reference adds the pairs of one event in order: the LAST pair carrying an engine key decides its
                    // mapping, and a request key met twice just has its entry refreshed twice (in_memory.go:159-203)
                    const uint64_t ehash = eh[base + lane];
                    const uint32_t ge = __match_any_sync(am, ehash), gr = __match_any_sync(am, mine);
                    do_add(t, evt.model, ehash, mine, &pt, 1, sb + 2 + 2ull * (base + lane),
                           lane == 31 - __clz(ge), lane == 31 - __clz(gr));
                }
                __syncwarp();
            }
        } else if (evt.op == KVIDX_EV_BLOCK_REMOVED) {
            const uint64_t* eh = hashes + evt.hash_off;
            for (uint32_t base = 0; base < evt.n_hashes; base += 32) {
                const bool act = base + lane < evt.n_hashes;
                const uint32_t am = __ballot_sync(0xffffffffu, act);
                if (act) {
                    const uint64_t ehash = eh[base + lane];
                    const uint32_t ge = __match_any_sync(am, ehash);
                    if (lane == 31 - __clz(ge)) do_evict(t, evt.model, ehash, &pt, 1, sb + 2 + 2ull * (base + lane));
                }
                __syncwarp();
            }
        }
        __syncwarp();
    }
}

// exact-LRU mode, kvidx_apply_events_dev: the largest n_hashes of a device-resident batch (sizes apply_events_kernel's stamp_stride)
__global__ void max_event_hashes_kernel(const kvidx_event_t* __restrict__ ev, int64_t n_ev, unsigned long long* out) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e < n_ev) atomicMax(out, (unsigned long long)ev[e].n_hashes);
}

// ---- exact key-LRU (InMemoryIndexConfig.Size, in_memory.go:59,64): evict the least recently used key -----------
// golang-lru evicts the back of its list when Len() exceeds the size.  Here recency is a stamp per slot; the oldest
// live slot is found with a grid-wide atomicMin and tombstoned.  Evicting a request key does NOT touch the engine map
// (the stale mapping is cleaned up lazily by Evict, in_memory.go:225-230), exactly as in the reference.
__global__ void lru_min_req_kernel(const ReqSlot* __restrict__ tab, const unsigned long long* __restrict__ stamp, uint64_t slots,
                                   unsigned long long* out_min) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < slots && meta_state(tab[i].meta) == kStateFull) atomicMin(out_min, stamp[i]);
}
__global__ void lru_drop_req_kernel(ReqSlot* tab, const unsigned long long* __restrict__ stamp, uint64_t slots,
                                    const unsigned long long* __restrict__ victim, Counters* cnt) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < slots && meta_state(tab[i].meta) == kStateFull && stamp[i] == *victim) {
        for (int j = 0; j < kMaxEnt; ++j) tab[i].ent[j] = 0;
        tab[i].meta = make_meta(kStateTomb, 0, meta_model(tab[i].meta));
        atomicAdd(&cnt->req_full, ~0ull); atomicAdd(&cnt->req_tomb, 1ull); atomicAdd(&cnt->cap_evicted[0], 1ull);
    }
}
__global__ void lru_min_eng_kernel(const EngSlot* __restrict__ tab, uint64_t slots, unsigned long long* out_min) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < slots && meta_state(tab[i].meta) == kStateFull) atomicMin(out_min, (unsigned long long)tab[i].stamp);
}
__global__ void lru_drop_eng_kernel(EngSlot* tab, uint64_t slots, const unsigned long long* __restrict__ victim, Counters* cnt) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < slots && meta_state(tab[i].meta) == kStateFull && tab[i].stamp == *victim) {
        tab[i].meta = make_meta(kStateTomb, 0, meta_model(tab[i].meta));
        atomicAdd(&cnt->eng_full, ~0ull); atomicAdd(&cnt->eng_tomb, 1ull); atomicAdd(&cnt->cap_evicted[1], 1ull);
    }
}

// Re-insert every FULL slot of an old table into a fresh one (drops tombstones).  Runs with the tables quiesced.  A CLOCK
// handle's reference bit moves with its key (old_ref / new_ref; nullptr otherwise).
__global__ void rebuild_req_kernel(const ReqSlot* __restrict__ old_tab, uint64_t old_slots, ReqSlot* new_tab, uint64_t new_mask,
                                   const unsigned long long* __restrict__ old_stamp, unsigned long long* new_stamp,
                                   const uint32_t* __restrict__ old_ref, uint32_t* new_ref) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= old_slots) return;
    const uint4* src = reinterpret_cast<const uint4*>(old_tab + i);
    const uint4 a = src[0];
    uint4 b = src[1];
    if (meta_state(b.w) != kStateFull) return;
    b.w &= ~kLockBit;
    const uint64_t tag = ((uint64_t)a.y << 32) | a.x;
    uint64_t j = slot_home(tag, meta_model(b.w), new_mask);
    for (;;) {
        if (atomicCAS(&new_tab[j].meta, 0u, make_meta(kStateBusy, 0, 0)) == 0u) {
            st_slot(new_tab + j, a, b);
            if (new_stamp) new_stamp[j] = old_stamp[i];
            if (old_ref && ((old_ref[i >> 5] >> (i & 31)) & 1u)) atomicOr(&new_ref[j >> 5], 1u << (j & 31));
            return;
        }
        j = (j + 1) & new_mask;
    }
}
__global__ void rebuild_eng_kernel(const EngSlot* __restrict__ old_tab, uint64_t old_slots, EngSlot* new_tab, uint64_t new_mask,
                                   const uint32_t* __restrict__ old_ref, uint32_t* new_ref) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= old_slots) return;
    const uint4* src = reinterpret_cast<const uint4*>(old_tab + i);
    const uint4 a = src[0];
    uint4 b = src[1];
    if (meta_state(b.x) != kStateFull) return;
    b.x &= ~kLockBit;
    const uint64_t ehash = ((uint64_t)a.y << 32) | a.x;
    uint64_t j = slot_home(ehash, meta_model(b.x), new_mask);
    for (;;) {
        if (atomicCAS(&new_tab[j].meta, 0u, make_meta(kStateBusy, 0, 0)) == 0u) {
            st_slot(new_tab + j, a, b);
            if (old_ref && ((old_ref[i >> 5] >> (i & 31)) & 1u)) atomicOr(&new_ref[j >> 5], 1u << (j & 31));
            return;
        }
        j = (j + 1) & new_mask;
    }
}

// all shards' counters in one buffer (sharded handles: the room check before a write batch looks at every owner)
__global__ void gather_counters_kernel(TableView t, Counters* out) {
    const uint32_t r = threadIdx.x;
    if (r < (1u << t.shard_bits)) {
        const volatile unsigned long long* c = reinterpret_cast<const volatile unsigned long long*>(t.cnt_peer[r]);
        unsigned long long* o = reinterpret_cast<unsigned long long*>(out + r);
        for (int i = 0; i < 8; ++i) o[i] = c[i];
    }
}

}  // namespace kvx
