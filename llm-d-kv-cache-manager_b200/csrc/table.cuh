// table.cuh -- HBM-resident open-addressed tables that replace the reference's two LRU maps
// (pkg/kvcache/kvblock/in_memory.go:77-84):
//   request table : Key{model, chunk hash} -> pod-entry set   (lru.Cache[Key,*PodCache])
//   engine  table : Key{model, engine hash} -> request hash    (lru.Cache[Key,Key])
//
// A slot of either table is exactly one naturally aligned 32-byte DRAM / L2 sector, so a probe that hits its home
// slot costs one sector.  Hopper's widest load / store is 16 bytes, so a slot moves as two halves
// (a = bytes 0..15, b = bytes 16..31), each a single 128-bit access:
//   request slot   bytes  0..7   tag      chunk hash
//                  bytes  8..27  ent[10]  packed (pod<<4|tier), physically ordered oldest -> newest, which is
//                                         the order golang-lru's Keys() returns (in_memory.go:128) and makes the
//                                         per-key pod LRU (in_memory.go:199-203, cap = PodCacheSize) a shift.
//                  bytes 28..31  meta     [1:0] state  [2] writer bit  [7:4] count  [15:8] publish count  [31:16] model id
//   engine slot    ehash, rhash, meta, pad, recency stamp
// Linear probing, power-of-two slot count >= 4 x capacity (load factor <= 0.25).  Deletion leaves a tombstone; the
// owner compacts when tombstones pile up (rebuild / kvidx_shard_compact in kvidx.cu).
//
// Concurrency (Index is called concurrently from gRPC goroutines and event workers, index.go:118):
//   * READERS (Score / Lookup / GetRequestKey kernels) never write.  The meta word is a sequence lock: a reader
//     loads half b (acquire), then half a (acquire), then the meta word again, and keeps the image only if the
//     meta word is unchanged and the writer bit clear; every publish bumps the publish count, so an unchanged meta
//     word means no writer touched the slot in between (the 8-bit count would alias only after 256 publishes of
//     one slot inside one three-load read, each a compare-and-swap round trip).  A reader waits only while a writer owns the very slot it
//     reads.  A BUSY slot (claimed by an insert that has not published yet) is stepped over like a slot of another
//     key.  A reader therefore linearises before or after each individual Add / Evict of a key -- the guarantee
//     the reference's per-key mutex gives (in_memory.go:199-203).
//   * WRITERS own a slot between a successful compare-and-swap on its meta word (FULL -> FULL|W, EMPTY -> BUSY) and
//     the publish of the complete new image: half a, then half b (which carries the meta word) with the bit cleared
//     and the publish count bumped, both release stores.  A writer looking for its key's slot loads half b (acquire)
//     before half a, so a FULL slot it sees always shows that key's tag.  Ownership is per slot, never nested, held for a handful of
//     instructions; there is no table-wide or per-pod lock and no host mutex between the read and the write path.
//     Slots may live in a peer GPU's shard: atomics and publishes are system scope.
//   * Every probe loop is bounded by the slot count: a full shard makes an insert fail (Counters::nospc) instead of
//     spinning.
#pragma once
#include <stdint.h>
#include "fnv_cbor.cuh"

namespace kvx {

constexpr uint32_t kStateEmpty = 0, kStateFull = 1, kStateTomb = 2, kStateBusy = 3;
constexpr uint32_t kStateMask = 3u, kLockBit = 4u;
constexpr uint32_t kPubShift = 8, kPubMask = 0xff00u;
constexpr int kMaxEnt = 10;

struct __align__(32) ReqSlot {
    uint64_t tag;
    uint16_t ent[kMaxEnt];
    uint32_t meta;
};
static_assert(sizeof(ReqSlot) == 32, "request slot must be one 32-byte sector");

struct __align__(32) EngSlot {
    uint64_t ehash;
    uint64_t rhash;
    uint32_t meta;     // [1:0] state [2] writer bit [31:16] model
    uint32_t pad;
    uint64_t stamp;    // recency stamp (exact-LRU mode)
};
static_assert(sizeof(EngSlot) == 32, "engine slot is 32 bytes");

// Home slot: even-aligned so that probe positions 0 and 1 share one 64-byte segment and the read path can
// fetch both with a single coalesced 64-byte access (then linear probing continues at home+2).
__host__ __device__ __forceinline__ uint64_t slot_home(uint64_t hash, uint32_t model, uint64_t mask) {
    return home_of(hash, model) & mask & ~1ull;
}
__host__ __device__ __forceinline__ uint32_t shard_of(uint64_t mixed, uint32_t shard_bits) {
    return shard_bits ? (uint32_t)(mixed >> (64 - shard_bits)) : 0u;
}
__host__ __device__ __forceinline__ uint32_t meta_state(uint32_t m) { return m & kStateMask; }
__host__ __device__ __forceinline__ uint32_t meta_count(uint32_t m) { return (m >> 4) & 0xfu; }
__host__ __device__ __forceinline__ uint32_t meta_model(uint32_t m) { return m >> 16; }
__host__ __device__ __forceinline__ uint32_t make_meta(uint32_t state, uint32_t count, uint32_t model) {
    return state | (count << 4) | (model << 16);
}

struct Counters {
    unsigned long long req_full, req_tomb, eng_full, eng_tomb;
    unsigned long long dropped_events;     // BlockStored with key-count mismatch (in_memory.go:153-155)
    unsigned long long nospc;              // inserts refused because the owning shard is full
    unsigned long long clock;              // recency clock (exact-LRU mode)
    unsigned long long rehashed;           // write path: events whose parent resolved differently from the prediction
    unsigned long long cap_evicted[2];     // request keys / engine mappings dropped by the capacity bound (CLOCK or exact LRU)
    unsigned long long hand[2];            // CLOCK mode: the sweep's hand in the request / engine table (a rebuild resets it)
    unsigned long long sweeps;             // CLOCK mode: sweeps that evicted (both tables) ...
    unsigned long long turns2;             // ... and those of them that went past a full turn of the hand
    unsigned long long rsv[2];
};
static_assert(sizeof(Counters) == 16 * 8, "counter block layout");

struct TableView {
    ReqSlot* req;
    EngSlot* eng;
    unsigned long long* req_stamp;   // per-request-slot recency stamp: exact-LRU mode only (else nullptr).  Engine
                                     // slots carry their stamp inline.  Larger = more recent (golang-lru front).
    uint32_t* req_ref;               // CLOCK mode only (else nullptr): a reference bit per request / engine slot, set where
    uint32_t* eng_ref;               // golang-lru refreshes recency, cleared by the sweep (kernels_clock.cuh)
    uint64_t req_mask, eng_mask;
    uint64_t capacity;
    uint64_t init_hash;
    uint32_t block_size;
    uint32_t pods_per_key;
    uint32_t max_pods;
    uint32_t filter_words;
    Counters* cnt;
    double weight[16];
    // hash-range sharding over the GPUs of one NVSwitch domain: shard = top bits of the mixed key, slot = low bits.
    // *_peer[r] is shard r's table mapped into this process (CUDA IPC); entry `shard_rank` is the local one.
    // Unsharded handles have shard_bits == 0 and *_peer[0] == the local tables.
    ReqSlot* req_peer[8];
    EngSlot* eng_peer[8];
    Counters* cnt_peer[8];
    uint32_t shard_bits, shard_rank;
    uint32_t peer_pair;              // 1: a probe of a peer's shard fetches the slot pair at once (64 B) like a local one; 0: the home slot
                                     // first, its neighbour only if needed (half the NVLink bytes, a second dependent round trip for ~1 probe in 10)
};

#ifdef __CUDACC__

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) { return *(const volatile uint32_t*)p; }

struct SlotWords { uint4 a, b; };   // a = {tag.lo, tag.hi, ent0|1, ent2|3}; b = {ent4|5, ent6|7, ent8|9, meta}

__device__ __forceinline__ void spin_pause() { __nanosleep(40); }

// 16-byte halves.  Not the read-only (.nc) path: writers may publish while a reader kernel runs, and a peer GPU's
// shard is NVLink-mapped memory, so a sharded handle (`sys`) orders its accesses at system scope.
__device__ __forceinline__ uint4 ld_half_acquire(const void* p, bool sys) {
    uint4 r;
    if (sys) asm volatile("ld.acquire.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    else     asm volatile("ld.acquire.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ uint32_t ld_word_relaxed(const void* p, bool sys) {
    uint32_t r;
    if (sys) asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    else     asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ uint4 ld_half_fresh(const void* p) {
    uint4 r;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ void st_half_release(void* p, const uint4& v) {
    asm volatile("st.release.sys.global.v4.u32 [%4], {%0,%1,%2,%3};" :: "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(p) : "memory");
}

// A consistent image of one published slot (the sequence-lock read described at the top).  kMeta is the index of the
// meta word in half b: 3 for a request slot, 0 for an engine slot.  A slot that is not FULL needs no image beyond its
// meta word; half a is then returned as zeros.
template <int kMeta>
__device__ __forceinline__ void ld_slot_t(const void* s, bool sys, uint4& a, uint4& b) {
    const char* p = static_cast<const char*>(s);
    for (;;) {
        b = ld_half_acquire(p + 16, sys);
        const uint32_t m = kMeta == 3 ? b.w : b.x;
        if (meta_state(m) != kStateFull) { a = make_uint4(0u, 0u, 0u, 0u); return; }
        if (m & kLockBit) { spin_pause(); continue; }
        a = ld_half_acquire(p, sys);
        if (ld_word_relaxed(p + 16 + 4 * kMeta, sys) == m) return;
    }
}
__device__ __forceinline__ void ld_slot(const void* s, bool peer, uint4& a, uint4& b) { ld_slot_t<3>(s, peer, a, b); }
// What a writer's acquire loop examines: half b (acquire), then half a.  A FULL meta word seen here was published
// after its tag (release stores, half a first), so the tag read afterwards is that key's; tag, state and model of a
// FULL slot then never change while it stays FULL.  Entries may still move: the owner re-reads them (ld_slot_fresh).
__device__ __forceinline__ void ld_slot_probe(const void* s, uint4& a, uint4& b) {
    b = ld_half_acquire(static_cast<const char*>(s) + 16, true);
    a = ld_half_fresh(s);
}
// Both halves with system-scope coherence (bypasses L1), no consistency check: what a writer reads under ownership.
__device__ __forceinline__ void ld_slot_fresh(const void* s, uint4& a, uint4& b) {
    a = ld_half_fresh(s);
    b = ld_half_fresh(static_cast<const char*>(s) + 16);
}
// publish: half a, then half b carrying the meta word.  The first release also orders the owning compare-and-swap
// before any byte of the new image.
__device__ __forceinline__ void st_slot(void* s, const uint4& a, const uint4& b) {
    st_half_release(s, a);
    st_half_release(static_cast<char*>(s) + 16, b);
}
// meta word of a publish: the caller's state / count / model, writer bit clear, publish count of `old` plus one
__device__ __forceinline__ uint32_t published_meta(uint32_t old, uint32_t new_meta) {
    return (new_meta & ~(kLockBit | kPubMask)) | ((old + (1u << kPubShift)) & kPubMask);
}
__device__ __forceinline__ SlotWords load_slot(const ReqSlot* s, bool peer = false) {
    SlotWords w;
    ld_slot(s, peer, w.a, w.b);
    return w;
}
__device__ __forceinline__ uint32_t slot_ent(const SlotWords& w, int j) {
    // j in [0,10): entries packed two per word starting at a.z
    const uint32_t word = j < 2 ? w.a.z : j < 4 ? w.a.w : j < 6 ? w.b.x : j < 8 ? w.b.y : w.b.z;
    return (j & 1) ? (word >> 16) : (word & 0xffffu);
}

// CLOCK mode: mark slot `slot` as referenced.  The word is read first and the atomic issued only when the bit is clear, so a
// hot key costs a load, not an atomic, per touch.
__device__ __forceinline__ void ref_touch(uint32_t* bits, uint64_t slot) {
    uint32_t* w = bits + (slot >> 5);
    const uint32_t m = 1u << (slot & 31);
    if (!(ld_word_relaxed(w, false) & m)) atomicOr(w, m);
}

// Exact-LRU mode: a touch of a slot's recency stamp.  One call may touch a key many times from many threads (prompts that
// share a prefix, pods that store the same block); every touch carries a stamp unique within the call and ordered as the
// reference applies the call, so the largest stamp is the last touch, whichever thread stores last.
__device__ __forceinline__ void stamp_touch(unsigned long long* p, unsigned long long stamp) { atomicMax(p, stamp); }
// An engine slot's stamp word is NOT part of the image an exact-LRU writer publishes (eng_publish_lru): eng_find touches it
// without owning the slot, and a publish of the whole half b would put back the stamp read when the writer acquired the
// slot.  Readers still see whole images: what they read is {ehash, rhash, meta}, checked by the meta word's sequence lock
// as before, and no reader uses the stamp -- only the LRU cut and the snapshot read it, after the call.
__device__ __forceinline__ void eng_stamp_touch(EngSlot* s, unsigned long long stamp) {
    stamp_touch(reinterpret_cast<unsigned long long*>(&s->stamp), stamp);
}

// ---- readers ------------------------------------------------------------------------------------------

// Finds the FULL slot holding (model, tag).  Returns false at the first EMPTY slot (or after a full cycle).
__device__ __forceinline__ bool req_find(const TableView& t, uint32_t model, uint64_t tag, SlotWords& w, uint64_t* slot_out = nullptr) {
    const uint64_t hm = home_of(tag, model);
    const ReqSlot* base = t.req_peer[shard_of(hm, t.shard_bits)];
    uint64_t i = hm & t.req_mask & ~1ull;
    const uint32_t tlo = (uint32_t)tag, thi = (uint32_t)(tag >> 32);
    for (uint64_t step = 0; step <= t.req_mask; ++step) {
        w = load_slot(base + i, t.shard_bits != 0);
        const uint32_t st = meta_state(w.b.w);
        if (st == kStateEmpty) return false;
        if (st == kStateFull && w.a.x == tlo && w.a.y == thi && meta_model(w.b.w) == model) {
            if (slot_out) *slot_out = i;
            return true;
        }
        i = (i + 1) & t.req_mask;
    }
    return false;
}

// engine -> request lookup (GetRequestKey, in_memory.go:264-270).  An engine slot image is {ehash, rhash | meta, pad, stamp}.
__device__ __forceinline__ bool eng_find(const TableView& t, uint32_t model, uint64_t ehash, uint64_t* rhash, uint64_t* slot_out = nullptr,
                                         unsigned long long stamp = 0, bool touch = false) {
    const uint64_t hm = home_of(ehash, model);
    const EngSlot* base = t.eng_peer[shard_of(hm, t.shard_bits)];
    uint64_t i = hm & t.eng_mask & ~1ull;
    const uint32_t elo = (uint32_t)ehash, ehi = (uint32_t)(ehash >> 32);
    for (uint64_t step = 0; step <= t.eng_mask; ++step) {
        const EngSlot* s = base + i;
        uint4 a, b;
        ld_slot_t<0>(s, t.shard_bits != 0, a, b);
        const uint32_t st = meta_state(b.x);
        if (st == kStateEmpty) return false;
        if (st == kStateFull && meta_model(b.x) == model && a.x == elo && a.y == ehi) {
            *rhash = ((uint64_t)a.w << 32) | a.z;
            if (slot_out) *slot_out = i;
            if (stamp && t.req_stamp) eng_stamp_touch(const_cast<EngSlot*>(s), stamp);               // lru Get refreshes recency
            if (touch && t.eng_ref) ref_touch(t.eng_ref, i);                                        // ... CLOCK: its bit
            return true;
        }
        i = (i + 1) & t.eng_mask;
    }
    return false;
}

// ---- writers ------------------------------------------------------------------------------------------
// Entry list of a request-slot image in registers (static indices only, so it stays in registers).
struct EntList {
    uint32_t e[kMaxEnt];
    __device__ __forceinline__ void unpack(const uint4& a, const uint4& b) {
        e[0] = a.z & 0xffffu; e[1] = a.z >> 16; e[2] = a.w & 0xffffu; e[3] = a.w >> 16; e[4] = b.x & 0xffffu; e[5] = b.x >> 16;
        e[6] = b.y & 0xffffu; e[7] = b.y >> 16; e[8] = b.z & 0xffffu; e[9] = b.z >> 16;
    }
    __device__ __forceinline__ void pack(uint4& a, uint4& b) const {
        a.z = e[0] | (e[1] << 16); a.w = e[2] | (e[3] << 16); b.x = e[4] | (e[5] << 16); b.y = e[6] | (e[7] << 16); b.z = e[8] | (e[9] << 16);
    }
    // remove position pos (< count): later entries move down, the vacated last position is zeroed so that slots with
    // equal live entries are bitwise equal (the score kernels compare slot images)
    __device__ __forceinline__ void remove_at(uint32_t pos) {
#pragma unroll
        for (int j = 0; j < kMaxEnt - 1; ++j) if ((uint32_t)j >= pos) e[j] = e[j + 1];
        e[kMaxEnt - 1] = 0;
    }
    __device__ __forceinline__ void set(uint32_t pos, uint32_t v) {
#pragma unroll
        for (int j = 0; j < kMaxEnt; ++j) if ((uint32_t)j == pos) e[j] = v;
    }
    __device__ __forceinline__ int find(uint32_t count, uint32_t pt) const {
        int pos = -1;
#pragma unroll
        for (int j = 0; j < kMaxEnt; ++j) if ((uint32_t)j < count && e[j] == pt) pos = j;
        return pos;
    }
    // PodCache.Add under podCache.mu (in_memory.go:199-203) with golang-lru semantics: an existing entry is refreshed
    // to newest, a new one is appended and the oldest dropped beyond the cap.  Returns the new count.
    __device__ __forceinline__ uint32_t add(uint32_t count, uint32_t pt, uint32_t cap) {
        const int pos = find(count, pt);
        if (pos >= 0) { remove_at((uint32_t)pos); set(count - 1, pt); return count; }
        if (count >= cap) { remove_at(0); --count; }
        set(count, pt);
        return count + 1;
    }
    // PodCache.Remove (in_memory.go:233-235): exact (pod,tier) match only.  Returns the new count.
    __device__ __forceinline__ uint32_t remove(uint32_t count, uint32_t pt) {
        const int pos = find(count, pt);
        if (pos < 0) return count;
        remove_at((uint32_t)pos);
        return count - 1;
    }
};

// Take ownership of the request slot of (model, tag); claim a fresh one if the key is absent (unless must_exist).
// On success the slot's current image is in (a, b) (for a fresh slot: tag set, no entries) and *created tells which.
// Returns nullptr if must_exist and the key is absent, or if the shard is full (*full set).
__device__ __forceinline__ ReqSlot* req_acquire(const TableView& t, uint32_t model, uint64_t tag, bool must_exist, bool* created,
                                                uint4& a, uint4& b, bool* full = nullptr) {
    const uint64_t hm = home_of(tag, model);
    ReqSlot* base = t.req_peer[shard_of(hm, t.shard_bits)];
    uint64_t i = hm & t.req_mask & ~1ull;
    const uint32_t tlo = (uint32_t)tag, thi = (uint32_t)(tag >> 32);
    *created = false;
    if (full) *full = false;
    for (uint64_t step = 0; step <= t.req_mask;) {
        ReqSlot* s = base + i;
        ld_slot_probe(s, a, b);
        const uint32_t m = b.w, st = meta_state(m);
        if (st == kStateBusy) { spin_pause(); continue; }              // another insert is publishing here: it may be this key
        if (st == kStateEmpty) {
            if (must_exist) return nullptr;
            if (atomicCAS_system(&s->meta, m, make_meta(kStateBusy, 0, model)) == m) {
                a = make_uint4(tlo, thi, 0u, 0u); b = make_uint4(0u, 0u, 0u, 0u);
                *created = true;
                return s;
            }
            continue;                                                  // lost the race: re-examine this slot
        }
        if (st == kStateFull && a.x == tlo && a.y == thi && meta_model(m) == model) {
            if (m & kLockBit) { spin_pause(); continue; }              // another writer owns it
            if (atomicCAS_system(&s->meta, m, m | kLockBit) == m) {
                ld_slot_fresh(s, a, b);                                // the image under ownership (entries may have moved
                return s;                                              //  since the first load even if meta looks the same)
            }
            continue;
        }
        i = (i + 1) & t.req_mask; ++step;
    }
    if (full) *full = true;
    return nullptr;
}
// publish the image with the given meta (writer bit clear) and give the slot up; b.w still holds the owned meta word
__device__ __forceinline__ void req_publish(ReqSlot* s, uint4& a, uint4& b, uint32_t new_meta) {
    b.w = published_meta(b.w, new_meta);
    st_slot(s, a, b);
}

// engine slot image: a = {ehash.lo, ehash.hi, rhash.lo, rhash.hi}, b = {meta, pad, stamp.lo, stamp.hi}
__device__ __forceinline__ EngSlot* eng_acquire(const TableView& t, uint32_t model, uint64_t ehash, bool must_exist, bool* created,
                                                uint4& a, uint4& b, bool* full = nullptr) {
    const uint64_t hm = home_of(ehash, model);
    EngSlot* base = t.eng_peer[shard_of(hm, t.shard_bits)];
    uint64_t i = hm & t.eng_mask & ~1ull;
    const uint32_t elo = (uint32_t)ehash, ehi = (uint32_t)(ehash >> 32);
    *created = false;
    if (full) *full = false;
    for (uint64_t step = 0; step <= t.eng_mask;) {
        EngSlot* s = base + i;
        ld_slot_probe(s, a, b);
        const uint32_t m = b.x, st = meta_state(m);
        if (st == kStateBusy) { spin_pause(); continue; }
        if (st == kStateEmpty) {
            if (must_exist) return nullptr;
            if (atomicCAS_system(&s->meta, m, make_meta(kStateBusy, 0, model)) == m) {
                a = make_uint4(elo, ehi, 0u, 0u); b = make_uint4(0u, 0u, 0u, 0u);
                *created = true;
                return s;
            }
            continue;
        }
        if (st == kStateFull && a.x == elo && a.y == ehi && meta_model(m) == model) {
            if (m & kLockBit) { spin_pause(); continue; }
            if (atomicCAS_system(&s->meta, m, m | kLockBit) == m) { ld_slot_fresh(s, a, b); return s; }
            continue;
        }
        i = (i + 1) & t.eng_mask; ++step;
    }
    if (full) *full = true;
    return nullptr;
}
__device__ __forceinline__ void eng_publish(EngSlot* s, uint4& a, uint4& b, uint32_t new_meta) {
    b.x = published_meta(b.x, new_meta);
    st_slot(s, a, b);
}
// exact-LRU mode: the same publish without the stamp word (eng_stamp_touch): half a, then meta and pad as one 8-byte release
__device__ __forceinline__ void eng_publish_lru(EngSlot* s, uint4& a, uint4& b, uint32_t new_meta) {
    b.x = published_meta(b.x, new_meta);
    st_half_release(s, a);
    asm volatile("st.release.sys.global.v2.u32 [%2], {%0,%1};" :: "r"(b.x), "r"(b.y), "l"(&s->meta) : "memory");
}

__device__ __forceinline__ Counters* cnt_of(const TableView& t, uint64_t hash, uint32_t model) {
    return t.cnt_peer[shard_of(home_of(hash, model), t.shard_bits)];
}

#endif  // __CUDACC__
}  // namespace kvx
