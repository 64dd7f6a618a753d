// kernels_text.cuh -- the device prefix store: prefixstore.LRUTokenStore (lru_store.go:54-190) on the GPU.
//
// Text is cut into B-byte blocks (a partial last block is never stored or looked up).  Block b's key is XXH64 (seed 0) of
// the previous block's key (8 bytes little-endian, 0 for block 0) followed by the block's bytes, bit-identical to the host
// store's chain (kvhost_xxhash64).  A block holds the tokens whose END offset is <= the block's end and that no earlier
// block took, in token order (lru_store.go:128-135).
//
// Storage: an open-addressed table of keys (linear probing, load <= 1/2, no deletions: eviction rebuilds it), a recency
// stamp per slot, and per slot one record (offset, length) into a u32 token arena.  Records are append-only; an update
// leaves the old one dead, and the arena is compacted when an append would not fit.
//
// Hashing: the chain is serial across a prompt's blocks, but XXH64's four accumulators are independent across 32-byte
// stripes.  A group of L lanes hashes one prompt (L = 4: lane j owns accumulator j; L = 1: a thread per prompt, for large
// batches).  Text is read bytewise: prompts start at arbitrary byte offsets.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace kvx {

constexpr int kTextThreads = 256;
constexpr uint64_t kXP1 = 0x9E3779B185EBCA87ull, kXP2 = 0xC2B2AE3D27D4EB4Full, kXP3 = 0x165667B19E3779F9ull,
                   kXP4 = 0x85EBCA77C2B2AE63ull, kXP5 = 0x27D4EB2F165667C5ull;
constexpr uint32_t kTextEmpty = 0, kTextBusy = 1, kTextFull = 2;      // slot states

// The store's table (device pointers; slots a power of two).
struct TextTable {
    uint64_t* key; uint32_t* state; unsigned long long* stamp; int64_t* off; int64_t* len;
    uint64_t mask;
};

__device__ __forceinline__ uint64_t xx_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t xx_round(uint64_t acc, uint64_t in) { return xx_rotl(acc + in * kXP2, 31) * kXP1; }
__device__ __forceinline__ uint64_t xx_merge(uint64_t h, uint64_t v) { return (h ^ xx_round(0, v)) * kXP1 + kXP4; }

__device__ __forceinline__ uint64_t ld_u64_bytes(const uint8_t* p) {
    uint64_t v = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) v |= (uint64_t)p[i] << (8 * i);
    return v;
}
__device__ __forceinline__ uint32_t ld_u32_bytes(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// The 8-byte word at message offset k (a multiple of 8) of prev || blk.
__device__ __forceinline__ uint64_t xx_word(uint64_t prev, const uint8_t* blk, uint32_t k) { return k == 0 ? prev : ld_u64_bytes(blk + (k - 8)); }

// XXH64(prev || blk[0 .. B)), seed 0, computed by the L lanes of a group (lane g in 0 .. L-1, all lanes get the result).
// `gmask` is the group's lanes in the warp.
template <int L>
__device__ __forceinline__ uint64_t xx_chain(uint64_t prev, const uint8_t* blk, uint32_t B, int g, unsigned gmask) {
    const uint32_t M = B + 8;
    uint64_t h;
    uint32_t k = 0;
    if (M >= 32) {
        uint64_t v0 = kXP1 + kXP2, v1 = kXP2, v2 = 0, v3 = 0ull - kXP1;
        if (L == 1) {
            for (; k + 32 <= M; k += 32) {
                v0 = xx_round(v0, xx_word(prev, blk, k));
                v1 = xx_round(v1, xx_word(prev, blk, k + 8));
                v2 = xx_round(v2, xx_word(prev, blk, k + 16));
                v3 = xx_round(v3, xx_word(prev, blk, k + 24));
            }
        } else {
            uint64_t a = g == 0 ? v0 : g == 1 ? v1 : g == 2 ? v2 : v3;
            for (; k + 32 <= M; k += 32) a = xx_round(a, xx_word(prev, blk, k + 8 * g));
            v0 = __shfl_sync(gmask, a, 0, L); v1 = __shfl_sync(gmask, a, 1, L);
            v2 = __shfl_sync(gmask, a, 2, L); v3 = __shfl_sync(gmask, a, 3, L);
        }
        h = xx_rotl(v0, 1) + xx_rotl(v1, 7) + xx_rotl(v2, 12) + xx_rotl(v3, 18);
        h = xx_merge(h, v0); h = xx_merge(h, v1); h = xx_merge(h, v2); h = xx_merge(h, v3);
    } else {
        h = kXP5;
    }
    h += (uint64_t)M;
    for (; k + 8 <= M; k += 8) h = xx_rotl(h ^ xx_round(0, xx_word(prev, blk, k)), 27) * kXP1 + kXP4;
    // the 4-byte and 1-byte tails lie past the first 8 bytes whenever they exist (k >= 8 here unless M < 8, impossible)
    if (k + 4 <= M) { h = xx_rotl(h ^ ((uint64_t)ld_u32_bytes(blk + (k - 8)) * kXP1), 23) * kXP2 + kXP3; k += 4; }
    for (; k < M; ++k) h = xx_rotl(h ^ ((uint64_t)blk[k - 8] * kXP5), 11) * kXP1;
    h ^= h >> 33; h *= kXP2; h ^= h >> 29; h *= kXP3; h ^= h >> 32;
    return h;
}

__device__ __forceinline__ uint64_t text_home(uint64_t key, uint64_t mask) {
    uint64_t h = key ^ (key >> 29);
    h *= 0xBF58476D1CE4E5B9ull;
    return (h ^ (h >> 32)) & mask;
}

// Read-only probe (no insert can run at the same time: store calls are serialised).  -> slot, or -1.
__device__ __forceinline__ int64_t text_probe(const TextTable& t, uint64_t key) {
    for (uint64_t s = text_home(key, t.mask);; s = (s + 1) & t.mask) {
        if (t.state[s] == kTextEmpty) return -1;
        if (t.key[s] == key) return (int64_t)s;
    }
}

// Find-or-insert; concurrent callers with the same key get the same slot.  *inserted = 1 for the thread that claimed it.
__device__ __forceinline__ uint64_t text_upsert(const TextTable& t, uint64_t key, int* inserted) {
    *inserted = 0;
    for (uint64_t s = text_home(key, t.mask);; s = (s + 1) & t.mask) {
        uint32_t st = atomicCAS(&t.state[s], kTextEmpty, kTextBusy);
        if (st == kTextEmpty) {
            t.key[s] = key;
            __threadfence();
            atomicExch(&t.state[s], kTextFull);
            *inserted = 1;
            return s;
        }
        while (st == kTextBusy) st = *(volatile uint32_t*)&t.state[s];
        __threadfence();
        if (*(volatile uint64_t*)&t.key[s] == key) return s;
    }
}

// Blocks per prompt: floor(len / B); with tok_off (an add call), 0 for a prompt without tokens (lru_store.go:96-98).
// Writes cnt[i + 1] (cnt[0] = 0 by the caller), to be scanned into the block offsets.
__global__ void text_block_counts_kernel(const int64_t* __restrict__ text_off, const int64_t* __restrict__ tok_off, int64_t n,
                                         uint32_t B, int64_t* __restrict__ cnt) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t len = text_off[i + 1] - text_off[i];
        cnt[i + 1] = (tok_off && tok_off[i + 1] == tok_off[i]) ? 0 : len / (int64_t)B;
    }
}

// Every block key of every prompt: key[blk_off[i] + b].  L lanes per prompt.
template <int L>
__global__ void __launch_bounds__(kTextThreads) text_hash_kernel(const uint8_t* __restrict__ text, const int64_t* __restrict__ text_off,
                                                                 int64_t text_base, int64_t n, uint32_t B,
                                                                 const int64_t* __restrict__ blk_off, uint64_t* __restrict__ key) {
    const int g = threadIdx.x % L;
    const unsigned gmask = L == 1 ? __activemask() : (((1u << L) - 1) << ((threadIdx.x & 31) & ~(L - 1)));
    const int64_t groups = (int64_t)gridDim.x * blockDim.x / L;
    for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / L; i < n; i += groups) {
        const uint8_t* p = text + (text_off[i] - text_base);
        const int64_t k0 = blk_off[i], nb = blk_off[i + 1] - k0;
        uint64_t prev = 0;
        for (int64_t b = 0; b < nb; ++b) {
            prev = xx_chain<L>(prev, p + b * B, B, g, gmask);
            if (g == 0) key[k0 + b] = prev;
        }
    }
}

// Find, pass one: walk each prompt's blocks until the first miss.  hit_slot[blk_off[i] + b] for the hits, nhit[i],
// tokens[i + 1] = their token count (the caller scans it), ratio[i] (may be NULL).  With min_ratio >= 0 (Score() from text)
// also score_tok[i + 1] = tokens of a prompt whose ratio passes, else 0, and tokenize[i] = !pass.
template <int L>
__global__ void __launch_bounds__(kTextThreads) text_find_kernel(const TextTable t, const uint8_t* __restrict__ text,
                                                                 const int64_t* __restrict__ text_off, int64_t text_base, int64_t n,
                                                                 uint32_t B, const int64_t* __restrict__ blk_off,
                                                                 uint32_t* __restrict__ hit_slot, int64_t* __restrict__ nhit,
                                                                 int64_t* __restrict__ tokens, double* __restrict__ ratio,
                                                                 double min_ratio, int64_t* __restrict__ score_tok,
                                                                 uint8_t* __restrict__ tokenize) {
    const int g = threadIdx.x % L;
    const unsigned gmask = L == 1 ? __activemask() : (((1u << L) - 1) << ((threadIdx.x & 31) & ~(L - 1)));
    const int64_t groups = (int64_t)gridDim.x * blockDim.x / L;
    for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / L; i < n; i += groups) {
        const int64_t len = text_off[i + 1] - text_off[i];
        const uint8_t* p = text + (text_off[i] - text_base);
        const int64_t k0 = blk_off[i], nb = blk_off[i + 1] - k0;
        uint64_t prev = 0;
        int64_t b = 0, ntok = 0;
        for (; b < nb; ++b) {
            prev = xx_chain<L>(prev, p + b * B, B, g, gmask);
            const int64_t s = text_probe(t, prev);           // every lane probes the same key: the same answer
            if (s < 0) break;
            if (g == 0) hit_slot[k0 + b] = (uint32_t)s;
            ntok += t.len[s];
        }
        if (g != 0) continue;
        const double r = b > 0 ? (double)(b * (int64_t)B) / (double)len : 0.0;
        nhit[i] = b;
        tokens[i + 1] = ntok;
        if (ratio) ratio[i] = r;
        if (score_tok) {
            const bool pass = r >= min_ratio;
            score_tok[i + 1] = pass ? ntok : 0;
            tokenize[i] = pass ? 0 : 1;
        }
    }
}

// Find, pass two: a warp per prompt refreshes its hits (stamp = base + blk_off[i] + b: prompt after prompt, block after
// block) and copies their tokens to out + out_off[i] (out NULL: refresh only).  With `gate`
// (Score() from text) only prompts whose gate[i] == 0 (not sent to the tokenizer) are copied; every prompt refreshes.
__global__ void __launch_bounds__(kTextThreads) text_gather_kernel(const TextTable t, const uint32_t* __restrict__ arena, int64_t n,
                                                                   const int64_t* __restrict__ blk_off, const uint32_t* __restrict__ hit_slot,
                                                                   const int64_t* __restrict__ nhit, unsigned long long stamp_base,
                                                                   const int64_t* __restrict__ out_off, const uint8_t* __restrict__ gate,
                                                                   uint32_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * blockDim.x / 32;
    for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32; i < n; i += warps) {
        const int64_t k0 = blk_off[i], nb = nhit[i];
        const bool copy = out && !(gate && gate[i]);
        int64_t o = copy ? out_off[i] : 0;
        for (int64_t b = 0; b < nb; ++b) {
            const uint32_t s = hit_slot[k0 + b];
            if (lane == 0) atomicMax(&t.stamp[s], stamp_base + (unsigned long long)(k0 + b));
            if (!copy) continue;
            const int64_t ro = t.off[s], rl = t.len[s];
            for (int64_t j = lane; j < rl; j += 32) out[o + j] = arena[ro + j];
            o += rl;
        }
    }
}

// Add, step one: a thread per prompt walks its tokens and gives each block its run [src, src + cnt) of the call's tokens
// (token index into tok, relative to tok_base).  tok_span holds [low, high) byte pairs; only `high` decides.
__global__ void text_add_ranges_kernel(const int64_t* __restrict__ tok_off, int64_t tok_base, const uint64_t* __restrict__ tok_span,
                                       int64_t n, uint32_t B, const int64_t* __restrict__ blk_off, int64_t* __restrict__ src,
                                       int64_t* __restrict__ cnt) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k0 = blk_off[i], nb = blk_off[i + 1] - k0;
        const int64_t t0 = tok_off[i] - tok_base, t1 = tok_off[i + 1] - tok_base;
        int64_t it = t0;
        for (int64_t b = 0; b < nb; ++b) {
            const uint64_t end = (uint64_t)(b + 1) * B;
            const int64_t lo = it;
            while (it < t1 && tok_span[2 * it + 1] <= end) ++it;
            src[k0 + b] = lo;
            cnt[k0 + b + 1] = it - lo;
        }
    }
}

// Add, step two: a warp per block copies its run to the arena at arena_base + pos[k] (pos: scanned cnt).
__global__ void __launch_bounds__(kTextThreads) text_add_copy_kernel(const uint32_t* __restrict__ tok, const int64_t* __restrict__ src,
                                                                     const int64_t* __restrict__ pos, int64_t nblk, int64_t arena_base,
                                                                     uint32_t* __restrict__ arena) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * blockDim.x / 32;
    for (int64_t k = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32; k < nblk; k += warps) {
        const int64_t s = src[k], c = pos[k + 1] - pos[k], d = arena_base + pos[k];
        for (int64_t j = lane; j < c; j += 32) arena[d + j] = tok[s + j];
    }
}

// Add, step three: every block touches its key (insert or update), stamp = stamp_base + k (the call's order: prompt after
// prompt, block after block).  slot_of[k] for step four; *inserted counts the new keys.
__global__ void text_add_touch_kernel(const TextTable t, const uint64_t* __restrict__ key, int64_t nblk, unsigned long long stamp_base,
                                      uint32_t* __restrict__ slot_of, unsigned long long* __restrict__ inserted) {
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nblk; k += (int64_t)gridDim.x * blockDim.x) {
        int ins;
        const uint64_t s = text_upsert(t, key[k], &ins);
        if (ins) atomicAdd(inserted, 1ull);
        atomicMax(&t.stamp[s], stamp_base + (unsigned long long)k);
        slot_of[k] = (uint32_t)s;
    }
}

// Add, step four: the last touch of a key in the call (the one whose stamp the slot kept) points the slot at its record.
__global__ void text_add_commit_kernel(const TextTable t, int64_t nblk, unsigned long long stamp_base, const uint32_t* __restrict__ slot_of,
                                       const int64_t* __restrict__ pos, int64_t arena_base) {
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nblk; k += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t s = slot_of[k];
        if (t.stamp[s] != stamp_base + (unsigned long long)k) continue;
        t.off[s] = arena_base + pos[k];
        t.len[s] = pos[k + 1] - pos[k];
    }
}

// The stamps of the full slots, in any order (*n counts them), for the eviction cut; with slot_out (a snapshot) each
// stamp's slot beside it; and the live token count.
__global__ void text_stamps_kernel(const TextTable t, unsigned long long* __restrict__ out, uint32_t* __restrict__ slot_out,
                                   unsigned long long* __restrict__ n, unsigned long long* __restrict__ live_tokens) {
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s <= t.mask; s += (uint64_t)gridDim.x * blockDim.x) {
        if (t.state[s] != kTextFull) continue;
        if (out) {
            const unsigned long long i = atomicAdd(n, 1ull);
            out[i] = t.stamp[s];
            if (slot_out) slot_out[i] = (uint32_t)s;
        }
        if (live_tokens) atomicAdd(live_tokens, (unsigned long long)t.len[s]);
    }
}

// ---- snapshot and restore: the image of kvidx_text_store_snapshot (include/kvidx.h) --------------------------------------
// Snapshot: cnt[i + 1] = the token count of the i-th slot in recency order (slot[], sorted by stamp), to be scanned.
__global__ void text_snap_len_kernel(const TextTable t, const uint32_t* __restrict__ slot, int64_t R, int64_t* __restrict__ cnt) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R; i += (int64_t)gridDim.x * blockDim.x)
        cnt[i + 1] = t.len[slot[i]];
}

// ... then a warp per record writes it (u64 key, u32 n_tok, u32 0) to rec + 16 i and copies its tokens to tok + tok_off[i].
__global__ void __launch_bounds__(kTextThreads) text_snapshot_kernel(const TextTable t, const uint32_t* __restrict__ arena,
                                                                     const uint32_t* __restrict__ slot, const int64_t* __restrict__ tok_off,
                                                                     int64_t R, uint4* __restrict__ rec, uint32_t* __restrict__ tok) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * blockDim.x / 32;
    for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32; i < R; i += warps) {
        const uint32_t s = slot[i];
        const int64_t o = t.off[s], c = t.len[s], d = tok_off[i];
        if (lane == 0) {
            const uint64_t k = t.key[s];
            rec[i] = make_uint4((uint32_t)k, (uint32_t)(k >> 32), (uint32_t)c, 0u);
        }
        for (int64_t j = lane; j < c; j += 32) tok[d + j] = arena[o + j];
    }
}

// Restore, check one: every record's key to key[i] and its token count to cnt[i + 1] (to be scanned); non-zero padding
// sets *bad.
__global__ void text_restore_records_kernel(const uint4* __restrict__ rec, int64_t R, uint64_t* __restrict__ key, int64_t* __restrict__ cnt,
                                            unsigned long long* __restrict__ bad) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R; i += (int64_t)gridDim.x * blockDim.x) {
        const uint4 r = rec[i];
        key[i] = (uint64_t)r.x | ((uint64_t)r.y << 32);
        cnt[i + 1] = r.z;
        if (r.w != 0) atomicOr(bad, 1ull);
    }
}

// Restore, check two: a key equal to its neighbour in the sorted copy appears twice in the image.
__global__ void text_restore_dups_kernel(const uint64_t* __restrict__ sorted, int64_t R, unsigned long long* __restrict__ bad) {
    for (int64_t i = 1 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R; i += (int64_t)gridDim.x * blockDim.x)
        if (sorted[i] == sorted[i - 1]) atomicOr(bad, 2ull);
}

// Rebuild: the full slots of `from` with stamp >= keep_from go into the empty table `to` (keys are distinct: no races on
// a key, only on slots).
__global__ void text_rebuild_kernel(const TextTable from, const TextTable to, unsigned long long keep_from) {
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s <= from.mask; s += (uint64_t)gridDim.x * blockDim.x) {
        if (from.state[s] != kTextFull || from.stamp[s] < keep_from) continue;
        const uint64_t k = from.key[s];
        for (uint64_t d = text_home(k, to.mask);; d = (d + 1) & to.mask) {
            if (atomicCAS(&to.state[d], kTextEmpty, kTextFull) != kTextEmpty) continue;
            to.key[d] = k; to.stamp[d] = from.stamp[s]; to.off[d] = from.off[s]; to.len[d] = from.len[s];
            break;
        }
    }
}

// Arena compaction: rec_len[s] = the record length of slot s (0 when not full), to be scanned into new offsets.
__global__ void text_rec_len_kernel(const TextTable t, int64_t* __restrict__ rec_len) {
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s <= t.mask; s += (uint64_t)gridDim.x * blockDim.x)
        rec_len[s + 1] = t.state[s] == kTextFull ? t.len[s] : 0;
}

// ... then a warp per slot moves its record to the new arena and repoints the slot.
__global__ void __launch_bounds__(kTextThreads) text_compact_kernel(const TextTable t, const int64_t* __restrict__ new_off,
                                                                    const uint32_t* __restrict__ from, uint32_t* __restrict__ to) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * blockDim.x / 32;
    for (uint64_t s = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) / 32; s <= t.mask; s += warps) {
        if (t.state[s] != kTextFull) continue;
        const int64_t o = t.off[s], d = new_off[s], c = t.len[s];
        for (int64_t j = lane; j < c; j += 32) to[d + j] = from[o + j];
        __syncwarp();
        if (lane == 0) t.off[s] = d;
    }
}

}  // namespace kvx
