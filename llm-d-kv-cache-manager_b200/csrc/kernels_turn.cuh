// kernels_turn.cuh -- Score() for a conversation turn: the request keys a caller holds, followed by the new turn's tokens.
//
// Prompt i is K_i = held_i ++ TokensToKVBlockKeys(parent = last held key, or init_hash, new tokens_i)
// (kvblock/token_processor.go:141-162); its row is LongestPrefixScorer.Score(K_i, Index.Lookup(K_i, pods))
// (kvblock_scorer.go:108-151, in_memory.go:105-146), and the keys of the new tokens are handed back so that the next turn
// holds them.  One warp per prompt at every batch size, with the coop kernel's shared memory:
//   * held-key phase: score_keys_kernel's chunk (keys_walk_chunk): lane j loads and probes key j, a ballot finds the first
//     miss, WarpWalk scores and marks.  The prompt's first token chunk is TMA-staged before it starts, so it lands while
//     the keys are walked;
//   * token phase: the coop kernel's chunk (coop_walk_chunk), chain seeded with the last held key, the walk state carried
//     on.  Probes stop where the walk stops, in either phase; the hashing goes on to the prompt's last full block only when
//     the new keys are wanted (lane j stores the key of the chunk's block j: one store of 512 / B keys per chunk).
// Built for block sizes B = 16, 32, 64 and 128, as the coop kernel.  Composed path (other block sizes, exact-LRU handles,
// KVIDX_SCORE_KERNEL=v1): hash_keys_kernel_v1 with each prompt's parent read on the device, turn_concat_kernel, then
// Score() from the concatenated keys.
#pragma once
#include <cuda_runtime.h>
#include "score_common.cuh"
#include "kernels_coop.cuh"
#include "kernels_keys.cuh"

namespace kvx {

// The parts of a turn besides ScoreArgs (whose tok_off / tok_base describe the held-key CSR): the held keys, the new tokens
// (prompt i owns tok[tok_off[i] - tok_base .. tok_off[i+1] - tok_base)), and where prompt i's new keys go
// (new_keys + new_off[i] - new_base; new_keys NULL: not wanted, new_off may be NULL too).
struct TurnArgs {
    const uint64_t* keys;
    const uint32_t* tok; const int64_t* tok_off; int64_t tok_base;
    uint64_t* new_keys; const int64_t* new_off; int64_t new_base;
};

template <int BS>
__global__ void __launch_bounds__(kCoopThreads, CoopGeom<BS>::kMinCtas)
score_turn_kernel(const TableView t, const ScoreArgs a, const TurnArgs ta) {
    constexpr int NB = CoopGeom<BS>::kBlocks;
    const uint64_t l2pol = l2_policy_stream();
    extern __shared__ __align__(128) unsigned char smem_raw_t[];
    CoopSmem<BS>& sm = *reinterpret_cast<CoopSmem<BS>*>(smem_raw_t);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
    typename CoopSmem<BS>::Warp& W = sm.w[wid];
    coop_setup<BS>(sm, W, lane);
    const bool peer = t.shard_bits != 0;
    uint32_t phases = 0;                                                  // bit s: parity the next wait on buffer s uses
    const long long total_warps = (long long)gridDim.x * kCoopWarps;
    for (long long pi = (long long)blockIdx.x * kCoopWarps + wid; pi < a.n_prompts; pi += total_warps) {
        const int64_t kb = a.tok_off[pi] - a.tok_base, nk = a.tok_off[pi + 1] - a.tok_base - kb;
        const int64_t tb0 = ta.tok_off[pi] - ta.tok_base, te = ta.tok_off[pi + 1] - ta.tok_base;
        const int nblk = (int)((te - tb0) / BS);
        const uint32_t* tokp = ta.tok + tb0;
        const bool aligned = (reinterpret_cast<uintptr_t>(tokp) & 15u) == 0;
        const uint32_t mdl = a.model ? a.model[pi] : a.model0;
        uint64_t* nkp = ta.new_keys ? ta.new_keys + (ta.new_off[pi] - ta.new_base) : nullptr;
        const uint64_t* kp = ta.keys + kb;
        uint64_t h = nk > 0 ? __ldg(kp + nk - 1) : t.init_hash;          // the chain's parent: the last held key
        coop_stage<BS>(W, tokp, nblk, 0, aligned, lane);                  // lands while the held keys are walked
        WarpWalk ws;
        // ---- held keys ----
        bool walking = true;
        uint64_t key = 0;
        if (lane < nk) key = ld_stream_u64(kp + lane, l2pol);
        for (int64_t c0 = 0; c0 < nk; c0 += kKeysChunk) {
            const int nb = nk - c0 < kKeysChunk ? (int)(nk - c0) : kKeysChunk;
            uint64_t next = 0;
            if (c0 + kKeysChunk + lane < nk) next = ld_stream_u64(kp + c0 + kKeysChunk + lane, l2pol);
            if (!keys_walk_chunk(t, ws, lane, key, nb, mdl, peer, c0 > 0, c0 == 0, a.filter, pi)) { walking = false; break; }
            key = next;
        }
        // ---- new tokens: hashed while the walk goes on, and to the end when the keys are wanted ----
        const int nchunks = (nblk + NB - 1) / NB;
        int consumed = 0;                                                 // chunks waited for (at most one more is in flight)
        for (int c = 0; c < nchunks && (walking || nkp); ++c) {
            __syncwarp();                                                 // every lane is done with buffer (c+1)&1 (chunk c-1)
            coop_stage<BS>(W, tokp, nblk, c + 1, aligned, lane);
            if (aligned) { mbar_wait(&W.bar[c & 1], (phases >> (c & 1)) & 1u); phases ^= 1u << (c & 1); }
            consumed = c + 1;
            __syncwarp();
            const int nb = min(NB, nblk - c * NB);
            const bool first = nk == 0 && c == 0;
            const int nhit = coop_walk_chunk<BS>(t, sm, W, W.tok[c & 1], h, nb, lane, lt, mdl, peer, nkp != nullptr, walking, ws, !first, first, a.filter, pi, key);
            if (nkp && lane < nb) nkp[c * NB + lane] = key;               // lane j: block j of the chunk
            if (!ws.alive || nhit < nb) walking = false;
        }
        warp_write_row(t, a, pi, ws.k, ws.pod, ws.sc, nk + nblk > 0, l2pol);
        // a chunk that was prefetched but never consumed (the walk ended before it, possibly still in the held keys) still
        // lands in its buffer: let it, so that the buffer and its barrier are free for the next prompt
        if (aligned && consumed < nchunks) { mbar_wait(&W.bar[consumed & 1], (phases >> (consumed & 1)) & 1u); phases ^= 1u << (consumed & 1); }
        __syncwarp();
    }
}

// ---- composed path ------------------------------------------------------------------------------------------------------
// Per prompt i: cat_off[i] = where K_i starts in the concatenated key CSR, new_dst[i] = where its new keys start there
// (cat_off[i] + held count), parent[i] = its last held key and pv[i] whether it holds one.  One CTA scans the counts.
constexpr int kTurnScanThreads = 1024;
__global__ void __launch_bounds__(kTurnScanThreads)
turn_offsets_kernel(const uint64_t* __restrict__ keys, const int64_t* __restrict__ key_off, int64_t key_base, const int64_t* __restrict__ tok_off,
                    int64_t n, uint32_t bs, int64_t* __restrict__ cat_off, int64_t* __restrict__ new_dst,
                    uint64_t* __restrict__ parent, uint8_t* __restrict__ pv) {
    __shared__ int64_t part[kTurnScanThreads];
    const int64_t per = (n + kTurnScanThreads - 1) / kTurnScanThreads;
    const int64_t i0 = min(n, (int64_t)threadIdx.x * per), i1 = min(n, i0 + per);
    auto count = [&](int64_t i) { return (key_off[i + 1] - key_off[i]) + (tok_off[i + 1] - tok_off[i]) / bs; };
    int64_t s = 0;
    for (int64_t i = i0; i < i1; ++i) s += count(i);
    part[threadIdx.x] = s;
    __syncthreads();
    for (int d = 1; d < kTurnScanThreads; d <<= 1) {                     // inclusive scan of the per-thread sums
        const int64_t v = threadIdx.x >= (unsigned)d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    int64_t at = part[threadIdx.x] - s;
    for (int64_t i = i0; i < i1; ++i) {
        const int64_t nh = key_off[i + 1] - key_off[i];
        cat_off[i] = at; new_dst[i] = at + nh;
        pv[i] = nh > 0;
        parent[i] = nh > 0 ? keys[key_off[i + 1] - key_base - 1] : 0;
        at += count(i);
    }
    if (threadIdx.x == kTurnScanThreads - 1) cat_off[n] = part[threadIdx.x];
}

// Warp per prompt: the held keys into the concatenated CSR (the new keys are already there, hashed in place), and the new
// keys out to the caller's new_keys when wanted.
__global__ void turn_concat_kernel(const uint64_t* __restrict__ keys, const int64_t* __restrict__ key_off, int64_t key_base,
                                   const int64_t* __restrict__ cat_off, const int64_t* __restrict__ new_dst, int64_t n,
                                   uint64_t* __restrict__ cat, uint64_t* __restrict__ new_keys, const int64_t* __restrict__ new_off, int64_t new_base) {
    const int lane = threadIdx.x & 31;
    const long long total_warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += total_warps) {
        const int64_t kb = key_off[i] - key_base, nh = key_off[i + 1] - key_off[i];
        for (int64_t j = lane; j < nh; j += 32) cat[cat_off[i] + j] = keys[kb + j];
        if (!new_keys) continue;
        const int64_t d = new_dst[i], nn = cat_off[i + 1] - d;
        uint64_t* o = new_keys + (new_off[i] - new_base);
        for (int64_t j = lane; j < nn; j += 32) o[j] = cat[d + j];
    }
}

template <int BS>
inline bool turn_init_one() {
    return cudaFuncSetAttribute(score_turn_kernel<BS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CoopSmem<BS>)) == cudaSuccess;
}
inline int turn_init() {
    return turn_init_one<16>() && turn_init_one<32>() && turn_init_one<64>() && turn_init_one<128>() ? 0 : -1;
}

}  // namespace kvx
