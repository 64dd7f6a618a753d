// kernels_score.cuh -- the fused Score() kernel for sm_90a.
//
// Replaces steps 2-4 of kvcache.Indexer.GetPodScores (pkg/kvcache/indexer.go:141-163):
//   TokensToKVBlockKeys  (kvblock/token_processor.go:141-162)   -> chain hash in registers
//   Index.Lookup         (kvblock/in_memory.go:105-146)         -> one 64-byte probe per key
//   LongestPrefixScorer  (kvblock_scorer.go:108-151)            -> in-order f64 accumulate
// Keys never touch memory: a key is produced in registers, turned into a slot address, and dropped.
//
// Shape (pure integer / HBM work -- no tensor cores):
//   * persistent grid; every LANE is an independent chain worker that owns one prompt at a time
//     (the FNV chain is serial per prompt, so the only parallelism is across prompts).  A lane that
//     finishes its prompt -- early, because its last active pod dropped, or at the end -- pulls the
//     next prompt index from a global counter, so early exits become throughput instead of idle lanes;
//   * token staging global->shared is COOPERATIVE: the per-lane source pointers are exchanged with
//     shuffles and each cp.async (LDGSTS, 16 B, L2-only) instruction moves 8 prompts x 64 B, so a
//     16-token block per lane costs 4 copy instructions per warp; double buffered one block ahead.
//     (The first version used one cp.async.bulk per lane; the profile showed it lowering to a serial
//     ELECT/R2UR/UBLKCP waterfall, 9 instructions per lane.)  Each lane's row is
//     padded to 80 B so the four LDS.128 of the hash loop are bank-conflict free;
//   * the hash itself is branch-free (Fnv::token): 33 issue slots per token for every lane;
//   * the probe for block b (home slot pair = one aligned 64-byte segment, 4 x LDG.128) is issued as
//     soon as key b exists and consumed after block b+1 has been hashed;
//   * per-prompt score state (<= 10 pods: the block-0 slot bounds the result map) lives in shared
//     memory, transposed [entry][lane]; when a slot repeats the previous block's entry pattern
//     (the common case: the same pods hold consecutive blocks) the per-pod max-weight tier is
//     reused and scoring is one DADD per live pod; at retirement the whole warp writes the dense row.
#pragma once
#include <cuda_runtime.h>
#include "score_common.cuh"

#ifndef KVX_ABLATE
#define KVX_ABLATE 0   // bitmask, timing experiments only: 1 no scoring, 2 no probe loads, 4 no token staging, 8 no hash
#endif

namespace kvx {

constexpr int kScoreWarps = 4;                 // warps per CTA
constexpr int kScoreThreads = kScoreWarps * 32;
constexpr int kScoreCtasPerSm = 5;
constexpr int kKeyRing = 4;                    // a lane may run this many blocks ahead of its probes

template <int BS> struct ScoreSmem {
    static constexpr int kRow = BS * 4 + 16;   // bytes per lane per stage (+16 pad -> conflict-free LDS.128)
    struct __align__(16) Warp {
        unsigned char tok[2][32 * kRow];
        LaneCols cols;                         // per-prompt score state of the warp's 32 lanes
        unsigned long long kq[kKeyRing][32];   // hashed-but-not-yet-probed keys (ring, indexed by block % kKeyRing)
    };
    Warp w[kScoreWarps];
    double weight[16];
};

template <int BS>
__global__ void __launch_bounds__(kScoreThreads, kScoreCtasPerSm)
score_kernel_tuned(const TableView t, const ScoreArgs a) {
    static_assert(BS == 16, "the cooperative staging pattern below is written for 16-token blocks");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using SM = ScoreSmem<BS>;
    SM& sm = *reinterpret_cast<SM*>(smem_raw);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t l2pol = l2_policy_stream();
    typename SM::Warp& W = sm.w[wid];
    if (threadIdx.x < 16) sm.weight[threadIdx.x] = t.weight[threadIdx.x];
    __syncthreads();
    const bool peer = t.shard_bits != 0;

    // ---- per-lane worker state ----
    long long pi = -1;                 // prompt index, -1 = no prompt
    bool exhausted = false;            // the global counter ran past n_prompts
    const uint32_t* tokp = nullptr;    // first token of the prompt
    int nblk = 0, cblk = 0, hblk = 0, iblk = 0;  // blocks: total, copies issued, hashed, probes issued
    bool aligned = true;               // prompt start is 16-byte aligned (cooperative cp.async) else own LDG+STS
    bool staged_cur = false, staged_next = false;
    uint64_t h = t.init_hash;
    bool pend = false; uint64_t pkey = 0, pslot = 0;
    const ReqSlot* pbase = t.req;      // table (shard) the pending probe goes to
    uint4 pa0 = {0, 0, 0, 0}, pb0 = {0, 0, 0, 0}, pa1 = {0, 0, 0, 0}, pb1 = {0, 0, 0, 0};
    int pblk = 0;
    SlotPat pv = {};                   // pattern of the previous block's slot
    uint32_t k = 0, alive = 0, mdl = a.model0;
    const uint64_t* frow = nullptr;
    bool finished = false;             // prompt result is final, waiting for the cooperative write-out

    auto refill = [&]() {
        // write out finished prompts and hand new prompts to lanes that need one
        for (;;) {
            __syncwarp();
            uint32_t dm = __ballot_sync(0xffffffffu, finished);
            while (dm) {
                const int p = __ffs(dm) - 1; dm &= dm - 1;
                const long long ppi = __shfl_sync(0xffffffffu, pi, p);
                const uint32_t pk = __shfl_sync(0xffffffffu, k, p);
                const int pn = __shfl_sync(0xffffffffu, nblk, p);
                const bool in = (uint32_t)lane < pk;
                warp_write_row(t, a, ppi, pk, in ? W.cols.pod[lane][p] : 0u, in ? W.cols.sc[lane][p] : 0.0, pn > 0, l2pol);
            }
            __syncwarp();
            const bool want = (finished || pi < 0) && !exhausted;
            const uint32_t wm = __ballot_sync(0xffffffffu, want);
            if (finished) { finished = false; pi = -1; }
            if (!wm) break;
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(a.next, (unsigned long long)__popc(wm));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (want) {
                const long long idx = (long long)base + __popc(wm & ((1u << lane) - 1u));
                if (idx >= a.n_prompts) { exhausted = true; pi = -1; }
                else {
                    pi = idx;
                    const int64_t b = a.tok_off[idx] - a.tok_base, e = a.tok_off[idx + 1] - a.tok_base;
                    tokp = a.tok + b;
                    nblk = (int)((e - b) / BS);
                    cblk = 0; hblk = 0; iblk = 0; h = t.init_hash; pend = false; staged_cur = false; staged_next = false; k = 0; alive = 0;
                    aligned = (reinterpret_cast<uintptr_t>(tokp) & 15u) == 0;
                    mdl = a.model ? a.model[idx] : a.model0;
                    frow = filter_row(a.filter, idx, t.filter_words);
                    finished = (nblk == 0);
                }
            }
            if (!__any_sync(0xffffffffu, finished)) break;
        }
    };

    // stage each lane's next block into buffer s; returns whether this lane staged one
    auto stage = [&](int s) -> bool {
        const bool issue = pi >= 0 && !finished && cblk < nblk;
        const uint32_t* src = tokp + (size_t)cblk * BS;
        const unsigned long long srcv = (issue && aligned) ? (unsigned long long)(uintptr_t)src : 0ull;
        __syncwarp();                                           // every lane is done reading buffer s
#pragma unroll
        for (int r = 0; r < 4; ++r) {                           // 8 prompts x 64 B per instruction
            const int p = 8 * r + (lane >> 2);
            const unsigned long long sp = __shfl_sync(0xffffffffu, srcv, p);
            if (sp && !(KVX_ABLATE & 4)) cp_async_16_stream(smem_addr(&W.tok[s][p * SM::kRow + (lane & 3) * 16]), reinterpret_cast<const char*>(sp) + (lane & 3) * 16, l2pol);
        }
        cp_async_commit();
        if (issue && !aligned) {                                // unaligned prompt start: this lane copies its own block
            uint32_t* dst = reinterpret_cast<uint32_t*>(&W.tok[s][lane * SM::kRow]);
            for (int j = 0; j < BS; ++j) dst[j] = __ldg(src + j);
        }
        if (issue) ++cblk;
        return issue;
    };

    refill();
    staged_next = stage(0);
    for (uint32_t it = 0;; ++it) {
        const int sC = it & 1, sN = sC ^ 1;
        staged_cur = staged_next;
        // 1. stage the following block; 2. the current one has landed
        staged_next = stage(sN);
        cp_async_wait<1>();
        __syncwarp();
        // 3. hash the current block -> request key   (uniform for all lanes; idle lanes hash stale bytes)
        uint64_t key;
        if (KVX_ABLATE & 8) { Fnv f; f.begin_block(h, BS); f.lo ^= W.tok[sC][lane * SM::kRow]; key = f.end_block(); }
        else key = hash_row16(h, &W.tok[sC][lane * SM::kRow]);
        if (staged_cur) {
            if (hblk - iblk >= kKeyRing - 1) {
                // (very rare) the ring is about to fill because several probes in a row needed a retry: resolve
                // the pending probe synchronously; steps 4/5 below then consume it and issue the oldest key,
                // so the slot written next (hblk % ring) is never one that still holds an unissued key
                uint4 A, B;
                bool hit;
                while (!pair_decides(pa0, pb0, pa1, pb1, pkey, mdl, A, B, hit)) {
                    pslot = (pslot + 2) & t.req_mask;
                    ld_slot_pair(pbase + pslot, peer, pa0, pb0, pa1, pb1);
                }
                // leave the resolved slot in the registers: step 4 consumes it without a retry (as slot 0 of the pair at
                // pslot, so a hit in slot 1 moves pslot on by one for the CLOCK marking)
                if (hit) { pslot += slot_matches(pa0, pb0, pkey, mdl) ? 0u : 1u; pa0 = A; pb0 = B; } else { pb0.w = 0; }
            }
            h = key;
            W.kq[hblk & (kKeyRing - 1)][lane] = key;
            ++hblk;
        }
        // 4. consume the probe issued earlier.  If neither slot of the fetched pair decides the lookup the next
        //    pair is requested and consumed one iteration later (the lane then runs one block ahead of its
        //    probes, keys waiting in W.kq) -- no lane ever blocks the warp on a dependent DRAM round trip.
        if (pend) {
            uint4 A, B;
            bool hit;
            if (!pair_decides(pa0, pb0, pa1, pb1, pkey, mdl, A, B, hit)) {
                pslot = (pslot + 2) & t.req_mask;                      // retry on the next pair
                ld_slot_pair(pbase + pslot, peer, pa0, pb0, pa1, pb1);
            } else if (!hit) {
                pend = false; finished = true;
            } else {
                pend = false;
                mark_hit(t, pslot, pa0, pb0, pkey, mdl);
                const SlotPat w = SlotPat::of(A, B);
                if (KVX_ABLATE & 1) { if (pblk == 0) { k = 0; alive = 1u; } }
                else {
                    if (pblk > 0 && w == pv) W.cols.repeat(lane, sm.weight, alive);
                    else if (pblk == 0) W.cols.first(lane, w, frow, sm.weight, k, alive);
                    else W.cols.next(lane, w, sm.weight, alive);
                    pv = w;
                }
                if (!alive || pblk == nblk - 1) finished = true;
            }
        }
        // 5. issue the probe for the oldest hashed-but-unprobed block: the aligned slot pair (home, home+1) = 64 bytes
        if (!pend && !finished && pi >= 0 && iblk < hblk) {
            pkey = (iblk == hblk - 1 && staged_cur) ? key : W.kq[iblk & (kKeyRing - 1)][lane];
            pblk = iblk;
            ++iblk;
            { const uint64_t hm = home_of(pkey, mdl); pbase = t.req_peer[shard_of(hm, t.shard_bits)]; pslot = hm & t.req_mask & ~1ull; }
            ld_slot_pair(pbase + pslot, peer, pa0, pb0, pa1, pb1);
            pend = true;
        }
        // 6. retire + refill
        if (__any_sync(0xffffffffu, finished)) {
            if (finished) { staged_next = false; pend = false; }
            refill();
        }
        if (!__any_sync(0xffffffffu, pi >= 0)) break;
    }
    cp_async_wait<0>();       // nothing may still be landing in this CTA's shared memory when it exits
}

// Host side -------------------------------------------------------------------------------------
inline int score_tuned_init() {
    cudaError_t e = cudaFuncSetAttribute(score_kernel_tuned<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ScoreSmem<16>));
    if (e != cudaSuccess) return -1;
    return 0;
}

// a.next is set to d_next, the work counter this launch zeroes
inline int launch_score_tuned(const TableView& t, int sm_count, ScoreArgs a, unsigned long long* d_next, cudaStream_t st,
                              uint64_t* launches) {
    if (cudaMemsetAsync(d_next, 0, sizeof(unsigned long long), st) != cudaSuccess) return -1;
    a.next = d_next;
    const int64_t lanes_per_cta = kScoreThreads;
    int64_t ctas = (a.n_prompts + lanes_per_cta - 1) / lanes_per_cta;
    const int64_t max_ctas = (int64_t)sm_count * kScoreCtasPerSm;
    if (ctas > max_ctas) ctas = max_ctas;
    score_kernel_tuned<16><<<(unsigned)ctas, kScoreThreads, sizeof(ScoreSmem<16>), st>>>(t, a);
    *launches += 1;
    if (cudaGetLastError() != cudaSuccess) return -1;
    return 0;
}

}  // namespace kvx
