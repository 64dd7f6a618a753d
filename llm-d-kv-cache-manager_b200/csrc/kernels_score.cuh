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
#include "kernels_v1.cuh"

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
        double sc[kMaxEnt][32];                // running score of block-0 pod q
        unsigned long long kq[kKeyRing][32];   // hashed-but-not-yet-probed keys (ring, indexed by block % kKeyRing)
        uint16_t pod[kMaxEnt][32];             // pod id of block-0 pod q
        uint8_t bt[kMaxEnt][32];               // tier giving pod q its max weight in the previous block (0xff: 0.0)
    };
    Warp w[kScoreWarps];
    double weight[16];
};

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
// L2 eviction policy for data that is read or written exactly once per step (the token stream, the dense result rows):
// evict_first keeps it from flushing what the latency-bound kernels of a round hand to each other (lists, walk states, keys)
// and the index slots out of the 50 MB L2.
#ifndef KVIDX_L2_STREAM
#define KVIDX_L2_STREAM 1
#endif
__device__ __forceinline__ uint64_t l2_policy_stream() {
    uint64_t pol = 0;
#if KVIDX_L2_STREAM
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
#endif
    return pol;
}
__device__ __forceinline__ void cp_async_16_stream(uint32_t dst, const void* src, uint64_t pol) {
#if KVIDX_L2_STREAM
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
#else
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
#endif
}
__device__ __forceinline__ void st_stream_f64x2(double* p, double a, double b, uint64_t pol) {
#if KVIDX_L2_STREAM
    asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(a), "d"(b), "l"(pol) : "memory");
#else
    *reinterpret_cast<double2*>(p) = make_double2(a, b);
#endif
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// ---- TMA (1-D bulk copy) + mbarrier: the sm_90 way to move a contiguous run of bytes into shared memory ----
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    asm volatile("{\n\t.reg .pred p;\n\tKVX_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra KVX_DONE;\n\tbra KVX_WAIT;\n\tKVX_DONE:\n\t}"
                 ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
// global -> shared bulk copy (TMA, 1-D): bytes a multiple of 16, both addresses 16-byte aligned; completes on `bar`
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

struct ScoreArgs {
    const uint32_t* tok; const int64_t* tok_off; int64_t tok_base; int64_t n_prompts;
    const uint32_t* model; uint32_t model0; const uint64_t* filter;
    double* dense; uint16_t* sp_pods; double* sp_scores; uint8_t* sp_cnt; uint8_t* has_keys;
    unsigned long long* next;      // global work counter (zeroed before launch)
};

__device__ __forceinline__ bool slot_matches(const uint4& a, const uint4& b, uint64_t key, uint32_t mdl) {
    return meta_state(b.w) == kStateFull && a.x == (uint32_t)key && a.y == (uint32_t)(key >> 32) && meta_model(b.w) == mdl;
}

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
    uint32_t pv0 = 0, pv1 = 0, pv2 = 0, pv3 = 0, pv4 = 0, pvc = 0;   // entry words + count of the previous block's slot
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
                if (a.dense) {
                    double* row = a.dense + ppi * (long long)t.max_pods;
                    const uint32_t P = t.max_pods;
                    if ((P & 1u) == 0 && ((reinterpret_cast<uintptr_t>(row) & 15u) == 0)) {
                        for (uint32_t c = lane * 2; c < P; c += 64) st_stream_f64x2(row + c, -1.0, -1.0, l2pol);
                    } else {
                        for (uint32_t c = lane; c < P; c += 32) row[c] = -1.0;
                    }
                    __syncwarp();
                    if ((uint32_t)lane < pk) { const uint32_t pd = W.pod[lane][p]; if (pd < P) row[pd] = W.sc[lane][p]; }
                }
                if (a.sp_cnt) {
                    if ((uint32_t)lane < pk) {
                        a.sp_pods[ppi * kMaxEnt + lane] = W.pod[lane][p];
                        a.sp_scores[ppi * kMaxEnt + lane] = W.sc[lane][p];
                    }
                    if (lane == 0) a.sp_cnt[ppi] = (uint8_t)pk;
                }
                if (a.has_keys && lane == 0) a.has_keys[ppi] = pn > 0;
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
        {
            Fnv f;
            f.begin_block(h, BS);
            if (KVX_ABLATE & 8) { f.lo ^= W.tok[sC][lane * SM::kRow]; key = f.end_block(); } else {
            const uint4* tp = reinterpret_cast<const uint4*>(&W.tok[sC][lane * SM::kRow]);
            const uint4 v0 = tp[0], v1 = tp[1];
            f.token(v0.x); f.token(v0.y); f.token(v0.z); f.token(v0.w);
            const uint4 v2 = tp[2];
            f.token(v1.x); f.token(v1.y); f.token(v1.z); f.token(v1.w);
            const uint4 v3 = tp[3];
            f.token(v2.x); f.token(v2.y); f.token(v2.z); f.token(v2.w);
            f.token(v3.x); f.token(v3.y); f.token(v3.z); f.token(v3.w);
            key = f.end_block();
            }
        }
        if (staged_cur) {
            if (hblk - iblk >= kKeyRing - 1) {
                // (very rare) the ring is about to fill because several probes in a row needed a retry: resolve
                // the pending probe synchronously; steps 4/5 below then consume it and issue the oldest key,
                // so the slot written next (hblk % ring) is never one that still holds an unissued key
                uint4 A, B; bool hit = false, term = false;
                for (;;) {
                    A = pa0; B = pb0; hit = slot_matches(A, B, pkey, mdl); term = !hit && meta_state(B.w) == kStateEmpty;
                    if (!hit && !term) { A = pa1; B = pb1; hit = slot_matches(A, B, pkey, mdl); term = !hit && meta_state(B.w) == kStateEmpty; }
                    if (hit || term) break;
                    pslot = (pslot + 2) & t.req_mask;
                    const uint4* sp = reinterpret_cast<const uint4*>(pbase + pslot);
                    ld_slot(reinterpret_cast<const ReqSlot*>(sp), peer, pa0, pb0); ld_slot(reinterpret_cast<const ReqSlot*>(sp) + 1, peer, pa1, pb1);
                }
                // leave the resolved slot in the registers: step 4 consumes it without a retry
                if (hit) { pa0 = A; pb0 = B; } else { pb0.w = 0; }
            }
            h = key;
            W.kq[hblk & (kKeyRing - 1)][lane] = key;
            ++hblk;
        }
        // 4. consume the probe issued earlier.  If neither slot of the fetched pair decides the lookup the next
        //    pair is requested and consumed one iteration later (the lane then runs one block ahead of its
        //    probes, keys waiting in W.kq) -- no lane ever blocks the warp on a dependent DRAM round trip.
        if (pend) {
            uint4 A = pa0, B = pb0;
            bool hit = slot_matches(A, B, pkey, mdl);
            bool term = !hit && meta_state(B.w) == kStateEmpty;
            if (!hit && !term) { A = pa1; B = pb1; hit = slot_matches(A, B, pkey, mdl); term = !hit && meta_state(B.w) == kStateEmpty; }
            if (!hit && !term) {
                pslot = (pslot + 2) & t.req_mask;                      // retry on the next pair
                const uint4* sp = reinterpret_cast<const uint4*>(pbase + pslot);
                ld_slot(reinterpret_cast<const ReqSlot*>(sp), peer, pa0, pb0); ld_slot(reinterpret_cast<const ReqSlot*>(sp) + 1, peer, pa1, pb1);
            } else if (!hit) {
                pend = false; finished = true;
            } else {
                pend = false;
                SlotWords w; w.a = A; w.b = B;
                const uint32_t cnt = meta_count(B.w);
                if (KVX_ABLATE & 1) { if (pblk == 0) { k = 0; alive = 1u; } }
                else {
                const bool same = pblk > 0 && (((pv0 ^ A.z) | (pv1 ^ A.w) | (pv2 ^ B.x) | (pv3 ^ B.y) | (pv4 ^ B.z) | (pvc ^ cnt)) == 0u);
                if (same) {
                    // same pod set as the previous block: add each live pod's cached max weight, in block order
                    uint32_t am = alive;
                    while (am) {
                        const int q = __ffs(am) - 1; am &= am - 1;
                        const uint32_t bt = W.bt[q][lane];
                        const double mx = bt == 0xffu ? 0.0 : sm.weight[bt];
                        W.sc[q][lane] = __dadd_rn(W.sc[q][lane], mx);
                    }
                } else if (pblk == 0) {
                    // activePods := pods of block 0 (after the filter); score = max weight   (kvblock_scorer.go:118-128)
                    k = 0;
                    for (uint32_t j = 0; j < cnt; ++j) {
                        const uint32_t pt = slot_ent(w, j), p = pt >> 4;
                        if (frow && !filter_has(frow, p)) continue;
                        const double wt = sm.weight[pt & 15u];
                        uint32_t q = 0;
                        for (; q < k; ++q) if (W.pod[q][lane] == p) break;
                        if (q == k) { W.pod[k][lane] = (uint16_t)p; W.sc[k][lane] = 0.0; W.bt[k][lane] = 0xffu; ++k; }
                        if (wt > W.sc[q][lane]) { W.sc[q][lane] = wt; W.bt[q][lane] = (uint8_t)(pt & 15u); }
                    }
                    alive = (1u << k) - 1u;
                } else {
                    // activePods &= pods(block); score[p] += max weight, in block order   (kvblock_scorer.go:130-147)
                    uint32_t am = alive;
                    while (am) {
                        const int q = __ffs(am) - 1; am &= am - 1;
                        const uint32_t want = W.pod[q][lane];
                        double mx = 0.0; bool present = false; uint32_t bt = 0xffu;
                        for (uint32_t j = 0; j < cnt; ++j) {
                            const uint32_t pt = slot_ent(w, j);
                            if ((pt >> 4) == want) {
                                present = true;
                                const double wt = sm.weight[pt & 15u];
                                if (wt > mx) { mx = wt; bt = pt & 15u; }
                            }
                        }
                        if (present) { W.sc[q][lane] = __dadd_rn(W.sc[q][lane], mx); W.bt[q][lane] = (uint8_t)bt; }
                        else alive &= ~(1u << q);
                    }
                }
                pv0 = A.z; pv1 = A.w; pv2 = B.x; pv3 = B.y; pv4 = B.z; pvc = cnt;
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
            const uint4* sp = reinterpret_cast<const uint4*>(pbase + pslot);
            ld_slot(reinterpret_cast<const ReqSlot*>(sp), peer, pa0, pb0); ld_slot(reinterpret_cast<const ReqSlot*>(sp) + 1, peer, pa1, pb1);
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

inline int launch_score_tuned(const TableView& t, int sm_count, const uint32_t* d_tok, const int64_t* d_off, int64_t tok_base, int64_t n,
                              const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter, double* dense, uint16_t* sp_pods,
                              double* sp_scores, uint8_t* sp_cnt, uint8_t* has_keys, unsigned long long* d_next, cudaStream_t st,
                              uint64_t* launches) {
    if (cudaMemsetAsync(d_next, 0, sizeof(unsigned long long), st) != cudaSuccess) return -1;
    ScoreArgs a{d_tok, d_off, tok_base, n, d_model, model0, d_filter, dense, sp_pods, sp_scores, sp_cnt, has_keys, d_next};
    const int64_t lanes_per_cta = kScoreThreads;
    int64_t ctas = (n + lanes_per_cta - 1) / lanes_per_cta;
    const int64_t max_ctas = (int64_t)sm_count * kScoreCtasPerSm;
    if (ctas > max_ctas) ctas = max_ctas;
    score_kernel_tuned<16><<<(unsigned)ctas, kScoreThreads, sizeof(ScoreSmem<16>), st>>>(t, a);
    *launches += 1;
    if (cudaGetLastError() != cudaSuccess) return -1;
    return 0;
}

}  // namespace kvx
