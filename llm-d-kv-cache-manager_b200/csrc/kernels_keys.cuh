// kernels_keys.cuh -- Score() from request keys the caller already holds: GetPodScores steps 3-4 (pkg/kvcache/indexer.go:150-159),
// Index.Lookup (kvblock/in_memory.go:105-146) followed by LongestPrefixScorer.Score (kvblock_scorer.go:108-151).
//
// Without tokens there is no hash chain: a prompt's keys are an array like any other, so one warp takes one prompt at
// every batch size and needs neither the round / class machinery of the large-batch pipelines nor their read-back of the
// longest prompt.  Per 32-key chunk: lane j loads key j (one coalesced 256-byte read, evict_first like the token stream)
// and probes it (HomeProbe: a local shard's slot pair at once, a peer's home slot first unless KVIDX_PEER_PAIR), a
// ballot finds the first miss, WarpWalk scores the hits in block order and marks what it looked at (CLOCK).  The next
// chunk's keys are loaded into registers while the current chunk is probed and walked; its probes are not issued before
// the walk has decided that it goes on, so a prompt whose walk ends early costs no slot reads past its end.  The probe,
// the walk and the result row are those of score_common.cuh: the same f64 addends in the same order as every other path.
#pragma once
#include <cuda_runtime.h>
#include "score_common.cuh"

namespace kvx {

constexpr int kKeysWarps = 4;
constexpr int kKeysThreads = kKeysWarps * 32;
constexpr int kKeysCtasPerSm = 6;                 // 80 registers, no spills: 24 warps per SM keep their probes in flight
constexpr int kKeysChunk = 32;                     // keys per probe / walk step: one per lane

__device__ __forceinline__ uint64_t ld_stream_u64(const uint64_t* p, uint64_t pol) {
    uint64_t v;
#if KVIDX_L2_STREAM
    asm volatile("ld.global.nc.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
#else
    v = __ldg(p);
#endif
    return v;
}

// One chunk of nb <= 32 held keys (lane j: key j): probe, ballot to the first miss, walk, mark.  `cont`: a block was scored
// before this chunk; `first_block`: the chunk's key 0 is the prompt's block 0.  True while the walk goes on past the chunk.
__device__ __forceinline__ bool keys_walk_chunk(const TableView& t, WarpWalk& ws, int lane, uint64_t key, int nb, uint32_t mdl, bool peer,
                                                bool cont, bool first_block, const uint64_t* filter, int64_t pi) {
    SlotPat mine = {};
    bool hit = false;
    uint64_t hslot = 0;                                           // CLOCK: slot of this lane's hit
    if (lane < nb) {
        HomeProbe pr;
        uint4 A, B;
        hit = pr.find(t, key, mdl, peer, A, B);
        if (hit) { mine = SlotPat::of(A, B); if (t.req_ref) hslot = pr.hit_slot(key, mdl); }
    }
    const uint32_t hm_ = __ballot_sync(0xffffffffu, hit);
    const int nhit = hm_ == 0xffffffffu ? 32 : __ffs(~hm_) - 1;   // consecutive hits from the chunk's first key
    const int nwalked = ws.walk<false>(t, lane, mine, nhit, ws.same_mask(lane, mine, cont, nhit), first_block, filter, pi, [](int) {});
    WarpWalk::mark_walked(t, lane, nwalked, hit, hslot);
    return ws.alive && nhit >= nb;                                // else a key not in the index, or no pod left
}

// a.tok_off / a.tok_base describe the key CSR: prompt i owns keys[a.tok_off[i] - a.tok_base .. a.tok_off[i+1] - a.tok_base)
__global__ void __launch_bounds__(kKeysThreads, kKeysCtasPerSm)
score_keys_kernel(const TableView t, const uint64_t* __restrict__ keys, const ScoreArgs a) {
    const uint64_t l2pol = l2_policy_stream();
    const int lane = threadIdx.x & 31;
    const bool peer = t.shard_bits != 0;
    const long long total_warps = (long long)gridDim.x * kKeysWarps;
    for (long long pi = (long long)blockIdx.x * kKeysWarps + (threadIdx.x >> 5); pi < a.n_prompts; pi += total_warps) {
        const int64_t kb = a.tok_off[pi] - a.tok_base, ke = a.tok_off[pi + 1] - a.tok_base;
        const int64_t nk = ke - kb;
        const uint64_t* kp = keys + kb;
        const uint32_t mdl = a.model ? a.model[pi] : a.model0;
        WarpWalk ws;
        uint64_t key = 0;
        if (lane < nk) key = ld_stream_u64(kp + lane, l2pol);
        for (int64_t c0 = 0; c0 < nk; c0 += kKeysChunk) {
            const int nb = nk - c0 < kKeysChunk ? (int)(nk - c0) : kKeysChunk;
            // the next chunk's keys, in flight while this chunk is probed and walked
            uint64_t next = 0;
            if (c0 + kKeysChunk + lane < nk) next = ld_stream_u64(kp + c0 + kKeysChunk + lane, l2pol);
            if (!keys_walk_chunk(t, ws, lane, key, nb, mdl, peer, c0 > 0, c0 == 0, a.filter, pi)) break;
            key = next;
        }
        warp_write_row(t, a, pi, ws.k, ws.pod, ws.sc, nk > 0, l2pol);
    }
}

}  // namespace kvx
