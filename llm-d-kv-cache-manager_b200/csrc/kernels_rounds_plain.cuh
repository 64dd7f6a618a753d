// kernels_rounds_plain.cuh -- Score() for MEDIUM batches: alternating hash / walk rounds, every prompt on its own.
//
// Same reference path as every Score() kernel (GetPodScores steps 2-4, pkg/kvcache/indexer.go:141-163), with the probe,
// the fold and the result row of score_common.cuh.  Two kernels per round and nothing else:
//
//   round r, kernel H (hash_round_kernel):  prompts that are still on the consecutive-prefix walk hash their next
//       kRoundBlocks blocks.  Lockstep, thin lanes (no score / probe state), the branch-free FNV/CBOR code at the
//       pipe-saturating occupancy measured by scripts/ubench_hash.cu.  Keys go to a per-round buffer in HBM (8 B per
//       block -- versus 64 B of tokens and 64 B of slot read).
//   round r, kernel P (probe_round_kernel): lane per prompt, a warp walks 32 prompts in lockstep one block per
//       iteration, the next block's slot pair in flight while this one is scored.  Prompts whose walk continues are
//       appended to the next round's list.
//
// The batch is radix-sorted by a fingerprint of the first block so that prompts sharing a prefix sit in neighbouring
// lanes and their probes coalesce.  kernels_rounds.cuh goes further for LARGE batches (it hashes and walks every
// distinct prefix once); its per-round bookkeeping is a fixed cost per round, which this path does not pay.
// Results are bit-identical on every path (tests run all of them against the oracle).
#pragma once
#include <cuda_runtime.h>
#include "score_common.cuh"
#include "kernels_rounds.cuh"      // PromptState, HashSmem, rounds_init_kernel

namespace kvx {
namespace plain {

// Blocks staged per copy step (2 = 128-byte accesses: fewer, longer DRAM accesses but only 24 resident warps/SM, and the
// kernel is pipe bound).  Always 1; kernel H's staging below keeps the general form because ptxas 12.9 compiles the
// one-block spelling of it to different code (40 / 56 registers instead of 48 / 52) that made the lane-walk step at 262 144
// prompts ~1.5 % slower (H100 80GB HBM3, 400 W power limit).
constexpr int kHashChunk = 1;

constexpr int kProbeThreads = 256;

struct RoundBufs {
    uint32_t* act[2];                    // active prompt lists (ping-pong)
    unsigned int* n_act;                 // [2] list lengths
    uint64_t* hstate;                    // chain hash after the last hashed block, per prompt
    uint64_t* keys;                      // [kRoundBlocks][n_prompts] keys of the current round, block-major: key of
                                         // block j of list slot i at keys[j * n_prompts + i] (coalesced both ways)
    uint32_t* nbr;                       // [n_act] per list slot: blocks hashed this round | (more blocks follow) << 8
    PromptState* pst;                    // per prompt
};

// ---- kernel H ---------------------------------------------------------------------------------
// PM (prompt-major keys): key of block j of list slot i at keys[i * 32 + j] -- what the warp-per-prompt kernel P reads in one
// coalesced 256-byte load; block-major (keys[j * n_prompts + i]) is what the lane-per-prompt kernel P wants.
// NS: token blocks staged per prompt (NS - 1 copies in flight ahead of the chain).  With 2 a launch lasts 32 x max(FNV of a block,
// one loaded DRAM round trip) -- fine when the list fills the machine, the floor of the round when it does not: the
// warp-per-prompt configuration stages 3 and runs 128-thread CTAs (55 KB each, four per SM).
template <int BS, bool PM>
__global__ void __launch_bounds__(kHashThreads, 4)
hash_round_kernel(const TableView t, const ScoreArgs a, const RoundBufs rb, const int cur, const int round) {
    static_assert(BS == 16, "staging pattern is written for 16-token blocks");
    constexpr int NS = PM ? 3 : 2;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using SM = HashSmem<BS>;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned char* const wtok = smem_raw + (size_t)wid * NS * 32 * SM::kRow;          // this warp's NS stages of 32 rows
    const uint32_t wbase = smem_addr(wtok);         // 32-bit shared-window address of the warp's stages
    const uint64_t l2pol = l2_policy_stream();      // created once, in uniform control flow (a policy built inside the divergent
                                                    // staging branch made ptxas 12.9 emit an LDGSTS with an unset descriptor: illegal instruction)
    const unsigned int n_act = rb.n_act[cur];
    if (blockIdx.x == 0 && threadIdx.x == 0) rb.n_act[cur ^ 1] = 0;      // next round's list starts empty
    const unsigned int total_warps = gridDim.x * (blockDim.x / 32);
    for (unsigned int w = blockIdx.x * (blockDim.x / 32) + wid; w * 32u < n_act; w += total_warps) {
        const unsigned int i = w * 32u + lane;                            // slot in the active list
        const bool have = i < n_act;
        const uint32_t p = have ? rb.act[cur][i] : 0u;
        int nb = 0;                                                      // blocks of this prompt in this round
        const uint32_t* src = nullptr;
        bool aligned = true;
        uint64_t h = 0;
        if (have) {
            const int64_t b = a.tok_off[p] - a.tok_base, e = a.tok_off[p + 1] - a.tok_base;
            const int64_t nblk = (e - b) / BS;
            const int64_t first = (int64_t)round * kRoundBlocks;
            nb = (int)max((int64_t)0, min((int64_t)kRoundBlocks, nblk - first));
            rb.nbr[i] = (uint32_t)nb | ((first + nb < nblk) ? 0x100u : 0u);
            src = a.tok + b + first * BS;
            aligned = (reinterpret_cast<uintptr_t>(src) & 15u) == 0;
            h = round == 0 ? t.init_hash : rb.hstate[p];
        }
        const int nb_max = __reduce_max_sync(0xffffffffu, nb);
        // stage chunk c (kHashChunk blocks) of every lane's prompt: 4*kHashChunk lanes move one prompt's contiguous bytes.
        auto stage = [&](int s, int c) {
            const int b0 = c * kHashChunk;
            const bool issue = b0 < nb;
            const int nbytes = issue ? min(kHashChunk, nb - b0) * BS * 4 : 0;
            const unsigned long long srcv = (issue && aligned) ? (unsigned long long)(uintptr_t)(src + (size_t)b0 * BS) : 0ull;
            __syncwarp();
            constexpr int LPP = 4 * kHashChunk;             // lanes that move one prompt's chunk (16 B each)
            constexpr int PPI = 32 / LPP;                   // prompts per copy instruction
#pragma unroll
            for (int r = 0; r < 32 / PPI; ++r) {
                const int q = PPI * r + lane / LPP;
                const unsigned long long sp = __shfl_sync(0xffffffffu, srcv, q);
                const int nby = kHashChunk == 1 ? BS * 4 : __shfl_sync(0xffffffffu, nbytes, q);
                if (sp && (lane % LPP) * 16 < nby)
                    cp_async_16_stream(wbase + (uint32_t)(s * 32 * SM::kRow + q * SM::kRow + (lane % LPP) * 16), reinterpret_cast<const char*>(sp) + (lane % LPP) * 16, l2pol);
            }
            cp_async_commit();
            if (issue && !aligned) {
                uint32_t* dst = reinterpret_cast<uint32_t*>(wtok + (size_t)s * 32 * SM::kRow + lane * SM::kRow);
                const uint32_t* g = src + (size_t)b0 * BS;
                for (int j = 0; j < nbytes / 4; ++j) dst[j] = __ldg(g + j);
            }
        };
#pragma unroll
        for (int c = 0; c < NS - 1; ++c) stage(c, c);
        const int nchunks = (nb_max + kHashChunk - 1) / kHashChunk;
        for (int c = 0; c < nchunks; ++c) {
            stage((c + NS - 1) % NS, c + NS - 1);
            cp_async_wait<NS - 1>();
            __syncwarp();
#pragma unroll
            for (int u = 0; u < kHashChunk; ++u) {
                const int b = c * kHashChunk + u;
                const uint64_t key = hash_row16(h, wtok + (size_t)(c % NS) * 32 * SM::kRow + lane * SM::kRow + u * BS * 4);
                if (b < nb) { h = key; rb.keys[PM ? (size_t)i * kRoundBlocks + b : (size_t)b * a.n_prompts + i] = key; }
            }
        }
        cp_async_wait<0>();
        __syncwarp();
        if (have && nb > 0) rb.hstate[p] = h;
    }
}

// ---- kernel P ---------------------------------------------------------------------------------
// Kernel P, lane-per-prompt.  (Two warp-per-prompt versions came first -- 32 lanes probing a prompt's 32 keys at
// once, then the same software-pipelined.  Both spent most issue slots idle because the walk itself
// runs on <= 10 lanes while the other 22 wait.)  Here a
// warp walks 32 prompts in lockstep, one block per iteration: every instruction serves 32 prompts, the 32 lanes'
// probes are 32 independent 64-byte reads, and the slot pair for block j+1 is in flight while block j is scored.
struct WalkSmem {
    LaneCols w[kProbeThreads / 32];
    double weight[16];
};

// kClock: CLOCK marking of the blocks walked (a template parameter: the default instance keeps its register allocation)
template <bool kClock>
__global__ void __launch_bounds__(kProbeThreads, 4)
probe_round_kernel(const TableView t, const ScoreArgs a, const RoundBufs rb, const int cur, const int round) {
    extern __shared__ __align__(16) unsigned char smem_raw_w[];
    WalkSmem& sm = *reinterpret_cast<WalkSmem*>(smem_raw_w);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    LaneCols& W = sm.w[wid];
    if (threadIdx.x < 16) sm.weight[threadIdx.x] = t.weight[threadIdx.x];
    __syncthreads();
    const unsigned int n_act = rb.n_act[cur];
    const uint64_t l2pol = l2_policy_stream();
    const size_t kstride = (size_t)a.n_prompts;
    const bool peer = t.shard_bits != 0;
    const unsigned int total_warps = gridDim.x * (kProbeThreads / 32);
    for (unsigned int w = blockIdx.x * (kProbeThreads / 32) + wid; w * 32u < n_act; w += total_warps) {
        const unsigned int i = w * 32u + lane;
        const bool have = i < n_act;
        const uint32_t p = have ? rb.act[cur][i] : 0u;
        const uint32_t meta = have ? rb.nbr[i] : 0u;
        const int nb = (int)(meta & 63u);
        const bool has_more = (meta >> 8) & 1u;
        const uint32_t mdl = (have && a.model) ? a.model[p] : a.model0;
        uint32_t k = 0, alive = 0;
        SlotPat pv = {};                                       // last scored pattern
        if (round > 0 && have) {
            const PromptState& ps = rb.pst[p];
            k = ps.k; alive = ps.alive;
#pragma unroll
            for (int x = 0; x < 6; ++x) pv.w[x] = ps.pat[x];
            for (uint32_t q = 0; q < k; ++q) { W.sc[q][lane] = ps.sc[q]; W.pod[q][lane] = ps.pod[q]; W.bt[q][lane] = ps.bt[q]; }
        }
        const int nb_max = __reduce_max_sync(0xffffffffu, nb);
        bool done = !have || nb == 0;                          // walk ended (miss / no live pod); scores are final
        // slot pair of block 0
        // (An L2 prefetch running 8 blocks ahead of the walk is a poor fit: it adds DRAM reads and
        //  lowers issue utilisation.  The SM's outstanding-miss capacity, not the
        //  DRAM latency of a single chain, is what bounds it; the batch is sorted by prefix instead so that lanes of
        //  a warp ask for the same slots.)
        uint64_t key = 0, slot = 0;
        const ReqSlot* base = t.req;                           // table (shard) of the current block's key
        uint4 A0 = {0, 0, 0, 0}, B0 = {0, 0, 0, 0}, A1 = {0, 0, 0, 0}, B1 = {0, 0, 0, 0};
        if (!done) {
            key = rb.keys[i];
            const uint64_t hm = home_of(key, mdl);
            base = t.req_peer[shard_of(hm, t.shard_bits)]; slot = hm & t.req_mask & ~1ull;
            ld_slot_pair(base + slot, peer, A0, B0, A1, B1);
        }
        uint64_t key1 = (!done && nb > 1) ? rb.keys[kstride + i] : 0ull;                        // key of block j+1
        for (int j = 0; j < nb_max; ++j) {
            // next block's pair is requested before this block is scored; keys are read one iteration ahead of their use
            uint64_t nkey = key1, nslot = 0;
            const ReqSlot* nbase = t.req;
            uint4 nA0 = {0, 0, 0, 0}, nB0 = {0, 0, 0, 0}, nA1 = {0, 0, 0, 0}, nB1 = {0, 0, 0, 0};
            const bool nextv = !done && (j + 1 < nb);
            if (nextv) {
                const uint64_t hm = home_of(nkey, mdl);
                nbase = t.req_peer[shard_of(hm, t.shard_bits)]; nslot = hm & t.req_mask & ~1ull;
                ld_slot_pair(nbase + nslot, peer, nA0, nB0, nA1, nB1);
            }
            key1 = (!done && j + 2 < nb) ? rb.keys[(size_t)(j + 2) * kstride + i] : 0ull;
            if (!done && j < nb) {
                uint4 A, B;
                bool hit;
                // (the loop `while (!pair_decides(..))`, spelled out: written that way, ptxas 12.9 spills 40 bytes more in this kernel)
                pair_decides(A0, B0, A1, B1, key, mdl, A, B, hit);
                while (!hit && meta_state(B.w) != kStateEmpty) {              // rare: displaced past the home pair
                    slot = (slot + 2) & t.req_mask;
                    ld_slot_pair(base + slot, peer, A0, B0, A1, B1);
                    pair_decides(A0, B0, A1, B1, key, mdl, A, B, hit);
                }
                if (!hit) { done = true; }
                else {
                    if (kClock) mark_hit(t, slot, A0, B0, key, mdl);
                    const SlotPat w = SlotPat::of(A, B);
                    const bool first_block = (round == 0 && j == 0);
                    if (!first_block && w == pv) W.repeat(lane, sm.weight, alive);
                    else if (first_block) W.first(lane, w, filter_row(a.filter, p, t.filter_words), sm.weight, k, alive);
                    else W.next(lane, w, sm.weight, alive);
                    pv = w;
                    if (!alive) done = true;
                }
            }
            key = nkey; slot = nslot; base = nbase; A0 = nA0; B0 = nB0; A1 = nA1; B1 = nB1;
        }
        // ---- continue next round, or write the result ----
        const bool more = have && !done && has_more;           // all blocks of the round hit, pods still live, blocks left
        const uint32_t mm = __ballot_sync(0xffffffffu, more);
        if (mm) {
            unsigned int base = 0;
            if (lane == 0) base = atomicAdd(&rb.n_act[cur ^ 1], (unsigned int)__popc(mm));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (more) {
                const unsigned int ns = base + __popc(mm & ((1u << lane) - 1u));
                rb.act[cur ^ 1][ns] = p;
                PromptState& ps = rb.pst[p];
                ps.k = (uint8_t)k; ps.alive = (uint16_t)alive;
#pragma unroll
                for (int x = 0; x < 6; ++x) ps.pat[x] = pv.w[x];
                for (uint32_t q = 0; q < k; ++q) { ps.sc[q] = W.sc[q][lane]; ps.pod[q] = W.pod[q][lane]; ps.bt[q] = W.bt[q][lane]; }
            }
        }
        __syncwarp();
        uint32_t dm = __ballot_sync(0xffffffffu, have && !more);
        while (dm) {                                           // the whole warp writes each finished prompt's row
            const int l = __ffs(dm) - 1; dm &= dm - 1;
            const uint32_t pp = __shfl_sync(0xffffffffu, p, l);
            const uint32_t pk = __shfl_sync(0xffffffffu, k, l);
            const uint32_t pmeta = __shfl_sync(0xffffffffu, meta, l);
            const bool in = (uint32_t)lane < pk;
            warp_write_row(t, a, pp, pk, in ? W.pod[lane][l] : 0u, in ? W.sc[lane][l] : 0.0, round > 0 || (pmeta & 63u) > 0, l2pol);
        }
        __syncwarp();
    }
}

// ---- kernel P, warp per prompt -----------------------------------------------------------------
// For batches of a few ten thousand prompts the lane-per-prompt kernel above is a latency chain: a warp walks its 32 prompts
// through 32 dependent probe -> score iterations while most of the machine idles (scripts/timeline.py shows DRAM and issue
// slots mostly idle in such launches).  Here a warp takes ONE prompt: the 32 lanes probe the
// round's 32 keys at once (one memory round trip for the whole chunk), a ballot finds the first miss, and the blocks before it
// are scored in order with lane q owning pod q (<= 10 pods); runs of blocks whose slot holds the same pods and tiers are runs of
// in-order additions of the same addend.  ~700 issue slots per prompt-round instead of ~1/32 of a lockstep warp's: worth it
// while the batch cannot fill the machine (kvidx.cu: rounds_warp_max).  Same arithmetic in the same order as every other path.
// The 8 warps of a CTA run in lock step over 8 consecutive list slots so that the survivors are appended with one atomic per CTA
// iteration, in list order.  Keys are prompt-major (hash_round_kernel<., true>).
struct WarpWalkSmem { uint32_t p[kProbeThreads / 32]; unsigned int base; };
__global__ void __launch_bounds__(kProbeThreads, 4)
probe_round_warp_kernel(const TableView t, const ScoreArgs a, const RoundBufs rb, const int cur, const int round) {
    __shared__ WarpWalkSmem sm;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    constexpr unsigned int WPC = kProbeThreads / 32;
    const unsigned int n_act = rb.n_act[cur];
    const uint64_t l2pol = l2_policy_stream();
    const bool peer = t.shard_bits != 0;
    for (unsigned int i0 = blockIdx.x * WPC; i0 < n_act; i0 += gridDim.x * WPC) {
        const unsigned int i = i0 + wid;
        const bool have = i < n_act;
        uint32_t p = 0, meta = 0;
        if (have) { p = rb.act[cur][i]; meta = rb.nbr[i]; }
        const int nb = (int)(meta & 63u);
        const bool has_more = (meta >> 8) & 1u;
        const uint32_t mdl = (have && a.model) ? a.model[p] : a.model0;
        uint64_t key = 0;
        if (lane < nb) key = rb.keys[(size_t)i * kRoundBlocks + lane];
        WarpWalk ws;
        if (round > 0 && have) ws.load(rb.pst[p], lane);
        // probe: lane j looks up block j's key
        SlotPat mine = {};
        bool hit = false;
        uint64_t hslot = 0;                                  // CLOCK: slot of this lane's hit
        if (lane < nb) {
            HomeProbe pr;
            uint4 A, B;
            hit = pr.find(t, key, mdl, peer, A, B);
            if (hit) { mine = SlotPat::of(A, B); if (t.req_ref) hslot = pr.hit_slot(key, mdl); }
        }
        const uint32_t hm_ = __ballot_sync(0xffffffffu, hit);
        const int nhit = hm_ == 0xffffffffu ? 32 : __ffs(~hm_) - 1;   // consecutive hits from block 0 (lanes >= nb never hit)
        const int nwalked = ws.walk<false>(t, lane, mine, nhit, ws.same_mask(lane, mine, round > 0, nhit), round == 0, a.filter, p, [](int) {});
        WarpWalk::mark_walked(t, lane, nwalked, hit, hslot);
        const bool done = nb == 0 || nhit < nb || !ws.alive;   // no block, a block of the round is not in the index, or no pod left
        const bool more = have && !done && has_more;
        // survivors of the CTA's 8 slots, in slot order
        if (lane == 0) sm.p[wid] = more ? p : 0xffffffffu;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned int c = 0;
            for (unsigned int w = 0; w < WPC; ++w) c += sm.p[w] != 0xffffffffu;
            sm.base = c ? atomicAdd(&rb.n_act[cur ^ 1], c) : 0u;
        }
        __syncthreads();
        if (more) {
            unsigned int rank = 0;
            for (int w = 0; w < wid; ++w) rank += sm.p[w] != 0xffffffffu;
            PromptState& ps = rb.pst[p];
            ws.store_lane(ps, lane);
            if (lane == 0) {
                rb.act[cur ^ 1][sm.base + rank] = p;
                ws.store_uniform(ps);
            }
        } else if (have) warp_write_row(t, a, p, ws.k, ws.pod, ws.sc, round > 0 || nb > 0, l2pol);
        __syncthreads();                                        // sm.p / sm.base are rewritten by the next iteration
    }
}

inline int rounds_init() {
    if (cudaFuncSetAttribute(hash_round_kernel<16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HashSmem<16>)) != cudaSuccess) return -1;
    if (cudaFuncSetAttribute(hash_round_kernel<16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HashSmem<16>)) != cudaSuccess) return -1;
    if (cudaFuncSetAttribute(probe_round_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WalkSmem)) != cudaSuccess) return -1;
    if (cudaFuncSetAttribute(probe_round_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WalkSmem)) != cudaSuccess) return -1;
    return 0;
}

}  // namespace plain
}  // namespace kvx
