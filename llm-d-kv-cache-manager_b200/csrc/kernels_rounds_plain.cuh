// kernels_rounds_plain.cuh -- Score() for MEDIUM batches: alternating hash / walk rounds, every prompt on its own.
//
// Same reference path as kernels_score.cuh (GetPodScores steps 2-4, pkg/kvcache/indexer.go:141-163).  Two kernels per
// round and nothing else:
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
#include "kernels_score.cuh"
#include "kernels_rounds.cuh"      // PromptState, HashSmem, rounds_init_kernel, ld_slot_pair, ent_of

namespace kvx {
namespace plain {

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
                Fnv f;
                f.begin_block(h, BS);
                const uint4* tp = reinterpret_cast<const uint4*>(wtok + (size_t)(c % NS) * 32 * SM::kRow + lane * SM::kRow + u * BS * 4);
                const uint4 v0 = tp[0], v1 = tp[1];
                f.token(v0.x); f.token(v0.y); f.token(v0.z); f.token(v0.w);
                const uint4 v2 = tp[2];
                f.token(v1.x); f.token(v1.y); f.token(v1.z); f.token(v1.w);
                const uint4 v3 = tp[3];
                f.token(v2.x); f.token(v2.y); f.token(v2.z); f.token(v2.w);
                f.token(v3.x); f.token(v3.y); f.token(v3.z); f.token(v3.w);
                const uint64_t key = f.end_block();
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
    struct Warp {
        double sc[kMaxEnt][32];
        uint16_t pod[kMaxEnt][32];
        uint8_t bt[kMaxEnt][32];
    };
    Warp w[kProbeThreads / 32];
    double weight[16];
};

__global__ void __launch_bounds__(kProbeThreads, 4)
probe_round_kernel(const TableView t, const ScoreArgs a, const RoundBufs rb, const int cur, const int round) {
    extern __shared__ __align__(16) unsigned char smem_raw_w[];
    WalkSmem& sm = *reinterpret_cast<WalkSmem*>(smem_raw_w);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    WalkSmem::Warp& W = sm.w[wid];
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
        uint32_t pv0 = 0, pv1 = 0, pv2 = 0, pv3 = 0, pv4 = 0, pvc = 0;      // last scored pattern
        if (round > 0 && have) {
            const PromptState& ps = rb.pst[p];
            k = ps.k; alive = ps.alive;
            pv0 = ps.pat[0]; pv1 = ps.pat[1]; pv2 = ps.pat[2]; pv3 = ps.pat[3]; pv4 = ps.pat[4]; pvc = ps.pat[5];
            for (uint32_t q = 0; q < k; ++q) { W.sc[q][lane] = ps.sc[q]; W.pod[q][lane] = ps.pod[q]; W.bt[q][lane] = ps.bt[q]; }
        }
        const uint64_t* frow = nullptr;
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
                uint4 A = A0, B = B0;
                bool hit = slot_matches(A, B, key, mdl);
                if (!hit && meta_state(B.w) != kStateEmpty) {
                    A = A1; B = B1;
                    hit = slot_matches(A, B, key, mdl);
                    while (!hit && meta_state(B.w) != kStateEmpty) {          // rare: displaced past the home pair
                        slot = (slot + 2) & t.req_mask;
                        ld_slot_pair(base + slot, peer, A0, B0, A1, B1);
                        A = A0; B = B0; hit = slot_matches(A, B, key, mdl);
                        if (!hit && meta_state(B.w) != kStateEmpty) { A = A1; B = B1; hit = slot_matches(A, B, key, mdl); }
                    }
                }
                if (!hit) { done = true; }
                else {
                    SlotWords sw; sw.a = A; sw.b = B;
                    const uint32_t cnt = meta_count(B.w);
                    const bool first_block = (round == 0 && j == 0);
                    const bool same = !first_block && (((pv0 ^ A.z) | (pv1 ^ A.w) | (pv2 ^ B.x) | (pv3 ^ B.y) | (pv4 ^ B.z) | (pvc ^ cnt)) == 0u);
                    if (same) {
                        uint32_t am = alive;
                        while (am) {
                            const int q = __ffs(am) - 1; am &= am - 1;
                            const uint32_t bt = W.bt[q][lane];
                            const double mx = bt == 0xffu ? 0.0 : sm.weight[bt];
                            W.sc[q][lane] = __dadd_rn(W.sc[q][lane], mx);
                        }
                    } else if (first_block) {
                        // activePods := pods of block 0 (after the filter); score = max weight   (kvblock_scorer.go:118-128)
                        frow = filter_row(a.filter, p, t.filter_words);
                        k = 0;
                        for (uint32_t e = 0; e < cnt; ++e) {
                            const uint32_t pt = slot_ent(sw, e), pd = pt >> 4;
                            if (frow && !filter_has(frow, pd)) continue;
                            const double wt = sm.weight[pt & 15u];
                            uint32_t q = 0;
                            for (; q < k; ++q) if (W.pod[q][lane] == pd) break;
                            if (q == k) { W.pod[k][lane] = (uint16_t)pd; W.sc[k][lane] = 0.0; W.bt[k][lane] = 0xffu; ++k; }
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
                            for (uint32_t e = 0; e < cnt; ++e) {
                                const uint32_t pt = slot_ent(sw, e);
                                if ((pt >> 4) == want) { present = true; const double wt = sm.weight[pt & 15u]; if (wt > mx) { mx = wt; bt = pt & 15u; } }
                            }
                            if (present) { W.sc[q][lane] = __dadd_rn(W.sc[q][lane], mx); W.bt[q][lane] = (uint8_t)bt; }
                            else alive &= ~(1u << q);
                        }
                    }
                    pv0 = A.z; pv1 = A.w; pv2 = B.x; pv3 = B.y; pv4 = B.z; pvc = cnt;
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
                ps.pat[0] = pv0; ps.pat[1] = pv1; ps.pat[2] = pv2; ps.pat[3] = pv3; ps.pat[4] = pv4; ps.pat[5] = pvc;
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
            if (a.dense) {
                double* row = a.dense + (long long)pp * t.max_pods;
                const uint32_t P = t.max_pods;
                if ((P & 1u) == 0 && ((reinterpret_cast<uintptr_t>(row) & 15u) == 0)) {
                    for (uint32_t c = lane * 2; c < P; c += 64) st_stream_f64x2(row + c, -1.0, -1.0, l2pol);
                } else {
                    for (uint32_t c = lane; c < P; c += 32) row[c] = -1.0;
                }
                __syncwarp();
                if ((uint32_t)lane < pk) { const uint32_t pd = W.pod[lane][l]; if (pd < P) row[pd] = W.sc[lane][l]; }
            }
            if (a.sp_cnt) {
                if ((uint32_t)lane < pk) { a.sp_pods[(long long)pp * kMaxEnt + lane] = W.pod[lane][l]; a.sp_scores[(long long)pp * kMaxEnt + lane] = W.sc[lane][l]; }
                if (lane == 0) a.sp_cnt[pp] = (uint8_t)pk;
            }
            if (a.has_keys && lane == 0) a.has_keys[pp] = (round > 0) || (pmeta & 63u) > 0;
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
        // walk state: lane q < k owns pod q
        uint32_t k = 0, alive = 0, mypod = 0xffffffffu, mybt = 0xffu;
        double mysc = 0.0;
        uint32_t pv0 = 0, pv1 = 0, pv2 = 0, pv3 = 0, pv4 = 0, pvc = 0xffffffffu;
        if (round > 0 && have) {
            const PromptState& ps = rb.pst[p];
            k = ps.k; alive = ps.alive;
            pv0 = ps.pat[0]; pv1 = ps.pat[1]; pv2 = ps.pat[2]; pv3 = ps.pat[3]; pv4 = ps.pat[4]; pvc = ps.pat[5];
            if ((uint32_t)lane < k) { mysc = ps.sc[lane]; mypod = ps.pod[lane]; mybt = ps.bt[lane]; }
        }
        // probe: lane j looks up block j's key
        uint32_t e0 = 0, e1 = 0, e2 = 0, e3 = 0, e4 = 0, cnt = 0;
        bool hit = false;
        if (lane < nb) {
            const uint64_t hm = home_of(key, mdl);
            const ReqSlot* base = t.req_peer[shard_of(hm, t.shard_bits)];
            uint64_t slot = hm & t.req_mask & ~1ull;
            const bool remote = base != t.req && !t.peer_pair;                  // a peer's shard: home slot first, its neighbour only if needed
            for (;;) {
                uint4 A0, B0, A1, B1;
                ld_slot(base + slot, peer, A0, B0);
                if (!remote) ld_slot(base + slot + 1, peer, A1, B1);
                uint4 A = A0, B = B0;
                hit = slot_matches(A, B, key, mdl);
                bool stop = hit || meta_state(B.w) == kStateEmpty;
                if (!stop) {
                    if (remote) ld_slot(base + slot + 1, peer, A1, B1);
                    A = A1; B = B1; hit = slot_matches(A, B, key, mdl); stop = hit || meta_state(B.w) == kStateEmpty;
                }
                if (hit) { e0 = A.z; e1 = A.w; e2 = B.x; e3 = B.y; e4 = B.z; cnt = meta_count(B.w); }
                if (stop) break;
                slot = (slot + 2) & t.req_mask;                 // rare: displaced past the home pair
            }
        }
        const uint32_t hm_ = __ballot_sync(0xffffffffu, hit);
        const int nhit = hm_ == 0xffffffffu ? 32 : __ffs(~hm_) - 1;   // consecutive hits from block 0 (lanes >= nb never hit)
        bool done = nb == 0;
        uint32_t samemask;                                      // block j's slot holds the same pods and tiers as block j-1's
        {
            const uint32_t u0 = __shfl_up_sync(0xffffffffu, e0, 1), u1 = __shfl_up_sync(0xffffffffu, e1, 1), u2 = __shfl_up_sync(0xffffffffu, e2, 1),
                           u3 = __shfl_up_sync(0xffffffffu, e3, 1), u4 = __shfl_up_sync(0xffffffffu, e4, 1), uc = __shfl_up_sync(0xffffffffu, cnt, 1);
            const bool sm_ = lane > 0 ? (((u0 ^ e0) | (u1 ^ e1) | (u2 ^ e2) | (u3 ^ e3) | (u4 ^ e4) | (uc ^ cnt)) == 0u)
                                      : (round > 0 && ((pv0 ^ e0) | (pv1 ^ e1) | (pv2 ^ e2) | (pv3 ^ e3) | (pv4 ^ e4) | (pvc ^ cnt)) == 0u);
            samemask = __ballot_sync(0xffffffffu, sm_ && lane < nhit);
        }
        int j = 0;
        while (j < nhit && !done) {
            if ((samemask >> j) & 1u) {
                const uint32_t rest = ~(samemask >> j);
                const int run = min(rest ? __ffs(rest) - 1 : 32, nhit - j);           // >= 1
                if ((alive >> lane) & 1u) {
                    const double add = mybt == 0xffu ? 0.0 : t.weight[mybt & 15u];
                    for (int u = 0; u < run; ++u) mysc = __dadd_rn(mysc, add);
                }
                j += run;
                continue;
            }
            const uint32_t w0 = __shfl_sync(0xffffffffu, e0, j), w1 = __shfl_sync(0xffffffffu, e1, j), w2 = __shfl_sync(0xffffffffu, e2, j),
                           w3 = __shfl_sync(0xffffffffu, e3, j), w4 = __shfl_sync(0xffffffffu, e4, j), c = __shfl_sync(0xffffffffu, cnt, j);
            if (round == 0 && j == 0) {
                // activePods := pods of block 0 (after the filter), in entry order; score = max weight   (kvblock_scorer.go:118-128)
                const uint64_t* frow = filter_row(a.filter, p, t.filter_words);
                k = 0;
                for (uint32_t e = 0; e < c; ++e) {
                    const uint32_t pt = ent_of(w0, w1, w2, w3, w4, (int)e), pd = pt >> 4;
                    if (frow && !filter_has(frow, pd)) continue;
                    const double wt = t.weight[pt & 15u];
                    const uint32_t own = __ballot_sync(0xffffffffu, (uint32_t)lane < k && mypod == pd);
                    const int q = own ? __ffs(own) - 1 : (int)k;
                    if (!own) { if (lane == q) { mypod = pd; mysc = 0.0; mybt = 0xffu; } ++k; }
                    if (lane == q && wt > mysc) { mysc = wt; mybt = pt & 15u; }
                }
                alive = (1u << k) - 1u;
            } else {
                // activePods &= pods(block); score[p] += max weight, in block order   (kvblock_scorer.go:130-147)
                bool present = false; double mx = 0.0; uint32_t bt = 0xffu;
                if ((alive >> lane) & 1u) {
                    for (uint32_t e = 0; e < c; ++e) {
                        const uint32_t pt = ent_of(w0, w1, w2, w3, w4, (int)e);
                        if ((pt >> 4) == mypod) { present = true; const double wt = t.weight[pt & 15u]; if (wt > mx) { mx = wt; bt = pt & 15u; } }
                    }
                    if (present) { mysc = __dadd_rn(mysc, mx); mybt = bt; }
                }
                alive = __ballot_sync(0xffffffffu, present);
            }
            if (!alive) done = true;
            ++j;
        }
        if (j > 0) {                                            // pattern of the last scored block, for the next round's first comparison
            const int lj = j - 1;
            pv0 = __shfl_sync(0xffffffffu, e0, lj); pv1 = __shfl_sync(0xffffffffu, e1, lj); pv2 = __shfl_sync(0xffffffffu, e2, lj);
            pv3 = __shfl_sync(0xffffffffu, e3, lj); pv4 = __shfl_sync(0xffffffffu, e4, lj); pvc = __shfl_sync(0xffffffffu, cnt, lj);
        }
        if (nhit < nb) done = true;                             // a block of the round is not in the index
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
            if ((uint32_t)lane < k) { ps.sc[lane] = mysc; ps.pod[lane] = (uint16_t)mypod; ps.bt[lane] = (uint8_t)mybt; }
            if (lane == 0) {
                rb.act[cur ^ 1][sm.base + rank] = p;
                ps.k = (uint8_t)k; ps.alive = (uint16_t)alive;
                ps.pat[0] = pv0; ps.pat[1] = pv1; ps.pat[2] = pv2; ps.pat[3] = pv3; ps.pat[4] = pv4; ps.pat[5] = pvc;
            }
        } else if (have) {
            if (a.dense) {
                double* row = a.dense + (long long)p * t.max_pods;
                const uint32_t P = t.max_pods;
                if ((P & 1u) == 0 && ((reinterpret_cast<uintptr_t>(row) & 15u) == 0)) {
                    for (uint32_t c2 = lane * 2; c2 < P; c2 += 64) st_stream_f64x2(row + c2, -1.0, -1.0, l2pol);
                } else {
                    for (uint32_t c2 = lane; c2 < P; c2 += 32) row[c2] = -1.0;
                }
                __syncwarp();
                if ((uint32_t)lane < k && mypod < P) row[mypod] = mysc;
            }
            if (a.sp_cnt) {
                if ((uint32_t)lane < k) { a.sp_pods[(long long)p * kMaxEnt + lane] = (uint16_t)mypod; a.sp_scores[(long long)p * kMaxEnt + lane] = mysc; }
                if (lane == 0) a.sp_cnt[p] = (uint8_t)k;
            }
            if (a.has_keys && lane == 0) a.has_keys[p] = (round > 0) || nb > 0;
        }
        __syncthreads();                                        // sm.p / sm.base are rewritten by the next iteration
    }
}

inline int rounds_init() {
    if (cudaFuncSetAttribute(hash_round_kernel<16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HashSmem<16>)) != cudaSuccess) return -1;
    if (cudaFuncSetAttribute(hash_round_kernel<16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HashSmem<16>)) != cudaSuccess) return -1;
    if (cudaFuncSetAttribute(probe_round_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WalkSmem)) != cudaSuccess) return -1;
    return 0;
}

}  // namespace plain
}  // namespace kvx
