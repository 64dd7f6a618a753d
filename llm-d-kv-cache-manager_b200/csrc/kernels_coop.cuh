// kernels_coop.cuh -- Score() for SMALL batches: one WARP per prompt, warp-cooperative FNV, TMA-staged tokens.
//
// Same reference path as every Score() kernel (GetPodScores steps 2-4, pkg/kvcache/indexer.go:141-163): chain keys
// (kvblock/token_processor.go:94-162), Lookup (in_memory.go:105-146), LongestPrefixScorer.Score (kvblock_scorer.go:108-151);
// the probe decision, the warp walk and the result row are the ones of score_common.cuh.
//
// The lane-per-prompt kernels need tens of thousands of prompts to fill the machine: one prompt is ONE serial FNV-1a
// chain (~19 K dependent byte steps at 4 K tokens), so a single GetPodScores RPC runs at the latency of that chain.  Here
// the 32 lanes of a warp evaluate one chain together:
//
//   * FNV-1a is h' = (h ^ b) * p (mod 2^64).  `h ^ b` only touches the low byte, so with L = h & 0xff and
//     d = ((L ^ b) & 0xff) - L,  h' = h*p + d*p, and over a payload of n bytes
//         h_n = h_0 * p^n  +  sum_j d_j * p^(n-j)            (mod 2^64)
//     -- a dot product with precomputed powers of p, lane-parallel, once the d_j are known;
//   * the d_j come from the 8-bit recurrence L' = ((L ^ b) * 0xb3) & 0xff.  Bit k of a product by an odd constant only
//     depends on bits <= k of the operand, so the recurrence is solved bit-plane by bit-plane: in plane k every byte
//     position contributes g = b_k ^ carry_k (carry from the planes below, known), and L_k at position j is the XOR of
//     all g before j -- ONE warp ballot and a popcount per plane, each lane owning P consecutive positions (P = 3 covers
//     the 28..92 CBOR bytes of a 16-token block; 6, 11 and 21 the <= 173, 333 and 653 of a 32-, 64- and 128-token block);
//   * every block's payload starts from the FNV offset basis (the parent hash enters as BYTES), so h_0 * p^n is a table.
//
//   A block then costs 8 ballot/popcount rounds plus one warp reduction instead of ~5 B dependent multiply steps, at
//   every block size B the kernel is built for (16, 32, 64, 128): a longer block costs more register work per lane and
//   plane, not more ballots.  The token bytes of a whole 512-token chunk are laid out in shared memory beforehand (lane =
//   block, off the chain's critical path); only the 8 parent bytes of a payload wait for the previous key.
//
// Tokens arrive by TMA: one elected lane issues a single cp.async.bulk per 2 KB chunk (the prompt's next 512 / B blocks,
// contiguous in HBM) onto an mbarrier, double buffered.  Probes: lane j looks up block j's key (the slot reads of a chunk
// are in flight together, issued 128 tokens' worth of blocks at a time while the chain runs on), a ballot finds the first
// miss, and the hits are scored in block order with lane q owning pod q -- the arithmetic of every other path, bit for bit.
// Block sizes other than these four take score_kernel_v1.
#pragma once
#include <cuda_runtime.h>
#include <type_traits>
#include "score_common.cuh"
#include "kernels_rounds.cuh"

namespace kvx {

constexpr int kCoopWarps = 4;
constexpr int kCoopThreads = kCoopWarps * 32;
constexpr int kCoopChunkTokens = kRoundBlocks * 16;  // tokens per staged chunk (2 KB) at every block size

// The shape of a BS-token block's payload and of a chunk, for BS in {16, 32, 64, 128}.  With a 9-byte parent head the
// array head is 0x90 (BS < 24) or 0x98 BS, so the token bytes start at payload position kHead (11 or 12) and the payload
// is n = tb + kHead + 1 bytes (tb token bytes, then 0xf6), at most 5 BS + kHead + 1.
template <int BS>
struct CoopGeom {
    static_assert(BS == 16 || BS == 32 || BS == 64 || BS == 128, "the cooperative kernels are built for 16/32/64/128-token blocks");
    static constexpr int kHead = BS < 24 ? 11 : 12;
    static constexpr int kPos = (5 * BS + kHead + 1 + 31) / 32;        // consecutive payload positions per lane: 3, 6, 11, 21
    static constexpr int kMaxPayload = 32 * kPos;
    static constexpr int kWords = (kPos + 2) / 3;                      // words of a lane's payload bytes, three to a word
    static constexpr int kHeadLanes = (kHead + kPos - 1) / kPos;       // lanes that own a head position (the parent's among them)
    static constexpr int kRow = 5 * BS + 4;                            // bytes per block row of CBOR token bytes (5 BS + 0xf6,
                                                                       // padded to an odd word count: conflict-free rows)
    static constexpr int kBlocks = kCoopChunkTokens / BS;              // blocks per chunk: 32, 16, 8, 4
    static constexpr int kLead = 128 / BS;                             // blocks per probe group (128 tokens): 8, 4, 2, 1
    static constexpr int kMinCtas = BS == 32 ? 4 : 0;                  // __launch_bounds__ CTAs per SM (0: ptxas's own register
                                                                       // budget, which spills at BS = 32 and holds 4 there)
};

template <int BS>
struct CoopTables { unsigned long long pw[CoopGeom<BS>::kMaxPayload + 1]; unsigned long long c0[CoopGeom<BS>::kMaxPayload + 1]; };
template <int BS>
struct CoopSmem {
    using G = CoopGeom<BS>;
    CoopTables<BS> tab;                                                 // p^j and offset_basis * p^j (mod 2^64)
    struct __align__(128) Warp {
        uint32_t tok[2][kCoopChunkTokens];                              // two 2 KB chunks (TMA destinations)
        unsigned char tokb[G::kBlocks][G::kRow];                        // CBOR bytes of the chunk's token arrays
        uint32_t tb[G::kBlocks];                                        // bytes per block
        uint32_t lanew[G::kBlocks][G::kWords][33];                      // per block, per lane: its payload bytes, three to a word,
                                                                        // each word | which of its three are inside the payload << 24
                                                                        // (rows padded to 33 words: conflict free both ways)
        unsigned long long bar[2];                                      // mbarriers of the two chunk buffers
    } w[kCoopWarps];
};

// ballot of "bit `bit` of z is set" (one LOP3 with predicate output + VOTE)
__device__ __forceinline__ uint32_t ballot_bit(uint32_t z, uint32_t bit) {
    uint32_t r;
    asm volatile("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\tand.b32 t, %1, %2;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 %0, p, 0xffffffff;\n\t}" : "=r"(r) : "r"(z), "r"(bit));
    return r;
}

// One BS-token block, all 32 lanes together.  parent >= 2^32 (9-byte CBOR head); payload = 0x83, 0x1b, 8 parent bytes,
// the array head (0x90, or 0x98 BS), tb token bytes, 0xf6: n = tb + kHead + 1 bytes.  Lane l owns the P = kPos CONSECUTIVE
// positions Pl .. Pl + P-1 (b[i]: the byte there as far as it does not depend on the parent -- 0 past the payload; vmask
// bit i: position Pl + i is inside it).
//
// Bit plane k of the 8-bit recurrence L' = ((L ^ b) * 0xb3) & 0xff: every position contributes g = bit k of (b ^ Y), Y the
// carry word (x mod 2^k) * 0xb3; L_k before a lane's first position is the XOR of all g of earlier lanes -- ONE ballot of
// the lanes' parities and a popcount -- and inside the lane P - 1 more register XORs.  The planes are inherently sequential
// (plane k+1's carries need plane k's x bits): a block is eight rounds of VOTE -> POPC -> (ALU) -> VOTE, whatever BS is; a
// longer block only makes each lane's ALU part longer.  The VOTE + POPC pair is the larger part of a plane at BS = 16;
// scripts/ubench_coop2.cu times a block with one warp, and with alternatives such as preparing the next plane's parity for
// both outcomes while the ballot is in flight, or a shuffle XOR scan instead of the ballot.
template <int BS>
__device__ __forceinline__ uint64_t coop_hash_block(const CoopTables<BS>& tab, uint64_t parent, uint32_t tb, uint32_t (&b)[CoopGeom<BS>::kPos],
                                                    uint32_t vmask, int lane, uint32_t lt) {
    using G = CoopGeom<BS>;
    constexpr int P = G::kPos;
    const uint32_t ph = (uint32_t)(parent >> 32), pl = (uint32_t)parent;
    auto parent_byte = [&](int q) -> uint32_t {                           // payload position q in 2..9: parent byte q - 2, MSB first
        return q < 6 ? (ph >> (8 * (5 - q))) & 0xffu : (pl >> (8 * (9 - q))) & 0xffu;
    };
    // positions 2..9 carry the parent, most significant byte first
#pragma unroll
    for (int l = 0; l < (10 + P - 1) / P; ++l)
        if (lane == l) {
#pragma unroll
            for (int i = 0; i < P; ++i)
                if (P * l + i >= 2 && P * l + i < 10) b[i] = parent_byte(P * l + i);
        }
    constexpr uint32_t L0 = (uint32_t)(kFnvOffset & 0xffu);
    uint32_t bs = 0;
#pragma unroll
    for (int i = 0; i < P; ++i) bs ^= b[i];
    // Y[i] = (x_i mod 2^k) * 0xb3: its bit k is the carry into plane k;  X[i] accumulates x_i = L_i ^ b_i
    uint32_t X[P], Y[P];
#pragma unroll
    for (int i = 0; i < P; ++i) X[i] = Y[i] = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t bit = 1u << k;
        uint32_t py = bs;
#pragma unroll
        for (int i = 0; i < P; ++i) py ^= Y[i];
        const uint32_t B = ballot_bit(py, bit);                               // lanes whose P positions flip the parity
        // x = L ^ b at each position: L before the lane's first position = par ^ L0, then L_{i+1} = L_i ^ g_i
        uint32_t L = ((uint32_t)__popc(B & lt) << k) ^ L0;
#pragma unroll
        for (int i = 0; i < P; ++i) {
            const uint32_t g = b[i] ^ Y[i];
            const uint32_t t = (L ^ b[i]) & bit;
            L ^= g;
            X[i] |= t;
            Y[i] += t * 0xb3u;
        }
    }
    // d = ((L ^ b) & 0xff) - L with L = X ^ b;  weight of position j is p^(n - j)
    const uint32_t n = tb + (uint32_t)G::kHead + 1u, j0 = (uint32_t)P * (uint32_t)lane;
    unsigned long long s = 0;
#pragma unroll
    for (int i = 0; i < P; ++i)
        if (vmask & (1u << i)) s += (unsigned long long)(long long)((int)X[i] - (int)(X[i] ^ b[i])) * tab.pw[n - j0 - i];
    // 64-bit sum over the warp as three limbs of 22 + 21 + 21 bits (each limb sum < 2^27)
    const uint32_t r0 = __reduce_add_sync(0xffffffffu, (uint32_t)s & 0x3fffffu), r1 = __reduce_add_sync(0xffffffffu, (uint32_t)(s >> 22) & 0x1fffffu);
    const uint32_t r2 = __reduce_add_sync(0xffffffffu, (uint32_t)(s >> 43));
    return tab.c0[n] + (unsigned long long)r0 + ((unsigned long long)r1 << 22) + ((unsigned long long)r2 << 43);
}

// The chunk's token arrays as CBOR bytes: lane = block.  Row layout: tb token bytes, then 0xf6.
template <int BS>
__device__ __forceinline__ void coop_layout_chunk(typename CoopSmem<BS>::Warp& W, const uint32_t* tk, int nb, int lane) {
    using G = CoopGeom<BS>;
    constexpr int P = G::kPos;
    if (lane < nb) {
        unsigned char* row = W.tokb[lane];
        uint32_t off = 0;
        const uint4* t4 = reinterpret_cast<const uint4*>(tk + lane * BS);
#pragma unroll 4
        for (int c = 0; c < BS / 4; ++c) {
            const uint4 v = t4[c];
            const uint32_t tv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                // shortest-form CBOR uint, branch free: head byte, then the low len-1 bytes of t, big endian.  Five bytes are
                // always stored; those past `len` are overwritten by the next token (or by the 0xf6 below).
                const uint32_t t = tv[u];
                const uint32_t len = t < 24u ? 1u : t < 256u ? 2u : t < 65536u ? 3u : 5u;
                const uint32_t head = t < 24u ? t : t < 256u ? 0x18u : t < 65536u ? 0x19u : 0x1au;
                const uint32_t be = t << (8u * (5u - len) & 31u);                  // the len-1 payload bytes, left aligned (len 1: unused)
                row[off] = (unsigned char)head;
                row[off + 1] = (unsigned char)(be >> 24); row[off + 2] = (unsigned char)(be >> 16);
                row[off + 3] = (unsigned char)(be >> 8); row[off + 4] = (unsigned char)be;
                off += len;
            }
        }
        row[off] = 0xf6;
        W.tb[lane] = off;
        // the same bytes once more, in the order the hash wants them: word w of lane l's slot in this block's row = the three
        // payload bytes of positions Pl + 3w .. Pl + 3w + 2 (parent bytes left 0) and which of the three are inside the
        // payload.  kWords LDS per block and lane in the chain instead of P dependent byte loads.
        const uint32_t tb = off;
        auto head_byte = [&](int q) -> uint32_t {                             // position q < kHead: the parent-independent head
            return q == 0 ? 0x83u : q == 1 ? 0x1bu : q < 10 ? 0u : q == 10 ? (BS < 24 ? 0x80u | BS : 0x98u) : (uint32_t)BS;
        };
#pragma unroll
        for (int l = 0; l < G::kHeadLanes; ++l) {                            // lanes that own head positions (compile-time bytes)
#pragma unroll
            for (int w = 0; w < G::kWords; ++w) {
                uint32_t word = 0;
#pragma unroll
                for (int u = 0; u < 3; ++u) {
                    const int q = P * l + 3 * w + u;
                    if (3 * w + u >= P) break;
                    word |= (q < G::kHead ? head_byte(q) : (uint32_t)row[q - G::kHead]) << (8 * u) | 1u << (24 + u);   // q - kHead < BS <= tb
                }
                W.lanew[lane][w][l] = word;
            }
        }
#pragma unroll 4
        for (int l = G::kHeadLanes; l < 32; ++l) {
#pragma unroll
            for (int w = 0; w < G::kWords; ++w) {
                const uint32_t i0 = (uint32_t)(P * l + 3 * w - G::kHead);
                uint32_t word = 0;
#pragma unroll
                for (int u = 0; u < 3; ++u) {
                    if (3 * w + u >= P) break;
                    const uint32_t v = i0 + u <= tb;                          // row[tb] is the 0xf6: the last payload byte
                    word |= (v ? (uint32_t)row[i0 + u] : 0u) << (8 * u) | v << (24 + u);
                }
                W.lanew[lane][w][l] = word;
            }
        }
    }
}

// this lane's parent-independent payload bytes of block blk (positions P*lane .. P*lane + P-1) and which of them exist
template <int BS>
__device__ __forceinline__ void coop_block_bytes(const typename CoopSmem<BS>::Warp& W, int blk, int lane, uint32_t& tb, uint32_t (&b)[CoopGeom<BS>::kPos],
                                                 uint32_t& vmask) {
    using G = CoopGeom<BS>;
    tb = W.tb[blk];
    vmask = 0;
#pragma unroll
    for (int w = 0; w < G::kWords; ++w) {
        const uint32_t v = W.lanew[blk][w][lane];
#pragma unroll
        for (int u = 0; u < 3; ++u)
            if (3 * w + u < G::kPos) b[3 * w + u] = (v >> (8 * u)) & 0xffu;
        vmask |= (v >> 24) << (3 * w);
    }
}

// keys of a prompt's next nb (<= kBlocks) blocks; lane j returns the key of block j (lanes >= nb: unspecified).  *last = key
// of block nb-1.  after(blocks_done) is asked every kLead blocks (128 tokens) and ends the chunk early when it says so.
template <int BS, class Probe>
__device__ __forceinline__ int coop_hash_chunk(const CoopSmem<BS>& sm, typename CoopSmem<BS>::Warp& W, const uint32_t* tk, uint64_t h, int nb, int lane, uint32_t lt,
                                               uint64_t& mykey, uint64_t& last, Probe&& after) {
    using G = CoopGeom<BS>;
    coop_layout_chunk<BS>(W, tk, nb, lane);
    __syncwarp();
    uint32_t tb, b[G::kPos], vm;
    coop_block_bytes<BS>(W, 0, lane, tb, b, vm);
    int j = 0;
    for (; j < nb; ++j) {
        uint32_t ntb = 0, nbx[G::kPos], nvm = 0;
#pragma unroll
        for (int i = 0; i < G::kPos; ++i) nbx[i] = 0;
        if (j + 1 < nb) coop_block_bytes<BS>(W, j + 1, lane, ntb, nbx, nvm);               // next block's bytes: off the chain
        uint64_t key;
        if (h >> 32) key = coop_hash_block<BS>(sm.tab, h, tb, b, vm, lane, lt);
        else {                                                                          // short parent head (< 2^32): plain chain, every lane
            Fnv f;
            f.begin_block(h, BS);
            for (int c = 0; c < BS; ++c) f.uint32(tk[j * BS + c]);
            key = f.end_block();
        }
        h = key;
        if (lane == j) mykey = key;
        tb = ntb; vm = nvm;
#pragma unroll
        for (int i = 0; i < G::kPos; ++i) b[i] = nbx[i];
        if (((j + 1) % G::kLead) == 0 && after(j + 1)) { ++j; break; }
    }
    last = h;
    return j;                                                                           // blocks hashed
}

// The CTA's FNV power tables and each warp's two chunk barriers (every thread of the CTA calls this once)
template <int BS>
__device__ __forceinline__ void coop_setup(CoopSmem<BS>& sm, typename CoopSmem<BS>::Warp& W, int lane) {
    for (int i = threadIdx.x; i <= CoopGeom<BS>::kMaxPayload; i += kCoopThreads) {
        unsigned long long p = 1;
        for (int q = 0; q < i; ++q) p *= kFnvPrime;
        sm.tab.pw[i] = p; sm.tab.c0[i] = kFnvOffset * p;
    }
    if (lane == 0) { mbar_init(&W.bar[0], 1); mbar_init(&W.bar[1], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async();
    __syncthreads();
}

// Chunk c of a prompt's nblk BS-token blocks at tokp -> buffer c & 1: one TMA bulk copy by lane 0 onto the buffer's
// barrier, or (tokp not 16-byte aligned) loads by every lane
template <int BS>
__device__ __forceinline__ void coop_stage(typename CoopSmem<BS>::Warp& W, const uint32_t* tokp, int nblk, int c, bool aligned, int lane) {
    constexpr int NB = CoopGeom<BS>::kBlocks;
    const int nbc = min(NB, nblk - c * NB);
    if (nbc <= 0) return;
    const uint32_t* src = tokp + (size_t)c * NB * BS;
    if (aligned) {
        if (lane == 0) { fence_proxy_async(); mbar_expect_tx(&W.bar[c & 1], (uint32_t)nbc * BS * 4); tma_load_1d(W.tok[c & 1], src, (uint32_t)nbc * BS * 4, &W.bar[c & 1]); }
    } else {
        for (int x = lane; x < nbc * BS; x += 32) W.tok[c & 1][x] = __ldg(src + x);
    }
}

// One chunk of nb <= kBlocks staged blocks (tk) of a warp-per-prompt token walk, chain seeded with h (left at the chunk's
// last key): lane j hashes with the warp and probes block j as soon as the kLead blocks (128 tokens) around it are hashed, a
// ballot finds the first miss, the hits are walked and marked.  `cont` / `first_block` as for WarpWalk::walk.  Returns the
// consecutive hits from the chunk's first block (0 when `probe` is false: no slot is read).  `all`: every block of the
// chunk is hashed (lane j's key in `key`) also once a miss is seen, probes still stop there; else a miss ends the hashing
// too (`probe` true).
template <int BS>
__device__ __forceinline__ int coop_walk_chunk(const TableView& t, const CoopSmem<BS>& sm, typename CoopSmem<BS>::Warp& W, const uint32_t* tk, uint64_t& h, int nb,
                                               int lane, uint32_t lt, uint32_t mdl, bool peer, bool all, bool probe, WarpWalk& ws, bool cont, bool first_block,
                                               const uint64_t* filter, int64_t pi, uint64_t& key) {
    constexpr int LEAD = CoopGeom<BS>::kLead;
    // ---- keys; lane j probes block j as soon as the kLead blocks around it are hashed ----
    uint64_t last = 0;
    key = 0;
    uint4 A0 = {0, 0, 0, 0}, B0 = {0, 0, 0, 0}, A1 = {0, 0, 0, 0}, B1 = {0, 0, 0, 0};
    const ReqSlot* base = t.req; uint64_t slot = 0;
    bool issued = false, hit = false, decided = false;
    int nprobe = all && !probe ? 0 : CoopGeom<BS>::kBlocks;             // all: the blocks probed before a miss was seen
    SlotPat mine = {};
    uint64_t hslot = 0;                                           // CLOCK: slot of this lane's hit
    auto resolve = [&]() {                                        // the slot pair has (or will have) arrived: hit or miss
        uint4 A, B;
        while (!pair_decides(A0, B0, A1, B1, key, mdl, A, B, hit)) {
            slot = (slot + 2) & t.req_mask;                       // rare: displaced past the home pair
            ld_slot_pair(base + slot, peer, A0, B0, A1, B1);
        }
        if (hit) { mine = SlotPat::of(A, B); if (t.req_ref) hslot = pair_hit_slot(slot, A0, B0, key, mdl); }
        decided = true;
    };
    const int nhashed = coop_hash_chunk<BS>(sm, W, tk, h, nb, lane, lt, key, last, [&](int ndone) -> bool {
        if (all && nprobe < ndone) return false;                            // past a miss (or not probing): hashing only
        if (lane >= ndone - LEAD && lane < ndone) {               // the keys just produced: request their slot pairs
            const uint64_t hm = home_of(key, mdl);
            base = t.req_peer[shard_of(hm, t.shard_bits)]; slot = hm & t.req_mask & ~1ull;
            ld_slot_pair(base + slot, peer, A0, B0, A1, B1);
            issued = true;
        }
        if (ndone < 2 * LEAD) return false;
        if (lane >= ndone - 2 * LEAD && lane < ndone - LEAD) resolve();    // the group before them has landed: a miss ends the prompt
        const bool miss = __any_sync(0xffffffffu, decided && !hit);
        if (all) { if (miss) nprobe = ndone; return false; }
        return miss;
    });
    const int np = all ? min(nhashed, nprobe) : nhashed;         // blocks that are probed
    // blocks hashed but not yet requested / resolved
    if (lane < np && !issued) {
        const uint64_t hm = home_of(key, mdl);
        base = t.req_peer[shard_of(hm, t.shard_bits)]; slot = hm & t.req_mask & ~1ull;
        ld_slot_pair(base + slot, peer, A0, B0, A1, B1);
        issued = true;
    }
    if (lane < np && !decided) resolve();
    const uint32_t hm_ = __ballot_sync(0xffffffffu, hit && lane < np);
    const int nhit = hm_ == 0xffffffffu ? 32 : __ffs(~hm_) - 1;   // consecutive hits from the chunk's first block
    // ---- ordered scoring of the hits (kvblock_scorer.go:108-151), lane q owns pod q ----
    const int nwalked = ws.walk<false>(t, lane, mine, nhit, ws.same_mask(lane, mine, cont, nhit), first_block, filter, pi, [](int) {});
    WarpWalk::mark_walked(t, lane, nwalked, hit, hslot);
    h = last;
    return nhit;
}

template <int BS>
__global__ void __launch_bounds__(kCoopThreads, CoopGeom<BS>::kMinCtas)
coop_score_kernel(const TableView t, const ScoreArgs a) {
    using G = CoopGeom<BS>;
    const uint64_t l2pol = l2_policy_stream();
    extern __shared__ __align__(128) unsigned char smem_raw_c[];
    CoopSmem<BS>& sm = *reinterpret_cast<CoopSmem<BS>*>(smem_raw_c);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
    typename CoopSmem<BS>::Warp& W = sm.w[wid];
    coop_setup<BS>(sm, W, lane);
    const bool peer = t.shard_bits != 0;
    uint32_t phases = 0;                                                  // bit s: parity the next wait on buffer s uses
    const long long total_warps = (long long)gridDim.x * kCoopWarps;
    for (long long pi = (long long)blockIdx.x * kCoopWarps + wid; pi < a.n_prompts; pi += total_warps) {
        const int64_t tb0 = a.tok_off[pi] - a.tok_base, te = a.tok_off[pi + 1] - a.tok_base;
        const int nblk = (int)((te - tb0) / BS);
        const uint32_t* tokp = a.tok + tb0;
        const bool aligned = (reinterpret_cast<uintptr_t>(tokp) & 15u) == 0;
        const uint32_t mdl = a.model ? a.model[pi] : a.model0;
        WarpWalk ws;
        uint64_t h = t.init_hash;
        auto stage = [&](int c) { coop_stage<BS>(W, tokp, nblk, c, aligned, lane); };
        stage(0);
        bool done = nblk == 0;
        const int nchunks = (nblk + G::kBlocks - 1) / G::kBlocks;
        int consumed = 0;                                                 // chunks waited for (at most one more is in flight)
        for (int c = 0; c < nchunks && !done; ++c) {
            __syncwarp();                                                 // every lane is done with buffer (c+1)&1 (chunk c-1)
            stage(c + 1);
            if (aligned) { mbar_wait(&W.bar[c & 1], (phases >> (c & 1)) & 1u); phases ^= 1u << (c & 1); }
            consumed = c + 1;
            __syncwarp();
            const int nb = min(G::kBlocks, nblk - c * G::kBlocks);
            const bool has_more = (c + 1) * G::kBlocks < nblk;
            uint64_t key;
            const int nhit = coop_walk_chunk<BS>(t, sm, W, W.tok[c & 1], h, nb, lane, lt, mdl, peer, false, true, ws, c > 0, c == 0, a.filter, pi, key);
            if (!ws.alive || nhit < nb || !has_more) done = true;
        }
        // ---- result ----
        warp_write_row(t, a, pi, ws.k, ws.pod, ws.sc, nblk > 0, l2pol);
        // a chunk that was prefetched but never consumed (the walk ended before it) still lands in its buffer: let it, so that
        // the buffer and its barrier are free for the next prompt
        if (aligned && consumed < nchunks && consumed > 0) { mbar_wait(&W.bar[consumed & 1], (phases >> (consumed & 1)) & 1u); phases ^= 1u << (consumed & 1); }
        __syncwarp();
    }
}

// The block sizes the cooperative kernels are built for (every other one takes score_kernel_v1)
inline bool coop_block_size(uint32_t bs) { return bs == 16 || bs == 32 || bs == 64 || bs == 128; }

// f(std::integral_constant<int, BS>{}) for BS = bs, one of the coop_block_size() sizes
template <class F>
inline auto coop_dispatch(uint32_t bs, F&& f) {
    switch (bs) {
    case 32: return f(std::integral_constant<int, 32>{});
    case 64: return f(std::integral_constant<int, 64>{});
    case 128: return f(std::integral_constant<int, 128>{});
    default: return f(std::integral_constant<int, 16>{});
    }
}

template <int BS>
inline bool coop_init_one() {
    return cudaFuncSetAttribute(coop_score_kernel<BS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CoopSmem<BS>)) == cudaSuccess;
}
inline int coop_init() {
    return coop_init_one<16>() && coop_init_one<32>() && coop_init_one<64>() && coop_init_one<128>() ? 0 : -1;
}

}  // namespace kvx
