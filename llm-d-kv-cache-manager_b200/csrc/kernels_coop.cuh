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
//     all g before j -- ONE warp ballot and a popcount per 32 positions.  8 planes x 3 ballots cover a 96-byte payload
//     (a 16-token block is 28..92 CBOR bytes);
//   * every block's payload starts from the FNV offset basis (the parent hash enters as BYTES), so h_0 * p^n is a table.
//
//   A block then costs 8 ballot/popcount rounds plus one warp reduction instead of ~90 dependent multiply steps.
//   The token bytes of a whole 32-block chunk are laid out in shared memory beforehand (lane = block, off the chain's
//   critical path); only the 8 parent bytes of a payload wait for the previous key.
//
// Tokens arrive by TMA: one elected lane issues a single cp.async.bulk per 2 KB chunk (the prompt's next 32 blocks,
// contiguous in HBM) onto an mbarrier, double buffered.  Probes: lane j looks up block j's key (the 32 slot reads of a
// chunk are in flight together, issued eight blocks at a time while the chain runs on), a ballot finds the first miss,
// and the hits are scored in block order with lane q owning pod q -- the arithmetic of every other path, bit for bit.
#pragma once
#include <cuda_runtime.h>
#include "score_common.cuh"
#include "kernels_rounds.cuh"

namespace kvx {

constexpr int kCoopWarps = 4;
constexpr int kCoopThreads = kCoopWarps * 32;
constexpr int kCoopRow = 84;                       // bytes per block row of CBOR token bytes (80 + 0xf6, padded: conflict-free rows)
constexpr int kCoopMaxPayload = 96;

struct CoopTables { unsigned long long pw[kCoopMaxPayload + 1]; unsigned long long c0[kCoopMaxPayload + 1]; };
struct CoopSmem {
    CoopTables tab;                                                     // p^j and offset_basis * p^j (mod 2^64)
    struct __align__(128) Warp {
        uint32_t tok[2][kRoundBlocks * 16];                             // two 2 KB chunks (TMA destinations)
        unsigned char tokb[kRoundBlocks][kCoopRow];                     // CBOR bytes of the chunk's token arrays
        uint32_t tb[kRoundBlocks];                                      // bytes per block
        uint32_t lanew[kRoundBlocks][33];                               // per block, per lane: its three payload bytes | vmask << 24
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

// One 16-token block, all 32 lanes together.  parent >= 2^32 (9-byte CBOR head); payload = 0x83, 0x1b, 8 parent bytes,
// 0x90, tb token bytes, 0xf6: n = tb + 12 bytes.  Lane l owns the three CONSECUTIVE positions 3l, 3l+1, 3l+2 (b0..b2: the
// bytes there as far as they do not depend on the parent -- 0 past the payload; vmask bit i: position 3l+i is inside it).
//
// Bit plane k of the 8-bit recurrence L' = ((L ^ b) * 0xb3) & 0xff: every position contributes g = bit k of (b ^ Y), Y the
// carry word (x mod 2^k) * 0xb3; L_k before a lane's first position is the XOR of all g of earlier lanes -- ONE ballot of
// the lanes' parities and a popcount -- and inside the lane two more register XORs.  The planes are inherently sequential
// (plane k+1's carries need plane k's x bits): a block is eight rounds of VOTE -> POPC -> (4 ALU) -> VOTE.  The VOTE + POPC
// pair is the larger part of a plane; scripts/ubench_coop2.cu times a block with one warp, and with alternatives such as
// preparing the next plane's parity for both outcomes while the ballot is in flight, or a shuffle XOR scan instead of the
// ballot.
__device__ __forceinline__ uint64_t coop_hash_block(const CoopTables& tab, uint64_t parent, uint32_t tb, uint32_t b0, uint32_t b1, uint32_t b2,
                                                    uint32_t vmask, int lane, uint32_t lt) {
    if (lane < 4) {                                         // positions 2..9 carry the parent, most significant byte first
        const uint32_t ph = (uint32_t)(parent >> 32), pl = (uint32_t)parent;
        if (lane == 0) b2 = ph >> 24;
        else if (lane == 1) { b0 = (ph >> 16) & 0xffu; b1 = (ph >> 8) & 0xffu; b2 = ph & 0xffu; }
        else if (lane == 2) { b0 = pl >> 24; b1 = (pl >> 16) & 0xffu; b2 = (pl >> 8) & 0xffu; }
        else b0 = pl & 0xffu;
    }
    constexpr uint32_t L0 = (uint32_t)(kFnvOffset & 0xffu);
    const uint32_t bs = b0 ^ b1 ^ b2;
    // Y_i = (x_i mod 2^k) * 0xb3: its bit k is the carry into plane k;  X_i accumulates x_i = L_i ^ b_i
    uint32_t X0 = 0, X1 = 0, X2 = 0, Y0 = 0, Y1 = 0, Y2 = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t bit = 1u << k;
        const uint32_t z0 = b0 ^ Y0, z01 = z0 ^ b1 ^ Y1;                      // g0, g0^g1 at bit k (needed only after the vote)
        const uint32_t B = ballot_bit(bs ^ Y0 ^ Y1 ^ Y2, bit);                // lanes whose three positions flip the parity
        const uint32_t par = (uint32_t)__popc(B & lt) << k;                   // L (before the lane's first position) ^ L0, at bit k
        // x = L ^ b at each position:  L_0 = par ^ L0,  L_1 = L_0 ^ g0,  L_2 = L_1 ^ g1
        const uint32_t t0 = (par ^ L0 ^ b0) & bit;
        const uint32_t t1 = (par ^ L0 ^ z0 ^ b1) & bit;
        const uint32_t t2 = (par ^ L0 ^ z01 ^ b2) & bit;
        X0 |= t0; X1 |= t1; X2 |= t2;
        Y0 += t0 * 0xb3u; Y1 += t1 * 0xb3u; Y2 += t2 * 0xb3u;
    }
    // d = ((L ^ b) & 0xff) - L with L = X ^ b;  weight of position j is p^(n - j)
    const uint32_t n = tb + 12u, j0 = 3u * (uint32_t)lane;
    unsigned long long s = 0;
    if (vmask & 1u) s += (unsigned long long)(long long)((int)X0 - (int)(X0 ^ b0)) * tab.pw[n - j0];
    if (vmask & 2u) s += (unsigned long long)(long long)((int)X1 - (int)(X1 ^ b1)) * tab.pw[n - j0 - 1];
    if (vmask & 4u) s += (unsigned long long)(long long)((int)X2 - (int)(X2 ^ b2)) * tab.pw[n - j0 - 2];
    // 64-bit sum over the warp as three limbs of 22 + 21 + 21 bits (each limb sum < 2^27)
    const uint32_t r0 = __reduce_add_sync(0xffffffffu, (uint32_t)s & 0x3fffffu), r1 = __reduce_add_sync(0xffffffffu, (uint32_t)(s >> 22) & 0x1fffffu);
    const uint32_t r2 = __reduce_add_sync(0xffffffffu, (uint32_t)(s >> 43));
    return tab.c0[n] + (unsigned long long)r0 + ((unsigned long long)r1 << 22) + ((unsigned long long)r2 << 43);
}

// The chunk's token arrays as CBOR bytes: lane = block.  Row layout: tb token bytes, then 0xf6.
__device__ __forceinline__ void coop_layout_chunk(CoopSmem::Warp& W, const uint32_t* tk, int nb, int lane) {
    if (lane < nb) {
        unsigned char* row = W.tokb[lane];
        uint32_t off = 0;
        const uint4* t4 = reinterpret_cast<const uint4*>(tk + lane * 16);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
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
        // the same bytes once more, in the order the hash wants them: word l of this block's row = the three payload bytes of
        // positions 3l .. 3l+2 (parent bytes left 0) and which of the three are inside the payload.  One LDS per block and lane
        // in the chain instead of three dependent byte loads.
        const uint32_t tb = off;
        W.lanew[lane][0] = 0x83u | (0x1bu << 8) | (7u << 24);
        W.lanew[lane][1] = 7u << 24;
        W.lanew[lane][2] = 7u << 24;
        W.lanew[lane][3] = (0x90u << 8) | ((uint32_t)row[0] << 16) | (7u << 24);
#pragma unroll 4
        for (int l = 4; l < 32; ++l) {
            const uint32_t i0 = 3u * (uint32_t)l - 11u;
            const uint32_t v0 = i0 <= tb, v1 = i0 + 1 <= tb, v2 = i0 + 2 <= tb;       // row[tb] is the 0xf6: the last payload byte
            const uint32_t r0 = v0 ? row[i0] : 0u, r1 = v1 ? row[i0 + 1] : 0u, r2 = v2 ? row[i0 + 2] : 0u;
            W.lanew[lane][l] = r0 | (r1 << 8) | (r2 << 16) | ((v0 | (v1 << 1) | (v2 << 2)) << 24);
        }
    }
}

// this lane's parent-independent payload bytes of block blk (positions 3*lane .. 3*lane+2) and which of them exist
__device__ __forceinline__ void coop_block_bytes(const CoopSmem::Warp& W, int blk, int lane, uint32_t& tb, uint32_t& b0, uint32_t& b1, uint32_t& b2, uint32_t& vmask) {
    const uint32_t w = W.lanew[blk][lane];
    tb = W.tb[blk];
    b0 = w & 0xffu; b1 = (w >> 8) & 0xffu; b2 = (w >> 16) & 0xffu; vmask = w >> 24;
}

// keys of a prompt's next nb (<= 32) blocks; lane j returns the key of block j (lanes >= nb: unspecified).  *last = key of
// block nb-1.  stop_after(blocks_done) is asked every eight blocks and ends the chunk early.
template <class Probe>
__device__ __forceinline__ int coop_hash_chunk(const CoopSmem& sm, CoopSmem::Warp& W, const uint32_t* tk, uint64_t h, int nb, int lane, uint32_t lt,
                                               uint64_t& mykey, uint64_t& last, Probe&& after8) {
    coop_layout_chunk(W, tk, nb, lane);
    __syncwarp();
    uint32_t tb, b0, b1, b2, vm;
    coop_block_bytes(W, 0, lane, tb, b0, b1, b2, vm);
    int j = 0;
    for (; j < nb; ++j) {
        uint32_t ntb = 0, nb0 = 0, nb1 = 0, nb2 = 0, nvm = 0;
        if (j + 1 < nb) coop_block_bytes(W, j + 1, lane, ntb, nb0, nb1, nb2, nvm);      // next block's bytes: off the chain
        uint64_t key;
        if (h >> 32) key = coop_hash_block(sm.tab, h, tb, b0, b1, b2, vm, lane, lt);
        else {                                                                          // short parent head (< 2^32): plain chain, every lane
            Fnv f;
            f.begin_block(h, 16);
            for (int c = 0; c < 16; ++c) f.uint32(tk[j * 16 + c]);
            key = f.end_block();
        }
        h = key;
        if (lane == j) mykey = key;
        tb = ntb; b0 = nb0; b1 = nb1; b2 = nb2; vm = nvm;
        if (((j + 1) & 7) == 0 && after8(j + 1)) { ++j; break; }
    }
    last = h;
    return j;                                                                           // blocks hashed
}

// The CTA's FNV power tables and each warp's two chunk barriers (every thread of the CTA calls this once)
__device__ __forceinline__ void coop_setup(CoopSmem& sm, CoopSmem::Warp& W, int lane) {
    for (int i = threadIdx.x; i <= kCoopMaxPayload; i += kCoopThreads) {
        unsigned long long p = 1;
        for (int q = 0; q < i; ++q) p *= kFnvPrime;
        sm.tab.pw[i] = p; sm.tab.c0[i] = kFnvOffset * p;
    }
    if (lane == 0) { mbar_init(&W.bar[0], 1); mbar_init(&W.bar[1], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async();
    __syncthreads();
}

// Chunk c of a prompt's nblk 16-token blocks at tokp -> buffer c & 1: one TMA bulk copy by lane 0 onto the buffer's
// barrier, or (tokp not 16-byte aligned) loads by every lane
__device__ __forceinline__ void coop_stage(CoopSmem::Warp& W, const uint32_t* tokp, int nblk, int c, bool aligned, int lane) {
    constexpr int BS = 16;
    const int nbc = min(kRoundBlocks, nblk - c * kRoundBlocks);
    if (nbc <= 0) return;
    const uint32_t* src = tokp + (size_t)c * kRoundBlocks * BS;
    if (aligned) {
        if (lane == 0) { fence_proxy_async(); mbar_expect_tx(&W.bar[c & 1], (uint32_t)nbc * BS * 4); tma_load_1d(W.tok[c & 1], src, (uint32_t)nbc * BS * 4, &W.bar[c & 1]); }
    } else {
        for (int x = lane; x < nbc * BS; x += 32) W.tok[c & 1][x] = __ldg(src + x);
    }
}

// One chunk of nb <= 32 staged blocks (tk) of a warp-per-prompt token walk, chain seeded with h (left at the chunk's last
// key): lane j hashes with the warp and probes block j as soon as the eight blocks around it are hashed, a ballot finds the
// first miss, the hits are walked and marked.  `cont` / `first_block` as for WarpWalk::walk.  Returns the consecutive hits
// from the chunk's first block (0 when `probe` is false: no slot is read).  `all`: every block of the chunk is hashed (lane
// j's key in `key`) also once a miss is seen, probes still stop there; else a miss ends the hashing too (`probe` true).
__device__ __forceinline__ int coop_walk_chunk(const TableView& t, const CoopSmem& sm, CoopSmem::Warp& W, const uint32_t* tk, uint64_t& h, int nb,
                                               int lane, uint32_t lt, uint32_t mdl, bool peer, bool all, bool probe, WarpWalk& ws, bool cont, bool first_block,
                                               const uint64_t* filter, int64_t pi, uint64_t& key) {
    // ---- keys; lane j probes block j as soon as the eight blocks around it are hashed ----
    uint64_t last = 0;
    key = 0;
    uint4 A0 = {0, 0, 0, 0}, B0 = {0, 0, 0, 0}, A1 = {0, 0, 0, 0}, B1 = {0, 0, 0, 0};
    const ReqSlot* base = t.req; uint64_t slot = 0;
    bool issued = false, hit = false, decided = false;
    int nprobe = all && !probe ? 0 : kRoundBlocks;                      // all: the blocks probed before a miss was seen
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
    const int nhashed = coop_hash_chunk(sm, W, tk, h, nb, lane, lt, key, last, [&](int ndone) -> bool {
        if (all && nprobe < ndone) return false;                            // past a miss (or not probing): hashing only
        if (lane >= ndone - 8 && lane < ndone) {                  // the eight keys just produced: request their slot pairs
            const uint64_t hm = home_of(key, mdl);
            base = t.req_peer[shard_of(hm, t.shard_bits)]; slot = hm & t.req_mask & ~1ull;
            ld_slot_pair(base + slot, peer, A0, B0, A1, B1);
            issued = true;
        }
        if (ndone < 16) return false;
        if (lane >= ndone - 16 && lane < ndone - 8) resolve();   // the eight before them have landed: a miss ends the prompt
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
__global__ void __launch_bounds__(kCoopThreads)
coop_score_kernel(const TableView t, const ScoreArgs a) {
    const uint64_t l2pol = l2_policy_stream();
    static_assert(BS == 16, "payload layout is written for 16-token blocks");
    extern __shared__ __align__(128) unsigned char smem_raw_c[];
    CoopSmem& sm = *reinterpret_cast<CoopSmem*>(smem_raw_c);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
    CoopSmem::Warp& W = sm.w[wid];
    coop_setup(sm, W, lane);
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
        auto stage = [&](int c) { coop_stage(W, tokp, nblk, c, aligned, lane); };
        stage(0);
        bool done = nblk == 0;
        const int nchunks = (nblk + kRoundBlocks - 1) / kRoundBlocks;
        int consumed = 0;                                                 // chunks waited for (at most one more is in flight)
        for (int c = 0; c < nchunks && !done; ++c) {
            __syncwarp();                                                 // every lane is done with buffer (c+1)&1 (chunk c-1)
            stage(c + 1);
            if (aligned) { mbar_wait(&W.bar[c & 1], (phases >> (c & 1)) & 1u); phases ^= 1u << (c & 1); }
            consumed = c + 1;
            __syncwarp();
            const int nb = min(kRoundBlocks, nblk - c * kRoundBlocks);
            const bool has_more = (c + 1) * kRoundBlocks < nblk;
            uint64_t key;
            const int nhit = coop_walk_chunk(t, sm, W, W.tok[c & 1], h, nb, lane, lt, mdl, peer, false, true, ws, c > 0, c == 0, a.filter, pi, key);
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

inline int coop_init() {
    return cudaFuncSetAttribute(coop_score_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CoopSmem)) == cudaSuccess ? 0 : -1;
}

}  // namespace kvx
