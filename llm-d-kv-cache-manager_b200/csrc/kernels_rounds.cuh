// kernels_rounds.cuh -- Score() for LARGE batches: rounds over PREFIX CLASSES.
//
// Same reference path as every Score() kernel (GetPodScores steps 2-4, pkg/kvcache/indexer.go:141-163): chain keys
// (token_processor.go:94-162), Lookup (in_memory.go:105-146), LongestPrefixScorer.Score (kvblock_scorer.go:108-151); the
// probe, the fold and the result row are the ones of score_common.cuh.
//
// A large batch repeats itself: thousands of prompts share a system prompt or a document, and the per-prompt kernels
// hash and probe that shared prefix once per prompt.  Here the batch is processed in rounds of kRoundBlocks blocks, and
// in every round the live prompts are partitioned into CLASSES -- same walk state, same model and filter, and a
// token-for-token identical next chunk.  One representative per class is hashed and walked; the other members take its
// outcome.  Class membership is never decided by a hash: every member has been compared with its class's chunk, so the
// results are bit-identical to the per-prompt kernels and the oracle for any input (tests run all paths).
//
//   G   group_round_kernel   stream every live prompt's chunk once, find the classes (compare with the running class's
//                            anchor chunk; election through a small map for the rest)
//   G2  group_lists_kernel   prompts that leave a class in the middle of the chunk become partial followers (class, d);
//                            compact the lists: representatives / followers / partial followers
//   H   hash_round_kernel    FNV-64a / CBOR chain keys of the representatives' chunks
//   P   walk_round_kernel    warp per representative: 32 probes at once, ordered scoring of the hits, run snapshots
//   R+D finish_round_kernel  followers copy their representative's fate; partial followers resume from its snapshot and
//                            walk their own blocks
//   C   compact_round_kernel next round's live list: the prompts that continue, in the order of this round's list
//
// What a prompt carries between rounds (position, chain state, where its walk state is) lives in a LiveRec per LIVE SLOT
// and moves with the slot; the walk states are stored by the slot of the round that wrote them.  So every kernel reads a
// live slot's state in list order, and the prompt id is only needed for the result row and the model / filter rows.
//
// Every round pays a fixed cost of short latency-bound kernels (hidden by running the batch as independent parts
// on separate streams), so medium batches use kernels_rounds_plain.cuh instead (see kvidx.cu: launch_score).
#pragma once
#include <cuda_runtime.h>
#include "score_common.cuh"

namespace kvx {

constexpr int kRoundBlocks = 32;         // blocks hashed per prompt per round (== lanes per warp in kernel P)
constexpr int kHashThreads = 256;
constexpr int kHashStages = 2;           // token blocks staged per prompt.  (4 stages x 4 warps is the alternative: what a launch of this kernel
                                         // waits for is room on an SM beside kernel G's CTAs, so the smaller footprint per warp is the choice)
constexpr int kGroupThreads = 256;
constexpr uint32_t kRoleSelf = 0xffffffffu;

struct __align__(8) PromptState {        // walk state carried between rounds (only for prompts that continue)
    double sc[kMaxEnt];
    uint16_t pod[kMaxEnt];
    uint32_t pat[6];                     // entry words + count of the last scored block's slot
    uint16_t alive;                      // bitmask over [0,k)
    uint8_t k;
    uint8_t pad;
    uint8_t bt[kMaxEnt];                 // tier giving pod q its max weight in that slot (0xff: 0.0)
    uint8_t pad2[2];
};

constexpr int kMaxParts = 16;             // the sorted batch runs as up to this many independent parts on their own streams

// What a live prompt carries from round to round, stored by LIVE SLOT: kernel C moves it into the next list together with
// the slot.  The kernels read one coalesced record per slot instead of gathering each field by prompt id.
struct __align__(16) LiveRec {
    int64_t tok;                         // token index of the prompt's next chunk (relative to tok_base)
    uint32_t left;                       // full blocks from there to the end of the prompt
    uint32_t src;                        // live slot of the previous round whose PromptState is this prompt's walk state:
                                         // its own, or its class representative's (round 0: kRoleSelf)
    uint64_t hstate;                     // chain hash after the last block of the previous round (round 0: the initial hash)
    uint32_t srcp;                       // the prompt in slot src (round 0: kRoleSelf).  Same state <=> same srcp; the class
                                         // election key hashes it
    uint32_t p;                          // prompt id: only for its result row, has_keys, model and filter row
};
static_assert(sizeof(LiveRec) == 32, "two 16-byte halves");
__device__ __forceinline__ LiveRec live_load(const LiveRec* r) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(r)), v = __ldg(reinterpret_cast<const uint4*>(r) + 1);
    LiveRec L;
    L.tok = (int64_t)(((uint64_t)u.y << 32) | u.x); L.left = u.z; L.src = u.w;
    L.hstate = ((uint64_t)v.y << 32) | v.x; L.srcp = v.z; L.p = v.w;
    return L;
}
// the record of a prompt that continues next round: tok / left advanced, walk state in slot src (prompt srcp), chain state h
__device__ __forceinline__ void live_store(LiveRec* r, int64_t tok, uint32_t left, uint32_t src, uint64_t h, uint32_t srcp, uint32_t p) {
    uint4* d = reinterpret_cast<uint4*>(r);
    d[0] = make_uint4((uint32_t)(uint64_t)tok, (uint32_t)((uint64_t)tok >> 32), left, src);
    d[1] = make_uint4((uint32_t)h, (uint32_t)(h >> 32), srcp, p);
}

struct RoundBufs {
    LiveRec* live[2];                    // live lists (ping-pong): one record per live slot, in the order of the round-0 sort
    unsigned int* n_act;                 // [2] list lengths
    uint32_t* nmap;                      // [n_act] written by kernel C: live slot of this round -> its slot next round (prompts that continue)
    PromptState* pst[2];                 // by live slot of the round that wrote it, by round parity (round r reads [r&1 ^ 1] at
                                         // LiveRec::src, writes [r&1])
    uint64_t* keys;                      // [kRoundBlocks][n_prompts] keys of the current round, block-major, by position in
                                         // the representative list: key of block j of entry a at keys[j * n_prompts + a]
    uint32_t* nbr;                       // [n_act] per live slot: blocks in this round | (more blocks follow) << 8
    // prefix classes (group_round_kernel): live prompts with the same walk state, model and filter whose next chunk of
    // tokens is identical get identical keys, probes, scores and fate this round.  One representative per class is
    // hashed and walked; the others wait in the follower list and take the representative's outcome.
    uint32_t* role;                      // [n_act] kRoleSelf: representative (or alone); else the live slot of its representative
    uint8_t* fate;                       // [n_act] kFateMore (continues next round) / kFateDone, for every live slot: written by
                                         // kernel P for representatives, R for followers, D for partial followers; read by C
    uint32_t* hl;                        // [n_act] representative list (live slots), compacted
    uint2* fl;                           // [n_act] follower list {live slot, its representative's live slot}, compacted
    unsigned int* n_hl;                  // [0] representatives, [1] followers, [2] partial followers (zeroed before every round)
    unsigned int* stat;                  // with KVIDX_ROUNDS_TRACE=1, running totals of the batch: [0] chunks kernel G streams,
                                         // [1] election losers that read two chunks again in G, [2] chunk compares in G2,
                                         // [3] blocks kernel H hashes
    // partial followers: a prompt alone in its class whose chunk starts like a neighbouring class's chunk (it leaves a
    // popular prefix inside this chunk) shares the first dmin blocks with that class -- keys and walk -- and continues on
    // its own from there (detach_round_kernel)
    uint8_t* nfol;                       // [n_act] live slot has followers (it must stay a representative); zeroed per round
    uint8_t* need_snap;                  // [n_act] representative must record its walk state after every block; zeroed per round
    uint32_t* anch;                      // [n_act] live slot of the representative it could share a chunk prefix with
    uint8_t* dmin;                       // [n_act] ... and the number of leading blocks it shares (0: none)
    uint32_t* apos;                      // [n_act] live slot -> position in the representative list
    unsigned long long* scan;            // [tiles of kernel C] per tile: round + 1 << 32 | prefix done << 31 | live slots (zeroed per batch)
    uint4* rec;                          // [n_hl] per representative {prompt, live slot, nbr word, src}: one load instead of a chain
    uint4* drec;                         // [n_dl] per partial follower {live slot, representative's live slot, shared blocks << 16 | nbr word, prompt}
    uint32_t* grp;                       // [n_act] by live slot of last round's representative R: a class of this round whose members
                                         // had R's state (kRoleSelf: none); cleared with the map
    uint8_t* nwalk;                      // [n_hl] blocks of the round after which the representative's walk was still alive
    // walk snapshots, one per RUN of blocks with the same slot pattern: state after the run's first block; the state after a
    // later block of the run is that plus (distance) in-order additions of the same per-pod addend
    uint8_t* snap_run;                   // [n_hl][32] first block of the run block j belongs to
    uint16_t* snap_alive;                // [n_hl][32] alive mask after block j (stored at run starts)
    uint8_t* snap_bt;                    // [n_hl][32][kMaxEnt] tier that gives pod q its addend (0xff: 0.0) (at run starts)
    double* snap_sc;                     // [n_hl][32][kMaxEnt] scores after block j (at run starts)
    uint32_t part_size;                  // prompts in this part (rounded up to 32): length of the per-slot arrays
    uint32_t* map;                       // class election: bucket -> live slot (kRoleSelf = empty), cleared before every round
    uint32_t map_mask;
};
constexpr uint8_t kFateMore = 1, kFateDone = 2;

// The counters of a round-pipeline batch, cleared by one memset per batch.  Part q's RoundBufs::n_act, n_hl and stat point
// into part[q] and stat[q] (the per-prompt rounds' two halves are parts 0 and 1); rounds_init_kernel sets the first list
// lengths and max_blocks.
struct RoundCounters {
    struct Part {
        unsigned int n_act[2];           // RoundBufs::n_act
        unsigned int n_hl[4];            // RoundBufs::n_hl; [3]: with KVIDX_ROUNDS_TRACE=1, blocks partial followers walked alone
        unsigned int unused[2];
    } part[kMaxParts];
    unsigned long long max_blocks;       // full blocks of the batch's longest prompt
    unsigned long long distinct;         // distinct first-block fingerprints (count_distinct_prefixes_kernel)
    unsigned int stat[kMaxParts][4];     // RoundBufs::stat
};
static_assert(sizeof(RoundCounters::Part) == 32 && offsetof(RoundCounters, max_blocks) == 4 * 8 * kMaxParts &&
              offsetof(RoundCounters, distinct) == offsetof(RoundCounters, max_blocks) + 8 &&
              offsetof(RoundCounters, stat) == 4 * (8 * kMaxParts + 4), "counter words: part q at 8 q, then max_blocks, distinct, stat");

template <int BS> struct HashSmem {
    static constexpr int kRow = BS * 4 + 16;                 // 80 B: the four LDS.128 of a block stay conflict free
    unsigned char tok[kHashThreads / 32][kHashStages][32 * kRow];     // [warps of the CTA]: a launch with fewer warps passes that much less
};

// ---- kernel G: prefix classes ------------------------------------------------------------------------------
// A warp takes 32 live slots.  Metadata is lane-parallel; each prompt's next chunk (<= 32 blocks = 2 KB) is then read by
// the whole warp (coalesced) and folded into a 64-bit fingerprint.  Lane-parallel again, every prompt tries to claim
// bucket hash(state source, chain state, model, fingerprint) of a small map: the winner represents the class; a loser
// compares itself with the bucket owner -- state source, chain state, block count, model, filter row, and the chunk
// token by token (warp-wide, 16 bytes per lane).  Only an exact match joins the class, so fingerprint and bucket
// collisions can cost sharing, never correctness.  Representatives and followers are compacted into two lists.
__device__ __forceinline__ void chunk_load(const uint32_t* sp, int nw, int lane, uint4 (&v)[4]) {
    const bool al = (reinterpret_cast<uintptr_t>(sp) & 15u) == 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int w0 = (c * 32 + lane) * 4;
        v[c] = make_uint4(0, 0, 0, 0);
        if (w0 < nw) {
            if (al) v[c] = __ldg(reinterpret_cast<const uint4*>(sp + w0));
            else { v[c].x = __ldg(sp + w0); v[c].y = __ldg(sp + w0 + 1); v[c].z = __ldg(sp + w0 + 2); v[c].w = __ldg(sp + w0 + 3); }
        }
    }
}

constexpr int kGroupTile = 32;           // live prompts a warp of kernel G takes at a time (their chunks stream through the warp one after the other)
constexpr int kGroupRing = 4;            // chunk slots per warp: one being examined, two in flight, the anchor (deeper rings cost occupancy)
struct GroupSmem {
    uint4 ring[kGroupThreads / 32][kGroupRing][4][32];                       // 64 KB
};

template <int BS>
__global__ void __launch_bounds__(kGroupThreads, 3)
group_round_kernel(const TableView t, const ScoreArgs a, const RoundBufs rb, const int cur, const int round, const int dedup, const int trace) {
    static_assert(BS == 16 && kRoundBlocks == 32, "a chunk is 4 x 32 lanes x 16 bytes");
    extern __shared__ __align__(128) unsigned char smem_raw_g[];
    uint4 (*ring)[4][32] = reinterpret_cast<GroupSmem*>(smem_raw_g)->ring[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const uint64_t l2pol = l2_policy_stream();
    const unsigned int n_act = rb.n_act[cur];
    if (blockIdx.x == 0 && threadIdx.x == 0) { rb.n_hl[0] = 0; rb.n_hl[1] = 0; rb.n_hl[2] = 0; rb.n_hl[3] = 0; }   // lists built by G2
    const unsigned int total_warps = gridDim.x * (kGroupThreads / 32);
    for (unsigned int w = blockIdx.x * (kGroupThreads / 32) + (threadIdx.x >> 5); w * (unsigned)kGroupTile < n_act; w += total_warps) {
        const unsigned int i = w * (unsigned)kGroupTile + lane;
        const bool have = lane < kGroupTile && i < n_act;
        uint32_t p = 0, srcp = kRoleSelf, mdl = a.model0;
        int nb = 0; bool more = false;
        uint64_t hprev = t.init_hash;
        const uint32_t* tp = a.tok;
        if (have) {
            const LiveRec L = live_load(rb.live[cur] + i);
            p = L.p;
            nb = (int)min(L.left, (uint32_t)kRoundBlocks);
            more = L.left > (uint32_t)nb;
            rb.nbr[i] = (uint32_t)nb | (more ? 0x100u : 0u);
            tp = a.tok + L.tok;
            srcp = L.srcp; hprev = L.hstate;
            if (a.model) mdl = a.model[p];
        }
        const bool cls = have && nb > 0 && dedup;
        uint64_t fsum = 0;
        if (cls && round == 0 && a.filter) { const uint64_t* fr = a.filter + (int64_t)p * t.filter_words; for (uint32_t x = 0; x < t.filter_words; ++x) fsum = (fsum ^ fr[x]) * 0x9E3779B97F4A7C15ull; }
        // The chunks stream through a 3-slot ring (one being examined, two in flight); a fourth slot keeps the ANCHOR: the chunk
        // of the class the list is currently running through (the list is sorted by prefix, so class-mates are neighbours).
        // A chunk equal to the anchor (and with the same walk state, model, filter, length) is a member of the anchor's
        // class: nothing else to do for it.  A chunk that starts like the anchor but differs is a prompt leaving that class
        // inside the chunk: it goes through the election like any new chunk, and remembers (class, shared blocks) as an exact
        // hint for kernel G2.  A chunk unrelated to the anchor -- or one that differs from an anchor nobody has joined yet --
        // becomes the anchor.
        uint32_t f0 = 0, f1 = 0;
        bool eqanch = false;                          // member of the class of lane `alane`
        int alane = -1;
        int dh = 0, hlane = -1;                       // hint: shares dh leading blocks with the chunk of lane hlane
        int anchor = -1, members = 0;                 // warp-uniform: the anchor's lane, prompts that matched it so far
        uint32_t todo = __ballot_sync(0xffffffffu, cls);
        if (trace && lane == 0 && todo) atomicAdd(&rb.stat[0], (unsigned int)__popc(todo));
        auto issue = [&](int slot, int qi) {
            if (qi >= 0) {
                const uint32_t* sp = reinterpret_cast<const uint32_t*>(__shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)tp, qi));
                const int nw = __shfl_sync(0xffffffffu, nb, qi) * BS;
                const bool al = (reinterpret_cast<uintptr_t>(sp) & 15u) == 0;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int w0 = (c * 32 + lane) * 4;
                    uint4* dst = &ring[slot][c][lane];
                    if (w0 < nw) {
                        if (al) cp_async_16_stream(smem_addr(dst), sp + w0, l2pol);
                        else *dst = make_uint4(__ldg(sp + w0), __ldg(sp + w0 + 1), __ldg(sp + w0 + 2), __ldg(sp + w0 + 3));
                    } else *dst = make_uint4(0, 0, 0, 0);
                }
            }
            cp_async_commit();
        };
        constexpr int RS = kGroupRing - 1;            // rotating slots; slot RS holds the anchor
        constexpr int PD = RS - 1;                    // chunks in flight
        uint32_t pend = todo;
        int issued = 0;
#pragma unroll
        for (int u = 0; u < PD; ++u) {
            const int qi = pend ? __ffs(pend) - 1 : -1;
            pend &= pend - 1;
            issue(issued % RS, qi); ++issued;
        }
        int ord = 0;
        while (todo) {
            const int q = __ffs(todo) - 1;
            todo &= todo - 1;
            {
                const int qi = pend ? __ffs(pend) - 1 : -1;
                pend &= pend - 1;
                issue(issued % RS, qi); ++issued;
            }
            cp_async_wait<PD>();
            uint4 v[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) v[c] = ring[ord % RS][c][lane];
            bool same = false, compat = false;
            int fbc = 0;
            if (anchor >= 0) {
                const int nb_q = __shfl_sync(0xffffffffu, nb, q), nb_a = __shfl_sync(0xffffffffu, nb, anchor);
                compat = __shfl_sync(0xffffffffu, mdl, q) == __shfl_sync(0xffffffffu, mdl, anchor) &&
                         __shfl_sync(0xffffffffu, srcp, q) == __shfl_sync(0xffffffffu, srcp, anchor) &&
                         __shfl_sync(0xffffffffu, hprev, q) == __shfl_sync(0xffffffffu, hprev, anchor) &&
                         __shfl_sync(0xffffffffu, fsum, q) == __shfl_sync(0xffffffffu, fsum, anchor);
                if (compat && round == 0 && a.filter) {           // equal filter fingerprints: compare the rows themselves
                    const uint32_t pq = __shfl_sync(0xffffffffu, p, q), pa = __shfl_sync(0xffffffffu, p, anchor);
                    bool eqr = true;
                    for (uint32_t x = lane; x < t.filter_words; x += 32) eqr = eqr && a.filter[(int64_t)pq * t.filter_words + x] == a.filter[(int64_t)pa * t.filter_words + x];
                    compat = __all_sync(0xffffffffu, eqr);
                }
                if (compat) {
                    int fb = 32;                                  // first block in which this lane's pieces differ
#pragma unroll
                    for (int c = 3; c >= 0; --c) {
                        const uint4 u = ring[RS][c][lane];
                        if (((v[c].x ^ u.x) | (v[c].y ^ u.y) | (v[c].z ^ u.z) | (v[c].w ^ u.w)) != 0u) fb = c * 8 + (lane >> 2);
                    }
                    fb = __reduce_min_sync(0xffffffffu, fb);
                    fbc = min(fb, min(nb_q, nb_a));
                    same = fb == 32 && nb_q == nb_a && __shfl_sync(0xffffffffu, (int)more, q) == __shfl_sync(0xffffffffu, (int)more, anchor);
                }
            }
            if (same) {
                if (lane == q) { eqanch = true; alane = anchor; }
                ++members;
            } else {
                uint32_t a0 = 0, a1 = 0;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const uint32_t w0 = (uint32_t)(c * 32 + lane) * 4u;
                    uint32_t x = (v[c].x ^ (w0 * 0x9E3779B1u + 0x7F4A7C15u)) * 0x85EBCA6Bu; x = (x ^ v[c].y) * 0xC2B2AE35u; x ^= x >> 15;
                    uint32_t y = (v[c].z ^ (w0 * 0x7FEB352Du + 0x165667B1u)) * 0x846CA68Bu; y = (y ^ v[c].w) * 0x9E3779B1u; y ^= y >> 13;
                    a0 ^= x + y; a1 ^= x * 0x27D4EB2Fu ^ y;
                }
                a0 = __reduce_xor_sync(0xffffffffu, a0);
                a1 = __reduce_xor_sync(0xffffffffu, a1);
                if (lane == q) { f0 = a0; f1 = a1; }
                bool take = true;                                // does this chunk become the anchor?
                if (anchor >= 0 && compat && fbc >= 1) {
                    if (members > 0) { take = false; if (lane == q) { dh = fbc; hlane = anchor; } }      // leaves the anchor's class
                    else if (lane == anchor) { dh = fbc; hlane = q; }                                      // ... or the old anchor leaves this one's
                }
                if (take) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) ring[RS][c][lane] = v[c];
                    anchor = q; members = 0;
                }
            }
            ++ord;
        }
        cp_async_wait<0>();
        // election among the prompts that are not members of an anchor's class
        uint32_t cand = kRoleSelf;
        if (cls && !eqanch) {
            const uint64_t key = mix64((((uint64_t)f1 << 32) | f0) ^ (hprev * 0xFF51AFD7ED558CCDull) ^ ((uint64_t)srcp << 17) ^ (uint64_t)(nb | (more ? 64 : 0)) ^
                                       ((uint64_t)mdl * 0xC2B2AE3D27D4EB4Full) ^ fsum);
            cand = atomicCAS(&rb.map[(uint32_t)key & rb.map_mask], kRoleSelf, i);
        }
        // a loser checks everything but the tokens lane-parallel ...
        bool okm = false;
        const uint32_t* lp = a.tok;
        if (cand != kRoleSelf) {
            const LiveRec Lc = live_load(rb.live[cur] + cand);      // (same state source => same position in the prompt)
            const int nbl = (int)min(Lc.left, (uint32_t)kRoundBlocks);
            okm = nbl == nb && (Lc.left > (uint32_t)nbl) == more && (a.model ? a.model[Lc.p] : a.model0) == mdl;
            if (round > 0) okm = okm && Lc.srcp == srcp && Lc.hstate == hprev;
            else if (a.filter) {
                const uint64_t* fa = a.filter + (int64_t)p * t.filter_words; const uint64_t* fb = a.filter + (int64_t)Lc.p * t.filter_words;
                for (uint32_t x = 0; x < t.filter_words; ++x) okm = okm && fa[x] == fb[x];
            }
            lp = a.tok + Lc.tok;
        }
        // ... and the tokens warp-wide
        bool shared = false;
        uint32_t vm = __ballot_sync(0xffffffffu, okm);
        if (trace && lane == 0 && vm) atomicAdd(&rb.stat[1], (unsigned int)__popc(vm));
        while (vm) {
            const int l = __ffs(vm) - 1; vm &= vm - 1;
            const uint32_t* s1 = reinterpret_cast<const uint32_t*>(__shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)tp, l));
            const uint32_t* s2 = reinterpret_cast<const uint32_t*>(__shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)lp, l));
            const int nw = __shfl_sync(0xffffffffu, nb, l) * BS;
            uint4 v[4], vn[4];
            chunk_load(s1, nw, lane, v);
            chunk_load(s2, nw, lane, vn);
            uint32_t d = 0;
#pragma unroll
            for (int c = 0; c < 4; ++c) d |= (v[c].x ^ vn[c].x) | (v[c].y ^ vn[c].y) | (v[c].z ^ vn[c].z) | (v[c].w ^ vn[c].w);
            const bool same = __all_sync(0xffffffffu, d == 0u);
            if (lane == l) shared = same;
        }
        // members take the outcome of their anchor (which went through the election); hints are resolved the same way
        {
            const int al_ = eqanch ? alane : lane;
            const uint32_t cand_h = __shfl_sync(0xffffffffu, cand, al_);
            const int shared_h = __shfl_sync(0xffffffffu, (int)shared, al_);
            const unsigned int i_h = __shfl_sync(0xffffffffu, i, al_);
            if (eqanch) { shared = true; cand = shared_h ? cand_h : i_h; }
        }
        if (have) { rb.role[i] = shared ? cand : kRoleSelf; if (shared) rb.nfol[cand] = 1; }
        // Every member of a class tells the prompts that shared its state last round (same src) where the class lives:
        // kernel G2 points the ones that stayed alone at this class.  (grp is by the state owner's slot in this round's list.)
        if (shared && round > 0) rb.grp[rb.nmap[rb.live[cur][i].src]] = cand;
        {
            const int hl_ = hlane >= 0 ? hlane : lane;
            const uint32_t cand_h = __shfl_sync(0xffffffffu, cand, hl_);
            const int shared_h = __shfl_sync(0xffffffffu, (int)shared, hl_);
            const unsigned int i_h = __shfl_sync(0xffffffffu, i, hl_);
            if (have) {
                const bool hint = cls && !shared && hlane >= 0 && dh > 0;
                rb.anch[i] = hint ? (shared_h ? cand_h : i_h) : kRoleSelf;
                rb.dmin[i] = (uint8_t)(hint ? (dh | 0x80) : 0);     // exact: measured against a chunk of that very class
            }
        }
    }
}

// ---- kernel G2: partial followers, and the three lists -----------------------------------------------------------
// A prompt that ended up alone in its class and that nobody follows looks for a class whose chunk starts like its own:
// the class that prompts with its state joined this round (grp), else last round's representative itself, else -- round
// 0, or nothing better -- the class of a list neighbour (kernel G's hint).  The shared prefix is then measured exactly,
// token by token against that class's chunk (warp-wide), so that the prompt detaches at the right block.
template <int BS>
__global__ void __launch_bounds__(256)
group_lists_kernel(const TableView t, const ScoreArgs a, const RoundBufs rb, const int cur, const int round, const int partial, const int trace) {
    const int lane = threadIdx.x & 31;
    const unsigned int n_act = rb.n_act[cur];
    const unsigned int total_warps = gridDim.x * (blockDim.x / 32);
    for (unsigned int w = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); w * 32u < n_act; w += total_warps) {
        const unsigned int i = w * 32u + lane;
        const bool have = i < n_act;
        int kind = -1;                               // 0 representative / alone, 1 follower, 2 partial follower
        uint32_t target = kRoleSelf;
        const uint32_t* tp = a.tok; const uint32_t* rp = a.tok;
        int nbc = 0;                                 // blocks both chunks have
        int dknown = 0;
        if (have) {
            kind = rb.role[i] == kRoleSelf ? 0 : 1;
            const int nb = (int)(rb.nbr[i] & 63u);
            if (kind == 0 && partial && nb > 0 && !rb.nfol[i]) {
                const LiveRec L = live_load(rb.live[cur] + i);
                // (Last round's representatives never become partial followers: the prompts that shared their state may be
                //  attaching to them right now.)
                bool allow = true;
                if (round > 0) {
                    allow = L.srcp != L.p;
                    if (allow) { const uint32_t rs = rb.nmap[L.src]; const uint32_t g = rb.grp[rs]; target = g != kRoleSelf ? g : rs; }
                }
                const uint32_t hint = rb.dmin[i];                  // kernel G: shared blocks with a neighbour's class | 0x80 if exact
                // a hinted class is only safe to lean on if it has followers (then its representative stays one)
                if (allow && target == kRoleSelf && (hint & 0x7fu) > 0 && rb.anch[i] != kRoleSelf && rb.nfol[rb.anch[i]]) target = rb.anch[i];
                if (target != kRoleSelf && rb.role[target] != kRoleSelf) target = rb.role[target];   // someone with the same chunk represents it
                if (target == i) target = kRoleSelf;
                if (target != kRoleSelf) {
                    const LiveRec Lt = live_load(rb.live[cur] + target);
                    nbc = min(nb, (int)min(Lt.left, (uint32_t)kRoundBlocks));
                    tp = a.tok + L.tok; rp = a.tok + Lt.tok;
                    // same walk state, model and filter as the class?  (grp / src: by construction; the neighbour hint: checked by kernel G)
                    // (same state source => same position in the prompt, so the two chunks start at the same block)
                    if (round > 0 && !(Lt.srcp == L.srcp && Lt.hstate == L.hstate)) nbc = 0;
                    // kernel G compared this prompt with a member of exactly this class already: no need to read the chunks again
                    if (nbc > 0 && (hint & 0x80u) && rb.anch[i] == target) { dknown = min((int)(hint & 0x7fu), nbc); nbc = 0; }
                }
            }
        }
        int dshare = dknown;
        uint32_t wm = __ballot_sync(0xffffffffu, nbc > 0);
        if (trace && lane == 0 && wm) atomicAdd(&rb.stat[2], (unsigned int)__popc(wm));
        while (wm) {
            const int l = __ffs(wm) - 1; wm &= wm - 1;
            const uint32_t* s1 = reinterpret_cast<const uint32_t*>(__shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)tp, l));
            const uint32_t* s2 = reinterpret_cast<const uint32_t*>(__shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)rp, l));
            const int nw = __shfl_sync(0xffffffffu, nbc, l) * BS;
            uint4 v[4], vn[4];
            chunk_load(s1, nw, lane, v);
            chunk_load(s2, nw, lane, vn);
            int fb = 32;
#pragma unroll
            for (int c = 3; c >= 0; --c)
                if (((v[c].x ^ vn[c].x) | (v[c].y ^ vn[c].y) | (v[c].z ^ vn[c].z) | (v[c].w ^ vn[c].w)) != 0u) fb = c * 8 + (lane >> 2);
            fb = __reduce_min_sync(0xffffffffu, fb);
            if (lane == l) dshare = min(fb, nw / BS);
        }
        if (dshare > 0) { kind = 2; rb.anch[i] = target; rb.dmin[i] = (uint8_t)dshare; rb.need_snap[target] = 1; }
        const uint32_t m0 = __ballot_sync(0xffffffffu, kind == 0), m1 = __ballot_sync(0xffffffffu, kind == 1), m2 = __ballot_sync(0xffffffffu, kind == 2);
        unsigned int b0 = 0, b1 = 0, b2 = 0;
        if (lane == 0) {
            if (m0) b0 = atomicAdd(&rb.n_hl[0], (unsigned int)__popc(m0));
            if (m1) b1 = atomicAdd(&rb.n_hl[1], (unsigned int)__popc(m1));
            if (m2) b2 = atomicAdd(&rb.n_hl[2], (unsigned int)__popc(m2));
        }
        b0 = __shfl_sync(0xffffffffu, b0, 0); b1 = __shfl_sync(0xffffffffu, b1, 0); b2 = __shfl_sync(0xffffffffu, b2, 0);
        const uint32_t below = (1u << lane) - 1u;
        if (kind == 0) {
            const unsigned int ap = b0 + __popc(m0 & below);
            rb.hl[ap] = i; rb.apos[i] = ap;
            rb.rec[ap] = make_uint4(rb.live[cur][i].p, i, rb.nbr[i], rb.live[cur][i].src);
        } else if (kind == 1) rb.fl[b1 + __popc(m1 & below)] = make_uint2(i, rb.role[i]);
        else if (kind == 2) rb.drec[b2 + __popc(m2 & below)] = make_uint4(i, target, ((uint32_t)dshare << 16) | rb.nbr[i], rb.live[cur][i].p);
    }
}

// ---- kernel H ---------------------------------------------------------------------------------
template <int BS>
__global__ void __launch_bounds__(kHashThreads, 3)
hash_round_kernel(const TableView t, const ScoreArgs a, const RoundBufs rb, const int cur, const int round, const int trace) {
    static_assert(BS == 16, "staging pattern is written for 16-token blocks");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using SM = HashSmem<BS>;
    SM& sm = *reinterpret_cast<SM*>(smem_raw);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const unsigned int n_hl = rb.n_hl[0];                                 // representatives this round (kernel G)
    const uint64_t l2pol = l2_policy_stream();
    {   // the election map, grp and nfol are dead until the next round's kernel G: clear them here instead of three memsets
        uint4* m4 = reinterpret_cast<uint4*>(rb.map);
        const size_t nm = ((size_t)rb.map_mask + 1 + rb.part_size) / 4;   // map + grp are contiguous; sizes are multiples of 4 words
        for (size_t x = blockIdx.x * (size_t)blockDim.x + threadIdx.x; x < nm; x += (size_t)gridDim.x * blockDim.x) m4[x] = make_uint4(~0u, ~0u, ~0u, ~0u);
        uint32_t* f4 = reinterpret_cast<uint32_t*>(rb.nfol);
        for (size_t x = blockIdx.x * (size_t)blockDim.x + threadIdx.x; x < rb.part_size / 4; x += (size_t)gridDim.x * blockDim.x) f4[x] = 0u;
    }
    const unsigned int total_warps = gridDim.x * (blockDim.x / 32);
    for (unsigned int w = blockIdx.x * (blockDim.x / 32) + wid; w * 32u < n_hl; w += total_warps) {
        const unsigned int i = w * 32u + lane;                            // position in the representative list
        const bool have = i < n_hl;
        int nb = 0;                                                      // blocks of this prompt in this round
        const uint32_t* src = nullptr;
        bool aligned = true;
        uint64_t h = 0;
        if (have) {
            const uint32_t li = rb.hl[i];
            const LiveRec L = live_load(rb.live[cur] + li);
            nb = (int)min(L.left, (uint32_t)kRoundBlocks);
            src = a.tok + L.tok;
            aligned = (reinterpret_cast<uintptr_t>(src) & 15u) == 0;
            h = L.hstate;                                                // (round 0: the initial hash)
            // the first half of its record for the next round, in case it continues: past this chunk, walk state in its own
            // slot (kernel P writes the other half).  Nothing reads a representative's position after this kernel.
            reinterpret_cast<uint4*>(rb.live[cur] + li)[0] = make_uint4((uint32_t)(uint64_t)(L.tok + (int64_t)nb * BS),
                                                                        (uint32_t)((uint64_t)(L.tok + (int64_t)nb * BS) >> 32), L.left - (uint32_t)nb, li);
        }
        const int nb_max = __reduce_max_sync(0xffffffffu, nb);
        if (trace) { const unsigned int nbs = __reduce_add_sync(0xffffffffu, (unsigned int)nb); if (lane == 0 && nbs) atomicAdd(&rb.stat[3], nbs); }
        // stage block c of every lane's prompt: 4 lanes move one prompt's 64 bytes, 8 prompts per copy instruction
        auto stage = [&](int s, int c) {
            const bool issue = c < nb;
            const unsigned long long srcv = (issue && aligned) ? (unsigned long long)(uintptr_t)(src + (size_t)c * BS) : 0ull;
            __syncwarp();
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int q = 8 * r + lane / 4;
                const unsigned long long sp = __shfl_sync(0xffffffffu, srcv, q);
                if (sp) cp_async_16_stream(smem_addr(&sm.tok[wid][s][q * SM::kRow + (lane % 4) * 16]), reinterpret_cast<const char*>(sp) + (lane % 4) * 16, l2pol);
            }
            cp_async_commit();
            if (issue && !aligned) {
                uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.tok[wid][s][lane * SM::kRow]);
                const uint32_t* g = src + (size_t)c * BS;
                for (int j = 0; j < BS; ++j) dst[j] = __ldg(g + j);
            }
        };
#pragma unroll
        for (int c = 0; c < kHashStages - 1; ++c) stage(c, c);
        for (int c = 0; c < nb_max; ++c) {
            stage((c + kHashStages - 1) % kHashStages, c + kHashStages - 1);
            cp_async_wait<kHashStages - 1>();
            __syncwarp();
            const uint64_t key = hash_row16(h, &sm.tok[wid][c % kHashStages][lane * SM::kRow]);
            if (c < nb) { h = key; rb.keys[(size_t)c * a.n_prompts + i] = key; }
        }
        cp_async_wait<0>();
        __syncwarp();
    }
}

// ---- kernel P: warp per representative ------------------------------------------------------------------------
// With prefix classes the representatives of a round are few (one per distinct prefix), so a lane-per-prompt walk
// (kernels_rounds_plain.cuh: 32 dependent iterations of divergent code per warp) would leave the machine idle: its time
// is a latency chain that does not shrink with the list.  Here a warp takes one representative: the 32 lanes probe the
// round's 32 keys at once (one DRAM latency for the whole chunk), a ballot finds the first miss, and the blocks before
// it are scored in order with lane q owning pod q of the first block (<= 10 pods), the block's entries broadcast by
// shuffle.  Same arithmetic in the same order as everywhere else: max weight per pod per block, added in block order.
// kClock: CLOCK marking of the blocks walked (a template parameter: the default instance keeps its register allocation)
template <bool kClock>
__global__ void __launch_bounds__(256)
walk_round_kernel(const TableView t, const ScoreArgs a, const RoundBufs rb, const int cur, const int round) {
    const int lane = threadIdx.x & 31;
    const unsigned int n_a = rb.n_hl[0];
    const uint64_t l2pol = l2_policy_stream();
    const size_t kstride = (size_t)a.n_prompts;
    const bool peer = t.shard_bits != 0;
    const PromptState* pst_prev = rb.pst[(round & 1) ^ 1];
    PromptState* pst_cur = rb.pst[round & 1];
    const unsigned int total_warps = gridDim.x * (blockDim.x / 32);
    for (unsigned int i = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); i < n_a; i += total_warps) {
        const uint4 rc = __ldg(rb.rec + i);
        const uint64_t key = rb.keys[(size_t)lane * kstride + i];   // lanes >= nb read a stale key and ignore it
        const unsigned int li = rc.y;
        const uint32_t p = rc.x;
        const uint32_t meta = rc.z;
        const int nb = (int)(meta & 63u);
        const bool has_more = (meta >> 8) & 1u;
        const uint32_t mdl = a.model ? a.model[p] : a.model0;
        const bool snapf = rb.need_snap[li];
        WarpWalk ws;
        if (round > 0) ws.load(pst_prev[rc.w], lane);       // by last round's live slot
        // probe: lane j looks up block j's key
        SlotPat mine = {};
        bool hit = false;
        uint64_t hslot = 0;                                  // CLOCK: slot of this lane's hit
        if (lane < nb) {
            HomeProbe pr;
            uint4 A, B;
            hit = pr.find(t, key, mdl, peer, A, B);
            if (hit) { mine = SlotPat::of(A, B); if (kClock) hslot = pr.hit_slot(key, mdl); }
        }
        const uint32_t hm_ = __ballot_sync(0xffffffffu, hit);
        const int nhit = hm_ == 0xffffffffu ? 32 : __ffs(~hm_) - 1;   // consecutive hits from block 0 (lanes >= nb never hit)
        const uint32_t samemask = ws.same_mask(lane, mine, round > 0, nhit);
        // snapshot of the walk state at every run start
        const int j = ws.walk<true>(t, lane, mine, nhit, samemask, round == 0, a.filter, p, [&](int b) {
            if (!snapf) return;
            const size_t sb = (size_t)i * kRoundBlocks + b;
            if ((uint32_t)lane < ws.k) { rb.snap_sc[sb * kMaxEnt + lane] = ws.sc; rb.snap_bt[sb * kMaxEnt + lane] = (uint8_t)ws.bt; }
            if (lane == 0) rb.snap_alive[sb] = (uint16_t)ws.alive;
        });
        // CLOCK: the representative's walk marks the blocks it looked at for its whole class (class-mates share model, filter,
        // walk state and these keys; a partial follower marks the blocks it walks alone in kernel D)
        if (kClock) WarpWalk::mark_walked(t, lane, j, hit, hslot);
        const uint32_t nwalk = (uint32_t)(j > 0 && !ws.alive ? j - 1 : j);      // blocks after which the walk was still alive
        if (snapf) {                                           // block -> first block of its run
            const uint32_t starts = ~samemask & ((2u << lane) - 1u);
            rb.snap_run[(size_t)i * kRoundBlocks + lane] = (uint8_t)(starts ? 31 - __clz(starts) : 0);
        }
        const bool done = nb == 0 || nhit < nb || !ws.alive;   // no block, a block of the round is not in the index, or no pod left
        const bool more = !done && has_more;
        PromptState& ps = pst_cur[li];
        ws.store_lane(ps, lane);
        if (lane == 0) {
            ws.store_uniform(ps);
            rb.fate[li] = more ? kFateMore : kFateDone; rb.nwalk[i] = (uint8_t)nwalk;
        }
        if (more) {           // chain state for the next round: key of the round's last block; its own walk state from here
            if (lane == nb - 1) reinterpret_cast<uint4*>(rb.live[cur] + li)[1] = make_uint4((uint32_t)key, (uint32_t)(key >> 32), p, p);
        } else warp_write_row(t, a, p, ws.k, ws.pod, ws.sc, round > 0 || nb > 0, l2pol);
        __syncwarp();
    }
}

// ---- kernel R: followers take their representative's outcome --------------------------------------------------
// Lane per follower.  Representative continues: so does the follower, with the representative's chain state, and its
// walk state stays where the representative left it (src: the representative's slot).  Representative finished: same pods, same scores -- the warp
// writes the follower's result from the representative's final state.  Either way the follower's slot takes the
// representative's fate, for kernel C.
__device__ __forceinline__ void resolve_round(const TableView& t, const ScoreArgs& a, const RoundBufs& rb, const int cur, const int round,
                                              const unsigned int bid, const unsigned int nbl, const uint64_t l2pol) {
    const int lane = threadIdx.x & 31;
    {   // kernel P is done with need_snap: clear it for the next round
        uint32_t* f4 = reinterpret_cast<uint32_t*>(rb.need_snap);
        for (size_t x = bid * (size_t)blockDim.x + threadIdx.x; x < rb.part_size / 4; x += (size_t)nbl * blockDim.x) f4[x] = 0u;
    }
    const unsigned int n_fl = rb.n_hl[1];
    const PromptState* pst_cur = rb.pst[round & 1];
    const unsigned int total_warps = nbl * (blockDim.x / 32);
    for (unsigned int w = bid * (blockDim.x / 32) + (threadIdx.x >> 5); w * 32u < n_fl; w += total_warps) {
        const unsigned int f = w * 32u + lane;
        const bool have = f < n_fl;
        uint32_t p = 0, lj = 0; uint8_t ft = 0;
        if (have) {
            const uint2 fr = rb.fl[f];
            const unsigned int li = fr.x;
            lj = fr.y;
            ft = rb.fate[lj];
            const LiveRec L = live_load(rb.live[cur] + li);
            const uint4 rs = __ldg(reinterpret_cast<const uint4*>(rb.live[cur] + lj) + 1);    // the representative's {hstate, srcp} as kernel P left them
            p = L.p;
            rb.fate[li] = ft;
            if (ft == kFateMore) {        // same chunk length as the representative: advance by the same blocks
                const uint32_t nb = rb.nbr[li] & 63u;
                live_store(rb.live[cur] + li, L.tok + (int64_t)nb * t.block_size, L.left - nb, lj, ((uint64_t)rs.y << 32) | rs.x, rs.z, p);
            }
        }
        const bool more = have && ft == kFateMore;
        uint32_t dm = __ballot_sync(0xffffffffu, have && !more);
        while (dm) {
            const int l = __ffs(dm) - 1; dm &= dm - 1;
            const uint32_t pp = __shfl_sync(0xffffffffu, p, l);
            const PromptState& ps = pst_cur[__shfl_sync(0xffffffffu, lj, l)];
            const uint32_t pk = ps.k;
            const bool in = (uint32_t)lane < pk;
            warp_write_row(t, a, pp, pk, in ? ps.pod[lane] : 0u, in ? ps.sc[lane] : 0.0, true, l2pol);   // followers always have a block in the round
        }
        __syncwarp();
    }
}

// ---- kernel D: partial followers leave their class inside the chunk ----------------------------------------------
// Lane per partial follower.  It shares the first d blocks of the chunk with representative R (same walk state before,
// same tokens): if R's walk ended inside those blocks, so does this one, with R's result.  Otherwise it resumes from
// R's snapshot after block d-1 and R's key of that block, and walks the rest of its chunk by itself -- hash one block,
// probe it, score it -- which normally ends at the first block it does not share.
__device__ __forceinline__ uint64_t hash_block16(uint64_t parent, const uint32_t* __restrict__ tk) {
    Fnv f;
    f.begin_block(parent, 16);
    if ((reinterpret_cast<uintptr_t>(tk) & 15u) == 0) {
        const uint4* t4 = reinterpret_cast<const uint4*>(tk);
#pragma unroll
        for (int c = 0; c < 4; ++c) { const uint4 v = __ldg(t4 + c); f.token(v.x); f.token(v.y); f.token(v.z); f.token(v.w); }
    } else {
#pragma unroll
        for (int c = 0; c < 16; ++c) f.token(__ldg(tk + c));
    }
    return f.end_block();
}
constexpr int kDetachBlocks = 3;         // blocks a partial follower walks alone inside the round before it is re-queued
struct DetachWarp { double sc[kMaxEnt][32]; uint16_t pod[kMaxEnt][32]; };     // per warp (dynamic shared memory: warps of the CTA x this)
template <int BS>
__device__ __forceinline__ void detach_round(const TableView& t, const ScoreArgs& a, const RoundBufs& rb, const int cur, const int round, const int trace, DetachWarp* smw,
                                             const unsigned int bid, const unsigned int nbl, const uint64_t l2pol) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    DetachWarp& sm = smw[wid];
    const unsigned int n_dl = rb.n_hl[2];
    const PromptState* pst_rd = rb.pst[round & 1];
    PromptState* pst_cur = rb.pst[round & 1];
    const size_t kstride = (size_t)a.n_prompts;
    const bool peer = t.shard_bits != 0;
    const unsigned int total_warps = nbl * (blockDim.x / 32);
    for (unsigned int w = bid * (blockDim.x / 32) + wid; w * 32u < n_dl; w += total_warps) {
        const unsigned int f = w * 32u + lane;
        const bool have = f < n_dl;
        uint32_t p = 0, meta = 0, li = 0;
        bool more = false;
        ScoreState s; s.k = 0; s.alive = 0;
        uint64_t h = 0;
        uint32_t adv = 0;
        uint4 pos0 = make_uint4(0, 0, 0, 0);                     // its LiveRec's {tok, left, src}
        if (have) {
            const uint4 rc = __ldg(rb.drec + f);
            li = rc.x; p = rc.w; meta = rc.z & 0xffffu;
            const unsigned int lr = rc.y;
            const int d = (int)(rc.z >> 16);
            const unsigned int ar = rb.apos[lr];
            const int nb = (int)(meta & 63u);
            const PromptState& R = pst_rd[lr];
            s.k = R.k;
            for (uint32_t q = 0; q < s.k; ++q) s.pod[q] = R.pod[q];
            if ((int)rb.nwalk[ar] < d) {                       // R stopped inside the shared blocks: same stop, same scores
                for (uint32_t q = 0; q < s.k; ++q) s.sc[q] = R.sc[q];
            } else {
                const int j0 = rb.snap_run[(size_t)ar * kRoundBlocks + (size_t)(d - 1)];
                const size_t sj = (size_t)ar * kRoundBlocks + (size_t)j0;
                s.alive = rb.snap_alive[sj];
                for (uint32_t q = 0; q < s.k; ++q) {
                    double v = rb.snap_sc[sj * kMaxEnt + q];
                    if (j0 < d - 1 && ((s.alive >> q) & 1u)) {          // later blocks of the run: the same addend again, in order
                        const uint32_t bt = rb.snap_bt[sj * kMaxEnt + q];
                        v = run_add(v, bt == 0xffu ? 0.0 : t.weight[bt & 15u], d - 1 - j0);
                    }
                    s.sc[q] = v;
                }
                h = rb.keys[(size_t)(d - 1) * kstride + ar];
                const uint32_t mdl = a.model ? a.model[p] : a.model0;
                pos0 = __ldg(reinterpret_cast<const uint4*>(rb.live[cur] + li));
                const uint32_t* tk = a.tok + (int64_t)(((uint64_t)pos0.y << 32) | pos0.x);
                bool walking = true;
                const int bend = min(nb, d + kDetachBlocks);          // walk at most this far alone; the rest waits for the next round
                uint64_t hk = d < nb ? hash_block16(h, tk + (size_t)d * BS) : 0ull;       // key of the first block of its own
                int b = d;
                for (; b < bend; ++b) {
                    if (trace) atomicAdd(&rb.n_hl[3], 1u);
                    HomeProbe pr;
                    pr.issue(t, hk, mdl, peer);
                    // the next key does not depend on the probe: hash it while the probe is in flight
                    const uint64_t hn = b + 1 < nb ? hash_block16(hk, tk + (size_t)(b + 1) * BS) : 0ull;
                    SlotWords sw;
                    if (!pr.resolve(t, hk, mdl, peer, sw.a, sw.b)) { walking = false; break; }
                    if (t.req_ref) ref_touch(t.req_ref, pr.hit_slot(hk, mdl));
                    s.next(t, sw);
                    if (!s.alive) { walking = false; break; }
                    h = hk; hk = hn;
                }
                more = walking && (b < nb || ((meta >> 8) & 1u));
                adv = (uint32_t)b;
            }
        }
        // continue on its own next round, or write the result
        if (have) rb.fate[li] = more ? kFateMore : kFateDone;
        if (more) {
            live_store(rb.live[cur] + li, (int64_t)(((uint64_t)pos0.y << 32) | pos0.x) + (int64_t)adv * BS, pos0.z - adv, li, h, p, p);
            PromptState& ps = pst_cur[li];
            ps.k = (uint8_t)s.k; ps.alive = (uint16_t)s.alive;
            ps.pat[5] = 0xffffffffu;                        // no cached slot pattern: the next block is scored the long way
            for (uint32_t q = 0; q < s.k; ++q) { ps.sc[q] = s.sc[q]; ps.pod[q] = s.pod[q]; ps.bt[q] = 0xffu; }
        }
        for (uint32_t q = 0; q < s.k; ++q) { sm.sc[q][lane] = s.sc[q]; sm.pod[q][lane] = s.pod[q]; }
        __syncwarp();
        uint32_t dm = __ballot_sync(0xffffffffu, have && !more);
        while (dm) {
            const int l = __ffs(dm) - 1; dm &= dm - 1;
            const uint32_t pp = __shfl_sync(0xffffffffu, p, l);
            const uint32_t pk = __shfl_sync(0xffffffffu, s.k, l);
            const bool in = (uint32_t)lane < pk;
            warp_write_row(t, a, pp, pk, in ? sm.pod[lane][l] : 0u, in ? sm.sc[lane][l] : 0.0, true, l2pol);
        }
        __syncwarp();
    }
}

// Kernels R and D in one launch (they work on different lists and neither reads what the other writes).
template <int BS>
__global__ void __launch_bounds__(256, 4)       // (4: 64 registers, what it used anyway; left free, ptxas picks 48 and spills)
finish_round_kernel(const TableView t, const ScoreArgs a, const RoundBufs rb, const int cur, const int round, const int detach, const int trace) {
    extern __shared__ __align__(16) unsigned char smem_raw_f[];
    DetachWarp* sm = reinterpret_cast<DetachWarp*>(smem_raw_f);
    const uint64_t l2pol = l2_policy_stream();
    if (!detach) { resolve_round(t, a, rb, cur, round, blockIdx.x, gridDim.x, l2pol); return; }
    // odd CTAs take the followers, even CTAs the partial followers: the two latency chains run side by side
    const unsigned int half = gridDim.x / 2;
    if (gridDim.x < 2) { resolve_round(t, a, rb, cur, round, 0, 1, l2pol); detach_round<BS>(t, a, rb, cur, round, trace, sm, 0, 1, l2pol); }
    else if (blockIdx.x & 1) { if (blockIdx.x / 2 < half) resolve_round(t, a, rb, cur, round, blockIdx.x / 2, half, l2pol); }
    else detach_round<BS>(t, a, rb, cur, round, trace, sm, blockIdx.x / 2, (gridDim.x + 1) / 2, l2pol);
}

// ---- kernel C: next round's live list --------------------------------------------------------------------------
// The prompts whose fate is kFateMore, in the order of this round's list.  A prompt that leaves never comes back, so a
// stable compaction keeps the round-0 order (sorted by prefix) in every round: class-mates stay list neighbours, and kernel
// G's anchor takes them without the election and its second read of two chunks.  One pass: a CTA counts its tile, publishes
// the count, adds up its predecessors' published counts (decoupled look-back) and writes its prompts from there.  A tile's
// status word carries round + 1 in its upper half, so a word of an earlier round of the batch reads as not yet published.
// Each continuing slot's LiveRec is copied to its place in the next list, and nmap records where it went.
constexpr int kCompactThreads = 256;
constexpr int kCompactItems = 8;                           // consecutive live slots per thread
constexpr int kCompactTile = kCompactThreads * kCompactItems;
constexpr unsigned long long kScanDone = 1ull << 31;       // the word holds the tile's inclusive prefix, not only its own count

__global__ void __launch_bounds__(kCompactThreads)
compact_round_kernel(const RoundBufs rb, const int cur, const int round) {
    __shared__ unsigned int s_warp[kCompactThreads / 32];
    __shared__ unsigned int s_base;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const unsigned int n_act = rb.n_act[cur];
    const unsigned int tile = blockIdx.x;
    const unsigned int i0 = tile * (unsigned)kCompactTile;
    if (tile > 0 && i0 >= n_act) return;                   // nothing of the list here, and no later tile looks back this far
    const unsigned int s0 = i0 + threadIdx.x * (unsigned)kCompactItems;
    uint32_t m = 0;                                        // bit k: slot s0 + k continues
    if (s0 + kCompactItems <= n_act) {
        const uint2 f = *reinterpret_cast<const uint2*>(rb.fate + s0);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (((f.x >> (8 * k)) & 0xffu) == kFateMore) m |= 1u << k;
            if (((f.y >> (8 * k)) & 0xffu) == kFateMore) m |= 16u << k;
        }
    } else {
        for (int k = 0; k < kCompactItems && s0 + k < n_act; ++k)
            if (rb.fate[s0 + k] == kFateMore) m |= 1u << k;
    }
    // offset of this thread's slots within the tile
    const unsigned int c = __popc(m);
    unsigned int incl = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const unsigned int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    unsigned int wbase = 0, agg = 0;
#pragma unroll
    for (int w = 0; w < kCompactThreads / 32; ++w) { const unsigned int v = s_warp[w]; wbase += w < wid ? v : 0u; agg += v; }
    // offset of the tile within the list
    if (wid == 0) {
        const unsigned long long tag = (unsigned long long)(round + 1) << 32;
        volatile unsigned long long* st = rb.scan;
        if (lane == 0) st[tile] = tag | (tile == 0 ? kScanDone : 0ull) | agg;
        unsigned int excl = 0;
        if (tile > 0) {
            for (int j = (int)tile - 1 - lane;; j -= 32) {          // lane l reads the (l+1)-th nearest predecessor not yet added
                unsigned long long s;
                for (;;) {
                    s = j >= 0 ? st[j] : (tag | kScanDone);         // before tile 0: a prefix of zero
                    if (__all_sync(0xffffffffu, (s & ~0xffffffffull) == tag)) break;
                    __nanosleep(64);
                }
                const uint32_t done = __ballot_sync(0xffffffffu, (s & kScanDone) != 0ull);
                const int last = done ? __ffs(done) - 1 : 31;       // nearest predecessor whose word is a full prefix
                excl += __reduce_add_sync(0xffffffffu, lane <= last ? (unsigned int)(s & (kScanDone - 1)) : 0u);
                if (done) break;
            }
            if (lane == 0) st[tile] = tag | kScanDone | (excl + agg);
        }
        if (lane == 0) s_base = excl;
    }
    __syncthreads();
    unsigned int at = s_base + wbase + incl - c;
    const uint4* lv = reinterpret_cast<const uint4*>(rb.live[cur]);
    uint4* nxt = reinterpret_cast<uint4*>(rb.live[cur ^ 1]);
    while (m) {                                            // the slot's record moves with it
        const int k = __ffs(m) - 1; m &= m - 1;
        const uint4 u = lv[2 * (s0 + k)], v = lv[2 * (s0 + k) + 1];
        nxt[2 * at] = u; nxt[2 * at + 1] = v;
        rb.nmap[s0 + k] = at; ++at;
    }
    if (threadIdx.x == 0 && (n_act == 0 || (n_act - 1) / (unsigned)kCompactTile == tile)) rb.n_act[cur ^ 1] = s_base + agg;
}

// List setup + a 64-bit fingerprint of every prompt's first block.  The batch is then radix-sorted by fingerprint so
// that prompts sharing a prefix sit in neighbouring lanes: their probes are the same 64-byte segments, which the
// load unit merges within a warp and L2 serves across warps.  (Any order gives the same results; this one lets the
// prefix sharing the system exists for -- system prompts, shared documents -- show up as memory locality.)
struct PartSizes { unsigned int n[kMaxParts]; };
__global__ void rounds_init_kernel(const ScoreArgs a, uint32_t block_size, RoundCounters* cnt, uint64_t* fp, uint32_t* idx,
                                   const PartSizes ps) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    unsigned long long nb = 0;
    if (i < a.n_prompts) {
        const int64_t b = a.tok_off[i] - a.tok_base, e = a.tok_off[i + 1] - a.tok_base;
        nb = (unsigned long long)((e - b) / block_size);
        uint64_t f = ~0ull;                                   // prompts without a full block sort last
        if (nb > 0) {
            f = 0x9E3779B97F4A7C15ull;
            const uint32_t* tk = a.tok + b;
            // (independent mixes of token pairs, not a chain: this kernel is one thread per prompt and latency bound)
            const uint32_t nt = block_size < 16u ? block_size : 16u;
            uint64_t g = 0;
            for (uint32_t j = 0; j + 1 < nt; j += 2) g ^= mix64(((uint64_t)__ldg(tk + j + 1) << 32 | __ldg(tk + j)) + 0xC2B2AE3D27D4EB4Full * (j + 1));
            if (nt & 1u) g ^= mix64(__ldg(tk + nt - 1) + 0x165667B19E3779F9ull);
            f = mix64(f ^ g);
            f &= ~(1ull << 63);
        }
        fp[i] = f; idx[i] = (uint32_t)i;
    }
    nb = __reduce_max_sync(0xffffffffu, (unsigned)min(nb, 0xffffffffull));
    if ((threadIdx.x & 31) == 0 && nb) atomicMax(&cnt->max_blocks, nb);
    if (i == 0) for (int q = 0; q < kMaxParts; ++q) { cnt->part[q].n_act[0] = ps.n[q]; cnt->part[q].n_act[1] = 0; }      // live-list lengths per part
}

// Distinct values among the sorted fingerprints (the sort orders by the top 32 bits, so those are compared).
__global__ void count_distinct_prefixes_kernel(const uint64_t* __restrict__ fp_sorted, int64_t n, unsigned long long* out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const bool edge = i < n && (i == 0 || (fp_sorted[i] >> 32) != (fp_sorted[i - 1] >> 32));
    const unsigned int m = __ballot_sync(0xffffffffu, edge);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(out, (unsigned long long)__popc(m));
}

// Round 0's live records, in the sorted order: slot i of the batch-wide list (part q's slots start at its offset) takes
// prompt idx[i].
__global__ void live_init_kernel(const ScoreArgs a, uint32_t block_size, const uint32_t* __restrict__ idx, LiveRec* live, uint64_t init_hash) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= a.n_prompts) return;
    const uint32_t p = idx[i];
    const int64_t b = a.tok_off[p] - a.tok_base, e = a.tok_off[p + 1] - a.tok_base;
    live_store(live + i, b, (uint32_t)max((int64_t)0, (e - b) / block_size), kRoleSelf, init_hash, kRoleSelf, p);
}

inline int rounds_init() {
    if (cudaFuncSetAttribute(hash_round_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HashSmem<16>)) != cudaSuccess) return -1;
    if (cudaFuncSetAttribute(group_round_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GroupSmem)) != cudaSuccess) return -1;
    return 0;
}

}  // namespace kvx
