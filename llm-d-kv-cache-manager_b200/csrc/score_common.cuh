// score_common.cuh -- what every Score() kernel shares: GetPodScores steps 2-4 (pkg/kvcache/indexer.go:141-163) once.
//
//   * the copy / TMA / cache-policy wrappers the staging loops use, and ScoreArgs;
//   * the home-pair probe of Index.Lookup (in_memory.go:105-146): the decision over one fetched slot pair, and for the
//     warp walks a probe that issues its loads and resolves them later;
//   * LongestPrefixScorer.Score (kvblock_scorer.go:108-151) in its three shapes: thread per prompt (ScoreState), lane per
//     prompt over transposed shared-memory columns (LaneCols), and warp per prompt with lane q owning pod q (WarpWalk);
//   * the result row: -1 for every pod, then the prompt's scores, plus the sparse form and has_keys.
// Every path adds the same f64 addends in the same order, so all of them give bit-identical results.
#pragma once
#include <cuda_runtime.h>
#include "table.cuh"

namespace kvx {

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
};

__device__ __forceinline__ bool filter_has(const uint64_t* __restrict__ frow, uint32_t pod) {
    return (frow[pod >> 6] >> (pod & 63)) & 1ull;
}
__device__ __forceinline__ const uint64_t* filter_row(const uint64_t* __restrict__ filter, int64_t i, uint32_t words) {
    if (!filter) return nullptr;
    const uint64_t* r = filter + i * words;
    uint64_t any = 0;
    for (uint32_t w = 0; w < words; ++w) any |= r[w];
    return any ? r : nullptr;      // empty set == all pods (in_memory.go:126)
}

// FNV/CBOR key of one 16-token block staged as a 16-byte aligned 64-byte row in shared memory (the loads interleaved with
// the chain)
__device__ __forceinline__ uint64_t hash_row16(uint64_t h, const unsigned char* rowp) {
    Fnv f;
    f.begin_block(h, 16);
    const uint4* row = reinterpret_cast<const uint4*>(rowp);
    const uint4 v0 = row[0], v1 = row[1];
    f.token(v0.x); f.token(v0.y); f.token(v0.z); f.token(v0.w);
    const uint4 v2 = row[2];
    f.token(v1.x); f.token(v1.y); f.token(v1.z); f.token(v1.w);
    const uint4 v3 = row[3];
    f.token(v2.x); f.token(v2.y); f.token(v2.z); f.token(v2.w);
    f.token(v3.x); f.token(v3.y); f.token(v3.z); f.token(v3.w);
    return f.end_block();
}

// ---- the home-pair probe -------------------------------------------------------------------------------------
__device__ __forceinline__ bool slot_matches(const uint4& a, const uint4& b, uint64_t key, uint32_t mdl) {
    return meta_state(b.w) == kStateFull && a.x == (uint32_t)key && a.y == (uint32_t)(key >> 32) && meta_model(b.w) == mdl;
}
// The decision over one fetched pair (slot 0, then slot 1): true when the pair decides the lookup -- hit, (A, B) the
// matching slot's image, or miss at an EMPTY slot; false when the key may be further on (the caller fetches the next
// pair, 2 slots on).
__device__ __forceinline__ bool pair_decides(const uint4& a0, const uint4& b0, const uint4& a1, const uint4& b1, uint64_t key, uint32_t mdl,
                                             uint4& A, uint4& B, bool& hit) {
    A = a0; B = b0;
    hit = slot_matches(A, B, key, mdl);
    if (!hit && meta_state(B.w) != kStateEmpty) { A = a1; B = b1; hit = slot_matches(A, B, key, mdl); }
    return hit || meta_state(B.w) == kStateEmpty;
}
// CLOCK mode (t.req_ref set): the slot of a hit that the pair at `slot` decided -- slot 0 if it holds the key, else slot 1
// -- is marked as referenced.  The Score() kernels mark exactly the blocks their walk looks at: block 0 up to and including
// the block that empties the active pod set, never a block fetched ahead of the walk's end.  One uniform branch on the
// pointer; default handles skip it.
__device__ __forceinline__ uint64_t pair_hit_slot(uint64_t slot, const uint4& a0, const uint4& b0, uint64_t key, uint32_t mdl) {
    return slot + (slot_matches(a0, b0, key, mdl) ? 0u : 1u);
}
__device__ __forceinline__ void mark_hit(const TableView& t, uint64_t slot, const uint4& a0, const uint4& b0, uint64_t key, uint32_t mdl) {
    if (t.req_ref) ref_touch(t.req_ref, pair_hit_slot(slot, a0, b0, key, mdl));
}
__device__ __forceinline__ void ld_slot_pair(const ReqSlot* s, bool peer, uint4& a0, uint4& b0, uint4& a1, uint4& b1) {
    ld_slot(s, peer, a0, b0);
    ld_slot(s + 1, peer, a1, b1);
}
// A probe whose loads are issued first and resolved later, so that independent work can run while they are in flight.
// A local probe fetches the aligned slot PAIR (one 64-byte DRAM access).  On a peer GPU's shard every byte crosses NVLink,
// and at load <= 0.25 the home slot alone decides ~9 probes out of 10: unless the table asks for pairs (peer_pair), the
// home slot is fetched first and its neighbour only if needed (halves the NVLink bytes of a sharded step).
struct HomeProbe {
    const ReqSlot* base;
    uint64_t slot;
    bool lazy;                       // slot 1 of the pair is fetched only when slot 0 does not decide
    uint4 a0, b0, a1, b1;
    __device__ __forceinline__ void load(bool peer) {
        ld_slot(base + slot, peer, a0, b0);
        if (!lazy) ld_slot(base + slot + 1, peer, a1, b1);
    }
    __device__ __forceinline__ void aim(const TableView& t, uint64_t key, uint32_t mdl) {
        const uint64_t hm = home_of(key, mdl);
        base = t.req_peer[shard_of(hm, t.shard_bits)];
        slot = hm & t.req_mask & ~1ull;
        lazy = base != t.req && !t.peer_pair;
    }
    // the fetched pair decides the lookup (hit: (A, B) the key's slot); else the probe moves on to the next pair
    __device__ __forceinline__ bool decide(const TableView& t, uint64_t key, uint32_t mdl, bool peer, uint4& A, uint4& B, bool& hit) {
        A = a0; B = b0;
        hit = slot_matches(A, B, key, mdl);
        if (!hit && meta_state(B.w) != kStateEmpty) {
            if (lazy) ld_slot(base + slot + 1, peer, a1, b1);
            A = a1; B = b1; hit = slot_matches(A, B, key, mdl);
        }
        if (hit || meta_state(B.w) == kStateEmpty) return true;
        slot = (slot + 2) & t.req_mask;                          // rare: displaced past the home pair
        return false;
    }
    // the loads now, the decision later (independent work may run in between)
    __device__ __forceinline__ void issue(const TableView& t, uint64_t key, uint32_t mdl, bool peer) { aim(t, key, mdl); load(peer); }
    __device__ __forceinline__ bool resolve(const TableView& t, uint64_t key, uint32_t mdl, bool peer, uint4& A, uint4& B) {
        bool hit;
        while (!decide(t, key, mdl, peer, A, B, hit)) load(peer);
        return hit;
    }
    // after a hit: the slot it was found in (CLOCK marking)
    __device__ __forceinline__ uint64_t hit_slot(uint64_t key, uint32_t mdl) const { return pair_hit_slot(slot, a0, b0, key, mdl); }
    // both at once, with the loads in one place (every ld_slot is a sequence-lock loop: fewer copies, shorter code)
    __device__ __forceinline__ bool find(const TableView& t, uint64_t key, uint32_t mdl, bool peer, uint4& A, uint4& B) {
        aim(t, key, mdl);
        bool hit;
        do load(peer); while (!decide(t, key, mdl, peer, A, B, hit));
        return hit;
    }
};

// The entry words and count of a slot image {ent 0|1, ent 2|3, ent 4|5, ent 6|7, ent 8|9, count}.  Two slots with equal
// patterns give every pod the same max-weight tier, so a block whose pattern repeats the previous block's adds the same
// addends again (most documents live on the same pods block after block).
struct SlotPat {
    uint32_t w[6];
    __device__ __forceinline__ static SlotPat of(const uint4& a, const uint4& b) { return {{a.z, a.w, b.x, b.y, b.z, meta_count(b.w)}}; }
    __device__ __forceinline__ uint32_t count() const { return w[5]; }
    __device__ __forceinline__ uint32_t ent(int j) const {
        const uint32_t word = j < 2 ? w[0] : j < 4 ? w[1] : j < 6 ? w[2] : j < 8 ? w[3] : w[4];
        return (j & 1) ? (word >> 16) : (word & 0xffffu);
    }
    __device__ __forceinline__ bool operator==(const SlotPat& o) const {
        return ((w[0] ^ o.w[0]) | (w[1] ^ o.w[1]) | (w[2] ^ o.w[2]) | (w[3] ^ o.w[3]) | (w[4] ^ o.w[4]) | (w[5] ^ o.w[5])) == 0u;
    }
    __device__ __forceinline__ SlotPat shfl(int src) const {
        SlotPat r;
#pragma unroll
        for (int x = 0; x < 6; ++x) r.w[x] = __shfl_sync(0xffffffffu, w[x], src);
        return r;
    }
    __device__ __forceinline__ SlotPat shfl_up() const {
        SlotPat r;
#pragma unroll
        for (int x = 0; x < 6; ++x) r.w[x] = __shfl_up_sync(0xffffffffu, w[x], 1);
        return r;
    }
};

// ---- LongestPrefixScorer.Score -----------------------------------------------------------------------------
// n in-order additions of the same addend (a run of blocks with the same slot pattern)
__device__ __forceinline__ double run_add(double sc, double add, int n) {
    for (int u = 0; u < n; ++u) sc = __dadd_rn(sc, add);
    return sc;
}

// Thread per prompt: the podScores / activePods of one prompt, restricted to the <= 10 pods block 0 can hold.
struct ScoreState {
    uint16_t pod[kMaxEnt];
    double sc[kMaxEnt];
    uint32_t k;        // pods present at block 0 (after the filter)
    uint32_t alive;    // bitmask over [0,k): still on the consecutive prefix

    __device__ __forceinline__ void first(const TableView& t, const SlotWords& w, const uint64_t* frow) {
        k = 0; alive = 0;
        const uint32_t cnt = meta_count(w.b.w);
        for (uint32_t j = 0; j < cnt; ++j) {
            const uint32_t pt = slot_ent(w, j);
            const uint32_t p = pt >> 4;
            if (frow && !filter_has(frow, p)) continue;
            const double wt = t.weight[pt & 15u];
            uint32_t q = 0;
            for (; q < k; ++q) if (pod[q] == p) break;
            if (q == k) { pod[k] = (uint16_t)p; sc[k] = 0.0; ++k; }
            if (wt > sc[q]) sc[q] = wt;                      // getMaxWeight starts at 0.0 (kvblock_scorer.go:90)
        }
        alive = (1u << k) - 1u;
    }
    __device__ __forceinline__ void next(const TableView& t, const SlotWords& w) {
        const uint32_t cnt = meta_count(w.b.w);
        for (uint32_t q = 0; q < k; ++q) {
            if (!((alive >> q) & 1u)) continue;
            double mx = 0.0; bool present = false;
            for (uint32_t j = 0; j < cnt; ++j) {
                const uint32_t pt = slot_ent(w, j);
                if ((pt >> 4) == pod[q]) { present = true; const double wt = t.weight[pt & 15u]; if (wt > mx) mx = wt; }
            }
            if (present) sc[q] = __dadd_rn(sc[q], mx);       // in-order f64 add (kvblock_scorer.go:143-146)
            else alive &= ~(1u << q);
        }
    }
    // the prompt's result row (the thread form of warp_write_row below)
    __device__ __forceinline__ void write_row(const TableView& t, int64_t i, bool has, double* dense_out, uint16_t* sp_pods, double* sp_scores,
                                              uint8_t* sp_cnt, uint8_t* has_keys) const {
        if (has_keys) has_keys[i] = has;
        if (dense_out) {
            double* row = dense_out + i * (int64_t)t.max_pods;
            for (uint32_t p = 0; p < t.max_pods; ++p) row[p] = -1.0;
            for (uint32_t q = 0; q < k; ++q) if (pod[q] < t.max_pods) row[pod[q]] = sc[q];
        }
        if (sp_cnt) {
            sp_cnt[i] = (uint8_t)k;
            for (uint32_t q = 0; q < k; ++q) { sp_pods[i * kMaxEnt + q] = pod[q]; sp_scores[i * kMaxEnt + q] = sc[q]; }
        }
    }
};

// Lane per prompt: the same state for the 32 prompts of a warp, transposed in shared memory ([entry][lane]: conflict free).
// bt caches the tier that gave pod q its max weight in the previous block, so a block with the previous block's pattern is
// one addition per live pod.
struct LaneCols {
    double sc[kMaxEnt][32];                // running score of block-0 pod q
    uint16_t pod[kMaxEnt][32];             // pod id of block-0 pod q
    uint8_t bt[kMaxEnt][32];               // tier giving pod q its max weight in the previous block (0xff: 0.0)

    // activePods := pods of block 0 (after the filter); score = max weight   (kvblock_scorer.go:118-128)
    __device__ __forceinline__ void first(int lane, const SlotPat& w, const uint64_t* frow, const double* weight, uint32_t& k, uint32_t& alive) {
        k = 0;
        for (uint32_t j = 0; j < w.count(); ++j) {
            const uint32_t pt = w.ent((int)j), p = pt >> 4;
            if (frow && !filter_has(frow, p)) continue;
            const double wt = weight[pt & 15u];
            uint32_t q = 0;
            for (; q < k; ++q) if (pod[q][lane] == p) break;
            if (q == k) { pod[k][lane] = (uint16_t)p; sc[k][lane] = 0.0; bt[k][lane] = 0xffu; ++k; }
            if (wt > sc[q][lane]) { sc[q][lane] = wt; bt[q][lane] = (uint8_t)(pt & 15u); }
        }
        alive = (1u << k) - 1u;
    }
    // activePods &= pods(block); score[p] += max weight, in block order   (kvblock_scorer.go:130-147)
    __device__ __forceinline__ void next(int lane, const SlotPat& w, const double* weight, uint32_t& alive) {
        uint32_t am = alive;
        while (am) {
            const int q = __ffs(am) - 1; am &= am - 1;
            const uint32_t want = pod[q][lane];
            double mx = 0.0; bool present = false; uint32_t b = 0xffu;
            for (uint32_t j = 0; j < w.count(); ++j) {
                const uint32_t pt = w.ent((int)j);
                if ((pt >> 4) == want) { present = true; const double wt = weight[pt & 15u]; if (wt > mx) { mx = wt; b = pt & 15u; } }
            }
            if (present) { sc[q][lane] = __dadd_rn(sc[q][lane], mx); bt[q][lane] = (uint8_t)b; }
            else alive &= ~(1u << q);
        }
    }
    // same pattern as the previous block: each live pod's cached max weight again, in block order
    __device__ __forceinline__ void repeat(int lane, const double* weight, uint32_t alive) {
        uint32_t am = alive;
        while (am) {
            const int q = __ffs(am) - 1; am &= am - 1;
            const uint32_t b = bt[q][lane];
            sc[q][lane] = __dadd_rn(sc[q][lane], b == 0xffu ? 0.0 : weight[b]);
        }
    }
};

// Warp per prompt: lane q < k owns pod q of the prompt's first block.  The lanes probe the blocks of a chunk at once
// (lane j: block j); the hits are then scored in block order, each block's slot pattern broadcast by shuffle.
struct WarpWalk {
    uint32_t k = 0, alive = 0;         // warp-uniform
    uint32_t pod = 0xffffffffu, bt = 0xffu;
    double sc = 0.0;
    SlotPat pat = {{0, 0, 0, 0, 0, 0xffffffffu}};   // pattern of the last scored block (warp-uniform)

    template <class PS> __device__ __forceinline__ void load(const PS& ps, int lane) {
        k = ps.k; alive = ps.alive;
#pragma unroll
        for (int x = 0; x < 6; ++x) pat.w[x] = ps.pat[x];
        if ((uint32_t)lane < k) { sc = ps.sc[lane]; pod = ps.pod[lane]; bt = ps.bt[lane]; }
    }
    // the per-lane part; the warp-uniform k, alive and pattern go to the state by store_uniform (lane 0)
    template <class PS> __device__ __forceinline__ void store_lane(PS& ps, int lane) const {
        if ((uint32_t)lane < k) { ps.sc[lane] = sc; ps.pod[lane] = (uint16_t)pod; ps.bt[lane] = (uint8_t)bt; }
    }
    template <class PS> __device__ __forceinline__ void store_uniform(PS& ps) const {
        ps.k = (uint8_t)k; ps.alive = (uint16_t)alive;
#pragma unroll
        for (int x = 0; x < 6; ++x) ps.pat[x] = pat.w[x];
    }

    // activePods := pods of block 0 (after the filter), in entry order; score = max weight   (kvblock_scorer.go:118-128)
    __device__ __forceinline__ void first(const TableView& t, int lane, const SlotPat& w, const uint64_t* frow) {
        k = 0;
        for (uint32_t e = 0; e < w.count(); ++e) {
            const uint32_t pt = w.ent((int)e), pd = pt >> 4;
            if (frow && !filter_has(frow, pd)) continue;
            const double wt = t.weight[pt & 15u];
            const uint32_t own = __ballot_sync(0xffffffffu, (uint32_t)lane < k && pod == pd);
            const int q = own ? __ffs(own) - 1 : (int)k;
            if (!own) { if (lane == q) { pod = pd; sc = 0.0; bt = 0xffu; } ++k; }
            if (lane == q && wt > sc) { sc = wt; bt = pt & 15u; }
        }
        alive = (1u << k) - 1u;
    }
    // activePods &= pods(block); score[p] += max weight, in block order   (kvblock_scorer.go:130-147)
    __device__ __forceinline__ void next(const TableView& t, int lane, const SlotPat& w) {
        bool present = false; double mx = 0.0; uint32_t b = 0xffu;
        if ((alive >> lane) & 1u) {
            for (uint32_t e = 0; e < w.count(); ++e) {
                const uint32_t pt = w.ent((int)e);
                if ((pt >> 4) == pod) { present = true; const double wt = t.weight[pt & 15u]; if (wt > mx) { mx = wt; b = pt & 15u; } }
            }
            if (present) { sc = __dadd_rn(sc, mx); bt = b; }
        }
        alive = __ballot_sync(0xffffffffu, present);
    }
    // CLOCK marking of a warp walk: lane l probed block l of the chunk and found it in slot `hslot`; walk() looked at the
    // chunk's first j blocks, so exactly those are marked (blocks fetched beyond the walk's end are not)
    __device__ __forceinline__ static void mark_walked(const TableView& t, int lane, int j, bool hit, uint64_t hslot) {
        if (t.req_ref && lane < j && hit) ref_touch(t.req_ref, hslot);
    }
    // n blocks that repeat the previous block's pattern: each live pod's addend n times more, in order
    __device__ __forceinline__ void run(const TableView& t, int lane, int n) {
        if ((alive >> lane) & 1u) sc = run_add(sc, bt == 0xffu ? 0.0 : t.weight[bt & 15u], n);
    }
    // bit j: block j of the chunk (lane j's pattern `mine`) repeats the block before it -- for block 0 the last block
    // scored before the chunk, if `cont` -- and is one of the first nhit blocks
    __device__ __forceinline__ uint32_t same_mask(int lane, const SlotPat& mine, bool cont, int nhit) const {
        const SlotPat up = mine.shfl_up();
        const bool s = lane > 0 ? up == mine : (cont && pat == mine);
        return __ballot_sync(0xffffffffu, s && lane < nhit);
    }
    // Scores the chunk's first nhit blocks (consecutive hits) in order, until no pod is left.  `first_block`: block 0 of the
    // chunk is the prompt's block 0 (then filter row `prompt` applies).  on_run_start(j) runs after block j is scored if the
    // walk is still alive and block j starts a run of equal patterns in this chunk: every block that is not a repeat, and,
    // with kRun0, block 0 also when it repeats the block before the chunk (that splits the run; a caller without snapshots
    // does without the extra code).  Returns the blocks looked at; the pattern of the last one is kept for the next chunk.
    template <bool kRun0, class Hook>
    __device__ __forceinline__ int walk(const TableView& t, int lane, const SlotPat& mine, int nhit, uint32_t samemask, bool first_block,
                                        const uint64_t* filter, int64_t prompt, Hook&& on_run_start) {
        int j = 0;
        bool dead = false;
        while (j < nhit && !dead) {
            if ((samemask >> j) & 1u) {
                const uint32_t rest = ~(samemask >> j);
                const int n = min(rest ? __ffs(rest) - 1 : 32, nhit - j);           // >= 1
                int u = 0;
                if (kRun0 && j == 0) { run(t, lane, 1); on_run_start(0); u = 1; }    // the chunk opens inside a run
                run(t, lane, n - u);
                j += n;
                continue;
            }
            const SlotPat w = mine.shfl(j);
            if (first_block && j == 0) first(t, lane, w, filter_row(filter, prompt, t.filter_words));
            else next(t, lane, w);
            if (!alive) dead = true;
            else on_run_start(j);
            ++j;
        }
        if (j > 0) pat = mine.shfl(j - 1);
        return j;
    }
};

// One finished prompt's result, written by the whole warp: every pod of the dense row -1, then the prompt's scores; the
// sparse form; has_keys.  Lane q passes entry q of the prompt's pod list (pod, sc: read only below k).
__device__ __forceinline__ void warp_write_row(const TableView& t, const ScoreArgs& a, int64_t prompt, uint32_t k, uint32_t pod, double sc, bool has,
                                               uint64_t l2pol) {
    const int lane = threadIdx.x & 31;
    if (a.dense) {
        double* row = a.dense + prompt * (int64_t)t.max_pods;
        const uint32_t P = t.max_pods;
        if ((P & 1u) == 0 && ((reinterpret_cast<uintptr_t>(row) & 15u) == 0)) {
            for (uint32_t c = lane * 2; c < P; c += 64) st_stream_f64x2(row + c, -1.0, -1.0, l2pol);
        } else {
            for (uint32_t c = lane; c < P; c += 32) row[c] = -1.0;
        }
        __syncwarp();
        if ((uint32_t)lane < k && pod < P) row[pod] = sc;
    }
    if (a.sp_cnt) {
        if ((uint32_t)lane < k) { a.sp_pods[prompt * kMaxEnt + lane] = (uint16_t)pod; a.sp_scores[prompt * kMaxEnt + lane] = sc; }
        if (lane == 0) a.sp_cnt[prompt] = (uint8_t)k;
    }
    if (a.has_keys && lane == 0) a.has_keys[prompt] = has;
}

}  // namespace kvx
