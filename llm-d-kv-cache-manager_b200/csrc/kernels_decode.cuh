// kernels_decode.cuh -- vLLM KVEvents msgpack messages decoded on the device into the write path's event records
// (include/kvidx.h kvidx_decode_event_payloads_dev).  The rules are host/kvhost.cpp's head / skip / hash_of / decode_event /
// decode_batch, one for one; the host decoder is the specification and the tests hold the two to byte equality.
//
// One thread per message, in two passes over the same code (d_decode_events, templated on what it does with an event):
//   count pass  validates the envelope, decodes every event and counts events, hashes and tokens, the admitted blocks and
//               removed hashes of the metrics, and the markers / unknown tier names that need the caller;
//   write pass  decodes again and writes the records, their hashes and tokens at the offsets the scans between the two
//               passes gave the message (events pod-sorted, hashes and tokens in message order).
// skip() cannot recurse on the device: it walks with an explicit stack of elements left per level, and fails past nesting
// depth 64 exactly where the host's recursion does.  Every read is checked against the end of the message (or of the event
// slice the envelope pass cut), so no input makes a thread read outside [msg_off[i], msg_off[i+1]).
#pragma once
#include <cstdint>
#include "../../include/kvidx.h"

namespace kvx {

constexpr int kDecThreads = 128;
constexpr int kDecMaxDepth = 64;                     // host skip(): depth > 64 fails
constexpr uint32_t kDecMaxTiers = KVIDX_MAX_TIERS;

// per-message flags (kvidx.h KVIDX_PAYLOAD_MSG_*)
constexpr uint8_t kMsgDecoded = 1, kMsgUnknownTier = 2, kMsgCleared = 4;

enum DKind : uint8_t { D_NIL, D_BOOL, D_INT, D_FLOAT, D_STR, D_BIN, D_ARRAY, D_MAP, D_EXT, D_BAD };
struct DVal { DKind k; uint8_t code; uint64_t u; const uint8_t* s; uint64_t n; };
struct DCur { const uint8_t* p; const uint8_t* e; };

// The tier table: name t is bytes[off[t] .. off[t+1]), lower-case.  gpu: the id of a Medium-less event (< 0: none).
struct TierTable { const uint8_t* bytes; uint64_t off[kDecMaxTiers + 1]; uint32_t n; int32_t gpu; };

// Totals the count pass accumulates (read back once by the host).
struct DecTotals {
    unsigned long long messages, events, hashes, tokens, queues, admitted, removed_hashes, markers;   // kvidx.h counts_out
    unsigned long long stored_hashes, max_ev_hashes;
    unsigned int unknown_tier, bad_pod, bad_model, bad_off;
};

__device__ __forceinline__ bool d_need(const DCur& c, uint64_t n) { return (uint64_t)(c.e - c.p) >= n; }
__device__ __forceinline__ uint64_t d_be(const uint8_t* p, int n) { uint64_t v = 0; for (int i = 0; i < n; ++i) v = (v << 8) | p[i]; return v; }

// host head(): scalars, strings and bins are consumed completely; containers leave the cursor at their first child
__device__ bool d_head(DCur& c, DVal& v) {
    if (!d_need(c, 1)) return false;
    const uint8_t b = *c.p++;
    v.code = b; v.u = 0; v.n = 0; v.s = nullptr; v.k = D_BAD;
    uint64_t t = 0;
    auto rd = [&](int n, uint64_t& out) { if (!d_need(c, n)) return false; out = d_be(c.p, n); c.p += n; return true; };
    auto blob = [&](uint64_t n, DKind k) { if (!d_need(c, n)) return false; v.k = k; v.s = c.p; v.n = n; c.p += n; return true; };
    if (b <= 0x7f) { v.k = D_INT; v.u = b; return true; }
    if (b >= 0xe0) { v.k = D_INT; v.u = (uint64_t)(int64_t)(int8_t)b; return true; }
    if (b >= 0xa0 && b <= 0xbf) return blob(b & 0x1f, D_STR);
    if (b >= 0x90 && b <= 0x9f) { v.k = D_ARRAY; v.n = b & 0x0f; return true; }
    if (b >= 0x80 && b <= 0x8f) { v.k = D_MAP; v.n = b & 0x0f; return true; }
    switch (b) {
        case 0xc0: v.k = D_NIL; return true;
        case 0xc2: case 0xc3: v.k = D_BOOL; v.u = b & 1; return true;
        case 0xc4: return rd(1, t) && blob(t, D_BIN);
        case 0xc5: return rd(2, t) && blob(t, D_BIN);
        case 0xc6: return rd(4, t) && blob(t, D_BIN);
        case 0xc7: return rd(1, t) && d_need(c, 1) && (c.p++, blob(t, D_EXT));
        case 0xc8: return rd(2, t) && d_need(c, 1) && (c.p++, blob(t, D_EXT));
        case 0xc9: return rd(4, t) && d_need(c, 1) && (c.p++, blob(t, D_EXT));
        case 0xca: if (!rd(4, t)) return false; v.k = D_FLOAT; return true;     // the value itself is never used
        case 0xcb: if (!rd(8, t)) return false; v.k = D_FLOAT; return true;
        case 0xcc: v.k = D_INT; return rd(1, v.u);
        case 0xcd: v.k = D_INT; return rd(2, v.u);
        case 0xce: v.k = D_INT; return rd(4, v.u);
        case 0xcf: v.k = D_INT; return rd(8, v.u);
        case 0xd0: v.k = D_INT; if (!rd(1, t)) return false; v.u = (uint64_t)(int64_t)(int8_t)t; return true;
        case 0xd1: v.k = D_INT; if (!rd(2, t)) return false; v.u = (uint64_t)(int64_t)(int16_t)t; return true;
        case 0xd2: v.k = D_INT; if (!rd(4, t)) return false; v.u = (uint64_t)(int64_t)(int32_t)t; return true;
        case 0xd3: v.k = D_INT; return rd(8, v.u);
        case 0xd4: return d_need(c, 1) && (c.p++, blob(1, D_EXT));
        case 0xd5: return d_need(c, 1) && (c.p++, blob(2, D_EXT));
        case 0xd6: return d_need(c, 1) && (c.p++, blob(4, D_EXT));
        case 0xd7: return d_need(c, 1) && (c.p++, blob(8, D_EXT));
        case 0xd8: return d_need(c, 1) && (c.p++, blob(16, D_EXT));
        case 0xd9: return rd(1, t) && blob(t, D_STR);
        case 0xda: return rd(2, t) && blob(t, D_STR);
        case 0xdb: return rd(4, t) && blob(t, D_STR);
        case 0xdc: v.k = D_ARRAY; if (!rd(2, t)) return false; v.n = t; return true;
        case 0xdd: v.k = D_ARRAY; if (!rd(4, t)) return false; v.n = t; return true;
        case 0xde: v.k = D_MAP; if (!rd(2, t)) return false; v.n = t; return true;
        case 0xdf: v.k = D_MAP; if (!rd(4, t)) return false; v.n = t; return true;
        default: return false;                       // 0xc1: never used
    }
}

// host skip(c, depth0), without recursion: left[l] = elements still to read at depth depth0 + l.  Every element takes at
// least one byte, so a container declaring more elements than bytes remain fails at once -- where the host fails too, only
// later; a failed skip's cursor position is never used.
__device__ bool d_skip(DCur& c, int depth0) {
    uint64_t left[kDecMaxDepth + 2];
    int l = 0;
    left[0] = 1;
    while (l >= 0) {
        if (left[l] == 0) { --l; continue; }
        --left[l];
        DVal v;
        if (depth0 + l > kDecMaxDepth || !d_head(c, v)) return false;
        if (v.k == D_ARRAY || v.k == D_MAP) {
            const uint64_t n = v.k == D_ARRAY ? v.n : 2 * v.n;
            if (n > (uint64_t)(c.e - c.p)) return false;
            left[++l] = n;
        }
    }
    return true;
}

// host hash_of(): only uint64- / int64-coded integers and non-empty bins are hashes
__device__ bool d_hash_of(DCur& c, uint64_t* out, bool* is_nil) {
    const uint8_t* start = c.p;
    DVal v;
    if (is_nil) *is_nil = false;
    DCur probe = c;
    if (!d_head(probe, v)) { c.p = c.e; return false; }
    if (v.k == D_ARRAY || v.k == D_MAP) { c.p = start; if (!d_skip(c, 0)) c.p = c.e; return false; }
    c = probe;
    if (v.k == D_NIL) { if (is_nil) *is_nil = true; return false; }
    if (v.k == D_INT && (v.code == 0xcf || v.code == 0xd3)) { *out = v.u; return true; }
    if (v.k == D_BIN) {
        if (v.n == 0) return false;
        *out = v.n >= 8 ? d_be(v.s + v.n - 8, 8) : d_be(v.s, (int)v.n);
        return true;
    }
    return false;
}

__device__ __forceinline__ bool d_tag_is(const DVal& t, const char* lit, uint64_t len) {
    if (t.n != len) return false;
    for (uint64_t i = 0; i < len; ++i) if (t.s[i] != (uint8_t)lit[i]) return false;
    return true;
}

// lower(Medium) (ASCII tolower, byte by byte) looked up in the tier table: its id, or -1
__device__ int d_tier_of(const TierTable& tt, const uint8_t* s, uint64_t n) {
    for (uint32_t t = 0; t < tt.n; ++t) {
        const uint64_t o = tt.off[t];
        if (tt.off[t + 1] - o != n) continue;
        uint64_t i = 0;
        for (; i < n; ++i) {
            uint8_t ch = s[i];
            if (ch >= 'A' && ch <= 'Z') ch += 'a' - 'A';
            if (ch != tt.bytes[o + i]) break;
        }
        if (i == n) return (int)t;
    }
    return -1;
}

// What a pass does with the decoded events of one message.  hash(i, h) / tok(i, t): the i-th hash / token of the event
// being decoded (relative to the committed ones); event(...) commits it with its counts.  An event that fails after some of
// its hashes or tokens were offered is simply never committed.
struct DecCount {
    int64_t n_ev = 0, n_hash = 0, n_tok = 0;
    uint64_t stored_hashes = 0, removed_hashes = 0, admitted = 0, markers = 0, max_ev_hashes = 0;
    uint32_t block_size;
    __device__ void hash(uint64_t, uint64_t) {}
    __device__ void tok(uint64_t, uint32_t) {}
    __device__ void marker() { ++markers; }
    __device__ void event(uint8_t op, bool, uint64_t, int, uint32_t nh, uint32_t nt) {
        ++n_ev; n_hash += nh; n_tok += nt;
        max_ev_hashes = max(max_ev_hashes, (uint64_t)nh);
        if (op == KVIDX_EV_BLOCK_STORED) { stored_hashes += nh; if (nh > 0) admitted += nt / block_size; }
        else removed_hashes += nh;
    }
};
struct DecWrite {
    kvidx_event_t* ev; uint64_t* hashes; uint32_t* toks;
    int64_t ev_at, h_at, t_at, h_end, t_end;         // next free positions; ends of this message's sections
    uint32_t pod, model;
    __device__ void marker() {}
    __device__ void hash(uint64_t i, uint64_t h) { if (h_at + (int64_t)i < h_end) hashes[h_at + i] = h; }
    __device__ void tok(uint64_t i, uint32_t t) { if (t_at + (int64_t)i < t_end) toks[t_at + i] = t; }
    __device__ void event(uint8_t op, bool has_parent, uint64_t parent, int tier, uint32_t nh, uint32_t nt) {
        kvidx_event_t e;
        e.op = op; e.has_parent = has_parent ? 1 : 0; e.podtier = KVIDX_PODTIER(pod, tier); e.model = model;
        e.parent_hash = has_parent ? parent : 0; e.hash_off = (uint64_t)h_at; e.tok_off = (uint64_t)t_at;
        e.n_hashes = nh; e.n_tokens = nt;
        ev[ev_at++] = e;
        h_at += nh; t_at += nt;
    }
};

// host decode_event() over one event slice [p, e).  *unknown: the event names a tier the table lacks (it is dropped, as
// the host drops an event whose name finds no room in the 16-id tier space).
template <class Sink>
__device__ void d_decode_event(const TierTable& tt, const uint8_t* p, const uint8_t* e, Sink& sk, bool* unknown) {
    DCur c{p, e};
    DVal v;
    if (!d_head(c, v)) return;
    if (v.k != D_ARRAY || v.n < 1) return;                               // not an array / no tag element: skipped
    const uint64_t rest = v.n - 1;
    DVal tag;
    if (!d_head(c, tag)) return;
    if (tag.k != D_STR && tag.k != D_BIN) return;                         // tag must decode as string
    const bool stored = d_tag_is(tag, "BlockStored", 11);
    if (!stored && !d_tag_is(tag, "BlockRemoved", 12)) {
        if (d_tag_is(tag, "AllBlocksCleared", 16)) sk.marker();           // decodes to nothing (pool.go:332-333)
        return;                                                           // unknown tags: skipped
    }
    bool ok = true, parent_bad = false, has_parent = false;
    uint64_t parent = 0, f = 0;
    uint32_t nh = 0, nt = 0;
    if (f < rest) {                                                       // BlockHashes []any
        DVal a;
        if (!d_head(c, a)) return;
        if (a.k == D_ARRAY) {
            for (uint64_t i = 0; i < a.n && ok; ++i) {
                uint64_t hv; const uint8_t* before = c.p;
                if (d_hash_of(c, &hv, nullptr)) sk.hash(nh++, hv);
                if (c.p == before || c.p > e) ok = false;
            }
        } else if (a.k != D_NIL) ok = false;
        ++f;
    }
    if (stored) {
        if (ok && f < rest) {                                             // ParentBlockHash any
            bool nil = false;
            if (d_hash_of(c, &parent, &nil)) has_parent = true;
            else if (!nil) parent_bad = true;                             // unsupported type: event skipped (pool.go:283-287)
            ++f;
        }
        if (ok && f < rest) {                                             // TokenIds []uint32
            DVal a;
            if (!d_head(c, a)) ok = false;
            else if (a.k == D_ARRAY) {
                for (uint64_t i = 0; i < a.n && ok; ++i) { DVal x; if (!d_head(c, x) || x.k != D_INT) ok = false; else sk.tok(nt++, (uint32_t)x.u); }
            } else if (a.k != D_NIL) ok = false;
            ++f;
        }
        if (ok && f < rest) { DVal x; if (!d_head(c, x) || (x.k != D_INT && x.k != D_NIL)) ok = false; ++f; }   // BlockSize int (ignored)
        if (ok && f < rest) { DVal x; if (!d_head(c, x) || (x.k != D_INT && x.k != D_NIL)) ok = false; ++f; }   // LoraID *int
    }
    int tier = 0;
    if (ok) {                                                             // Medium *string, lower-cased; default "gpu"
        int id = tt.gpu;
        if (f < rest) {
            DVal m;
            if (!d_head(c, m)) ok = false;
            else if (m.k == D_STR || m.k == D_BIN) id = d_tier_of(tt, m.s, m.n);
            else if (m.k != D_NIL) ok = false;
            ++f;
        }
        if (ok && id < 0) { *unknown = true; ok = false; }
        tier = id;
    }
    for (; ok && f < rest; ++f) ok = d_skip(c, 0);                        // extra fields are skipped
    if (!ok || parent_bad) return;
    sk.event(stored ? KVIDX_EV_BLOCK_STORED : KVIDX_EV_BLOCK_REMOVED, has_parent, parent, tier, nh, stored ? nt : 0);
}

// host decode_batch(): EventBatch = [ts, events[], dp_rank?, extra...]; any envelope error drops the whole message.  The
// event slices are cut (and skip()-validated) before any event is decoded, as the host does.  Returns false when dropped.
__device__ bool d_envelope(DCur& c, const uint8_t** ev0, uint64_t* n_ev) {
    DVal v;
    *n_ev = 0; *ev0 = nullptr;
    if (!d_head(c, v) || v.k != D_ARRAY) return false;
    const uint64_t n = v.n;
    if (n >= 1) { DVal ts; if (!d_head(c, ts) || (ts.k != D_FLOAT && ts.k != D_INT && ts.k != D_NIL)) return false; }
    if (n >= 2) {
        DVal a;
        if (!d_head(c, a)) return false;
        if (a.k == D_ARRAY) {
            *ev0 = c.p;
            for (uint64_t i = 0; i < a.n; ++i) if (!d_skip(c, 0)) return false;
            *n_ev = a.n;
        } else if (a.k != D_NIL) return false;
    }
    if (n >= 3) { DVal r; if (!d_head(c, r) || (r.k != D_INT && r.k != D_NIL)) return false; }
    for (uint64_t i = 3; i < n; ++i) if (!d_skip(c, 0)) return false;
    return true;
}

// Decodes message m's events into the sink (the envelope was validated: its events are n_ev consecutive valid elements).
template <class Sink>
__device__ void d_decode_events(const TierTable& tt, const uint8_t* ev0, uint64_t n_ev, const uint8_t* end, Sink& sk, bool* unknown) {
    DCur c{ev0, end};
    for (uint64_t i = 0; i < n_ev; ++i) {
        const uint8_t* s = c.p;
        d_skip(c, 0);
        d_decode_event(tt, s, c.p, sk, unknown);
    }
}

struct DecIn {
    const uint8_t* bytes; const int64_t* msg_off; const uint32_t* msg_pod; const uint32_t* msg_model;
    int64_t n_msgs; uint32_t max_pods; uint32_t block_size;
    TierTable tt;
};

// Count pass.  Per message: events, hashes, tokens, flags; per pod: events (pod_ev, zeroed by the caller); totals.
__global__ void __launch_bounds__(kDecThreads) decode_count_kernel(DecIn in, int64_t* ev_cnt, int64_t* hash_cnt, int64_t* tok_cnt,
                                                                   uint8_t* msg_flags, uint32_t* sort_key, uint32_t* sort_val,
                                                                   unsigned long long* pod_ev, DecTotals* tot) {
    const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= in.n_msgs) return;
    const uint32_t pod = in.msg_pod[m], model = in.msg_model[m];
    const bool pod_ok = pod < in.max_pods;
    if (!pod_ok) atomicOr(&tot->bad_pod, 1u);
    if (model > 0xffffu) atomicOr(&tot->bad_model, 1u);
    sort_key[m] = pod_ok ? pod : 0;
    sort_val[m] = (uint32_t)m;
    const int64_t o0 = in.msg_off[m], o1 = in.msg_off[m + 1];
    if (o1 < o0) { atomicOr(&tot->bad_off, 1u); msg_flags[m] = 0; ev_cnt[m] = hash_cnt[m] = tok_cnt[m] = 0; return; }
    const uint8_t* p = in.bytes + o0;
    const uint8_t* e = in.bytes + o1;
    DCur c{p, e};
    const uint8_t* ev0; uint64_t n_ev;
    DecCount k; k.block_size = in.block_size;
    uint8_t fl = 0;
    if (d_envelope(c, &ev0, &n_ev)) {
        bool unknown = false;
        d_decode_events(in.tt, ev0, n_ev, e, k, &unknown);
        fl = kMsgDecoded | (unknown ? kMsgUnknownTier : 0) | (k.markers ? kMsgCleared : 0);
    }
    ev_cnt[m] = k.n_ev; hash_cnt[m] = k.n_hash; tok_cnt[m] = k.n_tok;
    msg_flags[m] = fl;
    if (k.n_ev && pod_ok) atomicAdd(&pod_ev[pod], (unsigned long long)k.n_ev);
    if (fl & kMsgDecoded) atomicAdd(&tot->messages, 1ull);
    if (k.n_ev) atomicAdd(&tot->events, (unsigned long long)k.n_ev);
    if (k.n_hash) atomicAdd(&tot->hashes, (unsigned long long)k.n_hash);
    if (k.n_tok) atomicAdd(&tot->tokens, (unsigned long long)k.n_tok);
    if (fl & kMsgUnknownTier) atomicOr(&tot->unknown_tier, 1u);
    if (k.stored_hashes) atomicAdd(&tot->stored_hashes, (unsigned long long)k.stored_hashes);
    if (k.removed_hashes) atomicAdd(&tot->removed_hashes, (unsigned long long)k.removed_hashes);
    if (k.admitted) atomicAdd(&tot->admitted, (unsigned long long)k.admitted);
    if (k.markers) atomicAdd(&tot->markers, (unsigned long long)k.markers);
    if (k.max_ev_hashes) atomicMax(&tot->max_ev_hashes, (unsigned long long)k.max_ev_hashes);
}

// ev_cnt gathered into pod-sorted message order (the scan input of the events' positions)
__global__ void decode_gather_kernel(const uint32_t* sorted_val, const int64_t* ev_cnt, int64_t n, int64_t* out) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) out[j] = ev_cnt[sorted_val[j]];
}

// Queue offsets: queue q is the q-th pod (ascending) with events, starting at the events of all smaller pods.  One CTA of
// 1024 threads over max_pods (<= 4096) pods, four consecutive pods per thread; *n_queues: the queue count.
constexpr int kQueueThreads = 1024;
__global__ void __launch_bounds__(kQueueThreads) decode_queues_kernel(const unsigned long long* pod_ev, uint32_t max_pods,
                                                                      int64_t* queue_off, unsigned long long* n_queues) {
    __shared__ unsigned long long s_ev[kQueueThreads];
    __shared__ unsigned int s_q[kQueueThreads];
    const int t = threadIdx.x;
    unsigned long long e[4], evs = 0;
    unsigned int q = 0;
    for (int i = 0; i < 4; ++i) {
        const uint32_t p = (uint32_t)t * 4 + i;
        e[i] = p < max_pods ? pod_ev[p] : 0;
        evs += e[i]; q += e[i] ? 1 : 0;
    }
    s_ev[t] = evs; s_q[t] = q;
    __syncthreads();
    for (int d = 1; d < kQueueThreads; d <<= 1) {                 // inclusive Hillis-Steele scan
        const unsigned long long a = t >= d ? s_ev[t - d] : 0;
        const unsigned int b = t >= d ? s_q[t - d] : 0;
        __syncthreads();
        s_ev[t] += a; s_q[t] += b;
        __syncthreads();
    }
    unsigned long long at = s_ev[t] - evs;
    unsigned int qi = s_q[t] - q;
    for (int i = 0; i < 4; ++i) {
        if (e[i]) queue_off[qi++] = (int64_t)at;
        at += e[i];
    }
    if (t == kQueueThreads - 1) { queue_off[s_q[t]] = (int64_t)s_ev[t]; *n_queues = s_q[t]; }
}

// Write pass.  ev_base_sorted[j]: the first event position of the j-th message in pod order (scanned); hash_base /
// tok_base: the message's first hash / token (scanned in message order), hash_cnt / tok_cnt its counts.
__global__ void __launch_bounds__(kDecThreads) decode_write_kernel(DecIn in, const uint32_t* sorted_val, const int64_t* ev_base_sorted,
                                                                   const int64_t* hash_base, const int64_t* hash_cnt,
                                                                   const int64_t* tok_base, const int64_t* tok_cnt,
                                                                   const uint8_t* msg_flags, kvidx_event_t* ev_out,
                                                                   uint64_t* hash_out, uint32_t* tok_out) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= in.n_msgs) return;
    const int64_t m = sorted_val[j];
    if (!(msg_flags[m] & kMsgDecoded)) return;
    const uint8_t* p = in.bytes + in.msg_off[m];
    const uint8_t* e = in.bytes + in.msg_off[m + 1];
    DCur c{p, e};
    const uint8_t* ev0; uint64_t n_ev;
    d_envelope(c, &ev0, &n_ev);
    DecWrite w;
    w.ev = ev_out; w.hashes = hash_out; w.toks = tok_out;
    w.ev_at = ev_base_sorted[j]; w.h_at = hash_base[m]; w.t_at = tok_base[m];
    w.h_end = w.h_at + hash_cnt[m]; w.t_end = w.t_at + tok_cnt[m];
    w.pod = in.msg_pod[m]; w.model = in.msg_model[m];
    bool unknown = false;
    d_decode_events(in.tt, ev0, n_ev, e, w, &unknown);
}

}  // namespace kvx
