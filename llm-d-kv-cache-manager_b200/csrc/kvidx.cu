// kvidx.cu -- C ABI (include/kvidx.h) over the sm_90a kernels.  No torch types, no CPU fallback.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "../../include/kvidx.h"
#include "kernels_v1.cuh"
#include "kernels_write.cuh"
#include "kernels_clock.cuh"
#include "kernels_remove.cuh"
#include "kernels_snapshot.cuh"
#include "kernels_inventory.cuh"
#include "kernels_rounds.cuh"
#include "kernels_rounds_plain.cuh"
#include "kernels_coop.cuh"
#include "kernels_keys.cuh"
#include "kernels_turn.cuh"
#include "kernels_route.cuh"
#include "kernels_text.cuh"
#include "kernels_hits.cuh"
#include "kernels_decode.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

using namespace kvx;

namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    g_err = buf;
    return code;
}

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) return fail(KVIDX_ECUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

uint64_t pow2ceil(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return p; }

// A stream or event the handle created, destroyed with its owner.  It converts to the raw handle.
template <class T, cudaError_t (*Destroy)(T)> struct Owned {
    T h = nullptr;
    Owned() = default;
    Owned(const Owned&) = delete;
    Owned& operator=(const Owned&) = delete;
    ~Owned() { if (h) Destroy(h); }
    operator T() const { return h; }
};
using OwnStream = Owned<cudaStream_t, cudaStreamDestroy>;
using OwnEvent = Owned<cudaEvent_t, cudaEventDestroy>;

// growable device / pinned-host scratch, freed with its owner
struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    cudaError_t need(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = std::max(n, (size_t)4096);
        want = want + want / 4;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() { return static_cast<T*>(p); }
};
struct PinBuf {
    void* p = nullptr; size_t cap = 0;
    PinBuf() = default;
    PinBuf(const PinBuf&) = delete;
    PinBuf& operator=(const PinBuf&) = delete;
    ~PinBuf() { if (p) cudaFreeHost(p); }
    cudaError_t need(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        size_t want = std::max(n, (size_t)4096);
        want = want + want / 4;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    template <class T> T* as() { return static_cast<T*>(p); }
};

bool is_device_accessible_host(const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;     // pinned: cudaMemcpyAsync from it is truly async
}

// Every scratch buffer a call lays out is carved into sections by a Carver, twice: over a null base to size the buffer,
// then over the buffer itself (carve()), so each section's size is written once.  Sections start on 256-byte
// boundaries, as a cudaMalloc of their own would (TMA reads staged inputs in place and needs 16).  An empty section
// takes no bytes: its pointer is the next section's, and a caller never dereferences it.
struct Carver {
    static constexpr size_t kAlign = 256;
    uintptr_t base = 0; size_t at = 0;
    template <class T> T* take(size_t count) {
        static_assert(kAlign % alignof(T) == 0, "a section is aligned for its elements");
        T* p = reinterpret_cast<T*>(base + at);
        at += (count * sizeof(T) + kAlign - 1) & ~(kAlign - 1);
        return p;
    }
};

// Sizes buf for the sections `layout` takes (growing it as need() does; what it held is dropped) and carves them from it.
template <class Buf, class Layout> cudaError_t carve(Buf& buf, Layout&& layout) {
    Carver size;
    layout(size);
    if (cudaError_t e = buf.need(size.at)) return e;
    Carver c{reinterpret_cast<uintptr_t>(buf.p)};
    layout(c);
    return cudaSuccess;
}

// Moves bytes between the device and a caller's host buffer: one copy when the buffer is pinned, else through two pinned
// chunks that alternate (the copy engine fills or empties one while the host works on the other).
struct Stager {
    static constexpr size_t kChunk = 16u << 20;
    PinBuf buf[2];
    OwnEvent ev[2];
    cudaError_t init() {
        for (auto& e : ev) if (cudaError_t r = cudaEventCreateWithFlags(&e.h, cudaEventDisableTiming)) return r;
        return cudaSuccess;
    }
    // device -> host; every byte is in dst when it returns
    int d2h(void* dst, const void* src, size_t n, cudaStream_t st) {
        if (n == 0) return 0;
        if (is_device_accessible_host(dst)) {
            CK(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            return 0;
        }
        CK(buf[0].need(kChunk));
        CK(buf[1].need(kChunk));
        const size_t nc = (n + kChunk - 1) / kChunk;
        for (size_t k = 0; k <= nc; ++k) {
            if (k < nc) {
                const size_t off = k * kChunk, len = std::min(kChunk, n - off);
                CK(cudaMemcpyAsync(buf[k & 1].p, static_cast<const char*>(src) + off, len, cudaMemcpyDeviceToHost, st));
                CK(cudaEventRecord(ev[k & 1], st));
            }
            if (k > 0) {
                const size_t j = k - 1, off = j * kChunk, len = std::min(kChunk, n - off);
                CK(cudaEventSynchronize(ev[j & 1]));
                memcpy(static_cast<char*>(dst) + off, buf[j & 1].p, len);
            }
        }
        return 0;
    }
    // host -> device, queued on st
    int h2d(void* dst, const void* src, size_t n, cudaStream_t st) {
        if (n == 0) return 0;
        if (is_device_accessible_host(src)) { CK(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, st)); return 0; }
        CK(buf[0].need(kChunk));
        CK(buf[1].need(kChunk));
        const size_t nc = (n + kChunk - 1) / kChunk;
        for (size_t k = 0; k < nc; ++k) {
            const size_t off = k * kChunk, len = std::min(kChunk, n - off);
            CK(cudaEventSynchronize(ev[k & 1]));          // the copy out of this chunk two steps (or one call) ago is done
            memcpy(buf[k & 1].p, static_cast<const char*>(src) + off, len);
            CK(cudaMemcpyAsync(static_cast<char*>(dst) + off, buf[k & 1].p, len, cudaMemcpyHostToDevice, st));
            CK(cudaEventRecord(ev[k & 1], st));
        }
        return 0;
    }
};

}  // namespace

// Concurrent host-buffer Score() callers (one goroutine / OS thread per RPC, server.go:70-96) are coalesced: whoever finds
// no batch in progress becomes the leader, takes everything that has queued up meanwhile, runs it as ONE batch through the
// pipeline and wakes the owners.  No dedicated thread, no artificial delay: a lone caller goes straight through with its
// own buffers; under load the batch size grows by itself to what arrived during the previous launch.
struct SubmitReq {
    const uint32_t* tok; ScoreArgs a;              // the call in host memory (a.tok unused)
    int rc = 0; bool done = false, promote = false; std::string err;
    std::mutex m; std::condition_variable cv;      // each waiter sleeps on its OWN condition variable: finishing a batch wakes
                                                   // exactly its owners (and the next leader), not every queued thread
};
struct SubmitQueue {
    std::mutex mu;
    std::deque<SubmitReq*> pending;
    bool leader_active = false;
    bool enabled = true;
    int64_t max_prompts = 65536, max_tokens = 64ll << 20;
    std::atomic<uint64_t> coalesced{0}, batches{0};
    PinBuf h_in, h_out;                            // the combined batch and its rows, owned by the current leader
};

// the device prefix store (kvidx_text_store_*); the table and the arena are freed with it
struct TextStore {
    int64_t cap_blocks = 0; uint32_t B = 0;
    OwnStream stream;                         // kvidx_text_store_add / _find (Score() from text runs on the handle's stream)
    OwnEvent ev_last;                         // the end of the last store call, on whichever stream it ran: the next one waits
    Stager stage;                             // for pageable host buffers
    PinBuf h_misc;
    TextTable t{};
    void* tab = nullptr;                      // the table's arrays, one allocation
    uint32_t* arena = nullptr; int64_t arena_cap = 0, arena_used = 0;
    int64_t resident = 0;
    unsigned long long clock = 0;             // recency stamps handed out so far
    DevBuf d_in, d_blk, d_scr, d_tok, d_cub, d_out;
    TextStore() = default;
    TextStore(const TextStore&) = delete;
    TextStore& operator=(const TextStore&) = delete;
    ~TextStore() { if (tab) cudaFree(tab); if (arena) cudaFree(arena); }
};

struct kvidx {
    kvidx_config_t cfg{};
    TableView tv{};
    int device = 0;
    int sm_count = 132;
    // Read path (Score / Lookup / hash) and write path (Add / Evict / events) run on their own streams and behind their own
    // mutexes: a Score() call and an event batch overlap on the device (table.cuh: readers never wait for writers).
    // The streams and events below are the handle's own; `stream` is the read side's, which may be the caller's.
    OwnStream own_stream, copy_stream, d2h_stream, own_wstream;
    cudaStream_t stream = nullptr;
    OwnEvent ev_h2d[2], ev_done[2], ev_k[2];
    OwnEvent ev_write;                // last asynchronous (device-resident) write batch: later reads are ordered after it
    Counters* d_cnt = nullptr;
    Counters* h_cnt = nullptr;     // pinned mirror (write side)
    Counters* d_cnt_all = nullptr; // sharded: every owner's counters, gathered before a write batch
    Counters* h_cnt_all = nullptr;
    uint64_t rebuilds = 0;
    uint64_t grow_max = 0;          // grow_tables: the slot count the tables may grow to (C); 0: fixed tables
    std::atomic<uint64_t> launches{0};
    std::atomic<unsigned long long> clock{1};   // exact-LRU mode: recency stamps handed to kernels
    std::mutex mu_r, mu_w;          // read-side / write-side scratch and stream
    std::shared_mutex tables;       // shared: any call that launches on the tables; exclusive: rebuild swaps them
    // read-side scratch (guarded by mu_r)
    DevBuf d_tok[2], d_off[2], d_model[2], d_filter[2], d_out[2], d_aux[2], d_rmisc;
    PinBuf h_stage[2], h_out[2];
    DevBuf d_turn;                  // a conversation turn on the composed path: the concatenated key CSR and its setup
    DevBuf d_inv; PinBuf h_inv;     // kvidx_pod_inventory: the 64-bit histograms on the device and their pinned copy
    Stager rstage;                  // kvidx_lookup_hits*: a caller's host buffers to and from the device
    // write-side scratch (guarded by mu_w)
    DevBuf d_misc, d_ev, d_hash, d_evtok, d_qoff, d_wkeys, d_wpred, d_wready, d_wmap;
    DevBuf d_sweep;                 // CLOCK sweep scratch: bitmap image, per-tile counts, control block
    DevBuf d_dec, d_decin;          // KVEvents payload decode: its scratch, and the staged payloads of a host-buffer call
    PinBuf h_misc;
    // snapshot / restore (guarded by mu_w): the stager between the device and a caller's buffer, which may be pageable;
    // the device scratch (records, sort buffers) is released when the call returns
    DevBuf d_snap;
    Stager snap;
    // collective pod removal (kvidx_shard_remove_pods, guarded by mu_w): phase 0 ran on this handle with these masks and
    // neither phase 1 nor any write call has run since, so the removal bitmaps describe exactly that removal
    bool rm_armed = false;
    uint32_t rm_tiers = 0;
    uint64_t rm_pods[KVIDX_MAX_PODS / 64] = {};
    int write_phase1 = -1;          // -1: by batch size, 0: never, 1: always (phase 1 = hash_events_kernel)
    int64_t write_phase1_min = 1024; // engine hashes in a batch from which phase 1 pays
    int score_kernel = 2;          // 1 = v1 (thread per prompt, global tokens), 2 = tuned
    int score_path = 0;            // 0 = by batch size, 2 / 3 = always the plain / class round pipeline,
                                   // 4 = always the warp-per-prompt cooperative kernel
    int64_t coop_max = 2048;       // batches up to this many prompts use the warp-per-prompt cooperative kernel
    int64_t zerocopy_max = 32;     // host-buffer calls up to this many prompts skip the copy engine (tokens read from pinned host memory)
    std::unique_ptr<SubmitQueue> queue;    // coalesces concurrent host-buffer Score() callers (submit.cuh)
    // Batch-size thresholds, from a sweep of the forced paths on an H100 SXM (10 M-block index, bench.py's query mix): the
    // warp-per-prompt rounds beat the cooperative kernel from 4096 prompts (tie at 2048); the class pipeline beats them from
    // 131 072 prompts.
    int64_t classes_min = 131072;  // batches at least this large (and above coop_max) use the prefix-class round pipeline
    double classes_min_sharing = 0.85;   // ... if at least this fraction of the batch follows a representative in round 0
    DevBuf d_rounds;               // the round pipelines' scratch, carved per batch (ClassPlan / PlainPlan)
    int64_t host_chunk_tokens = 32ll << 20;   // tokens per H2D chunk of the host-buffer pipeline
    int rounds_trace = 0;
    int rounds_parts = 8;          // parts (streams) a large batch is split into
    int rounds_dedup = 2;          // round pipeline: 0 every prompt on its own, 1 prefix classes, 2 + partial followers
    int sort_prefix = 1;           // sort the batch by first-block fingerprint before the rounds
    int64_t rounds_overlap_min = 65536;   // batches from this size run as several parts (per-prompt rounds: two halves)
    OwnStream aux_stream[kMaxParts - 1]; OwnEvent ev_fork, ev_join[kMaxParts - 1];
    int64_t rounds_warp_max = 131072;      // per-prompt rounds: kernel P warp per prompt up to this many prompts
                                   // (faster than the lane-per-prompt kernel P at every size swept up to 131 072)
    // multi-part class pipeline: a part's kernel G on a low-priority stream, its short kernels (G2, H, P, R) on a high-priority one
    OwnStream hp_stream[kMaxParts], lp_stream[kMaxParts]; OwnEvent ev_g[kMaxParts], ev_r[kMaxParts];
    // the device prefix store (kvidx_text_store_*): its own lock, independent of the read and write sides
    std::mutex mu_text;
    std::unique_ptr<TextStore> text;
};

namespace {

// a sharded handle is usable once every peer shard has been mapped
int check_shards(kvidx* x) {
    for (uint32_t r = 0; r < (1u << x->tv.shard_bits); ++r)
        if (!x->tv.req_peer[r]) return fail(KVIDX_EINVAL, "shard %u of %u is not connected (kvidx_shard_import / kvidx_shard_attach)", r, 1u << x->tv.shard_bits);
    return 0;
}

unsigned long long reserve_stamps(kvidx* x, unsigned long long n) { return x->clock.fetch_add(n + 1); }

// removal bitmaps of a request table of `slots` slots: removed_slot (a bit per slot), then removed_home (a bit per home pair)
size_t remove_bitmap_bytes(uint64_t slots) { return slots / 8 + slots / 16; }

// The stream write kernels go to.  Exact-LRU mode keeps reads and writes on ONE stream (reads write recency stamps, so the
// two sides are not independent there); otherwise the write path has its own.
cudaStream_t wstream(kvidx* x) { return x->tv.req_stamp ? x->stream : x->own_wstream; }

int refresh_counters(kvidx* x) {
    CK(cudaMemcpyAsync(x->h_cnt, x->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, wstream(x)));
    CK(cudaStreamSynchronize(wstream(x)));
    return 0;
}

// req_tail: bytes allocated (and zeroed) behind the request slots -- a sharded handle keeps its removal bitmaps there
int alloc_tables(kvidx* x, uint64_t req_slots, uint64_t eng_slots, ReqSlot** req, EngSlot** eng, cudaStream_t st, size_t req_tail = 0) {
    *req = nullptr; *eng = nullptr;
    CK(cudaMalloc((void**)req, req_slots * sizeof(ReqSlot) + req_tail));
    cudaError_t e = cudaMalloc((void**)eng, eng_slots * sizeof(EngSlot));
    if (e != cudaSuccess) { cudaFree(*req); *req = nullptr; return fail(KVIDX_ENOMEM, "cudaMalloc of %llu engine slots: %s", (unsigned long long)eng_slots, cudaGetErrorString(e)); }
    CK(cudaMemsetAsync(*req, 0, req_slots * sizeof(ReqSlot) + req_tail, st));
    CK(cudaMemsetAsync(*eng, 0, eng_slots * sizeof(EngSlot), st));
    return 0;
}

// The fresh arrays of a rebuild: both tables of `slots` slots, and the exact-LRU stamps and CLOCK reference bits the handle
// keeps beside them.  Allocated all or nothing; whatever the rebuild has not handed to the handle is freed with this.
struct FreshTables {
    ReqSlot* req = nullptr; EngSlot* eng = nullptr;
    unsigned long long* stamp = nullptr;
    uint32_t *rref = nullptr, *eref = nullptr;
    FreshTables() = default;
    FreshTables(const FreshTables&) = delete;
    FreshTables& operator=(const FreshTables&) = delete;
    ~FreshTables() { cudaFree(req); cudaFree(eng); cudaFree(stamp); cudaFree(rref); cudaFree(eref); }
    int alloc(const TableView& tv, uint64_t slots, cudaStream_t st) {
        cudaError_t e = cudaMalloc((void**)&req, slots * sizeof(ReqSlot));
        if (e == cudaSuccess) e = cudaMalloc((void**)&eng, slots * sizeof(EngSlot));
        if (e == cudaSuccess && tv.req_stamp) e = cudaMalloc((void**)&stamp, slots * 8);
        if (e == cudaSuccess && tv.req_ref) e = cudaMalloc((void**)&rref, slots / 8);
        if (e == cudaSuccess && tv.req_ref) e = cudaMalloc((void**)&eref, slots / 8);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(KVIDX_ENOMEM, "cudaMalloc of two %llu-slot tables: %s", (unsigned long long)slots, cudaGetErrorString(e));
        }
        CK(cudaMemsetAsync(req, 0, slots * sizeof(ReqSlot), st));
        CK(cudaMemsetAsync(eng, 0, slots * sizeof(EngSlot), st));
        if (stamp) CK(cudaMemsetAsync(stamp, 0, slots * 8, st));
        if (rref) { CK(cudaMemsetAsync(rref, 0, slots / 8, st)); CK(cudaMemsetAsync(eref, 0, slots / 8, st)); }
        return 0;
    }
};

// Re-insert the live slots into fresh tables of `slots` slots each, dropping the tombstones: a compaction keeps the slot
// count, a growth (grow_tables, see ensure_room) raises it.  Exact-LRU stamps and CLOCK reference bits move with their keys.
// Caller holds mu_w and `tables` EXCLUSIVELY; every stream of the device is drained first (asynchronous Score() calls may
// still be reading the old tables).  A failed allocation (KVIDX_ENOMEM) leaves the handle exactly as it was.
//   unsharded: the fresh tables replace the old ones, which are freed only once the fresh ones are complete;
//   sharded  : peers have this shard mapped (CUDA IPC), so the fresh tables are copied back into the same allocation (same
//              slot count only).  The caller of kvidx_shard_compact guarantees that no rank touches the index meanwhile
//              (a barrier either side).
int rebuild(kvidx* x, bool in_place, uint64_t slots) {
    CK(cudaDeviceSynchronize());
    cudaStream_t st = wstream(x);
    const uint64_t rs = x->tv.req_mask + 1, es = x->tv.eng_mask + 1;
    FreshTables f;
    if (int rc = f.alloc(x->tv, slots, st)) return rc;
    const int T = 256;
    rebuild_req_kernel<<<(unsigned)((rs + T - 1) / T), T, 0, st>>>(x->tv.req, rs, f.req, slots - 1, x->tv.req_stamp, f.stamp, x->tv.req_ref, f.rref);
    rebuild_eng_kernel<<<(unsigned)((es + T - 1) / T), T, 0, st>>>(x->tv.eng, es, f.eng, slots - 1, x->tv.eng_ref, f.eref);
    x->launches += 2;
    CK(cudaGetLastError());
    // zero the tombstone counters on the device, and the CLOCK hands (slot positions of the old layout)
    CK(cudaMemsetAsync(&x->d_cnt->req_tomb, 0, sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(&x->d_cnt->eng_tomb, 0, sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(x->d_cnt->hand, 0, sizeof x->d_cnt->hand, st));
    if (in_place) {
        CK(cudaMemcpyAsync(x->tv.req, f.req, rs * sizeof(ReqSlot), cudaMemcpyDeviceToDevice, st));
        CK(cudaMemcpyAsync(x->tv.eng, f.eng, es * sizeof(EngSlot), cudaMemcpyDeviceToDevice, st));
        CK(cudaStreamSynchronize(st));
    } else {
        CK(cudaStreamSynchronize(st));
        cudaFree(x->tv.req); cudaFree(x->tv.eng); cudaFree(x->tv.req_stamp); cudaFree(x->tv.req_ref); cudaFree(x->tv.eng_ref);
        x->tv.req = f.req; x->tv.eng = f.eng; x->tv.req_stamp = f.stamp; x->tv.req_ref = f.rref; x->tv.eng_ref = f.eref;
        f.req = nullptr; f.eng = nullptr; f.stamp = nullptr; f.rref = nullptr; f.eref = nullptr;
        x->tv.req_mask = slots - 1; x->tv.eng_mask = slots - 1;
        x->tv.req_peer[0] = x->tv.req; x->tv.eng_peer[0] = x->tv.eng;
    }
    ++x->rebuilds;
    return refresh_counters(x);
}

// grow_tables: the slot count the growth rule gives for `live` keys and `incoming` new ones.  It is the current count when
// the tables are at their ceiling C (always, for fixed tables) or 4 (live + incoming) fits in them; otherwise
// min(C, the smallest power of two >= 4 (live + incoming)), which keeps the load at most 1/4, the fixed default's.
uint64_t grow_target(const kvidx* x, uint64_t live, uint64_t incoming) {
    const uint64_t s = x->tv.req_mask + 1, need = live + incoming;
    if (s >= x->grow_max) return s;
    if (need >= x->grow_max / 4) return x->grow_max;
    return 4 * need > s ? pow2ceil(4 * need) : s;
}

// Make room for up to `incoming` new keys in each table before a write batch.  Caller holds mu_w and NOT `tables`.
//   unsharded: this handle's counters decide.  A growable handle below its ceiling first grows both tables by the rule of
//              grow_target (one rebuild, however many doublings); then tombstones are compacted away when they are what
//              fills the table.  A growth that cannot allocate leaves the call on the old tables under these rules;
//   sharded  : the keys may land on any owner, so every owner's counters are read (through the mapped peer memory) and
//              each must have room for the whole batch; compaction is the collective kvidx_shard_compact.
int ensure_room(kvidx* x, uint64_t incoming) {
    // CLOCK: every eviction leaves a tombstone, so under churn tombstones are the steady state.  The host copy of the counters
    // is stale after an asynchronous batch (kvidx_apply_events_dev never reads them back): read them here, after the batches
    // queued before this call, so that the tombstones are compacted before they fill the table.  A growable handle below its
    // ceiling reads them for the same reason: the growth rule counts the live keys those batches added.
    const bool growable = x->tv.req_mask + 1 < x->grow_max;
    if (x->tv.req_ref || growable) { int rc = refresh_counters(x); if (rc) return rc; }
    std::string grow_failed;
    if (growable) {
        const uint64_t want = grow_target(x, std::max(x->h_cnt->req_full, x->h_cnt->eng_full), incoming);
        if (want > x->tv.req_mask + 1) {
            std::unique_lock<std::shared_mutex> tl(x->tables);
            if (int rc = rebuild(x, false, want)) {
                if (rc != KVIDX_ENOMEM) return rc;
                grow_failed = "; growing them to " + std::to_string(want) + " slots failed: " + g_err;
            }
        }
    }
    const uint64_t rs = x->tv.req_mask + 1, es = x->tv.eng_mask + 1;
    auto over = [&](uint64_t full, uint64_t tomb, uint64_t slots) { return (full + tomb + incoming) * 10 > slots * 8; };
    if (x->tv.shard_bits) {
        const uint32_t ns = 1u << x->tv.shard_bits;
        gather_counters_kernel<<<1, 32, 0, wstream(x)>>>(x->tv, x->d_cnt_all);
        x->launches += 1;
        CK(cudaMemcpyAsync(x->h_cnt_all, x->d_cnt_all, sizeof(Counters) * ns, cudaMemcpyDeviceToHost, wstream(x)));
        CK(cudaStreamSynchronize(wstream(x)));
        for (uint32_t r = 0; r < ns; ++r) {
            const Counters& c = x->h_cnt_all[r];
            if ((c.req_full + c.req_tomb + incoming) * 10 > rs * 9 || (c.eng_full + c.eng_tomb + incoming) * 10 > es * 9)
                return fail(KVIDX_ENOSPC, "shard %u full: %llu keys + %llu tombstones + %llu incoming in %llu slots%s", r,
                            (unsigned long long)c.req_full, (unsigned long long)c.req_tomb, (unsigned long long)incoming, (unsigned long long)rs,
                            (c.req_tomb || c.eng_tomb) ? " (kvidx_shard_compact on every rank drops the tombstones)" : "");
        }
        return 0;
    }
    const Counters& c = *x->h_cnt;
    if (over(c.req_full, c.req_tomb, rs) || over(c.eng_full, c.eng_tomb, es)) {
        if (c.req_tomb || c.eng_tomb) {
            std::unique_lock<std::shared_mutex> tl(x->tables);
            int rc = rebuild(x, false, rs);
            if (rc) return rc;
        }
        const Counters& d = *x->h_cnt;
        if ((d.req_full + incoming) * 10 > rs * 9 || (d.eng_full + incoming) * 10 > es * 9)
            return fail(KVIDX_ENOSPC, "table full: %llu request keys + %llu incoming in %llu slots%s",
                        (unsigned long long)d.req_full, (unsigned long long)incoming, (unsigned long long)rs, grow_failed.c_str());
    }
    return 0;
}

// exact-LRU mode: after a write call, evict least-recently-used keys until both maps respect InMemoryIndexConfig.Size
// (lru.Cache evicts the back of its list when Len() > size; in_memory.go:59,64).  Exact at call granularity.
int enforce_caps(kvidx* x) {
    if (!x->tv.req_stamp) return 0;
    int rc = refresh_counters(x);
    if (rc) return rc;
    CK(x->d_misc.need(64));
    unsigned long long* d_v = x->d_misc.as<unsigned long long>();
    const uint64_t rs = x->tv.req_mask + 1, es = x->tv.eng_mask + 1;
    const int T = 256;
    cudaStream_t st = wstream(x);
    while (x->h_cnt->req_full > x->tv.capacity) {
        CK(cudaMemsetAsync(d_v, 0xff, 8, st));
        lru_min_req_kernel<<<(unsigned)((rs + T - 1) / T), T, 0, st>>>(x->tv.req, x->tv.req_stamp, rs, d_v);
        lru_drop_req_kernel<<<(unsigned)((rs + T - 1) / T), T, 0, st>>>(x->tv.req, x->tv.req_stamp, rs, d_v, x->d_cnt);
        x->launches += 2;
        CK(cudaGetLastError());
        if ((rc = refresh_counters(x))) return rc;
    }
    while (x->h_cnt->eng_full > x->tv.capacity) {
        CK(cudaMemsetAsync(d_v, 0xff, 8, st));
        lru_min_eng_kernel<<<(unsigned)((es + T - 1) / T), T, 0, st>>>(x->tv.eng, es, d_v);
        lru_drop_eng_kernel<<<(unsigned)((es + T - 1) / T), T, 0, st>>>(x->tv.eng, es, d_v, x->d_cnt);
        x->launches += 2;
        CK(cudaGetLastError());
        if ((rc = refresh_counters(x))) return rc;
    }
    return 0;
}

// CLOCK mode: queue the sweeps that bring both tables back to `capacity` keys (kernels_clock.cuh) on the write stream.
// The excess is read from the counters on the device, so this never waits for the device.  Caller holds mu_w and
// `tables` (shared or exclusive).
int clock_sweep(kvidx* x) {
    if (!x->tv.req_ref) return 0;
    const uint64_t slots = x->tv.req_mask + 1;        // both tables have the same slot count
    const uint64_t words = slots / 32, tiles = (slots + kSweepTile - 1) / kSweepTile;
    uint32_t* snap; unsigned long long* tile_cnt; SweepCtl* ctl;
    CK(carve(x->d_sweep, [&](Carver& c) { snap = c.take<uint32_t>(words); tile_cnt = c.take<unsigned long long>(tiles * 2); ctl = c.take<SweepCtl>(1); }));
    cudaStream_t st = wstream(x);
    const unsigned grid = (unsigned)std::min<uint64_t>(tiles, (uint64_t)x->sm_count * 8);
    const unsigned wgrid = (unsigned)std::min<uint64_t>((words + 255) / 256, (uint64_t)x->sm_count * 8);
    Counters* c = x->d_cnt;
    const uint64_t cap = x->tv.capacity;
    sweep_snap_kernel<<<wgrid, 256, 0, st>>>(x->tv.req_ref, snap, words, &c->req_full, cap);
    sweep_count_kernel<ReqSlot><<<grid, kSweepThreads, 0, st>>>(x->tv.req, x->tv.req_mask, snap, &c->req_full, cap, &c->hand[0], tile_cnt);
    sweep_cut_kernel<ReqSlot><<<1, kCutThreads, 0, st>>>(x->tv.req, x->tv.req_mask, snap, &c->req_full, cap, &c->hand[0], tile_cnt, ctl, &c->sweeps, &c->turns2);
    sweep_apply_kernel<ReqSlot><<<grid, kSweepThreads, 0, st>>>(x->tv.req, x->tv.req_mask, x->tv.req_ref, snap, ctl, &c->req_full, &c->req_tomb, &c->cap_evicted[0]);
    sweep_snap_kernel<<<wgrid, 256, 0, st>>>(x->tv.eng_ref, snap, words, &c->eng_full, cap);
    sweep_count_kernel<EngSlot><<<grid, kSweepThreads, 0, st>>>(x->tv.eng, x->tv.eng_mask, snap, &c->eng_full, cap, &c->hand[1], tile_cnt);
    sweep_cut_kernel<EngSlot><<<1, kCutThreads, 0, st>>>(x->tv.eng, x->tv.eng_mask, snap, &c->eng_full, cap, &c->hand[1], tile_cnt, ctl, &c->sweeps, &c->turns2);
    sweep_apply_kernel<EngSlot><<<grid, kSweepThreads, 0, st>>>(x->tv.eng, x->tv.eng_mask, x->tv.eng_ref, snap, ctl, &c->eng_full, &c->eng_tomb, &c->cap_evicted[1]);
    x->launches += 8;
    CK(cudaGetLastError());
    return 0;
}

// The key cap of a synchronous write call: exact LRU or CLOCK, then the counters as the call leaves them.
int cap_keys(kvidx* x) {
    if (!x->tv.req_ref) return enforce_caps(x);
    int rc = clock_sweep(x);
    return rc ? rc : refresh_counters(x);
}

// ---- Call scopes ------------------------------------------------------------------------------------------------------
// Locks of a call.  Read-side calls take mu_r (+ mu_w in exact-LRU mode, where everything is serialised as in round 1),
// write-side calls mu_w; both hold `tables` shared while they launch.  Only rebuild() (through ensure_room, or a growable
// handle's restore) and the calls that swap or map tables take `tables` exclusively.
enum : unsigned {
    kShards = 1,          // begin: every peer shard must be mapped (check_shards)
    kAfterWrites = 2,     // begin (read): order the call's stream after the last asynchronous write batch (ev_write)
    kDisarm = 4,          // begin (write): a pending collective pod removal is void (kvidx_shard_remove_pods)
};

struct ReadCall {
    kvidx* x;
    std::unique_lock<std::mutex> w, r;
    std::shared_lock<std::shared_mutex> t;
    explicit ReadCall(kvidx* x) : x(x) {
        if (x->tv.req_stamp) w = std::unique_lock<std::mutex>(x->mu_w);
        r = std::unique_lock<std::mutex>(x->mu_r);
        t = std::shared_lock<std::shared_mutex>(x->tables);
    }
    int begin(unsigned flags) { return begin(flags, x->stream); }
    int begin(unsigned flags, cudaStream_t st) {
        CK(cudaSetDevice(x->device));
        if (flags & kShards) { if (int rc = check_shards(x)) return rc; }
        if (flags & kAfterWrites) CK(cudaStreamWaitEvent(st, x->ev_write, 0));
        return 0;
    }
    // after an error: copies may still read the caller's buffers and the handle's scratch, so the streams the call used are
    // drained before the caller gets its buffers back, and the sticky error is cleared (the call's error text is kept)
    static int end(int rc, std::initializer_list<cudaStream_t> streams) {
        if (!rc) return 0;
        const std::string keep = g_err;
        for (cudaStream_t s : streams) cudaStreamSynchronize(s);
        cudaGetLastError();
        g_err = keep;
        return rc;
    }
};

// The counters a synchronous write call compares after its launch
struct WriteTally { unsigned long long dropped, nospc; };

// A write call holds mu_w throughout, and takes `tables` shared (share) or exclusively (exclusive) for its launches.
// ensure_room may rebuild the tables, taking `tables` exclusively itself, so it runs only inside share_with_room: before
// the call holds them.
struct WriteCall {
    kvidx* x;
    std::unique_lock<std::mutex> w;
    std::shared_lock<std::shared_mutex> t;
    std::unique_lock<std::shared_mutex> tx;
    explicit WriteCall(kvidx* x) : x(x), w(x->mu_w) {}
    int begin(unsigned flags) {
        if (flags & kDisarm) x->rm_armed = false;
        CK(cudaSetDevice(x->device));
        if (flags & kShards) { if (int rc = check_shards(x)) return rc; }
        return 0;
    }
    void share() { t = std::shared_lock<std::shared_mutex>(x->tables); }
    int share_with_room(uint64_t incoming) {
        if (int rc = ensure_room(x, incoming)) return rc;
        share();
        return 0;
    }
    void exclusive() { tx = std::unique_lock<std::shared_mutex>(x->tables); }
    // grow_tables: rebuild into `slots` slots part way through a call that holds `tables` shared (kvidx_restore grows the
    // empty tables once the image has passed validation).  No other writer runs meanwhile: the call keeps mu_w.
    int grow_shared(uint64_t slots) {
        t.unlock();
        int rc;
        { std::unique_lock<std::shared_mutex> tl(x->tables); rc = rebuild(x, false, slots); }
        t.lock();
        return rc;
    }
    WriteTally tally() const { return WriteTally{x->h_cnt->dropped_events, x->h_cnt->nospc}; }
    // The end of a synchronous write batch: the counters read back, the events it dropped, the inserts a full shard refused,
    // then the key cap.
    int settle(const WriteTally& before, int64_t* n_dropped_out) {
        if (int rc = refresh_counters(x)) return rc;
        if (n_dropped_out) *n_dropped_out = (int64_t)(x->h_cnt->dropped_events - before.dropped);
        if (x->h_cnt->nospc != before.nospc) return fail(KVIDX_ENOSPC, "%llu inserts refused: the owning shard is full", x->h_cnt->nospc - before.nospc);
        return cap_keys(x);
    }
};

int launch_score_rounds_plain(kvidx* x, const ScoreArgs& a, cudaStream_t st, int64_t max_blocks);

// ---- Round-pipeline batch plans ------------------------------------------------------------------------------------
// Both round pipelines take a batch's scratch from one device arena, kvidx::d_rounds, carved by the plan.  Parts start on
// kPartSlots boundaries: the kernels' vector accesses of a part's slice stay aligned (kernel C reads fate 8 slots at a
// time; kernels H and P clear nfol and need_snap by words, map and grp by 4 words).

// A batch of n prompts in np parts: part q holds slots off[q] .. off[q] + size[q] of the sorted batch.  Every part but the
// last ones holds ceil(n / np) prompts rounded up to kPartSlots; the last ones hold fewer, or none.
constexpr int64_t kPartSlots = 32;
static_assert(kPartSlots % 8 == 0, "per-slot arrays are read 8 bytes and cleared 4 words at a time");
struct PartSplit {
    int np;
    int64_t per, off[kMaxParts] = {}, size[kMaxParts] = {};
    PartSplit(int64_t n, int parts) : np(parts), per(((n + parts - 1) / parts + kPartSlots - 1) / kPartSlots * kPartSlots) {
        for (int q = 0; q < np; ++q) { off[q] = std::min(n, q * per); size[q] = std::min(per, n - off[q]); }
    }
    PartSizes sizes() const { PartSizes ps{}; for (int q = 0; q < kMaxParts; ++q) ps.n[q] = (unsigned int)size[q]; return ps; }
};

// rounds_setup's sections, the first of both plans
struct SetupBufs {
    RoundCounters* cnt;
    uint32_t* order;                     // the batch's prompts in sorted order: round 0's list
    uint64_t* fp; uint64_t* fp_sorted; uint32_t* idx;    // first-block fingerprints by prompt, the same sorted, the prompt ids
    void* sort; size_t sort_bytes = 0;   // cub's scratch (sort_prefix)
    void carve(Carver& c, int64_t n) {
        cnt = c.take<RoundCounters>(1); order = c.take<uint32_t>(n);
        fp = c.take<uint64_t>(n); fp_sorted = c.take<uint64_t>(n); idx = c.take<uint32_t>(n);
        sort = c.take<uint8_t>(sort_bytes);
    }
};

// The class pipeline: `b` holds the batch-wide per-slot arrays (part q's slice starts at its offset) and, back to back, every
// part's election map and grp, nfol and need_snap, and kernel C's tile words.
struct ClassPlan {
    int64_t n; PartSplit s;
    int64_t ctiles;                      // kernel C's tiles per part (part 0 is the largest)
    uint64_t map_slots;                  // a part's election map: 4 buckets per prompt, at least 1024
    SetupBufs su{};
    RoundBufs b{};
    ClassPlan(int64_t n, int np) : n(n), s(n, np), ctiles((s.size[0] + kCompactTile - 1) / kCompactTile),
                                   map_slots(pow2ceil((uint64_t)std::max<int64_t>(4 * ((n + np - 1) / np), 1024))) {}
    size_t map_words() const { return (size_t)s.np * (map_slots + s.per); }      // each part's map, then its grp
    size_t flag_bytes() const { return (size_t)s.np * 2 * s.per; }               // each part's nfol, then its need_snap
    size_t scan_words() const { return (size_t)s.np * ctiles; }
    void carve(Carver& c) {
        su.carve(c, n);
        b.live[0] = c.take<LiveRec>(n); b.live[1] = c.take<LiveRec>(n);
        b.pst[0] = c.take<PromptState>(n); b.pst[1] = c.take<PromptState>(n);
        b.keys = c.take<uint64_t>((size_t)n * kRoundBlocks);
        b.nbr = c.take<uint32_t>(n); b.role = c.take<uint32_t>(n);
        b.fate = c.take<uint8_t>(n); b.dmin = c.take<uint8_t>(n);
        b.hl = c.take<uint32_t>(n); b.fl = c.take<uint2>(n);
        b.anch = c.take<uint32_t>(n); b.apos = c.take<uint32_t>(n); b.nmap = c.take<uint32_t>(n);
        b.rec = c.take<uint4>(n); b.drec = c.take<uint4>(n);
        b.nwalk = c.take<uint8_t>(n);
        b.snap_run = c.take<uint8_t>((size_t)n * kRoundBlocks); b.snap_alive = c.take<uint16_t>((size_t)n * kRoundBlocks);
        b.snap_bt = c.take<uint8_t>((size_t)n * kRoundBlocks * kMaxEnt); b.snap_sc = c.take<double>((size_t)n * kRoundBlocks * kMaxEnt);
        b.map = c.take<uint32_t>(map_words());
        b.nfol = c.take<uint8_t>(flag_bytes());
        b.scan = c.take<unsigned long long>(scan_words());
    }
    RoundBufs part(int q) const {
        const int64_t o = s.off[q];
        RoundBufs r = b;
        r.live[0] += o; r.live[1] += o; r.pst[0] += o; r.pst[1] += o;
        r.keys += o; r.nbr += o; r.role += o; r.fate += o; r.dmin += o; r.hl += o; r.fl += o;
        r.anch += o; r.apos += o; r.nmap += o; r.rec += o; r.drec += o; r.nwalk += o;
        r.snap_run += o * kRoundBlocks; r.snap_alive += o * kRoundBlocks;
        r.snap_bt += o * kRoundBlocks * kMaxEnt; r.snap_sc += o * kRoundBlocks * kMaxEnt;
        r.part_size = (uint32_t)((s.size[q] + kPartSlots - 1) / kPartSlots * kPartSlots);
        r.map = b.map + q * (map_slots + s.per); r.map_mask = (uint32_t)(map_slots - 1); r.grp = r.map + map_slots;
        r.nfol = b.nfol + q * 2 * s.per; r.need_snap = r.nfol + s.per;
        r.scan = b.scan + q * ctiles;
        r.n_act = su.cnt->part[q].n_act; r.n_hl = su.cnt->part[q].n_hl; r.stat = su.cnt->stat[q];
        return r;
    }
};

// The per-prompt rounds.  Keys are prompt-major for the warp-per-prompt kernel P (pm: a half's rows start at its offset
// times kRoundBlocks), block-major for the lane-per-prompt one.
struct PlainPlan {
    int64_t n; PartSplit s; bool pm;
    SetupBufs su{};
    plain::RoundBufs b{};
    PlainPlan(int64_t n, int np, bool pm) : n(n), s(n, np), pm(pm) {}
    void carve(Carver& c) {
        su.carve(c, n);
        b.act[0] = su.order; b.act[1] = c.take<uint32_t>(n);
        b.hstate = c.take<uint64_t>(n); b.pst = c.take<PromptState>(n);
        b.keys = c.take<uint64_t>((size_t)n * kRoundBlocks); b.nbr = c.take<uint32_t>(n);
    }
    plain::RoundBufs part(int q) const {
        const int64_t o = s.off[q];
        plain::RoundBufs r = b;
        r.act[0] += o; r.act[1] += o; r.keys += pm ? o * kRoundBlocks : o; r.nbr += o;
        r.n_act = su.cnt->part[q].n_act;
        return r;
    }
};

// Sizes d_rounds for plan p (growing it as DevBuf::need does; what it held is dropped) and carves p's sections from it.
template <class Plan> int carve_rounds(kvidx* x, const ScoreArgs& a, cudaStream_t st, Plan& p) {
    if (x->sort_prefix)
        CK(cub::DeviceRadixSort::SortPairs(nullptr, p.su.sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                           (uint32_t*)nullptr, (int)a.n_prompts, 32, 64, st));
    CK(carve(x->d_rounds, [&](Carver& c) { p.carve(c); }));
    return 0;
}

// Batch setup of both round pipelines: clear the counters, fingerprint every prompt's first block and set the parts' first
// list lengths (rounds_init_kernel), and with sort_prefix order the batch by fingerprint into su.order.
int rounds_setup(kvidx* x, const ScoreArgs& a, const SetupBufs& su, const PartSizes& ps, cudaStream_t st) {
    const int64_t n = a.n_prompts;
    CK(cudaMemsetAsync(su.cnt, 0, sizeof(RoundCounters), st));
    rounds_init_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, x->tv.block_size, su.cnt, su.fp, x->sort_prefix ? su.idx : su.order, ps);
    x->launches += 1;
    CK(cudaGetLastError());
    if (x->sort_prefix) {
        size_t tmp = su.sort_bytes;
        CK(cub::DeviceRadixSort::SortPairs(su.sort, tmp, su.fp, su.fp_sorted, su.idx, su.order, (int)n, 32, 64, st));
        x->launches += 5;     // cub: histogram + 4 onesweep passes (the top 32 fingerprint bits order the groups well enough)
    }
    return 0;
}

// Large batches: rounds of group / hash / walk / resolve / compact kernels (kernels_rounds.cuh).  max_blocks < 0: computed on the
// device.  The sorted batch is split into parts that run their rounds on separate streams, so that one part's
// latency-bound kernels (the serial FNV chain of few representatives, the dependent probes) share the SMs with
// another part's bandwidth-bound ones.
int launch_score_rounds(kvidx* x, const ScoreArgs& a, cudaStream_t st, int64_t max_blocks) {
    const int64_t n = a.n_prompts;
    ClassPlan p(n, n >= x->rounds_overlap_min ? std::max(1, std::min(kMaxParts, x->rounds_parts)) : 1);
    if (int rc = carve_rounds(x, a, st, p)) return rc;
    const int np = p.s.np;
    RoundBufs rb[kMaxParts]{};
    for (int q = 0; q < np; ++q) rb[q] = p.part(q);
    if (int rc = rounds_setup(x, a, p.su, p.s.sizes(), st)) return rc;
    // Is the batch worth it?  The class pipeline pays a token pass and five kernels per round; with few prompts per distinct
    // prefix the per-prompt rounds are faster.  The sorted first-block
    // fingerprints tell before anything is spent: count the distinct ones, and hand the batch over if more than 15 % of the
    // prompts start differently from their neighbour.  (The device-resident entry point waits for the block count here anyway.)
    const bool adaptive = x->score_path == 0 && x->rounds_dedup && x->sort_prefix && x->classes_min_sharing > 0.0;
    if (adaptive) {
        count_distinct_prefixes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p.su.fp_sorted, n, &p.su.cnt->distinct);
        x->launches += 1;
    }
    if (max_blocks < 0 || adaptive) {
        unsigned long long mb[2] = {0, 0};           // max_blocks, distinct
        CK(cudaMemcpyAsync(mb, &p.su.cnt->max_blocks, sizeof mb, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (max_blocks < 0) max_blocks = (int64_t)mb[0];
        if (adaptive && (double)mb[1] > (1.0 - x->classes_min_sharing) * (double)n) {
            if (x->rounds_trace) fprintf(stderr, "[kvidx rounds] %llu distinct first blocks among %lld prompts: per-prompt rounds instead\n", mb[1], (long long)n);
            return launch_score_rounds_plain(x, a, st, max_blocks);
        }
    }
    int64_t rounds = (max_blocks + kRoundBlocks - 1) / kRoundBlocks;
    if (x->rounds_dedup >= 2) rounds += 1;            // a prompt that left its class mid-chunk runs unaligned from there: one more round
    if (rounds < 1) rounds = 1;                       // round 0 also retires the prompts that have no full block
    live_init_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, x->tv.block_size, p.su.order, p.b.live[0], x->tv.init_hash);
    x->launches += 1;
    cudaStream_t strm[kMaxParts];
    strm[0] = st;
    for (int q = 1; q < kMaxParts; ++q) strm[q] = x->aux_stream[q - 1];
    CK(cudaMemsetAsync(p.b.map, 0xff, p.map_words() * 4, st));
    CK(cudaMemsetAsync(p.b.nfol, 0, p.flag_bytes(), st));
    CK(cudaMemsetAsync(p.b.scan, 0, p.scan_words() * 8, st));     // kernel C's tile words: nothing published
    if (np > 1) {
        CK(cudaEventRecord(x->ev_fork, st));
        for (int q = 1; q < np; ++q) CK(cudaStreamWaitEvent(strm[q], x->ev_fork, 0));
    }
    const auto t_enq = std::chrono::steady_clock::now();
    // With several parts, kernel G of a part runs on a low-priority stream and the part's short kernels on a high-priority one:
    // a CTA slot that frees up goes to a waiting latency-bound kernel before the next G CTA (otherwise the parts drift into lock
    // step: all in G sharing the bandwidth, then all in the short kernels with DRAM idle -- scripts/timeline.py).
    const bool prio = np > 1;
    cudaStream_t sS[kMaxParts], sG[kMaxParts];
    for (int q = 0; q < kMaxParts; ++q) { sS[q] = prio ? x->hp_stream[q] : strm[q]; sG[q] = prio ? x->lp_stream[q] : strm[q]; }
    if (prio) for (int q = 0; q < np; ++q) { CK(cudaStreamWaitEvent(sS[q], x->ev_fork, 0)); CK(cudaStreamWaitEvent(sG[q], x->ev_fork, 0)); }
    constexpr int T = 256, W = T / 32;                // threads / warps of the short kernels' CTAs
    const int trace = x->rounds_trace == 1;           // count the token work of every round (kernels_rounds.cuh: RoundBufs::stat)
    unsigned int stat0[kMaxParts][4] = {};            // ... the counts up to the last round, to print each round's own
    // The grids below are capped at CTAs per SM: what fills the machine with one part (two for the list and finish kernels),
    // less with more parts sharing it.
    for (int64_t r = 0; r < rounds; ++r) {
        const int cur = (int)(r & 1);
        for (int q = 0; q < np; ++q) {
            const int64_t m = p.s.size[q];
            if (m <= 0) continue;
            const unsigned ggrid = (unsigned)std::min<int64_t>((m + kGroupThreads / 32 * kGroupTile - 1) / (kGroupThreads / 32 * kGroupTile), (int64_t)x->sm_count * (np == 1 ? 3 : 2));
            if (prio && r > 0) CK(cudaStreamWaitEvent(sG[q], x->ev_r[q], 0));       // this part's previous round has built the live list
            group_round_kernel<16><<<ggrid, kGroupThreads, sizeof(GroupSmem), sG[q]>>>(x->tv, a, rb[q], cur, (int)r, x->rounds_dedup, trace);
            if (prio) { CK(cudaEventRecord(x->ev_g[q], sG[q])); CK(cudaStreamWaitEvent(sS[q], x->ev_g[q], 0)); }
            const unsigned lgrid = (unsigned)std::min<int64_t>((m + T - 1) / T, (int64_t)x->sm_count * (np <= 2 ? 8 : 4));
            group_lists_kernel<16><<<lgrid, T, 0, sS[q]>>>(x->tv, a, rb[q], cur, (int)r, x->rounds_dedup >= 2, trace);
        }
        for (int q = 0; q < np; ++q) {
            const int64_t m = p.s.size[q];
            if (m <= 0) continue;
            const unsigned hgrid = (unsigned)std::min<int64_t>((m + kHashThreads - 1) / kHashThreads, (int64_t)x->sm_count * (np == 1 ? 4 : 2));
            hash_round_kernel<16><<<hgrid, kHashThreads, sizeof(HashSmem<16>), sS[q]>>>(x->tv, a, rb[q], cur, (int)r, trace);
            const unsigned wgrid = (unsigned)std::min<int64_t>((m + W - 1) / W, (int64_t)x->sm_count * (np == 1 ? 8 : 4));
            if (x->tv.req_ref) walk_round_kernel<true><<<wgrid, T, 0, sS[q]>>>(x->tv, a, rb[q], cur, (int)r);
            else walk_round_kernel<false><<<wgrid, T, 0, sS[q]>>>(x->tv, a, rb[q], cur, (int)r);
            const unsigned rgrid = (unsigned)std::min<int64_t>((m + T - 1) / T, (int64_t)x->sm_count * (np <= 2 ? 8 : 4));
            finish_round_kernel<16><<<rgrid, T, sizeof(DetachWarp) * W, sS[q]>>>(x->tv, a, rb[q], cur, (int)r, x->rounds_dedup >= 2, x->rounds_trace);
            compact_round_kernel<<<(unsigned)((m + kCompactTile - 1) / kCompactTile), kCompactThreads, 0, sS[q]>>>(rb[q], cur, (int)r);
            if (prio && r + 1 < rounds) CK(cudaEventRecord(x->ev_r[q], sS[q]));
            x->launches += 6;
            if (trace) {      // debugging aid: list sizes and token work of this round (synchronises)
                RoundCounters c;
                CK(cudaMemcpyAsync(&c, p.su.cnt, sizeof c, cudaMemcpyDeviceToHost, sS[q]));
                CK(cudaStreamSynchronize(sS[q]));
                const RoundCounters::Part& l = c.part[q];
                const unsigned int* s = c.stat[q];
                fprintf(stderr, "[kvidx rounds] round %lld part %d: live %u -> representatives %u, followers %u, partial %u (%u blocks walked alone) -> next %u;"
                        " G streamed %u chunks, %u losers re-read, G2 compared %u, H hashed %u blocks\n",
                        (long long)r, q, l.n_act[cur], l.n_hl[0], l.n_hl[1], l.n_hl[2], l.n_hl[3], l.n_act[cur ^ 1], s[0] - stat0[q][0], s[1] - stat0[q][1], s[2] - stat0[q][2], s[3] - stat0[q][3]);
                for (int k = 0; k < 4; ++k) stat0[q][k] = s[k];
            }
        }
    }
    if (x->rounds_trace == 2) fprintf(stderr, "[kvidx rounds] host enqueue of %lld rounds x %d parts: %.3f ms\n", (long long)rounds, np,
                                      std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_enq).count());
    CK(cudaGetLastError());
    for (int q = 1; q < np; ++q) { CK(cudaEventRecord(x->ev_join[q - 1], sS[q])); CK(cudaStreamWaitEvent(st, x->ev_join[q - 1], 0)); }
    if (prio) { CK(cudaEventRecord(x->ev_g[0], sS[0])); CK(cudaStreamWaitEvent(st, x->ev_g[0], 0)); }
    return 0;
}

// Medium batches: hash / walk rounds, every prompt on its own (kernels_rounds_plain.cuh); two halves on two streams.
int launch_score_rounds_plain(kvidx* x, const ScoreArgs& a, cudaStream_t st, int64_t max_blocks) {
    const int64_t n = a.n_prompts;
    const bool warp_walk = n <= x->rounds_warp_max;      // kernel P: warp per prompt (batch too small to fill the machine lane per prompt)
    PlainPlan p(n, n >= x->rounds_overlap_min ? 2 : 1, warp_walk);
    if (int rc = carve_rounds(x, a, st, p)) return rc;
    const plain::RoundBufs rb[2] = {p.part(0), p.part(1)};
    if (int rc = rounds_setup(x, a, p.su, p.s.sizes(), st)) return rc;
    if (max_blocks < 0) {
        unsigned long long mb = 0;
        CK(cudaMemcpyAsync(&mb, &p.su.cnt->max_blocks, sizeof mb, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        max_blocks = (int64_t)mb;
    }
    int64_t rounds = (max_blocks + kRoundBlocks - 1) / kRoundBlocks;
    if (rounds < 1) rounds = 1;                       // round 0 also retires the prompts that have no full block
    const int nh = p.s.size[1] > 0 ? 2 : 1;
    const int per_sm = nh == 2 ? 2 : 4;               // CTAs per SM of a half's lane-per-prompt kernels H and P
    cudaStream_t strm[2] = {st, x->aux_stream[0]};
    if (nh == 2) { CK(cudaEventRecord(x->ev_fork, st)); CK(cudaStreamWaitEvent(x->aux_stream[0], x->ev_fork, 0)); }
    for (int64_t r = 0; r < rounds; ++r) {
        const int cur = (int)(r & 1);
        for (int hlf = 0; hlf < nh; ++hlf) {
            const int64_t m = p.s.size[hlf];
            if (warp_walk) {      // 128-thread CTAs, three stages: 55 KB, four CTAs per SM
                const unsigned hg = (unsigned)std::min<int64_t>((m + 127) / 128, (int64_t)x->sm_count * 4);
                plain::hash_round_kernel<16, true><<<hg, 128, 4 * 3 * 32 * HashSmem<16>::kRow, strm[hlf]>>>(x->tv, a, rb[hlf], cur, (int)r);
            } else {
                const unsigned hgrid = (unsigned)std::min<int64_t>((m + kHashThreads - 1) / kHashThreads, (int64_t)x->sm_count * per_sm);
                plain::hash_round_kernel<16, false><<<hgrid, kHashThreads, sizeof(HashSmem<16>), strm[hlf]>>>(x->tv, a, rb[hlf], cur, (int)r);
            }
        }
        for (int hlf = 0; hlf < nh; ++hlf) {
            const int64_t m = p.s.size[hlf];
            if (warp_walk) {      // warp per prompt: 8 prompts per CTA iteration
                const unsigned pgrid = (unsigned)std::min<int64_t>((m + 7) / 8, (int64_t)x->sm_count * 8);
                plain::probe_round_warp_kernel<<<pgrid, plain::kProbeThreads, 0, strm[hlf]>>>(x->tv, a, rb[hlf], cur, (int)r);
                continue;
            }
            const unsigned pgrid = (unsigned)std::min<int64_t>((m + plain::kProbeThreads - 1) / plain::kProbeThreads, (int64_t)x->sm_count * per_sm);
            if (x->tv.req_ref) plain::probe_round_kernel<true><<<pgrid, plain::kProbeThreads, sizeof(plain::WalkSmem), strm[hlf]>>>(x->tv, a, rb[hlf], cur, (int)r);
            else plain::probe_round_kernel<false><<<pgrid, plain::kProbeThreads, sizeof(plain::WalkSmem), strm[hlf]>>>(x->tv, a, rb[hlf], cur, (int)r);
        }
        x->launches += 2 * nh;
    }
    CK(cudaGetLastError());
    if (nh == 2) { CK(cudaEventRecord(x->ev_join[0], x->aux_stream[0])); CK(cudaStreamWaitEvent(st, x->ev_join[0], 0)); }
    return 0;
}

// The prompts of a Score() call: tokens (steps 2-4, `p` uint32) or request keys (steps 3-4, `p` uint64).  Prompt i owns
// elements tok_off[i] .. tok_off[i+1] of p, with the offsets and everything else about the call in a ScoreArgs.
// A conversation turn (kvidx_score_turn*) is keys followed by tokens: `t` holds the tokens' CSR and where the new keys go
// (t.keys unused: the held keys are at p).
//
// A host-buffer call moves as CSR sections (Csr): its inputs (tokens, keys, or a turn's keys then its tokens) and, for a
// turn that wants them, the new keys it returns.  A section moved elsewhere is a View: its elements from the first
// moved prompt's on, that prompt's offsets on, and the first offset (the base the kernels subtract).
struct Csr {
    const void* p; const int64_t* off; size_t esz;      // prompt i owns elements off[i] .. off[i+1] of p, esz bytes each
    size_t bytes(int64_t i0, int64_t i1) const { return (size_t)(off[i1] - off[i0]) * esz; }
    uint8_t* at(int64_t i) const { return p ? static_cast<uint8_t*>(const_cast<void*>(p)) + (size_t)off[i] * esz : nullptr; }
    // are the elements of prompts 0 .. n pinned host memory (or none at all)?
    bool pinned(int64_t n) const { return off[n] == off[0] || is_device_accessible_host(p); }
};
struct View { const void* p; const int64_t* off; int64_t base; };

struct ScoreIn {
    const void* p; bool keys;
    TurnArgs t = {};
    bool turn() const { return t.tok_off != nullptr; }
    // the sections of the host call h: s[0 .. inputs) the inputs, then s[inputs] the new keys when wanted; -> their count
    int sections(const ScoreArgs& h, Csr s[3], int* inputs) const {
        int k = 0;
        s[k++] = Csr{p, h.tok_off, keys ? 8u : 4u};
        if (turn()) s[k++] = Csr{t.tok, t.tok_off, 4};
        *inputs = k;
        if (t.new_keys) s[k++] = Csr{t.new_keys, t.new_off, 8};
        return k;
    }
    // this call with its sections at v (as sections() lists them); a's offsets are set
    ScoreIn moved(const View* v, ScoreArgs& a) const {
        ScoreIn r{v[0].p, keys, t};
        a.tok = nullptr; a.tok_off = v[0].off; a.tok_base = v[0].base;
        if (turn()) { r.t.tok = static_cast<const uint32_t*>(v[1].p); r.t.tok_off = v[1].off; r.t.tok_base = v[1].base; }
        if (t.new_keys) {
            const View& nk = v[turn() ? 2 : 1];
            r.t.new_keys = static_cast<uint64_t*>(const_cast<void*>(nk.p)); r.t.new_off = nk.off; r.t.new_base = nk.base;
        }
        return r;
    }
};

// A Score() call of n prompts (offsets off) with dense result rows (scores: n x max_pods) or sparse ones (pods, scores:
// n x kMaxEnt, cnt: n); the prompts' elements are set where the call is launched.
ScoreArgs dense_args(const int64_t* off, int64_t n, const uint32_t* model, uint32_t model0, const uint64_t* filter, double* scores,
                     uint8_t* has_keys) {
    ScoreArgs a{};
    a.tok_off = off; a.n_prompts = n; a.model = model; a.model0 = model0; a.filter = filter; a.dense = scores; a.has_keys = has_keys;
    return a;
}
ScoreArgs sparse_args(const int64_t* off, int64_t n, const uint32_t* model, uint32_t model0, const uint64_t* filter, uint16_t* pods,
                      double* scores, uint8_t* cnt, uint8_t* has_keys) {
    ScoreArgs a = dense_args(off, n, model, model0, filter, nullptr, has_keys);
    a.sp_pods = pods; a.sp_scores = scores; a.sp_cnt = cnt;
    return a;
}

// Exact-LRU handles take the thread-per-prompt kernel: Lookup must touch every present key of a prompt (no early exit).
// So does KVIDX_SCORE_KERNEL=v1 as the cross-check, and so do token prompts of a block size the other token kernels' staging
// is not written for: every size but 16, 32, 64 and 128.  At 32, 64 and 128 only the warp-per-prompt kernel
// (coop_score_kernel) is built, so a token batch of n prompts takes it where it would at 16 (n <= coop_max, or
// KVIDX_SCORE_PATH=coop) and v1 otherwise; the round pipelines are 16-token only.
bool score_takes_v1(const kvidx* x, bool keys, int64_t n) {
    if (x->score_kernel == 1 || x->tv.req_stamp) return true;
    if (keys || x->tv.block_size == 16) return false;
    return !coop_block_size(x->tv.block_size) || !(x->score_path == 4 || (x->score_path == 0 && n <= x->coop_max));
}

// Does a batch of n prompts take a warp-per-prompt kernel: score_keys_kernel (keys, every size) or coop_score_kernel (small
// token batches)?  Both read their inputs in place, so from pinned host memory as well (score_host_zerocopy).
bool score_warp_per_prompt(const kvidx* x, bool keys, int64_t n) {
    return !score_takes_v1(x, keys, n) && (keys || x->score_path == 4 || (x->score_path == 0 && n <= x->coop_max));
}

// Does a conversation turn take the fused kernel (score_turn_kernel, one warp per prompt at every batch size, inputs read in
// place)?  At every block size the kernel is built for, on default and CLOCK handles; elsewhere it is composed of the hash,
// a concatenation and Score() from keys.
bool score_turn_fused(const kvidx* x) { return x->score_kernel != 1 && !x->tv.req_stamp && coop_block_size(x->tv.block_size); }

// Does the kernel of a call of n prompts read its inputs in place (score_host_zerocopy)?
bool reads_in_place(const kvidx* x, const ScoreIn& in, int64_t n) { return in.turn() ? score_turn_fused(x) : score_warp_per_prompt(x, in.keys, n); }

template <class E>
int launch_score_v1(kvidx* x, const ScoreArgs& a, const E* src, cudaStream_t st) {
    const int T = 128;
    unsigned long long sb = 0;
    if (x->tv.req_stamp) {
        // exact-LRU: a stamp per element of the call (score_kernel_v1), counted from the offsets.  They may be device memory
        // (the _dev entry points, the host pipeline's chunks): read back -- this mode serialises its calls anyway
        int64_t e[2];
        CK(cudaMemcpyAsync(&e[0], a.tok_off, 8, cudaMemcpyDefault, st));
        CK(cudaMemcpyAsync(&e[1], a.tok_off + a.n_prompts, 8, cudaMemcpyDefault, st));
        CK(cudaStreamSynchronize(st));
        sb = reserve_stamps(x, (unsigned long long)(e[1] - e[0]));
    }
    score_kernel_v1<<<(unsigned)((a.n_prompts + T - 1) / T), T, 0, st>>>(x->tv, src, a.tok_off, a.tok_base, a.n_prompts, a.model, a.model0, a.filter,
                                                                        a.dense, a.sp_pods, a.sp_scores, a.sp_cnt, a.has_keys, sb);
    x->launches += 1;
    return 0;
}

// Launch Score() over device-addressable inputs: the prompts' elements at in.p (a.tok is set here), the rest of the call in
// `a`.  max_blocks: the token batch's largest block count, for the round pipelines; < 0 computes it on the device.  The
// callers order the launch after the asynchronous write batches issued before (ev_write), once per call.
int launch_turn(kvidx* x, const ScoreIn& in, const ScoreArgs& a, cudaStream_t st);

int launch_score(kvidx* x, const ScoreIn& in, ScoreArgs a, cudaStream_t st, int64_t max_blocks = -1) {
    const int64_t n = a.n_prompts;
    if (n <= 0) return 0;
    if (int rc = check_shards(x)) return rc;
    if (in.turn()) return launch_turn(x, in, a, st);
    a.tok = in.keys ? nullptr : static_cast<const uint32_t*>(in.p);
    if (score_takes_v1(x, in.keys, n)) {
        const int rc = in.keys ? launch_score_v1(x, a, static_cast<const uint64_t*>(in.p), st) : launch_score_v1(x, a, a.tok, st);
        if (rc) return rc;
    } else if (in.keys) {
        // request keys: one warp per prompt at every batch size (kernels_keys.cuh)
        const int64_t ctas = std::min<int64_t>((n + kKeysWarps - 1) / kKeysWarps, (int64_t)x->sm_count * kKeysCtasPerSm);
        score_keys_kernel<<<(unsigned)ctas, kKeysThreads, 0, st>>>(x->tv, static_cast<const uint64_t*>(in.p), a);
        x->launches += 1;
    } else if (score_warp_per_prompt(x, false, n)) {
        // small batches: a warp per prompt, warp-cooperative hashing, TMA-staged tokens (kernels_coop.cuh)
        const int64_t ctas = std::min<int64_t>((n + kCoopWarps - 1) / kCoopWarps, (int64_t)x->sm_count * 4);
        coop_dispatch(x->tv.block_size, [&](auto bs) {
            coop_score_kernel<bs.value><<<(unsigned)ctas, kCoopThreads, sizeof(CoopSmem<bs.value>), st>>>(x->tv, a);
        });
        x->launches += 1;
    } else if (n < (1ll << 31)) {
        // path 2: plain rounds, 3: prefix classes; automatic: by batch size (the class pipeline has a fixed cost per round)
        const bool classes = x->score_path == 3 || (x->score_path == 0 && n >= x->classes_min);
        return classes ? launch_score_rounds(x, a, st, max_blocks) : launch_score_rounds_plain(x, a, st, max_blocks);
    } else {
        // the round pipelines index prompts with 32 bits; the thread-per-prompt kernel indexes them with 64
        if (int rc = launch_score_v1(x, a, a.tok, st)) return rc;
    }
    CK(cudaGetLastError());
    return 0;
}

// A conversation turn: a.tok_off / a.tok_base the held keys' CSR (keys at in.p), in.t the tokens and the new keys.  The fused
// kernel, or (score_turn_fused false) the composed path: its scratch is sized from the batch's key and token counts, read
// back from the offsets, then hash_keys_kernel_v1 hashes every prompt's new blocks from its last held key straight into
// the concatenated key CSR, turn_concat_kernel adds the held keys (and hands the new ones out) and Score() runs on the keys.
int launch_turn(kvidx* x, const ScoreIn& in, const ScoreArgs& a, cudaStream_t st) {
    const int64_t n = a.n_prompts;
    TurnArgs ta = in.t;
    ta.keys = static_cast<const uint64_t*>(in.p);
    if (score_turn_fused(x)) {
        const int64_t ctas = std::min<int64_t>((n + kCoopWarps - 1) / kCoopWarps, (int64_t)x->sm_count * 4);
        coop_dispatch(x->tv.block_size, [&](auto bs) {
            score_turn_kernel<bs.value><<<(unsigned)ctas, kCoopThreads, sizeof(CoopSmem<bs.value>), st>>>(x->tv, a, ta);
        });
        x->launches += 1;
        CK(cudaGetLastError());
        return 0;
    }
    int64_t e[4];
    CK(cudaMemcpyAsync(&e[0], a.tok_off, 8, cudaMemcpyDefault, st));
    CK(cudaMemcpyAsync(&e[1], a.tok_off + n, 8, cudaMemcpyDefault, st));
    CK(cudaMemcpyAsync(&e[2], ta.tok_off, 8, cudaMemcpyDefault, st));
    CK(cudaMemcpyAsync(&e[3], ta.tok_off + n, 8, cudaMemcpyDefault, st));
    CK(cudaStreamSynchronize(st));
    const uint32_t B = x->tv.block_size;
    const int64_t cap = (e[1] - e[0]) + (e[3] - e[2]) / B;             // >= the concatenated key count
    int64_t *cat_off, *new_dst; uint64_t *parent, *cat; uint8_t* pv;
    CK(carve(x->d_turn, [&](Carver& c) {
        cat_off = c.take<int64_t>(n + 1); new_dst = c.take<int64_t>(n); parent = c.take<uint64_t>(n); pv = c.take<uint8_t>(n);
        cat = c.take<uint64_t>(std::max<int64_t>(cap, 1));
    }));
    turn_offsets_kernel<<<1, kTurnScanThreads, 0, st>>>(ta.keys, a.tok_off, a.tok_base, ta.tok_off, n, B, cat_off, new_dst, parent, pv);
    const int T = 128;
    hash_keys_kernel_v1<<<(unsigned)((n + T - 1) / T), T, 0, st>>>(x->tv, ta.tok, ta.tok_off, ta.tok_base, n, parent, pv, new_dst, 0, cat);
    const int64_t cw = std::min<int64_t>((n + 7) / 8, (int64_t)x->sm_count * 8);
    turn_concat_kernel<<<(unsigned)cw, 256, 0, st>>>(ta.keys, a.tok_off, a.tok_base, cat_off, new_dst, n, cat, ta.new_keys, ta.new_off, ta.new_base);
    x->launches += 3;
    CK(cudaGetLastError());
    ScoreArgs k = a;
    k.tok_off = cat_off; k.tok_base = 0;
    return launch_score(x, ScoreIn{cat, true}, k, st);
}

// The device-resident entry points: Score() on the handle's stream, after the asynchronous write batches issued before.
int score_dev(kvidx* x, const ScoreIn& in, const ScoreArgs& a) {
    ReadCall c(x);
    if (int rc = c.begin(kAfterWrites)) return rc;
    return launch_score(x, in, a, x->stream);
}

int check_csr(const int64_t* off, int64_t n, const char* what = "tok_off") {
    for (int64_t i = 0; i < n; ++i) if (off[i + 1] < off[i]) return fail(KVIDX_EINVAL, "%s not monotone at %lld", what, (long long)i);
    return 0;
}

// The result rows of a Score() call with P pods.  A buffer of n rows holds, dense: n x P f64 scores, then n has_keys bytes;
// sparse: n x kMaxEnt f64 scores, n x kMaxEnt u16 pods, n entry counts, then n has_keys bytes.
struct RowLayout {
    uint32_t P; bool sparse;
    size_t row() const { return sparse ? (size_t)kMaxEnt * (sizeof(double) + sizeof(uint16_t)) + 2 : (size_t)P * sizeof(double) + 1; }
    // f(array, bytes) for each array of c rows, in buffer order (array: the ScoreArgs member that points at it)
    template <class F> void each(int64_t c, F f) const {
        if (sparse) {
            f(&ScoreArgs::sp_scores, (size_t)c * kMaxEnt * sizeof(double));
            f(&ScoreArgs::sp_pods, (size_t)c * kMaxEnt * sizeof(uint16_t));
            f(&ScoreArgs::sp_cnt, (size_t)c);
        } else {
            f(&ScoreArgs::dense, (size_t)c * P * sizeof(double));
        }
        f(&ScoreArgs::has_keys, (size_t)c);
    }
    // point the outputs of `a` into a buffer of n rows
    void carve(void* buf, int64_t n, ScoreArgs& a) const {
        uint8_t* b = static_cast<uint8_t*>(buf);
        each(n, [&](auto m, size_t bytes) { a.*m = reinterpret_cast<std::remove_reference_t<decltype(a.*m)>>(b); b += bytes; });
    }
    // the outputs of `a` from row i on
    ScoreArgs at(ScoreArgs a, int64_t i) const {
        if (sparse) { a.sp_scores += i * kMaxEnt; a.sp_pods += i * kMaxEnt; a.sp_cnt += i; }
        else a.dense += i * (int64_t)P;
        if (a.has_keys) a.has_keys += i;
        return a;
    }
    // copy c rows from the outputs of src to those of dst: memcpy, or with st device to host on *st.  Only the arrays dst
    // has (has_keys is optional).
    int copy(const ScoreArgs& dst, const ScoreArgs& src, int64_t c, const cudaStream_t* st = nullptr) const {
        cudaError_t e = cudaSuccess;
        each(c, [&](auto m, size_t bytes) {
            if (!(dst.*m) || e != cudaSuccess) return;
            if (st) e = cudaMemcpyAsync(dst.*m, src.*m, bytes, cudaMemcpyDeviceToHost, *st);
            else memcpy(dst.*m, src.*m, bytes);
        });
        CK(e);
        return 0;
    }
    // are all of the outputs of `a` pinned host memory?
    bool pinned(const ScoreArgs& a) const {
        if (a.has_keys && !is_device_accessible_host(a.has_keys)) return false;
        return sparse ? is_device_accessible_host(a.sp_pods) && is_device_accessible_host(a.sp_scores) && is_device_accessible_host(a.sp_cnt)
                      : is_device_accessible_host(a.dense);
    }
};

// Stage prompts i0 .. i0+c of the host call h (sections s[0 .. ns), the inputs first) in one pinned buffer: each
// section's offsets, the model ids and filter rows when h has them, then the elements of each input that is not pinned.
// -> a: the chunk's call (the staged offsets, model ids and filter rows; h's outputs), v: each section's view (the
// elements of a pinned input and of the output stay in the caller's buffers).
int stage_inputs(PinBuf& buf, const ScoreArgs& h, const Csr* s, int ns, int nin, const bool* pinned, int64_t i0, int64_t c, uint32_t FW,
                 ScoreArgs& a, View* v) {
    int64_t* off[3]; uint32_t* model; uint64_t* filter; uint8_t* el[2];
    CK(carve(buf, [&](Carver& cv) {
        for (int k = 0; k < ns; ++k) off[k] = cv.take<int64_t>(c + 1);
        model = cv.take<uint32_t>(h.model ? c : 0);
        filter = cv.take<uint64_t>(h.filter ? c * FW : 0);
        for (int k = 0; k < nin; ++k) el[k] = cv.take<uint8_t>(pinned[k] ? 0 : s[k].bytes(i0, i0 + c));
    }));
    a = h; a.n_prompts = c;
    if (h.model) { memcpy(model, h.model + i0, (size_t)c * 4); a.model = model; }
    if (h.filter) { memcpy(filter, h.filter + i0 * FW, (size_t)c * FW * 8); a.filter = filter; }
    for (int k = 0; k < ns; ++k) {
        memcpy(off[k], s[k].off + i0, (size_t)(c + 1) * 8);
        v[k] = View{s[k].at(i0), off[k], s[k].off[i0]};
        if (k < nin && !pinned[k]) { memcpy(el[k], v[k].p, s[k].bytes(i0, i0 + c)); v[k].p = el[k]; }
    }
    return 0;
}

// Host-buffer scoring of the call `h` (host pointers; h.tok unused, the elements are at in.p).  Chunks of prompts flow
// through two slots and three streams so that the H2D copy of chunk c+1, the kernel of chunk c and the D2H of chunk c-1
// overlap (two DMA engines + SMs):
//   copy_stream : staging -> d_tok/d_off/...      (records ev_h2d[slot])
//   x->stream   : score kernel                      (waits ev_h2d, records ev_k[slot])
//   d2h_stream  : results -> pinned host            (waits ev_k, records ev_done[slot])
// Caller buffers that are already pinned are used directly (no staging memcpy).
int score_host_locked(kvidx* x, const ScoreIn& in, const ScoreArgs& h);

int score_host(kvidx* x, const ScoreIn& in, const ScoreArgs& h) {
    const int64_t n = h.n_prompts;
    if (n < 0 || !h.tok_off) return fail(KVIDX_EINVAL, "bad arguments");
    if (n == 0) return 0;
    int rc = check_csr(h.tok_off, n, in.keys ? "key_off" : "tok_off");
    if (rc) return rc;
    if (h.tok_off[n] > h.tok_off[0] && !in.p) return fail(KVIDX_EINVAL, in.keys ? "NULL keys" : "NULL tokens");
    ReadCall c(x);
    if ((rc = c.begin(kAfterWrites))) return rc;
    return c.end(score_host_locked(x, in, h), {x->copy_stream, x->stream, x->d2h_stream});
}

// A handful of prompts (the size of one RPC, or of what the submission queue gathers at low load) whose kernel reads its
// inputs in place: no copy engine, no second stream.  The cooperative kernel reads the tokens straight from PINNED HOST
// memory -- its TMA bulk copies fetch each 2 KB chunk over PCIe one chunk ahead of the chain -- and writes the result rows
// straight back into pinned host memory; the call is one launch and one stream synchronisation.  (cudaMallocHost memory
// is device-addressable under UVA.)  Request keys are read the same way by the key kernel, one coalesced 256-byte read per
// 32 keys.
int score_host_zerocopy(kvidx* x, const ScoreIn& in, const ScoreArgs& h) {
    const int64_t n = h.n_prompts;
    const RowLayout rows{x->tv.max_pods, h.sp_cnt != nullptr};
    Csr s[3]; int nin;
    const int ns = in.sections(h, s, &nin);
    bool pinned[3];
    for (int k = 0; k < ns; ++k) pinned[k] = s[k].pinned(n);
    ScoreArgs a; View v[3];
    if (int rc = stage_inputs(x->h_stage[0], h, s, ns, nin, pinned, 0, n, x->tv.filter_words, a, v)) return rc;
    // results: straight into the caller's buffers when those are pinned, else through the pinned staging (new keys after
    // the rows)
    const bool out_direct = rows.pinned(h), nk_direct = ns == nin || pinned[nin];
    if (!out_direct || !nk_direct) {
        uint8_t* r; uint64_t* nk;
        CK(carve(x->h_out[0], [&](Carver& c) { r = c.take<uint8_t>(n * rows.row()); nk = c.take<uint64_t>(ns > nin ? s[nin].bytes(0, n) / 8 : 0); }));
        if (!out_direct) rows.carve(r, n, a);
        if (!nk_direct) v[nin].p = nk;
    }
    const ScoreIn z = in.moved(v, a);
    if (int rc = launch_score(x, z, a, x->stream)) return rc;
    CK(cudaStreamSynchronize(x->stream));
    if (!nk_direct) memcpy(s[nin].at(0), v[nin].p, s[nin].bytes(0, n));
    return out_direct ? 0 : rows.copy(h, a, n);
}

int score_host_locked(kvidx* x, const ScoreIn& in, const ScoreArgs& h) {
    int rc = 0;
    const int64_t n = h.n_prompts;
    Csr s[3]; int nin;
    const int ns = in.sections(h, s, &nin);
    const Csr* nk = ns > nin ? &s[nin] : nullptr;      // a turn's new keys, when wanted
    // the zero-copy and chunk budgets are bytes of input: 16 MiB and host_chunk_tokens x 4 (32 Mi tokens, or as many bytes
    // of keys, or of a turn's keys and tokens)
    auto in_bytes = [&](int64_t i0, int64_t i1) { size_t b = 0; for (int k = 0; k < nin; ++k) b += s[k].bytes(i0, i1); return b; };
    if (n <= x->zerocopy_max && in_bytes(0, n) <= (16u << 20) && reads_in_place(x, in, n)) return score_host_zerocopy(x, in, h);
    const uint32_t FW = x->tv.filter_words;
    const RowLayout rows{x->tv.max_pods, h.sp_cnt != nullptr};
    // chunk = up to 128 MiB of input: the H2D copy of a chunk must outlast its kernel for the pipeline to be PCIe bound, and
    // smaller chunks leave the fixed cost of a launch exposed.
    const size_t kMaxChunkBytes = (size_t)x->host_chunk_tokens * 4;
    const int64_t kMaxRowsChunk = std::max<int64_t>(1, (128ll << 20) / (int64_t)rows.row());
    bool pinned[3];
    for (int k = 0; k < ns; ++k) pinned[k] = s[k].pinned(n);
    // dense rows are written straight into the caller's buffers when those are pinned; sparse rows are always staged
    const bool out_pinned = !rows.sparse && rows.pinned(h);
    cudaStream_t s_k = x->stream, s_in = x->copy_stream, s_out = x->d2h_stream;
    struct Pending { bool live = false; int64_t i0 = 0, cnt = 0; const uint64_t* nk = nullptr; } pend[2];   // nk: staged new keys
    auto drain = [&](int sl) -> int {
        if (!pend[sl].live) return 0;
        CK(cudaEventSynchronize(x->ev_done[sl]));
        pend[sl].live = false;
        const int64_t i0 = pend[sl].i0, c = pend[sl].cnt;
        if (pend[sl].nk) memcpy(nk->at(i0), pend[sl].nk, nk->bytes(i0, i0 + c));
        if (out_pinned) return 0;                 // results were written straight into the caller's buffers
        ScoreArgs staged{};
        rows.carve(x->h_out[sl].p, c, staged);
        return rows.copy(rows.at(h, i0), staged, c);
    };
    // the first chunk must see everything already queued on the handle's stream (asynchronous write batches issued before
    // included: score_host ordered it after them)
    CK(cudaEventRecord(x->ev_k[0], s_k));
    CK(cudaStreamWaitEvent(s_in, x->ev_k[0], 0));
    int64_t i0 = 0;
    int slot = 0;
    while (i0 < n) {
        int64_t i1 = i0;
        while (i1 < n && (i1 - i0) < kMaxRowsChunk && in_bytes(i0, i1 + 1) <= kMaxChunkBytes) ++i1;
        if (i1 == i0) i1 = i0 + 1;                // a single prompt larger than the chunk budget
        const int64_t c = i1 - i0, nnk = nk ? nk->off[i1] - nk->off[i0] : 0;
        rc = drain(slot);                         // slot's previous results are home; its device buffers are free
        if (rc) return rc;
        ScoreArgs d; View v[3];                   // the chunk staged, then on the device
        if ((rc = stage_inputs(x->h_stage[slot], h, s, ns, nin, pinned, i0, c, FW, d, v))) return rc;
        int64_t* doff[3]; uint8_t* del[2];
        CK(carve(x->d_off[slot], [&](Carver& cv) { for (int k = 0; k < ns; ++k) doff[k] = cv.take<int64_t>(c + 1); }));
        CK(carve(x->d_tok[slot], [&](Carver& cv) { for (int k = 0; k < nin; ++k) del[k] = cv.take<uint8_t>(s[k].bytes(i0, i1)); }));
        for (int k = 0; k < ns; ++k) {
            CK(cudaMemcpyAsync(doff[k], v[k].off, (size_t)(c + 1) * 8, cudaMemcpyHostToDevice, s_in));
            v[k].off = doff[k];
            if (k >= nin) continue;
            if (s[k].bytes(i0, i1) > 0) CK(cudaMemcpyAsync(del[k], v[k].p, s[k].bytes(i0, i1), cudaMemcpyHostToDevice, s_in));
            v[k].p = del[k];
        }
        if (d.model) {
            CK(x->d_model[slot].need((size_t)c * 4));
            CK(cudaMemcpyAsync(x->d_model[slot].p, d.model, (size_t)c * 4, cudaMemcpyHostToDevice, s_in));
            d.model = x->d_model[slot].as<uint32_t>();
        }
        if (d.filter) {
            CK(x->d_filter[slot].need((size_t)c * FW * 8));
            CK(cudaMemcpyAsync(x->d_filter[slot].p, d.filter, (size_t)c * FW * 8, cudaMemcpyHostToDevice, s_in));
            d.filter = x->d_filter[slot].as<uint64_t>();
        }
        CK(cudaEventRecord(x->ev_h2d[slot], s_in));
        // outputs: the rows, then (a turn that wants them) the new keys, on the device and in the pinned staging alike
        uint8_t *drow, *hrow = nullptr; uint64_t *dnk, *hnk = nullptr;
        CK(carve(x->d_out[slot], [&](Carver& cv) { drow = cv.take<uint8_t>(c * rows.row()); dnk = cv.take<uint64_t>(nnk); }));
        if (!out_pinned || (nnk > 0 && !pinned[nin]))
            CK(carve(x->h_out[slot], [&](Carver& cv) { hrow = cv.take<uint8_t>(c * rows.row()); hnk = cv.take<uint64_t>(nnk); }));
        if (nk) v[nin].p = dnk;
        rows.carve(drow, c, d);
        CK(cudaStreamWaitEvent(s_k, x->ev_h2d[slot], 0));
        int64_t maxb = 0;                         // the round pipelines' block count (tokens)
        if (!in.keys) for (int64_t q = i0; q < i1; ++q) maxb = std::max<int64_t>(maxb, (h.tok_off[q + 1] - h.tok_off[q]) / x->tv.block_size);
        const ScoreIn din = in.moved(v, d);
        rc = launch_score(x, din, d, s_k, maxb);
        if (rc) return rc;
        CK(cudaEventRecord(x->ev_k[slot], s_k));
        // (slot reuse is safe without further stream waits: drain(slot) host-waits on ev_done[slot], which is
        //  recorded after this kernel and its read-back)
        // read back
        CK(cudaStreamWaitEvent(s_out, x->ev_k[slot], 0));
        if (out_pinned) {
            if ((rc = rows.copy(rows.at(h, i0), d, c, &s_out))) return rc;
        } else {
            CK(cudaMemcpyAsync(hrow, drow, (size_t)c * rows.row(), cudaMemcpyDeviceToHost, s_out));
        }
        if (nnk > 0) CK(cudaMemcpyAsync(pinned[nin] ? static_cast<void*>(nk->at(i0)) : hnk, dnk, (size_t)nnk * 8, cudaMemcpyDeviceToHost, s_out));
        CK(cudaEventRecord(x->ev_done[slot], s_out));
        pend[slot].live = true; pend[slot].i0 = i0; pend[slot].cnt = c;
        pend[slot].nk = nnk > 0 && !pinned[nin] ? hnk : nullptr;
        slot ^= 1;
        i0 = i1;
    }
    rc = drain(slot); if (rc) return rc;
    rc = drain(slot ^ 1); if (rc) return rc;
    return 0;
}

// Several callers' requests as one batch: tokens are gathered into one pinned buffer (CSR rebuilt), per-prompt model ids and
// filter rows materialised if any request carries them, one pass through score_host, results scattered to the owners.
int run_combined(kvidx* x, SubmitQueue* q, const std::vector<SubmitReq*>& batch) {
    const uint32_t FW = x->tv.filter_words;
    const ScoreArgs& a0 = batch[0]->a;
    int64_t n = 0, nt = 0;
    bool any_model = false, any_filter = false;
    for (const SubmitReq* r : batch) {
        n += r->a.n_prompts; nt += r->a.tok_off[r->a.n_prompts] - r->a.tok_off[0];
        any_model |= r->a.model != nullptr || r->a.model0 != a0.model0; any_filter |= r->a.filter != nullptr;
    }
    const RowLayout rows{x->tv.max_pods, a0.sp_cnt != nullptr};
    int64_t* off; uint32_t* model; uint64_t* filter; uint32_t* tok;
    CK(carve(q->h_in, [&](Carver& c) {
        off = c.take<int64_t>(n + 1); model = c.take<uint32_t>(any_model ? n : 0); filter = c.take<uint64_t>(any_filter ? n * FW : 0);
        tok = c.take<uint32_t>(nt);
    }));
    CK(q->h_out.need((size_t)n * rows.row()));
    if (!any_model) model = nullptr;
    if (!any_filter) filter = nullptr;
    int64_t at = 0, tat = 0;
    off[0] = 0;
    for (const SubmitReq* r : batch) {
        const int64_t rn = r->a.n_prompts, tb = r->a.tok_off[0], rt = r->a.tok_off[rn] - tb;
        if (rt > 0) memcpy(tok + tat, r->tok + tb, (size_t)rt * 4);
        for (int64_t i = 0; i < rn; ++i) off[at + i + 1] = tat + (r->a.tok_off[i + 1] - tb);
        if (model) for (int64_t i = 0; i < rn; ++i) model[at + i] = r->a.model ? r->a.model[i] : r->a.model0;
        if (filter) { if (r->a.filter) memcpy(filter + (size_t)at * FW, r->a.filter, (size_t)rn * FW * 8); else memset(filter + (size_t)at * FW, 0, (size_t)rn * FW * 8); }
        at += rn; tat += rt;
    }
    ScoreArgs all = dense_args(off, n, model, a0.model0, filter, nullptr, nullptr);
    rows.carve(q->h_out.p, n, all);
    int rc = score_host(x, ScoreIn{tok, false}, all);
    if (rc) return rc;
    at = 0;
    for (const SubmitReq* r : batch) {
        rows.copy(r->a, rows.at(all, at), r->a.n_prompts);
        at += r->a.n_prompts;
    }
    return 0;
}

int submit_score(kvidx* x, const uint32_t* tok, const ScoreArgs& a) {
    SubmitQueue* q = x->queue.get();
    const int64_t n = a.n_prompts;
    // big batches and malformed calls go straight through (score_host validates); so does everything when the queue is off
    if (!q || !q->enabled || n <= 0 || !a.tok_off || n > q->max_prompts / 4) return score_host(x, ScoreIn{tok, false}, a);
    if (int rc = check_csr(a.tok_off, n)) return rc;
    if (a.tok_off[n] > a.tok_off[0] && !tok) return fail(KVIDX_EINVAL, "NULL tokens");
    SubmitReq me;
    me.tok = tok; me.a = a;
    bool lead;
    {
        std::lock_guard<std::mutex> lk(q->mu);
        q->pending.push_back(&me);
        lead = !q->leader_active;
        if (lead) q->leader_active = true;
    }
    if (!lead) {
        std::unique_lock<std::mutex> lk(me.m);
        me.cv.wait(lk, [&] { return me.done || me.promote; });
        if (me.done) { if (me.rc) g_err = me.err; return me.rc; }
        // promoted: the previous leader left with work still queued (this request among it)
    }
    for (;;) {
        std::vector<SubmitReq*> batch;
        {
            std::unique_lock<std::mutex> lk(q->mu);
            if (me.done) {                                    // my own request is served: hand the queue to the next owner
                SubmitReq* next = nullptr;
                if (q->pending.empty()) q->leader_active = false;
                else next = q->pending.front();
                lk.unlock();
                if (next) { std::lock_guard<std::mutex> g2(next->m); next->promote = true; next->cv.notify_one(); }
                if (me.rc) g_err = me.err;
                return me.rc;
            }
            const bool sparse = q->pending.front()->a.sp_cnt != nullptr;
            int64_t np = 0, ntok = 0;
            for (auto it = q->pending.begin(); it != q->pending.end();) {
                SubmitReq* r = *it;
                const int64_t rn = r->a.n_prompts, rt = r->a.tok_off[rn] - r->a.tok_off[0];
                if ((r->a.sp_cnt != nullptr) != sparse) { ++it; continue; }
                if (!batch.empty() && (np + rn > q->max_prompts || ntok + rt > q->max_tokens)) break;
                batch.push_back(r); np += rn; ntok += rt;
                it = q->pending.erase(it);
            }
        }
        int rc;
        if (batch.size() == 1) {
            rc = score_host(x, ScoreIn{batch[0]->tok, false}, batch[0]->a);
        } else {
            rc = run_combined(x, q, batch);
            q->coalesced += batch.size();
        }
        q->batches += 1;
        for (SubmitReq* r : batch) {
            if (r == &me) { me.rc = rc; if (rc) me.err = g_err; me.done = true; continue; }
            std::lock_guard<std::mutex> g2(r->m);             // (notify under the lock: the owner cannot return -- and destroy r -- before we are done with it)
            r->rc = rc; if (rc) r->err = g_err; r->done = true;
            r->cv.notify_one();
        }
    }
}

std::unique_ptr<SubmitQueue> new_submit_queue() {
    auto q = std::make_unique<SubmitQueue>();
    if (const char* k = getenv("KVIDX_SUBMIT_QUEUE")) q->enabled = atoi(k) != 0;
    return q;
}
uint64_t submit_queue_coalesced(SubmitQueue* q) { return q->coalesced.load(); }

// TokensToKVBlockKeys for a CSR batch on the device (token_processor.go:141-162)
int launch_hash_keys(kvidx* x, const uint32_t* d_tok, const int64_t* d_off, int64_t tok_base, int64_t n, const uint64_t* d_parent,
                     const uint8_t* d_pv, const int64_t* d_koff, uint64_t* d_keys, cudaStream_t st) {
    const int T = 128;
    hash_keys_kernel_v1<<<(unsigned)((n + T - 1) / T), T, 0, st>>>(x->tv, d_tok, d_off, tok_base, n, d_parent, d_pv, d_koff, 0, d_keys);
    x->launches += 1;
    CK(cudaGetLastError());
    return 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------
extern "C" {

int kvidx_abi_version(void) { return KVIDX_ABI_VERSION; }

void kvidx_config_default(kvidx_config_t* c) {
    if (!c) return;
    memset(c, 0, sizeof *c);
    c->struct_size = sizeof *c;
    c->device = 0;
    c->block_size = 16;                      // token_processor.go:31
    c->pods_per_key = KVIDX_MAX_PODS_PER_KEY; // in_memory.go:34
    c->init_hash = kFnvOffset;               // FNV64a("")  (HashSeed default "", token_processor.go:48)
    c->capacity = 1ull << 20;
    c->table_slots = 0;
    c->max_pods = 256;
    c->n_tier_weights = 2;
    for (auto& w : c->tier_weight) w = 1.0;
    c->tier_weight[0] = 1.0;                 // "gpu"  backend.go:28
    c->tier_weight[1] = 0.8;                 // "cpu"  backend.go:29
    c->lru_exact = 0;
}

const char* kvidx_last_error(kvidx_t*) { return g_err.c_str(); }

uint64_t kvidx_fnv64a(const void* data, size_t n) {
    const uint8_t* p = static_cast<const uint8_t*>(data);
    uint64_t h = kFnvOffset;
    for (size_t i = 0; i < n; ++i) h = (h ^ p[i]) * kFnvPrime;
    return h;
}
uint32_t kvidx_fnv32a(const void* data, size_t n) {
    const uint8_t* p = static_cast<const uint8_t*>(data);
    uint32_t h = 0x811C9DC5u;
    for (size_t i = 0; i < n; ++i) h = (h ^ p[i]) * 0x01000193u;
    return h;
}
uint32_t kvidx_queue_index(const char* pod, size_t n, uint32_t concurrency) {
    return concurrency ? kvidx_fnv32a(pod, n) % concurrency : 0;
}

void* kvidx_host_alloc(size_t bytes) { void* p = nullptr; if (cudaMallocHost(&p, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; } return p; }
void kvidx_host_free(void* p) { if (p) cudaFreeHost(p); }

namespace {
int create_impl(const kvidx_config_t& c, kvidx* x) {
    CK(cudaSetDevice(c.device));
    x->cfg = c;
    x->device = c.device;
    cudaDeviceProp prop{};
    CK(cudaGetDeviceProperties(&prop, c.device));
    x->sm_count = prop.multiProcessorCount;
    if (prop.major != 9 || prop.minor != 0) return fail(KVIDX_ECUDA, "device sm_%d%d is not Hopper; libkvidx is built for sm_90a only", prop.major, prop.minor);
    CK(cudaStreamCreateWithFlags(&x->own_stream.h, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&x->own_wstream.h, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&x->copy_stream.h, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&x->d2h_stream.h, cudaStreamNonBlocking));
    for (int q = 0; q < kMaxParts - 1; ++q) {
        CK(cudaStreamCreateWithFlags(&x->aux_stream[q].h, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&x->ev_join[q].h, cudaEventDisableTiming));
    }
    CK(cudaEventCreateWithFlags(&x->ev_fork.h, cudaEventDisableTiming));
    {
        int lo = 0, hi = 0;
        CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        for (int q = 0; q < kMaxParts; ++q) {
            CK(cudaStreamCreateWithPriority(&x->hp_stream[q].h, cudaStreamNonBlocking, hi));
            CK(cudaStreamCreateWithPriority(&x->lp_stream[q].h, cudaStreamNonBlocking, lo));
        }
    }
    for (int q = 0; q < kMaxParts; ++q) { CK(cudaEventCreateWithFlags(&x->ev_g[q].h, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&x->ev_r[q].h, cudaEventDisableTiming)); }
    CK(cudaEventCreateWithFlags(&x->ev_write.h, cudaEventDisableTiming));
    CK(x->snap.init());
    CK(x->rstage.init());
    x->stream = x->own_stream;
    for (int i = 0; i < 2; ++i) {
        CK(cudaEventCreateWithFlags(&x->ev_h2d[i].h, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&x->ev_done[i].h, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&x->ev_k[i].h, cudaEventDisableTiming));
    }
    uint32_t shard_bits = 0;
    if (c.shard_count > 1) {
        if (c.shard_count > 8 || (c.shard_count & (c.shard_count - 1)) || c.shard_rank >= c.shard_count) return fail(KVIDX_EINVAL, "shard_count must be a power of two <= 8 and shard_rank < shard_count");
        while ((1u << shard_bits) < c.shard_count) ++shard_bits;
    }
    const uint64_t per_shard = c.shard_count > 1 ? (c.capacity + c.shard_count - 1) / c.shard_count : c.capacity;
    const uint64_t full = pow2ceil(std::max<uint64_t>(4 * per_shard, 1024));
    uint64_t slots = c.table_slots ? pow2ceil(c.table_slots) : full;
    if (slots < 1024) slots = 1024;
    if (c.grow_tables) {                      // the tables start small and may grow up to what a fixed handle allocates
        x->grow_max = full;
        if (!c.table_slots) slots = std::min<uint64_t>(full, 1ull << 20);
    }
    TableView& t = x->tv;
    t.req_mask = slots - 1; t.eng_mask = slots - 1;
    t.capacity = c.capacity; t.init_hash = c.init_hash; t.block_size = c.block_size; t.pods_per_key = c.pods_per_key;
    t.max_pods = c.max_pods; t.filter_words = (c.max_pods + 63) / 64;
    for (int i = 0; i < 16; ++i) t.weight[i] = (uint32_t)i < c.n_tier_weights ? c.tier_weight[i] : 1.0;
    t.req_stamp = nullptr;
    t.req_ref = nullptr; t.eng_ref = nullptr;
    // a sharded handle's removal bitmaps (kvidx_shard_remove_pods) follow its request slots: its peers read them through
    // the mapping they already hold, and the in-place compaction rewrites only the slots
    int rc = alloc_tables(x, slots, slots, &t.req, &t.eng, x->stream, shard_bits ? remove_bitmap_bytes(slots) : 0);
    if (rc) return rc;
    if (c.lru_exact) {
        if (c.shard_count > 1) return fail(KVIDX_EINVAL, "lru_exact is not supported on a sharded index");
        CK(cudaMalloc((void**)&t.req_stamp, slots * 8));
        CK(cudaMemsetAsync(t.req_stamp, 0, slots * 8, x->stream));
    }
    if (c.evict_policy == KVIDX_EVICT_CLOCK) {
        CK(cudaMalloc((void**)&t.req_ref, slots / 8));
        CK(cudaMalloc((void**)&t.eng_ref, slots / 8));
        CK(cudaMemsetAsync(t.req_ref, 0, slots / 8, x->stream));
        CK(cudaMemsetAsync(t.eng_ref, 0, slots / 8, x->stream));
    }
    CK(cudaMalloc((void**)&x->d_cnt, sizeof(Counters)));
    CK(cudaMemsetAsync(x->d_cnt, 0, sizeof(Counters), x->stream));
    CK(cudaMallocHost((void**)&x->h_cnt, sizeof(Counters)));
    memset(x->h_cnt, 0, sizeof(Counters));
    CK(cudaMalloc((void**)&x->d_cnt_all, sizeof(Counters) * 8));
    CK(cudaMallocHost((void**)&x->h_cnt_all, sizeof(Counters) * 8));
    t.cnt = x->d_cnt;
    t.shard_bits = shard_bits; t.shard_rank = c.shard_count > 1 ? c.shard_rank : 0;
    for (int i = 0; i < 8; ++i) { t.req_peer[i] = nullptr; t.eng_peer[i] = nullptr; t.cnt_peer[i] = nullptr; }
    t.req_peer[t.shard_rank] = t.req; t.eng_peer[t.shard_rank] = t.eng; t.cnt_peer[t.shard_rank] = t.cnt;
    CK(cudaStreamSynchronize(x->stream));
    if (const char* k = getenv("KVIDX_SCORE_KERNEL")) x->score_kernel = (k[0] == 'v' ? atoi(k + 1) : atoi(k)) == 1 ? 1 : 2;
    if (const char* k = getenv("KVIDX_SCORE_PATH")) x->score_path = !strcmp(k, "rounds") ? 2 : !strcmp(k, "classes") ? 3 : !strcmp(k, "coop") ? 4 : 0;
    if (const char* k = getenv("KVIDX_COOP_MAX")) x->coop_max = atoll(k);
    if (const char* k = getenv("KVIDX_ZEROCOPY_MAX")) x->zerocopy_max = atoll(k);
    if (const char* k = getenv("KVIDX_CLASSES_MIN")) x->classes_min = atoll(k);
    if (const char* k = getenv("KVIDX_CLASSES_SHARING")) x->classes_min_sharing = atof(k);
    if (const char* k = getenv("KVIDX_SORT_PREFIX")) x->sort_prefix = atoi(k) != 0;
    if (const char* k = getenv("KVIDX_HOST_CHUNK_TOKENS")) x->host_chunk_tokens = std::max<int64_t>(1 << 16, atoll(k));
    if (const char* k = getenv("KVIDX_ROUNDS_TRACE")) x->rounds_trace = atoi(k);
    if (const char* k = getenv("KVIDX_ROUNDS_PARTS")) x->rounds_parts = atoi(k);
    if (const char* k = getenv("KVIDX_PEER_PAIR")) x->tv.peer_pair = atoi(k) != 0;
    if (const char* k = getenv("KVIDX_ROUNDS_WARP_MAX")) x->rounds_warp_max = atoll(k);
    if (const char* k = getenv("KVIDX_ROUNDS_DEDUP")) x->rounds_dedup = atoi(k);
    if (const char* k = getenv("KVIDX_ROUNDS_OVERLAP_MIN")) x->rounds_overlap_min = atoll(k);
    if (const char* k = getenv("KVIDX_WRITE_PHASE1")) x->write_phase1 = atoi(k);
    x->queue = new_submit_queue();
    if (rounds_init() || plain::rounds_init() || coop_init() || turn_init()) return fail(KVIDX_ECUDA, "kernel attribute setup failed: %s", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
}  // namespace

int kvidx_create(const kvidx_config_t* cfg_in, kvidx_t** out) {
    if (!out) return fail(KVIDX_EINVAL, "out is NULL");
    *out = nullptr;
    kvidx_config_t c;
    kvidx_config_default(&c);
    if (cfg_in) {
        if (cfg_in->struct_size == 0 || cfg_in->struct_size > sizeof c) return fail(KVIDX_EINVAL, "bad struct_size");
        memcpy(&c, cfg_in, cfg_in->struct_size);
        c.struct_size = sizeof c;
    }
    if (c.block_size == 0) c.block_size = 16;
    if (c.pods_per_key == 0) c.pods_per_key = KVIDX_MAX_PODS_PER_KEY;
    if (c.pods_per_key > KVIDX_MAX_PODS_PER_KEY) return fail(KVIDX_EINVAL, "pods_per_key %u > %d", c.pods_per_key, KVIDX_MAX_PODS_PER_KEY);
    if (c.capacity == 0) c.capacity = 1ull << 20;
    if (c.max_pods == 0) c.max_pods = 256;
    if (c.max_pods > KVIDX_MAX_PODS) return fail(KVIDX_ERANGE, "max_pods %u > %u", c.max_pods, KVIDX_MAX_PODS);
    if (c.n_tier_weights > KVIDX_MAX_TIERS) return fail(KVIDX_ERANGE, "n_tier_weights > 16");
    if (c.evict_policy > KVIDX_EVICT_CLOCK) return fail(KVIDX_EINVAL, "unknown evict_policy %u", c.evict_policy);
    if (c.evict_policy == KVIDX_EVICT_CLOCK && c.lru_exact) return fail(KVIDX_EINVAL, "evict_policy CLOCK and lru_exact exclude each other");
    if (c.evict_policy == KVIDX_EVICT_CLOCK && c.shard_count > 1) return fail(KVIDX_EINVAL, "evict_policy CLOCK is not supported on a sharded index");
    if (c.grow_tables > 1) return fail(KVIDX_EINVAL, "unknown grow_tables %u", c.grow_tables);
    if (c.grow_tables && c.shard_count > 1) return fail(KVIDX_EINVAL, "grow_tables is not supported on a sharded index");
    if (c.grow_tables && c.table_slots > pow2ceil(std::max<uint64_t>(4 * c.capacity, 1024)))
        return fail(KVIDX_EINVAL, "table_slots %llu is above the %llu slots grow_tables may reach with capacity %llu",
                    (unsigned long long)c.table_slots, (unsigned long long)pow2ceil(std::max<uint64_t>(4 * c.capacity, 1024)),
                    (unsigned long long)c.capacity);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(KVIDX_ECUDA, "no CUDA device: libkvidx has no CPU fallback");
    }
    if (c.device < 0 || c.device >= ndev) return fail(KVIDX_EINVAL, "device %d out of range (%d devices)", c.device, ndev);
    kvidx* x = new kvidx();
    const int rc = create_impl(c, x);
    if (rc) {                       // whatever was created so far (streams, events, tables) goes away with the handle
        const std::string keep = g_err;
        kvidx_destroy(x);
        cudaGetLastError();
        g_err = keep;
        return rc;
    }
    *out = x;
    return 0;
}

// The tables and counters are freed here; every other buffer, stream and event of the handle (and its prefix store) goes
// with its member, once the device is idle.
void kvidx_destroy(kvidx_t* x) {
    if (!x) return;
    cudaSetDevice(x->device);
    cudaDeviceSynchronize();
    if (x->tv.req) cudaFree(x->tv.req);
    if (x->tv.eng) cudaFree(x->tv.eng);
    if (x->tv.req_stamp) cudaFree(x->tv.req_stamp);
    if (x->tv.req_ref) cudaFree(x->tv.req_ref);
    if (x->tv.eng_ref) cudaFree(x->tv.eng_ref);
    if (x->d_cnt) cudaFree(x->d_cnt);
    if (x->h_cnt) cudaFreeHost(x->h_cnt);
    if (x->d_cnt_all) cudaFree(x->d_cnt_all);
    if (x->h_cnt_all) cudaFreeHost(x->h_cnt_all);
    delete x;
    cudaGetLastError();
}

int kvidx_set_tier_weight(kvidx_t* x, uint32_t tier, double w) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    if (tier >= KVIDX_MAX_TIERS) return fail(KVIDX_ERANGE, "tier %u out of range", tier);
    std::unique_lock<std::shared_mutex> tl(x->tables);
    x->tv.weight[tier] = w;
    return 0;
}

int kvidx_set_stream(kvidx_t* x, void* s) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    ReadCall c(x);
    x->stream = s ? static_cast<cudaStream_t>(s) : x->own_stream;
    return 0;
}
int kvidx_synchronize(kvidx_t* x) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    CK(cudaSetDevice(x->device));
    CK(cudaStreamSynchronize(x->stream));
    CK(cudaStreamSynchronize(x->own_wstream));
    return 0;
}

// ---- read path ------------------------------------------------------------------------------

int kvidx_hash_keys(kvidx_t* x, const uint32_t* tok, const int64_t* tok_off, int64_t n, const uint64_t* parent,
                    const uint8_t* parent_valid, uint64_t* keys_out, int64_t* key_off_out) {
    if (!x || !tok_off || !key_off_out || n < 0) return fail(KVIDX_EINVAL, "bad arguments");
    int rc = check_csr(tok_off, n);
    if (rc) return rc;
    const uint32_t B = x->tv.block_size;
    int64_t nk = 0;
    for (int64_t i = 0; i < n; ++i) { key_off_out[i] = nk; nk += (tok_off[i + 1] - tok_off[i]) / B; }
    key_off_out[n] = nk;
    if (n == 0 || nk == 0) return 0;
    if (!keys_out || !tok) return fail(KVIDX_EINVAL, "NULL buffer");
    ReadCall c(x);
    if ((rc = c.begin(0))) return rc;
    const int64_t tb = tok_off[0], nt = tok_off[n] - tb;
    CK(x->d_tok[0].need((size_t)nt * 4 + 64));
    CK(x->d_off[0].need((size_t)(n + 1) * 8));
    int64_t* d_koff; uint64_t* d_parent; uint8_t* d_pv;
    CK(carve(x->d_aux[0], [&](Carver& c) { d_koff = c.take<int64_t>(n + 1); d_parent = c.take<uint64_t>(n); d_pv = c.take<uint8_t>(n); }));
    CK(x->d_out[0].need((size_t)nk * 8));
    CK(cudaMemcpyAsync(x->d_tok[0].p, tok + tb, (size_t)nt * 4, cudaMemcpyHostToDevice, x->stream));
    CK(cudaMemcpyAsync(x->d_off[0].p, tok_off, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, x->stream));
    CK(cudaMemcpyAsync(d_koff, key_off_out, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, x->stream));
    if (parent) CK(cudaMemcpyAsync(d_parent, parent, (size_t)n * 8, cudaMemcpyHostToDevice, x->stream));
    if (parent && parent_valid) CK(cudaMemcpyAsync(d_pv, parent_valid, (size_t)n, cudaMemcpyHostToDevice, x->stream));
    if (!parent) d_parent = nullptr;
    if (!parent || !parent_valid) d_pv = nullptr;
    rc = launch_hash_keys(x, x->d_tok[0].as<uint32_t>(), x->d_off[0].as<int64_t>(), tb, n, d_parent, d_pv, d_koff, x->d_out[0].as<uint64_t>(), x->stream);
    if (rc) return rc;
    CK(cudaMemcpyAsync(keys_out, x->d_out[0].p, (size_t)nk * 8, cudaMemcpyDeviceToHost, x->stream));
    CK(cudaStreamSynchronize(x->stream));
    return 0;
}

int kvidx_hash_keys_dev(kvidx_t* x, const uint32_t* d_tok, const int64_t* d_tok_off, int64_t n, const uint64_t* d_parent,
                        const uint8_t* d_parent_valid, const int64_t* d_key_off, uint64_t* d_keys_out) {
    if (!x || n < 0) return fail(KVIDX_EINVAL, "bad arguments");
    if (n == 0) return 0;
    ReadCall c(x);
    if (int rc = c.begin(0)) return rc;
    return launch_hash_keys(x, d_tok, d_tok_off, 0, n, d_parent, d_parent_valid, d_key_off, d_keys_out, x->stream);
}

int kvidx_lookup(kvidx_t* x, uint32_t model, const uint64_t* keys, int64_t n, const uint64_t* filter,
                 kvidx_podtier_t* podtier_out, uint8_t* cnt_out) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    if (n <= 0 || !keys) return fail(KVIDX_EINVAL, "no requestKeys provided for lookup");   // in_memory.go:108-110
    if (!podtier_out || !cnt_out) return fail(KVIDX_EINVAL, "NULL output");
    if (model > 0xffffu) return fail(KVIDX_ERANGE, "model id %u > 65535", model);
    ReadCall c(x);
    if (int rc = c.begin(kShards | kAfterWrites)) return rc;
    const uint32_t FW = x->tv.filter_words;
    uint64_t *d_keys, *d_f; int* d_cut; uint16_t* d_pt; uint8_t* d_cnt;
    CK(carve(x->d_aux[0], [&](Carver& c) { d_keys = c.take<uint64_t>(n); d_f = c.take<uint64_t>(FW); d_cut = c.take<int>(1); }));
    CK(carve(x->d_out[0], [&](Carver& c) { d_pt = c.take<uint16_t>(n * kMaxEnt); d_cnt = c.take<uint8_t>(n); }));
    CK(cudaMemcpyAsync(d_keys, keys, (size_t)n * 8, cudaMemcpyHostToDevice, x->stream));
    if (filter) CK(cudaMemcpyAsync(d_f, filter, (size_t)FW * 8, cudaMemcpyHostToDevice, x->stream));
    else d_f = nullptr;
    const int big = 0x7fffffff;
    CK(cudaMemcpyAsync(d_cut, &big, sizeof(int), cudaMemcpyHostToDevice, x->stream));
    const int T = 128;
    lookup_kernel_v1<<<(unsigned)((n + T - 1) / T), T, 0, x->stream>>>(x->tv, model, d_keys, n, d_f, d_pt, d_cnt, d_cut,
                                                                      reserve_stamps(x, (unsigned long long)n));
    x->launches += 1;
    CK(cudaGetLastError());
    int cut = big;
    CK(cudaMemcpyAsync(podtier_out, d_pt, (size_t)n * kMaxEnt * 2, cudaMemcpyDeviceToHost, x->stream));
    CK(cudaMemcpyAsync(cnt_out, d_cnt, (size_t)n, cudaMemcpyDeviceToHost, x->stream));
    CK(cudaMemcpyAsync(&cut, d_cut, sizeof(int), cudaMemcpyDeviceToHost, x->stream));
    CK(cudaStreamSynchronize(x->stream));
    if (cut != big) for (int64_t i = cut; i < n; ++i) cnt_out[i] = 0;   // in_memory.go:119-122 early return
    return 0;
}

int kvidx_score_batch(kvidx_t* x, const uint32_t* tok, const int64_t* tok_off, int64_t n, const uint32_t* model, uint32_t model0,
                      const uint64_t* filter, double* scores_out, uint8_t* has_keys_out) {
    if (!x || !scores_out) return fail(KVIDX_EINVAL, "bad arguments");
    return submit_score(x, tok, dense_args(tok_off, n, model, model0, filter, scores_out, has_keys_out));
}

int kvidx_score_batch_sparse(kvidx_t* x, const uint32_t* tok, const int64_t* tok_off, int64_t n, const uint32_t* model, uint32_t model0,
                             const uint64_t* filter, uint16_t* pods_out, double* scores_out, uint8_t* cnt_out, uint8_t* has_keys_out) {
    if (!x || !pods_out || !scores_out || !cnt_out) return fail(KVIDX_EINVAL, "bad arguments");
    return submit_score(x, tok, sparse_args(tok_off, n, model, model0, filter, pods_out, scores_out, cnt_out, has_keys_out));
}

int kvidx_score_batch_dev(kvidx_t* x, const uint32_t* d_tok, const int64_t* d_tok_off, int64_t n, const uint32_t* d_model,
                          uint32_t model0, const uint64_t* d_filter, double* d_scores_out, uint8_t* d_has_keys_out) {
    if (!x || n < 0) return fail(KVIDX_EINVAL, "bad arguments");
    return score_dev(x, ScoreIn{d_tok, false}, dense_args(d_tok_off, n, d_model, model0, d_filter, d_scores_out, d_has_keys_out));
}

int kvidx_score_batch_sparse_dev(kvidx_t* x, const uint32_t* d_tok, const int64_t* d_tok_off, int64_t n, const uint32_t* d_model,
                                 uint32_t model0, const uint64_t* d_filter, uint16_t* d_pods_out, double* d_scores_out,
                                 uint8_t* d_cnt_out, uint8_t* d_has_keys_out) {
    if (!x || n < 0 || !d_pods_out || !d_scores_out || !d_cnt_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_dev(x, ScoreIn{d_tok, false}, sparse_args(d_tok_off, n, d_model, model0, d_filter, d_pods_out, d_scores_out, d_cnt_out, d_has_keys_out));
}

// ---- Score() from request keys (GetPodScores steps 3-4): not coalesced, every call goes straight through ----

int kvidx_score_keys(kvidx_t* x, const uint64_t* keys, const int64_t* key_off, int64_t n, const uint32_t* model, uint32_t model0,
                     const uint64_t* filter, double* scores_out, uint8_t* has_keys_out) {
    if (!x || !scores_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_host(x, ScoreIn{keys, true}, dense_args(key_off, n, model, model0, filter, scores_out, has_keys_out));
}

int kvidx_score_keys_sparse(kvidx_t* x, const uint64_t* keys, const int64_t* key_off, int64_t n, const uint32_t* model, uint32_t model0,
                            const uint64_t* filter, uint16_t* pods_out, double* scores_out, uint8_t* cnt_out, uint8_t* has_keys_out) {
    if (!x || !pods_out || !scores_out || !cnt_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_host(x, ScoreIn{keys, true}, sparse_args(key_off, n, model, model0, filter, pods_out, scores_out, cnt_out, has_keys_out));
}

int kvidx_score_keys_dev(kvidx_t* x, const uint64_t* d_keys, const int64_t* d_key_off, int64_t n, const uint32_t* d_model,
                         uint32_t model0, const uint64_t* d_filter, double* d_scores_out, uint8_t* d_has_keys_out) {
    if (!x || n < 0 || !d_key_off || !d_scores_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_dev(x, ScoreIn{d_keys, true}, dense_args(d_key_off, n, d_model, model0, d_filter, d_scores_out, d_has_keys_out));
}

int kvidx_score_keys_sparse_dev(kvidx_t* x, const uint64_t* d_keys, const int64_t* d_key_off, int64_t n, const uint32_t* d_model,
                                uint32_t model0, const uint64_t* d_filter, uint16_t* d_pods_out, double* d_scores_out,
                                uint8_t* d_cnt_out, uint8_t* d_has_keys_out) {
    if (!x || n < 0 || !d_key_off || !d_pods_out || !d_scores_out || !d_cnt_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_dev(x, ScoreIn{d_keys, true}, sparse_args(d_key_off, n, d_model, model0, d_filter, d_pods_out, d_scores_out, d_cnt_out, d_has_keys_out));
}

// ---- Score() for a conversation turn: held keys, then the new turn's tokens; not coalesced either ----

namespace {
// the host forms: check the token CSR, give the new keys' offsets (from 0), then the host-buffer pipeline
int score_turn_host(kvidx* x, const uint64_t* keys, const int64_t* key_off, const uint32_t* tok, const int64_t* tok_off, const ScoreArgs& h,
                    uint64_t* new_keys, int64_t* new_off) {
    const int64_t n = h.n_prompts;
    if (n < 0 || !key_off || !tok_off || (new_keys && !new_off)) return fail(KVIDX_EINVAL, "bad arguments");
    if (n == 0) return 0;
    int rc = check_csr(tok_off, n);
    if (rc) return rc;
    if (tok_off[n] > tok_off[0] && !tok) return fail(KVIDX_EINVAL, "NULL tokens");
    if (new_off) {
        const uint32_t B = x->tv.block_size;
        new_off[0] = 0;
        for (int64_t i = 0; i < n; ++i) new_off[i + 1] = new_off[i] + (tok_off[i + 1] - tok_off[i]) / B;
    }
    ScoreIn in{keys, true};
    in.t = TurnArgs{nullptr, tok, tok_off, 0, new_keys, new_keys ? new_off : nullptr, 0};
    return score_host(x, in, h);
}
ScoreIn turn_dev(const uint64_t* d_keys, const uint32_t* d_tok, const int64_t* d_tok_off, const int64_t* d_new_off, uint64_t* d_new_keys) {
    ScoreIn in{d_keys, true};
    in.t = TurnArgs{nullptr, d_tok, d_tok_off, 0, d_new_keys, d_new_off, 0};
    return in;
}
}  // namespace

int kvidx_score_turn(kvidx_t* x, const uint64_t* keys, const int64_t* key_off, const uint32_t* tok, const int64_t* tok_off, int64_t n,
                     const uint32_t* model, uint32_t model0, const uint64_t* filter, double* scores_out, uint8_t* has_keys_out,
                     uint64_t* new_keys_out, int64_t* new_key_off_out) {
    if (!x || !scores_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_turn_host(x, keys, key_off, tok, tok_off, dense_args(key_off, n, model, model0, filter, scores_out, has_keys_out),
                           new_keys_out, new_key_off_out);
}

int kvidx_score_turn_sparse(kvidx_t* x, const uint64_t* keys, const int64_t* key_off, const uint32_t* tok, const int64_t* tok_off, int64_t n,
                            const uint32_t* model, uint32_t model0, const uint64_t* filter, uint16_t* pods_out, double* scores_out,
                            uint8_t* cnt_out, uint8_t* has_keys_out, uint64_t* new_keys_out, int64_t* new_key_off_out) {
    if (!x || !pods_out || !scores_out || !cnt_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_turn_host(x, keys, key_off, tok, tok_off, sparse_args(key_off, n, model, model0, filter, pods_out, scores_out, cnt_out, has_keys_out),
                           new_keys_out, new_key_off_out);
}

int kvidx_score_turn_dev(kvidx_t* x, const uint64_t* d_keys, const int64_t* d_key_off, const uint32_t* d_tok, const int64_t* d_tok_off, int64_t n,
                         const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter, double* d_scores_out, uint8_t* d_has_keys_out,
                         const int64_t* d_new_key_off, uint64_t* d_new_keys_out) {
    if (!x || n < 0 || !d_key_off || !d_tok_off || !d_scores_out || (d_new_keys_out && !d_new_key_off)) return fail(KVIDX_EINVAL, "bad arguments");
    return score_dev(x, turn_dev(d_keys, d_tok, d_tok_off, d_new_key_off, d_new_keys_out),
                     dense_args(d_key_off, n, d_model, model0, d_filter, d_scores_out, d_has_keys_out));
}

int kvidx_score_turn_sparse_dev(kvidx_t* x, const uint64_t* d_keys, const int64_t* d_key_off, const uint32_t* d_tok, const int64_t* d_tok_off,
                                int64_t n, const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter, uint16_t* d_pods_out,
                                double* d_scores_out, uint8_t* d_cnt_out, uint8_t* d_has_keys_out, const int64_t* d_new_key_off,
                                uint64_t* d_new_keys_out) {
    if (!x || n < 0 || !d_key_off || !d_tok_off || !d_pods_out || !d_scores_out || !d_cnt_out || (d_new_keys_out && !d_new_key_off))
        return fail(KVIDX_EINVAL, "bad arguments");
    return score_dev(x, turn_dev(d_keys, d_tok, d_tok_off, d_new_key_off, d_new_keys_out),
                     sparse_args(d_key_off, n, d_model, model0, d_filter, d_pods_out, d_scores_out, d_cnt_out, d_has_keys_out));
}

// ---- Lookup hit counts: recordHitMetrics(Lookup(K_i, F_i)) per prompt (kernels_hits.cuh) ----

namespace {
int launch_lookup_hits(kvidx* x, const uint64_t* d_keys, const int64_t* d_key_off, int64_t key_base, int64_t n, const uint32_t* d_model,
                       uint32_t model0, const uint64_t* d_filter, uint32_t* d_hits, unsigned long long stamp_base, cudaStream_t st) {
    const int64_t ctas = std::min<int64_t>(n, (int64_t)x->sm_count * kHitsCtasPerSm);
    lookup_hits_kernel<<<(unsigned)ctas, kHitsThreads, hits_dyn_smem(x->tv.max_pods), st>>>(x->tv, d_keys, d_key_off, key_base, n, d_model,
                                                                                           model0, d_filter, d_hits, stamp_base);
    x->launches += 1;
    CK(cudaGetLastError());
    return 0;
}

// the first and last of n + 1 device offsets, read back on st
int read_ends(const int64_t* d_off, int64_t n, int64_t e[2], cudaStream_t st) {
    CK(cudaMemcpyAsync(&e[0], d_off, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&e[1], d_off + n, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return 0;
}

// The host forms: el / off the prompts' tokens (keys false) or request keys, staged to the device with the read side's
// stager (pinned buffers copied in place, pageable ones through its pinned chunks) into one carved buffer; tokens are
// hashed into the keys' CSR there, and the count runs on the keys.  Synchronous.
int lookup_hits_host_locked(kvidx* x, const void* el, bool keys, const int64_t* off, int64_t n, const uint32_t* model, uint32_t model0,
                            const uint64_t* filter, uint32_t* hits_out) {
    const uint32_t B = x->tv.block_size, FW = x->tv.filter_words;
    const size_t esz = keys ? 8 : 4;
    const int64_t e0 = off[0], ne = off[n] - e0;
    std::vector<int64_t> koff;                        // tokens: the keys' offsets, from 0
    if (!keys) {
        koff.resize(n + 1);
        koff[0] = 0;
        for (int64_t i = 0; i < n; ++i) koff[i + 1] = koff[i] + (off[i + 1] - off[i]) / B;
    }
    const int64_t nk = keys ? ne : koff[n];
    uint8_t* d_el; int64_t *d_off, *d_koff; uint32_t *d_model, *d_hits; uint64_t *d_filter, *d_keys;
    CK(carve(x->d_aux[0], [&](Carver& c) {
        d_el = c.take<uint8_t>((size_t)ne * esz); d_off = c.take<int64_t>(n + 1); d_model = c.take<uint32_t>(model ? n : 0);
        d_filter = c.take<uint64_t>(filter ? (size_t)n * FW : 0); d_hits = c.take<uint32_t>(n);
        d_koff = c.take<int64_t>(keys ? 0 : n + 1); d_keys = c.take<uint64_t>(keys ? 0 : nk);
    }));
    cudaStream_t st = x->stream;
    Stager& sg = x->rstage;
    int rc = sg.h2d(d_el, static_cast<const uint8_t*>(el) + (size_t)e0 * esz, (size_t)ne * esz, st);
    if (!rc) rc = sg.h2d(d_off, off, (size_t)(n + 1) * 8, st);
    if (!rc && model) rc = sg.h2d(d_model, model, (size_t)n * 4, st);
    if (!rc && filter) rc = sg.h2d(d_filter, filter, (size_t)n * FW * 8, st);
    if (!rc && !keys) rc = sg.h2d(d_koff, koff.data(), (size_t)(n + 1) * 8, st);
    if (rc) return rc;
    if (!keys && nk > 0) {
        rc = launch_hash_keys(x, reinterpret_cast<const uint32_t*>(d_el), d_off, e0, n, nullptr, nullptr, d_koff, d_keys, st);
        if (rc) return rc;
    }
    const unsigned long long sb = x->tv.req_stamp ? reserve_stamps(x, (unsigned long long)nk) : 0;
    rc = keys ? launch_lookup_hits(x, reinterpret_cast<const uint64_t*>(d_el), d_off, e0, n, model ? d_model : nullptr, model0,
                                   filter ? d_filter : nullptr, d_hits, sb, st)
              : launch_lookup_hits(x, d_keys, d_koff, 0, n, model ? d_model : nullptr, model0, filter ? d_filter : nullptr, d_hits, sb, st);
    if (rc) return rc;
    return sg.d2h(hits_out, d_hits, (size_t)n * 4, st);
}

int lookup_hits_host(kvidx* x, const void* el, bool keys, const int64_t* off, int64_t n, const uint32_t* model, uint32_t model0,
                     const uint64_t* filter, uint32_t* hits_out) {
    if (!x || n < 0 || !off || !hits_out) return fail(KVIDX_EINVAL, "bad arguments");
    if (n == 0) return 0;
    if (int rc = check_csr(off, n, keys ? "key_off" : "tok_off")) return rc;
    if (off[n] > off[0] && !el) return fail(KVIDX_EINVAL, keys ? "NULL keys" : "NULL tokens");
    ReadCall c(x);
    if (int rc = c.begin(kShards | kAfterWrites)) return rc;
    return c.end(lookup_hits_host_locked(x, el, keys, off, n, model, model0, filter, hits_out), {x->stream});
}
}  // namespace

int kvidx_lookup_hits(kvidx_t* x, const uint32_t* tok, const int64_t* tok_off, int64_t n, const uint32_t* model, uint32_t model0,
                      const uint64_t* filter, uint32_t* hits_out) {
    return lookup_hits_host(x, tok, false, tok_off, n, model, model0, filter, hits_out);
}

int kvidx_lookup_hits_keys(kvidx_t* x, const uint64_t* keys, const int64_t* key_off, int64_t n, const uint32_t* model, uint32_t model0,
                           const uint64_t* filter, uint32_t* hits_out) {
    return lookup_hits_host(x, keys, true, key_off, n, model, model0, filter, hits_out);
}

int kvidx_lookup_hits_keys_dev(kvidx_t* x, const uint64_t* d_keys, const int64_t* d_key_off, int64_t n, const uint32_t* d_model,
                               uint32_t model0, const uint64_t* d_filter, uint32_t* d_hits_out) {
    if (!x || n < 0 || !d_key_off || !d_hits_out) return fail(KVIDX_EINVAL, "bad arguments");
    if (n == 0) return 0;
    ReadCall c(x);
    if (int rc = c.begin(kShards | kAfterWrites)) return rc;
    unsigned long long sb = 0;
    if (x->tv.req_stamp) {                            // exact-LRU: a stamp per key, counted from the offsets (as Score() does)
        int64_t e[2];
        if (int rc = read_ends(d_key_off, n, e, x->stream)) return rc;
        sb = reserve_stamps(x, (unsigned long long)(e[1] - e[0]));
    }
    return launch_lookup_hits(x, d_keys, d_key_off, 0, n, d_model, model0, d_filter, d_hits_out, sb, x->stream);
}

int kvidx_lookup_hits_dev(kvidx_t* x, const uint32_t* d_tok, const int64_t* d_tok_off, int64_t n, const uint32_t* d_model, uint32_t model0,
                          const uint64_t* d_filter, uint32_t* d_hits_out) {
    if (!x || n < 0 || !d_tok_off || !d_hits_out) return fail(KVIDX_EINVAL, "bad arguments");
    if (n == 0) return 0;
    if (n >= (1ll << 31) - 1) return fail(KVIDX_EINVAL, "n_prompts %lld too large for one call", (long long)n);
    ReadCall c(x);
    if (int rc = c.begin(kShards | kAfterWrites)) return rc;
    cudaStream_t st = x->stream;
    int64_t e[2];                                     // the batch's token span sizes the key scratch: >= the keys it holds
    if (int rc = read_ends(d_tok_off, n, e, st)) return rc;
    const int64_t cap = (e[1] - e[0]) / x->tv.block_size;
    size_t scan_bytes = 0;                            // the keys' offsets: block counts, summed in place
    CK(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (int64_t*)nullptr, (int64_t*)nullptr, (int)n, st));
    int64_t* koff; uint64_t* keys; uint8_t* scan;
    CK(carve(x->d_aux[0], [&](Carver& c) {
        koff = c.take<int64_t>(n + 1); keys = c.take<uint64_t>(std::max<int64_t>(cap, 1)); scan = c.take<uint8_t>(scan_bytes);
    }));
    block_counts_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_tok_off, n, x->tv.block_size, koff);
    CK(cub::DeviceScan::InclusiveSum(scan, scan_bytes, koff + 1, koff + 1, (int)n, st));
    x->launches += 2;
    if (int rc = launch_hash_keys(x, d_tok, d_tok_off, 0, n, nullptr, nullptr, koff, keys, st)) return rc;
    const unsigned long long sb = x->tv.req_stamp ? reserve_stamps(x, (unsigned long long)cap) : 0;
    return launch_lookup_hits(x, keys, koff, 0, n, d_model, model0, d_filter, d_hits_out, sb, st);
}

// ---- routed (all-to-all) form of the sharded Score(): the device steps around the exchange (kernels_route.cuh) ----

int kvidx_key_owners_dev(kvidx_t* x, const uint64_t* d_keys, const uint32_t* d_model, uint32_t model0, int64_t n, uint8_t* d_owner_out) {
    if (!x || n < 0) return fail(KVIDX_EINVAL, "bad arguments");
    if (n == 0) return 0;
    ReadCall c(x);
    if (int rc = c.begin(0)) return rc;
    key_owners_kernel<<<(unsigned)((n + 255) / 256), 256, 0, x->stream>>>(x->tv, d_keys, d_model, model0, n, d_owner_out);
    x->launches += 1;
    CK(cudaGetLastError());
    return 0;
}

int kvidx_probe_slots_dev(kvidx_t* x, const uint64_t* d_keys, const uint32_t* d_model, uint32_t model0, int64_t n, void* d_slots_out) {
    if (!x || n < 0) return fail(KVIDX_EINVAL, "bad arguments");
    if (n == 0) return 0;
    ReadCall c(x);
    if (int rc = c.begin(kShards | kAfterWrites)) return rc;
    probe_slots_kernel<<<(unsigned)((n + 255) / 256), 256, 0, x->stream>>>(x->tv, d_keys, d_model, model0, n, static_cast<uint4*>(d_slots_out));
    x->launches += 1;
    CK(cudaGetLastError());
    return 0;
}

int kvidx_score_slots_dev(kvidx_t* x, const void* d_slots, const int64_t* d_key_off, int64_t n_prompts, const uint64_t* d_filter,
                          double* d_scores_out, uint8_t* d_has_keys_out) {
    if (!x || n_prompts < 0 || !d_scores_out) return fail(KVIDX_EINVAL, "bad arguments");
    if (n_prompts == 0) return 0;
    ReadCall c(x);
    if (int rc = c.begin(0)) return rc;
    score_slots_kernel<<<(unsigned)((n_prompts + 127) / 128), 128, 0, x->stream>>>(x->tv, static_cast<const uint4*>(d_slots), d_key_off, n_prompts, d_filter,
                                                                                   d_scores_out, d_has_keys_out);
    x->launches += 1;
    CK(cudaGetLastError());
    return 0;
}

// ---- write path -----------------------------------------------------------------------------

namespace {
int check_podtiers(kvidx* x, const kvidx_podtier_t* pts, int32_t m) {
    // dense score rows and filter rows are max_pods wide: a pod id beyond that cannot be scored or filtered
    for (int32_t j = 0; j < m; ++j)
        if (KVIDX_PT_POD(pts[j]) >= x->tv.max_pods) return fail(KVIDX_ERANGE, "pod id %u >= max_pods %u", KVIDX_PT_POD(pts[j]), x->tv.max_pods);
    return 0;
}
}  // namespace

int kvidx_add(kvidx_t* x, uint32_t model, const uint64_t* engine, const uint64_t* request, int64_t n,
              const kvidx_podtier_t* pts, int32_t m) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    if (n <= 0 || m <= 0 || !engine || !request || !pts) return fail(KVIDX_EINVAL, "no keys or entries provided for adding to index");
    if (model > 0xffffu) return fail(KVIDX_ERANGE, "model id %u > 65535", model);
    if (int rc0 = check_podtiers(x, pts, m)) return rc0;
    WriteCall w(x);
    if (int rc = w.begin(kDisarm | kShards)) return rc;
    if (int rc = w.share_with_room((uint64_t)n)) return rc;
    cudaStream_t st = wstream(x);
    uint64_t *d_engine, *d_request; uint16_t* d_pts; uint8_t* d_skip;
    CK(carve(x->d_misc, [&](Carver& c) { d_engine = c.take<uint64_t>(n); d_request = c.take<uint64_t>(n); d_pts = c.take<uint16_t>(m); d_skip = c.take<uint8_t>(n); }));
    CK(x->h_misc.need((size_t)n + 16));
    // pairs are added in order (in_memory.go:159): an engine key that appears again later in the call keeps the later mapping
    uint8_t* skip = x->h_misc.as<uint8_t>();
    bool any_dup = false;
    {
        std::unordered_map<uint64_t, int64_t> last;
        last.reserve((size_t)n * 2);
        for (int64_t i = 0; i < n; ++i) { skip[i] = 0; auto it = last.find(engine[i]); if (it != last.end()) { skip[it->second] = 1; any_dup = true; it->second = i; } else last.emplace(engine[i], i); }
    }
    CK(cudaMemcpyAsync(d_engine, engine, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_request, request, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_pts, pts, (size_t)m * 2, cudaMemcpyHostToDevice, st));
    if (any_dup) CK(cudaMemcpyAsync(d_skip, skip, (size_t)n, cudaMemcpyHostToDevice, st));
    const WriteTally t = w.tally();
    const int T = 128;
    add_kernel<<<(unsigned)((n + T - 1) / T), T, 0, st>>>(x->tv, model, d_engine, d_request, n, d_pts, m, any_dup ? d_skip : nullptr,
                                                         reserve_stamps(x, 2ull * (unsigned long long)n + 2));
    x->launches += 1;
    CK(cudaGetLastError());
    return w.settle(t, nullptr);
}

int kvidx_evict(kvidx_t* x, uint32_t model, uint64_t engine, const kvidx_podtier_t* pts, int32_t m) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    if (m <= 0 || !pts) return fail(KVIDX_EINVAL, "no entries provided for eviction from index");
    if (model > 0xffffu) return fail(KVIDX_ERANGE, "model id %u > 65535", model);
    if (int rc0 = check_podtiers(x, pts, m)) return rc0;
    WriteCall w(x);
    if (int rc = w.begin(kDisarm | kShards)) return rc;
    w.share();
    cudaStream_t st = wstream(x);
    CK(x->d_misc.need((size_t)m * 2 + 16));
    CK(cudaMemcpyAsync(x->d_misc.p, pts, (size_t)m * 2, cudaMemcpyHostToDevice, st));
    evict_kernel<<<1, 32, 0, st>>>(x->tv, model, engine, x->d_misc.as<uint16_t>(), m, reserve_stamps(x, 4));
    x->launches += 1;
    CK(cudaGetLastError());
    if (int rc = clock_sweep(x)) return rc;
    return refresh_counters(x);
}

int kvidx_get_request_key(kvidx_t* x, uint32_t model, uint64_t engine, uint64_t* out) {
    if (!x || !out) return fail(KVIDX_EINVAL, "bad arguments");
    ReadCall c(x);
    if (int rc = c.begin(kShards | kAfterWrites)) return rc;
    CK(x->d_rmisc.need(32));
    uint64_t* d_out = x->d_rmisc.as<uint64_t>();
    int* d_found = reinterpret_cast<int*>(d_out + 1);
    get_request_key_kernel<<<1, 32, 0, x->stream>>>(x->tv, model, engine, d_out, d_found, x->tv.req_stamp ? reserve_stamps(x, 1) : 0);
    x->launches += 1;
    CK(cudaGetLastError());
    struct { uint64_t r; int f; int pad; } h{};
    CK(cudaMemcpyAsync(&h, d_out, 16, cudaMemcpyDeviceToHost, x->stream));
    CK(cudaStreamSynchronize(x->stream));
    if (!h.f) return fail(KVIDX_ENOENT, "engine key not found: %u@%llu", model, (unsigned long long)engine);
    *out = h.r;
    return 0;
}

namespace {
// Both phases of a device-resident, pod-sorted event batch on the write stream (kernels_write.cuh).  Caller holds mu_w and
// `tables` shared.  max_ev_hashes: the batch's largest n_hashes (exact-LRU stamp stride), < 0: found on the device.
int launch_apply_events(kvidx* x, const kvidx_event_t* d_ev_sorted, const int64_t* d_queue_off, int64_t n_queues, int64_t n_events,
                        const uint64_t* d_hashes, int64_t n_hashes, const uint32_t* d_tokens, cudaStream_t st, int64_t max_ev_hashes) {
    unsigned long long sb = 0, stride = 0;
    if (x->tv.req_stamp) {
        if (max_ev_hashes < 0) {                      // read back: this mode serialises its calls anyway
            CK(x->d_misc.need(8));
            unsigned long long* d_max = x->d_misc.as<unsigned long long>();
            unsigned long long h_max = 0;
            CK(cudaMemsetAsync(d_max, 0, 8, st));
            max_event_hashes_kernel<<<(unsigned)((n_events + 255) / 256), 256, 0, st>>>(d_ev_sorted, n_events, d_max);
            x->launches += 1;
            CK(cudaMemcpyAsync(&h_max, d_max, 8, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            max_ev_hashes = (int64_t)h_max;
        }
        stride = 2ull + 2ull * (unsigned long long)max_ev_hashes;
        sb = reserve_stamps(x, stride * (unsigned long long)n_events);
    }
    const uint64_t* d_keys = nullptr; const uint64_t* d_pred = nullptr;
    const bool phase1 = x->write_phase1 == 1 || (x->write_phase1 < 0 && n_hashes >= x->write_phase1_min);
    if (phase1 && n_hashes > 0) {
        const uint64_t map_slots = pow2ceil((uint64_t)std::max<int64_t>(2 * n_events, 64));
        CK(x->d_wkeys.need((size_t)n_hashes * 8));
        CK(x->d_wpred.need((size_t)n_events * 8));
        // one zeroed block, cleared by one memset over its sections: work counter | ready[n] | next[n] | best[n]
        unsigned long long *d_next, *d_best; unsigned int *d_ready, *d_chain;
        size_t zbytes = 0;
        CK(carve(x->d_wready, [&](Carver& c) {
            d_next = c.take<unsigned long long>(2); d_ready = c.take<unsigned int>(n_events); d_chain = c.take<unsigned int>(n_events);
            d_best = c.take<unsigned long long>(n_events);
            zbytes = c.at;
        }));
        CK(x->d_wmap.need((size_t)map_slots * sizeof(WantEnt)));
        CK(cudaMemsetAsync(d_next, 0, zbytes, st));
        CK(cudaMemsetAsync(x->d_wmap.p, 0, (size_t)map_slots * sizeof(WantEnt), st));
        const int T = 256;
        want_parents_kernel<<<(unsigned)((n_events + T - 1) / T), T, 0, st>>>(d_ev_sorted, n_events, x->tv.block_size, x->d_wmap.as<WantEnt>(), (uint32_t)(map_slots - 1), d_chain);
        offer_blocks_kernel<<<(unsigned)((n_events * 32 + T - 1) / T), T, 0, st>>>(d_ev_sorted, n_events, x->tv.block_size, d_hashes, x->d_wmap.as<WantEnt>(), (uint32_t)(map_slots - 1), d_chain, d_best);
        const int64_t ctas = std::min<int64_t>((n_events + kHashEvThreads - 1) / kHashEvThreads, (int64_t)x->sm_count * 8);
        hash_events_kernel<<<(unsigned)ctas, kHashEvThreads, 0, st>>>(x->tv, d_ev_sorted, n_events, d_hashes, d_tokens, d_best,
                                                                     x->d_wkeys.as<uint64_t>(), x->d_wpred.as<uint64_t>(), d_ready, d_next);
        x->launches += 3;
        CK(cudaGetLastError());
        d_keys = x->d_wkeys.as<uint64_t>(); d_pred = x->d_wpred.as<uint64_t>();
    }
    const int T = 128;   // 4 queues per CTA
    apply_events_kernel<<<(unsigned)((n_queues * 32 + T - 1) / T), T, 0, st>>>(x->tv, d_ev_sorted, d_queue_off, n_queues, d_hashes, d_tokens, d_keys, d_pred,
                                                                               sb, stride);
    x->launches += 1;
    CK(cudaGetLastError());
    return 0;
}
}  // namespace

int kvidx_apply_events_dev(kvidx_t* x, const kvidx_event_t* d_ev_sorted, const int64_t* d_queue_off, int64_t n_queues, int64_t n_events,
                           const uint64_t* d_hashes, int64_t n_hashes, const uint32_t* d_tokens, int64_t* d_n_dropped) {
    if (!x || n_queues < 0 || n_events < 0 || n_hashes < 0) return fail(KVIDX_EINVAL, "bad arguments");
    if (n_queues == 0 || n_events == 0) return 0;
    WriteCall w(x);
    if (int rc = w.begin(kDisarm | kShards)) return rc;
    int rc = w.share_with_room((uint64_t)n_hashes);    // every hash of the batch may be a new key
    if (rc) return rc;
    cudaStream_t st = wstream(x);
    rc = launch_apply_events(x, d_ev_sorted, d_queue_off, n_queues, n_events, d_hashes, n_hashes, d_tokens, st, -1);
    if (rc) return rc;
    if ((rc = clock_sweep(x))) return rc;              // asynchronous too: the excess is read on the device
    // events dropped so far on this handle (cumulative, like the counter behind kvidx_apply_events' n_dropped_out)
    if (d_n_dropped) CK(cudaMemcpyAsync(d_n_dropped, &x->d_cnt->dropped_events, sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    CK(cudaEventRecord(x->ev_write, st));              // reads issued after this call are ordered after the batch
    return 0;
}

int kvidx_apply_events(kvidx_t* x, const kvidx_event_t* ev, int64_t n, const uint64_t* hashes, int64_t n_hashes,
                       const uint32_t* tokens, int64_t n_tokens, int64_t* n_dropped_out) {
    if (!x || n < 0) return fail(KVIDX_EINVAL, "bad arguments");
    if (n_dropped_out) *n_dropped_out = 0;
    if (n == 0) return 0;
    if (!ev) return fail(KVIDX_EINVAL, "NULL events");
    // validate + stable counting sort by pod -> per-pod FIFO queues (pool.go:129-144)
    std::vector<int64_t> qcount(KVIDX_MAX_PODS + 1, 0);
    uint64_t new_keys = 0;
    int64_t max_ev_hashes = 0;
    for (int64_t i = 0; i < n; ++i) {
        const kvidx_event_t& e = ev[i];
        max_ev_hashes = std::max<int64_t>(max_ev_hashes, e.n_hashes);
        if (e.op > KVIDX_EV_BLOCK_REMOVED) return fail(KVIDX_EINVAL, "event %lld: unknown op %u", (long long)i, e.op);
        if (e.model > 0xffffu) return fail(KVIDX_ERANGE, "event %lld: model id %u > 65535", (long long)i, e.model);
        if (KVIDX_PT_POD(e.podtier) >= x->tv.max_pods) return fail(KVIDX_ERANGE, "event %lld: pod id %u >= max_pods %u", (long long)i, KVIDX_PT_POD(e.podtier), x->tv.max_pods);
        if (e.hash_off + e.n_hashes > (uint64_t)n_hashes) return fail(KVIDX_EINVAL, "event %lld: hashes out of range", (long long)i);
        if (e.op == KVIDX_EV_BLOCK_STORED) {
            if (e.tok_off + e.n_tokens > (uint64_t)n_tokens) return fail(KVIDX_EINVAL, "event %lld: tokens out of range", (long long)i);
            new_keys += e.n_hashes;
        }
        qcount[KVIDX_PT_POD(e.podtier) + 1]++;
    }
    WriteCall w(x);
    if (int rc = w.begin(kDisarm | kShards)) return rc;
    if (int rc = w.share_with_room(new_keys)) return rc;
    cudaStream_t st = wstream(x);
    // compact non-empty queues
    std::vector<int64_t> start(KVIDX_MAX_PODS + 1, 0);
    for (uint32_t p = 0; p < KVIDX_MAX_PODS; ++p) start[p + 1] = start[p] + qcount[p + 1];
    CK(x->h_misc.need((size_t)n * sizeof(kvidx_event_t) + (size_t)(KVIDX_MAX_PODS + 2) * 8));
    kvidx_event_t* sorted = x->h_misc.as<kvidx_event_t>();
    int64_t* qoff = reinterpret_cast<int64_t*>(x->h_misc.as<uint8_t>() + (size_t)n * sizeof(kvidx_event_t));
    {
        std::vector<int64_t> cur(start.begin(), start.end() - 1);
        for (int64_t i = 0; i < n; ++i) sorted[cur[KVIDX_PT_POD(ev[i].podtier)]++] = ev[i];
    }
    int64_t nq = 0;
    for (uint32_t p = 0; p < KVIDX_MAX_PODS; ++p) if (qcount[p + 1]) { qoff[nq++] = start[p]; }
    qoff[nq] = n;
    CK(x->d_ev.need((size_t)n * sizeof(kvidx_event_t)));
    CK(x->d_qoff.need((size_t)(nq + 1) * 8));
    CK(x->d_hash.need((size_t)std::max<int64_t>(n_hashes, 1) * 8));
    CK(x->d_evtok.need((size_t)std::max<int64_t>(n_tokens, 1) * 4 + 16));
    CK(cudaMemcpyAsync(x->d_ev.p, sorted, (size_t)n * sizeof(kvidx_event_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(x->d_qoff.p, qoff, (size_t)(nq + 1) * 8, cudaMemcpyHostToDevice, st));
    if (n_hashes > 0) CK(cudaMemcpyAsync(x->d_hash.p, hashes, (size_t)n_hashes * 8, cudaMemcpyHostToDevice, st));
    if (n_tokens > 0) CK(cudaMemcpyAsync(x->d_evtok.p, tokens, (size_t)n_tokens * 4, cudaMemcpyHostToDevice, st));
    const WriteTally t = w.tally();
    if (int rc = launch_apply_events(x, x->d_ev.as<kvidx_event_t>(), x->d_qoff.as<int64_t>(), nq, n, x->d_hash.as<uint64_t>(), n_hashes,
                                     x->d_evtok.as<uint32_t>(), st, max_ev_hashes))
        return rc;
    return w.settle(t, n_dropped_out);
}

}  // extern "C"

namespace {
// ---- KVEvents payloads decoded on the device (kernels_decode.cuh) ---------------------------------------------------------
// A decode in two halves around the one read-back of its totals: decode_count runs the count pass, sorts the messages by pod
// and scans the counts into positions; decode_write runs the write pass into outputs sized from the totals.  Both on the
// write stream, under mu_w (the scratch, x->d_dec, is write-side).
struct DecodePlan {
    DecIn in{};
    int64_t *ev_cnt, *hash_cnt, *tok_cnt, *ev_base, *hash_base, *tok_base, *qoff;
    uint8_t* flags; uint32_t* sorted_val;
    DecTotals* d_tot; DecTotals tot{};
};

int check_tier_table(const uint8_t* tier_bytes, const int64_t* tier_off, uint32_t n_tiers, int32_t gpu_tier) {
    if (n_tiers == 0 || n_tiers > KVIDX_MAX_TIERS || !tier_off) return fail(KVIDX_EINVAL, "the tier table holds 1 to %u names", KVIDX_MAX_TIERS);
    for (uint32_t t = 0; t < n_tiers; ++t) if (tier_off[t + 1] < tier_off[t]) return fail(KVIDX_EINVAL, "tier offsets not monotone");
    if (tier_off[n_tiers] > tier_off[0] && !tier_bytes) return fail(KVIDX_EINVAL, "NULL tier names");
    if (gpu_tier >= (int32_t)n_tiers) return fail(KVIDX_EINVAL, "gpu_tier %d is not in the table", gpu_tier);
    return 0;
}

int check_payload_flags(uint32_t flags) {
    if (flags & ~(KVIDX_PAYLOAD_SKIP_UNKNOWN_TIER | KVIDX_PAYLOAD_STOP_AT_CLEARED)) return fail(KVIDX_EINVAL, "unknown flags 0x%x", flags);
    return 0;
}

int decode_count(kvidx* x, DecodePlan& pl, const uint8_t* tier_bytes, const int64_t* tier_off, uint32_t n_tiers, int32_t gpu_tier,
                 cudaStream_t st) {
    const int64_t n = pl.in.n_msgs;
    const uint32_t P = x->tv.max_pods;
    const uint64_t tb = (uint64_t)(tier_off[n_tiers] - tier_off[0]);
    size_t sort_bytes = 0, scan_bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                       (uint32_t*)nullptr, (int)n, 0, KVIDX_POD_BITS, st));
    CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int64_t*)nullptr, (int64_t*)nullptr, (int)n, st));
    uint8_t* d_tier; unsigned long long* pod_ev; uint32_t *key, *key2, *val; void* tmp;
    CK(carve(x->d_dec, [&](Carver& c) {
        d_tier = c.take<uint8_t>(tb); pod_ev = c.take<unsigned long long>(P); pl.d_tot = c.take<DecTotals>(1); pl.qoff = c.take<int64_t>(P + 1);
        pl.ev_cnt = c.take<int64_t>(n); pl.hash_cnt = c.take<int64_t>(n); pl.tok_cnt = c.take<int64_t>(n);
        pl.ev_base = c.take<int64_t>(n); pl.hash_base = c.take<int64_t>(n); pl.tok_base = c.take<int64_t>(n);
        pl.flags = c.take<uint8_t>(n); key = c.take<uint32_t>(n); key2 = c.take<uint32_t>(n); val = c.take<uint32_t>(n);
        pl.sorted_val = c.take<uint32_t>(n); tmp = c.take<uint8_t>(std::max(sort_bytes, scan_bytes));
    }));
    TierTable& tt = pl.in.tt;
    tt.bytes = d_tier; tt.n = n_tiers; tt.gpu = gpu_tier;
    for (uint32_t t = 0; t <= n_tiers; ++t) tt.off[t] = (uint64_t)(tier_off[t] - tier_off[0]);
    if (int rc = x->snap.h2d(d_tier, tier_bytes + tier_off[0], tb, st)) return rc;
    CK(cudaMemsetAsync(pod_ev, 0, (size_t)P * 8, st));
    CK(cudaMemsetAsync(pl.d_tot, 0, sizeof(DecTotals), st));
    const unsigned g = (unsigned)((n + kDecThreads - 1) / kDecThreads);
    decode_count_kernel<<<g, kDecThreads, 0, st>>>(pl.in, pl.ev_cnt, pl.hash_cnt, pl.tok_cnt, pl.flags, key, val, pod_ev, pl.d_tot);
    decode_queues_kernel<<<1, kQueueThreads, 0, st>>>(pod_ev, P, pl.qoff, &pl.d_tot->queues);
    size_t b = sort_bytes;
    CK(cub::DeviceRadixSort::SortPairs(tmp, b, key, key2, val, pl.sorted_val, (int)n, 0, KVIDX_POD_BITS, st));
    decode_gather_kernel<<<g, kDecThreads, 0, st>>>(pl.sorted_val, pl.ev_cnt, n, pl.ev_base);
    b = scan_bytes;
    CK(cub::DeviceScan::ExclusiveSum(tmp, b, pl.ev_base, pl.ev_base, (int)n, st));    // events: pod order
    b = scan_bytes;
    CK(cub::DeviceScan::ExclusiveSum(tmp, b, pl.hash_cnt, pl.hash_base, (int)n, st)); // hashes and tokens: message order
    b = scan_bytes;
    CK(cub::DeviceScan::ExclusiveSum(tmp, b, pl.tok_cnt, pl.tok_base, (int)n, st));
    x->launches += 3;
    CK(cudaGetLastError());
    CK(x->h_misc.need(sizeof(DecTotals)));
    CK(cudaMemcpyAsync(x->h_misc.p, pl.d_tot, sizeof(DecTotals), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    pl.tot = *x->h_misc.as<DecTotals>();
    return 0;
}

// counts_out of the ABI, and whether the batch can be applied as it is
int decode_verdict(kvidx* x, const DecTotals& t, uint32_t flags, int64_t* counts_out) {
    if (counts_out) {
        const unsigned long long c[KVIDX_PAYLOAD_COUNTS] = {t.messages, t.events, t.hashes, t.tokens, t.queues, t.admitted, t.removed_hashes, t.markers};
        for (int i = 0; i < KVIDX_PAYLOAD_COUNTS; ++i) counts_out[i] = (int64_t)c[i];
    }
    if (t.bad_off) return fail(KVIDX_EINVAL, "message offsets not monotone");
    if (t.bad_pod) return fail(KVIDX_ERANGE, "a message's pod id is >= max_pods %u", x->tv.max_pods);
    if (t.bad_model) return fail(KVIDX_ERANGE, "a message's model id is > 65535");
    if (t.unknown_tier && !(flags & KVIDX_PAYLOAD_SKIP_UNKNOWN_TIER))
        return fail(KVIDX_ENOENT, "a Medium names a tier the table lacks (messages flagged KVIDX_PAYLOAD_MSG_UNKNOWN_TIER)");
    if (t.markers && (flags & KVIDX_PAYLOAD_STOP_AT_CLEARED))
        return fail(KVIDX_ENOENT, "%llu AllBlocksCleared markers (messages flagged KVIDX_PAYLOAD_MSG_CLEARED)", t.markers);
    return 0;
}

int decode_write(kvidx* x, const DecodePlan& pl, kvidx_event_t* ev, int64_t* qoff, uint64_t* hashes, uint32_t* toks, cudaStream_t st) {
    const unsigned g = (unsigned)((pl.in.n_msgs + kDecThreads - 1) / kDecThreads);
    decode_write_kernel<<<g, kDecThreads, 0, st>>>(pl.in, pl.sorted_val, pl.ev_base, pl.hash_base, pl.hash_cnt, pl.tok_base, pl.tok_cnt,
                                                   pl.flags, ev, hashes, toks);
    x->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(qoff, pl.qoff, (size_t)(pl.tot.queues + 1) * 8, cudaMemcpyDeviceToDevice, st));
    return 0;
}
}  // namespace

extern "C" {

int kvidx_decode_event_payloads_dev(kvidx_t* x, const uint8_t* d_bytes, const int64_t* d_msg_off, int64_t n_msgs,
                                    const uint32_t* d_msg_pod, const uint32_t* d_msg_model, const uint8_t* tier_bytes,
                                    const int64_t* tier_off, uint32_t n_tiers, int32_t gpu_tier, uint32_t flags,
                                    kvidx_event_t* d_ev_out, int64_t ev_cap, int64_t* d_queue_off_out, int64_t queue_cap,
                                    uint64_t* d_hashes_out, int64_t hash_cap, uint32_t* d_tokens_out, int64_t tok_cap,
                                    uint8_t* d_msg_flags_out, int64_t counts_out[KVIDX_PAYLOAD_COUNTS]) {
    if (counts_out) for (int i = 0; i < KVIDX_PAYLOAD_COUNTS; ++i) counts_out[i] = 0;
    if (!x || n_msgs < 0 || n_msgs > INT32_MAX) return fail(KVIDX_EINVAL, "bad arguments");
    if (int rc = check_payload_flags(flags)) return rc;
    if (int rc = check_tier_table(tier_bytes, tier_off, n_tiers, gpu_tier)) return rc;
    if (n_msgs == 0) return 0;
    if (!d_bytes || !d_msg_off || !d_msg_pod || !d_msg_model) return fail(KVIDX_EINVAL, "NULL message arrays");
    WriteCall w(x);
    if (int rc = w.begin(0)) return rc;
    cudaStream_t st = wstream(x);
    DecodePlan pl;
    pl.in.bytes = d_bytes; pl.in.msg_off = d_msg_off; pl.in.msg_pod = d_msg_pod; pl.in.msg_model = d_msg_model;
    pl.in.n_msgs = n_msgs; pl.in.max_pods = x->tv.max_pods; pl.in.block_size = x->tv.block_size;
    if (int rc = decode_count(x, pl, tier_bytes, tier_off, n_tiers, gpu_tier, st)) return rc;
    const int rc = decode_verdict(x, pl.tot, flags, counts_out);
    if (d_msg_flags_out) CK(cudaMemcpyAsync(d_msg_flags_out, pl.flags, (size_t)n_msgs, cudaMemcpyDeviceToDevice, st));
    if (rc) return rc;
    const DecTotals& t = pl.tot;
    if ((int64_t)t.events > ev_cap || (int64_t)t.queues + 1 > queue_cap || (int64_t)t.hashes > hash_cap || (int64_t)t.tokens > tok_cap)
        return fail(KVIDX_ENOSPC, "outputs too small: %llu events, %llu queue offsets, %llu hashes, %llu tokens", t.events, t.queues + 1,
                    t.hashes, t.tokens);
    if ((t.events && !d_ev_out) || !d_queue_off_out || (t.hashes && !d_hashes_out) || (t.tokens && !d_tokens_out))
        return fail(KVIDX_EINVAL, "NULL output arrays");
    if (int rc2 = decode_write(x, pl, d_ev_out, d_queue_off_out, d_hashes_out, d_tokens_out, st)) return rc2;
    CK(cudaEventRecord(x->ev_write, st));              // reads issued after this call are ordered after it
    return 0;
}

int kvidx_apply_event_payloads(kvidx_t* x, const uint8_t* bytes, const int64_t* msg_off, int64_t n_msgs, const uint32_t* msg_pod,
                               const uint32_t* msg_model, const uint8_t* tier_bytes, const int64_t* tier_off, uint32_t n_tiers,
                               int32_t gpu_tier, uint32_t flags, uint8_t* msg_flags_out, int64_t counts_out[KVIDX_PAYLOAD_COUNTS],
                               int64_t* n_dropped_out) {
    if (counts_out) for (int i = 0; i < KVIDX_PAYLOAD_COUNTS; ++i) counts_out[i] = 0;
    if (n_dropped_out) *n_dropped_out = 0;
    if (!x || n_msgs < 0 || n_msgs > INT32_MAX) return fail(KVIDX_EINVAL, "bad arguments");
    if (int rc = check_payload_flags(flags)) return rc;
    if (int rc = check_tier_table(tier_bytes, tier_off, n_tiers, gpu_tier)) return rc;
    if (n_msgs == 0) return 0;
    if (!msg_off || !msg_pod || !msg_model) return fail(KVIDX_EINVAL, "NULL message arrays");
    for (int64_t i = 0; i < n_msgs; ++i) {
        if (msg_off[i + 1] < msg_off[i]) return fail(KVIDX_EINVAL, "message offsets not monotone at %lld", (long long)i);
        if (msg_pod[i] >= x->tv.max_pods) return fail(KVIDX_ERANGE, "message %lld: pod id %u >= max_pods %u", (long long)i, msg_pod[i], x->tv.max_pods);
        if (msg_model[i] > 0xffffu) return fail(KVIDX_ERANGE, "message %lld: model id %u > 65535", (long long)i, msg_model[i]);
    }
    const uint64_t nb = (uint64_t)(msg_off[n_msgs] - msg_off[0]);
    if (nb && !bytes) return fail(KVIDX_EINVAL, "NULL payload bytes");
    WriteCall w(x);
    if (int rc = w.begin(kShards)) return rc;
    cudaStream_t st = wstream(x);
    // the payloads on the device: bytes, offsets from 0, pods, models
    DecodePlan pl;
    uint8_t* d_bytes; int64_t* d_off; uint32_t *d_pod, *d_model;
    CK(carve(x->d_decin, [&](Carver& c) {
        d_bytes = c.take<uint8_t>(nb); d_off = c.take<int64_t>(n_msgs + 1); d_pod = c.take<uint32_t>(n_msgs); d_model = c.take<uint32_t>(n_msgs);
    }));
    std::vector<int64_t> off(msg_off, msg_off + n_msgs + 1);
    for (auto& o : off) o -= msg_off[0];
    if (int rc = x->snap.h2d(d_bytes, bytes + msg_off[0], nb, st)) return rc;
    if (int rc = x->snap.h2d(d_off, off.data(), off.size() * 8, st)) return rc;
    if (int rc = x->snap.h2d(d_pod, msg_pod, (size_t)n_msgs * 4, st)) return rc;
    if (int rc = x->snap.h2d(d_model, msg_model, (size_t)n_msgs * 4, st)) return rc;
    pl.in.bytes = d_bytes; pl.in.msg_off = d_off; pl.in.msg_pod = d_pod; pl.in.msg_model = d_model;
    pl.in.n_msgs = n_msgs; pl.in.max_pods = x->tv.max_pods; pl.in.block_size = x->tv.block_size;
    if (int rc = decode_count(x, pl, tier_bytes, tier_off, n_tiers, gpu_tier, st)) return rc;
    int rc = decode_verdict(x, pl.tot, flags, counts_out);
    if (msg_flags_out) if (int rc2 = x->snap.d2h(msg_flags_out, pl.flags, (size_t)n_msgs, st)) return rc2;
    if (rc) return rc;
    const DecTotals& t = pl.tot;
    if (t.events == 0) return 0;                       // as kvidx_apply_events with no event
    x->rm_armed = false;
    if ((rc = w.share_with_room(t.stored_hashes))) return rc;
    CK(x->d_ev.need((size_t)t.events * sizeof(kvidx_event_t)));
    CK(x->d_qoff.need((size_t)(t.queues + 1) * 8));
    CK(x->d_hash.need((size_t)std::max<uint64_t>(t.hashes, 1) * 8));
    CK(x->d_evtok.need((size_t)std::max<uint64_t>(t.tokens, 1) * 4 + 16));
    if ((rc = decode_write(x, pl, x->d_ev.as<kvidx_event_t>(), x->d_qoff.as<int64_t>(), x->d_hash.as<uint64_t>(), x->d_evtok.as<uint32_t>(), st)))
        return rc;
    const WriteTally tally = w.tally();
    rc = launch_apply_events(x, x->d_ev.as<kvidx_event_t>(), x->d_qoff.as<int64_t>(), (int64_t)t.queues, (int64_t)t.events,
                             x->d_hash.as<uint64_t>(), (int64_t)t.hashes, x->d_evtok.as<uint32_t>(), st, (int64_t)t.max_ev_hashes);
    return rc ? rc : w.settle(tally, n_dropped_out);
}

}  // extern "C"

namespace {
// Arguments shared by kvidx_remove_pods and kvidx_shard_remove_pods; 0 if they are usable.
int check_removal(kvidx* x, const uint64_t* pod_mask, uint32_t tier_mask) {
    if (!x || !pod_mask) return fail(KVIDX_EINVAL, "bad arguments");
    if ((tier_mask & 0xffffu) == 0) return fail(KVIDX_EINVAL, "empty tier mask");
    uint64_t any = 0;
    for (uint32_t w = 0; w < x->tv.filter_words; ++w) any |= pod_mask[w];
    if (!any) return fail(KVIDX_EINVAL, "empty pod mask");
    return 0;
}

// The two sweeps of a removal (kernels_remove.cuh).  Caller holds mu_w and `tables` shared.
//   d_misc: out[4] | pod mask | unsharded only: removed_slot (rs bits) | removed_home (rs / 2 bits)
//   sharded: this rank's bitmaps are the tail of its request-table allocation (alloc_tables), a peer's the tail of its own
// pass 1 (remove_req_kernel) clears and fills this handle's bitmaps; pass 2 (remove_eng_kernel) reads those of every
// request shard's owner.  removed_out: {entries, request keys, engine keys} removed by the passes that ran.
int run_removal(kvidx* x, const uint64_t* pod_mask, uint32_t tier_mask, bool pass1, bool pass2, uint64_t removed_out[3]) {
    cudaStream_t st = wstream(x);
    const uint64_t rs = x->tv.req_mask + 1;
    const uint32_t FW = x->tv.filter_words;
    const bool sharded = x->tv.shard_bits != 0;
    // the layout depends on the geometry and the mask width only: d_misc is not resized in phase 1 (phase 0 sized it and no
    // write call came between), so the bitmaps are where phase 0 left them
    unsigned long long* out; uint64_t* mask; uint32_t* bits;
    CK(carve(x->d_misc, [&](Carver& c) {
        out = c.take<unsigned long long>(4); mask = c.take<uint64_t>(FW); bits = c.take<uint32_t>(sharded ? 0 : remove_bitmap_bytes(rs) / 4);
    }));
    CK(x->h_misc.need(32));
    auto bits_of = [&](uint32_t r) { return sharded ? reinterpret_cast<uint32_t*>(x->tv.req_peer[r] + rs) : bits; };
    uint32_t* mine = bits_of(x->tv.shard_rank);
    RemoveArgs ra{mask, tier_mask & 0xffffu, mine, mine + rs / 32, out, {}, {}};
    for (uint32_t r = 0; r < (1u << x->tv.shard_bits); ++r) { ra.owner_slot[r] = bits_of(r); ra.owner_home[r] = bits_of(r) + rs / 32; }
    CK(cudaMemsetAsync(out, 0, 32, st));
    if (pass1) {
        CK(cudaMemsetAsync(mine, 0, remove_bitmap_bytes(rs), st));
        CK(cudaMemcpyAsync(mask, pod_mask, (size_t)FW * 8, cudaMemcpyHostToDevice, st));
    }
    const unsigned ctas = (unsigned)std::min<uint64_t>(rs / kRemoveThreads, (uint64_t)x->sm_count * 8);
    if (pass1) remove_req_kernel<<<ctas, kRemoveThreads, 0, st>>>(x->tv, ra);
    if (pass2) remove_eng_kernel<<<ctas, kRemoveThreads, 0, st>>>(x->tv, ra);
    x->launches += (pass1 ? 1 : 0) + (pass2 ? 1 : 0);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(x->h_misc.p, out, 24, cudaMemcpyDeviceToHost, st));
    int rc = refresh_counters(x);                      // synchronises the write stream: the removal has taken effect
    if (rc) return rc;
    if (removed_out) memcpy(removed_out, x->h_misc.p, 24);
    return 0;
}
}  // namespace

extern "C" {

int kvidx_remove_pods(kvidx_t* x, const uint64_t* pod_mask, uint32_t tier_mask, uint64_t removed_out[3]) {
    if (removed_out) removed_out[0] = removed_out[1] = removed_out[2] = 0;
    if (!x || !pod_mask) return fail(KVIDX_EINVAL, "bad arguments");
    // an engine mapping lives with its engine hash's owner and its request key with another rank: cleaning it up on a
    // sharded index needs the removal bitmaps of every rank, which the collective kvidx_shard_remove_pods provides
    if (x->tv.shard_bits) return fail(KVIDX_EINVAL, "kvidx_remove_pods is not supported on a sharded index (kvidx_shard_remove_pods is its collective form)");
    if (int rc = check_removal(x, pod_mask, tier_mask)) return rc;
    WriteCall w(x);
    if (int rc = w.begin(kDisarm)) return rc;
    w.share();
    return run_removal(x, pod_mask, tier_mask, true, true, removed_out);
}

int kvidx_shard_remove_pods(kvidx_t* x, const uint64_t* pod_mask, uint32_t tier_mask, uint32_t phase, uint64_t removed_out[3]) {
    if (removed_out) removed_out[0] = removed_out[1] = removed_out[2] = 0;
    if (phase > 1) return fail(KVIDX_EINVAL, "phase %u: a removal has phases 0 and 1", phase);
    if (int rc = check_removal(x, pod_mask, tier_mask)) return rc;
    const uint32_t FW = x->tv.filter_words;
    WriteCall w(x);
    if (int rc = w.begin(kShards)) return rc;
    if (phase == 1) {
        if (!x->rm_armed)
            return fail(KVIDX_EINVAL, "phase 1 without a preceding phase 0 on this handle, or a write call came between the phases");
        if (x->rm_tiers != (tier_mask & 0xffffu) || memcmp(x->rm_pods, pod_mask, (size_t)FW * 8) != 0)
            return fail(KVIDX_EINVAL, "phase 1 with other pod / tier masks than phase 0");
    }
    x->rm_armed = false;
    w.share();
    int rc = run_removal(x, pod_mask, tier_mask, phase == 0, phase == 1, removed_out);
    if (rc || phase == 1) return rc;
    x->rm_armed = true;
    x->rm_tiers = tier_mask & 0xffffu;
    memcpy(x->rm_pods, pod_mask, (size_t)FW * 8);
    return 0;
}

}  // extern "C"

namespace {
// ---- snapshot / restore (format v1, include/kvidx.h; kernels_snapshot.cuh) ----------------------------------------------
constexpr uint64_t kSnapHeaderBytes = 64;
constexpr uint32_t kSnapVersion = 1, kSnapFlagRecency = 1;
const char kSnapMagic[8] = {'K', 'V', 'I', 'D', 'X', 'S', 'N', 'P'};

struct SnapHeader {                               // the 64 header bytes (little-endian hosts: x86-64, aarch64)
    char magic[8];
    uint32_t version, flags, block_size, pods_per_key;
    uint64_t init_hash, n_request, n_engine;
    uint32_t pod_span, model_span;
    uint64_t zero;
};
static_assert(sizeof(SnapHeader) == kSnapHeaderBytes, "snapshot header is 64 bytes");

void release_snap(kvidx* x) { x->d_snap.release(); }

unsigned snap_ctas(kvidx* x, uint64_t n) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((n + kSnapThreads - 1) / kSnapThreads, (uint64_t)x->sm_count * 8));
}

// The sort buffers of up to N records (two of each: keys, slot indices, models) and the cub scratch
struct SnapSort {
    uint64_t* k[2]; uint32_t* i[2]; uint16_t* m[2]; void* tmp; size_t tmp_bytes;
    void carve(Carver& c, uint64_t N) {
        for (auto& p : k) p = c.take<uint64_t>(N);
        for (auto& p : i) p = c.take<uint32_t>(N);
        for (auto& p : m) p = c.take<uint16_t>(N);
        tmp = c.take<uint8_t>(tmp_bytes);
    }
};

// One table's FULL slots, sorted by (model, hash): slot indices in *sorted (inside `so`).  `misc` is zeroed by the caller.
// Slot indices are 32-bit: a table of 2^32 slots would be 128 GB.
template <int kMeta>
int snap_sort_table(kvidx* x, const void* tab, uint64_t slots, uint64_t expect, const SnapSort& so, SnapMisc* d_misc,
                    const uint32_t** sorted, const char* what, cudaStream_t st) {
    uint64_t *k0 = so.k[0], *k1 = so.k[1];
    uint32_t *i0 = so.i[0], *i1 = so.i[1];
    uint16_t *m0 = so.m[0], *m1 = so.m[1];
    void* tmp = so.tmp;
    const size_t sort_tmp = so.tmp_bytes;
    const unsigned ctas = (unsigned)std::min<uint64_t>(slots / kSnapThreads, (uint64_t)x->sm_count * 8);
    snap_compact_kernel<kMeta><<<ctas, kSnapThreads, 0, st>>>(static_cast<const uint4*>(tab), slots, expect, k0, i0, d_misc);
    x->launches += 1;
    CK(cudaGetLastError());
    SnapMisc* h = x->h_misc.as<SnapMisc>();
    CK(cudaMemcpyAsync(h, d_misc, sizeof(SnapMisc), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (h->n != expect)
        return fail(KVIDX_ECUDA, "snapshot: %llu FULL %s slots, but the handle counts %llu", (unsigned long long)h->n, what, (unsigned long long)expect);
    *sorted = i0;
    if (expect == 0) return 0;
    size_t tb = sort_tmp;
    CK(cub::DeviceRadixSort::SortPairs(tmp, tb, k0, k1, i0, i1, (int)expect, 0, 64, st));
    *sorted = i1;
    x->launches += 5;
    if (h->model_span > 1) {                          // more than one model: a stable pass over the model bits
        int bits = 0;
        while ((1u << bits) < h->model_span) ++bits;
        snap_models_kernel<kMeta><<<(unsigned)((expect + 255) / 256), 256, 0, st>>>(static_cast<const uint4*>(tab), i1, expect, m0);
        tb = sort_tmp;
        CK(cub::DeviceRadixSort::SortPairs(tmp, tb, m0, m1, i1, i0, (int)expect, 0, bits, st));
        *sorted = i0;
        x->launches += 4;
    }
    CK(cudaGetLastError());
    return 0;
}

int snapshot_impl(kvidx* x, void* buf, uint64_t R, uint64_t E, bool rec) {
    cudaStream_t st = wstream(x);
    const uint64_t N = std::max<uint64_t>(std::max(R, E), 1);
    SnapSort so{};
    size_t t2 = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, so.tmp_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)N, 0, 64, st));
    CK(cub::DeviceRadixSort::SortPairs(nullptr, t2, (uint16_t*)nullptr, (uint16_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)N, 0, 16, st));
    so.tmp_bytes = std::max(so.tmp_bytes, t2);
    // device scratch: misc (2 x SnapMisc) | image body (its byte layout, moved in one staged copy) | sort buffers
    const size_t body = (size_t)(32 * R + 24 * E + (rec ? 8 * (R + E) : 0));
    SnapMisc* d_req; uint8_t* out;
    CK(carve(x->d_snap, [&](Carver& c) { d_req = c.take<SnapMisc>(2); out = c.take<uint8_t>(body); so.carve(c, N); }));
    CK(x->h_misc.need(64));
    SnapMisc* d_eng = d_req + 1;
    CK(cudaMemsetAsync(d_req, 0, 2 * sizeof(SnapMisc), st));
    uint4* req_rec = reinterpret_cast<uint4*>(out);
    unsigned long long* eng_rec = reinterpret_cast<unsigned long long*>(out + 32 * R);
    unsigned long long* req_st = rec ? reinterpret_cast<unsigned long long*>(out + 32 * R + 24 * E) : nullptr;
    unsigned long long* eng_st = rec ? req_st + R : nullptr;
    const uint32_t* idx = nullptr;
    int rc = snap_sort_table<3>(x, x->tv.req, x->tv.req_mask + 1, R, so, d_req, &idx, "request", st);
    if (rc) return rc;
    const uint32_t model_span_req = x->h_misc.as<SnapMisc>()->model_span;
    if (R) {
        snap_req_records_kernel<<<snap_ctas(x, R), kSnapThreads, 0, st>>>(x->tv.req, idx, R, req_rec, x->tv.req_stamp, req_st, d_req);
        x->launches += 1;
        CK(cudaGetLastError());
    }
    rc = snap_sort_table<0>(x, x->tv.eng, x->tv.eng_mask + 1, E, so, d_eng, &idx, "engine", st);
    if (rc) return rc;
    const uint32_t model_span_eng = x->h_misc.as<SnapMisc>()->model_span;
    if (E) {
        snap_eng_records_kernel<<<(unsigned)((E + 255) / 256), 256, 0, st>>>(x->tv.eng, idx, E, eng_rec, eng_st);
        x->launches += 1;
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(x->h_misc.p, d_req, sizeof(SnapMisc), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    SnapHeader hd{};
    memcpy(hd.magic, kSnapMagic, 8);
    hd.version = kSnapVersion; hd.flags = rec ? kSnapFlagRecency : 0;
    hd.block_size = x->tv.block_size; hd.pods_per_key = x->tv.pods_per_key; hd.init_hash = x->tv.init_hash;
    hd.n_request = R; hd.n_engine = E;
    hd.pod_span = x->h_misc.as<SnapMisc>()->pod_span;
    hd.model_span = std::max(model_span_req, model_span_eng);
    memcpy(buf, &hd, sizeof hd);
    return x->snap.d2h(static_cast<char*>(buf) + kSnapHeaderBytes, out, body, st);
}

// slots: the size a growable handle's tables take before the insert (restore_call); the current size otherwise
int restore_impl(kvidx* x, WriteCall& w, const uint8_t* body, const SnapHeader& hd, uint64_t slots, uint64_t restored_out[2]) {
    cudaStream_t st = wstream(x);
    const uint64_t R = hd.n_request, E = hd.n_engine;
    const bool rec = hd.flags & kSnapFlagRecency;
    const size_t nbody = (size_t)(32 * R + 24 * E + (rec ? 8 * (R + E) : 0));
    // recency images: each section's stamps sorted (8 B per record) + the cub scratch
    size_t sort_tmp = 0;
    if (rec) CK(cub::DeviceRadixSort::SortKeys(nullptr, sort_tmp, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                               (int)std::max<uint64_t>(std::max(R, E), 1), 0, 64, st));
    // device scratch: the checks and, sharded, the records per owner (16 x 8 B) in one zeroed block | image body | sorted
    // stamps | cub scratch
    uint8_t *dchk, *dbody, *tmp; unsigned long long* sorted;
    CK(carve(x->d_snap, [&](Carver& c) {
        dchk = c.take<uint8_t>(2 * sizeof(SnapCheck) + 16 * 8); dbody = c.take<uint8_t>(nbody);
        sorted = c.take<unsigned long long>(rec ? R + E : 0); tmp = c.take<uint8_t>(sort_tmp);
    }));
    CK(x->h_misc.need(2 * sizeof(SnapCheck) + 16 + 16 * 8));
    SnapCheck* d_chk = reinterpret_cast<SnapCheck*>(dchk);
    unsigned long long* d_hist = reinterpret_cast<unsigned long long*>(d_chk + 2);
    CK(cudaMemsetAsync(dchk, 0, 2 * sizeof(SnapCheck) + 16 * 8, st));
    CK(cudaMemsetAsync(&d_chk[0].first_bad, 0xff, 8, st));
    CK(cudaMemsetAsync(&d_chk[1].first_bad, 0xff, 8, st));
    int rc = x->snap.h2d(dbody, body, nbody, st);
    if (rc) return rc;
    const uint4* req_rec = reinterpret_cast<const uint4*>(dbody);
    const unsigned long long* eng_rec = reinterpret_cast<const unsigned long long*>(dbody + 32 * R);
    const unsigned long long* req_st = rec ? reinterpret_cast<const unsigned long long*>(dbody + 32 * R + 24 * E) : nullptr;
    const unsigned long long* eng_st = rec ? req_st + R : nullptr;
    // 1. validate every record before anything is inserted
    if (R) snap_check_req_kernel<<<snap_ctas(x, R), kSnapThreads, 0, st>>>(req_rec, R, req_st, x->tv.pods_per_key, x->tv.max_pods, d_chk);
    if (E) snap_check_eng_kernel<<<snap_ctas(x, E), kSnapThreads, 0, st>>>(eng_rec, E, eng_st, d_chk + 1);
    x->launches += (R ? 1 : 0) + (E ? 1 : 0);
    const bool sharded = x->tv.shard_bits != 0;
    if (sharded) {                                    // the whole image's records per owner, for the room check below
        snap_owner_hist_kernel<<<snap_ctas(x, R + E), kSnapThreads, 0, st>>>(req_rec, R, eng_rec, E, x->tv.shard_bits, d_hist);
        x->launches += 1;
    }
    CK(cudaGetLastError());
    // recency: no value repeats within a section; in exact-LRU mode the `capacity` most recent keys of each table are kept,
    // which is what enforce_caps would leave, found here as the stamp of rank n - capacity instead of n - capacity sweeps
    const bool keep = x->tv.req_stamp != nullptr;
    SnapCheck* h = x->h_misc.as<SnapCheck>();
    unsigned long long* h_from = reinterpret_cast<unsigned long long*>(h + 2);
    unsigned long long* h_hist = h_from + 2;
    h_from[0] = h_from[1] = 0;
    if (rec) {
        const unsigned long long* sect[2] = {req_st, eng_st};
        const uint64_t cnt[2] = {R, E};
        for (int tb = 0; tb < 2; ++tb) {
            if (!cnt[tb]) continue;
            size_t tb_bytes = sort_tmp;
            CK(cub::DeviceRadixSort::SortKeys(tmp, tb_bytes, sect[tb], sorted, (int)cnt[tb], 0, 64, st));
            snap_check_ties_kernel<<<snap_ctas(x, cnt[tb]), kSnapThreads, 0, st>>>(sorted, cnt[tb], d_chk + tb);
            x->launches += 5;
            if (keep && cnt[tb] > x->tv.capacity)
                CK(cudaMemcpyAsync(&h_from[tb], sorted + (cnt[tb] - x->tv.capacity), 8, cudaMemcpyDeviceToHost, st));
            sorted += cnt[tb];
        }
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(h, d_chk, 2 * sizeof(SnapCheck), cudaMemcpyDeviceToHost, st));
    if (sharded) CK(cudaMemcpyAsync(h_hist, d_hist, 16 * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int tb = 0; tb < 2; ++tb) {
        const unsigned b = h[tb].bad;
        if (b)
            return fail(KVIDX_EINVAL, "malformed snapshot image: %s record %llu:%s%s%s%s%s%s", tb ? "engine" : "request", h[tb].first_bad,
                        b & kSnapBadOrder ? " not in strictly ascending (model, hash) order;" : "",
                        b & kSnapBadCount ? " entry count outside 1..pods_per_key;" : "",
                        b & kSnapBadEntry ? " repeated entry or pod id >= max_pods;" : "",
                        b & kSnapBadPad ? " non-zero padding or entry past the count;" : "",
                        b & kSnapBadStamp ? " recency value >= 2^63;" : "",
                        b & kSnapBadTie ? " a recency value repeats (index given in sorted order);" : "");
    }
    const uint32_t model_span = std::max(h[0].model_span, h[1].model_span);
    if (h[0].pod_span != hd.pod_span || model_span != hd.model_span)
        return fail(KVIDX_EINVAL, "malformed snapshot image: header pod_span %u / model_span %u, records %u / %u", hd.pod_span,
                    hd.model_span, h[0].pod_span, model_span);
    const unsigned long long stamp_max = std::max(h[0].stamp_max, h[1].stamp_max);
    // sharded: every owner's share against the write path's limit (90 % of a shard's slots; kvidx_shard_attach enforces
    // equal geometry on all shards), so that every rank refuses an image that does not fit before any rank inserts
    if (sharded) {
        const uint64_t rs = x->tv.req_mask + 1, es = x->tv.eng_mask + 1;
        for (uint32_t o = 0; o < (1u << x->tv.shard_bits); ++o)
            if (h_hist[o] * 10 > rs * 9 || h_hist[8 + o] * 10 > es * 9)
                return fail(KVIDX_ENOSPC, "shard %u full: it owns %llu request / %llu engine keys of the image, %llu / %llu slots", o,
                            h_hist[o], h_hist[8 + o], (unsigned long long)rs, (unsigned long long)es);
    }
    // 2. a growable handle's tables grow to the size the image needs: they hold no live key, so the rebuild only reallocates
    //    them (and drops their tombstones).  If that allocation fails, the image goes into the old tables if the write
    //    path's limit admits it there.
    if (slots > x->tv.req_mask + 1) {
        if ((rc = w.grow_shared(slots))) {
            if (rc != KVIDX_ENOMEM) return rc;
            const uint64_t rs = x->tv.req_mask + 1;
            if (R * 10 > rs * 9 || E * 10 > rs * 9)
                return fail(KVIDX_ENOSPC, "table full: %llu request / %llu engine keys in %llu slots; growing them to %llu slots failed: %s",
                            (unsigned long long)R, (unsigned long long)E, (unsigned long long)rs, (unsigned long long)slots,
                            std::string(g_err).c_str());
        }
    }
    // the target's tombstones go (it holds no live key, so this is clearing both tables)
    const Counters& c = *x->h_cnt;
    if (c.req_tomb || c.eng_tomb) {
        CK(cudaMemsetAsync(x->tv.req, 0, (x->tv.req_mask + 1) * sizeof(ReqSlot), st));
        CK(cudaMemsetAsync(x->tv.eng, 0, (x->tv.eng_mask + 1) * sizeof(EngSlot), st));
        if (x->tv.req_stamp) CK(cudaMemsetAsync(x->tv.req_stamp, 0, (x->tv.req_mask + 1) * 8, st));
        CK(cudaMemsetAsync(&x->d_cnt->req_tomb, 0, sizeof(unsigned long long), st));
        CK(cudaMemsetAsync(&x->d_cnt->eng_tomb, 0, sizeof(unsigned long long), st));
    }
    // restored keys start unreferenced on a CLOCK handle
    if (x->tv.req_ref) {
        CK(cudaMemsetAsync(x->tv.req_ref, 0, (x->tv.req_mask + 1) / 8, st));
        CK(cudaMemsetAsync(x->tv.eng_ref, 0, (x->tv.eng_mask + 1) / 8, st));
    }
    // 3. insert; recency is kept only by an exact-LRU handle
    const unsigned long long nospc_before = x->h_cnt->nospc, from_req = h_from[0], from_eng = h_from[1];
    if (R) restore_req_kernel<<<snap_ctas(x, R), kSnapThreads, 0, st>>>(x->tv, req_rec, R, keep ? req_st : nullptr, from_req);
    if (E) restore_eng_kernel<<<snap_ctas(x, E), kSnapThreads, 0, st>>>(x->tv, eng_rec, E, keep ? eng_st : nullptr, from_eng);
    x->launches += (R ? 1 : 0) + (E ? 1 : 0);
    CK(cudaGetLastError());
    if ((rc = refresh_counters(x))) return rc;
    if (x->h_cnt->nospc != nospc_before) return fail(KVIDX_ENOSPC, "%llu restored keys found no slot", x->h_cnt->nospc - nospc_before);
    if (keep) {                                       // later stamps must be newer than every restored one
        unsigned long long cur = x->clock.load();
        while (cur <= stamp_max && !x->clock.compare_exchange_weak(cur, stamp_max + 1)) {}
    }
    release_snap(x);
    if ((rc = cap_keys(x))) return rc;                // exact LRU: a no-op after the cut above; CLOCK: the sweep cuts the image
    if (restored_out) { restored_out[0] = x->h_cnt->req_full; restored_out[1] = x->h_cnt->eng_full; }
    return 0;
}

// Header and length of an image as kvidx_restore checks them before looking at the handle.
int check_image_header(const void* buf, uint64_t len, SnapHeader* out) {
    if (len < kSnapHeaderBytes) return fail(KVIDX_EINVAL, "malformed snapshot image: %llu bytes, shorter than the header", (unsigned long long)len);
    SnapHeader& hd = *out;
    memcpy(&hd, buf, sizeof hd);
    if (memcmp(hd.magic, kSnapMagic, 8) != 0) return fail(KVIDX_EINVAL, "malformed snapshot image: bad magic");
    if (hd.version != kSnapVersion) return fail(KVIDX_EINVAL, "unsupported snapshot version %u (this library reads %u)", hd.version, kSnapVersion);
    if ((hd.flags & ~kSnapFlagRecency) || hd.zero) return fail(KVIDX_EINVAL, "malformed snapshot image: unknown flags or non-zero header padding");
    const bool rec = hd.flags & kSnapFlagRecency;
    const uint64_t R = hd.n_request, E = hd.n_engine;
    if (R > (len >> 5) || E > len / 24 ||
        len != kSnapHeaderBytes + 32 * R + 24 * E + (rec ? 8 * (R + E) : 0))
        return fail(KVIDX_EINVAL, "malformed snapshot image: %llu bytes do not hold %llu request and %llu engine records%s",
                    (unsigned long long)len, (unsigned long long)R, (unsigned long long)E, rec ? " with recency" : "");
    return 0;
}

// The (model, hash) sort key of a record: model in the top bits of `hi`, so that pairs compare as one 80-bit number.
struct RecKey {
    uint64_t hi, lo;
    bool operator<(const RecKey& o) const { return hi < o.hi || (hi == o.hi && lo < o.lo); }
    bool operator==(const RecKey& o) const { return hi == o.hi && lo == o.lo; }
};
RecKey rec_key(const uint8_t* r, size_t model_off) {
    uint64_t h; uint16_t m;
    memcpy(&h, r, 8); memcpy(&m, r + model_off, 2);
    return RecKey{m, h};
}

// k-way merge of the parts' request sections, then of their engine sections, into dst (nullptr: check only).  Records of
// one part must be strictly ascending; a key in two parts is refused.  A linear scan over the part heads picks the next
// record: the parts are shards, at most 8 of them in a sharded index.
int merge_images(const void* const* parts, const std::vector<SnapHeader>& hd, uint8_t* dst) {
    const size_t np = hd.size();
    for (int sect = 0; sect < 2; ++sect) {
        const size_t rb = sect ? 24 : 32, moff = sect ? 16 : 8;
        const char* what = sect ? "engine" : "request";
        std::vector<const uint8_t*> cur(np);
        std::vector<uint64_t> left(np);
        for (size_t p = 0; p < np; ++p) {
            cur[p] = static_cast<const uint8_t*>(parts[p]) + kSnapHeaderBytes + (sect ? 32 * hd[p].n_request : 0);
            left[p] = sect ? hd[p].n_engine : hd[p].n_request;
        }
        std::vector<RecKey> head(np);
        for (size_t p = 0; p < np; ++p) if (left[p]) head[p] = rec_key(cur[p], moff);
        bool have_prev = false;
        RecKey prev{};
        size_t prev_part = 0;
        for (;;) {
            size_t best = np;
            for (size_t p = 0; p < np; ++p)
                if (left[p] && (best == np || head[p] < head[best])) best = p;
            if (best == np) break;
            if (have_prev && head[best] == prev)
                return fail(KVIDX_EINVAL, "%s key (model %llu, hash %#llx) is in parts %zu and %zu: parts must come from disjoint shards", what,
                            (unsigned long long)prev.hi, (unsigned long long)prev.lo, prev_part, best);
            if (dst) { memcpy(dst, cur[best], rb); dst += rb; }
            prev = head[best]; prev_part = best; have_prev = true;
            cur[best] += rb;
            if (--left[best]) {
                head[best] = rec_key(cur[best], moff);
                if (!(prev < head[best]))
                    return fail(KVIDX_EINVAL, "malformed snapshot image: part %zu %s record %llu: not in strictly ascending (model, hash) order", best,
                                what, (unsigned long long)((sect ? hd[best].n_engine : hd[best].n_request) - left[best]));
            }
        }
    }
    return 0;
}

int snapshot_call(kvidx* x, void* buf, uint64_t cap, uint64_t* size_out) {
    WriteCall w(x);
    if (int rc = w.begin(0)) return rc;
    w.share();
    int rc = refresh_counters(x);                     // synchronises the write stream: earlier asynchronous batches are in
    if (rc) return rc;
    const uint64_t R = x->h_cnt->req_full, E = x->h_cnt->eng_full;
    const bool rec = x->tv.req_stamp != nullptr;
    const uint64_t size = kSnapHeaderBytes + 32 * R + 24 * E + (rec ? 8 * (R + E) : 0);
    *size_out = size;
    if (!buf || cap < size) return fail(KVIDX_ENOSPC, "the snapshot needs %llu bytes, the buffer has %llu", (unsigned long long)size,
                                        (unsigned long long)(buf ? cap : 0));
    rc = snapshot_impl(x, buf, R, E, rec);
    release_snap(x);
    return rc;
}

// kvidx_restore after its argument checks; on a sharded handle only the records this shard owns are inserted, and the room
// check is every owner's (restore_impl)
int restore_call(kvidx* x, const void* buf, uint64_t len, uint64_t restored_out[2]) {
    SnapHeader hd;
    if (int rc = check_image_header(buf, len, &hd)) return rc;
    const bool rec = hd.flags & kSnapFlagRecency;
    const uint64_t R = hd.n_request, E = hd.n_engine;
    if (hd.block_size != x->tv.block_size || hd.init_hash != x->tv.init_hash || hd.pods_per_key != x->tv.pods_per_key)
        return fail(KVIDX_EINVAL, "snapshot of another configuration: block_size %u, init_hash %#llx, pods_per_key %u (this index: %u, %#llx, %u)",
                    hd.block_size, (unsigned long long)hd.init_hash, hd.pods_per_key, x->tv.block_size, (unsigned long long)x->tv.init_hash,
                    x->tv.pods_per_key);
    if (hd.pod_span > x->tv.max_pods) return fail(KVIDX_ERANGE, "snapshot holds pod ids up to %u, max_pods is %u", hd.pod_span - 1, x->tv.max_pods);
    if (hd.model_span > 65536) return fail(KVIDX_EINVAL, "malformed snapshot image: model_span %u", hd.model_span);
    if (x->tv.req_stamp && !rec) return fail(KVIDX_EINVAL, "an exact-LRU index needs an image with recency (taken from an exact-LRU index)");
    WriteCall w(x);
    if (int rc = w.begin(kDisarm)) return rc;
    w.share();
    int rc = refresh_counters(x);
    if (rc) return rc;
    if (x->h_cnt->req_full || x->h_cnt->eng_full)
        return fail(KVIDX_EINVAL, "restore needs an empty index: this one holds %llu request and %llu engine keys",
                    x->h_cnt->req_full, x->h_cnt->eng_full);
    // a growable handle is checked at the size its growth rule gives the image (as an empty handle: L = 0, I = max(R, E)),
    // which restore_impl allocates once every record has passed validation
    const uint64_t slots = x->tv.shard_bits ? x->tv.req_mask + 1 : grow_target(x, 0, std::max(R, E));
    if (!x->tv.shard_bits && (R * 10 > slots * 9 || E * 10 > slots * 9))   // the write path's limit: at most 90 % of a table's slots live
        return fail(KVIDX_ENOSPC, "table full: %llu request / %llu engine keys in %llu / %llu slots", (unsigned long long)R,
                    (unsigned long long)E, (unsigned long long)slots, (unsigned long long)slots);
    rc = restore_impl(x, w, static_cast<const uint8_t*>(buf) + kSnapHeaderBytes, hd, slots, restored_out);
    release_snap(x);
    return rc;
}
}  // namespace

extern "C" {

int kvidx_snapshot(kvidx_t* x, void* buf, uint64_t cap, uint64_t* size_out) {
    if (size_out) *size_out = 0;
    if (!x || !size_out) return fail(KVIDX_EINVAL, "bad arguments");
    // a sharded handle's keys live in several processes' tables: kvidx_shard_snapshot + kvidx_snapshot_merge is the collective export
    if (x->tv.shard_bits) return fail(KVIDX_EINVAL, "kvidx_snapshot is not supported on a sharded index (kvidx_shard_snapshot is its collective form)");
    return snapshot_call(x, buf, cap, size_out);
}

int kvidx_restore(kvidx_t* x, const void* buf, uint64_t len, uint64_t restored_out[2]) {
    if (restored_out) restored_out[0] = restored_out[1] = 0;
    if (!x || !buf) return fail(KVIDX_EINVAL, "bad arguments");
    if (x->tv.shard_bits) return fail(KVIDX_EINVAL, "kvidx_restore is not supported on a sharded index (kvidx_shard_restore is its collective form)");
    return restore_call(x, buf, len, restored_out);
}

int kvidx_shard_snapshot(kvidx_t* x, void* buf, uint64_t cap, uint64_t* size_out) {
    if (size_out) *size_out = 0;
    if (!x || !size_out) return fail(KVIDX_EINVAL, "bad arguments");
    return snapshot_call(x, buf, cap, size_out);
}

int kvidx_shard_restore(kvidx_t* x, const void* buf, uint64_t len, uint64_t restored_out[2]) {
    if (restored_out) restored_out[0] = restored_out[1] = 0;
    if (!x || !buf) return fail(KVIDX_EINVAL, "bad arguments");
    return restore_call(x, buf, len, restored_out);
}

int kvidx_snapshot_merge(const void* const* parts, const uint64_t* lens, uint32_t n_parts, void* out, uint64_t cap, uint64_t* size_out) {
    if (size_out) *size_out = 0;
    if (!size_out || (n_parts && (!parts || !lens))) return fail(KVIDX_EINVAL, "bad arguments");
    if (n_parts == 0) return fail(KVIDX_EINVAL, "no parts to merge");
    std::vector<SnapHeader> hd(n_parts);
    SnapHeader m{};
    for (uint32_t p = 0; p < n_parts; ++p) {
        if (!parts[p]) return fail(KVIDX_EINVAL, "part %u: NULL", p);
        if (int rc = check_image_header(parts[p], lens[p], &hd[p])) {
            const std::string why = g_err;
            return fail(rc, "part %u: %s", p, why.c_str());
        }
        const SnapHeader& h = hd[p];
        if (h.model_span > 65536) return fail(KVIDX_EINVAL, "part %u: malformed snapshot image: model_span %u", p, h.model_span);
        if (h.flags & kSnapFlagRecency)
            return fail(KVIDX_EINVAL, "part %u carries recency: parts come from sharded handles, which never track it", p);
        if (p && (h.block_size != m.block_size || h.init_hash != m.init_hash || h.pods_per_key != m.pods_per_key))
            return fail(KVIDX_EINVAL, "part %u is of another configuration: block_size %u, init_hash %#llx, pods_per_key %u (part 0: %u, %#llx, %u)",
                        p, h.block_size, (unsigned long long)h.init_hash, h.pods_per_key, m.block_size, (unsigned long long)m.init_hash, m.pods_per_key);
        if (!p) m = h;
        else { m.n_request += h.n_request; m.n_engine += h.n_engine; }
        m.pod_span = std::max(m.pod_span, h.pod_span);
        m.model_span = std::max(m.model_span, h.model_span);
    }
    // every record is checked before anything is written: order inside each part, no key in two parts
    if (int rc = merge_images(parts, hd, nullptr)) return rc;
    const uint64_t size = kSnapHeaderBytes + 32 * m.n_request + 24 * m.n_engine;
    *size_out = size;
    if (!out || cap < size) return fail(KVIDX_ENOSPC, "the merged image needs %llu bytes, the buffer has %llu", (unsigned long long)size,
                                        (unsigned long long)(out ? cap : 0));
    memcpy(out, &m, sizeof m);
    return merge_images(parts, hd, static_cast<uint8_t*>(out) + kSnapHeaderBytes);
}

int kvidx_shard_export(kvidx_t* x, void* out) {
    if (!x || !out) return fail(KVIDX_EINVAL, "bad arguments");
    WriteCall w(x);
    if (int rc = w.begin(0)) return rc;
    cudaIpcMemHandle_t h[3];
    CK(cudaIpcGetMemHandle(&h[0], x->tv.req));
    CK(cudaIpcGetMemHandle(&h[1], x->tv.eng));
    CK(cudaIpcGetMemHandle(&h[2], x->d_cnt));
    static_assert(sizeof(h) == KVIDX_SHARD_HANDLE_BYTES, "handle blob size");
    memcpy(out, h, sizeof h);
    return 0;
}

int kvidx_shard_import(kvidx_t* x, uint32_t rank, const void* handle) {
    if (!x || !handle) return fail(KVIDX_EINVAL, "bad arguments");
    if (rank >= (1u << x->tv.shard_bits)) return fail(KVIDX_ERANGE, "rank %u outside shard_count", rank);
    if (rank == x->tv.shard_rank) return 0;
    WriteCall w(x);
    w.exclusive();
    if (int rc = w.begin(0)) return rc;
    cudaIpcMemHandle_t h[3];
    memcpy(h, handle, sizeof h);
    void* p[3] = {nullptr, nullptr, nullptr};
    for (int i = 0; i < 3; ++i) CK(cudaIpcOpenMemHandle(&p[i], h[i], cudaIpcMemLazyEnablePeerAccess));
    x->tv.req_peer[rank] = static_cast<ReqSlot*>(p[0]); x->tv.eng_peer[rank] = static_cast<EngSlot*>(p[1]);
    x->tv.cnt_peer[rank] = static_cast<Counters*>(p[2]);
    return 0;
}

int kvidx_shard_attach(kvidx_t* x, uint32_t rank, kvidx_t* other) {
    if (!x || !other) return fail(KVIDX_EINVAL, "bad arguments");
    if (rank >= (1u << x->tv.shard_bits)) return fail(KVIDX_ERANGE, "rank %u outside shard_count", rank);
    if (rank == x->tv.shard_rank) return 0;
    if (other->tv.req_mask != x->tv.req_mask || other->tv.shard_bits != x->tv.shard_bits || other->tv.shard_rank != rank)
        return fail(KVIDX_EINVAL, "shard geometry mismatch");
    WriteCall w(x);
    w.exclusive();
    if (int rc = w.begin(0)) return rc;
    if (other->device != x->device) {
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, x->device, other->device));
        if (!can) return fail(KVIDX_ECUDA, "device %d cannot access device %d", x->device, other->device);
        cudaError_t e = cudaDeviceEnablePeerAccess(other->device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(KVIDX_ECUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e));
        cudaGetLastError();
    }
    x->tv.req_peer[rank] = other->tv.req; x->tv.eng_peer[rank] = other->tv.eng; x->tv.cnt_peer[rank] = other->d_cnt;
    return 0;
}

int kvidx_shard_compact(kvidx_t* x) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    WriteCall w(x);
    w.exclusive();
    if (int rc = w.begin(kDisarm)) return rc;
    return rebuild(x, x->tv.shard_bits != 0, x->tv.req_mask + 1);
}

// Counters of the device block read without the write lock, on no stream of the handle: a call never waits behind a write
// batch in flight (a metrics scrape), and sees the counts of the batches completed so far.
static int read_device_counters(kvidx* x, size_t off, uint64_t* out, int n) {
    CK(cudaSetDevice(x->device));
    CK(cudaMemcpy(out, reinterpret_cast<const uint8_t*>(x->d_cnt) + off, (size_t)n * 8, cudaMemcpyDeviceToHost));
    return 0;
}

int kvidx_get_evictions(kvidx_t* x, uint64_t out[2]) {
    if (!x || !out) return fail(KVIDX_EINVAL, "bad arguments");
    return read_device_counters(x, offsetof(Counters, cap_evicted), out, 2);
}

int kvidx_get_sweeps(kvidx_t* x, uint64_t out[2]) {
    if (!x || !out) return fail(KVIDX_EINVAL, "bad arguments");
    return read_device_counters(x, offsetof(Counters, sweeps), out, 2);
}

int kvidx_get_stats(kvidx_t* x, kvidx_stats_t* out) {
    if (!x || !out) return fail(KVIDX_EINVAL, "bad arguments");
    WriteCall w(x);
    if (int rc = w.begin(0)) return rc;
    if (int rc = refresh_counters(x)) return rc;
    out->request_keys = x->h_cnt->req_full; out->engine_keys = x->h_cnt->eng_full;
    out->request_tombs = x->h_cnt->req_tomb; out->engine_tombs = x->h_cnt->eng_tomb;
    out->request_slots = x->tv.req_mask + 1; out->engine_slots = x->tv.eng_mask + 1;
    out->rebuilds = x->rebuilds; out->kernel_launches = x->launches.load();
    out->rehashed_events = x->h_cnt->rehashed; out->coalesced_calls = x->queue ? submit_queue_coalesced(x->queue.get()) : 0;
    return 0;
}

// What each pod holds (kernels_inventory.cuh).  A read call: the read side's locks, stream and scratch.
//   d_inv: entries[P * 16] | keys[P] | sole[P] | sole_engine[P] | totals[4], all u64, zeroed by every call
int kvidx_pod_inventory(kvidx_t* x, uint32_t model, uint32_t flags, uint64_t* entries_out, uint64_t* keys_out, uint64_t* sole_out,
                        uint64_t* sole_engine_out, uint64_t totals_out[4]) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    if (!entries_out && !keys_out && !sole_out && !sole_engine_out && !totals_out) return fail(KVIDX_EINVAL, "every output is NULL");
    if (flags & ~KVIDX_INVENTORY_ENGINE) return fail(KVIDX_EINVAL, "unknown inventory flags 0x%x", flags);
    if (model != KVIDX_ANY_MODEL && model > 0xffffu) return fail(KVIDX_ERANGE, "model id %u > 65535", model);
    ReadCall c(x);
    if (int rc = c.begin(kShards | kAfterWrites)) return rc;
    const size_t P = x->tv.max_pods, n_ent = P * KVIDX_MAX_TIERS, words = n_ent + 3 * P + 4;
    CK(x->d_inv.need(words * 8));
    CK(x->h_inv.need(words * 8));
    unsigned long long* d = x->d_inv.as<unsigned long long>();
    InvArgs ia{model, d, d + n_ent, d + n_ent + P, d + n_ent + 2 * P, d + n_ent + 3 * P};
    CK(cudaMemsetAsync(d, 0, words * 8, x->stream));
    auto ctas = [&](uint64_t slots) { return (unsigned)std::min<uint64_t>((slots + kInvThreads - 1) / kInvThreads, (uint64_t)x->sm_count * 8); };
    inventory_req_kernel<<<ctas(x->tv.req_mask + 1), kInvThreads, inv_req_smem(x->tv.max_pods), x->stream>>>(x->tv, ia);
    if (flags & KVIDX_INVENTORY_ENGINE) inventory_eng_kernel<<<ctas(x->tv.eng_mask + 1), kInvThreads, P * 4, x->stream>>>(x->tv, ia);
    x->launches += (flags & KVIDX_INVENTORY_ENGINE) ? 2 : 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(x->h_inv.p, d, words * 8, cudaMemcpyDeviceToHost, x->stream));
    CK(cudaStreamSynchronize(x->stream));
    const uint64_t* h = x->h_inv.as<uint64_t>();
    if (entries_out) memcpy(entries_out, h, n_ent * 8);
    if (keys_out) memcpy(keys_out, h + n_ent, P * 8);
    if (sole_out) memcpy(sole_out, h + n_ent + P, P * 8);
    if (sole_engine_out) memcpy(sole_engine_out, h + n_ent + 2 * P, P * 8);
    if (totals_out) memcpy(totals_out, h + n_ent + 3 * P, 4 * 8);
    return 0;
}

}  // extern "C"

// ---- the device prefix store (kvidx_text_store_*, kernels_text.cuh) -----------------------------------------------------
namespace {

constexpr int64_t kTextLaneMax = 16384;       // batches below this many prompts hash with 4 lanes per prompt, larger ones with 1

int nomem(cudaError_t e, const char* what) {
    cudaGetLastError();
    return fail(e == cudaErrorMemoryAllocation ? KVIDX_ENOMEM : KVIDX_ECUDA, "prefix store: %s: %s", what, cudaGetErrorString(e));
}
#define TK(call, what) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return nomem(e_, what); } while (0)

unsigned text_grid(kvidx* x, int64_t threads) {
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>((threads + kTextThreads - 1) / kTextThreads, (int64_t)x->sm_count * 16));
}

// a fresh, empty table of `slots` slots
int text_table_alloc(TextStore* s, uint64_t slots, TextTable* t, void** mem, cudaStream_t st) {
    const size_t bytes = (size_t)slots * (8 + 8 + 8 + 8 + 4);
    TK(cudaMalloc(mem, bytes), "table");
    uint8_t* p = static_cast<uint8_t*>(*mem);
    t->key = reinterpret_cast<uint64_t*>(p);
    t->stamp = reinterpret_cast<unsigned long long*>(p + slots * 8);
    t->off = reinterpret_cast<int64_t*>(p + slots * 16);
    t->len = reinterpret_cast<int64_t*>(p + slots * 24);
    t->state = reinterpret_cast<uint32_t*>(p + slots * 32);
    t->mask = slots - 1;
    CK(cudaMemsetAsync(*mem, 0, bytes, st));
    return 0;
}

// Move the full slots whose stamp is >= keep_from into a fresh table of `slots` slots (growth: keep_from 0; eviction: the
// cut).  Records stay where they are in the arena.
int text_rebuild(kvidx* x, TextStore* s, uint64_t slots, unsigned long long keep_from, cudaStream_t st) {
    TextTable nt{}; void* mem = nullptr;
    if (int rc = text_table_alloc(s, slots, &nt, &mem, st)) return rc;
    text_rebuild_kernel<<<text_grid(x, (int64_t)s->t.mask + 1), kTextThreads, 0, st>>>(s->t, nt, keep_from);
    x->launches += 1;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    cudaFree(s->tab);
    s->tab = mem; s->t = nt;
    return 0;
}

// in-place inclusive sum of a[1 .. n] (a[0] = 0): CSR offsets from counts
int text_scan(kvidx* x, TextStore* s, int64_t* a, int64_t n, cudaStream_t st) {
    if (n <= 0) return 0;
    if (n >= (1ll << 31)) return fail(KVIDX_EINVAL, "prefix store: %lld elements in one call", (long long)n);
    size_t tb = 0;
    CK(cub::DeviceScan::InclusiveSum(nullptr, tb, a + 1, a + 1, (int)n, st));
    TK(s->d_cub.need(tb), "scan scratch");
    CK(cub::DeviceScan::InclusiveSum(s->d_cub.p, tb, a + 1, a + 1, (int)n, st));
    x->launches += 1;
    return 0;
}

// read n int64 values from the device (synchronises st)
int text_read(TextStore* s, const int64_t* const* src, int n, int64_t* out, cudaStream_t st) {
    CK(s->h_misc.need(64));
    int64_t* h = s->h_misc.as<int64_t>();
    for (int i = 0; i < n; ++i) CK(cudaMemcpyAsync(h + i, src[i], 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) out[i] = h[i];
    return 0;
}

// Block offsets of the call (d_blk: n + 1 int64, scanned) and their total.  tok_off (an add call): prompts without tokens
// have no blocks.
int text_blocks(kvidx* x, TextStore* s, const int64_t* text_off, const int64_t* tok_off, int64_t n, int64_t* nblk, cudaStream_t st) {
    TK(s->d_blk.need((size_t)(n + 1) * 8), "block offsets");
    int64_t* bo = s->d_blk.as<int64_t>();
    CK(cudaMemsetAsync(bo, 0, 8, st));
    text_block_counts_kernel<<<text_grid(x, n), kTextThreads, 0, st>>>(text_off, tok_off, n, s->B, bo);
    x->launches += 1;
    CK(cudaGetLastError());
    if (int rc = text_scan(x, s, bo, n, st)) return rc;
    const int64_t* p = bo + n;
    return text_read(s, &p, 1, nblk, st);
}

// Make room for `incoming` more tokens in the arena: compact the live records (into a larger arena when live + incoming
// would fill more than half of it).
int text_arena_room(kvidx* x, TextStore* s, int64_t incoming, cudaStream_t st) {
    if (s->arena_used + incoming <= s->arena_cap) return 0;
    const uint64_t slots = s->t.mask + 1;
    TK(s->d_scr.need((slots + 1) * 8 + 64), "compaction scratch");
    int64_t* newoff = s->d_scr.as<int64_t>();
    CK(cudaMemsetAsync(newoff, 0, 8, st));
    text_rec_len_kernel<<<text_grid(x, (int64_t)slots), kTextThreads, 0, st>>>(s->t, newoff);
    x->launches += 1;
    CK(cudaGetLastError());
    if (int rc = text_scan(x, s, newoff, (int64_t)slots, st)) return rc;
    int64_t live = 0;
    const int64_t* p = newoff + slots;
    if (int rc = text_read(s, &p, 1, &live, st)) return rc;
    const int64_t cap = std::max<int64_t>(s->arena_cap, 2 * (live + incoming));
    uint32_t* na = nullptr;
    TK(cudaMalloc((void**)&na, (size_t)std::max<int64_t>(cap, 1) * 4), "token arena");
    text_compact_kernel<<<text_grid(x, (int64_t)slots * 32), kTextThreads, 0, st>>>(s->t, newoff, s->arena, na);
    x->launches += 1;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    cudaFree(s->arena);
    s->arena = na; s->arena_cap = cap; s->arena_used = live;
    return 0;
}

// The device inputs of a store call: text (prompt i at text + text_off[i] - text_base) and its offsets.
struct TextIn { const uint8_t* text; const int64_t* off; int64_t base; int64_t n; };

template <class K> void text_launch_lanes(kvidx* x, int64_t n, K k) {
    if (n < kTextLaneMax) k(std::integral_constant<int, 4>{}, text_grid(x, n * 4));
    else k(std::integral_constant<int, 1>{}, text_grid(x, n));
}

// Find, pass one, for the call `in`: block offsets, hit slots, token counts (tok_off: n + 1, scanned), ratios; with
// min_ratio >= 0 also the Score() CSR counts (score_off, scanned) and tokenize flags.  totals = {tokens, score tokens}.
struct FindScratch { int64_t nblk = 0; uint32_t* hit = nullptr; int64_t* nhit = nullptr; int64_t* tok_off = nullptr; int64_t* score_off = nullptr;
                     double* ratio = nullptr; uint8_t* tokenize = nullptr; int64_t totals[2] = {0, 0}; };
int text_find_pass1(kvidx* x, TextStore* s, const TextIn& in, double min_ratio, FindScratch& f, cudaStream_t st) {
    const int64_t n = in.n;
    if (int rc = text_blocks(x, s, in.off, nullptr, n, &f.nblk, st)) return rc;
    TK(carve(s->d_scr, [&](Carver& c) {
        f.hit = c.take<uint32_t>(std::max<int64_t>(f.nblk, 1)); f.nhit = c.take<int64_t>(n); f.tok_off = c.take<int64_t>(n + 1);
        f.score_off = c.take<int64_t>(n + 1); f.ratio = c.take<double>(n); f.tokenize = c.take<uint8_t>(n);
    }), "find scratch");
    CK(cudaMemsetAsync(f.tok_off, 0, 8, st));
    CK(cudaMemsetAsync(f.score_off, 0, 8, st));
    const bool score = min_ratio >= 0;
    const int64_t* bo = s->d_blk.as<int64_t>();
    text_launch_lanes(x, n, [&](auto L, unsigned grid) {
        text_find_kernel<L.value><<<grid, kTextThreads, 0, st>>>(s->t, in.text, in.off, in.base, n, s->B, bo, f.hit, f.nhit, f.tok_off,
                                                                 f.ratio, min_ratio, score ? f.score_off : nullptr, f.tokenize);
    });
    x->launches += 1;
    CK(cudaGetLastError());
    if (int rc = text_scan(x, s, f.tok_off, n, st)) return rc;
    if (score) { if (int rc = text_scan(x, s, f.score_off, n, st)) return rc; }
    const int64_t* p[2] = {f.tok_off + n, f.score_off + n};
    return text_read(s, p, score ? 2 : 1, f.totals, st);
}

// Find, pass two: refresh every hit in call order and copy tokens to out (offsets out_off; gate: skip prompts flagged for
// the tokenizer; out NULL: refresh only).
int text_find_pass2(kvidx* x, TextStore* s, int64_t n, const FindScratch& f, const int64_t* out_off, const uint8_t* gate, uint32_t* out,
                    cudaStream_t st) {
    const unsigned long long base = s->clock + 1;
    s->clock += (unsigned long long)f.nblk + 1;
    text_gather_kernel<<<text_grid(x, n * 32), kTextThreads, 0, st>>>(s->t, s->arena, n, s->d_blk.as<int64_t>(), f.hit, f.nhit, base,
                                                                      out_off, gate, out);
    x->launches += 1;
    CK(cudaGetLastError());
    return 0;
}

// Steps two to four of an add, over keys already computed, then the cut down to cap_blocks keys: key k gets the
// tokens tok[src[k] .. src[k] + pos[k + 1] - pos[k]), touched in order k at fresh stamps, the last touch of a key winning.
// pos is scanned from pos0 (its first value, read back by the caller) and holds ntok = pos[nblk] - pos0 tokens in all.
// slot_of (nblk) and inserted (one counter) are the caller's scratch.  kvidx_text_store_add and _restore both insert here.
int text_insert(kvidx* x, TextStore* s, const uint64_t* key, int64_t nblk, const uint32_t* tok, const int64_t* src, const int64_t* pos,
                int64_t pos0, int64_t ntok, uint32_t* slot_of, unsigned long long* inserted, cudaStream_t st) {
    // room for every key of the call at load <= 1/2 before the cut
    const uint64_t want = pow2ceil((uint64_t)std::max<int64_t>(2 * (s->resident + nblk), 1024));
    if (want > s->t.mask + 1) { if (int rc = text_rebuild(x, s, want, 0, st)) return rc; }
    if (int rc = text_arena_room(x, s, ntok, st)) return rc;
    const int64_t arena_base = s->arena_used - pos0;
    const unsigned long long base = s->clock + 1;
    s->clock += (unsigned long long)nblk + 1;
    CK(cudaMemsetAsync(inserted, 0, 8, st));
    if (ntok > 0) text_add_copy_kernel<<<text_grid(x, nblk * 32), kTextThreads, 0, st>>>(tok, src, pos, nblk, arena_base, s->arena);
    text_add_touch_kernel<<<text_grid(x, nblk), kTextThreads, 0, st>>>(s->t, key, nblk, base, slot_of, inserted);
    text_add_commit_kernel<<<text_grid(x, nblk), kTextThreads, 0, st>>>(s->t, nblk, base, slot_of, pos, arena_base);
    x->launches += 3;
    CK(cudaGetLastError());
    s->arena_used += ntok;
    CK(cudaMemcpyAsync(s->h_misc.p, inserted, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    s->resident += (int64_t)*s->h_misc.as<unsigned long long>();
    if (s->resident <= s->cap_blocks) return 0;
    // the cut: keep the cap_blocks most recently touched keys (stamps are distinct: one sort finds the threshold)
    const int64_t R = s->resident;
    size_t tb = 0;
    CK(cub::DeviceRadixSort::SortKeys(nullptr, tb, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)R, 0, 64, st));
    unsigned long long *st0, *st1;
    TK(carve(s->d_scr, [&](Carver& c) { st0 = c.take<unsigned long long>(R); st1 = c.take<unsigned long long>(R); }), "eviction scratch");
    TK(s->d_cub.need(tb), "eviction sort scratch");
    CK(cudaMemsetAsync(inserted, 0, 8, st));
    text_stamps_kernel<<<text_grid(x, (int64_t)s->t.mask + 1), kTextThreads, 0, st>>>(s->t, st0, nullptr, inserted, nullptr);
    CK(cub::DeviceRadixSort::SortKeys(s->d_cub.p, tb, st0, st1, (int)R, 0, 64, st));
    x->launches += 5;
    const int64_t* tp = reinterpret_cast<const int64_t*>(st1 + (R - s->cap_blocks));
    int64_t thr = 0;
    if (int rc = text_read(s, &tp, 1, &thr, st)) return rc;
    // the kept keys go into a table sized for them (load <= 1/2), not for this call: one large add does not leave a large table
    const uint64_t keep_slots = pow2ceil((uint64_t)std::max<int64_t>(2 * s->cap_blocks, 1024));
    if (int rc = text_rebuild(x, s, std::min<uint64_t>(keep_slots, s->t.mask + 1), (unsigned long long)thr, st)) return rc;
    s->resident = s->cap_blocks;
    return 0;
}

// AddTokenization for every prompt of the call, in array order; then the cut down to cap_blocks keys.
int text_add(kvidx* x, TextStore* s, const TextIn& in, const uint32_t* tok, const uint64_t* span, const int64_t* tok_off, int64_t tok_base,
             cudaStream_t st) {
    const int64_t n = in.n;
    int64_t nblk = 0;
    if (int rc = text_blocks(x, s, in.off, tok_off, n, &nblk, st)) return rc;
    if (nblk == 0) return 0;
    uint64_t* key; int64_t *src, *pos; uint32_t* slot_of; unsigned long long* inserted;
    TK(carve(s->d_out, [&](Carver& c) {
        key = c.take<uint64_t>(nblk); src = c.take<int64_t>(nblk); pos = c.take<int64_t>(nblk + 1); slot_of = c.take<uint32_t>(nblk);
        inserted = c.take<unsigned long long>(1);
    }), "add scratch");
    const int64_t* bo = s->d_blk.as<int64_t>();
    text_launch_lanes(x, n, [&](auto L, unsigned grid) {
        text_hash_kernel<L.value><<<grid, kTextThreads, 0, st>>>(in.text, in.off, in.base, n, s->B, bo, key);
    });
    CK(cudaMemsetAsync(pos, 0, 8, st));
    text_add_ranges_kernel<<<text_grid(x, n), kTextThreads, 0, st>>>(tok_off, tok_base, span, n, s->B, bo, src, pos);
    x->launches += 2;
    CK(cudaGetLastError());
    if (int rc = text_scan(x, s, pos, nblk, st)) return rc;
    int64_t ntok = 0;
    const int64_t* pp = pos + nblk;
    if (int rc = text_read(s, &pp, 1, &ntok, st)) return rc;
    return text_insert(x, s, key, nblk, tok, src, pos, 0, ntok, slot_of, inserted, st);
}

// The store's image (kvidx_text_store_snapshot, format in include/kvidx.h): the full slots sorted by stamp, least recent
// first, each record's tokens behind the records in the same order.  Reads the store and refreshes nothing.
int text_snapshot(kvidx* x, TextStore* s, void* buf, uint64_t cap, uint64_t* size_out, cudaStream_t st) {
    const int64_t R = s->resident;
    if (R >= (1ll << 31)) return fail(KVIDX_EINVAL, "prefix store: %lld keys in one snapshot", (long long)R);
    size_t tb = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tb, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (uint32_t*)nullptr,
                                       (uint32_t*)nullptr, (int)R, 0, 64, st));
    unsigned long long *st0, *st1, *cnt; uint32_t *sl0, *sl1; int64_t* toff;
    TK(carve(s->d_scr, [&](Carver& c) {
        st0 = c.take<unsigned long long>(R); st1 = c.take<unsigned long long>(R); sl0 = c.take<uint32_t>(R); sl1 = c.take<uint32_t>(R);
        toff = c.take<int64_t>(R + 1); cnt = c.take<unsigned long long>(2);
    }), "snapshot scratch");
    // 1. the full slots as (stamp, slot) pairs, and the live token count, which sizes the image
    CK(cudaMemsetAsync(cnt, 0, 16, st));
    text_stamps_kernel<<<text_grid(x, (int64_t)s->t.mask + 1), kTextThreads, 0, st>>>(s->t, st0, sl0, cnt, cnt + 1);
    x->launches += 1;
    CK(cudaGetLastError());
    int64_t got[2];
    const int64_t* p[2] = {reinterpret_cast<const int64_t*>(cnt), reinterpret_cast<const int64_t*>(cnt + 1)};
    if (int rc = text_read(s, p, 2, got, st)) return rc;
    if (got[0] != R) return fail(KVIDX_ECUDA, "prefix store: %lld full slots, %lld keys resident", (long long)got[0], (long long)R);
    const uint64_t T = (uint64_t)got[1], body = 16 * (uint64_t)R + 4 * T;
    *size_out = 64 + body;
    if (!buf || cap < 64 + body)
        return fail(KVIDX_ENOSPC, "the prefix store image is %llu bytes, the buffer holds %llu", (unsigned long long)(64 + body),
                    (unsigned long long)(buf ? cap : 0));
    uint8_t* img = nullptr;
    if (R > 0) {
        TK(carve(s->d_out, [&](Carver& c) { img = c.take<uint8_t>(body); }), "snapshot image");
        TK(s->d_cub.need(tb), "snapshot sort scratch");
        // 2. recency order; 3. token offsets in that order; 4. the records and their tokens
        CK(cub::DeviceRadixSort::SortPairs(s->d_cub.p, tb, st0, st1, sl0, sl1, (int)R, 0, 64, st));
        CK(cudaMemsetAsync(toff, 0, 8, st));
        text_snap_len_kernel<<<text_grid(x, R), kTextThreads, 0, st>>>(s->t, sl1, R, toff);
        x->launches += 2;
        CK(cudaGetLastError());
        if (int rc = text_scan(x, s, toff, R, st)) return rc;
        text_snapshot_kernel<<<text_grid(x, R * 32), kTextThreads, 0, st>>>(s->t, s->arena, sl1, toff, R, reinterpret_cast<uint4*>(img),
                                                                          reinterpret_cast<uint32_t*>(img + 16 * R));
        x->launches += 1;
        CK(cudaGetLastError());
    }
    // 5. to the caller: the body through the stager, then the header
    if (int rc = s->stage.d2h(static_cast<uint8_t*>(buf) + 64, img, body, st)) return rc;
    uint8_t h[64] = {};
    const uint32_t ver = 1, bb = s->B;
    const uint64_t nr = (uint64_t)R;
    memcpy(h, "KVIDXTXT", 8); memcpy(h + 8, &ver, 4); memcpy(h + 16, &bb, 4); memcpy(h + 24, &nr, 8); memcpy(h + 32, &T, 8);
    memcpy(buf, h, 64);
    return 0;
}

// The header of a prefix store image, checked against a store of block_bytes B -> its record and token counts.
int text_image_head(const void* buf, uint64_t len, uint32_t B, uint64_t* R, uint64_t* T) {
    if (!buf || len < 64) return fail(KVIDX_EINVAL, "prefix store image: %llu bytes, shorter than its header", (unsigned long long)len);
    const uint8_t* p = static_cast<const uint8_t*>(buf);
    uint32_t ver, flags, bb, z;
    memcpy(&ver, p + 8, 4); memcpy(&flags, p + 12, 4); memcpy(&bb, p + 16, 4); memcpy(&z, p + 20, 4); memcpy(R, p + 24, 8); memcpy(T, p + 32, 8);
    if (memcmp(p, "KVIDXTXT", 8)) return fail(KVIDX_EINVAL, "prefix store image: bad magic");
    if (ver != 1 || flags != 0) return fail(KVIDX_EINVAL, "prefix store image: version %u flags %u (1 and 0 expected)", ver, flags);
    bool zero = z == 0;
    for (int i = 40; i < 64; ++i) zero = zero && p[i] == 0;
    if (!zero) return fail(KVIDX_EINVAL, "prefix store image: non-zero reserved header bytes");
    if (bb != B) return fail(KVIDX_EINVAL, "prefix store image: block_bytes %u, the store's is %u", bb, B);
    const uint64_t room = len - 64;
    if (*R > room / 16 || *T > room / 4 || 16 * *R + 4 * *T != room)
        return fail(KVIDX_EINVAL, "prefix store image: %llu bytes do not hold %llu records and %llu tokens", (unsigned long long)len,
                    (unsigned long long)*R, (unsigned long long)*T);
    return 0;
}

// Load the R records and T tokens of a checked image (img: the host bytes) into the empty store: check every record on
// the device, then insert the newest cap_blocks of them in record order through text_insert.
int text_restore(kvidx* x, TextStore* s, const uint8_t* img, uint64_t R64, uint64_t T, cudaStream_t st) {
    if (R64 == 0) return T ? fail(KVIDX_EINVAL, "prefix store image: no record holds its %llu tokens", (unsigned long long)T) : 0;
    if (R64 >= (1ull << 31)) return fail(KVIDX_EINVAL, "prefix store image: %llu records in one restore", (unsigned long long)R64);
    const int64_t R = (int64_t)R64;
    const uint64_t body = 16 * R64 + 4 * T;
    uint8_t* d_body; uint64_t *key, *sorted; int64_t* off; uint32_t* slot_of; unsigned long long* flags;
    TK(carve(s->d_in, [&](Carver& c) { d_body = c.take<uint8_t>(body); sorted = c.take<uint64_t>(R); }), "restore input");
    TK(carve(s->d_out, [&](Carver& c) {
        key = c.take<uint64_t>(R); off = c.take<int64_t>(R + 1); slot_of = c.take<uint32_t>(R); flags = c.take<unsigned long long>(2);
    }), "restore scratch");
    if (int rc = s->stage.h2d(d_body, img + 64, body, st)) return rc;
    // the records' keys and token counts, padding (flag 1) and duplicate keys (flag 2), the token offsets and their total
    CK(cudaMemsetAsync(off, 0, 8, st));
    CK(cudaMemsetAsync(flags, 0, 16, st));
    text_restore_records_kernel<<<text_grid(x, R), kTextThreads, 0, st>>>(reinterpret_cast<const uint4*>(d_body), R, key, off, flags);
    size_t tb = 0;
    unsigned long long* k0 = reinterpret_cast<unsigned long long*>(key);
    unsigned long long* k1 = reinterpret_cast<unsigned long long*>(sorted);
    CK(cub::DeviceRadixSort::SortKeys(nullptr, tb, k0, k1, (int)R, 0, 64, st));
    TK(s->d_cub.need(tb), "restore sort scratch");
    CK(cub::DeviceRadixSort::SortKeys(s->d_cub.p, tb, k0, k1, (int)R, 0, 64, st));
    text_restore_dups_kernel<<<text_grid(x, R), kTextThreads, 0, st>>>(sorted, R, flags);
    x->launches += 3;
    CK(cudaGetLastError());
    if (int rc = text_scan(x, s, off, R, st)) return rc;
    const int64_t first = std::max<int64_t>(R - s->cap_blocks, 0);         // a larger image keeps its newest cap_blocks records
    int64_t got[3];
    const int64_t* p[3] = {off + R, off + first, reinterpret_cast<const int64_t*>(flags)};
    if (int rc = text_read(s, p, 3, got, st)) return rc;
    if (got[2] & 1) return fail(KVIDX_EINVAL, "prefix store image: non-zero record padding");
    if (got[2] & 2) return fail(KVIDX_EINVAL, "prefix store image: a key appears twice");
    if ((uint64_t)got[0] != T) return fail(KVIDX_EINVAL, "prefix store image: records hold %lld tokens, the header says %llu", (long long)got[0],
                                           (unsigned long long)T);
    return text_insert(x, s, key + first, R - first, reinterpret_cast<const uint32_t*>(d_body + 16 * R), off + first, off + first, got[1],
                       got[0] - got[1], slot_of, flags + 1, st);
}

int text_check(kvidx* x, int64_t n, const void* text, const int64_t* text_off) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    if (n < 0 || (n > 0 && !text_off)) return fail(KVIDX_EINVAL, "bad arguments");
    if (!x->text) return fail(KVIDX_EINVAL, "prefix store not initialised (kvidx_text_store_init)");
    if (n == 0) return 0;
    if (int rc = check_csr(text_off, n, "text_off")) return rc;
    if (text_off[n] > text_off[0] && !text) return fail(KVIDX_EINVAL, "NULL text");
    return 0;
}

// Upload a host call's text and offsets to d_in, carved with the caller's own sections after them (more(Carver&)).
// -> the device view.
template <class More>
int text_upload(TextStore* s, const uint8_t* text, const int64_t* text_off, int64_t n, TextIn* out, cudaStream_t st, More&& more) {
    const int64_t tb = text_off[0], nb = text_off[n] - tb;
    uint8_t* d_text; int64_t* d_off;
    TK(carve(s->d_in, [&](Carver& c) { d_text = c.take<uint8_t>(nb); d_off = c.take<int64_t>(n + 1); more(c); }), "input buffer");
    if (int rc = s->stage.h2d(d_text, text + tb, (size_t)nb, st)) return rc;
    if (int rc = s->stage.h2d(d_off, text_off, (size_t)(n + 1) * 8, st)) return rc;
    *out = TextIn{d_text, d_off, tb, n};
    return 0;
}

// A store call: the store's lock, the device, and the order after the previous store call on stream st.
struct TextCall {
    std::unique_lock<std::mutex> lk;
    TextStore* s; cudaStream_t st;
    TextCall(kvidx* x, cudaStream_t stream) : lk(x->mu_text), s(x->text.get()), st(stream) {}
    int begin(kvidx* x) { CK(cudaSetDevice(x->device)); CK(cudaStreamWaitEvent(st, s->ev_last, 0)); return 0; }
    // after an error: let nothing of this call run on past the return (the caller's buffers, the store's scratch)
    int end(int rc) {
        ReadCall::end(rc, {st});
        cudaEventRecord(s->ev_last, st);
        return rc;
    }
};

// Score() from text: find with the min_ratio gate, then the Score() dispatch on the contained tokens of the passing prompts.
// `a` carries the model, filter and the result rows (device pointers); tokenize / ratio: device outputs (may be NULL).
int score_text_run(kvidx* x, TextStore* s, const TextIn& in, double min_ratio, ScoreArgs a, uint8_t* tokenize, double* ratio, cudaStream_t st) {
    FindScratch f;
    if (int rc = text_find_pass1(x, s, in, min_ratio, f, st)) return rc;
    TK(s->d_tok.need((size_t)std::max<int64_t>(f.totals[1], 1) * 4 + 64), "token buffer");
    if (int rc = text_find_pass2(x, s, in.n, f, f.score_off, f.tokenize, s->d_tok.as<uint32_t>(), st)) return rc;
    if (tokenize) CK(cudaMemcpyAsync(tokenize, f.tokenize, (size_t)in.n, cudaMemcpyDeviceToDevice, st));
    if (ratio) CK(cudaMemcpyAsync(ratio, f.ratio, (size_t)in.n * 8, cudaMemcpyDeviceToDevice, st));
    a.tok_off = f.score_off; a.tok_base = 0; a.n_prompts = in.n;
    ReadCall c(x);                                    // lock order: mu_text (the caller's TextCall), then the read side's
    if (int rc = c.begin(kAfterWrites, st)) return rc;
    return launch_score(x, ScoreIn{s->d_tok.p, false}, a, st);
}

int score_text_host(kvidx* x, const uint8_t* text, const int64_t* text_off, int64_t n, const uint32_t* model, uint32_t model0,
                    const uint64_t* filter, double min_ratio, const ScoreArgs& h, uint8_t* tokenize_out, double* ratio_out) {
    if (int rc = text_check(x, n, text, text_off)) return rc;
    if (n == 0) return 0;
    if (!(min_ratio >= 0)) return fail(KVIDX_EINVAL, "min_ratio must be >= 0");
    TextCall c(x, x->stream);
    if (int rc = c.begin(x)) return rc;
    TextStore* s = c.s;
    const uint32_t FW = x->tv.filter_words;
    const RowLayout rows{x->tv.max_pods, h.sp_cnt != nullptr};
    // on the device after the text: the model ids and filter rows (when the call has them), the rows, ratios and flags
    ScoreArgs a = dense_args(nullptr, n, nullptr, model0, nullptr, nullptr, nullptr);
    uint32_t* d_model; uint64_t* d_filter; double* d_ratio; uint8_t* d_tokz;
    TextIn in{};
    int rc = text_upload(s, text, text_off, n, &in, c.st, [&](Carver& cv) {
        d_model = cv.take<uint32_t>(model ? n : 0); d_filter = cv.take<uint64_t>(filter ? n * FW : 0);
        rows.carve(cv.take<uint8_t>(n * rows.row()), n, a);
        d_ratio = cv.take<double>(n); d_tokz = cv.take<uint8_t>(n);
    });
    if (!rc && model) { a.model = d_model; rc = s->stage.h2d(d_model, model, (size_t)n * 4, c.st); }
    if (!rc && filter) { a.filter = d_filter; rc = s->stage.h2d(d_filter, filter, (size_t)n * FW * 8, c.st); }
    if (rc) return c.end(rc);
    rc = score_text_run(x, s, in, min_ratio, a, d_tokz, d_ratio, c.st);
    auto back = [&](void* dst, const void* src, size_t b) { return dst && !rc ? (rc = s->stage.d2h(dst, src, b, c.st)) : rc; };
    rows.each(n, [&](auto m, size_t b) { back(h.*m, a.*m, b); });
    back(tokenize_out, d_tokz, (size_t)n);
    back(ratio_out, d_ratio, (size_t)n * 8);
    if (!rc) { CK(cudaStreamSynchronize(c.st)); }
    return c.end(rc);
}

int score_text_dev(kvidx* x, const uint8_t* d_text, const int64_t* d_text_off, int64_t n, double min_ratio, const ScoreArgs& a,
                   uint8_t* d_tokenize, double* d_ratio) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    if (n < 0 || (n > 0 && !d_text_off)) return fail(KVIDX_EINVAL, "bad arguments");
    if (!x->text) return fail(KVIDX_EINVAL, "prefix store not initialised (kvidx_text_store_init)");
    if (n == 0) return 0;
    if (!(min_ratio >= 0)) return fail(KVIDX_EINVAL, "min_ratio must be >= 0");
    TextCall c(x, x->stream);
    if (int rc = c.begin(x)) return rc;
    return c.end(score_text_run(x, c.s, TextIn{d_text, d_text_off, 0, n}, min_ratio, a, d_tokenize, d_ratio, c.st));
}

}  // namespace

extern "C" {

int kvidx_text_store_init(kvidx_t* x, int64_t cache_blocks, int32_t block_bytes) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    if (cache_blocks <= 0) return fail(KVIDX_EINVAL, "failed to initialize in-memory index: must provide a positive size");   // lru.New
    if (block_bytes <= 0) return fail(KVIDX_EINVAL, "block size must be positive");
    std::lock_guard<std::mutex> g(x->mu_text);
    if (x->text) return fail(KVIDX_EINVAL, "prefix store already initialised on this handle");
    CK(cudaSetDevice(x->device));
    auto s = std::make_unique<TextStore>();         // a store that fails to initialise is freed on the way out
    s->cap_blocks = cache_blocks; s->B = (uint32_t)block_bytes;
    if (cudaStreamCreateWithFlags(&s->stream.h, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&s->ev_last.h, cudaEventDisableTiming) != cudaSuccess ||
        s->stage.init() != cudaSuccess)
        return fail(KVIDX_ECUDA, "prefix store: stream / event creation failed");
    if (int rc = text_table_alloc(s.get(), 1024, &s->t, &s->tab, s->stream)) return rc;
    s->arena_cap = 1 << 16;
    if (cudaError_t e = cudaMalloc((void**)&s->arena, (size_t)s->arena_cap * 4)) return nomem(e, "token arena");
    if (s->h_misc.need(64) != cudaSuccess) return fail(KVIDX_ENOMEM, "prefix store: pinned scratch");
    if (cudaEventRecord(s->ev_last, s->stream) != cudaSuccess || cudaStreamSynchronize(s->stream) != cudaSuccess)
        return fail(KVIDX_ECUDA, "prefix store: initialisation failed");
    x->text = std::move(s);
    return 0;
}

int kvidx_text_store_len(kvidx_t* x, int64_t* blocks_out) {
    if (!x || !blocks_out) return fail(KVIDX_EINVAL, "bad arguments");
    std::lock_guard<std::mutex> g(x->mu_text);
    if (!x->text) return fail(KVIDX_EINVAL, "prefix store not initialised (kvidx_text_store_init)");
    *blocks_out = x->text->resident;
    return 0;
}

int kvidx_text_store_snapshot(kvidx_t* x, void* buf, uint64_t cap, uint64_t* size_out) {
    if (!x || !size_out) return fail(KVIDX_EINVAL, "bad arguments");
    TextCall c(x, nullptr);
    if (!c.s) return fail(KVIDX_EINVAL, "prefix store not initialised (kvidx_text_store_init)");
    c.st = c.s->stream;
    if (int rc = c.begin(x)) return rc;              // after the last store call, a Score() from text on the handle's stream too
    return c.end(text_snapshot(x, c.s, buf, cap, size_out, c.st));
}

int kvidx_text_store_restore(kvidx_t* x, const void* buf, uint64_t len, int64_t* blocks_out) {
    if (!x) return fail(KVIDX_EINVAL, "NULL handle");
    TextCall c(x, nullptr);
    if (!c.s) return fail(KVIDX_EINVAL, "prefix store not initialised (kvidx_text_store_init)");
    c.st = c.s->stream;
    uint64_t R = 0, T = 0;
    if (int rc = text_image_head(buf, len, c.s->B, &R, &T)) return rc;
    if (c.s->resident != 0) return fail(KVIDX_EINVAL, "prefix store restore needs an empty store (%lld keys resident)", (long long)c.s->resident);
    if (int rc = c.begin(x)) return rc;
    int rc = text_restore(x, c.s, static_cast<const uint8_t*>(buf), R, T, c.st);
    if (!rc && blocks_out) *blocks_out = c.s->resident;
    return c.end(rc);
}

int kvidx_text_store_add(kvidx_t* x, const uint8_t* text, const int64_t* text_off, int64_t n, const uint32_t* tok, const uint64_t* tok_span,
                         const int64_t* tok_off) {
    if (int rc = text_check(x, n, text, text_off)) return rc;
    if (n == 0) return 0;
    if (!tok_off) return fail(KVIDX_EINVAL, "NULL tok_off");
    if (int rc = check_csr(tok_off, n)) return rc;
    const int64_t tb = tok_off[0], nt = tok_off[n] - tb;
    if (nt > 0 && (!tok || !tok_span)) return fail(KVIDX_EINVAL, "NULL tokens or spans");
    TextCall c(x, nullptr);
    c.st = c.s->stream;
    if (int rc = c.begin(x)) return rc;
    TextStore* s = c.s;
    // the tokens and their spans after the text (empty when nt is 0: then no prompt has a block, and text_add reads neither)
    int64_t* d_toff; uint32_t* d_tok; uint64_t* d_span;
    TextIn in{};
    int rc = text_upload(s, text, text_off, n, &in, c.st, [&](Carver& cv) {
        d_toff = cv.take<int64_t>(n + 1); d_tok = cv.take<uint32_t>(nt); d_span = cv.take<uint64_t>(nt * 2);
    });
    if (!rc) rc = s->stage.h2d(d_toff, tok_off, (size_t)(n + 1) * 8, c.st);
    if (!rc && nt > 0) rc = s->stage.h2d(d_tok, tok + tb, (size_t)nt * 4, c.st);
    if (!rc && nt > 0) rc = s->stage.h2d(d_span, tok_span + 2 * tb, (size_t)nt * 16, c.st);
    if (!rc) rc = text_add(x, s, in, d_tok, d_span, d_toff, tb, c.st);
    if (!rc) { CK(cudaStreamSynchronize(c.st)); }
    return c.end(rc);
}

int kvidx_text_store_find(kvidx_t* x, const uint8_t* text, const int64_t* text_off, int64_t n, uint32_t* tok_out, int64_t tok_cap,
                          int64_t* tok_off_out, double* ratio_out) {
    if (int rc = text_check(x, n, text, text_off)) return rc;
    if (n == 0) return 0;
    if (!tok_off_out) return fail(KVIDX_EINVAL, "NULL tok_off_out");
    TextCall c(x, nullptr);
    c.st = c.s->stream;
    if (int rc = c.begin(x)) return rc;
    TextStore* s = c.s;
    TextIn in{};
    int rc = text_upload(s, text, text_off, n, &in, c.st, [](Carver&) {});
    FindScratch f;
    if (!rc) rc = text_find_pass1(x, s, in, -1.0, f, c.st);
    if (!rc) rc = s->stage.d2h(tok_off_out, f.tok_off, (size_t)(n + 1) * 8, c.st);
    if (!rc && ratio_out) rc = s->stage.d2h(ratio_out, f.ratio, (size_t)n * 8, c.st);
    if (rc) return c.end(rc);
    if (f.totals[0] > 0 && (!tok_out || tok_cap < f.totals[0]))       // nothing refreshed: the find has not happened
        return c.end(fail(KVIDX_ENOSPC, "tok_out holds %lld tokens, the find returns %lld", (long long)(tok_out ? tok_cap : 0), (long long)f.totals[0]));
    TK(s->d_tok.need((size_t)std::max<int64_t>(f.totals[0], 1) * 4 + 64), "token buffer");
    rc = text_find_pass2(x, s, n, f, f.tok_off, nullptr, s->d_tok.as<uint32_t>(), c.st);
    if (!rc && f.totals[0] > 0) rc = s->stage.d2h(tok_out, s->d_tok.p, (size_t)f.totals[0] * 4, c.st);
    if (!rc) { CK(cudaStreamSynchronize(c.st)); }
    return c.end(rc);
}

int kvidx_text_hash_keys(kvidx_t* x, const uint8_t* text, const int64_t* text_off, int64_t n, int32_t block_bytes, uint64_t* keys_out,
                         int64_t* key_off_out) {
    if (!x || n < 0 || (n > 0 && (!text_off || !key_off_out))) return fail(KVIDX_EINVAL, "bad arguments");
    if (block_bytes <= 0) return fail(KVIDX_EINVAL, "block size must be positive");
    if (n == 0) return 0;
    if (int rc = check_csr(text_off, n, "text_off")) return rc;
    if (text_off[n] > text_off[0] && !text) return fail(KVIDX_EINVAL, "NULL text");
    int64_t nk = 0;
    for (int64_t i = 0; i < n; ++i) { key_off_out[i] = nk; nk += (text_off[i + 1] - text_off[i]) / block_bytes; }
    key_off_out[n] = nk;
    if (nk == 0) return 0;
    if (!keys_out) return fail(KVIDX_EINVAL, "NULL keys_out");
    TextCall c(x, nullptr);
    if (!c.s) return fail(KVIDX_EINVAL, "prefix store not initialised (kvidx_text_store_init)");
    c.st = c.s->stream;
    if (int rc = c.begin(x)) return rc;
    TextStore* s = c.s;
    int64_t* d_koff; uint64_t* d_keys;
    TextIn in{};
    int rc = text_upload(s, text, text_off, n, &in, c.st, [&](Carver& cv) { d_koff = cv.take<int64_t>(n + 1); d_keys = cv.take<uint64_t>(nk); });
    if (rc) return c.end(rc);
    CK(cudaMemcpyAsync(d_koff, key_off_out, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, c.st));
    const uint32_t B = (uint32_t)block_bytes;
    text_launch_lanes(x, n, [&](auto L, unsigned grid) {
        text_hash_kernel<L.value><<<grid, kTextThreads, 0, c.st>>>(in.text, in.off, in.base, n, B, d_koff, d_keys);
    });
    x->launches += 1;
    rc = cudaGetLastError() == cudaSuccess ? 0 : fail(KVIDX_ECUDA, "text hash launch failed");
    if (!rc) rc = s->stage.d2h(keys_out, d_keys, (size_t)nk * 8, c.st);
    if (!rc) { CK(cudaStreamSynchronize(c.st)); }
    return c.end(rc);
}

int kvidx_score_text(kvidx_t* x, const uint8_t* text, const int64_t* text_off, int64_t n, const uint32_t* model, uint32_t model0,
                     const uint64_t* filter, double min_ratio, double* scores_out, uint8_t* has_keys_out, uint8_t* tokenize_out, double* ratio_out) {
    if (!x || !scores_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_text_host(x, text, text_off, n, model, model0, filter, min_ratio,
                           dense_args(nullptr, n, nullptr, model0, nullptr, scores_out, has_keys_out),
                           tokenize_out, ratio_out);
}

int kvidx_score_text_sparse(kvidx_t* x, const uint8_t* text, const int64_t* text_off, int64_t n, const uint32_t* model, uint32_t model0,
                            const uint64_t* filter, double min_ratio, uint16_t* pods_out, double* scores_out, uint8_t* cnt_out,
                            uint8_t* has_keys_out, uint8_t* tokenize_out, double* ratio_out) {
    if (!x || !pods_out || !scores_out || !cnt_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_text_host(x, text, text_off, n, model, model0, filter, min_ratio,
                           sparse_args(nullptr, n, nullptr, model0, nullptr, pods_out, scores_out, cnt_out, has_keys_out),
                           tokenize_out, ratio_out);
}

int kvidx_score_text_dev(kvidx_t* x, const uint8_t* d_text, const int64_t* d_text_off, int64_t n, const uint32_t* d_model, uint32_t model0,
                         const uint64_t* d_filter, double min_ratio, double* d_scores_out, uint8_t* d_has_keys_out, uint8_t* d_tokenize_out,
                         double* d_ratio_out) {
    if (!x || !d_scores_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_text_dev(x, d_text, d_text_off, n, min_ratio,
                          dense_args(nullptr, n, d_model, model0, d_filter, d_scores_out, d_has_keys_out),
                          d_tokenize_out, d_ratio_out);
}

int kvidx_score_text_sparse_dev(kvidx_t* x, const uint8_t* d_text, const int64_t* d_text_off, int64_t n, const uint32_t* d_model, uint32_t model0,
                                const uint64_t* d_filter, double min_ratio, uint16_t* d_pods_out, double* d_scores_out, uint8_t* d_cnt_out,
                                uint8_t* d_has_keys_out, uint8_t* d_tokenize_out, double* d_ratio_out) {
    if (!x || !d_pods_out || !d_scores_out || !d_cnt_out) return fail(KVIDX_EINVAL, "bad arguments");
    return score_text_dev(x, d_text, d_text_off, n, min_ratio,
                          sparse_args(nullptr, n, d_model, model0, d_filter, d_pods_out, d_scores_out, d_cnt_out, d_has_keys_out),
                          d_tokenize_out, d_ratio_out);
}

}  // extern "C"
