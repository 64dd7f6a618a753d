// kvhost.cpp -- host mirror of the reference's Go layer for the hot path (include/kvidx_host.h).
// String interning, FNV-32a sharded per-pod queues (kvevents.Pool) and the msgpack decoding of KVEvents, over the
// id-level C ABI of libkvidx.  No CUDA in this file; the decoder runs without a GPU.
#include <algorithm>
#include <cctype>
#include <cstring>
#include <chrono>
#include <deque>
#include <list>
#include <mutex>
#include <set>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/kvidx_host.h"

namespace {

thread_local std::string g_herr;
int hfail(int code, const std::string& m) { g_herr = m; return code; }

// name <-> id.  A released id is handed to the next new name, lowest first.  Names are kept for the life of the handle
// (node-based set: element addresses are stable), so a name pointer returned to a caller never dangles, even after its id
// has been reused.
struct Interner {
    std::unordered_map<std::string, uint32_t> ids;
    std::unordered_set<std::string> store;
    std::vector<const std::string*> names;           // id -> name; nullptr: released
    std::set<uint32_t> free_ids;
    int id(const std::string& s, uint32_t limit) {
        auto it = ids.find(s);
        if (it != ids.end()) return (int)it->second;
        uint32_t i;
        if (!free_ids.empty() && *free_ids.begin() < limit) { i = *free_ids.begin(); free_ids.erase(free_ids.begin()); }
        else if (names.size() < limit) { i = (uint32_t)names.size(); names.push_back(nullptr); }
        else return -1;
        names[i] = &*store.insert(s).first;
        ids.emplace(s, i);
        return (int)i;
    }
    int find(const std::string& s) const { auto it = ids.find(s); return it == ids.end() ? -1 : (int)it->second; }
    const char* name(uint32_t i) const { return names[i]->c_str(); }
    void release(uint32_t i) { ids.erase(*names[i]); names[i] = nullptr; free_ids.insert(i); }
};

// ---- minimal msgpack reader (vmihailenco/msgpack v5 type rules are applied by the callers) -------------------
enum Kind { K_NIL, K_BOOL, K_INT, K_FLOAT, K_STR, K_BIN, K_ARRAY, K_MAP, K_EXT, K_BAD };
struct Val { Kind k = K_BAD; uint8_t code = 0; uint64_t u = 0; double f = 0; const uint8_t* s = nullptr; size_t n = 0; };
struct Cur { const uint8_t* p; const uint8_t* e; };

bool need(Cur& c, size_t n) { return (size_t)(c.e - c.p) >= n; }
uint64_t be(const uint8_t* p, int n) { uint64_t v = 0; for (int i = 0; i < n; ++i) v = (v << 8) | p[i]; return v; }

// Reads one element head; scalars, strings and bins are consumed completely, containers leave the cursor at their
// first child (n = element count; maps count pairs).
bool head(Cur& c, Val& v) {
    if (!need(c, 1)) return false;
    const uint8_t b = *c.p++;
    v.code = b; v.u = 0; v.n = 0; v.s = nullptr;
    auto rd = [&](int n, uint64_t& out) { if (!need(c, n)) return false; out = be(c.p, n); c.p += n; return true; };
    auto blob = [&](size_t n, Kind k) { if (!need(c, n)) return false; v.k = k; v.s = c.p; v.n = n; c.p += n; return true; };
    uint64_t t = 0;
    if (b <= 0x7f) { v.k = K_INT; v.u = b; return true; }
    if (b >= 0xe0) { v.k = K_INT; v.u = (uint64_t)(int64_t)(int8_t)b; return true; }
    if (b >= 0xa0 && b <= 0xbf) return blob(b & 0x1f, K_STR);
    if (b >= 0x90 && b <= 0x9f) { v.k = K_ARRAY; v.n = b & 0x0f; return true; }
    if (b >= 0x80 && b <= 0x8f) { v.k = K_MAP; v.n = b & 0x0f; return true; }
    switch (b) {
        case 0xc0: v.k = K_NIL; return true;
        case 0xc2: case 0xc3: v.k = K_BOOL; v.u = b & 1; return true;
        case 0xc4: return rd(1, t) && blob(t, K_BIN);
        case 0xc5: return rd(2, t) && blob(t, K_BIN);
        case 0xc6: return rd(4, t) && blob(t, K_BIN);
        case 0xc7: return rd(1, t) && need(c, 1) && (c.p++, blob(t, K_EXT));
        case 0xc8: return rd(2, t) && need(c, 1) && (c.p++, blob(t, K_EXT));
        case 0xc9: return rd(4, t) && need(c, 1) && (c.p++, blob(t, K_EXT));
        case 0xca: { if (!rd(4, t)) return false; uint32_t w = (uint32_t)t; float f; memcpy(&f, &w, 4); v.k = K_FLOAT; v.f = f; return true; }
        case 0xcb: { if (!rd(8, t)) return false; double d; memcpy(&d, &t, 8); v.k = K_FLOAT; v.f = d; return true; }
        case 0xcc: v.k = K_INT; return rd(1, v.u);
        case 0xcd: v.k = K_INT; return rd(2, v.u);
        case 0xce: v.k = K_INT; return rd(4, v.u);
        case 0xcf: v.k = K_INT; return rd(8, v.u);
        case 0xd0: v.k = K_INT; if (!rd(1, t)) return false; v.u = (uint64_t)(int64_t)(int8_t)t; return true;
        case 0xd1: v.k = K_INT; if (!rd(2, t)) return false; v.u = (uint64_t)(int64_t)(int16_t)t; return true;
        case 0xd2: v.k = K_INT; if (!rd(4, t)) return false; v.u = (uint64_t)(int64_t)(int32_t)t; return true;
        case 0xd3: v.k = K_INT; return rd(8, v.u);
        case 0xd4: return need(c, 1) && (c.p++, blob(1, K_EXT));
        case 0xd5: return need(c, 1) && (c.p++, blob(2, K_EXT));
        case 0xd6: return need(c, 1) && (c.p++, blob(4, K_EXT));
        case 0xd7: return need(c, 1) && (c.p++, blob(8, K_EXT));
        case 0xd8: return need(c, 1) && (c.p++, blob(16, K_EXT));
        case 0xd9: return rd(1, t) && blob(t, K_STR);
        case 0xda: return rd(2, t) && blob(t, K_STR);
        case 0xdb: return rd(4, t) && blob(t, K_STR);
        case 0xdc: v.k = K_ARRAY; if (!rd(2, t)) return false; v.n = t; return true;
        case 0xdd: v.k = K_ARRAY; if (!rd(4, t)) return false; v.n = t; return true;
        case 0xde: v.k = K_MAP; if (!rd(2, t)) return false; v.n = t; return true;
        case 0xdf: v.k = K_MAP; if (!rd(4, t)) return false; v.n = t; return true;
        default: v.k = K_BAD; return false;     // 0xc1: never used
    }
}
bool skip(Cur& c, int depth = 0) {
    Val v;
    if (depth > 64 || !head(c, v)) return false;
    if (v.k == K_ARRAY) { for (size_t i = 0; i < v.n; ++i) if (!skip(c, depth + 1)) return false; }
    else if (v.k == K_MAP) { for (size_t i = 0; i < 2 * v.n; ++i) if (!skip(c, depth + 1)) return false; }
    return true;
}

// getHashAsUint64 (kvevents/pool.go:343-367) on a value decoded the way msgpack's DecodeInterface types it:
// only a uint64-coded (0xcf) or int64-coded (0xd3) integer or a byte slice (bin) is accepted.
bool hash_of(Cur& c, uint64_t* out, bool* is_nil) {
    const uint8_t* start = c.p;
    Val v;
    if (is_nil) *is_nil = false;
    Cur probe = c;
    if (!head(probe, v)) { c.p = c.e; return false; }
    if (v.k == K_ARRAY || v.k == K_MAP) { c.p = start; if (!skip(c)) c.p = c.e; return false; }
    c = probe;
    if (v.k == K_NIL) { if (is_nil) *is_nil = true; return false; }
    if (v.k == K_INT && (v.code == 0xcf || v.code == 0xd3)) { *out = v.u; return true; }
    if (v.k == K_BIN) {
        if (v.n == 0) return false;
        if (v.n >= 8) { *out = be(v.s + v.n - 8, 8); return true; }
        *out = be(v.s, (int)v.n);
        return true;
    }
    return false;
}

struct Msg { uint32_t pod, model; std::string payload; };

}  // namespace

struct kvhost {
    kvidx_t* ix = nullptr;
    kvhost_config_t cfg{};
    Interner models, pods, tiers;
    std::mutex mu;
    // Pod-id lifetime (kvhost_remove_pod frees ids).  read_mu: held shared by the read calls from their device call through
    // the id -> name mapping, exclusively while an id is freed, so that a reused id never puts a new pod's name on an old
    // pod's entries.  write_mu: held shared by the calls that intern a pod and then write its entries (pool_process from
    // the drain through the apply, index_add / index_evict), exclusively by remove_pod, so that no entry of a pod can be
    // written after its removal with the id it had.  Order: write_mu, read_mu, mu.
    std::shared_mutex read_mu, write_mu;
    std::vector<std::deque<Msg>> queues;
    uint32_t filter_words = 4;
    uint32_t pod_cap = 256;                          // == index.max_pods: ids of pods that own entries
    uint32_t cfg_tiers = 0;                          // tier ids interned from the configuration at create
    kvhost_metrics_t met{};              // guarded by mu
};

namespace {

std::string lower(std::string s) { for (auto& ch : s) ch = (char)tolower((unsigned char)ch); return s; }

// one event slice [p, e): a tagged union array ["BlockStored", ...]
void decode_event(kvhost* h, uint32_t pod, uint32_t model, const uint8_t* p, const uint8_t* e, std::vector<kvidx_event_t>& evs,
                  std::vector<uint64_t>& hashes, std::vector<uint32_t>& toks) {
    Cur c{p, e};
    Val v;
    if (!head(c, v)) return;
    if (v.k != K_ARRAY || v.n < 1) return;                               // not an array / no tag element: skipped
    size_t rest = v.n - 1;
    Val tag;
    if (!head(c, tag)) return;
    if (tag.k != K_STR && tag.k != K_BIN) return;                         // tag must decode as string
    const std::string t((const char*)tag.s, tag.n);
    auto medium_tier = [&](Cur& cc, bool present, int* tier_out) -> bool {  // *string, lower-cased; default "gpu"
        std::string name = "gpu";
        if (present) {
            Val m;
            if (!head(cc, m)) return false;
            if (m.k == K_STR || m.k == K_BIN) name = lower(std::string((const char*)m.s, m.n));
            else if (m.k != K_NIL) return false;
        }
        const int id = h->tiers.id(name, KVIDX_MAX_TIERS);
        if (id < 0) return false;
        *tier_out = id;
        return true;
    };
    if (t == "BlockStored") {
        const size_t h0 = hashes.size(), t0 = toks.size();
        kvidx_event_t ev{};
        ev.op = KVIDX_EV_BLOCK_STORED; ev.model = model; ev.hash_off = h0; ev.tok_off = t0;
        bool ok = true, parent_bad = false;
        size_t f = 0;
        if (f < rest) {                                                   // BlockHashes []any
            Val a;
            if (!head(c, a)) return;
            if (a.k == K_ARRAY) { for (size_t i = 0; i < a.n && ok; ++i) { uint64_t hv; const uint8_t* before = c.p; if (hash_of(c, &hv, nullptr)) hashes.push_back(hv); if (c.p == before || c.p > e) ok = false; } }
            else if (a.k != K_NIL) ok = false;
            ++f;
        }
        if (ok && f < rest) {                                             // ParentBlockHash any
            uint64_t hv; bool nil = false;
            if (hash_of(c, &hv, &nil)) { ev.has_parent = 1; ev.parent_hash = hv; }
            else if (!nil) parent_bad = true;                             // present but unsupported type: event skipped (pool.go:283-287)
            ++f;
        }
        if (ok && f < rest) {                                             // TokenIds []uint32
            Val a;
            if (!head(c, a)) ok = false;
            else if (a.k == K_ARRAY) { for (size_t i = 0; i < a.n && ok; ++i) { Val x; if (!head(c, x) || x.k != K_INT) ok = false; else toks.push_back((uint32_t)x.u); } }
            else if (a.k != K_NIL) ok = false;
            ++f;
        }
        if (ok && f < rest) { Val x; if (!head(c, x) || (x.k != K_INT && x.k != K_NIL)) ok = false; ++f; }   // BlockSize int (ignored)
        if (ok && f < rest) { Val x; if (!head(c, x) || (x.k != K_INT && x.k != K_NIL)) ok = false; ++f; }   // LoraID *int
        int tier = 0;
        if (ok) { ok = medium_tier(c, f < rest, &tier); if (f < rest) ++f; }
        for (; ok && f < rest; ++f) ok = skip(c);                         // extra fields are skipped
        if (!ok || parent_bad) { hashes.resize(h0); toks.resize(t0); return; }
        ev.podtier = KVIDX_PODTIER(pod, tier);
        ev.n_hashes = (uint32_t)(hashes.size() - h0); ev.n_tokens = (uint32_t)(toks.size() - t0);
        evs.push_back(ev);
    } else if (t == "BlockRemoved") {
        const size_t h0 = hashes.size();
        kvidx_event_t ev{};
        ev.op = KVIDX_EV_BLOCK_REMOVED; ev.model = model; ev.hash_off = h0; ev.tok_off = toks.size();
        bool ok = true;
        size_t f = 0;
        if (f < rest) {
            Val a;
            if (!head(c, a)) return;
            if (a.k == K_ARRAY) { for (size_t i = 0; i < a.n && ok; ++i) { uint64_t hv; const uint8_t* before = c.p; if (hash_of(c, &hv, nullptr)) hashes.push_back(hv); if (c.p == before || c.p > e) ok = false; } }
            else if (a.k != K_NIL) ok = false;
            ++f;
        }
        int tier = 0;
        if (ok) { ok = medium_tier(c, f < rest, &tier); if (f < rest) ++f; }
        for (; ok && f < rest; ++f) ok = skip(c);
        if (!ok) { hashes.resize(h0); return; }
        ev.podtier = KVIDX_PODTIER(pod, tier);
        ev.n_hashes = (uint32_t)(hashes.size() - h0);
        evs.push_back(ev);
    }
    else if (t == "AllBlocksCleared" && h->cfg.clear_on_all_blocks_cleared) {     // host-level marker, never applied as is
        kvidx_event_t ev{};
        ev.op = KVHOST_EV_ALL_BLOCKS_CLEARED; ev.model = model; ev.podtier = KVIDX_PODTIER(pod, 0);
        ev.hash_off = hashes.size(); ev.tok_off = toks.size();
        evs.push_back(ev);
    }
    // "AllBlocksCleared" otherwise: no-op (pool.go:332-333); unknown tags: skipped (pool.go:229-231)
}

// EventBatch = [ts, events[], data_parallel_rank?] (events.go:38-43).  Any decode error drops the whole message.
void decode_batch(kvhost* h, uint32_t pod, uint32_t model, const uint8_t* p, size_t len, std::vector<kvidx_event_t>& evs,
                  std::vector<uint64_t>& hashes, std::vector<uint32_t>& toks) {
    Cur c{p, p + len};
    Val v;
    if (!head(c, v) || v.k != K_ARRAY) return;
    const size_t n = v.n;
    std::vector<std::pair<const uint8_t*, const uint8_t*>> raw;
    if (n >= 1) { Val ts; if (!head(c, ts) || (ts.k != K_FLOAT && ts.k != K_INT && ts.k != K_NIL)) return; }
    if (n >= 2) {
        Val a;
        if (!head(c, a)) return;
        if (a.k == K_ARRAY) {
            for (size_t i = 0; i < a.n; ++i) { const uint8_t* s = c.p; if (!skip(c)) return; raw.emplace_back(s, c.p); }
        } else if (a.k != K_NIL) return;
    }
    if (n >= 3) { Val r; if (!head(c, r) || (r.k != K_INT && r.k != K_NIL)) return; }
    for (size_t i = 3; i < n; ++i) if (!skip(c)) return;
    for (auto& r : raw) decode_event(h, pod, model, r.first, r.second, evs, hashes, toks);
}

}  // namespace

static const double kLatencyBuckets[KVHOST_LATENCY_BUCKETS] = {0.005, 0.01, 0.025, 0.05, 0.1, 0.25, 0.5, 1.0, 2.5, 5.0, 10.0};   // prometheus.DefBuckets

extern "C" {

const char* kvhost_last_error(void) { return g_herr.c_str(); }

void kvhost_config_default(kvhost_config_t* c) {
    if (!c) return;
    memset(c, 0, sizeof *c);
    kvidx_config_default(&c->index);
    c->concurrency = 4;                      // kvevents/pool.go:52
    c->n_tiers = 2;
    c->tier_names[0] = "gpu"; c->tier_weights[0] = 1.0;     // backend.go:28
    c->tier_names[1] = "cpu"; c->tier_weights[1] = 0.8;     // backend.go:29
}

int kvhost_create(const kvhost_config_t* cfg_in, const char* hash_seed, kvhost_t** out) {
    if (!out) return hfail(KVIDX_EINVAL, "out is NULL");
    *out = nullptr;
    kvhost_config_t c;
    kvhost_config_default(&c);
    if (cfg_in) c = *cfg_in;
    if (c.concurrency == 0) c.concurrency = 4;
    if (c.n_tiers > KVIDX_MAX_TIERS) return hfail(KVIDX_ERANGE, "too many tiers");
    kvhost* h = new kvhost();
    h->cfg = c;
    h->queues.resize(c.concurrency);
    for (uint32_t i = 0; i < c.n_tiers; ++i) h->tiers.id(lower(c.tier_names[i] ? c.tier_names[i] : ""), KVIDX_MAX_TIERS);
    h->cfg_tiers = (uint32_t)h->tiers.names.size();
    const char* seed = hash_seed ? hash_seed : "";
    c.index.init_hash = kvidx_fnv64a(seed, strlen(seed));           // getInitHash, token_processor.go:81-90
    c.index.n_tier_weights = c.n_tiers;
    for (uint32_t i = 0; i < KVIDX_MAX_TIERS; ++i) c.index.tier_weight[i] = i < c.n_tiers ? c.tier_weights[i] : 1.0;
    h->filter_words = ((c.index.max_pods ? c.index.max_pods : 256) + 63) / 64;
    h->pod_cap = c.index.max_pods ? c.index.max_pods : 256;     // pods that own index entries must fit the score / filter row width
    if (!c.no_device) {
        const int rc = kvidx_create(&c.index, &h->ix);
        if (rc) { g_herr = kvidx_last_error(nullptr); delete h; return rc; }
    }
    *out = h;
    return 0;
}

void kvhost_destroy(kvhost_t* h) { if (!h) return; if (h->ix) kvidx_destroy(h->ix); delete h; }
kvidx_t* kvhost_index(kvhost_t* h) { return h ? h->ix : nullptr; }

int kvhost_get_metrics(kvhost_t* h, kvhost_metrics_t* out) {
    if (!h || !out) return hfail(KVIDX_EINVAL, "bad arguments");
    std::lock_guard<std::mutex> g(h->mu);
    *out = h->met;
    return 0;
}

int64_t kvhost_metrics_text(kvhost_t* h, char* buf, size_t cap) {
    kvhost_metrics_t m;
    if (kvhost_get_metrics(h, &m)) return KVIDX_EINVAL;
    std::string s;
    auto counter = [&](const char* name, const char* help, uint64_t v) {
        s += "# HELP kvcache_index_"; s += name; s += " "; s += help; s += "\n# TYPE kvcache_index_"; s += name; s += " counter\nkvcache_index_";
        s += name; s += " " + std::to_string(v) + "\n";
    };
    counter("admissions_total", "Total number of KV-block admissions", m.admissions_total);
    counter("evictions_total", "Total number of KV-block evictions", m.evictions_total);
    counter("lookup_requests_total", "Total number of lookup calls", m.lookup_requests_total);
    counter("max_pod_hit_count_total", "Maximum cache hits on a single pod on Lookup()", m.max_pod_hit_count_total);
    counter("lookup_hits_total", "Number of keys found in the cache on Lookup()", m.lookup_hits_total);
    uint64_t cap_ev[2] = {0, 0};                      // the index's own count (no device: none)
    if (h->ix && kvidx_get_evictions(h->ix, cap_ev)) cap_ev[0] = cap_ev[1] = 0;   // does not wait for a write batch
    counter("capacity_evictions_total", "Total number of request keys evicted to hold the index to its capacity", cap_ev[0]);
    counter("capacity_engine_evictions_total", "Total number of engine-key mappings evicted to hold the index to its capacity", cap_ev[1]);
    s += "# HELP kvcache_index_lookup_latency_seconds Latency of Lookup calls in seconds\n# TYPE kvcache_index_lookup_latency_seconds histogram\n";
    char tmp[96];
    for (int b = 0; b < KVHOST_LATENCY_BUCKETS; ++b) {
        snprintf(tmp, sizeof tmp, "kvcache_index_lookup_latency_seconds_bucket{le=\"%g\"} %llu\n", kLatencyBuckets[b], (unsigned long long)m.lookup_latency_bucket[b]);
        s += tmp;
    }
    snprintf(tmp, sizeof tmp, "kvcache_index_lookup_latency_seconds_bucket{le=\"+Inf\"} %llu\n", (unsigned long long)m.lookup_latency_count); s += tmp;
    snprintf(tmp, sizeof tmp, "kvcache_index_lookup_latency_seconds_sum %.9g\n", m.lookup_latency_sum); s += tmp;
    snprintf(tmp, sizeof tmp, "kvcache_index_lookup_latency_seconds_count %llu\n", (unsigned long long)m.lookup_latency_count); s += tmp;
    if (buf && cap) { const size_t n = std::min(cap - 1, s.size()); memcpy(buf, s.data(), n); buf[n] = 0; }
    return (int64_t)s.size();
}

int kvhost_pod_id(kvhost_t* h, const char* s) { std::lock_guard<std::mutex> g(h->mu); return h->pods.id(s, KVIDX_MAX_PODS); }
int kvhost_tier_id(kvhost_t* h, const char* s) { std::lock_guard<std::mutex> g(h->mu); return h->tiers.id(lower(s), KVIDX_MAX_TIERS); }
int kvhost_model_id(kvhost_t* h, const char* s) { std::lock_guard<std::mutex> g(h->mu); return h->models.id(s, 65536); }

static int need_dev(kvhost* h) { return h && h->ix ? 0 : hfail(KVIDX_ECUDA, "host-only instance: no device index (there is no CPU fallback)"); }

// One Lookup as the instrumented index sees it (instrumented_index.go:47-69): request + latency always, its hit count
// (0 for a failed Lookup) added to both hit counters.  Caller holds h->mu.
static void record_lookup_locked(kvhost* h, double seconds, uint64_t hits) {
    h->met.lookup_requests_total += 1;
    h->met.lookup_latency_count += 1; h->met.lookup_latency_sum += seconds;
    for (int b = 0; b < KVHOST_LATENCY_BUCKETS; ++b) if (seconds <= kLatencyBuckets[b]) h->met.lookup_latency_bucket[b] += 1;
    h->met.max_pod_hit_count_total += hits; h->met.lookup_hits_total += hits;
}
static void observe_hits(kvhost* h, double seconds, uint64_t hits) {
    if (!h->cfg.enable_metrics) return;
    std::lock_guard<std::mutex> g(h->mu);
    record_lookup_locked(h, seconds, hits);
}

// A Lookup whose result came back key by key.  recordHitMetrics counts entries per pod over the result MAP: without a filter
// (keys given) a repeated key is one map entry and counts once (in_memory.go:126-128); with one every occurrence appended
// its entries (:130-135).
static void observe_lookup(kvhost* h, double seconds, bool ok, const kvidx_podtier_t* pt, const uint8_t* cnt, size_t n, const uint64_t* keys) {
    if (!h->cfg.enable_metrics) return;
    uint64_t mx = 0;
    if (ok) {
        std::vector<uint32_t> per(KVIDX_MAX_PODS, 0);
        std::unordered_set<uint64_t> seen;
        for (size_t i = 0; i < n; ++i) {
            if (keys && cnt[i] && !seen.insert(keys[i]).second) continue;
            for (int j = 0; j < cnt[i]; ++j) { const uint32_t c = ++per[KVIDX_PT_POD(pt[i * KVIDX_MAX_PODS_PER_KEY + j])]; if (c > mx) mx = c; }
        }
    }
    observe_hits(h, seconds, mx);
}

static bool build_filter(kvhost* h, const char* const* pods, size_t n_pods, std::vector<uint64_t>& mask) {
    // sets.New(podIdentifiers...): a name never seen by the index cannot match any entry, but still makes the set non-empty
    mask.assign(h->filter_words, 0);
    if (n_pods == 0) return false;
    for (size_t i = 0; i < n_pods; ++i) {
        const int id = h->pods.id(pods[i], KVIDX_MAX_PODS);
        if (id >= 0 && (uint32_t)id < h->filter_words * 64) mask[id >> 6] |= 1ull << (id & 63);
    }
    return true;
}

// With enable_metrics: the instrumented Lookup of indexer.go:150 over every key of one prompt, given as its tokens
// (keys == nullptr, n = token count) or its request keys (n = key count): one kvidx_lookup_hits call.
static void observe_prompt(kvhost* h, const uint32_t* tokens, const uint64_t* keys, size_t n, uint32_t mid, const uint64_t* fm) {
    if (!h->cfg.enable_metrics) return;
    const int64_t off[2] = {0, (int64_t)n};
    uint32_t hits = 0;
    const auto t0 = std::chrono::steady_clock::now();
    const int r2 = keys ? kvidx_lookup_hits_keys(h->ix, keys, off, 1, nullptr, mid, fm, &hits)
                        : kvidx_lookup_hits(h->ix, tokens, off, 1, nullptr, mid, fm, &hits);
    observe_hits(h, std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(), r2 == 0 ? hits : 0);
}

// GetPodScores from step 3 on for one prompt given as its tokens (keys == nullptr, n = token count) or as its request
// keys (n = key count).
static int pod_scores(kvhost* h, const uint32_t* tokens, const uint64_t* keys, size_t n, const char* model, const char* const* pods, size_t n_pods,
                      const char** pod_out, double* score_out) {
    if (int rc = need_dev(h)) return rc;
    std::shared_lock<std::shared_mutex> rl(h->read_mu);
    std::vector<uint64_t> mask;
    bool filtered; int mid;
    { std::lock_guard<std::mutex> g(h->mu); filtered = build_filter(h, pods, n_pods, mask); mid = h->models.id(model, 65536); }
    if (mid < 0) return hfail(KVIDX_ERANGE, "too many models");
    if (filtered) {                                 // a filter whose pods all lie outside the mask width selects nothing
        bool any = false; for (uint64_t w : mask) any |= w != 0;
        if (!any) {
            const bool has_keys = keys ? n > 0 : n >= (h->cfg.index.block_size ? h->cfg.index.block_size : 16);
            if (has_keys) observe_hits(h, 0.0, 0);      // the Lookup still happens; it just finds no listed pod
            return has_keys ? 0 : -1000;
        }
    }
    const int64_t off[2] = {0, (int64_t)n};
    uint16_t ids[KVIDX_MAX_PODS_PER_KEY]; double sc[KVIDX_MAX_PODS_PER_KEY]; uint8_t cnt = 0, has = 0;
    const uint64_t* fm = filtered ? mask.data() : nullptr;
    const int rc = keys ? kvidx_score_keys_sparse(h->ix, keys, off, 1, nullptr, (uint32_t)mid, fm, ids, sc, &cnt, &has)
                        : kvidx_score_batch_sparse(h->ix, tokens, off, 1, nullptr, (uint32_t)mid, fm, ids, sc, &cnt, &has);
    if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
    if (!has) return -1000;                         // (nil, nil): no full block (indexer.go:142-146)
    observe_prompt(h, tokens, keys, n, (uint32_t)mid, fm);
    std::lock_guard<std::mutex> g(h->mu);
    for (int i = 0; i < cnt; ++i) { pod_out[i] = h->pods.name(ids[i]); score_out[i] = sc[i]; }
    return cnt;
}

// GetPodScores for a batch: prompt texts through the device prefix store (text != nullptr; tokenize_out flags the prompts
// whose cached prefix is too short) or a token CSR.  Like pod_scores, read_mu is held from the filter through the device
// call to the id -> name mapping, so a pod id freed and reused meanwhile cannot lend its new name to the old pod's entries.
static int batch_scores(kvhost* h, const uint8_t* text, const int64_t* text_off, const uint32_t* tok, const int64_t* tok_off, size_t n,
                        const char* model, const char* const* pods, size_t n_pods, double min_ratio, const char** pod_out, double* score_out,
                        int32_t* cnt_out, uint8_t* tokenize_out) {
    if (int rc = need_dev(h)) return rc;
    if (!model || !pod_out || !score_out || !cnt_out || (text_off ? !tokenize_out : !tok_off) || (n_pods && !pods))
        return hfail(KVIDX_EINVAL, "bad arguments");
    if (n == 0) return 0;
    std::shared_lock<std::shared_mutex> rl(h->read_mu);
    std::vector<uint64_t> mask;
    bool filtered; int mid;
    { std::lock_guard<std::mutex> g(h->mu); filtered = build_filter(h, pods, n_pods, mask); mid = h->models.id(model, 65536); }
    if (mid < 0) return hfail(KVIDX_ERANGE, "too many models");
    bool none = filtered;                           // a filter whose pods all lie outside the mask width selects nothing
    for (uint64_t w : mask) none = none && w == 0;
    std::vector<uint64_t> rows;
    if (filtered && !none) { rows.resize(n * h->filter_words); for (size_t i = 0; i < n; ++i) memcpy(&rows[i * h->filter_words], mask.data(), h->filter_words * 8); }
    const uint64_t* fm = rows.empty() ? nullptr : rows.data();
    std::vector<uint16_t> ids(n * KVIDX_MAX_PODS_PER_KEY); std::vector<double> sc(n * KVIDX_MAX_PODS_PER_KEY);
    std::vector<uint8_t> cnt(n), has(n);
    int rc = text ? kvidx_score_text_sparse(h->ix, text, text_off, (int64_t)n, nullptr, (uint32_t)mid, fm, min_ratio, ids.data(), sc.data(),
                                            cnt.data(), has.data(), tokenize_out, nullptr)
                  : kvidx_score_batch_sparse(h->ix, tok, tok_off, (int64_t)n, nullptr, (uint32_t)mid, fm, ids.data(), sc.data(), cnt.data(), has.data());
    if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
    if (h->cfg.enable_metrics) {                    // one instrumented Lookup per scored prompt, as pod_scores counts them
        std::vector<uint32_t> found;
        std::vector<int64_t> foff(n + 1, 0);
        const int64_t* to = tok_off;
        if (text) {
            // the tokens the score used: a second find over the same prompts touches the same keys in the same order, so the
            // store's recency order comes out as after one find
            rc = kvidx_text_store_find(h->ix, text, text_off, (int64_t)n, nullptr, 0, foff.data(), nullptr);
            if (rc == KVIDX_ENOSPC) { found.resize((size_t)foff[n]); rc = kvidx_text_store_find(h->ix, text, text_off, (int64_t)n, found.data(), foff[n], foff.data(), nullptr); }
            if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
            to = foff.data();
        }
        const uint32_t* tb = text ? found.data() : tok;
        // The hit counts of every scored prompt in ONE kvidx_lookup_hits call.  A prompt that was not scored but has a full
        // block (text left to the tokenizer) must not be looked up -- its keys would be touched -- so such a batch passes
        // its scored prompts' tokens, compacted; every other prompt has no key and may stay in the call.
        const uint32_t B = h->cfg.index.block_size ? h->cfg.index.block_size : 16;
        size_t m = 0; bool compact = false;
        for (size_t i = 0; i < n; ++i) { m += has[i] != 0; compact |= !has[i] && to[i + 1] - to[i] >= (int64_t)B; }
        std::vector<uint32_t> hits, ctok;
        std::vector<int64_t> coff;
        int r2 = 0;
        double secs = 0.0;
        if (!none && m > 0) {
            const uint32_t* ct = tb; const int64_t* co = to; size_t cn = n;
            if (compact) {
                coff.assign(1, 0);
                for (size_t i = 0; i < n; ++i) {
                    if (!has[i]) continue;
                    ctok.insert(ctok.end(), tb + to[i], tb + to[i + 1]);
                    coff.push_back((int64_t)ctok.size());
                }
                ct = ctok.data(); co = coff.data(); cn = m;
            }
            hits.resize(cn);
            const auto t0 = std::chrono::steady_clock::now();
            r2 = kvidx_lookup_hits(h->ix, ct, co, (int64_t)cn, nullptr, (uint32_t)mid, fm, hits.data());
            secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() / (double)m;
        }
        std::lock_guard<std::mutex> g(h->mu);
        for (size_t i = 0, j = 0; i < n; ++i) {
            if (!has[i]) continue;
            record_lookup_locked(h, secs, none || r2 ? 0 : hits[compact ? j : i]);
            ++j;
        }
    }
    std::lock_guard<std::mutex> g(h->mu);
    for (size_t i = 0; i < n; ++i) {
        cnt_out[i] = !has[i] ? -1 : none ? 0 : cnt[i];
        for (int j = 0; j < cnt_out[i]; ++j) {
            pod_out[i * KVIDX_MAX_PODS_PER_KEY + j] = h->pods.name(ids[i * KVIDX_MAX_PODS_PER_KEY + j]);
            score_out[i * KVIDX_MAX_PODS_PER_KEY + j] = sc[i * KVIDX_MAX_PODS_PER_KEY + j];
        }
    }
    return 0;
}

int kvhost_get_pod_scores_text(kvhost_t* h, const uint8_t* text, const int64_t* text_off, size_t n, const char* model, const char* const* pods,
                               size_t n_pods, double min_ratio, const char** pod_out, double* score_out, int32_t* cnt_out, uint8_t* tokenize_out) {
    if (!text_off && n) return hfail(KVIDX_EINVAL, "NULL text_off");
    return batch_scores(h, text, text_off, nullptr, nullptr, n, model, pods, n_pods, min_ratio, pod_out, score_out, cnt_out, tokenize_out);
}

int kvhost_get_pod_scores_batch(kvhost_t* h, const uint32_t* tokens, const int64_t* tok_off, size_t n, const char* model, const char* const* pods,
                                size_t n_pods, const char** pod_out, double* score_out, int32_t* cnt_out) {
    return batch_scores(h, nullptr, nullptr, tokens, tok_off, n, model, pods, n_pods, 0.0, pod_out, score_out, cnt_out, nullptr);
}

int kvhost_get_pod_scores(kvhost_t* h, const uint32_t* tokens, size_t n_tokens, const char* model, const char* const* pods, size_t n_pods,
                          const char** pod_out, double* score_out) {
    return pod_scores(h, tokens, nullptr, n_tokens, model, pods, n_pods, pod_out, score_out);
}

int kvhost_get_pod_scores_keys(kvhost_t* h, const uint64_t* keys, size_t n_keys, const char* model, const char* const* pods, size_t n_pods,
                               const char** pod_out, double* score_out) {
    if (n_keys && !keys) return hfail(KVIDX_EINVAL, "NULL keys");
    static const uint64_t none = 0;
    return pod_scores(h, nullptr, keys ? keys : &none, n_keys, model, pods, n_pods, pod_out, score_out);
}

int kvhost_get_pod_scores_turn(kvhost_t* h, const uint64_t* keys, size_t n_keys, const uint32_t* tokens, size_t n_tokens, const char* model,
                               const char* const* pods, size_t n_pods, const char** pod_out, double* score_out, uint64_t* new_keys_out) {
    if ((n_keys && !keys) || (n_tokens && !tokens)) return hfail(KVIDX_EINVAL, "NULL keys or tokens");
    if (int rc = need_dev(h)) return rc;
    std::shared_lock<std::shared_mutex> rl(h->read_mu);
    std::vector<uint64_t> mask;
    bool filtered; int mid;
    { std::lock_guard<std::mutex> g(h->mu); filtered = build_filter(h, pods, n_pods, mask); mid = h->models.id(model, 65536); }
    if (mid < 0) return hfail(KVIDX_ERANGE, "too many models");
    const size_t nn = n_tokens / (h->cfg.index.block_size ? h->cfg.index.block_size : 16);
    static const uint64_t none = 0;
    static const uint32_t none32 = 0;
    const uint64_t* kp = keys ? keys : &none;
    const uint32_t* tp = tokens ? tokens : &none32;
    const int64_t koff[2] = {0, (int64_t)n_keys}, toff[2] = {0, (int64_t)n_tokens};
    int64_t noff[2] = {0, 0};
    std::vector<uint64_t> all(n_keys + std::max<size_t>(nn, 1));     // K = held ++ new keys
    if (n_keys) memcpy(all.data(), keys, n_keys * 8);
    uint64_t* nk = all.data() + n_keys;
    const bool has_keys = n_keys + nn > 0;
    auto give_keys = [&] { if (new_keys_out && nn) memcpy(new_keys_out, nk, nn * 8); };
    if (filtered) {                                 // a filter whose pods all lie outside the mask width selects nothing
        bool any = false; for (uint64_t w : mask) any |= w != 0;
        if (!any) {
            if (nn) {                               // the new keys are still the caller's
                const uint64_t parent = n_keys ? keys[n_keys - 1] : 0;
                const uint8_t pv = n_keys > 0;
                if (kvidx_hash_keys(h->ix, tp, toff, 1, &parent, &pv, nk, noff)) { g_herr = kvidx_last_error(h->ix); return KVIDX_EINVAL; }
            }
            give_keys();
            if (has_keys) observe_hits(h, 0.0, 0);
            return has_keys ? 0 : -1000;
        }
    }
    uint16_t ids[KVIDX_MAX_PODS_PER_KEY]; double sc[KVIDX_MAX_PODS_PER_KEY]; uint8_t cnt = 0, has = 0;
    const uint64_t* fm = filtered ? mask.data() : nullptr;
    const int rc = kvidx_score_turn_sparse(h->ix, kp, koff, tp, toff, 1, nullptr, (uint32_t)mid, fm, ids, sc, &cnt, &has, nk, noff);
    if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
    give_keys();
    if (!has) return -1000;                         // (nil, nil): no key at all
    observe_prompt(h, nullptr, all.data(), n_keys + nn, (uint32_t)mid, fm);     // the instrumented Lookup of indexer.go:150: every key of K
    std::lock_guard<std::mutex> g(h->mu);
    for (int i = 0; i < cnt; ++i) { pod_out[i] = h->pods.name(ids[i]); score_out[i] = sc[i]; }
    return cnt;
}

static int entries_of(kvhost* h, const char* const* pods, const char* const* tiers, size_t n, std::vector<kvidx_podtier_t>& out) {
    out.clear();
    for (size_t i = 0; i < n; ++i) {
        const int p = h->pods.id(pods[i], h->pod_cap), t = h->tiers.id(lower(tiers[i]), KVIDX_MAX_TIERS);
        if (p < 0 || t < 0) return hfail(KVIDX_ERANGE, "pod / tier id space exhausted");
        out.push_back(KVIDX_PODTIER(p, t));
    }
    return 0;
}

int kvhost_index_add(kvhost_t* h, const char* model, const uint64_t* engine, size_t n_engine, const uint64_t* request, size_t n_request,
                     const char* const* pods, const char* const* tiers, size_t n_entries) {
    if (int rc = need_dev(h)) return rc;
    if (h->cfg.enable_metrics) { std::lock_guard<std::mutex> g(h->mu); h->met.admissions_total += n_request; }   // whatever Add returns
    if (n_engine == 0 || n_request == 0 || n_entries == 0) return hfail(KVIDX_EINVAL, "no keys or entries provided for adding to index");
    if (n_engine != n_request) return hfail(KVIDX_EINVAL, "mismatch between engine keys and request keys length");
    std::shared_lock<std::shared_mutex> wl(h->write_mu);
    std::vector<kvidx_podtier_t> pt; int mid;
    { std::lock_guard<std::mutex> g(h->mu); if (int rc = entries_of(h, pods, tiers, n_entries, pt)) return rc; mid = h->models.id(model, 65536); }
    const int rc = kvidx_add(h->ix, (uint32_t)mid, engine, request, (int64_t)n_engine, pt.data(), (int32_t)pt.size());
    if (rc) g_herr = kvidx_last_error(h->ix);
    return rc;
}

int kvhost_index_evict(kvhost_t* h, const char* model, uint64_t engine, const char* const* pods, const char* const* tiers, size_t n_entries) {
    if (int rc = need_dev(h)) return rc;
    if (h->cfg.enable_metrics) { std::lock_guard<std::mutex> g(h->mu); h->met.evictions_total += n_entries; }
    if (n_entries == 0) return hfail(KVIDX_EINVAL, "no entries provided for eviction from index");
    std::shared_lock<std::shared_mutex> wl(h->write_mu);
    std::vector<kvidx_podtier_t> pt; int mid;
    { std::lock_guard<std::mutex> g(h->mu); if (int rc = entries_of(h, pods, tiers, n_entries, pt)) return rc; mid = h->models.id(model, 65536); }
    const int rc = kvidx_evict(h->ix, (uint32_t)mid, engine, pt.data(), (int32_t)pt.size());
    if (rc) g_herr = kvidx_last_error(h->ix);
    return rc;
}

int kvhost_index_get_request_key(kvhost_t* h, const char* model, uint64_t engine, uint64_t* out) {
    if (int rc = need_dev(h)) return rc;
    int mid; { std::lock_guard<std::mutex> g(h->mu); mid = h->models.id(model, 65536); }
    const int rc = kvidx_get_request_key(h->ix, (uint32_t)mid, engine, out);
    if (rc) g_herr = kvidx_last_error(h->ix);
    return rc;
}

int kvhost_index_lookup(kvhost_t* h, const char* model, const uint64_t* keys, size_t n, const char* const* pods, size_t n_pods,
                        const char** pod_out, const char** tier_out, uint8_t* cnt_out) {
    if (int rc = need_dev(h)) return rc;
    const auto t0 = std::chrono::steady_clock::now();
    auto secs = [&] { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); };
    if (n == 0) { observe_hits(h, secs(), 0); return hfail(KVIDX_EINVAL, "no requestKeys provided for lookup"); }
    std::shared_lock<std::shared_mutex> rl(h->read_mu);
    std::vector<uint64_t> mask; bool filtered; int mid;
    { std::lock_guard<std::mutex> g(h->mu); filtered = build_filter(h, pods, n_pods, mask); mid = h->models.id(model, 65536); }
    std::vector<kvidx_podtier_t> pt(n * KVIDX_MAX_PODS_PER_KEY);
    if (filtered) { bool any = false; for (uint64_t w : mask) any |= w != 0; if (!any) { memset(cnt_out, 0, n); observe_hits(h, secs(), 0); return 0; } }
    const int rc = kvidx_lookup(h->ix, (uint32_t)mid, keys, (int64_t)n, filtered ? mask.data() : nullptr, pt.data(), cnt_out);
    observe_lookup(h, secs(), rc == 0, pt.data(), cnt_out, n, filtered ? nullptr : keys);
    if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
    std::lock_guard<std::mutex> g(h->mu);
    for (size_t i = 0; i < n; ++i)
        for (int j = 0; j < cnt_out[i]; ++j) {
            const kvidx_podtier_t e = pt[i * KVIDX_MAX_PODS_PER_KEY + j];
            pod_out[i * KVIDX_MAX_PODS_PER_KEY + j] = h->pods.name(KVIDX_PT_POD(e));
            tier_out[i * KVIDX_MAX_PODS_PER_KEY + j] = h->tiers.name(KVIDX_PT_TIER(e));
        }
    return 0;
}

int kvhost_pool_queue_index(kvhost_t* h, const char* pod) { return (int)kvidx_queue_index(pod, strlen(pod), h->cfg.concurrency); }

int kvhost_pool_add_task(kvhost_t* h, const char* pod, const char* model, const void* payload, size_t len) {
    if (!h || !pod || !model) return hfail(KVIDX_EINVAL, "bad arguments");
    std::lock_guard<std::mutex> g(h->mu);
    const int p = h->pods.id(pod, h->pod_cap), m = h->models.id(model, 65536);
    if (p < 0 || m < 0) return hfail(KVIDX_ERANGE, "pod / model id space exhausted");
    h->queues[kvidx_queue_index(pod, strlen(pod), h->cfg.concurrency)].push_back(Msg{(uint32_t)p, (uint32_t)m, std::string((const char*)payload, len)});
    return 0;
}

// clear_on_all_blocks_cleared: the drained batch cut at the AllBlocksCleared markers.  Segment k takes each pod's events
// after its k-th marker (and before its (k+1)-th); the pods whose k-th marker closes segment k are removed right after it.
static int64_t process_segments(kvhost* h, const std::vector<kvidx_event_t>& evs, const std::vector<uint64_t>& hashes,
                                const std::vector<uint32_t>& toks, int64_t* n_dropped_out) {
    std::vector<uint32_t> seg(evs.size()), cleared(KVIDX_MAX_PODS, 0);
    uint32_t n_seg = 1;
    for (size_t i = 0; i < evs.size(); ++i) {
        const uint32_t p = KVIDX_PT_POD(evs[i].podtier);
        seg[i] = cleared[p];
        if (evs[i].op == KVHOST_EV_ALL_BLOCKS_CLEARED) n_seg = std::max(n_seg, ++cleared[p] + 1);
    }
    int gpu;
    { std::lock_guard<std::mutex> g(h->mu); gpu = h->tiers.id("gpu", KVIDX_MAX_TIERS); }     // the tier of a Medium-less event
    if (gpu < 0) return hfail(KVIDX_ERANGE, "tier id space exhausted");
    int64_t applied = 0, dropped = 0;
    std::vector<kvidx_event_t> part;
    std::vector<uint64_t> mask(h->filter_words);
    for (uint32_t k = 0; k < n_seg; ++k) {
        part.clear();
        std::fill(mask.begin(), mask.end(), 0ull);
        bool any = false;
        for (size_t i = 0; i < evs.size(); ++i) {
            if (seg[i] != k) continue;
            if (evs[i].op != KVHOST_EV_ALL_BLOCKS_CLEARED) { part.push_back(evs[i]); continue; }
            const uint32_t p = KVIDX_PT_POD(evs[i].podtier);
            mask[p >> 6] |= 1ull << (p & 63);
            any = true;
        }
        if (!part.empty()) {
            int64_t d = 0;
            const int rc = kvidx_apply_events(h->ix, part.data(), (int64_t)part.size(), hashes.data(), (int64_t)hashes.size(), toks.data(),
                                              (int64_t)toks.size(), &d);
            if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
            applied += (int64_t)part.size(); dropped += d;
        }
        if (any) {
            const int rc = kvidx_remove_pods(h->ix, mask.data(), 1u << gpu, nullptr);
            if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
        }
    }
    if (n_dropped_out) *n_dropped_out = dropped;
    return applied;
}

// Drains of at least this many payload bytes are decoded on the device (kvidx_apply_event_payloads), smaller ones by
// decode_batch on the host.  scripts/bench_event_payloads.py (BASELINE config #5 events, 4 per message, 10 M-block index;
// NVIDIA H100 80GB HBM3 at 700 W, DESIGN section 6): the host path was faster at 52 KB (21 K vs 14 K events/s), the
// device path at 0.83 MB (130 K vs 96 K) and beyond; the device call has a floor of about 1.5 ms.
static constexpr size_t kDeviceDecodeMinBytes = size_t(1) << 20;

static void count_metrics(kvhost* h, const std::vector<kvidx_event_t>& evs) {
    const uint32_t bs = h->cfg.index.block_size ? h->cfg.index.block_size : 16;
    uint64_t adm = 0, evi = 0;
    for (const auto& e : evs) {
        if (e.op == KVIDX_EV_BLOCK_STORED) { if (e.n_hashes > 0) adm += e.n_tokens / bs; }      // Add(len(requestKeys)) only if there are engine keys
        else if (e.op == KVIDX_EV_BLOCK_REMOVED) evi += e.n_hashes;                             // one Evict with one entry per hash
    }
    std::lock_guard<std::mutex> g(h->mu);
    h->met.admissions_total += adm; h->met.evictions_total += evi;
}

// The host path's apply: the drained messages decoded (and interned) by decode_batch, then one kvidx_apply_events (or the
// segments of a drain with AllBlocksCleared markers).
static int64_t apply_decoded(kvhost* h, const std::vector<kvidx_event_t>& evs, const std::vector<uint64_t>& hashes,
                             const std::vector<uint32_t>& toks, int64_t* n_dropped_out) {
    if (h->cfg.enable_metrics) count_metrics(h, evs);  // digestEvents calls the instrumented Add / Evict (pool.go:299-330)
    if (evs.empty()) return 0;
    if (h->cfg.clear_on_all_blocks_cleared) return process_segments(h, evs, hashes, toks, n_dropped_out);
    const int rc = kvidx_apply_events(h->ix, evs.data(), (int64_t)evs.size(), hashes.data(), (int64_t)hashes.size(), toks.data(), (int64_t)toks.size(), n_dropped_out);
    if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
    return (int64_t)evs.size();
}

// The device path: the payloads packed in drain order and decoded by kvidx_apply_event_payloads against a copy of the tier
// table.  A message naming a tier the copy lacks is decoded on the host, under mu and in drain order, only to intern its
// names exactly as the host path would; the call is then repeated with the unknown tiers skipped (they are the names that
// found no room in the 16 ids).  A drain with AllBlocksCleared under clear_on_all_blocks_cleared goes to the host path.
static int64_t process_on_device(kvhost* h, std::vector<Msg>& msgs, int64_t* n_dropped_out) {
    const size_t n = msgs.size();
    std::vector<uint8_t> bytes; std::vector<int64_t> off(n + 1, 0); std::vector<uint32_t> pod(n), model(n);
    for (size_t i = 0; i < n; ++i) off[i + 1] = off[i] + (int64_t)msgs[i].payload.size();
    bytes.resize((size_t)off[n]);
    for (size_t i = 0; i < n; ++i) {
        memcpy(bytes.data() + off[i], msgs[i].payload.data(), msgs[i].payload.size());
        pod[i] = msgs[i].pod; model[i] = msgs[i].model;
    }
    std::vector<uint8_t> mflags(n);
    uint32_t flags = h->cfg.clear_on_all_blocks_cleared ? KVIDX_PAYLOAD_STOP_AT_CLEARED : 0u;
    int64_t counts[KVIDX_PAYLOAD_COUNTS];
    for (;;) {
        std::string tb; std::vector<int64_t> toff(1, 0); int gpu;
        {
            std::lock_guard<std::mutex> g(h->mu);
            for (const std::string* s : h->tiers.names) { tb += *s; toff.push_back((int64_t)tb.size()); }
            gpu = h->tiers.find("gpu");
        }
        const int rc = kvidx_apply_event_payloads(h->ix, bytes.data(), off.data(), (int64_t)n, pod.data(), model.data(), (const uint8_t*)tb.data(),
                                                  toff.data(), (uint32_t)(toff.size() - 1), gpu, flags, mflags.data(), counts, n_dropped_out);
        if (rc == KVIDX_ENOENT && (flags & KVIDX_PAYLOAD_STOP_AT_CLEARED) && counts[7] > 0) {
            std::vector<kvidx_event_t> evs; std::vector<uint64_t> hs; std::vector<uint32_t> ts;
            {
                std::lock_guard<std::mutex> g(h->mu);
                for (auto& m : msgs) decode_batch(h, m.pod, m.model, (const uint8_t*)m.payload.data(), m.payload.size(), evs, hs, ts);
            }
            return apply_decoded(h, evs, hs, ts, n_dropped_out);
        }
        if (rc == KVIDX_ENOENT && !(flags & KVIDX_PAYLOAD_SKIP_UNKNOWN_TIER)) {
            std::vector<kvidx_event_t> evs; std::vector<uint64_t> hs; std::vector<uint32_t> ts;
            std::lock_guard<std::mutex> g(h->mu);
            for (size_t i = 0; i < n; ++i)
                if (mflags[i] & KVIDX_PAYLOAD_MSG_UNKNOWN_TIER) decode_batch(h, pod[i], model[i], bytes.data() + off[i], (size_t)(off[i + 1] - off[i]), evs, hs, ts);
            flags |= KVIDX_PAYLOAD_SKIP_UNKNOWN_TIER;
            continue;
        }
        if (h->cfg.enable_metrics) {
            std::lock_guard<std::mutex> g(h->mu);
            h->met.admissions_total += (uint64_t)counts[5]; h->met.evictions_total += (uint64_t)counts[6];
        }
        if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
        return counts[1];
    }
}

int64_t kvhost_pool_process(kvhost_t* h, int64_t* n_dropped_out) {
    if (int rc = need_dev(h)) return rc;
    std::shared_lock<std::shared_mutex> wl(h->write_mu);
    std::vector<kvidx_event_t> evs; std::vector<uint64_t> hashes; std::vector<uint32_t> toks;
    std::vector<Msg> msgs;                               // a drain for the device path
    {
        std::lock_guard<std::mutex> g(h->mu);
        size_t bytes = 0;
        for (const auto& q : h->queues) for (const auto& m : q) bytes += m.payload.size();
        const bool device = bytes >= kDeviceDecodeMinBytes && !h->tiers.names.empty();
        for (auto& q : h->queues) {                      // each queue is FIFO; one pod always maps to one queue
            for (auto& m : q) {
                if (device) msgs.push_back(std::move(m));
                else decode_batch(h, m.pod, m.model, (const uint8_t*)m.payload.data(), m.payload.size(), evs, hashes, toks);
            }
            q.clear();
        }
    }
    if (n_dropped_out) *n_dropped_out = 0;
    if (!msgs.empty()) return process_on_device(h, msgs, n_dropped_out);
    return apply_decoded(h, evs, hashes, toks, n_dropped_out);
}

// Removes the pod's messages still waiting in its queue.  Caller holds mu.
static int drop_queued(kvhost* h, const char* pod, uint32_t id) {
    auto& q = h->queues[kvidx_queue_index(pod, strlen(pod), h->cfg.concurrency)];
    const size_t before = q.size();
    q.erase(std::remove_if(q.begin(), q.end(), [&](const Msg& m) { return m.pod == id; }), q.end());
    return (int)(before - q.size());
}

int kvhost_remove_pod(kvhost_t* h, const char* pod, const char* const* tiers, size_t n_tiers) {
    if (!h || !pod || (n_tiers && !tiers)) return hfail(KVIDX_EINVAL, "bad arguments");
    std::unique_lock<std::shared_mutex> wl(h->write_mu);     // no pool_process / index_add of any pod meanwhile
    int id, dropped;
    uint32_t tier_mask = n_tiers ? 0u : 0xFFFFu;
    {
        std::lock_guard<std::mutex> g(h->mu);
        for (size_t i = 0; i < n_tiers; ++i) {
            const int t = h->tiers.id(lower(tiers[i] ? tiers[i] : ""), KVIDX_MAX_TIERS);
            if (t < 0) return hfail(KVIDX_ERANGE, "tier id space exhausted");
            tier_mask |= 1u << t;
        }
        id = h->pods.find(pod);
        if (id < 0) return 0;                                    // never seen (or already removed): nothing to do
        dropped = drop_queued(h, pod, (uint32_t)id);
    }
    if (h->ix && (uint32_t)id < h->pod_cap) {                  // ids from pod_cap up (filter-only names) own no entries
        std::vector<uint64_t> mask(h->filter_words, 0);
        mask[id >> 6] |= 1ull << (id & 63);
        const int rc = kvidx_remove_pods(h->ix, mask.data(), tier_mask, nullptr);
        if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
    }
    if (n_tiers == 0) {
        std::unique_lock<std::shared_mutex> rl(h->read_mu);   // waits for the read calls that may still map this id
        std::lock_guard<std::mutex> g(h->mu);
        dropped += drop_queued(h, pod, (uint32_t)id);            // queued while the removal ran: they carry the old id
        h->pods.release((uint32_t)id);
    }
    return dropped;
}

}  // extern "C"

namespace {
const char kHostSnapMagic[8] = {'K', 'V', 'H', 'O', 'S', 'T', 'S', 'N'};
constexpr uint32_t kHostSnapVersion = 1, kReleased = 0xFFFFFFFFu;

void put32(std::string& s, uint32_t v) { s.append(reinterpret_cast<const char*>(&v), 4); }   // little-endian hosts
void put64(std::string& s, uint64_t v) { s.append(reinterpret_cast<const char*>(&v), 8); }
void put_names(std::string& s, const Interner& in) {
    put32(s, (uint32_t)in.names.size());
    for (const std::string* n : in.names) {
        if (!n) { put32(s, kReleased); continue; }
        put32(s, (uint32_t)n->size());
        s += *n;
    }
}
// one entry of a name table read back: the name of the id, or a released pod id
struct NameRec { std::string name; bool released; };
bool get_names(const uint8_t*& p, const uint8_t* e, std::vector<NameRec>& out) {
    uint32_t n;
    if (e - p < 4) return false;
    memcpy(&n, p, 4); p += 4;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t l;
        if (e - p < 4) return false;
        memcpy(&l, p, 4); p += 4;
        if (l == kReleased) { out.push_back({std::string(), true}); continue; }
        if ((uint64_t)(e - p) < l) return false;
        out.push_back({std::string(reinterpret_cast<const char*>(p), l), false});
        p += l;
    }
    return true;
}
bool distinct(const std::vector<NameRec>& v) {
    std::unordered_set<std::string> seen;
    for (const auto& r : v) if (!r.released && !seen.insert(r.name).second) return false;
    return true;
}
void install(Interner& in, const std::vector<NameRec>& v, size_t from) {      // the interner holds ids [0, from) already
    for (size_t i = from; i < v.size(); ++i) {
        if (v[i].released) { in.names.push_back(nullptr); in.free_ids.insert((uint32_t)i); continue; }
        in.names.push_back(&*in.store.insert(v[i].name).first);
        in.ids.emplace(v[i].name, (uint32_t)i);
    }
}
}  // namespace

extern "C" {

int kvhost_snapshot(kvhost_t* h, void* buf, uint64_t cap, uint64_t* size_out) {
    if (size_out) *size_out = 0;
    if (!h || !size_out) return hfail(KVIDX_EINVAL, "bad arguments");
    std::unique_lock<std::shared_mutex> wl(h->write_mu);     // no entry of any pod is written meanwhile
    std::string s(kHostSnapMagic, 8);
    put32(s, kHostSnapVersion); put32(s, 0);
    {
        std::lock_guard<std::mutex> g(h->mu);
        put_names(s, h->models); put_names(s, h->tiers); put_names(s, h->pods);
    }
    uint64_t isz = 0;
    if (h->ix) {
        const int rc = kvidx_snapshot(h->ix, nullptr, 0, &isz);             // size query
        if (rc != KVIDX_ENOSPC) { g_herr = kvidx_last_error(h->ix); return rc ? rc : KVIDX_ECUDA; }
    }
    const uint64_t total = s.size() + 8 + isz;
    *size_out = total;
    if (!buf || cap < total) return hfail(KVIDX_ENOSPC, "the snapshot needs " + std::to_string(total) + " bytes");
    put64(s, isz);
    memcpy(buf, s.data(), s.size());
    if (h->ix) {
        uint64_t got = 0;
        const int rc = kvidx_snapshot(h->ix, static_cast<char*>(buf) + s.size(), isz, &got);
        if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
    }
    return 0;
}

int kvhost_restore(kvhost_t* h, const void* buf, uint64_t len) {
    if (!h || (!buf && len)) return hfail(KVIDX_EINVAL, "bad arguments");
    const uint8_t* p = static_cast<const uint8_t*>(buf);
    const uint8_t* e = p + len;
    uint32_t ver = 0, zero = 1;
    if (len < 16 || memcmp(p, kHostSnapMagic, 8) != 0) return hfail(KVIDX_EINVAL, "malformed host snapshot: bad magic");
    memcpy(&ver, p + 8, 4); memcpy(&zero, p + 12, 4);
    if (ver != kHostSnapVersion || zero) return hfail(KVIDX_EINVAL, "unsupported host snapshot version " + std::to_string(ver));
    p += 16;
    std::vector<NameRec> models, tiers, pods;
    if (!get_names(p, e, models) || !get_names(p, e, tiers) || !get_names(p, e, pods))
        return hfail(KVIDX_EINVAL, "malformed host snapshot: truncated name table");
    uint64_t ilen = 0;
    if (e - p < 8) return hfail(KVIDX_EINVAL, "malformed host snapshot: truncated");
    memcpy(&ilen, p, 8); p += 8;
    if ((uint64_t)(e - p) != ilen) return hfail(KVIDX_EINVAL, "malformed host snapshot: index section length mismatch");
    for (const auto& r : models) if (r.released) return hfail(KVIDX_EINVAL, "malformed host snapshot: released model id");
    for (const auto& r : tiers) if (r.released) return hfail(KVIDX_EINVAL, "malformed host snapshot: released tier id");
    if (!distinct(models) || !distinct(tiers) || !distinct(pods)) return hfail(KVIDX_EINVAL, "malformed host snapshot: repeated name");
    if (models.size() > 65536 || tiers.size() > KVIDX_MAX_TIERS || pods.size() > KVIDX_MAX_PODS)
        return hfail(KVIDX_EINVAL, "malformed host snapshot: more ids than the id space holds");
    std::unique_lock<std::shared_mutex> wl(h->write_mu);
    std::lock_guard<std::mutex> g(h->mu);                    // held through the device restore: nothing interns meanwhile
    bool queued = false;
    for (const auto& q : h->queues) queued |= !q.empty();
    if (!h->pods.names.empty() || !h->models.names.empty() || h->tiers.names.size() != h->cfg_tiers || queued)
        return hfail(KVIDX_EINVAL, "restore needs a fresh host indexer (no pod or model seen, only the configured tiers, nothing queued)");
    if (tiers.size() < h->cfg_tiers) return hfail(KVIDX_EINVAL, "snapshot has fewer tiers than this indexer's configuration");
    for (uint32_t i = 0; i < h->cfg_tiers; ++i)
        if (tiers[i].name != *h->tiers.names[i])
            return hfail(KVIDX_EINVAL, "tier " + std::to_string(i) + " is \"" + tiers[i].name + "\" in the snapshot, \"" + *h->tiers.names[i] + "\" here");
    if (!h->ix && ilen) return hfail(KVIDX_EINVAL, "a host-only instance cannot restore an index section");
    if (ilen >= 64) {                                          // every pod owning an entry has a name (the rest is kvidx_restore's)
        uint64_t nreq = 0;
        memcpy(&nreq, p + 32, 8);
        if (nreq <= (ilen - 64) / 32) {
            for (uint64_t r = 0; r < nreq; ++r) {
                const uint8_t* rec = p + 64 + 32 * r;
                const uint32_t cnt = std::min<uint32_t>(rec[10], KVIDX_MAX_PODS_PER_KEY);
                for (uint32_t j = 0; j < cnt; ++j) {
                    uint16_t e;
                    memcpy(&e, rec + 12 + 2 * j, 2);
                    const uint32_t pod = KVIDX_PT_POD(e);
                    if (pod >= pods.size() || pods[pod].released)
                        return hfail(KVIDX_EINVAL, "malformed host snapshot: pod id " + std::to_string(pod) + " owns entries but has no name");
                }
            }
        }
    }
    if (ilen) {
        const int rc = kvidx_restore(h->ix, p, ilen, nullptr);
        if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
    }
    install(h->models, models, 0);
    install(h->tiers, tiers, h->cfg_tiers);
    install(h->pods, pods, 0);
    return 0;
}

int64_t kvhost_pod_inventory(kvhost_t* h, const char* model, int32_t engine, kvhost_pod_row_t* rows, size_t cap, const char** tier_names_out,
                             uint64_t totals_out[4]) {
    if (!h || (cap && !rows)) return hfail(KVIDX_EINVAL, "bad arguments");
    std::shared_lock<std::shared_mutex> wl(h->write_mu);     // no kvhost_remove_pod / kvhost_restore meanwhile: no id changes its name
    const size_t P = h->pod_cap;
    std::vector<uint64_t> ent(P * KVIDX_MAX_TIERS, 0), keys(P, 0), sole(P, 0), sole_eng(P, 0);
    uint64_t totals[4] = {0, 0, 0, 0};
    int mid = -1;
    if (model) { std::lock_guard<std::mutex> g(h->mu); mid = h->models.find(model); }
    if (h->ix && (!model || mid >= 0)) {
        const int rc = kvidx_pod_inventory(h->ix, model ? (uint32_t)mid : KVIDX_ANY_MODEL, engine ? KVIDX_INVENTORY_ENGINE : 0u, ent.data(),
                                           keys.data(), sole.data(), sole_eng.data(), totals);
        if (rc) { g_herr = kvidx_last_error(h->ix); return rc; }
    }
    // names after the counts: a writer interns a pod before it writes the pod's entries, so every id the device saw has its name
    std::lock_guard<std::mutex> g(h->mu);
    size_t n = 0;
    for (uint32_t id = 0; id < h->pods.names.size(); ++id) {
        if (!h->pods.names[id]) continue;                        // freed by kvhost_remove_pod
        if (n < cap) {
            kvhost_pod_row_t& r = rows[n];
            r = kvhost_pod_row_t{};
            r.pod = h->pods.name(id); r.pod_id = id;
            if (id < P) {                                        // ids from pod_cap up (filter-only names) own no entries
                r.keys = keys[id]; r.sole_keys = sole[id]; r.sole_engine_keys = sole_eng[id];
                memcpy(r.entries, &ent[(size_t)id * KVIDX_MAX_TIERS], sizeof r.entries);
            }
        }
        ++n;
    }
    if (tier_names_out)
        for (uint32_t t = 0; t < KVIDX_MAX_TIERS; ++t) tier_names_out[t] = t < h->tiers.names.size() ? h->tiers.name(t) : nullptr;
    if (totals_out) memcpy(totals_out, totals, sizeof totals);
    return (int64_t)n;
}

int64_t kvhost_inventory_text(kvhost_t* h, char* buf, size_t cap) {
    if (!h) return hfail(KVIDX_EINVAL, "bad arguments");
    std::vector<kvhost_pod_row_t> rows(KVIDX_MAX_PODS);
    const char* tier[KVIDX_MAX_TIERS];
    uint64_t totals[4];
    const int64_t n = kvhost_pod_inventory(h, nullptr, 1, rows.data(), rows.size(), tier, totals);
    if (n < 0) return n;
    auto label = [](const char* v) {                             // label value escaping of the text format
        std::string o;
        for (; *v; ++v) { if (*v == '\\' || *v == '"') o += '\\'; if (*v == '\n') { o += "\\n"; continue; } o += *v; }
        return o;
    };
    std::string s;
    auto gauge = [&](const char* name, const char* help) {
        s += "# HELP kvcache_index_"; s += name; s += " "; s += help; s += "\n# TYPE kvcache_index_"; s += name; s += " gauge\n";
    };
    gauge("pod_entries", "Request keys the index holds for a pod on a device tier");
    for (int64_t i = 0; i < n; ++i)
        for (uint32_t t = 0; t < KVIDX_MAX_TIERS; ++t)
            if (rows[i].entries[t])
                s += "kvcache_index_pod_entries{pod=\"" + label(rows[i].pod) + "\",tier=\"" + (tier[t] ? label(tier[t]) : std::to_string(t)) + "\"} " +
                     std::to_string(rows[i].entries[t]) + "\n";
    auto per_pod = [&](const char* name, const char* help, uint64_t kvhost_pod_row_t::*field) {
        gauge(name, help);
        for (int64_t i = 0; i < n; ++i)
            s += std::string("kvcache_index_") + name + "{pod=\"" + label(rows[i].pod) + "\"} " + std::to_string(rows[i].*field) + "\n";
    };
    per_pod("pod_keys", "Request keys with an entry of the pod on any tier", &kvhost_pod_row_t::keys);
    per_pod("pod_sole_keys", "Request keys held by the pod alone (removed with it)", &kvhost_pod_row_t::sole_keys);
    per_pod("pod_sole_engine_keys", "Engine-key mappings of the request keys held by the pod alone", &kvhost_pod_row_t::sole_engine_keys);
    gauge("stale_engine_keys", "Engine-key mappings whose request key is not resident");
    s += "kvcache_index_stale_engine_keys " + std::to_string(totals[3]) + "\n";
    if (buf && cap) { const size_t m = std::min(cap - 1, s.size()); memcpy(buf, s.data(), m); buf[m] = 0; }
    return (int64_t)s.size();
}

int64_t kvhost_decode_event_batch(kvhost_t* h, const char* pod, const char* model, const void* payload, size_t len, kvidx_event_t* ev_out,
                                  size_t ev_cap, uint64_t* hash_out, size_t hash_cap, size_t* n_hash_out, uint32_t* tok_out, size_t tok_cap,
                                  size_t* n_tok_out) {
    if (!h || !pod || !model) return hfail(KVIDX_EINVAL, "bad arguments");
    std::vector<kvidx_event_t> evs; std::vector<uint64_t> hashes; std::vector<uint32_t> toks;
    {
        std::lock_guard<std::mutex> g(h->mu);
        const int p = h->pods.id(pod, h->pod_cap), m = h->models.id(model, 65536);
        if (p < 0 || m < 0) return hfail(KVIDX_ERANGE, "pod / model id space exhausted");
        decode_batch(h, (uint32_t)p, (uint32_t)m, (const uint8_t*)payload, len, evs, hashes, toks);
    }
    if (evs.size() > ev_cap || hashes.size() > hash_cap || toks.size() > tok_cap) return hfail(KVIDX_ENOSPC, "output buffers too small");
    if (!evs.empty()) memcpy(ev_out, evs.data(), evs.size() * sizeof(kvidx_event_t));
    if (!hashes.empty()) memcpy(hash_out, hashes.data(), hashes.size() * 8);
    if (!toks.empty()) memcpy(tok_out, toks.data(), toks.size() * 4);
    if (n_hash_out) *n_hash_out = hashes.size();
    if (n_tok_out) *n_tok_out = toks.size();
    return (int64_t)evs.size();
}

}  // extern "C"

// ---- tokenization prefix store (prefixstore/lru_store.go) -------------------------------------------------------------
namespace {
constexpr uint64_t XP1 = 0x9E3779B185EBCA87ull, XP2 = 0xC2B2AE3D27D4EB4Full, XP3 = 0x165667B19E3779F9ull, XP4 = 0x85EBCA77C2B2AE63ull,
                   XP5 = 0x27D4EB2F165667C5ull;
inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
inline uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }      // little-endian hosts only (x86-64, aarch64)
inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint64_t xx_round(uint64_t acc, uint64_t in) { return rotl64(acc + in * XP2, 31) * XP1; }
inline uint64_t xx_merge(uint64_t h, uint64_t v) { return (h ^ xx_round(0, v)) * XP1 + XP4; }

// XXH64 as published (cespare/xxhash/v2 in the reference's go.mod); fed in two pieces (the 8-byte chain prefix, then the block)
uint64_t xxh64(const uint8_t* p, size_t n, uint64_t seed) {
    const uint8_t* e = p + n;
    uint64_t h;
    if (n >= 32) {
        uint64_t v1 = seed + XP1 + XP2, v2 = seed + XP2, v3 = seed, v4 = seed - XP1;
        for (; p + 32 <= e; p += 32) { v1 = xx_round(v1, rd64(p)); v2 = xx_round(v2, rd64(p + 8)); v3 = xx_round(v3, rd64(p + 16)); v4 = xx_round(v4, rd64(p + 24)); }
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = xx_merge(h, v1); h = xx_merge(h, v2); h = xx_merge(h, v3); h = xx_merge(h, v4);
    } else h = seed + XP5;
    h += (uint64_t)n;
    for (; p + 8 <= e; p += 8) h = rotl64(h ^ xx_round(0, rd64(p)), 27) * XP1 + XP4;
    if (p + 4 <= e) { h = rotl64(h ^ ((uint64_t)rd32(p) * XP1), 23) * XP2 + XP3; p += 4; }
    for (; p < e; ++p) h = rotl64(h ^ ((uint64_t)*p * XP5), 11) * XP1;
    h ^= h >> 33; h *= XP2; h ^= h >> 29; h *= XP3; h ^= h >> 32;
    return h;
}
}  // namespace

struct kvhost_prefix_store {
    int64_t cache_size; int32_t block_size;
    std::mutex mu;
    // golang-lru semantics: Add inserts at the front (or updates and refreshes), evicts the back beyond cache_size; Get refreshes
    std::list<std::pair<uint64_t, std::vector<uint32_t>>> order;
    std::unordered_map<uint64_t, std::list<std::pair<uint64_t, std::vector<uint32_t>>>::iterator> map;
    std::vector<uint8_t> scratch;

    uint64_t chain(uint64_t prev, const uint8_t* blk) {
        scratch.resize(8 + (size_t)block_size);
        memcpy(scratch.data(), &prev, 8);
        memcpy(scratch.data() + 8, blk, (size_t)block_size);
        return xxh64(scratch.data(), scratch.size(), 0);
    }
};

extern "C" {

uint64_t kvhost_xxhash64(const void* data, size_t len, uint64_t seed) { return xxh64((const uint8_t*)data, len, seed); }

int kvhost_prefix_store_create(int64_t cache_size, int32_t block_size, kvhost_prefix_store_t** out) {
    if (!out) return hfail(KVIDX_EINVAL, "bad arguments");
    if (cache_size <= 0) return hfail(KVIDX_EINVAL, "failed to initialize in-memory index: must provide a positive size");     // lru.New
    if (block_size <= 0) return hfail(KVIDX_EINVAL, "block size must be positive");
    auto* s = new kvhost_prefix_store();
    s->cache_size = cache_size; s->block_size = block_size;
    *out = s;
    return 0;
}

void kvhost_prefix_store_destroy(kvhost_prefix_store_t* s) { delete s; }

int64_t kvhost_prefix_store_len(kvhost_prefix_store_t* s) { if (!s) return KVIDX_EINVAL; std::lock_guard<std::mutex> g(s->mu); return (int64_t)s->map.size(); }

int kvhost_prefix_store_add(kvhost_prefix_store_t* s, const char* prompt, size_t prompt_len, const uint32_t* tokens, const uint64_t* offsets, size_t n_tokens) {
    if (!s || (prompt_len && !prompt) || (n_tokens && (!tokens || !offsets))) return hfail(KVIDX_EINVAL, "bad arguments");
    if (prompt_len == 0 || n_tokens == 0) return 0;                                  // lru_store.go:96-98
    std::lock_guard<std::mutex> g(s->mu);
    const size_t bs = (size_t)s->block_size;
    size_t it = 0;
    uint64_t prev = 0;
    for (size_t start = 0; start + bs <= prompt_len; start += bs) {                  // no partial blocks
        const size_t end = start + bs;
        prev = s->chain(prev, (const uint8_t*)prompt + start);
        std::vector<uint32_t> blk;
        for (; it < n_tokens && offsets[2 * it + 1] <= end; ++it) blk.push_back(tokens[it]);      // a token goes with the block its END falls in
        auto f = s->map.find(prev);
        if (f != s->map.end()) { f->second->second = std::move(blk); s->order.splice(s->order.begin(), s->order, f->second); }
        else {
            s->order.emplace_front(prev, std::move(blk));
            s->map[prev] = s->order.begin();
            if ((int64_t)s->map.size() > s->cache_size) { s->map.erase(s->order.back().first); s->order.pop_back(); }
        }
    }
    return 0;
}

int64_t kvhost_prefix_store_find(kvhost_prefix_store_t* s, const char* prompt, size_t prompt_len, uint32_t* tokens_out, size_t cap, double* ratio_out) {
    if (!s || (prompt_len && !prompt)) return hfail(KVIDX_EINVAL, "bad arguments");
    std::lock_guard<std::mutex> g(s->mu);
    const size_t bs = (size_t)s->block_size;
    uint64_t prev = 0;
    double ratio = 0.0;
    int64_t n = 0;
    for (size_t i = 0; i + bs <= prompt_len; i += bs) {
        prev = s->chain(prev, (const uint8_t*)prompt + i);
        auto f = s->map.find(prev);
        if (f == s->map.end()) break;                                                // early stop
        s->order.splice(s->order.begin(), s->order, f->second);                      // Get refreshes recency
        for (uint32_t t : f->second->second) { if (tokens_out && (size_t)n < cap) tokens_out[n] = t; ++n; }
        ratio = (double)(i + bs) / (double)prompt_len;
    }
    if (ratio_out) *ratio_out = ratio;
    return n;
}

int kvhost_prefix_store_snapshot(kvhost_prefix_store_t* s, void* buf, uint64_t cap, uint64_t* size_out) {
    if (!s || !size_out) return hfail(KVIDX_EINVAL, "bad arguments");
    std::lock_guard<std::mutex> g(s->mu);
    const uint64_t R = s->order.size();
    uint64_t T = 0;
    for (const auto& e : s->order) T += e.second.size();
    *size_out = 64 + 16 * R + 4 * T;
    if (!buf || cap < *size_out) return hfail(KVIDX_ENOSPC, "the prefix store image does not fit the buffer");
    uint8_t* p = static_cast<uint8_t*>(buf);
    memset(p, 0, 64);
    const uint32_t ver = 1, bb = (uint32_t)s->block_size;
    memcpy(p, "KVIDXTXT", 8); memcpy(p + 8, &ver, 4); memcpy(p + 16, &bb, 4); memcpy(p + 24, &R, 8); memcpy(p + 32, &T, 8);
    uint8_t* rec = p + 64;
    uint8_t* tok = rec + 16 * R;
    for (auto it = s->order.rbegin(); it != s->order.rend(); ++it) {        // least recent first
        const uint32_t nt = (uint32_t)it->second.size(), zero = 0;
        memcpy(rec, &it->first, 8); memcpy(rec + 8, &nt, 4); memcpy(rec + 12, &zero, 4);
        rec += 16;
        if (nt) memcpy(tok, it->second.data(), (size_t)nt * 4);
        tok += (size_t)nt * 4;
    }
    return 0;
}

int kvhost_prefix_store_restore(kvhost_prefix_store_t* s, const void* buf, uint64_t len) {
    if (!s || (!buf && len)) return hfail(KVIDX_EINVAL, "bad arguments");
    std::lock_guard<std::mutex> g(s->mu);
    if (!s->map.empty()) return hfail(KVIDX_EINVAL, "prefix store restore needs an empty store");
    if (len < 64) return hfail(KVIDX_EINVAL, "prefix store image: shorter than its header");
    const uint8_t* p = static_cast<const uint8_t*>(buf);
    uint32_t ver, flags, bb, z; uint64_t R, T;
    memcpy(&ver, p + 8, 4); memcpy(&flags, p + 12, 4); memcpy(&bb, p + 16, 4); memcpy(&z, p + 20, 4); memcpy(&R, p + 24, 8); memcpy(&T, p + 32, 8);
    if (memcmp(p, "KVIDXTXT", 8)) return hfail(KVIDX_EINVAL, "prefix store image: bad magic");
    if (ver != 1 || flags != 0) return hfail(KVIDX_EINVAL, "prefix store image: bad version or flags");
    bool zero = z == 0;
    for (int i = 40; i < 64; ++i) zero = zero && p[i] == 0;
    if (!zero) return hfail(KVIDX_EINVAL, "prefix store image: non-zero reserved header bytes");
    if (bb != (uint32_t)s->block_size) return hfail(KVIDX_EINVAL, "prefix store image: block_bytes differs from the store's");
    const uint64_t room = len - 64;
    if (R > room / 16 || T > room / 4 || 16 * R + 4 * T != room) return hfail(KVIDX_EINVAL, "prefix store image: length does not match the header");
    // every record checked before any is inserted
    const uint8_t* rec = p + 64;
    std::unordered_set<uint64_t> seen;
    uint64_t sum = 0;
    for (uint64_t i = 0; i < R; ++i) {
        uint64_t k; uint32_t nt, pad;
        memcpy(&k, rec + 16 * i, 8); memcpy(&nt, rec + 16 * i + 8, 4); memcpy(&pad, rec + 16 * i + 12, 4);
        if (pad) return hfail(KVIDX_EINVAL, "prefix store image: non-zero record padding");
        if (!seen.insert(k).second) return hfail(KVIDX_EINVAL, "prefix store image: a key appears twice");
        sum += nt;
    }
    if (sum != T) return hfail(KVIDX_EINVAL, "prefix store image: the records' token counts do not add up to the header's");
    // the replay of the records as adds, oldest first, leaves the newest cache_size of them
    const uint8_t* tok = rec + 16 * R;
    const uint64_t first = R > (uint64_t)s->cache_size ? R - (uint64_t)s->cache_size : 0;
    for (uint64_t i = 0; i < R; ++i) {
        uint64_t k; uint32_t nt;
        memcpy(&k, rec + 16 * i, 8); memcpy(&nt, rec + 16 * i + 8, 4);
        if (i >= first) {
            std::vector<uint32_t> blk(nt);
            if (nt) memcpy(blk.data(), tok, (size_t)nt * 4);
            s->order.emplace_front(k, std::move(blk));
            s->map[k] = s->order.begin();
        }
        tok += (size_t)nt * 4;
    }
    return 0;
}

}  // extern "C"
