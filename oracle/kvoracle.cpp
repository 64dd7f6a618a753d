// kvoracle.cpp -- fast CPU restatement of the reference's Go path (C++17, no GPU).
//
// TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may load the library built from this file.
// The product (libkvidx) never links or calls it.
//
// It mirrors the *structure* of the Go implementation so that it is a fair CPU
// baseline (kind "port"): map + doubly linked list LRUs behind one mutex each
// (hashicorp/golang-lru/v2 v2.0.7), a per-key pod LRU behind its own mutex, a
// Lookup that materialises map[Key][]PodEntry and a scorer that walks it with
// per-key pod sets.  It is deliberately allocation-light where Go is not
// (no reflection-based CBOR encoder), i.e. it is a *stronger* baseline than the
// real Go path.
//
// PARITY STATUS: hash values are "parity unpinned" against Go (see kvoracle.py
// header); this file is pinned against kvoracle.py and tests/golden/*.json.
//
// Reference citations are path:line under the reference root.

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <list>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../include/kvidx.h"

namespace {

constexpr uint64_t kFnvOffset = 0xCBF29CE484222325ull;
constexpr uint64_t kFnvPrime = 0x100000001B3ull;

inline uint64_t fnv_byte(uint64_t h, uint8_t b) { return (h ^ b) * kFnvPrime; }

// RFC 7049 shortest-form head, hashed on the fly (fxamacker/cbor CanonicalEncOptions).
inline uint64_t fnv_cbor_head(uint64_t h, uint8_t major, uint64_t v) {
    const uint8_t m = uint8_t(major << 5);
    if (v < 24) return fnv_byte(h, m | uint8_t(v));
    int nb;
    if (v < (1ull << 8)) { h = fnv_byte(h, m | 24); nb = 1; }
    else if (v < (1ull << 16)) { h = fnv_byte(h, m | 25); nb = 2; }
    else if (v < (1ull << 32)) { h = fnv_byte(h, m | 26); nb = 4; }
    else { h = fnv_byte(h, m | 27); nb = 8; }
    for (int i = nb - 1; i >= 0; --i) h = fnv_byte(h, uint8_t(v >> (8 * i)));
    return h;
}

// ChunkedTokenDatabase.hash (token_processor.go:94-112): FNV-64a(CBOR([parent, tokens, nil])).
inline uint64_t block_hash(uint64_t parent, const uint32_t* tok, uint32_t bs) {
    uint64_t h = kFnvOffset;
    h = fnv_byte(h, 0x83);
    h = fnv_cbor_head(h, 0, parent);
    h = fnv_cbor_head(h, 4, bs);
    for (uint32_t i = 0; i < bs; ++i) h = fnv_cbor_head(h, 0, tok[i]);
    return fnv_byte(h, 0xf6);
}

struct Key {
    uint32_t model;
    uint64_t hash;
    bool operator==(const Key& o) const { return model == o.model && hash == o.hash; }
};
struct KeyHash {
    size_t operator()(const Key& k) const {
        uint64_t x = k.hash ^ (uint64_t(k.model) * 0x9E3779B97F4A7C15ull);
        x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33;
        return size_t(x);
    }
};

// hashicorp/golang-lru/v2 Cache: simplelru (map + list) behind one mutex.
template <class K, class V, class H>
class Lru {
public:
    explicit Lru(size_t cap) : cap_(cap) {}
    // Add: update + refresh if present, else push front and evict the back when over size.
    void add(const K& k, const V& v) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = map_.find(k);
        if (it != map_.end()) { it->second->second = v; list_.splice(list_.begin(), list_, it->second); return; }
        list_.emplace_front(k, v);
        map_[k] = list_.begin();
        if (map_.size() > cap_) { auto last = std::prev(list_.end()); map_.erase(last->first); list_.pop_back(); }
    }
    bool get(const K& k, V* out) {   // Get refreshes recency
        std::lock_guard<std::mutex> g(mu_);
        auto it = map_.find(k);
        if (it == map_.end()) return false;
        list_.splice(list_.begin(), list_, it->second);
        if (out) *out = it->second->second;
        return true;
    }
    bool peek(const K& k, V* out) {   // Peek: no refresh
        std::lock_guard<std::mutex> g(mu_);
        auto it = map_.find(k);
        if (it == map_.end()) return false;
        *out = it->second->second;
        return true;
    }
    bool contains_or_add(const K& k, const V& v) {   // no refresh on hit
        std::lock_guard<std::mutex> g(mu_);
        if (map_.count(k)) return true;
        list_.emplace_front(k, v);
        map_[k] = list_.begin();
        if (map_.size() > cap_) { auto last = std::prev(list_.end()); map_.erase(last->first); list_.pop_back(); }
        return false;
    }
    bool remove(const K& k) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = map_.find(k);
        if (it == map_.end()) return false;
        list_.erase(it->second); map_.erase(it);
        return true;
    }
    size_t len() { std::lock_guard<std::mutex> g(mu_); return map_.size(); }
    template <class F> void keys_oldest_first(F f) {   // Keys(): oldest -> newest
        std::lock_guard<std::mutex> g(mu_);
        for (auto it = list_.rbegin(); it != list_.rend(); ++it) f(it->first);
    }
    template <class F> void items_oldest_first(F f) {   // (key, value), oldest -> newest
        std::lock_guard<std::mutex> g(mu_);
        for (auto it = list_.rbegin(); it != list_.rend(); ++it) f(it->first, it->second);
    }
private:
    size_t cap_;
    std::mutex mu_;
    std::list<std::pair<K, V>> list_;
    std::unordered_map<K, typename std::list<std::pair<K, V>>::iterator, H> map_;
};

struct PtHash { size_t operator()(uint16_t v) const { return v; } };
struct Empty {};
struct PodCache {                       // in_memory.go:89-95
    explicit PodCache(size_t cap) : cache(cap) {}
    Lru<uint16_t, Empty, PtHash> cache;
    std::mutex mu;
};
using PodCachePtr = std::shared_ptr<PodCache>;

struct Oracle {
    uint32_t block_size;
    uint64_t init_hash;
    size_t pod_cache_size;
    double weight[KVIDX_MAX_TIERS];
    Lru<Key, PodCachePtr, KeyHash> data;          // in_memory.go:80
    Lru<Key, Key, KeyHash> engine_to_request;     // in_memory.go:82
    Oracle(uint32_t bs, uint64_t ih, size_t size, size_t pcs)
        : block_size(bs), init_hash(ih), pod_cache_size(pcs), data(size), engine_to_request(size) {
        for (auto& w : weight) w = 1.0;
    }

    // TokensToKVBlockKeys (token_processor.go:141-162)
    void keys_for(const uint32_t* tok, int64_t n_tok, uint64_t parent, std::vector<uint64_t>& out) const {
        out.clear();
        for (int64_t i = 0; i + block_size <= n_tok; i += block_size) {
            parent = block_hash(parent, tok + i, block_size);
            out.push_back(parent);
        }
    }

    using HitMap = std::unordered_map<Key, std::vector<uint16_t>, KeyHash>;

    // Lookup (in_memory.go:105-146). filter == nullptr or empty -> all pods.
    int lookup(const std::vector<Key>& keys, const std::unordered_set<uint32_t>* filter, HitMap& out) {
        if (keys.empty()) return KVIDX_EINVAL;
        for (const Key& k : keys) {
            PodCachePtr pc;
            if (data.get(k, &pc)) {
                if (!pc || pc->cache.len() == 0) return 0;            // :119-122 cut
                if (!filter || filter->empty()) {
                    auto& v = out[k];
                    v.clear();                                        // :128 assigns (a repeated key overwrites)
                    pc->cache.keys_oldest_first([&](uint16_t e) { v.push_back(e); });
                } else {
                    pc->cache.keys_oldest_first([&](uint16_t e) {       // :130-135 appends (a repeated key accumulates)
                        if (filter->count(KVIDX_PT_POD(e))) out[k].push_back(e);
                    });
                }
            }
        }
        return 0;
    }

    // Add (in_memory.go:149-209)
    int add(uint32_t model, const uint64_t* engine, const uint64_t* request, int64_t n_e, int64_t n_r,
            const uint16_t* ent, int m) {
        if (n_e == 0 || n_r == 0 || m == 0) return KVIDX_EINVAL;
        if (n_e != n_r) return KVIDX_EINVAL;
        for (int64_t i = 0; i < n_r; ++i) {
            Key rk{model, request[i]}, ek{model, engine[i]};
            engine_to_request.add(ek, rk);
            PodCachePtr pc;
            if (!data.get(rk, &pc)) {
                auto npc = std::make_shared<PodCache>(pod_cache_size);
                if (data.contains_or_add(rk, npc)) {
                    if (!data.get(rk, &pc)) { data.add(rk, npc); pc = npc; }
                } else pc = npc;
            }
            std::lock_guard<std::mutex> g(pc->mu);
            for (int j = 0; j < m; ++j) pc->cache.add(ent[j], Empty{});
        }
        return 0;
    }

    // Evict (in_memory.go:212-260)
    int evict(uint32_t model, uint64_t engine, const uint16_t* ent, int m) {
        if (m == 0) return KVIDX_EINVAL;
        Key ek{model, engine}, rk{};
        if (!engine_to_request.get(ek, &rk)) return 0;
        PodCachePtr pc;
        if (!data.get(rk, &pc) || !pc) { engine_to_request.remove(ek); return 0; }
        bool empty;
        {
            std::lock_guard<std::mutex> g(pc->mu);
            for (int j = 0; j < m; ++j) pc->cache.remove(ent[j]);
            empty = pc->cache.len() == 0;
        }
        if (empty) {
            PodCachePtr cur;
            if (data.get(rk, &cur) && cur) {
                bool still;
                { std::lock_guard<std::mutex> g(cur->mu); still = cur->cache.len() == 0; }
                if (still) { data.remove(rk); engine_to_request.remove(ek); }
            }
        }
        return 0;
    }

    // getMaxWeight (kvblock_scorer.go:89-105)
    double max_weight(const std::vector<uint16_t>& ents, uint32_t pod) const {
        double mx = 0.0;
        for (uint16_t e : ents)
            if (KVIDX_PT_POD(e) == pod) { double w = weight[KVIDX_PT_TIER(e)]; if (w > mx) mx = w; }
        return mx;
    }

    // LongestPrefixScorer.Score (kvblock_scorer.go:108-151)
    void score(const std::vector<Key>& keys, const HitMap& hits, std::unordered_map<uint32_t, double>& out) const {
        out.clear();
        if (keys.empty()) return;
        static const std::vector<uint16_t> none;
        auto get = [&](const Key& k) -> const std::vector<uint16_t>& {
            auto it = hits.find(k); return it == hits.end() ? none : it->second;
        };
        const auto& first = get(keys[0]);
        std::unordered_set<uint32_t> active;
        for (uint16_t e : first) active.insert(KVIDX_PT_POD(e));
        for (uint32_t p : active) out[p] = max_weight(first, p);
        for (size_t i = 1; i < keys.size(); ++i) {
            if (active.empty()) break;
            const auto& cur = get(keys[i]);
            std::unordered_set<uint32_t> cs;
            for (uint16_t e : cur) cs.insert(KVIDX_PT_POD(e));
            std::unordered_set<uint32_t> inter;
            for (uint32_t p : active) if (cs.count(p)) inter.insert(p);
            active.swap(inter);
            for (uint32_t p : active) out[p] += max_weight(cur, p);   // in-order f64 add
        }
    }

    // GetPodScores steps 2-4 (indexer.go:141-163). Returns 0 keys -> has_keys=0.
    int get_pod_scores(const uint32_t* tok, int64_t n_tok, uint32_t model, const std::unordered_set<uint32_t>* filter,
                       std::unordered_map<uint32_t, double>& out, bool* has_keys) {
        std::vector<uint64_t> hs;
        keys_for(tok, n_tok, init_hash, hs);
        out.clear();
        *has_keys = !hs.empty();
        if (hs.empty()) return 0;
        std::vector<Key> keys(hs.size());
        for (size_t i = 0; i < hs.size(); ++i) keys[i] = Key{model, hs[i]};
        HitMap hits;
        int rc = lookup(keys, filter, hits);
        if (rc) return rc;
        score(keys, hits, out);
        return 0;
    }

    // digestEvents for one decoded event (kvevents/pool.go:246-338)
    bool apply_event(const kvidx_event_t& ev, const uint64_t* hashes, const uint32_t* tokens) {
        const uint16_t ent = ev.podtier;
        if (ev.op == KVIDX_EV_BLOCK_STORED) {
            uint64_t parent = init_hash;
            if (ev.has_parent) {
                Key rk{};
                if (engine_to_request.get(Key{ev.model, ev.parent_hash}, &rk)) parent = rk.hash;   // miss -> seed
            }
            std::vector<uint64_t> req;
            keys_for(tokens + ev.tok_off, ev.n_tokens, parent, req);
            if (ev.n_hashes > 0) {
                int rc = add(ev.model, hashes + ev.hash_off, req.data(), ev.n_hashes, (int64_t)req.size(), &ent, 1);
                return rc == 0;
            }
            return true;
        }
        if (ev.op == KVIDX_EV_BLOCK_REMOVED) {
            for (uint32_t i = 0; i < ev.n_hashes; ++i) evict(ev.model, hashes[ev.hash_off + i], &ent, 1);
        }
        return true;
    }
};

inline std::unordered_set<uint32_t> filter_from_mask(const uint64_t* mask, uint32_t words) {
    std::unordered_set<uint32_t> s;
    if (!mask) return s;
    for (uint32_t w = 0; w < words; ++w)
        for (int b = 0; b < 64; ++b) if ((mask[w] >> b) & 1) s.insert(w * 64 + b);
    return s;
}

}  // namespace

extern "C" {

void* ko_create(uint32_t block_size, uint64_t init_hash, uint64_t size, uint32_t pod_cache_size) {
    if (size == 0 || pod_cache_size == 0) return nullptr;     // lru.New(size<=0) errors
    return new Oracle(block_size ? block_size : 16, init_hash, size, pod_cache_size);
}
void ko_destroy(void* h) { delete static_cast<Oracle*>(h); }
void ko_set_tier_weight(void* h, uint32_t tier, double w) { static_cast<Oracle*>(h)->weight[tier & 15] = w; }
uint64_t ko_fnv64a(const uint8_t* p, size_t n) { uint64_t h = kFnvOffset; for (size_t i = 0; i < n; ++i) h = fnv_byte(h, p[i]); return h; }
uint64_t ko_block_hash(uint64_t parent, const uint32_t* tok, uint32_t bs) { return block_hash(parent, tok, bs); }

// keys for a CSR batch; returns number of keys written. key_off[n_prompts+1] filled.
int64_t ko_hash_keys(void* h, const uint32_t* tok, const int64_t* tok_off, int64_t n_prompts,
                     const uint64_t* parent, const uint8_t* parent_valid, uint64_t* keys_out, int64_t* key_off) {
    auto* o = static_cast<Oracle*>(h);
    std::vector<uint64_t> hs;
    int64_t w = 0;
    for (int64_t i = 0; i < n_prompts; ++i) {
        uint64_t p = o->init_hash;
        if (parent && (!parent_valid || parent_valid[i])) p = parent[i];
        o->keys_for(tok + tok_off[i], tok_off[i + 1] - tok_off[i], p, hs);
        key_off[i] = w;
        for (uint64_t k : hs) keys_out[w++] = k;
    }
    key_off[n_prompts] = w;
    return w;
}

int ko_add(void* h, uint32_t model, const uint64_t* engine, const uint64_t* request, int64_t n_e, int64_t n_r,
           const uint16_t* ent, int m) { return static_cast<Oracle*>(h)->add(model, engine, request, n_e, n_r, ent, m); }
int ko_evict(void* h, uint32_t model, uint64_t engine, const uint16_t* ent, int m) { return static_cast<Oracle*>(h)->evict(model, engine, ent, m); }
int ko_get_request_key(void* h, uint32_t model, uint64_t engine, uint64_t* out) {
    Key rk{};
    if (!static_cast<Oracle*>(h)->engine_to_request.get(Key{model, engine}, &rk)) return KVIDX_ENOENT;
    *out = rk.hash; return 0;
}
// GetRequestKey without the recency refresh: what a BlockStored event's parent lookup would find now.
int ko_peek_request_key(void* h, uint32_t model, uint64_t engine, uint64_t* out) {
    Key rk{};
    if (!static_cast<Oracle*>(h)->engine_to_request.peek(Key{model, engine}, &rk)) return KVIDX_ENOENT;
    *out = rk.hash; return 0;
}
uint64_t ko_len_request(void* h) { return static_cast<Oracle*>(h)->data.len(); }
uint64_t ko_len_engine(void* h) { return static_cast<Oracle*>(h)->engine_to_request.len(); }

// Lookup with the kvidx_lookup output convention.
int ko_lookup(void* h, uint32_t model, const uint64_t* keys, int64_t n, const uint64_t* filter, uint32_t filter_words,
              uint16_t* podtier_out, uint8_t* cnt_out) {
    auto* o = static_cast<Oracle*>(h);
    std::vector<Key> ks(n);
    for (int64_t i = 0; i < n; ++i) ks[i] = Key{model, keys[i]};
    auto fs = filter_from_mask(filter, filter_words);
    Oracle::HitMap hits;
    int rc = o->lookup(ks, filter ? &fs : nullptr, hits);
    if (rc) return rc;
    for (int64_t i = 0; i < n; ++i) {
        auto it = hits.find(ks[i]);
        cnt_out[i] = 0;
        if (it == hits.end()) continue;
        cnt_out[i] = (uint8_t)it->second.size();
        for (size_t j = 0; j < it->second.size() && j < KVIDX_MAX_PODS_PER_KEY; ++j) podtier_out[i * KVIDX_MAX_PODS_PER_KEY + j] = it->second[j];
    }
    return 0;
}

// GetPodScores for a CSR batch on n_threads OS threads (== concurrent goroutines calling
// Indexer.GetPodScores).  Dense rows of max_pods doubles, KVIDX_SCORE_ABSENT = not in map.
// lat_ns_out (nullable): per-prompt latency in ns.  Returns elapsed seconds via *elapsed_out.
int ko_score_batch(void* h, const uint32_t* tok, const int64_t* tok_off, int64_t n_prompts, const uint32_t* model,
                   uint32_t model0, const uint64_t* filter, uint32_t filter_words, uint32_t max_pods, int n_threads,
                   double* scores_out, uint8_t* has_keys_out, double* elapsed_out, int64_t* lat_ns_out) {
    auto* o = static_cast<Oracle*>(h);
    if (n_threads < 1) n_threads = 1;
    std::atomic<int64_t> next{0};
    std::atomic<int> err{0};
    auto t0 = std::chrono::steady_clock::now();
    auto work = [&]() {
        std::unordered_map<uint32_t, double> sc;
        for (;;) {
            int64_t i = next.fetch_add(1);
            if (i >= n_prompts) break;
            auto a = std::chrono::steady_clock::now();
            std::unordered_set<uint32_t> fs;
            if (filter) fs = filter_from_mask(filter + i * filter_words, filter_words);
            bool hk = false;
            int rc = o->get_pod_scores(tok + tok_off[i], tok_off[i + 1] - tok_off[i], model ? model[i] : model0,
                                       filter ? &fs : nullptr, sc, &hk);
            if (rc) err.store(rc);
            if (has_keys_out) has_keys_out[i] = hk;
            if (scores_out) {
                double* row = scores_out + i * (int64_t)max_pods;
                for (uint32_t p = 0; p < max_pods; ++p) row[p] = KVIDX_SCORE_ABSENT;
                for (auto& kv : sc) if (kv.first < max_pods) row[kv.first] = kv.second;
            }
            if (lat_ns_out) lat_ns_out[i] = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - a).count();
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; ++t) th.emplace_back(work);
    work();
    for (auto& t : th) t.join();
    if (elapsed_out) *elapsed_out = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return err.load();
}

// Apply events in array order (a valid schedule of the reference's per-pod FIFO queues).
int ko_apply_events(void* h, const kvidx_event_t* ev, int64_t n, const uint64_t* hashes, const uint32_t* tokens, int64_t* n_dropped) {
    auto* o = static_cast<Oracle*>(h);
    int64_t dropped = 0;
    for (int64_t i = 0; i < n; ++i) if (!o->apply_event(ev[i], hashes, tokens)) ++dropped;
    if (n_dropped) *n_dropped = dropped;
    return 0;
}

// The v1 index image (include/kvidx.h) of the oracle's contents: request records sorted by (model, hash) with their
// entries oldest -> newest, engine records sorted by (model, engine hash), stale mappings included.  With recency, one
// u64 per record: its 1-based position in its LRU (oldest = 1).  Returns the image size; writes nothing unless
// cap >= size.  Refreshes no recency.
int64_t ko_snapshot(void* h, int recency, uint8_t* buf, uint64_t cap) {
    auto* o = static_cast<Oracle*>(h);
    struct Req { uint32_t model; uint64_t hash; std::vector<uint16_t> ent; uint64_t rank; };
    struct Eng { uint32_t model; uint64_t hash, request; uint64_t rank; };
    std::vector<Req> reqs;
    std::vector<Eng> engs;
    o->data.items_oldest_first([&](const Key& k, const PodCachePtr& pc) {
        Req r{k.model, k.hash, {}, reqs.size() + 1};
        pc->cache.keys_oldest_first([&](uint16_t e) { r.ent.push_back(e); });
        reqs.push_back(std::move(r));
    });
    o->engine_to_request.items_oldest_first([&](const Key& ek, const Key& rk) {
        engs.push_back(Eng{ek.model, ek.hash, rk.hash, engs.size() + 1});
    });
    std::sort(reqs.begin(), reqs.end(), [](const Req& a, const Req& b) { return a.model != b.model ? a.model < b.model : a.hash < b.hash; });
    std::sort(engs.begin(), engs.end(), [](const Eng& a, const Eng& b) { return a.model != b.model ? a.model < b.model : a.hash < b.hash; });
    uint32_t pod_span = 0, model_span = 0;
    for (const Req& r : reqs) {
        model_span = std::max(model_span, r.model + 1);
        for (uint16_t e : r.ent) pod_span = std::max<uint32_t>(pod_span, KVIDX_PT_POD(e) + 1u);
    }
    for (const Eng& e : engs) model_span = std::max(model_span, e.model + 1);
    const uint64_t R = reqs.size(), E = engs.size();
    const uint64_t size = 64 + 32 * R + 24 * E + (recency ? 8 * (R + E) : 0);
    if (!buf || cap < size) return (int64_t)size;
    std::memset(buf, 0, size);
    auto put = [&](uint64_t off, const void* p, size_t n) { std::memcpy(buf + off, p, n); };
    const uint32_t version = 1, flags = recency ? 1u : 0u, bs = o->block_size, ppk = (uint32_t)o->pod_cache_size;
    put(0, "KVIDXSNP", 8); put(8, &version, 4); put(12, &flags, 4); put(16, &bs, 4); put(20, &ppk, 4);
    put(24, &o->init_hash, 8); put(32, &R, 8); put(40, &E, 8); put(48, &pod_span, 4); put(52, &model_span, 4);
    uint64_t off = 64;
    for (const Req& r : reqs) {
        const uint16_t model = (uint16_t)r.model;
        const uint8_t cnt = (uint8_t)r.ent.size();
        put(off, &r.hash, 8); put(off + 8, &model, 2); put(off + 10, &cnt, 1);
        for (size_t j = 0; j < r.ent.size() && j < KVIDX_MAX_PODS_PER_KEY; ++j) put(off + 12 + 2 * j, &r.ent[j], 2);
        off += 32;
    }
    for (const Eng& e : engs) {
        const uint16_t model = (uint16_t)e.model;
        put(off, &e.hash, 8); put(off + 8, &e.request, 8); put(off + 16, &model, 2);
        off += 24;
    }
    if (recency) {
        for (const Req& r : reqs) { put(off, &r.rank, 8); off += 8; }
        for (const Eng& e : engs) { put(off, &e.rank, 8); off += 8; }
    }
    return (int64_t)size;
}

}  // extern "C"
