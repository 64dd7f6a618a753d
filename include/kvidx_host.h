/*
 * kvidx_host.h -- string-level host mirror of the reference's Go interfaces for the hot path, in C++ behind a C ABI.
 *
 * The reference's host code is Go (kvcache.Indexer, kvblock.Index, kvevents.Pool); Go is not available in this build
 * image, so the layer a Go shim would provide -- string interning, the per-pod sharded event queues and the msgpack
 * decoding of KVEvents -- is provided here in C++ over libkvidx's id-level ABI (kvidx.h), with the same names, argument
 * meaning and error behaviour.  The decoder is pure host code and works without a GPU (tests/test_host_decode.py).
 *
 *   kvhost_create            <-> kvcache.NewKVCacheIndexer            pkg/kvcache/indexer.go:75-113
 *   kvhost_get_pod_scores    <-> Indexer.GetPodScores (steps 2-4)     pkg/kvcache/indexer.go:132-166
 *   kvhost_get_pod_scores_keys <-> GetPodScores steps 3-4 (from keys)  pkg/kvcache/indexer.go:150-159
 *   kvhost_index_*           <-> kvblock.Index Add/Evict/Lookup/GetRequestKey   pkg/kvcache/kvblock/index.go:119-135
 *   kvhost_pool_add_task     <-> kvevents.Pool.AddTask                pkg/kvcache/kvevents/pool.go:132-144
 *   kvhost_pool_process      <-> worker loop: processEvent + digestEvents       pkg/kvcache/kvevents/pool.go:149-338
 *   kvhost_decode_event_batch<-> processEvent's msgpack decoding      pkg/kvcache/kvevents/pool.go:177-244, events.go:38-96
 *   kvhost_remove_pod        <-> (no counterpart) drop a departed pod's entries and free its id (kvidx_remove_pods)
 *   kvhost_snapshot / _restore <-> (no counterpart) names + index image, warm start of a fresh mirror (kvidx_snapshot)
 *   kvhost_pod_inventory / kvhost_inventory_text <-> (no counterpart) what each pod holds, by name (kvidx_pod_inventory)
 *   kvhost_prefix_store_*    <-> prefixstore.LRUTokenStore            pkg/tokenization/prefixstore/lru_store.go:54-190
 *   kvhost_get_metrics / _text <-> InstrumentedIndex + collectors      pkg/kvcache/kvblock/instrumented_index.go:30-92, metrics/collector.go:28-59
 */
#ifndef KVIDX_HOST_H
#define KVIDX_HOST_H
#include "kvidx.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct kvhost kvhost_t;

typedef struct kvhost_config {
    kvidx_config_t index;            /* device index (tier weights are taken from tier_names / tier_weights below)      */
    uint32_t concurrency;            /* kvevents.Config.Concurrency (default 4): number of FNV-32a(pod) sharded queues  */
    uint32_t n_tiers;                /* KVCacheBackendConfig list: names[i] scores weights[i]; ids follow this order     */
    const char* tier_names[KVIDX_MAX_TIERS];
    double tier_weights[KVIDX_MAX_TIERS];
    int32_t no_device;               /* 1: host-only instance (interners, queues, decoder) without a kvidx handle       */
    int32_t enable_metrics;          /* IndexConfig.EnableMetrics (index.go:41-43): wrap the index in the instrumented one */
    int32_t clear_on_all_blocks_cleared; /* 1: an AllBlocksCleared from pod P removes P's entries on the tier of a
                                            Medium-less event ("gpu", pool.go:258-261) at its position in P's event order
                                            (vLLM sends it when the GPU prefix cache is reset; offloaded blocks survive).
                                            0 (default): a no-op, as in the reference (pool.go:332-333). */
} kvhost_config_t;

void kvhost_config_default(kvhost_config_t* cfg);       /* block 16, seed "", gpu 1.0 / cpu 0.8, concurrency 4 */
int  kvhost_create(const kvhost_config_t* cfg, const char* hash_seed, kvhost_t** out);
void kvhost_destroy(kvhost_t* h);
const char* kvhost_last_error(void);
kvidx_t* kvhost_index(kvhost_t* h);                      /* Indexer.KVBlockIndex(), indexer.go:121-123 */

/* Indexer.GetPodScores after tokenisation.  pods[n_pods] is the filter (n_pods == 0: all pods).  Results: up to 10
 * (pod name, score) pairs; the name pointers stay valid for the life of the handle.  Returns the number of pairs,
 * -1000 for "no full block" (the reference's (nil, nil)), or a negative KVIDX_E* code. */
int kvhost_get_pod_scores(kvhost_t* h, const uint32_t* tokens, size_t n_tokens, const char* model,
                          const char* const* pods, size_t n_pods, const char** pod_out, double* score_out);

/* Indexer.GetPodScores after step 2 (indexer.go:150-159): the prompt's request keys in block order instead of its tokens
 * (kvidx_score_keys).  Same filter, results and return values as kvhost_get_pod_scores; -1000 when n_keys == 0. */
int kvhost_get_pod_scores_keys(kvhost_t* h, const uint64_t* keys, size_t n_keys, const char* model,
                               const char* const* pods, size_t n_pods, const char** pod_out, double* score_out);

/* Indexer.GetPodScores for a conversation turn (kvidx_score_turn): the request keys held from earlier turns, then the new
 * turn's tokens, hashed from the last held key.  new_keys_out (may be NULL) receives the floor(n_tokens / B) new keys.  Same
 * filter, results and return values as kvhost_get_pod_scores; -1000 when there is no key at all.  With enable_metrics it
 * counts one Lookup over the held and the new keys. */
int kvhost_get_pod_scores_turn(kvhost_t* h, const uint64_t* keys, size_t n_keys, const uint32_t* tokens, size_t n_tokens,
                               const char* model, const char* const* pods, size_t n_pods, const char** pod_out, double* score_out,
                               uint64_t* new_keys_out);

/* GetPodScores for a batch of prompts (model and pod filter shared by the batch), read_mu held from the filter to the pod
 * names as in kvhost_get_pod_scores.  Results: pod_out / score_out hold n * KVIDX_MAX_PODS_PER_KEY entries, prompt i's at
 * i * KVIDX_MAX_PODS_PER_KEY; cnt_out[i] = its entry count, or -1 for (nil, nil) (no full block).  With enable_metrics each
 * scored prompt counts one Lookup, as kvhost_get_pod_scores does.
 * kvhost_get_pod_scores_text: prompt i is text[text_off[i] .. text_off[i+1]), looked up in the device prefix store of the
 *   index (kvidx_text_store_init on kvhost_index(h) first) and scored by kvidx_score_text_sparse: a prompt whose cached
 *   prefix covers less than min_ratio of its text gets cnt_out[i] = -1 and tokenize_out[i] = 1 (tokenize it,
 *   kvidx_text_store_add it, and score it with kvhost_get_pod_scores_batch).
 * kvhost_get_pod_scores_batch: prompt i is tokens[tok_off[i] .. tok_off[i+1]). */
int kvhost_get_pod_scores_text(kvhost_t* h, const uint8_t* text, const int64_t* text_off, size_t n, const char* model,
                               const char* const* pods, size_t n_pods, double min_ratio, const char** pod_out, double* score_out,
                               int32_t* cnt_out, uint8_t* tokenize_out);
int kvhost_get_pod_scores_batch(kvhost_t* h, const uint32_t* tokens, const int64_t* tok_off, size_t n, const char* model,
                                const char* const* pods, size_t n_pods, const char** pod_out, double* score_out, int32_t* cnt_out);

/* kvblock.Index with strings.  entries are (pod, tier) name pairs. */
int kvhost_index_add(kvhost_t* h, const char* model, const uint64_t* engine, size_t n_engine, const uint64_t* request, size_t n_request,
                     const char* const* pods, const char* const* tiers, size_t n_entries);
int kvhost_index_evict(kvhost_t* h, const char* model, uint64_t engine, const char* const* pods, const char* const* tiers, size_t n_entries);
int kvhost_index_get_request_key(kvhost_t* h, const char* model, uint64_t engine, uint64_t* out);
/* Lookup: for key i, cnt_out[i] entries; entry j's names at pod_out / tier_out [i*10 + j]. */
int kvhost_index_lookup(kvhost_t* h, const char* model, const uint64_t* keys, size_t n, const char* const* pods, size_t n_pods,
                        const char** pod_out, const char** tier_out, uint8_t* cnt_out);

/* kvevents.Pool.  add_task copies the payload into queue FNV-32a(pod) % concurrency; process drains every queue in
 * FIFO order, decodes the msgpack EventBatch of each message and applies all resulting events with ONE
 * kvidx_apply_events call.  Returns the number of events applied (or a negative code).
 * With clear_on_all_blocks_cleared, the drained batch is cut at the AllBlocksCleared markers: segment k holds each pod's
 * events between its (k-1)-th and k-th marker and is one kvidx_apply_events call, followed by one kvidx_remove_pods for
 * the pods that cleared at that boundary.  Per-pod order is kept; the order between pods stays unspecified.
 * A drain of 1 MiB of payloads or more is decoded on the GPU instead (kvidx_apply_event_payloads, one call), with the same
 * records, tier ids, metrics and result; a Medium new to the mirror is interned on the host first, in drain order, and a
 * drain holding an AllBlocksCleared marker under clear_on_all_blocks_cleared takes the host path. */
int kvhost_pool_add_task(kvhost_t* h, const char* pod, const char* model, const void* payload, size_t len);
int kvhost_pool_queue_index(kvhost_t* h, const char* pod);
int64_t kvhost_pool_process(kvhost_t* h, int64_t* n_dropped_out);

/* Pure host decoding of one message payload into kvidx_event_t records (+ flat hash / token arrays).  Writes at most
 * the given capacities and returns the number of events, or -KVIDX_ENOSPC-style negatives.  Malformed batches decode
 * to 0 events (poison pill dropped, pool.go:182-187); malformed events are skipped (pool.go:190-239).
 * Hashes rejected by getHashAsUint64 (pool.go:343-367) are left out of a BlockStored's list (pool.go:272-275); a rejected
 * parent hash skips the event (pool.go:283-287).  AllBlocksCleared decodes to nothing (pool.go:332-333), or, with
 * clear_on_all_blocks_cleared, to a KVHOST_EV_ALL_BLOCKS_CLEARED marker record at its position (pod and model set, no
 * hashes).  Markers are a host-level record: kvidx_apply_events rejects them. */
#define KVHOST_EV_ALL_BLOCKS_CLEARED 2
int64_t kvhost_decode_event_batch(kvhost_t* h, const char* pod, const char* model, const void* payload, size_t len,
                                  kvidx_event_t* ev_out, size_t ev_cap, uint64_t* hash_out, size_t hash_cap, size_t* n_hash_out,
                                  uint32_t* tok_out, size_t tok_cap, size_t* n_tok_out);

/* kvcache_index_* metrics (metrics/collector.go:28-59) with the instrumented index's semantics (instrumented_index.go:35-92):
 * Add counts len(requestKeys) admissions and Evict len(entries) evictions whatever the call returned; every Lookup counts
 * one request and one latency observation; a successful Lookup adds max over pods of that pod's entries in the result to
 * both max_pod_hit_count and lookup_hits.  The event pool goes through the same Add / Evict (one Evict per removed hash,
 * pool.go:317-330).  The hit count is taken over the result MAP: without a pod filter a key repeated in one Lookup counts
 * once, with one every occurrence counts (in_memory.go:126-135).  With enable_metrics, the GetPodScores entry points issue the
 * reference's full-depth Lookup next to the score call as kvidx_lookup_hits (the hit count needs every key of the prompt,
 * not only the consecutive prefix the scorer walks): one call (n = 1) for kvhost_get_pod_scores, _keys and _turn, and ONE
 * call over all scored prompts of a kvhost_get_pod_scores_batch / _text batch, each of which then records one request, one
 * latency observation of (call duration / scored prompts) and its own hit count.  kvhost_index_lookup counts from
 * kvidx_lookup's result.  All zero when enable_metrics is 0. */
#define KVHOST_LATENCY_BUCKETS 11          /* prometheus.DefBuckets: .005 .01 .025 .05 .1 .25 .5 1 2.5 5 10 (+Inf = count) */
typedef struct kvhost_metrics {
    uint64_t admissions_total, evictions_total, lookup_requests_total, max_pod_hit_count_total, lookup_hits_total;
    uint64_t lookup_latency_bucket[KVHOST_LATENCY_BUCKETS];      /* cumulative, le = bucket bound */
    uint64_t lookup_latency_count;
    double lookup_latency_sum;                                   /* seconds */
} kvhost_metrics_t;
int kvhost_get_metrics(kvhost_t* h, kvhost_metrics_t* out);
/* Prometheus text exposition of the above (same metric names and help strings as the reference).  Returns the number of
 * bytes needed (excluding the NUL); writes at most cap - 1 bytes + NUL. */
int64_t kvhost_metrics_text(kvhost_t* h, char* buf, size_t cap);

/* Tokenization prefix store (SURVEY 8(f3), the cache in front of the tokenizer; the tokenizer itself stays with the
 * embedding program).  Text is cut into block_size-BYTE blocks, block i is keyed by XXH64(seed 0) of the little-endian
 * previous key followed by the block's bytes (lru_store.go:111-121), and maps to the tokens whose END offset falls inside
 * the text up to the block's end (:124-137).  A partial last block is never stored or looked up.
 *   create: NewLRUTokenStore (:72-87); cache_size <= 0 is an error like lru.New; defaults 500000 blocks of 256 bytes.
 *   add:    AddTokenization (:89-141); offsets are n_tokens pairs [low, high) of byte offsets; empty prompt or no
 *           tokens is a no-op.
 *   find:   FindLongestContainedTokens (:143-190): walks the blocks until the first one missing from the cache (a hit
 *           refreshes its recency); returns the number of contained tokens (all of them are written if cap allows, else
 *           the first cap) and the covered fraction of the prompt, end of the last matched block / prompt length.
 * tokenization.Pool.processTask (pool.go:209-225) is: find; if the ratio is below 0.8 tokenize, add, use the fresh tokens. */
typedef struct kvhost_prefix_store kvhost_prefix_store_t;
int  kvhost_prefix_store_create(int64_t cache_size, int32_t block_size, kvhost_prefix_store_t** out);
void kvhost_prefix_store_destroy(kvhost_prefix_store_t* s);
int  kvhost_prefix_store_add(kvhost_prefix_store_t* s, const char* prompt, size_t prompt_len, const uint32_t* tokens,
                             const uint64_t* offsets, size_t n_tokens);
int64_t kvhost_prefix_store_find(kvhost_prefix_store_t* s, const char* prompt, size_t prompt_len, uint32_t* tokens_out, size_t cap,
                                 double* overlap_ratio_out);
int64_t kvhost_prefix_store_len(kvhost_prefix_store_t* s);           /* blocks resident */
/* Snapshot / restore of the store (no counterpart; the image of kvidx_text_store_snapshot, format in kvidx.h): snapshot
 * writes the resident blocks least recent first and refreshes nothing; buf == NULL or cap below the size -> KVIDX_ENOSPC
 * with *size_out set and nothing written.  restore needs an empty store of the image's block_bytes and equals adding the
 * records one by one, oldest first (the store keeps its cache_size: the newest cache_size records stay); a malformed image,
 * a non-empty store or another block_bytes -> KVIDX_EINVAL with the store unchanged.  The device store's image after the
 * same calls is byte-equal. */
int kvhost_prefix_store_snapshot(kvhost_prefix_store_t* s, void* buf, uint64_t cap, uint64_t* size_out);
int kvhost_prefix_store_restore(kvhost_prefix_store_t* s, const void* buf, uint64_t len);
uint64_t kvhost_xxhash64(const void* data, size_t len, uint64_t seed);

/* Remove a pod that has gone away (no counterpart in the reference, where a dead pod's blocks only age out of the LRU):
 * 1. drops the pod's messages still waiting in its queue; 2. removes its entries from the device index on the given tiers
 * (kvidx_remove_pods; n_tiers == 0: all tiers); 3. with all tiers, frees the pod's id once the removal has completed and
 * every read call that was already running has returned, so the next new pod name takes it (lowest freed id first) and
 * kvhost_pod_id of the old name gives a new interning.  Serialised with kvhost_pool_process.  On a no_device instance
 * steps 1 and 3 only.  An unknown pod name is a no-op.  Not counted in kvcache_index_evictions_total, which counts the
 * reference's Evict calls.  Returns the number of queued messages dropped, or a negative KVIDX_E* code. */
int kvhost_remove_pod(kvhost_t* h, const char* pod, const char* const* tiers, size_t n_tiers);

/* Snapshot / restore of the whole mirror (no counterpart; kvidx_snapshot / kvidx_restore).  Host image, little-endian:
 *   char[8] "KVHOSTSN", u32 version = 1, u32 0;
 *   three name tables -- models, tiers, pods -- each a u32 id count, then per id a u32 byte length and the bytes;
 *     0xFFFFFFFF (no bytes) marks a pod id freed by kvhost_remove_pod, so the lowest-first reuse order survives;
 *   u64 length, then the kvidx image as opaque bytes (length 0 for a no_device instance).
 * kvhost_snapshot holds the write side exclusively, as kvhost_remove_pod does, so names and entries agree; read calls keep
 * running.  Messages still queued (kvhost_pool_add_task without kvhost_pool_process) are not part of the image.
 * buf == NULL or cap too small -> KVIDX_ENOSPC with *size_out set.
 * kvhost_restore needs a fresh target: no pod or model interned, only the configured tiers, empty queues (else
 * KVIDX_EINVAL).  The image's tiers at the configured ids must carry the target's configured names (else KVIDX_EINVAL);
 * tier weights stay the target's.  Every pod id owning an entry in the index section must have a name in the pod table
 * (else KVIDX_EINVAL).  A no_device target accepts only an image without an index section.  The index section
 * goes through kvidx_restore and its error codes; on any error the target is left as it was. */
int kvhost_snapshot(kvhost_t* h, void* buf, uint64_t cap, uint64_t* size_out);
int kvhost_restore(kvhost_t* h, const void* buf, uint64_t len);

/* Pod inventory with names (no counterpart; kvidx_pod_inventory): for every interned pod its name and id, the request keys
 * it holds, those it alone holds (what kvhost_remove_pod of it would remove), with `engine` != 0 the engine mappings that
 * would go with them, and its entries per tier id.  model: a model name, or NULL for all models; a name never seen counts
 * nothing (it is not interned).  Pod ids freed by kvhost_remove_pod are skipped.  tier_names_out (may be NULL): the name of
 * every interned tier id, NULL for the others; name pointers stay valid for the life of the handle.  totals_out (may be
 * NULL): {request keys, entries, engine mappings, stale engine mappings}, the last two only with `engine`.
 * Writes at most `cap` rows, in pod id order, and returns the number of interned pods (call again with more room if it
 * exceeds cap), or a negative KVIDX_E* code.  Serialised with kvhost_remove_pod and kvhost_restore (it holds the write side
 * shared), so ids and names agree; read calls, index_add / index_evict and kvhost_pool_process keep running, and a pod
 * interned while the device counts is reported with whatever the device saw of it.  A no_device instance answers with
 * all-zero counts. */
typedef struct kvhost_pod_row {
    const char* pod;
    uint32_t pod_id, reserved;
    uint64_t keys, sole_keys, sole_engine_keys;
    uint64_t entries[KVIDX_MAX_TIERS];           /* by tier id */
} kvhost_pod_row_t;
int64_t kvhost_pod_inventory(kvhost_t* h, const char* model, int32_t engine, kvhost_pod_row_t* rows, size_t cap,
                             const char** tier_names_out /* KVIDX_MAX_TIERS */, uint64_t totals_out[4]);
/* The inventory over all models, engine pass included, in Prometheus text format, apart from kvhost_metrics_text (whose
 * output is the reference's metric set): gauges kvcache_index_pod_entries{pod,tier} (non-zero ones),
 * kvcache_index_pod_keys{pod}, kvcache_index_pod_sole_keys{pod}, kvcache_index_pod_sole_engine_keys{pod},
 * kvcache_index_stale_engine_keys.  Buffer conventions of kvhost_metrics_text; a negative KVIDX_E* code on failure. */
int64_t kvhost_inventory_text(kvhost_t* h, char* buf, size_t cap);

/* interning introspection.  Model and tier ids are never reused; a pod id is freed by kvhost_remove_pod (all tiers) and
 * reused lowest first.  Name pointers returned by the calls above stay valid for the life of the handle. */
int kvhost_pod_id(kvhost_t* h, const char* pod);
int kvhost_tier_id(kvhost_t* h, const char* tier);
int kvhost_model_id(kvhost_t* h, const char* model);

#ifdef __cplusplus
}
#endif
#endif
