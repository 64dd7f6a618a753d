/*
 * kvidx.h -- C ABI of libkvidx: the GPU-resident KV-block locality index.
 *
 * This is the drop-in boundary for ONE hot path of llm-d/llm-d-kv-cache-manager:
 * kvcache.Indexer.GetPodScores() steps 2-4 (token blocks -> chain-hashed request
 * keys -> index probe -> longest-consecutive-prefix per-pod score) and the
 * kvevents.Pool -> kvblock.Index.Add/Evict write path that feeds the same table.
 * Every entry point names the reference interface (path:line under the
 * reference root) it replaces.  A Go maintainer binds these with cgo
 * (INTEGRATION.md shows the stub); the tests bind them with ctypes.
 *
 * Conventions
 *   - plain C types only; caller owns every buffer; nothing is retained after
 *     return (cgo rule: no Go pointer survives the call);
 *   - return 0 on success or a negative KVIDX_E* code; kvidx_last_error() gives
 *     the message for the calling thread's last failure on that handle;
 *   - strings are interned on the host side of the boundary: model -> uint32,
 *     pod -> 12-bit id, device tier -> 4-bit id.  (pod,tier) travels packed in a
 *     kvidx_podtier_t.  The host mirror (kvidx_host.h) owns the string maps;
 *   - all entry points may be called concurrently from many OS threads (cgo
 *     pins one per call), as kvblock.Index requires (kvblock/index.go:118).
 *     The READ path (hash / lookup / score / get_request_key) and the WRITE path
 *     (add / evict / apply_events) run on separate CUDA streams and overlap on the
 *     device: a reader sees every slot either before or after an individual
 *     Add / Evict of that key (table.cuh), which is the guarantee the reference's
 *     per-key mutex gives.  A write call has taken effect when it returns, so a
 *     thread reads its own writes (index_test.go:214-278).  Concurrent host-buffer
 *     kvidx_score_batch* callers are coalesced into one launch (kvidx_score_keys* and kvidx_score_turn* calls are not);
 *   - there is NO CPU fallback: without a CUDA device kvidx_create fails with
 *     KVIDX_ECUDA.
 */
#ifndef KVIDX_H
#define KVIDX_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KVIDX_ABI_VERSION 2   /* 2: read and write path run concurrently; kvidx_apply_events_dev takes the batch sizes;
                                  kvidx_score_batch_sparse_dev, kvidx_shard_compact; two more stats fields */

/* error codes (negative errno style) */
#define KVIDX_OK        0
#define KVIDX_ENOENT   (-2)   /* engine key not found (in_memory.go:266-268)                 */
#define KVIDX_ECUDA    (-5)   /* CUDA runtime / device failure, or no device                  */
#define KVIDX_ENOMEM   (-12)
#define KVIDX_EINVAL   (-22)  /* empty args, length mismatch ... (in_memory.go:108-110,150-155,213-215) */
#define KVIDX_ENOSPC   (-28)  /* table full                                                    */
#define KVIDX_ERANGE   (-34)  /* id outside the configured pod / tier / model range            */

/* packed (pod, tier) entry == kvblock.PodEntry (index.go:149-154) after interning */
#define KVIDX_TIER_BITS        4
#define KVIDX_POD_BITS         12
#define KVIDX_MAX_TIERS        (1u << KVIDX_TIER_BITS)   /* 16   */
#define KVIDX_MAX_PODS         (1u << KVIDX_POD_BITS)    /* 4096 */
#define KVIDX_MAX_PODS_PER_KEY 10                        /* in_memory.go:34 defaultPodsPerKey */
typedef uint16_t kvidx_podtier_t;
#define KVIDX_PODTIER(pod, tier) ((kvidx_podtier_t)((((uint32_t)(pod)) << KVIDX_TIER_BITS) | ((uint32_t)(tier) & (KVIDX_MAX_TIERS - 1))))
#define KVIDX_PT_POD(pt)  ((uint32_t)(pt) >> KVIDX_TIER_BITS)
#define KVIDX_PT_TIER(pt) ((uint32_t)(pt) & (KVIDX_MAX_TIERS - 1))

/* value written into a dense score row for a pod that is NOT in the result map.
 * The reference's scores are sums of max(0, weight) (kvblock_scorer.go:90,100), so
 * every real score is >= 0 and -1.0 is unambiguous. */
#define KVIDX_SCORE_ABSENT (-1.0)

typedef struct kvidx kvidx_t;   /* opaque */

/* Configuration == TokenProcessorConfig (token_processor.go:34-42)
 *                + InMemoryIndexConfig  (in_memory.go:38-43)
 *                + KVCacheBackendConfig weights (backend.go:19-31). */
typedef struct kvidx_config {
    uint32_t struct_size;      /* sizeof(kvidx_config_t), for ABI growth                        */
    int32_t  device;           /* CUDA device ordinal                                           */
    uint32_t block_size;       /* tokens per block; 0 -> 16 (token_processor.go:31)             */
    uint32_t pods_per_key;     /* PodCacheSize; 0 -> 10; must be 1..10                          */
    uint64_t init_hash;        /* FNV-64a(HashSeed) (token_processor.go:81-90); use kvidx_fnv64a */
    uint64_t capacity;         /* InMemoryIndexConfig.Size: max resident keys; 0 -> 1<<20       */
    uint64_t table_slots;      /* open-addressing slots (power of two); 0 -> 4*capacity rounded up
                                  (load factor <= 0.25: a probe almost always ends in its home pair) */
    uint32_t max_pods;         /* dense score-row width P (1..4096); 0 -> 256                   */
    uint32_t n_tier_weights;   /* entries of tier_weight[] that are configured                  */
    double   tier_weight[KVIDX_MAX_TIERS]; /* weight of tier id i; ids >= n_tier_weights score 1.0
                                              (unknown tier => 1.0, kvblock_scorer.go:93-98)    */
    uint32_t lru_exact;        /* 1: track key recency (a stamp per slot, written by Lookup / Score / Add / Evict /
                                  GetRequestKey exactly where golang-lru refreshes) and evict the least recently used
                                  request / engine keys when a write call leaves more than `capacity` of them
                                  (in_memory.go:59,64,118,163,170).  A key touched several times in one call ranks
                                  as of its last touch in the order the reference applies the call:
                                    kvidx_lookup        keys in array order;
                                    Score() (batch, keys, turn; host and _dev)  prompt after prompt, and within a
                                                        prompt every present key in block order, also past the end
                                                        of the walk;
                                    kvidx_add           pairs in order, each one's engine mapping before its request key;
                                    apply_events[_dev]  each pod's events in array order, pods in ascending id (one of
                                                        the orders the reference's per-pod workers allow);
                                  every touch of a call gets its own stamp, however many keys a prompt or event holds.
                                  What stays at call granularity is eviction: it runs after the call, not inside it,
                                  so a call that takes a map past `capacity` may still see a key the reference would
                                  have evicted part way through it.  Score() probes
                                  every key of a prompt (the reference's Lookup has no early exit), so it is the slow,
                                  semantics-first mode.  0 (default): recency is not tracked and `capacity` only sizes
                                  the table -- right whenever the fleet's block count stays below Size (default 1e8). */
    uint32_t shard_rank;       /* hash-range sharding over the GPUs of one NVSwitch domain (SURVEY 8e): this handle */
    uint32_t shard_count;      /* owns shard `shard_rank` of `shard_count` (power of two <= 8; 0 or 1 = unsharded).   */
                               /* `capacity` stays the TOTAL key budget; each shard holds capacity/shard_count.        */
    uint32_t evict_policy;     /* KVIDX_EVICT_CLOCK: hold each map to `capacity` keys on the fast paths.  One reference bit per
                                  slot is set wherever golang-lru refreshes recency (Add, Evict, GetRequestKey, a BlockStored
                                  parent, Lookup) and, for Score(), on the present keys among the blocks the walk probes: block 0
                                  up to and including the block that empties the active pod set, or the last full block (the
                                  early exit stays).  After every write call (add, evict, apply_events[_dev], restore) a CLOCK
                                  sweep evicts keys until each map holds at most `capacity`: unreferenced keys go before referenced
                                  ones, whose bits are cleared as the hand passes them.  Request keys and engine mappings are
                                  evicted independently, as in the reference.  A read running at the same moment as a sweep sees
                                  each key before or after its eviction, and may or may not protect the keys it touches.
                                  KVIDX_EVICT_NONE (0, default): `capacity` only sizes the table.  Other values, CLOCK with
                                  lru_exact, or CLOCK on a sharded handle -> KVIDX_EINVAL. */
    uint32_t grow_tables;      /* 1: both tables grow on demand up to C = pow2ceil(max(4 * capacity, 1024)) slots, what a fixed
                                  handle with table_slots 0 allocates, so that `capacity` is a limit and not an up-front
                                  allocation (golang-lru's maps grow as keys arrive, in_memory.go:33).  The tables start at
                                  table_slots (rounded up to a power of two, at least 1024), or at min(C, 2^20) slots when
                                  table_slots is 0.  Before a write batch (add, apply_events[_dev], apply_event_payloads) with
                                  S slots, L = the larger of the live request keys and live engine mappings (tombstones do not
                                  count) and I = the batch's bound on new keys: if S < C and 4 (L + I) > S, both tables are
                                  rehashed, in one step, into min(C, the smallest power of two >= 4 (L + I)) slots, keeping
                                  the load at most 1/4 as on a fixed handle; exact-LRU stamps and CLOCK reference bits move
                                  with their keys, the CLOCK hands restart at slot 0.  Every other rule (compaction from
                                  80 %, KVIDX_ENOSPC beyond 90 %) then runs on the new size, so a handle grown to C behaves
                                  like the fixed one.  A growth takes the tables exclusively inside the write call that
                                  needs it and drains the device: read calls wait for it and see the index wholly before or
                                  after it, asynchronous reads already queued complete on the old tables (for
                                  kvidx_apply_events_dev the growth is synchronous, the batch stays asynchronous).  A growth
                                  whose allocation fails leaves the old tables in use under the fixed rules; its peak is old +
                                  new tables (3x the old size).  It counts in kvidx_stats_t.rebuilds.  0 (default): the
                                  tables are allocated whole at create.  Other values, table_slots > C, or a sharded handle
                                  -> KVIDX_EINVAL. */
    uint32_t reserved[3];
} kvidx_config_t;

#define KVIDX_EVICT_NONE  0u
#define KVIDX_EVICT_CLOCK 1u

void        kvidx_config_default(kvidx_config_t* cfg);
int         kvidx_create(const kvidx_config_t* cfg, kvidx_t** out);   /* NewInMemoryIndex + NewChunkedTokenDatabase + NewKVBlockScorer */
void        kvidx_destroy(kvidx_t* idx);
const char* kvidx_last_error(kvidx_t* idx);
int         kvidx_abi_version(void);

/* host-only helpers */
uint64_t kvidx_fnv64a(const void* data, size_t n);                 /* getInitHash, token_processor.go:81-90 */
uint32_t kvidx_fnv32a(const void* data, size_t n);
uint32_t kvidx_queue_index(const char* pod, size_t n, uint32_t concurrency); /* Pool.AddTask, kvevents/pool.go:132-144 */
int      kvidx_set_tier_weight(kvidx_t* idx, uint32_t tier, double weight);

/* pinned staging a caller may use for zero-copy submission (optional) */
void* kvidx_host_alloc(size_t bytes);
void  kvidx_host_free(void* p);

/* ---- read path ---------------------------------------------------------------- */

/* TokenProcessor.TokensToKVBlockKeys (token_processor.go:141-162) for a batch.
 * tok/tok_off: CSR, prompt i owns tok[tok_off[i] .. tok_off[i+1]).
 * parent: NULL -> every chain starts at init_hash; else parent[i] is the parent
 *         request-key hash of prompt i (parent_valid[i]==0 -> init_hash; parent_valid
 *         NULL -> all valid).
 * keys_out: sum_i floor(len_i/B) hashes, prompt-major; key_off_out[n_prompts+1]. */
int kvidx_hash_keys(kvidx_t* idx, const uint32_t* tok, const int64_t* tok_off, int64_t n_prompts,
                    const uint64_t* parent, const uint8_t* parent_valid,
                    uint64_t* keys_out, int64_t* key_off_out);

/* Index.Lookup (index.go:125, in_memory.go:105-146).  filter: NULL = all pods, else a
 * bitmask of ceil(max_pods/64) words over pod ids.  For key i, cnt_out[i] entries are
 * written to podtier_out[i*10 ..] oldest->newest (lru Keys() order); cnt_out[i]==0 means
 * "key absent from the result map" (missing, filtered to nothing, or after the
 * present-but-empty cut).  n==0 -> KVIDX_EINVAL (in_memory.go:108-110). */
int kvidx_lookup(kvidx_t* idx, uint32_t model, const uint64_t* keys, int64_t n,
                 const uint64_t* filter, kvidx_podtier_t* podtier_out, uint8_t* cnt_out);

/* The hit count of a full-depth Lookup for a batch of prompts: what the instrumented index adds to
 * kvcache_index_max_pod_hit_count_total and kvcache_index_lookup_hits_total (instrumented_index.go:71-92) for the Lookup
 * GetPodScores makes (indexer.go:150).  K_i are prompt i's request keys: for the tokens form TokensToKVBlockKeys(nil,
 * tokens_i), the keys kvidx_score_batch uses; for the keys form the given list (keys/key_off as for kvidx_score_keys).  With
 * F_i the prompt's filter row (NULL filter, or an all-zero row: all pods, as in Score()), hits_out[i] =
 * recordHitMetrics(Lookup(K_i, F_i)): for each pod the number of its entries in the result map, then the largest of those
 * counts (a pod with entries on two tiers of one key counts 2).  The map decides repeats: without a filter a key repeated in
 * K_i counts once (in_memory.go:126-128), with a filter once per occurrence (:130-135).  No key -> 0.  Lookup has no early
 * exit, so every key of every prompt is probed; its present-but-empty cut (:119-122) cannot trigger, since a present key
 * always holds an entry.
 * It IS a Lookup, and touches as kvidx_lookup does: exact-LRU handles stamp every present key in prompt-then-key order, with
 * the stamp layout of Score() (a repeated key ranks as of its last occurrence); CLOCK handles set the reference bit of every
 * present key.  A read call, ordered after kvidx_apply_events_dev batches issued before it; default, CLOCK, exact-LRU and
 * sharded handles (peers probed from the kernel, as Score() does).  n_prompts < 0, an offset array NULL or not monotone, an
 * element array NULL with a non-zero count, hits_out NULL -> KVIDX_EINVAL; n_prompts == 0 -> 0, nothing written;
 * key_off[0] / tok_off[0] may be non-zero.  model, model0 and filter mean what they mean for kvidx_score_batch.
 * The host forms are synchronous; pinned buffers are copied in place, pageable ones through pinned chunks.  The tokens
 * forms hash the keys into scratch first.  kvidx_lookup_hits_keys_dev is one asynchronous launch on the handle's stream (on
 * an exact-LRU handle it reads the first and last offsets back to reserve its stamps, as Score() does);
 * kvidx_lookup_hits_dev reads the batch's first and last token offsets back to size its key scratch, and is asynchronous
 * after that. */
int kvidx_lookup_hits(kvidx_t* idx, const uint32_t* tok, const int64_t* tok_off, int64_t n_prompts,
                      const uint32_t* model, uint32_t model0, const uint64_t* filter, uint32_t* hits_out);
int kvidx_lookup_hits_keys(kvidx_t* idx, const uint64_t* keys, const int64_t* key_off, int64_t n_prompts,
                           const uint32_t* model, uint32_t model0, const uint64_t* filter, uint32_t* hits_out);

/* Indexer.GetPodScores steps 2-4 fused (indexer.go:141-163) for a batch of prompts.
 * Callers that arrive while another call's batch is on the device are queued and served together by one launch
 * (each gets exactly the rows of its own prompts; KVIDX_SUBMIT_QUEUE=0 turns the coalescing off).
 * model: per-prompt model ids, or NULL to use model0 for all.
 * filter: NULL, or n_prompts * ceil(max_pods/64) words (all-zero row == empty set == all pods,
 *         indexer.go:151 / in_memory.go:126).
 * scores_out: n_prompts * max_pods doubles; KVIDX_SCORE_ABSENT where the pod is not in the
 *         reference's result map.  A prompt with no full block yields an all-absent row and
 *         has_keys_out[i]=0 (reference returns (nil,nil), indexer.go:142-146); has_keys_out
 *         may be NULL. */
int kvidx_score_batch(kvidx_t* idx, const uint32_t* tok, const int64_t* tok_off, int64_t n_prompts,
                      const uint32_t* model, uint32_t model0, const uint64_t* filter,
                      double* scores_out, uint8_t* has_keys_out);

/* Same, sparse result: for prompt i cnt_out[i] (<=10) pairs pods_out[i*10+j], scores_out[i*10+j]. */
int kvidx_score_batch_sparse(kvidx_t* idx, const uint32_t* tok, const int64_t* tok_off, int64_t n_prompts,
                             const uint32_t* model, uint32_t model0, const uint64_t* filter,
                             uint16_t* pods_out, double* scores_out, uint8_t* cnt_out, uint8_t* has_keys_out);

/* Indexer.GetPodScores steps 3-4 (indexer.go:150-159) for a batch of prompts whose request keys the caller already holds:
 * LongestPrefixScorer.Score(keys, Index.Lookup(keys, pods)) (kvblock_scorer.go:108-151, in_memory.go:105-146), e.g. a
 * conversation that kept turn k's keys and hashed only turn k+1's new blocks (kvidx_hash_keys with parent = last key), or
 * a deployment that keeps its own TokenProcessor.  keys/key_off: CSR, prompt i owns keys[key_off[i] .. key_off[i+1]),
 * request-key hashes in block order (any list: absent, repeated and other models' keys score as the reference scores
 * them); key_off[0] may be non-zero.  model, model0, filter, the dense / sparse result rows and KVIDX_SCORE_ABSENT mean what
 * they mean for kvidx_score_batch; has_keys_out[i] = (prompt i has at least one key) -- no key gives an all-absent row,
 * the reference's (nil, nil).  One warp per prompt at every batch size and block size; exact-LRU handles stamp every
 * present key of the prompt, as kvidx_score_batch does.  n_prompts < 0, key_off NULL or not monotone, keys NULL with a
 * non-zero key count -> KVIDX_EINVAL; n_prompts == 0 -> 0, nothing written.  Host buffers go through the same chunked
 * copy pipeline as kvidx_score_batch (pinned buffers directly; small calls read pinned keys in place), but calls are NOT
 * coalesced with other callers: each goes straight through. */
int kvidx_score_keys(kvidx_t* idx, const uint64_t* keys, const int64_t* key_off, int64_t n_prompts,
                     const uint32_t* model, uint32_t model0, const uint64_t* filter,
                     double* scores_out, uint8_t* has_keys_out);
int kvidx_score_keys_sparse(kvidx_t* idx, const uint64_t* keys, const int64_t* key_off, int64_t n_prompts,
                            const uint32_t* model, uint32_t model0, const uint64_t* filter,
                            uint16_t* pods_out, double* scores_out, uint8_t* cnt_out, uint8_t* has_keys_out);

/* GetPodScores steps 2-4 for a conversation turn, in one call: prompt i is the request keys the caller already holds
 * (keys[key_off[i] .. key_off[i+1]), block order) followed by new tokens (tok[tok_off[i] .. tok_off[i+1]), whose first
 * token starts a block).  With K_i = held_i ++ TokensToKVBlockKeys(parent = last held key, or init_hash when prompt i holds
 * none, new tokens_i), the row is LongestPrefixScorer.Score(K_i, Index.Lookup(K_i, pods)) and has_keys_out[i] = |K_i| > 0.
 * new_keys_out (may be NULL): the floor(len_i / B) new keys of every prompt, prompt-major; new_key_off_out[n_prompts+1] =
 * their offsets, from 0 (filled whenever it is given).  A trailing partial block is dropped, as in kvidx_hash_keys: the
 * caller re-sends it next turn.  Every other argument, KVIDX_SCORE_ABSENT and the result rows mean what they mean for
 * kvidx_score_keys; key_off[0] and tok_off[0] may be non-zero.  n_prompts < 0, NULL or non-monotone offsets, a NULL
 * element array with a non-zero count, new_keys_out without new_key_off_out -> KVIDX_EINVAL; n_prompts == 0 -> 0, nothing
 * written.  Block size 16, 32, 64 or 128 on default and CLOCK handles: one fused warp-per-prompt kernel at every batch size
 * (the held keys are walked, then the new tokens hashed warp-cooperatively from the last held key while the walk goes on).
 * Other block sizes, exact-LRU handles and KVIDX_SCORE_KERNEL=v1 hash, concatenate and score the keys (exact-LRU stamps as
 * kvidx_score_batch).  Host buffers as kvidx_score_keys: pinned ones in place, small calls zero-copy, the rest through the
 * chunked pipeline; not coalesced with other callers. */
int kvidx_score_turn(kvidx_t* idx, const uint64_t* keys, const int64_t* key_off, const uint32_t* tok, const int64_t* tok_off,
                     int64_t n_prompts, const uint32_t* model, uint32_t model0, const uint64_t* filter,
                     double* scores_out, uint8_t* has_keys_out, uint64_t* new_keys_out, int64_t* new_key_off_out);
int kvidx_score_turn_sparse(kvidx_t* idx, const uint64_t* keys, const int64_t* key_off, const uint32_t* tok, const int64_t* tok_off,
                            int64_t n_prompts, const uint32_t* model, uint32_t model0, const uint64_t* filter,
                            uint16_t* pods_out, double* scores_out, uint8_t* cnt_out, uint8_t* has_keys_out,
                            uint64_t* new_keys_out, int64_t* new_key_off_out);

/* ---- prefix store and Score() from text (tokenization.Pool.processTask, pool.go:198-237) ------------------------------
 * prefixstore.LRUTokenStore (lru_store.go:54-190) on the device, one per handle: cached tokenizations, so that a prompt
 * whose text repeats an earlier prompt's is scored without going back to the tokenizer.  Text is cut into block_bytes-byte
 * blocks; a partial last block is never stored or looked up.  Block b's key is XXH64 (seed 0) of the previous block's key
 * (little-endian u64; 0 for block 0) followed by the block's bytes -- the host store's chain (kvhost_xxhash64).  A block
 * holds the tokens whose END offset is <= the block's end and that no earlier block took (zero-width tokens included).
 * One map, no model in the key.  Add inserts or replaces a block's tokens and refreshes it; Find walks the blocks up to
 * the first miss, refreshes each hit, and returns their tokens with ratio = (end of the last hit block) / text length
 * (0.0 when nothing hits).  Exact LRU over cache_blocks keys.
 * A call holds many prompts (text / text_off: CSR of bytes, prompt i owns text[text_off[i] .. text_off[i+1]); text_off[0]
 * may be non-zero) and equals the host store applying them one after another in array order: an add's touches run prompt
 * by prompt, block by block, the last add of a key wins its tokens, and the eviction down to the cache_blocks most recently
 * touched keys runs once, after the add call (every touch of an add is an insert or an update, so the resident set and
 * every later find equal the sequential store's).  Finds never evict.
 * Store calls serialise on the store's own lock; the store is independent of the index's read and write sides, of its
 * capacity mode and of sharding (on a sharded handle it is rank-local).  Host buffers: pinned ones are copied in place,
 * pageable ones through pinned chunks.  Errors: NULL handle, negative n_prompts, NULL or non-monotone offsets, NULL arrays
 * with non-zero counts, a store call before kvidx_text_store_init, a second init, cache_blocks or block_bytes <= 0
 * -> KVIDX_EINVAL; a device allocation that fails -> KVIDX_ENOMEM.  n_prompts == 0 -> 0, nothing written.
 *
 * kvidx_text_store_init: NewLRUTokenStore (defaults there: cache_blocks 500000, block_bytes 256, lru_store.go:30-33).
 * kvidx_text_store_add: AddTokenization of every prompt.  tok / tok_off: CSR of the prompts' token ids (tok_off[0] may be
 *   non-zero); tok_span[2 t], tok_span[2 t + 1]: token t's [low, high) byte offsets in its prompt's text.  A prompt with no
 *   text or no tokens adds nothing (lru_store.go:96-98).
 * kvidx_text_store_find: FindLongestContainedTokens of every prompt.  tok_off_out[n_prompts + 1] (from 0) is always
 *   filled; tok_out NULL or tok_cap below the total -> KVIDX_ENOSPC, and the find refreshes nothing.  ratio_out may be NULL.
 * kvidx_text_store_len: keys resident.
 * kvidx_text_store_snapshot / _restore (no reference counterpart): the store as an image, for a warm start after a
 *   restart, an upgrade or a move to another GPU.  Image v1, little-endian, size 64 + 16 R + 4 T:
 *     header (64 bytes): char[8] "KVIDXTXT", u32 version = 1, u32 flags = 0, u32 block_bytes, u32 0, u64 R (records),
 *       u64 T (tokens), 24 zero bytes;
 *     R records of 16 bytes, least recent first (golang-lru Keys() order): u64 key, u32 n_tok, u32 0;
 *     T u32 token ids: record 0's n_tok tokens, then record 1's, ...
 *   The image depends only on the resident keys, their recency order and their tokens (not on table size, arena layout,
 *   stamps or cache_blocks), and equals kvhost_prefix_store_snapshot's after the same calls.  Records with n_tok 0 (a
 *   block in which no token ends) are legal.
 *   snapshot: runs after every earlier store call and every kvidx_score_text*_dev queued on the handle's stream, whose
 *   refreshes it includes; refreshes nothing itself.  buf == NULL or cap below the size -> KVIDX_ENOSPC with *size_out
 *   set and nothing written.  A pageable buffer is filled through pinned staging chunks, a pinned one directly.
 *   restore: into an initialised store holding no key (else KVIDX_EINVAL); equals adding the records one by one, oldest
 *   first: the store keeps its own cache_blocks, so a larger image leaves its newest cache_blocks records.  block_bytes
 *   other than the store's, a bad magic, version or flags, non-zero reserved bytes or record padding, a length that does
 *   not match the header, record token counts that do not add up to T, or a key appearing twice -> KVIDX_EINVAL.  Every
 *   record is checked before any is inserted: a refused image leaves the store as it was.  *blocks_out (may be NULL):
 *   keys resident afterwards.
 * kvidx_text_hash_keys: the block keys of every prompt at block_bytes (prompt-major, key_off_out[n_prompts + 1] from 0), as
 *   the store computes them; needs an initialised store (its stream and staging), whose contents it does not touch.
 * kvidx_score_text[_sparse]: processTask + GetPodScores steps 2-4.  One find over the batch (refreshing as above); prompt i
 *   is scored from its contained tokens when ratio_i >= min_ratio (the reference's `overlapRatio < min` test, negated),
 *   with the kvidx_score_batch dispatch at the batch's size, so its row equals kvidx_score_batch's of the same tokens on
 *   every handle mode.  Otherwise its row is all-absent, has_keys 0 and tokenize_out[i] = 1: the caller tokenizes it,
 *   adds it and scores it.  model, model0, filter and the result rows mean what they mean for kvidx_score_batch;
 *   has_keys_out, tokenize_out and ratio_out may be NULL.  min_ratio < 0 or NaN -> KVIDX_EINVAL.
 * kvidx_score_text[_sparse]_dev: the same over device-resident inputs and outputs, on the handle's stream.  It waits on the
 *   stream twice to size its scratch (the batch's block total, then its token totals), and is asynchronous after that. */
int kvidx_text_store_init(kvidx_t* idx, int64_t cache_blocks, int32_t block_bytes);
int kvidx_text_store_add(kvidx_t* idx, const uint8_t* text, const int64_t* text_off, int64_t n_prompts,
                         const uint32_t* tok, const uint64_t* tok_span, const int64_t* tok_off);
int kvidx_text_store_find(kvidx_t* idx, const uint8_t* text, const int64_t* text_off, int64_t n_prompts,
                          uint32_t* tok_out, int64_t tok_cap, int64_t* tok_off_out, double* ratio_out);
int kvidx_text_store_len(kvidx_t* idx, int64_t* blocks_out);
int kvidx_text_store_snapshot(kvidx_t* idx, void* buf, uint64_t cap, uint64_t* size_out);
int kvidx_text_store_restore(kvidx_t* idx, const void* buf, uint64_t len, int64_t* blocks_out);
int kvidx_text_hash_keys(kvidx_t* idx, const uint8_t* text, const int64_t* text_off, int64_t n_prompts, int32_t block_bytes,
                         uint64_t* keys_out, int64_t* key_off_out);
int kvidx_score_text(kvidx_t* idx, const uint8_t* text, const int64_t* text_off, int64_t n_prompts,
                     const uint32_t* model, uint32_t model0, const uint64_t* filter, double min_ratio,
                     double* scores_out, uint8_t* has_keys_out, uint8_t* tokenize_out, double* ratio_out);
int kvidx_score_text_sparse(kvidx_t* idx, const uint8_t* text, const int64_t* text_off, int64_t n_prompts,
                            const uint32_t* model, uint32_t model0, const uint64_t* filter, double min_ratio,
                            uint16_t* pods_out, double* scores_out, uint8_t* cnt_out, uint8_t* has_keys_out,
                            uint8_t* tokenize_out, double* ratio_out);
int kvidx_score_text_dev(kvidx_t* idx, const uint8_t* d_text, const int64_t* d_text_off, int64_t n_prompts,
                         const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter, double min_ratio,
                         double* d_scores_out, uint8_t* d_has_keys_out, uint8_t* d_tokenize_out, double* d_ratio_out);
int kvidx_score_text_sparse_dev(kvidx_t* idx, const uint8_t* d_text, const int64_t* d_text_off, int64_t n_prompts,
                                const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter, double min_ratio,
                                uint16_t* d_pods_out, double* d_scores_out, uint8_t* d_cnt_out, uint8_t* d_has_keys_out,
                                uint8_t* d_tokenize_out, double* d_ratio_out);

/* ---- write path --------------------------------------------------------------- */

/* Index.Add (index.go:127, in_memory.go:149-209): n (engine,request) key pairs of one model,
 * m entries added to every key in order.  n==0 or m==0 -> KVIDX_EINVAL. */
int kvidx_add(kvidx_t* idx, uint32_t model, const uint64_t* engine, const uint64_t* request, int64_t n,
              const kvidx_podtier_t* podtier, int32_t m);

/* Index.Evict (index.go:129, in_memory.go:212-260).  Unknown engine key is a silent no-op. */
int kvidx_evict(kvidx_t* idx, uint32_t model, uint64_t engine, const kvidx_podtier_t* podtier, int32_t m);

/* Index.GetRequestKey (index.go:131, in_memory.go:264-270); miss -> KVIDX_ENOENT. */
int kvidx_get_request_key(kvidx_t* idx, uint32_t model, uint64_t engine, uint64_t* request_out);

/* One decoded KV event == one element of Pool.digestEvents' loop (kvevents/pool.go:246-338)
 * after msgpack decoding, getHashAsUint64 (pool.go:343-367) and string interning. */
#define KVIDX_EV_BLOCK_STORED  0
#define KVIDX_EV_BLOCK_REMOVED 1
typedef struct kvidx_event {
    uint8_t  op;            /* KVIDX_EV_*                                                       */
    uint8_t  has_parent;    /* BlockStored: ParentBlockHash != nil                              */
    kvidx_podtier_t podtier;/* {pod of the message, lower(Medium) or "gpu"} (pool.go:258-265)   */
    uint32_t model;
    uint64_t parent_hash;   /* engine hash of the parent block                                  */
    uint64_t hash_off;      /* first engine hash of this event in `hashes`                      */
    uint64_t tok_off;       /* first token id of this event in `tokens` (BlockStored)           */
    uint32_t n_hashes;      /* engine hashes that survived getHashAsUint64                      */
    uint32_t n_tokens;
} kvidx_event_t;

/* Apply a batch of events.  Events of one pod are applied in array order (pool.go:129-144);
 * events of different pods are applied in an unspecified interleaving, as in the reference.
 * BlockStored whose request-key count differs from n_hashes is dropped (in_memory.go:153-155)
 * and counted in *n_dropped_out (may be NULL). */
int kvidx_apply_events(kvidx_t* idx, const kvidx_event_t* ev, int64_t n_events,
                       const uint64_t* hashes, int64_t n_hashes,
                       const uint32_t* tokens, int64_t n_tokens, int64_t* n_dropped_out);

/* ---- KVEvents wire payloads decoded on the device (no reference counterpart) ------------------------------------------
 * Pool.processEvent's msgpack decoding (kvevents/pool.go:177-244, events.go:38-96) of a drained batch of raw vLLM KVEvents
 * messages, run on the GPU: the payloads go in as they came off the wire and come out as the kvidx_event_t batch the write
 * path takes.  The rules are the host mirror's decoder (kvhost_decode_event_batch), and the records are byte-equal to its
 * records stably sorted by pod: EventBatch = [ts, events[], dp_rank?, extra...] (an envelope error drops the message);
 * unknown tags skipped; hashes = uint64- / int64-coded integers and non-empty bins (the last 8 bytes of a longer bin,
 * big-endian); a parent of another type skips the event; tokens truncated to u32; Medium lower-cased (ASCII), none or nil
 * = "gpu"; nesting deeper than 64 drops the message.
 *   bytes / msg_off: CSR of the payloads, message i is bytes[msg_off[i] .. msg_off[i+1]) (msg_off[0] may be non-zero);
 *   msg_pod[i] / msg_model[i]: the interned pod (< max_pods) and model (<= 65535) of message i (one pod per message);
 *   tier table: name t is tier_bytes[tier_off[t] .. tier_off[t+1]), lower-case, compared by length and bytes (no length
 *     cap); 1 <= n_tiers <= 16; gpu_tier: the id of a Medium-less event, or -1 when "gpu" has no id yet;
 *   flags: KVIDX_PAYLOAD_SKIP_UNKNOWN_TIER -- an event whose Medium is not in the table is skipped (what the host decoder
 *     does once the 16 tier ids are taken).  Without it such a batch applies nothing and the call returns KVIDX_ENOENT
 *     with the offending messages flagged: the caller interns their names (kvhost_decode_event_batch over them, in
 *     order) and calls again.  KVIDX_PAYLOAD_STOP_AT_CLEARED -- a batch holding an AllBlocksCleared event applies nothing
 *     and returns KVIDX_ENOENT with its messages flagged; without it the marker decodes to nothing (pool.go:332-333);
 *   msg_flags_out (may be NULL): n_msgs bytes, KVIDX_PAYLOAD_MSG_* per message; written whenever the decode ran;
 *   counts_out (may be NULL): {messages decoded, events, hashes, tokens, queues (pods with events), admitted blocks
 *     (sum of n_tokens / block_size over BlockStored events with hashes: kvcache_index_admissions_total), removed hashes
 *     (kvcache_index_evictions_total), AllBlocksCleared markers}; written whenever the decode ran.
 * Errors: n_msgs < 0, NULL or non-monotone offsets, a NULL array with a non-zero count, an empty tier table, gpu_tier >=
 * n_tiers, unknown flags -> KVIDX_EINVAL; a pod id >= max_pods or a model id > 65535 -> KVIDX_ERANGE; n_msgs == 0 -> 0.
 *
 * kvidx_decode_event_payloads_dev: decode only, device buffers in and out, in exactly the form kvidx_apply_events_dev
 *   takes: events stably sorted by pod (queue q owns d_ev_out[d_queue_off_out[q] .. d_queue_off_out[q+1])), hashes and
 *   tokens in message order.  Capacities are element counts (queue_cap counts offsets: queues + 1); an output below its
 *   total -> KVIDX_ENOSPC with counts_out filled and no output written.  The tier table and counts_out are host memory.
 *   The inputs must be complete when the call is made.  It runs on the handle's write stream, reads its totals back once
 *   (its only wait), and is asynchronous after that: a later kvidx_apply_events_dev and every later read call on the
 *   handle are ordered after it, kvidx_synchronize waits for it.
 * kvidx_apply_event_payloads: host buffers (pinned ones copied in place, pageable ones through pinned chunks): decode and
 *   apply in one synchronous write call, as kvidx_apply_events applies the decoded batch (*n_dropped_out the same).  It
 *   makes room for the decoded batch's BlockStored hashes and holds the write side for the whole call.  A device-resident
 *   caller composes kvidx_decode_event_payloads_dev and kvidx_apply_events_dev.
 * Both work on default, CLOCK, exact-LRU and sharded handles; the ingest rule is kvidx_apply_events': one rank per pod. */
#define KVIDX_PAYLOAD_SKIP_UNKNOWN_TIER 1u
#define KVIDX_PAYLOAD_STOP_AT_CLEARED   2u
#define KVIDX_PAYLOAD_MSG_DECODED       1u   /* the envelope decoded (else the whole message was dropped)        */
#define KVIDX_PAYLOAD_MSG_UNKNOWN_TIER  2u   /* an event names a Medium the tier table lacks                      */
#define KVIDX_PAYLOAD_MSG_CLEARED       4u   /* an AllBlocksCleared event                                          */
#define KVIDX_PAYLOAD_COUNTS            8
int kvidx_decode_event_payloads_dev(kvidx_t* idx, const uint8_t* d_bytes, const int64_t* d_msg_off, int64_t n_msgs,
                                    const uint32_t* d_msg_pod, const uint32_t* d_msg_model, const uint8_t* tier_bytes,
                                    const int64_t* tier_off, uint32_t n_tiers, int32_t gpu_tier, uint32_t flags,
                                    kvidx_event_t* d_ev_out, int64_t ev_cap, int64_t* d_queue_off_out, int64_t queue_cap,
                                    uint64_t* d_hashes_out, int64_t hash_cap, uint32_t* d_tokens_out, int64_t tok_cap,
                                    uint8_t* d_msg_flags_out, int64_t counts_out[KVIDX_PAYLOAD_COUNTS]);
int kvidx_apply_event_payloads(kvidx_t* idx, const uint8_t* bytes, const int64_t* msg_off, int64_t n_msgs, const uint32_t* msg_pod,
                               const uint32_t* msg_model, const uint8_t* tier_bytes, const int64_t* tier_off, uint32_t n_tiers,
                               int32_t gpu_tier, uint32_t flags, uint8_t* msg_flags_out, int64_t counts_out[KVIDX_PAYLOAD_COUNTS],
                               int64_t* n_dropped_out);

/* Drop every entry whose pod is in pod_mask (ceil(max_pods/64) words) and whose tier bit is set in tier_mask
 * (bit t = tier t; 0xFFFF = all tiers); request keys left without entries are removed together with the engine
 * mappings that point at them.  No reference counterpart: it removes the blocks of a pod that has gone away without
 * sending BlockRemoved events.  Survivors keep their order, no key's recency changes, and an engine mapping whose
 * request key was already absent before the call stays (Evict cleans those up, in_memory.go:225-230).  A concurrent
 * reader sees each key before or after its update, as with a sequence of Evict calls.  Synchronous like every write
 * call; works in both LRU modes; the tombstones it leaves are compacted by the usual rebuild policy.
 * All-zero pod_mask or tier_mask == 0 -> KVIDX_EINVAL; sharded handle -> KVIDX_EINVAL (kvidx_shard_remove_pods is the
 * collective form for those).
 * removed_out (may be NULL): {entries, request keys, engine keys} removed. */
int kvidx_remove_pods(kvidx_t* idx, const uint64_t* pod_mask, uint32_t tier_mask, uint64_t removed_out[3]);

/* ---- snapshot / restore (no reference counterpart) ------------------------------------------------------------------
 * The index's contents as a canonical image, and a bulk load of such an image into a fresh handle: an indexer that
 * restarts, is upgraded, moves to another GPU or is replicated keeps the blocks the fleet has already cached (vLLM
 * announces a block once, when it is first stored).  Restoring into a handle created with a larger capacity / table_slots
 * is also how an index outgrows its configuration; a handle with grow_tables grows by itself up to its capacity's table,
 * and needs this only to go beyond it.  Events sent while no indexer ran are not in any image: a block stored
 * or removed in that window is missed until Evict, kvidx_remove_pods or a later event of the same block corrects it.
 *
 * Image format v1, all values little-endian:
 *   header, 64 bytes
 *     0  char[8] "KVIDXSNP"      8  u32 version = 1     12  u32 flags (bit 0: recency section present; others 0)
 *    16  u32 block_size         20  u32 pods_per_key   24  u64 init_hash
 *    32  u64 n_request          40  u64 n_engine
 *    48  u32 pod_span (1 + highest pod id in any entry; 0 if none)   52  u32 model_span (1 + highest model id; 0 if none)
 *    56  u64 0
 *   n_request request records, 32 bytes each: u64 hash, u16 model, u8 count, u8 0, u16 ent[10] -- packed (pod<<4|tier),
 *     oldest -> newest (the slot's physical order, lru Keys()); positions >= count are 0
 *   n_engine engine records, 24 bytes each: u64 engine_hash, u64 request_hash, u16 model, 6 zero bytes
 *   recency section, only with flag bit 0 (exact-LRU handles): one u64 per request record, then one per engine record;
 *     larger = more recent, only the order carries meaning; every value is below 2^63 and no value repeats within a section
 * Request records are strictly ascending by (model, hash), engine records by (model, engine_hash): the image depends
 * only on the contents, not on the table size, insertion history, tombstones or rebuilds.  It holds every resident
 * request key and every engine mapping, including stale mappings whose request key is absent (GetRequestKey returns
 * them, a BlockStored parent resolves through them, Evict cleans them up, in_memory.go:225-230).  Tombstones, counters
 * and tier weights are not part of it: weights are configuration of the restoring process.
 * Size: 64 + 32 R + 24 E (+ 8 (R + E) with recency), R / E = kvidx_get_stats' request_keys / engine_keys.
 *
 * kvidx_snapshot writes the image to buf.  It holds the write side for the whole call (readers keep running; in exact-LRU
 * mode, where readers write recency, they wait) and refreshes no key's recency; a device-resident event batch issued
 * before it is included.  A pageable buffer is filled through pinned staging chunks, a pinned one (kvidx_host_alloc) directly.  buf == NULL or cap below the size -> KVIDX_ENOSPC with *size_out set and nothing written;
 * otherwise *size_out = bytes written.
 * kvidx_restore loads an image into a handle holding no live key (tombstones are dropped first; live keys ->
 * KVIDX_EINVAL).  block_size, init_hash and pods_per_key must equal the handle's (else KVIDX_EINVAL); pod_span > max_pods ->
 * KVIDX_ERANGE; a bad magic or version, a length that does not match the header, or any record failing validation (order,
 * 1 <= count <= pods_per_key, distinct entries with pod < max_pods, zero padding and entries past count, spans equal to
 * the header's) -> KVIDX_EINVAL, and the handle is left as it was.  Every record is validated before any is inserted.
 * table_slots / capacity may differ from the source's; more keys than the write path admits (90 % of a table's slots) ->
 * KVIDX_ENOSPC.  A grow_tables handle first applies its growth rule with L = 0 and I = max(R, E): the 90 % check is made
 * on the size the rule gives, and the (still empty) tables are reallocated at that size once every record has passed
 * validation, so a refused image leaves the handle at its old size.  An exact-LRU handle needs an image with recency (else KVIDX_EINVAL) and keeps the most recent `capacity`
 * keys of each map, as after any write call (found from the sorted recency values: the cut costs one sort, not one table
 * sweep per excess key); a default handle ignores recency, but a repeated value is still malformed.  A concurrent reader sees each key absent
 * or whole.  restored_out (may be NULL): {request keys, engine keys} resident after the call.
 * Both: synchronous like every write call; a sharded handle -> KVIDX_EINVAL (kvidx_shard_snapshot, kvidx_snapshot_merge
 * and kvidx_shard_restore are the collective forms for those). */
int kvidx_snapshot(kvidx_t* idx, void* buf, uint64_t cap, uint64_t* size_out);
int kvidx_restore(kvidx_t* idx, const void* buf, uint64_t len, uint64_t restored_out[2]);

/* ---- device-resident variants (inputs already in HBM; used by bench `value`, by the
 *      multi-GPU router and by callers that keep token buffers on the device) ------- */

/* Use an external CUDA stream (cudaStream_t as void*) for subsequent READ-path calls; NULL restores the
 * handle's own stream.  The write path always uses the handle's own write stream. */
int kvidx_set_stream(kvidx_t* idx, void* cuda_stream);
int kvidx_synchronize(kvidx_t* idx);

/* Score() over device-resident inputs and outputs, launched on the handle's stream.  Batches up to 2048 prompts
 * (KVIDX_COOP_MAX) are a single asynchronous kernel; larger ones run the round pipelines, which wait on the stream ONCE at the start (the number
 * of rounds is the longest prompt's block count, computed on the device) and are asynchronous after that.  Results are
 * complete when the stream reaches the point after the call (kvidx_synchronize, or an event recorded by the caller). */
int kvidx_score_batch_dev(kvidx_t* idx, const uint32_t* d_tok, const int64_t* d_tok_off, int64_t n_prompts,
                          const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter,
                          double* d_scores_out, uint8_t* d_has_keys_out);
int kvidx_score_batch_sparse_dev(kvidx_t* idx, const uint32_t* d_tok, const int64_t* d_tok_off, int64_t n_prompts,
                                 const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter,
                                 uint16_t* d_pods_out, double* d_scores_out, uint8_t* d_cnt_out, uint8_t* d_has_keys_out);
/* kvidx_score_keys[_sparse] over device-resident inputs and outputs: one asynchronous kernel on the handle's stream at
 * every batch size (no wait on the stream), ordered after kvidx_apply_events_dev batches issued before it. */
int kvidx_score_keys_dev(kvidx_t* idx, const uint64_t* d_keys, const int64_t* d_key_off, int64_t n_prompts,
                         const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter,
                         double* d_scores_out, uint8_t* d_has_keys_out);
int kvidx_score_keys_sparse_dev(kvidx_t* idx, const uint64_t* d_keys, const int64_t* d_key_off, int64_t n_prompts,
                                const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter,
                                uint16_t* d_pods_out, double* d_scores_out, uint8_t* d_cnt_out, uint8_t* d_has_keys_out);
/* kvidx_score_turn[_sparse] over device-resident inputs and outputs, asynchronous on the handle's stream, ordered after
 * kvidx_apply_events_dev batches issued before it.  The new keys' offsets are given (d_new_key_off[n_prompts+1], as in
 * kvidx_hash_keys_dev; may be NULL when d_new_keys_out is).  The fused kernel does not wait on the stream; the composed
 * path (see kvidx_score_turn) reads the batch's first and last offsets back to size its scratch. */
int kvidx_score_turn_dev(kvidx_t* idx, const uint64_t* d_keys, const int64_t* d_key_off, const uint32_t* d_tok,
                         const int64_t* d_tok_off, int64_t n_prompts, const uint32_t* d_model, uint32_t model0,
                         const uint64_t* d_filter, double* d_scores_out, uint8_t* d_has_keys_out,
                         const int64_t* d_new_key_off, uint64_t* d_new_keys_out);
int kvidx_score_turn_sparse_dev(kvidx_t* idx, const uint64_t* d_keys, const int64_t* d_key_off, const uint32_t* d_tok,
                                const int64_t* d_tok_off, int64_t n_prompts, const uint32_t* d_model, uint32_t model0,
                                const uint64_t* d_filter, uint16_t* d_pods_out, double* d_scores_out, uint8_t* d_cnt_out,
                                uint8_t* d_has_keys_out, const int64_t* d_new_key_off, uint64_t* d_new_keys_out);
/* kvidx_lookup_hits[_keys] over device-resident inputs and outputs (see there for when they wait on the stream). */
int kvidx_lookup_hits_dev(kvidx_t* idx, const uint32_t* d_tok, const int64_t* d_tok_off, int64_t n_prompts,
                          const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter, uint32_t* d_hits_out);
int kvidx_lookup_hits_keys_dev(kvidx_t* idx, const uint64_t* d_keys, const int64_t* d_key_off, int64_t n_prompts,
                               const uint32_t* d_model, uint32_t model0, const uint64_t* d_filter, uint32_t* d_hits_out);
int kvidx_hash_keys_dev(kvidx_t* idx, const uint32_t* d_tok, const int64_t* d_tok_off, int64_t n_prompts,
                        const uint64_t* d_parent, const uint8_t* d_parent_valid,
                        const int64_t* d_key_off, uint64_t* d_keys_out);
/* Pool.digestEvents for a device-resident batch: events stably sorted by pod (queue q owns
 * d_ev_sorted[d_queue_off[q] .. d_queue_off[q+1])), n_events in all, n_hashes engine hashes behind them.  Asynchronous on
 * the handle's WRITE stream; read calls issued after it returns are ordered after the batch.  d_n_dropped (may be NULL)
 * receives the handle's cumulative dropped-event count once the batch is done. */
int kvidx_apply_events_dev(kvidx_t* idx, const kvidx_event_t* d_ev_sorted, const int64_t* d_queue_off,
                           int64_t n_queues, int64_t n_events, const uint64_t* d_hashes, int64_t n_hashes,
                           const uint32_t* d_tokens, int64_t* d_n_dropped);

/* ---- hash-range sharding across GPUs (one process per GPU) ------------------------
 * The request and engine tables are partitioned by the top bits of the mixed key.  Every rank maps its peers'
 * shards (CUDA IPC over NVLink / NVSwitch peer memory) and the SAME kernels then probe, lock and update slots
 * wherever they live: a Score() probe of a remote key is a 64-byte peer load issued from the fused walk, an
 * Add / Evict is a system-scope CAS on the owner's slot.  No collective sits on the data path; NCCL (or any
 * transport) is only needed to exchange the 192-byte handle blobs once.
 * Ingest rule: all events of one pod must be applied through ONE rank (per-pod order, kvevents/pool.go:129-144).
 * Before a write batch every owner's fill level is read through the mapped memory; a full owner fails the call with
 * KVIDX_ENOSPC (and an insert that still finds no slot is refused and counted), nothing spins. */
#define KVIDX_SHARD_HANDLE_BYTES 192
int kvidx_shard_export(kvidx_t* idx, void* handle_out /* KVIDX_SHARD_HANDLE_BYTES */);
int kvidx_shard_import(kvidx_t* idx, uint32_t rank, const void* handle /* from that rank's kvidx_shard_export */);
/* same-process variant (several GPUs driven by one process, e.g. tests): map `other`'s shard directly */
int kvidx_shard_attach(kvidx_t* idx, uint32_t rank, kvidx_t* other);
/* Drop the tombstones of THIS rank's shard (steady BlockStored / BlockRemoved churn leaves them behind; a write call
 * answers KVIDX_ENOSPC when an owner runs out of room).  Collective by contract: every rank calls it between two barriers
 * of the embedding program, no rank touches the index meanwhile (kvidx.dist.compact_shards does exactly that).  On an
 * unsharded handle it is the compaction the write path runs by itself when needed. */
int kvidx_shard_compact(kvidx_t* idx);

/* Maintenance of a sharded index: pod removal, snapshot and restore.  Collective by contract, like kvidx_shard_compact:
 * every rank calls them between barriers of the embedding program and no rank writes to the index in the meantime (readers
 * keep running and see each key before or after its update).  kvidx.dist.remove_pods_shards / snapshot_shards /
 * restore_shards provide the barriers.  On an unsharded handle each does what its single-process counterpart does.
 *
 * kvidx_shard_remove_pods: kvidx_remove_pods over the whole sharded index, in two phases.  Phase 0 removes the entries
 *   of this rank's request shard and marks the keys it removes in two bitmaps (slots/8 + slots/16 bytes, kept behind the
 *   request slots, so that peers read them through the mapping they already hold); removed_out = {entries, request
 *   keys, 0}.  Phase 1, after every rank's phase 0, drops this rank's engine mappings whose request key phase 0 removed,
 *   on whichever rank owns it; removed_out = {0, 0, engine keys}.  Summed over ranks and phases the counters and the
 *   resulting contents equal kvidx_remove_pods on an unsharded index with the same contents (a stale mapping, whose key
 *   was absent before the call, stays).  KVIDX_EINVAL: phase 1 without a phase 0 on this handle, with other masks than
 *   phase 0, or after a write call (add, evict, apply_events, restore, compaction) on this handle since phase 0; an
 *   unconnected shard; an empty mask; phase > 1.
 * kvidx_shard_snapshot: the v1 image of the request keys and engine mappings THIS rank owns (stale mappings included),
 *   with kvidx_snapshot's buffer conventions.  Each part is a valid image on its own.
 * kvidx_snapshot_merge: host only (no device, no handle).  Merges the parts of disjoint shards into the one canonical
 *   image an unsharded index with the same contents would give: records in (model, hash) order, counts summed,
 *   pod_span / model_span the maxima.  KVIDX_EINVAL: n_parts == 0, a header or length kvidx_restore would refuse, parts
 *   of different block_size / init_hash / pods_per_key, a part with recency (sharded handles never track it, and stamps
 *   of different ranks do not compare), records out of order inside a part, a (model, hash) in two parts.  Every
 *   record is checked before anything is written.  out == NULL or cap below the size -> KVIDX_ENOSPC with *size_out set.
 *   The message is kvidx_last_error(NULL)'s.
 * kvidx_shard_restore: accepts any v1 image -- unsharded, merged, or a single part -- and inserts the records this rank
 *   owns, so the same call restarts a layout and reshards it (1 -> N, N -> M, N -> 1).  The handle must hold no live
 *   key (as kvidx_restore).  Every rank counts the records of every owner over the whole image and checks each owner's
 *   share against 90 % of a shard's slots (the geometry is equal on all shards), so a malformed image or one too
 *   large for any owner (KVIDX_ENOSPC) is refused by every rank before any rank inserts.  Recency is ignored, as on a
 *   default handle (a repeated value is still malformed).  restored_out: {request keys, engine keys} of this shard. */
int kvidx_shard_remove_pods(kvidx_t* idx, const uint64_t* pod_mask, uint32_t tier_mask, uint32_t phase, uint64_t removed_out[3]);
int kvidx_shard_snapshot(kvidx_t* idx, void* buf, uint64_t cap, uint64_t* size_out);
int kvidx_snapshot_merge(const void* const* parts, const uint64_t* lens, uint32_t n_parts, void* out, uint64_t cap, uint64_t* size_out);
int kvidx_shard_restore(kvidx_t* idx, const void* buf, uint64_t len, uint64_t restored_out[2]);

/* The ROUTED form of a sharded Score() (SURVEY 8(e): all-to-all of keys to their owners, slot images back), as three
 * device steps around an exchange the embedding program performs (kvidx.dist.score_alltoall does it with NCCL
 * all_to_all_single).  Provided so that the two designs can be measured against each other; the library's own sharded
 * Score() probes the owner's shard directly from the walk (see above) and needs none of this.
 *   key_owners : owner rank of every key (the routing decision)
 *   probe_slots: owner side -- the 32-byte slot image of every key of THIS shard (all zero: not in the index)
 *   score_slots: origin side -- consecutive-prefix walk + score over the returned images, prompt i owning images
 *                d_key_off[i] .. d_key_off[i+1]; dense rows like kvidx_score_batch_dev. */
int kvidx_key_owners_dev(kvidx_t* idx, const uint64_t* d_keys, const uint32_t* d_model, uint32_t model0, int64_t n, uint8_t* d_owner_out);
int kvidx_probe_slots_dev(kvidx_t* idx, const uint64_t* d_keys, const uint32_t* d_model, uint32_t model0, int64_t n, void* d_slots_out);
int kvidx_score_slots_dev(kvidx_t* idx, const void* d_slots, const int64_t* d_key_off, int64_t n_prompts, const uint64_t* d_filter,
                          double* d_scores_out, uint8_t* d_has_keys_out);

/* ---- introspection ------------------------------------------------------------ */
typedef struct kvidx_stats {
    uint64_t request_keys;      /* resident request keys (lru data.Len())       */
    uint64_t engine_keys;       /* resident engine->request mappings            */
    uint64_t request_tombs;
    uint64_t engine_tombs;
    uint64_t request_slots;
    uint64_t engine_slots;
    uint64_t rebuilds;
    uint64_t kernel_launches;   /* kernels this handle has launched so far      */
    uint64_t rehashed_events;   /* BlockStored events whose parent resolved differently at apply time than when their
                                   keys were precomputed (kernels_write.cuh phase 1): re-hashed in place             */
    uint64_t coalesced_calls;   /* host-buffer Score() calls that were served as part of another call's launch      */
} kvidx_stats_t;
int kvidx_get_stats(kvidx_t* idx, kvidx_stats_t* out);
/* {request keys, engine mappings} dropped by the capacity bound since the handle was created: CLOCK sweeps and exact-LRU
 * evictions.  Evict / BlockRemoved and kvidx_remove_pods are not counted.  On a CLOCK handle every write call reads the
 * device's counters before it runs (waiting for the batches queued before it), so that the tombstones evictions leave
 * are compacted by the usual rebuild also when only kvidx_apply_events_dev writes. */
int kvidx_get_evictions(kvidx_t* idx, uint64_t out[2]);
/* CLOCK mode: {sweeps that evicted, those of them whose hand went past a full turn} since the handle was created, over both
 * maps (a sweep makes at most two turns).  Both kvidx_get_evictions and this read the device's counters without waiting
 * for a write batch in flight: they report the batches completed so far. */
int kvidx_get_sweeps(kvidx_t* idx, uint64_t out[2]);

/* Pod inventory (no reference counterpart): what the index attributes to each pod, counted by one sweep of the request
 * table on the device, and -- with KVIDX_INVENTORY_ENGINE -- a second one of the engine table that makes it an exact dry
 * run of kvidx_remove_pods.  Over the resident request keys k of `model` (a 16-bit id, or KVIDX_ANY_MODEL for all), with
 * E(k) the key's (pod, tier) entries:
 *   entries_out[pod * 16 + tier]  keys with (pod, tier) in E(k)                              max_pods * KVIDX_MAX_TIERS u64
 *   keys_out[pod]                 keys with an entry of the pod on any tier (two tiers of one key count once)   max_pods u64
 *   sole_out[pod]                 keys all of whose entries belong to the pod                                    max_pods u64
 *   sole_engine_out[pod]          engine mappings (of `model`) whose request key is resident and counted in sole_out[pod];
 *                                 all zero without KVIDX_INVENTORY_ENGINE                                        max_pods u64
 *   totals_out                    {request keys, entries, engine mappings, stale engine mappings}; a mapping is stale when
 *                                 no resident request key (model, request hash) exists (Evict cleans those up lazily,
 *                                 in_memory.go:225-230; removal, snapshot and restore keep them, and they count against
 *                                 `capacity`).  The last two are zero without KVIDX_INVENTORY_ENGINE.
 * Any output may be NULL.  With KVIDX_ANY_MODEL, kvidx_remove_pods of the single pod p (all tiers) called right after it
 * returns removed_out = {sum over t of entries_out[p * 16 + t], sole_out[p], sole_engine_out[p]}, and totals_out[0] /
 * totals_out[2] equal kvidx_get_stats' request_keys / engine_keys.
 * A READER: it writes no slot, refreshes no recency stamp and sets no CLOCK reference bit, so taking an inventory never
 * changes what a later eviction picks.  It takes the locks of a read call (not the write side, except on an exact-LRU
 * handle, where every read call does), so writers and other readers keep running.  Ordered after every write call that has
 * returned and after the kvidx_apply_events_dev batches issued before it; synchronous.  With no writer running the counts
 * are exact; beside a writer every key is counted before or after each individual Add / Evict of that key.  Works in all
 * three capacity modes.  On a sharded handle it reports the request keys and engine mappings THIS rank owns (a mapping's
 * request key is probed on whichever rank owns it), needs no phases and no barrier, and the results of all ranks sum to
 * the unsharded answer (kvidx.dist.pod_inventory_shards).
 * All outputs NULL, or a flag other than KVIDX_INVENTORY_ENGINE -> KVIDX_EINVAL; model neither KVIDX_ANY_MODEL nor
 * <= 65535 -> KVIDX_ERANGE. */
#define KVIDX_ANY_MODEL        0xFFFFFFFFu
#define KVIDX_INVENTORY_ENGINE 1u
int kvidx_pod_inventory(kvidx_t* idx, uint32_t model, uint32_t flags, uint64_t* entries_out, uint64_t* keys_out,
                        uint64_t* sole_out, uint64_t* sole_engine_out, uint64_t totals_out[4]);

#ifdef __cplusplus
}
#endif
#endif /* KVIDX_H */
