/*
 * epp_engine.h -- C ABI of libepp_engine.so, the H100-native Endpoint-Picker scoring engine.
 *
 * The reference (llm-d/llm-d-inference-scheduler @ 520af478, pure Go, CGO_ENABLED=0) has NO FFI; this
 * header is the boundary the build introduces (SURVEY.md 8(b)).  Every entry point names the reference
 * interface it replaces (file:line relative to the reference root).  A thin cgo shim (go/eppcuda/,
 * INTEGRATION.md) binds exactly these symbols and keeps the Go plugin interfaces unchanged:
 *
 *   requestcontrol.DataProducer.Produce   pkg/epp/framework/interface/requestcontrol/plugins.go:69-72
 *   scheduling.Filter / Scorer / Picker    pkg/epp/framework/interface/scheduling/plugins.go:59-78
 *   requestcontrol.PreRequest              pkg/epp/framework/interface/requestcontrol/plugins.go:36-39
 *   Scheduler.Schedule                     pkg/epp/scheduling/scheduler.go:54-102
 *
 * Conventions: plain C, no exceptions cross the boundary.  Every function returns int32_t: 0 = EPP_OK,
 * negative = epp_status error; epp_last_error() returns a thread-local message.  The caller owns every
 * host buffer and may free it on return (cgo forbids retaining Go pointers); the engine owns all device
 * memory.  Every entry point is thread-safe (calls on one engine are serialised internally; goroutines
 * should batch requests before calling, see INTEGRATION.md).  Handles are opaque.
 *
 * Streams: the engine launches on its own CUDA streams.  With EPP_BATCH_DEVICE_PTRS (and in the epp_shard_* calls)
 * every device buffer passed IN must be complete before the call (the engine does not wait on the caller's
 * streams); every output is complete when the call returns (EPP_BATCH_ASYNC: when epp_synchronize returns).
 *
 * Endpoint identity: the reference keys servers by NamespacedName strings.  The shim maps each endpoint
 * to a dense SLOT id in [0, max_endpoints); all arrays below are indexed by slot id.
 *
 * Batch semantics (SURVEY.md App. A.8): the reference schedules one request at a time; a batch evaluates
 * all R requests against ONE frozen snapshot (pool state + prefix index).  Index updates (PreRequest)
 * are applied between batches.  The same holds for the no-hit-lru scorer's LRU: every scheduling call (epp_schedule[_topk],
 * epp_schedule_with_match[_topk], the micro-batcher's flushes) scores against the LRU as it stood when the call started
 * and then applies its cold requests' Adds in request order (on the device, in enqueue order for async batches), so cold
 * requests inside one batch do not rotate; epp_score, epp_prefix_match and epp_hash_prompts never update it.  The same
 * holds for the in-flight counters of the inflight-load producer (below).
 *
 * In-flight load (epp_config.inflight_load = 1; the inflight-load-producer, requestcontrol/dataproducer/inflightload/
 * producer.go): the engine keeps per slot the InFlightLoad{Requests, Tokens} that the token-load and active-request
 * scorers read, as int64 counters on the device.  Negative counts are kept (a release on a slot reset since its add).
 *   PreRequest (:110-129): every scheduling call, after its last pick, adds for every request with status 0 one request
 *       and est(L) tokens to each stage that ran and found an endpoint: pick, prefill_pick and the encode pick (only
 *       entry 0 of a first-k list; the same slot picked by two stages counts twice).  Status -1 requests add nothing.
 *       The call scores against the counters as they stood when it started (frozen snapshot, like the no-hit-lru LRU);
 *       async batches apply their adds in enqueue order.
 *   est(L) = i + round(1.5 i), i = max(floor(L / 4), 1), halves away from zero (SimpleTokenEstimator, token_estimator.go
 *       :55-56, 70-71), with L = the request's true prompt length in bytes (lengths[r] / the row length; input_len_bytes[r]
 *       for epp_schedule_with_match, 0 when NULL).  The reference feeds it the whole HTTP body size.
 *   ResponseBody (:131-168): epp_inflight_release; endpoint deletion (:86-97): epp_inflight_reset.  Both are folded on the
 *       host, cost no CUDA call and take effect in call order, before the next scheduling call or epp_inflight_get.
 * Not available in the endpoint-sharded and peer-memory modes.
 *
 * Tie rule: the reference's max-score picker shuffles with math/rand before its stable sort, i.e. it returns a
 * uniformly random member of the arg-max set (picker/maxscore/picker.go:91-102).  The engine always returns the bit
 * pattern of the max score and the size of the set, and as the pick
 *   epp_config.tie_seed == 0: the LOWEST slot id of the set (deterministic; what the parity tests compare), or
 *   epp_config.tie_seed != 0: the member of rank ((mix64(tie_seed ^ mix64(key)) >> 32) * |set|) >> 32 of the set in
 *       ascending slot order, mix64 = the SplitMix64 output function, key = 4 * (ordinal of the request since the
 *       engine was created = epp_stats.n_decisions before the call + index in the batch) + profile index (0 primary /
 *       decode, 1 prefill, 2 encode): uniform over the set like the reference, reproducible by the oracle
 *       (oracle/epp_oracle.c: orc_tie_rank).  Without it every tied request of a batch (cold prompts on a balanced
 *       pool) would land on the same endpoint.  The P/D decider reads the match count of the member picked, as the
 *       reference does (disagg_profile_handler.go:300).  Endpoint-sharded mode uses the lowest slot unless it was set
 *       with epp_shard_set_seeded (see "Seeded ties").
 *
 * Top-k (epp_config.pick_k > 1, epp_schedule_topk): maxscore/picker.go:91-110 shuffles, stable-sorts by score descending
 * and keeps the first k, i.e. the endpoints come out group by group in descending score order and every group of equal
 * scores in uniformly random order.  The engine emits pick j (j = 0 .. k-1) as the member of rank
 *   tie_seed == 0: 0 (the lowest remaining slot), or
 *   tie_seed != 0: ((mix64((tie_seed + j * 0x9E3779B97F4A7C15) ^ mix64(key)) >> 32) * n_j) >> 32
 * among the n_j members of the current group not emitted yet (ascending slot order); pick 0 is the pick of the rule above.
 *
 * Exploration draw of the prefix-cache-affinity-filter (rand.Float64() < explorationProbability,
 * filter/prefixcacheaffinity/plugin.go:113): u = (mix64((tie_seed ^ 0xA0761D6478BD642F) ^ mix64(key)) >> 11) * 2^-53 when
 * tie_seed != 0; with tie_seed == 0 (the deterministic mode) the filter never explores.
 *
 * Random pickers (epp_profile_cfg.picker): the draw u = (mix64((tie_seed ^ 0xE7037ED1A0B428DB) ^
 * mix64(key)) >> 11) * 2^-53 (same key as the tie rule) is made for every tie_seed, 0 included.  The population is the
 * profile's candidates c_0 < c_1 < ... < c_{n-1} (ascending slot order, after the affinity filter); s(c) is c's weighted score.
 *   random-picker: c_min(floor(u * n), n - 1)  (u * n rounded to nearest).
 *   weighted-random-picker: P(c_i) = s_i+ / W.  s+ = s when 0 < s < +inf (times sigma = 2^-128 when the profile's
 *       sum of |weight| exceeds 2^960, which keeps every sum finite; exact, a power of two), 0 when s <= 0 or NaN.
 *       The sequence folded is: the request's EXPLICIT candidates (matchBlocks > 0, or the request's LoRA adapter is
 *       active / waiting on them; under a narrowing affinity filter every candidate) with their own s+, and between
 *       them the GAPS, runs [a, b) of the other candidates, whose mass is wcum[b] - wcum[a], wcum[i] = the left fold
 *       (+0.0 first, round-to-nearest) of s+(base) over c_0 .. c_{i-1}, base = the score with no match (computed once
 *       per pool snapshot / no-hit-lru update).  W = the left fold of that sequence.
 *       - some candidate scores +inf: the pick is the one of rank min(floor(u * N), N - 1) among the N +inf candidates;
 *       - else W == 0 (every score <= 0): the random-picker's pick (weightedrandom/picker.go:113-116);
 *       - else t = u * W (rounded; t >= W becomes the largest double below W); the pick is the first item whose
 *         running sum exceeds t -- inside a gap [a, b) that followed the running sum S, the first c_i (a <= i < b) with
 *         S + (wcum[i+1] - wcum[a]) > t (the last one reproduces the gap's own sum, so the search stays inside it).
 *       The draw has the distribution of A-Res's largest key (picker.go:121-154) and costs O(explicit + log n).
 *   First k (pick_k > 1): draw j = 0 .. min(k, n) - 1 is the draw above with the seed tie_seed + j * 0x9E3779B97F4A7C15 over
 *       the candidates not emitted yet (the random rank counts only those); the emitted ones stay in the weighted sequence
 *       as explicit items of mass 0, so once the positive scores are used up W == 0 and the rest follow in uniform random
 *       order.  Pick 0 is the one-endpoint pick.
 */
#ifndef EPP_ENGINE_H
#define EPP_ENGINE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define EPP_API __attribute__((visibility("default")))
#else
#define EPP_API
#endif

#define EPP_ABI_VERSION 5
#define EPP_MAX_SCORERS 8
#define EPP_NO_ENDPOINT 0xFFFFFFFFu

typedef struct epp_engine epp_engine;

typedef enum {
    EPP_OK = 0,
    EPP_ERR_INVALID = -1,     /* bad argument / configuration                                       */
    EPP_ERR_CUDA = -2,        /* a CUDA runtime call failed (message has the CUDA error string)     */
    EPP_ERR_NO_DEVICE = -3,   /* no usable CUDA device: the engine NEVER falls back to a CPU path   */
    EPP_ERR_CAPACITY = -4,    /* batch / index larger than the configured or available capacity     */
    EPP_ERR_STATE = -5,       /* call order violation (e.g. schedule before pool_set)               */
    EPP_ERR_NCCL = -6
} epp_status;

/* Scorer kinds (plugin type strings of the reference in comments). */
typedef enum {
    EPP_SCORER_PREFIX = 0,     /* "prefix-cache-scorer"          scorer/prefix/plugin.go:95-117               */
    EPP_SCORER_KV_UTIL = 1,    /* "kv-cache-utilization-scorer"  scorer/kvcacheutilization/kvcache_utilization.go:76-82 */
    EPP_SCORER_QUEUE = 2,      /* "queue-scorer"                 scorer/queuedepth/queue.go:78-108            */
    EPP_SCORER_LOAD_AWARE = 3, /* "load-aware-scorer"            scorer/loadaware/load_aware.go:84-100; param = threshold */
    EPP_SCORER_EXTERNAL = 4,   /* host-computed per-endpoint column (param = column index): lets the Go
                                  side keep any other Scorer (lora-affinity, session-affinity, ...) */
    EPP_SCORER_RUNNING = 5,    /* "running-requests-size-scorer" scorer/runningrequests/runningrequest.go:78-108 */
    EPP_SCORER_TOKEN_LOAD = 6, /* "token-load-scorer"            scorer/tokenload/token_load.go:84-112; column = ext column
                                  holding InFlightLoad.Tokens (ignored with inflight_load: the engine's counters),
                                  param = queueThresholdTokens (<= 0: 4194304)                                    */
    EPP_SCORER_ACTIVE_REQUEST = 7, /* "active-request-scorer"    scorer/activerequest/active_request.go:140-173; column = ext
                                  column holding InFlightLoad.Requests (ignored with inflight_load: the engine's
                                  counters), param = maxBusyScore (outside [0,1]: 1.0),
                                  param2 = idleThreshold (< 0: 0)                                                 */
    EPP_SCORER_LORA_AFFINITY = 8, /* "lora-affinity-scorer"      scorer/loraaffinity/lora_affinity.go:76-100; the adapter is the
                                  request's model id; residency comes from epp_pool_set_lora                     */
    EPP_SCORER_NO_HIT_LRU = 9, /* "no-hit-lru-scorer"          scorer/nohitlru/no_hit_lru.go:259-321; param = lruSize (<= 0:
                                  1024), the same in every profile that lists it (they share ONE LRU).  A request is cold
                                  for a profile when no candidate holds a block of its prompt (the engine's own match is
                                  the producer).  Every scheduling call scores against the LRU as it stood when the call
                                  started and then Adds, for each cold request in request order, its pick and its
                                  prefill pick (PreRequest, :279-321): inside one batch cold requests do not rotate.
                                  Not available in the endpoint-sharded and peer-memory modes.                    */
    EPP_SCORER_LATENCY = 10,   /* "latency-scorer"               scorer/latency/plugin.go:144-395; reads the request's latency
                                  predictions, configured by epp_latency_profile_set (see "Latency predictions")  */
    EPP_SCORER_CONTEXT_LENGTH = 11 /* "context-length-aware"     scorer/contextlengthaware/context_length_aware.go; scorer and
                                  filter, configured by epp_context_length_set (see "Context length")            */
} epp_scorer_kind;

/* Value of the llm-d.ai/role label (filter/bylabel/roles.go:25-44). */
typedef enum {
    EPP_ROLE_NONE = 0,         /* label absent */
    EPP_ROLE_DECODE = 1,
    EPP_ROLE_PREFILL = 2,
    EPP_ROLE_PREFILL_DECODE = 3,
    EPP_ROLE_BOTH = 4,
    EPP_ROLE_ENCODE = 5,
    EPP_ROLE_ENCODE_PREFILL = 6,
    EPP_ROLE_ENCODE_PREFILL_DECODE = 7,
    EPP_ROLE_OTHER = 8         /* label present, value not in the tables */
} epp_role;

/* Role filters (filter/bylabel/roles.go:46-70, filter.go:104-117). */
typedef enum {
    EPP_FILTER_NONE = 0,
    EPP_FILTER_DECODE = 1,     /* "decode-filter": decode, prefill-decode, both, encode-prefill-decode, or no label */
    EPP_FILTER_PREFILL = 2,    /* "prefill-filter": prefill, encode-prefill, prefill-decode, both, e-p-d; label required */
    EPP_FILTER_ENCODE = 3      /* "encode-filter": encode, encode-prefill, e-p-d; label required */
} epp_filter_kind;

/* Profile handlers. */
typedef enum {
    EPP_HANDLER_SINGLE = 0,    /* profilehandler/single/single_profile_handler.go:66-99     */
    EPP_HANDLER_DISAGG = 1     /* profilehandler/disagg/disagg_profile_handler.go:246-354 (decode -> decider -> prefill) */
} epp_handler_kind;

typedef struct {
    int32_t kind;              /* epp_scorer_kind */
    int32_t column;            /* ext column read by TOKEN_LOAD / ACTIVE_REQUEST (raw attribute values, not scores) */
    double weight;             /* WeightedScorer.weight, scheduling/weighted_scorer.go:24-40 */
    double param;
    double param2;
} epp_scorer_cfg;

/* Pickers (the last plugin of a profile).  Under the random pickers an epp_decision's score is the pick's own weighted
 * score (bit-exact), tie_count the size of the population the draw was made from (the profile's candidates), and
 * match_blocks / the P/D decider read the pick's match count, as under max-score.  See "Random pickers" above. */
typedef enum {
    EPP_PICKER_MAX_SCORE = 0,        /* "max-score-picker"       picker/maxscore/picker.go:87-115                    */
    EPP_PICKER_RANDOM = 1,           /* "random-picker"          picker/random/picker.go:86-104                      */
    EPP_PICKER_WEIGHTED_RANDOM = 2   /* "weighted-random-picker" picker/weightedrandom/picker.go:111-155             */
} epp_picker_kind;

/* One SchedulerProfile (scheduling/scheduler_profile.go:117-128): role filter -> [prefix-cache-affinity-filter] ->
 * scorers IN ORDER -> picker. */
typedef struct {
    int32_t filter;            /* epp_filter_kind */
    int32_t n_scorers;
    epp_scorer_cfg scorers[EPP_MAX_SCORERS];
    /* "prefix-cache-affinity-filter" after the role filter (filter/prefixcacheaffinity/plugin.go:105-151): with
     * probability 1 - exploration_probability the candidates are narrowed to the STICKY endpoints (matchBlocks /
     * totalBlocks >= affinity_threshold) unless there is none, or the best predicted TTFT among them exceeds the best
     * among the others by more than max_ttft_penalty_ms.  The scorers then normalise over the narrowed set
     * (queue / running min-max, active-request max).  affinity_threshold <= 0: no such filter (plugin.go:108).
     * The reference's defaults are 0.80 / 0.01 / 5000 (plugin.go:62-66). */
    double affinity_threshold;
    double exploration_probability;    /* [0, 1]                                                              */
    double max_ttft_penalty_ms;        /* >= 0; 0 = always stick                                              */
    int32_t ttft_column;               /* ext column holding LatencyPredictionInfo.TTFT per endpoint; < 0 = no
                                          prediction attached (the gate then never breaks stickiness, :169-180) */
    int32_t picker;                    /* epp_picker_kind of the profile (0 = max-score)                      */
} epp_profile_cfg;

/* Mirrors the EndpointPickerConfig fields that define this path (apix/config/v1alpha1, and
 * approximateprefix/types.go:78-142 for the prefix producer defaults). */
typedef struct {
    uint32_t struct_size;          /* sizeof(epp_config), for ABI evolution                              */
    int32_t device;                /* CUDA device ordinal                                                */
    int32_t max_endpoints;         /* slot-id capacity                                                   */
    int32_t block_size_tokens;     /* blockSizeTokens (default 16); block bytes = 4 * this (hashing.go:49) */
    int32_t max_prefix_blocks;     /* maxPrefixBlocksToMatch (default 256)                               */
    int32_t lru_capacity_per_server; /* lruCapacityPerServer (default 31250)                             */
    int32_t handler;               /* epp_handler_kind                                                   */
    int32_t always_disagg;         /* always-disagg-pd-decider (always_disagg_pd_decider.go:48-50)        */
    int64_t non_cached_tokens;     /* prefix-based-pd-decider nonCachedTokens (0 disables)               */
    int32_t n_ext_cols;            /* number of EPP_SCORER_EXTERNAL columns                              */
    int32_t pick_k;                /* max-score-picker maxNumOfEndpoints (picker/common.go:36, maxscore/picker.go:104-115);
                                      0 or 1 = one endpoint; 2..64: epp_schedule_topk / epp_schedule_with_match_topk also
                                      return the k best of every profile that ran                                     */
    epp_profile_cfg primary;       /* the single profile, or the decode profile under EPP_HANDLER_DISAGG */
    epp_profile_cfg prefill;       /* the prefill profile (EPP_HANDLER_DISAGG only)                      */
    epp_profile_cfg encode;        /* the encode profile (EPP_HANDLER_DISAGG with encode_enabled != 0):
                                      disagg_profile_handler.go:284-295                                   */
    uint64_t tie_seed;             /* seed of every reproducible random draw (ties, top-k order, exploration); 0 = the
                                      deterministic mode: lowest slot of the arg-max set, no exploration              */
    int32_t encode_enabled;        /* an "encode" profile + always-disagg-multimodal-decider are configured */
    int32_t index_commit_interval_us; /* 0: every scheduling call first makes all earlier index updates (epp_index_add,
                                      epp_index_add_picked) visible -- exact sequential semantics, what the parity tests use;
                                      > 0: a scheduling call does that only if the last one that did is at least this long
                                      ago, i.e. picks become visible to later requests with a bounded delay, like the
                                      reference's asynchronous PreRequest (approximateprefix/plugin.go:189-194).
                                      epp_index_commit / epp_index_get always commit.                              */
    int32_t inflight_load;         /* 1: the inflight-load producer runs on the device (see "In-flight load" above) and
                                      every TOKEN_LOAD / ACTIVE_REQUEST scorer reads its counters (`column` ignored);
                                      0: off (default)                                                              */
    uint32_t reserved0;
    uint64_t reserved1;
} epp_config;

/* One routing decision (32 bytes).  status: 0 = ok, -1 = no endpoint available for the primary profile
 * (Schedule error: scheduler_profile.go:119-121 / disagg_profile_handler.go:335-338), EPP_STATUS_REJECTED (-2) = an
 * admitter rejected the request (see "Admission"). */
typedef struct {
    int32_t status;
    uint32_t pick;             /* primary (decode) pick: lowest slot id of the arg-max set, or EPP_NO_ENDPOINT */
    double score;              /* max weighted score (bit-exact vs the reference arithmetic)        */
    uint32_t prefill_pick;     /* prefill pick, EPP_NO_ENDPOINT when the prefill stage did not run / found nobody */
    uint32_t tie_count;        /* size of the primary arg-max set                                   */
    int32_t total_blocks;      /* PrefixCacheMatchInfo.totalBlocks (= number of prefix hashes)      */
    int32_t match_blocks;      /* PrefixCacheMatchInfo.matchBlocks of the primary pick              */
} epp_decision;

/* Optional second record per decision (40 bytes): the other stages of the disagg handler, for the shim's
 * SchedulingResult.ProfileResults, tests and metrics. */
typedef struct {
    double prefill_score;
    uint32_t prefill_tie_count;
    uint32_t prefill_ran;      /* the P/D decider asked for the prefill stage                        */
    double encode_score;
    uint32_t encode_pick;      /* encode pick, EPP_NO_ENDPOINT when the stage did not run / found nobody */
    uint32_t encode_tie_count;
    uint32_t encode_ran;       /* the encode decider asked for the encode stage (multimodal request) */
    uint32_t reserved;
} epp_decision_detail;

#define EPP_BATCH_DEVICE_PTRS 1u   /* data / offsets / model_ids and all outputs are DEVICE pointers */
#define EPP_BATCH_ASYNC 2u         /* epp_schedule + DEVICE_PTRS: enqueue and return; outputs (and epp_stats.last_*)
                                    * are complete after epp_synchronize().  Batches enqueue in call order.       */
#define EPP_BATCH_LENGTHS_EXCEED_ROWS 4u /* lengths[r] may exceed the row offsets[r+1] - offsets[r]: a row then holds only the
                                    * first min(lengths[r], max_prefix_blocks * block_size_tokens * 4) bytes of its prompt --
                                    * everything hashPrompt reads (hashing.go:63-66) -- while lengths[r] stays the prompt's
                                    * true length (input of the P/D decider).  Saves shipping the tail of long prompts.  */

/* A batch of prompts.  Prompt r is data[offsets[r] .. offsets[r+1]) (bytes), or data[offsets[r] .. offsets[r] +
 * lengths[r]) when `lengths` is given (lets ragged prompts START on 32-byte boundaries, which selects the 256-bit-load
 * kernel; offsets[r] + lengths[r] <= offsets[r+1] must hold).  A uint32 token array viewed as little-endian bytes is
 * a prompt with 4 bytes/token (hashing.go:49, types.go:113). */
typedef struct {
    int64_t n_requests;
    const void *data;
    const uint64_t *offsets;       /* [n_requests+1]; NULL => uniform: prompt r = data[r*uniform_len ..) */
    uint64_t uniform_len;
    const uint32_t *model_ids;     /* [n_requests] ids from epp_model_register; NULL => model 0       */
    uint32_t flags;                /* EPP_BATCH_* */
    uint32_t reserved;
    const uint64_t *lengths;       /* [n_requests] or NULL */
    const uint8_t *multimodal;     /* [n_requests] or NULL: != 0 = the request carries image / video / audio content blocks
                                      (hasMultimodalContent, disagg/multimodal_helpers.go): input of the encode decider */
} epp_batch;

typedef struct {
    uint64_t n_batches, n_decisions;
    uint64_t index_pairs, index_hashes, index_slots;   /* device table occupancy */
    double last_h2d_ms, last_kernels_ms, last_d2h_ms;  /* CUDA-event times of the last batch */
    double last_hash_ms, last_match_pick_ms;
    uint64_t last_kernel_launches;
    uint64_t device_bytes;
    /* device-pointer batches only: CUDA-event time of each kernel of the last batch on the launch stream.
     * [0] prompt lengths  [1] block digests (dominant: reads every token once)  [2] chain  [3] match+score+pick
     * [4] the no-hit-lru update after the picks (engines with that scorer; 0 otherwise)
     * [5] the in-flight counters' update after the picks (engines with inflight_load; 0 otherwise)
     * [6] the subset pick kernel (calls with restricted requests; 0 otherwise)
     * [7] the admission kernel (calls with a row an admitter can reject, see "Admission"; 0 otherwise) */
    double last_kernel_ms[8];
    /* algorithmic work of the last batch (SURVEY.md 8(d)): table probes P = sum_r min(stop_r+1, B_r) and
     * postings consumed M = sum_r sum_{i<stop_r} |servers(h_i)| */
    uint64_t last_probes, last_postings;
    /* write side (index_store.cu): the last epp_index_add_picked / queued-Add flush and the last read-table build */
    double last_index_apply_ms;        /* Add + eviction kernels incl. their two small read-backs (host clock)   */
    double last_index_build_ms;        /* export of the inverted map + bulk build of the read table (host clock) */
    uint64_t last_index_items;         /* hashes added by the last applied batch                               */
    uint64_t last_index_launches;      /* kernels launched by it                                               */
    uint64_t last_index_patched;       /* 1: the last commit patched the read table from the change log; 0: bulk build */
    /* bytes of hash rows k_hash_fused stored for the last synchronous device batch (8 per hash; a Schedule batch without
     * keep_hashes stores each row only up to the first block the index cannot hold, EPP_HASH_TRIM; 0 when another hash
     * kernel ran) */
    uint64_t last_hash_bytes_stored;
    /* prompt bytes k_hash_fused read for the last synchronous device batch or epp_hash_prompts call: every byte the
     * hashes need, or, for a trimmed Schedule batch, each prompt only up to shortly past its first absent block
     * (EPP_HASH_SKIP); 0 when another hash kernel ran */
    uint64_t last_prompt_bytes_read;
} epp_stats;

/* ---- lifecycle --------------------------------------------------------------------------------- */
EPP_API int32_t epp_abi_version(void);
EPP_API const char *epp_last_error(void);
/* plugin factories + EndpointPickerConfig (framework/interface/plugin/registry.go:25-30). */
EPP_API int32_t epp_engine_create(const epp_config *cfg, epp_engine **out);
EPP_API int32_t epp_engine_destroy(epp_engine *h);
EPP_API void epp_config_default(epp_config *cfg);   /* types.go:136-142 + config/loader/defaults.go:47-49,78-87 */

/* Pinned host staging buffers for the shim (C memory, so cgo may keep them). */
EPP_API int32_t epp_host_alloc(size_t bytes, void **out);
EPP_API int32_t epp_host_free(void *p);

/* request.TargetModel (+ Body.CacheSalt()): registers the seed h_{-1} = XXH64(model || salt)
 * (hashing.go:71-78), computed on the device.  Returns a small id used in epp_batch.model_ids. */
EPP_API int32_t epp_model_register(epp_engine *h, const uint8_t *model, size_t model_len, const uint8_t *salt,
                           size_t salt_len, uint32_t *out_model_id);
EPP_API int32_t epp_model_seed(epp_engine *h, uint32_t model_id, uint64_t *out_seed);

/* ---- pool state (fwkdl.Metrics framework/interface/datalayer/metrics.go:26-42, EndpointMetadata.Labels) --
 * Replaces the snapshot (called by the 50 ms scrape loop).  n entries; ids[i] is the slot id of entry i;
 * slots not listed are absent from the pool.  role: epp_role.  ext may be NULL when n_ext_cols == 0, else
 * [n_ext_cols][n].  Also derives, ON THE DEVICE, every request-independent quantity of the scorers
 * (queue min/max over each profile's candidates, per-scorer contributions, ordered base sums). */
EPP_API int32_t epp_pool_set(epp_engine *h, int32_t n, const uint32_t *ids, const uint8_t *role, const double *kv_usage,
                     const int32_t *waiting, const int32_t *running, const double *ext);

/* LoRA adapter residency for EPP_SCORER_LORA_AFFINITY (fwkdl.Metrics.ActiveModels / WaitingModels / MaxActiveModels,
 * scorer/loraaffinity/lora_affinity.go:76-100).  n entries by slot id: MaxActiveModels and len(ActiveModels) +
 * len(WaitingModels); n_members triples (endpoint slot, model id from epp_model_register, state 1 = active /
 * 2 = waiting) list where each adapter is resident.  Replaces the previous LoRA state and re-derives the scorer terms;
 * call it after epp_pool_set of the same scrape (slots absent here have capacity 0 and nothing resident). */
EPP_API int32_t epp_pool_set_lora(epp_engine *h, int32_t n, const uint32_t *ids, const int32_t *max_active_models,
                          const int32_t *n_models_loaded, int64_t n_members, const uint32_t *member_ep,
                          const uint32_t *member_model, const uint8_t *member_state);

/* ---- Label filters (filter/bylabel/selector.go:34-101 "label-selector-filter" / deprecated "by-label-selector", and
 * filter/bylabel/filter.go:34-117 "by-label") ---------------------------------------------------------------------------
 * Each profile may hold label requirements besides its role filter.  A slot is a candidate of the profile when it is in
 * the pool, passes the role filter and matches EVERY requirement (AND; an empty list keeps everything).  The chain is
 * [role and label filters, any order] [prefix-cache-affinity-filter]: label and role filters are pure per-endpoint
 * predicates, so their order does not matter; a label filter after the affinity filter is not supported.  Labels are the
 * endpoint's EndpointMetadata.Labels; a requirement on key k reads labels[k]:
 *   EPP_LABEL_IN            k present and its value among `values` (an absent key never matches, even with "" listed)
 *   EPP_LABEL_NOT_IN        k absent, or its value not among `values` (an absent key always matches)
 *   EPP_LABEL_EXISTS        k present (any value, "" included)
 *   EPP_LABEL_DOES_NOT_EXIST k absent
 *   EPP_LABEL_BY_LABEL      by-label with allowsNoLabel = false: labels[k] among `values`, where an ABSENT key reads as ""
 *                           (filter.go:108-111), so "" among `values` also admits slots without the key
 *   EPP_LABEL_BY_LABEL_OR_ABSENT  by-label with allowsNoLabel = true: k absent, or labels[k] among `values`
 * matchLabels {k: v} is k In [v].  IN / NOT_IN / BY_LABEL need at least one value, EXISTS / DOES_NOT_EXIST take none,
 * BY_LABEL_OR_ABSENT any number.  The IN / NOT_IN rules for absent keys and the key / value syntax come from
 * k8s.io/apimachinery's Requirement.Matches and validation, which the reference does not pin in its own tests; this
 * engine states them as its contract.  The C side checks structure only (a key is non-empty and holds no '=' or newline,
 * a value holds no newline); the shims validate label syntax as LabelSelectorAsSelector does.
 * Caps: EPP_LABEL_MAX_REQS requirements per profile, 16 distinct keys over all profiles, 62 distinct named values per key.
 * Over a cap is EPP_ERR_INVALID.  Every rejected call changes no state.
 * Cost: the filters are decided when the pool kernels derive each profile's candidates (per snapshot), not per request. */
#define EPP_LABEL_MAX_REQS 32
typedef enum {
    EPP_LABEL_IN = 0,
    EPP_LABEL_NOT_IN = 1,
    EPP_LABEL_EXISTS = 2,
    EPP_LABEL_DOES_NOT_EXIST = 3,
    EPP_LABEL_BY_LABEL = 4,            /* by-label, allowsNoLabel = false: value in the set, an absent key reads "" */
    EPP_LABEL_BY_LABEL_OR_ABSENT = 5   /* by-label, allowsNoLabel = true                                          */
} epp_label_op;
typedef struct {
    const char *key;                   /* NUL-terminated                                                           */
    int32_t op;                        /* epp_label_op                                                             */
    int32_t n_values;
    const char *const *values;         /* [n_values] NUL-terminated; duplicates allowed                            */
} epp_label_req;
/* profile: 0 primary / decode, 1 prefill, 2 encode (a profile the configuration has).  Replaces that profile's label
 * requirements.  Only before the engine's first successful epp_pool_set / epp_pool_set_labels (EPP_ERR_STATE after). */
EPP_API int32_t epp_label_filters_set(epp_engine *h, int32_t profile, int32_t n, const epp_label_req *reqs);
/* EndpointMetadata.Labels of the listed slots: text[offsets[i] .. offsets[i+1]) holds entry i's labels as "key=value\n"
 * lines (each split at its first '=').  offsets: [n + 1], non-decreasing.  Replaces every slot's labels (slots not listed
 * have none) and re-derives every profile, as epp_pool_set does; batches enqueued before the call decide on the labels
 * they were enqueued under, and epp_pool_set alone keeps the labels.  Rejected: a NULL array, a slot id >= max_endpoints
 * or listed twice, a line without '=' or newline, an empty key, a key repeated within one slot.  On an engine without
 * label requirements the call only validates: nothing on the device reads labels. */
EPP_API int32_t epp_pool_set_labels(epp_engine *h, int32_t n, const uint32_t *ids, const uint64_t *offsets,
                                    const uint8_t *text);

/* ---- prefix index write side (approximateprefix/indexer.go:52-83, 105-115, 167-182; plugin.go:164-211) --
 * The LRU bookkeeping lives in HBM (index_store.cu): epp_index_add calls are queued and applied as ONE device batch,
 * in call order, by the next commit / lookup / remove; epp_index_add_picked never leaves the device.  The read table
 * is rebuilt on the device by epp_index_commit (also called implicitly by the next lookup when dirty). */
EPP_API int32_t epp_index_add(epp_engine *h, uint32_t ep, int32_t n, const uint64_t *hashes, int32_t num_gpu_blocks);
EPP_API int32_t epp_index_remove_endpoint(epp_engine *h, uint32_t ep);
/* CleanUpInactivePods (approximateprefix/plugin.go:99-122): RemovePod for every indexed endpoint NOT in active_ids. */
EPP_API int32_t epp_index_retain_endpoints(epp_engine *h, int32_t n, const uint32_t *active_ids);
/* Bulk-replace the index with a frozen snapshot of UNIQUE-or-not (hash, endpoint) pairs (host pointers);
 * bypasses LRU bookkeeping.  Duplicates are removed on the device. */
EPP_API int32_t epp_index_load_snapshot(epp_engine *h, uint64_t n_pairs, const uint64_t *hashes, const uint32_t *eps);
EPP_API int32_t epp_index_commit(epp_engine *h);
/* indexer.Get (indexer.go:86-102), read from the DEVICE table; returns the set size in *out_n. */
EPP_API int32_t epp_index_get(epp_engine *h, uint64_t hash, uint32_t *out_eps, int32_t cap, int32_t *out_n);

/* ---- a1: hashPrompt (approximateprefix/hashing.go:35-99) -----------------------------------------
 * out_hashes: [R][max_prefix_blocks] (row-major, unused tail undefined); out_nblocks: [R]. */
EPP_API int32_t epp_hash_prompts(epp_engine *h, const epp_batch *batch, uint64_t *out_hashes, int32_t *out_nblocks);

/* ---- a1-a4: Produce (approximateprefix/plugin.go:135-160) -- plugin-parity mode ---------------------
 * out_match: dense [R][max_endpoints] matchBlocks (0 for unmatched); out_total: [R] totalBlocks. */
EPP_API int32_t epp_prefix_match(epp_engine *h, const epp_batch *batch, int32_t *out_match, int32_t *out_total);

/* ---- a5-a9: Scorer.Score / runScorerPlugins (scheduler_profile.go:151-174) -- plugin-parity mode ----
 * match: [R][max_endpoints], total: [R] (as produced by epp_prefix_match or injected by a test).
 * profile: 0 = primary, 1 = prefill.  scorer_index >= 0: raw column of that scorer (what Scorer.Score
 * returns, 0 for non-candidates); -1: weighted, clamped, ordered sum (-1.0 for filtered-out endpoints).
 * out_scores: [R][max_endpoints].  flags: EPP_BATCH_DEVICE_PTRS.
 * model_ids: [R] model (= LoRA adapter) of each request, NULL = model 0 (only lora-affinity reads it). */
EPP_API int32_t epp_score(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                  const uint32_t *model_ids, int32_t profile, int32_t scorer_index, double *out_scores, uint32_t flags);

/* ---- a1-a14 fused: Scheduler.Schedule for a batch (scheduling/scheduler.go:54-102) ---------------
 * out: [R]; detail: [R] or NULL; keep_hashes != 0 keeps the batch's prefix hashes resident on the device
 * for epp_index_add_picked (the PluginState stash of plugin.go:150-157).  Without it the engine may store each row
 * only up to the first block the index cannot hold (EPP_HASH_TRIM). */
EPP_API int32_t epp_schedule(epp_engine *h, const epp_batch *batch, epp_decision *out, epp_decision_detail *detail,
                     int32_t keep_hashes);

/* Same decision logic with PrefixCacheMatchInfo injected by the caller (how the reference's own scheduler
 * tests drive it: disagg/scheduler_test.go:264-268): match [R][max_endpoints], total [R],
 * model_ids [R] or NULL, input_len_bytes [R] (prompt length for the P/D decider), block_size_tokens override
 * (0 = config). */
EPP_API int32_t epp_schedule_with_match(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                const uint32_t *model_ids, const int64_t *input_len_bytes, int32_t block_size_tokens, epp_decision *out,
                                epp_decision_detail *detail, uint32_t flags);

/* maxNumOfEndpoints > 1 (maxscore/picker.go:104-115): the k = epp_config.pick_k best endpoints of every profile that ran
 * for the request, in picker order (see "Top-k" above); rows are padded with EPP_NO_ENDPOINT / 0.0 when a profile has
 * fewer candidates than k or did not run.  primary[r*k] == out[r].pick, prefill[r*k] == out[r].prefill_pick,
 * encode[r*k] == detail[r].encode_pick.  Host pointers for host batches, device pointers with EPP_BATCH_DEVICE_PTRS;
 * any of the arrays may be NULL. */
typedef struct {
    uint32_t struct_size;          /* sizeof(epp_topk_out)                                              */
    int32_t k;                     /* row stride; must equal epp_config.pick_k                           */
    uint32_t *primary;             /* [R][k] slot ids                                                    */
    double *primary_scores;        /* [R][k] their weighted scores                                       */
    uint32_t *prefill;             /* [R][k]                                                             */
    uint32_t *encode;              /* [R][k]                                                             */
} epp_topk_out;
EPP_API int32_t epp_schedule_topk(epp_engine *h, const epp_batch *batch, epp_decision *out, epp_decision_detail *detail,
                          int32_t keep_hashes, const epp_topk_out *topk);
EPP_API int32_t epp_schedule_with_match_topk(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                     const uint32_t *model_ids, const int64_t *input_len_bytes, int32_t block_size_tokens,
                                     epp_decision *out, epp_decision_detail *detail, uint32_t flags,
                                     const epp_topk_out *topk);

/* ---- Endpoint subsets (requestcontrol/candidates.go:98-167, director.go:222-243) -------------------------------------
 * When Envoy attaches x-gateway-destination-endpoint-subset metadata, Scheduler.Schedule receives only that subset's
 * endpoints.  A request with a subset is decided exactly as the reference decides it when Schedule is called with the
 * subset's endpoints:
 *   - Candidates: every profile's candidates are the subset's slots that are in the pool and pass the profile's role
 *     filter; the affinity filter, scorers and picker run over those.  Subset slots not in the pool are ignored.
 *   - Everything normalised over "the candidates" uses the narrowed set: the queue / running min-max, the active-request
 *     max, the no-hit-lru cold test (no SUBSET candidate holds a block) and its cold ranks (never-used index in slot
 *     order, neverUsedCount + the position in the engine's one LRU, over totalEndpoints = |candidates|), the affinity
 *     filter's len(endpoints) <= 1 gate and its sticky / TTFT sets, tie_count, the tie rank, the first-k ranks and the
 *     random pickers' population.
 *   - The prefix match is NOT narrowed (matchLongestPrefix walks the whole index, approximateprefix/plugin.go:214-230):
 *     totalBlocks, the global stop (the first block no endpoint holds) and each member's matchBlocks are those of the
 *     whole pool.  The P/D decider reads the pick's match count, as without a subset.
 *   - Random pickers: every subset candidate is an EXPLICIT item (no gaps; wcum is not read), the rule stated above for a
 *     set narrowed by the affinity filter.  W is the left fold of s+ in ascending slot order; the +inf and 2^-128 rules are
 *     unchanged.  So an explicit subset listing the whole pool gives the max-score decisions of no subset; under the
 *     weighted-random picker its W may differ from the gap fold's in the last bits (a different summation order).
 *   - Ordinal, tie key (4 * ordinal + profile index) and the after-pick updates (no-hit-lru Adds, in-flight adds,
 *     epp_index_add_picked) read subset picks like any other.
 *   - An empty subset (counts[r] == 0) gives status -1 (the director answers ServiceUnavailable before Schedule).
 * The subset arrays are HOST memory for every batch kind (EPP_BATCH_DEVICE_PTRS / EPP_BATCH_ASYNC included), validated and
 * copied before the call returns.  A slot >= max_endpoints, a slot list that is not strictly ascending or a wrong
 * struct_size fails the call with EPP_ERR_INVALID before anything is launched and before any LRU, counter or ordinal state
 * changes; so does any subset call on an endpoint-sharded or peer-memory engine.  EPP_SUBSET_ALL rows are decided exactly as
 * by epp_schedule; a batch without a restricted row IS epp_schedule.  Restricted rows are re-decided by a kernel of their
 * own after the batch's match kernels (so such batches never take the small-batch single-launch path); its device time is
 * epp_stats.last_kernel_ms[6] on device-pointer batches (0 otherwise).
 * On an engine with latency profiles ("Latency predictions" below) epp_schedule_subset and epp_submit_subset refuse
 * subsets with EPP_ERR_INVALID; epp_schedule_subset_predicted and epp_submit_subset_predicted take them, with or without
 * predictions, and decide a restricted request's latency profiles over its subset candidates (the rules are stated
 * there).  Non-latency profiles of such an engine follow the rules above. */
#define EPP_SUBSET_ALL 0xFFFFFFFFu
typedef struct {
    uint32_t struct_size;          /* sizeof(epp_subset)                                                                 */
    uint32_t reserved;
    const uint32_t *counts;        /* [R] slots of request r, or EPP_SUBSET_ALL = the whole pool (decided as by epp_schedule) */
    const uint64_t *offsets;       /* [R] request r's slots are slots[offsets[r] .. offsets[r] + counts[r])             */
    const uint32_t *slots;         /* strictly ascending within a request, each < max_endpoints                          */
} epp_subset;
EPP_API int32_t epp_schedule_subset(epp_engine *h, const epp_batch *batch, const epp_subset *subset, epp_decision *out,
                                    epp_decision_detail *detail, int32_t keep_hashes, const epp_topk_out *topk /* or NULL */);

/* ---- Latency predictions (datalayer/attribute/latency/data_types.go; filter/sloheadroomtier/plugin.go:84-138;
 * scorer/latency/plugin.go:144-395) ---------------------------------------------------------------------------------
 * The predicted-latency producer computes a LatencyPredictionInfo per (request, endpoint): headroom = the request's SLO
 * minus a prediction that depends on its prompt.  The caller passes those per request:
 *   - Request r carries entries (slot, ttft, ttft_headroom, tpot_headroom, dispatched): TTFT(), TTFTHeadroom(),
 *     TPOTHeadroom() and DispatchedRequestCount() of the endpoint in that slot, for that request.  Nothing else of the
 *     attribute is read by the plugins.  A candidate without an entry has no attribute.  A request without entries, and
 *     every request of a call without predictions, has no attribute anywhere.  Every profile of the request sees the same
 *     entries (decode, prefill and encode).  Entries for slots that are not candidates are ignored.
 *   - A profile has a latency piece when epp_latency_profile_set enables its tier filter or its first affinity filter, or
 *     when it lists EPP_SCORER_LATENCY (which, without that call, uses the defaults of epp_latency_cfg_default).  Profiles
 *     without one are decided exactly as on any other engine.
 * Filter chain of a latency profile:
 *     [role + label filters] -> [affinity A1] -> [tier filter T] -> [affinity A2] -> scorers in order -> picker
 *   A1 (the epp_latency_cfg a1_* fields) needs T.  A2 is the profile's own prefix-cache-affinity-filter (epp_profile_cfg
 *   affinity_*, with today's exploration draw).  Each stage works on the set it receives; everything after the chain uses
 *   the final set: the len(endpoints) <= 1 gates, the sticky sets, the queue / running min-max, the active-request max,
 *   the latency scorer's buckets, tie_count, and the random pickers' population, where every candidate is an EXPLICIT item
 *   (no gaps, as for a set narrowed by the affinity filter).  Both affinity filters read TTFT from the entries: bestTTFT
 *   skips candidates without one.  ttft_column must be < 0 on a latency profile.
 * Tier filter: a set of <= 1 is kept.  Else positive = has an entry with both headrooms >= 0, negative = has an entry with
 *   either headroom < 0, no-prediction = no entry.  No entry anywhere: keep all.  Else the no-prediction endpoints join
 *   negative; with both tiers non-empty negative is kept when u < epsilon_explore_neg, else positive; otherwise the
 *   non-empty tier.
 * Draws: A1 and T each draw u = (mix64((tie_seed ^ D) ^ mix64(key)) >> 11) * 2^-53 with key = 4 * ordinal + profile index
 *   and D = 0x8EBC6AF09C88C6E3 (A1), 0x589965CC75374CC3 (T).  With tie_seed == 0 neither explores.
 * Latency scorer (Go amd64 arithmetic: no fused multiply-add):
 *   - No candidate of the final set has an entry: composite fallback.  Weights divided by their sum ((1, 0, 0) when the sum
 *     is <= 0); maxQ = the set's largest waiting count (from 0); relQueue = (maxQ - q) / maxQ (1 when maxQ == 0); prefix =
 *     match / total (0 when total == 0); composite = wkv * (1 - kv) + wq * relQueue + wprefix * prefix, left to right;
 *     score = int(math.Round(100 * composite)) / 100.
 *   - Else negative = has an entry with either headroom < 0; positive = every other candidate, those without an entry
 *     included.  The scored bucket is positive (configured strategy) when non-empty, else the negative candidates with
 *     dispatched == 0 when there are any, else the first non-empty of TPOT-only-negative, TTFT-only-negative,
 *     both-negative; negative buckets use "least".  Candidates outside the bucket score 0.
 *   - In the bucket: alpha, beta = the normalised ttft / tpot weights ((1, 0) when their sum is <= 0); ranges of |headroom|
 *     per dimension over the bucket; eps = 1e-9; a range <= eps with the other > eps moves all weight to the other;
 *     n = (|h| - min) / range, or 0.5 when range <= eps; combined = alpha * nT + beta * nP; score =
 *     float64(int(x * 100) + 1) / 100 with x = combined ("most") or 1 - combined ("least"), int truncating toward zero.
 *   The latency scorer enters the ordered, clamped weighted sum like every other scorer.  A latency profile may not list
 *   the no-hit-lru scorer (its cold test over a tier-narrowed set is not built); epp_score rejects a latency scorer index,
 *   and -1 on a latency profile.
 * Predictions are HOST memory for every batch kind, validated and copied before the call returns.  A slot list that is not
 * strictly ascending, a slot >= max_endpoints, a non-finite ttft or headroom, a wrong struct_size, or predictions on an
 * engine without a latency profile fail the call with EPP_ERR_INVALID before anything is launched and before any LRU,
 * counter or ordinal state changes.  The endpoint-sharded modes are not available on a latency engine, and neither are
 * epp_schedule_subset and epp_submit_subset: endpoint subsets go through epp_schedule_subset_predicted /
 * epp_submit_subset_predicted.  Plain epp_schedule* on a latency engine decides every request without predictions.
 * A restricted request on a latency engine is decided exactly as the reference decides it when Schedule receives the
 * subset's endpoints and the producer has attached that request's predictions:
 *   - A profile's candidates are the subset slots that are in the pool and pass its role and label filters; the chain
 *     [A1] -> [T] -> [A2] -> scorers -> picker runs over those only.  Everything taken "over the set" uses the narrowed set:
 *     A1's and A2's len(endpoints) <= 1 gates, sticky sets and best-TTFT sets; T's tiers and its "no entry anywhere: keep
 *     all" rule; the queue / running min-max and the active-request max; the latency scorer's bucket, its |headroom|
 *     ranges and the composite fallback's maxQ; tie_count, the tie and first-k ranks and the random pickers' population
 *     (every candidate an explicit item, as on every latency profile).
 *   - The prefix match is not narrowed: totalBlocks, the global stop and each member's matchBlocks are whole-pool values,
 *     in the sticky tests and the composite prefix term as everywhere else.
 *   - Entries for slots outside the subset are ignored; a subset slot without an entry has no attribute.
 *   - Draw keys and domains are unchanged.  Since latency profiles fold every candidate explicitly in ascending slot order,
 *     a request whose subset lists the whole pool gets bit-identical decisions to the same request without a subset, for
 *     all three pickers.
 *   - An empty subset gives status -1; ordinals, the in-flight adds and epp_index_add_picked read subset picks like any
 *     other.  No-hit-lru stays refused on latency profiles. */
enum { EPP_HEADROOM_LEAST = 0, EPP_HEADROOM_MOST = 1 };
typedef struct {
    uint32_t struct_size;              /* sizeof(epp_latency_cfg)                                                      */
    int32_t tier_filter;               /* 1: the slo-headroom-tier-filter T runs between A1 and A2                     */
    double epsilon_explore_neg;        /* T's EpsilonExploreNeg, [0, 1] (default 0.01)                                 */
    double a1_affinity_threshold;      /* > 0: affinity filter A1 before T (needs tier_filter); <= 1                   */
    double a1_exploration_probability; /* [0, 1]                                                                       */
    double a1_max_ttft_penalty_ms;     /* >= 0                                                                         */
    double ttft_weight;                /* latency-scorer TTFTWeight (default 0.8)                                      */
    double tpot_weight;                /* TPOTWeight (default 0.2)                                                     */
    int32_t strategy;                  /* EPP_HEADROOM_LEAST (default) or EPP_HEADROOM_MOST                            */
    int32_t reserved;
    double composite_kv_weight;        /* CompositeKVWeight / QueueWeight / PrefixWeight (default 1, 1, 1)             */
    double composite_queue_weight;
    double composite_prefix_weight;
} epp_latency_cfg;
EPP_API void epp_latency_cfg_default(epp_latency_cfg *cfg);
/* Sets profile's latency configuration (0 = primary / decode, 1 = prefill, 2 = encode).  Only before the engine's first
 * successful epp_pool_set / epp_pool_set_labels (EPP_ERR_STATE after), and not on an endpoint-sharded engine. */
EPP_API int32_t epp_latency_profile_set(epp_engine *h, int32_t profile, const epp_latency_cfg *cfg);

typedef struct {                       /* 32 bytes */
    uint32_t slot;
    int32_t dispatched;                /* DispatchedRequestCount()                                                     */
    double ttft;                       /* TTFT()                                                                       */
    double ttft_headroom;              /* TTFTHeadroom()                                                               */
    double tpot_headroom;              /* TPOTHeadroom()                                                               */
} epp_prediction;
typedef struct {
    uint32_t struct_size;              /* sizeof(epp_predictions)                                                      */
    uint32_t reserved;
    const uint32_t *counts;            /* [R] entries of request r                                                     */
    const uint64_t *offsets;           /* [R] request r's entries are entries[offsets[r] .. offsets[r] + counts[r])    */
    const epp_prediction *entries;     /* slots strictly ascending within a request                                    */
} epp_predictions;
/* epp_schedule_topk / epp_schedule_with_match_topk with predictions (preds may be NULL: no predictions; topk may be NULL). */
EPP_API int32_t epp_schedule_predicted(epp_engine *h, const epp_batch *batch, const epp_predictions *preds, epp_decision *out,
                                       epp_decision_detail *detail, int32_t keep_hashes, const epp_topk_out *topk);
EPP_API int32_t epp_schedule_with_match_predicted(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                                  const uint32_t *model_ids, const int64_t *input_len_bytes,
                                                  int32_t block_size_tokens, epp_decision *out, epp_decision_detail *detail,
                                                  uint32_t flags, const epp_topk_out *topk, const epp_predictions *preds);
/* Endpoint subsets and predictions in one call.  subset == NULL is exactly epp_schedule_predicted; preds == NULL is
 * epp_schedule_subset, except that a latency engine is accepted (its restricted requests are then decided without
 * entries).  Both arrays are validated, with every rule of the two calls, before anything is launched: a rejected call
 * changes no ordinal, LRU or counter state. */
EPP_API int32_t epp_schedule_subset_predicted(epp_engine *h, const epp_batch *batch, const epp_subset *subset,
                                              const epp_predictions *preds, epp_decision *out, epp_decision_detail *detail,
                                              int32_t keep_hashes, const epp_topk_out *topk /* or NULL */);

/* ---- Context length (scorer/contextlengthaware/context_length_aware.go, "context-length-aware") ---------------------
 * One plugin that is both a scorer and a filter: it sends long prompts to endpoints whose range label covers them.  A
 * profile lists it as EPP_SCORER_CONTEXT_LENGTH with its weight (at most one per profile) and is then a CHAIN profile,
 * decided by the evaluation of "Latency predictions" (it counts as a latency profile wherever that section says so:
 * subsets through epp_schedule_subset_predicted / epp_schedule_ctx, predictions accepted, no endpoint-sharded mode):
 *     [role + label + context-length filters] -> [A1] -> [T] -> [A2] -> scorers in order -> picker
 *   The context-length filter is a per-endpoint predicate on the request's context length, so it joins the role and label
 *   filters in the first stage.  Everything taken "over the set" uses the final set: the affinity filters' gates and sticky
 *   sets, the queue / running min-max, the active-request max, the latency scorer's buckets, tie_count, and the random
 *   pickers' population (every candidate an explicit item).
 * Range label: each profile names a label key (default "llm-d.ai/context-length-range"; profiles may name different keys);
 *   epp_pool_set_labels parses the value of every slot (parseContextRange): split on "-" into exactly 2 parts, each part
 *   trimmed of Unicode white space (strings.TrimSpace) and read by strconv.Atoi (base 10, optional sign, int64 range), and
 *   min <= max; anything else, the empty value included, is an INVALID label.  Slots without the key have NO label.  The
 *   ranges follow the label snapshot rule: batches enqueued before an epp_pool_set_labels decide on the ranges they were
 *   enqueued under.
 * Filter (enable_filtering != 0): no label keeps, an invalid label drops, else keep iff min <= ctx <= max.  A request whose
 *   filter empties its decode set gets status -1 (that request only); an empty prefill or encode set omits that stage.
 * Score: no label 0.5; invalid label 0.0; in range with w = max - min: 1.0 when w == 0, else 0.3 + raw * 0.7 with raw =
 *   0.7 * (1 / (1 + w / 10000)) + 0.3 * ((max - ctx) / w); out of range 0.3 / (1 + d / 1000), d = the distance to the nearer
 *   bound.  Integers convert to double rounding to nearest; every operation rounds on its own (no fused multiply-add).
 * Request context length ctx: the caller's token count (len(TokenizedPrompt.TokenIDs), or its chat estimate) when it passes
 *   one; else the reference's estimate of a completions request, ctx = int(float64(L) * 0.25) = floor(L / 4) for L < 2^53,
 *   with L the true prompt length as est(L) of "In-flight load" reads it (lengths[r], the row length, input_len_bytes[r]).
 *   Every scheduling call decides context-length profiles with that default.
 * Refused (EPP_ERR_INVALID): a second context-length scorer in one profile; the no-hit-lru scorer or ttft_column >= 0 on a
 *   profile that lists it; the endpoint-sharded and peer-memory modes; epp_score naming its index, or -1 on its profile. */
#define EPP_CONTEXT_LENGTH_LABEL "llm-d.ai/context-length-range"
/* Sets profile's label key (NUL-terminated, non-empty; NULL = the default) and filtering (0 or 1, default 0).  Only
 * before the engine's first successful epp_pool_set / epp_pool_set_labels (EPP_ERR_STATE after), and only on a profile
 * that lists the scorer. */
EPP_API int32_t epp_context_length_set(epp_engine *h, int32_t profile, const char *label, int32_t enable_filtering);
/* Per-request context lengths: tokens[r] >= 0 is request r's ctx, -1 the default above.  HOST memory for every batch kind,
 * validated and copied before anything is launched; an entry < -1 or a wrong struct_size is EPP_ERR_INVALID and the call
 * then changes no ordinal, LRU or counter state.  Accepted on every engine (read only by context-length profiles). */
typedef struct {
    uint32_t struct_size;              /* sizeof(epp_context_tokens)                                                   */
    uint32_t reserved;
    const int64_t *tokens;             /* [R]                                                                          */
} epp_context_tokens;
/* epp_schedule_subset_predicted plus context lengths; subset, preds, ctx and topk may each be NULL. */
EPP_API int32_t epp_schedule_ctx(epp_engine *h, const epp_batch *batch, const epp_subset *subset, const epp_predictions *preds,
                                 const epp_context_tokens *ctx, epp_decision *out, epp_decision_detail *detail,
                                 int32_t keep_hashes, const epp_topk_out *topk);
/* epp_schedule_with_match_predicted plus context lengths (ctx may be NULL). */
EPP_API int32_t epp_schedule_with_match_ctx(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                            const uint32_t *model_ids, const int64_t *input_len_bytes, int32_t block_size_tokens,
                                            epp_decision *out, epp_decision_detail *detail, uint32_t flags,
                                            const epp_topk_out *topk, const epp_predictions *preds,
                                            const epp_context_tokens *ctx);

/* ---- Admission (requestcontrol/admitter/latencyslo/plugin.go:99-158 "latency-slo-admitter",
 * requestcontrol/admitter/probabilisticadmitter/plugin.go:125-162 "probabilistic-admitter") ---------------------------
 * The director runs the Admitter plugins after the data producers and before Scheduler.Schedule, over the same candidate
 * snapshot (requestcontrol/director.go:230-243); a rejected request is never scheduled.  The engine decides admission on
 * the device after the picks of a call and rewrites the rows it rejects, so a rejected request makes none of the
 * after-pick updates (no in-flight adds, no no-hit-lru Adds, nothing for epp_index_add_picked).
 *   Candidates of a request: the pool slots, or, for a request with an endpoint subset, the subset's slots that are in the
 *     pool.  Role, label, context-length and affinity filters do NOT apply (admission runs before any profile).  A request
 *     without a candidate keeps status -1 (the director answers ServiceUnavailable before admission); every other row may
 *     be rejected, a row whose decode profile found nobody included.
 *   Per-request inputs (epp_admission): priority (< 0 = sheddable; both admitters admit priority >= 0), ttft_slo / tpot_slo
 *     (parseFloatHeaderValue of x-slo-ttft-ms / x-slo-tpot-ms: 0 when absent, unparsable or out of range; only > 0 is
 *     tested, any double is accepted), and pred_valid: one byte per entry of the call's epp_predictions, same layout,
 *     bit 0 TTFTValid, bit 1 TPOTValid; IsValid() = both.  Validity is not derived from the headrooms (the producer
 *     neutralises TPOT with headroom 0, and a streaming prediction at the buffered SLO has headroom 0 but is invalid).
 *   latency-slo-admitter rejects iff the request is sheddable, ttft_slo > 0 || tpot_slo > 0, some candidate has an entry
 *     (entries for other slots are ignored), no candidate's entry has both bits set, no candidate has running == 0 and no
 *     candidate has kv_usage < 0.02.
 *   probabilistic-admitter, for a sheddable request: sat = the left fold from +0.0, in ascending slot order over the
 *     candidates, of math.Max(float64(waiting) / float64(queue_depth_threshold), kv_usage / kv_cache_util_threshold),
 *     divided by the number of candidates; p = math.Min(math.Pow(sat, power) * k, 1.0); rejected iff u < p with
 *     u = (mix64((tie_seed ^ 0x1D8E4E27C47D124F) ^ mix64(key)) >> 11) * 2^-53, key = 4 * ordinal + 3 (the one index of the
 *     key space no profile uses), drawn for every tie_seed, 0 included.  math.Pow is Go's algorithm restated (special
 *     cases, Modf, Exp(yf * Log(x)) for the fraction, the binary loop on Frexp's mantissa, Ldexp): bit-exact for an
 *     integer power; with a fractional one Exp and Log are CUDA's exp and log.
 *   Both admitters may be on: a row is rejected when either rejects it (the draw is keyed, so their order is irrelevant).
 *   A rejected row: status EPP_STATUS_REJECTED, pick = prefill_pick = EPP_NO_ENDPOINT, score 0.0, tie_count 0,
 *     match_blocks 0, total_blocks unchanged (the prefix producer ran before admission); its detail EPP_NO_ENDPOINT / 0 with
 *     every *_ran 0; its first-k rows EPP_NO_ENDPOINT / 0.0.  It keeps its ordinal (n_decisions counts it), so every
 *     admitted row is byte-identical to the same call made without admission inputs.
 *   The whole-pool candidate set's idle and cold flags, count and saturation fold are derived by epp_pool_set and follow
 *   the snapshot rule: an async batch decides on the pool it was enqueued under.  Only rows an admitter can reject are
 *   examined, one warp each, by a kernel behind the call's picks (and before its after-pick updates); a call without such
 *   a row launches nothing more and may take the small-batch path.  Its device time is epp_stats.last_kernel_ms[7] on
 *   device-pointer batches (0 otherwise).
 * The arrays are HOST memory for every batch kind, validated and copied before anything is launched.  A wrong struct_size,
 * a NULL pred_valid on an engine with the latency-slo-admitter for a call with predictions, or epp_admission on an
 * engine without admitters is EPP_ERR_INVALID; a refused call changes no ordinal, LRU, counter or index state.  With the
 * latency-slo-admitter on, predictions are accepted on every engine (on an engine without a latency profile only the
 * admitter reads them). */
#define EPP_STATUS_REJECTED (-2)
typedef struct {
    uint32_t struct_size;              /* sizeof(epp_admission_cfg)                                                    */
    int32_t latency_slo;               /* 1: the latency-slo-admitter                                                  */
    int32_t probabilistic;             /* 1: the probabilistic-admitter                                                */
    int32_t queue_depth_threshold;     /* queueDepthThreshold, > 0 (default 5)                                         */
    double kv_cache_util_threshold;    /* kvCacheUtilThreshold, finite and > 0 (default 0.8)                           */
    double power;                      /* power, finite and > 0 (default 5.0)                                          */
    double k;                          /* k, finite and > 0 (default 300)                                              */
} epp_admission_cfg;
EPP_API void epp_admission_cfg_default(epp_admission_cfg *cfg);
/* Sets the engine's admitters.  Only before the first successful epp_pool_set / epp_pool_set_labels (EPP_ERR_STATE after);
 * refused on endpoint-sharded and peer-memory engines. */
EPP_API int32_t epp_admission_set(epp_engine *h, const epp_admission_cfg *cfg);
typedef struct {
    uint32_t struct_size;              /* sizeof(epp_admission)                                                        */
    uint32_t reserved;
    const int32_t *priority;           /* [R] Objectives.Priority, or NULL = all 0                                     */
    const double *ttft_slo;            /* [R] or NULL = all 0                                                          */
    const double *tpot_slo;            /* [R] or NULL = all 0                                                          */
    const uint8_t *pred_valid;         /* one byte per entry of the call's epp_predictions (entries[offsets[r] + i]), or NULL */
} epp_admission;
/* epp_schedule_ctx / epp_schedule_with_match_ctx with admission inputs (adm may be NULL: the call is then exactly the
 * _ctx call). */
EPP_API int32_t epp_schedule_admit(epp_engine *h, const epp_batch *batch, const epp_subset *subset, const epp_predictions *preds,
                                   const epp_context_tokens *ctx, const epp_admission *adm, epp_decision *out,
                                   epp_decision_detail *detail, int32_t keep_hashes, const epp_topk_out *topk);
EPP_API int32_t epp_schedule_with_match_admit(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                              const uint32_t *model_ids, const int64_t *input_len_bytes,
                                              int32_t block_size_tokens, epp_decision *out, epp_decision_detail *detail,
                                              uint32_t flags, const epp_topk_out *topk, const epp_predictions *preds,
                                              const epp_context_tokens *ctx, const epp_admission *adm);

/* PreRequest (approximateprefix/plugin.go:164-200): index the hashes of the LAST epp_schedule batch
 * (keep_hashes=1) for each request's primary pick and prefill pick. */
EPP_API int32_t epp_index_add_picked(epp_engine *h);

/* The no-hit-lru scorer's LRU, oldest first (golang-lru Cache.Keys): *out_n = its length, the first min(cap, *out_n)
 * slot ids go to out_eps.  Waits for the batches in flight.  EPP_ERR_STATE when no profile has the scorer. */
EPP_API int32_t epp_nohit_lru_get(epp_engine *h, uint32_t *out_eps, int32_t cap, int32_t *out_n);

/* ResponseBody of the inflight-load producer (producer.go:131-168): entry i takes 1 request and est(prompt_lens[i]) tokens
 * off slot eps[i] (the prefill target at the first chunk, the other targets at the end of the stream).  EPP_NO_ENDPOINT
 * entries are skipped; a slot >= max_endpoints fails the whole call with EPP_ERR_INVALID.  EPP_ERR_STATE when the engine
 * was created without inflight_load.  No CUDA call: applied before the next scheduling call or epp_inflight_get. */
EPP_API int32_t epp_inflight_release(epp_engine *h, int32_t n, const uint32_t *eps, const uint64_t *prompt_lens);
/* Endpoint deletion (producer.go:86-97, 189-192): both counters of slots ids[0 .. n) become 0, after every earlier
 * release and before every later one.  Call it before a slot id is given to another endpoint. */
EPP_API int32_t epp_inflight_reset(epp_engine *h, int32_t n, const uint32_t *ids);
/* The counters of the first min(cap, max_endpoints) slots (InFlightLoad.Requests / .Tokens).  Applies the pending
 * releases and resets and waits for the batches in flight.  EPP_ERR_STATE without inflight_load. */
EPP_API int32_t epp_inflight_get(epp_engine *h, int32_t cap, int64_t *out_requests, int64_t *out_tokens);

EPP_API int32_t epp_get_stats(epp_engine *h, epp_stats *out);

/* Waits for everything the engine has enqueued (EPP_BATCH_ASYNC batches). */
EPP_API int32_t epp_synchronize(epp_engine *h);
/* CUDA events on the engine's launch stream: record event `which` (0 = start, 1 = stop) after the work enqueued so
 * far; epp_event_elapsed_ms waits for the stop event and returns stop - start in milliseconds (device time). */
EPP_API int32_t epp_event_record(epp_engine *h, int32_t which);
EPP_API int32_t epp_event_elapsed_ms(epp_engine *h, double *out_ms);

/* ---- endpoint-sharded multi-GPU mode (SURVEY.md 8(e)) ----------------------------------------------
 * Each rank holds the postings of the endpoints of its shard and the full pool state.  Phase 1 probes
 * the local table and produces per-request block-presence masks (ceil(max_prefix_blocks/32) words per
 * request); the caller ORs the masks of all ranks (NCCL all-gather / bitwise OR); phase 2 applies the
 * global stop rule (plugin.go:219-223), counts local matches and returns the local best record; the caller
 * all-gathers the records and epp_shard_merge reduces them.  All pointers are DEVICE pointers. */
typedef struct {
    double score;
    uint32_t pick;
    uint32_t tie_count;
    int32_t match_blocks;
    int32_t status;            /* 0 = this shard has a candidate, -1 = none */
} epp_shard_best;              /* 24 bytes */
EPP_API int32_t epp_shard_set(epp_engine *h, uint32_t ep_begin, uint32_t ep_end);
EPP_API int32_t epp_shard_probe(epp_engine *h, const epp_batch *batch, uint32_t *out_masks);
/* Scores the batch of the last epp_shard_probe.  Its per-request model ids (the lora-affinity scorer's adapters) are the
 * engine's own copy, taken by epp_shard_probe: the caller's model_ids array need not outlive that call. */
EPP_API int32_t epp_shard_pick(epp_engine *h, int64_t n_requests, const uint32_t *global_masks, epp_shard_best *out_best);
EPP_API int32_t epp_shard_merge(epp_engine *h, int64_t n_requests, int32_t n_ranks, const epp_shard_best *all_best,
                        epp_decision *out);

/* Staged records: the disagg profile handler (decode -> P/D decider -> prefill, with the optional encode stage) in the
 * endpoint-sharded mode, with the same three phases and two exchanges.  epp_shard_set_staged does what epp_shard_set does,
 * also accepts EPP_HANDLER_DISAGG (with or without encode_enabled) and returns S in *out_stages: 1 for the single-profile
 * handler, 2 for decode + prefill, 3 with the encode profile.  Every other refusal of epp_shard_set stays.
 * epp_shard_pick then writes S records per request, request-major ([R][S]: stage 0 decode, 1 prefill, 2 encode), so the
 * all-gather yields [n_ranks][R][S] and epp_shard_merge(_detail) reads that.  For request r on one rank:
 *   stage 0  the local best decode record (as with one stage);
 *   stage 1  the local best prefill record whenever the P/D decider can still say yes, i.e. always_disagg, or
 *            non_cached_tokens != 0 and (request bytes / 4) >= non_cached_tokens -- whether it runs depends on the merged
 *            decode pick's match_blocks, which no rank knows yet; it is evaluated even when this rank has no decode
 *            candidate; status -1 otherwise;
 *   stage 2  the local best encode record for multimodal requests, status -1 otherwise.
 * The merge reduces each stage alone (max score, lowest slot id among equals, ties summed), then applies the handler as
 * epp_schedule does: no decode pick anywhere -> status -1 and no other stage; encode_ran = multimodal[r]; prefill_ran =
 * always_disagg || the P/D decider on the merged decode pick's match_blocks; the stage fields come from the reduced
 * records (EPP_NO_ENDPOINT when no rank has one).  The request lengths (lengths[r] when given, the decider's input) and
 * multimodal flags are the engine's own copies, kept by epp_shard_probe.  On a peer-memory engine epp_shard_set_staged
 * must come before epp_shard_p2p_export: the buffer holds max_requests * S records, and a call after an export made for
 * another S is EPP_ERR_STATE.
 * out_detail ([R] device, or NULL) receives the prefill and encode fields; with an encode profile and a batch that flags
 * multimodal requests it must not be NULL (EPP_ERR_INVALID), as in epp_schedule.  epp_shard_merge, epp_shard_schedule_p2p
 * and epp_shard_p2p_phase are these calls with out_detail = NULL. */
EPP_API int32_t epp_shard_set_staged(epp_engine *h, uint32_t ep_begin, uint32_t ep_end, int32_t *out_stages);
EPP_API int32_t epp_shard_merge_detail(epp_engine *h, int64_t n_requests, int32_t n_ranks, const epp_shard_best *all_best,
                                       epp_decision *out, epp_decision_detail *out_detail);

/* The same protocol with both exchanges done by the ranks' own kernels over NVLink PEER MEMORY (no NCCL): every rank
 * exports one exchange buffer (CUDA IPC handle, 64 bytes; out_ptr is the raw device pointer for ranks that share a
 * process), connects to all peers' buffers (peers: n_ranks x 64-byte handles when ipc_handles != 0, else n_ranks
 * uint64 pointers), then calls epp_shard_schedule_p2p with the SAME device batch on every rank: presence masks are
 * OR-reduced and best records merged straight out of the peers' memory, ordered by release/acquire flags (the two halves
 * of a batch pipelined through the exchange on the engine's two streams); `out`
 * ([R] device) is identical on every rank.  A peer that does not show up within 20 s (EPP_P2P_TIMEOUT_MS) yields EPP_ERR_NCCL. */
EPP_API int32_t epp_shard_p2p_export(epp_engine *h, int64_t max_requests, uint8_t *out_handle, uint64_t *out_ptr);
EPP_API int32_t epp_shard_p2p_connect(epp_engine *h, int32_t n_ranks, int32_t rank, const void *peers, int32_t ipc_handles);
EPP_API int32_t epp_shard_schedule_p2p(epp_engine *h, const epp_batch *batch, epp_decision *out);
/* The same batch ONE phase at a time (0: hashes + local masks + flag 1; 1: OR of the peers' masks + local best records +
 * flag 2; 2: gather + merge -> out), each call synchronising before it returns: for ranks that share a GPU, whose
 * device-side waits could starve each other -- step all ranks through phase 0, then all through 1, then 2.
 * A peer that times out (or whose flags are poisoned) breaks the exchange for good: every later call fails with
 * EPP_ERR_STATE until epp_shard_p2p_export / _connect are called again on every rank. */
EPP_API int32_t epp_shard_p2p_phase(epp_engine *h, const epp_batch *batch, epp_decision *out, int32_t phase);
/* The two calls above with the detail of the staged records (see "Staged records"); the batch's multimodal flags are a
 * device array. */
EPP_API int32_t epp_shard_schedule_p2p_detail(epp_engine *h, const epp_batch *batch, epp_decision *out,
                                              epp_decision_detail *out_detail);
EPP_API int32_t epp_shard_p2p_phase_detail(epp_engine *h, const epp_batch *batch, epp_decision *out,
                                           epp_decision_detail *out_detail, int32_t phase);

/* Seeded ties: the tie rule of epp_config.tie_seed != 0 (see "Tie rule") in the endpoint-sharded mode, with a third
 * exchange.  epp_shard_set_seeded does what epp_shard_set_staged does (same *out_stages) and selects the seeded rule; it
 * is EPP_ERR_INVALID when tie_seed == 0 and for every configuration epp_shard_set_staged refuses.  A later epp_shard_set
 * or epp_shard_set_staged returns the engine to the lowest-slot rule.
 * Phase 2 is unchanged: each record holds this rank's max, its lowest tied slot and its local tie count.  For request r
 * and stage st every rank then computes from the gathered records the global max, N = the sum of the tied counts and
 * rho = tie_rank(tie_seed, 4 * (n_decisions + r) + st, N).  The shard ranges are disjoint, so the arg-max set in
 * ascending slot order is the ranks' local sets taken in the order of their records' picks; that order gives the OWNER
 * rank of member rho and its rank in the owner's local set.  The owner selects that member (its match kernel again, the
 * rank forced) and publishes {pick, match_blocks}; every other rank publishes EPP_NO_ENDPOINT for that entry.  The
 * decisions are then built from the selected members, the P/D decider reading the seeded decode member's match_blocks,
 * and are bit for bit those of an unsharded engine with the same tie_seed and ordinal.
 * Host-driven exchanges: probe -> OR of the masks -> epp_shard_pick -> all-gather of the records -> epp_shard_select
 * (writes this rank's [R][S] entries to out_sel) -> all-gather of the entries -> epp_shard_finish (the decisions; it
 * advances epp_stats.n_decisions by R, the ordinal of the next batch).  epp_shard_merge(_detail) is EPP_ERR_STATE on a
 * seeded engine.  all_best and all_sel are stacked in the same rank order.
 * Peer memory: epp_shard_set_seeded must come before epp_shard_p2p_export, which then also sizes the entries (an export
 * made for the other rule is EPP_ERR_STATE for both set calls).  A batch is four phases: 0 and 1 as above; 2 waits for
 * the records, resolves, selects and raises flag 3; 3 waits for flag 3, gathers the entries and writes the decisions.
 * epp_shard_p2p_phase(_detail) takes phase 0..3 on a seeded engine (0..2 otherwise: 3 is EPP_ERR_INVALID). */
typedef struct {
    uint32_t pick;             /* the selected member, EPP_NO_ENDPOINT on the ranks that do not own the entry */
    int32_t match_blocks;      /* its match count */
} epp_shard_sel;               /* 8 bytes */
EPP_API int32_t epp_shard_set_seeded(epp_engine *h, uint32_t ep_begin, uint32_t ep_end, int32_t *out_stages);
EPP_API int32_t epp_shard_select(epp_engine *h, int64_t n_requests, int32_t n_ranks, const epp_shard_best *all_best,
                                 epp_shard_sel *out_sel);
EPP_API int32_t epp_shard_finish(epp_engine *h, int64_t n_requests, int32_t n_ranks, const epp_shard_best *all_best,
                                 const epp_shard_sel *all_sel, epp_decision *out, epp_decision_detail *out_detail);

/* The configuration the engine was created with. */
EPP_API int32_t epp_get_config(epp_engine *h, epp_config *out);

/* ---- micro-batcher: one request in, one decision out (SURVEY.md 8(f).2) ------------------------------------------
 * The reference calls Scheduler.Schedule(ctx, *InferenceRequest, []Endpoint) once per in-flight request, from one
 * goroutine each (requestcontrol/director.go:69-71, 243; handlers/server.go:168).  epp_submit / epp_wait give a shim
 * exactly that shape: any number of threads submit single prompts; a flusher thread inside the library closes a batch
 * when it holds max_batch requests or its oldest request has waited max_delay_us, evaluates it against ONE frozen
 * snapshot (epp_schedule), hands out the decisions and -- with index_picks -- applies PreRequest (epp_index_add_picked,
 * approximateprefix/plugin.go:164-200; off the request path like the reference's, :189-194) before the next batch;
 * epp_wait blocks until the ticket's batch is done.
 * A batcher must be destroyed before its engine; other threads may keep calling epp_pool_set etc. on the engine
 * (the scrape loop) -- every flush sees the snapshot current at its start. */
typedef struct epp_batcher epp_batcher;
typedef struct {
    uint32_t struct_size;
    int32_t max_batch;             /* requests per flush at most                                          */
    int32_t max_delay_us;          /* a batch closes when its oldest request has waited this long (0 = flush at once) */
    int32_t index_picks;           /* != 0: PreRequest after every flush (the picks' prefix hashes enter the index) */
} epp_batcher_cfg;
typedef struct {
    uint64_t n_flushes, n_requests, n_full_flushes, n_pending;
    uint64_t n_index_errors;       /* flushes whose PreRequest (epp_index_add_picked) failed: it runs after the decisions
                                      were handed out, so its error reaches epp_batcher_stats / the log, not the waiters */
} epp_batcher_stats_t;
EPP_API int32_t epp_batcher_create(epp_engine *h, const epp_batcher_cfg *cfg, epp_batcher **out);
EPP_API int32_t epp_batcher_destroy(epp_batcher *b);     /* flushes what is pending, then stops the flusher   */
/* prompt: the request's bytes (a uint32 token array = 4 bytes per token, hashing.go:49), copied before the call returns
 * (only the first max_prefix_blocks blocks are kept); multimodal: hasMultimodalContent (encode decider).  A ticket can
 * be waited for (any number of times, from any thread) until 4096 later batches have been flushed; after that
 * epp_wait returns EPP_ERR_STATE.  Every epp_wait must have returned before epp_batcher_destroy.
 * Neither call takes a lock: a submit is one compare-and-swap + the copy, a wait polls / sleeps on the flush counter. */
EPP_API int32_t epp_submit(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len,
                           uint32_t multimodal, uint64_t *out_ticket);
/* epp_submit for a request whose candidates are the n_slots endpoints slots[0 .. n_slots) (see "Endpoint subsets"; any
 * order, duplicates allowed: the batcher sorts and deduplicates them).  Up to EPP_SUBSET_MAX_SLOTS slots, kept in the
 * batcher's staging next to the prompt; more is EPP_ERR_CAPACITY, a slot >= max_endpoints EPP_ERR_INVALID, and so is an
 * engine with latency profiles (use epp_submit_subset_predicted there).  A flush holding a request submitted this way
 * runs epp_schedule_subset, every other flush epp_schedule. */
#define EPP_SUBSET_MAX_SLOTS 1024
EPP_API int32_t epp_submit_subset(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len,
                                  uint32_t multimodal, uint32_t n_slots, const uint32_t *slots, uint64_t *out_ticket);
/* epp_submit with the request's latency predictions (include "Latency predictions"): n entries, in any slot order (the
 * batcher sorts them), staged next to the prompt; a flush that holds such a request runs epp_schedule_predicted.  More
 * than EPP_PRED_MAX_SLOTS entries is EPP_ERR_CAPACITY; two entries for one slot, a slot >= max_endpoints, a non-finite
 * value, or an engine without a latency profile is EPP_ERR_INVALID, refused here so that no flush fails for it. */
#define EPP_PRED_MAX_SLOTS 1024
EPP_API int32_t epp_submit_predicted(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len,
                                     uint32_t multimodal, uint32_t n, const epp_prediction *entries, uint64_t *out_ticket);
/* epp_submit for a request on a latency engine with both an endpoint subset (n_slots slots, as for epp_submit_subset) and
 * its predictions (n_pred entries, as for epp_submit_predicted).  Both lists are checked here with every rule of those two
 * calls (so a latency engine is required) and staged next to the prompt.  On a latency engine every flush that holds a
 * subset or a prediction row runs epp_schedule_subset_predicted. */
EPP_API int32_t epp_submit_subset_predicted(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len,
                                            uint32_t multimodal, uint32_t n_slots, const uint32_t *slots, uint32_t n_pred,
                                            const epp_prediction *entries, uint64_t *out_ticket);
/* epp_submit with everything a request may carry (see "Context length"): an endpoint subset (slots == NULL: none, then
 * n_slots must be 0), predictions (n_pred entries; a latency engine is required when n_pred > 0) and context_tokens (-1 =
 * the default, < -1 EPP_ERR_INVALID), each checked here with the rules of epp_submit_subset_predicted.  A flush that holds
 * such a request runs epp_schedule_ctx. */
EPP_API int32_t epp_submit_ctx(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len, uint32_t multimodal,
                               uint32_t n_slots, const uint32_t *slots, uint32_t n_pred, const epp_prediction *entries,
                               int64_t context_tokens, uint64_t *out_ticket);
/* epp_submit_ctx plus the request's admission inputs (see "Admission"): pred_valid holds one byte per entry of `entries`
 * (required when n_pred > 0 and the engine has the latency-slo-admitter), priority (< 0 = sheddable) and the two SLOs.  An
 * engine without admitters is EPP_ERR_INVALID; predictions are accepted on an engine with the latency-slo-admitter.  A
 * flush that holds such a request runs epp_schedule_admit; its rejected requests get status EPP_STATUS_REJECTED from
 * epp_wait / epp_wait_topk like any other row. */
EPP_API int32_t epp_submit_admit(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len, uint32_t multimodal,
                                 uint32_t n_slots, const uint32_t *slots, uint32_t n_pred, const epp_prediction *entries,
                                 const uint8_t *pred_valid, int64_t context_tokens, int32_t priority, double ttft_slo,
                                 double tpot_slo, uint64_t *out_ticket);
EPP_API int32_t epp_wait(epp_batcher *b, uint64_t ticket, epp_decision *out, epp_decision_detail *out_detail);
/* The same on an engine created with pick_k > 1, plus the request's first-k lists (ProfileRunResult.TargetEndpoints of
 * each profile, see epp_topk_out): primary / prefill / encode receive pick_k slot ids each (EPP_NO_ENDPOINT padded); any
 * of them may be NULL. */
EPP_API int32_t epp_wait_topk(epp_batcher *b, uint64_t ticket, epp_decision *out, epp_decision_detail *out_detail,
                              uint32_t *primary, uint32_t *prefill, uint32_t *encode);
EPP_API int32_t epp_batcher_stats(epp_batcher *b, epp_batcher_stats_t *out);
EPP_API const char *epp_batcher_last_error(void);

#ifdef __cplusplus
}
#endif
#endif
