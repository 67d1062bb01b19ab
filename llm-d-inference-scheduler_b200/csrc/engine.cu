// engine.cu -- the C ABI of libepp_engine.so (include/epp_engine.h) and the host logic above the kernels:
// configuration, pool-state snapshot, prefix-index store + device table, batch staging (H2D / D2H pipelined
// against the kernels on two streams) and the per-batch launch sequence.
//
// There is NO CPU compute path in this file: without a CUDA device epp_engine_create fails with
// EPP_ERR_NO_DEVICE, and every data-path entry point only stages buffers and launches kernels.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "devbuf.h"
#include "index_store.h"
#include "kernels.h"

using namespace epp;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;

static int32_t fail(int32_t code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

#define CUDA_TRY(expr)                                                                             \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return fail(EPP_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

#define EPP_TRY(expr)            \
    do {                         \
        int32_t _r = (expr);     \
        if (_r != EPP_OK) return _r; \
    } while (0)

struct ProfileState {
    DevBuf cand, contrib, base, order, grp_size, sort_key, n_cand, qminmax;
    DevBuf cands, wcum, icum;       // random pickers only (ProfileDerived)
};

struct LabelReq {                   // one epp_label_req, copied
    std::string key;
    int32_t op;
    std::vector<std::string> values;
};
// Every profile's label requirements compiled against one interning of keys and values (epp_label_filters_set).
struct LabelPlan {
    std::vector<std::string> keys;                                  // row k of lcode
    std::vector<std::unordered_map<std::string, uint8_t>> codes;    // per key: named value -> code 1..62
    LabelFilterDev dev[kMaxProfiles] = {};                          // lcode filled in by label_dev
};
static constexpr int kMaxLabelKeys = 16, kMaxLabelValues = 62;

struct Slot {                       // per-stream staging for host-pointer batches
    cudaStream_t stream = nullptr;
    DevBuf data;
    DevBuf overflow_list, overflow_n;   // requests handed from a sparse pass to the dense-counter pass (per stream);
                                        // overflow_n[1] is the sparse pass's request counter
    DevBuf hash_next;                   // k_hash_fused's request counter
    DevBuf pick_scratch;                // zeroed global match counters of the dense-counter kernel when max_endpoints is too
                                        // large for shared memory: per stream, two streams may run that kernel at once
    cudaEvent_t done = nullptr;
};

// Event pairs bracketing the launches of one kernel in the device batch in flight; their elapsed times are summed once
// it completes.
struct EventSpans {
    std::vector<cudaEvent_t> ev;
    int used = 0;                   // events recorded for the batch in flight
    EventSpans() = default;
    EventSpans(const EventSpans &) = delete;
    EventSpans &operator=(const EventSpans &) = delete;
    ~EventSpans() { for (cudaEvent_t e : ev) cudaEventDestroy(e); }
    cudaError_t begin(cudaStream_t s) {
        while ((int)ev.size() < used + 2) {
            cudaEvent_t e;
            cudaError_t err = cudaEventCreate(&e);
            if (err != cudaSuccess) return err;
            ev.push_back(e);
        }
        return cudaEventRecord(ev[used], s);
    }
    cudaError_t end(cudaStream_t s) {
        const cudaError_t err = cudaEventRecord(ev[used + 1], s);
        if (err == cudaSuccess) used += 2;
        return err;
    }
    double take_ms() {
        double t = 0.0;
        for (int i = 0; i + 1 < used; i += 2) {
            float t1 = 0;
            cudaEventElapsedTime(&t1, ev[i], ev[i + 1]);
            t += t1;
        }
        used = 0;
        return t;
    }
};

// The side inputs of one scheduling call: validated on the host by check_inputs before any engine state changes, then
// staged to the device by stage_inputs.  A call without them stages nothing.
struct CallInputs {
    int64_t R = 0;
    const epp_topk_out *topk = nullptr;
    const epp_subset *subset = nullptr;         // the caller's arrays, packed by stage_inputs
    const epp_predictions *preds = nullptr;
    const epp_context_tokens *ctx = nullptr;
    std::vector<SubsetRow> sub_rows;            // the restricted requests, ascending
    uint64_t sub_n_slots = 0;
    bool use_pred = false;                      // staged: without a latency profile only the admitter reads predictions
    bool use_ctx = false;                       // staged: only a context-length profile reads the token counts
    uint64_t n_ent = 0;                         // prediction entries
    std::vector<AdmitRow> adm_rows;             // the rows an admitter can reject, ascending
    std::vector<uint32_t> adm_ent;
    // the staged sections on the device (nullptr: not staged)
    const SubsetRow *d_sub_rows = nullptr;
    const uint32_t *d_sub_slots = nullptr, *d_cnt = nullptr, *d_adm_ent = nullptr;
    const uint64_t *d_off = nullptr;
    const epp_prediction *d_ent = nullptr;
    const int64_t *d_ctx = nullptr;
    const AdmitRow *d_adm_rows = nullptr;
    bool staged() const { return !sub_rows.empty() || use_pred || use_ctx || !adm_rows.empty(); }
};

struct epp_engine {
    std::mutex mu;
    epp_config cfg;
    int n_profiles = 1;             // profiles of the P/D handler: 1 (single) or 2 (decode + prefill)
    int n_alloc_profiles = 1;       // + the encode profile ([2]) when configured
    int sm_count = 132;
    int32_t Epad = 0;
    size_t dev_bytes = 0;
    size_t max_smem_optin = 0;

    Slot slot[2];
    cudaEvent_t ev[9] = {};
    // post-pick update u (0 = no-hit-lru, 1 = inflight) of the device batch in flight is bracketed by ev[5 + 2u] /
    // ev[6 + 2u]: epp_stats.last_kernel_ms[4 + u]
    bool post_pick_timed[2] = {};
    cudaEvent_t user_ev[2] = {};    // epp_event_record / epp_event_elapsed_ms
    unsigned long long *wc_host = nullptr;   // pinned: work counters of an async batch
    bool async_pending = false;     // an EPP_BATCH_ASYNC batch whose stats have not been read back yet
    bool s1_unjoined = false;       // chunk-pipelined async batches left work on stream 1 that stream 0 has not waited for
    int64_t pipe_R = 0, pipe_per = 0;   // chunk layout of the pipelined batches in flight (row ranges are per stream)
    int async_launches = 0;
    DevBuf work_counters;           // u64[4] probes, postings, hash bytes stored, prompt bytes read

    // models
    DevBuf seeds;                   // u64[kMaxModels]
    DevBuf seed_msg;
    int n_models = 0;
    std::vector<uint64_t> host_seeds;

    // pool state
    bool pool_ready = false;
    DevBuf role, kv, waiting, running, ext;
    DevBuf lora_max, lora_cnt, lora_ptr, lora_ep, lora_state, score_models;   // LoRA residency (epp_pool_set_lora)
    bool lora_set = false, lora_enabled = false;
    int32_t lora_models = 0;
    // label filters: the requirements of each profile, their compiled form and the interned labels of every slot
    std::vector<LabelReq> label_reqs[kMaxProfiles];
    LabelPlan labels;
    DevBuf lcode;                   // uint8 [labels.keys.size()][E] (LabelFilterDev)
    bool pool_called = false;       // epp_pool_set / epp_pool_set_labels succeeded once: the label filters are fixed
    // latency predictions (include/epp_engine.h "Latency predictions"): each profile's configuration and the profiles with
    // a latency piece
    epp_latency_cfg lat_cfg[kMaxProfiles] = {};
    int lat_mask = 0;
    // context length (include/epp_engine.h "Context length"): the profiles listing the plugin (they are in lat_mask too),
    // each one's label key, filtering and per-slot ranges
    int cl_mask = 0, cl_filter = 0;
    std::string cl_label[kMaxProfiles];
    DevBuf cl_rng[kMaxProfiles];    // longlong2 [E] (kernels.h LatView::rng)
    ProfileState prof[kMaxProfiles];
    // no-hit-lru scorer (nohit_lru.cu), allocated only when a profile lists it
    int nohit_mask = 0;             // bit pi: profile pi has the scorer
    int32_t nohit_lru = 0;          // lruSize
    uint64_t nohit_seq = 1;         // sequence number of the next call's first Add (0 = not in the LRU)
    ProfileState prof_cold[kMaxProfiles];   // cold sets: base / order / groups with the LRU column
    DevBuf nh_last_seq, nh_pos, nh_misc, nh_sort_key, nh_order, nh_cold, nh_col[kMaxProfiles];
    DevBuf nh_prof;                 // ProfileDev[kMaxProfiles] of the cold sets (NoHitView::cold)
    // inflight-load producer (inflight.cu), allocated only with cfg.inflight_load
    bool inflight = false;
    int inflight_mask = 0;          // bit pi: profile pi lists a token-load or active-request scorer (they read the counters)
    int32_t n_ext_total = 0;        // the caller's ext columns, then (with inflight) the token and request count columns
    DevBuf if_req, if_tok;
    std::mutex if_mu;               // guards if_pending only: releases and resets never wait for a batch
    std::unordered_map<uint32_t, InflightDelta> if_pending;   // folded releases / resets not applied yet
    // two staging sets for the folded deltas: a set is refilled once the apply kernel that read it has run (if_ev)
    HostBuf if_host[2];
    DevBuf if_dev[2];
    cudaEvent_t if_ev[2] = {};
    int if_flip = 0;
    epp_config cfg_user;            // the configuration as given (cfg has the counter columns filled in)

    // index
    std::unique_ptr<IndexStore> store;          // write side: LRU bookkeeping in HBM (index_store.cu)
    // indexer.Add calls queued by epp_index_add until the next commit / read (applied as ONE device batch)
    std::vector<uint32_t> q_ep, q_n;
    std::vector<int32_t> q_nb;
    std::vector<uint64_t> q_src, q_hashes;
    DevBuf q_ep_dev, q_n_dev, q_nb_dev, q_src_dev, q_hashes_dev, kept_dec;
    bool snapshot_mode = false;
    DevBuf slots, postings, idx_scratch, idx_cursor, idx_special, pair_hash, pair_ep, get_out, intern_keys, intern_vals;
    uint64_t idx_capacity = 0, idx_pairs = 0;
    // incremental maintenance of the read table (IndexStore::patch_read_table)
    bool rt_from_store = false;     // the table mirrors the store's inverted map (bulk-built from its export)
    uint64_t post_cap = 0, post_used = 0, rt_slots_used = 0, rt_intern_used = 0;
    int patches_since_build = 0;
    int patch_enabled = 1;          // EPP_INDEX_PATCH=0: always rebuild
    IndexSlot idx_special_host{};
    // presence bitmap of the read table (index.cuh presence_maybe): rebuilt by every bulk build, bits added by patches
    DevBuf presence;
    int presence_log2 = 0;          // log2 of its bits
    int presence_log2_env = 0;      // EPP_PRESENCE_LOG2BITS=n (6..30): fixed size instead of 16 bits per table slot
    int hash_trim = 1;              // EPP_HASH_TRIM=0: Schedule batches store whole hash rows
    int hash_skip = 1;              // EPP_HASH_SKIP=0: trimmed batches still read and hash every prompt byte
    uint32_t shard_begin = 0, shard_end = 0xFFFFFFFFu;

    // batch buffers (sized for the largest batch seen)
    DevBuf offsets, lengths, model_ids, multimodal, hashes, nblocks, bound, eff_len, in_len, decisions, details, flag;
    DevBuf dense_match, dense_total, dense_scores;
    int index_load = 0;             // EPP_INDEX_LOAD=n: read-table slots per distinct hash (2 = load factor <= 0.5, 4 = <= 0.25);
                                    // 0 = automatic: 4 while the table stays L2-sized (<= l2_table_bytes), else 2
    uint64_t l2_table_bytes = 24ull << 20;  // half the device's L2: the other half stays for the streamed prompts
    int dev_chunks = 2;             // EPP_DEV_CHUNKS=N: async device batches run as N chunks over both streams (1 = off)
    int pick_grid = 0;
    bool pick_global = false;
    size_t pick_smem = 0;
    // small host batches: one zero-copy kernel, no copy engine, no stream synchronisation (cycle_small.cu)
    int small_max = 1024;           // EPP_SMALL_BATCH=n: largest batch that takes the path (0 = off)
    int small_zc_max = 8;           // EPP_SMALL_ZEROCOPY=n: largest batch whose prompts the kernel reads over PCIe itself
    int64_t small_cap = 0;          // requests the pinned staging below is sized for
    uint8_t *small_host = nullptr;  // one pinned + mapped allocation: 2 x {offsets, lengths, model_ids, multimodal}, dec, det, flags
    uint64_t *small_offsets[2] = {}, *small_lengths[2] = {};
    uint32_t *small_models[2] = {};
    uint8_t *small_mm[2] = {};
    epp_decision *small_dec = nullptr;
    epp_decision_detail *small_det = nullptr;
    uint32_t *small_flags = nullptr;
    uint32_t small_epoch = 0;
    DevBuf small_overflow_n;        // stays zero between batches (reset by the overflow pass)
    int small_pipe_min = 1;         // EPP_SMALL_PIPELINE=n: DMA-copied batches of >= n requests start their kernel BEFORE the copy
                                    // lands (copy on the second stream, one stream-ordered flag write behind it); 0 = off
    DevBuf small_arrive;            // epoch word: the prompts of the batch have arrived
    uint32_t *small_epoch_host = nullptr;   // pinned source of that word when the driver has no stream write-value
    bool small_no_write_value = false;
    bool small_stats_pending = false;   // ev[0] / ev[1] bracket the last small batch; read lazily by epp_get_stats
    std::chrono::steady_clock::time_point last_commit{};   // last commit done by a scheduling call (index_commit_interval_us)
    bool committed_once = false;
    bool general = false;           // a profile configures the prefix-cache-affinity-filter or pick_k > 1: every batch takes
                                    // the dense-counter kernel with the full-scan evaluation of pick_general.cuh
    // the side inputs of the scheduling call in progress (under mu): set by schedule_impl and with_match_impl for the whole
    // call (CallScope), nullptr otherwise
    const CallInputs *cur = nullptr;
    HostBuf in_host;                // pinned staging of the call's side inputs (stage_inputs)
    DevBuf in_dev;
    cudaEvent_t in_ev = nullptr;    // behind the last copy from in_host
    DevBuf sub_hits, sub_scratch;   // endpoint subsets (subset_pick.cu): written by the subset kernel, parallel to its slots
    EventSpans sub_spans;           // the subset launches of the device batch in flight (last_kernel_ms[6])
    DevBuf topk_picks[kMaxProfiles], topk_scores;   // device staging of the lists for host batches
    // admission (include/epp_engine.h "Admission", admit.cu): the admitters and the whole pool's candidate aggregates of the
    // current snapshot (derived by epp_pool_set)
    epp_admission_cfg adm{};
    bool adm_on = false;
    int32_t adm_pool_n = 0, adm_idle = 0, adm_cold = 0;
    double adm_sat = 0.0;
    EventSpans adm_spans;           // the admission launches of the device batch in flight (last_kernel_ms[7])
    int64_t kept_R = 0;             // rows of `hashes` valid for epp_index_add_picked
    int64_t shard_R = 0;            // rows of `hashes` valid for epp_shard_pick / epp_shard_merge
    bool shard_models = false;      // the probed batch had model ids: its copy in `model_ids` feeds epp_shard_pick
    bool shard_mm = false;          // the probed batch had multimodal flags: its copy in `multimodal` feeds pick and merge
    int32_t shard_stages = 1;       // records per request of the sharded protocol (epp_shard_set_staged)
    bool shard_seeded = false;      // the seeded tie rule (epp_shard_set_seeded): resolve, select, finish
    bool shard_picked = false;      // epp_shard_pick ran on the probed batch: its global masks are in sel_gmasks
    DevBuf sel_gmasks;              // seeded host-driven exchanges: the OR of the masks, kept for epp_shard_select
    DevBuf sel_work, sel_dense;     // seeded: [R][S] work items of k_shard_resolve and the dense-select list (slot counters
                                    // overflow_n[2] and [3])
    // endpoint-sharded mode over NVLink peer memory (shard_p2p.cu)
    void *p2p_buf = nullptr;        // this rank's exchange buffer {flags, masks, records} (cudaMalloc, IPC-exported)
    size_t p2p_bytes = 0, p2p_masks_off = 0, p2p_best_off = 0, p2p_sel_off = 0;
    bool p2p_seeded = false;        // the buffer was exported for the seeded tie rule (it holds the selected entries)
    int64_t p2p_R = 0;              // requests the buffer was sized for
    int32_t p2p_stages = 1;         // records per request the buffer was sized for
    int p2p_ranks = 0, p2p_rank = 0;
    bool p2p_ipc = false;
    std::vector<void *> p2p_peer;   // peers' buffers in this process's address space (own buffer at [p2p_rank])
    DevBuf p2p_peer_dev, p2p_gmasks, p2p_allbest, p2p_allsel, p2p_err;
    unsigned long long p2p_epoch = 0;
    uint64_t p2p_or_bits = 0;       // offsets alignment of the batch being stepped through epp_shard_p2p_phase
    bool p2p_broken = false;        // a wait timed out: the ranks are out of step until the buffers are connected again
    int p2p_launches = 0;

    epp_stats stats{};
};

static constexpr int kMaxModels = 4096;

static int32_t set_device(epp_engine *e) {
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    return EPP_OK;
}

// Orders stream 0 after whatever chunk-pipelined async batches left on stream 1 (no host synchronisation).  Every entry
// point that enqueues on stream 0 calls it first, so everything outside the pipelined path stays in call order.
static int32_t join_streams(epp_engine *e) {
    if (!e->s1_unjoined) return EPP_OK;
    CUDA_TRY(cudaEventRecord(e->slot[1].done, e->slot[1].stream));
    CUDA_TRY(cudaStreamWaitEvent(e->slot[0].stream, e->slot[1].done, 0));
    e->s1_unjoined = false;
    return EPP_OK;
}

// The endpoint-sharded mode (epp_shard_set): this rank's table and candidates cover a range of the endpoints only.
static bool sharded(const epp_engine *e) { return e->shard_begin != 0 || e->shard_end != 0xFFFFFFFFu; }

// ------------------------------------------------------------------------------------------------
// config
// ------------------------------------------------------------------------------------------------
extern "C" int32_t epp_abi_version(void) { return EPP_ABI_VERSION; }
extern "C" const char *epp_last_error(void) { return g_last_error.c_str(); }

extern "C" void epp_config_default(epp_config *cfg) {
    if (!cfg) return;
    memset(cfg, 0, sizeof *cfg);
    cfg->struct_size = sizeof(epp_config);
    cfg->device = 0;
    cfg->max_endpoints = 4096;
    cfg->block_size_tokens = 16;            // types.go:92
    cfg->max_prefix_blocks = 256;           // types.go:99
    cfg->lru_capacity_per_server = 31250;   // types.go:110
    cfg->handler = EPP_HANDLER_SINGLE;
    // config/loader/defaults.go:47-49, 78-87: queue 2, kv-cache-utilization 2, prefix 3 -- in that order
    cfg->primary.filter = EPP_FILTER_NONE;
    cfg->primary.n_scorers = 3;
    cfg->primary.scorers[0] = {EPP_SCORER_QUEUE, 0, 2.0, 0.0, 0.0};
    cfg->primary.scorers[1] = {EPP_SCORER_KV_UTIL, 0, 2.0, 0.0, 0.0};
    cfg->primary.scorers[2] = {EPP_SCORER_PREFIX, 0, 3.0, 0.0, 0.0};
    cfg->primary.ttft_column = cfg->prefill.ttft_column = cfg->encode.ttft_column = -1;   // no affinity filter, no TTFT column
}

// inflight: the token-load / active-request scorers read the engine's counters, whatever their column.
static int32_t validate_profile(const epp_profile_cfg &p, int n_ext, bool inflight, const char *name) {
    if (p.filter < EPP_FILTER_NONE || p.filter > EPP_FILTER_ENCODE) return fail(EPP_ERR_INVALID, "%s: bad filter %d", name, p.filter);
    if (p.n_scorers < 0 || p.n_scorers > EPP_MAX_SCORERS) return fail(EPP_ERR_INVALID, "%s: n_scorers %d out of range", name, p.n_scorers);
    for (int s = 0; s < p.n_scorers; s++) {
        const epp_scorer_cfg &sc = p.scorers[s];
        if (sc.kind < EPP_SCORER_PREFIX || sc.kind > EPP_SCORER_CONTEXT_LENGTH) return fail(EPP_ERR_INVALID, "%s: scorer %d has unknown kind %d", name, s, sc.kind);
        if (!std::isfinite(sc.weight)) return fail(EPP_ERR_INVALID, "%s: scorer %d weight is not finite", name, s);
        if (!inflight && (sc.kind == EPP_SCORER_TOKEN_LOAD || sc.kind == EPP_SCORER_ACTIVE_REQUEST) && (sc.column < 0 || sc.column >= n_ext))
            return fail(EPP_ERR_INVALID, "%s: scorer %d reads ext column %d, out of range [0,%d)", name, s, sc.column, n_ext);
        if (sc.kind == EPP_SCORER_EXTERNAL && (sc.param < 0 || sc.param >= n_ext)) return fail(EPP_ERR_INVALID, "%s: scorer %d external column %g out of range [0,%d)", name, s, sc.param, n_ext);
    }
    // prefix-cache-affinity-filter: Config.validate, filter/prefixcacheaffinity/plugin.go:87-98
    if (std::isnan(p.affinity_threshold) || p.affinity_threshold > 1.0) return fail(EPP_ERR_INVALID, "%s: affinityThreshold must be <= 1.0, got %f", name, p.affinity_threshold);
    if (!(p.exploration_probability >= 0.0 && p.exploration_probability <= 1.0)) return fail(EPP_ERR_INVALID, "%s: explorationProbability must be in [0, 1], got %f", name, p.exploration_probability);
    if (!(p.max_ttft_penalty_ms >= 0.0)) return fail(EPP_ERR_INVALID, "%s: maxTTFTPenaltyMs must be >= 0, got %f", name, p.max_ttft_penalty_ms);
    if (p.affinity_threshold > 0.0 && p.ttft_column >= n_ext) return fail(EPP_ERR_INVALID, "%s: ttft_column %d out of range [0,%d)", name, p.ttft_column, n_ext);
    if (p.picker < EPP_PICKER_MAX_SCORE || p.picker > EPP_PICKER_WEIGHTED_RANDOM) return fail(EPP_ERR_INVALID, "%s: unknown picker %d", name, p.picker);
    int n_cl = 0;
    for (int s = 0; s < p.n_scorers; s++) n_cl += p.scorers[s].kind == EPP_SCORER_CONTEXT_LENGTH;
    if (n_cl > 1) return fail(EPP_ERR_INVALID, "%s: the context-length scorer is listed %d times (at most once per profile)", name, n_cl);
    return EPP_OK;
}

static bool lists_scorer(const epp_profile_cfg &p, int kind) {
    for (int s = 0; s < p.n_scorers; s++)
        if (p.scorers[s].kind == kind) return true;
    return false;
}
static bool latency_piece(const epp_profile_cfg &p, const epp_latency_cfg &c) {
    return c.tier_filter || c.a1_affinity_threshold > 0.0 || lists_scorer(p, EPP_SCORER_LATENCY);
}
// A profile decided by the chain of pick_latency.cuh: a latency piece or the context-length plugin ("Context length").
static bool chain_profile(const epp_profile_cfg &p, const epp_latency_cfg &c) {
    return latency_piece(p, c) || lists_scorer(p, EPP_SCORER_CONTEXT_LENGTH);
}
// The rules a chain profile adds to validate_profile ("Latency predictions", "Context length").
static int32_t validate_latency(const epp_profile_cfg &p, const epp_latency_cfg &c, const char *name) {
    if (c.struct_size != sizeof(epp_latency_cfg)) return fail(EPP_ERR_INVALID, "epp_latency_cfg.struct_size %u != %zu", c.struct_size, sizeof(epp_latency_cfg));
    if (c.tier_filter != 0 && c.tier_filter != 1) return fail(EPP_ERR_INVALID, "%s: tier_filter %d must be 0 or 1", name, c.tier_filter);
    if (!(c.epsilon_explore_neg >= 0.0 && c.epsilon_explore_neg <= 1.0)) return fail(EPP_ERR_INVALID, "%s: epsilonExploreNeg must be in [0, 1], got %f", name, c.epsilon_explore_neg);
    if (std::isnan(c.a1_affinity_threshold) || c.a1_affinity_threshold > 1.0) return fail(EPP_ERR_INVALID, "%s: A1 affinityThreshold must be <= 1.0, got %f", name, c.a1_affinity_threshold);
    if (!(c.a1_exploration_probability >= 0.0 && c.a1_exploration_probability <= 1.0)) return fail(EPP_ERR_INVALID, "%s: A1 explorationProbability must be in [0, 1], got %f", name, c.a1_exploration_probability);
    if (!(c.a1_max_ttft_penalty_ms >= 0.0)) return fail(EPP_ERR_INVALID, "%s: A1 maxTTFTPenaltyMs must be >= 0, got %f", name, c.a1_max_ttft_penalty_ms);
    if (c.a1_affinity_threshold > 0.0 && !c.tier_filter) return fail(EPP_ERR_INVALID, "%s: an affinity filter before the tier filter needs the tier filter", name);
    if (c.strategy != EPP_HEADROOM_LEAST && c.strategy != EPP_HEADROOM_MOST) return fail(EPP_ERR_INVALID, "%s: unknown headroom strategy %d", name, c.strategy);
    const double w[5] = {c.ttft_weight, c.tpot_weight, c.composite_kv_weight, c.composite_queue_weight, c.composite_prefix_weight};
    for (double x : w) if (!std::isfinite(x)) return fail(EPP_ERR_INVALID, "%s: latency-scorer weights must be finite", name);
    const bool piece = chain_profile(p, c);
    if (piece && lists_scorer(p, EPP_SCORER_NO_HIT_LRU)) return fail(EPP_ERR_INVALID, "%s: the no-hit-lru scorer is not available on a latency or context-length profile", name);
    if (piece && p.ttft_column >= 0) return fail(EPP_ERR_INVALID, "%s: a latency or context-length profile reads TTFT from the predictions: ttft_column must be < 0", name);
    return EPP_OK;
}

static int32_t alloc_profile(epp_engine *e, ProfileState &ps, bool random_picker) {
    size_t E = (size_t)e->cfg.max_endpoints, Ep = (size_t)e->Epad;
    if (random_picker) {
        CUDA_TRY(ps.cands.reserve(sizeof(uint32_t) * E, &e->dev_bytes));
        CUDA_TRY(ps.wcum.reserve(sizeof(double) * (E + 1), &e->dev_bytes));
        CUDA_TRY(ps.icum.reserve(sizeof(uint32_t) * (E + 1), &e->dev_bytes));
    }
    CUDA_TRY(ps.cand.reserve(E, &e->dev_bytes));
    CUDA_TRY(ps.contrib.reserve(sizeof(double) * EPP_MAX_SCORERS * E, &e->dev_bytes));
    CUDA_TRY(ps.base.reserve(sizeof(double) * E, &e->dev_bytes));
    CUDA_TRY(ps.order.reserve(sizeof(uint32_t) * Ep, &e->dev_bytes));
    CUDA_TRY(ps.grp_size.reserve(sizeof(uint32_t) * Ep, &e->dev_bytes));
    CUDA_TRY(ps.sort_key.reserve(sizeof(uint64_t) * Ep, &e->dev_bytes));
    CUDA_TRY(ps.n_cand.reserve(sizeof(int32_t) * 4, &e->dev_bytes));
    CUDA_TRY(ps.qminmax.reserve(sizeof(int64_t) * (4 + EPP_MAX_SCORERS), &e->dev_bytes));
    return EPP_OK;
}

static int32_t rebuild_presence(epp_engine *h);
static ProfileDev profile_dev(epp_engine *h, int p, bool cold = false);
static epp_profile_cfg &profile_cfg(epp_engine *h, int p) {
    return p == 0 ? h->cfg.primary : (p == 1 ? h->cfg.prefill : h->cfg.encode);
}
static const epp_profile_cfg &profile_cfg(const epp_engine *h, int p) { return profile_cfg(const_cast<epp_engine *>(h), p); }
// Does any profile of the handler use a random picker?
static bool any_random_picker(const epp_engine *h) {
    for (int p = 0; p < h->n_alloc_profiles; p++)
        if (profile_cfg(h, p).picker != EPP_PICKER_MAX_SCORE) return true;
    return false;
}

extern "C" int32_t epp_engine_create(const epp_config *cfg, epp_engine **out) {
    if (!cfg || !out) return fail(EPP_ERR_INVALID, "cfg/out is NULL");
    *out = nullptr;
    if (cfg->struct_size != sizeof(epp_config)) return fail(EPP_ERR_INVALID, "epp_config.struct_size %u != %zu (ABI mismatch)", cfg->struct_size, sizeof(epp_config));
    if (cfg->max_endpoints <= 0 || cfg->max_endpoints > (1 << 24)) return fail(EPP_ERR_INVALID, "max_endpoints %d out of range", cfg->max_endpoints);
    if (cfg->block_size_tokens <= 0 || cfg->block_size_tokens > (1 << 20)) return fail(EPP_ERR_INVALID, "block_size_tokens %d must be > 0 (plugin.go:75-77)", cfg->block_size_tokens);
    if (cfg->max_prefix_blocks <= 0 || cfg->max_prefix_blocks > 65535) return fail(EPP_ERR_INVALID, "max_prefix_blocks %d out of range [1,65535]", cfg->max_prefix_blocks);
    if (cfg->lru_capacity_per_server <= 0) return fail(EPP_ERR_INVALID, "lru_capacity_per_server must be > 0");
    if (cfg->handler != EPP_HANDLER_SINGLE && cfg->handler != EPP_HANDLER_DISAGG) return fail(EPP_ERR_INVALID, "bad handler %d", cfg->handler);
    if (cfg->n_ext_cols < 0 || cfg->n_ext_cols > 64) return fail(EPP_ERR_INVALID, "n_ext_cols %d out of range", cfg->n_ext_cols);
    if (cfg->non_cached_tokens < 0) return fail(EPP_ERR_INVALID, "non_cached_tokens must be >= 0");
    if (cfg->inflight_load != 0 && cfg->inflight_load != 1) return fail(EPP_ERR_INVALID, "inflight_load %d must be 0 or 1", cfg->inflight_load);
    const bool inflight = cfg->inflight_load != 0;
    EPP_TRY(validate_profile(cfg->primary, cfg->n_ext_cols, inflight, "primary profile"));
    if (cfg->handler == EPP_HANDLER_DISAGG) EPP_TRY(validate_profile(cfg->prefill, cfg->n_ext_cols, inflight, "prefill profile"));
    if (cfg->encode_enabled) {
        if (cfg->handler != EPP_HANDLER_DISAGG) return fail(EPP_ERR_INVALID, "encode_enabled needs the disagg handler");
        EPP_TRY(validate_profile(cfg->encode, cfg->n_ext_cols, inflight, "encode profile"));
    }
    if (cfg->index_commit_interval_us < 0) return fail(EPP_ERR_INVALID, "index_commit_interval_us must be >= 0");
    if (cfg->pick_k < 0 || cfg->pick_k > 64) return fail(EPP_ERR_INVALID, "pick_k %d out of range [0,64]", cfg->pick_k);

    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    if (ce != cudaSuccess || ndev == 0)
        return fail(EPP_ERR_NO_DEVICE, "no CUDA device available (%s); the engine has no CPU fallback", ce == cudaSuccess ? "device count 0" : cudaGetErrorString(ce));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(EPP_ERR_INVALID, "device %d out of range [0,%d)", cfg->device, ndev);

    std::unique_ptr<epp_engine> e(new epp_engine());
    e->cfg = *cfg;
    e->cfg_user = *cfg;
    e->n_profiles = cfg->handler == EPP_HANDLER_DISAGG ? 2 : 1;
    e->n_alloc_profiles = cfg->encode_enabled ? 3 : e->n_profiles;
    e->n_ext_total = cfg->n_ext_cols;
    if (inflight) {
        // the counters live in two engine-owned ext columns behind the caller's: every kernel that reads a token-load /
        // active-request column reads them unchanged
        e->inflight = true;
        e->n_ext_total = cfg->n_ext_cols + 2;
        for (int pi = 0; pi < e->n_alloc_profiles; pi++) {
            epp_profile_cfg &pc = profile_cfg(e.get(), pi);
            for (int si = 0; si < pc.n_scorers; si++) {
                if (pc.scorers[si].kind == EPP_SCORER_TOKEN_LOAD) pc.scorers[si].column = cfg->n_ext_cols;
                else if (pc.scorers[si].kind == EPP_SCORER_ACTIVE_REQUEST) pc.scorers[si].column = cfg->n_ext_cols + 1;
                else continue;
                e->inflight_mask |= 1 << pi;
            }
        }
    }
    CUDA_TRY(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
    e->sm_count = prop.multiProcessorCount;
    e->max_smem_optin = prop.sharedMemPerBlockOptin;
    if (prop.l2CacheSize > 0) e->l2_table_bytes = (uint64_t)prop.l2CacheSize / 2;
    int32_t Ep = 1;
    while (Ep < cfg->max_endpoints) Ep <<= 1;
    e->Epad = Ep;
    for (int i = 0; i < 2; i++) {
        CUDA_TRY(cudaStreamCreateWithFlags(&e->slot[i].stream, cudaStreamNonBlocking));
        CUDA_TRY(cudaEventCreateWithFlags(&e->slot[i].done, cudaEventDisableTiming));
    }
    for (auto &ev : e->ev) CUDA_TRY(cudaEventCreate(&ev));
    for (auto &ev : e->user_ev) CUDA_TRY(cudaEventCreate(&ev));
    CUDA_TRY(cudaHostAlloc(reinterpret_cast<void **>(&e->wc_host), sizeof(unsigned long long) * 4, cudaHostAllocDefault));
    size_t E = (size_t)cfg->max_endpoints;
    CUDA_TRY(e->seeds.reserve(sizeof(uint64_t) * kMaxModels, &e->dev_bytes));
    CUDA_TRY(e->seed_msg.reserve(4096, &e->dev_bytes));
    CUDA_TRY(e->role.reserve(E, &e->dev_bytes));
    CUDA_TRY(e->kv.reserve(sizeof(double) * E, &e->dev_bytes));
    CUDA_TRY(e->waiting.reserve(sizeof(int32_t) * E, &e->dev_bytes));
    CUDA_TRY(e->running.reserve(sizeof(int32_t) * E, &e->dev_bytes));
    if (e->n_ext_total) CUDA_TRY(e->ext.reserve(sizeof(double) * E * (size_t)e->n_ext_total, &e->dev_bytes));
    if (e->inflight) {
        CUDA_TRY(e->if_req.reserve(sizeof(int64_t) * E, &e->dev_bytes));
        CUDA_TRY(e->if_tok.reserve(sizeof(int64_t) * E, &e->dev_bytes));
        CUDA_TRY(cudaMemset(e->if_req.p, 0, sizeof(int64_t) * E));
        CUDA_TRY(cudaMemset(e->if_tok.p, 0, sizeof(int64_t) * E));
        CUDA_TRY(cudaMemset(e->ext.as<double>() + E * (size_t)cfg->n_ext_cols, 0, sizeof(double) * E * 2));
        for (auto &ev : e->if_ev) CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    }
    for (int p = 0; p < e->n_alloc_profiles; p++) EPP_TRY(alloc_profile(e.get(), e->prof[p], profile_cfg(e.get(), p).picker != 0));
    CUDA_TRY(e->idx_cursor.reserve(sizeof(uint32_t) * 4, &e->dev_bytes));
    CUDA_TRY(e->idx_special.reserve(sizeof(IndexSlot), &e->dev_bytes));
    CUDA_TRY(e->get_out.reserve(sizeof(uint32_t) * 4096 + 16, &e->dev_bytes));
    CUDA_TRY(e->flag.reserve(sizeof(int) * 4, &e->dev_bytes));
    CUDA_TRY(e->work_counters.reserve(sizeof(unsigned long long) * 4, &e->dev_bytes));
    memset(&e->idx_special_host, 0, sizeof(IndexSlot));
    e->idx_special_host.key = kEmptyKey;
    for (int pi = 0; pi < e->n_alloc_profiles; pi++) {
        const epp_profile_cfg &pc = profile_cfg(e.get(), pi);
        for (int si = 0; si < pc.n_scorers; si++) if (pc.scorers[si].kind == EPP_SCORER_LORA_AFFINITY) e->lora_enabled = true;
    }
    for (int pi = 0; pi < e->n_alloc_profiles; pi++) {
        const epp_profile_cfg &pc = profile_cfg(e.get(), pi);
        for (int si = 0; si < pc.n_scorers; si++) {
            if (pc.scorers[si].kind != EPP_SCORER_NO_HIT_LRU) continue;
            if (e->nohit_mask & (1 << pi)) return fail(EPP_ERR_INVALID, "profile %d lists the no-hit-lru scorer twice", pi);
            const double p = pc.scorers[si].param;
            if (std::isnan(p) || p > (double)(1 << 30) || (p > 0.0 && p != std::floor(p)))
                return fail(EPP_ERR_INVALID, "no-hit-lru lruSize %g must be an integer <= 2^30 (<= 0: 1024)", p);
            const int32_t lru = p <= 0.0 ? 1024 : (int32_t)p;             // no_hit_lru.go:93-95
            if (e->nohit_mask && lru != e->nohit_lru)
                return fail(EPP_ERR_INVALID, "the no-hit-lru scorer has lruSize %d in one profile and %d in another: the profiles share one LRU", e->nohit_lru, lru);
            e->nohit_mask |= 1 << pi;
            e->nohit_lru = lru;
        }
    }
    if (e->nohit_mask) {
        CUDA_TRY(e->nh_last_seq.reserve(sizeof(uint64_t) * E, &e->dev_bytes));
        CUDA_TRY(e->nh_pos.reserve(sizeof(int32_t) * E, &e->dev_bytes));
        CUDA_TRY(e->nh_misc.reserve(sizeof(int32_t) * 4, &e->dev_bytes));
        CUDA_TRY(e->nh_sort_key.reserve(sizeof(uint64_t) * (size_t)e->Epad, &e->dev_bytes));
        CUDA_TRY(e->nh_order.reserve(sizeof(uint32_t) * (size_t)e->Epad, &e->dev_bytes));
        CUDA_TRY(cudaMemset(e->nh_last_seq.p, 0, sizeof(uint64_t) * E));
        CUDA_TRY(cudaMemset(e->nh_pos.p, 0xFF, sizeof(int32_t) * E));
        CUDA_TRY(cudaMemset(e->nh_misc.p, 0, sizeof(int32_t) * 4));
        for (int pi = 0; pi < e->n_alloc_profiles; pi++)
            if (e->nohit_mask & (1 << pi)) {
                EPP_TRY(alloc_profile(e.get(), e->prof_cold[pi], profile_cfg(e.get(), pi).picker != 0));
                CUDA_TRY(e->nh_col[pi].reserve(sizeof(double) * E, &e->dev_bytes));
            }
    }
    e->general = cfg->pick_k > 1;
    for (int pi = 0; pi < e->n_alloc_profiles; pi++)
        if (profile_cfg(e.get(), pi).affinity_threshold > 0.0) e->general = true;
    for (int pi = 0; pi < e->n_alloc_profiles; pi++) {
        epp_latency_cfg_default(&e->lat_cfg[pi]);
        const epp_profile_cfg &pc = profile_cfg(e.get(), pi);
        EPP_TRY(validate_latency(pc, e->lat_cfg[pi], pi == 0 ? "primary profile" : (pi == 1 ? "prefill profile" : "encode profile")));
        if (chain_profile(pc, e->lat_cfg[pi])) e->lat_mask |= 1 << pi;
        if (!lists_scorer(pc, EPP_SCORER_CONTEXT_LENGTH)) continue;
        e->cl_mask |= 1 << pi;
        e->cl_label[pi] = EPP_CONTEXT_LENGTH_LABEL;
        const std::vector<longlong2> absent(E, longlong2{kRangeAbsent, 0});     // no labels yet
        CUDA_TRY(e->cl_rng[pi].reserve(sizeof(longlong2) * E, &e->dev_bytes));
        CUDA_TRY(cudaMemcpy(e->cl_rng[pi].p, absent.data(), sizeof(longlong2) * E, cudaMemcpyHostToDevice));
    }
    if (e->lat_mask) e->general = true;
    e->store.reset(new IndexStore((uint32_t)cfg->max_endpoints, cfg->lru_capacity_per_server, e->sm_count));
    { const char *v1 = getenv("EPP_INDEX_PATCH"); e->patch_enabled = v1 ? atoi(v1) : 1; }
    { const char *v1 = getenv("EPP_INDEX_LOAD"); e->index_load = v1 ? std::max(2, atoi(v1)) : 0; }
    { const char *v1 = getenv("EPP_DEV_CHUNKS"); e->dev_chunks = v1 ? std::max(1, atoi(v1)) : 2; }
    { const char *v1 = getenv("EPP_HASH_TRIM"); e->hash_trim = v1 ? atoi(v1) : 1; }
    { const char *v1 = getenv("EPP_HASH_SKIP"); e->hash_skip = v1 ? atoi(v1) : 1; }
    { const char *v1 = getenv("EPP_PRESENCE_LOG2BITS"); e->presence_log2_env = v1 ? std::min(30, std::max(6, atoi(v1))) : 0; }
    { const char *v1 = getenv("EPP_SMALL_BATCH"); e->small_max = v1 ? std::max(0, atoi(v1)) : 1024; }
    { const char *v1 = getenv("EPP_SMALL_ZEROCOPY"); e->small_zc_max = v1 ? std::max(0, atoi(v1)) : 8; }
    { const char *v1 = getenv("EPP_SMALL_PIPELINE"); e->small_pipe_min = v1 ? std::max(0, atoi(v1)) : 1; }
    CUDA_TRY(e->small_arrive.reserve(sizeof(uint32_t) * 16, &e->dev_bytes));
    CUDA_TRY(cudaMemset(e->small_arrive.p, 0, sizeof(uint32_t) * 16));
    CUDA_TRY(cudaHostAlloc(reinterpret_cast<void **>(&e->small_epoch_host), 64, cudaHostAllocDefault));
    CUDA_TRY(e->small_overflow_n.reserve(sizeof(int32_t) * 4, &e->dev_bytes));
    CUDA_TRY(cudaMemset(e->small_overflow_n.p, 0, sizeof(int32_t) * 4));
    for (int i = 0; i < 2; i++) CUDA_TRY(e->slot[i].overflow_n.reserve(sizeof(int32_t) * 4, &e->dev_bytes));
    for (int i = 0; i < 2; i++) CUDA_TRY(e->slot[i].hash_next.reserve(sizeof(uint32_t), &e->dev_bytes));
    EPP_TRY(rebuild_presence(e.get()));              // the empty index: every bit clear
    if (e->nohit_mask) {
        ProfileDev cold[kMaxProfiles];
        memset(cold, 0, sizeof cold);
        for (int pi = 0; pi < e->n_alloc_profiles; pi++)
            if (e->nohit_mask & (1 << pi)) cold[pi] = profile_dev(e.get(), pi, true);
        CUDA_TRY(e->nh_prof.reserve(sizeof cold, &e->dev_bytes));
        CUDA_TRY(cudaMemcpy(e->nh_prof.p, cold, sizeof cold, cudaMemcpyHostToDevice));
    }

    // match/pick launch geometry: counters in shared memory when they fit, else zeroed global scratch
    size_t smem_local = match_pick_smem_bytes(cfg->max_endpoints, false);
    e->pick_global = smem_local > std::min<size_t>(e->max_smem_optin, 200 * 1024);
    e->pick_smem = match_pick_smem_bytes(cfg->max_endpoints, e->pick_global);
    int ctas_per_sm = e->pick_global ? 4 : std::max<int>(1, (int)((size_t)(220 * 1024) / (e->pick_smem + 1024)));
    ctas_per_sm = std::min(ctas_per_sm, 8);
    e->pick_grid = e->sm_count * ctas_per_sm;
    if (e->pick_global) {
        size_t words = (size_t)e->pick_grid * match_pick_warps_per_cta() * (size_t)((cfg->max_endpoints + 1) / 2);
        for (int i = 0; i < 2; i++) {
            CUDA_TRY(e->slot[i].pick_scratch.reserve(words * sizeof(uint32_t), &e->dev_bytes));
            CUDA_TRY(cudaMemset(e->slot[i].pick_scratch.p, 0, words * sizeof(uint32_t)));
        }
    }
    CUDA_TRY(cudaDeviceSynchronize());
    *out = e.release();
    return EPP_OK;
}

extern "C" int32_t epp_engine_destroy(epp_engine *h) {
    if (!h) return EPP_OK;
    cudaSetDevice(h->cfg.device);
    cudaDeviceSynchronize();
    if (h->in_ev) cudaEventDestroy(h->in_ev);
    for (int i = 0; i < 2; i++) {
        if (h->slot[i].stream) cudaStreamDestroy(h->slot[i].stream);
        if (h->slot[i].done) cudaEventDestroy(h->slot[i].done);
    }
    for (auto &ev : h->ev) if (ev) cudaEventDestroy(ev);
    for (auto &ev : h->user_ev) if (ev) cudaEventDestroy(ev);
    if (h->wc_host) cudaFreeHost(h->wc_host);
    if (h->small_host) cudaFreeHost(h->small_host);
    if (h->small_epoch_host) cudaFreeHost(h->small_epoch_host);
    for (auto &ev : h->if_ev) if (ev) cudaEventDestroy(ev);
    for (int g = 0; g < (int)h->p2p_peer.size(); g++)
        if (h->p2p_ipc && g != h->p2p_rank && h->p2p_peer[g]) cudaIpcCloseMemHandle(h->p2p_peer[g]);
    if (h->p2p_buf) cudaFree(h->p2p_buf);
    delete h;
    return EPP_OK;
}

extern "C" int32_t epp_host_alloc(size_t bytes, void **out) {
    if (!out) return fail(EPP_ERR_INVALID, "out is NULL");
    CUDA_TRY(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
    return EPP_OK;
}
extern "C" int32_t epp_host_free(void *p) {
    if (p) CUDA_TRY(cudaFreeHost(p));
    return EPP_OK;
}

// ------------------------------------------------------------------------------------------------
// models: h_{-1} = XXH64(model || salt) on the device (hashing.go:71-78)
// ------------------------------------------------------------------------------------------------
extern "C" int32_t epp_model_register(epp_engine *h, const uint8_t *model, size_t model_len, const uint8_t *salt,
                                      size_t salt_len, uint32_t *out_model_id) {
    if (!h || !out_model_id) return fail(EPP_ERR_INVALID, "NULL argument");
    if ((model_len && !model) || (salt_len && !salt)) return fail(EPP_ERR_INVALID, "NULL model/salt with non-zero length");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (h->n_models >= kMaxModels) return fail(EPP_ERR_CAPACITY, "too many registered models (max %d)", kMaxModels);
    size_t n = model_len + salt_len;
    std::vector<uint8_t> msg(n ? n : 1);
    if (model_len) memcpy(msg.data(), model, model_len);
    if (salt_len) memcpy(msg.data() + model_len, salt, salt_len);
    CUDA_TRY(h->seed_msg.reserve(n + 16, &h->dev_bytes));
    cudaStream_t s = h->slot[0].stream;
    if (n) CUDA_TRY(cudaMemcpyAsync(h->seed_msg.p, msg.data(), n, cudaMemcpyHostToDevice, s));
    CUDA_TRY(launch_hash_bytes(h->seed_msg.as<uint8_t>(), n, h->seeds.as<uint64_t>() + h->n_models, s));
    uint64_t seed = 0;
    CUDA_TRY(cudaMemcpyAsync(&seed, h->seeds.as<uint64_t>() + h->n_models, sizeof seed, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    h->host_seeds.push_back(seed);
    *out_model_id = (uint32_t)h->n_models++;
    return EPP_OK;
}

extern "C" int32_t epp_model_seed(epp_engine *h, uint32_t model_id, uint64_t *out_seed) {
    if (!h || !out_seed) return fail(EPP_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(h->mu);
    if ((int)model_id >= h->n_models) return fail(EPP_ERR_INVALID, "unknown model id %u", model_id);
    *out_seed = h->host_seeds[model_id];
    return EPP_OK;
}

// ------------------------------------------------------------------------------------------------
// pool state
// ------------------------------------------------------------------------------------------------
static LoraDev lora_dev(epp_engine *h) {
    LoraDev L{};
    L.enabled = h->lora_enabled ? 1 : 0;
    if (h->lora_set) {
        L.max_active = h->lora_max.as<int32_t>();
        L.n_loaded = h->lora_cnt.as<int32_t>();
        L.ptr = h->lora_ptr.as<uint32_t>();
        L.ep = h->lora_ep.as<uint32_t>();
        L.state = h->lora_state.as<uint8_t>();
        L.n_models = h->lora_models;
    }
    return L;
}

static PoolArrays pool_arrays(epp_engine *h) {
    PoolArrays pa;
    pa.E = h->cfg.max_endpoints;
    pa.n_ext_cols = h->n_ext_total;
    pa.role = h->role.as<uint8_t>();
    pa.kv_usage = h->kv.as<double>();
    pa.waiting = h->waiting.as<int32_t>();
    pa.running = h->running.as<int32_t>();
    pa.ext = h->ext.as<double>();
    pa.lora = lora_dev(h);
    return pa;
}

// Profile p's warm set, or (cold) its no-hit-lru cold set: the cold set has the warm set's candidates (cand / n_cand /
// qminmax) and its own contributions, base sums, order, groups and random-picker arrays.
static ProfileDerived profile_derived(epp_engine *h, int p, bool cold) {
    const ProfileState &w = h->prof[p], &x = cold ? h->prof_cold[p] : w;
    ProfileDerived d{};
    d.cand = w.cand.as<uint8_t>();
    d.n_cand = w.n_cand.as<int32_t>();
    d.qminmax = w.qminmax.as<int64_t>();
    d.contrib = x.contrib.as<double>();
    d.base = x.base.as<double>();
    d.order = x.order.as<uint32_t>();
    d.grp_size = x.grp_size.as<uint32_t>();
    d.sort_key = x.sort_key.as<uint64_t>();
    d.cands = x.cands.as<uint32_t>();
    d.wcum = x.wcum.as<double>();
    d.icum = x.icum.as<uint32_t>();
    return d;
}

// What the pick kernels read of the same set.
static ProfileDev profile_dev(epp_engine *h, int p, bool cold) {
    const ProfileDerived d = profile_derived(h, p, cold);
    ProfileDev pd;
    pd.cfg = profile_cfg(h, p);
    pd.cand = d.cand;
    pd.contrib = d.contrib;
    pd.base = d.base;
    pd.order = d.order;
    pd.grp_size = d.grp_size;
    pd.n_cand = d.n_cand;
    pd.cands = d.cands;
    pd.wcum = d.wcum;
    pd.icum = d.icum;
    return pd;
}

static NoHitState nohit_state(epp_engine *h) {
    NoHitState st;
    st.last_seq = h->nh_last_seq.as<uint64_t>();
    st.pos = h->nh_pos.as<int32_t>();
    st.n_members = h->nh_misc.as<int32_t>();
    st.dirty = h->nh_misc.as<int32_t>() + 1;
    st.sort_key = h->nh_sort_key.as<uint64_t>();
    st.order = h->nh_order.as<uint32_t>();
    st.lru_size = h->nohit_lru;
    return st;
}

// The cold set of every profile with the no-hit-lru scorer: its LRU column over the profile's candidates, and the base
// sums / order / groups with that column (the warm set holds 0.5).  gated: only if an Add happened since the last time.
static int32_t nohit_derive(epp_engine *h, cudaStream_t s, bool gated, int *launches) {
    if (!h->nohit_mask) return EPP_OK;
    const NoHitState st = nohit_state(h);
    PoolArrays pa = pool_arrays(h);
    for (int p = 0; p < h->n_alloc_profiles; p++) {
        if (!(h->nohit_mask & (1 << p))) continue;
        const ProfileDerived d = profile_derived(h, p, true);
        double *col = h->nh_col[p].as<double>();
        CUDA_TRY(launch_nohit_column(st, h->cfg.max_endpoints, d.cand, d.n_cand, col, gated, s, launches));
        CUDA_TRY(launch_pool_order(pa, profile_cfg(h, p), d, h->Epad, col, gated ? st.dirty : nullptr, s, launches));
    }
    return EPP_OK;
}

// PreRequest of the no-hit-lru scorer for one scheduling call (no_hit_lru.go:279-321), enqueued on s behind the call's
// last pick kernel: the cold requests' picks are Added in request order, then the LRU is trimmed and re-ranked and the
// cold sets re-derived -- all on the device, and all but the first kernel return at once when no request was cold.
// dec / the cold scratch hold the call's R requests.
static int32_t nohit_update(epp_engine *h, const epp_decision *dec, int64_t R, cudaStream_t s, int *launches) {
    if (!h->nohit_mask || R <= 0) return EPP_OK;
    const NoHitState st = nohit_state(h);
    CUDA_TRY(launch_nohit_touch(st, dec, h->nh_cold.as<uint8_t>(), R, h->nohit_seq, s, launches));
    h->nohit_seq += 2 * (uint64_t)R;
    CUDA_TRY(launch_nohit_rank(st, h->cfg.max_endpoints, h->Epad, true, s, launches));
    EPP_TRY(nohit_derive(h, s, true, launches));
    CUDA_TRY(launch_nohit_clear(st, s, launches));
    return EPP_OK;
}

// The no-hit-lru view of a pick launch whose first request is r0.
static NoHitView nohit_view(epp_engine *h, int64_t r0) {
    NoHitView v;
    memset(&v, 0, sizeof v);
    v.mask = h->nohit_mask;
    if (!v.mask) return v;
    v.cold = h->nh_prof.as<ProfileDev>();
    v.cold_out = h->nh_cold.as<uint8_t>() + r0;
    return v;
}

static LabelFilterDev label_dev(epp_engine *h, int p) {
    LabelFilterDev d = h->labels.dev[p];
    d.lcode = h->lcode.as<uint8_t>();
    return d;
}

// Request-independent scorer terms of profile p from the current pool (+ LoRA, + labels) snapshot, on the device.
static int32_t derive_profile(epp_engine *h, int p, cudaStream_t s, int *launches) {
    CUDA_TRY(launch_pool_prepare(pool_arrays(h), profile_cfg(h, p), label_dev(h, p), profile_derived(h, p, false), h->Epad,
                                 h->shard_begin, h->shard_end, s, launches));
    return EPP_OK;
}

static int32_t derive_pool(epp_engine *h) {
    cudaStream_t s = h->slot[0].stream;
    int launches = 0;
    for (int p = 0; p < h->n_alloc_profiles; p++) EPP_TRY(derive_profile(h, p, s, &launches));
    return nohit_derive(h, s, false, &launches);
}

// ---- inflight-load producer (inflight.cu) ---------------------------------------------------------------------------
static InflightState inflight_state(epp_engine *h) {
    InflightState st;
    const size_t E = (size_t)h->cfg.max_endpoints;
    st.req = h->if_req.as<int64_t>();
    st.tok = h->if_tok.as<int64_t>();
    st.col_tok = h->ext.as<double>() + E * (size_t)h->cfg.n_ext_cols;
    st.col_req = st.col_tok + E;
    st.E = h->cfg.max_endpoints;
    return st;
}

// After the counters changed: their columns, and every term derived from them -- the profiles that list a token-load or
// active-request scorer (launch_pool_prepare, random pickers' cumulative arrays included) and the no-hit-lru cold sets,
// which are built on those profiles' candidates and load maxima.
static int32_t inflight_rederive(epp_engine *h, cudaStream_t s, int *launches) {
    if (!h->inflight_mask) return EPP_OK;
    CUDA_TRY(launch_inflight_columns(inflight_state(h), s, launches));
    for (int p = 0; p < h->n_alloc_profiles; p++)
        if (h->inflight_mask & (1 << p)) EPP_TRY(derive_profile(h, p, s, launches));
    if (h->inflight_mask & h->nohit_mask) EPP_TRY(nohit_derive(h, s, false, launches));
    return EPP_OK;
}

// PreRequest of the producer for one scheduling call (producer.go:110-129), enqueued on s behind the call's last pick
// kernel.  dec / det / in_len hold the call's R requests (det, in_len may be nullptr).
static int32_t inflight_update(epp_engine *h, const epp_decision *dec, const epp_decision_detail *det, const int64_t *in_len,
                               int64_t R, cudaStream_t s, int *launches) {
    if (!h->inflight || R <= 0) return EPP_OK;
    CUDA_TRY(launch_inflight_add(inflight_state(h), dec, det, in_len, R, s, launches));
    return inflight_rederive(h, s, launches);
}

// Everything a scheduling call updates behind its last pick kernel, in this order: the no-hit-lru LRU, then the in-flight
// counters.  Per-call state that a pick changes is updated here and only here, so that every scheduling path carries it
// alike.  timed (the device batch in flight): each update that is on is bracketed by its event pair for finish_async
// (post_pick_timed).
static int32_t after_picks(epp_engine *h, const epp_decision *dec, const epp_decision_detail *det, const int64_t *in_len,
                           int64_t R, cudaStream_t s, int *launches, bool timed) {
    if (h->nohit_mask) {
        if (timed) CUDA_TRY(cudaEventRecord(h->ev[5], s));
        EPP_TRY(nohit_update(h, dec, R, s, launches));
        if (timed) { CUDA_TRY(cudaEventRecord(h->ev[6], s)); h->post_pick_timed[0] = true; }
    }
    if (h->inflight) {
        if (timed) CUDA_TRY(cudaEventRecord(h->ev[7], s));
        EPP_TRY(inflight_update(h, dec, det, in_len, R, s, launches));
        if (timed) { CUDA_TRY(cudaEventRecord(h->ev[8], s)); h->post_pick_timed[1] = true; }
    }
    return EPP_OK;
}

// Applies the releases and resets folded since the last time (one copy + one kernel on s), then re-derives.
static int32_t inflight_flush(epp_engine *h, cudaStream_t s, int *launches) {
    if (!h->inflight) return EPP_OK;
    std::vector<InflightDelta> d;
    {
        std::lock_guard<std::mutex> lk(h->if_mu);
        if (h->if_pending.empty()) return EPP_OK;
        d.reserve(h->if_pending.size());
        for (const auto &kv : h->if_pending) d.push_back(kv.second);
        h->if_pending.clear();
    }
    const int k = h->if_flip;
    h->if_flip ^= 1;
    CUDA_TRY(cudaEventSynchronize(h->if_ev[k]));      // the apply kernel that last read staging set k has run
    const size_t bytes = sizeof(InflightDelta) * d.size();
    CUDA_TRY(h->if_host[k].reserve(bytes));
    memcpy(h->if_host[k].p, d.data(), bytes);
    CUDA_TRY(h->if_dev[k].reserve(bytes, &h->dev_bytes));
    CUDA_TRY(cudaMemcpyAsync(h->if_dev[k].p, h->if_host[k].p, bytes, cudaMemcpyHostToDevice, s));
    CUDA_TRY(launch_inflight_apply(inflight_state(h), h->if_dev[k].as<InflightDelta>(), (int32_t)d.size(), s, launches));
    CUDA_TRY(cudaEventRecord(h->if_ev[k], s));
    return inflight_rederive(h, s, launches);
}

// ---- admission (admit.cu) ------------------------------------------------------------------------------------------
// Go's math.Max (Inf, then NaN, then the sign of zero): the probabilistic-admitter's per-endpoint saturation term.
static double go_max(double x, double y) {
    if (std::isinf(x) && x > 0) return x;
    if (std::isinf(y) && y > 0) return y;
    if (std::isnan(x) || std::isnan(y)) return std::nan("");
    if (x == 0 && x == y) return std::signbit(x) ? y : x;
    return x > y ? x : y;
}

// The whole pool's candidate aggregates of a new snapshot (slot-indexed arrays, role 0xFF = absent): the count, whether
// one is idle (running == 0) or cold (kv < 0.02), and the saturation terms folded from +0.0 in ascending slot order.  They
// reach k_admit as launch arguments, so a batch enqueued before the next epp_pool_set keeps deciding on these.
static void admission_derive(epp_engine *h, const std::vector<uint8_t> &role, const std::vector<double> &kv,
                             const std::vector<int32_t> &waiting, const std::vector<int32_t> &running) {
    const double qdt = (double)h->adm.queue_depth_threshold, kvt = h->adm.kv_cache_util_threshold;
    int32_t n = 0, idle = 0, cold = 0;
    double sat = 0.0;
    for (size_t e = 0; e < role.size(); e++) {
        if (role[e] == 0xFF) continue;
        n++;
        idle |= running[e] == 0;
        cold |= kv[e] < 0.02;
        sat += go_max((double)waiting[e] / qdt, kv[e] / kvt);
    }
    h->adm_pool_n = n;
    h->adm_idle = idle;
    h->adm_cold = cold;
    h->adm_sat = sat;
}

extern "C" void epp_admission_cfg_default(epp_admission_cfg *cfg) {
    if (!cfg) return;
    memset(cfg, 0, sizeof *cfg);
    cfg->struct_size = sizeof(epp_admission_cfg);
    cfg->queue_depth_threshold = 5;                   // probabilisticadmitter/plugin.go:38-41
    cfg->kv_cache_util_threshold = 0.8;
    cfg->power = 5.0;
    cfg->k = 300.0;
}

extern "C" int32_t epp_admission_set(epp_engine *h, const epp_admission_cfg *cfg) {
    if (!h || !cfg) return fail(EPP_ERR_INVALID, "NULL engine or configuration");
    if (cfg->struct_size != sizeof(epp_admission_cfg))
        return fail(EPP_ERR_INVALID, "epp_admission_cfg.struct_size %u != %zu", cfg->struct_size, sizeof(epp_admission_cfg));
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->pool_called) return fail(EPP_ERR_STATE, "the admitters are fixed once the pool has been set");
    if (sharded(h) || h->p2p_buf)
        return fail(EPP_ERR_INVALID, "admission is not available in the endpoint-sharded and peer-memory modes");
    if ((cfg->latency_slo != 0 && cfg->latency_slo != 1) || (cfg->probabilistic != 0 && cfg->probabilistic != 1))
        return fail(EPP_ERR_INVALID, "latency_slo and probabilistic must be 0 or 1");
    // probabilisticadmitter.Factory's checks and messages (plugin.go:71-84); the finiteness checks are the C side's own
    if (cfg->queue_depth_threshold <= 0)
        return fail(EPP_ERR_INVALID, "plugin 'probabilistic-admitter': queueDepthThreshold must be > 0, got %d", cfg->queue_depth_threshold);
    if (!(cfg->kv_cache_util_threshold > 0.0) || !std::isfinite(cfg->kv_cache_util_threshold))
        return fail(EPP_ERR_INVALID, "plugin 'probabilistic-admitter': kvCacheUtilThreshold must be > 0, got %g", cfg->kv_cache_util_threshold);
    if (!(cfg->power > 0) || !std::isfinite(cfg->power))
        return fail(EPP_ERR_INVALID, "plugin 'probabilistic-admitter': power must be > 0, got %g", cfg->power);
    if (!(cfg->k > 0) || !std::isfinite(cfg->k))
        return fail(EPP_ERR_INVALID, "plugin 'probabilistic-admitter': k must be > 0, got %g", cfg->k);
    h->adm = *cfg;
    h->adm_on = cfg->latency_slo || cfg->probabilistic;
    return EPP_OK;
}

extern "C" int32_t epp_pool_set(epp_engine *h, int32_t n, const uint32_t *ids, const uint8_t *role,
                                const double *kv_usage, const int32_t *waiting, const int32_t *running,
                                const double *ext) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    if (n < 0 || (n > 0 && (!ids || !role || !kv_usage || !waiting))) return fail(EPP_ERR_INVALID, "NULL pool arrays");
    if (h->cfg.n_ext_cols > 0 && n > 0 && !ext) return fail(EPP_ERR_INVALID, "ext columns configured but ext is NULL");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    const int32_t E = h->cfg.max_endpoints;
    std::vector<uint8_t> r(E, 0xFF);
    std::vector<double> kv(E, 0.0);
    std::vector<int32_t> w(E, 0), run(E, 0);
    std::vector<double> ex((size_t)E * (size_t)std::max(1, h->cfg.n_ext_cols), 0.0);
    for (int32_t i = 0; i < n; i++) {
        uint32_t id = ids[i];
        if (id >= (uint32_t)E) return fail(EPP_ERR_INVALID, "pool entry %d: slot id %u >= max_endpoints %d", i, id, E);
        if (r[id] != 0xFF) return fail(EPP_ERR_INVALID, "pool entry %d: duplicate slot id %u", i, id);
        if (role[i] > EPP_ROLE_OTHER) return fail(EPP_ERR_INVALID, "pool entry %d: bad role %u", i, role[i]);
        if (std::isnan(kv_usage[i])) return fail(EPP_ERR_INVALID, "pool entry %d: kv_usage is NaN", i);
        r[id] = role[i];
        kv[id] = kv_usage[i];
        w[id] = waiting[i];
        run[id] = running ? running[i] : 0;
        for (int c = 0; c < h->cfg.n_ext_cols; c++) {
            double v = ext[(size_t)c * (size_t)n + (size_t)i];
            if (std::isnan(v)) return fail(EPP_ERR_INVALID, "pool entry %d: ext column %d is NaN", i, c);
            ex[(size_t)c * (size_t)E + id] = v;
        }
    }
    cudaStream_t s = h->slot[0].stream;
    CUDA_TRY(cudaMemcpyAsync(h->role.p, r.data(), E, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(h->kv.p, kv.data(), sizeof(double) * E, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(h->waiting.p, w.data(), sizeof(int32_t) * E, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(h->running.p, run.data(), sizeof(int32_t) * E, cudaMemcpyHostToDevice, s));
    if (h->cfg.n_ext_cols)
        CUDA_TRY(cudaMemcpyAsync(h->ext.p, ex.data(), sizeof(double) * E * (size_t)h->cfg.n_ext_cols, cudaMemcpyHostToDevice, s));
    EPP_TRY(derive_pool(h));
    CUDA_TRY(cudaStreamSynchronize(s));
    if (h->adm_on) admission_derive(h, r, kv, w, run);
    h->pool_ready = true;
    h->pool_called = true;
    return EPP_OK;
}

extern "C" int32_t epp_pool_set_lora(epp_engine *h, int32_t n, const uint32_t *ids, const int32_t *max_active_models,
                                     const int32_t *n_models_loaded, int64_t n_members, const uint32_t *member_ep,
                                     const uint32_t *member_model, const uint8_t *member_state) {
    if (!h || n < 0 || n_members < 0) return fail(EPP_ERR_INVALID, "bad arguments");
    if (n > 0 && (!ids || !max_active_models || !n_models_loaded)) return fail(EPP_ERR_INVALID, "NULL LoRA arrays");
    if (n_members > 0 && (!member_ep || !member_model || !member_state)) return fail(EPP_ERR_INVALID, "NULL LoRA member arrays");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    const uint32_t E = (uint32_t)h->cfg.max_endpoints;
    std::vector<int32_t> mx(E, 0), cnt(E, 0);
    for (int32_t i = 0; i < n; i++) {
        if (ids[i] >= E) return fail(EPP_ERR_INVALID, "LoRA entry %d: slot id %u >= max_endpoints %u", i, ids[i], E);
        mx[ids[i]] = max_active_models[i];
        cnt[ids[i]] = n_models_loaded[i];
    }
    const int32_t n_models = std::max(1, h->n_models);
    struct Mem { uint32_t model, ep; uint8_t st; };
    std::vector<Mem> mem;
    mem.reserve((size_t)n_members);
    for (int64_t i = 0; i < n_members; i++) {
        if (member_ep[i] >= E) return fail(EPP_ERR_INVALID, "LoRA member %lld: slot id %u >= max_endpoints %u", (long long)i, member_ep[i], E);
        if (member_model[i] >= (uint32_t)n_models) return fail(EPP_ERR_INVALID, "LoRA member %lld: model id %u is not registered", (long long)i, member_model[i]);
        if (member_state[i] != 1 && member_state[i] != 2) return fail(EPP_ERR_INVALID, "LoRA member %lld: state %u (1 = active, 2 = waiting)", (long long)i, member_state[i]);
        mem.push_back({member_model[i], member_ep[i], member_state[i]});
    }
    // CSR by adapter, endpoints ascending; an adapter both active and waiting on an endpoint counts as active
    // (the `case active` branch comes first, lora_affinity.go:85-87)
    std::sort(mem.begin(), mem.end(), [](const Mem &a, const Mem &b) {
        return a.model != b.model ? a.model < b.model : (a.ep != b.ep ? a.ep < b.ep : a.st < b.st);
    });
    std::vector<uint32_t> ptr((size_t)n_models + 1, 0), eps;
    std::vector<uint8_t> sts;
    for (size_t i = 0; i < mem.size(); i++) {
        if (i && mem[i].model == mem[i - 1].model && mem[i].ep == mem[i - 1].ep) continue;
        eps.push_back(mem[i].ep);
        sts.push_back(mem[i].st);
        ptr[mem[i].model + 1]++;
    }
    for (int32_t a = 0; a < n_models; a++) ptr[a + 1] += ptr[a];
    cudaStream_t s = h->slot[0].stream;
    CUDA_TRY(h->lora_max.reserve(sizeof(int32_t) * E, &h->dev_bytes));
    CUDA_TRY(h->lora_cnt.reserve(sizeof(int32_t) * E, &h->dev_bytes));
    CUDA_TRY(h->lora_ptr.reserve(sizeof(uint32_t) * ptr.size(), &h->dev_bytes));
    CUDA_TRY(h->lora_ep.reserve(sizeof(uint32_t) * std::max<size_t>(1, eps.size()), &h->dev_bytes));
    CUDA_TRY(h->lora_state.reserve(std::max<size_t>(1, sts.size()), &h->dev_bytes));
    CUDA_TRY(cudaMemcpyAsync(h->lora_max.p, mx.data(), sizeof(int32_t) * E, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(h->lora_cnt.p, cnt.data(), sizeof(int32_t) * E, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(h->lora_ptr.p, ptr.data(), sizeof(uint32_t) * ptr.size(), cudaMemcpyHostToDevice, s));
    if (!eps.empty()) {
        CUDA_TRY(cudaMemcpyAsync(h->lora_ep.p, eps.data(), sizeof(uint32_t) * eps.size(), cudaMemcpyHostToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(h->lora_state.p, sts.data(), sts.size(), cudaMemcpyHostToDevice, s));
    }
    h->lora_models = n_models;
    h->lora_set = true;
    if (h->pool_ready) EPP_TRY(derive_pool(h));
    CUDA_TRY(cudaStreamSynchronize(s));
    return EPP_OK;
}

// ---- label filters ----------------------------------------------------------------------------------------------------
// Interns the keys and named values of every profile's requirements and compiles each requirement to one mask of the
// codes it admits (include/epp_engine.h "Label filters").  Fails on a cap; `out` is then unusable.
static int32_t compile_labels(const std::vector<LabelReq> (&reqs)[kMaxProfiles], LabelPlan &out) {
    out = LabelPlan{};
    for (int p = 0; p < kMaxProfiles; p++) {
        LabelFilterDev &d = out.dev[p];
        d.n = (int32_t)reqs[p].size();
        for (int i = 0; i < d.n; i++) {
            const LabelReq &q = reqs[p][i];
            size_t k = std::find(out.keys.begin(), out.keys.end(), q.key) - out.keys.begin();
            if (k == out.keys.size()) {
                if ((int)k == kMaxLabelKeys) return fail(EPP_ERR_INVALID, "label filters reference more than %d distinct keys", kMaxLabelKeys);
                out.keys.push_back(q.key);
                out.codes.emplace_back();
            }
            auto &codes = out.codes[k];
            uint64_t named = 0;
            bool empty_named = false;
            for (const std::string &v : q.values) {
                auto it = codes.find(v);
                if (it == codes.end()) {
                    if ((int)codes.size() == kMaxLabelValues)
                        return fail(EPP_ERR_INVALID, "label key \"%s\": more than %d distinct values named", q.key.c_str(), kMaxLabelValues);
                    it = codes.emplace(v, (uint8_t)(codes.size() + 1)).first;
                }
                named |= 1ull << it->second;
                empty_named |= v.empty();
            }
            const uint64_t absent = 1ull, all = ~0ull;
            uint64_t m = 0;
            switch (q.op) {
                case EPP_LABEL_IN: m = named; break;                                 // absent never matches
                case EPP_LABEL_NOT_IN: m = all & ~named; break;                      // absent always matches
                case EPP_LABEL_EXISTS: m = all & ~absent; break;
                case EPP_LABEL_DOES_NOT_EXIST: m = absent; break;
                case EPP_LABEL_BY_LABEL: m = named | (empty_named ? absent : 0); break;   // absent reads ""
                case EPP_LABEL_BY_LABEL_OR_ABSENT: m = named | absent; break;
            }
            d.key[i] = (uint8_t)k;
            d.mask[i] = m;
        }
    }
    return EPP_OK;
}

extern "C" int32_t epp_label_filters_set(epp_engine *h, int32_t profile, int32_t n, const epp_label_req *reqs) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    if (profile < 0 || profile >= h->n_alloc_profiles) return fail(EPP_ERR_INVALID, "profile %d is not configured", profile);
    if (n < 0 || n > EPP_LABEL_MAX_REQS) return fail(EPP_ERR_INVALID, "%d label requirements, out of range [0,%d]", n, EPP_LABEL_MAX_REQS);
    if (n > 0 && !reqs) return fail(EPP_ERR_INVALID, "NULL requirements");
    std::vector<LabelReq> mine;
    for (int32_t i = 0; i < n; i++) {
        const epp_label_req &r = reqs[i];
        if (!r.key || !r.key[0]) return fail(EPP_ERR_INVALID, "requirement %d: empty key", i);
        if (strpbrk(r.key, "=\n")) return fail(EPP_ERR_INVALID, "requirement %d: key holds '=' or a newline", i);
        if (r.op < EPP_LABEL_IN || r.op > EPP_LABEL_BY_LABEL_OR_ABSENT) return fail(EPP_ERR_INVALID, "requirement %d: unknown op %d", i, r.op);
        const bool takes = r.op != EPP_LABEL_EXISTS && r.op != EPP_LABEL_DOES_NOT_EXIST;
        const bool needs = r.op == EPP_LABEL_IN || r.op == EPP_LABEL_NOT_IN || r.op == EPP_LABEL_BY_LABEL;
        if (r.n_values < 0 || (!takes && r.n_values != 0) || (needs && r.n_values == 0))
            return fail(EPP_ERR_INVALID, "requirement %d: %d values do not fit op %d", i, r.n_values, r.op);
        if (r.n_values > 0 && !r.values) return fail(EPP_ERR_INVALID, "requirement %d: NULL values", i);
        LabelReq q{r.key, r.op, {}};
        for (int32_t j = 0; j < r.n_values; j++) {
            if (!r.values[j]) return fail(EPP_ERR_INVALID, "requirement %d: value %d is NULL", i, j);
            if (strchr(r.values[j], '\n')) return fail(EPP_ERR_INVALID, "requirement %d: value %d holds a newline", i, j);
            q.values.emplace_back(r.values[j]);
        }
        mine.push_back(std::move(q));
    }
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->pool_called) return fail(EPP_ERR_STATE, "label filters are fixed once the pool has been set");
    std::vector<LabelReq> all[kMaxProfiles];
    for (int p = 0; p < kMaxProfiles; p++) all[p] = p == profile ? mine : h->label_reqs[p];
    LabelPlan plan;
    EPP_TRY(compile_labels(all, plan));
    EPP_TRY(set_device(h));
    const size_t bytes = plan.keys.size() * (size_t)h->cfg.max_endpoints;
    if (bytes) {
        CUDA_TRY(h->lcode.reserve(bytes, &h->dev_bytes));
        cudaStream_t s = h->slot[0].stream;                      // the stream every later upload and derive runs on
        CUDA_TRY(cudaMemsetAsync(h->lcode.p, 0, bytes, s));      // no labels yet: every key absent
        CUDA_TRY(cudaStreamSynchronize(s));
    }
    h->label_reqs[profile] = std::move(mine);
    h->labels = std::move(plan);
    return EPP_OK;
}

// ---- context length ---------------------------------------------------------------------------------------------------
// unicode.IsSpace
static bool go_is_space(uint32_t r) {
    if (r < 0x80) return r == ' ' || (r >= '\t' && r <= '\r');
    return r == 0x85 || r == 0xA0 || r == 0x1680 || (r >= 0x2000 && r <= 0x200A) || r == 0x2028 || r == 0x2029 ||
           r == 0x202F || r == 0x205F || r == 0x3000;
}
// The rune encoded by exactly the bytes [p, end), or -1 when they are not one valid UTF-8 sequence.
static int64_t utf8_rune(const unsigned char *p, const unsigned char *end) {
    const size_t n = (size_t)(end - p);
    if (n == 1) return p[0] < 0x80 ? p[0] : -1;
    const size_t want = (p[0] & 0xE0) == 0xC0 ? 2 : (p[0] & 0xF0) == 0xE0 ? 3 : (p[0] & 0xF8) == 0xF0 ? 4 : 0;
    if (want != n) return -1;
    uint32_t r = p[0] & (0x7F >> n);
    for (size_t i = 1; i < n; i++) {
        if ((p[i] & 0xC0) != 0x80) return -1;
        r = (r << 6) | (p[i] & 0x3F);
    }
    static const uint32_t min_of[5] = {0, 0, 0x80, 0x800, 0x10000};
    if (r < min_of[n] || r > 0x10FFFF || (r >= 0xD800 && r <= 0xDFFF)) return -1;
    return r;
}
// strings.TrimSpace: white-space runes off both ends (an invalid byte stops the trim, as utf8.RuneError is no space).
static std::string go_trim_space(const std::string &v) {
    const unsigned char *b = reinterpret_cast<const unsigned char *>(v.data()), *e = b + v.size();
    while (b < e) {
        const ptrdiff_t want = *b < 0x80 ? 1 : (*b & 0xE0) == 0xC0 ? 2 : (*b & 0xF0) == 0xE0 ? 3 : 4;
        const unsigned char *q = e - b < want ? e : b + want;
        const int64_t r = utf8_rune(b, q);
        if (r < 0 || !go_is_space((uint32_t)r)) break;
        b = q;
    }
    while (e > b) {
        const unsigned char *q = e - 1;
        while (q > b && e - q < 4 && (*q & 0xC0) == 0x80) q--;
        const int64_t r = utf8_rune(q, e);
        if (r < 0 || !go_is_space((uint32_t)r)) break;
        e = q;
    }
    return std::string(reinterpret_cast<const char *>(b), (size_t)(e - b));
}
// strconv.Atoi on a 64-bit platform: optional sign, then at least one decimal digit and nothing else, within int64.
static bool go_atoi(const std::string &v, long long *out) {
    size_t i = 0;
    bool neg = false;
    if (i < v.size() && (v[i] == '+' || v[i] == '-')) neg = v[i++] == '-';
    if (i == v.size()) return false;
    const unsigned long long lim = neg ? (1ull << 63) : (1ull << 63) - 1;
    unsigned long long x = 0;
    for (; i < v.size(); i++) {
        if (v[i] < '0' || v[i] > '9') return false;
        const unsigned d = (unsigned)(v[i] - '0');
        if (x > (lim - d) / 10) return false;
        x = x * 10 + d;
    }
    *out = neg ? (long long)(0ull - x) : (long long)x;
    return true;
}
// parseContextRange: "min-max" split on "-" into exactly 2 parts, each TrimSpace + Atoi, min <= max.
static bool parse_context_range(const std::string &v, long long *lo, long long *hi) {
    const size_t dash = v.find('-');
    if (v.empty() || dash == std::string::npos || v.find('-', dash + 1) != std::string::npos) return false;
    if (!go_atoi(go_trim_space(v.substr(0, dash)), lo) || !go_atoi(go_trim_space(v.substr(dash + 1)), hi)) return false;
    return *lo <= *hi;
}

extern "C" int32_t epp_context_length_set(epp_engine *h, int32_t profile, const char *label, int32_t enable_filtering) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    if (profile < 0 || profile >= h->n_alloc_profiles) return fail(EPP_ERR_INVALID, "profile %d is not configured", profile);
    if (label && !label[0]) return fail(EPP_ERR_INVALID, "the context-length label must not be empty");
    if (label && strpbrk(label, "=\n")) return fail(EPP_ERR_INVALID, "the context-length label holds '=' or a newline");
    if (enable_filtering != 0 && enable_filtering != 1) return fail(EPP_ERR_INVALID, "enable_filtering %d must be 0 or 1", enable_filtering);
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->pool_called) return fail(EPP_ERR_STATE, "context-length profiles are fixed once the pool has been set");
    if (sharded(h) || h->p2p_buf) return fail(EPP_ERR_INVALID, "endpoint-sharded mode does not support the context-length scorer");
    if (!((h->cl_mask >> profile) & 1)) return fail(EPP_ERR_INVALID, "profile %d does not list the context-length scorer", profile);
    h->cl_label[profile] = label ? label : EPP_CONTEXT_LENGTH_LABEL;
    if (enable_filtering) h->cl_filter |= 1 << profile;
    else h->cl_filter &= ~(1 << profile);
    return EPP_OK;
}

extern "C" int32_t epp_pool_set_labels(epp_engine *h, int32_t n, const uint32_t *ids, const uint64_t *offsets,
                                       const uint8_t *text) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    if (n < 0 || (n > 0 && (!ids || !offsets || !text))) return fail(EPP_ERR_INVALID, "NULL label arrays");
    std::lock_guard<std::mutex> lk(h->mu);
    const uint32_t E = (uint32_t)h->cfg.max_endpoints;
    const size_t K = h->labels.keys.size();
    std::vector<uint8_t> seen(E, 0), lc(K * (size_t)E, 0);
    std::unordered_map<std::string, size_t> key_row;
    for (size_t k = 0; k < K; k++) key_row.emplace(h->labels.keys[k], k);
    std::vector<std::string> slot_keys;
    std::vector<longlong2> rng[kMaxProfiles];          // context-length ranges of the profiles listing the plugin
    for (int pi = 0; pi < kMaxProfiles; pi++)
        if ((h->cl_mask >> pi) & 1) rng[pi].assign(E, longlong2{kRangeAbsent, 0});
    for (int32_t i = 0; i < n; i++) {
        const uint32_t id = ids[i];
        if (id >= E) return fail(EPP_ERR_INVALID, "label entry %d: slot id %u >= max_endpoints %u", i, id, E);
        if (seen[id]) return fail(EPP_ERR_INVALID, "label entry %d: duplicate slot id %u", i, id);
        seen[id] = 1;
        if (offsets[i + 1] < offsets[i]) return fail(EPP_ERR_INVALID, "label entry %d: offsets decrease", i);
        slot_keys.clear();
        const char *p = reinterpret_cast<const char *>(text) + offsets[i], *end = reinterpret_cast<const char *>(text) + offsets[i + 1];
        while (p < end) {
            const char *nl = static_cast<const char *>(memchr(p, '\n', (size_t)(end - p)));
            if (!nl) return fail(EPP_ERR_INVALID, "label entry %d: a label is not terminated by a newline", i);
            const char *eq = static_cast<const char *>(memchr(p, '=', (size_t)(nl - p)));
            if (!eq) return fail(EPP_ERR_INVALID, "label entry %d: a label has no '='", i);
            if (eq == p) return fail(EPP_ERR_INVALID, "label entry %d: a label has an empty key", i);
            std::string key(p, eq);
            if (std::find(slot_keys.begin(), slot_keys.end(), key) != slot_keys.end())
                return fail(EPP_ERR_INVALID, "label entry %d: key \"%s\" repeated", i, key.c_str());
            slot_keys.push_back(key);
            for (int pi = 0; pi < kMaxProfiles; pi++) {
                if (!((h->cl_mask >> pi) & 1) || key != h->cl_label[pi]) continue;
                long long lo, hi;
                rng[pi][id] = parse_context_range(std::string(eq + 1, nl), &lo, &hi) ? longlong2{lo, hi} : longlong2{kRangeInvalid, 0};
            }
            auto kr = key_row.find(key);
            if (kr != key_row.end()) {                     // keys no requirement references are dropped here
                const auto &codes = h->labels.codes[kr->second];
                auto c = codes.find(std::string(eq + 1, nl));
                lc[kr->second * (size_t)E + id] = c == codes.end() ? 63 : c->second;
            }
            p = nl + 1;
        }
    }
    h->pool_called = true;
    if (!K && !h->cl_mask) return EPP_OK;                  // no label filter or range: nothing on the device reads labels
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    cudaStream_t s = h->slot[0].stream;
    for (int pi = 0; pi < kMaxProfiles; pi++)
        if ((h->cl_mask >> pi) & 1)
            CUDA_TRY(cudaMemcpyAsync(h->cl_rng[pi].p, rng[pi].data(), sizeof(longlong2) * E, cudaMemcpyHostToDevice, s));
    if (K) {
        CUDA_TRY(cudaMemcpyAsync(h->lcode.p, lc.data(), lc.size(), cudaMemcpyHostToDevice, s));
        if (h->pool_ready) EPP_TRY(derive_pool(h));
    }
    CUDA_TRY(cudaStreamSynchronize(s));
    return EPP_OK;
}

// ------------------------------------------------------------------------------------------------
// prefix index
// ------------------------------------------------------------------------------------------------
// Clears the presence bitmap and sets the bits of every key the read table holds.  16 bits per table slot, which is
// >= 26 per distinct key at the load factors the build and the patches allow, up to 2^26 bits (8 MiB, L2-resident) while
// the table fits its L2 budget.  A larger table is read from DRAM anyway: its bitmap may grow to 2^30 bits (128 MiB), as
// 2^26 bits over 1.3e8 keys would be mostly set and prove few misses (the lookup's latency hides behind its window).
static int32_t rebuild_presence(epp_engine *h) {
    const int cap = h->idx_capacity * sizeof(IndexSlot) > h->l2_table_bytes ? 30 : 26;
    int l = 6;
    while (l < cap && (1ull << l) < 16 * h->idx_capacity) l++;
    if (h->presence_log2_env) l = h->presence_log2_env;
    h->presence_log2 = l;
    CUDA_TRY(h->presence.reserve(((size_t)1 << l) / 8, &h->dev_bytes));
    int launches = 0;
    CUDA_TRY(launch_presence_build(h->idx_capacity ? h->slots.as<IndexSlot>() : nullptr, h->idx_capacity,
                                   h->presence.as<uint32_t>(), l, h->slot[0].stream, &launches));
    return EPP_OK;
}

// Bulk build of the read table from n (hash, endpoint) pairs already in h->pair_hash / h->pair_ep.
static int32_t build_index_from_device_pairs(epp_engine *h, uint64_t n, uint64_t n_distinct_hint, bool from_store = false) {
    cudaStream_t s = h->slot[0].stream;
    if (n >= 0xFFFFFFF0ull) return fail(EPP_ERR_CAPACITY, "index snapshot of %llu pairs exceeds the u32 posting space", (unsigned long long)n);
    // posting space: the lists of this build + room for the copy-on-write lists of later patches
    uint64_t post_entries = std::max<uint64_t>(n, 1);
    if (from_store) post_entries = std::min<uint64_t>(0xFFFFFFF0ull, n + std::max<uint64_t>(n / 2, 1ull << 20));
    CUDA_TRY(h->postings.reserve(sizeof(uint32_t) * post_entries, &h->dev_bytes));
    uint64_t distinct = std::max<uint64_t>(1, n_distinct_hint);
    uint32_t cursor[4] = {0, 0, 0, 0};
    uint64_t cap = 16;
    for (int pass = 0; pass < 2; pass++) {
        // load factor <= 0.5 over the distinct hashes (<= 0.25 while the table stays L2-sized: shorter probe chains, a faster
        // step on H100, profiles/h100_index_load_ab.jsonl); the first pass only knows an upper bound (the pair count)
        const uint64_t load = h->index_load ? (uint64_t)h->index_load : (4 * distinct * sizeof(IndexSlot) <= h->l2_table_bytes ? 4 : 2);
        uint64_t want = std::max<uint64_t>(16, load * distinct);
        cap = 16;
        while (cap < want) cap <<= 1;
        CUDA_TRY(h->slots.reserve(sizeof(IndexSlot) * cap, &h->dev_bytes));
        CUDA_TRY(h->idx_scratch.reserve(sizeof(uint32_t) * cap, &h->dev_bytes));
        CUDA_TRY(h->intern_keys.reserve(sizeof(uint64_t) * cap, &h->dev_bytes));
        CUDA_TRY(h->intern_vals.reserve(sizeof(uint32_t) * cap, &h->dev_bytes));
        int launches = 0;
        CUDA_TRY(launch_index_build(h->pair_hash.as<uint64_t>(), h->pair_ep.as<uint32_t>(), n, h->slots.as<IndexSlot>(), cap,
                                    h->postings.as<uint32_t>(), h->idx_scratch.as<uint32_t>(), h->idx_cursor.as<uint32_t>(),
                                    h->idx_special.as<IndexSlot>(), h->intern_keys.as<uint64_t>(), h->intern_vals.as<uint32_t>(), s, &launches));
        CUDA_TRY(cudaMemcpyAsync(&h->idx_special_host, h->idx_special.p, sizeof(IndexSlot), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaMemcpyAsync(cursor, h->idx_cursor.p, sizeof cursor, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        uint64_t true_distinct = std::max<uint64_t>(1, cursor[2]);
        const uint64_t load2 = h->index_load ? (uint64_t)h->index_load : (4 * true_distinct * sizeof(IndexSlot) <= h->l2_table_bytes ? 4 : 2);
        uint64_t tight = 16;
        while (tight < load2 * true_distinct) tight <<= 1;
        if (tight >= cap) break;            // already as small as the load factor allows
        distinct = true_distinct;           // rebuild once into a table a quarter (or less) of the size
    }
    h->idx_capacity = cap;
    h->idx_pairs = n;
    h->stats.index_pairs = n;
    h->stats.index_hashes = cursor[2];
    h->stats.index_slots = cap;
    // patch bookkeeping: pending-list heads idle, posting cursor, used slots
    CUDA_TRY(cudaMemsetAsync(h->idx_scratch.p, 0xFF, sizeof(uint32_t) * cap, s));
    h->post_cap = h->postings.cap / sizeof(uint32_t);
    h->post_used = cursor[0];
    h->rt_slots_used = cursor[2];
    h->rt_intern_used = cursor[3];
    h->rt_from_store = from_store;
    h->patches_since_build = 0;
    return rebuild_presence(h);
}

static int32_t build_device_index(epp_engine *h, const uint64_t *hashes, const uint32_t *eps, uint64_t n,
                                  uint64_t n_distinct_hint) {
    cudaStream_t s = h->slot[0].stream;
    CUDA_TRY(h->pair_hash.reserve(sizeof(uint64_t) * std::max<uint64_t>(n, 1), &h->dev_bytes));
    CUDA_TRY(h->pair_ep.reserve(sizeof(uint32_t) * std::max<uint64_t>(n, 1), &h->dev_bytes));
    if (n) {
        CUDA_TRY(cudaMemcpyAsync(h->pair_hash.p, hashes, sizeof(uint64_t) * n, cudaMemcpyHostToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(h->pair_ep.p, eps, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, s));
    }
    return build_index_from_device_pairs(h, n, n_distinct_hint);
}

// Applies the queued epp_index_add calls to the device store as one batch (sub-batches bound the ordering scratch).
static int32_t flush_add_queue(epp_engine *h) {
    const size_t M = h->q_ep.size();
    if (M == 0) return EPP_OK;
    cudaStream_t s = h->slot[0].stream;
    CUDA_TRY(h->q_ep_dev.reserve(sizeof(uint32_t) * M, &h->dev_bytes));
    CUDA_TRY(h->q_n_dev.reserve(sizeof(uint32_t) * M, &h->dev_bytes));
    CUDA_TRY(h->q_nb_dev.reserve(sizeof(int32_t) * M, &h->dev_bytes));
    CUDA_TRY(h->q_src_dev.reserve(sizeof(uint64_t) * M, &h->dev_bytes));
    CUDA_TRY(h->q_hashes_dev.reserve(sizeof(uint64_t) * std::max<size_t>(1, h->q_hashes.size()), &h->dev_bytes));
    CUDA_TRY(cudaMemcpyAsync(h->q_ep_dev.p, h->q_ep.data(), sizeof(uint32_t) * M, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(h->q_n_dev.p, h->q_n.data(), sizeof(uint32_t) * M, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(h->q_nb_dev.p, h->q_nb.data(), sizeof(int32_t) * M, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(h->q_src_dev.p, h->q_src.data(), sizeof(uint64_t) * M, cudaMemcpyHostToDevice, s));
    if (!h->q_hashes.empty())
        CUDA_TRY(cudaMemcpyAsync(h->q_hashes_dev.p, h->q_hashes.data(), sizeof(uint64_t) * h->q_hashes.size(), cudaMemcpyHostToDevice, s));
    const size_t kSub = 1u << 18;
    for (size_t c0 = 0; c0 < M; c0 += kSub) {
        StoreCalls c;
        c.M = (uint32_t)std::min(kSub, M - c0);
        c.ep = h->q_ep_dev.as<uint32_t>() + c0;
        c.n = h->q_n_dev.as<uint32_t>() + c0;
        c.nb = h->q_nb_dev.as<int32_t>() + c0;
        c.src = h->q_src_dev.as<uint64_t>() + c0;
        c.hashes = h->q_hashes_dev.as<uint64_t>();
        CUDA_TRY(h->store->apply(c, s));
    }
    h->q_ep.clear();
    h->q_n.clear();
    h->q_nb.clear();
    h->q_src.clear();
    h->q_hashes.clear();
    return EPP_OK;
}

static double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

static int32_t commit_locked(epp_engine *h) {
    if (h->snapshot_mode) return EPP_OK;
    if (!h->q_ep.empty() || h->store->dirty()) EPP_TRY(join_streams(h));     // the table is about to change under stream 1
    EPP_TRY(flush_add_queue(h));
    if (!h->store->dirty()) return EPP_OK;
    auto t0 = std::chrono::steady_clock::now();
    cudaStream_t s = h->slot[0].stream;
    bool patched = false;
    if (h->patch_enabled && h->rt_from_store && h->idx_capacity && h->patches_since_build < 256) {
        ReadTableRef rt;
        rt.slots = h->slots.as<IndexSlot>();
        rt.capacity = h->idx_capacity;
        rt.slots_used = h->rt_slots_used;
        rt.postings = h->postings.as<uint32_t>();
        rt.post_cap = h->post_cap;
        rt.post_used = h->post_used;
        rt.head = h->idx_scratch.as<uint32_t>();
        rt.intern_keys = h->intern_keys.as<uint64_t>();
        rt.intern_vals = h->intern_vals.as<uint32_t>();
        rt.intern_used = h->rt_intern_used;
        rt.presence = h->presence.as<uint32_t>();
        rt.presence_shift = 64 - h->presence_log2;
        uint64_t np = 0, nu = 0, npost = 0, ni = 0;
        CUDA_TRY(h->store->patch_read_table(rt, h->idx_pairs, s, &patched, &np, &nu, &npost, &ni));
        if (patched) {
            h->idx_pairs = np;
            h->rt_slots_used = nu;
            h->rt_intern_used = ni;
            h->post_used = npost;
            h->stats.index_pairs = np;
            h->stats.index_hashes = nu;
            h->patches_since_build++;
            h->stats.last_index_patched = 1;
        }
    }
    if (!patched) {
        uint64_t n = 0;
        CUDA_TRY(h->store->export_pairs(h->pair_hash, h->pair_ep, &n, &h->dev_bytes, s));
        EPP_TRY(build_index_from_device_pairs(h, n, n, true));
        h->stats.last_index_patched = 0;
    }
    CUDA_TRY(h->store->touch_reset(s));
    h->store->mark_clean();
    h->stats.last_index_build_ms = ms_since(t0);
    return EPP_OK;
}

static IndexView index_view(epp_engine *h) {
    IndexView v;
    v.slots = h->idx_capacity ? h->slots.as<IndexSlot>() : nullptr;
    v.postings = h->postings.as<uint32_t>();
    v.mask = h->idx_capacity ? h->idx_capacity - 1 : 0;
    v.special = h->idx_special_host;
    if (!h->idx_capacity) v.special.cnt = 0;
    v.ep_begin = h->shard_begin;
    v.ep_end = h->shard_end;
    return v;
}

extern "C" int32_t epp_index_add(epp_engine *h, uint32_t ep, int32_t n, const uint64_t *hashes, int32_t num_gpu_blocks) {
    if (!h || n < 0 || (n > 0 && !hashes)) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->snapshot_mode) return fail(EPP_ERR_STATE, "index holds a bulk snapshot; incremental adds need an empty or incrementally built index");
    if (ep >= (uint32_t)h->cfg.max_endpoints) return fail(EPP_ERR_INVALID, "endpoint slot %u out of range [0,%d)", ep, h->cfg.max_endpoints);
    h->q_ep.push_back(ep);
    h->q_n.push_back((uint32_t)n);
    h->q_nb.push_back(num_gpu_blocks);
    h->q_src.push_back((uint64_t)h->q_hashes.size());
    h->q_hashes.insert(h->q_hashes.end(), hashes, hashes + n);
    if (h->q_hashes.size() >= (1u << 26) || h->q_ep.size() >= (1u << 22)) {      // bound the host queue
        EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
        EPP_TRY(flush_add_queue(h));
    }
    return EPP_OK;
}

extern "C" int32_t epp_index_remove_endpoint(epp_engine *h, uint32_t ep) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->snapshot_mode) return fail(EPP_ERR_STATE, "index holds a bulk snapshot; reload it without the endpoint instead");
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    EPP_TRY(flush_add_queue(h));                    // calls apply in the order they were made
    CUDA_TRY(h->store->remove_endpoint(ep, h->slot[0].stream));
    return EPP_OK;
}

// CleanUpInactivePods (approximateprefix/plugin.go:99-122).
extern "C" int32_t epp_index_retain_endpoints(epp_engine *h, int32_t n, const uint32_t *active_ids) {
    if (!h || n < 0 || (n > 0 && !active_ids)) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->snapshot_mode) return fail(EPP_ERR_STATE, "index holds a bulk snapshot; reload it without the endpoints instead");
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    EPP_TRY(flush_add_queue(h));
    const size_t E = (size_t)h->cfg.max_endpoints;
    std::vector<uint8_t> active(E, 0);
    for (int32_t i = 0; i < n; i++) {
        if (active_ids[i] >= E) return fail(EPP_ERR_INVALID, "endpoint slot %u out of range [0,%zu)", active_ids[i], E);
        active[active_ids[i]] = 1;
    }
    cudaStream_t s = h->slot[0].stream;
    CUDA_TRY(h->q_ep_dev.reserve(E, &h->dev_bytes));
    CUDA_TRY(cudaMemcpyAsync(h->q_ep_dev.p, active.data(), E, cudaMemcpyHostToDevice, s));
    CUDA_TRY(h->store->retain_endpoints(h->q_ep_dev.as<uint8_t>(), s));
    return EPP_OK;
}

extern "C" int32_t epp_index_load_snapshot(epp_engine *h, uint64_t n_pairs, const uint64_t *hashes, const uint32_t *eps) {
    if (!h || (n_pairs && (!hashes || !eps))) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    h->q_ep.clear(); h->q_n.clear(); h->q_nb.clear(); h->q_src.clear(); h->q_hashes.clear();
    CUDA_TRY(h->store->clear(h->slot[0].stream));
    h->store->mark_clean();
    EPP_TRY(build_device_index(h, hashes, eps, n_pairs, n_pairs));
    h->snapshot_mode = n_pairs > 0;
    return EPP_OK;
}

extern "C" int32_t epp_index_commit(epp_engine *h) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    return commit_locked(h);
}

extern "C" int32_t epp_index_get(epp_engine *h, uint64_t hash, uint32_t *out_eps, int32_t cap, int32_t *out_n) {
    if (!h || !out_n || cap < 0 || (cap > 0 && !out_eps)) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    EPP_TRY(commit_locked(h));
    cudaStream_t s = h->slot[0].stream;
    int32_t dcap = std::min(cap, 4096);
    uint32_t *d_eps = h->get_out.as<uint32_t>();
    int32_t *d_n = reinterpret_cast<int32_t *>(d_eps + 4096);
    CUDA_TRY(launch_index_get(index_view(h), hash, d_eps, dcap, d_n, s));
    CUDA_TRY(cudaMemcpyAsync(out_n, d_n, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    int32_t ncopy = std::min(*out_n, dcap);
    if (ncopy > 0) CUDA_TRY(cudaMemcpy(out_eps, d_eps, sizeof(uint32_t) * ncopy, cudaMemcpyDeviceToHost));
    return EPP_OK;
}

// ------------------------------------------------------------------------------------------------
// batches
// ------------------------------------------------------------------------------------------------
struct BatchView {
    int64_t R = 0;
    bool device = false;
    bool async = false;            // EPP_BATCH_ASYNC (device batches, epp_schedule only)
    const uint8_t *data = nullptr;
    const uint64_t *offsets = nullptr;
    const uint64_t *lengths = nullptr;
    uint64_t uniform_len = 0;
    const uint32_t *model_ids = nullptr;
    const uint8_t *multimodal = nullptr;
    uint64_t total_bytes = 0;      // host batches only
    uint64_t offsets_or_bits = 0;
};

static int32_t check_batch(epp_engine *h, const epp_batch *b, BatchView &v) {
    if (!b) return fail(EPP_ERR_INVALID, "batch is NULL");
    if (b->n_requests < 0) return fail(EPP_ERR_INVALID, "n_requests < 0");
    if (h->n_models == 0) return fail(EPP_ERR_STATE, "no model registered (epp_model_register)");
    v.R = b->n_requests;
    v.device = (b->flags & EPP_BATCH_DEVICE_PTRS) != 0;
    v.async = (b->flags & EPP_BATCH_ASYNC) != 0;
    if (v.async && !v.device) return fail(EPP_ERR_INVALID, "EPP_BATCH_ASYNC needs EPP_BATCH_DEVICE_PTRS");
    v.data = reinterpret_cast<const uint8_t *>(b->data);
    v.offsets = b->offsets;
    v.lengths = b->lengths;
    if (v.lengths && !v.offsets) return fail(EPP_ERR_INVALID, "lengths needs offsets");
    v.uniform_len = b->uniform_len;
    v.model_ids = b->model_ids;
    v.multimodal = b->multimodal;
    if (v.R == 0) return EPP_OK;
    if (!v.offsets && v.uniform_len > 0 && !v.data) return fail(EPP_ERR_INVALID, "data is NULL");
    if (!v.device) {
        if (v.offsets) {
            uint64_t bits = 0;
            for (int64_t r = 0; r < v.R; r++) {
                if (v.offsets[r + 1] < v.offsets[r]) return fail(EPP_ERR_INVALID, "offsets not monotonic at request %lld", (long long)r);
                if (v.lengths && v.offsets[r] + v.lengths[r] > v.offsets[r + 1]) {
                    // EPP_BATCH_LENGTHS_EXCEED_ROWS: the row must still hold every byte hashPrompt reads
                    const uint64_t cap = (uint64_t)h->cfg.max_prefix_blocks * (uint64_t)h->cfg.block_size_tokens * 4;
                    const uint64_t need = std::min<uint64_t>(v.lengths[r], cap);
                    if (!(b->flags & EPP_BATCH_LENGTHS_EXCEED_ROWS) || v.offsets[r] + need > v.offsets[r + 1])
                        return fail(EPP_ERR_INVALID, "request %lld: offsets[r] + lengths[r] exceeds offsets[r+1]", (long long)r);
                }
                bits |= v.offsets[r];
            }
            v.offsets_or_bits = bits;
            v.total_bytes = v.offsets[v.R] - v.offsets[0];
            if (v.total_bytes && !v.data) return fail(EPP_ERR_INVALID, "data is NULL");
        } else {
            v.total_bytes = (uint64_t)v.R * v.uniform_len;
        }
        if (v.model_ids)
            for (int64_t r = 0; r < v.R; r++)
                if ((int)v.model_ids[r] >= h->n_models) return fail(EPP_ERR_INVALID, "request %lld: unknown model id %u", (long long)r, v.model_ids[r]);
    }
    return EPP_OK;
}

static int32_t reserve_batch(epp_engine *h, int64_t R) {
    size_t B = (size_t)h->cfg.max_prefix_blocks;
    size_t n = (size_t)std::max<int64_t>(R, 1);
    CUDA_TRY(h->hashes.reserve(sizeof(uint64_t) * n * B, &h->dev_bytes));
    CUDA_TRY(h->nblocks.reserve(sizeof(int32_t) * n, &h->dev_bytes));
    CUDA_TRY(h->bound.reserve(sizeof(int32_t) * n, &h->dev_bytes));
    CUDA_TRY(h->eff_len.reserve(sizeof(int64_t) * n, &h->dev_bytes));
    CUDA_TRY(h->in_len.reserve(sizeof(int64_t) * n, &h->dev_bytes));
    CUDA_TRY(h->decisions.reserve(sizeof(epp_decision) * n, &h->dev_bytes));
    CUDA_TRY(h->details.reserve(sizeof(epp_decision_detail) * n, &h->dev_bytes));
    CUDA_TRY(h->offsets.reserve(sizeof(uint64_t) * (n + 1), &h->dev_bytes));
    CUDA_TRY(h->lengths.reserve(sizeof(uint64_t) * n, &h->dev_bytes));
    CUDA_TRY(h->model_ids.reserve(sizeof(uint32_t) * n, &h->dev_bytes));
    for (int i = 0; i < 2; i++) CUDA_TRY(h->slot[i].overflow_list.reserve(sizeof(int32_t) * n, &h->dev_bytes));
    if (h->nohit_mask) CUDA_TRY(h->nh_cold.reserve(n, &h->dev_bytes));
    return EPP_OK;
}

// What one launch sequence works on: requests [r0, r1) whose bytes are resident at `data_base + offsets[r]`.
struct Work {
    int64_t r0, r1;
    const uint8_t *data_base;
    const uint64_t *offsets_dev;   // indexed by absolute request id, or nullptr
    const uint64_t *lengths_dev;   // absolute, or nullptr
    uint64_t uniform_len;
    const uint32_t *model_ids_dev; // absolute, or nullptr
    uint64_t offsets_or_bits;      // OR of all offsets (alignment of the batch layout)
    uint64_t *hashes_out;          // row r0 of the destination
    int32_t *nblocks_out;
    const uint8_t *multimodal_dev = nullptr;   // absolute, or nullptr
};

static HashParams hash_params(epp_engine *h, const Work &w, Slot &sl) {
    HashParams p;
    int64_t n = w.r1 - w.r0;
    p.data = w.data_base;
    p.offsets = w.offsets_dev ? w.offsets_dev + w.r0 : nullptr;
    p.lengths = w.lengths_dev ? w.lengths_dev + w.r0 : nullptr;
    p.uniform_len = w.uniform_len;
    p.model_ids = w.model_ids_dev ? w.model_ids_dev + w.r0 : nullptr;
    p.seeds = h->seeds.as<uint64_t>();
    p.R = n;
    p.block_bytes = h->cfg.block_size_tokens * 4;
    p.max_blocks = h->cfg.max_prefix_blocks;
    p.hashes = w.hashes_out;
    p.nblocks = w.nblocks_out;
    p.eff_len = h->eff_len.as<int64_t>() + w.r0;
    p.in_len = h->in_len.as<int64_t>() + w.r0;
    p.offsets_or_bits = w.offsets_or_bits;
    p.sm_count = h->sm_count;
    p.presence = nullptr;
    p.presence_shift = 0;
    p.bound = nullptr;
    p.stored = nullptr;
    p.skip = 0;
    p.read = nullptr;
    p.req_next = sl.hash_next.as<uint32_t>();
    return p;
}

// General-evaluation view; the top-k rows are attached by the caller (they depend on where the batch's rows live).
static GenView gen_view(epp_engine *h) {
    GenView g;
    memset(&g, 0, sizeof g);
    g.on = h->general ? 1 : 0;
    g.pool = pool_arrays(h);
    return g;
}
// Rows [r0, ...) of the top-k lists of the call in progress, in `base` arrays of row stride k.
static void attach_topk(epp_engine *h, GenView &g, uint32_t *const picks[kMaxProfiles], double *scores, int64_t r0) {
    const int32_t k = h->cfg.pick_k;
    g.topk = k;
    for (int i = 0; i < kMaxProfiles; i++) g.topk_picks[i] = picks[i] ? picks[i] + (size_t)r0 * (size_t)k : nullptr;
    g.topk_scores = scores ? scores + (size_t)r0 * (size_t)k : nullptr;
}

// The top-k lists of a scheduling call: the caller's arrays (dst), and the device rows the pick kernels write (picks /
// scores) -- the caller's own arrays for a device batch, engine staging for a host batch.
struct TopkRows {
    bool on = false;
    uint32_t *dst[kMaxProfiles] = {};
    double *dst_scores = nullptr;
    uint32_t *picks[kMaxProfiles] = {};
    double *scores = nullptr;
};

static int32_t topk_rows(epp_engine *h, const epp_topk_out *out, bool device, int64_t R, TopkRows &t) {
    if (!out) return EPP_OK;
    const size_t n = (size_t)R * (size_t)h->cfg.pick_k;
    t.on = true;
    t.dst[0] = out->primary; t.dst[1] = out->prefill; t.dst[2] = out->encode;
    t.dst_scores = out->primary_scores;
    for (int i = 0; i < kMaxProfiles; i++) {
        t.picks[i] = t.dst[i];
        if (!device && t.dst[i]) {
            CUDA_TRY(h->topk_picks[i].reserve(sizeof(uint32_t) * n, &h->dev_bytes));
            t.picks[i] = h->topk_picks[i].as<uint32_t>();
        }
    }
    t.scores = t.dst_scores;
    if (!device && t.scores) {
        CUDA_TRY(h->topk_scores.reserve(sizeof(double) * n, &h->dev_bytes));
        t.scores = h->topk_scores.as<double>();
    }
    return EPP_OK;
}

// Copies rows [r0, r0 + n) of a host batch's lists from the staging to the caller's arrays on s.
static int32_t topk_copy_back(epp_engine *h, const TopkRows &t, int64_t r0, int64_t n, cudaStream_t s) {
    const size_t K = (size_t)h->cfg.pick_k, o = (size_t)r0 * K, m = (size_t)n * K;
    for (int i = 0; i < kMaxProfiles; i++)
        if (t.dst[i]) CUDA_TRY(cudaMemcpyAsync(t.dst[i] + o, t.picks[i] + o, sizeof(uint32_t) * m, cudaMemcpyDeviceToHost, s));
    if (t.scores) CUDA_TRY(cudaMemcpyAsync(t.dst_scores + o, t.scores + o, sizeof(double) * m, cudaMemcpyDeviceToHost, s));
    return EPP_OK;
}

// The decision fields that every pick launch (PickParams, DensePickParams) fills alike, for a launch whose first request
// is r0.  Each caller sets the rest, and may override block_size_tokens.
template <class P> static void fill_decision_fields(epp_engine *h, P &p, int64_t r0) {
    p.E = h->cfg.max_endpoints;
    p.block_size_tokens = h->cfg.block_size_tokens;
    p.n_profiles = h->n_profiles;
    p.always_disagg = h->cfg.always_disagg;
    p.non_cached_tokens = h->cfg.non_cached_tokens;
    for (int i = 0; i < h->n_alloc_profiles; i++) p.prof[i] = profile_dev(h, i);
    p.lora = lora_dev(h);
    p.tie_base = h->stats.n_decisions + (uint64_t)r0;
    p.gen = gen_view(h);
    p.nohit = nohit_view(h, r0);
}

static PickParams pick_params(epp_engine *h, const Work &w, epp_decision *out, epp_decision_detail *detail,
                              int32_t *out_match) {
    PickParams p;
    fill_decision_fields(h, p, w.r0);
    p.R = w.r1 - w.r0;
    p.max_blocks = h->cfg.max_prefix_blocks;
    p.encode_on = h->cfg.encode_enabled ? 1 : 0;
    p.multimodal = w.multimodal_dev ? w.multimodal_dev + w.r0 : nullptr;
    p.tie_seed = sharded(h) ? 0 : h->cfg.tie_seed;      // sharded mode: the records hold the lowest slot
    p.hashes = w.hashes_out;
    p.nblocks = w.nblocks_out;
    p.bound = nullptr;
    p.in_len = h->in_len.as<int64_t>() + w.r0;
    p.model_ids = w.model_ids_dev ? w.model_ids_dev + w.r0 : nullptr;
    p.index = index_view(h);
    p.out = out;
    p.detail = detail;
    p.out_match = out_match;
    p.work_counters = nullptr;
    p.global_masks = nullptr;
    p.mask_words = 0;
    p.shard_out = nullptr;
    p.req_list = nullptr;
    p.req_list_n = nullptr;
    p.overflow_list = nullptr;
    p.overflow_n = nullptr;
    p.req_next = nullptr;
    return p;
}

// Device-side offsets alignment probe for device-pointer batches.
static int32_t device_offsets_or_bits(epp_engine *h, const uint64_t *offsets_dev, int64_t n, cudaStream_t s, uint64_t *out) {
    CUDA_TRY(cudaMemsetAsync(h->flag.p, 0, sizeof(int), s));
    CUDA_TRY(launch_check_offsets_aligned(offsets_dev, n, h->flag.as<int>(), s));
    int res = 0;
    CUDA_TRY(cudaMemcpyAsync(&res, h->flag.p, sizeof res, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    *out = (uint64_t)res;
    return EPP_OK;
}

enum class Mode { HashOnly, Match, Schedule };

// Dense-counter kernel over the requests a sparse kernel could not finish (their matched-endpoint set overflowed its
// per-request map).  No host round trip: the kernel reads the list length on the device, at n.
static int32_t launch_overflow_pass(epp_engine *h, Slot &sl, PickParams pp, const int32_t *n, int *launches) {
    cudaStream_t s = sl.stream;
    pp.req_list = sl.overflow_list.as<int32_t>();
    pp.req_list_n = n;
    pp.overflow_list = nullptr;
    pp.overflow_n = nullptr;
    pp.work_counters = nullptr;            // already counted by the sparse pass
    CUDA_TRY(launch_match_pick(pp, h->pick_global ? sl.pick_scratch.as<uint32_t>() : nullptr, h->pick_grid, h->pick_smem, s, launches));
    return EPP_OK;
}

// Standalone match/pick over hashes already in HBM: warp-per-request sparse kernel + overflow pass (or the dense
// kernel alone for Produce-parity rows / A-B runs).
// The latency view of a launch whose request 0 is row r0 of the call in progress.
static LatView lat_view(epp_engine *h, int64_t r0) {
    LatView v;
    memset(&v, 0, sizeof v);
    v.mask = h->lat_mask;
    v.r0 = r0;
    for (int i = 0; i < kMaxProfiles; i++) v.cfg[i] = h->lat_cfg[i];
    for (int i = 0; i < kMaxProfiles; i++) v.rng[i] = (h->cl_mask >> i) & 1 ? h->cl_rng[i].as<longlong2>() : nullptr;
    v.cl_filter = h->cl_filter;
    v.ctx = h->cur->d_ctx;
    v.cnt = h->cur->d_cnt;
    v.off = h->cur->d_off;
    v.ent = h->cur->d_ent;
    return v;
}

// r0: row of pp's request 0 in the call (reads the call's latency predictions).
static int32_t launch_match(epp_engine *h, Slot &sl, PickParams pp, int *launches, int64_t r0 = 0) {
    cudaStream_t s = sl.stream;
    uint32_t *gs = h->pick_global ? sl.pick_scratch.as<uint32_t>() : nullptr;
    if (pp.gen.on && h->lat_mask && !pp.out_match) {
        CUDA_TRY(launch_match_pick_lat(pp, lat_view(h, r0), gs, h->pick_grid, h->pick_smem, s, launches));
        return EPP_OK;
    }
    if (pp.out_match || pp.gen.on) {
        CUDA_TRY(launch_match_pick(pp, gs, h->pick_grid, h->pick_smem, s, launches));
        return EPP_OK;
    }
    // overflow_n[0]: the overflow count, [1]: the sparse kernel's request counter; one memset clears both
    CUDA_TRY(cudaMemsetAsync(sl.overflow_n.p, 0, sizeof(int32_t) * 2, s));
    pp.overflow_list = sl.overflow_list.as<int32_t>();
    pp.overflow_n = sl.overflow_n.as<int32_t>();
    pp.req_next = sl.overflow_n.as<int32_t>() + 1;
    CUDA_TRY(launch_match_pick_sparse(pp, h->sm_count, s, launches));
    return launch_overflow_pass(h, sl, pp, sl.overflow_n.as<int32_t>(), launches);
}

// A Schedule batch's hash rows are read by nothing but its match kernel, whose global stop never lies beyond the first
// block the presence bitmap proves absent: k_hash_fused stores each row only up to there and both match kernels honour
// the bound.  Only on the k_hash_fused + k_match_pick_sparse path (not the dense-counter or general evaluation).  Since
// a block hash depends on the blocks before it alone, the kernel also stops reading each prompt there (EPP_HASH_SKIP).
static void trim_rows(epp_engine *h, const Work &w, HashParams &hp, PickParams &pp) {
    if (!hash_fused_selected(hp) || pp.out_match || pp.gen.on) return;
    hp.skip = h->hash_skip;
    hp.presence = h->presence.as<uint32_t>();
    hp.presence_shift = 64 - h->presence_log2;
    hp.bound = h->bound.as<int32_t>() + w.r0;
    pp.bound = hp.bound;
}

// What run_batch settles for a call before it takes the device, small or host path.
struct Call {
    Mode mode;
    uint64_t *out_hashes;          // the caller's arrays (nullptr: not asked for)
    int32_t *out_nblocks, *out_match, *out_total;
    epp_decision *out_dec;
    epp_decision_detail *out_detail;
    epp_decision_detail *det_out;  // out_detail, or the engine's rows when the inflight producer needs the stage records
    TopkRows tk;
    bool pipelined = false;        // an async Schedule device batch run as chunks over both streams
    bool trim = false;             // trim_rows applies
    int launches = 0;
};

// Rows [r0, r1) of a device-pointer batch, hashed into the same rows of the engine's buffers.
static Work device_work(epp_engine *h, const BatchView &v, int64_t r0, int64_t r1, uint64_t or_bits) {
    return Work{r0, r1, v.offsets ? v.data : v.data + (uint64_t)r0 * v.uniform_len, v.offsets, v.lengths, v.uniform_len,
                v.model_ids, or_bits, h->hashes.as<uint64_t>() + (size_t)r0 * (size_t)h->cfg.max_prefix_blocks,
                h->nblocks.as<int32_t>() + r0, v.multimodal};
}

// The launch sequence of one row range on sl's stream: the hash kernel, then (unless HashOnly) the standalone match /
// score / pick kernel (every fused or concurrently scheduled arrangement of the two was measured slower), writing dec,
// det and out_match from row w.r0 on.  counted: the one-pass device launch, which adds to the work counters and brackets
// the hash kernel with ev[0..3].  pp: the match kernel's parameters, for the subset launch of the same rows.
static int32_t launch_rows(epp_engine *h, Slot &sl, const Work &w, const Call &call, epp_decision *dec,
                           epp_decision_detail *det, int32_t *out_match, bool counted, PickParams &pp, int *launches) {
    unsigned long long *wc = counted ? h->work_counters.as<unsigned long long>() : nullptr;
    HashParams hp = hash_params(h, w, sl);
    if (wc) hp.read = wc + 3;
    if (call.mode != Mode::HashOnly) {
        pp = pick_params(h, w, dec, det, out_match);
        if (call.tk.on) attach_topk(h, pp.gen, call.tk.picks, call.tk.scores, w.r0);
        if (wc) {
            pp.work_counters = wc;
            hp.stored = wc + 2;
        }
        if (call.trim) trim_rows(h, w, hp, pp);
    }
    CUDA_TRY(launch_hash_prompts(hp, sl.stream, launches, counted ? h->ev : nullptr));
    return call.mode == Mode::HashOnly ? EPP_OK : launch_match(h, sl, pp, launches, w.r0);
}

// Completes the device batch in flight on stream 0 and reads its per-kernel CUDA-event times and work counters.
static int32_t finish_async(epp_engine *h) {
    EPP_TRY(join_streams(h));
    CUDA_TRY(cudaStreamSynchronize(h->slot[0].stream));
    if (!h->async_pending) return EPP_OK;
    h->async_pending = false;
    float t[4] = {0, 0, 0, 0};
    for (int i = 0; i < 4; i++) cudaEventElapsedTime(&t[i], h->ev[i], h->ev[i + 1]);
    for (int i = 0; i < 8; i++) h->stats.last_kernel_ms[i] = i < 4 ? t[i] : 0.0;
    h->stats.last_hash_ms = t[0] + t[1] + t[2];
    h->stats.last_match_pick_ms = t[3];
    h->stats.last_kernels_ms = t[0] + t[1] + t[2] + t[3];
    h->stats.last_h2d_ms = h->stats.last_d2h_ms = 0;
    h->stats.last_probes = h->wc_host[0];
    h->stats.last_postings = h->wc_host[1];
    h->stats.last_hash_bytes_stored = h->wc_host[2];
    h->stats.last_prompt_bytes_read = h->wc_host[3];
    h->stats.last_kernel_launches = (uint64_t)h->async_launches;
    for (int u = 0; u < 2; u++) {
        if (!h->post_pick_timed[u]) continue;
        float tu = 0;
        cudaEventElapsedTime(&tu, h->ev[5 + 2 * u], h->ev[6 + 2 * u]);
        h->stats.last_kernel_ms[4 + u] = tu;
        h->post_pick_timed[u] = false;
    }
    h->stats.last_kernel_ms[6] = h->sub_spans.take_ms();
    h->stats.last_kernel_ms[7] = h->adm_spans.take_ms();
    return EPP_OK;
}

// The restricted requests among rows [r0, r1) of a Schedule batch, re-decided on s by the subset kernel after the match
// kernels of the same rows (pp: their PickParams, trimmed rows included).  timed: bracket it for last_kernel_ms[6].
static int32_t launch_subset(epp_engine *h, const PickParams &pp, int64_t r0, int64_t r1, cudaStream_t s, int *launches,
                             bool timed) {
    const std::vector<SubsetRow> &rows = h->cur->sub_rows;
    auto below = [](const SubsetRow &a, int64_t r) { return (int64_t)a.row < r; };
    const size_t lo = std::lower_bound(rows.begin(), rows.end(), r0, below) - rows.begin();
    const size_t hi = std::lower_bound(rows.begin(), rows.end(), r1, below) - rows.begin();
    if (lo == hi) return EPP_OK;
    SubsetView sv;
    sv.rows = h->cur->d_sub_rows + lo;
    sv.n_rows = (int32_t)(hi - lo);
    sv.r0 = r0;
    sv.slots = h->cur->d_sub_slots;
    sv.hits = h->sub_hits.as<int32_t>();
    sv.scratch = h->sub_scratch.as<int32_t>();
    sv.nohit_pos = h->nohit_mask ? h->nh_pos.as<int32_t>() : nullptr;
    if (timed) CUDA_TRY(h->sub_spans.begin(s));
    const LatView lv = lat_view(h, r0);
    CUDA_TRY(launch_subset_pick(pp, sv, h->lat_mask ? &lv : nullptr, s, launches));
    if (timed) CUDA_TRY(h->sub_spans.end(s));
    return EPP_OK;
}

// The listed admission rows among rows [r0, r1) of a call, decided on s by k_admit after the picks (subset launch
// included) of the same rows.  dec / det / tk: the call's rows from request 0 on.  timed: bracket it for last_kernel_ms[7].
static int32_t launch_admission(epp_engine *h, int64_t r0, int64_t r1, epp_decision *dec, epp_decision_detail *det,
                                const TopkRows &tk, cudaStream_t s, int *launches, bool timed) {
    const std::vector<AdmitRow> &rows = h->cur->adm_rows;
    auto below = [](const AdmitRow &a, int64_t r) { return (int64_t)a.row < r; };
    const size_t lo = std::lower_bound(rows.begin(), rows.end(), r0, below) - rows.begin();
    const size_t hi = std::lower_bound(rows.begin(), rows.end(), r1, below) - rows.begin();
    if (lo == hi) return EPP_OK;
    AdmitParams p;
    memset(&p, 0, sizeof p);
    p.rows = h->cur->d_adm_rows + lo;
    p.n_rows = (int32_t)(hi - lo);
    p.E = h->cfg.max_endpoints;
    p.ent = h->cur->d_adm_ent;
    p.sub_slots = h->cur->d_sub_slots;
    p.role = h->role.as<uint8_t>();
    p.kv = h->kv.as<double>();
    p.waiting = h->waiting.as<int32_t>();
    p.running = h->running.as<int32_t>();
    p.pool_n = h->adm_pool_n;
    p.pool_idle = h->adm_idle;
    p.pool_cold = h->adm_cold;
    p.pool_sat = h->adm_sat;
    p.qdt = (double)h->adm.queue_depth_threshold;
    p.kvt = h->adm.kv_cache_util_threshold;
    p.power = h->adm.power;
    p.k = h->adm.k;
    p.tie_seed = h->cfg.tie_seed;
    p.ord_base = h->stats.n_decisions;
    p.dec = dec;
    p.det = det;
    if (tk.on) {
        p.topk = h->cfg.pick_k;
        for (int i = 0; i < kMaxProfiles; i++) p.topk_picks[i] = tk.picks[i];
        p.topk_scores = tk.scores;
    }
    if (timed) CUDA_TRY(h->adm_spans.begin(s));
    CUDA_TRY(launch_admit(p, s, launches));
    if (timed) CUDA_TRY(h->adm_spans.end(s));
    return EPP_OK;
}

// ---- small host batches (cycle_small.cu) -------------------------------------------------------------------------
static int32_t small_reserve(epp_engine *h, int64_t R) {
    if (R <= h->small_cap) return EPP_OK;
    const int64_t cap = std::max<int64_t>(64, std::min<int64_t>(h->small_max, R * 2));
    if (h->small_host) { CUDA_TRY(cudaStreamSynchronize(h->slot[0].stream)); CUDA_TRY(cudaFreeHost(h->small_host)); h->small_host = nullptr; h->small_cap = 0; }
    const size_t n = (size_t)cap;
    const size_t per_set = sizeof(uint64_t) * (n + 1) + sizeof(uint64_t) * n + sizeof(uint32_t) * n + ((n + 7) & ~(size_t)7);
    const size_t total = 2 * per_set + sizeof(epp_decision) * n + sizeof(epp_decision_detail) * n + sizeof(uint32_t) * n + 64;
    CUDA_TRY(cudaHostAlloc(reinterpret_cast<void **>(&h->small_host), total, cudaHostAllocMapped | cudaHostAllocPortable));
    memset(h->small_host, 0, total);
    uint8_t *q = h->small_host;
    for (int i = 0; i < 2; i++) {
        h->small_offsets[i] = reinterpret_cast<uint64_t *>(q); q += sizeof(uint64_t) * (n + 1);
        h->small_lengths[i] = reinterpret_cast<uint64_t *>(q); q += sizeof(uint64_t) * n;
        h->small_models[i] = reinterpret_cast<uint32_t *>(q); q += sizeof(uint32_t) * n;
        h->small_mm[i] = q; q += (n + 7) & ~(size_t)7;
    }
    q = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(q) + 15) & ~(uintptr_t)15);
    h->small_dec = reinterpret_cast<epp_decision *>(q); q += sizeof(epp_decision) * n;
    h->small_det = reinterpret_cast<epp_decision_detail *>(q); q += sizeof(epp_decision_detail) * n;
    h->small_flags = reinterpret_cast<uint32_t *>(q);
    h->small_cap = cap;
    return EPP_OK;
}

// Device view of a pointer into pinned host memory (cudaHostAlloc / cudaHostRegister), or nullptr.
static const uint8_t *device_view_of_pinned(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    if (a.type != cudaMemoryTypeHost || !a.devicePointer) return nullptr;
    return reinterpret_cast<const uint8_t *>(a.devicePointer);
}

// Is this host batch one for the single-launch path?  Returns 0 = no; 1 = the kernel reads the prompts from the
// caller's pinned memory over PCIe (*data_dev = their device view); 2 = one DMA copy into HBM first (SM-issued PCIe
// reads are slower than the copy engine: beyond a handful of prompts the copy wins).
static int small_batch_mode(epp_engine *h, const BatchView &v, const uint8_t **data_dev) {
    if (v.device || h->small_max <= 0 || v.R > h->small_max || h->general) return 0;
    if (sharded(h)) return 0;
    const int64_t bs = (int64_t)h->cfg.block_size_tokens * 4;
    if ((bs & 31) || bs > 64 * 1024 || (size_t)h->cfg.max_prefix_blocks > cycle_small_max_blocks()) return 0;
    const uint64_t layout_bits = v.offsets ? v.offsets_or_bits : v.uniform_len;
    if (v.R <= h->small_zc_max || !v.total_bytes) {
        *data_dev = v.total_bytes ? device_view_of_pinned(v.data) : nullptr;
        if (*data_dev || !v.total_bytes) {
            const uint64_t bits = reinterpret_cast<uintptr_t>(*data_dev) | layout_bits;
            if ((bits & 15) == 0) return 1;
        }
    }
    // the staged copy keeps the caller's layout modulo 32 (see run_small), so only the layout decides the alignment
    return (layout_bits & 15) == 0 ? 2 : 0;
}

// cuStreamWriteValue32 through the runtime's driver-entry-point lookup (no link against libcuda); nullptr when absent.
typedef CUresult (*StreamWriteValue32)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
static StreamWriteValue32 stream_write_value32() {
    static const StreamWriteValue32 fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuStreamWriteValue32", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            p = nullptr;
        }
        return reinterpret_cast<StreamWriteValue32>(p);
    }();
    return fn;
}

// Waits for the flag word of every request of small batch `epoch` (written after a system-scope fence behind its
// decision) on the host; *overflowed: some request was left to the overflow pass.
static int32_t wait_small_flags(epp_engine *h, int64_t R, uint32_t epoch, uint32_t *overflowed) {
    volatile uint32_t *flags = h->small_flags;
    uint32_t spins = 0;
    bool finished_once = false;
    for (int64_t next = 0; next < R;) {
        const uint32_t x = flags[next];
        if ((x & 0x7fffffffu) == epoch) { *overflowed |= x >> 31; next++; continue; }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
        if ((++spins & 0x3fff) == 0) {             // a faulted launch never raises its flags
            const cudaError_t q = cudaStreamQuery(h->slot[0].stream);
            if (q == cudaSuccess) {
                if (finished_once) return fail(EPP_ERR_CUDA, "small-batch kernel finished without publishing request %lld", (long long)next);
                finished_once = true;
            } else if (q != cudaErrorNotReady) {
                return fail(EPP_ERR_CUDA, "small-batch kernel failed: %s", cudaGetErrorString(q));
            }
        }
    }
    return EPP_OK;
}

static int32_t run_small(epp_engine *h, const BatchView &v, int mode, const uint8_t *data_dev, epp_decision *out_dec,
                         epp_decision_detail *out_detail) {
    const int64_t R = v.R;
    cudaStream_t s0 = h->slot[0].stream;
    EPP_TRY(reserve_batch(h, R));
    EPP_TRY(small_reserve(h, R));
    uint32_t epoch = h->small_epoch + 1;
    if (epoch > 0x7fffffffu) {
        epoch = 1;
        CUDA_TRY(cudaMemsetAsync(h->small_arrive.p, 0, sizeof(uint32_t), s0));
        CUDA_TRY(cudaStreamSynchronize(s0));
    }
    h->small_epoch = epoch;
    const uint32_t *arrive = nullptr;
    if (mode == 2) {
        const uint64_t start = v.offsets ? v.offsets[0] : 0;
        CUDA_TRY(h->slot[0].data.reserve(v.total_bytes + 64, &h->dev_bytes));
        uint8_t *stage = h->slot[0].data.as<uint8_t>() + (start & 31);
        data_dev = reinterpret_cast<const uint8_t *>(reinterpret_cast<uintptr_t>(stage) - (uintptr_t)start);   // + offsets[r]
        if (h->small_pipe_min > 0 && R >= h->small_pipe_min &&
            cycle_small_stages_prompt(h->cfg.max_prefix_blocks, h->cfg.block_size_tokens * 4)) {
            // The copy goes to the second stream with a stream-ordered 32-bit write of the epoch behind it; the kernel is
            // launched on s0 at once and thread 0 of every CTA waits for that word, so the launch latency (and the stream's
            // copy -> kernel hand-over) hides under the transfer.  The staging buffer is free although the kernel of the batch
            // before may still be walking chains: it keeps a whole prompt in shared memory (cycle_small_stages_prompt),
            // so every request raised its flag after its last read of these bytes.
            cudaStream_t s1 = h->slot[1].stream;
            uint32_t *arr = h->small_arrive.as<uint32_t>();
            CUDA_TRY(cudaMemcpyAsync(stage, v.data + start, v.total_bytes, cudaMemcpyHostToDevice, s1));
            const StreamWriteValue32 wv = h->small_no_write_value ? nullptr : stream_write_value32();
            if (!wv || wv(s1, reinterpret_cast<CUdeviceptr>(arr), epoch, 0) != CUDA_SUCCESS) {
                h->small_no_write_value = true;    // no stream memory operations in this driver / context: a 4-byte copy does it
                *h->small_epoch_host = epoch;      // read by the copy below before this (synchronous) call returns
                CUDA_TRY(cudaMemcpyAsync(arr, h->small_epoch_host, sizeof(uint32_t), cudaMemcpyHostToDevice, s1));
            }
            arrive = arr;
            h->s1_unjoined = true;
        } else {
            CUDA_TRY(cudaMemcpyAsync(stage, v.data + start, v.total_bytes, cudaMemcpyHostToDevice, s0));
        }
    }
    const int set = (int)(epoch & 1);              // the kernel of the batch before may still be finishing its chains
    if (v.offsets) memcpy(h->small_offsets[set], v.offsets, sizeof(uint64_t) * (size_t)(R + 1));
    if (v.lengths) memcpy(h->small_lengths[set], v.lengths, sizeof(uint64_t) * (size_t)R);
    if (v.model_ids) memcpy(h->small_models[set], v.model_ids, sizeof(uint32_t) * (size_t)R);
    if (v.multimodal) memcpy(h->small_mm[set], v.multimodal, (size_t)R);
    // the per-request arrays are pinned + mapped: host address == device address (UVA)
    const Work w{0, R, data_dev, v.offsets ? h->small_offsets[set] : nullptr, v.lengths ? h->small_lengths[set] : nullptr,
                 v.uniform_len, v.model_ids ? h->small_models[set] : nullptr, v.offsets_or_bits, h->hashes.as<uint64_t>(),
                 h->nblocks.as<int32_t>(), v.multimodal ? h->small_mm[set] : nullptr};
    PickParams pp = pick_params(h, w, h->decisions.as<epp_decision>(), h->details.as<epp_decision_detail>(), nullptr);
    pp.overflow_list = h->slot[0].overflow_list.as<int32_t>();
    pp.overflow_n = h->small_overflow_n.as<int32_t>();
    SmallOut so{h->small_dec, h->small_det, h->small_flags, epoch, arrive};
    int launches = 0;
    CUDA_TRY(cudaEventRecord(h->ev[0], s0));
    CUDA_TRY(launch_cycle_small(hash_params(h, w, h->slot[0]), pp, so, s0, &launches));
    CUDA_TRY(cudaEventRecord(h->ev[1], s0));
    uint32_t overflowed = 0;
    EPP_TRY(wait_small_flags(h, R, epoch, &overflowed));
    if (overflowed) {
        // > 32 endpoints hold a part of some prompt: those requests go through the dense-counter kernel, then the whole
        // batch is read back the ordinary way
        EPP_TRY(launch_overflow_pass(h, h->slot[0], pp, h->small_overflow_n.as<int32_t>(), &launches));
        CUDA_TRY(cudaMemsetAsync(h->small_overflow_n.p, 0, sizeof(int32_t), s0));
        CUDA_TRY(cudaMemcpyAsync(h->small_dec, h->decisions.p, sizeof(epp_decision) * (size_t)R, cudaMemcpyDeviceToHost, s0));
        CUDA_TRY(cudaMemcpyAsync(h->small_det, h->details.p, sizeof(epp_decision_detail) * (size_t)R, cudaMemcpyDeviceToHost, s0));
        CUDA_TRY(cudaStreamSynchronize(s0));
    }
    // reads the decisions from the pinned copies (UVA)
    EPP_TRY(after_picks(h, h->small_dec, h->small_det, h->in_len.as<int64_t>(), R, s0, &launches, false));
    memcpy(out_dec, h->small_dec, sizeof(epp_decision) * (size_t)R);
    if (out_detail) memcpy(out_detail, h->small_det, sizeof(epp_decision_detail) * (size_t)R);
    h->small_stats_pending = true;
    h->stats.last_hash_ms = h->stats.last_match_pick_ms = 0;
    h->stats.last_kernel_launches = (uint64_t)launches;
    return EPP_OK;
}

// A device-pointer batch: an async Schedule batch of at least two chunks runs chunk-pipelined over both streams, any other
// in one pass on stream 0.  An async batch (not Match) returns with its results and stats pending (finish_async).
static int32_t run_device(epp_engine *h, const BatchView &v, Call &call) {
    const int64_t R = v.R;
    cudaStream_t s0 = h->slot[0].stream;
    uint64_t or_bits = 0;
    if (v.offsets) EPP_TRY(device_offsets_or_bits(h, v.offsets, R, s0, &or_bits));
    CUDA_TRY(cudaMemsetAsync(h->work_counters.p, 0, sizeof(unsigned long long) * 4, s0));
    const int64_t min_chunk = 4096;
    h->sub_spans.used = 0;
    h->adm_spans.used = 0;
    epp_decision *dec = call.out_dec ? call.out_dec : h->decisions.as<epp_decision>();
    PickParams pp;                                 // the rows of the last launch_rows, for their subset launch
    if (call.pipelined) {
        // Throughput mode: the batch runs as C chunks alternating between the engine's two streams, so the hash
        // kernel of one chunk (HBM / integer bound) shares the SMs with the match kernel of another (latency bound).
        // Consecutive pipelined batches of the same shape are not joined: every row range of the engine's buffers is
        // only ever touched by one stream, and the next entry point of any other kind joins the streams first.
        const int64_t C = std::min<int64_t>(h->dev_chunks, R / min_chunk);
        const int64_t per = ((R + C - 1) / C + 31) & ~(int64_t)31;
        cudaStream_t s1 = h->slot[1].stream;
        if (h->s1_unjoined && (h->inflight || h->pipe_R != R || h->pipe_per != per)) EPP_TRY(join_streams(h));
        for (int i = 0; i < 4; i++) CUDA_TRY(cudaEventRecord(h->ev[i], s0));
        if (!h->s1_unjoined) {
            CUDA_TRY(cudaEventRecord(h->slot[0].done, s0));
            CUDA_TRY(cudaStreamWaitEvent(s1, h->slot[0].done, 0));
        }
        int k = 0;
        for (int64_t r0 = 0; r0 < R; r0 += per, k++) {
            const int64_t r1 = std::min(R, r0 + per);
            Slot &sl = h->slot[k & 1];
            EPP_TRY(launch_rows(h, sl, device_work(h, v, r0, r1, or_bits), call, dec + r0,
                                call.det_out ? call.det_out + r0 : nullptr, nullptr, false, pp, &call.launches));
            EPP_TRY(launch_subset(h, pp, r0, r1, sl.stream, &call.launches, true));
            EPP_TRY(launch_admission(h, r0, r1, dec, call.det_out, call.tk, sl.stream, &call.launches, true));
        }
        h->s1_unjoined = true;
        // the next call's picks must see both chunks' Adds: join the chunks on stream 0 for the update (below), and the
        // next call's stream-1 chunk waits for stream 0 again (engines without the scorer or the producer stay unjoined)
        if (h->nohit_mask || h->inflight) EPP_TRY(join_streams(h));
        h->pipe_R = R;
        h->pipe_per = per;
    } else {
        Work w = device_work(h, v, 0, R, or_bits);
        if (call.mode == Mode::HashOnly && call.out_hashes) w.hashes_out = call.out_hashes;
        if (call.mode == Mode::HashOnly && call.out_nblocks) w.nblocks_out = call.out_nblocks;
        if (call.mode == Mode::Match && call.out_total) w.nblocks_out = call.out_total;
        EPP_TRY(launch_rows(h, h->slot[0], w, call, dec, call.mode == Mode::Schedule ? call.det_out : nullptr,
                            call.mode == Mode::Match ? call.out_match : nullptr, true, pp, &call.launches));
    }
    CUDA_TRY(cudaEventRecord(h->ev[4], s0));
    if (call.mode == Mode::Schedule) {             // after ev[4]: last_kernel_ms[3] stays the match + pick time
        if (!call.pipelined) {
            EPP_TRY(launch_subset(h, pp, 0, R, s0, &call.launches, true));
            EPP_TRY(launch_admission(h, 0, R, dec, call.det_out, call.tk, s0, &call.launches, true));
        }
        EPP_TRY(after_picks(h, dec, call.det_out, h->in_len.as<int64_t>(), R, s0, &call.launches, true));
    }
    CUDA_TRY(cudaMemcpyAsync(h->wc_host, h->work_counters.p, sizeof(unsigned long long) * 4, cudaMemcpyDeviceToHost, s0));
    h->async_pending = true;
    h->async_launches = call.launches;
    if (v.async && call.mode != Mode::Match) return EPP_OK;    // epp_synchronize() (or the next call that needs the
                                                               // results on the host) completes it
    return finish_async(h);
}

// A host batch: the small per-request arrays are uploaded once, then the prompt bytes go in chunks whose H2D copy
// overlaps the kernels of the previous chunk (two streams, two staging buffers); each chunk's results are copied back
// behind its kernels.
static int32_t run_host(epp_engine *h, const BatchView &v, Call &call) {
    const int64_t R = v.R;
    const size_t B = (size_t)h->cfg.max_prefix_blocks;
    cudaStream_t s0 = h->slot[0].stream;
    if (v.offsets) CUDA_TRY(cudaMemcpyAsync(h->offsets.p, v.offsets, sizeof(uint64_t) * (size_t)(R + 1), cudaMemcpyHostToDevice, s0));
    if (v.lengths) CUDA_TRY(cudaMemcpyAsync(h->lengths.p, v.lengths, sizeof(uint64_t) * (size_t)R, cudaMemcpyHostToDevice, s0));
    if (v.model_ids) CUDA_TRY(cudaMemcpyAsync(h->model_ids.p, v.model_ids, sizeof(uint32_t) * (size_t)R, cudaMemcpyHostToDevice, s0));
    if (v.multimodal) {
        CUDA_TRY(h->multimodal.reserve((size_t)R, &h->dev_bytes));
        CUDA_TRY(cudaMemcpyAsync(h->multimodal.p, v.multimodal, (size_t)R, cudaMemcpyHostToDevice, s0));
    }
    CUDA_TRY(cudaEventRecord(h->slot[0].done, s0));
    CUDA_TRY(cudaStreamWaitEvent(h->slot[1].stream, h->slot[0].done, 0));

    // chunk plan: at least one request per chunk, about kChunkBytes of prompt bytes
    const uint64_t kChunkBytes = 48ull << 20;
    struct Chunk { int64_t r0, r1; uint64_t start, bytes; };
    std::vector<Chunk> chunks;
    uint64_t max_bytes = 0;
    for (int64_t r = 0; r < R;) {
        int64_t r_end = r;
        uint64_t start, bytes;
        if (v.offsets) {
            while (r_end < R && (r_end == r || (v.offsets[r_end + 1] - v.offsets[r]) <= kChunkBytes)) r_end++;
            start = v.offsets[r];
            bytes = v.offsets[r_end] - start;
        } else {
            int64_t per = v.uniform_len ? (int64_t)std::max<uint64_t>(1, kChunkBytes / v.uniform_len) : R;
            r_end = std::min(R, r + per);
            start = (uint64_t)r * v.uniform_len;
            bytes = (uint64_t)(r_end - r) * v.uniform_len;
        }
        chunks.push_back({r, r_end, start, bytes});
        max_bytes = std::max(max_bytes, bytes);
        r = r_end;
    }
    for (int i = 0; i < 2; i++) CUDA_TRY(h->slot[i].data.reserve(max_bytes + 64, &h->dev_bytes));
    const size_t E = (size_t)h->cfg.max_endpoints;
    if (call.mode == Mode::Match) CUDA_TRY(h->dense_match.reserve(sizeof(int32_t) * (size_t)R * E, &h->dev_bytes));

    CUDA_TRY(cudaEventRecord(h->ev[0], s0));
    for (size_t k = 0; k < chunks.size(); k++) {
        const Chunk &c = chunks[k];
        Slot &sl = h->slot[k & 1];
        cudaStream_t s = sl.stream;
        const size_t nreq = (size_t)(c.r1 - c.r0);
        // keep the staged copy aligned (mod 32) like the caller's layout
        uint8_t *stage = sl.data.as<uint8_t>() + (c.start & 31);
        if (c.bytes) CUDA_TRY(cudaMemcpyAsync(stage, v.data + c.start, c.bytes, cudaMemcpyHostToDevice, s));
        // the kernels address  data_base + offsets[r]  with ABSOLUTE offsets, or  data_base + chunk-local index * uniform_len
        const uint8_t *base = v.offsets ? reinterpret_cast<const uint8_t *>(reinterpret_cast<uintptr_t>(stage) - (uintptr_t)c.start)
                                        : stage;
        const Work w{c.r0, c.r1, base, v.offsets ? h->offsets.as<uint64_t>() : nullptr,
                     v.offsets && v.lengths ? h->lengths.as<uint64_t>() : nullptr, v.uniform_len,
                     v.model_ids ? h->model_ids.as<uint32_t>() : nullptr, v.offsets ? v.offsets_or_bits : 0,
                     h->hashes.as<uint64_t>() + (size_t)c.r0 * B, h->nblocks.as<int32_t>() + c.r0,
                     v.multimodal ? h->multimodal.as<uint8_t>() : nullptr};
        int32_t *dm = call.mode == Mode::Match ? h->dense_match.as<int32_t>() + (size_t)c.r0 * E : nullptr;
        epp_decision *dec = h->decisions.as<epp_decision>() + c.r0;
        epp_decision_detail *det = h->details.as<epp_decision_detail>() + c.r0;
        PickParams pp;
        EPP_TRY(launch_rows(h, sl, w, call, dec, det, dm, false, pp, &call.launches));
        if (call.mode == Mode::HashOnly) {
            if (call.out_hashes) CUDA_TRY(cudaMemcpyAsync(call.out_hashes + (size_t)c.r0 * B, w.hashes_out, sizeof(uint64_t) * nreq * B, cudaMemcpyDeviceToHost, s));
            if (call.out_nblocks) CUDA_TRY(cudaMemcpyAsync(call.out_nblocks + c.r0, w.nblocks_out, sizeof(int32_t) * nreq, cudaMemcpyDeviceToHost, s));
        } else if (call.mode == Mode::Schedule) {
            EPP_TRY(launch_subset(h, pp, c.r0, c.r1, s, &call.launches, false));
            EPP_TRY(launch_admission(h, c.r0, c.r1, h->decisions.as<epp_decision>(), h->details.as<epp_decision_detail>(),
                                     call.tk, s, &call.launches, false));
            if (call.out_dec) CUDA_TRY(cudaMemcpyAsync(call.out_dec + c.r0, dec, sizeof(epp_decision) * nreq, cudaMemcpyDeviceToHost, s));
            if (call.out_detail) CUDA_TRY(cudaMemcpyAsync(call.out_detail + c.r0, det, sizeof(epp_decision_detail) * nreq, cudaMemcpyDeviceToHost, s));
            if (call.tk.on) EPP_TRY(topk_copy_back(h, call.tk, c.r0, (int64_t)nreq, s));
        } else {
            if (call.out_match) CUDA_TRY(cudaMemcpyAsync(call.out_match + (size_t)c.r0 * E, dm, sizeof(int32_t) * nreq * E, cudaMemcpyDeviceToHost, s));
            if (call.out_total) CUDA_TRY(cudaMemcpyAsync(call.out_total + c.r0, w.nblocks_out, sizeof(int32_t) * nreq, cudaMemcpyDeviceToHost, s));
        }
    }
    CUDA_TRY(cudaStreamSynchronize(h->slot[1].stream));
    if (call.mode == Mode::Schedule)
        EPP_TRY(after_picks(h, h->decisions.as<epp_decision>(), h->details.as<epp_decision_detail>(), h->in_len.as<int64_t>(), R,
                            s0, &call.launches, false));
    CUDA_TRY(cudaEventRecord(h->ev[1], s0));
    CUDA_TRY(cudaStreamSynchronize(s0));
    float t_all = 0;
    cudaEventElapsedTime(&t_all, h->ev[0], h->ev[1]);
    h->stats.last_kernels_ms = t_all;
    h->stats.last_kernel_ms[6] = 0.0;              // the subset and admission kernels are timed on device batches only
    h->stats.last_kernel_ms[7] = 0.0;
    h->stats.last_hash_ms = h->stats.last_match_pick_ms = 0;
    h->stats.last_kernel_launches = (uint64_t)call.launches;
    return EPP_OK;
}

// Runs hashing (+ match/pick) for a batch: device batches in run_device, small host batches in pinned memory in
// run_small, every other host batch in run_host.
// keep_hashes: the hash rows of a Schedule batch stay for epp_index_add_picked (whole rows, no trimming).
static int32_t run_batch(epp_engine *h, const BatchView &v, Mode mode, uint64_t *out_hashes, int32_t *out_nblocks,
                         epp_decision *out_dec, epp_decision_detail *out_detail, int32_t *out_match,
                         int32_t *out_total, bool keep_hashes = false) {
    const int64_t R = v.R;
    if (R == 0) return EPP_OK;
    if (mode != Mode::HashOnly) {
        if (!h->pool_ready) return fail(EPP_ERR_STATE, "epp_pool_set has not been called");
        // index updates become visible here -- or, with index_commit_interval_us, at most that much later: the reference
        // applies PreRequest in a goroutine of its own "to avoid blocking the request path" (approximateprefix/plugin.go:189-194),
        // so a scheduling cycle may well run against an index that lacks the last few picks
        const bool due = h->cfg.index_commit_interval_us <= 0 || !h->committed_once ||
                         ms_since(h->last_commit) * 1000.0 >= (double)h->cfg.index_commit_interval_us;
        if (due) {
            EPP_TRY(commit_locked(h));
            h->last_commit = std::chrono::steady_clock::now();
            h->committed_once = true;
        }
    }
    if (h->async_pending && !(v.device && v.async)) EPP_TRY(finish_async(h));
    Call call{mode, out_hashes, out_nblocks, out_match, out_total, out_dec, out_detail, out_detail};
    EPP_TRY(topk_rows(h, mode == Mode::Schedule ? h->cur->topk : nullptr, v.device, R, call.tk));
    call.pipelined = v.device && v.async && mode == Mode::Schedule && h->dev_chunks > 1 && R >= 2 * 4096 && !h->pick_global;
    // the endpoint-sharded mode's local table is not the global one: its rows stay whole
    call.trim = mode == Mode::Schedule && !keep_hashes && h->hash_trim && !sharded(h);
    if (!call.pipelined) EPP_TRY(join_streams(h));
    EPP_TRY(reserve_batch(h, R));
    // releases / resets since the last call, on stream 0 before any pick kernel (a pipelined batch's stream 1 waits
    // for stream 0 in run_device)
    if (mode == Mode::Schedule) EPP_TRY(inflight_flush(h, h->slot[0].stream, &call.launches));
    // the stage records reach the producer's add kernel even when the caller asked for none
    if (mode == Mode::Schedule && !out_detail && h->inflight) call.det_out = h->details.as<epp_decision_detail>();
    if (v.device) return run_device(h, v, call);

    // small host batch in pinned memory: one zero-copy launch, no copy engine, no stream synchronisation (not for a batch
    // with restricted requests or admission rows: the kernel hands the decisions to the host before a subset or admission
    // launch could rewrite them)
    if (mode == Mode::Schedule && !call.tk.on && out_dec && h->cur->sub_rows.empty() && h->cur->adm_rows.empty()) {
        const uint8_t *data_dev = nullptr;
        const int sm = small_batch_mode(h, v, &data_dev);
        if (sm) return run_small(h, v, sm, data_dev, out_dec, out_detail);
    }
    return run_host(h, v, call);
}

extern "C" int32_t epp_hash_prompts(epp_engine *h, const epp_batch *batch, uint64_t *out_hashes, int32_t *out_nblocks) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    BatchView v;
    EPP_TRY(check_batch(h, batch, v));
    v.async = false;                               // EPP_BATCH_ASYNC is an epp_schedule flag: hashes are complete on return
    h->kept_R = 0;
    return run_batch(h, v, Mode::HashOnly, out_hashes, out_nblocks, nullptr, nullptr, nullptr, nullptr);
}

extern "C" int32_t epp_prefix_match(epp_engine *h, const epp_batch *batch, int32_t *out_match, int32_t *out_total) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    if (!out_match) return fail(EPP_ERR_INVALID, "out_match is NULL");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    BatchView v;
    EPP_TRY(check_batch(h, batch, v));
    h->kept_R = 0;
    return run_batch(h, v, Mode::Match, nullptr, nullptr, nullptr, nullptr, out_match, out_total);
}

static int32_t check_topk(epp_engine *h, const epp_topk_out *topk) {
    if (!topk) return fail(EPP_ERR_INVALID, "topk is NULL");
    if (topk->struct_size != sizeof(epp_topk_out)) return fail(EPP_ERR_INVALID, "epp_topk_out.struct_size %u != %zu", topk->struct_size, sizeof(epp_topk_out));
    if (h->cfg.pick_k <= 1) return fail(EPP_ERR_STATE, "the engine was created with pick_k = %d: nothing but the pick to return", h->cfg.pick_k);
    if (topk->k != h->cfg.pick_k) return fail(EPP_ERR_INVALID, "epp_topk_out.k %d != epp_config.pick_k %d", topk->k, h->cfg.pick_k);
    return EPP_OK;
}

// Validates the subsets of a batch of R requests on the host and lists the restricted ones in ascending request order,
// each with its offset in the packed slot array (*n_slots entries in all).  Nothing of the engine changes.
// latency_ok: the call may also carry predictions (epp_schedule_subset_predicted), so a latency engine is accepted.
static int32_t check_subset(const epp_engine *h, int64_t R, const epp_subset *s, std::vector<SubsetRow> &rows,
                            uint64_t *n_slots, bool latency_ok) {
    if (s->struct_size != sizeof(epp_subset)) return fail(EPP_ERR_INVALID, "epp_subset.struct_size %u != %zu", s->struct_size, sizeof(epp_subset));
    if (sharded(h) || h->p2p_buf)
        return fail(EPP_ERR_INVALID, "endpoint subsets are not available in the endpoint-sharded and peer-memory modes");
    if (h->lat_mask && !latency_ok)
        return fail(EPP_ERR_INVALID, "endpoint subsets on an engine with latency profiles go through epp_schedule_subset_predicted");
    if (R > 0 && !s->counts) return fail(EPP_ERR_INVALID, "epp_subset.counts is NULL");
    const uint32_t E = (uint32_t)h->cfg.max_endpoints;
    int64_t n_rows = 0;
    for (int64_t r = 0; r < R; r++) n_rows += s->counts[r] != EPP_SUBSET_ALL;
    rows.reserve((size_t)n_rows);
    uint64_t total = 0;
    for (int64_t r = 0; r < R; r++) {
        const uint32_t n = s->counts[r];
        if (n == EPP_SUBSET_ALL) continue;
        if (n > E) return fail(EPP_ERR_INVALID, "request %lld: %u slots, more than max_endpoints %u", (long long)r, n, E);
        if (n) {
            if (!s->offsets || !s->slots) return fail(EPP_ERR_INVALID, "epp_subset.offsets / slots is NULL");
            const uint32_t *src = s->slots + s->offsets[r];
            for (uint32_t i = 0; i < n; i++) {
                if (src[i] >= E) return fail(EPP_ERR_INVALID, "request %lld: slot %u >= max_endpoints %u", (long long)r, src[i], E);
                if (i && src[i] <= src[i - 1]) return fail(EPP_ERR_INVALID, "request %lld: slots not strictly ascending at entry %u", (long long)r, i);
            }
        }
        rows.push_back({total, (uint32_t)r, n});
        total += n;
    }
    *n_slots = total;
    return EPP_OK;
}

// For the batcher (batcher.cu), which refuses subsets and checks predictions at submit time.  The mask is fixed once the
// pool is set, and no batch is scheduled before that.
int32_t engine_latency_mask(const epp_engine *h) { return h->lat_mask; }
// The admitters (kAdmitProbabilistic | kAdmitLatencySlo), for the batcher's submit-time checks; fixed once the pool is set.
int32_t engine_admission(const epp_engine *h) {
    if (!h->adm_on) return 0;
    return (h->adm.probabilistic ? (int32_t)kAdmitProbabilistic : 0) | (h->adm.latency_slo ? (int32_t)kAdmitLatencySlo : 0);
}

extern "C" void epp_latency_cfg_default(epp_latency_cfg *cfg) {
    if (!cfg) return;
    memset(cfg, 0, sizeof *cfg);
    cfg->struct_size = sizeof(epp_latency_cfg);
    cfg->epsilon_explore_neg = 0.01;                  // sloheadroomtier/plugin.go:50-52
    cfg->a1_affinity_threshold = 0.0;                 // no A1
    cfg->a1_exploration_probability = 0.01;           // prefixcacheaffinity/plugin.go:62-66
    cfg->a1_max_ttft_penalty_ms = 5000.0;
    cfg->ttft_weight = 0.8;                           // scorer/latency/plugin.go:83-90
    cfg->tpot_weight = 0.2;
    cfg->strategy = EPP_HEADROOM_LEAST;
    cfg->composite_kv_weight = cfg->composite_queue_weight = cfg->composite_prefix_weight = 1.0;
}

extern "C" int32_t epp_latency_profile_set(epp_engine *h, int32_t profile, const epp_latency_cfg *cfg) {
    if (!h || !cfg) return fail(EPP_ERR_INVALID, "NULL engine or configuration");
    if (profile < 0 || profile >= h->n_alloc_profiles) return fail(EPP_ERR_INVALID, "profile %d is not configured", profile);
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->pool_called) return fail(EPP_ERR_STATE, "latency profiles are fixed once the pool has been set");
    if (sharded(h) || h->p2p_buf)
        return fail(EPP_ERR_INVALID, "endpoint-sharded mode does not support latency profiles");
    const epp_profile_cfg &pc = profile_cfg(h, profile);
    EPP_TRY(validate_latency(pc, *cfg, profile == 0 ? "primary profile" : (profile == 1 ? "prefill profile" : "encode profile")));
    h->lat_cfg[profile] = *cfg;
    if (chain_profile(pc, *cfg)) h->lat_mask |= 1 << profile;
    else h->lat_mask &= ~(1 << profile);
    if (h->lat_mask) h->general = true;
    return EPP_OK;
}

// Validates the predictions of a batch of R requests on the host (*n_ent entries in all).  Nothing of the engine changes.
static int32_t check_predictions(const epp_engine *h, int64_t R, const epp_predictions *p, uint64_t *n_ent) {
    if (p->struct_size != sizeof(epp_predictions)) return fail(EPP_ERR_INVALID, "epp_predictions.struct_size %u != %zu", p->struct_size, sizeof(epp_predictions));
    if (!h->lat_mask && !(h->adm_on && h->adm.latency_slo))
        return fail(EPP_ERR_INVALID, "predictions passed to an engine without a latency profile or the latency-slo-admitter");
    if (R > 0 && !p->counts) return fail(EPP_ERR_INVALID, "epp_predictions.counts is NULL");
    const uint32_t E = (uint32_t)h->cfg.max_endpoints;
    uint64_t total = 0;
    for (int64_t r = 0; r < R; r++) {
        const uint32_t n = p->counts[r];
        if (!n) continue;
        if (n > E) return fail(EPP_ERR_INVALID, "request %lld: %u predictions, more than max_endpoints %u", (long long)r, n, E);
        if (!p->offsets || !p->entries) return fail(EPP_ERR_INVALID, "epp_predictions.offsets / entries is NULL");
        const epp_prediction *src = p->entries + p->offsets[r];
        for (uint32_t i = 0; i < n; i++) {
            if (src[i].slot >= E) return fail(EPP_ERR_INVALID, "request %lld: slot %u >= max_endpoints %u", (long long)r, src[i].slot, E);
            if (i && src[i].slot <= src[i - 1].slot) return fail(EPP_ERR_INVALID, "request %lld: prediction slots not strictly ascending at entry %u", (long long)r, i);
            if (!std::isfinite(src[i].ttft) || !std::isfinite(src[i].ttft_headroom) || !std::isfinite(src[i].tpot_headroom))
                return fail(EPP_ERR_INVALID, "request %lld: prediction %u is not finite", (long long)r, i);
        }
        total += n;
    }
    *n_ent = total;
    return EPP_OK;
}

// Validates a call's context lengths (R entries, each >= -1).  Nothing of the engine changes.
static int32_t check_ctx(int64_t R, const epp_context_tokens *c) {
    if (c->struct_size != sizeof(epp_context_tokens)) return fail(EPP_ERR_INVALID, "epp_context_tokens.struct_size %u != %zu", c->struct_size, sizeof(epp_context_tokens));
    if (R > 0 && !c->tokens) return fail(EPP_ERR_INVALID, "epp_context_tokens.tokens is NULL");
    for (int64_t r = 0; r < R; r++)
        if (c->tokens[r] < -1) return fail(EPP_ERR_INVALID, "request %lld: context tokens %lld < -1", (long long)r, (long long)c->tokens[r]);
    return EPP_OK;
}

// Validates a call's admission inputs (R requests; preds: the call's predictions, validated, or nullptr; sub: its
// restricted rows, ascending) and lists, in ascending request order, the rows an admitter can reject, with the packed
// entries of the latency-slo-admitter's rows (slot | both validity bits << 31).  Nothing of the engine changes.
static int32_t check_admission(const epp_engine *h, int64_t R, const epp_admission *a, const epp_predictions *preds,
                               const std::vector<SubsetRow> &sub, std::vector<AdmitRow> &rows, std::vector<uint32_t> &ent) {
    if (a->struct_size != sizeof(epp_admission)) return fail(EPP_ERR_INVALID, "epp_admission.struct_size %u != %zu", a->struct_size, sizeof(epp_admission));
    if (!h->adm_on) return fail(EPP_ERR_INVALID, "admission inputs passed to an engine without admitters (epp_admission_set)");
    const bool lat = h->adm.latency_slo != 0, with_pred = lat && preds && R > 0;
    if (with_pred && !a->pred_valid)
        return fail(EPP_ERR_INVALID, "epp_admission.pred_valid is NULL: the latency-slo-admitter needs it for a call with predictions");
    if (!a->priority) return EPP_OK;              // nobody is sheddable
    size_t si = 0;
    for (int64_t r = 0; r < R; r++) {
        while (si < sub.size() && (int64_t)sub[si].row < r) si++;
        if (a->priority[r] >= 0) continue;
        const bool restricted = si < sub.size() && (int64_t)sub[si].row == r;
        if (restricted && sub[si].n == 0) continue;    // no candidate: status -1 stands
        AdmitRow row{(uint32_t)r, 0u, restricted ? sub[si].off : 0ull, restricted ? sub[si].n : EPP_SUBSET_ALL, 0u, 0ull};
        if (h->adm.probabilistic) row.flags |= kAdmitProbabilistic;
        const double ttft = a->ttft_slo ? a->ttft_slo[r] : 0.0, tpot = a->tpot_slo ? a->tpot_slo[r] : 0.0;
        if (with_pred && preds->counts[r] && (ttft > 0 || tpot > 0)) {
            row.flags |= kAdmitLatencySlo;
            row.pred_off = ent.size();
            row.pred_n = preds->counts[r];
            const uint64_t o = preds->offsets[r];
            for (uint32_t i = 0; i < row.pred_n; i++)
                ent.push_back(preds->entries[o + i].slot | ((a->pred_valid[o + i] & 3u) == 3u ? 0x80000000u : 0u));
        }
        if (row.flags) rows.push_back(row);
    }
    return EPP_OK;
}

// Validates a call's side inputs (R requests; each input nullptr when not passed) into in: subsets, predictions, context
// lengths, then admission, and which of them the engine reads.  Nothing of the engine changes.
// latency_ok: as check_subset.
static int32_t check_inputs(const epp_engine *h, int64_t R, const epp_subset *subset, bool latency_ok,
                            const epp_predictions *preds, const epp_context_tokens *ctx, const epp_admission *adm,
                            CallInputs &in) {
    in.R = R;
    in.subset = subset;
    in.preds = preds;
    in.ctx = ctx;
    if (subset) EPP_TRY(check_subset(h, R, subset, in.sub_rows, &in.sub_n_slots, latency_ok));
    if (preds) EPP_TRY(check_predictions(h, R, preds, &in.n_ent));
    if (ctx) EPP_TRY(check_ctx(R, ctx));
    if (adm) EPP_TRY(check_admission(h, R, adm, preds, in.sub_rows, in.adm_rows, in.adm_ent));
    in.use_pred = preds && R && h->lat_mask;
    in.use_ctx = ctx && R && h->cl_mask;
    return EPP_OK;
}

// A validated call's staged inputs to the device on stream 0, behind everything enqueued so far (a pipelined batch's
// stream 1 joins first): the sections are packed into the engine's pinned staging, each from a 256-byte boundary (the
// alignment of a cudaMalloc), and go over in one copy.  The staging is refilled only once the previous call's copy has
// run (in_ev).  Sets in's device pointers.
static int32_t stage_inputs(epp_engine *h, CallInputs &in) {
    if (!in.staged()) return EPP_OK;
    const size_t R = (size_t)in.R;
    size_t total = 0;
    auto section = [&total](size_t bytes) {
        const size_t at = (total + 255) & ~(size_t)255;
        total = at + bytes;
        return at;
    };
    const size_t at_rows = section(sizeof(SubsetRow) * in.sub_rows.size());
    const size_t at_slots = section(sizeof(uint32_t) * (size_t)in.sub_n_slots);
    const size_t at_cnt = section(in.use_pred ? sizeof(uint32_t) * R : 0);
    const size_t at_off = section(in.use_pred ? sizeof(uint64_t) * R : 0);
    const size_t at_ent = section(in.use_pred ? sizeof(epp_prediction) * (size_t)in.n_ent : 0);
    const size_t at_ctx = section(in.use_ctx ? sizeof(int64_t) * R : 0);
    const size_t at_adm = section(sizeof(AdmitRow) * in.adm_rows.size());
    const size_t at_adm_ent = section(sizeof(uint32_t) * in.adm_ent.size());
    cudaStream_t s0 = h->slot[0].stream;
    EPP_TRY(join_streams(h));
    CUDA_TRY(h->in_dev.reserve(total, &h->dev_bytes));
    if (!in.sub_rows.empty()) {
        const size_t ns = (size_t)std::max<uint64_t>(in.sub_n_slots, 1);
        CUDA_TRY(h->sub_hits.reserve(sizeof(int32_t) * ns, &h->dev_bytes));
        CUDA_TRY(h->sub_scratch.reserve(sizeof(int32_t) * ns, &h->dev_bytes));
    }
    if (!h->in_ev) CUDA_TRY(cudaEventCreateWithFlags(&h->in_ev, cudaEventDisableTiming));
    else CUDA_TRY(cudaEventSynchronize(h->in_ev));
    CUDA_TRY(h->in_host.reserve(total));
    uint8_t *stage = h->in_host.as<uint8_t>();
    const uint8_t *dev = h->in_dev.as<uint8_t>();
    if (!in.sub_rows.empty()) {
        memcpy(stage + at_rows, in.sub_rows.data(), sizeof(SubsetRow) * in.sub_rows.size());
        uint32_t *slots = reinterpret_cast<uint32_t *>(stage + at_slots);
        for (const SubsetRow &row : in.sub_rows)
            if (row.n) memcpy(slots + row.off, in.subset->slots + in.subset->offsets[row.row], sizeof(uint32_t) * row.n);
        in.d_sub_rows = reinterpret_cast<const SubsetRow *>(dev + at_rows);
        in.d_sub_slots = reinterpret_cast<const uint32_t *>(dev + at_slots);
    }
    if (in.use_pred) {
        uint32_t *cnt = reinterpret_cast<uint32_t *>(stage + at_cnt);
        uint64_t *off = reinterpret_cast<uint64_t *>(stage + at_off);
        epp_prediction *ent = reinterpret_cast<epp_prediction *>(stage + at_ent);
        uint64_t o = 0;
        for (size_t r = 0; r < R; r++) {
            const uint32_t n = in.preds->counts[r];
            cnt[r] = n;
            off[r] = o;
            if (n) memcpy(ent + o, in.preds->entries + in.preds->offsets[r], sizeof(epp_prediction) * n);
            o += n;
        }
        in.d_cnt = reinterpret_cast<const uint32_t *>(dev + at_cnt);
        in.d_off = reinterpret_cast<const uint64_t *>(dev + at_off);
        in.d_ent = reinterpret_cast<const epp_prediction *>(dev + at_ent);
    }
    if (in.use_ctx) {
        memcpy(stage + at_ctx, in.ctx->tokens, sizeof(int64_t) * R);
        in.d_ctx = reinterpret_cast<const int64_t *>(dev + at_ctx);
    }
    if (!in.adm_rows.empty()) {
        memcpy(stage + at_adm, in.adm_rows.data(), sizeof(AdmitRow) * in.adm_rows.size());
        if (!in.adm_ent.empty()) memcpy(stage + at_adm_ent, in.adm_ent.data(), sizeof(uint32_t) * in.adm_ent.size());
        in.d_adm_rows = reinterpret_cast<const AdmitRow *>(dev + at_adm);
        in.d_adm_ent = reinterpret_cast<const uint32_t *>(dev + at_adm_ent);
    }
    CUDA_TRY(cudaMemcpyAsync(h->in_dev.p, stage, total, cudaMemcpyHostToDevice, s0));
    CUDA_TRY(cudaEventRecord(h->in_ev, s0));
    return EPP_OK;
}

// The engine's call in progress (epp_engine::cur) for the life of a scheduling call, whichever way it returns.
struct CallScope {
    epp_engine *h;
    CallScope(epp_engine *e, const CallInputs *in) : h(e) { h->cur = in; }
    ~CallScope() { h->cur = nullptr; }
};

static int32_t schedule_impl(epp_engine *h, const epp_batch *batch, epp_decision *out, epp_decision_detail *detail,
                             int32_t keep_hashes, const epp_topk_out *topk, const epp_subset *subset = nullptr,
                             const epp_predictions *preds = nullptr, bool subset_latency_ok = false,
                             const epp_context_tokens *ctx = nullptr, const epp_admission *adm = nullptr) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    if (!out) return fail(EPP_ERR_INVALID, "out is NULL");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    BatchView v;
    EPP_TRY(check_batch(h, batch, v));
    if (topk) EPP_TRY(check_topk(h, topk));
    if (h->cfg.encode_enabled && v.multimodal && !detail) return fail(EPP_ERR_INVALID, "an encode profile is configured and the batch flags multimodal requests: `detail` (which carries the encode pick) must not be NULL");
    CallInputs in;
    in.topk = topk;
    EPP_TRY(check_inputs(h, v.R, subset, subset_latency_ok, preds, ctx, adm, in));
    if (in.staged() && !h->pool_ready) return fail(EPP_ERR_STATE, "epp_pool_set has not been called");
    EPP_TRY(stage_inputs(h, in));
    h->kept_R = 0;
    const CallScope scope(h, &in);
    EPP_TRY(run_batch(h, v, Mode::Schedule, nullptr, nullptr, out, detail, nullptr, nullptr, keep_hashes != 0));
    h->stats.n_batches++;
    h->stats.n_decisions += (uint64_t)v.R;
    if (keep_hashes && v.R) {
        // the decisions stay on the device next to the hashes; host batches already have them in h->decisions
        cudaStream_t s0 = h->slot[0].stream;
        EPP_TRY(join_streams(h));
        CUDA_TRY(h->kept_dec.reserve(sizeof(epp_decision) * (size_t)v.R, &h->dev_bytes));
        const void *src = v.device ? (const void *)out : (const void *)h->decisions.p;
        CUDA_TRY(cudaMemcpyAsync(h->kept_dec.p, src, sizeof(epp_decision) * (size_t)v.R, cudaMemcpyDeviceToDevice, s0));
        if (v.device && !v.async) CUDA_TRY(cudaStreamSynchronize(s0));     // `out` is the caller's again when we return
        h->kept_R = v.R;
    }
    return EPP_OK;
}

extern "C" int32_t epp_schedule(epp_engine *h, const epp_batch *batch, epp_decision *out, epp_decision_detail *detail,
                                int32_t keep_hashes) {
    return schedule_impl(h, batch, out, detail, keep_hashes, nullptr);
}

extern "C" int32_t epp_schedule_topk(epp_engine *h, const epp_batch *batch, epp_decision *out, epp_decision_detail *detail,
                                     int32_t keep_hashes, const epp_topk_out *topk) {
    if (!topk) return fail(EPP_ERR_INVALID, "topk is NULL");
    return schedule_impl(h, batch, out, detail, keep_hashes, topk);
}

extern "C" int32_t epp_schedule_predicted(epp_engine *h, const epp_batch *batch, const epp_predictions *preds, epp_decision *out,
                                          epp_decision_detail *detail, int32_t keep_hashes, const epp_topk_out *topk) {
    return schedule_impl(h, batch, out, detail, keep_hashes, topk, nullptr, preds);
}

extern "C" int32_t epp_schedule_subset(epp_engine *h, const epp_batch *batch, const epp_subset *subset, epp_decision *out,
                                       epp_decision_detail *detail, int32_t keep_hashes, const epp_topk_out *topk) {
    if (!subset) return fail(EPP_ERR_INVALID, "subset is NULL");
    return schedule_impl(h, batch, out, detail, keep_hashes, topk, subset);
}

extern "C" int32_t epp_schedule_subset_predicted(epp_engine *h, const epp_batch *batch, const epp_subset *subset,
                                                 const epp_predictions *preds, epp_decision *out, epp_decision_detail *detail,
                                                 int32_t keep_hashes, const epp_topk_out *topk) {
    return schedule_impl(h, batch, out, detail, keep_hashes, topk, subset, preds, true);
}

extern "C" int32_t epp_schedule_ctx(epp_engine *h, const epp_batch *batch, const epp_subset *subset, const epp_predictions *preds,
                                    const epp_context_tokens *ctx, epp_decision *out, epp_decision_detail *detail,
                                    int32_t keep_hashes, const epp_topk_out *topk) {
    return schedule_impl(h, batch, out, detail, keep_hashes, topk, subset, preds, true, ctx);
}

extern "C" int32_t epp_schedule_admit(epp_engine *h, const epp_batch *batch, const epp_subset *subset, const epp_predictions *preds,
                                      const epp_context_tokens *ctx, const epp_admission *adm, epp_decision *out,
                                      epp_decision_detail *detail, int32_t keep_hashes, const epp_topk_out *topk) {
    return schedule_impl(h, batch, out, detail, keep_hashes, topk, subset, preds, true, ctx, adm);
}

// PreRequest: approximateprefix/plugin.go:164-200 (primary target + "prefill" profile target).
extern "C" int32_t epp_index_add_picked(epp_engine *h) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (h->kept_R == 0) return fail(EPP_ERR_STATE, "no batch kept (call epp_schedule with keep_hashes=1 first)");
    if (h->snapshot_mode) return fail(EPP_ERR_STATE, "index holds a bulk snapshot; incremental adds need an incrementally built index");
    EPP_TRY(flush_add_queue(h));
    auto t0 = std::chrono::steady_clock::now();
    CUDA_TRY(h->store->apply_picks(h->kept_dec.as<epp_decision>(), h->hashes.as<uint64_t>(), h->nblocks.as<int32_t>(), h->kept_R,
                                   h->cfg.max_prefix_blocks, h->slot[0].stream));
    h->stats.last_index_apply_ms = ms_since(t0);
    h->stats.last_index_items = h->store->last_items;
    h->stats.last_index_launches = (uint64_t)h->store->last_launches;
    h->kept_R = 0;
    return EPP_OK;
}

// ------------------------------------------------------------------------------------------------
// plugin-parity entry points on injected match info
// ------------------------------------------------------------------------------------------------
struct MatchRows {
    const int32_t *match, *total;
    const uint32_t *model_ids;
};

// The injected rows of a call (match [R][E], total [R], model_ids [R] or nullptr) on the device: a host call's are
// copied to engine buffers on s, a device call's are used as they are.
static int32_t match_rows(epp_engine *h, int64_t R, const int32_t *match, const int32_t *total, const uint32_t *model_ids,
                          bool dev, cudaStream_t s, MatchRows &m) {
    m = {match, total, model_ids};
    if (dev) return EPP_OK;
    const size_t n = (size_t)R * (size_t)h->cfg.max_endpoints;
    CUDA_TRY(h->dense_match.reserve(sizeof(int32_t) * n, &h->dev_bytes));
    CUDA_TRY(h->dense_total.reserve(sizeof(int32_t) * (size_t)R, &h->dev_bytes));
    CUDA_TRY(cudaMemcpyAsync(h->dense_match.p, match, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(h->dense_total.p, total, sizeof(int32_t) * (size_t)R, cudaMemcpyHostToDevice, s));
    m.match = h->dense_match.as<int32_t>();
    m.total = h->dense_total.as<int32_t>();
    if (model_ids) {
        CUDA_TRY(h->score_models.reserve(sizeof(uint32_t) * (size_t)R, &h->dev_bytes));
        CUDA_TRY(cudaMemcpyAsync(h->score_models.p, model_ids, sizeof(uint32_t) * (size_t)R, cudaMemcpyHostToDevice, s));
        m.model_ids = h->score_models.as<uint32_t>();
    }
    return EPP_OK;
}

extern "C" int32_t epp_score(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                             const uint32_t *model_ids, int32_t profile, int32_t scorer_index, double *out_scores,
                             uint32_t flags) {
    if (!h || n_requests < 0 || (n_requests && (!match || !total || !out_scores))) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (!h->pool_ready) return fail(EPP_ERR_STATE, "epp_pool_set has not been called");
    if (profile < 0 || profile >= h->n_alloc_profiles) return fail(EPP_ERR_INVALID, "profile %d out of range", profile);
    if (scorer_index < -1 || scorer_index >= profile_cfg(h, profile).n_scorers) return fail(EPP_ERR_INVALID, "scorer_index %d out of range", scorer_index);
    if (((h->lat_mask >> profile) & 1) &&
        (scorer_index < 0 || profile_cfg(h, profile).scorers[scorer_index].kind == EPP_SCORER_LATENCY ||
         profile_cfg(h, profile).scorers[scorer_index].kind == EPP_SCORER_CONTEXT_LENGTH))
        return fail(EPP_ERR_INVALID, "epp_score does not evaluate chain pieces (the weighted sum of a latency or context-length profile, the latency and context-length scorers)");
    if (n_requests == 0) return EPP_OK;
    const size_t E = (size_t)h->cfg.max_endpoints, n = (size_t)n_requests * E;
    cudaStream_t s = h->slot[0].stream;
    const bool dev = (flags & EPP_BATCH_DEVICE_PTRS) != 0;
    MatchRows m;
    EPP_TRY(match_rows(h, n_requests, match, total, model_ids, dev, s, m));
    double *d_out = out_scores;
    if (!dev) {
        CUDA_TRY(h->dense_scores.reserve(sizeof(double) * n, &h->dev_bytes));
        d_out = h->dense_scores.as<double>();
    }
    int launches = 0;
    // no-hit-lru: each request's cold bit for this profile selects its cold set (no_hit_lru.go:259-275)
    const bool nh = (h->nohit_mask >> profile) & 1;
    const ProfileDev pw = profile_dev(h, profile);
    uint8_t *cold = nullptr;
    if (nh) {
        CUDA_TRY(h->nh_cold.reserve((size_t)n_requests, &h->dev_bytes));
        cold = h->nh_cold.as<uint8_t>();
        CUDA_TRY(launch_nohit_cold_rows(n_requests, h->cfg.max_endpoints, pw.cand, m.match, cold, s, &launches));
    }
    CUDA_TRY(launch_score_dense(n_requests, h->cfg.max_endpoints, pw, nh ? profile_dev(h, profile, true) : pw, cold,
                                nh ? h->nh_col[profile].as<double>() : nullptr, pool_arrays(h),
                                h->prof[profile].qminmax.as<int64_t>(), m.match, m.total, m.model_ids, scorer_index, d_out, s,
                                &launches));
    if (!dev) CUDA_TRY(cudaMemcpyAsync(out_scores, d_out, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return EPP_OK;
}

static int32_t with_match_impl(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                               const uint32_t *model_ids, const int64_t *input_len_bytes, int32_t block_size_tokens, epp_decision *out,
                               epp_decision_detail *detail, uint32_t flags, const epp_topk_out *topk,
                               const epp_predictions *preds = nullptr, const epp_context_tokens *ctx = nullptr,
                               const epp_admission *adm = nullptr) {
    if (!h || n_requests < 0 || (n_requests && (!match || !total || !out))) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (topk) EPP_TRY(check_topk(h, topk));
    CallInputs in;
    in.topk = topk;
    EPP_TRY(check_inputs(h, n_requests, nullptr, false, preds, ctx, adm, in));
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (!h->pool_ready) return fail(EPP_ERR_STATE, "epp_pool_set has not been called");
    if (n_requests == 0) return EPP_OK;
    EPP_TRY(stage_inputs(h, in));
    const CallScope scope(h, &in);
    const size_t R = (size_t)n_requests;
    cudaStream_t s = h->slot[0].stream;
    const bool dev = (flags & EPP_BATCH_DEVICE_PTRS) != 0;
    int launches = 0;
    EPP_TRY(inflight_flush(h, s, &launches));
    DensePickParams p;
    fill_decision_fields(h, p, 0);
    p.R = n_requests;
    if (block_size_tokens > 0) p.block_size_tokens = block_size_tokens;
    p.encode_on = 0;                              // the injected-match entry point has no multimodal flags
    p.multimodal = nullptr;
    p.tie_seed = h->cfg.tie_seed;
    if (h->nohit_mask) {
        CUDA_TRY(h->nh_cold.reserve(R, &h->dev_bytes));
        p.nohit.cold_out = h->nh_cold.as<uint8_t>();
    }
    TopkRows tk;
    EPP_TRY(topk_rows(h, topk, dev, n_requests, tk));
    if (tk.on) attach_topk(h, p.gen, tk.picks, tk.scores, 0);
    if (!dev) EPP_TRY(reserve_batch(h, n_requests));
    MatchRows m;
    EPP_TRY(match_rows(h, n_requests, match, total, model_ids, dev, s, m));
    p.match = m.match;
    p.total = m.total;
    p.model_ids = m.model_ids;
    if (dev) {
        p.in_len = input_len_bytes; p.out = out; p.detail = detail;
    } else {
        if (input_len_bytes) CUDA_TRY(cudaMemcpyAsync(h->in_len.p, input_len_bytes, sizeof(int64_t) * R, cudaMemcpyHostToDevice, s));
        else CUDA_TRY(cudaMemsetAsync(h->in_len.p, 0, sizeof(int64_t) * R, s));
        p.in_len = h->in_len.as<int64_t>();
        p.out = h->decisions.as<epp_decision>();
        p.detail = h->details.as<epp_decision_detail>();
    }
    if (h->lat_mask) {
        CUDA_TRY(launch_dense_pick_lat(p, lat_view(h, 0), s, &launches));
    } else {
        CUDA_TRY(launch_dense_pick(p, s, &launches));
    }
    EPP_TRY(launch_admission(h, 0, n_requests, p.out, p.detail, tk, s, &launches, false));
    EPP_TRY(after_picks(h, p.out, p.detail, p.in_len, n_requests, s, &launches, false));
    if (!dev) {
        CUDA_TRY(cudaMemcpyAsync(out, p.out, sizeof(epp_decision) * R, cudaMemcpyDeviceToHost, s));
        if (detail) CUDA_TRY(cudaMemcpyAsync(detail, p.detail, sizeof(epp_decision_detail) * R, cudaMemcpyDeviceToHost, s));
        if (tk.on) EPP_TRY(topk_copy_back(h, tk, 0, n_requests, s));
    }
    CUDA_TRY(cudaStreamSynchronize(s));
    h->kept_R = 0;
    h->stats.n_decisions += (uint64_t)n_requests;          // request ordinals (tie rule) advance here too
    return EPP_OK;
}

extern "C" int32_t epp_schedule_with_match(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                           const uint32_t *model_ids, const int64_t *input_len_bytes, int32_t block_size_tokens, epp_decision *out,
                                           epp_decision_detail *detail, uint32_t flags) {
    return with_match_impl(h, n_requests, match, total, model_ids, input_len_bytes, block_size_tokens, out, detail, flags, nullptr);
}

extern "C" int32_t epp_schedule_with_match_predicted(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                                     const uint32_t *model_ids, const int64_t *input_len_bytes,
                                                     int32_t block_size_tokens, epp_decision *out, epp_decision_detail *detail,
                                                     uint32_t flags, const epp_topk_out *topk, const epp_predictions *preds) {
    return with_match_impl(h, n_requests, match, total, model_ids, input_len_bytes, block_size_tokens, out, detail, flags, topk, preds);
}

extern "C" int32_t epp_schedule_with_match_ctx(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                               const uint32_t *model_ids, const int64_t *input_len_bytes,
                                               int32_t block_size_tokens, epp_decision *out, epp_decision_detail *detail,
                                               uint32_t flags, const epp_topk_out *topk, const epp_predictions *preds,
                                               const epp_context_tokens *ctx) {
    return with_match_impl(h, n_requests, match, total, model_ids, input_len_bytes, block_size_tokens, out, detail, flags, topk,
                           preds, ctx);
}

extern "C" int32_t epp_schedule_with_match_admit(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                                 const uint32_t *model_ids, const int64_t *input_len_bytes,
                                                 int32_t block_size_tokens, epp_decision *out, epp_decision_detail *detail,
                                                 uint32_t flags, const epp_topk_out *topk, const epp_predictions *preds,
                                                 const epp_context_tokens *ctx, const epp_admission *adm) {
    return with_match_impl(h, n_requests, match, total, model_ids, input_len_bytes, block_size_tokens, out, detail, flags, topk,
                           preds, ctx, adm);
}

extern "C" int32_t epp_schedule_with_match_topk(epp_engine *h, int64_t n_requests, const int32_t *match, const int32_t *total,
                                                const uint32_t *model_ids, const int64_t *input_len_bytes, int32_t block_size_tokens,
                                                epp_decision *out, epp_decision_detail *detail, uint32_t flags,
                                                const epp_topk_out *topk) {
    if (!topk) return fail(EPP_ERR_INVALID, "topk is NULL");
    return with_match_impl(h, n_requests, match, total, model_ids, input_len_bytes, block_size_tokens, out, detail, flags, topk);
}

extern "C" int32_t epp_nohit_lru_get(epp_engine *h, uint32_t *out_eps, int32_t cap, int32_t *out_n) {
    if (!h || !out_n || cap < 0 || (cap > 0 && !out_eps)) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    if (!h->nohit_mask) return fail(EPP_ERR_STATE, "no profile has the no-hit-lru scorer");
    EPP_TRY(finish_async(h));
    const size_t E = (size_t)h->cfg.max_endpoints;
    std::vector<uint64_t> seq(E);
    CUDA_TRY(cudaMemcpy(seq.data(), h->nh_last_seq.p, sizeof(uint64_t) * E, cudaMemcpyDeviceToHost));
    std::vector<std::pair<uint64_t, uint32_t>> m;
    for (size_t e = 0; e < E; e++) if (seq[e]) m.push_back({seq[e], (uint32_t)e});
    std::sort(m.begin(), m.end());
    *out_n = (int32_t)m.size();
    for (int32_t i = 0; i < std::min<int32_t>(cap, (int32_t)m.size()); i++) out_eps[i] = m[(size_t)i].second;
    return EPP_OK;
}

// The producer's token estimate of a prompt of L bytes (the device copy is inflight_est in inflight.cu).
static int64_t inflight_est_host(int64_t L) {
    const int64_t i = L < 8 ? 1 : L / 4;
    return 2 * i + (i + 1) / 2;
}

extern "C" int32_t epp_inflight_release(epp_engine *h, int32_t n, const uint32_t *eps, const uint64_t *prompt_lens) {
    if (!h || n < 0 || (n > 0 && (!eps || !prompt_lens))) return fail(EPP_ERR_INVALID, "bad arguments");
    if (!h->inflight) return fail(EPP_ERR_STATE, "the engine was created without inflight_load");
    for (int32_t i = 0; i < n; i++)
        if (eps[i] != EPP_NO_ENDPOINT && eps[i] >= (uint32_t)h->cfg.max_endpoints)
            return fail(EPP_ERR_INVALID, "entry %d: slot id %u >= max_endpoints %d", i, eps[i], h->cfg.max_endpoints);
    std::lock_guard<std::mutex> lk(h->if_mu);
    for (int32_t i = 0; i < n; i++) {
        if (eps[i] == EPP_NO_ENDPOINT) continue;
        InflightDelta &d = h->if_pending.try_emplace(eps[i], InflightDelta{eps[i], 0, 0, 0}).first->second;
        d.req -= 1;
        d.tok -= inflight_est_host((int64_t)std::min<uint64_t>(prompt_lens[i], (uint64_t)INT64_MAX));
    }
    return EPP_OK;
}

extern "C" int32_t epp_inflight_reset(epp_engine *h, int32_t n, const uint32_t *ids) {
    if (!h || n < 0 || (n > 0 && !ids)) return fail(EPP_ERR_INVALID, "bad arguments");
    if (!h->inflight) return fail(EPP_ERR_STATE, "the engine was created without inflight_load");
    for (int32_t i = 0; i < n; i++)
        if (ids[i] >= (uint32_t)h->cfg.max_endpoints)
            return fail(EPP_ERR_INVALID, "entry %d: slot id %u >= max_endpoints %d", i, ids[i], h->cfg.max_endpoints);
    std::lock_guard<std::mutex> lk(h->if_mu);
    for (int32_t i = 0; i < n; i++) h->if_pending[ids[i]] = InflightDelta{ids[i], 1, 0, 0};   // drops earlier pending releases
    return EPP_OK;
}

extern "C" int32_t epp_inflight_get(epp_engine *h, int32_t cap, int64_t *out_requests, int64_t *out_tokens) {
    if (!h || cap < 0 || (cap > 0 && (!out_requests || !out_tokens))) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (!h->inflight) return fail(EPP_ERR_STATE, "the engine was created without inflight_load");
    EPP_TRY(set_device(h));
    EPP_TRY(finish_async(h));
    cudaStream_t s = h->slot[0].stream;
    int launches = 0;
    EPP_TRY(inflight_flush(h, s, &launches));
    const size_t n = (size_t)std::min<int32_t>(cap, h->cfg.max_endpoints);
    if (n) {
        CUDA_TRY(cudaMemcpyAsync(out_requests, h->if_req.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaMemcpyAsync(out_tokens, h->if_tok.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, s));
    }
    CUDA_TRY(cudaStreamSynchronize(s));
    return EPP_OK;
}

extern "C" int32_t epp_get_config(epp_engine *h, epp_config *out) {
    if (!h || !out) return fail(EPP_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(h->mu);
    *out = h->cfg_user;
    return EPP_OK;
}

extern "C" int32_t epp_get_stats(epp_engine *h, epp_stats *out) {
    if (!h || !out) return fail(EPP_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->async_pending) { EPP_TRY(set_device(h)); EPP_TRY(finish_async(h)); }
    if (h->small_stats_pending) {
        EPP_TRY(set_device(h));
        float t = 0;
        CUDA_TRY(cudaEventSynchronize(h->ev[1]));
        cudaEventElapsedTime(&t, h->ev[0], h->ev[1]);
        h->stats.last_kernels_ms = t;
        for (int i = 0; i < 8; i++) h->stats.last_kernel_ms[i] = i == 0 ? t : 0.0;
        h->small_stats_pending = false;
    }
    h->stats.device_bytes = h->dev_bytes + h->store->device_bytes();
    *out = h->stats;
    return EPP_OK;
}

extern "C" int32_t epp_synchronize(epp_engine *h) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL engine");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    EPP_TRY(finish_async(h));
    CUDA_TRY(cudaStreamSynchronize(h->slot[1].stream));
    return EPP_OK;
}

extern "C" int32_t epp_event_record(epp_engine *h, int32_t which) {
    if (!h || which < 0 || which > 1) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    CUDA_TRY(cudaEventRecord(h->user_ev[which], h->slot[0].stream));
    return EPP_OK;
}

extern "C" int32_t epp_event_elapsed_ms(epp_engine *h, double *out_ms) {
    if (!h || !out_ms) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    CUDA_TRY(cudaEventSynchronize(h->user_ev[1]));
    float ms = 0;
    CUDA_TRY(cudaEventElapsedTime(&ms, h->user_ev[0], h->user_ev[1]));
    *out_ms = ms;
    return EPP_OK;
}

// ------------------------------------------------------------------------------------------------
// endpoint-sharded mode (kernels: pick_kernels.cu k_shard_*, shard_p2p.cu)
// ------------------------------------------------------------------------------------------------
// Per-call state that no rank can keep from its own shard alone.
static int32_t check_shardable(const epp_engine *h) {
    if (h->lat_mask) return fail(EPP_ERR_INVALID, "endpoint-sharded mode does not support latency profiles");
    if (h->nohit_mask) return fail(EPP_ERR_INVALID, "endpoint-sharded mode does not support the no-hit-lru scorer (coldness needs every rank's match)");
    if (any_random_picker(h)) return fail(EPP_ERR_INVALID, "endpoint-sharded mode does not support the random pickers (a weighted draw needs every rank's scores)");
    if (h->inflight) return fail(EPP_ERR_INVALID, "endpoint-sharded mode does not support the inflight-load producer");
    if (h->adm_on) return fail(EPP_ERR_INVALID, "endpoint-sharded mode does not support the admitters");
    return EPP_OK;
}

// epp_shard_set (staged == false: the single-profile handler only), epp_shard_set_staged and (seeded)
// epp_shard_set_seeded.
static int32_t shard_set(epp_engine *h, uint32_t ep_begin, uint32_t ep_end, bool staged, int32_t *out_stages,
                         bool seeded = false) {
    if (!h || ep_begin > ep_end) return fail(EPP_ERR_INVALID, "bad shard range");
    std::lock_guard<std::mutex> lk(h->mu);
    if (seeded && h->cfg.tie_seed == 0) return fail(EPP_ERR_INVALID, "epp_shard_set_seeded needs epp_config.tie_seed != 0");
    if (!staged && h->cfg.handler != EPP_HANDLER_SINGLE) return fail(EPP_ERR_INVALID, "endpoint-sharded mode supports the single-profile handler only");
    if (h->general) return fail(EPP_ERR_INVALID, "endpoint-sharded mode supports neither pick_k > 1 nor the prefix-cache-affinity-filter (both need every candidate's score on one rank)");
    EPP_TRY(check_shardable(h));
    // the kernels write handler_stages records (kernels.h); the same count from the configuration
    const int32_t stages = h->cfg.encode_enabled ? 3 : h->n_profiles;
    if (h->p2p_buf && h->p2p_stages != stages)
        return fail(EPP_ERR_STATE, "the exchange buffer was exported for %d record(s) per request, this handler needs %d: call epp_shard_set_staged before epp_shard_p2p_export", (int)h->p2p_stages, (int)stages);
    if (h->p2p_buf && h->p2p_seeded != seeded)
        return fail(EPP_ERR_STATE, "the exchange buffer was exported for the %s tie rule: set the rule before epp_shard_p2p_export",
                    h->p2p_seeded ? "seeded" : "lowest-slot");
    h->shard_begin = ep_begin;
    h->shard_end = ep_end;
    h->shard_stages = stages;
    h->shard_seeded = seeded;
    h->pool_ready = false;          // candidates are derived per shard: epp_pool_set must follow
    if (out_stages) *out_stages = stages;
    return EPP_OK;
}

extern "C" int32_t epp_shard_set(epp_engine *h, uint32_t ep_begin, uint32_t ep_end) {
    return shard_set(h, ep_begin, ep_end, false, nullptr);
}
extern "C" int32_t epp_shard_set_staged(epp_engine *h, uint32_t ep_begin, uint32_t ep_end, int32_t *out_stages) {
    if (!out_stages) return fail(EPP_ERR_INVALID, "NULL argument");
    return shard_set(h, ep_begin, ep_end, true, out_stages);
}
extern "C" int32_t epp_shard_set_seeded(epp_engine *h, uint32_t ep_begin, uint32_t ep_end, int32_t *out_stages) {
    if (!out_stages) return fail(EPP_ERR_INVALID, "NULL argument");
    return shard_set(h, ep_begin, ep_end, true, out_stages, true);
}

static int32_t mask_words_of(const epp_engine *h) { return (h->cfg.max_prefix_blocks + 31) / 32; }

extern "C" int32_t epp_shard_probe(epp_engine *h, const epp_batch *batch, uint32_t *out_masks) {
    if (!h || !out_masks) return fail(EPP_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    BatchView v;
    EPP_TRY(check_batch(h, batch, v));
    if (!v.device) return fail(EPP_ERR_INVALID, "epp_shard_probe takes device-pointer batches (EPP_BATCH_DEVICE_PTRS)");
    h->kept_R = 0;
    h->shard_R = 0;
    h->shard_models = false;
    h->shard_mm = false;
    h->shard_picked = false;
    EPP_TRY(commit_locked(h));
    EPP_TRY(run_batch(h, v, Mode::HashOnly, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr));
    int launches = 0;
    cudaStream_t s = h->slot[0].stream;
    // the pick (a later call) scores lora-affinity with the batch's adapters: keep a copy, the caller's ids may be gone.
    // Likewise the multimodal flags (encode stage); the request lengths (P/D decider) stay in `in_len` from the hashing.
    if (v.model_ids && v.R)
        CUDA_TRY(cudaMemcpyAsync(h->model_ids.p, v.model_ids, sizeof(uint32_t) * (size_t)v.R, cudaMemcpyDeviceToDevice, s));
    if (v.multimodal && v.R) {
        CUDA_TRY(h->multimodal.reserve((size_t)v.R, &h->dev_bytes));
        CUDA_TRY(cudaMemcpyAsync(h->multimodal.p, v.multimodal, (size_t)v.R, cudaMemcpyDeviceToDevice, s));
    }
    CUDA_TRY(launch_shard_probe(v.R, h->cfg.max_prefix_blocks, h->hashes.as<uint64_t>(), h->nblocks.as<int32_t>(),
                                index_view(h), out_masks, mask_words_of(h), s, &launches));
    CUDA_TRY(cudaStreamSynchronize(s));
    h->shard_R = v.R;
    h->shard_models = v.model_ids != nullptr;
    h->shard_mm = v.multimodal != nullptr;
    return EPP_OK;
}

// The merge of rows [r0, r0 + R) of the batch in progress, whose lengths are in_len[r0 ..] and flags multimodal (absolute
// rows, or nullptr).
static ShardMergeParams shard_merge_params(epp_engine *h, int64_t r0, int64_t R, int32_t n_ranks, const epp_shard_best *all_best,
                                           const uint8_t *multimodal, epp_decision *out, epp_decision_detail *detail) {
    ShardMergeParams p;
    p.R = R;
    p.n_ranks = n_ranks;
    p.stages = h->shard_stages;
    p.all_best = all_best;
    p.nblocks = h->nblocks.as<int32_t>() + r0;
    p.out = out;
    p.detail = detail;
    p.always_disagg = h->cfg.always_disagg;
    p.block_size_tokens = h->cfg.block_size_tokens;
    p.non_cached_tokens = h->cfg.non_cached_tokens;
    p.in_len = h->in_len.as<int64_t>() + r0;
    p.multimodal = multimodal ? multimodal + r0 : nullptr;
    return p;
}

// Only the detail carries the encode pick (the rule of epp_schedule).
static int32_t check_encode_detail(const epp_engine *h, bool multimodal, const epp_decision_detail *detail) {
    if (h->cfg.encode_enabled && multimodal && !detail)
        return fail(EPP_ERR_INVALID, "an encode profile is configured and the batch flags multimodal requests: `out_detail` (which carries the encode pick) must not be NULL");
    return EPP_OK;
}

extern "C" int32_t epp_shard_pick(epp_engine *h, int64_t n_requests, const uint32_t *global_masks, epp_shard_best *out_best) {
    if (!h || !global_masks || !out_best) return fail(EPP_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (!h->pool_ready) return fail(EPP_ERR_STATE, "epp_pool_set has not been called (after epp_shard_set)");
    if (n_requests != h->shard_R) return fail(EPP_ERR_STATE, "epp_shard_pick: n_requests %lld does not match the probed batch (%lld)", (long long)n_requests, (long long)h->shard_R);
    if (n_requests == 0) return EPP_OK;
    Work w{0, n_requests, nullptr, nullptr, nullptr, 0, h->shard_models ? h->model_ids.as<uint32_t>() : nullptr, 0,
           h->hashes.as<uint64_t>(), h->nblocks.as<int32_t>(), h->shard_mm ? h->multimodal.as<uint8_t>() : nullptr};
    PickParams pp = pick_params(h, w, h->decisions.as<epp_decision>(), nullptr, nullptr);
    pp.global_masks = global_masks;
    pp.mask_words = mask_words_of(h);
    pp.shard_out = out_best;
    int launches = 0;
    cudaStream_t s = h->slot[0].stream;
    EPP_TRY(reserve_batch(h, n_requests));
    EPP_TRY(launch_match(h, h->slot[0], pp, &launches));
    if (h->shard_seeded) {          // epp_shard_select walks the same prompts again: keep the OR of the masks
        const size_t bytes = sizeof(uint32_t) * (size_t)n_requests * (size_t)pp.mask_words;
        CUDA_TRY(h->sel_gmasks.reserve(bytes, &h->dev_bytes));
        CUDA_TRY(cudaMemcpyAsync(h->sel_gmasks.p, global_masks, bytes, cudaMemcpyDeviceToDevice, s));
    }
    CUDA_TRY(cudaStreamSynchronize(s));
    h->shard_picked = true;
    return EPP_OK;
}

extern "C" int32_t epp_shard_merge_detail(epp_engine *h, int64_t n_requests, int32_t n_ranks, const epp_shard_best *all_best,
                                          epp_decision *out, epp_decision_detail *out_detail) {
    if (!h || !all_best || !out || n_ranks <= 0) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (h->shard_seeded) return fail(EPP_ERR_STATE, "the engine was set with epp_shard_set_seeded: epp_shard_select and epp_shard_finish replace epp_shard_merge");
    if (n_requests != h->shard_R) return fail(EPP_ERR_STATE, "epp_shard_merge: n_requests does not match the probed batch");
    EPP_TRY(check_encode_detail(h, h->shard_mm, out_detail));
    int launches = 0;
    cudaStream_t s = h->slot[0].stream;
    CUDA_TRY(launch_shard_merge(shard_merge_params(h, 0, n_requests, n_ranks, all_best,
                                                   h->shard_mm ? h->multimodal.as<uint8_t>() : nullptr, out, out_detail),
                                s, &launches));
    CUDA_TRY(cudaStreamSynchronize(s));
    return EPP_OK;
}
extern "C" int32_t epp_shard_merge(epp_engine *h, int64_t n_requests, int32_t n_ranks, const epp_shard_best *all_best, epp_decision *out) {
    return epp_shard_merge_detail(h, n_requests, n_ranks, all_best, out, nullptr);
}

// ---- seeded ties (include/epp_engine.h, "Seeded ties") ------------------------------------------------------------
static ShardSeedParams shard_seed_params(const epp_engine *h, int64_t r0) {
    ShardSeedParams sp;
    memset(&sp, 0, sizeof sp);
    sp.tie_seed = h->cfg.tie_seed;
    sp.tie_base = h->stats.n_decisions + (uint64_t)r0;
    sp.ep_begin = h->shard_begin;
    sp.ep_end = h->shard_end;
    return sp;
}

static int32_t reserve_select(epp_engine *h, int64_t R) {
    const size_t n = (size_t)std::max<int64_t>(R, 1) * (size_t)h->shard_stages;
    CUDA_TRY(h->sel_work.reserve(sizeof(uint2) * n, &h->dev_bytes));
    CUDA_TRY(h->sel_dense.reserve(sizeof(int32_t) * n, &h->dev_bytes));
    return EPP_OK;
}

// Resolve rows [r0, r0 + mp.R) over the gathered records and select the members this rank owns: k_shard_resolve, the
// sparse select, the dense-counter select over its overflows.  pp: the rows' match launch (global masks set); own_sel:
// this rank's [R][S] entries of the rows.  Work items at sel_work[r0 * S ..], counters in the slot's overflow_n[2], [3].
static int32_t launch_select(epp_engine *h, Slot &sl, const ShardMergeParams &mp, const PickParams &pp, int64_t r0,
                             epp_shard_sel *own_sel, int *launches) {
    cudaStream_t s = sl.stream;
    const size_t at = (size_t)r0 * (size_t)h->shard_stages;
    int32_t *counts = sl.overflow_n.as<int32_t>() + 2;
    CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(int32_t) * 2, s));
    ShardSeedParams sp = shard_seed_params(h, r0);
    sp.sel = own_sel;
    sp.work = h->sel_work.as<uint2>() + at;
    sp.work_n = counts;
    CUDA_TRY(launch_shard_resolve(mp, sp, s, launches));
    ShardSelView sv;
    sv.work = sp.work;
    sv.work_n = counts;
    sv.stages = h->shard_stages;
    sv.sel = own_sel;
    sv.dense_list = h->sel_dense.as<int32_t>() + at;
    sv.dense_n = counts + 1;
    CUDA_TRY(launch_match_pick_sparse_select(pp, sv, h->sm_count, s, launches));
    CUDA_TRY(launch_match_pick_select(pp, sv, h->pick_global ? sl.pick_scratch.as<uint32_t>() : nullptr, h->pick_grid,
                                      h->pick_smem, s, launches));
    return EPP_OK;
}

extern "C" int32_t epp_shard_select(epp_engine *h, int64_t n_requests, int32_t n_ranks, const epp_shard_best *all_best,
                                    epp_shard_sel *out_sel) {
    if (!h || !all_best || !out_sel || n_ranks <= 0) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (!h->shard_seeded) return fail(EPP_ERR_STATE, "epp_shard_select needs an engine set with epp_shard_set_seeded");
    if (!h->pool_ready) return fail(EPP_ERR_STATE, "epp_pool_set has not been called (after epp_shard_set_seeded)");
    if (n_requests != h->shard_R || (n_requests && !h->shard_picked))
        return fail(EPP_ERR_STATE, "epp_shard_select: n_requests %lld does not match the picked batch", (long long)n_requests);
    if (n_requests == 0) return EPP_OK;
    Work w{0, n_requests, nullptr, nullptr, nullptr, 0, h->shard_models ? h->model_ids.as<uint32_t>() : nullptr, 0,
           h->hashes.as<uint64_t>(), h->nblocks.as<int32_t>(), h->shard_mm ? h->multimodal.as<uint8_t>() : nullptr};
    PickParams pp = pick_params(h, w, h->decisions.as<epp_decision>(), nullptr, nullptr);
    pp.global_masks = h->sel_gmasks.as<uint32_t>();
    pp.mask_words = mask_words_of(h);
    EPP_TRY(reserve_select(h, n_requests));
    int launches = 0;
    cudaStream_t s = h->slot[0].stream;
    EPP_TRY(launch_select(h, h->slot[0], shard_merge_params(h, 0, n_requests, n_ranks, all_best, nullptr, nullptr, nullptr),
                          pp, 0, out_sel, &launches));
    CUDA_TRY(cudaStreamSynchronize(s));
    return EPP_OK;
}

extern "C" int32_t epp_shard_finish(epp_engine *h, int64_t n_requests, int32_t n_ranks, const epp_shard_best *all_best,
                                    const epp_shard_sel *all_sel, epp_decision *out, epp_decision_detail *out_detail) {
    if (!h || !all_best || !all_sel || !out || n_ranks <= 0) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (!h->shard_seeded) return fail(EPP_ERR_STATE, "epp_shard_finish needs an engine set with epp_shard_set_seeded");
    if (n_requests != h->shard_R) return fail(EPP_ERR_STATE, "epp_shard_finish: n_requests does not match the probed batch");
    EPP_TRY(check_encode_detail(h, h->shard_mm, out_detail));
    int launches = 0;
    cudaStream_t s = h->slot[0].stream;
    ShardSeedParams sp = shard_seed_params(h, 0);
    sp.all_sel = all_sel;
    CUDA_TRY(launch_shard_finish(shard_merge_params(h, 0, n_requests, n_ranks, all_best,
                                                    h->shard_mm ? h->multimodal.as<uint8_t>() : nullptr, out, out_detail),
                                 sp, s, &launches));
    CUDA_TRY(cudaStreamSynchronize(s));
    h->stats.n_batches++;
    h->stats.n_decisions += (uint64_t)n_requests;    // the next batch's ordinals follow this one's
    return EPP_OK;
}

// ---- endpoint-sharded mode with the exchanges over NVLink peer memory (shard_p2p.cu) ------------------------------
// flags of chunk c of a batch: flag 1 at c * 256, flag 2 at c * 256 + 128, and with the seeded tie rule flag 3 at
// c * 256 + 64 (two chunks: the halves of a batch travel through the exchange on the engine's two streams, so that a rank
// computes on one half while it waits for its peers on the other)
static constexpr size_t kP2pFlag1 = 0, kP2pFlag2 = 128, kP2pFlag3 = 64, kP2pChunkFlags = 256, kP2pChunks = 2,
                        kP2pHeader = kP2pChunkFlags * kP2pChunks;

extern "C" int32_t epp_shard_p2p_export(epp_engine *h, int64_t max_requests, uint8_t *out_handle, uint64_t *out_ptr) {
    if (!h || max_requests <= 0 || !out_handle || !out_ptr) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (h->p2p_buf && !h->p2p_broken) return fail(EPP_ERR_STATE, "the exchange buffer is already exported");
    if (h->p2p_buf) {                                           // broken exchange: start over with a fresh buffer
        for (int g = 0; g < (int)h->p2p_peer.size(); g++)
            if (h->p2p_ipc && g != h->p2p_rank && h->p2p_peer[g]) cudaIpcCloseMemHandle(h->p2p_peer[g]);
        h->p2p_peer.clear();
        cudaFree(h->p2p_buf);
        h->dev_bytes -= h->p2p_bytes;
        h->p2p_buf = nullptr;
        h->p2p_broken = false;
        h->p2p_epoch = 0;
    }
    const size_t W = (size_t)mask_words_of(h);
    h->p2p_masks_off = kP2pHeader;
    h->p2p_best_off = (kP2pHeader + (size_t)max_requests * W * sizeof(uint32_t) + 255) & ~(size_t)255;
    h->p2p_bytes = (h->p2p_best_off + (size_t)max_requests * (size_t)h->shard_stages * sizeof(epp_shard_best) + 255) & ~(size_t)255;
    h->p2p_seeded = h->shard_seeded;
    h->p2p_sel_off = h->p2p_bytes;                              // seeded: the selected entries follow the records
    if (h->p2p_seeded) h->p2p_bytes += ((size_t)max_requests * (size_t)h->shard_stages * sizeof(epp_shard_sel) + 255) & ~(size_t)255;
    CUDA_TRY(cudaMalloc(&h->p2p_buf, h->p2p_bytes));
    CUDA_TRY(cudaMemset(h->p2p_buf, 0, h->p2p_bytes));
    h->dev_bytes += h->p2p_bytes;
    h->p2p_R = max_requests;
    h->p2p_stages = h->shard_stages;
    cudaIpcMemHandle_t hd;
    CUDA_TRY(cudaIpcGetMemHandle(&hd, h->p2p_buf));
    static_assert(sizeof(hd) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(out_handle, &hd, sizeof hd);
    *out_ptr = (uint64_t)(uintptr_t)h->p2p_buf;
    return EPP_OK;
}

extern "C" int32_t epp_shard_p2p_connect(epp_engine *h, int32_t n_ranks, int32_t rank, const void *peers, int32_t ipc_handles) {
    if (!h || n_ranks <= 0 || n_ranks > 64 || rank < 0 || rank >= n_ranks || !peers) return fail(EPP_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    EPP_TRY(check_shardable(h));
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (!h->p2p_buf) return fail(EPP_ERR_STATE, "epp_shard_p2p_export has not been called");
    if (!h->p2p_peer.empty()) return fail(EPP_ERR_STATE, "peers are already connected");
    h->p2p_peer.assign((size_t)n_ranks, nullptr);
    h->p2p_ipc = ipc_handles != 0;
    for (int g = 0; g < n_ranks; g++) {
        if (g == rank) { h->p2p_peer[g] = h->p2p_buf; continue; }
        if (ipc_handles) {
            cudaIpcMemHandle_t hd;
            memcpy(&hd, static_cast<const uint8_t *>(peers) + (size_t)g * 64, sizeof hd);
            CUDA_TRY(cudaIpcOpenMemHandle(&h->p2p_peer[g], hd, cudaIpcMemLazyEnablePeerAccess));
        } else {
            h->p2p_peer[g] = (void *)(uintptr_t)static_cast<const uint64_t *>(peers)[g];    // same process: plain pointers
        }
    }
    h->p2p_ranks = n_ranks;
    h->p2p_rank = rank;
    CUDA_TRY(h->p2p_peer_dev.reserve(sizeof(void *) * (size_t)n_ranks, &h->dev_bytes));
    CUDA_TRY(cudaMemcpy(h->p2p_peer_dev.p, h->p2p_peer.data(), sizeof(void *) * (size_t)n_ranks, cudaMemcpyHostToDevice));
    CUDA_TRY(h->p2p_err.reserve(sizeof(int), &h->dev_bytes));
    CUDA_TRY(cudaMemset(h->p2p_err.p, 0, sizeof(int)));
    // everything the batches need is allocated now: no cudaMalloc / cudaFree (device-wide synchronisation) may happen
    // while a peer-wait kernel is spinning
    const size_t W = (size_t)mask_words_of(h);
    CUDA_TRY(h->p2p_gmasks.reserve(((size_t)h->p2p_R * W * sizeof(uint32_t) + 15) & ~(size_t)15, &h->dev_bytes));
    CUDA_TRY(h->p2p_allbest.reserve(sizeof(epp_shard_best) * (size_t)h->p2p_R * (size_t)h->p2p_stages * (size_t)n_ranks,
                                     &h->dev_bytes));
    if (h->p2p_seeded) {
        CUDA_TRY(h->p2p_allsel.reserve(sizeof(epp_shard_sel) * (size_t)h->p2p_R * (size_t)h->p2p_stages * (size_t)n_ranks,
                                        &h->dev_bytes));
        EPP_TRY(reserve_select(h, h->p2p_R));
    }
    EPP_TRY(reserve_batch(h, h->p2p_R));
    return EPP_OK;
}

// One batch of the sharded protocol with both exchanges done by this rank's own kernels over peer memory.  Every rank
// calls it with the same batch; the decisions (identical on every rank) land in `out` (device pointer).
// The protocol is three phases (four with the seeded tie rule); epp_shard_schedule_p2p runs them back to back (the waits happen ON THE DEVICE, the host
// only waits at the end), epp_shard_p2p_phase runs ONE phase and synchronises, so that ranks which share a GPU -- whose
// spin-wait kernels could starve each other -- can be stepped phase by phase from one host thread (tests, small setups).
static constexpr unsigned long long kP2pPoison = ~0ull;

static unsigned long long p2p_timeout_ns() {
    unsigned long long timeout_ns = 20ull * 1000 * 1000 * 1000;
    if (const char *tv = getenv("EPP_P2P_TIMEOUT_MS")) timeout_ns = (unsigned long long)std::max(1, atoi(tv)) * 1000ull * 1000ull;
    return timeout_ns;
}

// A wait that timed out (or met a poisoned flag) leaves the ranks out of step for good: the exchange is marked broken,
// this rank's flags are poisoned so that the peers fail too instead of reading half-written buffers, and every later
// call fails until the buffers are exported / connected again.
static int32_t p2p_check(epp_engine *h, cudaStream_t s, unsigned long long epoch) {
    int err = 0;
    CUDA_TRY(cudaMemcpyAsync(&err, h->p2p_err.p, sizeof err, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    if (!err) return EPP_OK;
    h->p2p_broken = true;
    uint8_t *own = static_cast<uint8_t *>(h->p2p_buf);
    for (size_t c = 0; c < kP2pChunks; c++) {
        CUDA_TRY(launch_p2p_signal(reinterpret_cast<unsigned long long *>(own + c * kP2pChunkFlags + kP2pFlag1), kP2pPoison, s));
        CUDA_TRY(launch_p2p_signal(reinterpret_cast<unsigned long long *>(own + c * kP2pChunkFlags + kP2pFlag2), kP2pPoison, s));
        CUDA_TRY(launch_p2p_signal(reinterpret_cast<unsigned long long *>(own + c * kP2pChunkFlags + kP2pFlag3), kP2pPoison, s));
    }
    CUDA_TRY(cudaMemsetAsync(h->p2p_err.p, 0, sizeof(int), s));
    CUDA_TRY(cudaStreamSynchronize(s));
    const bool poisoned = err > 64;
    return fail(EPP_ERR_NCCL, poisoned ? "peer rank %d reported a broken sharded exchange (batch %llu); re-export and re-connect the exchange buffers"
                                       : "peer rank %d did not reach batch %llu of the sharded exchange within %llu ms; the exchange is broken until the buffers are exported and connected again",
                (poisoned ? err - 64 : err) - 1, epoch, p2p_timeout_ns() / 1000000ull);
}

// One phase of the exchange for rows [r0, r1) of the batch (chunk c: its own flag words, stream of slot c).  Phase 0
// expects ++p2p_epoch and the commit to have happened; the caller checks p2p_err after the last phase of every chunk.
static int32_t p2p_phase_rows(epp_engine *h, const BatchView &v, epp_decision *out, epp_decision_detail *detail, int phase,
                              int c, int64_t r0, int64_t r1, uint64_t or_bits) {
    const int64_t R = r1 - r0;
    const int n = h->p2p_ranks;
    const size_t S = (size_t)h->p2p_stages;
    const size_t W = (size_t)mask_words_of(h);
    Slot &sl = h->slot[c];
    cudaStream_t s = sl.stream;
    uint8_t *own = static_cast<uint8_t *>(h->p2p_buf);
    unsigned char *const *peers = h->p2p_peer_dev.as<unsigned char *>();
    const size_t flag1 = (size_t)c * kP2pChunkFlags + kP2pFlag1, flag2 = (size_t)c * kP2pChunkFlags + kP2pFlag2;
    const size_t mask_off = h->p2p_masks_off + (size_t)r0 * W * sizeof(uint32_t);
    const size_t mask_bytes = ((size_t)R * W * sizeof(uint32_t) + 15) & ~(size_t)15;
    const size_t best_off = h->p2p_best_off + (size_t)r0 * S * sizeof(epp_shard_best);
    const unsigned long long timeout_ns = p2p_timeout_ns();
    const unsigned long long epoch = h->p2p_epoch;
    const Work w = device_work(h, v, r0, r1, or_bits);
    uint32_t *gmasks = h->p2p_gmasks.as<uint32_t>() + (size_t)r0 * W;
    epp_shard_best *allbest = h->p2p_allbest.as<epp_shard_best>() + (size_t)r0 * (size_t)n * S;   // this chunk's own [n][R][S] records
    int launches = 0;
    if (phase == 0) {
        // hashes + local presence masks -> own exchange buffer, raise flag 1
        CUDA_TRY(launch_hash_prompts(hash_params(h, w, sl), s, &launches));
        CUDA_TRY(launch_shard_probe(R, h->cfg.max_prefix_blocks, w.hashes_out, w.nblocks_out, index_view(h),
                                    reinterpret_cast<uint32_t *>(own + mask_off), (int32_t)W, s, &launches));
        CUDA_TRY(launch_p2p_signal(reinterpret_cast<unsigned long long *>(own + flag1), epoch, s));
        h->p2p_launches += launches + 1;
        return EPP_OK;
    }
    if (phase == 1) {
        // exchange 1: OR of every rank's masks, read straight from the peers; then the global stop rule on the local counts ->
        // local best record in the own exchange buffer, raise flag 2
        CUDA_TRY(launch_p2p_wait(peers, n, flag1, epoch, h->p2p_err.as<int>(), timeout_ns, s));
        CUDA_TRY(launch_p2p_or_masks(peers, n, mask_off, mask_bytes, gmasks, s));
        PickParams pp = pick_params(h, w, h->decisions.as<epp_decision>() + r0, nullptr, nullptr);
        pp.global_masks = gmasks;
        pp.mask_words = (int32_t)W;
        pp.shard_out = reinterpret_cast<epp_shard_best *>(own + best_off);
        EPP_TRY(launch_match(h, sl, pp, &launches));
        // a rank whose wait failed must NOT publish records computed from an incomplete OR: the signal kernel checks
        CUDA_TRY(launch_p2p_signal_unless(reinterpret_cast<unsigned long long *>(own + flag2), epoch, h->p2p_err.as<int>(), s));
        h->p2p_launches += launches + 3;
        return EPP_OK;
    }
    const ShardMergeParams mp = shard_merge_params(h, r0, R, n, allbest, v.multimodal, out + r0, detail ? detail + r0 : nullptr);
    const size_t flag3 = (size_t)c * kP2pChunkFlags + kP2pFlag3;
    const size_t sel_off = h->p2p_sel_off + (size_t)r0 * S * sizeof(epp_shard_sel);
    if (phase == 2) {
        // exchange 2: gather every rank's records from the peers; then merge (lowest slot), or (seeded) resolve the tie
        // rule, select the members this rank owns into the own exchange buffer and raise flag 3
        CUDA_TRY(launch_p2p_wait(peers, n, flag2, epoch, h->p2p_err.as<int>(), timeout_ns, s));
        CUDA_TRY(launch_p2p_gather(peers, n, best_off, sizeof(epp_shard_best) * S * (size_t)R, allbest, s));
        if (!h->p2p_seeded) {
            CUDA_TRY(launch_shard_merge(mp, s, &launches));
            h->p2p_launches += launches + 2;
            return EPP_OK;
        }
        PickParams pp = pick_params(h, w, h->decisions.as<epp_decision>() + r0, nullptr, nullptr);
        pp.global_masks = gmasks;
        pp.mask_words = (int32_t)W;
        EPP_TRY(launch_select(h, sl, mp, pp, r0, reinterpret_cast<epp_shard_sel *>(own + sel_off), &launches));
        CUDA_TRY(launch_p2p_signal_unless(reinterpret_cast<unsigned long long *>(own + flag3), epoch, h->p2p_err.as<int>(), s));
        h->p2p_launches += launches + 3;
        return EPP_OK;
    }
    // exchange 3 (seeded): gather every rank's selected entries and build the decisions
    epp_shard_sel *allsel = h->p2p_allsel.as<epp_shard_sel>() + (size_t)r0 * (size_t)n * S;
    CUDA_TRY(launch_p2p_wait(peers, n, flag3, epoch, h->p2p_err.as<int>(), timeout_ns, s));
    CUDA_TRY(launch_p2p_gather(peers, n, sel_off, sizeof(epp_shard_sel) * S * (size_t)R, allsel, s));
    ShardSeedParams sp = shard_seed_params(h, r0);
    sp.all_sel = allsel;
    CUDA_TRY(launch_shard_finish(mp, sp, s, &launches));
    h->p2p_launches += launches + 2;
    return EPP_OK;
}

// Phases of a batch: the seeded tie rule adds the third exchange.
static int p2p_phases(const epp_engine *h) { return h->p2p_seeded ? 4 : 3; }

// Start / end of a batch of the exchange.
static int32_t p2p_begin(epp_engine *h, const BatchView &v, uint64_t *or_bits) {
    h->kept_R = 0;
    h->shard_R = 0;
    EPP_TRY(commit_locked(h));
    if (h->async_pending) EPP_TRY(finish_async(h));
    EPP_TRY(join_streams(h));
    EPP_TRY(reserve_batch(h, v.R));
    *or_bits = 0;
    if (v.offsets) EPP_TRY(device_offsets_or_bits(h, v.offsets, v.R, h->slot[0].stream, or_bits));
    ++h->p2p_epoch;
    h->p2p_launches = 0;
    return EPP_OK;
}
static int32_t p2p_end(epp_engine *h, int64_t R) {
    h->stats.last_kernel_launches = (uint64_t)h->p2p_launches;
    EPP_TRY(p2p_check(h, h->slot[0].stream, h->p2p_epoch));
    h->stats.n_batches++;
    h->stats.n_decisions += (uint64_t)R;
    return EPP_OK;
}
static int32_t p2p_prepare(epp_engine *h, const epp_batch *batch, epp_decision *out, const epp_decision_detail *detail,
                           BatchView &v) {
    if (!h || !out) return fail(EPP_ERR_INVALID, "NULL argument");
    EPP_TRY(set_device(h));
    EPP_TRY(join_streams(h));
    if (h->p2p_peer.empty()) return fail(EPP_ERR_STATE, "epp_shard_p2p_connect has not been called");
    if (h->p2p_broken) return fail(EPP_ERR_STATE, "the sharded exchange is broken (an earlier batch timed out): export and connect the buffers again");
    if (!sharded(h)) return fail(EPP_ERR_STATE, "epp_shard_set has not been called: every rank would count every endpoint");
    if (!h->pool_ready) return fail(EPP_ERR_STATE, "epp_pool_set has not been called (after epp_shard_set)");
    EPP_TRY(check_batch(h, batch, v));
    if (!v.device) return fail(EPP_ERR_INVALID, "the sharded peer-memory entry points take device-pointer batches (EPP_BATCH_DEVICE_PTRS)");
    if (v.R > h->p2p_R) return fail(EPP_ERR_CAPACITY, "batch of %lld requests exceeds the exported exchange buffer (%lld)", (long long)v.R, (long long)h->p2p_R);
    EPP_TRY(check_encode_detail(h, v.multimodal != nullptr, detail));
    v.async = false;
    return EPP_OK;
}

extern "C" int32_t epp_shard_schedule_p2p_detail(epp_engine *h, const epp_batch *batch, epp_decision *out,
                                                 epp_decision_detail *out_detail) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(h->mu);
    BatchView v;
    EPP_TRY(p2p_prepare(h, batch, out, out_detail, v));
    if (v.R == 0) return EPP_OK;
    uint64_t or_bits = 0;
    EPP_TRY(p2p_begin(h, v, &or_bits));
    // two halves on the engine's two streams: while one half waits for the peers' flags, the other half computes
    const bool split = h->dev_chunks > 1 && v.R >= 2 * 4096;       // (the dense-counter scratch is per stream)
    const int64_t half = split ? (((v.R + 1) / 2 + 31) & ~(int64_t)31) : v.R;
    if (split) {
        CUDA_TRY(cudaEventRecord(h->slot[0].done, h->slot[0].stream));
        CUDA_TRY(cudaStreamWaitEvent(h->slot[1].stream, h->slot[0].done, 0));
    }
    for (int phase = 0; phase < p2p_phases(h); phase++) {
        EPP_TRY(p2p_phase_rows(h, v, out, out_detail, phase, 0, 0, half, or_bits));
        if (split) EPP_TRY(p2p_phase_rows(h, v, out, out_detail, phase, 1, half, v.R, or_bits));
    }
    if (split) {
        h->s1_unjoined = true;
        EPP_TRY(join_streams(h));
    }
    return p2p_end(h, v.R);
}
extern "C" int32_t epp_shard_schedule_p2p(epp_engine *h, const epp_batch *batch, epp_decision *out) {
    return epp_shard_schedule_p2p_detail(h, batch, out, nullptr);
}
extern "C" int32_t epp_shard_p2p_phase_detail(epp_engine *h, const epp_batch *batch, epp_decision *out,
                                              epp_decision_detail *out_detail, int32_t phase) {
    if (!h) return fail(EPP_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(h->mu);
    if (phase < 0 || phase >= p2p_phases(h)) return fail(EPP_ERR_INVALID, "phase %d out of range [0,%d]", phase, p2p_phases(h) - 1);
    BatchView v;
    EPP_TRY(p2p_prepare(h, batch, out, out_detail, v));
    if (v.R == 0) return EPP_OK;
    if (phase == 0) EPP_TRY(p2p_begin(h, v, &h->p2p_or_bits));
    EPP_TRY(p2p_phase_rows(h, v, out, out_detail, phase, 0, 0, v.R, h->p2p_or_bits));
    if (phase == p2p_phases(h) - 1) return p2p_end(h, v.R);
    CUDA_TRY(cudaStreamSynchronize(h->slot[0].stream));
    return EPP_OK;
}
extern "C" int32_t epp_shard_p2p_phase(epp_engine *h, const epp_batch *batch, epp_decision *out, int32_t phase) {
    return epp_shard_p2p_phase_detail(h, batch, out, nullptr, phase);
}
