// kernels.h -- host-callable launchers of the sm_90a kernels (internal to libepp_engine.so).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/epp_engine.h"

namespace epp {

// ------------------------------------------------------------------------------------------------
// hashing (a1)
// ------------------------------------------------------------------------------------------------
struct HashParams {
    const uint8_t *data;        // prompt bytes (device)
    const uint64_t *offsets;    // [R+1] device, or nullptr => uniform_len
    const uint64_t *lengths;    // [R] device or nullptr => offsets[r+1] - offsets[r]
    uint64_t uniform_len;
    const uint32_t *model_ids;  // [R] device or nullptr
    const uint64_t *seeds;      // device table of h_{-1} per registered model
    int64_t R;
    int32_t block_bytes;        // blockSizeTokens * 4
    int32_t max_blocks;         // row pitch of `hashes`
    uint64_t *hashes;           // [R][max_blocks]
    int32_t *nblocks;           // [R]
    int64_t *eff_len;           // [R] bytes hashed after truncation (hashing.go:63-66)
    int64_t *in_len;            // [R] untruncated prompt length in bytes (P/D decider), may be nullptr
    uint64_t offsets_or_bits;   // OR of every offsets[r] (low bits decide the common alignment)
    int32_t sm_count;
    // k_hash_fused only: presence != nullptr trims the rows to the read table's reach.  bound[r] = the first block at a
    // window start (every 8th block is looked up) whose presence bit is clear (index.cuh), else nblocks[r]: the global
    // stop is <= bound[r].  Hashes [0, bound[r]) are stored.
    const uint32_t *presence;
    int32_t presence_shift;
    int32_t *bound;             // [R]
    unsigned long long *stored; // += bytes of hash rows stored by k_hash_fused, or nullptr
    // with presence: stop loading each prompt at its closing window (bound's window; the trailing partial block only
    // while no block is proven absent).  0: every prompt byte is read and hashed.
    int32_t skip;
    unsigned long long *read;   // += prompt bytes loaded by k_hash_fused, or nullptr
    uint32_t *req_next;         // k_hash_fused's request counter (device; zeroed by its launcher): one per stream
};
// Common alignment (0, 16, 32) of every block start; >= 16 (and block_bytes % 32 == 0) enables the fused kernel.
int hash_batch_alignment(const HashParams &p);
// Does launch_hash_prompts run k_hash_fused for this batch (the only kernel that trims rows and counts stored bytes)?
bool hash_fused_selected(const HashParams &p);
// Generic single-message XXH64 (model || salt seeds).  msg on device.
cudaError_t launch_hash_bytes(const uint8_t *msg, size_t len, uint64_t *out, cudaStream_t s);
cudaError_t launch_check_offsets_aligned(const uint64_t *offsets, int64_t n, int *flag_dev, cudaStream_t s);
// Whole hashPrompt for a batch.  Returns number of kernels launched via *launches.
// ev (optional, 4 events): [1]..[2] brackets the kernel(s) that read the prompt bytes.
cudaError_t launch_hash_prompts(const HashParams &p, cudaStream_t s, int *launches, cudaEvent_t *ev = nullptr);

// ------------------------------------------------------------------------------------------------
// prefix index (a2): open-addressed table  hash -> (posting offset, count)
// ------------------------------------------------------------------------------------------------
constexpr int kInlineIds = 5;
// One 32-byte slot = one DRAM/L2 sector, fetched by two 128-bit loads.  Posting lists of up to kInlineIds
// endpoints live IN the slot (no dependent load); longer lists live in `postings` at offset ids[0].  Lists are
// sorted by endpoint id and duplicate-free.
struct __align__(32) IndexSlot {
    uint64_t key;
    uint32_t cnt;                 // endpoints holding the block; 0 with a real key = every holder was evicted
                                  // (tombstone left by the incremental patch); a FREE slot has key == kEmptyKey
    uint32_t ids[kInlineIds];     // cnt <= kInlineIds: the endpoints; else ids[0] = offset into postings
};
constexpr uint64_t kEmptyKey = 0xFFFFFFFFFFFFFFFFULL;   // free-slot sentinel (ends probe chains); a real key equal to it
                                                        // lives in IndexView::special
struct IndexView {
    const IndexSlot *slots;
    const uint32_t *postings;
    uint64_t mask;            // capacity - 1 (capacity is a power of two); slots == nullptr => empty index
    IndexSlot special;        // record for key == kEmptyKey (cnt 0 when absent)
    uint32_t ep_begin, ep_end;  // shard range (postings outside are ignored for counting but keep the walk alive)
};
// Builds table + postings from n pairs (device arrays).  slots must hold `capacity` entries, postings n,
// scratch `capacity` uint32, cursor 4 uint32 (cursor[2] returns the number of distinct hashes, cursor[3] the keys
// claimed in the interning table).  *special_dev
// receives the record of key == kEmptyKey.  Deduplicates pairs, sorts every posting list and interns equal spilled
// lists (intern_keys / intern_vals: `capacity` entries each).
cudaError_t launch_index_build(const uint64_t *pair_hash, const uint32_t *pair_ep, uint64_t n, IndexSlot *slots,
                               uint64_t capacity, uint32_t *postings, uint32_t *scratch, uint32_t *cursor,
                               IndexSlot *special_dev, uint64_t *intern_keys, uint32_t *intern_vals,
                               cudaStream_t s, int *launches);
cudaError_t launch_index_get(const IndexView &ix, uint64_t hash, uint32_t *out_eps, int32_t cap, int32_t *out_n,
                             cudaStream_t s);
// Presence bitmap of 2^log2bits bits (6..30) over the table's keys (index.cuh presence_maybe); slots == nullptr: clear.
cudaError_t launch_presence_build(const IndexSlot *slots, uint64_t capacity, uint32_t *bits, int log2bits, cudaStream_t s,
                                  int *launches);

// ------------------------------------------------------------------------------------------------
// pool state -> request-independent scorer terms (a5-a9 precompute)
// ------------------------------------------------------------------------------------------------
constexpr int kMaxProfiles = 3;            // [0] primary / decode, [1] prefill, [2] encode
// LoRA adapter residency (fwkdl.Metrics.ActiveModels / WaitingModels / MaxActiveModels) for lora-affinity-scorer:
// per endpoint the adapter capacity, per adapter (= registered model id) the endpoints where it is active (1) or
// waiting (2), sorted by endpoint.  ptr == nullptr: no LoRA state (every endpoint scores 0.0 / its capacity tier).
struct LoraDev {
    const int32_t *max_active;   // [E] MaxActiveModels
    const int32_t *n_loaded;     // [E] len(ActiveModels) + len(WaitingModels)
    const uint32_t *ptr;         // [n_models + 1]
    const uint32_t *ep;          // [ptr[n_models]] endpoint slot ids, ascending within an adapter
    const uint8_t *state;        // 1 = active, 2 = waiting
    int32_t n_models;
    int32_t enabled;             // some profile has a lora-affinity scorer
};
struct PoolArrays {
    int32_t E;                 // slot capacity (max_endpoints)
    int32_t n_ext_cols;
    const uint8_t *role;       // [E] epp_role, 0xFF = absent
    const double *kv_usage;    // [E]
    const int32_t *waiting;    // [E]
    const int32_t *running;    // [E]
    const double *ext;         // [n_ext_cols][E]
    LoraDev lora;
};
struct ProfileDerived {
    // per profile, device arrays
    uint8_t *cand;             // [E] 1 = passes the role and label filters
    double *contrib;           // [EPP_MAX_SCORERS][E] clamp(score)*weight of every request-independent scorer
    double *base;              // [E] ordered weighted sum with every prefix term = clamp(0)*w
    uint32_t *order;           // [Epad] candidates sorted by (base desc, slot asc); then non-candidates
    uint32_t *grp_size;        // [Epad] size of the equal-base group of order[k]
    uint64_t *sort_key;        // [Epad] scratch
    int32_t *n_cand;           // [1]
    int64_t *qminmax;          // [4] waiting min,max, running min,max over candidates
    // random pickers only (nullptr otherwise): the candidates in ascending slot order, and over them the prefix sums of
    // the weighted-random masses of their bases (pick_random.cuh) and the prefix counts of +inf bases
    uint32_t *cands;           // [E]
    double *wcum;              // [E + 1]
    uint32_t *icum;            // [E + 1]
};
// A profile's label filters (include/epp_engine.h "Label filters"), compiled on the host: slot e passes requirement i
// when bit lcode[key[i]][e] of mask[i] is set.  lcode codes: 0 = key absent, 1..62 = a value some requirement names,
// 63 = any other value.  n == 0: no label filter (lcode is not read).
struct LabelFilterDev {
    const uint8_t *lcode;      // [keys][E]
    int32_t n;
    uint8_t key[EPP_LABEL_MAX_REQS];
    uint64_t mask[EPP_LABEL_MAX_REQS];
};
// [shard_begin, shard_end): only these slots become candidates (queue min/max still span the whole pool).
// A no-hit-lru scorer gets its warm score 0.5 here (the cold set comes from launch_pool_order).
cudaError_t launch_pool_prepare(const PoolArrays &pool, const epp_profile_cfg &prof, const LabelFilterDev &labels,
                                const ProfileDerived &d, int32_t Epad, uint32_t shard_begin, uint32_t shard_end,
                                cudaStream_t s, int *launches);
// The contribution rows, base sums, (base desc, slot asc) order and groups of d over d.cand / d.n_cand / d.qminmax (already
// derived), with the raw no-hit-lru score of slot e = nohit_col[e] (nullptr: the warm 0.5).  gate != nullptr: every kernel
// returns at once unless *gate != 0.
// With d.wcum != nullptr (a random picker) also d.cands / d.wcum / d.icum.
// (key asc, order asc) sort of Epad (a power of two) entries by one CTA; gate as below.
cudaError_t launch_pool_sort(uint64_t *key, uint32_t *order, int32_t Epad, const int32_t *gate, cudaStream_t s);
cudaError_t launch_pool_order(const PoolArrays &pool, const epp_profile_cfg &prof, const ProfileDerived &d, int32_t Epad,
                              const double *nohit_col, const int32_t *gate, cudaStream_t s, int *launches);

// ------------------------------------------------------------------------------------------------
// no-hit-lru scorer state (nohit_lru.cu): the LRU of endpoints that received a cold request
// ------------------------------------------------------------------------------------------------
struct NoHitState {
    uint64_t *last_seq;        // [E] sequence number of the endpoint's last Add, 0 = not in the LRU
    int32_t *pos;              // [E] position in the LRU (oldest = 0), -1 = not in it
    int32_t *n_members;        // [1] LRU length
    int32_t *dirty;            // [1] some Add happened since the cold sets were derived
    uint64_t *sort_key;        // [Epad] scratch
    uint32_t *order;           // [Epad] scratch
    int32_t lru_size;
};
// Applies the Adds of one scheduling call's decisions (request r: its pick, then its prefill pick, when cold[r] != 0) as
// last_seq[e] = max(last_seq[e], seq0 + 2r (+1)), then trims the LRU to lru_size members and re-ranks it.
// dec / cold are indexed by r in [0, R).
cudaError_t launch_nohit_touch(const NoHitState &st, const epp_decision *dec, const uint8_t *cold, int64_t R, uint64_t seq0,
                               cudaStream_t s, int *launches);
cudaError_t launch_nohit_rank(const NoHitState &st, int32_t E, int32_t Epad, bool gated, cudaStream_t s, int *launches);
// The raw cold no-hit-lru column of one profile (no_hit_lru.go:198-242) over its candidates -> col[E].
cudaError_t launch_nohit_column(const NoHitState &st, int32_t E, const uint8_t *cand, const int32_t *n_cand, double *col,
                                bool gated, cudaStream_t s, int *launches);
cudaError_t launch_nohit_clear(const NoHitState &st, cudaStream_t s, int *launches);
// Cold bit of each request of a dense match matrix for one profile (epp_score): no candidate has match > 0.
cudaError_t launch_nohit_cold_rows(int64_t R, int32_t E, const uint8_t *cand, const int32_t *match, uint8_t *cold,
                                   cudaStream_t s, int *launches);

// ------------------------------------------------------------------------------------------------
// inflight-load producer (inflight.cu): per-slot in-flight request and token counts
// ------------------------------------------------------------------------------------------------
struct InflightState {
    int64_t *req;              // [E] InFlightLoad.Requests
    int64_t *tok;              // [E] InFlightLoad.Tokens
    double *col_tok;           // [E] the ext column the token-load scorers read
    double *col_req;           // [E] the ext column the active-request scorers read
    int32_t E;
};
// Releases and resets of one slot folded on the host: set != 0 replaces the counters, else adds to them.
struct InflightDelta {
    uint32_t slot;
    uint32_t set;
    int64_t req, tok;
};
// PreRequest of one scheduling call: for every request with status 0, +1 request and +est(in_len[r]) tokens on its
// pick, its prefill pick and (det != nullptr) its encode pick, each that is not EPP_NO_ENDPOINT.  in_len == nullptr: 0.
cudaError_t launch_inflight_add(const InflightState &st, const epp_decision *dec, const epp_decision_detail *det,
                                const int64_t *in_len, int64_t R, cudaStream_t s, int *launches);
cudaError_t launch_inflight_apply(const InflightState &st, const InflightDelta *d, int32_t n, cudaStream_t s, int *launches);
// col_tok / col_req <- the counters.
cudaError_t launch_inflight_columns(const InflightState &st, cudaStream_t s, int *launches);

// ------------------------------------------------------------------------------------------------
// match + score + pick (a3-a14)
// ------------------------------------------------------------------------------------------------
struct ProfileDev {            // what the pick kernels read (device pointers + config by value)
    epp_profile_cfg cfg;
    const uint8_t *cand;
    const double *contrib;
    const double *base;
    const uint32_t *order;
    const uint32_t *grp_size;
    const int32_t *n_cand;
    const uint32_t *cands;     // random pickers (cfg.picker != 0): ProfileDerived::cands / wcum / icum
    const double *wcum;
    const uint32_t *icum;
};
// no-hit-lru scorer (nohitlru/no_hit_lru.go): a profile whose bit is set in `mask` evaluates a cold request (no candidate
// holds a block of its prompt) with cold[pi] -- the same candidates, with the LRU column in place of the warm 0.5 -- and
// every decision writes the cold bit of the last such profile that ran (decode -> encode -> prefill) to cold_out[r].
struct NoHitView {
    int32_t mask;              // 0: no profile has the scorer
    const ProfileDev *cold;    // [kMaxProfiles] in device memory (keeps the launch parameters of the default builds small)
    uint8_t *cold_out;         // [R] (this launch's rows), or nullptr
};
// General evaluation (pick_general.cuh): set when a profile configures the prefix-cache-affinity-filter or pick_k > 1.
struct GenView {
    int32_t on;                // every profile evaluation of the launch goes through gen::eval
    int32_t topk;              // k of the lists below (<= 1: no lists)
    PoolArrays pool;           // raw pool arrays (scores over a narrowed candidate set are not in the snapshot columns)
    uint32_t *topk_picks[kMaxProfiles];   // [R][topk] per profile, or nullptr
    double *topk_scores;       // [R][topk] scores of the primary list, or nullptr
};
struct PickParams {
    int64_t R;
    int32_t E;
    int32_t max_blocks;
    int32_t block_size_tokens;
    int32_t n_profiles;        // 1 or 2 (2 => disagg: [0]=decode, [1]=prefill)
    int32_t encode_on;         // disagg with an encode profile ([2]): runs for requests flagged in `multimodal`
    const uint8_t *multimodal; // [R] or nullptr (encode decider input: hasMultimodalContent)
    int32_t always_disagg;
    int64_t non_cached_tokens;
    ProfileDev prof[kMaxProfiles];
    const uint64_t *hashes;    // [R][max_blocks]
    const int32_t *nblocks;    // [R]
    // [R] rows trimmed by k_hash_fused (HashParams::bound): hashes [bound, nblocks) were not stored and block `bound`
    // (< nblocks) is a proven miss.  nullptr: every row is whole.
    const int32_t *bound;
    const int64_t *in_len;     // [R] prompt bytes (decider)
    const uint32_t *model_ids; // [R] registered model (= LoRA adapter) of each request, or nullptr => model 0
    LoraDev lora;
    IndexView index;
    epp_decision *out;         // [R]
    epp_decision_detail *detail;  // [R] or nullptr
    int32_t *out_match;        // dense [R][E] or nullptr (Produce parity mode)
    unsigned long long *work_counters;  // [2] += (probes, postings) of this launch, or nullptr
    // endpoint-sharded mode (nullptr otherwise): the stop rule comes from the OR of all ranks' presence masks
    const uint32_t *global_masks;       // [R][mask_words]
    int32_t mask_words;
    epp_shard_best *shard_out;          // [R][handler_stages] local best records instead of `out`
    // dense-counter kernel (k_match_pick) only: process the requests listed in req_list[0 .. *req_list_n) (the sparse kernel's overflows)
    const int32_t *req_list;
    const int32_t *req_list_n;
    // sparse kernels only: requests whose matched-endpoint set overflowed the per-warp map are appended here
    int32_t *overflow_list;
    int32_t *overflow_n;
    // k_match_pick_sparse only: requests taken beyond each warp's first one (zero at launch; R < 2^31)
    int32_t *req_next;
    // tie rule: 0 = lowest slot of the arg-max set; else the member of rank tie_rank(seed, 4 * (tie_base + r) + profile)
    uint64_t tie_seed;
    uint64_t tie_base;         // ordinal of request 0 of this launch
    GenView gen;
    NoHitView nohit;
};
// Fused lookup + match + score + pick, one warp per request.  Per-warp match counters live in shared memory
// (smem = match_pick_smem_bytes(E, false)) or, when E is too large for that, in a zero-initialised global
// scratch of grid * warps * ceil(E/2) words (smem = match_pick_smem_bytes(E, true)).
size_t match_pick_smem_bytes(int32_t E, bool global_counts);
int match_pick_warps_per_cta();
cudaError_t launch_match_pick(const PickParams &p, uint32_t *gscratch, int grid, size_t smem, cudaStream_t s,
                              int *launches);
// The same decision per request with a lane-distributed register map of the matched endpoints (requests whose set
// overflows it are appended to p.overflow_list for the dense-counter kernel).  8 warps per CTA, 6-8 CTAs per SM.
cudaError_t launch_match_pick_sparse(const PickParams &p, int sm_count, cudaStream_t s, int *launches);
// Does some profile of the launch (PickParams, DensePickParams) have a random picker?  Then the sparse, small-batch,
// dense-counter and injected-match paths launch their _rand builds.
// Stages of the handler of a launch (PickParams, DensePickParams): 1 = single profile, 2 = decode + prefill, 3 = + encode.
// In the endpoint-sharded mode it is also the number of records per request (include/epp_engine.h, "Staged records").
template <class Params> __host__ __device__ inline int handler_stages(const Params &p) {
    return p.encode_on ? 3 : (p.n_profiles >= 2 ? 2 : 1);
}
template <class Params> inline bool any_random_picker(const Params &p) {
    const int np = handler_stages(p);
    for (int i = 0; i < np; i++)
        if (p.prof[i].cfg.picker) return true;
    return false;
}
// cycle_small.cu: a1-a14 of a small host batch in ONE launch, one CTA per request, prompts read from and decisions
// written to PINNED HOST memory (zero-copy); flags[r] = epoch (| 0x80000000 when the request overflowed the sparse map and
// was appended to pp.overflow_list instead of being decided) is written last, after a system-scope fence.
struct SmallOut {
    epp_decision *dec;             // [R] device view of pinned host memory
    epp_decision_detail *det;      // [R]
    uint32_t *flags;               // [R]
    uint32_t epoch;                // 1 .. 0x7fffffff
    // Prompts still on their way when the kernel starts (the copy runs on another stream): the rows may be read once
    // *arrive == epoch (a stream-ordered 32-bit write behind the copy).  nullptr: resident at launch.
    const uint32_t *arrive;        // device
};
size_t cycle_small_max_blocks();
// Does the kernel bring a whole prompt into shared memory (one bulk copy) before it hashes?  Then a request's flag is
// raised only after its last read of the prompt bytes, and the staging buffer may be refilled as soon as all flags are up.
bool cycle_small_stages_prompt(int32_t max_blocks, int32_t block_bytes);
cudaError_t launch_cycle_small(const HashParams &hp, const PickParams &pp, const SmallOut &so, cudaStream_t s, int *launches);
// Decision logic on injected dense match info (plugin parity / KAT mode).
struct DensePickParams {
    int64_t R;
    int32_t E;
    int32_t block_size_tokens;
    int32_t n_profiles;
    int32_t encode_on;
    const uint8_t *multimodal;
    int32_t always_disagg;
    int64_t non_cached_tokens;
    ProfileDev prof[kMaxProfiles];
    const int32_t *match;      // [R][E]
    const int32_t *total;      // [R]
    const int64_t *in_len;     // [R]
    const uint32_t *model_ids; // [R] or nullptr
    LoraDev lora;
    epp_decision *out;
    epp_decision_detail *detail;
    uint64_t tie_seed;
    uint64_t tie_base;
    GenView gen;
    NoHitView nohit;
};
cudaError_t launch_dense_pick(const DensePickParams &p, cudaStream_t s, int *launches);
// Latency predictions (include/epp_engine.h, "Latency predictions"): the general evaluation of pick_latency.cuh for the
// profiles whose bit is set in `mask`, with request r's entries at ent[off[r0 + r] .. + cnt[r0 + r]) (cnt == nullptr: no
// request has any).  The _lat builds of the dense-counter, injected-match and subset kernels take it as an extra
// argument, so the parameters of every other kernel stay as they are.
struct LatView {
    const uint32_t *cnt;       // [batch R] absolute request rows
    const uint64_t *off;
    const epp_prediction *ent;
    int64_t r0;                // row of this launch's request 0
    int32_t mask;              // chain profiles: a latency piece or the context-length scorer
    epp_latency_cfg cfg[kMaxProfiles];
    // context length ("Context length"): the call's per-row token counts ([batch R] absolute rows, -1 = the default from
    // the prompt length; nullptr: all default), and per profile listing the scorer its slots' ranges ([E]: x = min, y = max
    // when x >= 0; x = kRangeAbsent / kRangeInvalid otherwise) and whether it filters
    const int64_t *ctx;
    const longlong2 *rng[kMaxProfiles];
    int32_t cl_filter;         // bit pi: profile pi's context-length filter is on
};
constexpr long long kRangeAbsent = -1, kRangeInvalid = -2;
cudaError_t launch_match_pick_lat(const PickParams &p, const LatView &lv, uint32_t *gscratch, int grid, size_t smem,
                                  cudaStream_t s, int *launches);
cudaError_t launch_dense_pick_lat(const DensePickParams &p, const LatView &lv, cudaStream_t s, int *launches);
// subset_pick.cu: per-request endpoint subsets (include/epp_engine.h, "Endpoint subsets").  One warp re-decides one
// restricted request of a launch whose ordinary match kernel has run: it walks the request's stored hash row up to the
// global stop counting only the listed holders, then evaluates every profile over the listed slots (full evaluation:
// affinity filter, scorer normalisation, no-hit-lru cold ranks, first-k and random draws over the narrowed set).
// lv != nullptr (an engine with latency profiles): k_subset_pick_lat, whose latency profiles run the chain of
// pick_latency.cuh over the listed slots with the request's predictions.
struct SubsetRow {
    uint64_t off;              // the request's slots are slots[off .. off + n), ascending
    uint32_t row;              // absolute request index in the batch
    uint32_t n;
};
struct SubsetView {
    const SubsetRow *rows;     // [n_rows] restricted requests of this launch
    int32_t n_rows;
    int64_t r0;                // the PickParams rows start at request r0
    const uint32_t *slots;
    int32_t *hits;             // parallel to slots: the request's matchBlocks on each listed slot (written here)
    int32_t *scratch;          // parallel to slots: no-hit-lru cold ranks (written here)
    const int32_t *nohit_pos;  // [E] position in the no-hit-lru LRU (oldest 0, -1 = never used), or nullptr
};
cudaError_t launch_subset_pick(const PickParams &p, const SubsetView &sv, const LatView *lv, cudaStream_t s, int *launches);

// ------------------------------------------------------------------------------------------------
// admission (admit.cu, include/epp_engine.h "Admission"): k_admit rewrites the rows an admitter rejects, one warp per
// listed row, behind the call's picks and before its after-pick updates.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kAdmitProbabilistic = 1u, kAdmitLatencySlo = 2u;
struct AdmitRow {
    uint32_t row;              // absolute request index in the call
    uint32_t flags;            // kAdmitProbabilistic: sheddable; kAdmitLatencySlo: sheddable with an SLO and entries
    uint64_t sub_off;          // subset slots sub_slots[sub_off .. + sub_n), ascending
    uint32_t sub_n;            // EPP_SUBSET_ALL: the whole pool
    uint32_t pred_n;           // entries ent[pred_off .. + pred_n)
    uint64_t pred_off;
};
struct AdmitParams {
    const AdmitRow *rows;      // [n_rows] ascending by row
    int32_t n_rows;
    int32_t E;
    const uint32_t *ent;       // slot | (both validity bits set) << 31
    const uint32_t *sub_slots;
    const uint8_t *role;       // the pool snapshot (PoolArrays)
    const double *kv;
    const int32_t *waiting, *running;
    int32_t pool_n, pool_idle, pool_cold;   // the whole pool's candidates, idle and cold flags, saturation fold
    double pool_sat;
    double qdt, kvt, power, k;
    uint64_t tie_seed, ord_base;            // ordinal of row r = ord_base + r
    epp_decision *dec;                      // [R] of the call
    epp_decision_detail *det;               // [R] or nullptr
    int32_t topk;                           // row stride of the lists (0 = none)
    uint32_t *topk_picks[kMaxProfiles];
    double *topk_scores;
};
cudaError_t launch_admit(const AdmitParams &p, cudaStream_t s, int *launches);

// Scorer.Score parity: out[R][E].  scorer_index -1 => weighted ordered sum (-1.0 for non-candidates).
// cold != nullptr (the profile has a no-hit-lru scorer): cold[r] selects prof_cold and the raw cold column nohit_col
// for request r.
cudaError_t launch_score_dense(int64_t R, int32_t E, const ProfileDev &prof, const ProfileDev &prof_cold,
                               const uint8_t *cold, const double *nohit_col, const PoolArrays &pool,
                               const int64_t *qminmax, const int32_t *match, const int32_t *total,
                               const uint32_t *model_ids, int32_t scorer_index, double *out, cudaStream_t s,
                               int *launches);

// endpoint-sharded mode: per-request block-presence masks of the LOCAL table (bit i of word i/32 = block i held
// by some endpoint of this shard), and the cross-rank reduction of the per-shard best records.
cudaError_t launch_shard_probe(int64_t R, int32_t max_blocks, const uint64_t *hashes, const int32_t *nblocks,
                               const IndexView &index, uint32_t *out_masks, int32_t mask_words, cudaStream_t s,
                               int *launches);
// The merge: per stage, max score, lowest slot id among equals, ties summed; then the disagg handler's deciders on the
// merged decode pick (score.cuh: pd_decide).  stages == 1 is the single-profile handler.
struct ShardMergeParams {
    int64_t R;
    int32_t n_ranks;
    int32_t stages;                     // records per request and rank
    const epp_shard_best *all_best;     // [n_ranks][R][stages]
    const int32_t *nblocks;             // [R]
    epp_decision *out;                  // [R]
    epp_decision_detail *detail;        // [R] or nullptr
    // decider inputs (stages >= 2)
    int32_t always_disagg;
    int32_t block_size_tokens;
    int64_t non_cached_tokens;
    const int64_t *in_len;              // [R] prompt bytes
    const uint8_t *multimodal;          // [R] or nullptr (stages == 3)
};
cudaError_t launch_shard_merge(const ShardMergeParams &p, cudaStream_t s, int *launches);

// Seeded ties (include/epp_engine.h, "Seeded ties"): every rank resolves the global tie rule over the gathered records
// (k_shard_resolve: the owner of each arg-max member and its rank in the owner's local set), the owner selects that
// member (the _select builds of the match kernels), and k_shard_finish builds the decisions from the gathered selects.
// A work item is x = r * stages + st (r: row of the launch), y = the member's rank in this rank's local set (>= 1).
struct ShardSeedParams {
    uint64_t tie_seed;
    uint64_t tie_base;                  // ordinal of request 0 of the launch
    uint32_t ep_begin, ep_end;          // resolve: this rank's shard (the owner's pick lies in its range)
    epp_shard_sel *sel;                 // resolve: [R][stages] this rank's entries (EPP_NO_ENDPOINT where it owns none)
    uint2 *work;                        // resolve: the selects this rank owns, appended at work[*work_n]
    int32_t *work_n;
    const epp_shard_sel *all_sel;       // finish: [n_ranks][R][stages], in the order of all_best
};
cudaError_t launch_shard_resolve(const ShardMergeParams &p, const ShardSeedParams &sp, cudaStream_t s, int *launches);
cudaError_t launch_shard_finish(const ShardMergeParams &p, const ShardSeedParams &sp, cudaStream_t s, int *launches);
struct ShardSelView {
    const uint2 *work;                  // [*work_n] items of k_shard_resolve
    const int32_t *work_n;
    int32_t stages;
    epp_shard_sel *sel;                 // [R][stages]: the selected member and its match count
    int32_t *dense_list;                // items whose lane map overflowed, for the dense-counter select
    int32_t *dense_n;
};
// The sparse select (one warp per item; overflows to sv.dense_list) and the dense-counter select over sv.dense_list.
cudaError_t launch_match_pick_sparse_select(const PickParams &p, const ShardSelView &sv, int sm_count, cudaStream_t s,
                                            int *launches);
cudaError_t launch_match_pick_select(const PickParams &p, const ShardSelView &sv, uint32_t *gscratch, int grid, size_t smem,
                                     cudaStream_t s, int *launches);

// shard_p2p.cu: exchanges of the endpoint-sharded mode over NVLink peer memory (no NCCL)
cudaError_t launch_p2p_signal(unsigned long long *flag, unsigned long long epoch, cudaStream_t s);
cudaError_t launch_p2p_signal_unless(unsigned long long *flag, unsigned long long epoch, const int *err_dev, cudaStream_t s);
cudaError_t launch_p2p_wait(unsigned char *const *peers_dev, int n, size_t flag_off, unsigned long long epoch, int *err_dev,
                            unsigned long long timeout_ns, cudaStream_t s);
cudaError_t launch_p2p_or_masks(unsigned char *const *peers_dev, int n, size_t masks_off, unsigned long long n_bytes,
                                void *out, cudaStream_t s);
cudaError_t launch_p2p_gather(unsigned char *const *peers_dev, int n, size_t best_off, unsigned long long n_bytes,
                              void *out, cudaStream_t s);

}  // namespace epp
