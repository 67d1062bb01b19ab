// batcher.cu -- the micro-batcher of the drop-in boundary (SURVEY 8(f).2): the reference calls
// Scheduler.Schedule(ctx, *InferenceRequest, []Endpoint) once per in-flight HTTP request, concurrently from one
// goroutine each (pkg/epp/requestcontrol/director.go:243, handlers/server.go:168); the engine decides batches.  This
// layer turns the one into the other INSIDE the library, so that a cgo shim is a two-call wrapper
// (epp_submit + epp_wait) with no batching logic of its own:
//
//   epp_submit   reserves a row of the batch being filled with ONE atomic compare-and-swap (no lock), copies the prompt
//                into the batch's pinned staging buffer and returns a ticket;
//   the flusher  (one thread per batcher) closes a batch when it holds max_batch requests or its oldest request has
//                waited max_delay_us, runs epp_schedule on it (ONE frozen snapshot per flush, App. A.8), publishes the
//                decisions, then -- when index_picks is set -- runs epp_index_add_picked (PreRequest,
//                approximateprefix/plugin.go:164-200), so index updates land BETWEEN flushes; meanwhile the submitters fill
//                the next staging buffers;
//   epp_wait     returns the ticket's decision once its batch has been flushed: a few waiters poll the flush counter
//                (a flush is ONE 30-130 us kernel launch), the others sleep on it (futex) -- nobody takes a lock.
//
// Hot-path synchronisation is three atomics: `fill` = (sequence number of the batch being filled << 20 | rows reserved),
// `ready` (per staging buffer) = rows whose prompt copy is complete, `done` = batches flushed.  Batch k uses staging
// buffer k % 4 and result slot k % 4096; a submitter of batch k waits until batch k - 4 has been flushed.
//
// It is built on the public C ABI only (include/epp_engine.h): no engine internals, no CPU compute path.
#include <linux/futex.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/epp_engine.h"
#include "kernels.h"

// engine.cu: the engine's profiles with a latency piece (0: none)
int32_t engine_latency_mask(const epp_engine *h);
int32_t engine_admission(const epp_engine *h);

namespace {
constexpr int kBufs = 4;                       // staging buffers: batches k .. k+3 can be filling / in flight at once
constexpr int kResults = 4096;                 // flushed batches whose results are kept for epp_wait (ring)
constexpr uint64_t kCountMask = (1ull << 20) - 1;
using Clock = std::chrono::steady_clock;

inline void cpu_relax() {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
}
inline void futex_wait(std::atomic<uint32_t> *a, uint32_t expected, const timespec *timeout) {
    syscall(SYS_futex, reinterpret_cast<uint32_t *>(a), FUTEX_WAIT_PRIVATE, expected, timeout, nullptr, 0);
}
inline void futex_wake_all(std::atomic<uint32_t> *a) {
    syscall(SYS_futex, reinterpret_cast<uint32_t *>(a), FUTEX_WAKE_PRIVATE, INT_MAX, nullptr, nullptr, 0);
}
inline int64_t now_ns() {
    return std::chrono::duration_cast<std::chrono::nanoseconds>(Clock::now().time_since_epoch()).count();
}

struct Staging {
    uint8_t *data = nullptr;                   // [max_batch][row_cap] pinned
    uint64_t *offsets = nullptr;               // [max_batch + 1]
    uint64_t *lengths = nullptr;               // [max_batch] true prompt lengths (may exceed the row)
    uint32_t *model_ids = nullptr;
    uint8_t *multimodal = nullptr;
    epp_decision *dec = nullptr;
    epp_decision_detail *det = nullptr;
    uint32_t *topk[3] = {nullptr, nullptr, nullptr};   // [max_batch][pick_k] primary / prefill / encode lists (pick_k > 1)
    // endpoint subsets (epp_submit_subset): per row EPP_SUBSET_ALL or its slot count, its slots at row * EPP_SUBSET_MAX_SLOTS
    std::vector<uint32_t> sub_counts;          // [max_batch]
    std::vector<uint64_t> sub_offsets;         // [max_batch]
    std::vector<uint32_t> sub_slots;           // [max_batch][EPP_SUBSET_MAX_SLOTS], allocated by the first subset submit
    std::atomic<int32_t> any_subset{0};        // some row of the batch using this buffer has a subset
    // latency predictions (epp_submit_predicted): per row its entry count, its entries at row * EPP_PRED_MAX_SLOTS
    std::vector<uint32_t> pred_counts;         // [max_batch]
    std::vector<uint64_t> pred_offsets;        // [max_batch]
    std::vector<epp_prediction> pred_entries;  // [max_batch][EPP_PRED_MAX_SLOTS], allocated by the first predicted submit
    std::atomic<int32_t> any_pred{0};          // some row of the batch using this buffer has predictions
    // context lengths (epp_submit_ctx): per row its token count, -1 = the default
    std::vector<int64_t> ctx;                  // [max_batch]
    std::atomic<int32_t> any_ctx{0};           // some row of the batch using this buffer has a token count
    // admission (epp_submit_admit): per row its priority and SLOs, and its entries' validity bytes next to pred_entries
    std::vector<int32_t> priority;             // [max_batch], 0 for rows submitted any other way
    std::vector<double> ttft_slo, tpot_slo;    // [max_batch]
    std::vector<uint8_t> pred_valid;           // [max_batch][EPP_PRED_MAX_SLOTS], allocated with pred_entries
    std::atomic<int32_t> any_adm{0};           // some row of the batch using this buffer came through epp_submit_admit
    std::atomic<int32_t> ready{0};             // rows of the batch using this buffer whose copy is complete
    std::atomic<int64_t> first_arrival_ns{0};  // when row 0 of that batch was reserved
};
// Results of one flushed batch, kept until kResults later batches were flushed.
struct Result {
    std::atomic<uint64_t> seq{~0ull};          // which batch the arrays hold (~0: being rewritten)
    std::atomic<int32_t> readers{0};           // epp_wait calls copying out of the arrays: the flusher waits for them before
                                               // it rewrites the slot (4096 flushes later)
    int32_t status = EPP_OK;                   // return code of the batch's epp_schedule / epp_index_add_picked
    int32_t n = 0;
    std::vector<epp_decision> dec;
    std::vector<epp_decision_detail> det;
    std::vector<uint32_t> topk;                // [3][n][pick_k] when the engine's pick_k > 1
};
}  // namespace

struct epp_batcher {
    epp_engine *eng = nullptr;
    epp_batcher_cfg cfg{};
    uint64_t row_cap = 0;                      // bytes of a prompt that hashPrompt can read (hashing.go:63-66)
    int32_t pick_k = 0;                        // the engine's maxNumOfEndpoints (> 1: flushes also fetch the first-k lists)
    uint32_t max_endpoints = 0;
    std::once_flag sub_once;                   // the subset slot staging of every buffer, allocated on first use
    bool sub_alloc_failed = false;
    std::once_flag pred_once;                  // the prediction staging of every buffer, allocated on first use
    bool pred_alloc_failed = false;
    Staging buf[kBufs];
    std::vector<Result> results;
    std::atomic<uint64_t> fill{0};             // (sequence number of the batch being filled << 20) | rows reserved in it
    std::atomic<uint64_t> done{0};             // batches [0, done) have been flushed
    std::atomic<uint32_t> done32{0};           // low word of `done` (futex word of the waiters)
    std::atomic<uint32_t> work32{0};           // bumped by whoever gives the flusher something to do (its futex word)
    std::atomic<int32_t> sleepers{0};          // waiters asleep on done32
    std::atomic<int32_t> spinners{0};          // waiters polling `done`
    std::atomic<bool> flusher_asleep{false};
    std::atomic<bool> stop{false};
    std::thread flusher;
    std::atomic<uint64_t> n_flushes{0}, n_requests{0}, n_full{0}, index_errors{0};
    std::mutex err_mu;
    std::string last_error;
};

static thread_local std::string g_batcher_error;

static void wake_flusher(epp_batcher *b) {
    b->work32.fetch_add(1, std::memory_order_seq_cst);
    if (b->flusher_asleep.load(std::memory_order_seq_cst)) futex_wake_all(&b->work32);
}

static void flusher_main(epp_batcher *b) {
    const int64_t delay_ns = (int64_t)b->cfg.max_delay_us * 1000;
    for (;;) {
        // ---- wait for a batch to close: full, or non-empty and its oldest request has waited max_delay_us
        uint64_t f;
        for (int idle = 0;; idle++) {
            f = b->fill.load(std::memory_order_acquire);
            const uint64_t n = f & kCountMask;
            const bool stopping = b->stop.load(std::memory_order_acquire);
            if (n >= (uint64_t)b->cfg.max_batch || (n > 0 && stopping)) break;
            if (n == 0 && stopping) return;
            if (n > 0) {
                const int64_t t0 = b->buf[(f >> 20) % kBufs].first_arrival_ns.load(std::memory_order_acquire);
                if (delay_ns == 0 || (t0 && now_ns() - t0 >= delay_ns)) break;
                cpu_relax();                                   // the deadline is microseconds away: poll
                continue;
            }
            if (idle < 2000) { cpu_relax(); continue; }        // some tens of microseconds of polling before sleeping
            const uint32_t w = b->work32.load(std::memory_order_acquire);
            b->flusher_asleep.store(true, std::memory_order_seq_cst);
            if ((b->fill.load(std::memory_order_seq_cst) & kCountMask) == 0 && !b->stop.load(std::memory_order_acquire)) {
                timespec ts{0, 50 * 1000 * 1000};              // a lost wake-up costs 50 ms at most
                futex_wait(&b->work32, w, &ts);
            }
            b->flusher_asleep.store(false, std::memory_order_release);
            idle = 0;
        }
        // ---- close it: from now on submitters reserve rows of batch seq + 1
        const uint64_t seq = f >> 20;
        f = b->fill.exchange((seq + 1) << 20, std::memory_order_acq_rel);
        const int32_t n = (int32_t)std::min<uint64_t>(f & kCountMask, (uint64_t)b->cfg.max_batch);
        Staging &st = b->buf[seq % kBufs];
        while (st.ready.load(std::memory_order_acquire) < n) cpu_relax();     // rows reserved before the close: a 16 KiB memcpy each
        if (n >= b->cfg.max_batch) b->n_full.fetch_add(1, std::memory_order_relaxed);

        epp_batch batch;
        memset(&batch, 0, sizeof batch);
        batch.n_requests = n;
        batch.data = st.data;
        batch.offsets = st.offsets;
        batch.lengths = st.lengths;
        batch.model_ids = st.model_ids;
        batch.multimodal = st.multimodal;
        batch.flags = EPP_BATCH_LENGTHS_EXCEED_ROWS;
        epp_topk_out tk;
        memset(&tk, 0, sizeof tk);
        tk.struct_size = sizeof tk;
        tk.k = b->pick_k;
        tk.primary = st.topk[0]; tk.prefill = st.topk[1]; tk.encode = st.topk[2];
        const bool any_pred = st.any_pred.load(std::memory_order_acquire) != 0;
        const bool any_sub = st.any_subset.load(std::memory_order_acquire) != 0;
        const bool any_ctx = st.any_ctx.load(std::memory_order_acquire) != 0;
        const bool any_adm = st.any_adm.load(std::memory_order_acquire) != 0;
        // each input is passed exactly when some row carries it; predictions only reach a latency engine or the
        // latency-slo-admitter (every predicted submit checks it)
        epp_predictions pr;
        memset(&pr, 0, sizeof pr);
        pr.struct_size = sizeof pr;
        pr.counts = st.pred_counts.data();
        pr.offsets = st.pred_offsets.data();
        pr.entries = st.pred_entries.data();
        epp_subset sub;
        memset(&sub, 0, sizeof sub);
        sub.struct_size = sizeof sub;
        sub.counts = st.sub_counts.data();
        sub.offsets = st.sub_offsets.data();
        sub.slots = st.sub_slots.data();
        epp_context_tokens ct;
        memset(&ct, 0, sizeof ct);
        ct.struct_size = sizeof ct;
        ct.tokens = st.ctx.data();
        epp_admission adm;
        memset(&adm, 0, sizeof adm);
        adm.struct_size = sizeof adm;
        adm.priority = st.priority.data();
        adm.ttft_slo = st.ttft_slo.data();
        adm.tpot_slo = st.tpot_slo.data();
        adm.pred_valid = st.pred_valid.empty() ? nullptr : st.pred_valid.data();
        const int32_t rc = epp_schedule_admit(b->eng, &batch, any_sub ? &sub : nullptr, any_pred ? &pr : nullptr,
                                              any_ctx ? &ct : nullptr, any_adm ? &adm : nullptr, st.dec, st.det,
                                              b->cfg.index_picks ? 1 : 0, b->pick_k > 1 ? &tk : nullptr);
        st.any_pred.store(0, std::memory_order_relaxed);
        st.any_subset.store(0, std::memory_order_relaxed);
        st.any_ctx.store(0, std::memory_order_relaxed);
        st.any_adm.store(0, std::memory_order_relaxed);
        if (rc != EPP_OK) {
            std::lock_guard<std::mutex> lk(b->err_mu);
            b->last_error = epp_last_error();
        }
        // ---- publish the results, then the flush counter
        Result &res = b->results[seq % kResults];
        res.seq.store(~0ull, std::memory_order_seq_cst);           // late readers of the slot's previous batch see it expire ...
        while (res.readers.load(std::memory_order_seq_cst) != 0) cpu_relax();   // ... and those inside finish first
        res.status = rc;
        res.n = n;
        res.dec.assign(st.dec, st.dec + n);                       // the vectors keep their capacity from lap to lap of the ring
        res.det.assign(st.det, st.det + n);
        res.topk.clear();
        if (b->pick_k > 1)
            for (int q = 0; q < 3; q++) res.topk.insert(res.topk.end(), st.topk[q], st.topk[q] + (size_t)n * (size_t)b->pick_k);
        res.seq.store(seq, std::memory_order_release);
        st.ready.store(0, std::memory_order_relaxed);
        st.first_arrival_ns.store(0, std::memory_order_relaxed);
        b->n_flushes.fetch_add(1, std::memory_order_relaxed);
        b->n_requests.fetch_add((uint64_t)n, std::memory_order_relaxed);
        b->done.store(seq + 1, std::memory_order_seq_cst);        // also frees staging buffer seq % kBufs for batch seq + kBufs
        b->done32.store((uint32_t)(seq + 1), std::memory_order_seq_cst);
        if (b->sleepers.load(std::memory_order_seq_cst) > 0) futex_wake_all(&b->done32);
        // ---- PreRequest for the whole batch, off the waiters' path like the reference's (plugin.go:189-194: "Update
        // indexer asynchronously to avoid blocking the request path"); the next flush sees it (or a later one, see
        // epp_config.index_commit_interval_us)
        if (rc == EPP_OK && b->cfg.index_picks) {
            const int32_t rc2 = epp_index_add_picked(b->eng);
            if (rc2 != EPP_OK) {
                std::lock_guard<std::mutex> lk(b->err_mu);
                b->last_error = epp_last_error();
                b->index_errors.fetch_add(1, std::memory_order_relaxed);
            }
        }
    }
}

static int32_t bfail(int32_t code, const char *msg) {
    g_batcher_error = msg;
    return code;
}

extern "C" const char *epp_batcher_last_error(void) { return g_batcher_error.c_str(); }

extern "C" int32_t epp_batcher_create(epp_engine *h, const epp_batcher_cfg *cfg, epp_batcher **out) {
    if (!h || !cfg || !out) return bfail(EPP_ERR_INVALID, "NULL argument");
    *out = nullptr;
    if (cfg->struct_size != sizeof(epp_batcher_cfg)) return bfail(EPP_ERR_INVALID, "epp_batcher_cfg.struct_size mismatch");
    if (cfg->max_batch <= 0 || cfg->max_batch > (1 << 19)) return bfail(EPP_ERR_INVALID, "max_batch out of range [1, 2^19]");
    if (cfg->max_delay_us < 0) return bfail(EPP_ERR_INVALID, "max_delay_us must be >= 0");
    epp_config ec;
    int32_t rc = epp_get_config(h, &ec);
    if (rc != EPP_OK) return bfail(rc, epp_last_error());
    epp_batcher *b = new epp_batcher();
    b->eng = h;
    b->cfg = *cfg;
    // every byte hashPrompt can read: maxPrefixBlocks blocks of blockSizeTokens * 4 bytes (hashing.go:49, 63-66);
    // rows start on 32-byte boundaries (selects the aligned hash kernels)
    b->row_cap = ((uint64_t)ec.max_prefix_blocks * (uint64_t)ec.block_size_tokens * 4 + 31) & ~31ull;
    b->pick_k = ec.pick_k;
    b->max_endpoints = (uint32_t)ec.max_endpoints;
    b->results = std::vector<Result>(kResults);
    const size_t mb = (size_t)cfg->max_batch;
    for (int i = 0; i < kBufs; i++) {
        Staging &st = b->buf[i];
        void *p = nullptr;
        const size_t sizes[7] = {mb * b->row_cap, sizeof(uint64_t) * (mb + 1), sizeof(uint64_t) * mb, sizeof(uint32_t) * mb,
                                 mb, sizeof(epp_decision) * mb, sizeof(epp_decision_detail) * mb};
        void **dst[7] = {(void **)&st.data, (void **)&st.offsets, (void **)&st.lengths, (void **)&st.model_ids,
                         (void **)&st.multimodal, (void **)&st.dec, (void **)&st.det};
        for (int k = 0; k < 7; k++) {
            rc = epp_host_alloc(sizes[k], &p);
            if (rc != EPP_OK) {
                g_batcher_error = epp_last_error();
                epp_batcher_destroy(b);
                return rc;
            }
            *dst[k] = p;
        }
        for (size_t r = 0; r <= mb; r++) st.offsets[r] = (uint64_t)r * b->row_cap;
        st.sub_counts.assign(mb, EPP_SUBSET_ALL);
        st.sub_offsets.resize(mb);
        for (size_t r = 0; r < mb; r++) st.sub_offsets[r] = (uint64_t)r * EPP_SUBSET_MAX_SLOTS;
        st.pred_counts.assign(mb, 0);
        st.pred_offsets.resize(mb);
        for (size_t r = 0; r < mb; r++) st.pred_offsets[r] = (uint64_t)r * EPP_PRED_MAX_SLOTS;
        st.ctx.assign(mb, -1);
        st.priority.assign(mb, 0);
        st.ttft_slo.assign(mb, 0.0);
        st.tpot_slo.assign(mb, 0.0);
        if (b->pick_k > 1)
            for (int q = 0; q < 3; q++) {
                rc = epp_host_alloc(sizeof(uint32_t) * mb * (size_t)b->pick_k, &p);
                if (rc != EPP_OK) {
                    g_batcher_error = epp_last_error();
                    epp_batcher_destroy(b);
                    return rc;
                }
                st.topk[q] = (uint32_t *)p;
            }
    }
    b->flusher = std::thread(flusher_main, b);
    *out = b;
    return EPP_OK;
}

extern "C" int32_t epp_batcher_destroy(epp_batcher *b) {
    if (!b) return EPP_OK;
    b->stop.store(true, std::memory_order_seq_cst);
    wake_flusher(b);
    futex_wake_all(&b->work32);
    if (b->flusher.joinable()) b->flusher.join();            // drains the batch being filled
    futex_wake_all(&b->done32);
    for (int i = 0; i < kBufs; i++) {
        Staging &st = b->buf[i];
        void *ps[10] = {st.data, st.offsets, st.lengths, st.model_ids, st.multimodal, st.dec, st.det, st.topk[0], st.topk[1], st.topk[2]};
        for (void *p : ps) if (p) epp_host_free(p);
    }
    delete b;
    return EPP_OK;
}

// The admission inputs of one request (epp_submit_admit): its entries' validity bytes in the order of its sorted predictions.
struct AdmitIn {
    int32_t priority;
    double ttft_slo, tpot_slo;
    const std::vector<uint8_t> *valid;
};

// sub: the request's slots, sorted and deduplicated, or nullptr (the whole pool); pred: its predictions, validated and
// sorted by slot, or nullptr (none); ctx: its context tokens, -1 = the default; adm: its admission inputs, or nullptr
static int32_t submit_impl(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len, uint32_t multimodal,
                           const std::vector<uint32_t> *sub, uint64_t *out_ticket,
                           const std::vector<epp_prediction> *pred = nullptr, int64_t ctx = -1, const AdmitIn *adm = nullptr) {
    const uint64_t max_batch = (uint64_t)b->cfg.max_batch;
    uint64_t seq, idx;
    for (int spin = 0;; spin++) {
        if (b->stop.load(std::memory_order_acquire)) return bfail(EPP_ERR_STATE, "the batcher is shutting down");
        uint64_t f = b->fill.load(std::memory_order_acquire);
        // full: the flusher is about to close it; or its staging buffer is still in flight (batch seq - 4 not flushed yet)
        if ((f & kCountMask) >= max_batch || (f >> 20) >= b->done.load(std::memory_order_acquire) + kBufs) {
            if (spin == 0) wake_flusher(b);
            if (spin < 200) {
                cpu_relax();
            } else {                                           // sleep until the next flush completes (it frees a batch)
                const uint32_t d = b->done32.load(std::memory_order_seq_cst);
                b->sleepers.fetch_add(1, std::memory_order_seq_cst);
                if (b->fill.load(std::memory_order_seq_cst) == f) {
                    timespec ts{0, 2 * 1000 * 1000};
                    futex_wait(&b->done32, d, &ts);
                }
                b->sleepers.fetch_sub(1, std::memory_order_seq_cst);
            }
            continue;
        }
        if (!b->fill.compare_exchange_weak(f, f + 1, std::memory_order_seq_cst)) continue;
        seq = f >> 20;
        idx = f & kCountMask;
        break;
    }
    Staging &st = b->buf[seq % kBufs];
    if (idx == 0) st.first_arrival_ns.store(now_ns(), std::memory_order_release);
    if (idx == 0 || idx + 1 >= max_batch) wake_flusher(b);
    st.lengths[idx] = prompt_len;                  // the TRUE length: the P/D decider counts it (prefix_based_pd_decider.go:152-167)
    st.model_ids[idx] = model_id;
    st.multimodal[idx] = multimodal ? 1 : 0;
    const uint64_t n_copy = prompt_len < b->row_cap ? prompt_len : b->row_cap;
    if (n_copy) memcpy(st.data + (size_t)idx * b->row_cap, prompt, n_copy);
    if (sub) {
        if (!sub->empty()) memcpy(st.sub_slots.data() + (size_t)idx * EPP_SUBSET_MAX_SLOTS, sub->data(), sizeof(uint32_t) * sub->size());
        st.sub_counts[idx] = (uint32_t)sub->size();
        st.any_subset.store(1, std::memory_order_relaxed);         // published by the release below
    } else {
        st.sub_counts[idx] = EPP_SUBSET_ALL;
    }
    if (pred && !pred->empty()) {
        memcpy(st.pred_entries.data() + (size_t)idx * EPP_PRED_MAX_SLOTS, pred->data(), sizeof(epp_prediction) * pred->size());
        st.pred_counts[idx] = (uint32_t)pred->size();
        st.any_pred.store(1, std::memory_order_relaxed);           // published by the release below
    } else {
        st.pred_counts[idx] = 0;
    }
    st.ctx[idx] = ctx;
    if (ctx != -1) st.any_ctx.store(1, std::memory_order_relaxed);   // published by the release below
    st.priority[idx] = adm ? adm->priority : 0;
    st.ttft_slo[idx] = adm ? adm->ttft_slo : 0.0;
    st.tpot_slo[idx] = adm ? adm->tpot_slo : 0.0;
    if (adm) {
        if (adm->valid && !adm->valid->empty())
            memcpy(st.pred_valid.data() + (size_t)idx * EPP_PRED_MAX_SLOTS, adm->valid->data(), adm->valid->size());
        st.any_adm.store(1, std::memory_order_relaxed);            // published by the release below
    }
    st.ready.fetch_add(1, std::memory_order_release);              // the flusher waits for this before it reads the row
    *out_ticket = (seq << 20) | idx;
    return EPP_OK;
}

extern "C" int32_t epp_submit(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len,
                              uint32_t multimodal, uint64_t *out_ticket) {
    if (!b || !out_ticket || (prompt_len && !prompt)) return bfail(EPP_ERR_INVALID, "NULL argument");
    return submit_impl(b, model_id, prompt, prompt_len, multimodal, nullptr, out_ticket);
}

// A subset's slots checked (every rule epp_schedule_subset applies, bar the engine's kind), sorted and deduplicated into
// *sub, and the subset staging allocated.  Checked here rather than at the flush, where a bad list would fail every
// request of the batch.
static int32_t take_subset(epp_batcher *b, uint32_t n_slots, const uint32_t *slots, std::vector<uint32_t> *sub) {
    if (n_slots > EPP_SUBSET_MAX_SLOTS) return bfail(EPP_ERR_CAPACITY, "more than EPP_SUBSET_MAX_SLOTS slots in one subset");
    sub->assign(slots, slots + n_slots);
    for (uint32_t e : *sub)
        if (e >= b->max_endpoints) return bfail(EPP_ERR_INVALID, "subset slot >= max_endpoints");
    std::sort(sub->begin(), sub->end());
    sub->erase(std::unique(sub->begin(), sub->end()), sub->end());
    std::call_once(b->sub_once, [b] {
        try {
            for (int i = 0; i < kBufs; i++) b->buf[i].sub_slots.resize((size_t)b->cfg.max_batch * EPP_SUBSET_MAX_SLOTS);
        } catch (...) {
            b->sub_alloc_failed = true;
        }
    });
    if (b->sub_alloc_failed) return bfail(EPP_ERR_CAPACITY, "cannot allocate the batcher's subset staging");
    return EPP_OK;
}

// A request's predictions checked with every rule epp_schedule_predicted applies, sorted by slot into *pred, and the
// prediction staging allocated.
static int32_t take_predictions(epp_batcher *b, uint32_t n, const epp_prediction *entries, std::vector<epp_prediction> *pred) {
    if (n > EPP_PRED_MAX_SLOTS) return bfail(EPP_ERR_CAPACITY, "more than EPP_PRED_MAX_SLOTS predictions for one request");
    if (!engine_latency_mask(b->eng) && !(engine_admission(b->eng) & epp::kAdmitLatencySlo))
        return bfail(EPP_ERR_INVALID, "predictions passed to an engine without a latency profile or the latency-slo-admitter");
    pred->assign(entries, entries + n);
    for (const epp_prediction &p : *pred) {
        if (p.slot >= b->max_endpoints) return bfail(EPP_ERR_INVALID, "prediction slot >= max_endpoints");
        if (!std::isfinite(p.ttft) || !std::isfinite(p.ttft_headroom) || !std::isfinite(p.tpot_headroom))
            return bfail(EPP_ERR_INVALID, "a prediction is not finite");
    }
    std::sort(pred->begin(), pred->end(), [](const epp_prediction &x, const epp_prediction &y) { return x.slot < y.slot; });
    for (size_t i = 1; i < pred->size(); i++)
        if ((*pred)[i].slot == (*pred)[i - 1].slot) return bfail(EPP_ERR_INVALID, "two predictions for one slot");
    std::call_once(b->pred_once, [b] {
        try {
            for (int i = 0; i < kBufs; i++) {
                b->buf[i].pred_entries.resize((size_t)b->cfg.max_batch * EPP_PRED_MAX_SLOTS);
                b->buf[i].pred_valid.resize((size_t)b->cfg.max_batch * EPP_PRED_MAX_SLOTS);
            }
        } catch (...) {
            b->pred_alloc_failed = true;
        }
    });
    if (b->pred_alloc_failed) return bfail(EPP_ERR_CAPACITY, "cannot allocate the batcher's prediction staging");
    return EPP_OK;
}

extern "C" int32_t epp_submit_subset(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len,
                                     uint32_t multimodal, uint32_t n_slots, const uint32_t *slots, uint64_t *out_ticket) {
    if (!b || !out_ticket || (prompt_len && !prompt) || (n_slots && !slots)) return bfail(EPP_ERR_INVALID, "NULL argument");
    if (n_slots > EPP_SUBSET_MAX_SLOTS) return bfail(EPP_ERR_CAPACITY, "more than EPP_SUBSET_MAX_SLOTS slots in one subset");
    if (engine_latency_mask(b->eng))
        return bfail(EPP_ERR_INVALID, "endpoint subsets on an engine with latency profiles go through epp_submit_subset_predicted");
    std::vector<uint32_t> sub;
    const int32_t rc = take_subset(b, n_slots, slots, &sub);
    if (rc != EPP_OK) return rc;
    return submit_impl(b, model_id, prompt, prompt_len, multimodal, &sub, out_ticket);
}

extern "C" int32_t epp_submit_predicted(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len,
                                        uint32_t multimodal, uint32_t n, const epp_prediction *entries, uint64_t *out_ticket) {
    if (!b || !out_ticket || (prompt_len && !prompt) || (n && !entries)) return bfail(EPP_ERR_INVALID, "NULL argument");
    std::vector<epp_prediction> pred;
    const int32_t rc = take_predictions(b, n, entries, &pred);
    if (rc != EPP_OK) return rc;
    return submit_impl(b, model_id, prompt, prompt_len, multimodal, nullptr, out_ticket, &pred);
}

extern "C" int32_t epp_submit_subset_predicted(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len,
                                               uint32_t multimodal, uint32_t n_slots, const uint32_t *slots, uint32_t n_pred,
                                               const epp_prediction *entries, uint64_t *out_ticket) {
    if (!b || !out_ticket || (prompt_len && !prompt) || (n_slots && !slots) || (n_pred && !entries))
        return bfail(EPP_ERR_INVALID, "NULL argument");
    std::vector<uint32_t> sub;
    std::vector<epp_prediction> pred;
    int32_t rc = take_subset(b, n_slots, slots, &sub);
    if (rc == EPP_OK) rc = take_predictions(b, n_pred, entries, &pred);
    if (rc != EPP_OK) return rc;
    return submit_impl(b, model_id, prompt, prompt_len, multimodal, &sub, out_ticket, &pred);
}

extern "C" int32_t epp_submit_ctx(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len, uint32_t multimodal,
                                  uint32_t n_slots, const uint32_t *slots, uint32_t n_pred, const epp_prediction *entries,
                                  int64_t context_tokens, uint64_t *out_ticket) {
    if (!b || !out_ticket || (prompt_len && !prompt) || (n_slots && !slots) || (n_pred && !entries))
        return bfail(EPP_ERR_INVALID, "NULL argument");
    if (context_tokens < -1) return bfail(EPP_ERR_INVALID, "context tokens < -1");
    std::vector<uint32_t> sub;
    std::vector<epp_prediction> pred;
    int32_t rc = slots ? take_subset(b, n_slots, slots, &sub) : EPP_OK;
    if (rc == EPP_OK && n_pred) rc = take_predictions(b, n_pred, entries, &pred);
    if (rc != EPP_OK) return rc;
    return submit_impl(b, model_id, prompt, prompt_len, multimodal, slots ? &sub : nullptr, out_ticket, &pred, context_tokens);
}

extern "C" int32_t epp_submit_admit(epp_batcher *b, uint32_t model_id, const void *prompt, uint64_t prompt_len, uint32_t multimodal,
                                    uint32_t n_slots, const uint32_t *slots, uint32_t n_pred, const epp_prediction *entries,
                                    const uint8_t *pred_valid, int64_t context_tokens, int32_t priority, double ttft_slo,
                                    double tpot_slo, uint64_t *out_ticket) {
    if (!b || !out_ticket || (prompt_len && !prompt) || (n_slots && !slots) || (n_pred && !entries))
        return bfail(EPP_ERR_INVALID, "NULL argument");
    if (context_tokens < -1) return bfail(EPP_ERR_INVALID, "context tokens < -1");
    const int32_t admitters = engine_admission(b->eng);
    if (!admitters) return bfail(EPP_ERR_INVALID, "admission inputs passed to an engine without admitters (epp_admission_set)");
    if (n_pred && (admitters & epp::kAdmitLatencySlo) && !pred_valid)
        return bfail(EPP_ERR_INVALID, "pred_valid is NULL: the latency-slo-admitter needs it for a request with predictions");
    if (n_pred > EPP_PRED_MAX_SLOTS) return bfail(EPP_ERR_CAPACITY, "more than EPP_PRED_MAX_SLOTS predictions for one request");
    // the entries and their validity bytes sorted together by slot (take_predictions keeps an ascending list as it is)
    std::vector<uint32_t> order(n_pred);
    for (uint32_t i = 0; i < n_pred; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [entries](uint32_t x, uint32_t y) { return entries[x].slot < entries[y].slot; });
    std::vector<epp_prediction> sorted(n_pred);
    std::vector<uint8_t> valid(n_pred, 0);
    for (uint32_t i = 0; i < n_pred; i++) {
        sorted[i] = entries[order[i]];
        if (pred_valid) valid[i] = pred_valid[order[i]];
    }
    std::vector<uint32_t> sub;
    std::vector<epp_prediction> pred;
    int32_t rc = slots ? take_subset(b, n_slots, slots, &sub) : EPP_OK;
    if (rc == EPP_OK && n_pred) rc = take_predictions(b, n_pred, sorted.data(), &pred);
    if (rc != EPP_OK) return rc;
    const AdmitIn adm{priority, ttft_slo, tpot_slo, &valid};
    return submit_impl(b, model_id, prompt, prompt_len, multimodal, slots ? &sub : nullptr, out_ticket, &pred, context_tokens, &adm);
}

extern "C" int32_t epp_wait(epp_batcher *b, uint64_t ticket, epp_decision *out, epp_decision_detail *out_detail) {
    return epp_wait_topk(b, ticket, out, out_detail, nullptr, nullptr, nullptr);
}

extern "C" int32_t epp_wait_topk(epp_batcher *b, uint64_t ticket, epp_decision *out, epp_decision_detail *out_detail,
                                 uint32_t *primary, uint32_t *prefill, uint32_t *encode) {
    if (!b || !out) return bfail(EPP_ERR_INVALID, "NULL argument");
    if ((primary || prefill || encode) && b->pick_k <= 1) return bfail(EPP_ERR_STATE, "the engine was created with pick_k <= 1: there are no lists");
    const uint64_t seq = ticket >> 20;
    const uint32_t idx = (uint32_t)(ticket & kCountMask);
    {
        const uint64_t f = b->fill.load(std::memory_order_acquire);
        if (seq > (f >> 20) || (seq == (f >> 20) && idx >= (f & kCountMask))) return bfail(EPP_ERR_INVALID, "unknown ticket");
    }
    // a flush is one 30-130 us launch: up to four waiters poll the flush counter for about that long, everybody else
    // (and they, afterwards) sleeps on it -- more pollers than that only take cores away from the flusher
    if (b->done.load(std::memory_order_acquire) <= seq) {
        if (b->spinners.fetch_add(1, std::memory_order_acq_rel) < 4)
            for (int spin = 0; spin < 4000 && b->done.load(std::memory_order_acquire) <= seq; spin++) cpu_relax();
        b->spinners.fetch_sub(1, std::memory_order_acq_rel);
        while (b->done.load(std::memory_order_seq_cst) <= seq) {      // a closing batcher still flushes what is pending
            const uint32_t d = b->done32.load(std::memory_order_seq_cst);
            b->sleepers.fetch_add(1, std::memory_order_seq_cst);
            if (b->done.load(std::memory_order_seq_cst) <= seq) {
                timespec ts{0, 20 * 1000 * 1000};
                futex_wait(&b->done32, d, &ts);
            }
            b->sleepers.fetch_sub(1, std::memory_order_seq_cst);
        }
    }
    Result &res = b->results[seq % kResults];
    res.readers.fetch_add(1, std::memory_order_seq_cst);
    if (res.seq.load(std::memory_order_seq_cst) != seq) {
        res.readers.fetch_sub(1, std::memory_order_seq_cst);
        return bfail(EPP_ERR_STATE, "ticket expired: its batch was flushed more than 4096 flushes ago");
    }
    if ((int32_t)idx >= res.n) {
        res.readers.fetch_sub(1, std::memory_order_seq_cst);
        return bfail(EPP_ERR_INVALID, "unknown ticket");
    }
    const int32_t rc = res.status;
    epp_decision d{};
    epp_decision_detail dd{};
    uint32_t lists[3][64];
    const size_t k = (size_t)b->pick_k, n = (size_t)res.n;
    if (rc == EPP_OK) {
        d = res.dec[idx];
        dd = res.det[idx];
        if (k > 1 && res.topk.size() >= 3 * n * k)
            for (int q = 0; q < 3; q++) memcpy(lists[q], res.topk.data() + ((size_t)q * n + idx) * k, sizeof(uint32_t) * k);
    }
    res.readers.fetch_sub(1, std::memory_order_seq_cst);
    if (rc != EPP_OK) {
        std::lock_guard<std::mutex> lk(b->err_mu);
        g_batcher_error = b->last_error;
        return rc;
    }
    *out = d;
    if (out_detail) *out_detail = dd;
    uint32_t *dst[3] = {primary, prefill, encode};
    for (int q = 0; q < 3; q++)
        if (dst[q]) memcpy(dst[q], lists[q], sizeof(uint32_t) * k);
    return EPP_OK;
}

extern "C" int32_t epp_batcher_stats(epp_batcher *b, epp_batcher_stats_t *out) {
    if (!b || !out) return bfail(EPP_ERR_INVALID, "NULL argument");
    out->n_flushes = b->n_flushes.load(std::memory_order_relaxed);
    out->n_requests = b->n_requests.load(std::memory_order_relaxed);
    out->n_full_flushes = b->n_full.load(std::memory_order_relaxed);
    out->n_pending = b->fill.load(std::memory_order_acquire) & kCountMask;
    out->n_index_errors = b->index_errors.load(std::memory_order_relaxed);
    return EPP_OK;
}
