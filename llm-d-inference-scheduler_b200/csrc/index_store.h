// index_store.h -- the WRITE side of the prefix index, resident in HBM (SURVEY.md 8(f).1):
//   indexer.Add + per-server LRU eviction   approximateprefix/indexer.go:52-83, 105-115
//   indexer.RemovePod                        approximateprefix/indexer.go:167-182
//   PreRequest (index the picks of a batch)  approximateprefix/plugin.go:164-200
//
// The reference keeps, per server, a golang-lru (v2.0.7) cache of block hashes and an inverted map hash -> podSet that
// the cache's eviction callback prunes.  With Add as the only operation that touches recency (Get never does), the
// cache content after any sequence of Adds is "the C most recently added distinct hashes"; a batch of Add calls is
// therefore applied in parallel:
//
//   pair table   open-addressed (hash, endpoint) -> {seq of the latest Add, in_map}; 32-byte entries, one sector
//   endpoint log per endpoint, append-only in Add order: (hash, seq).  An entry is LIVE iff the pair table still holds
//                its seq; eviction walks the log from the tail and removes the oldest live entries until the endpoint
//                is back at its capacity -- O(evicted + stale), never O(index)
//   sequencing   seq of item i of call c = next_seq[ep] + (items of earlier calls of the batch for the same endpoint)
//                + i, from a per-chunk histogram and an ordered scan, so "most recent" means exactly what it means
//                when the calls run one after another
//
// One corner of the reference is kept bit for bit: a single Add of MORE hashes than the LRU holds evicts hashes of the
// same call and then re-inserts them into the inverted map (indexer.go:76-83) without putting them back into the LRU;
// such pairs stay visible to Get until the hash is added again and evicted normally -- they survive RemovePod too.
// They are the LEAKED pairs below (in_map = 1, seq = 0).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "devbuf.h"
#include "kernels.h"

namespace epp {

constexpr uint32_t kNoEp = 0xFFFFFFFFu;

// A batch of indexer.Add calls in the order the reference would run them (device arrays).
struct StoreCalls {
    uint32_t M = 0;
    const uint32_t *ep = nullptr;     // [M] endpoint slot; kNoEp = the call does not happen
    const uint32_t *n = nullptr;      // [M] number of hashes of the call (0 still creates the endpoint's LRU)
    const int32_t *nb = nullptr;      // [M] NumOfGPUBlocks argument: LRU size if this call creates it (<= 0: default)
    const uint64_t *src = nullptr;    // [M] index of the call's first hash in `hashes`
    const uint64_t *hashes = nullptr;
};

// What patch_read_table needs to know about the read table (index_kernels.cu layout, owned by the engine).
struct ReadTableRef {
    IndexSlot *slots = nullptr;
    uint64_t capacity = 0;        // power of two
    uint64_t slots_used = 0;      // claimed keys incl. tombstones
    uint32_t *postings = nullptr;
    uint64_t post_cap = 0;        // allocated posting entries
    uint64_t post_used = 0;       // posting entries handed out so far
    uint32_t *head = nullptr;     // device: [capacity], all 0xFFFFFFFF between patches
    uint64_t *intern_keys = nullptr;
    uint32_t *intern_vals = nullptr;
    uint64_t intern_used = 0;     // claimed keys of the interning table, retired ones included (`capacity` entries)
    uint32_t *presence = nullptr; // presence bitmap (index.cuh): the patch sets the bits of keys whose list is not empty
    int32_t presence_shift = 0;
};

class IndexStore {
  public:
    // sm_count: SMs of the engine's device; sizes the persistent grids of the compaction and eviction kernels.
    IndexStore(uint32_t max_endpoints, int32_t default_lru_size, int sm_count)
        : E_(max_endpoints), default_cap_(default_lru_size), sm_count_(sm_count > 0 ? sm_count : 1) {}

    // Applies the calls (Add + eviction).  Synchronises `s` (two small read-backs size the tables).
    cudaError_t apply(const StoreCalls &calls, cudaStream_t s);
    // PreRequest for a scheduled batch: call 2r = (pick_r, hashes of r), call 2r+1 = (prefill_pick_r, same hashes).
    cudaError_t apply_picks(const epp_decision *decisions, const uint64_t *hashes, const int32_t *nblocks, int64_t R,
                            int32_t max_blocks, cudaStream_t s);
    cudaError_t remove_endpoint(uint32_t ep, cudaStream_t s);
    // CleanUpInactivePods: active_dev[e] != 0 keeps endpoint e (device array of max_endpoints bytes).
    cudaError_t retain_endpoints(const uint8_t *active_dev, cudaStream_t s);
    cudaError_t clear(cudaStream_t s);
    // Every (hash, endpoint) pair of the inverted map, for the bulk build of the read table.
    // Incremental read-table maintenance from the log of changed (hash, endpoint) pairs (see index_store.cu).
    cudaError_t patch_read_table(const ReadTableRef &rt, uint64_t table_pairs, cudaStream_t s, bool *patched,
                                 uint64_t *new_pairs, uint64_t *new_slots_used, uint64_t *new_post_used,
                                 uint64_t *new_intern_used);
    cudaError_t touch_reset(cudaStream_t s);
    uint64_t last_patch_touches = 0, last_patch_dirty = 0;
    cudaError_t export_pairs(DevBuf &pair_hash, DevBuf &pair_ep, uint64_t *n_pairs, size_t *accounted, cudaStream_t s);

    bool dirty() const { return dirty_; }
    void mark_clean() { dirty_ = false; }
    bool empty() const { return !used_; }
    uint64_t pairs_in_map() const { return in_map_; }
    size_t device_bytes() const { return bytes_; }
    struct View;                       // device pointers handed to the kernels (index_store.cu)
    // launch / timing record of the last apply() for stats and the bench
    int last_launches = 0;
    uint64_t last_items = 0;
    bool last_repacked = false, last_rehashed = false;

  private:
    cudaError_t ensure_init(cudaStream_t s);
    cudaError_t grow_pair_table(uint64_t incoming, cudaStream_t s);
    cudaError_t repack_logs(cudaStream_t s);
    cudaError_t reserve_touch(uint64_t more, cudaStream_t s);
    void fill_view(View &v) const;

    uint32_t E_;
    int32_t default_cap_;
    int sm_count_;
    bool init_ = false, dirty_ = false, used_ = false;
    size_t bytes_ = 0;
    uint64_t pt_cap_ = 0, log_cap_ = 0, in_map_ = 0, pt_used_ = 0;
    DevBuf pt_, log_hash_, log_seq_;
    DevBuf pt_spare_, log_hash_spare_, log_seq_spare_;   // the previous generation of the three big buffers: rehash / repack
                                                          // ping-pong between the pairs instead of cudaMalloc + cudaFree
    DevBuf cap_, live_, firstcall_, seg_off_, seg_cap_, head_, tail_, inc_, next_seq_, sp_seq_, sp_in_map_, ctr_;
    DevBuf hist_, off_, new_off_, new_cap_, cut_, blockcnt_, blockmask_, list_e_, list_start_;
    // touch log + scratch of patch_read_table
    DevBuf touch_hash_, touch_ep_, patch_next_, patch_dirty_;
    uint64_t touch_cap_ = 0, touch_upper_ = 0;      // allocated entries; host upper bound of the entries logged so far
    bool touch_disabled_ = false;                   // too many changes to log: the next commit rebuilds
    DevBuf call_ep_, call_n_, call_nb_, call_src_;
    std::vector<uint64_t> h_live_, h_inc_, h_off_, h_cap_;
    unsigned long long *ctr_host_ = nullptr;   // pinned
};

}  // namespace epp
