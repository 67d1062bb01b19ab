// cycle_small.cu -- the whole scheduling cycle (a1-a14) of a SMALL host batch as ONE kernel launch that writes the
// decisions straight into pinned host memory: no copy back, no stream synchronisation -- the host polls one flag word
// per request.  The prompts of a handful of requests are read straight from the caller's pinned memory over PCIe (no
// copy engine at all); a larger batch is DMA-copied into HBM on the engine's second stream while this kernel, launched
// at the same time, waits for the word the copy stream writes behind the copy (SmallOut::arrive).
// This is the latency path of the micro-batcher (csrc/batcher.cu): a flush of 1 .. 1024 requests.
//
// One CTA per request, 9 warps:
//   thread 0   stages the prompt: ONE cp.async.bulk (TMA) + mbarrier brings all its full blocks -- 16 KiB for a 4 096-token
//              prompt -- into shared memory, from HBM or straight from the caller's pinned host memory over PCIe;
//   warps 0-7  digest: every thread hashes the 32-byte stripes of "its" blocks out of shared memory and leaves the merged
//              stripe state of each FULL block there (256 blocks = one per thread);
//   warp 8     chain: ONE lane walks the blocks in order (the serial part of hashPrompt, hashing.go:80-96; five
//              dependent 64-bit multiplies per block), stores every hash to the request's row in HBM (the stash
//              PreRequest needs) and over the block's stripe state in shared memory, and publishes its progress there
//              every 32 blocks (no global fence on the critical path);
//   warp 1     match: after its digests, runs sparse::match_request in FOLLOW mode -- it probes the index 32 blocks at
//              a time as soon as the chain has produced them, so the table and posting-list latencies hide under the
//              chain, and the global-stop rule (plugin.go:219-223) lets it decide a cold prompt after the first chunk
//              while the chain is still hashing.  It then copies the decision to host memory and raises the flag.
// Every prompt byte is consumed before the chain starts (the trailing partial block is parked in shared memory by the idle
// chain warp): once a request's flag is up, its input may be overwritten.
// The critical path is the chain (256 dependent blocks for a 16 KiB prompt) + one PCIe round trip each way.
#include "hash_blocks.cuh"
#include "match_sparse.cuh"

namespace epp {

namespace {
constexpr int kDigestThreads = 256;
constexpr int kThreads = kDigestThreads + 32;

// Hand-over of the hashes from the chain lane to the match warp: plain shared-memory stores published by a release
// store of the progress word, consumed behind an acquire load (CTA scope).  compute-sanitizer's racecheck models
// barriers only and reports this flag protocol as hazards.
__device__ __forceinline__ void st_release_cta(int32_t *p, int32_t v) {
    asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(p)), "r"(v) : "memory");
}
__device__ __forceinline__ int32_t ld_acquire_cta(const int32_t *p) {
    int32_t v;
    asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(v) : "r"((uint32_t)__cvta_generic_to_shared(p)) : "memory");
    return v;
}
// Poll word written by the copy stream (device memory, so L2 is the point of coherence).  Relaxed on purpose: an acquire at
// system scope is a MEMBAR.SYS per poll, and a thousand CTAs issuing those while the copy engine streams the prompts in
// slow it down; one GPU-scope fence after the wait orders the reads behind it.
__device__ __forceinline__ uint32_t ld_relaxed_gpu(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// ---- bulk-copy (TMA) staging of the request's prompt: one cp.async.bulk brings all its full blocks into shared memory
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *b, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *b, uint32_t tx) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(tx) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *b, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(b)), "r"(parity)
            : "memory");
    } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// Stripe rounds + merge of one full block whose bytes are in shared memory (part A of xxh64.cuh).
__device__ __forceinline__ uint64_t block_digest_smem(const uint8_t *src, int n_stripes) {
    uint64_t v[4];
    xxh_init(v);
    const uint32_t a = smem_u32(src);
    for (int st = 0; st < n_stripes; st++) {
        uint64_t x[4];
        asm volatile("ld.shared.v2.u64 {%0,%1}, [%2];" : "=l"(x[0]), "=l"(x[1]) : "r"(a + 32u * st));
        asm volatile("ld.shared.v2.u64 {%0,%1}, [%2];" : "=l"(x[2]), "=l"(x[3]) : "r"(a + 32u * st + 16u));
#pragma unroll
        for (int q = 0; q < 4; q++) v[q] = xxh_round(v[q], x[q]);
    }
    return xxh_merge_all(v);
}

struct ChainFollower {
    static constexpr bool kOn = true;
    const int32_t *progress;                   // hashes [0, *progress) are in `h`
    const uint64_t *h;                         // shared memory: the chain overwrites every stripe state with the block's hash
    __device__ __forceinline__ void wait(int32_t n) const {
        while (ld_acquire_cta(progress) < n) {}
    }
    __device__ __forceinline__ uint64_t hash(int32_t i) const { return h[i]; }
};

// kStage: the prompt is staged into shared memory by ONE bulk copy (TMA) per request; else the digest threads load their
// blocks themselves (prompts too long for the staging buffer).
// kNoHit: a profile has the no-hit-lru scorer (match_sparse.cuh match_request); those engines launch k_cycle_small_nohit.
// kRand: some profile has a random picker (k_cycle_small_rand, which also carries the no-hit-lru logic).
template <bool kStage, bool kNoHit, bool kRand = false>
__device__ __forceinline__ void cycle_small(const HashParams &hp, const PickParams &pp, const SmallOut &so, uint32_t stage_off) {
    extern __shared__ __align__(128) uint64_t s_m[];   // [max_blocks] merged stripe state of every full block; then, at byte
                                                       // stage_off, (kStage) the prompt's full blocks and its trailing partial block
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ uint64_t s_off;
    __shared__ int64_t s_eff;
    __shared__ int32_t s_nfull, s_nb;
    __shared__ int32_t s_progress;                 // hashes [0, s_progress) are in s_m (release / acquire, CTA scope)
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int64_t r = blockIdx.x;
    const int64_t bs = hp.block_bytes;

    if (t == 0) {                                  // hashing.go:58-66 (the same arithmetic as tile_lengths, hash_fused.cu)
        uint64_t off, len;
        if (hp.offsets) { off = hp.offsets[r]; len = hp.lengths ? hp.lengths[r] : hp.offsets[r + 1] - off; }
        else { off = (uint64_t)r * hp.uniform_len; len = hp.uniform_len; }
        int64_t eff = (int64_t)len;
        int32_t nfull = 0, nb = 0;
        if (eff < bs) {
            eff = 0;
        } else {
            const int64_t cap = bs * (int64_t)hp.max_blocks;
            if (eff > cap) eff = cap;
            nfull = (int32_t)(eff / bs);
            nb = nfull + ((eff % bs) ? 1 : 0);
        }
        if (hp.in_len) hp.in_len[r] = (int64_t)len;
        hp.nblocks[r] = nb;
        hp.eff_len[r] = eff;
        s_off = off; s_eff = eff; s_nfull = nfull; s_nb = nb;
        s_progress = 0;
        __threadfence();                           // the match warp reads nblocks / in_len at L2
        if (so.arrive) {                           // the prompts may still be in flight: wait for the copy that carries them
            while (ld_relaxed_gpu(so.arrive) != so.epoch) __nanosleep(100);
            __threadfence();
        }
        if (kStage) {
            mbar_init(&s_bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("fence.proxy.async;" ::: "memory");        // barrier init (shared) and, behind `arrive`, the copied prompt (global)
            if (nfull > 0) {                       // every full block of the prompt in one transaction (16-byte aligned, size % 32 == 0)
                const uint32_t bytes = (uint32_t)nfull * (uint32_t)bs;
                mbar_arrive_expect_tx(&s_bar, bytes);
                bulk_g2s(reinterpret_cast<uint8_t *>(s_m) + stage_off, hp.data + off, bytes, &s_bar);
            }
        }
    }
    __syncthreads();
    const int32_t nfull = s_nfull;
    if (warp < kDigestThreads / 32) {
        const int n_stripes = (int)(bs >> 5);
        if (kStage) {
            if (nfull > 0) {
                mbar_wait(&s_bar, 0);
                const uint8_t *base = reinterpret_cast<const uint8_t *>(s_m) + stage_off;
                for (int32_t b = t; b < nfull; b += kDigestThreads)
                    s_m[b] = block_digest_smem(base + (size_t)b * (size_t)bs, n_stripes);
            }
        } else {
            const uint8_t *base = hp.data + s_off;
            for (int32_t b = t; b < nfull; b += kDigestThreads)
                s_m[b] = block_digest(base + (uint64_t)b * (uint64_t)bs, n_stripes);
        }
    } else if (warp == kDigestThreads / 32) {
        // The trailing partial block is hashed LAST, long after a cold request may have raised its flag (global stop), and
        // the caller -- or the next batch's copy into the staging buffer -- may rewrite the prompt bytes from then on: the
        // chain warp, idle until the digests are done, brings them into shared memory now (behind the full blocks of the
        // staged prompt, else behind the stripe states).
        const int64_t tail_n = s_eff - (int64_t)nfull * bs;
        if (tail_n > 0) {
            const uint8_t *src = hp.data + s_off + (uint64_t)nfull * (uint64_t)bs;
            uint8_t *dst = reinterpret_cast<uint8_t *>(s_m) + stage_off + (kStage ? (size_t)nfull * (size_t)bs : 0);
            const int64_t n16 = tail_n >> 4;       // rows and blocks are 16-byte aligned on this path
            for (int64_t i = lane; i < n16; i += 32)
                reinterpret_cast<uint4 *>(dst)[i] = reinterpret_cast<const uint4 *>(src)[i];
            for (int64_t i = (n16 << 4) + lane; i < tail_n; i += 32) dst[i] = src[i];
        }
    }
    __syncthreads();                               // the prompt bytes are consumed: nothing below reads host input data

    if (warp == kDigestThreads / 32) {
        if (lane == 0 && s_nb > 0) {
            uint64_t prev = hp.seeds[hp.model_ids ? hp.model_ids[r] : 0];
            uint64_t *row = hp.hashes + r * (int64_t)hp.max_blocks;
            const uint64_t lenp8 = (uint64_t)bs + 8;
            uint64_t *sh = s_m;
            int32_t b = 0;
            for (; b + 32 <= nfull; b += 32) {     // 32 blocks per hand-over, nothing but the dependent multiplies inside
#pragma unroll 8
                for (int j = 0; j < 32; j++) {
                    prev = xxh_chain_step32_lat(s_m[b + j], lenp8, prev);
                    row[b + j] = prev;             // the stash PreRequest reads (stream-ordered, after this kernel)
                    sh[b + j] = prev;              // what the match warp of this CTA reads
                }
                st_release_cta(&s_progress, b + 32);
            }
            for (; b < nfull; b++) {
                prev = xxh_chain_step32_lat(s_m[b], lenp8, prev);
                row[b] = prev;
                sh[b] = prev;
            }
            if ((int64_t)nfull * bs < s_eff) {     // trailing partial block (hashing.go:90-96)
                const uint8_t *tail = reinterpret_cast<const uint8_t *>(s_m) + stage_off + (kStage ? (size_t)nfull * (size_t)bs : 0);
                prev = hash_block_generic(tail, s_eff - (int64_t)nfull * bs, prev);
                row[nfull] = prev;
                sh[nfull] = prev;
            }
            st_release_cta(&s_progress, s_nb);
        }
        return;
    }
    if (warp != 1) return;                         // not warp 0: that one shares its scheduler with the chain warp (8 % 4)

    int32_t unused = 0;
    const ChainFollower fw{&s_progress, s_m};
    const bool decided = sparse::match_request<true, false, true, 3, ChainFollower, kNoHit, kRand>(pp, r, lane, false, nullptr, nullptr, unused, fw);
    if (lane == 0) {
        if (decided) {
            so.dec[r] = pp.out[r];
            so.det[r] = pp.detail[r];
        }
        __threadfence_system();
        *reinterpret_cast<volatile uint32_t *>(so.flags + r) = decided ? so.epoch : (so.epoch | 0x80000000u);
    }
}

template <bool kStage>
__global__ void __launch_bounds__(kThreads) k_cycle_small(HashParams hp, PickParams pp, SmallOut so, uint32_t stage_off) {
    cycle_small<kStage, false>(hp, pp, so, stage_off);
}
template <bool kStage>
__global__ void __launch_bounds__(kThreads) k_cycle_small_nohit(HashParams hp, PickParams pp, SmallOut so, uint32_t stage_off) {
    cycle_small<kStage, true>(hp, pp, so, stage_off);
}
template <bool kStage>
__global__ void __launch_bounds__(kThreads) k_cycle_small_rand(HashParams hp, PickParams pp, SmallOut so, uint32_t stage_off) {
    cycle_small<kStage, true, true>(hp, pp, so, stage_off);
}
}  // namespace

size_t cycle_small_max_blocks() { return 8192; }   // 64 KiB of stripe states per CTA

bool cycle_small_stages_prompt(int32_t max_blocks, int32_t block_bytes) {
    const size_t m_bytes = (sizeof(uint64_t) * (size_t)max_blocks + 127) & ~(size_t)127;
    return m_bytes + (size_t)max_blocks * (size_t)block_bytes <= 160 * 1024;
}

cudaError_t launch_cycle_small(const HashParams &hp, const PickParams &pp, const SmallOut &so, cudaStream_t s,
                               int *launches) {
    if (hp.R <= 0) return cudaSuccess;
    const size_t m_bytes = (sizeof(uint64_t) * (size_t)hp.max_blocks + 127) & ~(size_t)127;
    const size_t stage_bytes = (size_t)hp.max_blocks * (size_t)hp.block_bytes;
    const bool stage = cycle_small_stages_prompt(hp.max_blocks, hp.block_bytes);   // longer prompts: the digest threads load their blocks themselves
    const size_t smem = m_bytes + (stage ? stage_bytes : (size_t)hp.block_bytes);     // unstaged: room for the trailing partial block
    if (smem > 160 * 1024) return cudaErrorInvalidValue;
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_set[64] = {};                 // function attributes are per device: engines of one process may sit on several GPUs
    if (!attr_set[dev & 63]) {
        cudaError_t e = cudaFuncSetAttribute(k_cycle_small<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cycle_small<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cycle_small_nohit<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cycle_small_nohit<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cycle_small_rand<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cycle_small_rand<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        if (e != cudaSuccess) return e;
        attr_set[dev & 63] = true;
    }
    const unsigned grid = (unsigned)hp.R;
    const uint32_t off = (uint32_t)m_bytes;
    if (any_random_picker(pp)) {                   // random-picker builds (match_sparse.cuh eval_random_lanes)
        if (stage) k_cycle_small_rand<true><<<grid, kThreads, smem, s>>>(hp, pp, so, off);
        else k_cycle_small_rand<false><<<grid, kThreads, smem, s>>>(hp, pp, so, off);
    } else if (pp.nohit.mask) {                    // no-hit-lru builds (match_sparse.cuh match_request)
        if (stage) k_cycle_small_nohit<true><<<grid, kThreads, smem, s>>>(hp, pp, so, off);
        else k_cycle_small_nohit<false><<<grid, kThreads, smem, s>>>(hp, pp, so, off);
    } else if (stage) {
        k_cycle_small<true><<<grid, kThreads, smem, s>>>(hp, pp, so, off);
    } else {
        k_cycle_small<false><<<grid, kThreads, smem, s>>>(hp, pp, so, off);
    }
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace epp
