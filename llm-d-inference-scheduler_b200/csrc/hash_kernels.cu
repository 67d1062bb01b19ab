// hash_kernels.cu -- a1: batched chained XXH64 prefix-block hashing (approximateprefix/hashing.go:35-99): the dispatcher
// and the generic path.
//   launch_hash_prompts : block sizes that are a multiple of 32 bytes + 16-byte aligned prompts (every BASELINE
//                         config) -> hash_fused.cu; anything else -> the two kernels below
//   k_prompt_lengths    : per request, truncation + block count                     (hashing.go:58-66)
//   k_hash_generic      : any block size / alignment, one thread per request, fully serial
//   k_hash_bytes        : XXH64 of one message (the model || salt seed, hashing.go:71-78)
#include "kernels.h"
#include "xxh64.cuh"

namespace epp {

__device__ __forceinline__ void request_span(const HashParams &p, int64_t r, uint64_t &off, uint64_t &len) {
    if (p.offsets) {
        off = p.offsets[r];
        len = p.lengths ? p.lengths[r] : p.offsets[r + 1] - off;
    } else {
        off = (uint64_t)r * p.uniform_len;
        len = p.uniform_len;
    }
}

__global__ void k_hash_bytes(const uint8_t *msg, size_t len, uint64_t *out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint64_t v[4];
    bool have_v = false;
    size_t i = 0;
    if (len >= 32) {
        xxh_init(v);
        have_v = true;
        for (; i + 32 <= len; i += 32) {
            v[0] = xxh_round(v[0], load_le64(msg + i));
            v[1] = xxh_round(v[1], load_le64(msg + i + 8));
            v[2] = xxh_round(v[2], load_le64(msg + i + 16));
            v[3] = xxh_round(v[3], load_le64(msg + i + 24));
        }
    }
    uint8_t tail[32];
    int t = 0;
    for (; i < len; i++) tail[t++] = msg[i];
    *out = xxh_finish(v, have_v, (uint64_t)len, tail, t);
}

cudaError_t launch_hash_bytes(const uint8_t *msg, size_t len, uint64_t *out, cudaStream_t s) {
    k_hash_bytes<<<1, 32, 0, s>>>(msg, len, out);
    return cudaGetLastError();
}

__global__ void k_prompt_lengths(HashParams p) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= p.R) return;
    uint64_t off, len;
    request_span(p, r, off, len);
    if (p.in_len) p.in_len[r] = (int64_t)len;
    int64_t bs = p.block_bytes;
    int64_t eff = (int64_t)len;
    int32_t nb = 0;
    if (bs <= 0 || eff < bs) {            // hashing.go:51-61 -> nil
        eff = 0;
    } else {
        int64_t cap = bs * (int64_t)p.max_blocks;
        if (eff > cap) eff = cap;         // hashing.go:63-66
        nb = (int32_t)(eff / bs) + ((eff % bs) ? 1 : 0);
    }
    p.nblocks[r] = nb;
    p.eff_len[r] = eff;
}

__global__ void __launch_bounds__(128) k_hash_generic(HashParams p) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= p.R) return;
    int32_t nb = p.nblocks[r];
    if (nb == 0) return;
    int64_t eff = p.eff_len[r];
    int64_t bs = p.block_bytes;
    uint64_t off, len;
    request_span(p, r, off, len);
    const uint8_t *base = p.data + off;
    uint64_t prev = p.seeds[p.model_ids ? p.model_ids[r] : 0];
    uint64_t *row = p.hashes + r * (int64_t)p.max_blocks;
    for (int32_t b = 0; b < nb; b++) {
        int64_t start = (int64_t)b * bs;
        int64_t n = eff - start < bs ? eff - start : bs;
        prev = hash_block_generic(base + start, n, prev);
        row[b] = prev;
    }
}

// Common alignment (0, 16 or 32 bytes) of every block start of the batch; the vectorised paths need
// block_bytes % 32 == 0 and alignment >= 16 (128-bit loads).
int hash_batch_alignment(const HashParams &p) {
    if (p.block_bytes <= 0 || (p.block_bytes % 32) != 0) return 0;
    uint64_t bits = reinterpret_cast<uintptr_t>(p.data);
    bits |= p.offsets ? p.offsets_or_bits : p.uniform_len;
    if ((bits & 31) == 0) return 32;
    if ((bits & 15) == 0) return 16;
    return 0;
}
// *flag |= low bits of every offset (device-pointer batches).
__global__ void k_offsets_aligned(const uint64_t *offsets, int64_t n, int *flag) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n && (offsets[r] & 31)) atomicOr(flag, (int)(offsets[r] & 31));
}
cudaError_t launch_check_offsets_aligned(const uint64_t *offsets, int64_t n, int *flag_dev, cudaStream_t s) {
    k_offsets_aligned<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(offsets, n, flag_dev);
    return cudaGetLastError();
}

cudaError_t launch_hash_fused(const HashParams &p, int sm_count, cudaStream_t s, int *launches);

bool hash_fused_selected(const HashParams &p) {
    return hash_batch_alignment(p) >= 16;
}

// ev (optional, 4 events): recorded around the hash kernel(s): [1]..[2] brackets the kernel that reads the prompt bytes.
cudaError_t launch_hash_prompts(const HashParams &p, cudaStream_t s, int *launches, cudaEvent_t *ev) {
    if (p.R <= 0) return cudaSuccess;
    if (hash_fused_selected(p)) {               // one kernel: lengths + digests + chain
        if (ev) { cudaEventRecord(ev[0], s); cudaEventRecord(ev[1], s); }
        cudaError_t e = launch_hash_fused(p, p.sm_count, s, launches);
        if (ev) { cudaEventRecord(ev[2], s); cudaEventRecord(ev[3], s); }
        return e;
    }
    const unsigned gR = (unsigned)((p.R + 127) / 128);
    if (ev) { cudaEventRecord(ev[0], s); cudaEventRecord(ev[1], s); }
    k_prompt_lengths<<<gR, 128, 0, s>>>(p);
    k_hash_generic<<<gR, 128, 0, s>>>(p);
    if (ev) { cudaEventRecord(ev[2], s); cudaEventRecord(ev[3], s); }
    if (launches) *launches += 2;
    return cudaGetLastError();
}

}  // namespace epp
