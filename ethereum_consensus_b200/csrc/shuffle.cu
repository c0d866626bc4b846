// Committee shuffling on the device (SURVEY.md §8f-3): the step immediately BEFORE the BLS hot path — every
// `process_attestation` resolves its committee through `get_beacon_committee`
// (ethereum-consensus/src/phase0/helpers.rs:775-806), which scans the registry for active validators
// (:646-676) and runs the 90-round swap-or-not shuffle (:249-283 per index, :287-360 for a whole list).
//
// Device formulation (not the reference's in-place swap walk, which is inherently sequential):
//   k_shuffle_sources : every SHA-256 the shuffle can need is independent of the data: for each round r the pivot
//                       hash(seed || r) and one "source" block hash(seed || r || le32(b)) per 256 positions —
//                       rounds x (ceil(n/256) + 1) single-block hashes, one thread each (ALU-pipe bound).
//   k_shuffle_map     : one thread per OUTPUT position i runs the forward per-index map of `compute_shuffled_index`
//                       (90 dependent steps: flip, position = max(index, flip), one bit of the source table) and
//                       writes out[i] = indices[map(i)] — exactly `compute_committee`'s definition, and equal to the
//                       list walk `compute_shuffled_indices` produces (tests pin both formulations against each other).
//                       The source table (rounds x n/8 bytes: 11.8 MB at n = 2^20) is L2-resident; the kernel is bound
//                       by dependent L2 gathers, not by HBM.
//   k_active_*        : `get_active_validator_indices` as an order-preserving stream compaction over the 121-byte
//                       Validator records (activation_epoch <= epoch < exit_epoch, phase0/validator.rs:10-26).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>

#include "engine.h"
#include "sha256.cuh"
#include "shuffle.h"

namespace b200 {
namespace {

constexpr int kThreads = 256;

// SHA-256 of seed(32) || extra[0..n_extra) for n_extra <= 5: one padded block
__device__ __forceinline__ void sha256_seed_plus(const uint32_t seed_w[8], uint32_t round, uint32_t pos_block, bool with_pos, uint32_t out[8]) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = seed_w[i];
    if (with_pos) {   // 37 bytes: seed | round | le32(pos_block) | 0x80
        w[8] = (round << 24) | ((pos_block & 0xffu) << 16) | (((pos_block >> 8) & 0xffu) << 8) | ((pos_block >> 16) & 0xffu);
        w[9] = ((pos_block >> 24) << 24) | 0x00800000u;
        w[15] = 37 * 8;
    } else {          // 33 bytes: seed | round | 0x80
        w[8] = (round << 24) | 0x00800000u;
        w[9] = 0;
        w[15] = 33 * 8;
    }
#pragma unroll
    for (int i = 10; i < 15; i++) w[i] = 0;
    sha256_init(out);
    sha256_compress(out, w);
}

// grid covers rounds x (nblk + 1): slot b < nblk -> source block b; slot nblk -> the round's pivot
__global__ void __launch_bounds__(kThreads) k_shuffle_sources(const uint32_t* __restrict__ seed_words, uint32_t rounds, uint32_t nblk,
                                                                uint64_t n, uint32_t* __restrict__ sources, uint64_t* __restrict__ pivots) {
    const uint64_t t = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const uint64_t per = uint64_t(nblk) + 1;
    if (t >= per * rounds) return;
    const uint32_t r = uint32_t(t / per), b = uint32_t(t % per);
    uint32_t sw[8], h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) sw[i] = seed_words[i];
    if (b == nblk) {
        sha256_seed_plus(sw, r, 0, false, h);
        // first 8 digest bytes as a little-endian u64
        const uint64_t v = uint64_t(bswap32(h[0])) | (uint64_t(bswap32(h[1])) << 32);
        pivots[r] = v % n;
    } else {
        sha256_seed_plus(sw, r, b, true, h);
        uint32_t* dst = sources + (uint64_t(r) * nblk + b) * 8;
#pragma unroll
        for (int i = 0; i < 8; i++) dst[i] = h[i];
    }
}

template <class Idx>
__global__ void __launch_bounds__(kThreads) k_shuffle_map(const uint64_t* __restrict__ indices, uint64_t n, uint32_t rounds, uint32_t nblk,
                                                            const uint32_t* __restrict__ sources, const uint64_t* __restrict__ pivots,
                                                            uint64_t* __restrict__ out) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Idx idx = Idx(i);
    const Idx nn = Idx(n);
#pragma unroll 1
    for (uint32_t r = 0; r < rounds; r++) {
        const Idx p = Idx(pivots[r]);
        Idx flip = p + (nn - idx);          // in (0, 2n): fits u32 for n <= 2^31
        if (flip >= nn) flip -= nn;
        const Idx pos = idx > flip ? idx : flip;
        // bit (pos % 8) of digest byte (pos % 256) / 8 of source block pos / 256; digest kept as big-endian words
        const uint32_t word = __ldg(sources + (uint64_t(r) * nblk + uint64_t(pos >> 8)) * 8 + ((uint32_t(pos) & 255u) >> 5));
        const uint32_t byte_in_word = (uint32_t(pos) & 31u) >> 3;
        const uint32_t bit = (word >> (24u - 8u * byte_in_word + (uint32_t(pos) & 7u))) & 1u;
        idx = bit ? flip : idx;
    }
    out[i] = indices ? indices[idx] : uint64_t(idx);
}

__device__ __forceinline__ uint64_t load_le64_unaligned(const uint8_t* p) {
    uint64_t v = 0;
#pragma unroll
    for (int k = 7; k >= 0; k--) v = (v << 8) | p[k];
    return v;
}
// is_active_validator(v, epoch): activation_epoch <= epoch < exit_epoch; record layout phase0/validator.rs:10-26:
// pubkey 0..48, withdrawal_credentials 48..80, effective_balance 80..88, slashed 88, activation_eligibility_epoch 89..97,
// activation_epoch 97..105, exit_epoch 105..113, withdrawable_epoch 113..121
__global__ void __launch_bounds__(kThreads) k_active_count(const uint8_t* __restrict__ recs, uint64_t n, uint64_t epoch,
                                                             uint32_t* __restrict__ block_counts) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    bool act = false;
    if (i < n) {
        const uint8_t* r = recs + i * 121;
        act = load_le64_unaligned(r + 97) <= epoch && epoch < load_le64_unaligned(r + 105);
    }
    const int c = __syncthreads_count(act ? 1 : 0);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = uint32_t(c);
}
// exclusive scan of the per-block counts by one CTA (n_blocks <= a few thousand); total -> block_off[n_blocks]
__global__ void __launch_bounds__(1024) k_active_scan(const uint32_t* __restrict__ block_counts, uint32_t n_blocks, uint64_t* __restrict__ block_off) {
    __shared__ uint64_t part[1024];
    const uint32_t per = (n_blocks + 1023) / 1024;
    const uint32_t lo = threadIdx.x * per, hi = min(n_blocks, lo + per);
    uint64_t s = 0;
    for (uint32_t k = lo; k < hi; k++) s += block_counts[k];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {   // Hillis-Steele inclusive scan
        uint64_t v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    uint64_t run = threadIdx.x ? part[threadIdx.x - 1] : 0;
    for (uint32_t k = lo; k < hi; k++) { block_off[k] = run; run += block_counts[k]; }
    if (threadIdx.x == 1023) block_off[n_blocks] = part[1023];
}
__global__ void __launch_bounds__(kThreads) k_active_scatter(const uint8_t* __restrict__ recs, uint64_t n, uint64_t epoch,
                                                               const uint64_t* __restrict__ block_off, uint64_t* __restrict__ out) {
    __shared__ uint32_t warp_cnt[kThreads / 32];
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    bool act = false;
    if (i < n) {
        const uint8_t* r = recs + i * 121;
        act = load_le64_unaligned(r + 97) <= epoch && epoch < load_le64_unaligned(r + 105);
    }
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t m = __ballot_sync(0xffffffffu, act);
    if (lane == 0) warp_cnt[warp] = __popc(m);
    __syncthreads();
    uint32_t before = 0;
    for (uint32_t w = 0; w < warp; w++) before += warp_cnt[w];
    if (act) out[block_off[blockIdx.x] + before + __popc(m & ((1u << lane) - 1u))] = i;
}

}  // namespace

struct ShuffleScratch {
    DevBuf sources, pivots, seed, idx_in, out, counts, offs, recs;
};
static ShuffleScratch g_sh;

static uint32_t be32h(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }

// out_dev[0..n) = shuffled `idx_dev` (nullptr: identity) on the engine stream; all device pointers
int32_t shuffle_on_device(Engine& e, const uint64_t* idx_dev, uint64_t n, const uint8_t seed[32], uint32_t rounds, uint64_t* out_dev) {
    if (n == 0) return B200_SUCCESS;
    // the block index of a source hash is a u32 and the table is rounds x n / 8 bytes: 2^31 positions (24 GB at 90 rounds) is
    // the ceiling of this formulation, three orders of magnitude above any registry
    if (rounds > 255 || n > (uint64_t(1) << 31)) { e.last_error = "shuffle: more than 255 rounds or 2^31 positions"; return B200_ERR_BAD_ARG; }
    const uint32_t nblk = uint32_t((n + 255) / 256);
    B200_CUDA_TRY(g_sh.sources.reserve(uint64_t(rounds ? rounds : 1) * nblk * 32));
    B200_CUDA_TRY(g_sh.pivots.reserve(256 * 8));
    B200_CUDA_TRY(g_sh.seed.reserve(64));
    B200_CUDA_TRY(e.staging.reserve(64));
    uint32_t* hw = static_cast<uint32_t*>(e.staging.p);
    for (int i = 0; i < 8; i++) hw[i] = be32h(seed + 4 * i);
    cudaStream_t s = e.stream;
    B200_CUDA_TRY(cudaMemcpyAsync(g_sh.seed.p, hw, 32, cudaMemcpyHostToDevice, s));
    B200_CUDA_TRY(cudaStreamSynchronize(s));   // staging is shared scratch: do not let a later call overwrite it in flight
    if (rounds) {
        const uint64_t items = (uint64_t(nblk) + 1) * rounds;
        k_shuffle_sources<<<unsigned((items + kThreads - 1) / kThreads), kThreads, 0, s>>>(
            static_cast<const uint32_t*>(g_sh.seed.p), rounds, nblk, n, static_cast<uint32_t*>(g_sh.sources.p),
            static_cast<uint64_t*>(g_sh.pivots.p));
        e.launches++;
    }
    const unsigned grid = unsigned((n + kThreads - 1) / kThreads);
    k_shuffle_map<uint32_t><<<grid, kThreads, 0, s>>>(idx_dev, n, rounds, nblk, static_cast<const uint32_t*>(g_sh.sources.p),
                                                      static_cast<const uint64_t*>(g_sh.pivots.p), out_dev);
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    return B200_SUCCESS;
}

// out_dev (capacity n) = indices of the active validators, in order; *count_dev-side total copied to *out_n (host)
int32_t active_indices_on_device(Engine& e, const uint8_t* recs_dev, uint64_t n, uint64_t epoch, uint64_t* out_dev, uint64_t* out_n) {
    *out_n = 0;
    if (n == 0) return B200_SUCCESS;
    const uint32_t n_blocks = uint32_t((n + kThreads - 1) / kThreads);
    B200_CUDA_TRY(g_sh.counts.reserve(uint64_t(n_blocks) * 4 + 16));
    B200_CUDA_TRY(g_sh.offs.reserve(uint64_t(n_blocks + 1) * 8 + 16));
    B200_CUDA_TRY(e.staging.reserve(64));
    cudaStream_t s = e.stream;
    k_active_count<<<n_blocks, kThreads, 0, s>>>(recs_dev, n, epoch, static_cast<uint32_t*>(g_sh.counts.p));
    k_active_scan<<<1, 1024, 0, s>>>(static_cast<const uint32_t*>(g_sh.counts.p), n_blocks, static_cast<uint64_t*>(g_sh.offs.p));
    k_active_scatter<<<n_blocks, kThreads, 0, s>>>(recs_dev, n, epoch, static_cast<const uint64_t*>(g_sh.offs.p), out_dev);
    e.launches += 3;
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaMemcpyAsync(e.staging.p, static_cast<const uint64_t*>(g_sh.offs.p) + n_blocks, 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA_TRY(cudaStreamSynchronize(s));
    *out_n = *static_cast<const uint64_t*>(e.staging.p);
    return B200_SUCCESS;
}

int32_t shuffle_scratch(Engine& e, uint64_t n, uint64_t** a, uint64_t** b) {
    B200_CUDA_TRY(g_sh.idx_in.reserve(n * 8 + 64));
    B200_CUDA_TRY(g_sh.out.reserve(n * 8 + 64));
    *a = static_cast<uint64_t*>(g_sh.idx_in.p);
    *b = static_cast<uint64_t*>(g_sh.out.p);
    return B200_SUCCESS;
}

}  // namespace b200

using namespace b200;

extern "C" {

int32_t b200_compute_shuffled_indices(const uint64_t* indices, size_t n, const uint8_t seed[32], uint32_t rounds, uint64_t* out) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    if (!e.ready) { e.last_error = "b200_init has not been called (or failed)"; return B200_ERR_NOT_INITIALIZED; }
    if (!seed || (n && !out)) return B200_ERR_BAD_ARG;
    if (n == 0) return B200_SUCCESS;
    B200_CUDA_TRY(cudaSetDevice(e.device));
    uint64_t *d_in, *d_out;
    int32_t rc = shuffle_scratch(e, n, &d_in, &d_out);
    if (rc) return rc;
    B200_CUDA_TRY(cudaEventRecord(e.ev0, e.stream));
    if (indices) B200_CUDA_TRY(cudaMemcpyAsync(d_in, indices, n * 8, cudaMemcpyHostToDevice, e.stream));
    rc = shuffle_on_device(e, indices ? d_in : nullptr, n, seed, rounds, d_out);
    if (rc) return rc;
    B200_CUDA_TRY(cudaEventRecord(e.ev1, e.stream));
    B200_CUDA_TRY(cudaMemcpyAsync(out, d_out, n * 8, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, e.ev0, e.ev1));
    return B200_SUCCESS;
}

int32_t b200_get_active_validator_indices(const uint8_t* validators_ssz, size_t n, uint64_t epoch, uint64_t* out, size_t* out_n) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    if (!e.ready) { e.last_error = "b200_init has not been called (or failed)"; return B200_ERR_NOT_INITIALIZED; }
    if (!out_n || (n && (!validators_ssz || !out))) return B200_ERR_BAD_ARG;
    *out_n = 0;
    if (n == 0) return B200_SUCCESS;
    B200_CUDA_TRY(cudaSetDevice(e.device));
    uint64_t *d_in, *d_out;
    int32_t rc = shuffle_scratch(e, n, &d_in, &d_out);
    if (rc) return rc;
    B200_CUDA_TRY(g_sh.recs.reserve(n * 121 + 64));
    B200_CUDA_TRY(cudaMemcpyAsync(g_sh.recs.p, validators_ssz, n * 121, cudaMemcpyHostToDevice, e.stream));
    uint64_t cnt = 0;
    rc = active_indices_on_device(e, static_cast<const uint8_t*>(g_sh.recs.p), n, epoch, d_out, &cnt);
    if (rc) return rc;
    if (cnt) B200_CUDA_TRY(cudaMemcpy(out, d_out, cnt * 8, cudaMemcpyDeviceToHost));
    *out_n = size_t(cnt);
    return B200_SUCCESS;
}

}  // extern "C"
