// Integer-pipe peak microbenchmarks: the roofline denominators for the two hot paths, MEASURED on the GPU the bench
// runs on.  kind 0: IMAD.WIDE.U32 (32x32+64, the Montgomery
// multiply-add), kind 1: IMAD.U32 lo, kind 2: LOP3/SHF/IADD3 mix (the SHA-256 round ops), all dependency-limited
// only by 8 independent chains per thread with the SMs fully occupied.
// kind 7 / 8 (round 2): IMAD.WIDE.U32 whose multiplicand is the low word of ANOTHER chain's accumulator, multiplier in a
// register (7) or an immediate (8), instead of the addend's own low word — kind 0 reads its 64-bit accumulator pair as BOTH a source and the addend, which a profile
// showed saturating below the pipe's real issue rate (the FMA-heavy pipe two-thirds busy while kind 0 said "peak").
#include <cuda_runtime.h>

#include "engine.h"

namespace b200 {
namespace {

template <int KIND>
__global__ void __launch_bounds__(256) k_int_peak(uint32_t iters, uint32_t seed, uint64_t* out) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t acc[8];
    uint32_t y = seed * 2654435761u + tid * 40503u + 12345u;
#pragma unroll
    for (int k = 0; k < 8; k++) acc[k] = (uint64_t(tid) << 32) ^ (0x9e3779b97f4a7c15ull * (k + 1));
#pragma unroll 1
    for (uint32_t it = 0; it < iters; it++) {
#pragma unroll
        for (int rep = 0; rep < 4; rep++) {
#pragma unroll
            for (int k = 0; k < 8; k++) {
                if (KIND == 0) {
                    acc[k] = uint64_t(uint32_t(acc[k])) * y + acc[k];                         // IMAD.WIDE.U32
                } else if (KIND == 7) {
                    acc[k] = uint64_t(uint32_t(acc[(k + 4) & 7])) * y + acc[k];
                } else if (KIND == 8) {
                    acc[k] = uint64_t(uint32_t(acc[(k + 4) & 7])) * 0xb9feffffu + acc[k];
                } else if (KIND == 1) {
                    uint32_t lo = uint32_t(acc[k]);
                    lo = lo * y + uint32_t(acc[k] >> 32);                                        // IMAD
                    acc[k] = (acc[k] & 0xffffffff00000000ull) | lo;
                } else if (KIND == 3) {
                    uint32_t lo = uint32_t(acc[k]);
                    lo = __umulhi(lo, y) + uint32_t(acc[k] >> 32);                               // IMAD.HI.U32
                    acc[k] = (acc[k] & 0xffffffff00000000ull) | lo;
                } else if (KIND == 5) {
                    // one 52x52->104-bit product by the sampled-FMA trick + integer accumulation of both halves
                    const double C1 = 20282409603651670423947251286016.0;            // 2^104
                    const double C2 = 20282409603651670423947251286016.0 + 4503599627370496.0;  // 2^104 + 2^52
                    double x = __longlong_as_double((acc[k] & 0x000fffffffffffffull) | 0x4330000000000000ull) - 4503599627370496.0;
                    double yd = double(y);
                    double hi = __fma_rz(x, yd, C1);
                    double lo = __fma_rz(x, yd, C2 - hi);
                    acc[k] += uint64_t(__double_as_longlong(hi)) + uint64_t(__double_as_longlong(lo));
                } else if (KIND == 6) {
                    double x = __longlong_as_double(acc[k] | 0x3ff0000000000000ull);
                    x = __fma_rz(x, 1.0000001, 0.5);                                              // DFMA
                    acc[k] = uint64_t(__double_as_longlong(x)) & 0x000fffffffffffffull;
                } else if (KIND == 4) {
                    uint32_t lo = uint32_t(acc[k]), hi = uint32_t(acc[k] >> 32);
                    lo = lo + hi + y; hi = hi + lo + y;                                          // 2 x IADD3
                    acc[k] = (uint64_t(hi) << 32) | lo;
                } else {
                    uint32_t a = uint32_t(acc[k]), b = uint32_t(acc[k] >> 32);
                    uint32_t r = __funnelshift_r(a, a, 7) ^ (a & b) ^ (~a & y);                 // SHF + LOP3 (+LOP3)
                    b = b + r + y;                                                               // IADD3
                    acc[k] = (uint64_t(r) << 32) | b;
                }
            }
        }
    }
    uint64_t x = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) x ^= acc[k];
    out[tid] = x;
}

}  // namespace
}  // namespace b200

using namespace b200;

// -> operations of the named kind per second (1e9 units) in *gops; ops counted = threads * iters * 32
extern "C" int32_t b200_measure_int_peak(int32_t kind, double* gops) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    if (!e.ready) return B200_ERR_NOT_INITIALIZED;
    if (!gops || kind < 0 || kind > 8) return B200_ERR_BAD_ARG;
    B200_CUDA_TRY(cudaSetDevice(e.device));
    int sms = 0;
    B200_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e.device));
    const uint32_t blocks = uint32_t(sms) * 8, threads = 256, iters = 4096;
    uint64_t* d = nullptr;
    B200_CUDA_TRY(cudaMalloc(&d, size_t(blocks) * threads * 8));
    float best = 1e30f;
    for (int rep = 0; rep < 4; rep++) {
        B200_CUDA_TRY(cudaEventRecord(e.ev0, e.stream));
        if (kind == 0) k_int_peak<0><<<blocks, threads, 0, e.stream>>>(iters, 1 + rep, d);
        else if (kind == 1) k_int_peak<1><<<blocks, threads, 0, e.stream>>>(iters, 1 + rep, d);
        else if (kind == 2) k_int_peak<2><<<blocks, threads, 0, e.stream>>>(iters, 1 + rep, d);
        else if (kind == 3) k_int_peak<3><<<blocks, threads, 0, e.stream>>>(iters, 1 + rep, d);
        else if (kind == 4) k_int_peak<4><<<blocks, threads, 0, e.stream>>>(iters, 1 + rep, d);
        else if (kind == 5) k_int_peak<5><<<blocks, threads, 0, e.stream>>>(iters, 1 + rep, d);
        else if (kind == 6) k_int_peak<6><<<blocks, threads, 0, e.stream>>>(iters, 1 + rep, d);
        else if (kind == 7) k_int_peak<7><<<blocks, threads, 0, e.stream>>>(iters, 1 + rep, d);
        else k_int_peak<8><<<blocks, threads, 0, e.stream>>>(iters, 1 + rep, d);
        e.launches++;
        B200_CUDA_TRY(cudaEventRecord(e.ev1, e.stream));
        B200_CUDA_TRY(cudaGetLastError());
        B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
        float ms = 0;
        B200_CUDA_TRY(cudaEventElapsedTime(&ms, e.ev0, e.ev1));
        if (rep > 0 && ms < best) best = ms;
    }
    cudaFree(d);
    const double ops_per_thread = double(iters) * 32.0 * (kind == 2 ? 4.0 : kind == 4 ? 2.0 : 1.0);  // kind 2: SHF + 2 LOP3 + IADD3 per step; kind 4: 2 IADD3
    *gops = double(blocks) * threads * ops_per_thread / (double(best) * 1e-3) / 1e9;
    return B200_SUCCESS;
}
