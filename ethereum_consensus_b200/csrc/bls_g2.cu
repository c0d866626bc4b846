// G2 side of the BLS pipeline: signature decompression + subgroup check (blst `Signature::from_bytes` and the
// `sig_groupcheck = true` of ethereum-consensus/src/crypto/bls.rs:71,106,126) and hash_to_G2 of
// the signing roots.  One thread per signature / message; these kernels see only T (thousands) of items, so
// they run concurrently with the wide G1 kernels on a second stream.
#define B200_FP_MUL_CALL 1
// Fp2 products are INLINED into the curve routines here and the kernels may use 255 registers: these kernels run one or two
// warps per SM, so the only thing that matters is the length of one thread's dependent chain — and at T = 4096 the 3-5 KB
// stack frames of the earlier build (Fp2 products as calls, 128 registers) overflowed L1.  In strict mode they hide under the
// per-key kernel either way; in registry mode the step waits for them.
// -DB200_G2_FP2_CALLS / -DB200_G2_MAXREG=128 restore the earlier build.
#if defined(B200_G2_FP2_CALLS)
#define B200_FP2_NOINLINE 1
#endif
#define B200_TOWER_NOINLINE 1   // (a build with the curve routines inlined as well returned wrong verdicts on the GPU — not investigated, not offered)
#include <cuda_runtime.h>

#include "bls_kernels.cuh"
#include "h2c.cuh"

namespace b200 {
namespace {

// One warp per CTA: with only T items there is at most a warp or two per SM, so these kernels are latency-bound and
// spread as 32-thread CTAs over every SM (128-thread CTAs when they run under a big per-key kernel, capi_bls.cu).
// With Fp2 products as calls, more registers in the caller meant more saves / restores around every product.  Round 2 inlines the Fp2 products and lifts the cap
// (see the top of this file).
constexpr int kSmallCta = 32;
#if !defined(B200_G2_MAXREG)
#define B200_G2_MAXREG 255
#endif
#define B200_G2_BOUNDS __maxnreg__(B200_G2_MAXREG)
__global__ void B200_G2_BOUNDS k_g2_sig_decode(const uint8_t* __restrict__ sigs, uint32_t n, G2Aff* __restrict__ out,
                                                       int32_t* __restrict__ sig_code) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    __align__(16) uint8_t b[96];  // written through uint4*
    const uint4* src = reinterpret_cast<const uint4*>(sigs + size_t(i) * 96);
    uint4* dst = reinterpret_cast<uint4*>(b);
#pragma unroll
    for (int k = 0; k < 6; k++) dst[k] = src[k];
    G2Aff q;
    int32_t rc = g2_uncompress(q, b);
    if (rc == BLS_SUCCESS) {
        out[i] = q;
        if (!g2_in_subgroup(q)) rc = SIG_NOT_IN_GROUP;
    }
    sig_code[i] = rc;
}

// hash_to_G2 in two launches: the two SSWU maps of a message are independent (2n threads), then one thread per message
// adds them, clears the cofactor and normalises.
__global__ void B200_G2_BOUNDS k_hash_to_g2_map(const uint8_t* __restrict__ msgs, const uint32_t* __restrict__ moff,
                                                        uint32_t n, G2Jac* __restrict__ tmp) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 * n) return;
    const uint32_t m = i >> 1;
    G2Jac q;
    hash_to_g2_map(q, msgs + moff[m], size_t(moff[m + 1] - moff[m]), int(i & 1));
    tmp[i] = q;
}
__global__ void B200_G2_BOUNDS k_hash_to_g2_finish(const G2Jac* __restrict__ tmp, uint32_t n, G2Aff* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G2Jac q0 = tmp[2 * i], q1 = tmp[2 * i + 1];
    G2Aff h;
    hash_to_g2_finish(h, q0, q1);
    out[i] = h;
}

// `aggregate` (crypto/bls.rs:79-93): every signature decoded already; group-check each (first failure in order
// wins), sum, compress.  One warp: lanes stride, shared-memory tree.
__global__ void __launch_bounds__(32) k_g2_sum_compress(const G2Aff* __restrict__ sigs, const int32_t* __restrict__ sig_code,
                                                         uint32_t n, uint8_t* out96, int32_t* out_code) {
    __shared__ G2Jac part[32];
    const uint32_t lane = threadIdx.x;
    uint32_t first_bad = 0xffffffffu;
    for (uint32_t k = lane; k < n; k += 32)
        if (sig_code[k] != SIG_OK) { first_bad = k; break; }
    for (int s = 16; s > 0; s >>= 1) first_bad = min(first_bad, __shfl_xor_sync(0xffffffffu, first_bad, s));
    // decode errors take precedence over group-check errors (all signatures are decoded before any is checked)
    uint32_t first_dec = 0xffffffffu;
    for (uint32_t k = lane; k < n; k += 32)
        if (sig_code[k] > 0) { first_dec = k; break; }
    for (int s = 16; s > 0; s >>= 1) first_dec = min(first_dec, __shfl_xor_sync(0xffffffffu, first_dec, s));
    if (first_dec != 0xffffffffu) { if (lane == 0) *out_code = sig_code[first_dec]; return; }
    if (first_bad != 0xffffffffu) { if (lane == 0) *out_code = BLS_POINT_NOT_IN_GROUP; return; }
    G2Jac acc;
    jac_set_inf(acc);
    for (uint32_t k = lane; k < n; k += 32) {
        const G2Aff q = sigs[k];
        if (!q.inf) jac_add_mixed(acc, acc, q.x, q.y);
    }
    part[lane] = acc;
    __syncwarp();
    for (int s = 16; s > 0; s >>= 1) {
        if (lane < s) {
            G2Jac a = part[lane], b = part[lane + s];
            jac_add(a, a, b);
            part[lane] = a;
        }
        __syncwarp();
    }
    if (lane == 0) {
        G2Aff a;
        jac_to_aff(a, part[0]);
        g2_compress(out96, a);
        *out_code = BLS_SUCCESS;
    }
}

}  // namespace

constexpr size_t kPowTab = 0;  // thread-local table here (see above)
// CTA size of the signature / message kernels: 32 spreads them over all SMs (lowest latency when they run alone, before
// the per-key kernel); larger CTAs pack them onto few SMs for runs UNDER the per-key kernel (B200_SMALL_ORDER=0)
static int g_small_cta = kSmallCta;
void set_small_cta(int threads) { if (threads >= 32 && threads <= 512 && threads % 32 == 0) g_small_cta = threads; }

void launch_g2_sig_decode(const uint8_t* sigs, uint32_t n, G2Aff* out, int32_t* sig_code, void* stream) {
    if (!n) return;
    const int threads = g_small_cta;
    k_g2_sig_decode<<<(n + threads - 1) / threads, threads, kPowTab, static_cast<cudaStream_t>(stream)>>>(sigs, n, out, sig_code);
}
void launch_hash_to_g2(const uint8_t* msgs, const uint32_t* moff, uint32_t n, G2Aff* out, void* tmp_jac, void* stream) {
    if (!n) return;
    const int threads = g_small_cta;
    G2Jac* tmp = static_cast<G2Jac*>(tmp_jac);
    k_hash_to_g2_map<<<(2 * n + threads - 1) / threads, threads, kPowTab, static_cast<cudaStream_t>(stream)>>>(msgs, moff, n, tmp);
    k_hash_to_g2_finish<<<(n + threads - 1) / threads, threads, kPowTab, static_cast<cudaStream_t>(stream)>>>(tmp, n, out);
}
void launch_g2_sum_compress(const G2Aff* sigs, const int32_t* sig_code, uint32_t n, uint8_t* out96, int32_t* out_code, void* stream) {
    k_g2_sum_compress<<<1, 32, kPowTab, static_cast<cudaStream_t>(stream)>>>(sigs, sig_code, n, out96, out_code);
}

}  // namespace b200
