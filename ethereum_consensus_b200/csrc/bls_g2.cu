// G2 side of the BLS pipeline: signature decompression + subgroup check (blst `Signature::from_bytes` and the
// `sig_groupcheck = true` of ethereum-consensus/src/crypto/bls.rs:71,106,126) and hash_to_G2 of
// the signing roots.  One thread per signature / message; these kernels see only T (thousands) of items, so
// they run concurrently with the wide G1 kernels on a second stream.
#define B200_FP_MUL_CALL 1
// Fp2 products are INLINED into the curve routines here and the kernels may use 255 registers: these kernels run one or two
// warps per SM, so the only thing that matters is the length of one thread's dependent chain — and at T = 4096 the 3-5 KB
// stack frames of the earlier build (Fp2 products as calls, 128 registers) overflowed L1.  In strict mode they hide under the
// per-key kernel either way; in registry mode the step waits for them.
#define B200_TOWER_NOINLINE 1   // (a build with the curve routines inlined as well returned wrong verdicts on the GPU — not investigated, not offered)
#include <cuda_runtime.h>

#include <algorithm>

#include "../../include/b200_consensus.h"
#include "bls_kernels.cuh"
#include "h2c.cuh"

namespace b200 {
namespace {

// One warp per CTA: with only T items there is at most a warp or two per SM, so these kernels are latency-bound and
// spread as 32-thread CTAs over every SM (128-thread CTAs when they run under a big per-key kernel, capi_bls.cu).
// With Fp2 products as calls, more registers in the caller meant more saves / restores around every product.  Round 2 inlines the Fp2 products and lifts the cap
// (see the top of this file).
constexpr int kSmallCta = 32;
__global__ void __maxnreg__(255) k_g2_sig_decode(const uint8_t* __restrict__ sigs, uint32_t n, G2Aff* __restrict__ out,
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
__global__ void __maxnreg__(255) k_hash_to_g2_map(const uint8_t* __restrict__ msgs, const uint32_t* __restrict__ moff,
                                                        uint32_t n, G2Jac* __restrict__ tmp) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 * n) return;
    const uint32_t m = i >> 1;
    G2Jac q;
    hash_to_g2_map(q, msgs + moff[m], size_t(moff[m + 1] - moff[m]), int(i & 1));
    tmp[i] = q;
}
__global__ void __maxnreg__(255) k_hash_to_g2_finish(const G2Jac* __restrict__ tmp, uint32_t n, G2Aff* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G2Jac q0 = tmp[2 * i], q1 = tmp[2 * i + 1];
    G2Aff h;
    hash_to_g2_finish(h, q0, q1);
    out[i] = h;
}

// `aggregate` (crypto/bls.rs:79-93) over T groups, every signature decoded already (k_g2_sig_decode).  Group g is split
// into chunks of `chunk` signatures; one warp per chunk, so that a group of 32 768 signatures is summed by hundreds of
// warps instead of one.  Chunks of a group are numbered chunk_off[g] .. chunk_off[g+1]-1, chunk_group[c] names the group.
__device__ __forceinline__ void warp_min(uint32_t& v) {
    for (int s = 16; s > 0; s >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, s));
}
__device__ __forceinline__ void shfl_xor_fp(Fp& d, const Fp& a, int s) {
#pragma unroll
    for (int k = 0; k < 12; k++) d.l[k] = __shfl_xor_sync(0xffffffffu, a.l[k], s);
}
// butterfly: every lane ends with the warp's sum (as a possibly different Jacobian representative of the same point)
__device__ __forceinline__ void warp_sum(G2Jac& acc) {
    for (int s = 16; s > 0; s >>= 1) {
        G2Jac o;
        shfl_xor_fp(o.x.c0, acc.x.c0, s); shfl_xor_fp(o.x.c1, acc.x.c1, s);
        shfl_xor_fp(o.y.c0, acc.y.c0, s); shfl_xor_fp(o.y.c1, acc.y.c1, s);
        shfl_xor_fp(o.z.c0, acc.z.c0, s); shfl_xor_fp(o.z.c1, acc.z.c1, s);
        jac_add(acc, acc, o);
    }
}

// The chunks' partial results are read back by another warp of the same launch: through L2 (ld.global.cg), never from a
// possibly stale L1 line
__device__ __forceinline__ void load_cg(G2Jac& q, const G2Jac* p) {
    const uint4* s = reinterpret_cast<const uint4*>(p);
    uint4* d = reinterpret_cast<uint4*>(&q);
#pragma unroll
    for (int k = 0; k < int(sizeof(G2Jac) / 16); k++) d[k] = __ldcg(s + k);
}

// One warp per chunk.  part_code[c] = the code of the chunk's first decode failure (> 0), else SIG_NOT_IN_GROUP if any of
// its signatures failed the group check, else SIG_OK and part[c] = the Jacobian sum of its signatures.  The warp that
// completes a group's last outstanding chunk (counter done[g], zero at launch) then finishes the group: decode errors take
// precedence over group-check errors (every signature is decoded before any is checked, as blst's aggregate does), else
// the chunk sums are added, normalised and compressed.  A failed or empty group's 96 bytes are zero.  Every group, empty
// ones included, has at least one chunk.
__global__ void __maxnreg__(255) k_g2_aggregate(const G2Aff* __restrict__ sigs, const int32_t* __restrict__ sig_code,
                                              const uint32_t* __restrict__ off, const uint32_t* __restrict__ chunk_group,
                                              const uint32_t* __restrict__ chunk_off, uint32_t n_chunks, uint32_t chunk,
                                              G2Jac* part, int32_t* part_code, uint32_t* done, uint8_t* __restrict__ out96,
                                              int32_t* __restrict__ out_code) {
    const uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (c >= n_chunks) return;  // whole warp exits together
    const uint32_t g = chunk_group[c];
    const uint32_t lo = off[g] + (c - chunk_off[g]) * chunk, hi = min(off[g + 1], lo + chunk);
    uint32_t first_dec = 0xffffffffu, first_bad = 0xffffffffu;
    for (uint32_t k = lo + lane; k < hi; k += 32) {
        const int32_t rc = sig_code[k];
        if (rc != SIG_OK && first_bad == 0xffffffffu) first_bad = k;
        if (rc > 0) { first_dec = k; break; }
    }
    warp_min(first_dec);
    warp_min(first_bad);
    G2Jac acc;
    jac_set_inf(acc);
    if (first_bad == 0xffffffffu) {
        for (uint32_t k = lo + lane; k < hi; k += 32) {
            const G2Aff q = sigs[k];
            if (!q.inf) jac_add_mixed(acc, acc, q.x, q.y);
        }
        warp_sum(acc);
    }
    uint32_t last = 0;
    if (lane == 0) {
        part[c] = acc;
        part_code[c] = first_bad == 0xffffffffu ? SIG_OK : first_dec != 0xffffffffu ? sig_code[first_dec] : SIG_NOT_IN_GROUP;
        __threadfence();   // this chunk's result is visible before the counter says so
        last = atomicAdd(done + g, 1u) == chunk_off[g + 1] - chunk_off[g] - 1;
    }
    if (!__shfl_sync(0xffffffffu, last, 0)) return;
    __threadfence();
    // the group's finish
    const uint32_t clo = chunk_off[g], chi = chunk_off[g + 1];
    first_dec = 0xffffffffu;
    bool bad = false;
    for (uint32_t k = clo + lane; k < chi; k += 32) {
        const int32_t rc = __ldcg(part_code + k);
        bad = bad || rc != SIG_OK;
        if (rc > 0) { first_dec = k; break; }
    }
    warp_min(first_dec);
    bad = __any_sync(0xffffffffu, bad);
    uint8_t* o = out96 + size_t(g) * 96;
    if (off[g] == off[g + 1] || bad) {
        if (lane == 0) out_code[g] = off[g] == off[g + 1] ? B200_EMPTY_AGGREGATE
                                     : first_dec != 0xffffffffu ? __ldcg(part_code + first_dec) : int32_t(BLS_POINT_NOT_IN_GROUP);
        o[3 * lane] = 0; o[3 * lane + 1] = 0; o[3 * lane + 2] = 0;
        return;
    }
    jac_set_inf(acc);
    for (uint32_t k = clo + lane; k < chi; k += 32) {
        G2Jac q;
        load_cg(q, part + k);
        jac_add(acc, acc, q);
    }
    warp_sum(acc);
    if (lane == 0) {
        G2Aff a;
        jac_to_aff(a, acc);
        g2_compress(o, a);
        out_code[g] = BLS_SUCCESS;
    }
}

// Fp2 self-test against big integers (b200_fp_eval): compiled here so that it runs this unit's inlined Fp2 products,
// register cap and ptxas level
__global__ void __maxnreg__(255) k_fp2_eval(int32_t op, uint32_t n, const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                                          uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fp2 x, y, r = fp2_zero();
    for (int k = 0; k < 12; k++) {
        x.c0.l[k] = a[size_t(i) * kFpEvalIn + k]; x.c1.l[k] = a[size_t(i) * kFpEvalIn + 12 + k];
        y.c0.l[k] = b[size_t(i) * kFpEvalIn + k]; y.c1.l[k] = b[size_t(i) * kFpEvalIn + 12 + k];
    }
    uint32_t flag = 0;
    switch (op) {
    case FP2_EVAL_MUL: fp2_mul(r, x, y); break;
    case FP2_EVAL_SQR: fp2_sqr(r, x); break;
    case FP2_EVAL_INV: fp2_inv(r, x); break;
    case FP2_EVAL_SQRT: flag = fp2_sqrt(r, x) ? 1u : 0u; if (!flag) r = fp2_zero(); break;
    case FP2_EVAL_SGN0: flag = fp2_sgn0(x); break;
    default: break;
    }
    uint32_t* o = out + size_t(i) * kFpEvalOut;
    for (int k = 0; k < 12; k++) { o[k] = r.c0.l[k]; o[12 + k] = r.c1.l[k]; }
    o[24] = flag;
}

// Curve stages of the signature / hash kernels against the big-integer oracle (b200_curve_eval), one per launch, as this
// unit compiles them: the Jacobian formulas, the subgroup check, psi, cofactor clearing, the map and hash_to_G2's second
// half on Jacobian inputs
__device__ __forceinline__ void curve2_load(G2Jac& p, const uint32_t* w) {
    for (int k = 0; k < 12; k++) {
        p.x.c0.l[k] = w[k]; p.x.c1.l[k] = w[12 + k];
        p.y.c0.l[k] = w[24 + k]; p.y.c1.l[k] = w[36 + k];
        p.z.c0.l[k] = w[48 + k]; p.z.c1.l[k] = w[60 + k];
    }
}
__global__ void __maxnreg__(255) k_curve2_eval(int32_t op, uint32_t n, const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                                             uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* pa = a + size_t(i) * kCurveEvalWords;
    G2Jac p, q, r;
    curve2_load(p, pa);
    curve2_load(q, b + size_t(i) * kCurveEvalWords);
    jac_set_inf(r);
    uint32_t flag = 0;
    switch (op) {
    case CURVE_G2_ADD: jac_add(r, p, q); break;
    case CURVE_G2_ADD_MIXED: jac_add_mixed(r, p, q.x, q.y); break;
    case CURVE_G2_DOUBLE: jac_double(r, p); break;
    case CURVE_G2_IN_SUBGROUP: {
        G2Aff s;
        s.x = p.x; s.y = p.y; s.inf = pa[72];
        flag = g2_in_subgroup(s) ? 1u : 0u;
        break;
    }
    case CURVE_G2_PSI: g2_psi(r, p); break;
    case CURVE_G2_CLEAR_COFACTOR: g2_clear_cofactor(r, p); break;
    case CURVE_G2_SSWU_ISO: B200_SSWU_ISO(r, p.x); break;
    case CURVE_G2_H2C_FINISH: {
        G2Aff h;
        hash_to_g2_finish(h, p, q);
        r.x = h.x; r.y = h.y; r.z = h.inf ? fp2_zero() : fp2_one();
        flag = h.inf;
        break;
    }
    default: break;
    }
    uint32_t* o = out + size_t(i) * kCurveEvalWords;
    for (int k = 0; k < 12; k++) {
        o[k] = r.x.c0.l[k]; o[12 + k] = r.x.c1.l[k];
        o[24 + k] = r.y.c0.l[k]; o[36 + k] = r.y.c1.l[k];
        o[48 + k] = r.z.c0.l[k]; o[60 + k] = r.z.c1.l[k];
    }
    o[72] = flag;
}

}  // namespace

constexpr size_t kPowTab = 0;  // thread-local table here (see above)
// CTA size of the signature / message kernels: 32 spreads them over all SMs (lowest latency when they run alone, without
// a per-key kernel); larger CTAs pack them onto few SMs for runs UNDER the per-key kernel
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
// Warps of one launch of the aggregation kernels: 32-thread CTAs spread a few warps over every SM; from four per SM on,
// 128-thread CTAs
static uint32_t sm_count() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1)
            n = 132;
    }
    return uint32_t(n);
}
static int agg_cta(uint32_t warps) { return warps >= 4 * sm_count() ? 128 : 32; }

// About eight warps per SM over the whole call, in whole warps' strides (the sum is ~1 % of the decode's work, so only its
// latency matters); a group gets one chunk per `chunk` signatures
uint32_t g2_aggregate_chunk(uint32_t n_sigs) {
    const uint32_t warps = 8 * sm_count();
    return 32u * std::max<uint32_t>(1u, (n_sigs + 32u * warps - 1) / (32u * warps));
}
void launch_g2_aggregate(const G2Aff* sigs, const int32_t* sig_code, const uint32_t* off, const uint32_t* chunk_group,
                         const uint32_t* chunk_off, uint32_t n_chunks, uint32_t chunk, G2Jac* part, int32_t* part_code,
                         uint32_t* done, uint8_t* out96, int32_t* out_code, void* stream) {
    if (!n_chunks) return;
    const int t = agg_cta(n_chunks);
    k_g2_aggregate<<<(n_chunks + t / 32 - 1) / (t / 32), t, kPowTab, static_cast<cudaStream_t>(stream)>>>(
        sigs, sig_code, off, chunk_group, chunk_off, n_chunks, chunk, part, part_code, done, out96, out_code);
}
void launch_fp2_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream) {
    if (!n) return;
    k_fp2_eval<<<(n + kSmallCta - 1) / kSmallCta, kSmallCta, kPowTab, static_cast<cudaStream_t>(stream)>>>(op, n, a, b, out);
}
void launch_curve2_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream) {
    if (!n) return;
    k_curve2_eval<<<(n + kSmallCta - 1) / kSmallCta, kSmallCta, kPowTab, static_cast<cudaStream_t>(stream)>>>(op, n, a, b, out);
}

}  // namespace b200
