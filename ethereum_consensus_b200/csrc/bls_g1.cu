// G1 side of the BLS pipeline: per-public-key validation (the dominant cost of the reference's
// fast_aggregate_verify, ethereum-consensus/src/crypto/bls.rs:119-123 -> :283) and the per-tuple
// aggregation blst performs in `AggregatePublicKey::aggregate`.
//
// k_g1_validate : one thread per key, Fp limbs in registers; 48 B in, 100 B out.  Integer-pipe bound.
// k_g1_aggregate: one warp per tuple; lanes stride over the tuple's keys with mixed additions, then a
//                 5-round shared-memory tree of Jacobian additions; lane 0 normalises to affine.
// Squarings (~75 % of this kernel's products) use the dedicated PTX square (222 wide MADs instead of 288).  It pays
// with 256-thread CTAs at 224 registers; with the 168-register cap the square's wider live range spills, and at ptxas'
// default level it loses to predicate spills.  -DB200_G1_SQR_VIA_MUL restores squares-by-product.
#if defined(B200_G1_SQR_VIA_MUL)
#define B200_FP_SQR_VIA_MUL 1
#endif
// Products as by-value function CALLS (operands and result in registers, 0-byte frames) instead of ~70 inlined copies:
// the inlined kernel is 0.5 MB of straight-line code, far beyond the instruction caches, and only pays at 8 warps per SM
// where the warps stay in step.  With calls the kernel body is about a third of that and 12 warps per SM
// win.  -DB200_G1_INLINE_MUL restores the inlined products.
#if !defined(B200_G1_INLINE_MUL)
#define B200_FP_MUL_CALL 1
#endif
// fp_pow's window table in dynamic shared memory (fp.cuh): every kernel here that can reach fp_pow is launched through
// with_pow_tab() below.  Thread-local storage made the per-key kernel's speed depend on what else the process had run.
#define B200_POW_TAB_SMEM 1
#include <cuda_runtime.h>

#include "bls_kernels.cuh"

namespace b200 {
namespace {

__device__ __forceinline__ void g1_validate_body(const uint8_t* __restrict__ keys, uint32_t n, G1Aff* __restrict__ out,
                                                 int32_t* __restrict__ codes) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    __align__(16) uint8_t b[48];  // written through uint4*
    const uint4* src = reinterpret_cast<const uint4*>(keys + size_t(i) * 48);
    uint4* dst = reinterpret_cast<uint4*>(b);
    dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
    G1Aff p;
    const int32_t rc = g1_key_validate(p, b);
    codes[i] = rc;
    if (rc == BLS_SUCCESS) out[i] = p;
}
// Default (variant 7): 384 threads capped at 168 registers = 12 warps per SM (with call-based products, see the top of
// this file).  Variant 0: 256-thread CTAs at 224 registers (8 warps per SM, no spills).  Variant 6: 512 threads at 128
// registers = 16 warps per SM.  The register budgets follow from the SM's 64 K-entry register file;
// B200_G1_VARIANT selects a variant at run time for A/B runs.  (__maxnreg__ cannot be combined with __launch_bounds__.)
__global__ void __maxnreg__(224) k_g1_validate_main(const uint8_t* __restrict__ keys, uint32_t n, G1Aff* __restrict__ out,
                                                    int32_t* __restrict__ codes) {
    g1_validate_body(keys, n, out, codes);
}
__global__ void __maxnreg__(168) k_g1_validate_r168(const uint8_t* __restrict__ keys, uint32_t n, G1Aff* __restrict__ out,
                                                    int32_t* __restrict__ codes) {
    g1_validate_body(keys, n, out, codes);
}
// (Occupancies between 8 and 12 warps per SM do not exist for this kernel: the register file is handed out in units of
// four warps, so 9-, 10- and 11-warp CTAs at 224 / 200 / 184 registers all fail to launch — measured, "too many
// resources requested" — and the choice is 8 warps at <= 256 registers or 12 warps at <= 168.)
__global__ void __maxnreg__(128) k_g1_validate_r128(const uint8_t* __restrict__ keys, uint32_t n, G1Aff* __restrict__ out,
                                                    int32_t* __restrict__ codes) {
    g1_validate_body(keys, n, out, codes);
}
constexpr int kAggWarps = 4;

__global__ void __launch_bounds__(32 * kAggWarps) k_g1_aggregate(const G1Aff* __restrict__ keys,
                                                                  const int32_t* __restrict__ key_codes,
                                                                  const uint32_t* __restrict__ index,
                                                                  const uint32_t* __restrict__ off, uint32_t n_tuples,
                                                                  G1Aff* __restrict__ agg, G1Pre* __restrict__ agg_pre,
                                                                  int32_t* __restrict__ pk_code,
                                                                  uint32_t* __restrict__ flags, uint32_t extra_flags,
                                                                  G1Jac* __restrict__ agg_jac) {
    __shared__ G1Jac part[kAggWarps][32];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t t = blockIdx.x * kAggWarps + warp;
    if (t >= n_tuples) return;  // whole warp exits together
    const uint32_t lo = off[t], hi = off[t + 1];
    // first failing key in order
    uint32_t first_bad = 0xffffffffu;
    for (uint32_t k = lo + lane; k < hi; k += 32) {
        const uint32_t id = index ? index[k] : k;
        if (key_codes[id] != BLS_SUCCESS) { first_bad = k; break; }
    }
    for (int s = 16; s > 0; s >>= 1) first_bad = min(first_bad, __shfl_xor_sync(0xffffffffu, first_bad, s));
    if (first_bad != 0xffffffffu) {
        if (lane == 0) {
            pk_code[t] = key_codes[index ? index[first_bad] : first_bad];
            flags[t] = 0;
        }
        return;
    }
    if (agg == nullptr && agg_pre == nullptr) {  // code scan only
        if (lane == 0) { pk_code[t] = BLS_SUCCESS; flags[t] = (hi == lo ? TUPLE_FLAG_EMPTY : 0u) | extra_flags; }
        return;
    }
    G1Jac acc;
    jac_set_inf(acc);
    for (uint32_t k = lo + lane; k < hi; k += 32) {
        const G1Aff q = keys[index ? index[k] : k];
        jac_add_mixed(acc, acc, q.x, q.y);
    }
    part[warp][lane] = acc;
    __syncwarp();
    for (int s = 16; s > 0; s >>= 1) {
        if (lane < s) {
            G1Jac a = part[warp][lane], b = part[warp][lane + s];
            jac_add(a, a, b);
            part[warp][lane] = a;
        }
        __syncwarp();
    }
    if (lane == 0) {
        bool inf;
        if (agg_pre) {   // hand the Jacobian sum to the Miller VM: (X Z, Y, Z^3), no inversion
            const G1Jac s = part[warp][0];
            G1Pre p;
            inf = jac_is_inf(s);
            Fp zz;
            fp_sqr(zz, s.z);
            fp_mul(p.z3, zz, s.z);
            fp_mul(p.xz, s.x, s.z);
            p.y = s.y;
            p.inf = inf ? 1u : 0u;
            agg_pre[t] = p;
            if (agg_jac) agg_jac[t] = s;   // the RLC batch check scales the sum itself (bls_rlc.cu)
        } else {
            G1Aff a;
            jac_to_aff(a, part[warp][0]);
            agg[t] = a;
            inf = a.inf != 0;
        }
        pk_code[t] = BLS_SUCCESS;
        flags[t] = (hi == lo ? TUPLE_FLAG_EMPTY : 0u) | (inf ? TUPLE_FLAG_AGG_INF : 0u) | extra_flags;
    }
}

__global__ void k_g1_compress(const G1Aff* p, uint8_t* out48) {
    if (threadIdx.x == 0 && blockIdx.x == 0) g1_compress(out48, *p);
}
__global__ void k_neg_g1(G1Aff* out, G1Pre* out_pre) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        G1Aff g;
        const Fp x = B200_FP_G1_X, y = B200_FP_G1_NEG_Y;
        g.x = x; g.y = y; g.inf = 0;
        *out = g;
        G1Pre p;
        p.xz = x; p.y = y; p.z3 = fp_one(); p.inf = 0;
        *out_pre = p;
    }
}

// Fp self-test: random a, b; checks (a*b)*c == a*(b*c), a*(b+c) == a*b + a*c, a * a^-1 == 1 for a few values
__global__ void k_fp_selftest(uint32_t n, uint32_t seed, uint32_t* out_mismatch) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t s = (uint64_t(seed) << 32) | i;
    auto next = [&]() { s += 0x9e3779b97f4a7c15ull; uint64_t z = s; z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
                        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull; return uint32_t((z ^ (z >> 31)) >> 16); };
    Fp a, b, c;
    for (int k = 0; k < 12; k++) { a.l[k] = next(); b.l[k] = next(); c.l[k] = next(); }
    a.l[11] &= 0x0fffffffu; b.l[11] &= 0x0fffffffu; c.l[11] &= 0x0fffffffu;  // < p
    if ((i & 7) == 1) { const Fp pp = fp_p(); Fp one; for (int k = 0; k < 12; k++) one.l[k] = 0; one.l[0] = 1 + (i >> 3); fp_sub_raw(a, pp, one); }  // near p
    Fp ab, bc, l, r, t;
    uint32_t bad = 0;
    fp_mul(ab, a, b); fp_mul(l, ab, c); fp_mul(bc, b, c); fp_mul(r, a, bc);
    if (!fp_eq(l, r)) bad++;
    fp_add(t, b, c); fp_mul(l, a, t); fp_mul(r, a, c); fp_add(r, r, ab);
    if (!fp_eq(l, r)) bad++;
    fp_sqr(l, a); fp_mul(r, a, a);
    if (!fp_eq(l, r)) bad++;
    fp_mul_portable(r, a, b);  // tuned PTX product / square vs the portable product
    if (!fp_eq(ab, r)) bad++;
    fp_mul_portable(r, a, a); fp_sqr(l, a);
    if (!fp_eq(l, r)) bad++;
    {   // carry-chain add / subtract (fp.cuh) vs the portable 64-bit emulation, incl. equal operands, zero and p - 1
        Fp x = a, y = b;
        if ((i & 15) == 3) y = a;
        if ((i & 15) == 5) x = fp_zero();
        if ((i & 15) == 7) { y = fp_zero(); }
        Fp u, v;
        const uint32_t cu = fp_add_raw(u, x, y), cv = fp_add_raw_portable(v, x, y);
        if (cu != cv || !fp_eq(u, v)) bad++;
        const uint32_t bu = fp_sub_raw(u, x, y), bv = fp_sub_raw_portable(v, x, y);
        if (bu != bv || !fp_eq(u, v)) bad++;
        // field-level: (x + y) - y == x, x - y == -(y - x), 2x == x + x, x + (-x) == 0
        fp_add(u, x, y); fp_sub(u, u, y);
        if (!fp_eq(u, x)) bad++;
        fp_sub(u, x, y); fp_sub(v, y, x); fp_neg(v, v);
        if (!fp_eq(u, v)) bad++;
        fp_dbl(u, x); fp_add(v, x, x);
        if (!fp_eq(u, v)) bad++;
        fp_neg(u, x); fp_add(u, u, x);
        if (!fp_is_zero(u)) bad++;
        fp_add_masked_raw(u, x, y, 0u);
        if (!fp_eq(u, x)) bad++;
        fp_add_masked_raw(u, x, y, 0xffffffffu); fp_add_raw_portable(v, x, y);
        if (!fp_eq(u, v)) bad++;
    }
    if ((i & 63) == 0 && !fp_is_zero(a)) {
        fp_inv(t, a); fp_mul(t, t, a);
        if (!fp_eq(t, fp_one())) bad++;
        Fp k, f;                       // the shift-and-add inverse (the device's fp_inv) against the exponentiation
        fp_inv_kaliski(k, a); fp_inv_fermat(f, a);
        if (!fp_eq(k, f)) bad++;
        fp_inv_kaliski(k, fp_zero());
        if (!fp_is_zero(k)) bad++;
    }
    if (bad) atomicAdd(out_mismatch, bad);
}

}  // namespace

// dynamic shared memory for fp_pow's table; opts the kernel in to > 48 KiB once
template <class K>
static size_t with_pow_tab(K kernel, unsigned threads) {
    const size_t bytes = fp_pow_smem_bytes(threads);
    static const void* seen[16];  // kernels of equal signature share this instantiation: key by address
    static size_t granted[16];    // opt-in already made for that kernel (one kernel may be launched at several CTA sizes)
    static int n_seen = 0;
    const void* key = reinterpret_cast<const void*>(kernel);
    for (int i = 0; i < n_seen; i++)
        if (seen[i] == key) {
            if (granted[i] < bytes) { cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes)); granted[i] = bytes; }
            return bytes;
        }
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes));
    if (n_seen < 16) { seen[n_seen] = key; granted[n_seen++] = bytes; }
    return bytes;
}
// tuning knob (B200_G1_VARIANT): 7: 384 threads, 168 registers (default); 0: 256 threads, 224 registers; 6: 512 threads, 128 registers
static int g_g1_variant = 7;
static uint32_t g_g1_small_n = 3u * 148u * 384u;   // B200_G1_SMALL_N overrides (0: always 384-thread CTAs)
void set_g1_small_n(uint32_t n) { g_g1_small_n = n; }
void set_g1_variant(int v) { if (v >= 0 && v <= 7) g_g1_variant = v; }
void launch_g1_validate(const uint8_t* keys, uint32_t n, G1Aff* out, int32_t* codes, void* stream, int cta) {
    if (!n) return;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (g_g1_variant) {
    case 6: k_g1_validate_r128<<<(n + 511) / 512, 512, with_pow_tab(k_g1_validate_r128, 512), st>>>(keys, n, out, codes); break;
    case 0: k_g1_validate_main<<<(n + 255) / 256, 256, with_pow_tab(k_g1_validate_main, 256), st>>>(keys, n, out, codes); break;
    default:
        // 12 warps per SM either way; below ~3 full waves of 384-thread CTAs the same kernel goes out as three 128-thread
        // CTAs per SM, so that the last, partial wave spreads over all SMs instead of leaving most of them idle
        if (cta == 128 || (cta != 384 && n <= g_g1_small_n))
            k_g1_validate_r168<<<(n + 127) / 128, 128, with_pow_tab(k_g1_validate_r168, 128), st>>>(keys, n, out, codes);
        else
            k_g1_validate_r168<<<(n + 383) / 384, 384, with_pow_tab(k_g1_validate_r168, 384), st>>>(keys, n, out, codes);
        break;
    }
}
void launch_g1_aggregate(const G1Aff* keys, const int32_t* key_codes, const uint32_t* index, const uint32_t* off,
                         uint32_t n_tuples, G1Aff* agg, G1Pre* agg_pre, int32_t* pk_code, uint32_t* flags,
                         uint32_t extra_flags, void* stream, G1Jac* agg_jac) {
    if (!n_tuples) return;
    k_g1_aggregate<<<(n_tuples + kAggWarps - 1) / kAggWarps, 32 * kAggWarps, with_pow_tab(k_g1_aggregate, 32 * kAggWarps),
                     static_cast<cudaStream_t>(stream)>>>(
        keys, key_codes, index, off, n_tuples, agg, agg_pre, pk_code, flags, extra_flags, agg_jac);
}
void launch_g1_compress(const G1Aff* p, uint8_t* out48, void* stream) {
    k_g1_compress<<<1, 32, with_pow_tab(k_g1_compress, 32), static_cast<cudaStream_t>(stream)>>>(p, out48);
}
void launch_neg_g1(G1Aff* out, G1Pre* out_pre, void* stream) { k_neg_g1<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(out, out_pre); }
void launch_fp_selftest(uint32_t n, uint32_t seed, uint32_t* out_mismatch, void* stream) {
    k_fp_selftest<<<(n + 127) / 128, 128, with_pow_tab(k_fp_selftest, 128), static_cast<cudaStream_t>(stream)>>>(n, seed, out_mismatch);
}

}  // namespace b200
