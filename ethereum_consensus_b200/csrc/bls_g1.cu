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

#include "../../include/b200_consensus.h"
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
// The default launch of 384-thread CTAs (variant 7): the same 168-register budget split by role, so that both multiply
// pipes of an SM work on the same keys.  Warps 0-7 run the subgroup checks of the CTA's 256 keys on the integer pipe
// (g1_in_subgroup_iso, which needs x only); warps 8-11 run their square roots on the FP64 pipe (g1_y_from_x_fpd), two
// keys per thread, one after the other.  One barrier, then each integer thread merges its key's code in the
// reference's order and writes the point.  (Separate kernels on two streams would not share an SM: either one fills its
// register file.)
constexpr int kSplitIntThreads = 256, kSplitThreads = 384;
__global__ void __maxnreg__(168) k_g1_validate_split(const uint8_t* __restrict__ keys, uint32_t n, G1Aff* __restrict__ out,
                                                     int32_t* __restrict__ codes) {
    __shared__ Fp s_y[kSplitIntThreads];
    __shared__ uint8_t s_on_curve[kSplitIntThreads];
    const uint32_t base = blockIdx.x * kSplitIntThreads;
    __align__(16) uint8_t b[48];  // written through uint4*
    Fp x;
    uint32_t inf = 0;
    bool largest = false, in_group = true;
    int32_t rc = BLS_SUCCESS;
    if (threadIdx.x < kSplitIntThreads) {
        const uint32_t i = base + threadIdx.x;
        if (i < n) {
            const uint4* src = reinterpret_cast<const uint4*>(keys + size_t(i) * 48);
            uint4* dst = reinterpret_cast<uint4*>(b);
            dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
            rc = g1_parse(x, inf, largest, b);
            if (rc == BLS_SUCCESS && !inf) in_group = g1_in_subgroup_iso(x);
        }
    } else {
#pragma unroll 1
        for (uint32_t j = threadIdx.x - kSplitIntThreads; j < kSplitIntThreads; j += kSplitThreads - kSplitIntThreads) {
            const uint32_t i = base + j;
            if (i >= n) break;
            const uint4* src = reinterpret_cast<const uint4*>(keys + size_t(i) * 48);
            uint4* dst = reinterpret_cast<uint4*>(b);
            dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
            Fp y = fp_zero();
            bool on_curve = true;
            if (g1_parse(x, inf, largest, b) == BLS_SUCCESS && !inf) on_curve = g1_y_from_x_fpd(y, x, largest);
            s_y[j] = y;
            s_on_curve[j] = on_curve;
        }
    }
    __syncthreads();
    const uint32_t i = base + threadIdx.x;
    if (threadIdx.x >= kSplitIntThreads || i >= n) return;
    rc = g1_key_validate_code(rc, inf, s_on_curve[threadIdx.x] != 0, in_group);
    codes[i] = rc;
    if (rc == BLS_SUCCESS) {
        G1Aff p;
        p.x = x; p.y = s_y[threadIdx.x]; p.inf = 0;
        out[i] = p;
    }
}
constexpr int kAggWarps = 4;

__global__ void __launch_bounds__(32 * kAggWarps) k_g1_aggregate(const G1Aff* __restrict__ keys,
                                                                  const int32_t* __restrict__ key_codes,
                                                                  const uint32_t* __restrict__ index,
                                                                  const uint32_t* __restrict__ off, uint32_t n_tuples,
                                                                  G1Aff* __restrict__ agg, G1Pre* __restrict__ agg_pre,
                                                                  int32_t* __restrict__ pk_code,
                                                                  uint32_t* __restrict__ flags, uint32_t extra_flags,
                                                                  G1Jac* __restrict__ agg_jac,
                                                                  const uint32_t* __restrict__ tuple_flags) {
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
    if (tuple_flags) extra_flags |= tuple_flags[t];
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

// `eth_aggregate_public_keys` (crypto/bls.rs:135-148) after K2: one thread per group.  The first failing key's code, else
// EMPTY_AGGREGATE for a group without keys, else the compressed sum; a failed or empty group's 48 bytes are zero.
__global__ void k_g1_compress_groups(const G1Aff* __restrict__ agg, const int32_t* __restrict__ pk_code,
                                     const uint32_t* __restrict__ flags, uint32_t n_groups, uint8_t* __restrict__ out48,
                                     int32_t* __restrict__ out_code) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_groups) return;
    uint8_t* o = out48 + size_t(g) * 48;
    const int32_t rc = pk_code[g] != BLS_SUCCESS ? pk_code[g] : (flags[g] & TUPLE_FLAG_EMPTY) ? int32_t(B200_EMPTY_AGGREGATE) : BLS_SUCCESS;
    out_code[g] = rc;
    if (rc == BLS_SUCCESS) g1_compress(o, agg[g]);
    else for (int k = 0; k < 48; k++) o[k] = 0;
}
// aggregate_verify batches: one thread per key of the call, its pair's G1 operand (launch_g1_pair_operands).  Keys that
// failed validation are converted as well; their tuples are dead and no pairing kernel reads them.
__global__ void k_g1_pair_operands(const G1Aff* __restrict__ keys, const uint32_t* __restrict__ index, uint32_t n,
                                   G1Pre* __restrict__ pre, G1Aff* __restrict__ aff) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G1Aff a = keys[index ? index[i] : i];
    if (pre) {
        G1Pre p;
        p.xz = a.x; p.y = a.y; p.z3 = fp_one(); p.inf = a.inf;
        pre[i] = p;
    }
    if (aff) aff[i] = a;
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

// Field self-test against big integers (b200_fp_eval): one operation per launch on raw operands, so that the host can
// check the exact representative.  Compiled here so that it runs the per-key kernel's products (fp_mul_call /
// fpl_mul_call), its shared-memory pow table and this unit's ptxas level.
__global__ void k_fp_eval(int32_t op, uint32_t n, const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                          uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fp x, y, x1, y1, r = fp_zero();
    for (int k = 0; k < 12; k++) { x.l[k] = a[size_t(i) * kFpEvalIn + k]; y.l[k] = b[size_t(i) * kFpEvalIn + k]; }
    for (int k = 0; k < 12; k++) { x1.l[k] = a[size_t(i) * kFpEvalIn + 12 + k]; y1.l[k] = b[size_t(i) * kFpEvalIn + 12 + k]; }
    const FpL xl = fpl_from_fp(x), yl = fpl_from_fp(y), x1l = fpl_from_fp(x1), y1l = fpl_from_fp(y1);
    FpL rl;
    uint32_t flag = 0;
    // FpD operands and result: words 0..15 as 8 binary64 limbs, bit for bit
    auto fpd_load = [](const uint32_t* w) {
        FpD d;
        for (int k = 0; k < 8; k++) d.l[k] = __hiloint2double(int(w[2 * k + 1]), int(w[2 * k]));
        return d;
    };
    const FpD xd = fpd_load(a + size_t(i) * kFpEvalIn), yd = fpd_load(b + size_t(i) * kFpEvalIn);
    FpD rd;
    bool fpd_out = false;
    switch (op) {
    case FP_EVAL_MUL: fp_mul(r, x, y); break;
    case FP_EVAL_SQR: fp_sqr(r, x); break;
    case FPL_EVAL_MUL: f_mul(rl, xl, yl); r = rl.v; break;
    case FPL_EVAL_SQR: f_sqr(rl, xl); r = rl.v; break;
    case FP_EVAL_ADD: fp_add(r, x, y); break;
    case FP_EVAL_SUB: fp_sub(r, x, y); break;
    case FP_EVAL_NEG: fp_neg(r, x); break;
    case FPL_EVAL_ADD: f_add(rl, xl, yl); r = rl.v; break;
    case FPL_EVAL_SUB: f_sub(rl, xl, yl); r = rl.v; break;
    case FPL_EVAL_NEG: f_neg(rl, xl); r = rl.v; break;
    case FP_EVAL_ADD_RAW: flag = fp_add_raw(r, x, y); break;
    case FP_EVAL_SUB_RAW: flag = fp_sub_raw(r, x, y); break;
    case FP_EVAL_INV_KALISKI: fp_inv_kaliski(r, x); break;
    case FP_EVAL_INV_FERMAT: fp_inv_fermat(r, x); break;
    case FP_EVAL_SQRT: flag = fp_sqrt(r, x) ? 1u : 0u; break;
    case FPL_EVAL_POW_SQRT: fpl_pow(rl, xl, B200_EXP_TABLE(exp_sqrt)); r = rl.v; break;
    case FPL_EVAL_SQRT_CHAIN: fpl_sqrt_chain(rl, xl); r = rl.v; break;
    case FPL_EVAL_MUL_SUB_MUL: f_mul_sub_mul(rl, xl, x1l, yl, y1l); r = rl.v; break;
    case FPL_EVAL_MUL_SUB_8SQR: f_mul_sub_8sqr(rl, xl, x1l, yl); r = rl.v; break;
    case FP_EVAL_IS_LEX_LARGEST: flag = fp_is_lex_largest(x) ? 1u : 0u; break;
    case FPD_EVAL_MUL: fpd_mul(rd, xd, yd); fpd_out = true; break;
    case FPD_EVAL_SQR: fpd_sqr(rd, xd); fpd_out = true; break;
    case FPD_EVAL_ADD: fpd_add(rd, xd, yd); fpd_out = true; break;
    case FPD_EVAL_FROM_FP: rd = fpd_from_fp(x); fpd_out = true; break;
    case FPD_EVAL_TO_FPL: r = fpd_to_fpl(xd).v; break;
    case FPD_EVAL_SQRT_CHAIN: fpd_sqrt_chain(rd, fpd_from_fp(x)); r = fpd_to_fpl(rd).v; break;
    case FPD_EVAL_Y_FROM_X: flag = g1_y_from_x_fpd(r, x, y.l[0] != 0) ? 1u : 0u; break;
    default: break;
    }
    uint32_t* o = out + size_t(i) * kFpEvalOut;
    for (int k = 0; k < 12; k++) { o[k] = r.l[k]; o[12 + k] = 0; }
    if (fpd_out)
        for (int k = 0; k < 8; k++) {
            o[2 * k] = uint32_t(__double2loint(rd.l[k]));
            o[2 * k + 1] = uint32_t(__double2hiint(rd.l[k]));
        }
    o[24] = flag;
}

// Curve stages on FpL against the big-integer oracle (b200_curve_eval): the per-key kernel's Jacobian formulas and
// subgroup check with this unit's products.  Operands are taken as given, any representative in [0, 2p), so that a test
// can hand the exceptional branches a coordinate difference equal to p instead of 0.
__global__ void k_curve_eval(int32_t op, uint32_t n, const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                             uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* pa = a + size_t(i) * kCurveEvalWords;
    const uint32_t* pb = b + size_t(i) * kCurveEvalWords;
    Jac<FpL> p, q, r;
    for (int k = 0; k < 12; k++) {
        p.x.v.l[k] = pa[k]; p.y.v.l[k] = pa[24 + k]; p.z.v.l[k] = pa[48 + k];
        q.x.v.l[k] = pb[k]; q.y.v.l[k] = pb[24 + k]; q.z.v.l[k] = pb[48 + k];
    }
    jac_set_inf(r);
    uint32_t flag = 0;
    switch (op) {
    case CURVE_G1L_ADD_MIXED: jac_add_mixed(r, p, q.x, q.y); break;
    case CURVE_G1L_ADD: jac_add(r, p, q); break;
    case CURVE_G1L_DOUBLE: jac_double(r, p); break;
    case CURVE_G1L_IN_SUBGROUP: {
        G1Aff s;
        s.x = p.x.v; s.y = p.y.v; s.inf = pa[72];
        flag = g1_in_subgroup_lazy(s) ? 1u : 0u;
        break;
    }
    case CURVE_G1_IN_SUBGROUP_ISO: flag = g1_in_subgroup_iso(p.x.v) ? 1u : 0u; break;
    default: break;
    }
    uint32_t* o = out + size_t(i) * kCurveEvalWords;
    for (int k = 0; k < 72; k++) o[k] = 0;
    for (int k = 0; k < 12; k++) { o[k] = r.x.v.l[k]; o[24 + k] = r.y.v.l[k]; o[48 + k] = r.z.v.l[k]; }
    o[72] = flag;
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
// Shared memory of a per-key kernel launch.  Its square root is a fixed chain in registers (fpl_sqrt_chain), so it reaches
// no pow table: no dynamic shared memory, and the carve-out asks for all of the SM's unified L1 / shared array as L1,
// where the 168-register kernel's stack frames (384 threads x 280 B at 12 warps per SM) have to stay.
template <class K>
static size_t k1_smem(K kernel, unsigned threads) {
#if defined(B200_G1_CANONICAL_FP)
    return with_pow_tab(kernel, threads);   // fp_sqrt -> fp_pow
#else
    (void)threads;
    static const void* done[4];
    static int n_done = 0;
    const void* key = reinterpret_cast<const void*>(kernel);
    for (int i = 0; i < n_done; i++)
        if (done[i] == key) return 0;
    cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 0);
    if (n_done < 4) done[n_done++] = key;
    return 0;
#endif
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
    case 6: k_g1_validate_r128<<<(n + 511) / 512, 512, k1_smem(k_g1_validate_r128, 512), st>>>(keys, n, out, codes); break;
    case 0: k_g1_validate_main<<<(n + 255) / 256, 256, k1_smem(k_g1_validate_main, 256), st>>>(keys, n, out, codes); break;
    default:
        // 12 warps per SM either way; below ~3 full waves of 384-thread CTAs the keys go out as three 128-thread CTAs per
        // SM of the unsplit kernel, so that the last, partial wave spreads over all SMs instead of leaving most of them
        // idle; larger launches run the role-split kernel
        if (cta == 128 || (cta != 384 && n <= g_g1_small_n))
            k_g1_validate_r168<<<(n + 127) / 128, 128, k1_smem(k_g1_validate_r168, 128), st>>>(keys, n, out, codes);
        else
            k_g1_validate_split<<<(n + kSplitIntThreads - 1) / kSplitIntThreads, kSplitThreads,
                                  k1_smem(k_g1_validate_split, kSplitThreads), st>>>(keys, n, out, codes);
        break;
    }
}
// The registry's key staging from a resident state: the 48-byte public key at the head of each 121-byte Validator record,
// packed back to back so that K1 reads every key as three 16-byte words.  Records sit at odd byte offsets: byte loads.
// `index` (device, optional): key i is that of record index[i] (a sync committee's members) instead of record i.
static __global__ void k_gather_validator_keys(const uint8_t* __restrict__ records, const uint64_t* __restrict__ index, uint32_t n,
                                               uint4* __restrict__ keys) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* r = records + (index ? index[i] : uint64_t(i)) * 121;
    uint32_t w[12];
#pragma unroll
    for (int k = 0; k < 12; k++)
        w[k] = uint32_t(r[4 * k]) | uint32_t(r[4 * k + 1]) << 8 | uint32_t(r[4 * k + 2]) << 16 | uint32_t(r[4 * k + 3]) << 24;
#pragma unroll
    for (int k = 0; k < 3; k++) keys[size_t(i) * 3 + k] = make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
}
void launch_gather_validator_keys(const uint8_t* records, uint32_t n, uint8_t* keys, void* stream, const uint64_t* index) {
    if (!n) return;
    k_gather_validator_keys<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(records, index, n, reinterpret_cast<uint4*>(keys));
}
void launch_g1_aggregate(const G1Aff* keys, const int32_t* key_codes, const uint32_t* index, const uint32_t* off,
                         uint32_t n_tuples, G1Aff* agg, G1Pre* agg_pre, int32_t* pk_code, uint32_t* flags,
                         uint32_t extra_flags, void* stream, G1Jac* agg_jac, const uint32_t* tuple_flags) {
    if (!n_tuples) return;
    k_g1_aggregate<<<(n_tuples + kAggWarps - 1) / kAggWarps, 32 * kAggWarps, with_pow_tab(k_g1_aggregate, 32 * kAggWarps),
                     static_cast<cudaStream_t>(stream)>>>(
        keys, key_codes, index, off, n_tuples, agg, agg_pre, pk_code, flags, extra_flags, agg_jac, tuple_flags);
}
void launch_g1_pair_operands(const G1Aff* keys, const uint32_t* index, uint32_t n, G1Pre* pre, G1Aff* aff, void* stream) {
    if (!n) return;
    k_g1_pair_operands<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(keys, index, n, pre, aff);
}
void launch_g1_compress_groups(const G1Aff* agg, const int32_t* pk_code, const uint32_t* flags, uint32_t n_groups, uint8_t* out48,
                               int32_t* out_code, void* stream) {
    if (!n_groups) return;
    const unsigned t = n_groups <= 32 ? 32 : 128;
    k_g1_compress_groups<<<(n_groups + t - 1) / t, t, with_pow_tab(k_g1_compress_groups, t), static_cast<cudaStream_t>(stream)>>>(
        agg, pk_code, flags, n_groups, out48, out_code);
}
void launch_neg_g1(G1Aff* out, G1Pre* out_pre, void* stream) { k_neg_g1<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(out, out_pre); }
void launch_fp_selftest(uint32_t n, uint32_t seed, uint32_t* out_mismatch, void* stream) {
    k_fp_selftest<<<(n + 127) / 128, 128, with_pow_tab(k_fp_selftest, 128), static_cast<cudaStream_t>(stream)>>>(n, seed, out_mismatch);
}
void launch_fp_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream) {
    if (!n) return;
    k_fp_eval<<<(n + 127) / 128, 128, with_pow_tab(k_fp_eval, 128), static_cast<cudaStream_t>(stream)>>>(op, n, a, b, out);
}
void launch_curve_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream) {
    if (!n) return;
    k_curve_eval<<<(n + 127) / 128, 128, with_pow_tab(k_curve_eval, 128), static_cast<cudaStream_t>(stream)>>>(op, n, a, b, out);
}

}  // namespace b200
