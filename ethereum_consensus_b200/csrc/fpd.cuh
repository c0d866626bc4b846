// FpD: base-field elements on the FP64 pipe, for the per-key kernel's decompression square root (bls_g1.cu).
//
// Why: the per-key kernel's integer products keep the FMA-heavy pipe about 90 % busy while the FP64 pipe idles.  The
// square root is a third of the kernel's wide multiply-adds and depends on nothing the subgroup check computes, so
// it runs here, on warps of its own, as exact integer arithmetic in doubles.
//
// Representation: 8 limbs of 48 bits in the same Montgomery domain as Fp / FpL (R = 2^384).  Limb k is held at its
// true magnitude: l[k] is an integer multiple of 2^(48k) (the double's exponent does the scaling, so no multiply by a
// radix power is ever needed), balanced: |l[k]| <= 2^(48k+47) for k < 7.  Values are signed representatives: the
// quotient digits of the reduction are balanced too, so a product of |a|, |b| < 2p lies in (-0.91 p, 0.91 p).
//
// Exactness: every partial product a_i b_j (|.| <= 2^(48(i+j)+94)) is split into hi, a multiple of 2^(48(i+j+1)), and
// lo = a_i b_j - hi with |lo| <= 2^(48(i+j)+47): hi = fma(a, b, K) - K rounds to that multiple because K = 1.5 *
// 2^(48(i+j)+100) puts the sum in a binade whose ulp is 2^(48(i+j+1)), and fma(a, b, -hi) is then exact.  A column
// collects fewer than 2^52 units of its weight, so every sum of the product is exact and order-independent: the host
// build (std::fma) computes the same bits as the device's DFMA sequence.  No int <-> double conversion inside a
// product; conversions happen only in fpd_from_fp / fpd_to_fpl, once per chain.
#pragma once
#include <cmath>
#include <cstring>

#include "fpl.cuh"

namespace b200 {

struct FpD {
    double l[8];
};

// 2^e from its bits (the unrolled loops below fold it to a constant)
B200_HD double fpd_pow2(int e) {
    const uint64_t bits = uint64_t(1023 + e) << 52;
#if defined(__CUDA_ARCH__)
    return __longlong_as_double(static_cast<long long>(bits));
#else
    double d;
    std::memcpy(&d, &bits, sizeof d);
    return d;
#endif
}
// 1.5 * 2^(48c+100): split and carry constant of column c
B200_HD double fpd_k(int c) { return 1.5 * fpd_pow2(48 * c + 100); }
// p in balanced 48-bit limbs, p_j at weight 2^(48j)
B200_HD constexpr double fpd_p(int j) {
    return j == 0 ? -21845.0
         : j == 1 ? -86500641359361.0 * 0x1p48
         : j == 2 ? -10839982866433.0 * 0x1p96
         : j == 3 ? 113459389855409.0 * 0x1p144
         : j == 4 ? 83034393350847.0 * 0x1p192
         : j == 5 ? 73992301405303.0 * 0x1p240
         : j == 6 ? -27924617254986.0 * 0x1p288
         : 28591897852288.0 * 0x1p336;
}
// -p^-1 mod 2^48, balanced
constexpr double kFpdPinv = -12885098499.0;

#if defined(__CUDA_ARCH__)
B200_HD double fpd_fma(double a, double b, double c) { return __fma_rn(a, b, c); }
#else
B200_HD double fpd_fma(double a, double b, double c) { return std::fma(a, b, c); }
#endif

// t[c] += lo, t[c+1] += hi for the product a b of column c
B200_HD void fpd_mac(double* t, int c, double a, double b) {
    const double k = fpd_k(c);
    const double hi = fpd_fma(a, b, k) - k;
    t[c] += fpd_fma(a, b, -hi);
    t[c + 1] += hi;
}

// Montgomery reduction of the 16 columns (t[c] at weight 2^(48c), |t[c]| < 2^(48c+52)) into r = t / R
B200_HD void fpd_redc(FpD& r, double* t) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const double v = t[i];
        const double h = fpd_fma(v, kFpdPinv, fpd_k(i)) - fpd_k(i);
        const double q = fpd_fma(v, kFpdPinv, -h);   // q = (v p') mod 2^(48(i+1)), balanced, at weight 2^(48i)
        t[i + 1] += fpd_fma(q, fpd_p(0), v);         // v + q p_0 is a multiple of 2^(48(i+1)) with 47 bits: exact
#pragma unroll
        for (int j = 1; j < 8; j++) fpd_mac(t, i + j, q, fpd_p(j));
    }
#pragma unroll
    for (int c = 8; c < 15; c++) {
        const double cy = (t[c] + fpd_k(c)) - fpd_k(c);
        t[c] -= cy;
        t[c + 1] += cy;
    }
#pragma unroll
    for (int k = 0; k < 8; k++) r.l[k] = t[8 + k] * 0x1p-384;
}

B200_HD void fpd_mul_core(FpD& r, const FpD& a, const FpD& b) {
    double t[16];
#pragma unroll
    for (int c = 0; c < 16; c++) t[c] = -0.0;
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) fpd_mac(t, i + j, a.l[i], b.l[j]);
    fpd_redc(r, t);
}
B200_HD void fpd_sqr_core(FpD& r, const FpD& a) {
    double t[16], a2[8];
#pragma unroll
    for (int c = 0; c < 16; c++) t[c] = -0.0;
#pragma unroll
    for (int j = 1; j < 8; j++) a2[j] = a.l[j] + a.l[j];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        fpd_mac(t, 2 * i, a.l[i], a.l[i]);
#pragma unroll
        for (int j = i + 1; j < 8; j++) fpd_mac(t, i + j, a.l[i], a2[j]);
    }
    fpd_redc(r, t);
}

#if defined(__CUDA_ARCH__)
// by-value calls like fpl_mul_call: one copy of each body (about 11 KB and 9 KB of code) instead of one per chain step
static __device__ __noinline__ FpD fpd_mul_call(FpD a, FpD b) { FpD r; fpd_mul_core(r, a, b); return r; }
static __device__ __noinline__ FpD fpd_sqr_call(FpD a) { FpD r; fpd_sqr_core(r, a); return r; }
B200_HD void fpd_mul(FpD& r, const FpD& a, const FpD& b) { r = fpd_mul_call(a, b); }
B200_HD void fpd_sqr(FpD& r, const FpD& a) { r = fpd_sqr_call(a); }
#else
B200_HD void fpd_mul(FpD& r, const FpD& a, const FpD& b) { fpd_mul_core(r, a, b); }
B200_HD void fpd_sqr(FpD& r, const FpD& a) { fpd_sqr_core(r, a); }
#endif
// a = a^(2^n): the squaring runs of the chain, one call site per run
B200_HD void fpd_sqr_n(FpD& a, int n) {
#pragma unroll 1
    for (int k = 0; k < n; k++) fpd_sqr(a, a);
}

// carries of limbs 0..6 into the next limb: back to balanced limbs (after an addition, whose limbs reach 2^(48k+48))
B200_HD void fpd_normalize(FpD& a) {
#pragma unroll
    for (int k = 0; k < 7; k++) {
        const double cy = (a.l[k] + fpd_k(k)) - fpd_k(k);
        a.l[k] -= cy;
        a.l[k + 1] += cy;
    }
}
B200_HD void fpd_add(FpD& r, const FpD& a, const FpD& b) {
#pragma unroll
    for (int k = 0; k < 8; k++) r.l[k] = a.l[k] + b.l[k];
    fpd_normalize(r);
}

// Fp limbs (any value below 2^384 - 2^383, here representatives in [0, 2p)) -> balanced FpD.  The conversions of the chain.
B200_HD FpD fpd_from_fp(const Fp& a) {
    FpD r;
    int64_t carry = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int w = 3 * (k >> 1);
        const uint64_t chunk = (k & 1) ? (a.l[w + 1] >> 16) | (uint64_t(a.l[w + 2]) << 16)
                                       : a.l[w] | (uint64_t(a.l[w + 1] & 0xffffu) << 32);
        int64_t d = int64_t(chunk) + carry;
        carry = 0;
        if (k < 7 && d >= (int64_t(1) << 47)) { d -= int64_t(1) << 48; carry = 1; }
        r.l[k] = double(d) * fpd_pow2(48 * k);
    }
    return r;
}
// FpD with |a| < 2p -> the FpL representative in [0, 2p)
B200_HD FpL fpd_to_fpl(const FpD& a) {
    FpL r;
    int64_t carry = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int64_t d = int64_t(a.l[k] * fpd_pow2(-48 * k)) + carry;   // an integer below 2^53: exact
        const uint64_t chunk = uint64_t(d) & ((uint64_t(1) << 48) - 1);
        carry = d >> 48;   // arithmetic: floor
        const int w = 3 * (k >> 1);
        if (k & 1) {
            r.v.l[w + 1] |= uint32_t(chunk << 16);
            r.v.l[w + 2] = uint32_t(chunk >> 16);
        } else {
            r.v.l[w] = uint32_t(chunk);
            r.v.l[w + 1] = uint32_t(chunk >> 32);
        }
    }
    // carry is 0 for a >= 0 and -1 for a < 0, whose 384-bit two's complement 2^384 + a plus 2p wraps to a + 2p
    Fp t;
    fp_add_masked_raw(t, r.v, fp_2p(), 0u - uint32_t(carry != 0));
    r.v = t;
    return r;
}

}  // namespace b200

// fpd_sqrt_chain(r, a): r = a^((p+1)/4) on the FP64 pipe
#include "fpd_sqrt_chain.cuh"

namespace b200 {

// The decompression's square root on FpD: y with y^2 = x^3 + 4 for x (Montgomery, canonical), canonical and with the
// sign the flag asks for; BLS_POINT_NOT_ON_CURVE when x^3 + 4 is not a square.  Same result as g1_uncompress_lazy.
B200_HD bool g1_y_from_x_fpd(Fp& y, const Fp& x, bool largest) {
    const Fp four = B200_FP_B_G1;
    FpD xd = fpd_from_fp(x), y2, yd, c;
    fpd_sqr(y2, xd);
    fpd_mul(y2, y2, xd);
    fpd_add(y2, y2, fpd_from_fp(four));
    fpd_sqrt_chain(yd, y2);
    fpd_sqr(c, yd);
    if (!fp_eq(fpl_canon(fpd_to_fpl(c)), fpl_canon(fpd_to_fpl(y2)))) return false;
    y = fpl_canon(fpd_to_fpl(yd));
    if (fp_is_lex_largest(y) != largest) fp_neg(y, y);
    return true;
}

}  // namespace b200
