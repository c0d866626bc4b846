// FpL: "lazily reduced" base-field elements for the per-key kernel (bls_g1.cu) — any representative in [0, 2p).
//
// Why: a profile of the per-key kernel shows the FMA-heavy pipe only two-thirds busy with
// `wait` as the top stall; the SASS explains it: every IMAD.WIDE carries a 4-cycle issue stall, so ONE warp streaming
// wide MADs already saturates its scheduler's share of the pipe, and the pipe idles exactly while warps run the
// ALU-only glue between products — the conditional subtraction after every Montgomery product and the add/sub/select
// chains of the group law.  With R = 2^384 and p < 2^381 the product has three bits of slack: for a, b < 2p,
// a*b/R + p < (4p/R) p + p < 1.41 p, so products of [0, 2p) inputs land in [0, 2p) again WITHOUT any final
// subtraction.  FpL keeps every intermediate in [0, 2p): mul / sqr are the bare PTX sequences, add / sub / neg reduce
// modulo 2p (same instruction count as modulo p), and only comparisons and the final outputs canonicalise.
// A distinct type (not a flag) so that the compiler rejects any mixing with canonical Fp; the templated curve code
// (curve.cuh) is reused unchanged through the f_* overloads.
#pragma once
#include "curve.cuh"

namespace b200 {

struct FpL {
    Fp v;
};

B200_HD Fp fp_2p() { Fp r = B200_FP_2P; return r; }

// r in [0, 4p) -> [0, 2p)
B200_HD void fpl_reduce_2p(Fp& r) {
    const Fp pp = fp_2p();
    Fp t;
    const uint32_t borrow = fp_sub_raw(t, r, pp);
    fp_select(r, t, borrow == 0);
}
B200_HD FpL fpl_from_fp(const Fp& a) { FpL r; r.v = a; return r; }
// canonical representative in [0, p)
B200_HD Fp fpl_canon(const FpL& a) { Fp r = a.v; fp_reduce_once(r); return r; }

B200_HD void f_add(FpL& r, const FpL& a, const FpL& b) {
    fp_add_raw(r.v, a.v, b.v);  // < 4p < 2^384: no carry out
    fpl_reduce_2p(r.v);
}
B200_HD void f_sub(FpL& r, const FpL& a, const FpL& b) {
    Fp t;
    const uint32_t borrow = fp_sub_raw(t, a.v, b.v);
    fp_add_masked_raw(r.v, t, fp_2p(), 0u - borrow);
}
B200_HD void f_dbl(FpL& r, const FpL& a) { f_add(r, a, a); }
B200_HD void f_neg(FpL& r, const FpL& a) {
    FpL z; z.v = fp_zero();
    f_sub(r, z, a);   // 0 -> 0, otherwise 2p - a in (0, 2p)
}
#if defined(__CUDA_ARCH__) && defined(B200_FP_MUL_CALL)
// A/B knob (-DB200_G1_CALL_MUL): the two products as real functions, operands and result by value in registers — one
// ~4 KB copy of each instead of ~70 inlined copies (the per-key kernel is 0.5 MB of straight-line code otherwise)
static __device__ __noinline__ Fp fpl_mul_call(Fp a, Fp b) { Fp out; fp_mul_ptx_core(out.l, a.l, b.l); return out; }
static __device__ __noinline__ Fp fpl_sqr_call(Fp a) {
    Fp out;
#if defined(B200_FP_SQR_VIA_MUL)
    fp_mul_ptx_core(out.l, a.l, a.l);
#else
    fp_sqr_ptx_core(out.l, a.l);
#endif
    return out;
}
#endif
// products without the final conditional subtraction: [0, 2p) x [0, 2p) -> [0, 1.41 p)
B200_HD void f_mul(FpL& r, const FpL& a, const FpL& b) {
    Fp out;
#if defined(__CUDA_ARCH__) && defined(B200_FP_MUL_CALL)
    out = fpl_mul_call(a.v, b.v);
#elif defined(__CUDA_ARCH__) && !defined(B200_FP_PORTABLE)
    fp_mul_ptx_core(out.l, a.v.l, b.v.l);
#else
    fp_mul_emul_core(out.l, a.v.l, b.v.l);   // host: the C emulation of the very same instruction list
#endif
    r.v = out;
}
B200_HD void f_sqr(FpL& r, const FpL& a) {
    Fp out;
#if defined(__CUDA_ARCH__) && defined(B200_FP_MUL_CALL)
    out = fpl_sqr_call(a.v);
#elif defined(__CUDA_ARCH__) && !defined(B200_FP_PORTABLE)
#if defined(B200_FP_SQR_VIA_MUL)
    fp_mul_ptx_core(out.l, a.v.l, a.v.l);
#else
    fp_sqr_ptx_core(out.l, a.v.l);
#endif
#else
#if defined(B200_FP_SQR_VIA_MUL)
    fp_mul_emul_core(out.l, a.v.l, a.v.l);
#else
    fp_sqr_emul_core(out.l, a.v.l);
#endif
#endif
    r.v = out;
}
B200_HD bool f_is_zero(const FpL& a) { return fp_is_zero(fpl_canon(a)); }
B200_HD bool f_eq(const FpL& a, const FpL& b) { return fp_eq(fpl_canon(a), fpl_canon(b)); }
template <> B200_HD FpL f_one<FpL>() { return fpl_from_fp(fp_one()); }
template <> B200_HD FpL f_zero<FpL>() { return fpl_from_fp(fp_zero()); }
template <> B200_HD FpL curve_b<FpL>() { Fp b = B200_FP_B_G1; return fpl_from_fp(b); }

// a^e with lazily reduced squarings / products (same sliding 4-bit windows and table placement as fp_pow, fp.cuh)
B200_BIG void fpl_pow(FpL& r, const FpL& a, const uint32_t* e) {
    PowTab tab;  // tab[k] = a^(2k+1), entries in [0, 2p)
    tab.set(0, a.v);
    {
        FpL a2, cur = a;
        f_sqr(a2, a);
#pragma unroll 1
        for (int k = 1; k < kPowTabEntries; k++) { f_mul(cur, cur, a2); tab.set(k, cur.v); }
    }
    int i = 383;
    while (i >= 0 && !((e[i >> 5] >> (i & 31)) & 1u)) i--;
    if (i < 0) { r = f_one<FpL>(); return; }
    FpL acc, t;
    bool started = false;
#pragma unroll 1
    while (i >= 0) {
        if (!((e[i >> 5] >> (i & 31)) & 1u)) {
            f_sqr(acc, acc);
            i--;
            continue;
        }
        int l = i + 1 < 4 ? i + 1 : 4;
        const int lo = i - l + 1;
        uint64_t two = e[lo >> 5];
        if ((lo >> 5) + 1 < 12) two |= uint64_t(e[(lo >> 5) + 1]) << 32;
        uint32_t w = uint32_t(two >> (lo & 31)) & ((1u << l) - 1u);
        while (!(w & 1u)) { w >>= 1; l--; }
        if (started) {
#pragma unroll 1
            for (int k = 0; k < l; k++) f_sqr(acc, acc);
            tab.get(t.v, int(w >> 1));
            f_mul(acc, acc, t);
        } else {
            tab.get(acc.v, int(w >> 1));
            started = true;
        }
        i -= l;
    }
    r = acc;
}

}  // namespace b200
