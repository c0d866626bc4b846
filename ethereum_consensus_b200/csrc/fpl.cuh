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
// B200_FP_MUL_CALL (fp.cuh): the two products as real functions, operands and result by value in registers — one
// ~4 KB copy of each instead of ~70 inlined copies (the per-key kernel is 0.5 MB of straight-line code otherwise)
static __device__ __noinline__ Fp fpl_mul_call(Fp a, Fp b) { Fp out; fp_mul_ptx_core(out.l, a.l, b.l); return out; }
static __device__ __noinline__ Fp fpl_sqr_call(Fp a) { Fp out; fp_sqr_ptx_core(out.l, a.l); return out; }
#endif
// products without the final conditional subtraction: [0, 2p) x [0, 2p) -> [0, 1.41 p)
B200_HD void f_mul(FpL& r, const FpL& a, const FpL& b) {
    Fp out;
#if defined(__CUDA_ARCH__) && defined(B200_FP_MUL_CALL)
    out = fpl_mul_call(a.v, b.v);
#elif defined(__CUDA_ARCH__)
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
#elif defined(__CUDA_ARCH__)
    fp_sqr_ptx_core(out.l, a.v.l);
#else
    fp_sqr_emul_core(out.l, a.v.l);
#endif
    r.v = out;
}

// ---- one Montgomery reduction for a difference of products (the Y3 of the Jacobian formulas below) ----------------
// R = 2^384 and p/R < 0.102, so REDC(T) = (T + m p)/R < T/R + p for any T < 2^768 (m < R).  Operands in [0, 2p).
// f_mul_sub_mul: r = (a b - c d)/R.  T = a b + c (2p - d): the offset 2p c is a multiple of p, 2p - d lies in (0, 2p],
//   so T is in [0, 8p^2) and r < 8 (p/R) p + p < 1.82 p.  No fix-up.  2 x 144 + 144 wide MADs instead of 2 x 288.
// f_mul_sub_8sqr: r = (a b - 8 c^2)/R.  T = a b + 32p^2 - 8c^2 is in (0, 36p^2) < 2^767, so REDC < 36 (p/R) p + p < 4.66 p;
//   subtracting 4p, then 2p, where they fit brings r to [0, 2p).  144 + 78 + 144 wide MADs instead of 222 + 288.
B200_HD Fp fp_4p() {
    Fp r = {{0xfffeaaacu, 0xe7fbffffu, 0xc54ffffeu, 0x7aaffffau, 0xdac3d890u, 0x9cc34a83u, 0xce144afdu, 0x91dd2e13u,
             0x0d2eb35du, 0x2c6e9ed9u, 0xe5ff9a69u, 0x680447a8u}};
    return r;
}
// r in [0, 8p) -> [0, 4p)
B200_HD void fpl_reduce_4p(Fp& r) {
    const Fp pp = fp_4p();
    Fp t;
    const uint32_t borrow = fp_sub_raw(t, r, pp);
    fp_select(r, t, borrow == 0);
}
B200_HD Fp fpl_mul_sub_mul_core(const Fp& a, const Fp& b, const Fp& c, const Fp& d) {
    Fp nd, out;
    fp_sub_raw(nd, fp_2p(), d);
#if defined(__CUDA_ARCH__)
    fp_mul_add_mul_ptx_core(out.l, a.l, b.l, c.l, nd.l);
#else
    fp_mul_add_mul_emul_core(out.l, a.l, b.l, c.l, nd.l);
#endif
    return out;
}
B200_HD Fp fpl_mul_sub_8sqr_core(const Fp& a, const Fp& b, const Fp& c) {
    Fp out;
#if defined(__CUDA_ARCH__)
    fp_mul_sub_8sqr_ptx_core(out.l, a.l, b.l, c.l);
#else
    fp_mul_sub_8sqr_emul_core(out.l, a.l, b.l, c.l);
#endif
    fpl_reduce_4p(out);
    fpl_reduce_2p(out);
    return out;
}
#if defined(__CUDA_ARCH__) && defined(B200_FP_MUL_CALL)
// by-value call units like fpl_mul_call: no 24-word value crosses a function boundary
static __device__ __noinline__ Fp fpl_mul_sub_mul_call(Fp a, Fp b, Fp c, Fp d) { return fpl_mul_sub_mul_core(a, b, c, d); }
static __device__ __noinline__ Fp fpl_mul_sub_8sqr_call(Fp a, Fp b, Fp c) { return fpl_mul_sub_8sqr_core(a, b, c); }
#endif
B200_HD void f_mul_sub_mul(FpL& r, const FpL& a, const FpL& b, const FpL& c, const FpL& d) {
#if defined(__CUDA_ARCH__) && defined(B200_FP_MUL_CALL)
    r.v = fpl_mul_sub_mul_call(a.v, b.v, c.v, d.v);
#else
    r.v = fpl_mul_sub_mul_core(a.v, b.v, c.v, d.v);
#endif
}
B200_HD void f_mul_sub_8sqr(FpL& r, const FpL& a, const FpL& b, const FpL& c) {
#if defined(__CUDA_ARCH__) && defined(B200_FP_MUL_CALL)
    r.v = fpl_mul_sub_8sqr_call(a.v, b.v, c.v);
#else
    r.v = fpl_mul_sub_8sqr_core(a.v, b.v, c.v);
#endif
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

// a = a^(2^n): the squaring runs of the fixed chains, one call site per run
B200_HD void fpl_sqr_n(FpL& a, int n) {
#pragma unroll 1
    for (int k = 0; k < n; k++) f_sqr(a, a);
}

// ---- FpL overloads of curve.cuh's doubling and additions: Y3 by one fused reduction --------------------------------
// Same formulas, branches and canonicalising comparisons as the templates (which Fp and Fp2 keep); the templated ladders
// (jac_mul_u64*, jac_add) reach these through argument-dependent lookup, where a non-template overload wins.
// dbl-2009-l (a = 0) with D = 4 X B, which equals 2((X + B)^2 - A - C): C = B^2 is then only needed in Y3 = E (D - X3) - 8C,
// and f_mul_sub_8sqr forms it from B without reducing B^2.  2M + 3S + one fused step = 1 608 wide MADs instead of 1 686.
B200_BIG void jac_double(Jac<FpL>& r, const Jac<FpL>& p) {
    FpL A, B, D, E, Fq, t;
    f_sqr(A, p.x);
    f_sqr(B, p.y);
    f_mul(D, p.x, B);
    f_dbl(D, D); f_dbl(D, D);
    f_dbl(E, A);
    f_add(E, E, A);
    f_sqr(Fq, E);
    FpL z3;
    f_mul(z3, p.y, p.z);
    f_dbl(z3, z3);
    FpL x3;
    f_dbl(t, D);
    f_sub(x3, Fq, t);
    f_sub(t, D, x3);
    f_mul_sub_8sqr(r.y, E, t, B);
    r.x = x3;
    r.z = z3;
}

B200_BIG void jac_add_mixed(Jac<FpL>& r, const Jac<FpL>& p, const FpL& qx, const FpL& qy) {
    if (jac_is_inf(p)) { r.x = qx; r.y = qy; r.z = f_one<FpL>(); return; }
    FpL zz, zzz, u2, s2, h, rr;
    f_sqr(zz, p.z);
    f_mul(zzz, zz, p.z);
    f_mul(u2, qx, zz);
    f_mul(s2, qy, zzz);
    f_sub(h, u2, p.x);
    f_sub(rr, s2, p.y);
    if (f_is_zero(h)) {
        if (f_is_zero(rr)) { Jac<FpL> t; t.x = qx; t.y = qy; t.z = f_one<FpL>(); jac_double(r, t); }
        else jac_set_inf(r);
        return;
    }
    FpL hh, hhh, v, x3, t;
    f_sqr(hh, h);
    f_mul(hhh, hh, h);
    f_mul(v, p.x, hh);
    f_sqr(x3, rr);
    f_sub(x3, x3, hhh);
    f_dbl(t, v);
    f_sub(x3, x3, t);
    f_sub(t, v, x3);
    f_mul_sub_mul(r.y, rr, t, p.y, hhh);   // rr (V - X3) - Y1 HHH
    f_mul(r.z, p.z, h);
    r.x = x3;
}

B200_HD void jac_add_zz(Jac<FpL>& r, const Jac<FpL>& p, const Jac<FpL>& q, const FpL& z2z2, const FpL& z2z3) {
    if (jac_is_inf(p)) { r = q; return; }
    if (jac_is_inf(q)) { r = p; return; }
    FpL z1z1, u1, u2, s1, s2, h, rr, t;
    f_sqr(z1z1, p.z);
    f_mul(u1, p.x, z2z2);
    f_mul(u2, q.x, z1z1);
    f_mul(s1, p.y, z2z3);
    f_mul(t, p.z, z1z1);
    f_mul(s2, q.y, t);
    f_sub(h, u2, u1);
    f_sub(rr, s2, s1);
    if (f_is_zero(h)) {
        if (f_is_zero(rr)) jac_double(r, p); else jac_set_inf(r);
        return;
    }
    FpL hh, hhh, v, x3;
    f_sqr(hh, h);
    f_mul(hhh, hh, h);
    f_mul(v, u1, hh);
    f_sqr(x3, rr);
    f_sub(x3, x3, hhh);
    f_dbl(t, v);
    f_sub(x3, x3, t);
    f_sub(t, v, x3);
    f_mul_sub_mul(r.y, rr, t, s1, hhh);    // rr (V - X3) - S1 HHH
    f_mul(t, p.z, q.z);
    f_mul(r.z, t, h);
    r.x = x3;
}

}  // namespace b200

// fpl_sqrt_chain(r, a): r = a^((p+1)/4), no table (what the per-key kernel's decompression runs)
#include "fpl_sqrt_chain.cuh"
