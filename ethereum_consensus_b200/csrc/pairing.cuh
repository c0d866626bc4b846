// Optimal-ate pairing check for BLS12-381: Miller loop over |z| with Jacobian line functions on the M-twist and
// the final exponentiation (easy part + Hayashida-Hayasaka-Teruya hard part, exponent 3(p^4-p^2+1)/r).
// This is what blst runs under `Signature::{verify, fast_aggregate_verify, aggregate_verify}` for
// ethereum-consensus/src/crypto/bls.rs:64-132.
//
// Line through T (Jacobian X,Y,Z on E') evaluated at P = (xP, yP) in G1, scaled by factors in Fp2 (killed by the
// final exponentiation), in the basis 1, v, v*w of Fp12:
//   doubling:  A = 3X^3 - 2Y^2,        B = -3X^2 Z^2 * xP,  C = Z3 Z^2 * yP   (Z3 = 2YZ)
//   addition:  A = Rr*x2 - y2*Z3,      B = -Rr * xP,        C = Z3 * yP       (H = x2 Z^2 - X, Rr = y2 Z^3 - Y, Z3 = Z H)
#pragma once
#include "fp12.cuh"
#include "groups.cuh"

namespace b200 {

B200_BIG void miller_double_step(G2Jac& t, Fp2& A, Fp2& B, Fp2& C, const Fp& xp, const Fp& yp) {
    Fp2 xx, yy, zz, e, tmp;
    fp2_sqr(xx, t.x);
    fp2_sqr(yy, t.y);
    fp2_sqr(zz, t.z);
    fp2_dbl(e, xx);
    fp2_add(e, e, xx);             // 3X^2
    fp2_mul(A, e, t.x);
    fp2_dbl(tmp, yy);
    fp2_sub(A, A, tmp);            // 3X^3 - 2Y^2
    fp2_mul(tmp, e, zz);
    fp2_mul_fp(tmp, tmp, xp);
    fp2_neg(B, tmp);               // -3X^2 Z^2 xP
    jac_double(t, t);
    fp2_mul(tmp, t.z, zz);
    fp2_mul_fp(C, tmp, yp);        // Z3 Z^2 yP
}

B200_BIG void miller_add_step(G2Jac& t, Fp2& A, Fp2& B, Fp2& C, const G2Aff& q, const Fp& xp, const Fp& yp) {
    Fp2 zz, zzz, h, rr, hh, hhh, v, x3, tmp, z3;
    fp2_sqr(zz, t.z);
    fp2_mul(zzz, zz, t.z);
    fp2_mul(h, q.x, zz);
    fp2_sub(h, h, t.x);
    fp2_mul(rr, q.y, zzz);
    fp2_sub(rr, rr, t.y);
    fp2_mul(z3, t.z, h);
    fp2_mul(A, rr, q.x);
    fp2_mul(tmp, q.y, z3);
    fp2_sub(A, A, tmp);
    fp2_mul_fp(tmp, rr, xp);
    fp2_neg(B, tmp);
    fp2_mul_fp(C, z3, yp);
    fp2_sqr(hh, h);
    fp2_mul(hhh, hh, h);
    fp2_mul(v, t.x, hh);
    fp2_sqr(x3, rr);
    fp2_sub(x3, x3, hhh);
    fp2_dbl(tmp, v);
    fp2_sub(x3, x3, tmp);
    fp2_sub(tmp, v, x3);
    fp2_mul(tmp, rr, tmp);
    fp2_mul(hhh, t.y, hhh);
    fp2_sub(t.y, tmp, hhh);
    t.x = x3;
    t.z = z3;
}

// f_{z,Q}(P); 1 if either point is the point at infinity
B200_BIG void miller_loop(Fp12& f, const G1Aff& p, const G2Aff& q) {
    f = fp12_one();
    if (p.inf || q.inf) return;
    G2Jac t;
    jac_from_aff(t, q);
    Fp2 A, B, C;
    const uint64_t z = B200_Z_ABS;
    bool first = true;
#pragma unroll 1
    for (int bit = 62; bit >= 0; bit--) {
        if (!first) fp12_sqr(f, f);
        first = false;
        miller_double_step(t, A, B, C, p.x, p.y);
        fp12_mul_by_line(f, f, A, B, C);
        if ((z >> bit) & 1) {
            miller_add_step(t, A, B, C, q, p.x, p.y);
            fp12_mul_by_line(f, f, A, B, C);
        }
    }
    fp12_conj(f, f);  // z < 0
}

// g^|z| by square-and-multiply; g must lie in the cyclotomic subgroup (true after the easy part)
B200_BIG void fp12_pow_z(Fp12& r, const Fp12& g) {
    Fp12 acc = g;
    const uint64_t z = B200_Z_ABS;
#pragma unroll 1
    for (int bit = 62; bit >= 0; bit--) {
        fp12_cyclotomic_sqr(acc, acc);
        if ((z >> bit) & 1) fp12_mul(acc, acc, g);
    }
    r = acc;
}

// c = f^((p^12-1)/r * 3); the inverse path maps 0 to 0
B200_BIG void final_exp(Fp12& c, const Fp12& f_in) {
    Fp12 f, t0, t1, a, b;
    // easy part: f^((p^6-1)(p^2+1))
    fp12_inv(t0, f_in);
    fp12_conj(t1, f_in);
    fp12_mul(t0, t1, t0);
    fp12_frobenius<2>(t1, t0);
    fp12_mul(f, t1, t0);
    // hard part: (x-1)^2 (x+p)(x^2+p^2-1) + 3, x = -|z|; inverse = conjugate in the cyclotomic subgroup
    fp12_pow_z(t0, f); fp12_mul(t0, t0, f); fp12_conj(t0, t0);        // f^(x-1)
    fp12_pow_z(a, t0); fp12_mul(a, a, t0); fp12_conj(a, a);           // f^((x-1)^2)
    fp12_pow_z(t0, a); fp12_conj(t0, t0);                             // a^x
    fp12_frobenius<1>(t1, a);
    fp12_mul(b, t0, t1);                                              // a^(x+p)
    fp12_pow_z(t0, b); fp12_pow_z(t0, t0);                            // b^(x^2)
    fp12_frobenius<2>(t1, b);
    fp12_mul(c, t0, t1);
    fp12_conj(t1, b);
    fp12_mul(c, c, t1);                                               // b^(x^2+p^2-1)
    fp12_sqr(t0, f); fp12_mul(t0, t0, f);                             // f^3
    fp12_mul(c, c, t0);
}

// f^((p^12-1)/r * 3) == 1 ?
B200_BIG bool final_exp_is_one(const Fp12& f_in) {
    Fp12 c;
    final_exp(c, f_in);
    return fp12_is_one(c);
}

}  // namespace b200
