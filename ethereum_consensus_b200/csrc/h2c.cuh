// hash_to_G2 for the ciphersuite BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_ (the DST at
// ethereum-consensus/src/crypto/bls.rs:22): RFC 9380 hash_to_curve =
// expand_message_xmd(SHA-256) -> 2 x Fp2 -> simplified SWU on the 3-isogenous curve E'' -> 3-isogeny to E' ->
// add -> clear cofactor.  blst computes the same function for every `verify`/`sign` of the reference.
#pragma once
#include "groups.cuh"
#include "sha256_hd.cuh"

namespace b200 {

B200_HD void bls_dst_prime(uint8_t out[44]) {
    const char dst[44] = "BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_";  // 43 chars + NUL
    for (int i = 0; i < 43; i++) out[i] = uint8_t(dst[i]);
    out[43] = 43;  // I2OSP(len(DST), 1)
}

// 64 big-endian bytes -> integer mod p, Montgomery form: hi(16 B) * 2^384 + lo(48 B)
B200_HD void fp_from_be64_mod_p(Fp& r, const uint8_t* b) {
    Fp lo, hi, t;
    fp_from_be_bytes_raw(lo, b + 16);
    for (int i = 0; i < 12; i++) hi.l[i] = 0;
    for (int i = 0; i < 4; i++) {
        const uint8_t* q = b + 12 - 4 * i;
        hi.l[i] = (uint32_t(q[0]) << 24) | (uint32_t(q[1]) << 16) | (uint32_t(q[2]) << 8) | q[3];
    }
    const Fp r2 = B200_FP_R2, r3 = B200_FP_R3;
    fp_mul_portable(lo, lo, r2);   // lo * R  (lo < 2^384 may exceed p: the portable product accepts it)
    fp_mul(t, hi, r3);    // hi * R * R
    fp_add(r, lo, t);
}

// hash_to_field(msg, count = 2) over Fp2: u0 = e0 + e1 u, u1 = e2 + e3 u
B200_BIG void hash_to_field_fp2(Fp2& u0, Fp2& u1, const uint8_t* msg, size_t len) {
    uint8_t dstp[44], b0[32], bi[32], tmp[32];
    bls_dst_prime(dstp);
    Sha256Ctx c;
    sha_init(c);
    const uint8_t zero64[64] = {0};
    sha_update(c, zero64, 64);
    sha_update(c, msg, len);
    const uint8_t lib[3] = {1, 0, 0};  // I2OSP(256, 2) || I2OSP(0, 1)
    sha_update(c, lib, 3);
    sha_update(c, dstp, 44);
    sha_final(c, b0);
    uint8_t uniform[256];
    for (int i = 1; i <= 8; i++) {
        sha_init(c);
        if (i == 1) sha_update(c, b0, 32);
        else {
            for (int k = 0; k < 32; k++) tmp[k] = b0[k] ^ bi[k];
            sha_update(c, tmp, 32);
        }
        const uint8_t idx = uint8_t(i);
        sha_update(c, &idx, 1);
        sha_update(c, dstp, 44);
        sha_final(c, bi);
        for (int k = 0; k < 32; k++) uniform[32 * (i - 1) + k] = bi[k];
    }
    fp_from_be64_mod_p(u0.c0, uniform);
    fp_from_be64_mod_p(u0.c1, uniform + 64);
    fp_from_be64_mod_p(u1.c0, uniform + 128);
    fp_from_be64_mod_p(u1.c1, uniform + 192);
}

// g(x) = x^3 + A'x + B' on E''
B200_HD void sswu_g(Fp2& r, const Fp2& x) {
    const Fp2 A = B200_FP2_SSWU_A, B = B200_FP2_SSWU_B;
    Fp2 t;
    fp2_sqr(t, x);
    fp2_add(t, t, A);
    fp2_mul(t, t, x);
    fp2_add(r, t, B);
}
// simplified SWU: t -> (x, y) on E''
B200_BIG void sswu_map(Fp2& x, Fp2& y, const Fp2& t) {
    const Fp2 Zc = B200_FP2_SSWU_Z;
    Fp2 t2, zt2, tv1, x1, gx, yy;
    fp2_sqr(t2, t);
    fp2_mul(zt2, Zc, t2);          // Z t^2
    fp2_sqr(tv1, zt2);             // Z^2 t^4
    fp2_add(tv1, tv1, zt2);
    if (fp2_is_zero(tv1)) {
        const Fp2 c = B200_FP2_SSWU_B_OVER_ZA;
        x1 = c;
    } else {
        const Fp2 c = B200_FP2_SSWU_NEG_B_OVER_A;
        Fp2 inv, one = fp2_one();
        fp2_inv(inv, tv1);
        fp2_add(inv, inv, one);
        fp2_mul(x1, c, inv);
    }
    sswu_g(gx, x1);
    // y = sqrt(g(x1)) if that is a square, else x = Z t^2 x1 and y = sqrt(g(x)) = t^3 sqrt(Z^3 g(x1)).  One shared
    // exponentiation s = norm(g(x1))^((p+1)/4) decides which: s^2 = norm (square) or s^2 = -norm, and then
    // s * sqrt(-norm(Z^3)) is the root of norm(Z^3 g(x1)).  A second one finishes the complex-method root: two
    // exponentiations per map and no divergent retry.
    Fp n, tt, s, c;
    fp_sqr(n, gx.c0);
    fp_sqr(tt, gx.c1);
    fp_add(n, n, tt);
    fp_pow(s, n, B200_EXP_TABLE(exp_sqrt));
    fp_sqr(c, s);
    const bool is_sq = fp_eq(c, n);
    Fp2 w = gx;
    if (!is_sq) {
        const Fp2 z3 = B200_FP2_SSWU_Z3;
        const Fp cs = B200_FP_SSWU_SQRT_NEG_NORM_Z3;
        fp2_mul(w, z3, gx);
        fp_mul(s, s, cs);
    }
    bool ok = !fp_is_zero(w.c1) && fp2_sqrt_with_norm_root(yy, w, s);
    if (!ok) fp2_sqrt(yy, w);      // real w (probability ~2^-381): the general routine
    if (is_sq) {
        x = x1;
    } else {
        Fp2 t3;
        fp2_mul(x, zt2, x1);
        fp2_mul(t3, t2, t);
        fp2_mul(yy, yy, t3);
    }
    if (fp2_sgn0(t) != fp2_sgn0(yy)) fp2_neg(yy, yy);
    y = yy;
}

#define B200_HORNER4(r, x, c0, c1, c2, c3) \
    { const Fp2 k0 = c0, k1 = c1, k2 = c2, k3 = c3; r = k3; fp2_mul(r, r, x); fp2_add(r, r, k2); fp2_mul(r, r, x); fp2_add(r, r, k1); fp2_mul(r, r, x); fp2_add(r, r, k0); }
#define B200_HORNER3(r, x, c0, c1, c2) \
    { const Fp2 k0 = c0, k1 = c1, k2 = c2; r = k2; fp2_mul(r, r, x); fp2_add(r, r, k1); fp2_mul(r, r, x); fp2_add(r, r, k0); }

// 3-isogeny E'' -> E', output in Jacobian coordinates (no inversion): Z = xd*yd
B200_BIG void iso3_map(G2Jac& out, const Fp2& x, const Fp2& y) {
    Fp2 xn, xd, yn, yd, t, yd2;
    B200_HORNER4(xn, x, B200_FP2_ISO_XNUM0, B200_FP2_ISO_XNUM1, B200_FP2_ISO_XNUM2, B200_FP2_ISO_XNUM3);
    B200_HORNER3(xd, x, B200_FP2_ISO_XDEN0, B200_FP2_ISO_XDEN1, B200_FP2_ISO_XDEN2);
    B200_HORNER4(yn, x, B200_FP2_ISO_YNUM0, B200_FP2_ISO_YNUM1, B200_FP2_ISO_YNUM2, B200_FP2_ISO_YNUM3);
    B200_HORNER4(yd, x, B200_FP2_ISO_YDEN0, B200_FP2_ISO_YDEN1, B200_FP2_ISO_YDEN2, B200_FP2_ISO_YDEN3);
    fp2_mul(out.z, xd, yd);
    fp2_sqr(yd2, yd);
    fp2_mul(t, xn, xd);
    fp2_mul(out.x, t, yd2);          // X = xn * xd * yd^2
    fp2_sqr(t, xd);
    fp2_mul(t, t, xd);               // xd^3
    fp2_mul(t, t, yd2);
    fp2_mul(t, t, yn);
    fp2_mul(out.y, t, y);            // Y = y * yn * xd^3 * yd^2
    if (fp2_is_zero(out.z)) jac_set_inf(out);
}

#if defined(B200_SSWU_FRACTION)
// ---- A/B variant (default off; round-2 experiment): simplified SWU with x kept as a fraction, so the Fp2 inversion
// (one of the three exponentiations of the map) disappears.  RFC 9380 F.2 straight-line shape:
//   x1 = N/D, N = B (tv1 + 1), D = -A tv1 (D = Z A when tv1 = 0);  g(x1) = U/V, U = N^3 + A N D^2 + B D^3, V = D^3.
// Square root of W = U/V without inverting V: with V~ = conj(V), nV = norm(V):  W = W'/nV^2 for W' = U V~ nV, so
// sqrt(W) = sqrt(W')/nV.  Complex method on W' (norm root s' = s_n nV with s_n^2 = +-norm(U V~)), d = (W'_0 + s')/2,
// and ONE exponentiation of q = d nV^2:  r = q^((p-3)/4) = t chi(nV)/nV  with t = d^((p-3)/4).  Up to the irrelevant
// global sign chi(nV) the affine root is (d r, W'_1 r/2) if (d r nV)^2 = d, else (-W'_1 r/2, d r)  [cf. fp2.cuh].
// Output: x as the fraction xn/xd, y affine (so sgn0 can fix its sign).
B200_BIG void sswu_map_frac(Fp2& xn, Fp2& xd, Fp2& y, const Fp2& t) {
    const Fp2 Zc = B200_FP2_SSWU_Z, A = B200_FP2_SSWU_A, B = B200_FP2_SSWU_B;
    Fp2 t2, zt2, tv1, N, D, one = fp2_one();
    fp2_sqr(t2, t);
    fp2_mul(zt2, Zc, t2);
    fp2_sqr(tv1, zt2);
    fp2_add(tv1, tv1, zt2);
    fp2_add(N, tv1, one);
    fp2_mul(N, N, B);
    if (fp2_is_zero(tv1)) fp2_mul(D, Zc, A); else { fp2_mul(D, A, tv1); fp2_neg(D, D); }
    Fp2 N2, D2, D3, U, u1;
    fp2_sqr(N2, N); fp2_sqr(D2, D); fp2_mul(D3, D2, D);
    fp2_mul(U, N2, N);                 // N^3
    fp2_mul(u1, A, N); fp2_mul(u1, u1, D2);
    fp2_add(U, U, u1);
    fp2_mul(u1, B, D3);
    fp2_add(U, U, u1);                 // U;  V = D3
    Fp nV, tt;
    fp_sqr(nV, D3.c0); fp_sqr(tt, D3.c1); fp_add(nV, nV, tt);
    Fp2 Vc = D3, Wn, W;
    fp_neg(Vc.c1, Vc.c1);
    fp2_mul(Wn, U, Vc);                // U conj(V)
    Fp n, s, c;
    fp_sqr(n, Wn.c0); fp_sqr(tt, Wn.c1); fp_add(n, n, tt);
    fp_pow(s, n, B200_EXP_TABLE(exp_sqrt));
    fp_sqr(c, s);
    const bool is_sq = fp_eq(c, n);
    if (!is_sq) {
        const Fp2 z3 = B200_FP2_SSWU_Z3;
        const Fp cs = B200_FP_SSWU_SQRT_NEG_NORM_Z3;
        fp2_mul(Wn, z3, Wn);
        fp_mul(s, s, cs);
    }
    fp_mul(W.c0, Wn.c0, nV); fp_mul(W.c1, Wn.c1, nV);   // W' = (Z^3) U conj(V) nV
    fp_mul(s, s, nV);                                   // s' = sqrt(norm(W'))
    Fp2 yy;
    bool ok = false;
    if (!fp_is_zero(W.c1)) {
        Fp d, q, r, u, chk, h, dr;
        fp_add(d, W.c0, s); fp_half(d, d);
        fp_sqr(q, nV); fp_mul(q, q, d);
        fp_pow(r, q, B200_EXP_TABLE(exp_p_minus_3_div_4));
        fp_mul(dr, d, r);
        fp_mul(u, dr, nV);
        fp_sqr(chk, u);
        fp_mul(h, W.c1, r); fp_half(h, h);
        if (fp_eq(chk, d)) { yy.c0 = dr; yy.c1 = h; } else { fp_neg(yy.c0, h); yy.c1 = dr; }
        // verify in fraction form: yy^2 nV^2 == W'  (yy = sqrt(W')/nV)
        Fp2 sq; Fp nV2;
        fp2_sqr(sq, yy); fp_sqr(nV2, nV);
        fp_mul(sq.c0, sq.c0, nV2); fp_mul(sq.c1, sq.c1, nV2);
        ok = fp2_eq(sq, W);
    }
    if (!ok) {   // real W' (probability ~2^-381) or an inconsistency: the general affine routine
        Fp2 xa, ya;
        sswu_map(xa, ya, t);
        xn = xa; xd = fp2_one(); y = ya;
        return;
    }
    if (is_sq) {
        xn = N;
    } else {
        Fp2 t3;
        fp2_mul(xn, zt2, N);
        fp2_mul(t3, t2, t);
        fp2_mul(yy, yy, t3);
    }
    xd = D;
    if (fp2_sgn0(t) != fp2_sgn0(yy)) fp2_neg(yy, yy);
    y = yy;
}
// 3-isogeny with x = xn/xd: homogeneous Horner forms, Jacobian output Z = xd XD YD
//   x' = XN / (xd XD),  y' = y YN / YD   with XN, YN, YD cubic forms and XD a quadratic form in (xn, xd)
B200_BIG void iso3_map_frac(G2Jac& out, const Fp2& xn, const Fp2& xd, const Fp2& y) {
    Fp2 z2, z3, t, XN, XD, YN, YD;
    fp2_sqr(z2, xd); fp2_mul(z3, z2, xd);
    auto cubic = [&](Fp2& r, const Fp2& k0, const Fp2& k1, const Fp2& k2, const Fp2& k3) {
        Fp2 a;                                  // ((k3 xn + k2 xd) xn + k1 xd^2) xn + k0 xd^3
        fp2_mul(r, k3, xn); fp2_mul(a, k2, xd); fp2_add(r, r, a);
        fp2_mul(r, r, xn); fp2_mul(a, k1, z2); fp2_add(r, r, a);
        fp2_mul(r, r, xn); fp2_mul(a, k0, z3); fp2_add(r, r, a);
    };
    { const Fp2 k0 = B200_FP2_ISO_XNUM0, k1 = B200_FP2_ISO_XNUM1, k2 = B200_FP2_ISO_XNUM2, k3 = B200_FP2_ISO_XNUM3; cubic(XN, k0, k1, k2, k3); }
    { const Fp2 k0 = B200_FP2_ISO_YNUM0, k1 = B200_FP2_ISO_YNUM1, k2 = B200_FP2_ISO_YNUM2, k3 = B200_FP2_ISO_YNUM3; cubic(YN, k0, k1, k2, k3); }
    { const Fp2 k0 = B200_FP2_ISO_YDEN0, k1 = B200_FP2_ISO_YDEN1, k2 = B200_FP2_ISO_YDEN2, k3 = B200_FP2_ISO_YDEN3; cubic(YD, k0, k1, k2, k3); }
    {
        const Fp2 k0 = B200_FP2_ISO_XDEN0, k1 = B200_FP2_ISO_XDEN1, k2 = B200_FP2_ISO_XDEN2;
        Fp2 a;                                  // (k2 xn + k1 xd) xn + k0 xd^2
        fp2_mul(XD, k2, xn); fp2_mul(a, k1, xd); fp2_add(XD, XD, a);
        fp2_mul(XD, XD, xn); fp2_mul(a, k0, z2); fp2_add(XD, XD, a);
    }
    Fp2 zx, yd2;
    fp2_mul(zx, xd, XD);                        // xd XD
    fp2_mul(out.z, zx, YD);
    fp2_sqr(yd2, YD);
    fp2_mul(t, XN, zx);
    fp2_mul(out.x, t, yd2);                     // X = XN (xd XD) YD^2
    fp2_sqr(t, zx); fp2_mul(t, t, zx);          // (xd XD)^3
    fp2_mul(t, t, yd2);
    fp2_mul(t, t, YN);
    fp2_mul(out.y, t, y);                       // Y = y YN (xd XD)^3 YD^2
    if (fp2_is_zero(out.z)) jac_set_inf(out);
}
#define B200_SSWU_ISO(out, u) { Fp2 xn_, xd_, y_; sswu_map_frac(xn_, xd_, y_, u); iso3_map_frac(out, xn_, xd_, y_); }
#else
#define B200_SSWU_ISO(out, u) { Fp2 x_, y_; sswu_map(x_, y_, u); iso3_map(out, x_, y_); }
#endif

// first half, for j in {0, 1}: u_j = hash_to_field(msg)[j], Q_j = iso3(sswu(u_j)) in Jacobian coordinates
B200_BIG void hash_to_g2_map(G2Jac& out, const uint8_t* msg, size_t len, int j) {
    Fp2 u0, u1;
    hash_to_field_fp2(u0, u1, msg, len);
    B200_SSWU_ISO(out, j ? u1 : u0);
}
// second half: Q_0 + Q_1, clear the cofactor, normalise
B200_BIG void hash_to_g2_finish(G2Aff& out, const G2Jac& q0, const G2Jac& q1) {
    G2Jac s, c;
    jac_add(s, q0, q1);
    g2_clear_cofactor(c, s);
    jac_to_aff(out, c);
}

// full hash_to_curve -> affine G2 point
B200_BIG void hash_to_g2(G2Aff& out, const uint8_t* msg, size_t len) {
    Fp2 u0, u1;
    hash_to_field_fp2(u0, u1, msg, len);
    G2Jac q0, q1;
    B200_SSWU_ISO(q0, u0);
    B200_SSWU_ISO(q1, u1);
    jac_add(q0, q0, q1);
    g2_clear_cofactor(q1, q0);
    jac_to_aff(out, q1);
}

}  // namespace b200
