// G1 / G2 of BLS12-381: ZCash (de)compression with blst's error taxonomy, subgroup membership, psi, cofactor
// clearing.  Semantics restated from the reference wrapper (the checks blst runs for
// ethereum-consensus/src/crypto/bls.rs:279-285 `key_validate` and :330-336 `from_bytes`):
//   BAD_ENCODING(1): compression bit clear, infinity flag with payload, coordinate >= p
//   POINT_NOT_ON_CURVE(2), POINT_NOT_IN_GROUP(3), PK_IS_INFINITY(6)
#pragma once
#include "curve.cuh"
#include "fpl.cuh"

namespace b200 {

enum : int32_t {
    BLS_SUCCESS = 0, BLS_BAD_ENCODING = 1, BLS_POINT_NOT_ON_CURVE = 2, BLS_POINT_NOT_IN_GROUP = 3,
    BLS_AGGR_TYPE_MISMATCH = 4, BLS_VERIFY_FAIL = 5, BLS_PK_IS_INFINITY = 6, BLS_BAD_SCALAR = 7
};

typedef Aff<Fp> G1Aff;
typedef Jac<Fp> G1Jac;
typedef Aff<Fp2> G2Aff;
typedef Jac<Fp2> G2Jac;

// 48 big-endian bytes with the 3 flag bits cleared -> Montgomery Fp; false if the integer is >= p
B200_HD bool fp_from_be48_masked(Fp& r, const uint8_t* b, bool mask_flags) {
    Fp raw;
    fp_from_be_bytes_raw(raw, b);
    if (mask_flags) raw.l[11] &= 0x1fffffffu;
    const Fp p = fp_p();
    if (fp_geq_raw(raw, p)) return false;
    fp_to_mont(r, raw);
    return true;
}
B200_HD bool bytes_all_zero(const uint8_t* b, int n) {
    uint32_t acc = 0;
    for (int i = 0; i < n; i++) acc |= b[i];
    return acc == 0;
}

// -> BLS_* code; out.inf = 1 for the (valid) infinity encoding
B200_HD int32_t g1_uncompress(G1Aff& out, const uint8_t b[48]) {
    const uint8_t f = b[0];
    out.inf = 0;
    if (!(f & 0x80)) return BLS_BAD_ENCODING;
    if (f & 0x40) {
        if ((f & 0x3f) == 0 && bytes_all_zero(b + 1, 47)) { out.inf = 1; out.x = fp_zero(); out.y = fp_zero(); return BLS_SUCCESS; }
        return BLS_BAD_ENCODING;
    }
    Fp x, y2, y;
    if (!fp_from_be48_masked(x, b, true)) return BLS_BAD_ENCODING;
    fp_sqr(y2, x);
    fp_mul(y2, y2, x);
    const Fp four = B200_FP_B_G1;
    fp_add(y2, y2, four);
    if (!fp_sqrt(y, y2)) return BLS_POINT_NOT_ON_CURVE;
    if (fp_is_lex_largest(y) != ((f & 0x20) != 0)) fp_neg(y, y);
    out.x = x; out.y = y;
    return BLS_SUCCESS;
}

// phi(P) == -[z^2]P  (Scott 2021; beta chosen by tools/gen_bls_consts.py so that this holds on G1)
B200_HD bool g1_in_subgroup(const G1Aff& p) {
    if (p.inf) return true;
    G1Jac t, t2;
    jac_mul_u64(t, p.x, p.y, B200_Z_ABS);
    jac_mul_u64_jac(t2, t, B200_Z_ABS);
    const Fp beta = B200_FP_BETA;
    Fp bx, ny;
    fp_mul(bx, p.x, beta);
    fp_neg(ny, p.y);
    return jac_eq_aff(t2, bx, ny);
}

// ---- the same two steps on lazily reduced field elements (fpl.cuh): what the per-key kernel runs ----------------
// decompression: identical checks and codes as g1_uncompress; y = (x^3 + 4)^((p+1)/4) with no reduction inside the chain
B200_HD int32_t g1_uncompress_lazy(G1Aff& out, const uint8_t b[48]) {
    const uint8_t f = b[0];
    out.inf = 0;
    if (!(f & 0x80)) return BLS_BAD_ENCODING;
    if (f & 0x40) {
        if ((f & 0x3f) == 0 && bytes_all_zero(b + 1, 47)) { out.inf = 1; out.x = fp_zero(); out.y = fp_zero(); return BLS_SUCCESS; }
        return BLS_BAD_ENCODING;
    }
    Fp x;
    if (!fp_from_be48_masked(x, b, true)) return BLS_BAD_ENCODING;
    FpL xl = fpl_from_fp(x), y2, yl, c;
    f_sqr(y2, xl);
    f_mul(y2, y2, xl);
    f_add(y2, y2, curve_b<FpL>());
    fpl_pow(yl, y2, B200_EXP_TABLE(exp_sqrt));
    f_sqr(c, yl);
    if (!f_eq(c, y2)) return BLS_POINT_NOT_ON_CURVE;
    Fp y = fpl_canon(yl);
    if (fp_is_lex_largest(y) != ((f & 0x20) != 0)) fp_neg(y, y);
    out.x = x; out.y = y;
    return BLS_SUCCESS;
}
// phi(P) == -[z^2]P on FpL (the templated Jacobian formulas of curve.cuh, every intermediate in [0, 2p))
B200_HD bool g1_in_subgroup_lazy(const G1Aff& p) {
    if (p.inf) return true;
    const FpL px = fpl_from_fp(p.x), py = fpl_from_fp(p.y);
    Jac<FpL> t, t2;
    jac_mul_u64(t, px, py, B200_Z_ABS);
    jac_mul_u64_jac(t2, t, B200_Z_ABS);
    const Fp beta = B200_FP_BETA;
    FpL bx, ny;
    f_mul(bx, px, fpl_from_fp(beta));
    f_neg(ny, py);
    return jac_eq_aff(t2, bx, ny);
}

// blst `PublicKey::key_validate`.  -DB200_G1_CANONICAL_FP selects the fully reduced arithmetic (round 1's path).
B200_HD int32_t g1_key_validate(G1Aff& out, const uint8_t b[48]) {
#if defined(B200_G1_CANONICAL_FP)
    int32_t rc = g1_uncompress(out, b);
    if (rc) return rc;
    if (out.inf) return BLS_PK_IS_INFINITY;
    if (!g1_in_subgroup(out)) return BLS_POINT_NOT_IN_GROUP;
#else
    int32_t rc = g1_uncompress_lazy(out, b);
    if (rc) return rc;
    if (out.inf) return BLS_PK_IS_INFINITY;
    if (!g1_in_subgroup_lazy(out)) return BLS_POINT_NOT_IN_GROUP;
#endif
    return BLS_SUCCESS;
}

B200_HD void g1_compress(uint8_t out[48], const G1Aff& a) {
    if (a.inf) { for (int i = 0; i < 48; i++) out[i] = 0; out[0] = 0xc0; return; }
    Fp raw;
    fp_from_mont(raw, a.x);
    fp_to_be_bytes_raw(out, raw);
    out[0] |= 0x80;
    if (fp_is_lex_largest(a.y)) out[0] |= 0x20;
}

B200_BIG int32_t g2_uncompress(G2Aff& out, const uint8_t b[96]) {
    const uint8_t f = b[0];
    out.inf = 0;
    if (!(f & 0x80)) return BLS_BAD_ENCODING;
    if (f & 0x40) {
        if ((f & 0x3f) == 0 && bytes_all_zero(b + 1, 95)) { out.inf = 1; out.x = fp2_zero(); out.y = fp2_zero(); return BLS_SUCCESS; }
        return BLS_BAD_ENCODING;
    }
    Fp2 x, y2, y;
    if (!fp_from_be48_masked(x.c1, b, true)) return BLS_BAD_ENCODING;
    if (!fp_from_be48_masked(x.c0, b + 48, false)) return BLS_BAD_ENCODING;
    fp2_sqr(y2, x);
    fp2_mul(y2, y2, x);
    const Fp2 bb = B200_FP2_B_G2;
    fp2_add(y2, y2, bb);
    if (!fp2_sqrt(y, y2)) return BLS_POINT_NOT_ON_CURVE;
    if (fp2_is_lex_largest(y) != ((f & 0x20) != 0)) fp2_neg(y, y);
    out.x = x; out.y = y;
    return BLS_SUCCESS;
}

B200_HD void g2_compress(uint8_t out[96], const G2Aff& a) {
    if (a.inf) { for (int i = 0; i < 96; i++) out[i] = 0; out[0] = 0xc0; return; }
    Fp raw;
    fp_from_mont(raw, a.x.c1);
    fp_to_be_bytes_raw(out, raw);
    fp_from_mont(raw, a.x.c0);
    fp_to_be_bytes_raw(out + 48, raw);
    out[0] |= 0x80;
    if (fp2_is_lex_largest(a.y)) out[0] |= 0x20;
}

// psi = twist^-1 o frobenius o twist on Jacobian coordinates: (conj(X)*cx, conj(Y)*cy, conj(Z))
B200_BIG void g2_psi(G2Jac& r, const G2Jac& p) {
    const Fp2 cx = B200_FP2_PSI_X, cy = B200_FP2_PSI_Y;
    Fp2 t;
    fp2_conj(t, p.x); fp2_mul(r.x, t, cx);
    fp2_conj(t, p.y); fp2_mul(r.y, t, cy);
    fp2_conj(r.z, p.z);
}
// psi^2: (X * c, -Y, Z) with c in Fp
B200_HD void g2_psi2(G2Jac& r, const G2Jac& p) {
    const Fp c = B200_FP_PSI2_X;
    fp2_mul_fp(r.x, p.x, c);
    fp2_neg(r.y, p.y);
    r.z = p.z;
}

// psi(Q) == [z]Q, z = -|z|  (Scott 2021)
B200_BIG bool g2_in_subgroup(const G2Aff& q) {
    if (q.inf) return true;
    G2Jac t, qj, ps;
    jac_mul_u64(t, q.x, q.y, B200_Z_ABS);  // [|z|]Q
    jac_from_aff(qj, q);
    g2_psi(ps, qj);                         // Z = 1 stays 1
    Fp2 ny;
    fp2_neg(ny, ps.y);
    return jac_eq_aff(t, ps.x, ny);         // [|z|]Q == -psi(Q)
}

// h_eff * P via Budroni-Pintore (RFC 9380 G.3); equality with the scalar h_eff is asserted in the generator
B200_BIG void g2_clear_cofactor(G2Jac& r, const G2Jac& p) {
    G2Jac t1, t2, t3, np;
    jac_mul_u64_jac(t1, p, B200_Z_ABS);
    jac_neg(t1, t1);                 // t1 = [z]P
    g2_psi(t2, p);                   // t2 = psi(P)
    jac_double(t3, p);
    g2_psi2(t3, t3);                 // t3 = psi^2(2P)
    G2Jac nt2;
    jac_neg(nt2, t2);
    jac_add(t3, t3, nt2);            // t3 -= t2
    jac_add(t2, t1, t2);             // t2 = t1 + t2
    jac_mul_u64_jac(t2, t2, B200_Z_ABS);
    jac_neg(t2, t2);                 // t2 = [z]t2
    jac_add(t3, t3, t2);
    jac_neg(t1, t1);
    jac_add(t3, t3, t1);             // t3 -= t1
    jac_neg(np, p);
    jac_add(r, t3, np);              // Q = t3 - P
}

}  // namespace b200
