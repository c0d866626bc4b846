// TEST INFRASTRUCTURE: compiles the product's __host__ __device__ BLS math (ethereum_consensus_b200/csrc/*.cuh)
// for the CPU so that every layer above the PTX-free Fp arithmetic can be diffed against the big-int oracle
// without a GPU.  Nothing here is linked into libb200_consensus.so; the product path launches kernels only.
#include <cstdint>
#include <cstring>

#include "../../ethereum_consensus_b200/csrc/h2c.cuh"
#include "../../ethereum_consensus_b200/csrc/pairing.cuh"

using namespace b200;
#define HM __attribute__((visibility("default")))

static void fp_in(Fp& r, const uint8_t* be48) { Fp raw; fp_from_be_bytes_raw(raw, be48); fp_to_mont(r, raw); }
static void fp_out(uint8_t* be48, const Fp& a) { Fp raw; fp_from_mont(raw, a); fp_to_be_bytes_raw(be48, raw); }
static void fp2_in(Fp2& r, const uint8_t* b) { fp_in(r.c0, b); fp_in(r.c1, b + 48); }
static void fp2_out(uint8_t* b, const Fp2& a) { fp_out(b, a.c0); fp_out(b + 48, a.c1); }
static void g1_in(G1Aff& p, const uint8_t* b, int inf) { p.inf = inf; fp_in(p.x, b); fp_in(p.y, b + 48); }
static void g2_in(G2Aff& p, const uint8_t* b, int inf) { p.inf = inf; fp2_in(p.x, b); fp2_in(p.y, b + 96); }
static void g2_out(uint8_t* b, const G2Aff& p) { fp2_out(b, p.x); fp2_out(b + 96, p.y); }

extern "C" {

// op: 0 add, 1 sub, 2 mul, 3 inv(a), 4 sqrt(a) (returns ok), 5 neg(a)
HM int hm_fp_op(int op, const uint8_t* a48, const uint8_t* b48, uint8_t* out48) {
    Fp a, b, r;
    fp_in(a, a48); fp_in(b, b48);
    int ok = 1;
    switch (op) {
    case 0: fp_add(r, a, b); break;
    case 1: fp_sub(r, a, b); break;
    case 2: fp_mul(r, a, b); break;
    case 3: fp_inv(r, a); break;
    case 4: ok = fp_sqrt(r, a); break;
    default: fp_neg(r, a); break;
    }
    fp_out(out48, r);
    return ok;
}
// op: 0 mul, 1 sqr(a), 2 inv(a), 3 sqrt(a) (returns ok), 4 sgn0(a) (returned), 5 lex_largest(a) (returned)
HM int hm_fp2_op(int op, const uint8_t* a96, const uint8_t* b96, uint8_t* out96) {
    Fp2 a, b, r = fp2_zero();
    fp2_in(a, a96); fp2_in(b, b96);
    int ret = 1;
    switch (op) {
    case 0: fp2_mul(r, a, b); break;
    case 1: fp2_sqr(r, a); break;
    case 2: fp2_inv(r, a); break;
    case 3: ret = fp2_sqrt(r, a); break;
    case 4: ret = int(fp2_sgn0(a)); break;
    default: ret = fp2_is_lex_largest(a); break;
    }
    fp2_out(out96, r);
    return ret;
}
HM int hm_g1_key_validate(const uint8_t* in48, uint8_t* out_xy96, uint8_t* recompressed48) {
    G1Aff p;
    int rc = g1_key_validate(p, in48);
    if (rc == 0) { fp_out(out_xy96, p.x); fp_out(out_xy96 + 48, p.y); g1_compress(recompressed48, p); }
    return rc;
}
HM int hm_g1_uncompress(const uint8_t* in48, uint8_t* out_xy96, int* inf) {
    G1Aff p;
    int rc = g1_uncompress(p, in48);
    if (rc == 0) { fp_out(out_xy96, p.x); fp_out(out_xy96 + 48, p.y); *inf = int(p.inf); }
    return rc;
}
HM int hm_g2_uncompress(const uint8_t* in96, uint8_t* out192, int* inf, int* in_group, uint8_t* recompressed96) {
    G2Aff p;
    int rc = g2_uncompress(p, in96);
    if (rc == 0) { g2_out(out192, p); *inf = int(p.inf); *in_group = g2_in_subgroup(p); g2_compress(recompressed96, p); }
    return rc;
}
HM void hm_hash_to_field(const uint8_t* msg, size_t len, uint8_t* out192) {
    Fp2 u0, u1;
    hash_to_field_fp2(u0, u1, msg, len);
    fp2_out(out192, u0); fp2_out(out192 + 96, u1);
}
HM void hm_sswu_iso(const uint8_t* t96, uint8_t* out192, int* inf) {
    Fp2 t, x, y;
    fp2_in(t, t96);
    sswu_map(x, y, t);
    G2Jac j;
    iso3_map(j, x, y);
    G2Aff a;
    jac_to_aff(a, j);
    g2_out(out192, a);
    *inf = int(a.inf);
}
HM void hm_hash_to_g2(const uint8_t* msg, size_t len, uint8_t* out192, int* inf) {
    G2Aff h;
    hash_to_g2(h, msg, len);
    g2_out(out192, h);
    *inf = int(h.inf);
}
// prod e(P_i, Q_i) == 1 ?   g1: n x 96 bytes (x,y), g2: n x 192 bytes, inf flags per point (bit0 g1, bit1 g2)
HM int hm_pairing_check(int n, const uint8_t* g1, const uint8_t* g2, const uint8_t* inf) {
    Fp12 acc = fp12_one(), f;
    for (int i = 0; i < n; i++) {
        G1Aff p; G2Aff q;
        g1_in(p, g1 + 96 * i, inf[i] & 1);
        g2_in(q, g2 + 192 * i, (inf[i] >> 1) & 1);
        miller_loop(f, p, q);
        fp12_mul(acc, acc, f);
    }
    return final_exp_is_one(acc);
}
// fp12 self-consistency: returns bitmask of passed checks (inverse, frobenius^12... ) on a = miller_loop(g1, g2 gens)
HM int hm_fp12_selftest(void) {
    G1Aff p; p.inf = 0; { const Fp x = B200_FP_G1_X, y = B200_FP_G1_Y; p.x = x; p.y = y; }
    G2Aff q;
    uint8_t msg[3] = {1, 2, 3};
    hash_to_g2(q, msg, 3);
    Fp12 a, b, c;
    miller_loop(a, p, q);
    int ok = 0;
    fp12_inv(b, a); fp12_mul(c, a, b); if (fp12_is_one(c)) ok |= 1;
    fp12_sqr(b, a); fp12_mul(c, a, a);
    bool same = fp2_eq(b.c0.c0, c.c0.c0) && fp2_eq(b.c1.c2, c.c1.c2) && fp2_eq(b.c0.c1, c.c0.c1) && fp2_eq(b.c1.c0, c.c1.c0) &&
                fp2_eq(b.c0.c2, c.c0.c2) && fp2_eq(b.c1.c1, c.c1.c1);
    if (same) ok |= 2;
    // frobenius^1 applied 12 times is the identity; frobenius<2> == frobenius<1> twice; <3> == thrice
    b = a;
    for (int i = 0; i < 12; i++) { fp12_frobenius<1>(c, b); b = c; }
    fp12_inv(c, a); fp12_mul(c, c, b); if (fp12_is_one(c)) ok |= 4;
    fp12_frobenius<1>(b, a); fp12_frobenius<1>(c, b); fp12_frobenius<2>(b, a);
    { Fp12 d; fp12_inv(d, c); fp12_mul(d, d, b); if (fp12_is_one(d)) ok |= 8; }
    fp12_frobenius<1>(b, c); fp12_frobenius<3>(c, a);
    { Fp12 d; fp12_inv(d, c); fp12_mul(d, d, b); if (fp12_is_one(d)) ok |= 16; }
    // cyclotomic squaring == generic squaring on the cyclotomic subgroup (after the easy part)
    { Fp12 e, t0, t1, s1, s2;
      fp12_inv(t0, a); fp12_conj(t1, a); fp12_mul(t0, t1, t0); fp12_frobenius<2>(t1, t0); fp12_mul(e, t1, t0);
      fp12_sqr(s1, e); fp12_cyclotomic_sqr(s2, e);
      fp12_inv(t0, s1); fp12_mul(t0, t0, s2); if (fp12_is_one(t0)) ok |= 32; }
    return ok;
}

// the reference wrapper's fast_aggregate_verify (crypto/bls.rs:114-132), sequentially, from the HD pieces
HM int hm_fast_aggregate_verify(const uint8_t* pks, size_t k, const uint8_t* msg, size_t len, const uint8_t* sig) {
    G1Jac acc;
    jac_set_inf(acc);
    for (size_t i = 0; i < k; i++) {
        G1Aff p;
        int rc = g1_key_validate(p, pks + 48 * i);
        if (rc) return rc;
        jac_add_mixed(acc, acc, p.x, p.y);
    }
    G2Aff s;
    int rc = g2_uncompress(s, sig);
    if (rc) return rc;
    if (k == 0) return BLS_VERIFY_FAIL;
    if (!g2_in_subgroup(s)) return BLS_VERIFY_FAIL;
    G1Aff agg;
    jac_to_aff(agg, acc);
    if (agg.inf) return BLS_VERIFY_FAIL;
    G2Aff h;
    hash_to_g2(h, msg, len);
    G1Aff ng; ng.inf = 0; { const Fp x = B200_FP_G1_X, y = B200_FP_G1_NEG_Y; ng.x = x; ng.y = y; }
    Fp12 f1, f2;
    miller_loop(f1, agg, h);
    miller_loop(f2, ng, s);
    fp12_mul(f1, f1, f2);
    return final_exp_is_one(f1) ? BLS_SUCCESS : BLS_VERIFY_FAIL;
}

}  // extern "C"

// the C emulation of the generated PTX instruction list vs the portable product (raw Montgomery-domain limbs)
extern "C" HM int hm_fp_mul_emul_matches(const uint32_t* a, const uint32_t* b) {
    Fp x, y, want, got;
    for (int i = 0; i < 12; i++) { x.l[i] = a[i]; y.l[i] = b[i]; }
    fp_mul_portable(want, x, y);
    fp_mul_emul_core(got.l, x.l, y.l);
    fp_reduce_once(got);
    if (!fp_eq(want, got)) return 0;
    fp_mul_portable(want, x, x);
    fp_sqr_emul_core(got.l, x.l);
    fp_reduce_once(got);
    return fp_eq(want, got);
}

// raw outputs of the emulated PTX product (op 0) / square (op 1) WITHOUT the final conditional subtraction: what the lazily
// reduced per-key path (fpl.cuh) consumes; operands may be anywhere in [0, 2p)
extern "C" HM void hm_fp_emul_raw(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) {
    if (op == 0) fp_mul_emul_core(out, a, b);
    else fp_sqr_emul_core(out, a);
}
// FpL add / sub / neg on raw limbs (operands and results in [0, 2p))
extern "C" HM void hm_fpl_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) {
    FpL x, y, r;
    for (int i = 0; i < 12; i++) { x.v.l[i] = a[i]; y.v.l[i] = b[i]; }
    if (op == 0) f_add(r, x, y); else if (op == 1) f_sub(r, x, y); else f_neg(r, x);
    for (int i = 0; i < 12; i++) out[i] = r.v.l[i];
}

// ---- Kaliski inverse (fp.cuh, the device's fp_inv) against the Fermat exponentiation: out = [kaliski | fermat], 12 limbs each
extern "C" HM void hm_fp_inv_both(const uint32_t* a, uint32_t* out) {
    Fp x, k, f;
    for (int i = 0; i < 12; i++) x.l[i] = a[i];
    fp_inv_kaliski(k, x);
    fp_inv_fermat(f, x);
    for (int i = 0; i < 12; i++) { out[i] = k.l[i]; out[12 + i] = f.l[i]; }
}

// ---- Fp2 VM (lane-parallel pairing programs) on the host: scheduled program == direct evaluation, bit for bit
#include "../../ethereum_consensus_b200/csrc/pairing_vm.cuh"
static void vm_consts(Fp2* c) { for (int i = 0; i < kVmConsts; i++) vm_const_to_mont(c[i], h_vm_consts[i]); }
template <int TEAM>
static int vm_matches_direct(const uint8_t* g1a, const uint8_t* g2a, const uint8_t* g1b, const uint8_t* g2b) {
    typedef VmProg<TEAM> P;
    Fp2 consts[kVmConsts];
    vm_consts(consts);
    G1Aff p[2]; G2Aff q[2];
    g1_in(p[0], g1a, 0); g2_in(q[0], g2a, 0); g1_in(p[1], g1b, 0); g2_in(q[1], g2b, 0);
    Fp12 direct[2], viavm[2];
    int ok = 1;
    for (int k = 0; k < 2; k++) {
        miller_loop(direct[k], p[k], q[k]);
        static Fp2 rf[256];
        rf[0].c0 = p[k].x; rf[0].c1 = fp_zero(); rf[1].c0 = p[k].y; rf[1].c1 = fp_zero();
        rf[2].c0 = fp_one(); rf[2].c1 = fp_zero(); rf[3] = q[k].x; rf[4] = q[k].y;   // affine P: (x, y, 1)
        vm_run_host<TEAM>(P::miller_code(), P::miller_rounds, consts, rf);
        Fp12& f = viavm[k];
        f.c0.c0 = rf[P::miller_out[0]]; f.c1.c0 = rf[P::miller_out[1]]; f.c0.c1 = rf[P::miller_out[2]];
        f.c1.c1 = rf[P::miller_out[3]]; f.c0.c2 = rf[P::miller_out[4]]; f.c1.c2 = rf[P::miller_out[5]];
        const Fp2* d = &direct[k].c0.c0; const Fp2* v = &viavm[k].c0.c0;
        for (int i = 0; i < 6; i++) if (!fp2_eq(d[i], v[i])) ok = 0;
    }
    // final exponentiation program: verdict and value
    Fp12 prod;
    fp12_mul(prod, direct[0], direct[1]);
    const int want_one = final_exp_is_one(prod);
    static Fp2 rf[256];
    const Fp12* fs[2] = {&viavm[0], &viavm[1]};
    for (int k = 0; k < 2; k++) {
        rf[6 * k + 0] = fs[k]->c0.c0; rf[6 * k + 1] = fs[k]->c1.c0; rf[6 * k + 2] = fs[k]->c0.c1;
        rf[6 * k + 3] = fs[k]->c1.c1; rf[6 * k + 4] = fs[k]->c0.c2; rf[6 * k + 5] = fs[k]->c1.c2;
    }
    vm_run_host<TEAM>(P::final_code(), P::final_rounds, consts, rf);
    int is_one = fp2_eq(rf[P::final_out[0]], fp2_one());
    for (int i = 1; i < 6; i++) is_one = is_one && fp2_is_zero(rf[P::final_out[i]]);
    if (is_one != want_one) ok = 0;
    return ok | (is_one << 1);
}
// both program pairs (teams of 8 and of 16 lanes) must agree with the direct evaluation: 3 = match + pairing product is one
extern "C" HM int hm_vm_matches_direct(const uint8_t* g1a, const uint8_t* g2a, const uint8_t* g1b, const uint8_t* g2b) {
    const int r8 = vm_matches_direct<8>(g1a, g2a, g1b, g2b), r16 = vm_matches_direct<16>(g1a, g2a, g1b, g2b);
    return r8 == r16 ? r8 : 0;
}

// ---- b200_pairing_eval's operations on the host build of the same headers, on the same 145-word records (the folds
// excepted): the one-thread ops, and the scheduled VM programs through vm_run_host with G1Pre inputs of any Z
template <int TEAM>
static void hm_vm_miller(Fp12& f, const Fp* pre, const Fp2* q) {
    typedef VmProg<TEAM> P;
    Fp2 consts[kVmConsts];
    vm_consts(consts);
    static Fp2 rf[256];
    for (int k = 0; k < 3; k++) { rf[k].c0 = pre[k]; rf[k].c1 = fp_zero(); }
    rf[3] = q[0]; rf[4] = q[1];
    vm_run_host<TEAM>(P::miller_code(), P::miller_rounds, consts, rf);
    Fp2* d = &f.c0.c0;
    const int tower_pos[6] = {0, 3, 1, 4, 2, 5};
    for (int k = 0; k < 6; k++) d[tower_pos[k]] = rf[P::miller_out[k]];
}
template <int TEAM>
static uint32_t hm_vm_final(Fp12& f, const Fp12& f0, const Fp12& f1) {
    typedef VmProg<TEAM> P;
    Fp2 consts[kVmConsts];
    vm_consts(consts);
    static Fp2 rf[256];
    const int tower_pos[6] = {0, 3, 1, 4, 2, 5};
    for (int k = 0; k < 6; k++) { rf[k] = (&f0.c0.c0)[tower_pos[k]]; rf[6 + k] = (&f1.c0.c0)[tower_pos[k]]; }
    vm_run_host<TEAM>(P::final_code(), P::final_rounds, consts, rf);
    Fp2* d = &f.c0.c0;
    for (int k = 0; k < 6; k++) d[tower_pos[k]] = rf[P::final_out[k]];
    return fp12_is_one(f) ? 1u : 0u;
}
extern "C" HM void hm_pairing_eval(int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out) {
    const size_t W = 145;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t* pa = a + i * W;
        const uint32_t* pb = b + i * W;
        Fp12 x, y, r = fp12_one();
        memcpy(&x, pa, sizeof(Fp12));
        memcpy(&y, pb, sizeof(Fp12));
        uint32_t flag = 0;
        switch (op) {
        case 0: fp6_mul(r.c0, x.c0, y.c0); r.c1 = x.c1; break;
        case 1: fp6_inv(r.c0, x.c0); r.c1 = x.c1; break;
        case 2: fp12_mul(r, x, y); break;
        case 3: fp12_sqr(r, x); break;
        case 4: fp12_inv(r, x); break;
        case 5: fp12_mul_by_line(r, x, y.c0.c0, y.c0.c1, y.c0.c2); break;
        case 6: fp12_frobenius<1>(r, x); break;
        case 7: fp12_frobenius<2>(r, x); break;
        case 8: fp12_cyclotomic_sqr(r, x); break;
        case 9: fp12_pow_z(r, x); break;
        case 10: case 11: {
            G2Jac t; t.x = x.c0.c0; t.y = x.c0.c1; t.z = x.c0.c2;
            G2Aff q; q.x = y.c0.c0; q.y = y.c0.c1; q.inf = 0;
            if (op == 10) miller_double_step(t, r.c1.c0, r.c1.c1, r.c1.c2, y.c0.c2.c0, y.c0.c2.c1);
            else miller_add_step(t, r.c1.c0, r.c1.c1, r.c1.c2, q, y.c0.c2.c0, y.c0.c2.c1);
            r.c0.c0 = t.x; r.c0.c1 = t.y; r.c0.c2 = t.z;
            break;
        }
        case 12: {
            G1Aff p; p.x = x.c0.c0.c0; p.y = x.c0.c0.c1; p.inf = pa[144];
            G2Aff q; q.x = y.c0.c0; q.y = y.c0.c1; q.inf = pb[144];
            miller_loop(r, p, q);
            break;
        }
        case 13: final_exp(r, x); flag = fp12_is_one(r) ? 1u : 0u; break;
        case 32: case 33:   // the kernels bypass the program for a point at infinity: the pair contributes one
            if (!pa[144] && !pb[144]) {
                if (op == 32) hm_vm_miller<8>(r, &x.c0.c0.c0, &y.c0.c0); else hm_vm_miller<16>(r, &x.c0.c0.c0, &y.c0.c0);
            }
            break;
        case 34: flag = hm_vm_final<8>(r, x, y); break;
        case 35: flag = hm_vm_final<16>(r, x, y); break;
        default: break;
        }
        memcpy(out + i * W, &r, sizeof(Fp12));
        out[i * W + 144] = flag;
    }
}
