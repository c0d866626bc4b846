/*
 * BLS12-381 signature oracle in plain C (6 x 64-bit limbs, unsigned __int128 Montgomery).  TEST INFRASTRUCTURE:
 * only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference, workload generation) may
 * load this.  The product path never does.
 *
 * What it restates: the byte-level behaviour of ethereum-consensus/src/crypto/bls.rs
 *   verify_signature :64-77, aggregate :79-93, aggregate_verify :95-112, fast_aggregate_verify :114-132,
 *   eth_aggregate_public_keys :135-148, eth_fast_aggregate_verify :150-160, key_validate :279-285,
 *   Signature::from_bytes :330-336, SecretKey::{public_key,sign} :212-220,
 * whose arithmetic the reference takes from the un-vendored crate blst 0.3.11 (Cargo.toml:21).
 * Algorithms are the published ones (IETF BLS signatures with the DST at crypto/bls.rs:22, RFC 9380
 * hash_to_curve, ZCash serialization, optimal-ate pairing).  Every derived constant (Frobenius coefficients, psi,
 * the G1 endomorphism) is computed at start-up from first principles; only the RFC 9380 isogeny coefficients
 * and the curve/generator definitions are literals.
 *
 * Pinned by tests/test_oracle_bls.py: reference KATs B-1 (bin/ec/validator/keystores.rs:239-249) and B-2
 * (crypto/bls.rs:530-544), and diffed against the independent big-int oracle (oracle/bls_oracle.py).
 * It is also the timed CPU baseline ("port", not blst): expect blst's assembly to be ~2x faster per core.
 */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>

#define ORC_EXPORT __attribute__((visibility("default")))
typedef unsigned __int128 u128;

void orc_sha256(const uint8_t *data, size_t len, uint8_t out[32]); /* ssz_oracle.c */

enum { OK = 0, BAD_ENCODING = 1, NOT_ON_CURVE = 2, NOT_IN_GROUP = 3, AGGR_TYPE_MISMATCH = 4, VERIFY_FAIL = 5,
       PK_IS_INFINITY = 6, BAD_SCALAR = 7, EMPTY_AGGREGATE = 16 };

/* ================================================================================================ Fp */
typedef struct { uint64_t l[6]; } fp;
static const fp P = {{0xb9feffffffffaaabull, 0x1eabfffeb153ffffull, 0x6730d2a0f6b0f624ull, 0x64774b84f38512bfull,
                      0x4b1ba7b6434bacd7ull, 0x1a0111ea397fe69aull}};
static const uint64_t N0 = 0x89f3fffcfffcfffdull; /* -p^-1 mod 2^64 */
static fp R1, R2;                                  /* 2^384 mod p, 2^768 mod p (computed at init) */
/* instrumented Fp-product counter (SURVEY.md §8d): enabled only between reset() and count(), single-threaded use */
static uint64_t g_fp_mul_count, g_fp_sqr_count;
static int g_count_on;
ORC_EXPORT uint64_t orc_fp_mul_count(void) { g_count_on = 0; return g_fp_mul_count; }
ORC_EXPORT uint64_t orc_fp_sqr_count(void) { return g_fp_sqr_count; }   /* how many of those products were squarings */
ORC_EXPORT void orc_fp_mul_count_reset(void) { g_fp_mul_count = 0; g_fp_sqr_count = 0; g_count_on = 1; }

static int fp_is_zero(const fp *a) { uint64_t x = 0; for (int i = 0; i < 6; i++) x |= a->l[i]; return x == 0; }
static int fp_eq(const fp *a, const fp *b) { uint64_t x = 0; for (int i = 0; i < 6; i++) x |= a->l[i] ^ b->l[i]; return x == 0; }
static uint64_t raw_sub(fp *r, const fp *a, const fp *b) {
    u128 br = 0;
    for (int i = 0; i < 6; i++) { u128 d = (u128)a->l[i] - b->l[i] - (uint64_t)br; r->l[i] = (uint64_t)d; br = (d >> 64) & 1; }
    return (uint64_t)br;
}
static uint64_t raw_add(fp *r, const fp *a, const fp *b) {
    u128 c = 0;
    for (int i = 0; i < 6; i++) { c += (u128)a->l[i] + b->l[i]; r->l[i] = (uint64_t)c; c >>= 64; }
    return (uint64_t)c;
}
static int raw_geq(const fp *a, const fp *b) { fp t; return raw_sub(&t, a, b) == 0; }
static void fp_add(fp *r, const fp *a, const fp *b) { fp t; raw_add(r, a, b); if (!raw_sub(&t, r, &P)) *r = t; }
static void fp_sub(fp *r, const fp *a, const fp *b) { fp t; if (raw_sub(&t, a, b)) raw_add(&t, &t, &P); *r = t; }
static void fp_neg(fp *r, const fp *a) { if (fp_is_zero(a)) *r = *a; else raw_sub(r, &P, a); }
static void fp_mul(fp *r, const fp *a, const fp *b) {
    uint64_t t[8] = {0};
    if (g_count_on) g_fp_mul_count++;
    for (int i = 0; i < 6; i++) {
        u128 c = 0;
        for (int j = 0; j < 6; j++) { c += (u128)a->l[j] * b->l[i] + t[j]; t[j] = (uint64_t)c; c >>= 64; }
        c += t[6]; t[6] = (uint64_t)c; t[7] = (uint64_t)(c >> 64);
        uint64_t m = t[0] * N0;
        c = (u128)m * P.l[0] + t[0]; c >>= 64;
        for (int j = 1; j < 6; j++) { c += (u128)m * P.l[j] + t[j]; t[j - 1] = (uint64_t)c; c >>= 64; }
        c += t[6]; t[5] = (uint64_t)c; t[6] = t[7] + (uint64_t)(c >> 64);
    }
    fp o, s; /* result < 2p < 2^382, so t[6] == 0 */
    memcpy(o.l, t, 48);
    if (!raw_sub(&s, &o, &P)) o = s;
    *r = o;
}
/* Dedicated squaring (round 2: the CPU arm should not pay 36 limb products where 21 do): the 15 off-diagonal products
 * once, doubled, plus the 6 squares, then a separate 6-round Montgomery reduction.  Counted as one product. */
static void fp_sqr(fp *r, const fp *a) {
    uint64_t t[13] = {0};
    if (g_count_on) { g_fp_mul_count++; g_fp_sqr_count++; }
    for (int i = 0; i < 5; i++) {                      /* off-diagonal a_i a_j, i < j */
        u128 c = 0;
        for (int j = i + 1; j < 6; j++) { c += (u128)a->l[i] * a->l[j] + t[i + j]; t[i + j] = (uint64_t)c; c >>= 64; }
        t[i + 6] = (uint64_t)c;
    }
    uint64_t top = 0;                                   /* double */
    for (int k = 1; k < 12; k++) { uint64_t v = t[k]; t[k] = (v << 1) | top; top = v >> 63; }
    u128 c = 0;                                        /* + diagonal squares */
    for (int i = 0; i < 6; i++) {
        u128 sq = (u128)a->l[i] * a->l[i];
        c += (u128)t[2 * i] + (uint64_t)sq; t[2 * i] = (uint64_t)c; c >>= 64;
        c += (u128)t[2 * i + 1] + (uint64_t)(sq >> 64); t[2 * i + 1] = (uint64_t)c; c >>= 64;
    }
    for (int i = 0; i < 6; i++) {                      /* Montgomery reduction, one limb per round */
        uint64_t m = t[i] * N0;
        u128 cc = 0;
        for (int j = 0; j < 6; j++) { cc += (u128)m * P.l[j] + t[i + j]; t[i + j] = (uint64_t)cc; cc >>= 64; }
        for (int k = i + 6; k < 13 && cc; k++) { cc += t[k]; t[k] = (uint64_t)cc; cc >>= 64; }
    }
    fp o, s; /* a < p  =>  result < 2p < 2^382 */
    memcpy(o.l, t + 6, 48);
    if (!raw_sub(&s, &o, &P)) o = s;
    *r = o;
}
/* r = a^e, e little-endian 64-bit words.  Sliding 4-bit windows over the 8 odd powers a, a^3 .. a^15 — the same
 * exponentiation the CUDA path runs (csrc/fp.cuh fp_pow), so that the instrumented product counter below reports the
 * work of the algorithm that is actually executed (~465 products for the 381-bit exponents here, not ~570). */
static void fp_pow(fp *r, const fp *a, const uint64_t *e, int nw) {
    fp tab[8], a2, acc, t;
    tab[0] = *a;
    fp_sqr(&a2, a);
    for (int k = 1; k < 8; k++) fp_mul(&tab[k], &tab[k - 1], &a2);
    int i = 64 * nw - 1;
    while (i >= 0 && !((e[i >> 6] >> (i & 63)) & 1)) i--;
    if (i < 0) { *r = R1; return; }
    int started = 0;
    acc = R1;
    while (i >= 0) {
        if (!((e[i >> 6] >> (i & 63)) & 1)) { fp_sqr(&acc, &acc); i--; continue; }
        int l = i + 1 < 4 ? i + 1 : 4;
        unsigned w = 0;
        for (int k = 0; k < l; k++) w = (w << 1) | (unsigned)((e[(i - k) >> 6] >> ((i - k) & 63)) & 1);
        while (!(w & 1)) { w >>= 1; l--; }
        if (started) {
            for (int k = 0; k < l; k++) fp_sqr(&acc, &acc);
            t = tab[w >> 1];
            fp_mul(&acc, &acc, &t);
        } else { acc = tab[w >> 1]; started = 1; }
        i -= l;
    }
    *r = acc;
}
static uint64_t E_PM2[6], E_SQRT[6], E_PM3D4[6], E_PM1D2[6], E_PM1D3[6], E_PM1D6[6];
static void fp_inv(fp *r, const fp *a) { fp_pow(r, a, E_PM2, 6); }
static int fp_sqrt(fp *r, const fp *a) { fp s, c; fp_pow(&s, a, E_SQRT, 6); fp_sqr(&c, &s); *r = s; return fp_eq(&c, a); }
static void fp_to_mont(fp *r, const fp *a) { fp_mul(r, a, &R2); }
static void fp_from_mont(fp *r, const fp *a) { fp one = {{1, 0, 0, 0, 0, 0}}; fp_mul(r, a, &one); }
static void raw_from_be(fp *r, const uint8_t *b) {
    for (int i = 0; i < 6; i++) { uint64_t v = 0; for (int k = 0; k < 8; k++) v = (v << 8) | b[40 - 8 * i + k]; r->l[i] = v; }
}
static void raw_to_be(uint8_t *b, const fp *a) {
    for (int i = 0; i < 6; i++) for (int k = 0; k < 8; k++) b[40 - 8 * i + k] = (uint8_t)(a->l[i] >> (56 - 8 * k));
}
static int fp_from_be(fp *r, const uint8_t *b, int mask) { /* 0 if >= p */
    fp raw; raw_from_be(&raw, b);
    if (mask) raw.l[5] &= 0x1fffffffffffffffull;
    if (raw_geq(&raw, &P)) return 0;
    fp_to_mont(r, &raw); return 1;
}
static void fp_to_be(uint8_t *b, const fp *a) { fp raw; fp_from_mont(&raw, a); raw_to_be(b, &raw); }
static fp HALF_P;
static int fp_lex_largest(const fp *a) { fp raw; fp_from_mont(&raw, a); return !raw_geq(&HALF_P, &raw); }
static int fp_parity(const fp *a) { fp raw; fp_from_mont(&raw, a); return (int)(raw.l[0] & 1); }
static void fp_set_u64(fp *r, uint64_t v) { fp raw = {{v, 0, 0, 0, 0, 0}}; fp_to_mont(r, &raw); }
static void fp_from_hex(fp *r, const char *hex) { /* big-endian hex, up to 96 digits */
    uint8_t b[48] = {0};
    size_t n = strlen(hex);
    for (size_t i = 0; i < n; i++) {
        char c = hex[n - 1 - i];
        int v = (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : c - 'A' + 10;
        b[47 - i / 2] |= (uint8_t)(v << (4 * (i & 1)));
    }
    fp_from_be(r, b, 0);
}

/* ================================================================================================ Fp2 */
typedef struct { fp c0, c1; } fp2;
static fp2 F2_ZERO, F2_ONE;
static int f2_is_zero(const fp2 *a) { return fp_is_zero(&a->c0) && fp_is_zero(&a->c1); }
static int f2_eq(const fp2 *a, const fp2 *b) { return fp_eq(&a->c0, &b->c0) && fp_eq(&a->c1, &b->c1); }
static void f2_add(fp2 *r, const fp2 *a, const fp2 *b) { fp_add(&r->c0, &a->c0, &b->c0); fp_add(&r->c1, &a->c1, &b->c1); }
static void f2_sub(fp2 *r, const fp2 *a, const fp2 *b) { fp_sub(&r->c0, &a->c0, &b->c0); fp_sub(&r->c1, &a->c1, &b->c1); }
static void f2_neg(fp2 *r, const fp2 *a) { fp_neg(&r->c0, &a->c0); fp_neg(&r->c1, &a->c1); }
static void f2_conj(fp2 *r, const fp2 *a) { r->c0 = a->c0; fp_neg(&r->c1, &a->c1); }
static void f2_mul(fp2 *r, const fp2 *a, const fp2 *b) {
    fp t0, t1, s0, s1, m;
    fp_mul(&t0, &a->c0, &b->c0); fp_mul(&t1, &a->c1, &b->c1);
    fp_add(&s0, &a->c0, &a->c1); fp_add(&s1, &b->c0, &b->c1);
    fp_mul(&m, &s0, &s1); fp_sub(&m, &m, &t0); fp_sub(&m, &m, &t1);
    fp_sub(&r->c0, &t0, &t1); r->c1 = m;
}
static void f2_sqr(fp2 *r, const fp2 *a) {
    fp s, d, m;
    fp_add(&s, &a->c0, &a->c1); fp_sub(&d, &a->c0, &a->c1); fp_mul(&m, &a->c0, &a->c1);
    fp_mul(&r->c0, &s, &d); fp_add(&r->c1, &m, &m);
}
static void f2_mul_fp(fp2 *r, const fp2 *a, const fp *k) { fp_mul(&r->c0, &a->c0, k); fp_mul(&r->c1, &a->c1, k); }
static void f2_mul_xi(fp2 *r, const fp2 *a) { fp t0, t1; fp_sub(&t0, &a->c0, &a->c1); fp_add(&t1, &a->c0, &a->c1); r->c0 = t0; r->c1 = t1; }
static void f2_inv(fp2 *r, const fp2 *a) {
    fp n, t;
    fp_sqr(&n, &a->c0); fp_sqr(&t, &a->c1); fp_add(&n, &n, &t); fp_inv(&n, &n);
    fp_mul(&r->c0, &a->c0, &n); fp_mul(&t, &a->c1, &n); fp_neg(&r->c1, &t);
}
static void f2_pow(fp2 *r, const fp2 *a, const uint64_t *e, int nw) {
    fp2 acc = F2_ONE;
    int started = 0;
    for (int w = nw - 1; w >= 0; w--)
        for (int b = 63; b >= 0; b--) {
            if (started) f2_sqr(&acc, &acc);
            if ((e[w] >> b) & 1) { if (started) f2_mul(&acc, &acc, a); else { acc = *a; started = 1; } }
        }
    *r = acc;
}
static int f2_sqrt(fp2 *r, const fp2 *a) {
    if (f2_is_zero(a)) { *r = *a; return 1; }
    fp2 a1, alpha, x0, x, chk, m1;
    f2_pow(&a1, a, E_PM3D4, 6);
    f2_sqr(&alpha, &a1); f2_mul(&alpha, &alpha, a);
    f2_mul(&x0, &a1, a);
    fp_neg(&m1.c0, &R1); memset(&m1.c1, 0, sizeof(fp));
    if (f2_eq(&alpha, &m1)) { fp_neg(&x.c0, &x0.c1); x.c1 = x0.c0; }
    else { fp2 b; f2_add(&b, &F2_ONE, &alpha); f2_pow(&b, &b, E_PM1D2, 6); f2_mul(&x, &b, &x0); }
    f2_sqr(&chk, &x); *r = x;
    return f2_eq(&chk, a);
}
static int f2_sgn0(const fp2 *a) { int s0 = fp_parity(&a->c0), z0 = fp_is_zero(&a->c0), s1 = fp_parity(&a->c1); return s0 | (z0 & s1); }
static int f2_lex_largest(const fp2 *a) { return fp_is_zero(&a->c1) ? fp_lex_largest(&a->c0) : fp_lex_largest(&a->c1); }

/* ================================================================================================ Fp6 / Fp12 */
typedef struct { fp2 c0, c1, c2; } fp6;
typedef struct { fp6 c0, c1; } fp12;
static void f6_add(fp6 *r, const fp6 *a, const fp6 *b) { f2_add(&r->c0, &a->c0, &b->c0); f2_add(&r->c1, &a->c1, &b->c1); f2_add(&r->c2, &a->c2, &b->c2); }
static void f6_sub(fp6 *r, const fp6 *a, const fp6 *b) { f2_sub(&r->c0, &a->c0, &b->c0); f2_sub(&r->c1, &a->c1, &b->c1); f2_sub(&r->c2, &a->c2, &b->c2); }
static void f6_neg(fp6 *r, const fp6 *a) { f2_neg(&r->c0, &a->c0); f2_neg(&r->c1, &a->c1); f2_neg(&r->c2, &a->c2); }
static void f6_mul_v(fp6 *r, const fp6 *a) { fp2 t; f2_mul_xi(&t, &a->c2); r->c2 = a->c1; r->c1 = a->c0; r->c0 = t; }
static void f6_mul(fp6 *r, const fp6 *a, const fp6 *b) {
    fp2 v0, v1, v2, t0, t1, x0, x1, x2;
    f2_mul(&v0, &a->c0, &b->c0); f2_mul(&v1, &a->c1, &b->c1); f2_mul(&v2, &a->c2, &b->c2);
    f2_add(&t0, &a->c1, &a->c2); f2_add(&t1, &b->c1, &b->c2); f2_mul(&x0, &t0, &t1);
    f2_sub(&x0, &x0, &v1); f2_sub(&x0, &x0, &v2); f2_mul_xi(&x0, &x0); f2_add(&x0, &x0, &v0);
    f2_add(&t0, &a->c0, &a->c1); f2_add(&t1, &b->c0, &b->c1); f2_mul(&x1, &t0, &t1);
    f2_sub(&x1, &x1, &v0); f2_sub(&x1, &x1, &v1); f2_mul_xi(&t0, &v2); f2_add(&x1, &x1, &t0);
    f2_add(&t0, &a->c0, &a->c2); f2_add(&t1, &b->c0, &b->c2); f2_mul(&x2, &t0, &t1);
    f2_sub(&x2, &x2, &v0); f2_sub(&x2, &x2, &v2); f2_add(&x2, &x2, &v1);
    r->c0 = x0; r->c1 = x1; r->c2 = x2;
}
static void f6_inv(fp6 *r, const fp6 *a) {
    fp2 c0, c1, c2, t, d;
    f2_sqr(&c0, &a->c0); f2_mul(&t, &a->c1, &a->c2); f2_mul_xi(&t, &t); f2_sub(&c0, &c0, &t);
    f2_sqr(&c1, &a->c2); f2_mul_xi(&c1, &c1); f2_mul(&t, &a->c0, &a->c1); f2_sub(&c1, &c1, &t);
    f2_sqr(&c2, &a->c1); f2_mul(&t, &a->c0, &a->c2); f2_sub(&c2, &c2, &t);
    f2_mul(&d, &a->c2, &c1); f2_mul(&t, &a->c1, &c2); f2_add(&d, &d, &t); f2_mul_xi(&d, &d);
    f2_mul(&t, &a->c0, &c0); f2_add(&d, &d, &t); f2_inv(&d, &d);
    f2_mul(&r->c0, &c0, &d); f2_mul(&r->c1, &c1, &d); f2_mul(&r->c2, &c2, &d);
}
static fp12 F12_ONE;
static int f12_is_one(const fp12 *a) { return memcmp(a, &F12_ONE, sizeof(fp12)) == 0; }
static void f12_conj(fp12 *r, const fp12 *a) { r->c0 = a->c0; f6_neg(&r->c1, &a->c1); }
static void f12_mul(fp12 *r, const fp12 *a, const fp12 *b) {
    fp6 v0, v1, t0, t1, x1;
    f6_mul(&v0, &a->c0, &b->c0); f6_mul(&v1, &a->c1, &b->c1);
    f6_add(&t0, &a->c0, &a->c1); f6_add(&t1, &b->c0, &b->c1); f6_mul(&x1, &t0, &t1);
    f6_sub(&x1, &x1, &v0); f6_sub(&x1, &x1, &v1);
    f6_mul_v(&t0, &v1); f6_add(&r->c0, &v0, &t0); r->c1 = x1;
}
static void f12_sqr(fp12 *r, const fp12 *a) { fp12 t = *a; f12_mul(r, &t, &t); }
static void f12_inv(fp12 *r, const fp12 *a) {
    fp6 t0, t1;
    f6_mul(&t0, &a->c0, &a->c0); f6_mul(&t1, &a->c1, &a->c1); f6_mul_v(&t1, &t1); f6_sub(&t0, &t0, &t1);
    f6_inv(&t0, &t0);
    f6_mul(&r->c0, &a->c0, &t0); f6_mul(&t1, &a->c1, &t0); f6_neg(&r->c1, &t1);
}
static fp2 GAMMA1[6]; /* xi^(i (p-1)/6) */
static void f12_frob(fp12 *r, const fp12 *a) {
    fp2 *dst[6] = {&r->c0.c0, &r->c1.c0, &r->c0.c1, &r->c1.c1, &r->c0.c2, &r->c1.c2};
    const fp2 *src[6] = {&a->c0.c0, &a->c1.c0, &a->c0.c1, &a->c1.c1, &a->c0.c2, &a->c1.c2};
    for (int i = 0; i < 6; i++) { fp2 t; f2_conj(&t, src[i]); if (i) f2_mul(dst[i], &t, &GAMMA1[i]); else *dst[i] = t; }
}

/* ================================================================================================ curves */
#define DEFINE_CURVE(N, F, ZERO, ONE, add, sub, mul, sqr, neg, inv, is_zero, eq)                               \
    typedef struct { F x, y; int inf; } N##_aff;                                                                \
    typedef struct { F x, y, z; } N##_jac;                                                                      \
    static int N##_is_inf(const N##_jac *p) { return is_zero(&p->z); }                                          \
    static void N##_set_inf(N##_jac *p) { p->x = ONE; p->y = ONE; p->z = ZERO; }                                \
    static void N##_from_aff(N##_jac *p, const N##_aff *a) {                                                    \
        if (a->inf) N##_set_inf(p); else { p->x = a->x; p->y = a->y; p->z = ONE; } }                            \
    static void N##_jneg(N##_jac *r, const N##_jac *p) { r->x = p->x; neg(&r->y, &p->y); r->z = p->z; }         \
    static void N##_dbl(N##_jac *r, const N##_jac *p) {                                                         \
        if (N##_is_inf(p)) { *r = *p; return; }                                                                 \
        F A, B, C, D, E, G, t, x3, z3;                                                                          \
        sqr(&A, &p->x); sqr(&B, &p->y); sqr(&C, &B);                                                            \
        add(&t, &p->x, &B); sqr(&t, &t); sub(&t, &t, &A); sub(&t, &t, &C); add(&D, &t, &t);                     \
        add(&E, &A, &A); add(&E, &E, &A); sqr(&G, &E);                                                          \
        mul(&z3, &p->y, &p->z); add(&z3, &z3, &z3);                                                             \
        add(&t, &D, &D); sub(&x3, &G, &t); sub(&t, &D, &x3); mul(&t, &E, &t);                                   \
        add(&C, &C, &C); add(&C, &C, &C); add(&C, &C, &C);                                                      \
        sub(&r->y, &t, &C); r->x = x3; r->z = z3; }                                                             \
    static void N##_jadd(N##_jac *r, const N##_jac *p, const N##_jac *q) {                                      \
        if (N##_is_inf(p)) { *r = *q; return; }                                                                 \
        if (N##_is_inf(q)) { *r = *p; return; }                                                                 \
        F z1z1, z2z2, u1, u2, s1, s2, h, rr, t, hh, hhh, v, x3;                                                 \
        sqr(&z1z1, &p->z); sqr(&z2z2, &q->z); mul(&u1, &p->x, &z2z2); mul(&u2, &q->x, &z1z1);                   \
        mul(&t, &q->z, &z2z2); mul(&s1, &p->y, &t); mul(&t, &p->z, &z1z1); mul(&s2, &q->y, &t);                 \
        sub(&h, &u2, &u1); sub(&rr, &s2, &s1);                                                                  \
        if (is_zero(&h)) { if (is_zero(&rr)) N##_dbl(r, p); else N##_set_inf(r); return; }                      \
        sqr(&hh, &h); mul(&hhh, &hh, &h); mul(&v, &u1, &hh);                                                    \
        sqr(&x3, &rr); sub(&x3, &x3, &hhh); add(&t, &v, &v); sub(&x3, &x3, &t);                                 \
        sub(&t, &v, &x3); mul(&t, &rr, &t); mul(&s1, &s1, &hhh); sub(&r->y, &t, &s1);                           \
        mul(&t, &p->z, &q->z); mul(&r->z, &t, &h); r->x = x3; }                                                 \
    static void N##_add_aff(N##_jac *r, const N##_jac *p, const N##_aff *q) {                                   \
        N##_jac qj; N##_from_aff(&qj, q); N##_jadd(r, p, &qj); }                                                \
    static void N##_to_aff(N##_aff *a, const N##_jac *p) {                                                      \
        if (N##_is_inf(p)) { a->inf = 1; a->x = ZERO; a->y = ZERO; return; }                                    \
        F zi, zi2, zi3; inv(&zi, &p->z); sqr(&zi2, &zi); mul(&zi3, &zi2, &zi);                                  \
        mul(&a->x, &p->x, &zi2); mul(&a->y, &p->y, &zi3); a->inf = 0; }                                         \
    static void N##_mul(N##_jac *r, const N##_jac *p, const uint64_t *k, int nw) {                              \
        N##_jac acc; N##_set_inf(&acc);                                                                         \
        for (int w = nw - 1; w >= 0; w--) for (int b = 63; b >= 0; b--) {                                       \
            N##_dbl(&acc, &acc); if ((k[w] >> b) & 1) N##_jadd(&acc, &acc, p); }                                \
        *r = acc; }                                                                                             \
    static int N##_jeq(const N##_jac *p, const N##_jac *q) {                                                    \
        if (N##_is_inf(p) || N##_is_inf(q)) return N##_is_inf(p) && N##_is_inf(q);                              \
        F a, b, z1z1, z2z2, t; sqr(&z1z1, &p->z); sqr(&z2z2, &q->z);                                            \
        mul(&a, &p->x, &z2z2); mul(&b, &q->x, &z1z1); if (!eq(&a, &b)) return 0;                                \
        mul(&t, &z2z2, &q->z); mul(&a, &p->y, &t); mul(&t, &z1z1, &p->z); mul(&b, &q->y, &t); return eq(&a, &b); }

static fp FP_ZERO;
DEFINE_CURVE(g1, fp, FP_ZERO, R1, fp_add, fp_sub, fp_mul, fp_sqr, fp_neg, fp_inv, fp_is_zero, fp_eq)
DEFINE_CURVE(g2, fp2, F2_ZERO, F2_ONE, f2_add, f2_sub, f2_mul, f2_sqr, f2_neg, f2_inv, f2_is_zero, f2_eq)

static const uint64_t Z_ABS[1] = {0xd201000000010000ull};
static const uint64_t R_ORDER[4] = {0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull};
static g1_aff G1_GEN, G1_GEN_NEG;
static g2_aff G2_GEN;
static fp BETA, B1;          /* G1 endomorphism constant; curve b = 4 */
static fp2 B2, PSI_X, PSI_Y; /* twist b' = 4(1+u); psi coefficients */
static fp PSI2_X;

/* ---- decoding (ZCash format, blst error taxonomy) */
static int all_zero(const uint8_t *b, int n) { uint8_t x = 0; for (int i = 0; i < n; i++) x |= b[i]; return x == 0; }
static int g1_uncompress(g1_aff *o, const uint8_t b[48]) {
    o->inf = 0;
    if (!(b[0] & 0x80)) return BAD_ENCODING;
    if (b[0] & 0x40) { if ((b[0] & 0x3f) == 0 && all_zero(b + 1, 47)) { o->inf = 1; o->x = FP_ZERO; o->y = FP_ZERO; return OK; } return BAD_ENCODING; }
    fp x, y2, y;
    if (!fp_from_be(&x, b, 1)) return BAD_ENCODING;
    fp_sqr(&y2, &x); fp_mul(&y2, &y2, &x); fp_add(&y2, &y2, &B1);
    if (!fp_sqrt(&y, &y2)) return NOT_ON_CURVE;
    if (fp_lex_largest(&y) != ((b[0] & 0x20) != 0)) fp_neg(&y, &y);
    o->x = x; o->y = y;
    return OK;
}
static int g2_uncompress(g2_aff *o, const uint8_t b[96]) {
    o->inf = 0;
    if (!(b[0] & 0x80)) return BAD_ENCODING;
    if (b[0] & 0x40) { if ((b[0] & 0x3f) == 0 && all_zero(b + 1, 95)) { o->inf = 1; o->x = F2_ZERO; o->y = F2_ZERO; return OK; } return BAD_ENCODING; }
    fp2 x, y2, y;
    if (!fp_from_be(&x.c1, b, 1) || !fp_from_be(&x.c0, b + 48, 0)) return BAD_ENCODING;
    f2_sqr(&y2, &x); f2_mul(&y2, &y2, &x); f2_add(&y2, &y2, &B2);
    if (!f2_sqrt(&y, &y2)) return NOT_ON_CURVE;
    if (f2_lex_largest(&y) != ((b[0] & 0x20) != 0)) f2_neg(&y, &y);
    o->x = x; o->y = y;
    return OK;
}
static void g1_compress(uint8_t out[48], const g1_aff *a) {
    if (a->inf) { memset(out, 0, 48); out[0] = 0xc0; return; }
    fp_to_be(out, &a->x); out[0] |= 0x80; if (fp_lex_largest(&a->y)) out[0] |= 0x20;
}
static void g2_compress(uint8_t out[96], const g2_aff *a) {
    if (a->inf) { memset(out, 0, 96); out[0] = 0xc0; return; }
    fp_to_be(out, &a->x.c1); fp_to_be(out + 48, &a->x.c0); out[0] |= 0x80; if (f2_lex_largest(&a->y)) out[0] |= 0x20;
}
/* ---- subgroup membership: definition ([r]P = inf) and the endomorphism shortcuts blst-class libraries use */
static int g1_in_group_def(const g1_aff *a) { g1_jac p, t; g1_from_aff(&p, a); g1_mul(&t, &p, R_ORDER, 4); return g1_is_inf(&t); }
static int g2_in_group_def(const g2_aff *a) { g2_jac p, t; g2_from_aff(&p, a); g2_mul(&t, &p, R_ORDER, 4); return g2_is_inf(&t); }
static int g1_in_group(const g1_aff *a) { /* phi(P) == -[z^2]P */
    if (a->inf) return 1;
    g1_jac p, t, ph;
    g1_from_aff(&p, a); g1_mul(&t, &p, Z_ABS, 1); g1_mul(&t, &t, Z_ABS, 1);
    fp_mul(&ph.x, &a->x, &BETA); fp_neg(&ph.y, &a->y); ph.z = R1;
    return g1_jeq(&t, &ph);
}
static void g2_psi(g2_jac *r, const g2_jac *p) {
    fp2 t; f2_conj(&t, &p->x); f2_mul(&r->x, &t, &PSI_X); f2_conj(&t, &p->y); f2_mul(&r->y, &t, &PSI_Y); f2_conj(&r->z, &p->z);
}
static void g2_psi2(g2_jac *r, const g2_jac *p) { f2_mul_fp(&r->x, &p->x, &PSI2_X); f2_neg(&r->y, &p->y); r->z = p->z; }
static int g2_in_group(const g2_aff *a) { /* psi(Q) == [z]Q = -[|z|]Q */
    if (a->inf) return 1;
    g2_jac q, t, ps;
    g2_from_aff(&q, a); g2_mul(&t, &q, Z_ABS, 1); g2_psi(&ps, &q); g2_jneg(&ps, &ps);
    return g2_jeq(&t, &ps);
}
static int key_validate(g1_aff *o, const uint8_t b[48]) {
    int rc = g1_uncompress(o, b);
    if (rc) return rc;
    if (o->inf) return PK_IS_INFINITY;
    return g1_in_group(o) ? OK : NOT_IN_GROUP;
}

/* ================================================================================================ hash to G2 */
static const char DST[] = "BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_"; /* crypto/bls.rs:22 */
static void expand_message_xmd256(const uint8_t *msg, size_t len, uint8_t out[256]) {
    size_t dl = sizeof(DST) - 1;
    uint8_t *buf = malloc(64 + len + 3 + dl + 1 + 64);
    uint8_t b0[32], bi[32];
    memset(buf, 0, 64); memcpy(buf + 64, msg, len);
    buf[64 + len] = 1; buf[65 + len] = 0; buf[66 + len] = 0;
    memcpy(buf + 67 + len, DST, dl); buf[67 + len + dl] = (uint8_t)dl;
    orc_sha256(buf, 68 + len + dl, b0);
    for (int i = 1; i <= 8; i++) {
        uint8_t t[32 + 1 + 64];
        for (int k = 0; k < 32; k++) t[k] = (i == 1) ? b0[k] : (uint8_t)(b0[k] ^ bi[k]);
        t[32] = (uint8_t)i; memcpy(t + 33, DST, dl); t[33 + dl] = (uint8_t)dl;
        orc_sha256(t, 34 + dl, bi);
        memcpy(out + 32 * (i - 1), bi, 32);
    }
    free(buf);
}
static fp R3; /* 2^1152 mod p: to_mont(x * 2^384) = mont_mul(x, R3) */
static void fp_from_be64(fp *r, const uint8_t *b) { /* 64 bytes mod p */
    fp lo, hi = {{0}}, t;
    raw_from_be(&lo, b + 16);
    for (int i = 0; i < 2; i++) { uint64_t v = 0; for (int k = 0; k < 8; k++) v = (v << 8) | b[8 - 8 * i + k]; hi.l[i] = v; }
    fp_mul(&lo, &lo, &R2); fp_mul(&t, &hi, &R3); fp_add(r, &lo, &t);
}
static fp2 SSWU_A, SSWU_B, SSWU_Z, ISO_XN[4], ISO_XD[3], ISO_YN[4], ISO_YD[4];
static void sswu_g(fp2 *r, const fp2 *x) { fp2 t; f2_sqr(&t, x); f2_add(&t, &t, &SSWU_A); f2_mul(&t, &t, x); f2_add(r, &t, &SSWU_B); }
static void sswu(fp2 *xo, fp2 *yo, const fp2 *t) {
    fp2 t2, zt2, tv1, x1, gx, y, tmp;
    f2_sqr(&t2, t); f2_mul(&zt2, &SSWU_Z, &t2); f2_sqr(&tv1, &zt2); f2_add(&tv1, &tv1, &zt2);
    if (f2_is_zero(&tv1)) { f2_mul(&tmp, &SSWU_Z, &SSWU_A); f2_inv(&tmp, &tmp); f2_mul(&x1, &SSWU_B, &tmp); }
    else { f2_inv(&tmp, &tv1); f2_add(&tmp, &tmp, &F2_ONE); fp2 nb, ia; f2_neg(&nb, &SSWU_B); f2_inv(&ia, &SSWU_A); f2_mul(&nb, &nb, &ia); f2_mul(&x1, &nb, &tmp); }
    sswu_g(&gx, &x1);
    if (f2_sqrt(&y, &gx)) *xo = x1;
    else { f2_mul(xo, &zt2, &x1); sswu_g(&gx, xo); f2_sqrt(&y, &gx); }
    if (f2_sgn0(t) != f2_sgn0(&y)) f2_neg(&y, &y);
    *yo = y;
}
static void horner(fp2 *r, const fp2 *c, int n, const fp2 *x) { *r = c[n - 1]; for (int i = n - 2; i >= 0; i--) { f2_mul(r, r, x); f2_add(r, r, &c[i]); } }
static void iso3(g2_aff *o, const fp2 *x, const fp2 *y) {
    fp2 xn, xd, yn, yd;
    horner(&xn, ISO_XN, 4, x); horner(&xd, ISO_XD, 3, x); horner(&yn, ISO_YN, 4, x); horner(&yd, ISO_YD, 4, x);
    if (f2_is_zero(&xd) || f2_is_zero(&yd)) { o->inf = 1; o->x = F2_ZERO; o->y = F2_ZERO; return; }
    f2_inv(&xd, &xd); f2_inv(&yd, &yd);
    f2_mul(&o->x, &xn, &xd); f2_mul(&yn, &yn, &yd); f2_mul(&o->y, y, &yn); o->inf = 0;
}
static void clear_cofactor(g2_jac *r, const g2_jac *p) { /* RFC 9380 G.3 */
    g2_jac t1, t2, t3, n;
    g2_mul(&t1, p, Z_ABS, 1); g2_jneg(&t1, &t1);
    g2_psi(&t2, p);
    g2_dbl(&t3, p); g2_psi2(&t3, &t3);
    g2_jneg(&n, &t2); g2_jadd(&t3, &t3, &n);
    g2_jadd(&t2, &t1, &t2);
    g2_mul(&t2, &t2, Z_ABS, 1); g2_jneg(&t2, &t2);
    g2_jadd(&t3, &t3, &t2);
    g2_jneg(&n, &t1); g2_jadd(&t3, &t3, &n);
    g2_jneg(&n, p); g2_jadd(r, &t3, &n);
}
static void hash_to_g2(g2_aff *o, const uint8_t *msg, size_t len) {
    uint8_t u[256];
    expand_message_xmd256(msg, len, u);
    fp2 u0, u1, x, y;
    fp_from_be64(&u0.c0, u); fp_from_be64(&u0.c1, u + 64); fp_from_be64(&u1.c0, u + 128); fp_from_be64(&u1.c1, u + 192);
    g2_aff q0, q1; g2_jac j0, j1;
    sswu(&x, &y, &u0); iso3(&q0, &x, &y);
    sswu(&x, &y, &u1); iso3(&q1, &x, &y);
    g2_from_aff(&j0, &q0); g2_from_aff(&j1, &q1); g2_jadd(&j0, &j0, &j1);
    clear_cofactor(&j1, &j0);
    g2_to_aff(o, &j1);
}

/* ================================================================================================ pairing */
/* line through T (Jacobian) at P, scaled into Fp2-multiples: A + B v + C v w (see DESIGN.md "Miller loop") */
static void f12_mul_line(fp12 *f, const fp2 *A, const fp2 *B, const fp2 *C) {
    fp12 l; memset(&l, 0, sizeof l);
    l.c0.c0 = *A; l.c0.c1 = *B; l.c1.c1 = *C;
    f12_mul(f, f, &l);
}
static void miller_loop(fp12 *f, const g1_aff *p, const g2_aff *q) {
    *f = F12_ONE;
    if (p->inf || q->inf) return;
    g2_jac t; g2_from_aff(&t, q);
    for (int bit = 62; bit >= 0; bit--) {
        fp2 A, B, C, xx, yy, zz, e, tmp;
        if (bit != 62) f12_sqr(f, f);
        f2_sqr(&xx, &t.x); f2_sqr(&yy, &t.y); f2_sqr(&zz, &t.z);
        f2_add(&e, &xx, &xx); f2_add(&e, &e, &xx);
        f2_mul(&A, &e, &t.x); f2_add(&tmp, &yy, &yy); f2_sub(&A, &A, &tmp);
        f2_mul(&tmp, &e, &zz); f2_mul_fp(&tmp, &tmp, &p->x); f2_neg(&B, &tmp);
        g2_dbl(&t, &t);
        f2_mul(&tmp, &t.z, &zz); f2_mul_fp(&C, &tmp, &p->y);
        f12_mul_line(f, &A, &B, &C);
        if ((Z_ABS[0] >> bit) & 1) {
            fp2 zzz, h, rr, z3;
            f2_sqr(&zz, &t.z); f2_mul(&zzz, &zz, &t.z);
            f2_mul(&h, &q->x, &zz); f2_sub(&h, &h, &t.x);
            f2_mul(&rr, &q->y, &zzz); f2_sub(&rr, &rr, &t.y);
            f2_mul(&z3, &t.z, &h);
            f2_mul(&A, &rr, &q->x); f2_mul(&tmp, &q->y, &z3); f2_sub(&A, &A, &tmp);
            f2_mul_fp(&tmp, &rr, &p->x); f2_neg(&B, &tmp);
            f2_mul_fp(&C, &z3, &p->y);
            g2_add_aff(&t, &t, q);
            f12_mul_line(f, &A, &B, &C);
        }
    }
    f12_conj(f, f);
}
static void f12_pow_z(fp12 *r, const fp12 *g) {
    fp12 acc = *g;
    for (int bit = 62; bit >= 0; bit--) { f12_sqr(&acc, &acc); if ((Z_ABS[0] >> bit) & 1) f12_mul(&acc, &acc, g); }
    *r = acc;
}
static int final_exp_is_one(const fp12 *fin) {
    fp12 f, t0, t1, a, b, c;
    f12_inv(&t0, fin); f12_conj(&t1, fin); f12_mul(&t0, &t1, &t0);
    f12_frob(&t1, &t0); f12_frob(&t1, &t1); f12_mul(&f, &t1, &t0);
    f12_pow_z(&t0, &f); f12_mul(&t0, &t0, &f); f12_conj(&t0, &t0);
    f12_pow_z(&a, &t0); f12_mul(&a, &a, &t0); f12_conj(&a, &a);
    f12_pow_z(&t0, &a); f12_conj(&t0, &t0); f12_frob(&t1, &a); f12_mul(&b, &t0, &t1);
    f12_pow_z(&t0, &b); f12_pow_z(&t0, &t0); f12_frob(&t1, &b); f12_frob(&t1, &t1); f12_mul(&c, &t0, &t1);
    f12_conj(&t1, &b); f12_mul(&c, &c, &t1);
    f12_sqr(&t0, &f); f12_mul(&t0, &t0, &f); f12_mul(&c, &c, &t0);
    return f12_is_one(&c);
}

/* ================================================================================================ init */
static void bn_div_small(uint64_t out[6], const uint64_t in[6], uint64_t d) {
    u128 rem = 0;
    for (int i = 5; i >= 0; i--) { u128 cur = (rem << 64) | in[i]; out[i] = (uint64_t)(cur / d); rem = cur % d; }
}
static void f2_from_hex(fp2 *r, const char *c0, const char *c1) { fp_from_hex(&r->c0, c0); fp_from_hex(&r->c1, c1); }
static pthread_once_t init_once = PTHREAD_ONCE_INIT;
static void do_init(void) {
    /* R1 = 2^384 mod p by 384 doublings of 1; R2 = R1^2 * R^-1 ... computed with plain modular doubling */
    fp one = {{1, 0, 0, 0, 0, 0}}, t = one;
    for (int i = 0; i < 384; i++) { fp s; if (raw_add(&s, &t, &t) || raw_geq(&s, &P)) raw_sub(&s, &s, &P); t = s; }
    R1 = t;
    for (int i = 0; i < 384; i++) { fp s; if (raw_add(&s, &t, &t) || raw_geq(&s, &P)) raw_sub(&s, &s, &P); t = s; }
    R2 = t;
    fp_mul(&R3, &R2, &R2); /* R2*R2/R = R^3 mod p */
    memset(&FP_ZERO, 0, sizeof FP_ZERO);
    F2_ZERO.c0 = FP_ZERO; F2_ZERO.c1 = FP_ZERO; F2_ONE.c0 = R1; F2_ONE.c1 = FP_ZERO;
    memset(&F12_ONE, 0, sizeof F12_ONE); F12_ONE.c0.c0 = F2_ONE;
    /* exponents */
    uint64_t pm1[6], pm3[6], pp1[6];
    memcpy(pm1, P.l, 48); pm1[0] -= 1;
    memcpy(E_PM2, P.l, 48); E_PM2[0] -= 2;
    memcpy(pm3, P.l, 48); pm3[0] -= 3;
    memcpy(pp1, P.l, 48); pp1[0] += 1;
    bn_div_small(E_SQRT, pp1, 4); bn_div_small(E_PM3D4, pm3, 4); bn_div_small(E_PM1D2, pm1, 2);
    bn_div_small(E_PM1D3, pm1, 3); bn_div_small(E_PM1D6, pm1, 6);
    memcpy(HALF_P.l, E_PM1D2, 48);
    fp_set_u64(&B1, 4);
    B2.c0 = B1; B2.c1 = B1;
    /* generators (SURVEY.md Appendix A) */
    fp_from_hex(&G1_GEN.x, "17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb");
    fp_from_hex(&G1_GEN.y, "08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1");
    G1_GEN.inf = 0; G1_GEN_NEG = G1_GEN; fp_neg(&G1_GEN_NEG.y, &G1_GEN.y);
    f2_from_hex(&G2_GEN.x, "024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8",
                "13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e");
    f2_from_hex(&G2_GEN.y, "0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801",
                "0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be");
    G2_GEN.inf = 0;
    /* Frobenius: gamma1[i] = xi^(i (p-1)/6) */
    fp2 xi = F2_ONE, g; xi.c1 = R1;
    f2_pow(&g, &xi, E_PM1D6, 6);
    GAMMA1[0] = F2_ONE; GAMMA1[1] = g;
    for (int i = 2; i < 6; i++) f2_mul(&GAMMA1[i], &GAMMA1[i - 1], &g);
    f2_inv(&PSI_X, &GAMMA1[2]); f2_inv(&PSI_Y, &GAMMA1[3]);
    { fp2 c, n; f2_conj(&c, &PSI_X); f2_mul(&n, &c, &PSI_X); PSI2_X = n.c0; }
    /* beta: the non-trivial cube root of unity with phi(G) == -[z^2]G */
    { fp two, b; fp_set_u64(&two, 2); fp_pow(&b, &two, E_PM1D3, 6);
      g1_jac G, tz; g1_from_aff(&G, &G1_GEN); g1_mul(&tz, &G, Z_ABS, 1); g1_mul(&tz, &tz, Z_ABS, 1); g1_jneg(&tz, &tz);
      g1_aff want; g1_to_aff(&want, &tz);
      fp cand = b, x;
      fp_mul(&x, &G1_GEN.x, &cand);
      if (!fp_eq(&x, &want.x)) { fp_sqr(&cand, &b); }
      BETA = cand; }
    /* SSWU / isogeny (RFC 9380 8.8.2, E.3; SURVEY.md Appendix A) */
    fp z0; memset(&z0, 0, sizeof z0);
    fp_set_u64(&SSWU_A.c1, 240); SSWU_A.c0 = z0;
    fp_set_u64(&SSWU_B.c0, 1012); SSWU_B.c1 = SSWU_B.c0;
    { fp a, b; fp_set_u64(&a, 2); fp_set_u64(&b, 1); fp_neg(&SSWU_Z.c0, &a); fp_neg(&SSWU_Z.c1, &b); }
    const char *k10 = "5c759507e8e333ebb5b7a9a47d7ed8532c52d39fd3a042a88b58423c50ae15d5c2638e343d9c71c6238aaaaaaaa97d6";
    f2_from_hex(&ISO_XN[0], k10, k10);
    f2_from_hex(&ISO_XN[1], "0", "11560bf17baa99bc32126fced787c88f984f87adf7ae0c7f9a208c6b4f20a4181472aaa9cb8d555526a9ffffffffc71a");
    f2_from_hex(&ISO_XN[2], "11560bf17baa99bc32126fced787c88f984f87adf7ae0c7f9a208c6b4f20a4181472aaa9cb8d555526a9ffffffffc71e",
                "8ab05f8bdd54cde190937e76bc3e447cc27c3d6fbd7063fcd104635a790520c0a395554e5c6aaaa9354ffffffffe38d");
    f2_from_hex(&ISO_XN[3], "171d6541fa38ccfaed6dea691f5fb614cb14b4e7f4e810aa22d6108f142b85757098e38d0f671c7188e2aaaaaaaa5ed1", "0");
    { fp a; fp_set_u64(&a, 72); ISO_XD[0].c0 = z0; fp_neg(&ISO_XD[0].c1, &a);
      fp_set_u64(&ISO_XD[1].c0, 12); fp_set_u64(&a, 12); fp_neg(&ISO_XD[1].c1, &a);
      ISO_XD[2] = F2_ONE; }
    const char *k30 = "1530477c7ab4113b59a4c18b076d11930f7da5d4a07f649bf54439d87d27e500fc8c25ebf8c92f6812cfc71c71c6d706";
    f2_from_hex(&ISO_YN[0], k30, k30);
    f2_from_hex(&ISO_YN[1], "0", "5c759507e8e333ebb5b7a9a47d7ed8532c52d39fd3a042a88b58423c50ae15d5c2638e343d9c71c6238aaaaaaaa97be");
    f2_from_hex(&ISO_YN[2], "11560bf17baa99bc32126fced787c88f984f87adf7ae0c7f9a208c6b4f20a4181472aaa9cb8d555526a9ffffffffc71c",
                "8ab05f8bdd54cde190937e76bc3e447cc27c3d6fbd7063fcd104635a790520c0a395554e5c6aaaa9354ffffffffe38f");
    f2_from_hex(&ISO_YN[3], "124c9ad43b6cf79bfbf7043de3811ad0761b0f37a1e26286b0e977c69aa274524e79097a56dc4bd9e1b371c71c718b10", "0");
    { fp a; fp_set_u64(&a, 432); fp_neg(&ISO_YD[0].c0, &a); ISO_YD[0].c1 = ISO_YD[0].c0;
      fp_set_u64(&a, 216); ISO_YD[1].c0 = z0; fp_neg(&ISO_YD[1].c1, &a);
      fp_set_u64(&ISO_YD[2].c0, 18); fp_set_u64(&a, 18); fp_neg(&ISO_YD[2].c1, &a);
      ISO_YD[3] = F2_ONE; }
}
static void init(void) { pthread_once(&init_once, do_init); }

/* ================================================================================================ API */
static int core_verify(g1_aff *pks, const g2_aff *hs, size_t n, const g2_aff *sig) {
    /* blst Signature::aggregate_verify(sig_groupcheck = true, ...) on decoded inputs */
    if (!sig->inf && !g2_in_group(sig)) return VERIFY_FAIL;
    fp12 acc = F12_ONE, f;
    for (size_t i = 0; i < n; i++) {
        if (pks[i].inf) return VERIFY_FAIL;
        miller_loop(&f, &pks[i], &hs[i]); f12_mul(&acc, &acc, &f);
    }
    miller_loop(&f, &G1_GEN_NEG, sig); f12_mul(&acc, &acc, &f);
    return final_exp_is_one(&acc) ? OK : VERIFY_FAIL;
}

ORC_EXPORT int orc_fast_aggregate_verify(const uint8_t *pks, size_t k, const uint8_t *msg, size_t len, const uint8_t *sig) {
    init();
    g1_jac acc; g1_set_inf(&acc);
    for (size_t i = 0; i < k; i++) {
        g1_aff a; int rc = key_validate(&a, pks + 48 * i);
        if (rc) return rc;
        g1_add_aff(&acc, &acc, &a);
    }
    g2_aff s; int rc = g2_uncompress(&s, sig);
    if (rc) return rc;
    if (k == 0) return VERIFY_FAIL;
    g1_aff agg; g1_to_aff(&agg, &acc);
    g2_aff h; hash_to_g2(&h, msg, len);
    return core_verify(&agg, &h, 1, &s);
}
ORC_EXPORT int orc_verify_signature(const uint8_t *pk, const uint8_t *msg, size_t len, const uint8_t *sig) {
    return orc_fast_aggregate_verify(pk, 1, msg, len, sig);
}
ORC_EXPORT int orc_eth_fast_aggregate_verify(const uint8_t *pks, size_t k, const uint8_t *msg, size_t len, const uint8_t *sig) {
    if (k == 0 && sig[0] == 0xc0 && all_zero(sig + 1, 95)) return OK;
    return orc_fast_aggregate_verify(pks, k, msg, len, sig);
}
ORC_EXPORT int orc_aggregate_verify(const uint8_t *pks, size_t n_pks, const uint8_t *const *msgs, const size_t *lens,
                                    size_t n_msgs, const uint8_t *sig) {
    init();
    g1_aff *a = malloc(sizeof(g1_aff) * (n_pks + 1));
    g2_aff *h = malloc(sizeof(g2_aff) * (n_msgs + 1));
    int rc = OK;
    for (size_t i = 0; i < n_pks && !rc; i++) rc = key_validate(&a[i], pks + 48 * i);
    g2_aff s;
    if (!rc) rc = g2_uncompress(&s, sig);
    if (!rc) {
        if (n_pks == 0 || n_pks != n_msgs) rc = VERIFY_FAIL;
        else { for (size_t i = 0; i < n_msgs; i++) hash_to_g2(&h[i], msgs[i], lens[i]); rc = core_verify(a, h, n_pks, &s); }
    }
    free(a); free(h);
    return rc;
}
ORC_EXPORT int orc_aggregate(const uint8_t *sigs, size_t n, uint8_t out[96]) {
    init();
    if (n == 0) return EMPTY_AGGREGATE;
    g2_aff *a = malloc(sizeof(g2_aff) * n);
    int rc = OK;
    for (size_t i = 0; i < n && !rc; i++) rc = g2_uncompress(&a[i], sigs + 96 * i);
    g2_jac acc; g2_set_inf(&acc);
    for (size_t i = 0; i < n && !rc; i++) { if (!a[i].inf && !g2_in_group(&a[i])) rc = NOT_IN_GROUP; else g2_add_aff(&acc, &acc, &a[i]); }
    if (!rc) { g2_aff r; g2_to_aff(&r, &acc); g2_compress(out, &r); }
    free(a);
    return rc;
}
ORC_EXPORT int orc_eth_aggregate_public_keys(const uint8_t *pks, size_t n, uint8_t out[48]) {
    init();
    if (n == 0) return EMPTY_AGGREGATE;
    g1_jac acc; g1_set_inf(&acc);
    for (size_t i = 0; i < n; i++) { g1_aff a; int rc = key_validate(&a, pks + 48 * i); if (rc) return rc; g1_add_aff(&acc, &acc, &a); }
    g1_aff r; g1_to_aff(&r, &acc); g1_compress(out, &r);
    return OK;
}
ORC_EXPORT int orc_key_validate(const uint8_t *pk) { init(); g1_aff a; return key_validate(&a, pk); }
/* cross-checks of the endomorphism shortcuts against the definition; returns 1 if they agree on this input */
ORC_EXPORT int orc_g1_group_checks_agree(const uint8_t *pk) {
    init(); g1_aff a; if (g1_uncompress(&a, pk) || a.inf) return 1; return g1_in_group(&a) == g1_in_group_def(&a);
}
ORC_EXPORT int orc_g2_group_checks_agree(const uint8_t *sig) {
    init(); g2_aff a; if (g2_uncompress(&a, sig) || a.inf) return 1; return g2_in_group(&a) == g2_in_group_def(&a);
}
ORC_EXPORT void orc_hash_to_g2(const uint8_t *msg, size_t len, uint8_t out192[192]) {
    init(); g2_aff h; hash_to_g2(&h, msg, len);
    fp_to_be(out192, &h.x.c0); fp_to_be(out192 + 48, &h.x.c1); fp_to_be(out192 + 96, &h.y.c0); fp_to_be(out192 + 144, &h.y.c1);
}
static void scalar_from_be32(uint64_t k[4], const uint8_t *b) {
    for (int i = 0; i < 4; i++) { uint64_t v = 0; for (int j = 0; j < 8; j++) v = (v << 8) | b[24 - 8 * i + j]; k[i] = v; }
}
/* SecretKey::public_key / sign (crypto/bls.rs:212-220) — used for KATs and to synthesise benchmark workloads */
ORC_EXPORT void orc_sk_to_pk(const uint8_t sk[32], uint8_t out[48]) {
    init(); uint64_t k[4]; scalar_from_be32(k, sk);
    g1_jac g, r; g1_from_aff(&g, &G1_GEN); g1_mul(&r, &g, k, 4);
    g1_aff a; g1_to_aff(&a, &r); g1_compress(out, &a);
}
ORC_EXPORT void orc_sign(const uint8_t sk[32], const uint8_t *msg, size_t len, uint8_t out[96]) {
    init(); uint64_t k[4]; scalar_from_be32(k, sk);
    g2_aff h; hash_to_g2(&h, msg, len);
    g2_jac hj, r; g2_from_aff(&hj, &h); g2_mul(&r, &hj, k, 4);
    g2_aff a; g2_to_aff(&a, &r); g2_compress(out, &a);
}

/* ---- batch + threads (the reference is single-threaded per call; the all-core variant is "the best the host can do") */
typedef struct { const uint8_t *pks; const uint32_t *off; const uint8_t *msgs; const uint8_t *sigs; int32_t *out; size_t lo, hi; } batch_task;
static void *batch_run(void *p) {
    batch_task *t = p;
    for (size_t i = t->lo; i < t->hi; i++)
        t->out[i] = orc_fast_aggregate_verify(t->pks + 48 * (size_t)t->off[i], t->off[i + 1] - t->off[i], t->msgs + 32 * i, 32, t->sigs + 96 * i);
    return NULL;
}
ORC_EXPORT void orc_fast_aggregate_verify_batch(const uint8_t *pks, const uint32_t *off, const uint8_t *msgs32, const uint8_t *sigs,
                                                size_t n, int32_t *out, int nthreads) {
    init();
    if (nthreads < 1) nthreads = 1;
    if ((size_t)nthreads > n) nthreads = n ? (int)n : 1;
    pthread_t th[256]; batch_task tk[256];
    if (nthreads > 256) nthreads = 256;
    size_t per = (n + nthreads - 1) / nthreads;
    int started = 0;
    for (int i = 0; i < nthreads; i++) {
        size_t lo = i * per, hi = lo + per > n ? n : lo + per;
        if (lo >= hi) break;
        tk[i] = (batch_task){pks, off, msgs32, sigs, out, lo, hi};
        if (nthreads == 1) batch_run(&tk[i]); else { pthread_create(&th[i], NULL, batch_run, &tk[i]); started++; }
    }
    for (int i = 0; i < started; i++) pthread_join(th[i], NULL);
}
/* sign a batch: sig_t = sk_t * H(msg_t), sk_t given as 32 big-endian bytes (already the sum of the signers' keys mod r) */
typedef struct { const uint8_t *sks, *msgs; uint8_t *out; size_t lo, hi; } sign_task;
static void *sign_run(void *p) { sign_task *t = p; for (size_t i = t->lo; i < t->hi; i++) orc_sign(t->sks + 32 * i, t->msgs + 32 * i, 32, t->out + 96 * i); return NULL; }
ORC_EXPORT void orc_sign_batch(const uint8_t *sks32, const uint8_t *msgs32, size_t n, uint8_t *out96, int nthreads) {
    init();
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    pthread_t th[256]; sign_task tk[256];
    size_t per = (n + nthreads - 1) / nthreads;
    int started = 0;
    for (int i = 0; i < nthreads; i++) {
        size_t lo = i * per, hi = lo + per > n ? n : lo + per;
        if (lo >= hi) break;
        tk[i] = (sign_task){sks32, msgs32, out96, lo, hi};
        pthread_create(&th[i], NULL, sign_run, &tk[i]); started++;
    }
    for (int i = 0; i < started; i++) pthread_join(th[i], NULL);
}
/* pk_i = (sk0 + i*delta) * g1 for i < n, by repeated addition + one inversion per key (workload synthesis) */
ORC_EXPORT void orc_pk_sequence(const uint8_t sk0[32], const uint8_t delta[32], size_t n, uint8_t *out48) {
    init(); uint64_t k[4];
    g1_jac g, cur, d; g1_from_aff(&g, &G1_GEN);
    scalar_from_be32(k, sk0); g1_mul(&cur, &g, k, 4);
    scalar_from_be32(k, delta); g1_mul(&d, &g, k, 4);
    g1_aff da; g1_to_aff(&da, &d);
    for (size_t i = 0; i < n; i++) { g1_aff a; g1_to_aff(&a, &cur); g1_compress(out48 + 48 * i, &a); g1_add_aff(&cur, &cur, &da); }
}
