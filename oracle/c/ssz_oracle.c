/*
 * SSZ / SHA-256 Merkle oracle in plain C.  TEST INFRASTRUCTURE — only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may link or load this.  The product path never does.
 *
 * Restates, for the CPU, the merkleization the reference gets from the un-vendored `ssz_rs @ 84ef2b71`
 * (Cargo.toml:20; surface re-exported at ethereum-consensus/src/ssz/mod.rs:4-7)
 * and the one-shot SHA-256 of ethereum-consensus/src/crypto/bls.rs:12-20 (sha2 0.10.8, which
 * dispatches to SHA-NI at run time — so does this file).  Container shapes:
 *   deneb::BeaconState   ethereum-consensus/src/deneb/beacon_state.rs:13-64
 *   Validator            ethereum-consensus/src/phase0/validator.rs:10-26
 * Validated against oracle/ssz_oracle.py (hashlib) and the reference KAT B-3 in tests/test_oracle_ssz.py.
 */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <cpuid.h>
#include <immintrin.h>

#define ORC_EXPORT __attribute__((visibility("default")))

/* ------------------------------------------------------------------ SHA-256 (portable) */
static const uint32_t K256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
static const uint32_t H256[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a,
                                 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};

static inline uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
static inline uint32_t be32(const uint8_t *p) {
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
static inline void put_be32(uint8_t *p, uint32_t v) { p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v; }

static void compress_portable(uint32_t st[8], const uint8_t blk[64]) {
    uint32_t w[64], a, b, c, d, e, f, g, h;
    for (int i = 0; i < 16; i++) w[i] = be32(blk + 4 * i);
    for (int i = 16; i < 64; i++) {
        uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
        uint32_t s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
        w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    a = st[0]; b = st[1]; c = st[2]; d = st[3]; e = st[4]; f = st[5]; g = st[6]; h = st[7];
    for (int i = 0; i < 64; i++) {
        uint32_t t1 = h + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + K256[i] + w[i];
        uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

/* ------------------------------------------------------------------ SHA-256 (SHA-NI) */
__attribute__((target("sha,sse4.1,ssse3")))
static void compress_shani(uint32_t state[8], const uint8_t *data) {
    __m128i STATE0, STATE1, MSG, TMP, MSG0, MSG1, MSG2, MSG3, ABEF_SAVE, CDGH_SAVE;
    const __m128i MASK = _mm_set_epi64x(0x0c0d0e0f08090a0bULL, 0x0405060700010203ULL);
    TMP = _mm_loadu_si128((const __m128i *)&state[0]);
    STATE1 = _mm_loadu_si128((const __m128i *)&state[4]);
    TMP = _mm_shuffle_epi32(TMP, 0xB1);
    STATE1 = _mm_shuffle_epi32(STATE1, 0x1B);
    STATE0 = _mm_alignr_epi8(TMP, STATE1, 8);
    STATE1 = _mm_blend_epi16(STATE1, TMP, 0xF0);
    ABEF_SAVE = STATE0; CDGH_SAVE = STATE1;
#define RND4(Ma, i)                                                                          \
    MSG = _mm_add_epi32(Ma, _mm_loadu_si128((const __m128i *)&K256[4 * (i)]));                \
    STATE1 = _mm_sha256rnds2_epu32(STATE1, STATE0, MSG);                                      \
    MSG = _mm_shuffle_epi32(MSG, 0x0E);                                                       \
    STATE0 = _mm_sha256rnds2_epu32(STATE0, STATE1, MSG);
    MSG0 = _mm_shuffle_epi8(_mm_loadu_si128((const __m128i *)(data + 0)), MASK);
    MSG1 = _mm_shuffle_epi8(_mm_loadu_si128((const __m128i *)(data + 16)), MASK);
    MSG2 = _mm_shuffle_epi8(_mm_loadu_si128((const __m128i *)(data + 32)), MASK);
    MSG3 = _mm_shuffle_epi8(_mm_loadu_si128((const __m128i *)(data + 48)), MASK);
    RND4(MSG0, 0); RND4(MSG1, 1); RND4(MSG2, 2); RND4(MSG3, 3);
    for (int i = 4; i < 16; i++) {
        /* W[4i..4i+3] from the previous four quads */
        __m128i t = _mm_sha256msg1_epu32(MSG0, MSG1);
        t = _mm_add_epi32(t, _mm_alignr_epi8(MSG3, MSG2, 4));
        t = _mm_sha256msg2_epu32(t, MSG3);
        MSG0 = MSG1; MSG1 = MSG2; MSG2 = MSG3; MSG3 = t;
        RND4(MSG3, i);
    }
#undef RND4
    STATE0 = _mm_add_epi32(STATE0, ABEF_SAVE);
    STATE1 = _mm_add_epi32(STATE1, CDGH_SAVE);
    TMP = _mm_shuffle_epi32(STATE0, 0x1B);
    STATE1 = _mm_shuffle_epi32(STATE1, 0xB1);
    STATE0 = _mm_blend_epi16(TMP, STATE1, 0xF0);
    STATE1 = _mm_alignr_epi8(STATE1, TMP, 8);
    _mm_storeu_si128((__m128i *)&state[0], STATE0);
    _mm_storeu_si128((__m128i *)&state[4], STATE1);
}

static int g_have_shani = -1;
static int g_force_portable = 0;
static int have_shani(void) {
    if (g_have_shani < 0) {
        unsigned a, b, c, d;
        g_have_shani = 0;
        if (__get_cpuid_count(7, 0, &a, &b, &c, &d)) g_have_shani = (b >> 29) & 1;
    }
    return g_have_shani && !g_force_portable;
}
ORC_EXPORT int orc_sha_backend(void) { return have_shani(); }
ORC_EXPORT void orc_force_portable(int on) { g_force_portable = on; }

static inline void compress(uint32_t st[8], const uint8_t blk[64]) {
    if (have_shani()) compress_shani(st, blk); else compress_portable(st, blk);
}

ORC_EXPORT void orc_sha256(const uint8_t *data, size_t len, uint8_t out[32]) {
    uint32_t st[8];
    uint8_t blk[128];
    memcpy(st, H256, sizeof st);
    size_t n = len;
    while (n >= 64) { compress(st, data); data += 64; n -= 64; }
    memset(blk, 0, sizeof blk);
    memcpy(blk, data, n);
    blk[n] = 0x80;
    size_t tot = (n + 9 <= 64) ? 64 : 128;
    uint64_t bits = (uint64_t)len * 8;
    for (int i = 0; i < 8; i++) blk[tot - 1 - i] = (uint8_t)(bits >> (8 * i));
    compress(st, blk);
    if (tot == 128) compress(st, blk + 64);
    for (int i = 0; i < 8; i++) put_be32(out + 4 * i, st[i]);
}

static const uint8_t PAD64[64] = {0x80, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                  0,    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                  0,    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 0};

/* sha256 of exactly 64 bytes (one Merkle pair) */
static inline void hash64(const uint8_t in[64], uint8_t out[32]) {
    uint32_t st[8];
    memcpy(st, H256, sizeof st);
    compress(st, in);
    compress(st, PAD64);
    for (int i = 0; i < 8; i++) put_be32(out + 4 * i, st[i]);
}
ORC_EXPORT void orc_hash_pair(const uint8_t a[32], const uint8_t b[32], uint8_t out[32]) {
    uint8_t buf[64];
    memcpy(buf, a, 32); memcpy(buf + 32, b, 32);
    hash64(buf, out);
}

/* ------------------------------------------------------------------ zero hashes */
static uint8_t ZERO[65][32];
static pthread_once_t zero_once = PTHREAD_ONCE_INIT;
static void zero_init(void) {
    memset(ZERO[0], 0, 32);
    for (int i = 0; i < 64; i++) orc_hash_pair(ZERO[i], ZERO[i], ZERO[i + 1]);
}
ORC_EXPORT void orc_zero_hash(int depth, uint8_t out[32]) {
    pthread_once(&zero_once, zero_init);
    memcpy(out, ZERO[depth], 32);
}
static int depth_for(uint64_t n) { int d = 0; while (((uint64_t)1 << d) < n) d++; return d; }

/* ------------------------------------------------------------------ tiny parallel-for */
typedef void (*range_fn)(void *ctx, size_t lo, size_t hi);
typedef struct { range_fn fn; void *ctx; size_t lo, hi; } pf_task;
static void *pf_run(void *p) { pf_task *t = p; t->fn(t->ctx, t->lo, t->hi); return NULL; }
static void parallel_for(size_t n, int nthreads, size_t grain, range_fn fn, void *ctx) {
    if (nthreads <= 1 || n < 2 * grain) { fn(ctx, 0, n); return; }
    if ((size_t)nthreads > n / grain) nthreads = (int)(n / grain);
    pthread_t th[256]; pf_task tk[256];
    if (nthreads > 256) nthreads = 256;
    size_t per = (n + nthreads - 1) / nthreads;
    int started = 0;
    for (int i = 0; i < nthreads; i++) {
        size_t lo = i * per, hi = lo + per > n ? n : lo + per;
        if (lo >= hi) break;
        tk[i] = (pf_task){fn, ctx, lo, hi};
        pthread_create(&th[i], NULL, pf_run, &tk[i]);
        started++;
    }
    for (int i = 0; i < started; i++) pthread_join(th[i], NULL);
}

/* ------------------------------------------------------------------ merkleize */
typedef struct { const uint8_t *in; uint8_t *out; } level_ctx;
static void level_range(void *c, size_t lo, size_t hi) {
    level_ctx *x = c;
    for (size_t i = lo; i < hi; i++) hash64(x->in + 64 * i, x->out + 32 * i);
}

/* Root of `n` 32-byte chunks in `buf` (clobbered; needs room for n+1 chunks), virtually padded to `limit`
 * chunks (limit==0: next pow2 of n). */
static int merkleize_inplace(uint8_t *buf, size_t n, uint64_t limit, int nthreads, uint8_t out[32]) {
    pthread_once(&zero_once, zero_init);
    if (limit == 0) limit = n ? n : 1;
    if (n > limit) return -1;
    int depth = depth_for(limit);
    if (n == 0) { memcpy(out, ZERO[depth], 32); return 0; }
    for (int d = 0; d < depth; d++) {
        if (n & 1) { memcpy(buf + 32 * n, ZERO[d], 32); n++; }
        level_ctx c = {buf, buf};
        if (nthreads > 1 && n >= 4096) {
            /* out-of-place halves are safe in place only sequentially; use a temp for the parallel case */
            uint8_t *tmp = malloc(16 * n + 32);
            c.out = tmp;
            parallel_for(n / 2, nthreads, 1024, level_range, &c);
            memcpy(buf, tmp, 16 * n);
            free(tmp);
        } else {
            level_range(&c, 0, n / 2); /* in-place: out[i] written after in[2i],in[2i+1] are consumed */
        }
        n /= 2;
    }
    memcpy(out, buf, 32);
    return 0;
}

ORC_EXPORT int orc_merkleize(const uint8_t *chunks, size_t n, uint64_t limit, int nthreads, uint8_t out[32]) {
    uint8_t *buf = malloc(32 * (n + 2));
    if (!buf) return -2;
    memcpy(buf, chunks, 32 * n);
    int rc = merkleize_inplace(buf, n, limit, nthreads, out);
    free(buf);
    return rc;
}

ORC_EXPORT void orc_mix_in_length(const uint8_t root[32], uint64_t len, uint8_t out[32]) {
    uint8_t l[32] = {0};
    for (int i = 0; i < 8; i++) l[i] = (uint8_t)(len >> (8 * i));
    orc_hash_pair(root, l, out);
}

/* packed basic list/vector: `nbytes` of little-endian data -> chunks; limit in chunks; mixes length if is_list */
ORC_EXPORT int orc_htr_packed(const uint8_t *data, size_t nbytes, uint64_t limit_chunks, int is_list,
                              uint64_t length, int nthreads, uint8_t out[32]) {
    size_t n = (nbytes + 31) / 32;
    uint8_t *buf = calloc(n + 2, 32);
    if (!buf) return -2;
    memcpy(buf, data, nbytes);
    int rc = merkleize_inplace(buf, n, limit_chunks, nthreads, out);
    free(buf);
    if (rc) return rc;
    if (is_list) orc_mix_in_length(out, length, out);
    return 0;
}

/* ------------------------------------------------------------------ Validator (121 bytes) */
static void validator_root(const uint8_t *v, uint8_t out[32]) {
    uint8_t leaf[8][32];
    uint8_t blk[64];
    memset(leaf, 0, sizeof leaf);
    memcpy(blk, v, 48); memset(blk + 48, 0, 16);
    hash64(blk, leaf[0]);                 /* pubkey: 2 chunks */
    memcpy(leaf[1], v + 48, 32);          /* withdrawal_credentials */
    memcpy(leaf[2], v + 80, 8);           /* effective_balance */
    leaf[3][0] = v[88];                   /* slashed */
    memcpy(leaf[4], v + 89, 8);
    memcpy(leaf[5], v + 97, 8);
    memcpy(leaf[6], v + 105, 8);
    memcpy(leaf[7], v + 113, 8);
    uint8_t l1[4][32], l2[2][32];
    /* adjacent 32-byte rows are one contiguous 64-byte block */
    for (int i = 0; i < 4; i++) hash64((const uint8_t *)leaf + 64 * i, l1[i]);
    for (int i = 0; i < 2; i++) hash64((const uint8_t *)l1 + 64 * i, l2[i]);
    hash64((const uint8_t *)l2, out);
}
typedef struct { const uint8_t *in; uint8_t *out; size_t stride; int kind; } elem_ctx;
static void elem_range(void *c, size_t lo, size_t hi) {
    elem_ctx *x = c;
    uint8_t blk[64];
    for (size_t i = lo; i < hi; i++) {
        const uint8_t *p = x->in + x->stride * i;
        switch (x->kind) {
        case 0: validator_root(p, x->out + 32 * i); break;
        case 1: memcpy(blk, p, 48); memset(blk + 48, 0, 16); hash64(blk, x->out + 32 * i); break; /* pubkey */
        case 2: hash64(p, x->out + 32 * i); break;                 /* 64-byte, two-chunk container */
        case 3: {                                                  /* Eth1Data: root,u64,root */
            uint8_t l[4][32], m[2][32];
            memset(l, 0, sizeof l);
            memcpy(l[0], p, 32); memcpy(l[1], p + 32, 8); memcpy(l[2], p + 40, 32);
            hash64((const uint8_t *)l, m[0]); hash64((const uint8_t *)l + 64, m[1]);
            orc_hash_pair(m[0], m[1], x->out + 32 * i);
        } break;
        }
    }
}
ORC_EXPORT void orc_validator_root(const uint8_t v[121], uint8_t out[32]) { validator_root(v, out); }

/* List/Vector of composite elements: kind 0 Validator(121) 1 pubkey(48) 2 pair(64) 3 Eth1Data(72) */
static int htr_elems(const uint8_t *data, size_t n, size_t stride, int kind, uint64_t limit, int is_list,
                     int nthreads, uint8_t out[32]) {
    uint8_t *roots = malloc(32 * (n + 2));
    if (!roots) return -2;
    elem_ctx c = {data, roots, stride, kind};
    parallel_for(n, nthreads, 256, elem_range, &c);
    int rc = merkleize_inplace(roots, n, limit, nthreads, out);
    free(roots);
    if (rc) return rc;
    if (is_list) orc_mix_in_length(out, n, out);
    return 0;
}
ORC_EXPORT int orc_htr_validators(const uint8_t *ssz, size_t n, uint64_t limit, int nthreads, uint8_t out[32]) {
    return htr_elems(ssz, n, 121, 0, limit, 1, nthreads, out);
}

/* ------------------------------------------------------------------ deneb BeaconState from SSZ bytes */
typedef struct {
    uint64_t slots_per_historical_root, historical_roots_limit, eth1_data_votes_bound, validator_registry_limit,
        epochs_per_historical_vector, epochs_per_slashings_vector, sync_committee_size;
} preset_t;
static const preset_t PRESET[2] = {
    {8192, 1ull << 24, 2048, 1ull << 40, 65536, 8192, 512}, /* mainnet */
    {64, 1ull << 24, 32, 1ull << 40, 64, 64, 32},           /* minimal */
};
static uint32_t le32(const uint8_t *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
static void chunk_u64(const uint8_t *p, uint8_t out[32]) { memset(out, 0, 32); memcpy(out, p, 8); }

static int small_container(uint8_t (*leaves)[32], size_t n, uint8_t out[32]) {
    uint8_t buf[40][32];
    memcpy(buf, leaves, 32 * n);
    return merkleize_inplace(&buf[0][0], n, 0, 1, out);
}

static int htr_sync_committee(const uint8_t *p, uint64_t size, int nthreads, uint8_t out[32]) {
    uint8_t l[2][32], blk[64];
    int rc = htr_elems(p, size, 48, 1, size, 0, nthreads, l[0]);
    if (rc) return rc;
    memcpy(blk, p + 48 * size, 48); memset(blk + 48, 0, 16);
    hash64(blk, l[1]);
    orc_hash_pair(l[0], l[1], out);
    return 0;
}

static int htr_payload_header(const uint8_t *p, size_t len, uint8_t out[32]) {
    /* fixed part: 32+20+32+32+256+32+8*4+4(offset)+32+32+32+32+8+8 = 584 */
    if (len < 584) return -3;
    uint8_t l[17][32];
    memset(l, 0, sizeof l);
    size_t o = 0;
    memcpy(l[0], p + o, 32); o += 32;       /* parent_hash */
    memcpy(l[1], p + o, 20); o += 20;       /* fee_recipient */
    memcpy(l[2], p + o, 32); o += 32;       /* state_root */
    memcpy(l[3], p + o, 32); o += 32;       /* receipts_root */
    { uint8_t b[9 * 32]; memcpy(b, p + o, 256); merkleize_inplace(b, 8, 8, 1, l[4]); o += 256; }
    memcpy(l[5], p + o, 32); o += 32;       /* prev_randao */
    for (int i = 0; i < 4; i++) { memcpy(l[6 + i], p + o, 8); o += 8; }
    uint32_t off = le32(p + o); o += 4;
    if (off != 584 || len - off > 32) return -3;
    { uint8_t b[2 * 32]; memset(b, 0, sizeof b); memcpy(b, p + off, len - off);
      uint8_t r[32]; merkleize_inplace(b, (len - off + 31) / 32, 1, 1, r); orc_mix_in_length(r, len - off, l[10]); }
    memcpy(l[11], p + o, 32); o += 32;      /* base_fee_per_gas (U256 LE) */
    memcpy(l[12], p + o, 32); o += 32;      /* block_hash */
    memcpy(l[13], p + o, 32); o += 32;      /* transactions_root */
    memcpy(l[14], p + o, 32); o += 32;      /* withdrawals_root */
    memcpy(l[15], p + o, 8); o += 8;
    memcpy(l[16], p + o, 8); o += 8;
    return small_container(l, 17, out);
}

ORC_EXPORT int orc_htr_beacon_state_deneb(const uint8_t *s, size_t len, int preset, int nthreads, uint8_t out[32]) {
    if (preset < 0 || preset > 1) return -1;
    const preset_t *P = &PRESET[preset];
    uint8_t f[28][32];
    memset(f, 0, sizeof f);
    size_t o = 0;
    uint32_t off_hist_roots, off_votes, off_validators, off_balances, off_prev, off_cur, off_inact, off_header,
        off_summaries;
    size_t fixed = 8 + 32 + 8 + 16 + 112 + 2 * 32 * P->slots_per_historical_root + 4 + 72 + 4 + 8 + 4 + 4 +
                   32 * P->epochs_per_historical_vector + 8 * P->epochs_per_slashings_vector + 4 + 4 + 1 + 3 * 40 + 4 +
                   2 * (48 * P->sync_committee_size + 48) + 4 + 8 + 8 + 4;
    if (len < fixed) return -3;
    chunk_u64(s + o, f[0]); o += 8;
    memcpy(f[1], s + o, 32); o += 32;
    chunk_u64(s + o, f[2]); o += 8;
    { uint8_t l[3][32]; memset(l, 0, sizeof l); memcpy(l[0], s + o, 4); memcpy(l[1], s + o + 4, 4);
      memcpy(l[2], s + o + 8, 8); small_container(l, 3, f[3]); o += 16; }
    { uint8_t l[5][32]; memset(l, 0, sizeof l); memcpy(l[0], s + o, 8); memcpy(l[1], s + o + 8, 8);
      memcpy(l[2], s + o + 16, 32); memcpy(l[3], s + o + 48, 32); memcpy(l[4], s + o + 80, 32);
      small_container(l, 5, f[4]); o += 112; }
    orc_merkleize(s + o, P->slots_per_historical_root, P->slots_per_historical_root, nthreads, f[5]);
    o += 32 * P->slots_per_historical_root;
    orc_merkleize(s + o, P->slots_per_historical_root, P->slots_per_historical_root, nthreads, f[6]);
    o += 32 * P->slots_per_historical_root;
    off_hist_roots = le32(s + o); o += 4;
    { elem_ctx c = {s + o, f[8], 72, 3}; elem_range(&c, 0, 1); o += 72; }
    off_votes = le32(s + o); o += 4;
    chunk_u64(s + o, f[10]); o += 8;
    off_validators = le32(s + o); o += 4;
    off_balances = le32(s + o); o += 4;
    orc_merkleize(s + o, P->epochs_per_historical_vector, P->epochs_per_historical_vector, nthreads, f[13]);
    o += 32 * P->epochs_per_historical_vector;
    orc_htr_packed(s + o, 8 * P->epochs_per_slashings_vector, P->epochs_per_slashings_vector / 4, 0, 0, nthreads, f[14]);
    o += 8 * P->epochs_per_slashings_vector;
    off_prev = le32(s + o); o += 4;
    off_cur = le32(s + o); o += 4;
    f[17][0] = s[o]; o += 1;
    for (int i = 0; i < 3; i++) {
        uint8_t l[2][32]; memset(l, 0, sizeof l); memcpy(l[0], s + o, 8); memcpy(l[1], s + o + 8, 32);
        orc_hash_pair(l[0], l[1], f[18 + i]); o += 40;
    }
    off_inact = le32(s + o); o += 4;
    htr_sync_committee(s + o, P->sync_committee_size, nthreads, f[22]); o += 48 * P->sync_committee_size + 48;
    htr_sync_committee(s + o, P->sync_committee_size, nthreads, f[23]); o += 48 * P->sync_committee_size + 48;
    off_header = le32(s + o); o += 4;
    chunk_u64(s + o, f[25]); o += 8;
    chunk_u64(s + o, f[26]); o += 8;
    off_summaries = le32(s + o); o += 4;
    if (o != fixed) return -4;
    /* variable part: offsets must be ascending and in range */
    uint32_t offs[10] = {off_hist_roots, off_votes, off_validators, off_balances, off_prev, off_cur, off_inact,
                         off_header, off_summaries, (uint32_t)len};
    if (len > 0xffffffffu || offs[0] != fixed) return -3;
    for (int i = 0; i < 9; i++) if (offs[i] > offs[i + 1]) return -3;
    size_t n;
    /* historical_roots */
    n = offs[1] - offs[0]; if (n % 32) return -3;
    if (orc_merkleize(s + offs[0], n / 32, P->historical_roots_limit, nthreads, f[7])) return -3;
    orc_mix_in_length(f[7], n / 32, f[7]);
    /* eth1_data_votes */
    n = offs[2] - offs[1]; if (n % 72 || n / 72 > P->eth1_data_votes_bound) return -3;
    if (htr_elems(s + offs[1], n / 72, 72, 3, P->eth1_data_votes_bound, 1, nthreads, f[9])) return -3;
    /* validators */
    n = offs[3] - offs[2]; if (n % 121) return -3;
    size_t nval = n / 121;
    if (htr_elems(s + offs[2], nval, 121, 0, P->validator_registry_limit, 1, nthreads, f[11])) return -3;
    /* balances */
    n = offs[4] - offs[3]; if (n % 8) return -3;
    if (orc_htr_packed(s + offs[3], n, P->validator_registry_limit / 4, 1, n / 8, nthreads, f[12])) return -3;
    /* participation */
    n = offs[5] - offs[4];
    if (orc_htr_packed(s + offs[4], n, P->validator_registry_limit / 32, 1, n, nthreads, f[15])) return -3;
    n = offs[6] - offs[5];
    if (orc_htr_packed(s + offs[5], n, P->validator_registry_limit / 32, 1, n, nthreads, f[16])) return -3;
    /* inactivity_scores */
    n = offs[7] - offs[6]; if (n % 8) return -3;
    if (orc_htr_packed(s + offs[6], n, P->validator_registry_limit / 4, 1, n / 8, nthreads, f[21])) return -3;
    /* latest_execution_payload_header */
    if (htr_payload_header(s + offs[7], offs[8] - offs[7], f[24])) return -3;
    /* historical_summaries */
    n = offs[9] - offs[8]; if (n % 64) return -3;
    if (htr_elems(s + offs[8], n / 64, 64, 2, P->historical_roots_limit, 1, nthreads, f[27])) return -3;
    return small_container(f, 28, out);
}

/* bulk pair hashing: out[i] = sha256(in[64i..64i+64)) — used to time raw SHA-256 throughput on the host */
ORC_EXPORT void orc_hash_pairs(const uint8_t *in, size_t n, int nthreads, uint8_t *out) {
    level_ctx c = {in, out};
    parallel_for(n, nthreads, 1024, level_range, &c);
}
