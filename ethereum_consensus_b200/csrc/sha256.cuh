// SHA-256 device primitives for the SSZ Merkle kernels and hash_to_field (sm_90a).
//
// Replaces, on the device, what the reference gets from `sha2 0.10.8` through `ssz_rs` (merkleization,
// ethereum-consensus/src/ssz/mod.rs:4-7) and `crypto::hash`
// (ethereum-consensus/src/crypto/bls.rs:12-20).
//
// Node representation: a 32-byte Merkle node is kept in HBM as 8 big-endian-decoded 32-bit words ("word
// form"), i.e. exactly the SHA-256 state words, so a parent = compress(compress(IV, left||right), PAD) needs
// no byte swaps between levels.  Raw SSZ bytes are swapped once on load (`bswap32`).
//
// Everything is 32-bit integer work on the ALU pipe (LOP3 / SHF / IADD3); no tensor cores.
#pragma once
#include <cstdint>

namespace b200 {

struct Sha256Consts {
    uint32_t k[64];
    uint32_t kw_pad[64];  // K[i] + W_pad[i] for the constant second block of a 64-byte message
};

constexpr uint32_t c_rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

constexpr Sha256Consts make_consts() {
    Sha256Consts c{};
    const uint32_t k[64] = {
        0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
        0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
        0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
        0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
        0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
        0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
        0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
        0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
    uint32_t w[64] = {};
    w[0] = 0x80000000u;
    w[15] = 512;
    for (int i = 16; i < 64; i++) {
        uint32_t s0 = c_rotr(w[i - 15], 7) ^ c_rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
        uint32_t s1 = c_rotr(w[i - 2], 17) ^ c_rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
        w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    for (int i = 0; i < 64; i++) {
        c.k[i] = k[i];
        c.kw_pad[i] = k[i] + w[i];
    }
    return c;
}

// constexpr table: with the round loops fully unrolled every use becomes an immediate operand.
static constexpr Sha256Consts kSha = make_consts();

#if defined(__CUDACC__)
#define B200_DEV __device__ __forceinline__

// device copy of the tables; after unrolling every access is a constant-bank operand of the ALU instruction
static __constant__ Sha256Consts dSha = make_consts();

B200_DEV uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }
B200_DEV uint32_t rotr32(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

#define B200_SHA_ROUND(a, b, c, d, e, f, g, h, kw)                                        \
    {                                                                                     \
        uint32_t t1 = h + (rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25)) + ((e & f) ^ (~e & g)) + (kw); \
        uint32_t t2 = (rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));   \
        d += t1;                                                                          \
        h = t1 + t2;                                                                      \
    }

// One compression of `st` with the 16 message words in w (w is clobbered: rolling schedule).
B200_DEV void sha256_compress(uint32_t st[8], uint32_t w[16]) {
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
    for (int i = 0; i < 64; i += 8) {
        if (i >= 16) {
#pragma unroll
            for (int j = 0; j < 8; j++) {
                int t = (i + j) & 15;
                uint32_t w15 = w[(t + 1) & 15], w2 = w[(t + 14) & 15];
                uint32_t s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
                uint32_t s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
                w[t] = w[t] + s0 + w[(t + 9) & 15] + s1;
            }
        }
        B200_SHA_ROUND(a, b, c, d, e, f, g, h, dSha.k[i + 0] + w[(i + 0) & 15]);
        B200_SHA_ROUND(h, a, b, c, d, e, f, g, dSha.k[i + 1] + w[(i + 1) & 15]);
        B200_SHA_ROUND(g, h, a, b, c, d, e, f, dSha.k[i + 2] + w[(i + 2) & 15]);
        B200_SHA_ROUND(f, g, h, a, b, c, d, e, dSha.k[i + 3] + w[(i + 3) & 15]);
        B200_SHA_ROUND(e, f, g, h, a, b, c, d, dSha.k[i + 4] + w[(i + 4) & 15]);
        B200_SHA_ROUND(d, e, f, g, h, a, b, c, dSha.k[i + 5] + w[(i + 5) & 15]);
        B200_SHA_ROUND(c, d, e, f, g, h, a, b, dSha.k[i + 6] + w[(i + 6) & 15]);
        B200_SHA_ROUND(b, c, d, e, f, g, h, a, dSha.k[i + 7] + w[(i + 7) & 15]);
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// Second block of a 64-byte message: padding only, schedule folded into constants.
B200_DEV void sha256_compress_pad64(uint32_t st[8]) {
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
    for (int i = 0; i < 64; i += 8) {
        B200_SHA_ROUND(a, b, c, d, e, f, g, h, dSha.kw_pad[i + 0]);
        B200_SHA_ROUND(h, a, b, c, d, e, f, g, dSha.kw_pad[i + 1]);
        B200_SHA_ROUND(g, h, a, b, c, d, e, f, dSha.kw_pad[i + 2]);
        B200_SHA_ROUND(f, g, h, a, b, c, d, e, dSha.kw_pad[i + 3]);
        B200_SHA_ROUND(e, f, g, h, a, b, c, d, dSha.kw_pad[i + 4]);
        B200_SHA_ROUND(d, e, f, g, h, a, b, c, dSha.kw_pad[i + 5]);
        B200_SHA_ROUND(c, d, e, f, g, h, a, b, dSha.kw_pad[i + 6]);
        B200_SHA_ROUND(b, c, d, e, f, g, h, a, dSha.kw_pad[i + 7]);
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

B200_DEV void sha256_init(uint32_t st[8]) {
    st[0] = 0x6a09e667u; st[1] = 0xbb67ae85u; st[2] = 0x3c6ef372u; st[3] = 0xa54ff53au;
    st[4] = 0x510e527fu; st[5] = 0x9b05688cu; st[6] = 0x1f83d9abu; st[7] = 0x5be0cd19u;
}

// out = SHA-256(m[0..16)) for a 64-byte message given as 16 big-endian-decoded words (m clobbered).
B200_DEV void sha256_msg64(uint32_t m[16], uint32_t out[8]) {
    sha256_init(out);
    sha256_compress(out, m);
    sha256_compress_pad64(out);
}

// parent = H(left || right), all in word form.
B200_DEV void hash_pair_words(const uint32_t l[8], const uint32_t r[8], uint32_t out[8]) {
    uint32_t m[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { m[i] = l[i]; m[8 + i] = r[i]; }
    sha256_msg64(m, out);
}
#endif  // __CUDACC__

}  // namespace b200
