// Fp: the BLS12-381 base field, 381-bit, 12 x 32-bit limbs kept in registers, Montgomery form (R = 2^384).
//
// This is the arithmetic blst implements in x86-64 assembly for the reference
// (ethereum-consensus/src/crypto/bls.rs:4 `use blst::{min_pk as bls_impl, ..}`), re-designed for
// the GPU integer pipe: a Montgomery product is 2 x 12 x 12 32x32->64 multiply-adds (IMAD.WIDE on the fma
// pipe) plus carry propagation on the ALU pipe.  No tensor cores: this is modular integer arithmetic.
//
// The same source compiles for the host (`B200_HD` = inline) so that every layer above Fp (towers, curves,
// pairing, hash-to-curve) is unit-tested on the CPU against the big-int oracle before it ever runs on a GPU;
// the host build exists only inside tests/host_math — the product library launches kernels, nothing else.
#pragma once
#include <cstdint>

#include "bls_consts.cuh"

#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#define B200_HD_NOINLINE static __host__ __device__ __noinline__
#else
#define B200_HD inline
#define B200_HD_NOINLINE static inline
#endif
// B200_BIG: tower / curve-level routines.  Inlined in the wide per-key kernels (limbs stay in registers); real
// functions (operands in local memory) in the low-parallelism pairing kernels, which keeps their code size and
// ptxas time bounded.
#if defined(B200_TOWER_NOINLINE)
#define B200_BIG B200_HD_NOINLINE
#else
#define B200_BIG B200_HD
#endif

namespace b200 {

struct Fp {
    uint32_t l[12];
};

B200_HD Fp fp_p() { Fp r = B200_FP_P; return r; }
B200_HD Fp fp_zero() { Fp r = B200_FP_ZERO; return r; }
B200_HD Fp fp_one() { Fp r = B200_FP_ONE; return r; }

B200_HD bool fp_is_zero(const Fp& a) {
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) acc |= a.l[i];
    return acc == 0;
}
B200_HD bool fp_eq(const Fp& a, const Fp& b) {
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) acc |= a.l[i] ^ b.l[i];
    return acc == 0;
}
// a >= b as 384-bit integers
B200_HD bool fp_geq_raw(const Fp& a, const Fp& b) {
    uint64_t borrow = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) {
        uint64_t d = uint64_t(a.l[i]) - b.l[i] - borrow;
        borrow = (d >> 32) & 1;
    }
    return borrow == 0;
}
// Raw 384-bit add / subtract.  On the device: hardware carry chains (add.cc / addc.cc -> one IADD3.X per limb); the
// portable 64-bit emulation below compiles to THREE dependent instructions per limb (IADD3 + IADD3.X + LOP3, several of them
// IMAD.X / IMAD.IADD on the FMA pipe the products need), which made a plain Fp2 addition ~150 SASS instructions in the
// pairing VM's light rounds.  The emulation stays the host's code and the device self-test's reference.  Outputs may
// alias inputs: asm operands are distinct PTX virtual registers.
B200_HD uint32_t fp_sub_raw_portable(Fp& r, const Fp& a, const Fp& b) {
    uint64_t borrow = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) {
        uint64_t d = uint64_t(a.l[i]) - b.l[i] - borrow;
        r.l[i] = uint32_t(d);
        borrow = (d >> 32) & 1;
    }
    return uint32_t(borrow);
}
B200_HD uint32_t fp_add_raw_portable(Fp& r, const Fp& a, const Fp& b) {
    uint64_t carry = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) {
        uint64_t s = uint64_t(a.l[i]) + b.l[i] + carry;
        r.l[i] = uint32_t(s);
        carry = s >> 32;
    }
    return uint32_t(carry);
}
#if defined(__CUDA_ARCH__)
// r = a - b (mod 2^384), returns the borrow (0 / 1)
__device__ __forceinline__ uint32_t fp_sub_raw(Fp& r, const Fp& a, const Fp& b) {
    uint32_t c;
    asm("sub.cc.u32 %0, %13, %25;\n\t"
        "subc.cc.u32 %1, %14, %26;\n\t"
        "subc.cc.u32 %2, %15, %27;\n\t"
        "subc.cc.u32 %3, %16, %28;\n\t"
        "subc.cc.u32 %4, %17, %29;\n\t"
        "subc.cc.u32 %5, %18, %30;\n\t"
        "subc.cc.u32 %6, %19, %31;\n\t"
        "subc.cc.u32 %7, %20, %32;\n\t"
        "subc.cc.u32 %8, %21, %33;\n\t"
        "subc.cc.u32 %9, %22, %34;\n\t"
        "subc.cc.u32 %10, %23, %35;\n\t"
        "subc.cc.u32 %11, %24, %36;\n\t"
        "subc.u32 %12, 0, 0;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7]), "=r"(r.l[8]), "=r"(r.l[9]), "=r"(r.l[10]), "=r"(r.l[11]), "=r"(c)
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]), "r"(a.l[8]), "r"(a.l[9]), "r"(a.l[10]), "r"(a.l[11]), "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]), "r"(b.l[8]), "r"(b.l[9]), "r"(b.l[10]), "r"(b.l[11]));
    return c & 1u;   // 0 - 0 - borrow
}
// r = a + b (mod 2^384), returns the carry
__device__ __forceinline__ uint32_t fp_add_raw(Fp& r, const Fp& a, const Fp& b) {
    uint32_t c;
    asm("add.cc.u32 %0, %13, %25;\n\t"
        "addc.cc.u32 %1, %14, %26;\n\t"
        "addc.cc.u32 %2, %15, %27;\n\t"
        "addc.cc.u32 %3, %16, %28;\n\t"
        "addc.cc.u32 %4, %17, %29;\n\t"
        "addc.cc.u32 %5, %18, %30;\n\t"
        "addc.cc.u32 %6, %19, %31;\n\t"
        "addc.cc.u32 %7, %20, %32;\n\t"
        "addc.cc.u32 %8, %21, %33;\n\t"
        "addc.cc.u32 %9, %22, %34;\n\t"
        "addc.cc.u32 %10, %23, %35;\n\t"
        "addc.cc.u32 %11, %24, %36;\n\t"
        "addc.u32 %12, 0, 0;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7]), "=r"(r.l[8]), "=r"(r.l[9]), "=r"(r.l[10]), "=r"(r.l[11]), "=r"(c)
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]), "r"(a.l[8]), "r"(a.l[9]), "r"(a.l[10]), "r"(a.l[11]), "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]), "r"(b.l[8]), "r"(b.l[9]), "r"(b.l[10]), "r"(b.l[11]));
    return c;
}
// r = a + (m & mask) (mod 2^384), mask = 0 or 0xffffffff: the branch-free "add the modulus back after a borrow"
__device__ __forceinline__ void fp_add_masked_raw(Fp& r, const Fp& a, const Fp& m, uint32_t mask) {
    asm("{\n\t"
        ".reg .u32 m<12>;\n\t"
        "and.b32 m0, %24, %36;\n\t"
        "and.b32 m1, %25, %36;\n\t"
        "and.b32 m2, %26, %36;\n\t"
        "and.b32 m3, %27, %36;\n\t"
        "and.b32 m4, %28, %36;\n\t"
        "and.b32 m5, %29, %36;\n\t"
        "and.b32 m6, %30, %36;\n\t"
        "and.b32 m7, %31, %36;\n\t"
        "and.b32 m8, %32, %36;\n\t"
        "and.b32 m9, %33, %36;\n\t"
        "and.b32 m10, %34, %36;\n\t"
        "and.b32 m11, %35, %36;\n\t"
        "add.cc.u32 %0, %12, m0;\n\t"
        "addc.cc.u32 %1, %13, m1;\n\t"
        "addc.cc.u32 %2, %14, m2;\n\t"
        "addc.cc.u32 %3, %15, m3;\n\t"
        "addc.cc.u32 %4, %16, m4;\n\t"
        "addc.cc.u32 %5, %17, m5;\n\t"
        "addc.cc.u32 %6, %18, m6;\n\t"
        "addc.cc.u32 %7, %19, m7;\n\t"
        "addc.cc.u32 %8, %20, m8;\n\t"
        "addc.cc.u32 %9, %21, m9;\n\t"
        "addc.cc.u32 %10, %22, m10;\n\t"
        "addc.u32 %11, %23, m11;\n\t"
        "}"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7]), "=r"(r.l[8]), "=r"(r.l[9]), "=r"(r.l[10]), "=r"(r.l[11])
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]), "r"(a.l[8]), "r"(a.l[9]), "r"(a.l[10]), "r"(a.l[11]), "r"(m.l[0]), "r"(m.l[1]), "r"(m.l[2]), "r"(m.l[3]), "r"(m.l[4]), "r"(m.l[5]), "r"(m.l[6]), "r"(m.l[7]), "r"(m.l[8]), "r"(m.l[9]), "r"(m.l[10]), "r"(m.l[11]), "r"(mask));
}
#else
B200_HD uint32_t fp_sub_raw(Fp& r, const Fp& a, const Fp& b) { return fp_sub_raw_portable(r, a, b); }
B200_HD uint32_t fp_add_raw(Fp& r, const Fp& a, const Fp& b) { return fp_add_raw_portable(r, a, b); }
B200_HD void fp_add_masked_raw(Fp& r, const Fp& a, const Fp& m, uint32_t mask) {
    Fp t;
#pragma unroll
    for (int i = 0; i < 12; i++) t.l[i] = m.l[i] & mask;
    fp_add_raw_portable(r, a, t);
}
#endif
// select without a branch: r = take_t ? t : r
B200_HD void fp_select(Fp& r, const Fp& t, bool take_t) {
#pragma unroll
    for (int i = 0; i < 12; i++) r.l[i] = take_t ? t.l[i] : r.l[i];
}
// conditional final subtraction: r in [0, 2p) -> [0, p)
B200_HD void fp_reduce_once(Fp& r) {
    const Fp p = fp_p();
    Fp t;
    uint32_t borrow = fp_sub_raw(t, r, p);
    fp_select(r, t, borrow == 0);
}
B200_HD void fp_add(Fp& r, const Fp& a, const Fp& b) {
    fp_add_raw(r, a, b);  // p < 2^381: no carry out of 384 bits
    fp_reduce_once(r);
}
B200_HD void fp_sub(Fp& r, const Fp& a, const Fp& b) {
    const Fp p = fp_p();
    Fp t;
    uint32_t borrow = fp_sub_raw(t, a, b);
    fp_add_masked_raw(r, t, p, 0u - borrow);
}
B200_HD void fp_neg(Fp& r, const Fp& a) {   // 0 -> 0, otherwise p - a; no branch
    const Fp p = fp_p();
    const uint32_t nz = fp_is_zero(a) ? 0u : 0xffffffffu;
    Fp t;
    fp_sub_raw(t, p, a);
#pragma unroll
    for (int i = 0; i < 12; i++) r.l[i] = t.l[i] & nz;
}
B200_HD void fp_dbl(Fp& r, const Fp& a) { fp_add(r, a, a); }

// Montgomery product r = a*b/R mod p (CIOS, operand scanning).  Portable C++: identical on host and device.
// Accepts a < 2^384 (not only a < p) as long as b < p: used where an unreduced integer enters the field.
B200_HD void fp_mul_portable(Fp& r, const Fp& a, const Fp& b) {
    const Fp p = fp_p();
    uint32_t t[14];
#pragma unroll
    for (int i = 0; i < 14; i++) t[i] = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) {
        uint64_t carry = 0;
#pragma unroll
        for (int j = 0; j < 12; j++) {
            uint64_t cur = uint64_t(a.l[j]) * b.l[i] + t[j] + carry;
            t[j] = uint32_t(cur);
            carry = cur >> 32;
        }
        uint64_t cur = uint64_t(t[12]) + carry;
        t[12] = uint32_t(cur);
        t[13] = uint32_t(cur >> 32);
        const uint32_t m = t[0] * B200_FP_N0;
        cur = uint64_t(m) * p.l[0] + t[0];
        carry = cur >> 32;
#pragma unroll
        for (int j = 1; j < 12; j++) {
            cur = uint64_t(m) * p.l[j] + t[j] + carry;
            t[j - 1] = uint32_t(cur);
            carry = cur >> 32;
        }
        cur = uint64_t(t[12]) + carry;
        t[11] = uint32_t(cur);
        t[12] = t[13] + uint32_t(cur >> 32);
    }
    Fp out;
#pragma unroll
    for (int i = 0; i < 12; i++) out.l[i] = t[i];
    fp_reduce_once(out);  // t < 2p
    r = out;
}
}  // namespace b200
#include "fp_mul_ptx.cuh"
namespace b200 {

// The product used everywhere: on the device the generated inline-PTX sequences (mad.lo.cc/madc.hi.cc pairs that
// ptxas fuses into IMAD.WIDE.U32.X carry chains, inputs must be < p); on the host the portable code above.
// B200_FP_MUL_CALL: emit them as real functions taking/returning Fp BY VALUE — the ABI keeps all 36 limbs in
// registers (0-byte stack frame), so a call costs ~40 register moves but every warp of the kernel shares one ~13 KB
// instruction footprint instead of hundreds of inlined copies (the per-key kernel was instruction-fetch limited).
#if defined(__CUDA_ARCH__)
#if defined(B200_FP_MUL_CALL)
static __device__ __noinline__ Fp fp_mul_call(Fp a, Fp b) {
    Fp out;
    fp_mul_ptx_core(out.l, a.l, b.l);
    fp_reduce_once(out);
    return out;
}
static __device__ __noinline__ Fp fp_sqr_call(Fp a) {
    Fp out;
    fp_sqr_ptx_core(out.l, a.l);   // dedicated square: 222 wide multiply-adds instead of 288
    fp_reduce_once(out);
    return out;
}
B200_HD void fp_mul(Fp& r, const Fp& a, const Fp& b) { r = fp_mul_call(a, b); }
B200_HD void fp_sqr(Fp& r, const Fp& a) { r = fp_sqr_call(a); }
#else
B200_HD void fp_mul(Fp& r, const Fp& a, const Fp& b) {
    Fp out;
    fp_mul_ptx_core(out.l, a.l, b.l);
    fp_reduce_once(out);
    r = out;
}
B200_HD void fp_sqr(Fp& r, const Fp& a) {
    Fp out;
    fp_sqr_ptx_core(out.l, a.l);
    fp_reduce_once(out);
    r = out;
}
#endif
#else
B200_HD void fp_mul(Fp& r, const Fp& a, const Fp& b) { fp_mul_portable(r, a, b); }
B200_HD void fp_sqr(Fp& r, const Fp& a) { fp_mul_portable(r, a, a); }
#endif

B200_HD void fp_to_mont(Fp& r, const Fp& a) { const Fp r2 = B200_FP_R2; fp_mul(r, a, r2); }
B200_HD void fp_from_mont(Fp& r, const Fp& a) {
    Fp one;
#pragma unroll
    for (int i = 0; i < 12; i++) one.l[i] = 0;
    one.l[0] = 1;
    fp_mul(r, a, one);
}

// 48 big-endian bytes -> raw integer limbs (no reduction, not Montgomery)
B200_HD void fp_from_be_bytes_raw(Fp& r, const uint8_t* b) {
#pragma unroll
    for (int i = 0; i < 12; i++) {
        const uint8_t* q = b + 44 - 4 * i;
        r.l[i] = (uint32_t(q[0]) << 24) | (uint32_t(q[1]) << 16) | (uint32_t(q[2]) << 8) | q[3];
    }
}
B200_HD void fp_to_be_bytes_raw(uint8_t* b, const Fp& a) {
#pragma unroll
    for (int i = 0; i < 12; i++) {
        uint8_t* q = b + 44 - 4 * i;
        q[0] = uint8_t(a.l[i] >> 24); q[1] = uint8_t(a.l[i] >> 16); q[2] = uint8_t(a.l[i] >> 8); q[3] = uint8_t(a.l[i]);
    }
}

// "lexicographically largest": plain integer value > (p-1)/2.  `a` in Montgomery form.
B200_HD bool fp_is_lex_largest(const Fp& a) {
    Fp raw;
    fp_from_mont(raw, a);
    const Fp half = B200_FP_HALF_P;
    return !fp_geq_raw(half, raw);  // raw > half
}
// parity of the plain integer value (sgn0 building block)
B200_HD uint32_t fp_parity(const Fp& a) {
    Fp raw;
    fp_from_mont(raw, a);
    return raw.l[0] & 1;
}

// exponent tables: device code reads them from the constant bank, host code from static storage
#if defined(__CUDACC__)
static __constant__ uint32_t d_exp_p_minus_2[12] = B200_EXP_P_MINUS_2;
static __constant__ uint32_t d_exp_sqrt[12] = B200_EXP_P_PLUS_1_DIV_4;
static __constant__ uint32_t d_exp_p_minus_3_div_4[12] = B200_EXP_P_MINUS_3_DIV_4;
static __constant__ uint32_t d_exp_p_minus_1_div_2[12] = B200_EXP_P_MINUS_1_DIV_2;
#endif
static const uint32_t h_exp_p_minus_2[12] = B200_EXP_P_MINUS_2;
static const uint32_t h_exp_sqrt[12] = B200_EXP_P_PLUS_1_DIV_4;
static const uint32_t h_exp_p_minus_3_div_4[12] = B200_EXP_P_MINUS_3_DIV_4;
static const uint32_t h_exp_p_minus_1_div_2[12] = B200_EXP_P_MINUS_1_DIV_2;

#if defined(__CUDA_ARCH__)
#define B200_EXP_TABLE(name) d_##name
#else
#define B200_EXP_TABLE(name) h_##name
#endif

// r = a^e, e given as 12 little-endian words.  Sliding 4-bit windows over a table of the 8 odd powers a, a^3 .. a^15:
// for the dense 381-bit exponents used here ((p+1)/4, (p-3)/4, p-2) that is ~380 squarings + ~76 table products + 8 to
// build the table (plain square-and-multiply: ~570; fixed 4-bit windows: ~490).  The exponent is the same constant for
// every thread, so the window logic is uniform (no divergence).  `a` is public data: variable-time is fine.
//
// Where the table (8 x 48 B per thread) lives:
//  * default: thread-local memory.  Its L1 residency depends on how the driver has laid out the context's local-memory
//    pool, and that layout changes once ANY other CUDA module has launched a kernel in the process (the per-key
//    kernel then slows down by a sixth).
//  * B200_POW_TAB_SMEM (defined by a TU before including this header): dynamic shared memory, word-interleaved
//    [(entry*12 + limb) * blockDim.x + threadIdx.x] so every access is bank-conflict-free.  Every kernel of that TU that
//    reaches fp_pow must be launched with fp_pow_smem_bytes(threads) of dynamic shared memory.
constexpr int kPowTabEntries = 8;
#if defined(__CUDA_ARCH__) && defined(B200_POW_TAB_SMEM)
extern __shared__ uint32_t b200_pow_tab[];
struct PowTab {
    __device__ __forceinline__ void set(int i, const Fp& v) {
        uint32_t* q = b200_pow_tab + i * 12 * blockDim.x + threadIdx.x;
#pragma unroll
        for (int k = 0; k < 12; k++) q[k * blockDim.x] = v.l[k];
    }
    __device__ __forceinline__ void get(Fp& v, int i) const {
        const uint32_t* q = b200_pow_tab + i * 12 * blockDim.x + threadIdx.x;
#pragma unroll
        for (int k = 0; k < 12; k++) v.l[k] = q[k * blockDim.x];
    }
};
#else
struct PowTab {
    Fp t[kPowTabEntries];
    B200_HD void set(int i, const Fp& v) { t[i] = v; }
    B200_HD void get(Fp& v, int i) const { v = t[i]; }
};
#endif
constexpr size_t fp_pow_smem_bytes(unsigned threads) { return size_t(threads) * kPowTabEntries * 12 * 4; }

B200_BIG void fp_pow(Fp& r, const Fp& a, const uint32_t* e) {
    PowTab tab;  // tab[k] = a^(2k+1)
    tab.set(0, a);
    {
        Fp a2, cur = a;
        fp_sqr(a2, a);
#pragma unroll 1
        for (int k = 1; k < kPowTabEntries; k++) { fp_mul(cur, cur, a2); tab.set(k, cur); }
    }
    int i = 383;
    while (i >= 0 && !((e[i >> 5] >> (i & 31)) & 1u)) i--;
    if (i < 0) { r = fp_one(); return; }
    Fp acc, t;
    bool started = false;
#pragma unroll 1
    while (i >= 0) {
        if (!((e[i >> 5] >> (i & 31)) & 1u)) {
            fp_sqr(acc, acc);  // started is always true here: the scan begins at the top set bit
            i--;
            continue;
        }
        int l = i + 1 < 4 ? i + 1 : 4;  // window = bits i .. i-l+1, then trimmed to end in a 1
        const int lo = i - l + 1;
        uint64_t two = e[lo >> 5];
        if ((lo >> 5) + 1 < 12) two |= uint64_t(e[(lo >> 5) + 1]) << 32;
        uint32_t w = uint32_t(two >> (lo & 31)) & ((1u << l) - 1u);
        while (!(w & 1u)) { w >>= 1; l--; }
        if (started) {
#pragma unroll 1
            for (int k = 0; k < l; k++) fp_sqr(acc, acc);
            tab.get(t, int(w >> 1));
            fp_mul(acc, acc, t);
        } else {
            tab.get(acc, int(w >> 1));
            started = true;
        }
        i -= l;
    }
    r = acc;
}
B200_HD void fp_inv_fermat(Fp& r, const Fp& a) { fp_pow(r, a, B200_EXP_TABLE(exp_p_minus_2)); }

// Inverse by Kaliski's "almost Montgomery inverse": 381..762 rounds of 384-bit shifts, adds and selects (no products),
// then two products to fix the power of two.  a^(p-2) is 461 DEPENDENT products — for one thread (hash_to_G2's
// normalisation) or one lane of a pairing-VM team (the Fp12 inversion of the final exponentiation: over a quarter of its
// latency floor) that chain is pure latency; this loop is ~70 k short-latency ALU instructions with 12-way limb parallelism.
// Branch-free inside the loop (a conditional swap keeps "the side to halve" in slot 1), so the lanes of a warp stay together.
// Invariants (Kaliski 1995), x = the input integer: x*r = -u*2^k, x*s = v*2^k (mod p); u, v end at (1, 0) or (0, 1).
// Same value as fp_inv_fermat for every input (0 -> 0); tests/host_math + b200_fp_selftest compare the two.
B200_HD void fp_inv_kaliski(Fp& out, const Fp& a) {
    if (fp_is_zero(a)) { out = fp_zero(); return; }
    const Fp p = fp_p();
    Fp a1 = p, b1 = fp_zero();   // (u, r)
    Fp a2 = a, b2 = fp_zero();   // (v, s)
    b2.l[0] = 1;
    bool fl = false;             // true: slot 1 currently holds the (v, s) side
    uint32_t k = 0;
#pragma unroll 1
    for (;;) {
        if (fp_is_zero(a1) || fp_is_zero(a2)) break;
        const bool o1 = (a1.l[0] & 1u) != 0, o2 = (a2.l[0] & 1u) != 0;
        Fp t;
        const uint32_t borrow = fp_sub_raw(t, a1, a2);
        // halve slot 1 this round; swap first when slot 1 is odd and (slot 2 is even, or both are odd and slot 1 is the smaller)
        const bool sw = o1 && (!o2 || borrow != 0);
#pragma unroll
        for (int i = 0; i < 12; i++) {
            const uint32_t x1 = a1.l[i], x2 = a2.l[i], y1 = b1.l[i], y2 = b2.l[i];
            a1.l[i] = sw ? x2 : x1; a2.l[i] = sw ? x1 : x2;
            b1.l[i] = sw ? y2 : y1; b2.l[i] = sw ? y1 : y2;
        }
        fl ^= sw;
        const uint32_t both = (o1 && o2) ? 0xffffffffu : 0u;
        Fp m;
#pragma unroll
        for (int i = 0; i < 12; i++) m.l[i] = a2.l[i] & both;
        fp_sub_raw(a1, a1, m);                        // both odd: a1 >= a2 after the swap
        fp_add_masked_raw(b1, b1, b2, both);          // coefficients stay below 2p < 2^382
#pragma unroll
        for (int i = 0; i < 11; i++) a1.l[i] = (a1.l[i] >> 1) | (a1.l[i + 1] << 31);
        a1.l[11] >>= 1;
#pragma unroll
        for (int i = 11; i > 0; i--) b2.l[i] = (b2.l[i] << 1) | (b2.l[i - 1] >> 31);
        b2.l[0] <<= 1;
        k++;
    }
    // the surviving side holds gcd = 1; its coefficient c gives x^-1 2^k = -c on the u side, +c on the v side
    const bool one_in_slot1 = fp_is_zero(a2);
    Fp c = one_in_slot1 ? b1 : b2;
    const bool v_side = one_in_slot1 ? fl : !fl;
    fp_reduce_once(c);                                // [0, 2p) -> [0, p)
    Fp y;
    if (v_side) y = c; else fp_neg(y, c);
    // y = x^-1 2^k with x = a_real * R: multiply by 2^(768-k) to reach a_real^-1 * R (Montgomery form of the inverse)
    uint32_t j = 768u - k;                            // 6..387
#pragma unroll 1
    while (j > 380u) { fp_dbl(y, y); j--; }           // keep the power-of-two factor below p
    Fp pw = fp_zero();
    pw.l[j >> 5] = 1u << (j & 31u);
    Fp tt;
    fp_mul(tt, y, pw);                                // y 2^j / R
    const Fp r2 = B200_FP_R2;
    fp_mul(out, tt, r2);                              // y 2^j
}
// Device: Kaliski; host: the exponentiation (reference for the tests)
B200_HD void fp_inv(Fp& r, const Fp& a) {
#if defined(__CUDA_ARCH__)
    fp_inv_kaliski(r, a);
#else
    fp_inv_fermat(r, a);
#endif
}
// candidate square root a^((p+1)/4); returns whether it is one
B200_HD bool fp_sqrt(Fp& r, const Fp& a) {
    Fp s, c;
    fp_pow(s, a, B200_EXP_TABLE(exp_sqrt));
    fp_sqr(c, s);
    r = s;
    return fp_eq(c, a);
}

}  // namespace b200
