// Random-linear-combination (RLC) whole-batch check — the `north_star`'s "Miller loops fused across the batch, partial Gt
// products reduced with warp shuffles, one NCCL exchange of the per-shard Gt result" (SURVEY.md §7 step 7, §8e).
//
// For T tuples (agg_t, H_t = hash_to_G2(msg_t), sig_t) whose points already passed the per-point checks, draw 64-bit
// scalars r_t and test ONE product instead of T:
//        prod_t e(r_t agg_t, H_t)  *  e(-g1, sum_t r_t sig_t)  ==  1
// T Miller loops instead of 2T, one final exponentiation instead of T.  If every tuple is valid the product is 1 for any
// r; if some tuple is invalid it is 1 with probability <= 2^-64 over the r_t (all points are in the r-order subgroups, so
// the left side is g^(sum r_t d_t) for the tuples' discrete-log defects d_t).  The answer is therefore a whole-batch
// boolean — exactly what `process_block` needs in the common case (every signature valid); when it is 0 the caller asks
// the per-tuple path, which stays the only source of per-tuple codes (bit-exact by construction).
//
// Kernels here: k_rlc_scale (per tuple: r_t agg_t in G1, r_t sig_t in G2), k_rlc_reduce (warp-shuffle trees: product of
// Miller values in Fp12, sum of the scaled signatures in G2), k_rlc_finish (sum -> affine for the last Miller loop).
// The T Miller loops and the final exponentiation reuse the lane-parallel VM kernels (bls_vm.cu).
#define B200_FP_MUL_CALL 1
#define B200_FP2_NOINLINE 1
#define B200_TOWER_NOINLINE 1
#include <cuda_runtime.h>

#include "bls_kernels.cuh"
#include "pairing.cuh"
#include "sha256.cuh"

namespace b200 {
namespace {

// r_t = first 8 bytes (little-endian) of SHA-256(seed || le64(t)), forced non-zero
__device__ __forceinline__ uint64_t rlc_scalar(const uint32_t* __restrict__ seed_words, uint64_t t) {
    uint32_t w[16], h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = seed_words[i];
    w[8] = bswap32(uint32_t(t)); w[9] = bswap32(uint32_t(t >> 32));   // le64(t) as big-endian words of the byte stream
    w[10] = 0x80000000u;
#pragma unroll
    for (int i = 11; i < 15; i++) w[i] = 0;
    w[15] = 40 * 8;
    sha256_init(h);
    sha256_compress(h, w);
    const uint64_t r = uint64_t(bswap32(h[0])) | (uint64_t(bswap32(h[1])) << 32);
    return r ? r : 1;
}

// One thread per (tuple, group): the first half of the grid scales the aggregate keys (G1Pre of r_t * agg_t), the second
// half the signatures (Jacobian r_t * sig_t) — block-uniform roles, so the two scalar multiplications of a tuple run on
// different SMs at the same time instead of back to back in one thread.  A tuple that already failed a per-point check
// makes the whole batch fail (*bad = 1) — its code comes from the per-tuple path.
__global__ void __launch_bounds__(64) k_rlc_scale(const G1Jac* __restrict__ agg, const G2Aff* __restrict__ sig,
                                                   const int32_t* __restrict__ pk_code, const uint32_t* __restrict__ flags,
                                                   const int32_t* __restrict__ sig_code, const uint32_t* __restrict__ seed_words,
                                                   uint64_t t0, uint32_t n, uint32_t blocks_per_role, G1Pre* __restrict__ out_g1,
                                                   G2Jac* __restrict__ out_g2, int32_t* __restrict__ bad) {
    const bool g2_role = blockIdx.x >= blocks_per_role;
    const uint32_t t = (blockIdx.x - (g2_role ? blocks_per_role : 0u)) * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const bool dead = pk_code[t] != BLS_SUCCESS || flags[t] != 0 || sig_code[t] != SIG_OK;
    const uint64_t r = rlc_scalar(seed_words, t0 + t);
    if (!g2_role) {
        G1Pre p;
        if (dead) {
            atomicExch(bad, 1);
            p.xz = fp_one(); p.y = fp_one(); p.z3 = fp_zero(); p.inf = 1;   // neutral contribution
        } else {
            const G1Jac a = agg[t];
            G1Jac ra;
            jac_mul_u64_jac(ra, a, r);
            p.inf = jac_is_inf(ra) ? 1u : 0u;
            Fp zz;
            fp_sqr(zz, ra.z);
            fp_mul(p.z3, zz, ra.z);
            fp_mul(p.xz, ra.x, ra.z);
            p.y = ra.y;
        }
        out_g1[t] = p;
    } else {
        G2Jac rs;
        jac_set_inf(rs);
        if (!dead) {
            const G2Aff s = sig[t];
            if (!s.inf) jac_mul_u64(rs, s.x, s.y, r);
        }
        out_g2[t] = rs;
    }
}

// warp-shuffle exchange of a struct of 32-bit words
template <class T>
__device__ __forceinline__ void shfl_down_words(T& dst, const T& src, int delta) {
    static_assert(sizeof(T) % 4 == 0, "word-sized struct");
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&src);
    uint32_t* d = reinterpret_cast<uint32_t*>(&dst);
#pragma unroll 4
    for (unsigned k = 0; k < sizeof(T) / 4; k++) d[k] = __shfl_down_sync(0xffffffffu, s[k], delta);
}

// One warp folds 32 consecutive Fp12 values (product) or G2 points (sum) with a shuffle tree: lane l combines lane l+s's
// partial for s = 16, 8, 4, 2, 1; lane 0 writes the warp's partial.  Inputs beyond n are the neutral elements.
__global__ void __launch_bounds__(32) k_rlc_reduce(const Fp12* __restrict__ f_in, const G2Jac* __restrict__ q_in, uint32_t n,
                                                    Fp12* __restrict__ f_out, G2Jac* __restrict__ q_out) {
    const uint32_t lane = threadIdx.x, i = blockIdx.x * 32 + lane;
    if (f_in) {   // Gt product (the launch folds either the Miller values or the scaled signatures, never both)
        Fp12 f = fp12_one();
        if (i < n) f = f_in[i];
#pragma unroll 1
        for (int s = 16; s > 0; s >>= 1) {
            Fp12 fo;
            shfl_down_words(fo, f, s);
            if (lane < uint32_t(s)) fp12_mul(f, f, fo);
        }
        if (lane == 0) f_out[blockIdx.x] = f;
    }
    if (q_in) {   // G2 sum
        G2Jac q;
        jac_set_inf(q);
        if (i < n) q = q_in[i];
#pragma unroll 1
        for (int s = 16; s > 0; s >>= 1) {
            G2Jac qo;
            shfl_down_words(qo, q, s);
            if (lane < uint32_t(s)) jac_add(q, q, qo);
        }
        if (lane == 0) q_out[blockIdx.x] = q;
    }
}
// Segmented Gt product for aggregate_verify batches (launch_fold_segments): k_rlc_reduce's warp and shuffles, with the
// tree replaced by a segmented suffix scan, so that one warp serves every segment its 32 values touch.  Step d = 1, 2, ..,
// 16: lane l multiplies in lane l + d's partial while l + d is still in l's segment; afterwards the first lane of each piece
// holds the piece's product.  Five dependent products per level, whatever the segments' lengths; a segment of n values
// needs about log32(n) levels.
__global__ void __launch_bounds__(64) k_fold_segments(const Fp12* __restrict__ in, uint32_t n_in, const uint32_t* __restrict__ seg_of,
                                                       const uint32_t* __restrict__ seg_in, const uint32_t* __restrict__ seg_out,
                                                       const int32_t* __restrict__ pk_code, const uint32_t* __restrict__ flags,
                                                       const int32_t* __restrict__ sig_code, Fp12* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31u, chunk = i >> 5;
    bool live = i < n_in;
    uint32_t t = 0, last = 0;   // the segment, and the lane of its last value in this chunk
    if (live) {
        t = seg_of[i];
        last = min(seg_in[t + 1], (chunk + 1) * 32u) - 1 - chunk * 32u;
        if (pk_code && (pk_code[t] != BLS_SUCCESS || flags[t] != 0 || sig_code[t] != SIG_OK)) live = false;   // failed tuple
    }
    Fp12 f = fp12_one();
    if (live) f = in[i];
#pragma unroll 1
    for (uint32_t d = 1; d < 32; d <<= 1) {   // every lane shuffles: the whole warp takes part in each step
        Fp12 fo;
        shfl_down_words(fo, f, int(d));
        if (live && lane + d <= last) fp12_mul(f, f, fo);
    }
    if (!live) return;
    const uint32_t first = seg_in[t];
    if (i != first && lane != 0) return;   // not the head of a piece
    const uint32_t k = chunk - first / 32u;
    if (seg_out) {
        out[seg_out[t] + k] = f;
    } else {
        out[2 * size_t(t) + k] = f;
        if ((seg_in[t + 1] - 1) / 32u == first / 32u) out[2 * size_t(t) + 1] = fp12_one();   // one piece: pad with one
    }
}
__global__ void k_fp12_one(Fp12* out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *out = fp12_one();
}

// the reduced signature sum as an affine point for the last Miller loop (Q = infinity: that pair contributes 1)
__global__ void k_rlc_finish(const G2Jac* __restrict__ q, G2Aff* __restrict__ out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    G2Aff a;
    jac_to_aff(a, *q);
    *out = a;
}

}  // namespace

void launch_rlc_scale(const G1Jac* agg, const G2Aff* sig, const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code,
                      const uint32_t* seed_words, uint64_t t0, uint32_t n, G1Pre* out_g1, G2Jac* out_g2, int32_t* bad, void* stream) {
    if (!n) return;
    const uint32_t per_role = (n + 63) / 64;
    k_rlc_scale<<<2 * per_role, 64, 0, static_cast<cudaStream_t>(stream)>>>(agg, sig, pk_code, flags, sig_code, seed_words, t0, n,
                                                                            per_role, out_g1, out_g2, bad);
}
// folds n inputs to ceil(n / 32) partials
uint32_t launch_rlc_reduce(const Fp12* f_in, const G2Jac* q_in, uint32_t n, Fp12* f_out, G2Jac* q_out, void* stream) {
    const uint32_t blocks = (n + 31) / 32;
    if (blocks) k_rlc_reduce<<<blocks, 32, 0, static_cast<cudaStream_t>(stream)>>>(f_in, q_in, n, f_out, q_out);
    return blocks;
}
void launch_fold_segments(const Fp12* in, uint32_t n_in, const uint32_t* seg_of, const uint32_t* seg_in, const uint32_t* seg_out,
                          const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code, Fp12* out, void* stream) {
    if (!n_in) return;
    k_fold_segments<<<(n_in + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(in, n_in, seg_of, seg_in, seg_out, pk_code, flags,
                                                                                     sig_code, out);
}
void launch_fp12_one(Fp12* out, void* stream) { k_fp12_one<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(out); }
void launch_rlc_finish(const G2Jac* q, G2Aff* out, void* stream) { k_rlc_finish<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(q, out); }

}  // namespace b200
