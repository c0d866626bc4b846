// Pairing side of the BLS pipeline: one Miller loop per (G1, G2) pair and, per tuple, the Gt product + final
// exponentiation + comparison with one — the check blst performs inside `fast_aggregate_verify` /
// `aggregate_verify` (ethereum-consensus/src/crypto/bls.rs:106,126), plus the code merge that
// reproduces the wrapper's precedence: first bad public key -> signature decoding error -> verification.
#define B200_FP_MUL_CALL 1
#define B200_FP2_NOINLINE 1
#define B200_TOWER_NOINLINE 1
#include <cuda_runtime.h>

#include "bls_kernels.cuh"
#include "pairing.cuh"

namespace b200 {
namespace {

__device__ __forceinline__ bool tuple_dead(uint32_t t, const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code) {
    return pk_code[t] != BLS_SUCCESS || flags[t] != 0 || sig_code[t] != SIG_OK;
}

__global__ void __launch_bounds__(64) k_miller(const G1Aff* __restrict__ g1, const uint32_t* __restrict__ g1_idx,
                                                const G2Aff* __restrict__ g2, const uint32_t* __restrict__ g2_idx,
                                                const uint32_t* __restrict__ pair_tuple, const int32_t* __restrict__ pk_code,
                                                const uint32_t* __restrict__ flags, const int32_t* __restrict__ sig_code,
                                                uint32_t n_pairs, Fp12* __restrict__ f) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pairs) return;
    if (tuple_dead(pair_tuple[i], pk_code, flags, sig_code)) return;
    const G1Aff p = g1[g1_idx[i]];
    const G2Aff q = g2[g2_idx[i]];
    Fp12 r;
    miller_loop(r, p, q);
    f[i] = r;
}

__global__ void __launch_bounds__(64) k_final(const Fp12* __restrict__ f, const uint32_t* __restrict__ pair_off,
                                               const int32_t* __restrict__ pk_code, const uint32_t* __restrict__ flags,
                                               const int32_t* __restrict__ sig_code, uint32_t n_tuples,
                                               int32_t* __restrict__ out_codes) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tuples) return;
    int32_t code;
    if (pk_code[t] != BLS_SUCCESS) code = pk_code[t];               // Err(Error::BLST(..)) from key_validate
    else if (sig_code[t] > 0) code = sig_code[t];                    // Err(Error::BLST(..)) from Signature::from_bytes
    else if (flags[t] != 0 || sig_code[t] == SIG_NOT_IN_GROUP) code = BLS_VERIFY_FAIL;
    else {
        Fp12 acc = f[pair_off[t]];
        for (uint32_t k = pair_off[t] + 1; k < pair_off[t + 1]; k++) {
            const Fp12 x = f[k];
            fp12_mul(acc, acc, x);
        }
        code = final_exp_is_one(acc) ? BLS_SUCCESS : BLS_VERIFY_FAIL;
    }
    out_codes[t] = code;
}

}  // namespace

void launch_miller(const G1Aff* g1, const uint32_t* g1_idx, const G2Aff* g2, const uint32_t* g2_idx,
                   const uint32_t* pair_tuple, const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code,
                   uint32_t n_pairs, Fp12* f, void* stream) {
    if (!n_pairs) return;
    k_miller<<<(n_pairs + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(g1, g1_idx, g2, g2_idx, pair_tuple, pk_code,
                                                                                    flags, sig_code, n_pairs, f);
}
void launch_final(const Fp12* f, const uint32_t* pair_off, const int32_t* pk_code, const uint32_t* flags,
                  const int32_t* sig_code, uint32_t n_tuples, int32_t* out_codes, void* stream) {
    if (!n_tuples) return;
    k_final<<<(n_tuples + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(f, pair_off, pk_code, flags, sig_code, n_tuples,
                                                                                  out_codes);
}

}  // namespace b200
