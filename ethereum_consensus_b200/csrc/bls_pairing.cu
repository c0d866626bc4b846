// The device reference of the pairing: pairing.cuh's tower operations, Miller loop and final exponentiation, one thread
// per record, behind b200_pairing_eval.  No verification path runs these kernels; the device tests compare the
// lane-parallel VM (bls_vm.cu) against them, the Miller loop with Z = 1 bit for bit.
#define B200_FP_MUL_CALL 1
#define B200_FP2_NOINLINE 1
#define B200_TOWER_NOINLINE 1
#include <cuda_runtime.h>

#include "bls_kernels.cuh"
#include "pairing.cuh"

namespace b200 {
namespace {

// Tower operations, Miller steps and the final exponentiation against big integers (b200_pairing_eval), one per launch,
// as this unit compiles them: products through calls, non-inlined tower functions, ptxas at its default level
__device__ __forceinline__ void pe_load(Fp* v, const uint32_t* w, int n_slots) {
    for (int s = 0; s < n_slots; s++)
        for (int k = 0; k < 12; k++) v[s].l[k] = w[12 * s + k];
}
__global__ void __launch_bounds__(64) k_pairing_eval(int32_t op, uint32_t n, const uint32_t* __restrict__ a,
                                                      const uint32_t* __restrict__ b, uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* pa = a + size_t(i) * kPairingEvalWords;
    const uint32_t* pb = b + size_t(i) * kPairingEvalWords;
    Fp12 x, y, r = fp12_one();
    pe_load(&x.c0.c0.c0, pa, 12);
    pe_load(&y.c0.c0.c0, pb, 12);
    uint32_t flag = 0;
    switch (op) {
    case PAIRING_EVAL_FP6_MUL: fp6_mul(r.c0, x.c0, y.c0); r.c1 = x.c1; break;
    case PAIRING_EVAL_FP6_INV: fp6_inv(r.c0, x.c0); r.c1 = x.c1; break;
    case PAIRING_EVAL_FP12_MUL: fp12_mul(r, x, y); break;
    case PAIRING_EVAL_FP12_SQR: fp12_sqr(r, x); break;
    case PAIRING_EVAL_FP12_INV: fp12_inv(r, x); break;
    case PAIRING_EVAL_FP12_MUL_BY_LINE: fp12_mul_by_line(r, x, y.c0.c0, y.c0.c1, y.c0.c2); break;
    case PAIRING_EVAL_FP12_FROB1: fp12_frobenius<1>(r, x); break;
    case PAIRING_EVAL_FP12_FROB2: fp12_frobenius<2>(r, x); break;
    case PAIRING_EVAL_FP12_CYCLO_SQR: fp12_cyclotomic_sqr(r, x); break;
    case PAIRING_EVAL_FP12_POW_Z: fp12_pow_z(r, x); break;
    case PAIRING_EVAL_MILLER_DOUBLE:
    case PAIRING_EVAL_MILLER_ADD: {
        G2Jac t;
        t.x = x.c0.c0; t.y = x.c0.c1; t.z = x.c0.c2;
        G2Aff q;
        q.x = y.c0.c0; q.y = y.c0.c1; q.inf = 0;
        const Fp xp = y.c0.c2.c0, yp = y.c0.c2.c1;
        if (op == PAIRING_EVAL_MILLER_DOUBLE) miller_double_step(t, r.c1.c0, r.c1.c1, r.c1.c2, xp, yp);
        else miller_add_step(t, r.c1.c0, r.c1.c1, r.c1.c2, q, xp, yp);
        r.c0.c0 = t.x; r.c0.c1 = t.y; r.c0.c2 = t.z;
        break;
    }
    case PAIRING_EVAL_MILLER_LOOP: {
        G1Aff p;
        p.x = x.c0.c0.c0; p.y = x.c0.c0.c1; p.inf = pa[144];
        G2Aff q;
        q.x = y.c0.c0; q.y = y.c0.c1; q.inf = pb[144];
        miller_loop(r, p, q);
        break;
    }
    case PAIRING_EVAL_FINAL_EXP: final_exp(r, x); flag = fp12_is_one(r) ? 1u : 0u; break;
    default: break;
    }
    uint32_t* o = out + size_t(i) * kPairingEvalWords;
    const Fp* v = &r.c0.c0.c0;
    for (int s = 0; s < 12; s++)
        for (int k = 0; k < 12; k++) o[12 * s + k] = v[s].l[k];
    o[144] = flag;
}

}  // namespace

void launch_pairing_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream) {
    if (!n) return;
    k_pairing_eval<<<(n + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(op, n, a, b, out);
}

}  // namespace b200
