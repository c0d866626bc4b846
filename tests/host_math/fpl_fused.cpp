// TEST INFRASTRUCTURE: the per-key kernel's fused reductions (fpl.cuh) and its FpL Jacobian formulas, compiled for the CPU
// from the same headers (the C emulations of the generated PTX), for tests/test_fpl_fused.py.
#include <cstddef>
#include <cstdint>

#include "../../ethereum_consensus_b200/csrc/groups.cuh"

using namespace b200;
#define HM extern "C" __attribute__((visibility("default")))

static Fp load(const uint32_t* w) { Fp r; for (int k = 0; k < 12; k++) r.l[k] = w[k]; return r; }

// n records of four 12-word operands (a, b, c, d) -> 12-word results
//   op 0: fp_mul_add_mul_emul_core(a, b, c, d) = REDC(a b + c d)        op 2: f_mul_sub_mul(a, b, c, d)
//   op 1: fp_mul_sub_8sqr_emul_core(a, b, c) = REDC(a b + 32p^2 - 8c^2)   op 3: f_mul_sub_8sqr(a, b, c)
HM void hm_fused(int op, uint32_t n, const uint32_t* in, uint32_t* out) {
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t* w = in + 48 * std::size_t(i);
        uint32_t* o = out + 12 * std::size_t(i);
        FpL a = fpl_from_fp(load(w)), b = fpl_from_fp(load(w + 12)), c = fpl_from_fp(load(w + 24)),
            d = fpl_from_fp(load(w + 36)), r;
        switch (op) {
        case 0: fp_mul_add_mul_emul_core(o, w, w + 12, w + 24, w + 36); break;
        case 1: fp_mul_sub_8sqr_emul_core(o, w, w + 12, w + 24); break;
        case 2: f_mul_sub_mul(r, a, b, c, d); for (int k = 0; k < 12; k++) o[k] = r.v.l[k]; break;
        default: f_mul_sub_8sqr(r, a, b, c); for (int k = 0; k < 12; k++) o[k] = r.v.l[k]; break;
        }
    }
}

// n Jacobian points on FpL (X, Y, Z as 12-word raw limbs each): op 0 jac_double(p), 1 jac_add_mixed(p, (q.x, q.y)),
// 2 jac_add(p, q)
HM void hm_g1l_curve(int op, uint32_t n, const uint32_t* pa, const uint32_t* pb, uint32_t* out) {
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t* a = pa + 36 * std::size_t(i);
        const uint32_t* b = pb + 36 * std::size_t(i);
        Jac<FpL> p, q, r;
        p.x.v = load(a); p.y.v = load(a + 12); p.z.v = load(a + 24);
        q.x.v = load(b); q.y.v = load(b + 12); q.z.v = load(b + 24);
        if (op == 0) jac_double(r, p);
        else if (op == 1) jac_add_mixed(r, p, q.x, q.y);
        else jac_add(r, p, q);
        uint32_t* o = out + 36 * std::size_t(i);
        for (int k = 0; k < 12; k++) { o[k] = r.x.v.l[k]; o[12 + k] = r.y.v.l[k]; o[24 + k] = r.z.v.l[k]; }
    }
}
