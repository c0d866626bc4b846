// Host build of the per-key kernel's fixed square-root chain (fpl_sqrt_chain) and of the subgroup check's second ladder
// with the base point's Z^2 / Z^3 cached (jac_mul_u64_jac_cached), for tests/test_sqrt_chain.py.  The lazily reduced
// products run the C emulation of the device's instruction list (fpl.cuh), so representatives match the device's.
#include <cstddef>
#include <cstdint>

#include "../../ethereum_consensus_b200/csrc/groups.cuh"

using namespace b200;

#define HM __attribute__((visibility("default")))

static FpL load(const uint32_t* a) { FpL r; for (int k = 0; k < 12; k++) r.v.l[k] = a[k]; return r; }
static void store(uint32_t* o, const FpL& a) { for (int k = 0; k < 12; k++) o[k] = a.v.l[k]; }

// n inputs of 12 limbs each (any representative in [0, 2p)) -> a^((p+1)/4) by the chain and by the windowed fpl_pow
extern "C" HM void hm_fpl_sqrt_chain(uint32_t n, const uint32_t* in, uint32_t* out_chain, uint32_t* out_pow) {
    for (uint32_t i = 0; i < n; i++) {
        const FpL a = load(in + 12 * i);
        FpL r;
        fpl_sqrt_chain(r, a);
        store(out_chain + 12 * i, r);
        fpl_pow(r, a, B200_EXP_TABLE(exp_sqrt));
        store(out_pow + 12 * i, r);
    }
}

// affine (x, y), Montgomery limbs: t = [|z|](x, y), then [|z|]t by jac_mul_u64_jac and by jac_mul_u64_jac_cached;
// out: the two results as X | Y | Z (36 limbs each)
extern "C" HM void hm_second_ladder(const uint32_t* x, const uint32_t* y, uint32_t* out_plain, uint32_t* out_cached) {
    Jac<FpL> t, a, b;
    jac_mul_u64(t, load(x), load(y), B200_Z_ABS);
    jac_mul_u64_jac(a, t, B200_Z_ABS);
    jac_mul_u64_jac_cached(b, t, B200_Z_ABS);
    store(out_plain, a.x); store(out_plain + 12, a.y); store(out_plain + 24, a.z);
    store(out_cached, b.x); store(out_cached + 12, b.y); store(out_cached + 24, b.z);
}
