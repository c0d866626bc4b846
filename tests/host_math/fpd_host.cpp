// Host build of the FP64 field (fpd.cuh) and of the per-key kernel's split validation (groups.cuh), for
// tests/test_fpd.py and tests/test_fpd_device_gpu.py.  std::fma is the same IEEE binary64 fused operation as the
// device's DFMA, and every other rounding in fpd.cuh is exact or spelled out, so these are meant to be the device's bits:
// test_fpd_device_gpu.py compares products, squares, sums, the conversions and the square-root chain with the device
// build limb for limb, and test_fpd.py checks that a build which contracts freely (-mfma -ffp-contract=fast) gives the
// same bits as this one.
#include <cstddef>
#include <cstdint>

#include "../../ethereum_consensus_b200/csrc/groups.cuh"

using namespace b200;

#define HM __attribute__((visibility("default")))

static Fp load(const uint32_t* a) { Fp r; for (int k = 0; k < 12; k++) r.l[k] = a[k]; return r; }
static void store(uint32_t* o, const Fp& a) { for (int k = 0; k < 12; k++) o[k] = a.l[k]; }
static FpD loadd(const double* a) { FpD r; for (int k = 0; k < 8; k++) r.l[k] = a[k]; return r; }
static void stored(double* o, const FpD& a) { for (int k = 0; k < 8; k++) o[k] = a.l[k]; }

// op 0: a b, 1: a^2, 2: a + b, on raw limbs (8 doubles each)
extern "C" HM void hm_fpd_op(int op, uint32_t n, const double* a, const double* b, double* out) {
    for (uint32_t i = 0; i < n; i++) {
        FpD r;
        const FpD x = loadd(a + 8 * i), y = loadd(b + 8 * i);
        if (op == 0) fpd_mul(r, x, y); else if (op == 1) fpd_sqr(r, x); else fpd_add(r, x, y);
        stored(out + 8 * i, r);
    }
}
// Fp limbs in [0, 2p) -> FpD -> FpL representative in [0, 2p), and the FpD limbs
extern "C" HM void hm_fpd_roundtrip(uint32_t n, const uint32_t* a, double* d, uint32_t* back) {
    for (uint32_t i = 0; i < n; i++) {
        const FpD x = fpd_from_fp(load(a + 12 * i));
        stored(d + 8 * i, x);
        store(back + 12 * i, fpd_to_fpl(x).v);
    }
}
// a^((p+1)/4) by fpd_sqrt_chain and by fpl_sqrt_chain, both as FpL representatives
extern "C" HM void hm_fpd_sqrt_chain(uint32_t n, const uint32_t* a, uint32_t* out_fpd, uint32_t* out_fpl) {
    for (uint32_t i = 0; i < n; i++) {
        const Fp x = load(a + 12 * i);
        FpD r;
        fpd_sqrt_chain(r, fpd_from_fp(x));
        store(out_fpd + 12 * i, fpd_to_fpl(r).v);
        FpL l;
        fpl_sqrt_chain(l, fpl_from_fp(x));
        store(out_fpl + 12 * i, l.v);
    }
}
// 48-byte keys: g1_key_validate's code and point, and the split kernel's (g1_parse, g1_y_from_x_fpd,
// g1_in_subgroup_iso, g1_key_validate_code); points as x | y (24 limbs), written on success only
extern "C" HM void hm_key_validate_split(uint32_t n, const uint8_t* keys, int32_t* code_ref, uint32_t* pt_ref,
                                         int32_t* code_split, uint32_t* pt_split) {
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t* b = keys + 48 * i;
        G1Aff p;
        code_ref[i] = g1_key_validate(p, b);
        if (code_ref[i] == BLS_SUCCESS) { store(pt_ref + 24 * i, p.x); store(pt_ref + 24 * i + 12, p.y); }
        Fp x, y = fp_zero();
        uint32_t inf;
        bool largest, on_curve = true, in_group = true;
        int32_t rc = g1_parse(x, inf, largest, b);
        if (rc == BLS_SUCCESS && !inf) {
            on_curve = g1_y_from_x_fpd(y, x, largest);
            in_group = g1_in_subgroup_iso(x);
        }
        code_split[i] = g1_key_validate_code(rc, inf, on_curve, in_group);
        if (code_split[i] == BLS_SUCCESS) { store(pt_split + 24 * i, x); store(pt_split + 24 * i + 12, y); }
    }
}
// affine (x, y) on E, Montgomery limbs: g1_in_subgroup_lazy and g1_in_subgroup_iso(x)
extern "C" HM void hm_subgroup_iso(const uint32_t* x, const uint32_t* y, int32_t* lazy, int32_t* iso) {
    G1Aff p;
    p.x = load(x); p.y = load(y); p.inf = 0;
    *lazy = g1_in_subgroup_lazy(p);
    *iso = g1_in_subgroup_iso(p.x);
}
