// Lane-parallel "Fp2 VM": executes the statically scheduled Miller-loop / final-exponentiation programs produced by
// tools/gen_pairing_vm.py.  A TEAM of kVmTeam lanes shares one register file of Fp2 slots (shared memory on the
// device); in every round each lane executes at most one Fp2 instruction, rounds are separated by a barrier.
// Register allocation guarantees that no slot is both read and written in the same round.
#pragma once
#include "fp12.cuh"
#include "pairing_vm_prog.cuh"    // teams of 8 lanes: the higher throughput (batches that fill the machine)
#include "pairing_vm_prog16.cuh"  // teams of 16 lanes: the shorter critical path (1 918 / 3 094 rounds instead of 2 493 / 3 842)

namespace b200 {

enum VmOp : uint32_t { VM_NOP = 0, VM_MUL, VM_SQR, VM_MULFP, VM_INV, VM_ADD, VM_SUB, VM_NEG, VM_DBL, VM_CONJ, VM_MULXI, VM_COPY, VM_LDC };

// register-file accessors: dense array of Fp2 (host) or 25-word-strided shared memory (device, bank-conflict free)
struct VmRfDense {
    Fp2* p;
    B200_HD Fp2 load(uint32_t i) const { return p[i]; }
    B200_HD void store(uint32_t i, const Fp2& v) const { p[i] = v; }
};
// Slot stride in words.  28 (default) / 24: 16-byte aligned slots moved with 128-bit LDS/STS; 25 (round 1, -DB200_VM_SLOT_WORDS=25):
// scalar LDS/STS, conflict-free for any slot pattern.  28 had the shortest Miller loop and final exponentiation of the three.
// 16-byte aligned slots moved with 128-bit LDS/STS — 6 + 6 + 6 wide accesses per light op instead of 24 + 24 + 24.
#if !defined(B200_VM_SLOT_WORDS)
#define B200_VM_SLOT_WORDS 28
#endif
constexpr int kVmSlotWords = B200_VM_SLOT_WORDS;
// -DB200_VM_SLOT_PAD4 (A/B): 24-word slots with 16 bytes of padding after every fourth (100 B per slot on average instead of 112):
// any 8 consecutive slots still fall into 8 different 16-byte bank groups, and 12 % more teams fit an SM.
#if defined(B200_VM_SLOT_PAD4)
B200_HD constexpr uint32_t vm_slot_word(uint32_t i) { return i * 24u + (i >> 2) * 4u; }
B200_HD constexpr uint32_t vm_team_words(uint32_t n_slots) { return n_slots * 24u + ((n_slots + 3u) >> 2) * 4u; }
#else
B200_HD constexpr uint32_t vm_slot_word(uint32_t i) { return i * uint32_t(kVmSlotWords); }
B200_HD constexpr uint32_t vm_team_words(uint32_t n_slots) { return n_slots * uint32_t(kVmSlotWords); }
#endif
constexpr int kVmMaxSmemBytes = 227 * 1024;          // opt-in dynamic shared memory per CTA on sm_90 (H100)
constexpr uint32_t kVmBlobMagic = 0xB200564Du;       // run-time program blobs (vm_load_programs)
struct VmRfStrided {
    uint32_t* p;
    B200_HD Fp2 load(uint32_t i) const {
        Fp2 v;
#if defined(__CUDA_ARCH__) && (B200_VM_SLOT_WORDS % 4 == 0)
        const uint4* q = reinterpret_cast<const uint4*>(p + vm_slot_word(i));
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const uint4 a = q[k], b = q[3 + k];
            v.c0.l[4 * k] = a.x; v.c0.l[4 * k + 1] = a.y; v.c0.l[4 * k + 2] = a.z; v.c0.l[4 * k + 3] = a.w;
            v.c1.l[4 * k] = b.x; v.c1.l[4 * k + 1] = b.y; v.c1.l[4 * k + 2] = b.z; v.c1.l[4 * k + 3] = b.w;
        }
#else
        const uint32_t* q = p + vm_slot_word(i);
#pragma unroll
        for (int k = 0; k < 12; k++) { v.c0.l[k] = q[k]; v.c1.l[k] = q[12 + k]; }
#endif
        return v;
    }
    B200_HD void store(uint32_t i, const Fp2& v) const {
#if defined(__CUDA_ARCH__) && (B200_VM_SLOT_WORDS % 4 == 0)
        uint4* q = reinterpret_cast<uint4*>(p + vm_slot_word(i));
#pragma unroll
        for (int k = 0; k < 3; k++) {
            q[k] = make_uint4(v.c0.l[4 * k], v.c0.l[4 * k + 1], v.c0.l[4 * k + 2], v.c0.l[4 * k + 3]);
            q[3 + k] = make_uint4(v.c1.l[4 * k], v.c1.l[4 * k + 1], v.c1.l[4 * k + 2], v.c1.l[4 * k + 3]);
        }
#else
        uint32_t* q = p + vm_slot_word(i);
#pragma unroll
        for (int k = 0; k < 12; k++) { q[k] = v.c0.l[k]; q[12 + k] = v.c1.l[k]; }
#endif
    }
};

// one instruction: result into `res`, returns false for NOP
template <class RF>
B200_HD bool vm_exec(uint32_t w, const RF& rf, const Fp2* consts, Fp2& res) {
    const uint32_t op = w & 0xffu, a = (w >> 16) & 0xffu, b = w >> 24;
    switch (op) {
    case VM_NOP: return false;
    case VM_MUL: { const Fp2 x = rf.load(a), y = rf.load(b); fp2_mul(res, x, y); } break;
    case VM_SQR: { const Fp2 x = rf.load(a); fp2_sqr(res, x); } break;
    case VM_MULFP: { const Fp2 x = rf.load(a); const Fp k = rf.load(b).c0; fp2_mul_fp(res, x, k); } break;
    case VM_INV: { const Fp2 x = rf.load(a); fp2_inv(res, x); } break;
    case VM_ADD: { const Fp2 x = rf.load(a), y = rf.load(b); fp2_add(res, x, y); } break;
    case VM_SUB: { const Fp2 x = rf.load(a), y = rf.load(b); fp2_sub(res, x, y); } break;
    case VM_NEG: { const Fp2 x = rf.load(a); fp2_neg(res, x); } break;
    case VM_DBL: { const Fp2 x = rf.load(a); fp2_dbl(res, x); } break;
    case VM_CONJ: { const Fp2 x = rf.load(a); fp2_conj(res, x); } break;
    case VM_MULXI: { const Fp2 x = rf.load(a); fp2_mul_xi(res, x); } break;
    case VM_COPY: res = rf.load(a); break;
    default: res = consts[a]; break;  // VM_LDC
    }
    return true;
}

// The two scheduled program pairs behind one name: VmProg<8>, VmProg<16>
template <int TEAM> struct VmProg;
template <> struct VmProg<8> {
    static constexpr int team = 8, miller_rounds = kMillerRounds, miller_slots = kMillerSlots, final_rounds = kFinalRounds, final_slots = kFinalSlots;
    static constexpr const int* miller_out = kMillerOut;
    static constexpr const int* final_out = kFinalOut;
    static const uint32_t* miller_code() { return h_miller_code; }
    static const uint32_t* final_code() { return h_final_code; }
    static constexpr size_t miller_code_bytes = sizeof(h_miller_code), final_code_bytes = sizeof(h_final_code);
};
template <> struct VmProg<16> {
    static constexpr int team = 16, miller_rounds = kMillerRounds16, miller_slots = kMillerSlots16, final_rounds = kFinalRounds16, final_slots = kFinalSlots16;
    static constexpr const int* miller_out = kMillerOut16;
    static constexpr const int* final_out = kFinalOut16;
    static const uint32_t* miller_code() { return h_miller_code16; }
    static const uint32_t* final_code() { return h_final_code16; }
    static constexpr size_t miller_code_bytes = sizeof(h_miller_code16), final_code_bytes = sizeof(h_final_code16);
};

// Sequential reference executor (host tests): all lanes of a round read before any writes.
template <int TEAM>
inline void vm_run_host(const uint32_t* code, int n_rounds, const Fp2* consts, Fp2* rf_mem) {
    VmRfDense rf{rf_mem};
    for (int r = 0; r < n_rounds; r++) {
        Fp2 res[TEAM];
        bool live[TEAM];
        for (int l = 0; l < TEAM; l++) live[l] = vm_exec(code[r * TEAM + l], rf, consts, res[l]);
        for (int l = 0; l < TEAM; l++)
            if (live[l]) rf.store((code[r * TEAM + l] >> 8) & 0xffu, res[l]);
    }
}

// plain-integer constant table -> Montgomery form
B200_HD void vm_const_to_mont(Fp2& out, const uint32_t limbs[24]) {
    Fp a, b;
#pragma unroll
    for (int i = 0; i < 12; i++) { a.l[i] = limbs[i]; b.l[i] = limbs[12 + i]; }
    fp_to_mont(out.c0, a);
    fp_to_mont(out.c1, b);
}

}  // namespace b200
