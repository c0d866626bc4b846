// Lane-parallel pairing kernels: a TEAM of 8 or 16 lanes per (G1, G2) pair / per tuple replays the statically
// scheduled Fp2 programs of tools/gen_pairing_vm.py (Miller loop, final exponentiation) on a shared-memory register
// file.  Every verification call pairs here.  One thread per pair, as bls_pairing.cu's reference kernels run, would expose
// only 2T threads (a latency floor of tens of ms at T = 4096); here 16x more lanes work on the same tuples, products stay
// inlined PTX.
#include <cuda_runtime.h>

#include <algorithm>

#include "bls_kernels.cuh"
#include "pairing_vm.cuh"

namespace b200 {
namespace {

__global__ void k_vm_consts(const uint32_t* __restrict__ plain, Fp2* __restrict__ out) {
    const int i = threadIdx.x;
    if (i < kVmConsts) {
        uint32_t l[24];
        for (int k = 0; k < 24; k++) l[k] = plain[i * 24 + k];
        Fp2 v;
        vm_const_to_mont(v, l);
        out[i] = v;
    }
}

struct VmOuts { int v[6]; };   // register-file slots of a program's six output coefficients (w-power order)

template <int TEAM>
__device__ __forceinline__ void vm_run(const uint32_t* __restrict__ code, int n_rounds, const Fp2* __restrict__ consts,
                                       const VmRfStrided& rf, uint32_t lane, bool active) {
    // the next round's instruction word is fetched while the current round executes: with one or two warps per scheduler
    // (small batches) the load's latency would otherwise sit on the critical path of every one of the ~2 500 / ~3 800 rounds
    // A warp with no live team (failed or padding tuples) skips the rounds; all its lanes leave together.
    if (!__any_sync(~0u, active)) return;
    uint32_t w = __ldg(code + lane);
#pragma unroll 1
    for (int r = 0; r < n_rounds; r++) {
        const uint32_t w_next = (r + 1 < n_rounds) ? __ldg(code + (r + 1) * TEAM + lane) : 0u;
        if (active && (w & 0xffu) != VM_NOP) {
            Fp2 res;
            vm_exec(w, rf, consts, res);
            rf.store((w >> 8) & 0xffu, res);
        }
        __syncwarp();
        w = w_next;
    }
}

__device__ __forceinline__ bool tuple_dead(uint32_t t, const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code) {
    return pk_code[t] != BLS_SUCCESS || flags[t] != 0 || sig_code[t] != SIG_OK;
}

// one team per pair
template <int TEAM>
__global__ void __launch_bounds__(128) k_vm_miller(const uint32_t* __restrict__ code, const Fp2* __restrict__ consts,
                                                    const G1Pre* __restrict__ g1, const uint32_t* __restrict__ g1_idx,
                                                    const G2Aff* __restrict__ g2, const uint32_t* __restrict__ g2_idx,
                                                    const uint32_t* __restrict__ pair_tuple, const int32_t* __restrict__ pk_code,
                                                    const uint32_t* __restrict__ flags, const int32_t* __restrict__ sig_code,
                                                    uint32_t n_pairs, Fp12* __restrict__ f, int n_rounds, int n_slots, VmOuts outs6) {
    extern __shared__ uint32_t smem[];
    const uint32_t team_in_block = threadIdx.x / TEAM, lane = threadIdx.x % TEAM;
    const uint32_t i = blockIdx.x * (blockDim.x / TEAM) + team_in_block;
    VmRfStrided rf{smem + team_in_block * vm_team_words(uint32_t(n_slots))};
    bool active = i < n_pairs && !tuple_dead(pair_tuple[i], pk_code, flags, sig_code);
    bool trivial = false;  // a point at infinity: the pair contributes 1
    if (active) {
        const G1Pre* p = g1 + g1_idx[i];
        const G2Aff* q = g2 + g2_idx[i];
        trivial = p->inf || q->inf;
        if (!trivial) {  // program inputs: slots 0..4 = X Z, Y, Z^3 (as Fp2 with c1 = 0), Qx, Qy
            if (lane == 0) { Fp2 v; v.c0 = p->xz; v.c1 = fp_zero(); rf.store(0, v); }
            if (lane == 1) { Fp2 v; v.c0 = p->y; v.c1 = fp_zero(); rf.store(1, v); }
            if (lane == 2) { Fp2 v; v.c0 = p->z3; v.c1 = fp_zero(); rf.store(2, v); }
            if (lane == 3) rf.store(3, q->x);
            if (lane == 4) rf.store(4, q->y);
        }
    }
    __syncwarp();
    vm_run<TEAM>(code, n_rounds, consts, rf, lane, active && !trivial);
    static_assert(TEAM >= 6, "team must cover the six output coefficients");
    if (active && lane < 6) {
        // w-power order of the program outputs -> tower slots c0.c0, c1.c0, c0.c1, c1.c1, c0.c2, c1.c2
        Fp2 v;
        if (trivial) v = (lane == 0) ? fp2_one() : fp2_zero();
        else v = rf.load(uint32_t(outs6.v[lane]));
        Fp2* dst = reinterpret_cast<Fp2*>(f + i);
        const int tower_pos[6] = {0, 3, 1, 4, 2, 5};  // Fp12 memory order: c0.{c0,c1,c2}, c1.{c0,c1,c2}
        dst[tower_pos[lane]] = v;
    }
}

// one team per tuple (two Miller values per tuple: pairs pair_off[t], pair_off[t]+1)
// STORE (self-test only, b200_pairing_eval): also write the program's six outputs to f_out[t] in Fp12 memory order
template <int TEAM, bool STORE = false>
__global__ void __launch_bounds__(128) k_vm_final(const uint32_t* __restrict__ code, const Fp2* __restrict__ consts,
                                                  const Fp12* __restrict__ f, const uint32_t* __restrict__ pair_off,
                                                  const int32_t* __restrict__ pk_code, const uint32_t* __restrict__ flags,
                                                  const int32_t* __restrict__ sig_code, uint32_t n_tuples,
                                                  int32_t* __restrict__ out_codes, int n_rounds, int n_slots, VmOuts outs6,
                                                  Fp12* __restrict__ f_out = nullptr) {
    extern __shared__ uint32_t smem[];
    const uint32_t team_in_block = threadIdx.x / TEAM, lane = threadIdx.x % TEAM;
    const uint32_t t = blockIdx.x * (blockDim.x / TEAM) + team_in_block;
    VmRfStrided rf{smem + team_in_block * vm_team_words(uint32_t(n_slots))};
    int32_t code_out = BLS_SUCCESS;
    bool active = false;
    if (t < n_tuples) {
        if (pk_code[t] != BLS_SUCCESS) code_out = pk_code[t];
        else if (sig_code[t] > 0) code_out = sig_code[t];
        else if (flags[t] != 0 || sig_code[t] == SIG_NOT_IN_GROUP) code_out = BLS_VERIFY_FAIL;
        else active = true;
    }
    if (active) {
        const int tower_pos[6] = {0, 3, 1, 4, 2, 5};
        for (uint32_t k = lane; k < 12; k += TEAM) {
            const Fp2* src = reinterpret_cast<const Fp2*>(f + pair_off[t] + k / 6);
            rf.store(k, src[tower_pos[k % 6]]);
        }
    }
    __syncwarp();
    vm_run<TEAM>(code, n_rounds, consts, rf, lane, active);
    if (STORE && active && lane < 6) {
        const int tower_pos[6] = {0, 3, 1, 4, 2, 5};
        reinterpret_cast<Fp2*>(f_out + t)[tower_pos[lane]] = rf.load(uint32_t(outs6.v[lane]));
    }
    if (t < n_tuples && lane == 0) {
        if (active) {
            bool one = fp2_eq(rf.load(uint32_t(outs6.v[0])), fp2_one());
#pragma unroll 1
            for (int k = 1; k < 6; k++) one = one && fp2_is_zero(rf.load(uint32_t(outs6.v[k])));
            code_out = one ? BLS_SUCCESS : BLS_VERIFY_FAIL;
        }
        out_codes[t] = code_out;
    }
}

}  // namespace

// The scheduled programs live on the device as data: [0] teams of 8 lanes, [1] teams of 16.  The compiled-in defaults come
// from pairing_vm_prog*.cuh; vm_load_programs() swaps in another schedule of the same formulas at run time (schedule
// tuning: tools/gen_pairing_vm.py --blob writes one after its numeric self-check; the GPU parity tests then pin it).
struct VmProgramDev {
    uint32_t* d_code = nullptr;
    int rounds = 0, slots = 0;
    VmOuts outs{};
};
static VmProgramDev g_miller_prog[2], g_final_prog[2];
static Fp2* g_d_consts = nullptr;
// Batches with at most this many teams' worth of work run on 16-lane teams: they cannot fill the machine anyway, so the
// shorter critical path (1 918 / 3 094 rounds instead of 2 493 / 3 842) wins; above it the 8-lane programs' higher
// throughput does.  b200_tune("vm_team16_max") / B200_VM_TEAM16_MAX overrides (0: never).
static uint32_t g_team16_max = 2048;
// threads per CTA of the VM kernels (32 | 64 | 128): teams never synchronise across warps, so this only sets how finely the
// shared-memory register files pack an SM and how the last wave spreads (b200_tune("vm_cta") / B200_VM_CTA)
static int g_vm_cta = 32;   // the registry step was fastest with 32-thread CTAs at T = 2048 and 4096
void set_vm_team16_max(uint32_t n) { g_team16_max = n; }
void set_vm_cta(int threads) { if (threads == 32 || threads == 64 || threads == 128) g_vm_cta = threads; }

static int vm_set_program(VmProgramDev& p, const uint32_t* code, size_t bytes, int rounds, int slots, const int* outs, cudaStream_t st) {
    uint32_t* d = nullptr;
    if (cudaMalloc(&d, bytes) != cudaSuccess) return 1;
    if (cudaMemcpyAsync(d, code, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return 1;
    if (cudaStreamSynchronize(st) != cudaSuccess) return 1;   // `code` may be a caller buffer
    if (p.d_code) cudaFree(p.d_code);
    p.d_code = d; p.rounds = rounds; p.slots = slots;
    for (int k = 0; k < 6; k++) p.outs.v[k] = outs[k];
    return 0;
}
template <int TEAM>
static int vm_upload(int slot, cudaStream_t st) {
    typedef VmProg<TEAM> P;
    if (vm_set_program(g_miller_prog[slot], P::miller_code(), P::miller_code_bytes, P::miller_rounds, P::miller_slots, P::miller_out, st)) return 1;
    if (vm_set_program(g_final_prog[slot], P::final_code(), P::final_code_bytes, P::final_rounds, P::final_slots, P::final_out, st)) return 1;
    // any schedule that fits an SM's shared memory may be loaded later
    cudaFuncSetAttribute(k_vm_miller<TEAM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kVmMaxSmemBytes);
    cudaFuncSetAttribute(k_vm_final<TEAM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kVmMaxSmemBytes);
    cudaFuncSetAttribute(k_vm_final<TEAM, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kVmMaxSmemBytes);
    return 0;
}

// blob: [magic, team, m_rounds, m_slots, m_out x6, f_rounds, f_slots, f_out x6, m_code (m_rounds x team), f_code (f_rounds x team)]
int vm_load_programs(const uint32_t* blob, size_t n_words, void* stream) {
    if (!blob || n_words < 18 || blob[0] != kVmBlobMagic) return 1;
    const uint32_t team = blob[1], mr = blob[2], ms = blob[3], fr = blob[10], fs = blob[11];
    if (team != 8 && team != 16) return 1;
    if (!mr || !fr || mr > (1u << 20) || fr > (1u << 20) || ms < 12 || fs < 12 || ms > 255 || fs > 255) return 1;
    if (n_words != 18 + size_t(mr) * team + size_t(fr) * team) return 1;
    // one team's register file must fit a CTA's shared memory at the smallest CTA (one warp)
    if (size_t(32 / team) * vm_team_words(std::max(ms, fs)) * 4 > size_t(kVmMaxSmemBytes)) return 1;
    auto check = [&](const uint32_t* code, uint32_t rounds, uint32_t slots, const uint32_t* outs) {
        for (int k = 0; k < 6; k++) if (outs[k] >= slots) return false;
        for (size_t i = 0; i < size_t(rounds) * team; i++) {
            const uint32_t w = code[i], op = w & 0xffu, d = (w >> 8) & 0xffu, a = (w >> 16) & 0xffu, b = w >> 24;
            if (op > VM_LDC) return false;
            if (op == VM_NOP) continue;
            if (d >= slots) return false;
            if (op == VM_LDC) { if (a >= uint32_t(kVmConsts)) return false; continue; }
            if (a >= slots) return false;
            const bool binary = op == VM_MUL || op == VM_MULFP || op == VM_ADD || op == VM_SUB;
            if (binary && b >= slots) return false;
        }
        return true;
    };
    const uint32_t* mcode = blob + 18;
    const uint32_t* fcode = mcode + size_t(mr) * team;
    if (!check(mcode, mr, ms, blob + 4) || !check(fcode, fr, fs, blob + 12)) return 1;
    int mo[6], fo[6];
    for (int k = 0; k < 6; k++) { mo[k] = int(blob[4 + k]); fo[k] = int(blob[12 + k]); }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int slot = team == 8 ? 0 : 1;
    if (vm_set_program(g_miller_prog[slot], mcode, size_t(mr) * team * 4, int(mr), int(ms), mo, st)) return 1;
    if (vm_set_program(g_final_prog[slot], fcode, size_t(fr) * team * 4, int(fr), int(fs), fo, st)) return 1;
    return 0;
}

int vm_init(void* stream) {
    if (g_d_consts) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint32_t* d_plain = nullptr;
    if (vm_upload<8>(0, st) || vm_upload<16>(1, st)) return 1;
    if (cudaMalloc(&g_d_consts, sizeof(Fp2) * kVmConsts) != cudaSuccess) return 1;
    if (cudaMalloc(&d_plain, sizeof(h_vm_consts)) != cudaSuccess) return 1;
    cudaMemcpyAsync(d_plain, h_vm_consts, sizeof(h_vm_consts), cudaMemcpyHostToDevice, st);
    k_vm_consts<<<1, 32, 0, st>>>(d_plain, g_d_consts);
    if (cudaStreamSynchronize(st) != cudaSuccess) return 1;
    cudaFree(d_plain);
    return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

template <int TEAM>
static void launch_vm_miller_t(int slot, const G1Pre* g1, const uint32_t* g1_idx, const G2Aff* g2, const uint32_t* g2_idx,
                               const uint32_t* pair_tuple, const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code,
                               uint32_t n_pairs, Fp12* f, cudaStream_t st) {
    const VmProgramDev& p = g_miller_prog[slot];
    int threads = g_vm_cta;
    while (threads > 32 && size_t(threads / TEAM) * vm_team_words(uint32_t(p.slots)) * 4 > size_t(kVmMaxSmemBytes)) threads >>= 1;
    const int teams = threads / TEAM;
    const size_t smem = size_t(teams) * vm_team_words(uint32_t(p.slots)) * 4;
    k_vm_miller<TEAM><<<(n_pairs + teams - 1) / teams, threads, smem, st>>>(
        p.d_code, g_d_consts, g1, g1_idx, g2, g2_idx, pair_tuple, pk_code, flags, sig_code, n_pairs, f, p.rounds, p.slots, p.outs);
}
template <int TEAM, bool STORE = false>
static void launch_vm_final_t(int slot, const Fp12* f, const uint32_t* pair_off, const int32_t* pk_code, const uint32_t* flags,
                              const int32_t* sig_code, uint32_t n_tuples, int32_t* out_codes, cudaStream_t st,
                              Fp12* f_out = nullptr) {
    const VmProgramDev& p = g_final_prog[slot];
    int threads = g_vm_cta;
    while (threads > 32 && size_t(threads / TEAM) * vm_team_words(uint32_t(p.slots)) * 4 > size_t(kVmMaxSmemBytes)) threads >>= 1;
    const int teams = threads / TEAM;
    const size_t smem = size_t(teams) * vm_team_words(uint32_t(p.slots)) * 4;
    k_vm_final<TEAM, STORE><<<(n_tuples + teams - 1) / teams, threads, smem, st>>>(
        p.d_code, g_d_consts, f, pair_off, pk_code, flags, sig_code, n_tuples, out_codes, p.rounds, p.slots, p.outs, f_out);
}

void launch_vm_miller(const G1Pre* g1, const uint32_t* g1_idx, const G2Aff* g2, const uint32_t* g2_idx,
                      const uint32_t* pair_tuple, const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code,
                      uint32_t n_pairs, Fp12* f, void* stream) {
    if (!n_pairs) return;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n_pairs <= g_team16_max) launch_vm_miller_t<16>(1, g1, g1_idx, g2, g2_idx, pair_tuple, pk_code, flags, sig_code, n_pairs, f, st);
    else launch_vm_miller_t<8>(0, g1, g1_idx, g2, g2_idx, pair_tuple, pk_code, flags, sig_code, n_pairs, f, st);
}
void launch_vm_final(const Fp12* f, const uint32_t* pair_off, const int32_t* pk_code, const uint32_t* flags,
                     const int32_t* sig_code, uint32_t n_tuples, int32_t* out_codes, void* stream) {
    if (!n_tuples) return;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n_tuples <= g_team16_max) launch_vm_final_t<16>(1, f, pair_off, pk_code, flags, sig_code, n_tuples, out_codes, st);
    else launch_vm_final_t<8>(0, f, pair_off, pk_code, flags, sig_code, n_tuples, out_codes, st);
}

void launch_vm_miller_team(int team, const G1Pre* g1, const uint32_t* idx, const G2Aff* g2, const uint32_t* zeros, uint32_t n,
                           Fp12* f, void* stream) {
    if (!n) return;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int32_t* z = reinterpret_cast<const int32_t*>(zeros);
    if (team == 16) launch_vm_miller_t<16>(1, g1, idx, g2, idx, zeros, z, zeros, z, n, f, st);
    else launch_vm_miller_t<8>(0, g1, idx, g2, idx, zeros, z, zeros, z, n, f, st);
}
void launch_vm_final_team(int team, const Fp12* f, const uint32_t* pair_off, const uint32_t* zeros, uint32_t n, Fp12* f_out,
                          int32_t* codes, void* stream) {
    if (!n) return;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int32_t* z = reinterpret_cast<const int32_t*>(zeros);
    if (team == 16) launch_vm_final_t<16, true>(1, f, pair_off, z, zeros, z, n, codes, st, f_out);
    else launch_vm_final_t<8, true>(0, f, pair_off, z, zeros, z, n, codes, st, f_out);
}

}  // namespace b200
