// deneb process_epoch on a device-resident state (deneb/spec/mod.rs:965-1003): the per-validator sub-steps as three
// kernels over the Validator records, balances, inactivity scores and both participation lists in HBM.
//   k_epoch_totals    : one pass, one thread per validator; per-CTA partials of every sum the host step needs (active
//                       balance, participating balance per flag, current target balance), the active counts at the current
//                       and next epochs, the ejections and the head of the exit queue.
//   k_epoch_reduce    : one CTA folds the partials and scans the per-CTA ejection counts (an ejection's rank in index order
//                       is its CTA's offset plus its rank inside the CTA).
//   k_epoch_apply     : one thread per validator, in the reference's order: inactivity update, the four (reward, penalty)
//                       pairs, activation eligibility and ejection, the slashing penalty, the effective-balance hysteresis.
//                       Each CTA also leaves its best activation candidates by (activation_eligibility_epoch, index).
//   k_activation_select: one CTA merges the candidates and activates at most MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT.
//   k_epoch_deltas    : one thread per validator, read-only: the four (reward, penalty) pairs k_epoch_apply would add, as
//                       eight lists of n u64 (the spec-test Deltas of source, target, head and the inactivity penalty).
// Everything the kernels compute is integer arithmetic in wrapping u64 (a release build of the reference), decrease_balance
// saturating at zero; the sums are order-independent, so the result does not depend on the launch shape.
#include <cuda_runtime.h>

#include "engine.h"
#include "epoch.h"
#include "records.cuh"

namespace b200 {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxActivations = 8;   // MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT of the mainnet preset, the larger of the two
constexpr uint64_t kFar = ~uint64_t(0);   // FAR_FUTURE_EPOCH; also the "no key" sentinel (no index reaches it)
__device__ __forceinline__ uint64_t flag_weight(int f) { return f == 1 ? 26 : 14; }   // PARTICIPATION_FLAG_WEIGHTS (altair)
constexpr uint64_t kWeightDenominator = 64;
// B200_EPOCH_* bits (include/b200_consensus.h)
constexpr uint32_t kInactivity = 1u << 1, kRewards = 1u << 2, kRegistry = 1u << 3, kSlashings = 1u << 4, kEffective = 1u << 6;

struct BlockPart {
    uint64_t lo[5], hi[5];
    uint64_t key, key_count;         // 1 + largest non-FAR exit epoch of the CTA (0: none), and how many have it
    uint32_t n_cur, n_next, n_eject, pad;
};

__device__ __forceinline__ void add128(uint64_t& lo, uint64_t& hi, uint64_t vlo, uint64_t vhi) {
    lo += vlo;
    hi += vhi + (lo < vlo ? 1 : 0);
}
__device__ __forceinline__ void max_key(uint64_t& k, uint64_t& c, uint64_t k2, uint64_t c2) {
    if (k2 > k) { k = k2; c = c2; }
    else if (k2 == k) c += c2;
}

// the BlockPart of one CTA (or one thread's range) reduced over the CTA; the result is valid in thread 0
template <int NT>
__device__ void reduce_part(BlockPart& v) {
    __shared__ BlockPart s_warp[NT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
#pragma unroll
        for (int k = 0; k < 5; k++)
            add128(v.lo[k], v.hi[k], __shfl_down_sync(0xffffffffu, v.lo[k], d), __shfl_down_sync(0xffffffffu, v.hi[k], d));
        max_key(v.key, v.key_count, __shfl_down_sync(0xffffffffu, v.key, d), __shfl_down_sync(0xffffffffu, v.key_count, d));
        v.n_cur += __shfl_down_sync(0xffffffffu, v.n_cur, d);
        v.n_next += __shfl_down_sync(0xffffffffu, v.n_next, d);
        v.n_eject += __shfl_down_sync(0xffffffffu, v.n_eject, d);
    }
    if (lane == 0) s_warp[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < NT / 32; w++) {
            const BlockPart& o = s_warp[w];
            for (int k = 0; k < 5; k++) add128(v.lo[k], v.hi[k], o.lo[k], o.hi[k]);
            max_key(v.key, v.key_count, o.key, o.key_count);
            v.n_cur += o.n_cur; v.n_next += o.n_next; v.n_eject += o.n_eject;
        }
}

__global__ void __launch_bounds__(kThreads) k_epoch_totals(const uint8_t* __restrict__ recs, const uint8_t* __restrict__ prev_part,
                                                             const uint8_t* __restrict__ cur_part, uint64_t n, uint64_t cur, uint64_t prev,
                                                             uint64_t ejection_balance, BlockPart* __restrict__ parts) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    BlockPart v = {};
    if (i < n) {
        const uint8_t* r = recs + i * 121;
        const uint64_t eb = load_le64_unaligned(r + kRecEffectiveBalance);
        const bool slashed = r[kRecSlashed] != 0;
        const uint64_t act = load_le64_unaligned(r + kRecActivation), exit = load_le64_unaligned(r + kRecExit);
        const bool a_cur = act <= cur && cur < exit, a_prev = act <= prev && prev < exit;
        const uint8_t pf = prev_part[i], cf = cur_part[i];
        v.lo[0] = a_cur ? eb : 0;
#pragma unroll
        for (int f = 0; f < 3; f++) v.lo[1 + f] = (a_prev && !slashed && ((pf >> f) & 1)) ? eb : 0;
        v.lo[4] = (a_cur && !slashed && (cf & 2)) ? eb : 0;
        v.n_cur = a_cur;
        v.n_next = record_active(r, cur + 1);
        v.n_eject = exit == kFar && act <= cur && eb <= ejection_balance;   // active, and not exiting yet
        if (exit != kFar) { v.key = exit + 1; v.key_count = 1; }
    }
    reduce_part<kThreads>(v);
    if (threadIdx.x == 0) parts[blockIdx.x] = v;
}

// one CTA: totals of all CTAs, and eject_off[b] = ejections in CTAs before b
constexpr int kReduceThreads = 512;
__global__ void __launch_bounds__(kReduceThreads) k_epoch_reduce(const BlockPart* __restrict__ parts, uint32_t nb, EpochTotals* __restrict__ out,
                                                         uint64_t* __restrict__ eject_off) {
    __shared__ uint64_t scan[kReduceThreads];
    const uint32_t per = (nb + kReduceThreads - 1) / kReduceThreads;
    const uint32_t lo = threadIdx.x * per, hi = min(nb, lo + per);
    BlockPart v = {};
    uint64_t ej = 0;
    for (uint32_t b = lo; b < hi; b++) {
        const BlockPart& o = parts[b];
        for (int k = 0; k < 5; k++) add128(v.lo[k], v.hi[k], o.lo[k], o.hi[k]);
        max_key(v.key, v.key_count, o.key, o.key_count);
        v.n_cur += o.n_cur; v.n_next += o.n_next;
        ej += o.n_eject;
    }
    scan[threadIdx.x] = ej;
    __syncthreads();
    for (int d = 1; d < kReduceThreads; d <<= 1) {   // Hillis-Steele inclusive scan
        const uint64_t x = threadIdx.x >= d ? scan[threadIdx.x - d] : 0;
        __syncthreads();
        scan[threadIdx.x] += x;
        __syncthreads();
    }
    uint64_t run = threadIdx.x ? scan[threadIdx.x - 1] : 0;
    for (uint32_t b = lo; b < hi; b++) { eject_off[b] = run; run += parts[b].n_eject; }
    // the counts of a range can exceed 32 bits only past 2^32 validators; the u32 fields hold per-CTA values
    reduce_part<kReduceThreads>(v);
    if (threadIdx.x == 0) {
        for (int k = 0; k < 5; k++) { out->lo[k] = v.lo[k]; out->hi[k] = v.hi[k]; }
        out->n_active_cur = v.n_cur;
        out->n_active_next = v.n_next;
        out->n_eject = scan[kReduceThreads - 1];
        out->max_exit_plus1 = v.key;
        out->n_at_max_exit = v.key_count;
    }
}

__device__ __forceinline__ uint64_t sat_sub(uint64_t a, uint64_t b) { return b > a ? 0 : a - b; }

// The terms of get_flag_index_deltas (altair/helpers.rs:265) and get_inactivity_penalty_deltas (bellatrix/helpers.rs:13)
// for one eligible validator, in wrapping u64 as the reference's release build: k_epoch_apply folds them into the balance
// one by one, k_epoch_deltas stores them as the eight lists.
__device__ __forceinline__ uint64_t base_reward(uint64_t eb, const EpochParams& p) { return eb / p.increment * p.base_per_inc; }
__device__ __forceinline__ uint64_t flag_reward(uint64_t base, int f, const EpochParams& p) {
    return base * flag_weight(f) * p.part_inc[f] / (p.active_inc * kWeightDenominator);
}
__device__ __forceinline__ uint64_t flag_penalty(uint64_t base, int f) { return base * flag_weight(f) / kWeightDenominator; }
__device__ __forceinline__ uint64_t inactivity_penalty(uint64_t eb, uint64_t score, const EpochParams& p) {
    return eb * score / p.inactivity_denominator;
}

// (eligibility epoch, index) keys of activation candidates; lexicographic
__device__ __forceinline__ bool key_less(uint64_t e1, uint64_t i1, uint64_t e2, uint64_t i2) {
    return e1 < e2 || (e1 == e2 && i1 < i2);
}
// the smallest key (e, i) among the CTA's valid ones, above (le, li) unless `first`; (kFar, kFar) when none.  All threads.
template <int NT>
__device__ void block_min_above(bool valid, uint64_t e, uint64_t i, bool first, uint64_t le, uint64_t li, uint64_t* out_e,
                                uint64_t* out_i) {
    __shared__ uint64_t s_e[NT / 32], s_i[NT / 32];
    uint64_t be = kFar, bi = kFar;
    if (valid && (first || key_less(le, li, e, i))) { be = e; bi = i; }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const uint64_t oe = __shfl_down_sync(0xffffffffu, be, d), oi = __shfl_down_sync(0xffffffffu, bi, d);
        if (key_less(oe, oi, be, bi)) { be = oe; bi = oi; }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_e[warp] = be; s_i[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < NT / 32; w++)
            if (key_less(s_e[w], s_i[w], be, bi)) { be = s_e[w]; bi = s_i[w]; }
        s_e[0] = be; s_i[0] = bi;
    }
    __syncthreads();
    *out_e = s_e[0];
    *out_i = s_i[0];
    __syncthreads();
}

// append record index i to the changed list (warp-aggregated)
__device__ __forceinline__ void push_changed(bool changed, uint64_t i, uint32_t* list, unsigned long long* count) {
    const uint32_t m = __ballot_sync(0xffffffffu, changed);
    if (!m) return;
    const uint32_t lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(count, static_cast<unsigned long long>(__popc(m)));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (changed) list[base + __popc(m & ((1u << lane) - 1u))] = uint32_t(i);
}

__global__ void __launch_bounds__(kThreads) k_epoch_apply(uint8_t* __restrict__ recs, uint64_t* __restrict__ balances,
                                                            uint64_t* __restrict__ scores, const uint8_t* __restrict__ prev_part,
                                                            uint64_t n, EpochParams p,
                                                            const uint64_t* __restrict__ eject_off, uint64_t* __restrict__ cand_e,
                                                            uint64_t* __restrict__ cand_i, uint32_t* __restrict__ cand_n,
                                                            uint32_t* __restrict__ changed, unsigned long long* __restrict__ n_changed) {
    __shared__ uint32_t warp_ej[kThreads / 32];
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool valid = i < n;
    uint8_t* r = recs + (valid ? i : 0) * 121;
    const uint64_t eb = valid ? load_le64_unaligned(r + kRecEffectiveBalance) : 0;
    const bool slashed = valid && r[kRecSlashed] != 0;
    const uint64_t elig0 = valid ? load_le64_unaligned(r + kRecEligibility) : 0;
    const uint64_t act = valid ? load_le64_unaligned(r + kRecActivation) : kFar;
    const uint64_t exit0 = valid ? load_le64_unaligned(r + kRecExit) : 0;
    const uint64_t wd0 = valid ? load_le64_unaligned(r + kRecWithdrawable) : 0;
    const uint64_t bal0 = valid ? balances[i] : 0, score0 = valid ? scores[i] : 0;
    const uint8_t pf = valid ? prev_part[i] : 0;
    const bool a_prev = act <= p.prev && p.prev < exit0;
    const bool eligible = valid && (a_prev || (slashed && p.prev + 1 < wd0));   // get_eligible_validator_indices
    const bool target = a_prev && !slashed && (pf & 2);
    uint64_t bal = bal0, score = score0;
    // process_inactivity_updates (:1135-1186)
    if ((p.steps & kInactivity) && eligible) {
        if (target) score -= score < 1 ? score : 1;
        else score += p.score_bias;
        if (!p.leak) score -= score < p.score_recovery ? score : p.score_recovery;
    }
    // process_rewards_and_penalties (:1187-1230): flags 0, 1, 2, then the inactivity pair, each applied in turn
    if ((p.steps & kRewards) && eligible) {
        const uint64_t base = base_reward(eb, p);
#pragma unroll
        for (int f = 0; f < 3; f++) {
            if (a_prev && !slashed && ((pf >> f) & 1)) {
                if (!p.leak) bal += flag_reward(base, f, p);
            } else if (f != 2) {
                bal = sat_sub(bal, flag_penalty(base, f));
            }
        }
        if (!target) bal = sat_sub(bal, inactivity_penalty(eb, score, p));
    }
    // process_registry_updates (deneb/epoch_processing.rs:11-55): eligibility, then ejection through the exit queue's
    // closed form (the k-th ejection in index order, k = eject_off[cta] + rank in the CTA)
    uint64_t elig = elig0, exit = exit0, wd = wd0;
    bool rec_changed = false;
    const bool ej = valid && (p.steps & kRegistry) && exit0 == kFar && act <= p.cur && eb <= p.ejection_balance;
    {
        const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const uint32_t m = __ballot_sync(0xffffffffu, ej);
        if (lane == 0) warp_ej[warp] = __popc(m);
        __syncthreads();
        if (ej) {
            uint64_t k = eject_off[blockIdx.x] + __popc(m & ((1u << lane) - 1u));
            for (uint32_t w = 0; w < warp; w++) k += warp_ej[w];
            exit = p.c0 < p.churn ? p.exit0 + (p.c0 + k) / p.churn : p.exit0 + 1 + k / p.churn;
            wd = exit + p.withdraw_delay;
            rec_changed = true;
        }
    }
    if (valid && (p.steps & kRegistry) && elig0 == kFar && eb == p.max_effective) {
        elig = p.cur + 1;
        rec_changed = true;
    }
    // process_slashings (:1005-1050), withdrawable_epoch as the registry step left it
    if (valid && (p.steps & kSlashings) && slashed && p.slash_epoch == wd)
        bal = sat_sub(bal, eb / p.increment * p.adjusted_slashing / p.total_active * p.increment);
    // process_effective_balance_updates (:1329-1350)
    uint64_t neb = eb;
    if (valid && (p.steps & kEffective) && (bal + p.hysteresis_down < eb || eb + p.hysteresis_up < bal)) {
        neb = bal - bal % p.increment;
        if (neb > p.max_effective) neb = p.max_effective;
        rec_changed = rec_changed || neb != eb;
    }
    if (valid) {
        if (bal != bal0) balances[i] = bal;
        if (score != score0) scores[i] = score;
        if (neb != eb) store_le64_unaligned(r + kRecEffectiveBalance, neb);
        if (elig != elig0) store_le64_unaligned(r + kRecEligibility, elig);
        if (exit != exit0) {
            store_le64_unaligned(r + kRecExit, exit);
            store_le64_unaligned(r + kRecWithdrawable, wd);
        }
    }
    push_changed(rec_changed, i, changed, n_changed);
    // this CTA's first activation_limit candidates of the queue (is_eligible_for_activation after the first loop)
    const bool cand = valid && p.activation_limit && elig <= p.finalized_epoch && act == kFar;
    const int nc = __syncthreads_count(cand);
    const uint32_t take = min(uint32_t(nc), p.activation_limit);
    uint64_t le = 0, li = 0;
    for (uint32_t k = 0; k < take; k++) {
        uint64_t be, bi;
        block_min_above<kThreads>(cand, elig, i, k == 0, le, li, &be, &bi);
        if (threadIdx.x == 0) { cand_e[uint64_t(blockIdx.x) * kMaxActivations + k] = be; cand_i[uint64_t(blockIdx.x) * kMaxActivations + k] = bi; }
        le = be; li = bi;
    }
    if (threadIdx.x == 0) cand_n[blockIdx.x] = take;
}

// one CTA: the first `limit` keys of all CTAs' candidate lists get activation_epoch
__global__ void __launch_bounds__(1024) k_activation_select(uint8_t* __restrict__ recs, const uint64_t* __restrict__ cand_e,
                                                              const uint64_t* __restrict__ cand_i, const uint32_t* __restrict__ cand_n,
                                                              uint32_t nb, uint32_t limit, uint64_t activation_epoch,
                                                              uint32_t* __restrict__ changed, unsigned long long* __restrict__ n_changed) {
    uint64_t le = 0, li = 0;
    for (uint32_t k = 0; k < limit; k++) {
        uint64_t be = kFar, bi = kFar;   // this thread's smallest key above the last one taken
        for (uint32_t b = threadIdx.x; b < nb; b += 1024)
            for (uint32_t j = 0; j < cand_n[b]; j++) {
                const uint64_t ce = cand_e[uint64_t(b) * kMaxActivations + j], ci = cand_i[uint64_t(b) * kMaxActivations + j];
                if ((k == 0 || key_less(le, li, ce, ci)) && key_less(ce, ci, be, bi)) { be = ce; bi = ci; }
            }
        block_min_above<1024>(bi != kFar, be, bi, true, 0, 0, &le, &li);
        if (li == kFar) break;   // the queue is shorter than the limit
        if (threadIdx.x == 0) {
            store_le64_unaligned(recs + li * 121 + kRecActivation, activation_epoch);
            changed[atomicAdd(n_changed, 1ull)] = uint32_t(li);
        }
    }
}

// The pairs k_epoch_apply adds, without applying them (process_rewards_and_penalties' order and conditions, on the terms
// above).  List-major: out[2 k n + i] the reward and out[(2 k + 1) n + i] the penalty of pair k for validator i, so that
// each of the eight stores of a warp is one coalesced 256-byte segment.
__global__ void __launch_bounds__(kThreads) k_epoch_deltas(const uint8_t* __restrict__ recs, const uint64_t* __restrict__ scores,
                                                             const uint8_t* __restrict__ part, uint64_t n, EpochParams p,
                                                             uint64_t* __restrict__ out) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* r = recs + i * 121;
    const uint64_t eb = load_le64_unaligned(r + kRecEffectiveBalance);
    const bool slashed = r[kRecSlashed] != 0;
    const uint64_t act = load_le64_unaligned(r + kRecActivation), exit = load_le64_unaligned(r + kRecExit);
    const uint64_t wd = load_le64_unaligned(r + kRecWithdrawable);
    const uint8_t pf = part[i];
    const bool a_prev = act <= p.prev && p.prev < exit;
    uint64_t d[8] = {};   // pair k: d[2 k] reward, d[2 k + 1] penalty; zero for a validator that is not eligible
    if (a_prev || (slashed && p.prev + 1 < wd)) {   // get_eligible_validator_indices
        const uint64_t base = base_reward(eb, p);
#pragma unroll
        for (int f = 0; f < 3; f++) {
            if (a_prev && !slashed && ((pf >> f) & 1)) {
                if (!p.leak) d[2 * f] = flag_reward(base, f, p);
            } else if (f != 2) {
                d[2 * f + 1] = flag_penalty(base, f);
            }
        }
        if (!(a_prev && !slashed && (pf & 2))) d[7] = inactivity_penalty(eb, scores[i], p);
    }
#pragma unroll
    for (int k = 0; k < 8; k++) out[k * n + i] = d[k];
}

struct EpochScratch {
    DevBuf parts, totals, eject_off, cand_e, cand_i, cand_n, changed, n_changed, deltas;
};
EpochScratch g_ep;

}  // namespace

int32_t epoch_totals_on_device(Engine& e, const uint8_t* recs, const uint8_t* prev_part, const uint8_t* cur_part, uint64_t n,
                               uint64_t cur, uint64_t prev, uint64_t ejection_balance, EpochTotals* out) {
    *out = EpochTotals{};
    if (n == 0) return B200_SUCCESS;
    const uint32_t nb = uint32_t((n + kThreads - 1) / kThreads);
    B200_CUDA_TRY(g_ep.parts.reserve(size_t(nb) * sizeof(BlockPart)));
    B200_CUDA_TRY(g_ep.totals.reserve(sizeof(EpochTotals)));
    B200_CUDA_TRY(g_ep.eject_off.reserve(size_t(nb) * 8));
    B200_CUDA_TRY(e.staging.reserve(sizeof(EpochTotals)));
    cudaStream_t s = e.stream;
    k_epoch_totals<<<nb, kThreads, 0, s>>>(recs, prev_part, cur_part, n, cur, prev, ejection_balance,
                                           static_cast<BlockPart*>(g_ep.parts.p));
    k_epoch_reduce<<<1, kReduceThreads, 0, s>>>(static_cast<const BlockPart*>(g_ep.parts.p), nb, static_cast<EpochTotals*>(g_ep.totals.p),
                                      static_cast<uint64_t*>(g_ep.eject_off.p));
    e.launches += 2;
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaMemcpyAsync(e.staging.p, g_ep.totals.p, sizeof(EpochTotals), cudaMemcpyDeviceToHost, s));
    B200_CUDA_TRY(cudaStreamSynchronize(s));
    *out = *static_cast<const EpochTotals*>(e.staging.p);
    return B200_SUCCESS;
}

int32_t epoch_apply_on_device(Engine& e, uint8_t* recs, uint64_t* balances, uint64_t* scores, const uint8_t* prev_part,
                              uint64_t n, const EpochParams& p, const uint32_t** changed_dev,
                              uint64_t* n_changed) {
    *n_changed = 0;
    *changed_dev = nullptr;
    if (n == 0) return B200_SUCCESS;
    if (p.activation_limit > kMaxActivations) { e.last_error = "process_epoch: activation churn above 8"; return B200_ERR_BAD_ARG; }
    const uint32_t nb = uint32_t((n + kThreads - 1) / kThreads);
    B200_CUDA_TRY(g_ep.cand_e.reserve(size_t(nb) * kMaxActivations * 8));
    B200_CUDA_TRY(g_ep.cand_i.reserve(size_t(nb) * kMaxActivations * 8));
    B200_CUDA_TRY(g_ep.cand_n.reserve(size_t(nb) * 4));
    B200_CUDA_TRY(g_ep.changed.reserve(size_t(n + kMaxActivations) * 4));
    B200_CUDA_TRY(g_ep.n_changed.reserve(8));
    B200_CUDA_TRY(e.staging.reserve(8));
    cudaStream_t s = e.stream;
    auto* cnt = static_cast<unsigned long long*>(g_ep.n_changed.p);
    B200_CUDA_TRY(cudaMemsetAsync(cnt, 0, 8, s));
    k_epoch_apply<<<nb, kThreads, 0, s>>>(recs, balances, scores, prev_part, n, p,
                                          static_cast<const uint64_t*>(g_ep.eject_off.p), static_cast<uint64_t*>(g_ep.cand_e.p),
                                          static_cast<uint64_t*>(g_ep.cand_i.p), static_cast<uint32_t*>(g_ep.cand_n.p),
                                          static_cast<uint32_t*>(g_ep.changed.p), cnt);
    e.launches++;
    if (p.activation_limit) {
        k_activation_select<<<1, 1024, 0, s>>>(recs, static_cast<const uint64_t*>(g_ep.cand_e.p), static_cast<const uint64_t*>(g_ep.cand_i.p),
                                               static_cast<const uint32_t*>(g_ep.cand_n.p), nb, p.activation_limit, p.activation_epoch,
                                               static_cast<uint32_t*>(g_ep.changed.p), cnt);
        e.launches++;
    }
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaMemcpyAsync(e.staging.p, cnt, 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA_TRY(cudaStreamSynchronize(s));
    *n_changed = *static_cast<const uint64_t*>(e.staging.p);
    *changed_dev = static_cast<const uint32_t*>(g_ep.changed.p);
    return B200_SUCCESS;
}

int32_t epoch_deltas_on_device(Engine& e, const uint8_t* recs, const uint64_t* scores, const uint8_t* part, uint64_t n,
                               const EpochParams& p, const uint64_t** out_dev) {
    *out_dev = nullptr;
    if (n == 0) return B200_SUCCESS;
    const uint32_t nb = uint32_t((n + kThreads - 1) / kThreads);
    B200_CUDA_TRY(g_ep.deltas.reserve(size_t(n) * 64));
    k_epoch_deltas<<<nb, kThreads, 0, e.stream>>>(recs, scores, part, n, p, static_cast<uint64_t*>(g_ep.deltas.p));
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    *out_dev = static_cast<const uint64_t*>(g_ep.deltas.p);
    return B200_SUCCESS;
}

}  // namespace b200
