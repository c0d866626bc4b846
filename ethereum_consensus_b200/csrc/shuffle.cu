// Committee shuffling on the device (SURVEY.md §8f-3): the step immediately BEFORE the BLS hot path — every
// `process_attestation` resolves its committee through `get_beacon_committee`
// (ethereum-consensus/src/phase0/helpers.rs:775-806), which scans the registry for active validators
// (:646-676) and runs the 90-round swap-or-not shuffle (:249-283 per index, :287-360 for a whole list).
//
// Device formulation (not the reference's in-place swap walk, which is inherently sequential):
//   k_shuffle_sources : every SHA-256 the shuffle can need is independent of the data: for each round r the pivot
//                       hash(seed || r) and one "source" block hash(seed || r || le32(b)) per 256 positions —
//                       rounds x (ceil(n/256) + 1) single-block hashes, one thread each (ALU-pipe bound).
//   k_shuffle_map     : one thread per OUTPUT position i runs the forward per-index map of `compute_shuffled_index`
//                       (90 dependent steps: flip, position = max(index, flip), one bit of the source table) and
//                       writes out[i] = indices[map(i)] — exactly `compute_committee`'s definition, and equal to the
//                       list walk `compute_shuffled_indices` produces (tests pin both formulations against each other).
//                       The source table (rounds x n/8 bytes: 11.8 MB at n = 2^20) is L2-resident; the kernel is bound
//                       by dependent L2 gathers, not by HBM.
//   k_active_*        : `get_active_validator_indices` as an order-preserving stream compaction over the 121-byte
//                       Validator records (activation_epoch <= epoch < exit_epoch, phase0/validator.rs:10-26).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "engine.h"
#include "records.cuh"
#include "sha256.cuh"
#include "shuffle.h"

namespace b200 {
namespace {

constexpr int kThreads = 256;

// SHA-256 of seed(32) || extra[0..n_extra) for n_extra <= 5: one padded block
__device__ __forceinline__ void sha256_seed_plus(const uint32_t seed_w[8], uint32_t round, uint32_t pos_block, bool with_pos, uint32_t out[8]) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = seed_w[i];
    if (with_pos) {   // 37 bytes: seed | round | le32(pos_block) | 0x80
        w[8] = (round << 24) | ((pos_block & 0xffu) << 16) | (((pos_block >> 8) & 0xffu) << 8) | ((pos_block >> 16) & 0xffu);
        w[9] = ((pos_block >> 24) << 24) | 0x00800000u;
        w[15] = 37 * 8;
    } else {          // 33 bytes: seed | round | 0x80
        w[8] = (round << 24) | 0x00800000u;
        w[9] = 0;
        w[15] = 33 * 8;
    }
#pragma unroll
    for (int i = 10; i < 15; i++) w[i] = 0;
    sha256_init(out);
    sha256_compress(out, w);
}

// grid covers rounds x (nblk + 1): slot b < nblk -> source block b; slot nblk -> the round's pivot
__global__ void __launch_bounds__(kThreads) k_shuffle_sources(const uint32_t* __restrict__ seed_words, uint32_t rounds, uint32_t nblk,
                                                                uint64_t n, uint32_t* __restrict__ sources, uint64_t* __restrict__ pivots) {
    const uint64_t t = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const uint64_t per = uint64_t(nblk) + 1;
    if (t >= per * rounds) return;
    const uint32_t r = uint32_t(t / per), b = uint32_t(t % per);
    uint32_t sw[8], h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) sw[i] = seed_words[i];
    if (b == nblk) {
        sha256_seed_plus(sw, r, 0, false, h);
        // first 8 digest bytes as a little-endian u64
        const uint64_t v = uint64_t(bswap32(h[0])) | (uint64_t(bswap32(h[1])) << 32);
        pivots[r] = v % n;
    } else {
        sha256_seed_plus(sw, r, b, true, h);
        uint32_t* dst = sources + (uint64_t(r) * nblk + b) * 8;
#pragma unroll
        for (int i = 0; i < 8; i++) dst[i] = h[i];
    }
}

// One round of compute_shuffled_index (phase0/helpers.rs:249-283): flip = (pivot + n - idx) mod n, position =
// max(idx, flip), and idx moves to flip when bit (position % 8) of byte (position % 256) / 8 of the round's source block
// position / 256 is set.  `source_word(position)` returns the big-endian digest word (position % 256) / 32 of that block:
// a table lookup in the list shuffle, a hash on demand in the candidate sampler.
template <class Idx, class SourceWord>
__device__ __forceinline__ Idx shuffle_round(Idx idx, Idx pivot, Idx nn, SourceWord source_word) {
    Idx flip = pivot + (nn - idx);          // in (0, 2n): fits u32 for n <= 2^31
    if (flip >= nn) flip -= nn;
    const Idx pos = idx > flip ? idx : flip;
    const uint32_t word = source_word(pos);
    const uint32_t byte_in_word = (uint32_t(pos) & 31u) >> 3;
    const uint32_t bit = (word >> (24u - 8u * byte_in_word + (uint32_t(pos) & 7u))) & 1u;
    return bit ? flip : idx;
}

template <class Idx>
__global__ void __launch_bounds__(kThreads) k_shuffle_map(const uint64_t* __restrict__ indices, uint64_t n, uint32_t rounds, uint32_t nblk,
                                                            const uint32_t* __restrict__ sources, const uint64_t* __restrict__ pivots,
                                                            uint64_t* __restrict__ out) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Idx idx = Idx(i);
    const Idx nn = Idx(n);
#pragma unroll 1
    for (uint32_t r = 0; r < rounds; r++)
        idx = shuffle_round(idx, Idx(pivots[r]), nn, [&](Idx pos) {
            return __ldg(sources + (uint64_t(r) * nblk + uint64_t(pos >> 8)) * 8 + ((uint32_t(pos) & 255u) >> 5));
        });
    out[i] = indices ? indices[idx] : uint64_t(idx);
}

// is_active_validator(v, epoch) over the records (records.cuh)
__global__ void __launch_bounds__(kThreads) k_active_count(const uint8_t* __restrict__ recs, uint64_t n, uint64_t epoch,
                                                             uint32_t* __restrict__ block_counts) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    bool act = false;
    if (i < n) {
        act = record_active(recs + i * 121, epoch);
    }
    const int c = __syncthreads_count(act ? 1 : 0);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = uint32_t(c);
}
// exclusive scan of the per-block counts by one CTA (n_blocks <= a few thousand); total -> block_off[n_blocks]
__global__ void __launch_bounds__(1024) k_active_scan(const uint32_t* __restrict__ block_counts, uint32_t n_blocks, uint64_t* __restrict__ block_off) {
    __shared__ uint64_t part[1024];
    const uint32_t per = (n_blocks + 1023) / 1024;
    const uint32_t lo = threadIdx.x * per, hi = min(n_blocks, lo + per);
    uint64_t s = 0;
    for (uint32_t k = lo; k < hi; k++) s += block_counts[k];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {   // Hillis-Steele inclusive scan
        uint64_t v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    uint64_t run = threadIdx.x ? part[threadIdx.x - 1] : 0;
    for (uint32_t k = lo; k < hi; k++) { block_off[k] = run; run += block_counts[k]; }
    if (threadIdx.x == 1023) block_off[n_blocks] = part[1023];
}
__global__ void __launch_bounds__(kThreads) k_active_scatter(const uint8_t* __restrict__ recs, uint64_t n, uint64_t epoch,
                                                               const uint64_t* __restrict__ block_off, uint64_t* __restrict__ out) {
    __shared__ uint32_t warp_cnt[kThreads / 32];
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    bool act = false;
    if (i < n) {
        act = record_active(recs + i * 121, epoch);
    }
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t m = __ballot_sync(0xffffffffu, act);
    if (lane == 0) warp_cnt[warp] = __popc(m);
    __syncthreads();
    uint32_t before = 0;
    for (uint32_t w = 0; w < warp; w++) before += warp_cnt[w];
    if (act) out[block_off[blockIdx.x] + before + __popc(m & ((1u << lane) - 1u))] = i;
}


// ---- proposer and sync-committee selection: compute_proposer_index (deneb/spec/mod.rs:2420-2518) and
//      get_next_sync_committee_indices (:1973-2013)
// Candidate i of a sampling seed is active[compute_shuffled_index(i mod n, n, seed)]; it is accepted when
// effective_balance * 255 >= MAX_EFFECTIVE_BALANCE * random_byte, in wrapping u64 as a release build of the reference
// computes it, with random_byte = SHA-256(seed || le64(i / 32))[i % 32].  Lane j of a warp takes candidate 32w + j of
// window w, so a window's random-byte block is one hash per warp, computed by the warp in lockstep.  Few candidates are
// ever drawn (32 per slot, about SIZE for the committee), so each runs its rounds with the round's source block hashed on
// demand instead of building the list shuffle's rounds x n/256 table; the pivots are hashed once per warp (proposers:
// one seed per warp) or per CTA (committee: one seed per call) into shared memory.
constexpr int kSampleWarps = 4;
constexpr uint64_t kMaxEffectiveBalance = 32000000000ull;   // MAX_EFFECTIVE_BALANCE, both presets

// SHA-256 of seed(32) || le64(v): one padded block
__device__ __forceinline__ void sha256_seed_le64(const uint32_t seed_w[8], uint64_t v, uint32_t out[8]) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = seed_w[i];
    w[8] = bswap32(uint32_t(v));
    w[9] = bswap32(uint32_t(v >> 32));
    w[10] = 0x80000000u;
#pragma unroll
    for (int i = 11; i < 15; i++) w[i] = 0;
    w[15] = 40 * 8;
    sha256_init(out);
    sha256_compress(out, w);
}
// word k of a digest held in registers (a select chain: no local-memory indexing)
__device__ __forceinline__ uint32_t digest_word(const uint32_t h[8], uint32_t k) {
    uint32_t v = h[0];
#pragma unroll
    for (int j = 1; j < 8; j++) v = k == uint32_t(j) ? h[j] : v;
    return v;
}
// pivots of rounds t, t + stride, ... (t: this thread's rank among `stride` threads sharing piv)
__device__ __forceinline__ void hash_pivots(const uint32_t sw[8], uint32_t rounds, uint32_t n, uint32_t t, uint32_t stride, uint32_t* piv) {
    for (uint32_t r = t; r < rounds; r += stride) {
        uint32_t h[8];
        sha256_seed_plus(sw, r, 0, false, h);
        piv[r] = uint32_t((uint64_t(bswap32(h[0])) | (uint64_t(bswap32(h[1])) << 32)) % n);
    }
}
// candidate 32 * window + lane of seed `sw` (n <= 2^31 active validators): *cand is this lane's candidate, the result
// the warp's ballot of accepted lanes
__device__ __forceinline__ uint32_t sample_window(const uint32_t sw[8], const uint32_t* piv, uint32_t rounds,
                                                  const uint64_t* __restrict__ active, uint32_t n, const uint8_t* __restrict__ recs,
                                                  uint64_t window, uint64_t* cand) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t idx = uint32_t((window * 32 + lane) % n);
#pragma unroll 1
    for (uint32_t r = 0; r < rounds; r++)
        idx = shuffle_round(idx, piv[r], n, [&](uint32_t pos) {
            uint32_t h[8];
            sha256_seed_plus(sw, r, pos >> 8, true, h);
            return digest_word(h, (pos & 255u) >> 5);
        });
    const uint64_t c = active[idx];
    const uint64_t eff = load_le64_unaligned(recs + c * 121 + kRecEffectiveBalance);
    uint32_t h[8];
    sha256_seed_le64(sw, window, h);
    const uint64_t byte = (digest_word(h, lane >> 2) >> (24u - 8u * (lane & 3u))) & 0xffu;
    *cand = c;
    return __ballot_sync(0xffffffffu, eff * 255u >= kMaxEffectiveBalance * byte);
}

// compute_proposer_index for n_seeds slot seeds (8 big-endian words each): warp s draws windows 0, 1, ... of seed s until
// one accepts, and its first accepted lane is the proposer; out[s] = UINT64_MAX after max_windows windows without one
__global__ void __launch_bounds__(32 * kSampleWarps) k_sample_proposers(const uint32_t* __restrict__ seeds_w, uint32_t n_seeds, uint32_t rounds,
                                                                          const uint64_t* __restrict__ active, uint32_t n,
                                                                          const uint8_t* __restrict__ recs, uint64_t max_windows,
                                                                          uint64_t* __restrict__ out) {
    __shared__ uint32_t piv[kSampleWarps][256];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t s = blockIdx.x * kSampleWarps + warp;
    if (s >= n_seeds) return;   // whole warps
    uint32_t sw[8];
#pragma unroll
    for (int i = 0; i < 8; i++) sw[i] = seeds_w[s * 8 + i];
    hash_pivots(sw, rounds, n, lane, 32, piv[warp]);
    __syncwarp();
    uint64_t found = ~0ull;
#pragma unroll 1
    for (uint64_t w = 0; w < max_windows; w++) {
        uint64_t c;
        const uint32_t m = sample_window(sw, piv[warp], rounds, active, n, recs, w, &c);
        if (m) { found = __shfl_sync(0xffffffffu, c, __ffs(m) - 1); break; }
    }
    if (lane == 0) out[s] = found;
}

// windows first .. first + n_windows - 1 of one seed, a warp each: every lane's candidate and each window's ballot
__global__ void __launch_bounds__(32 * kSampleWarps) k_sample_windows(const uint32_t* __restrict__ seed_w, uint32_t rounds,
                                                                        const uint64_t* __restrict__ active, uint32_t n,
                                                                        const uint8_t* __restrict__ recs, uint64_t first,
                                                                        uint32_t n_windows, uint64_t* __restrict__ cand,
                                                                        uint32_t* __restrict__ accept) {
    __shared__ uint32_t piv[256];
    uint32_t sw[8];
#pragma unroll
    for (int i = 0; i < 8; i++) sw[i] = seed_w[i];
    hash_pivots(sw, rounds, n, threadIdx.x, blockDim.x, piv);
    __syncthreads();
    const uint32_t k = blockIdx.x * kSampleWarps + (threadIdx.x >> 5);
    if (k >= n_windows) return;   // whole warps
    uint64_t c;
    const uint32_t m = sample_window(sw, piv, rounds, active, n, recs, first + k, &c);
    cand[uint64_t(k) * 32 + (threadIdx.x & 31)] = c;
    if ((threadIdx.x & 31) == 0) accept[k] = m;
}

// The first `size` accepted candidates in candidate order: one CTA walks the window's ballots 1024 at a time, a block
// scan of their popcounts placing each accepted candidate at out[rank] while rank < size; *have (accepted before this
// window) advances, saturating at size.
__global__ void __launch_bounds__(1024) k_select_accepted(const uint32_t* __restrict__ accept, const uint64_t* __restrict__ cand,
                                                            uint32_t n_words, uint32_t size, uint64_t* __restrict__ out,
                                                            uint32_t* __restrict__ have) {
    __shared__ uint32_t warp_sum[32];
    __shared__ uint32_t base;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) base = *have;
    __syncthreads();
    for (uint32_t w0 = 0; w0 < n_words && base < size; w0 += 1024) {
        const uint32_t k = w0 + threadIdx.x;
        const uint32_t m = k < n_words ? accept[k] : 0u, c = __popc(m);
        uint32_t x = c;   // inclusive warp scan, then the warps' totals
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= uint32_t(d)) x += y;
        }
        if (lane == 31) warp_sum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint32_t v = warp_sum[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, v, d);
                if (lane >= uint32_t(d)) v += y;
            }
            warp_sum[lane] = v;
        }
        __syncthreads();
        uint32_t rank = base + (warp ? warp_sum[warp - 1] : 0u) + x - c;
        for (uint32_t mm = m; mm && rank < size; mm &= mm - 1) out[rank++] = cand[uint64_t(k) * 32 + uint32_t(__ffs(mm) - 1)];
        __syncthreads();
        if (threadIdx.x == 0) base += warp_sum[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) *have = min(base, size);
}

// process_sync_aggregate's key -> validator index map (deneb/spec/mod.rs:463-473).  The m <= 512 committee keys, sorted by
// their first 8 bytes (`prefix`, big-endian), are staged in shared memory; each Validator record binary-searches its own
// first 8 bytes and, on a full 48-byte match, raises every committee position holding that key to i + 1.  atomicMax keeps
// the largest index, as the reference's HashMap built in registry order keeps the last insert; 0 is left for a key no
// validator holds.
constexpr uint32_t kMaxCommittee = 512;
__global__ void __launch_bounds__(kThreads) k_match_committee_keys(const uint8_t* __restrict__ recs, uint64_t n,
                                                                     const uint4* __restrict__ keys, const uint64_t* __restrict__ prefix,
                                                                     const uint32_t* __restrict__ pos, uint32_t m,
                                                                     unsigned long long* __restrict__ out) {
    __shared__ uint64_t s_prefix[kMaxCommittee];
    __shared__ uint4 s_keys[kMaxCommittee * 3];
    for (uint32_t k = threadIdx.x; k < m; k += blockDim.x) s_prefix[k] = prefix[k];
    for (uint32_t k = threadIdx.x; k < m * 3; k += blockDim.x) s_keys[k] = keys[k];
    __syncthreads();
    for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x) {
        const uint8_t* r = recs + i * 121;
        uint64_t p = 0;
#pragma unroll
        for (int b = 0; b < 8; b++) p = (p << 8) | r[b];
        uint32_t lo = 0, hi = m;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (s_prefix[mid] < p) lo = mid + 1; else hi = mid;
        }
        for (uint32_t k = lo; k < m && s_prefix[k] == p; k++) {
            const uint8_t* key = reinterpret_cast<const uint8_t*>(s_keys + 3 * k);
            bool eq = true;
            for (int b = 8; b < 48; b++) eq = eq && key[b] == r[b];
            if (eq) atomicMax(out + pos[k], static_cast<unsigned long long>(i + 1));
        }
    }
}

// ---- beacon committees over an epoch's cached shuffled active list (phase0/helpers.rs:459-483, 741-806) ----
// Committee k of C = SLOTS_PER_EPOCH x committees_per_slot is positions [n k / C, n (k + 1) / C) of the list.
// k_committee_positions inverts the list: pos[shuffled[p]] = p over a map pre-filled with kNotActive.  A duty row is then
// arithmetic on p: the committee holding p is k = ((p + 1) C - 1) / n, the largest k with n k / C <= p, so never an empty
// one; (p + 1) C fits u64 (C <= 2048, p < 2^31).
__global__ void __launch_bounds__(kThreads) k_committee_positions(const uint64_t* __restrict__ shuffled, uint64_t n,
                                                                    uint32_t* __restrict__ pos) {
    const uint64_t p = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (p < n) pos[shuffled[p]] = uint32_t(p);
}
// AttestationDuty rows (slot, committee_index, committee_length, committees_at_slot, validator_committee_index) for
// validators[r] (nullptr: r itself); UINT64_MAX x 5 for a validator not active at the epoch
__global__ void __launch_bounds__(kThreads) k_attester_duties(const uint32_t* __restrict__ pos, const uint64_t* __restrict__ validators,
                                                                uint64_t n_rows, uint64_t n, uint64_t cps, uint64_t spe,
                                                                uint64_t epoch, uint64_t* __restrict__ out) {
    const uint64_t r = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const uint32_t p = pos[validators ? validators[r] : r];
    uint64_t* row = out + r * 5;
    if (p == kNotActive) {
#pragma unroll
        for (int f = 0; f < 5; f++) row[f] = ~uint64_t(0);
        return;
    }
    const uint64_t c = spe * cps;
    const uint64_t k = ((uint64_t(p) + 1) * c - 1) / n;
    const uint64_t start = n * k / c, end = n * (k + 1) / c;
    row[0] = epoch * spe + k / cps;
    row[1] = k % cps;
    row[2] = end - start;
    row[3] = cps;
    row[4] = p - start;
}

// get_attesting_indices + get_indexed_attestation's sort (phase0/helpers.rs:896-974), one CTA per attestation that passed
// the host's checks: the set bits of its committee slice are compacted by warp ballot into shared memory (committee order
// is lost, the sort restores a canonical one), padded with UINT64_MAX to a power of two and bitonic-sorted ascending, then
// written at the job's prefix-summed offset.  A committee member appears once, so the sorted set is the sorted list.
constexpr int kAttThreads = 256;
__global__ void __launch_bounds__(kAttThreads) k_attesting_indices(const AttestingJob* __restrict__ jobs, const uint8_t* __restrict__ bits,
                                                                     uint64_t* __restrict__ out) {
    __shared__ uint64_t s[kMaxCommitteeBits];
    __shared__ uint32_t count;
    const AttestingJob j = jobs[blockIdx.x];
    const uint32_t lane = threadIdx.x & 31;
    if (threadIdx.x == 0) count = 0;
    __syncthreads();
    const uint8_t* b = bits + j.bits_off;
    for (uint32_t i0 = 0; i0 < j.len; i0 += kAttThreads) {   // uniform trip count: whole warps reach the ballot
        const uint32_t i = i0 + threadIdx.x;
        const bool set = i < j.len && ((b[i >> 3] >> (i & 7)) & 1u);
        const uint32_t m = __ballot_sync(0xffffffffu, set);
        uint32_t base = 0;
        if (lane == 0 && m) base = atomicAdd(&count, uint32_t(__popc(m)));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (set) s[base + __popc(m & ((1u << lane) - 1u))] = j.committee[i];
    }
    __syncthreads();
    const uint32_t n = count;
    uint32_t size = 1;
    while (size < n) size <<= 1;
    for (uint32_t i = n + threadIdx.x; i < size; i += kAttThreads) s[i] = ~uint64_t(0);
    __syncthreads();
    for (uint32_t k = 2; k <= size; k <<= 1)
        for (uint32_t d = k >> 1; d > 0; d >>= 1) {
            for (uint32_t i = threadIdx.x; i < size; i += kAttThreads) {
                const uint32_t l = i ^ d;
                if (l > i) {
                    const uint64_t a = s[i], c = s[l];
                    if ((a > c) == ((i & k) == 0)) { s[i] = c; s[l] = a; }
                }
            }
            __syncthreads();
        }
    for (uint32_t i = threadIdx.x; i < n; i += kAttThreads) out[uint64_t(j.out_off) + i] = s[i];
}

}  // namespace

struct ShuffleScratch {
    DevBuf sources, pivots, seed, idx_in, out, counts, offs, recs;
    DevBuf sample;   // proposer / committee sampling and key matching: seeds, ballots, candidates, results
};
static ShuffleScratch g_sh;

static uint32_t be32h(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }

// out_dev[0..n) = shuffled `idx_dev` (nullptr: identity) on the engine stream; all device pointers
int32_t shuffle_on_device(Engine& e, const uint64_t* idx_dev, uint64_t n, const uint8_t seed[32], uint32_t rounds, uint64_t* out_dev) {
    if (n == 0) return B200_SUCCESS;
    // the block index of a source hash is a u32 and the table is rounds x n / 8 bytes: 2^31 positions (24 GB at 90 rounds) is
    // the ceiling of this formulation, three orders of magnitude above any registry
    if (rounds > 255 || n > (uint64_t(1) << 31)) { e.last_error = "shuffle: more than 255 rounds or 2^31 positions"; return B200_ERR_BAD_ARG; }
    const uint32_t nblk = uint32_t((n + 255) / 256);
    B200_CUDA_TRY(g_sh.sources.reserve(uint64_t(rounds ? rounds : 1) * nblk * 32));
    B200_CUDA_TRY(g_sh.pivots.reserve(256 * 8));
    B200_CUDA_TRY(g_sh.seed.reserve(64));
    B200_CUDA_TRY(e.staging.reserve(64));
    uint32_t* hw = static_cast<uint32_t*>(e.staging.p);
    for (int i = 0; i < 8; i++) hw[i] = be32h(seed + 4 * i);
    cudaStream_t s = e.stream;
    B200_CUDA_TRY(cudaMemcpyAsync(g_sh.seed.p, hw, 32, cudaMemcpyHostToDevice, s));
    B200_CUDA_TRY(cudaStreamSynchronize(s));   // staging is shared scratch: do not let a later call overwrite it in flight
    if (rounds) {
        const uint64_t items = (uint64_t(nblk) + 1) * rounds;
        k_shuffle_sources<<<unsigned((items + kThreads - 1) / kThreads), kThreads, 0, s>>>(
            static_cast<const uint32_t*>(g_sh.seed.p), rounds, nblk, n, static_cast<uint32_t*>(g_sh.sources.p),
            static_cast<uint64_t*>(g_sh.pivots.p));
        e.launches++;
    }
    const unsigned grid = unsigned((n + kThreads - 1) / kThreads);
    k_shuffle_map<uint32_t><<<grid, kThreads, 0, s>>>(idx_dev, n, rounds, nblk, static_cast<const uint32_t*>(g_sh.sources.p),
                                                      static_cast<const uint64_t*>(g_sh.pivots.p), out_dev);
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    return B200_SUCCESS;
}

// out_dev (capacity n) = indices of the active validators, in order; *count_dev-side total copied to *out_n (host)
int32_t active_indices_on_device(Engine& e, const uint8_t* recs_dev, uint64_t n, uint64_t epoch, uint64_t* out_dev, uint64_t* out_n) {
    *out_n = 0;
    if (n == 0) return B200_SUCCESS;
    const uint32_t n_blocks = uint32_t((n + kThreads - 1) / kThreads);
    B200_CUDA_TRY(g_sh.counts.reserve(uint64_t(n_blocks) * 4 + 16));
    B200_CUDA_TRY(g_sh.offs.reserve(uint64_t(n_blocks + 1) * 8 + 16));
    B200_CUDA_TRY(e.staging.reserve(64));
    cudaStream_t s = e.stream;
    k_active_count<<<n_blocks, kThreads, 0, s>>>(recs_dev, n, epoch, static_cast<uint32_t*>(g_sh.counts.p));
    k_active_scan<<<1, 1024, 0, s>>>(static_cast<const uint32_t*>(g_sh.counts.p), n_blocks, static_cast<uint64_t*>(g_sh.offs.p));
    k_active_scatter<<<n_blocks, kThreads, 0, s>>>(recs_dev, n, epoch, static_cast<const uint64_t*>(g_sh.offs.p), out_dev);
    e.launches += 3;
    B200_CUDA_TRY(cudaGetLastError());
    B200_CUDA_TRY(cudaMemcpyAsync(e.staging.p, static_cast<const uint64_t*>(g_sh.offs.p) + n_blocks, 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA_TRY(cudaStreamSynchronize(s));
    *out_n = *static_cast<const uint64_t*>(e.staging.p);
    return B200_SUCCESS;
}

int32_t shuffle_scratch(Engine& e, uint64_t n, uint64_t** a, uint64_t** b) {
    B200_CUDA_TRY(g_sh.idx_in.reserve(n * 8 + 64));
    B200_CUDA_TRY(g_sh.out.reserve(n * 8 + 64));
    *a = static_cast<uint64_t*>(g_sh.idx_in.p);
    *b = static_cast<uint64_t*>(g_sh.out.p);
    return B200_SUCCESS;
}


// Safety cap of the sampling loops, which have no bound in the reference: they end with probability 1 (a random byte of 0
// accepts any candidate), and the expected worst case, every balance 0, draws 256 candidates per proposer and about
// 131 072 for a 512-member committee.  Past the cap the call returns B200_ERR_LIMIT.
constexpr uint64_t kMaxSampleCandidates = uint64_t(1) << 26;

static void seed_words(const uint8_t seed[32], uint32_t* w) {
    for (int i = 0; i < 8; i++) w[i] = be32h(seed + 4 * i);
}

int32_t sample_proposers_on_device(Engine& e, const uint8_t* seeds, uint32_t n_seeds, uint32_t rounds, const uint64_t* active_dev,
                                   uint64_t n, const uint8_t* recs_dev, uint64_t* out) {
    if (!n || n > (uint64_t(1) << 31) || rounds > 255) { e.last_error = "proposer sampling: 0 or more than 2^31 active validators"; return B200_ERR_BAD_ARG; }
    const size_t seed_bytes = size_t(n_seeds) * 32;
    B200_CUDA_TRY(g_sh.sample.reserve(seed_bytes + size_t(n_seeds) * 8 + 64));
    B200_CUDA_TRY(e.staging.reserve(seed_bytes + size_t(n_seeds) * 8));
    uint32_t* hw = static_cast<uint32_t*>(e.staging.p);
    for (uint32_t s = 0; s < n_seeds; s++) seed_words(seeds + 32 * s, hw + 8 * s);
    uint32_t* d_seeds = static_cast<uint32_t*>(g_sh.sample.p);
    uint64_t* d_out = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(g_sh.sample.p) + seed_bytes);
    cudaStream_t st = e.stream;
    B200_CUDA_TRY(cudaMemcpyAsync(d_seeds, hw, seed_bytes, cudaMemcpyHostToDevice, st));
    k_sample_proposers<<<(n_seeds + kSampleWarps - 1) / kSampleWarps, 32 * kSampleWarps, 0, st>>>(
        d_seeds, n_seeds, rounds, active_dev, uint32_t(n), recs_dev, kMaxSampleCandidates / 32, d_out);
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    uint64_t* h_out = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(e.staging.p) + seed_bytes);
    B200_CUDA_TRY(cudaMemcpyAsync(h_out, d_out, size_t(n_seeds) * 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA_TRY(cudaStreamSynchronize(st));
    for (uint32_t s = 0; s < n_seeds; s++) {
        if (h_out[s] == ~uint64_t(0)) { e.last_error = "proposer sampling: no candidate accepted within the candidate cap"; return B200_ERR_LIMIT; }
        out[s] = h_out[s];
    }
    return B200_SUCCESS;
}

// Windows of candidates until `size` are accepted: the first window holds `size` candidates (when every balance is 32 ETH
// all of them are accepted: one window), each further one twice the previous, up to kMaxSampleCandidates in all.
// Sampling scratch: seed words (32 B) | accepted so far (4 B) | the window's ballots | its candidates.
int32_t sample_committee_on_device(Engine& e, const uint8_t seed[32], uint32_t size, uint32_t rounds, const uint64_t* active_dev,
                                   uint64_t n, const uint8_t* recs_dev, uint64_t* out_dev) {
    if (!n || n > (uint64_t(1) << 31) || rounds > 255) { e.last_error = "committee sampling: 0 or more than 2^31 active validators"; return B200_ERR_BAD_ARG; }
    const uint64_t max_words = kMaxSampleCandidates / 32;
    B200_CUDA_TRY(e.staging.reserve(64));
    uint32_t* hw = static_cast<uint32_t*>(e.staging.p);
    cudaStream_t st = e.stream;
    uint64_t done = 0;   // windows of 32 candidates drawn so far
    uint32_t words = (size + 31) / 32, have = 0;
    bool staged = false;
    while (have < size) {
        if (done >= max_words) { e.last_error = "committee sampling: fewer than SIZE accepted within the candidate cap"; return B200_ERR_LIMIT; }
        words = uint32_t(std::min<uint64_t>(words, max_words - done));
        const size_t o_cand = 64 + ((size_t(words) * 4 + 15) & ~size_t(15));
        if (!staged || g_sh.sample.cap < o_cand + size_t(words) * 256) {   // (re)allocated: the seed and the count again
            B200_CUDA_TRY(g_sh.sample.reserve(o_cand + size_t(words) * 256));
            seed_words(seed, hw);
            hw[8] = have;
            B200_CUDA_TRY(cudaMemcpyAsync(g_sh.sample.p, hw, 36, cudaMemcpyHostToDevice, st));
            staged = true;
        }
        uint8_t* base = static_cast<uint8_t*>(g_sh.sample.p);
        uint32_t* d_have = reinterpret_cast<uint32_t*>(base + 32);
        uint32_t* d_acc = reinterpret_cast<uint32_t*>(base + 64);
        uint64_t* d_cand = reinterpret_cast<uint64_t*>(base + o_cand);
        k_sample_windows<<<(words + kSampleWarps - 1) / kSampleWarps, 32 * kSampleWarps, 0, st>>>(
            reinterpret_cast<const uint32_t*>(base), rounds, active_dev, uint32_t(n), recs_dev, done, words, d_cand, d_acc);
        k_select_accepted<<<1, 1024, 0, st>>>(d_acc, d_cand, words, size, out_dev, d_have);
        e.launches += 2;
        B200_CUDA_TRY(cudaGetLastError());
        B200_CUDA_TRY(cudaMemcpyAsync(hw + 8, d_have, 4, cudaMemcpyDeviceToHost, st));
        B200_CUDA_TRY(cudaStreamSynchronize(st));
        have = hw[8];
        done += words;
        words = uint32_t(std::min<uint64_t>(uint64_t(words) * 2, max_words));
    }
    return B200_SUCCESS;
}

int32_t match_committee_keys_on_device(Engine& e, const uint8_t* recs_dev, uint64_t n, const uint8_t* keys, uint32_t m, uint64_t* out) {
    if (m == 0 || m > kMaxCommittee) { e.last_error = "committee key match: 1 to 512 keys"; return B200_ERR_BAD_ARG; }
    std::vector<uint32_t> order(m);
    std::vector<uint64_t> prefix(m);
    for (uint32_t k = 0; k < m; k++) {
        order[k] = k;
        uint64_t p = 0;
        for (int b = 0; b < 8; b++) p = (p << 8) | keys[48 * k + b];
        prefix[k] = p;
    }
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return prefix[a] < prefix[b]; });
    // keys (16-byte aligned) | prefixes | positions | results
    const size_t o_pre = size_t(m) * 48, o_pos = o_pre + size_t(m) * 8, o_out = (o_pos + size_t(m) * 4 + 15) & ~size_t(15);
    const size_t total = o_out + size_t(m) * 8;
    B200_CUDA_TRY(g_sh.sample.reserve(total + 64));
    B200_CUDA_TRY(e.staging.reserve(total));
    uint8_t* hs = static_cast<uint8_t*>(e.staging.p);
    for (uint32_t k = 0; k < m; k++) {
        memcpy(hs + 48 * size_t(k), keys + 48 * size_t(order[k]), 48);
        memcpy(hs + o_pre + 8 * size_t(k), &prefix[order[k]], 8);
        memcpy(hs + o_pos + 4 * size_t(k), &order[k], 4);
    }
    memset(hs + o_out, 0, size_t(m) * 8);
    uint8_t* d = static_cast<uint8_t*>(g_sh.sample.p);
    cudaStream_t st = e.stream;
    B200_CUDA_TRY(cudaMemcpyAsync(d, hs, total, cudaMemcpyHostToDevice, st));
    if (n) {
        int sms = 132;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e.device);
        const uint64_t blocks = std::min<uint64_t>((n + kThreads - 1) / kThreads, uint64_t(sms) * 4);
        k_match_committee_keys<<<unsigned(blocks), kThreads, 0, st>>>(recs_dev, n, reinterpret_cast<const uint4*>(d),
                                                                      reinterpret_cast<const uint64_t*>(d + o_pre),
                                                                      reinterpret_cast<const uint32_t*>(d + o_pos), m,
                                                                      reinterpret_cast<unsigned long long*>(d + o_out));
        e.launches++;
        B200_CUDA_TRY(cudaGetLastError());
    }
    B200_CUDA_TRY(cudaMemcpyAsync(hs + o_out, d + o_out, size_t(m) * 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA_TRY(cudaStreamSynchronize(st));
    for (uint32_t k = 0; k < m; k++) {
        uint64_t v;
        memcpy(&v, hs + o_out + 8 * size_t(k), 8);
        out[k] = v ? v - 1 : ~uint64_t(0);
    }
    return B200_SUCCESS;
}

int32_t committee_positions_on_device(Engine& e, const uint64_t* shuffled_dev, uint64_t n_active, uint64_t n_validators, uint32_t* pos_dev) {
    if (n_active > n_validators || n_validators > (uint64_t(1) << 32)) { e.last_error = "committee positions: bad list sizes"; return B200_ERR_BAD_ARG; }
    cudaStream_t st = e.stream;
    if (n_validators) B200_CUDA_TRY(cudaMemsetAsync(pos_dev, 0xff, n_validators * 4, st));
    if (n_active) {
        k_committee_positions<<<unsigned((n_active + kThreads - 1) / kThreads), kThreads, 0, st>>>(shuffled_dev, n_active, pos_dev);
        e.launches++;
        B200_CUDA_TRY(cudaGetLastError());
    }
    return B200_SUCCESS;
}

int32_t attester_duties_on_device(Engine& e, const uint32_t* pos_dev, const uint64_t* validators_dev, uint64_t n_rows, uint64_t n_active,
                                  uint64_t cps, uint64_t slots_per_epoch, uint64_t epoch, uint64_t* out_dev) {
    if (!n_rows) return B200_SUCCESS;
    k_attester_duties<<<unsigned((n_rows + kThreads - 1) / kThreads), kThreads, 0, e.stream>>>(pos_dev, validators_dev, n_rows, n_active,
                                                                                                cps, slots_per_epoch, epoch, out_dev);
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    return B200_SUCCESS;
}

int32_t attesting_indices_on_device(Engine& e, const AttestingJob* jobs_dev, uint32_t n_jobs, const uint8_t* bits_dev, uint64_t* out_dev) {
    if (!n_jobs) return B200_SUCCESS;
    k_attesting_indices<<<n_jobs, kAttThreads, 0, e.stream>>>(jobs_dev, bits_dev, out_dev);
    e.launches++;
    B200_CUDA_TRY(cudaGetLastError());
    return B200_SUCCESS;
}
}  // namespace b200

using namespace b200;

extern "C" {

int32_t b200_compute_shuffled_indices(const uint64_t* indices, size_t n, const uint8_t seed[32], uint32_t rounds, uint64_t* out) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    if (!e.ready) { e.last_error = "b200_init has not been called (or failed)"; return B200_ERR_NOT_INITIALIZED; }
    if (!seed || (n && !out)) return B200_ERR_BAD_ARG;
    if (n == 0) return B200_SUCCESS;
    B200_CUDA_TRY(cudaSetDevice(e.device));
    uint64_t *d_in, *d_out;
    int32_t rc = shuffle_scratch(e, n, &d_in, &d_out);
    if (rc) return rc;
    B200_CUDA_TRY(cudaEventRecord(e.ev0, e.stream));
    if (indices) B200_CUDA_TRY(cudaMemcpyAsync(d_in, indices, n * 8, cudaMemcpyHostToDevice, e.stream));
    rc = shuffle_on_device(e, indices ? d_in : nullptr, n, seed, rounds, d_out);
    if (rc) return rc;
    B200_CUDA_TRY(cudaEventRecord(e.ev1, e.stream));
    B200_CUDA_TRY(cudaMemcpyAsync(out, d_out, n * 8, cudaMemcpyDeviceToHost, e.stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e.stream));
    B200_CUDA_TRY(cudaEventElapsedTime(&e.last_kernel_ms, e.ev0, e.ev1));
    return B200_SUCCESS;
}

int32_t b200_get_active_validator_indices(const uint8_t* validators_ssz, size_t n, uint64_t epoch, uint64_t* out, size_t* out_n) {
    Engine& e = engine();
    std::unique_lock<std::mutex> lk(e.mu);
    if (!e.ready) { e.last_error = "b200_init has not been called (or failed)"; return B200_ERR_NOT_INITIALIZED; }
    if (!out_n || (n && (!validators_ssz || !out))) return B200_ERR_BAD_ARG;
    *out_n = 0;
    if (n == 0) return B200_SUCCESS;
    B200_CUDA_TRY(cudaSetDevice(e.device));
    uint64_t *d_in, *d_out;
    int32_t rc = shuffle_scratch(e, n, &d_in, &d_out);
    if (rc) return rc;
    B200_CUDA_TRY(g_sh.recs.reserve(n * 121 + 64));
    B200_CUDA_TRY(cudaMemcpyAsync(g_sh.recs.p, validators_ssz, n * 121, cudaMemcpyHostToDevice, e.stream));
    uint64_t cnt = 0;
    rc = active_indices_on_device(e, static_cast<const uint8_t*>(g_sh.recs.p), n, epoch, d_out, &cnt);
    if (rc) return rc;
    if (cnt) B200_CUDA_TRY(cudaMemcpy(out, d_out, cnt * 8, cudaMemcpyDeviceToHost));
    *out_n = size_t(cnt);
    return B200_SUCCESS;
}

}  // extern "C"
