// SSZ hash_tree_root kernels for sm_90a.
//
// One `k_merkle_stage` launch processes one step of *every* big field of the container at once (a stage is a
// list of jobs; blocks find their job through `block_begin`), so a full deneb BeaconState root is
// ~6 wide launches + one single-CTA finisher for the small containers, the virtual zero-hash padding chains
// (List limits of 2^40 => 40 levels, only the populated part is ever hashed), the length mix-ins and the
// 28-field top tree.  Replaces ssz_rs' `merkleize` / derived `hash_tree_root`
// (ethereum-consensus/src/deneb/beacon_state.rs:10-64, called at
// ethereum-consensus/src/deneb/spec/mod.rs:3215,3288).
//
// Work decomposition: every thread owns a complete small subtree (8 leaves -> 1 node = 7 hashes, or one
// 121-byte Validator -> 8 hashes) and runs it entirely in registers: no idle lanes on the upper levels, no
// inter-thread traffic.  The kernel is bound by the 32-bit ALU pipe (LOP3/SHF/IADD3), not by HBM: 96 B of
// traffic per ~2.3 k integer instructions.
#include "sha256.cuh"
#include "ssz_kernels.cuh"

#include <cuda_runtime.h>

namespace b200 {

namespace {

__device__ __forceinline__ void load_node(const uint32_t* p, uint32_t out[8]) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = q[0], b = q[1];
    out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w;
    out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
}
__device__ __forceinline__ void load_node_raw(const uint32_t* p, uint32_t out[8]) {
    load_node(p, out);
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = bswap32(out[i]);
}
__device__ __forceinline__ void store_node(uint32_t* p, const uint32_t v[8]) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(v[0], v[1], v[2], v[3]);
    q[1] = make_uint4(v[4], v[5], v[6], v[7]);
}

// input node `idx` of a REDUCE job (zero-subtree hash of `level` beyond the populated range)
__device__ __forceinline__ void fetch(const Job& jb, const uint32_t* zero_nodes, uint64_t idx, uint32_t out[8]) {
    if (idx < jb.n_in) {
        const uint32_t* p = reinterpret_cast<const uint32_t*>(jb.src) + idx * 8;
        if (jb.raw) load_node_raw(p, out); else load_node(p, out);
    } else {
        load_node(zero_nodes + jb.level * 8, out);
    }
}

template <int NLEV>
__device__ __forceinline__ void subtree(const Job& jb, const uint32_t* zero_nodes, uint64_t first, uint32_t out[8]) {
    if constexpr (NLEV == 0) {
        fetch(jb, zero_nodes, first, out);
    } else {
        uint32_t l[8], r[8];
        subtree<NLEV - 1>(jb, zero_nodes, first, l);
        subtree<NLEV - 1>(jb, zero_nodes, first + (1ull << (NLEV - 1)), r);
        hash_pair_words(l, r, out);
    }
}

// big-endian word at byte offset `off` of a record staged in shared memory (any alignment)
__device__ __forceinline__ uint32_t smem_be_word(const uint32_t* sm, uint32_t off) {
    uint32_t k = off >> 2, s = off & 3;
    uint32_t lo = sm[k], hi = sm[k + 1];
    // bytes s..s+3 of (lo | hi<<32), most significant first
    uint32_t sel = ((s + 3) | ((s + 2) << 4) | ((s + 1) << 8) | (s << 12));
    return __byte_perm(lo, hi, sel);
}

// hash_tree_root(Validator) of the 121-byte record staged at byte offset `base` of `smem`
__device__ __forceinline__ void validator_root(const uint32_t* smem, uint32_t base, uint32_t root[8]) {
    uint32_t m[16], x[8], y[8], ab[8];
    // pubkey: 48 bytes -> 2 chunks -> 1 hash
#pragma unroll
    for (int i = 0; i < 12; i++) m[i] = smem_be_word(smem, base + 4 * i);
    m[12] = m[13] = m[14] = m[15] = 0;
    sha256_msg64(m, x);
    // (pubkey_root, withdrawal_credentials)
#pragma unroll
    for (int i = 0; i < 8; i++) { m[i] = x[i]; m[8 + i] = smem_be_word(smem, base + 48 + 4 * i); }
    sha256_msg64(m, x);
    // (effective_balance, slashed)
#pragma unroll
    for (int i = 0; i < 16; i++) m[i] = 0;
    m[0] = smem_be_word(smem, base + 80); m[1] = smem_be_word(smem, base + 84);
    m[8] = smem_be_word(smem, base + 88) & 0xff000000u;
    sha256_msg64(m, y);
    hash_pair_words(x, y, ab);
    // (activation_eligibility_epoch, activation_epoch)
#pragma unroll
    for (int i = 0; i < 16; i++) m[i] = 0;
    m[0] = smem_be_word(smem, base + 89); m[1] = smem_be_word(smem, base + 93);
    m[8] = smem_be_word(smem, base + 97); m[9] = smem_be_word(smem, base + 101);
    sha256_msg64(m, x);
    // (exit_epoch, withdrawable_epoch)
#pragma unroll
    for (int i = 0; i < 16; i++) m[i] = 0;
    m[0] = smem_be_word(smem, base + 105); m[1] = smem_be_word(smem, base + 109);
    m[8] = smem_be_word(smem, base + 113); m[9] = smem_be_word(smem, base + 117);
    sha256_msg64(m, y);
    hash_pair_words(x, y, x);
    hash_pair_words(ab, x, root);
}

template <int MINB>
__global__ void __launch_bounds__(kStageThreads, MINB) k_validator_roots(const __grid_constant__ Job jb) {
    __shared__ __align__(16) uint32_t smem[(kStageThreads * 121 + 16) / 4 + 4];
    const uint32_t blk = blockIdx.x;
    // stage 256 x 121 B (30 976 B, a multiple of 16) with coalesced 16-byte loads
    const uint64_t first = uint64_t(blk) * kStageThreads;
    const uint64_t nrec = min(uint64_t(kStageThreads), jb.n_in - first);
    const uint32_t nbytes = uint32_t(nrec) * 121u;
    const uint4* g = reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(jb.src) + first * 121u);
    uint4* s4 = reinterpret_cast<uint4*>(smem);
    const uint32_t nvec = (nbytes + 15) >> 4;  // the field buffer is padded to a 16-byte multiple
    for (uint32_t i = threadIdx.x; i < nvec; i += kStageThreads) s4[i] = g[i];
    __syncthreads();
    if (threadIdx.x >= nrec) return;
    uint32_t root[8];
    validator_root(smem, threadIdx.x * 121u, root);
    store_node(jb.dst + (first + threadIdx.x) * 8, root);
}

template <int MINB>
__global__ void __launch_bounds__(kStageThreads, MINB) k_merkle_stage(const __grid_constant__ StageDesc sd) {
    // locate this block's job (njobs is small; block_begin ascending)
    int j = 0;
#pragma unroll 1
    for (int k = 1; k < sd.njobs; k++)
        if (blockIdx.x >= sd.jobs[k].block_begin) j = k;
    const Job& jb = sd.jobs[j];
    const uint32_t blk = blockIdx.x - jb.block_begin;
    const uint64_t t = uint64_t(blk) * kStageThreads + threadIdx.x;

    switch (jb.type) {
    case JOB_REDUCE: {
        const uint64_t n_out = (jb.n_in + (1ull << jb.nlev) - 1) >> jb.nlev;
        if (t >= n_out) return;
        uint32_t out[8];
        switch (jb.nlev) {
        case 0: subtree<0>(jb, sd.zero_nodes, t, out); break;
        case 1: subtree<1>(jb, sd.zero_nodes, t << 1, out); break;
        case 2: subtree<2>(jb, sd.zero_nodes, t << 2, out); break;
        default: subtree<3>(jb, sd.zero_nodes, t << 3, out); break;
        }
        store_node(jb.dst + t * 8, out);
    } break;
    case JOB_PUBKEY48: {
        if (t >= jb.n_in) return;
        const uint4* p = reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(jb.src) + t * 48);
        uint4 x0 = p[0], x1 = p[1], x2 = p[2];
        uint32_t m[16] = {bswap32(x0.x), bswap32(x0.y), bswap32(x0.z), bswap32(x0.w),
                          bswap32(x1.x), bswap32(x1.y), bswap32(x1.z), bswap32(x1.w),
                          bswap32(x2.x), bswap32(x2.y), bswap32(x2.z), bswap32(x2.w), 0, 0, 0, 0};
        uint32_t out[8];
        sha256_msg64(m, out);
        store_node(jb.dst + t * 8, out);
    } break;
    case JOB_PAIR64: {
        if (t >= jb.n_in) return;
        const uint32_t* p = reinterpret_cast<const uint32_t*>(jb.src) + t * 16;
        uint32_t m[16], out[8];
        load_node_raw(p, m);
        load_node_raw(p + 8, m + 8);
        sha256_msg64(m, out);
        store_node(jb.dst + t * 8, out);
    } break;
    case JOB_ETH1DATA: {
        if (t >= jb.n_in) return;
        const uint2* p = reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(jb.src) + t * 72);
        uint32_t r[18];
#pragma unroll
        for (int i = 0; i < 9; i++) { uint2 v = p[i]; r[2 * i] = bswap32(v.x); r[2 * i + 1] = bswap32(v.y); }
        uint32_t m[16], h0[8], h1[8], out[8];
        // (deposit_root, deposit_count)
#pragma unroll
        for (int i = 0; i < 8; i++) { m[i] = r[i]; m[8 + i] = 0; }
        m[8] = r[8]; m[9] = r[9];
        sha256_msg64(m, h0);
        // (block_hash, zero chunk)
#pragma unroll
        for (int i = 0; i < 8; i++) { m[i] = r[10 + i]; m[8 + i] = 0; }
        sha256_msg64(m, h1);
        hash_pair_words(h0, h1, out);
        store_node(jb.dst + t * 8, out);
    } break;
    default:
        break;
    }
}


// ---- folded upper levels: one pair-hash per thread per level, levels separated by __syncthreads (CoopJob, ssz_kernels.cuh)
__global__ void __launch_bounds__(kStageThreads) k_merkle_coop(const __grid_constant__ CoopDesc cd) {
    __shared__ uint32_t buf[2][kStageThreads][8];
    int j = 0;
#pragma unroll 1
    for (int k = 1; k < cd.njobs; k++)
        if (blockIdx.x >= cd.jobs[k].block_begin) j = k;
    const CoopJob& cj = cd.jobs[j];
    const uint32_t L = cj.nlev[0] + cj.nlev[1] + cj.nlev[2];     // 1..9
    const uint64_t cta = blockIdx.x - cj.block_begin;
    const uint32_t t = threadIdx.x;
    Job first{};   // the first job's input side, for fetch()
    first.src = cj.src; first.n_in = cj.n_in; first.level = cj.level; first.raw = cj.raw;
    uint32_t done = 0;          // levels completed
    int slot = 0;               // which of the folded jobs the next boundary belongs to
    uint32_t boundary = cj.nlev[0];
#pragma unroll 1
    for (uint32_t lv = 1; lv <= L; lv++) {
        const uint32_t width = 1u << (L - lv);              // nodes this CTA produces at this level
        uint32_t out[8];
        if (t < width) {
            uint32_t l[8], r[8];
            if (lv == 1) {
                const uint64_t i0 = (cta << L) + 2ull * t;
                fetch(first, cd.zero_nodes, i0, l);
                fetch(first, cd.zero_nodes, i0 + 1, r);
            } else {
#pragma unroll
                for (int w = 0; w < 8; w++) { l[w] = buf[lv & 1][2 * t][w]; r[w] = buf[lv & 1][2 * t + 1][w]; }
            }
            hash_pair_words(l, r, out);
#pragma unroll
            for (int w = 0; w < 8; w++) buf[(lv + 1) & 1][t][w] = out[w];
        }
        done = lv;
        if (done == boundary) {                              // a folded job ends here: its outputs go to the arena
            if (t < width) {
                const uint64_t idx = cta * width + t;
                const uint64_t n_out = (cj.n_in + (1ull << done) - 1) >> done;
                if (idx < n_out) store_node(cj.dst[slot] + idx * 8, out);
            }
            slot++;
            if (slot < 3) boundary += cj.nlev[slot];
        }
        __syncthreads();
    }
}

// ---- dirty-path variants (incremental re-hash of a device-resident state, SURVEY.md §8f-2) --------------------
// Same per-thread work as the dense kernels, but thread t handles output sel[t] of the job instead of output t.
__global__ void __launch_bounds__(kStageThreads) k_validator_roots_sparse(const __grid_constant__ Job jb,
                                                                          const uint32_t* __restrict__ sel, uint32_t n_sel) {
    __shared__ __align__(16) uint32_t smem[(kStageThreads * 121 + 16) / 4 + 4];
    const uint32_t t = blockIdx.x * kStageThreads + threadIdx.x;
    const bool valid = t < n_sel;
    const uint32_t rec = valid ? sel[t] : 0u;
    if (valid) {
        const uint8_t* g = reinterpret_cast<const uint8_t*>(jb.src) + uint64_t(rec) * 121u;
        uint8_t* sb = reinterpret_cast<uint8_t*>(smem) + threadIdx.x * 121u;
        for (int i = 0; i < 121; i++) sb[i] = g[i];  // each thread stages its own record
    }
    // smem_be_word loads whole words, which straddle the neighbouring threads' records (only this record's bytes are selected):
    // a block-wide barrier, not a warp one, so that no neighbour is still storing into a word this thread reads
    // (compute-sanitizer racecheck flagged the warp-level version; byte stores never clobbered the selected bytes, but it was a hazard)
    __syncthreads();
    if (!valid) return;
    uint32_t root[8];
    validator_root(smem, threadIdx.x * 121u, root);
    store_node(jb.dst + uint64_t(rec) * 8, root);
}
__global__ void __launch_bounds__(kStageThreads) k_merkle_reduce_sparse(const __grid_constant__ Job jb,
                                                                        const uint32_t* __restrict__ zero_nodes,
                                                                        const uint32_t* __restrict__ sel, uint32_t n_sel) {
    const uint32_t t = blockIdx.x * kStageThreads + threadIdx.x;
    if (t >= n_sel) return;
    const uint64_t o = sel[t];
    uint32_t out[8];
    switch (jb.nlev) {
    case 0: subtree<0>(jb, zero_nodes, o, out); break;
    case 1: subtree<1>(jb, zero_nodes, o << 1, out); break;
    case 2: subtree<2>(jb, zero_nodes, o << 2, out); break;
    default: subtree<3>(jb, zero_nodes, o << 3, out); break;
    }
    store_node(jb.dst + o * 8, out);
}
// REDUCE jobs of one tree level of several lists in one launch
__global__ void __launch_bounds__(kStageThreads) k_merkle_reduce_sparse_multi(const __grid_constant__ SparseDesc sd) {
    int j = 0;
#pragma unroll 1
    for (int k = 1; k < sd.njobs; k++)
        if (blockIdx.x >= sd.block_begin[k]) j = k;
    const Job& jb = sd.jobs[j];
    const uint32_t t = (blockIdx.x - sd.block_begin[j]) * kStageThreads + threadIdx.x;
    if (t >= sd.n_sel[j]) return;
    const uint64_t o = sd.sel[sd.sel_begin[j] + t];
    uint32_t out[8];
    switch (jb.nlev) {
    case 0: subtree<0>(jb, sd.zero_nodes, o, out); break;
    case 1: subtree<1>(jb, sd.zero_nodes, o << 1, out); break;
    case 2: subtree<2>(jb, sd.zero_nodes, o << 2, out); break;
    default: subtree<3>(jb, sd.zero_nodes, o << 3, out); break;
    }
    store_node(jb.dst + o * 8, out);
}
// dst[idx[i] * elem .. +elem) = vals[i * elem .. +elem)   (elem in {1, 8, 121}: byte copies, any alignment)
__global__ void k_scatter_elements(uint8_t* __restrict__ dst, const uint64_t* __restrict__ idx, const uint8_t* __restrict__ vals,
                                   uint32_t n, uint32_t elem) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint8_t* d = dst + idx[t] * elem;
    const uint8_t* v = vals + uint64_t(t) * elem;
    for (uint32_t i = 0; i < elem; i++) d[i] = v[i];
}

// Single-CTA finisher: executes the planner's op list wave by wave (all ops of a wave are independent).
__global__ void __launch_bounds__(kFinisherThreads) k_merkle_finisher(uint32_t* arena, const FinOp* ops,
                                                                        const uint32_t* wave_end, int nwaves, uint32_t first_op) {
    uint32_t begin = first_op;
#pragma unroll 1
    for (int w = 0; w < nwaves; w++) {
        const uint32_t end = wave_end[w];
#pragma unroll 1
        for (uint32_t i = begin + threadIdx.x; i < end; i += kFinisherThreads) {
            const FinOp op = ops[i];
            uint32_t l[8], r[8], out[8];
            load_node(arena + uint64_t(op.a) * 8, l);
            if (op.kind == FIN_COPY) {
                store_node(arena + uint64_t(op.dst) * 8, l);
                continue;
            }
            load_node(arena + uint64_t(op.b) * 8, r);
            hash_pair_words(l, r, out);
            store_node(arena + uint64_t(op.dst) * 8, out);
        }
        begin = end;
        __syncthreads();
    }
}

}  // namespace

// occupancy knobs (registers per thread vs resident warps); set once from B200_SSZ_MINB_{VALIDATORS,STAGE}
int g_minb_validators = 4;
int g_minb_stage = 4;
void set_ssz_tuning(int minb_validators, int minb_stage) {
    if (minb_validators >= 2 && minb_validators <= 4) g_minb_validators = minb_validators;
    if (minb_stage >= 2 && minb_stage <= 4) g_minb_stage = minb_stage;
}

void launch_validators(const Job& jb, void* stream) {
    if (jb.n_in == 0) return;
    const uint32_t nblocks = uint32_t((jb.n_in + kStageThreads - 1) / kStageThreads);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (g_minb_validators) {
    case 2: k_validator_roots<2><<<nblocks, kStageThreads, 0, st>>>(jb); break;
    case 4: k_validator_roots<4><<<nblocks, kStageThreads, 0, st>>>(jb); break;
    default: k_validator_roots<3><<<nblocks, kStageThreads, 0, st>>>(jb); break;
    }
}

void launch_stage(const StageDesc& sd, void* stream) {
    if (sd.nblocks == 0) return;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (g_minb_stage) {
    case 2: k_merkle_stage<2><<<sd.nblocks, kStageThreads, 0, st>>>(sd); break;
    case 4: k_merkle_stage<4><<<sd.nblocks, kStageThreads, 0, st>>>(sd); break;
    default: k_merkle_stage<3><<<sd.nblocks, kStageThreads, 0, st>>>(sd); break;
    }
}

void launch_coop(const CoopDesc& cd, void* stream) {
    if (cd.nblocks == 0) return;
    k_merkle_coop<<<cd.nblocks, kStageThreads, 0, static_cast<cudaStream_t>(stream)>>>(cd);
}

void launch_sparse(const Job& jb, const uint32_t* zero_nodes, const uint32_t* sel, uint32_t n_sel, void* stream) {
    if (!n_sel) return;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uint32_t nb = (n_sel + kStageThreads - 1) / kStageThreads;
    if (jb.type == JOB_VALIDATORS) k_validator_roots_sparse<<<nb, kStageThreads, 0, st>>>(jb, sel, n_sel);
    else k_merkle_reduce_sparse<<<nb, kStageThreads, 0, st>>>(jb, zero_nodes, sel, n_sel);
}
void launch_sparse_multi(const SparseDesc& sd, void* stream) {
    if (sd.njobs == 0 || sd.block_begin[sd.njobs] == 0) return;
    k_merkle_reduce_sparse_multi<<<sd.block_begin[sd.njobs], kStageThreads, 0, static_cast<cudaStream_t>(stream)>>>(sd);
}
void launch_scatter(uint8_t* dst, const uint64_t* idx, const uint8_t* vals, uint32_t n, uint32_t elem, void* stream) {
    if (!n) return;
    k_scatter_elements<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(dst, idx, vals, n, elem);
}

void launch_finisher(uint32_t* arena, const FinOp* ops, const uint32_t* wave_end, int nwaves, void* stream, uint32_t first_op) {
    if (nwaves == 0) return;
    k_merkle_finisher<<<1, kFinisherThreads, 0, static_cast<cudaStream_t>(stream)>>>(arena, ops, wave_end, nwaves, first_op);
}

}  // namespace b200
