// SSZ Merkle stage kernels: job descriptors shared by the host planner (ssz_plan.cu) and the kernels.
#pragma once
#include <cstdint>

namespace b200 {

enum JobType : uint32_t {
    JOB_REDUCE = 0,      // nodes/chunks -> nodes, nlev in {0,1,2,3} levels per thread, zero-hash padding
    JOB_VALIDATORS = 1,  // 121-byte SSZ Validator records -> hash_tree_root(Validator)
    JOB_PUBKEY48 = 2,    // 48-byte records -> hash_tree_root(ByteVector<48>) (1 hash)
    JOB_PAIR64 = 3,      // 64-byte records (two-chunk containers, e.g. HistoricalSummary) -> 1 hash
    JOB_ETH1DATA = 4,    // 72-byte Eth1Data records -> 3 hashes
};

struct Job {
    const void* src;      // device pointer (16-byte aligned)
    uint32_t* dst;        // device pointer into the node arena (word form, 8 words per node)
    uint64_t n_in;        // input elements
    uint32_t type;
    uint32_t level;       // REDUCE: tree level of the inputs (selects the zero-hash used as padding)
    uint32_t nlev;        // REDUCE: levels folded per thread (0 = convert only)
    uint32_t raw;         // REDUCE: inputs are raw SSZ bytes (byte-swap on load) instead of word-form nodes
    uint32_t block_begin; // first block of this job inside the stage launch
    uint32_t pad_;
};

constexpr int kMaxJobsPerStage = 24;
constexpr int kStageThreads = 256;

// Up to three CONSECUTIVE reduce jobs of one field (job k+1 reads what job k wrote) folded into one launch: a CTA owns
// 2^L inputs (L = sum of the jobs' levels <= 9), hashes them level by level in shared memory — one pair-hash per thread
// per level, __syncthreads between levels — and writes every job's output nodes where the separate launches would have.
// 9 levels cost 9 pair-hash latencies instead of the 21 of three thread-per-subtree stages: the upper, latency-bound
// part of a big list's tree (k_merkle_stage stays for the wide, throughput-bound lower stages).
struct CoopJob {
    const void* src;       // inputs of the first job
    uint32_t* dst[3];      // outputs of each folded job (node arena)
    uint64_t n_in;         // inputs of the first job
    uint32_t level;        // tree level of those inputs
    uint32_t nlev[3];      // levels folded by each job (0 = unused slot)
    uint32_t raw;          // first job's inputs are raw SSZ bytes
    uint32_t block_begin;
};
constexpr int kMaxCoopJobs = 12;
struct CoopDesc {
    CoopJob jobs[kMaxCoopJobs];
    int njobs;
    uint32_t nblocks;
    const uint32_t* zero_nodes;
};
void launch_coop(const CoopDesc& cd, void* stream);

struct StageDesc {
    Job jobs[kMaxJobsPerStage];
    int njobs;
    uint32_t nblocks;
    const uint32_t* zero_nodes;  // device: zero-subtree hashes, word form, 65 x 8 words
};

// One dirty-path launch for the same tree level of several lists (incremental re-hash): job k recomputes outputs
// sel[sel_begin[k] .. sel_begin[k] + n_sel[k]) — blocks [block_begin[k], block_begin[k+1]) belong to job k.
constexpr int kMaxSparseJobs = 12;
struct SparseDesc {
    Job jobs[kMaxSparseJobs];
    uint32_t sel_begin[kMaxSparseJobs];
    uint32_t n_sel[kMaxSparseJobs];
    uint32_t block_begin[kMaxSparseJobs + 1];
    int njobs;
    const uint32_t* zero_nodes;
    const uint32_t* sel;
};

// finisher op: arena[dst] = H(arena[a] || arena[b]) (kind 0) or arena[dst] = arena[a] (kind 1: gathers nodes into the
// contiguous send region of a multi-GPU exchange); indices are node indices into the arena
struct FinOp {
    uint32_t a, b, dst, kind;
};
enum FinKind : uint32_t { FIN_HASH = 0, FIN_COPY = 1 };

constexpr int kFinisherThreads = 1024;
constexpr int kMaxWaves = 256;

void launch_validators(const Job& jb, void* stream);
void launch_stage(const StageDesc& sd, void* stream);
// dirty-path variants: thread t handles output sel[t] (JOB_VALIDATORS or JOB_REDUCE only)
void launch_sparse(const Job& jb, const uint32_t* zero_nodes, const uint32_t* sel, uint32_t n_sel, void* stream);
void launch_sparse_multi(const SparseDesc& sd, void* stream);
void launch_scatter(uint8_t* dst, const uint64_t* idx, const uint8_t* vals, uint32_t n, uint32_t elem, void* stream);
// waves [0, nwaves) of `wave_end` (cumulative op counts); the first wave starts at op `first_op`
void launch_finisher(uint32_t* arena, const FinOp* ops, const uint32_t* wave_end, int nwaves, void* stream, uint32_t first_op = 0);

}  // namespace b200
