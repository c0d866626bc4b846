// Host-side planner for SSZ hash_tree_root on the device: turns a container instance into
//   (a) H2D copies of its big fields into 256-byte-aligned device regions,
//   (b) wide stage launches (ssz_kernels.cu) over those regions,
//   (c) a finisher op list for everything small (tops of trees, zero-hash chains, mix-ins, small containers).
// The planner does no hashing itself; all SHA-256 work happens on the device.
#pragma once
#include <cstdint>
#include <cstring>
#include <unordered_map>
#include <vector>

#include "engine.h"
#include "ssz_kernels.cuh"

namespace b200 {

// source of a wide job: either a region of the field buffer (raw SSZ bytes) or nodes in the arena
struct PSrc {
    bool in_arena = false;
    uint64_t off = 0;  // byte offset in the field buffer, or node index in the arena
};

struct PJob {
    uint32_t type = JOB_REDUCE;
    PSrc src;
    uint64_t dst = 0;  // node index in the arena
    uint64_t n_in = 0;
    uint32_t level = 0, nlev = 0, raw = 0;
    int chain = -1;  // index into SszPlan::chains_ for the jobs of a big list (dirty-path re-hash), else -1
    int copy = -1;   // index into SszPlan::copies_ of the staged field this job (transitively) reads, else -1
};

struct HostCopy {
    const uint8_t* src;
    size_t nbytes;
    uint64_t field_off;
    size_t zero_tail;  // bytes to clear after the copy (keeps the last partial chunk zero-padded)
    bool validators = false;  // the big Validator list: copied in slices so hashing overlaps the PCIe transfer
    int chain = -1;
};

// One big list of a device-resident state: its staged bytes and the sequence of jobs that reduces them to <= kHandoff
// nodes.  `jobs[k]` = (stage, index in that stage), stage -1 = validator_jobs_.  Job k+1 reads exactly job k's output.
struct PChain {
    int copy = -1;
    std::vector<std::pair<int, size_t>> jobs;
};

enum CopyMode { COPY_ALL = 0, COPY_NONE = 1, COPY_SMALL_ONLY = 2 };

class SszPlan {
public:
    static constexpr uint32_t kZeroBase = 0;   // arena[0..65) = zero-subtree hashes
    static constexpr uint64_t kHandoff = 64;   // <= this many nodes: finish in the single-CTA finisher

    SszPlan() = default;

    // ---- building blocks (return arena node indices) ----
    uint32_t zero(int depth) const { return kZeroBase + uint32_t(depth); }
    uint32_t leaf(const uint8_t chunk[32]);              // small leaf uploaded with the plan
    uint32_t leaf_u64(uint64_t v);
    uint32_t leaf_bytes(const uint8_t* p, size_t n);     // n <= 32, right-padded
    uint32_t hash2(uint32_t a, uint32_t b);              // finisher op
    uint32_t mix_in_length(uint32_t root, uint64_t len) { return hash2(root, leaf_u64(len)); }
    // ---- multi-GPU exchange (one per plan): `n` local nodes are gathered into a contiguous send region by the last
    // wave of finisher pass 1, one all-gather fills world x n remote nodes, and every op that depends on a remote node
    // runs in finisher pass 2.  Returns the first remote node; rank r's copy of local[i] is remote + r*n + i.
    uint32_t exchange(const std::vector<uint32_t>& local, int world);
    // root (at `depth_target`) of explicit nodes sitting at `level`
    uint32_t merkle_small(std::vector<uint32_t> nodes, int level, int depth_target);
    // container of small field roots
    uint32_t container(const std::vector<uint32_t>& field_roots);
    // stage a host region into the field buffer (16-byte padded, 256-byte aligned)
    uint64_t stage_field(const uint8_t* src, size_t nbytes);
    // root at depth_target of `n` chunks/records living in the field buffer
    uint32_t wide_chunks(uint64_t field_off, uint64_t n_chunks, int depth_target);
    uint32_t wide_records(uint32_t type, uint64_t field_off, uint64_t n, int depth_target);
    // generic: n nodes at `level`, located at src, reduced to depth_target starting at stage `s`
    uint32_t wide_nodes(PSrc src, bool raw, uint64_t n, int level, int depth_target, size_t s);

    // n+1 48-byte records (n vector elements + 1 extra key) hashed by one job; returns the vector root
    uint32_t wide_pubkeys_with_extra(uint64_t field_off, uint64_t n, int depth_target, uint32_t* extra);

    // jobs and staged bytes added between begin_chain() and end_chain() belong to one big list
    int begin_chain() { chains_.emplace_back(); cur_chain_ = int(chains_.size()) - 1; return cur_chain_; }
    void end_chain() { cur_chain_ = -1; }
    size_t n_chains() const { return chains_.size(); }
    // device byte offset (in the field buffer) and byte length of chain c's staged list; false if the list is empty
    bool chain_field(int c, uint64_t* field_off, size_t* nbytes) const;

    // ---- execution ----
    // Uploads fields (+plan) and runs; `copy`: which staged fields to copy H2D first (COPY_NONE: device-resident state,
    // COPY_SMALL_ONLY: everything except the chains' lists).
    // `dirty` (optional, one sorted-unique vector per chain: indices of changed first-job inputs — Validator records, or
    // 32-byte chunks of a packed list): the chains' jobs then only recompute the paths above those inputs.
    // `changed_host_ranges` (COPY_SMALL_ONLY): copy only the staged fields whose host bytes intersect one of these ranges.
    // `outputs`: arena nodes to read back (32 bytes each, SSZ byte order) into `out`.
    int32_t run(Engine& e, DevBuf& arena, DevBuf& fields, DevBuf& planbuf, CopyMode copy,
                const std::vector<uint32_t>& outputs, uint8_t* out,
                const std::vector<std::vector<uint32_t>>* dirty = nullptr, DevBuf* selbuf = nullptr,
                const std::vector<std::pair<const uint8_t*, const uint8_t*>>* changed_host_ranges = nullptr);
    bool has_exchange() const { return xch_n_ != 0; }

    size_t field_bytes() const { return field_next_; }
    uint64_t arena_nodes() const { return arena_next_; }
    uint64_t h2d_bytes() const;

private:
    uint64_t arena_alloc(uint64_t n) { uint64_t r = arena_next_; arena_next_ += n; return r; }
    void add_job(size_t stage, const PJob& j);

    std::vector<PJob> validator_jobs_;
    std::vector<std::vector<PJob>> stages_;
    std::vector<FinOp> ops_;
    std::vector<int> op_wave_;
    std::unordered_map<uint32_t, int> ready_;  // finisher-produced node -> first wave in which it is readable
    std::vector<uint32_t> small_words_; // word-form image of small leaves
    std::vector<uint32_t> small_idx_;   // arena idx of each small leaf
    std::vector<HostCopy> copies_;
    std::vector<PChain> chains_;
    int cur_chain_ = -1;
    int cur_copy_ = -1;   // staged field of the wide_* call being planned (stamped on its jobs)
    int copy_of(uint64_t field_off) const;
    // exchange(): send region, receive region, nodes per rank, world
    uint32_t xch_send_ = 0, xch_recv_ = 0, xch_n_ = 0;
    int xch_world_ = 0;
    static constexpr int kRemoteWave = 1 << 20;  // readiness wave of a remote node: splits the finisher in two passes
    uint64_t arena_next_ = 65 + 8192;  // [0,65) zero hashes, [65, 65+8192) small leaves uploaded with the plan
    size_t field_next_ = 0;

    int ready_wave(uint32_t idx) const;
};

int depth_for(uint64_t n);

// deneb BeaconState (ethereum-consensus/src/deneb/beacon_state.rs:26-63): byte offsets of the
// fixed-size fields and of the nine variable-size fields inside the SSZ serialization.
struct StateOffsets {
    size_t fixed = 0;
    size_t block_roots = 0, state_roots = 0, eth1_data = 0, eth1_deposit_index = 0, randao_mixes = 0, slashings = 0,
           justification_bits = 0, checkpoints = 0, current_sync_committee = 0, next_sync_committee = 0,
           next_withdrawal_index = 0, next_withdrawal_validator_index = 0;
    // historical_roots, eth1_data_votes, validators, balances, previous/current participation, inactivity_scores,
    // latest_execution_payload_header, historical_summaries, end
    uint32_t var[10] = {0};
};
bool parse_beacon_state(const uint8_t* ssz, size_t len, int preset, StateOffsets& so);
int32_t build_beacon_state_plan(SszPlan& plan, const uint8_t* ssz, size_t len, int preset, std::vector<uint32_t>& outputs);
int32_t build_beacon_state_shard_plan(SszPlan& plan, const uint8_t* ssz, size_t len, int preset, int rank, int world,
                                      std::vector<uint32_t>& outputs);
int32_t build_beacon_state_sharded_plan(SszPlan& plan, const uint8_t* ssz, size_t len, int preset, int rank, int world,
                                        std::vector<uint32_t>& outputs);
int32_t build_beacon_state_combine_plan(SszPlan& plan, const uint8_t* ssz, size_t len, int preset, int world,
                                        const uint8_t* all_roots, std::vector<uint32_t>& outputs);

int32_t ensure_zero_nodes(Engine& e);

}  // namespace b200
