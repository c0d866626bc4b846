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
    bool reserved = false;    // region sized for a capacity beyond nbytes: the whole tail is cleared on upload
};

// One big list of a device-resident state: its staged bytes and the sequence of jobs that reduces them to <= kHandoff
// nodes.  `jobs[k]` = (stage, index in that stage), stage -1 = validator_jobs_.  Job k+1 reads exactly job k's output.
// `arena` = every node range allocated for the chain (all levels, at capacity when the list was planned with one).
struct PChain {
    int copy = -1;
    std::vector<std::pair<int, size_t>> jobs;
    std::vector<std::pair<uint64_t, uint64_t>> arena;  // (first node, node count)
};

// A wide list reduced to <= kHandoff nodes at `level`; SszPlan::finish() adds the finisher ops up to `depth`.
struct Handoff {
    std::vector<uint32_t> nodes;
    int level = 0, depth = 0;
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
    // stage a host region into the field buffer (16-byte padded, 256-byte aligned); `reserve_bytes` > nbytes sizes the
    // region for a list that may grow in place (the tail is zeroed when the region is uploaded)
    uint64_t stage_field(const uint8_t* src, size_t nbytes, size_t reserve_bytes = 0);
    // root at depth_target of `n` chunks/records living in the field buffer
    uint32_t wide_chunks(uint64_t field_off, uint64_t n_chunks, int depth_target);
    uint32_t wide_records(uint32_t type, uint64_t field_off, uint64_t n, int depth_target);
    // generic: n nodes at `level`, located at src, reduced to depth_target starting at stage `s`
    uint32_t wide_nodes(PSrc src, bool raw, uint64_t n, int level, int depth_target, size_t s);

    // The same two reductions without their finisher ops, so that a resident plan can allocate every chain's arena
    // levels before any finisher node.  `cap` (> 0): inputs the arena levels are sized for (>= n, every level of a
    // cap-input tree is allocated, plus a kHandoff-node region for the word-form conversion of a short raw list): the
    // positions then depend on `cap` only, and a list that grows up to `cap` keeps them.
    Handoff chunks_to_handoff(uint64_t field_off, uint64_t n_chunks, int depth_target, uint64_t cap_chunks = 0);
    Handoff records_to_handoff(uint32_t type, uint64_t field_off, uint64_t n, int depth_target, uint64_t cap = 0);
    uint32_t finish(const Handoff& h) { return merkle_small(h.nodes, h.level, h.depth); }

    // n+1 48-byte records (n vector elements + 1 extra key) hashed by one job; returns the vector root
    uint32_t wide_pubkeys_with_extra(uint64_t field_off, uint64_t n, int depth_target, uint32_t* extra);

    // jobs and staged bytes added between begin_chain() and end_chain() belong to one big list
    int begin_chain() { chains_.emplace_back(); cur_chain_ = int(chains_.size()) - 1; return cur_chain_; }
    void end_chain() { cur_chain_ = -1; }
    size_t n_chains() const { return chains_.size(); }
    // device byte offset (in the field buffer) and byte length of chain c's staged list; false if the list is empty
    bool chain_field(int c, uint64_t* field_off, size_t* nbytes) const;
    // byte size of chain c's field-buffer region (reserved capacity included) and its arena node ranges
    size_t chain_region_bytes(int c) const;
    const std::vector<std::pair<uint64_t, uint64_t>>& chain_arena(int c) const { return chains_[size_t(c)].arena; }
    // chain c sits at the same field-buffer region and arena ranges in both plans
    bool same_chain_layout(const SszPlan& o, int c) const;
    // chain c runs the same job sequence (stages, levels, sources, destinations) in both plans; input counts may differ
    bool same_chain_jobs(const SszPlan& o, int c) const;

    // ---- execution ----
    // Uploads fields (+plan) and runs; `copy`: which staged fields to copy H2D first (COPY_NONE: device-resident state,
    // COPY_SMALL_ONLY: everything except the chains' lists).
    // `dirty` (optional, one sorted-unique vector per chain: indices of changed first-job inputs — Validator records, or
    // 32-byte chunks of a packed list): the chains' jobs then only recompute the paths above those inputs.
    // `changed_host_ranges` (COPY_SMALL_ONLY): copy only the staged fields whose host bytes intersect one of these ranges.
    // `outputs`: arena nodes to read back (32 bytes each, SSZ byte order) into `out`.
    // `rehash` (with `dirty`, one flag per chain): these chains are re-hashed in full from their resident data instead
    // of along dirty paths (their job sequence changed, or they were relocated).
    int32_t run(Engine& e, DevBuf& arena, DevBuf& fields, DevBuf& planbuf, CopyMode copy,
                const std::vector<uint32_t>& outputs, uint8_t* out,
                const std::vector<std::vector<uint32_t>>* dirty = nullptr, DevBuf* selbuf = nullptr,
                const std::vector<std::pair<const uint8_t*, const uint8_t*>>* changed_host_ranges = nullptr,
                const std::vector<char>* rehash = nullptr);
    bool has_exchange() const { return xch_n_ != 0; }

    size_t field_bytes() const { return field_next_; }
    uint64_t arena_nodes() const { return arena_next_; }
    uint64_t h2d_bytes() const;

private:
    uint64_t arena_alloc(uint64_t n) {
        uint64_t r = arena_next_; arena_next_ += n;
        if (cur_chain_ >= 0) chains_[size_t(cur_chain_)].arena.emplace_back(r, n);
        return r;
    }
    void add_job(size_t stage, const PJob& j);
    Handoff reduce_to_handoff(PSrc src, bool raw, uint64_t n, int level, int depth_target, size_t s, uint64_t cap);
    const PJob& chain_job(int c, size_t k) const {
        const auto& ref = chains_[size_t(c)].jobs[k];
        return ref.first < 0 ? validator_jobs_[ref.second] : stages_[size_t(ref.first)][ref.second];
    }

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

inline uint32_t le32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | (uint32_t(p[3]) << 24); }
inline uint64_t le64(const uint8_t* p) { return uint64_t(le32(p)) | (uint64_t(le32(p + 4)) << 32); }

// The constants of a preset that the state plans, the duties and process_epoch read
struct Preset {
    uint64_t slots_per_epoch, slots_per_historical_root, historical_roots_limit, eth1_data_votes_bound,
        validator_registry_limit, epochs_per_historical_vector, epochs_per_slashings_vector, sync_committee_size;
    uint64_t epochs_per_sync_committee_period, shuffle_round_count;
    // process_epoch
    uint64_t epochs_per_eth1_voting_period, min_per_epoch_churn_limit, max_per_epoch_activation_churn_limit,
        churn_limit_quotient;
    uint64_t effective_balance_increment, max_effective_balance, ejection_balance;
    uint64_t hysteresis_quotient, hysteresis_downward_multiplier, hysteresis_upward_multiplier;
    uint64_t inactivity_score_bias, inactivity_score_recovery_rate, inactivity_penalty_quotient_bellatrix;
    uint64_t proportional_slashing_multiplier_bellatrix, base_reward_factor, min_epochs_to_inactivity_penalty;
    uint64_t max_seed_lookahead, min_validator_withdrawability_delay;
    // beacon committees (phase0/helpers.rs:741-806) and process_attestation (deneb/block_processing.rs:53-100)
    uint64_t target_committee_size, max_committees_per_slot, max_validators_per_committee, min_attestation_inclusion_delay;
};
const Preset& preset_of(int preset);   // B200_PRESET_MAINNET or B200_PRESET_MINIMAL

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
    uint32_t var_word[9] = {0};  // byte position of each offset word in the fixed part
};
bool parse_beacon_state(const uint8_t* ssz, size_t len, int preset, StateOffsets& so);

// The nine chains of a resident state plan: 0..4 the five big lists in B200_FIELD_* order (validators, balances,
// previous / current epoch participation, inactivity_scores), 5..8 the four big vectors (block_roots, state_roots,
// randao_mixes, slashings).  The sharded plans slice the five lists the same way.
struct StateChain {
    int var;            // StateOffsets::var index of a big list, -1 for a vector
    uint64_t lo, hi;    // byte range in the serialization
    uint32_t elem;      // element size in bytes
    uint32_t unit;      // bytes per first-job input: a 121-byte Validator record or a 32-byte chunk
    uint64_t len;       // elements
    uint64_t n_inputs;  // first-job inputs
    int depth;          // Merkle depth of the data (below a list's length mix-in)
    uint64_t bytes() const { return hi - lo; }
    uint32_t input_of(uint64_t i) const { return uint32_t(i * elem / unit); }   // the input covering element i
};
StateChain state_chain(const StateOffsets& so, const Preset& P, int c);

// The two small lists that grow by appending (B200_FIELD_ETH1_DATA_VOTES, B200_FIELD_HISTORICAL_SUMMARIES): their
// StateOffsets::var index, element size and limit.  var = -1 for any other field id.
struct SmallList {
    int var = -1;
    uint32_t elem = 0;
    uint64_t limit = 0;
};
SmallList appendable_small_list(int field, const Preset& P);

// `caps` (optional, element counts of the five big lists, each >= the list's length): the lists' field regions and arena
// levels are reserved for that many elements and are laid out, with the four big vectors, ahead of everything whose size
// depends on a small variable-size field — a device-resident state can then grow or reshape without moving them.
int32_t build_beacon_state_plan(SszPlan& plan, const uint8_t* ssz, size_t len, int preset, std::vector<uint32_t>& outputs,
                                const uint64_t* caps = nullptr);
int32_t build_beacon_state_shard_plan(SszPlan& plan, const uint8_t* ssz, size_t len, int preset, int rank, int world,
                                      std::vector<uint32_t>& outputs);
int32_t build_beacon_state_sharded_plan(SszPlan& plan, const uint8_t* ssz, size_t len, int preset, int rank, int world,
                                        std::vector<uint32_t>& outputs);
int32_t build_beacon_state_combine_plan(SszPlan& plan, const uint8_t* ssz, size_t len, int preset, int world,
                                        const uint8_t* all_roots, std::vector<uint32_t>& outputs);

int32_t ensure_zero_nodes(Engine& e);

}  // namespace b200
