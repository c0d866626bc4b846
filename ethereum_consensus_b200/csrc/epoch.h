// Device half of deneb process_epoch on a resident state (epoch.cu), driven by b200_state_process_epoch in capi_ssz.cu,
// and of the read-only b200_state_epoch_deltas beside it.
#pragma once
#include "engine.h"

namespace b200 {

// k_epoch_totals + k_epoch_reduce: every quantity the host step needs, from one pass over the records and both
// participation lists.  Sums are 128-bit (lo, hi) so that get_total_balance's overflow is visible.
struct EpochTotals {
    uint64_t lo[5], hi[5];   // 0 active effective balance at `cur`; 1..3 unslashed participating at `prev`, flags 0..2;
                             // 4 unslashed timely-target at `cur` (current participation)
    uint64_t n_active_cur, n_active_next, n_eject;
    uint64_t max_exit_plus1;  // 1 + the largest exit_epoch != FAR_FUTURE_EPOCH, 0 when there is none
    uint64_t n_at_max_exit;   // validators whose exit_epoch is that epoch
};

// What the host step decided, passed by value to k_epoch_apply (and to k_epoch_deltas, which reads the reward fields)
struct EpochParams {
    uint32_t steps;               // the B200_EPOCH_* bits whose per-validator work runs
    uint32_t leak;                // is_in_inactivity_leak, after justification
    uint64_t cur, prev;
    uint64_t base_per_inc;        // get_base_reward_per_increment
    uint64_t part_inc[3];         // unslashed participating increments per flag
    uint64_t active_inc;          // total active increments
    uint64_t finalized_epoch;     // after justification
    uint64_t exit0, c0, churn;    // exit queue: E0, c0, L
    uint64_t slash_epoch;         // cur + EPOCHS_PER_SLASHINGS_VECTOR / 2
    uint64_t adjusted_slashing, total_active;
    uint32_t activation_limit;    // min(MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT, L); 0 without the registry step
    uint64_t activation_epoch;    // compute_activation_exit_epoch(cur)
    // constants of the handle's preset (ssz_plan.h: preset_of)
    uint64_t increment, max_effective, ejection_balance, hysteresis_down, hysteresis_up;
    uint64_t score_bias, score_recovery, inactivity_denominator, withdraw_delay;
};

// Pass 1.  recs / participation are the resident lists (n entries each); *out (host) gets the totals.
int32_t epoch_totals_on_device(Engine& e, const uint8_t* recs, const uint8_t* prev_part, const uint8_t* cur_part, uint64_t n,
                               uint64_t cur, uint64_t prev, uint64_t ejection_balance, EpochTotals* out);
// Pass 2 (after epoch_totals_on_device on the same state): the fused per-validator step, then the activation queue.
// *n_changed (host) gets the number of Validator records written; their indices, possibly repeated, are at *changed_dev.
int32_t epoch_apply_on_device(Engine& e, uint8_t* recs, uint64_t* balances, uint64_t* scores, const uint8_t* prev_part,
                              uint64_t n, const EpochParams& p, const uint32_t** changed_dev, uint64_t* n_changed);
// The (reward, penalty) pairs of k_epoch_apply without applying them (after epoch_totals_on_device with the same
// participation list): *out_dev (device, valid until the next call) holds eight lists of n u64, source rewards, source
// penalties, target ..., head ..., inactivity rewards (zero), inactivity penalties.  Reads p's prev, leak, base_per_inc,
// part_inc, active_inc, increment and inactivity_denominator.
int32_t epoch_deltas_on_device(Engine& e, const uint8_t* recs, const uint64_t* scores, const uint8_t* part, uint64_t n,
                               const EpochParams& p, const uint64_t** out_dev);

}  // namespace b200
