// Device-side building blocks of shuffle.cu used by the resident-state entry point in capi_ssz.cu.
#pragma once
#include "engine.h"

namespace b200 {
int32_t shuffle_on_device(Engine& e, const uint64_t* idx_dev, uint64_t n, const uint8_t seed[32], uint32_t rounds, uint64_t* out_dev);
int32_t active_indices_on_device(Engine& e, const uint8_t* recs_dev, uint64_t n, uint64_t epoch, uint64_t* out_dev, uint64_t* out_n);
int32_t shuffle_scratch(Engine& e, uint64_t n, uint64_t** a, uint64_t** b);
// compute_proposer_index for n_seeds 32-byte slot seeds (host) over the n active indices at active_dev: out (host) gets one
// validator index per seed.  B200_ERR_LIMIT past the candidate cap.
int32_t sample_proposers_on_device(Engine& e, const uint8_t* seeds, uint32_t n_seeds, uint32_t rounds, const uint64_t* active_dev,
                                   uint64_t n, const uint8_t* recs_dev, uint64_t* out);
// get_next_sync_committee_indices' loop: the first `size` accepted candidates of `seed` into out_dev (device, size entries)
int32_t sample_committee_on_device(Engine& e, const uint8_t seed[32], uint32_t size, uint32_t rounds, const uint64_t* active_dev,
                                   uint64_t n, const uint8_t* recs_dev, uint64_t* out_dev);
// out[k] (host) = the largest i with record i's public key == keys[k] (host, m <= 512 keys of 48 bytes), UINT64_MAX if none
int32_t match_committee_keys_on_device(Engine& e, const uint8_t* recs_dev, uint64_t n, const uint8_t* keys, uint32_t m, uint64_t* out);

// ---- beacon committees over an epoch's shuffled active list (n_active entries, device) ----
constexpr uint32_t kNotActive = 0xffffffffu;      // position-map entry of a validator not active at the epoch
constexpr uint32_t kMaxCommitteeBits = 2048;       // MAX_VALIDATORS_PER_COMMITTEE, both presets
// pos_dev (device, n_validators u32) = each validator's position in the shuffled list, kNotActive for the others
int32_t committee_positions_on_device(Engine& e, const uint64_t* shuffled_dev, uint64_t n_active, uint64_t n_validators, uint32_t* pos_dev);
// out_dev (device, n_rows x 5 u64) = the AttestationDuty row of validators_dev[r] (device; nullptr: r) from pos_dev
int32_t attester_duties_on_device(Engine& e, const uint32_t* pos_dev, const uint64_t* validators_dev, uint64_t n_rows, uint64_t n_active,
                                  uint64_t cps, uint64_t slots_per_epoch, uint64_t epoch, uint64_t* out_dev);
// One attestation's gather: its committee slice (device, len <= kMaxCommitteeBits members), its Bitlist's first byte in
// the bits buffer, and where its sorted attesting indices go in the output
struct AttestingJob {
    const uint64_t* committee;
    uint32_t len, bits_off, out_off, pad;
};
int32_t attesting_indices_on_device(Engine& e, const AttestingJob* jobs_dev, uint32_t n_jobs, const uint8_t* bits_dev, uint64_t* out_dev);
}  // namespace b200
