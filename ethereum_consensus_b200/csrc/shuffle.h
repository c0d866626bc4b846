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
}  // namespace b200
