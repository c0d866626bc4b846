// Field reads of the 121-byte SSZ Validator records resident in HBM (phase0/validator.rs:10-26): pubkey 0..48,
// withdrawal_credentials 48..80, effective_balance 80..88, slashed 88, activation_eligibility_epoch 89..97,
// activation_epoch 97..105, exit_epoch 105..113, withdrawable_epoch 113..121.  Records are byte-aligned, so every u64 is
// assembled from bytes.  Shared by the active-index compaction (shuffle.cu) and the epoch kernels (epoch.cu).
#pragma once
#include <cstdint>

namespace b200 {

constexpr uint32_t kRecEffectiveBalance = 80, kRecSlashed = 88, kRecEligibility = 89, kRecActivation = 97, kRecExit = 105,
                   kRecWithdrawable = 113;

__device__ __forceinline__ uint64_t load_le64_unaligned(const uint8_t* p) {
    uint64_t v = 0;
#pragma unroll
    for (int k = 7; k >= 0; k--) v = (v << 8) | p[k];
    return v;
}
__device__ __forceinline__ void store_le64_unaligned(uint8_t* p, uint64_t v) {
#pragma unroll
    for (int k = 0; k < 8; k++) p[k] = uint8_t(v >> (8 * k));
}
// is_active_validator(v, epoch): activation_epoch <= epoch < exit_epoch
__device__ __forceinline__ bool record_active(const uint8_t* r, uint64_t epoch) {
    return load_le64_unaligned(r + kRecActivation) <= epoch && epoch < load_le64_unaligned(r + kRecExit);
}

}  // namespace b200
