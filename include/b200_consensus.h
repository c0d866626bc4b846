/*
 * b200_consensus.h — C ABI of the H100-native batch-crypto engine.
 *
 * This is the drop-in boundary for ralexstokes/ethereum_consensus' hot path (SURVEY.md §8b):
 *   - BLS:  the seven free functions re-exported at
 *           ethereum-consensus/src/crypto/mod.rs:4-8 (bodies in crypto/bls.rs:64-160), whose only
 *           backend today is `use blst::{min_pk as bls_impl, BLST_ERROR}` (crypto/bls.rs:4);
 *   - SSZ:  `HashTreeRoot::hash_tree_root` / `merkleize` / `is_valid_merkle_branch` from
 *           `pub use ssz_rs::prelude::*` (ethereum-consensus/src/ssz/mod.rs:6).
 * Plain pointers and sizes only; the caller owns every buffer; calls are synchronous and thread-safe (one
 * process-global context per device).  INTEGRATION.md shows the Rust `extern "C"` block that binds these.
 *
 * Return codes: 0..7 are blst's BLST_ERROR values (order pinned by
 * ethereum-consensus/src/crypto/bls.rs:48-62); >= 0x100 are engine failures (CUDA, bad
 * arguments, malformed SSZ) and are NEVER conflated with a signature verdict.  There is no CPU fallback: if
 * the device or the CUDA library is unavailable every entry point returns B200_ERR_NO_DEVICE / B200_ERR_CUDA.
 */
#ifndef B200_CONSENSUS_H
#define B200_CONSENSUS_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ---- return codes -------------------------------------------------------------------------------- */
enum {
    B200_SUCCESS = 0,            /* BLST_SUCCESS */
    B200_BAD_ENCODING = 1,       /* BLST_BAD_ENCODING */
    B200_POINT_NOT_ON_CURVE = 2, /* BLST_POINT_NOT_ON_CURVE */
    B200_POINT_NOT_IN_GROUP = 3, /* BLST_POINT_NOT_IN_GROUP */
    B200_AGGR_TYPE_MISMATCH = 4, /* BLST_AGGR_TYPE_MISMATCH */
    B200_VERIFY_FAIL = 5,        /* BLST_VERIFY_FAIL  -> Error::InvalidSignature (crypto/bls.rs:127-131) */
    B200_PK_IS_INFINITY = 6,     /* BLST_PK_IS_INFINITY */
    B200_BAD_SCALAR = 7,         /* BLST_BAD_SCALAR */
    B200_EMPTY_AGGREGATE = 16,   /* Error::EmptyAggregate (crypto/bls.rs:80-82,136-138) */
    B200_ERR_CUDA = 0x100,
    B200_ERR_NO_DEVICE = 0x101,
    B200_ERR_BAD_ARG = 0x102,
    B200_ERR_SSZ_MALFORMED = 0x103, /* offsets / lengths inconsistent with the container schema */
    B200_ERR_NOT_INITIALIZED = 0x104,
    B200_ERR_LIMIT = 0x105,         /* more chunks than the declared limit (MerkleizationError) */
    B200_ERR_COMM = 0x106           /* NCCL missing / communicator failure (multi-GPU entry points) */
};

enum { B200_PRESET_MAINNET = 0, B200_PRESET_MINIMAL = 1 };

/* ---- life cycle ------------------------------------------------------------------------------------ */
/* Binds the calling process to CUDA device `device` (one process per GPU).  Idempotent. */
B200_API int32_t b200_init(int32_t device);
B200_API void b200_shutdown(void);
/* Human-readable text for the last engine failure (>= 0x100) on this thread's context. */
B200_API const char* b200_last_error(void);
/* Number of kernel launches issued by the library since b200_init (bench.py's gpu_launches). */
B200_API uint64_t b200_launch_count(void);
/* Device time (ms, CUDA events on the library stream) of the kernels of the last SSZ / BLS call. */
B200_API float b200_last_kernel_ms(void);

/* ---- SSZ / SHA-256 Merkle (replaces ssz_rs merkleize / hash_tree_root; sha2 one-shot) -------------- */
/* crypto::hash — ethereum-consensus/src/crypto/bls.rs:12-20 (computed on the device). */
B200_API int32_t b200_sha256(const uint8_t* data, size_t len, uint8_t out[32]);

/* merkleize(chunks, limit): `n_chunks` 32-byte chunks, virtually zero-padded to `limit` chunks
 * (limit == 0: next power of two of n_chunks).  ssz_rs `merkleize`. */
B200_API int32_t b200_merkleize(const uint8_t* chunks, size_t n_chunks, uint64_t limit, uint8_t out[32]);
/* mix_in_length(root, len) */
B200_API int32_t b200_mix_in_length(const uint8_t root[32], uint64_t length, uint8_t out[32]);
/* is_valid_merkle_branch(leaf, branch[depth], depth, index, root): *ok = 1/0.
 * Used at ethereum-consensus/src/phase0/block_processing.rs:428-437 and deneb/blob_sidecar.rs:58-63. */
B200_API int32_t b200_is_valid_merkle_branch(const uint8_t leaf[32], const uint8_t* branch, size_t depth, uint64_t index,
                                    const uint8_t root[32], int32_t* ok);

/* hash_tree_root(List<Validator, limit>) from N x 121 bytes of SSZ (phase0/validator.rs:10-26). */
B200_API int32_t b200_htr_validators(const uint8_t* ssz, size_t n, uint64_t limit, uint8_t out[32]);
/* hash_tree_root of a packed basic List (is_list=1, mixes `length`) or Vector (is_list=0):
 * `nbytes` of little-endian elements, limit in chunks. */
B200_API int32_t b200_htr_packed(const uint8_t* data, size_t nbytes, uint64_t limit_chunks, int32_t is_list, uint64_t length,
                        uint8_t out[32]);

/* hash_tree_root(deneb::BeaconState) from its SSZ serialization
 * (ethereum-consensus/src/deneb/beacon_state.rs:13-64; called at deneb/spec/mod.rs:3215,3288). */
B200_API int32_t b200_htr_beacon_state_deneb(const uint8_t* ssz, size_t len, int32_t preset, uint8_t out[32]);

/* Device-resident state: upload once, re-hash many times (kernel-only cost; SURVEY.md §8f-2 groundwork). */
typedef struct b200_state b200_state;
B200_API int32_t b200_state_upload_deneb(const uint8_t* ssz, size_t len, int32_t preset, b200_state** out_handle);
B200_API int32_t b200_state_root(b200_state* handle, uint8_t out[32]);
B200_API void b200_state_free(b200_state* handle);

/* Incremental re-hash of a device-resident state (SURVEY.md §8b `b200_state_update_leaves`, §8f-2): the two
 * `state.hash_tree_root()` calls per block (deneb/spec/mod.rs:3215,3288) then cost O(changed x depth), not O(N).
 *  - b200_state_update_elements: overwrite elements `indices[i]` of one of the five big lists with `values`
 *    (n x 121 / 8 / 1 bytes, SSZ encoding of Validator / u64 / participation flags).  List lengths do not change;
 *    an index may appear more than once only with identical values (elements are written in parallel).
 *  - b200_state_update_bytes: overwrite bytes [ssz_offset, ssz_offset + n) of the serialization that was uploaded
 *    (any field; must not change a variable-size field's offset or length — the two reshaping calls below do that).
 *    Offsets refer to the serialization as it is now, after any reshape.
 *  - b200_state_root_incremental: root after the updates.  Dirty paths of the big lists only; everything small
 *    (~1 % of the hashes) is re-hashed in full.  b200_state_root stays the full O(N) re-hash. */
#define B200_FIELD_VALIDATORS 0
#define B200_FIELD_BALANCES 1
#define B200_FIELD_PREVIOUS_EPOCH_PARTICIPATION 2
#define B200_FIELD_CURRENT_EPOCH_PARTICIPATION 3
#define B200_FIELD_INACTIVITY_SCORES 4
#define B200_FIELD_ETH1_DATA_VOTES 5
#define B200_FIELD_HISTORICAL_SUMMARIES 6
#define B200_FIELD_LATEST_EXECUTION_PAYLOAD_HEADER 7
B200_API int32_t b200_state_update_elements(b200_state* handle, int32_t field, const uint64_t* indices, const uint8_t* values, size_t n);
B200_API int32_t b200_state_update_bytes(b200_state* handle, uint64_t ssz_offset, const uint8_t* data, size_t n);
B200_API int32_t b200_state_root_incremental(b200_state* handle, uint8_t out[32]);

/* Shape changes of a device-resident state (single-GPU handles; a sharded handle gets B200_ERR_BAD_ARG).  The library
 * rewrites the offset words of the fixed part; b200_state_update_bytes, b200_state_update_elements,
 * b200_state_shuffled_active_indices and both roots then see the state as reshaped.
 *  - b200_state_append_elements: the spec's `.push` of `n` elements, SSZ-encoded back to back in `values`, onto one of
 *    the five big lists (121 / 8 / 1 / 1 / 8-byte elements; the lists grow independently: a deposit appends to all five),
 *    B200_FIELD_ETH1_DATA_VOTES (72-byte Eth1Data) or B200_FIELD_HISTORICAL_SUMMARIES (64-byte HistoricalSummary).
 *    A big list's device regions hold its length plus max(2^16, length / 16) elements: an append within them copies
 *    only the appended bytes; past them the list is relocated on the device (device-to-device copy) and re-hashed in
 *    full from HBM at the next root.
 *  - b200_state_set_field: replace a whole small variable-size value: B200_FIELD_ETH1_DATA_VOTES (`len` a multiple of
 *    72; 0 is the voting-period reset) or B200_FIELD_LATEST_EXECUTION_PAYLOAD_HEADER (584 fixed bytes whose
 *    extra_data offset, at byte 436, is 584, then 0..32 bytes of extra_data).
 * Errors: beyond VALIDATOR_REGISTRY_LIMIT, ETH1_DATA_VOTES_BOUND or HISTORICAL_ROOTS_LIMIT (or a serialization past the
 * 4 GiB its offsets can address) -> B200_ERR_LIMIT; a length that is not a multiple of the element size or a malformed
 * header -> B200_ERR_SSZ_MALFORMED; any other field id -> B200_ERR_BAD_ARG.  A refused call leaves the handle as it was. */
B200_API int32_t b200_state_append_elements(b200_state* handle, int32_t field, const uint8_t* values, size_t n);
B200_API int32_t b200_state_set_field(b200_state* handle, int32_t field, const uint8_t* ssz, size_t len);

/* Multi-GPU sharding of hash_tree_root(BeaconState) (SURVEY.md §8e): rank r of `world` hashes its contiguous
 * power-of-two-aligned slice of the five big lists and returns one subtree root per list
 * (out_roots: 5 x 32 bytes, order validators, balances, previous/current participation, inactivity_scores);
 * after an allgather of those roots, b200_htr_beacon_state_deneb_combine finishes the tree on any rank. */
B200_API int32_t b200_htr_beacon_state_deneb_shard(const uint8_t* ssz, size_t len, int32_t preset, int32_t rank, int32_t world,
                                          uint8_t* out_roots /* 5*32 */);
B200_API int32_t b200_htr_beacon_state_deneb_combine(const uint8_t* ssz, size_t len, int32_t preset, int32_t world,
                                            const uint8_t* all_roots /* world*5*32 */, uint8_t out[32]);

/* ---- committee shuffling (SURVEY.md §8f-3): the step before the BLS hot path ---------------------------------- */
/* compute_shuffled_indices — ethereum-consensus/src/phase0/helpers.rs:287-360 (whole list; equal to
 * mapping every position through compute_shuffled_index, :249-283): out[i] = indices[shuffled_index(i, n, seed)].
 * `indices` == NULL means the identity list 0..n-1; `rounds` = SHUFFLE_ROUND_COUNT (90 on mainnet, 10 on minimal). */
B200_API int32_t b200_compute_shuffled_indices(const uint64_t* indices, size_t n, const uint8_t seed[32], uint32_t rounds,
                                               uint64_t* out);
/* get_active_validator_indices — phase0/helpers.rs:646-676 over n x 121 bytes of SSZ Validator records
 * (activation_epoch <= epoch < exit_epoch); `out` must hold n entries, *out_n receives the count. */
B200_API int32_t b200_get_active_validator_indices(const uint8_t* validators_ssz, size_t n, uint64_t epoch, uint64_t* out,
                                                   size_t* out_n);
/* Both steps on a device-resident state (b200_state_upload_deneb): the registry never leaves HBM, only the shuffled
 * active-index list returns.  get_beacon_committee (phase0/helpers.rs:775-806) is then the slice
 * [len*index/count, len*(index+1)/count) of `out` (compute_committee, :459-483). */
B200_API int32_t b200_state_shuffled_active_indices(b200_state* handle, uint64_t epoch, const uint8_t seed[32], uint32_t rounds,
                                                    uint64_t* out, size_t* out_n);

/* Duties on a device-resident state (single-GPU handles; a NULL, not uploaded or sharded handle gets B200_ERR_BAD_ARG and
 * is left as it was): who proposes each slot and who sits on the sync committee, computed where the Validator records
 * are.  Preset constants follow the handle's preset: SLOTS_PER_EPOCH 32 / 8, SHUFFLE_ROUND_COUNT 90 / 10,
 * EPOCHS_PER_HISTORICAL_VECTOR 65536 / 64, SYNC_COMMITTEE_SIZE 512 / 32, EPOCHS_PER_SYNC_COMMITTEE_PERIOD 256 / 8
 * (mainnet / minimal); MAX_EFFECTIVE_BALANCE is 32 ETH in both.
 *  - b200_state_get_seed: get_seed (deneb/spec/mod.rs:2713-2748), SHA-256(domain_type || le64(epoch) ||
 *    randao_mixes[(epoch + EPHV - 2) mod EPHV]).  domain_type: the 4 bytes of DomainType::as_bytes (domains.rs:19-30), e.g.
 *    {1,0,0,0} BeaconAttester for b200_state_shuffled_active_indices' seed.
 *  - b200_state_proposer_indices: out[j] (SLOTS_PER_EPOCH entries) = get_beacon_proposer_index (:2822-2856) on this state
 *    with slot = epoch * SLOTS_PER_EPOCH + j: one call gives the epoch's whole proposer table (the active set and the
 *    effective balances do not change inside an epoch).  No active validator at `epoch`, or an epoch * SLOTS_PER_EPOCH
 *    that overflows u64 -> B200_ERR_BAD_ARG.
 *  - b200_state_next_sync_committee: get_next_sync_committee (:1973-2060) at epoch slot / SLOTS_PER_EPOCH + 1.
 *    out_indices (SIZE) are the members in selection order, repeats kept; out_committee (SIZE x 48 + 48 bytes) is the
 *    SSZ SyncCommittee: their public keys, gathered from the records in HBM, then eth_aggregate_public_keys of them
 *    (strict: every key validated as b200_eth_aggregate_public_keys does).  *out_code is that aggregation's code; on a
 *    non-zero code out_committee is zero-filled and out_indices still returned.  No active validator -> B200_ERR_BAD_ARG.
 *  - b200_state_sync_committee_updates: process_sync_committee_updates (:1263-1297).  When (slot / SLOTS_PER_EPOCH + 1) is
 *    a multiple of EPOCHS_PER_SYNC_COMMITTEE_PERIOD, current_sync_committee <- next_sync_committee <- the result of
 *    b200_state_next_sync_committee, written as b200_state_update_bytes writes (both roots follow) and *rotated = 1;
 *    otherwise nothing changes and *rotated = 0.  A non-zero aggregation code is returned in *out_code with *rotated = 0
 *    and the state unchanged.
 *  - b200_state_sync_committee_indices: the committee-key -> validator-index map of process_sync_aggregate (:463-473) for
 *    which = 0 (current_sync_committee) or 1 (next): out[j] (SIZE entries) is the LARGEST i with
 *    validators[i].pubkey == pubkeys[j] (the reference's HashMap keeps the last insert), UINT64_MAX when no validator
 *    holds the key (the reference panics).
 * The sampling loops, unbounded in the reference (each candidate is accepted with probability >= 1/256), stop after
 * 2^26 candidates with B200_ERR_LIMIT.  effective_balance * 255 is computed in wrapping u64, as a release build of the
 * reference does.  b200_last_kernel_ms: the device time of the call. */
B200_API int32_t b200_state_get_seed(b200_state* handle, uint64_t epoch, const uint8_t domain_type[4], uint8_t out[32]);
B200_API int32_t b200_state_proposer_indices(b200_state* handle, uint64_t epoch, uint64_t* out);
B200_API int32_t b200_state_next_sync_committee(b200_state* handle, uint64_t* out_indices, uint8_t* out_committee, int32_t* out_code);
B200_API int32_t b200_state_sync_committee_updates(b200_state* handle, int32_t* rotated, int32_t* out_code);
B200_API int32_t b200_state_sync_committee_indices(b200_state* handle, int32_t which, uint64_t* out);

/* Beacon committees on a device-resident state (single-GPU handles; a NULL, not uploaded or sharded handle gets
 * B200_ERR_BAD_ARG and is left as it was): who attests where, and who signed an attestation, computed where the Validator
 * records are.  These calls read the state and never write it.  Preset constants follow the handle's preset:
 * SLOTS_PER_EPOCH 32 / 8, TARGET_COMMITTEE_SIZE 128 / 4, MAX_COMMITTEES_PER_SLOT 64 / 4, SHUFFLE_ROUND_COUNT 90 / 10
 * (mainnet / minimal); MAX_VALIDATORS_PER_COMMITTEE 2048 and MIN_ATTESTATION_INCLUSION_DELAY 1 in both.
 * An epoch's committees are the slices [n k / C, n (k + 1) / C), k = 0 .. C - 1 with C = SLOTS_PER_EPOCH x cps, of its n
 * active validators shuffled by get_seed(epoch, BeaconAttester = {1,0,0,0}) (compute_committee, phase0/helpers.rs:459-483);
 * get_beacon_committee(slot, index) (:775-806) is committee k = (slot mod SLOTS_PER_EPOCH) x cps + index of slot's epoch,
 * and cps = get_committee_count_per_slot = max(1, min(MAX_COMMITTEES_PER_SLOT, n / SLOTS_PER_EPOCH / TARGET_COMMITTEE_SIZE))
 * (:741-773).  A committee is empty when n < C.
 * The handle caches the shuffled active lists of the last four epochs asked, in HBM.  An entry is used only while its
 * epoch's seed (recomputed from the host copy on every call) and the Validator records are what it was built from: any
 * write into the records (b200_state_update_elements or b200_state_update_bytes on them, an append to the validator list,
 * a relocation, or a b200_state_process_epoch that changes a record) makes every entry stale.  A cached epoch costs no
 * shuffle.  b200_last_kernel_ms: the device time of the call's kernels, without the copy of the results to the host.
 *  - b200_state_committee_count_per_slot: *out = cps of `epoch` (1 when no validator is active).
 *  - b200_state_beacon_committees: every committee of `epoch`: out_indices (room for n entries; the registry length always
 *    suffices) receives the shuffled active list, out_offsets (SLOTS_PER_EPOCH x cps + 1 <= 2049 entries) the committee
 *    bounds, *out_cps and *out_n = n.  No active validator at `epoch` -> B200_ERR_BAD_ARG.
 *  - b200_state_attester_duties: get_committee_assignment of the validator guide for each of the n validators named
 *    (validators == NULL with n == the registry length: every validator), as out[5 i .. 5 i + 4] = the AttestationDuty
 *    fields slot, committee_index, committee_length, committees_at_slot, validator_committee_index; a validator not
 *    active at `epoch` gets five UINT64_MAX.  B200_ERR_BAD_ARG before any work: an index >= the registry length, NULL with
 *    another n, n > 2^32 - 1, an epoch after the state's next epoch (the guide's `assert epoch <= next_epoch`), or an
 *    epoch x SLOTS_PER_EPOCH that overflows u64.
 *  - b200_state_attesting_indices: for n_att attestations, data (n_att x 128 bytes, SSZ AttestationData) and the SSZ
 *    Bitlist[MAX_VALIDATORS_PER_COMMITTEE] aggregation_bits of attestation a at bytes [bits_offsets[a], bits_offsets[a+1])
 *    of `bits`: the attesting_indices of get_indexed_attestation (:896-974), the committee members whose bit is set in
 *    ascending order, as out_indices[out_offsets[a] .. out_offsets[a+1]) (out_offsets: n_att + 1 entries; out_indices: room
 *    for the sum of the Bitlists' lengths in bits), and out_codes[a].  An attestation that fails gets its code and an empty
 *    slice.  The checks run in deneb process_attestation's order (deneb/block_processing.rs:53-100), after the Bitlist's
 *    decoding and before is_valid_indexed_attestation's emptiness test; the source checkpoint (participation flags) and
 *    the signature are not checked here:
 *      B200_ATTESTATION_MALFORMED_BITS        no delimiter bit (no bytes, or a zero last byte), or more than 2048 bits;
 *      B200_ATTESTATION_INVALID_TARGET_EPOCH  target.epoch neither the previous nor the current epoch (InvalidTargetEpoch);
 *      B200_ATTESTATION_INVALID_SLOT          target.epoch != compute_epoch_at_slot(slot) (InvalidSlot);
 *      B200_ATTESTATION_NO_DELAY              slot + MIN_ATTESTATION_INCLUSION_DELAY > state.slot, the sum wrapping in u64 as
 *                                             a release build computes it (NoDelay);
 *      B200_ATTESTATION_INVALID_INDEX         index >= get_committee_count_per_slot(target.epoch) (InvalidIndex);
 *      B200_ATTESTATION_BITFIELD              the Bitlist's length != the committee's length (Bitfield);
 *      B200_ATTESTATION_INDICES_EMPTY         no bit set (InvalidIndexedAttestation::AttestingIndicesEmpty).
 *    These codes are neither blst codes nor engine errors.  B200_ERR_BAD_ARG before any work: a NULL pointer (bits may be
 *    NULL when bits_offsets[n_att] == 0), bits_offsets not starting at 0 or decreasing, or n_att > 2^20.  n_att == 0
 *    succeeds and sets out_offsets[0] = 0 when out_offsets is not NULL. */
enum {
    B200_ATTESTATION_INVALID_TARGET_EPOCH = 0x201,
    B200_ATTESTATION_INVALID_SLOT = 0x202,
    B200_ATTESTATION_NO_DELAY = 0x203,
    B200_ATTESTATION_INVALID_INDEX = 0x204,
    B200_ATTESTATION_BITFIELD = 0x205,
    B200_ATTESTATION_INDICES_EMPTY = 0x206,
    B200_ATTESTATION_MALFORMED_BITS = 0x207
};
B200_API int32_t b200_state_committee_count_per_slot(b200_state* handle, uint64_t epoch, uint64_t* out);
B200_API int32_t b200_state_beacon_committees(b200_state* handle, uint64_t epoch, uint64_t* out_indices, uint32_t* out_offsets,
                                              uint64_t* out_cps, size_t* out_n);
B200_API int32_t b200_state_attester_duties(b200_state* handle, uint64_t epoch, const uint64_t* validators, size_t n,
                                            uint64_t* out /* n x 5 */);
B200_API int32_t b200_state_attesting_indices(b200_state* handle, size_t n_att, const uint8_t* data, const uint8_t* bits,
                                              const uint32_t* bits_offsets, uint64_t* out_indices, uint32_t* out_offsets,
                                              int32_t* out_codes);

/* Epoch processing on a device-resident state (single-GPU handles, as the duties above).  Sub-steps of deneb
 * process_epoch (deneb/spec/mod.rs:991-1002), in the reference's order: */
#define B200_EPOCH_JUSTIFICATION_AND_FINALIZATION  (1u << 0)
#define B200_EPOCH_INACTIVITY_UPDATES              (1u << 1)
#define B200_EPOCH_REWARDS_AND_PENALTIES           (1u << 2)
#define B200_EPOCH_REGISTRY_UPDATES                (1u << 3)
#define B200_EPOCH_SLASHINGS                       (1u << 4)
#define B200_EPOCH_ETH1_DATA_RESET                 (1u << 5)
#define B200_EPOCH_EFFECTIVE_BALANCE_UPDATES       (1u << 6)
#define B200_EPOCH_SLASHINGS_RESET                 (1u << 7)
#define B200_EPOCH_RANDAO_MIXES_RESET              (1u << 8)
#define B200_EPOCH_HISTORICAL_SUMMARIES_UPDATE     (1u << 9)
#define B200_EPOCH_PARTICIPATION_FLAG_UPDATES      (1u << 10)
#define B200_EPOCH_SYNC_COMMITTEE_UPDATES          (1u << 11)
#define B200_EPOCH_ALL                             0xfffu
/*  - b200_state_process_epoch applies the selected sub-steps, each with exactly the effect of the reference function of
 *    that name; one bit is one handler of spec-tests/runners/epoch_processing.rs, B200_EPOCH_ALL is process_epoch.  The
 *    mask only skips work.  Afterwards b200_state_root_incremental and b200_state_root both give the post-epoch root.
 *    A NULL, not uploaded or sharded handle, a NULL out_code, a mask bit above bit 11, or a state whose five big lists
 *    differ in length -> B200_ERR_BAD_ARG.  b200_last_kernel_ms: the device time of the call.
 *    Where the reference returns Err, the call refuses before writing anything (the state stays byte for byte as it was):
 *      - get_block_root out of range (:2582), asked only when a 2/3 target test passes -> B200_ERR_BAD_ARG;
 *      - get_total_balance's checked_add overflowing u64 (:2857-2868), for any sum a selected sub-step reads -> B200_ERR_LIMIT;
 *      - the checked_add of an ejected validator's withdrawable_epoch (:3106-3109) -> B200_ERR_LIMIT;
 *      - no validator active at the next epoch when the sync committees are due to rotate -> B200_ERR_BAD_ARG (the active
 *        set at the next epoch does not depend on this epoch's registry changes);
 *      - historical_summaries already at HISTORICAL_ROOTS_LIMIT when a summary is due -> B200_ERR_LIMIT.
 *    One failure comes after the writes: the sync-committee aggregation, which runs last.  Its code is returned in
 *    *out_code with B200_SUCCESS; every earlier sub-step stays applied and the committees stay as they were (what the
 *    reference's `&mut state` holds at its `?`).
 *    All other arithmetic wraps in u64, as a release build of the reference does: increase_balance,
 *    effective_balance * inactivity_score, the reward numerators, base_reward * weight, the slashings sum and its
 *    multiple, current_epoch + 1, balance + threshold, get_finality_delay.  decrease_balance saturates at zero.
 *    integer_sqrt of the total active balance is the exact floor.  Inside a validator: the inactivity score updates before
 *    the inactivity penalty reads it; the (reward, penalty) pairs apply in turn, flags 0, 1, 2, then inactivity, each
 *    penalty saturating; ejection and the slashing test read withdrawable_epoch after the registry step; effective
 *    balances read balances after the slashing penalty; the leak test and activation eligibility read
 *    finalized_checkpoint after justification whenever that step runs.
 *    The exit queue in closed form: ejections are assigned in index order; with E0 = max(the largest exit_epoch !=
 *    FAR_FUTURE_EPOCH, compute_activation_exit_epoch(current)), c0 = the validators whose exit_epoch is E0 and
 *    L = max(MIN_PER_EPOCH_CHURN_LIMIT, active / CHURN_LIMIT_QUOTIENT), the k-th ejection exits at E0 + (c0 + k) / L when
 *    c0 < L and E0 + 1 + k / L otherwise, as initiate_validator_exit (:3062-3111) called once per ejection gives.  The
 *    activation queue takes the first min(MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT, L) validators by
 *    (activation_eligibility_epoch, index), the eligibility epochs as the first loop left them.
 *    Preset constants: those of the duties, and SLOTS_PER_HISTORICAL_ROOT 8192 / 64, EPOCHS_PER_SLASHINGS_VECTOR
 *    8192 / 64, EPOCHS_PER_ETH1_VOTING_PERIOD 64 / 4, MIN_PER_EPOCH_CHURN_LIMIT 4 / 2,
 *    MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT 8 / 4, CHURN_LIMIT_QUOTIENT 65536 / 32 (mainnet / minimal); the rest are
 *    equal in both (EJECTION_BALANCE 16 ETH, INACTIVITY_PENALTY_QUOTIENT_BELLATRIX 2^24,
 *    PROPORTIONAL_SLASHING_MULTIPLIER_BELLATRIX 3, ...).
 *  - b200_state_serialized_len / b200_state_read_bytes read the serialization back in the coordinates
 *    b200_state_update_bytes takes, after any updates, reshapes or epochs: bytes inside the five big lists come from
 *    HBM, the rest from the host copy.  A range past the end -> B200_ERR_BAD_ARG. */
B200_API int32_t b200_state_process_epoch(b200_state* handle, uint32_t steps, int32_t* out_code);
/*  - b200_state_epoch_deltas: the reward and penalty deltas of process_rewards_and_penalties on the state as it is, without
 *    applying them: get_flag_index_deltas (altair/helpers.rs:265) for flags 0, 1, 2 and get_inactivity_penalty_deltas
 *    (bellatrix/helpers.rs:13), the four spec-test Deltas pairs of the `rewards` handler.  `out` is list-major, eight
 *    lists of n u64: source rewards, source penalties, target rewards, target penalties, head rewards, head penalties,
 *    inactivity rewards (always zero), inactivity penalties; list j is out[j n .. j n + n).  Each is the Vec<Gwei> the
 *    reference returns.  The call reads the state and never writes it: the serialization, both roots, the incremental
 *    root's pending work and the committee cache stay as they were.
 *    Semantics of the reference functions as they stand, with no other sub-step run first: previous = max(current - 1,
 *    0); the leak test reads the state's finalized_checkpoint (get_finality_delay wraps); the inactivity penalty reads
 *    the state's scores; only get_eligible_validator_indices receive deltas; there is no genesis shortcut.  At the
 *    current epoch 0, previous == current and get_unslashed_participating_indices reads current_epoch_participation.
 *    Arithmetic wraps in u64 as in b200_state_process_epoch (base_reward * weight * increments, effective_balance *
 *    inactivity_score).  Refusals before any write: a NULL, not uploaded or sharded handle, out == NULL with n > 0,
 *    n != the validator count, or five big lists of different lengths -> B200_ERR_BAD_ARG; get_total_balance's
 *    checked_add overflowing u64 for the total active balance or any flag's unslashed participating balance ->
 *    B200_ERR_LIMIT (the reference's Err, which its rewards handler unwraps).  n == 0 succeeds and launches nothing.
 *    Three launches (the totals pass, its fold, k_epoch_deltas).  b200_last_kernel_ms: the device time of the call's
 *    kernels, without the copy of the lists to the host. */
B200_API int32_t b200_state_epoch_deltas(b200_state* handle, uint64_t* out /* 8 x n */, size_t n);
B200_API int32_t b200_state_serialized_len(b200_state* handle, uint64_t* out_len);
B200_API int32_t b200_state_read_bytes(b200_state* handle, uint64_t ssz_offset, uint8_t* out, size_t n);

/* ---- multi-GPU: one process per GPU, the exchange step lives INSIDE the library (SURVEY.md §8b `b200_init(n_gpus)`,
 * §8e).  The reference is single-process (no counterpart, SURVEY.md §2a); a Rust host with one process per GPU calls:
 *   rank 0:   b200_comm_unique_id(id)  -> ships the 128 bytes to the other ranks by any means it likes (pipe, file, TCP)
 *   all ranks: b200_init(local_gpu); b200_comm_init(id, rank, world)       (collective; NCCL over NVLink / NVSwitch)
 * and then the *_sharded entry points below, which every rank must call with the same arguments.  world == 1 is
 * legal (no NCCL needed) and makes the sharded calls equivalent to the single-GPU ones. */
#define B200_COMM_ID_BYTES 128
B200_API int32_t b200_comm_unique_id(uint8_t out_id[B200_COMM_ID_BYTES]);
B200_API int32_t b200_comm_init(const uint8_t id[B200_COMM_ID_BYTES], int32_t rank, int32_t world);
B200_API int32_t b200_comm_info(int32_t* rank, int32_t* world, int32_t* nccl_version);
B200_API void b200_comm_destroy(void);
/* all-gather of `bytes_per_rank` host bytes per rank into recv[world * bytes_per_rank] (rank-major): for the host's own
 * small exchanges, e.g. verdict vectors when every rank verified a different batch (weak scaling). */
B200_API int32_t b200_comm_all_gather_bytes(const uint8_t* send, size_t bytes_per_rank, uint8_t* recv);
/* NCCL collectives issued by the library since start-up (bench.py reports it next to gpu_launches); loopback
 * all-gathers count too. */
B200_API uint64_t b200_collective_count(void);
/* Test use only: a communicator of `world` processes that may share ONE GPU, for running the sharded entry points at
 * world > 1 without NCCL.  Every all-gather goes through the file `path`, which all ranks map (MAP_SHARED) and which must
 * be new for each communicator: a 64-byte header (magic, world, slot size, arrival counter), then two generations of
 * world x `slot_bytes` slots.  Same preconditions as b200_comm_init (b200_init first; a second init with another rank or
 * world is refused; b200_comm_destroy resets).  A rank that finds a header with another world or slot size gets
 * B200_ERR_COMM.  An all-gather larger than `slot_bytes` per rank returns B200_ERR_COMM; one that waits longer than
 * `timeout_ms` for the other ranks returns B200_ERR_COMM (b200_last_error names the generation and how many ranks
 * arrived), and every later collective of the communicator then fails at once. */
B200_API int32_t b200_comm_init_loopback(const char* path, int32_t rank, int32_t world, uint64_t slot_bytes, uint32_t timeout_ms);

/* hash_tree_root(deneb::BeaconState) computed by all ranks of the communicator in ONE call (deneb/spec/mod.rs:3215,3288):
 * every rank passes the same serialization, uploads and hashes only its power-of-two-aligned slice of the five big
 * lists (parallel H2D over every GPU's own PCIe link) together with all small fields, the 5 x 32-byte slice roots are
 * exchanged with one ncclAllGather on the engine stream, and the finisher completes the tree on every rank: no host
 * round trip between the phases.  world must be a power of two.  Every rank gets the same `out`. */
B200_API int32_t b200_htr_beacon_state_deneb_sharded(const uint8_t* ssz, size_t len, int32_t preset, uint8_t out[32]);
/* The same, resident: every rank uploads its slices (and the small fields) once; b200_state_root on the returned handle is
 * then a collective of kernels + one ncclAllGather with no PCIe traffic (all ranks call it together; b200_state_free per
 * rank).  Root only — the update / incremental / shuffling entry points take single-GPU handles. */
B200_API int32_t b200_state_upload_deneb_sharded(const uint8_t* ssz, size_t len, int32_t preset, b200_state** out_handle);

/* b200_fast_aggregate_verify_batch over all ranks (BASELINE configs[4]: an epoch's attestation batch sharded over
 * 8 GPUs): every rank passes the same T tuples, verifies the contiguous block parallel.tuple_shard(T, world, rank)
 * names (only that block's keys cross PCIe), and one ncclAllGather of the int32 verdicts leaves all T codes in
 * `out_codes` on every rank — what process_block needs to pick the first failure. */
B200_API int32_t b200_fast_aggregate_verify_batch_sharded(const uint8_t* pks_flat, const uint32_t* pk_offsets,
                                                          const uint8_t* msgs32, const uint8_t* sigs, size_t n_tuples,
                                                          int32_t* out_codes);

/* ---- BLS12-381 signatures, min-pk (replaces the blst calls of crypto/bls.rs) ------------------------- */
/* Public keys are 48-byte and signatures 96-byte ZCash-compressed points (crypto/bls.rs:23-25,227-239,287-290);
 * the ciphersuite / DST is the one at crypto/bls.rs:22.  Results: 0 = Ok(()), 5 = Err(InvalidSignature),
 * 1,2,3,6 = Err(Error::BLST(..)) from key_validate / Signature::from_bytes, first offending input in order. */

/* verify_signature — crypto/bls.rs:64-77 */
B200_API int32_t b200_verify_signature(const uint8_t pk[48], const uint8_t* msg, size_t msg_len, const uint8_t sig[96]);
/* fast_aggregate_verify — crypto/bls.rs:114-132; `pks` is the array of K pointers the reference passes
 * (`&[&PublicKey]`, gathered from state.validators at phase0/helpers.rs:123-131) */
B200_API int32_t b200_fast_aggregate_verify(const uint8_t* const* pks, size_t k, const uint8_t* msg, size_t msg_len,
                                            const uint8_t sig[96]);
/* eth_fast_aggregate_verify — crypto/bls.rs:150-160 */
B200_API int32_t b200_eth_fast_aggregate_verify(const uint8_t* const* pks, size_t k, const uint8_t* msg, size_t msg_len,
                                                const uint8_t sig[96]);
/* aggregate_verify — crypto/bls.rs:95-112; n_pks x 48 contiguous bytes, n_msgs (pointer,length) messages */
B200_API int32_t b200_aggregate_verify(const uint8_t* pks_flat, size_t n_pks, const uint8_t* const* msgs,
                                       const size_t* msg_lens, size_t n_msgs, const uint8_t sig[96]);
/* aggregate_verify (crypto/bls.rs:95-112) over T tuples in one call.  Tuple t: keys [pk_offsets[t], pk_offsets[t+1]) of
 * pks_flat (48 B each), messages [msg_group[t], msg_group[t+1]) where message j is bytes [msg_offsets[j], msg_offsets[j+1])
 * of msgs, signature sigs[96 t ..].  out_codes[t] = what b200_aggregate_verify returns for that tuple alone: the first
 * invalid key's code, else the signature's decode code, else 5 (VERIFY_FAIL) for a tuple without keys or with as many
 * keys as messages not holding, for a signature outside G2 or a pairing product other than one; else 0.  Duplicate keys and
 * messages, empty messages and tuples without keys or messages are allowed.  All pairs of all tuples run on the
 * lane-parallel pairing kernels together, and each tuple's n + 1 Miller values are multiplied by a segmented warp-shuffle
 * product before its final exponentiation.
 * B200_ERR_BAD_ARG, nothing changed: a NULL pointer with a non-zero count; an offset array (T + 1 key offsets, T + 1
 * message groups, n_msgs + 1 byte offsets) that does not start at 0 or decreases; more than 0x3fffffff keys or messages;
 * T > 2^26.  n_tuples == 0 succeeds and changes nothing.  Each call sets b200_last_kernel_ms. */
B200_API int32_t b200_aggregate_verify_batch(const uint8_t* pks_flat, const uint32_t* pk_offsets, const uint8_t* msgs,
                                             const uint32_t* msg_offsets, const uint32_t* msg_group, const uint8_t* sigs,
                                             size_t n_tuples, int32_t* out_codes);
/* The same with keys named by validator index into the resident registry (b200_registry_load / _append / _load_state):
 * each key keeps the code it was validated with, so the codes equal the strict call's on the same key bytes.  Also
 * B200_ERR_BAD_ARG: no registry loaded, or an index >= the registry's size. */
B200_API int32_t b200_aggregate_verify_batch_indexed(const uint32_t* indices, const uint32_t* offsets, const uint8_t* msgs,
                                                     const uint32_t* msg_offsets, const uint32_t* msg_group,
                                                     const uint8_t* sigs, size_t n_tuples, int32_t* out_codes);
/* aggregate — crypto/bls.rs:79-93; n == 0 -> B200_EMPTY_AGGREGATE; out = compressed sum */
B200_API int32_t b200_aggregate(const uint8_t* sigs_flat, size_t n, uint8_t out[96]);
/* eth_aggregate_public_keys — crypto/bls.rs:135-148 */
B200_API int32_t b200_eth_aggregate_public_keys(const uint8_t* pks_flat, size_t n, uint8_t out[48]);
/* aggregate (crypto/bls.rs:79-93) over T groups: group t is signatures offsets[t] .. offsets[t+1]-1 of sigs_flat
 * (96 bytes each).  out_codes[t] and out96[96t..] are exactly what b200_aggregate returns for that group's bytes:
 * 0 and the compressed sum; 16 (EMPTY_AGGREGATE) for an empty group; otherwise the decode code of the first
 * signature that does not decode, else 3 (POINT_NOT_IN_GROUP).  out96 of a failed group is zero-filled.
 * b200_aggregate and b200_eth_aggregate_public_keys are the T = 1 case of these calls.
 * Arguments as on the verify batches: T + 1 non-decreasing offsets, T <= 2^26, offsets[T] <= 0x3fffffff items, and a
 * NULL pointer with a non-zero count -> B200_ERR_BAD_ARG; n_groups == 0 succeeds and changes nothing.  The return value
 * is B200_SUCCESS or an engine error (>= 0x100); each call sets b200_last_kernel_ms to the device time of its kernels. */
B200_API int32_t b200_aggregate_batch(const uint8_t* sigs_flat, const uint32_t* offsets, size_t n_groups,
                                      uint8_t* out96, int32_t* out_codes);
/* eth_aggregate_public_keys (crypto/bls.rs:135-148) over T groups of 48-byte keys; per group exactly
 * b200_eth_aggregate_public_keys. */
B200_API int32_t b200_eth_aggregate_public_keys_batch(const uint8_t* pks_flat, const uint32_t* offsets, size_t n_groups,
                                                      uint8_t* out48, int32_t* out_codes);
/* The same over keys named by registry (validator) index: no key crosses PCIe or is validated again.  Each key keeps
 * the code it was given at load / append, so out_codes[t] equals b200_eth_aggregate_public_keys on the same key bytes,
 * invalid keys included.  An index >= reg_n -> B200_ERR_BAD_ARG for the call. */
B200_API int32_t b200_registry_aggregate_public_keys(const uint32_t* indices, const uint32_t* offsets, size_t n_groups,
                                                     uint8_t* out48, int32_t* out_codes);

/* The throughput path: T independent fast_aggregate_verify tuples in one call (the batch of attestation checks
 * `process_block` issues one by one at deneb/block_processing.rs:104-108).  Tuple t uses public keys
 * pk_offsets[t] .. pk_offsets[t+1] of `pks_flat`, the 32-byte signing root msgs32[32t..] and sigs[96t..];
 * out_codes[t] is exactly what b200_fast_aggregate_verify would return for that tuple (strict mode: every key is
 * decompressed and validated in every call, as crypto/bls.rs:119-123 does). */
B200_API int32_t b200_fast_aggregate_verify_batch(const uint8_t* pks_flat, const uint32_t* pk_offsets, const uint8_t* msgs32,
                                                  const uint8_t* sigs, size_t n_tuples, int32_t* out_codes);
/* Optimistic WHOLE-BATCH check by random linear combination (north_star: "Miller loops fused across the batch, partial Gt
 * products reduced with warp shuffles"): *all_ok = 1 iff every tuple of the batch would return 0 above — decided with
 * T Miller loops and ONE final exponentiation instead of 2T and T:  prod_t e(r_t agg_t, H(msg_t)) * e(-g1, sum_t r_t sig_t) == 1
 * for 64-bit scalars r_t = the first 8 bytes, little-endian, of SHA-256(seed || le64(t)) (forced non-zero).  Valid batches
 * are always accepted; a batch with an invalid tuple is accepted with probability <= 2^-64 over the seed (seed32 == NULL:
 * the library draws one from the OS; tests pass a fixed seed).  A caller-supplied seed must be unpredictable to whoever
 * produced the signatures: anyone who knows the seed can build a batch in which every tuple is invalid and the defects
 * cancel, and that batch is accepted.  This is the normal-case path of process_block (every signature of a block is
 * expected to verify); on *all_ok == 0 the caller asks b200_fast_aggregate_verify_batch, which remains the only source of
 * per-tuple codes. */
B200_API int32_t b200_fast_aggregate_verify_batch_all(const uint8_t* pks_flat, const uint32_t* pk_offsets, const uint8_t* msgs32,
                                                      const uint8_t* sigs, size_t n_tuples, const uint8_t* seed32, int32_t* all_ok);
/* Registry mode: validate the (append-only, immutable-pubkey) validator registry once, keep the affine keys in
 * HBM, then verify tuples that name their signers by validator index.  Same per-tuple codes as the strict path. */
B200_API int32_t b200_registry_load(const uint8_t* pks_flat, size_t n);
/* The registry follows the growing validator list (deposits, phase0/block_processing.rs:394-401).  Registry indices are
 * validator indices, and keys are never validated twice: each key keeps the code and point it was given, so the key codes
 * and every verdict are exactly those of b200_registry_load over the concatenated key list, invalid keys included (a
 * tuple that names an invalid key gets its code).  The `..._batch_mixed` extra-key tail follows reg_n: after an append,
 * index i >= reg_n names extra key i - reg_n with the new reg_n.
 *  - b200_registry_append: validate n more keys; they become indices reg_n .. reg_n + n - 1.  Keys already in the
 *    registry are neither copied from the host nor validated again.  n == 0 succeeds and changes nothing.
 *  - b200_registry_load_state: replace the registry with the public keys of every validator of a single-GPU resident
 *    state (b200_state_upload_deneb), read from its Validator records in HBM: no key crosses PCIe.
 *  - b200_registry_sync_state: append the state's validators reg_n .. n_validators - 1, i.e. those that
 *    b200_state_append_elements added since the registry last matched the state.  Keys 0 .. reg_n - 1 are taken to be
 *    the state's first reg_n public keys (pubkeys are immutable, phase0/validator.rs:10-13) and are not compared again;
 *    a sync with nothing new succeeds and changes nothing.
 * The registry holds its own copy of the keys: freeing the state afterwards leaves it intact.  Each call sets
 * b200_last_kernel_ms to the device time of its kernels.  B200_ERR_BAD_ARG, with the registry left as it was (size, keys,
 * codes): a NULL pointer with n > 0; reg_n + n > 0x7fffffff (the bound of b200_registry_load); a state handle that is
 * NULL, not uploaded or sharded; a sync against a state with fewer validators than the registry. */
B200_API int32_t b200_registry_append(const uint8_t* pks_flat, size_t n);
B200_API int32_t b200_registry_load_state(b200_state* handle);
B200_API int32_t b200_registry_sync_state(b200_state* handle);
B200_API int32_t b200_registry_key_codes(int32_t* out_codes, size_t n);
B200_API int32_t b200_fast_aggregate_verify_batch_indexed(const uint32_t* indices, const uint32_t* offsets,
                                                          const uint8_t* msgs32, const uint8_t* sigs, size_t n_tuples,
                                                          int32_t* out_codes);
/* Registry mode for a whole block's signature set in ONE call: `extra_pks` are the n_extra (<= 65 536) 48-byte keys that
 * are not in the registry because they arrive in the block itself (deposits `phase0/block_processing.rs:387-392`, bls-to-
 * execution changes `capella/block_processing.rs:43-56`); they are decompressed + validated by this call exactly like
 * the strict path does, and an index i >= n_registry names extra key i - n_registry.  Codes as the strict path's. */
B200_API int32_t b200_fast_aggregate_verify_batch_mixed(const uint8_t* extra_pks, size_t n_extra, const uint32_t* indices,
                                                        const uint32_t* offsets, const uint8_t* msgs32, const uint8_t* sigs,
                                                        size_t n_tuples, int32_t* out_codes);
/* RLC whole-batch check over registry indices, and over all ranks of the communicator: every rank passes the same batch
 * and the same (non-NULL) seed, verifies its block, and ONE ncclAllGather moves the per-rank Gt partial (576 B) and the
 * rank's bad flag (16 B); every rank then finishes the same final exponentiation and returns the same boolean.  Rank k scales
 * its tuples with r_t of their global index t.  The sharded call requires the caller's seed, so the caller must draw it
 * unpredictably (for instance from the OS after the signatures are fixed) and share it among the ranks: a seed known to
 * whoever produced the signatures lets them build an all-invalid batch that is accepted. */
B200_API int32_t b200_fast_aggregate_verify_batch_indexed_all(const uint32_t* indices, const uint32_t* offsets,
                                                              const uint8_t* msgs32, const uint8_t* sigs, size_t n_tuples,
                                                              const uint8_t* seed32, int32_t* all_ok);
B200_API int32_t b200_fast_aggregate_verify_batch_all_sharded(const uint8_t* pks_flat, const uint32_t* pk_offsets,
                                                              const uint8_t* msgs32, const uint8_t* sigs, size_t n_tuples,
                                                              const uint8_t seed32[32], int32_t* all_ok);
/* Device time (ms) of the dominant kernel (per-key validation) of the last BLS call. */
B200_API float b200_last_dominant_kernel_ms(void);
/* Measured integer-pipe peak on this device, 1e9 ops/s: kind 0 IMAD.WIDE.U32 (Montgomery multiply-add), 1 IMAD.U32,
 * 2 LOP3/SHF/IADD3 mix (SHA-256 round ops).  Roofline denominators for bench.py. */
B200_API int32_t b200_measure_int_peak(int32_t kind, double* gops);
/* Scheduling knobs of the BLS batch pipeline, settable at run time (the same names, upper-cased with a B200_ prefix, are
 * read from the environment when the pipeline is first used).  They change launch shapes only, never a result:
 *   "bls_small_cta" (0 = by batch size | 32 | 64 | 128: CTA size of the signature / message kernels), "vm_team16_max",
 *   "vm_cta" (32 | 64 | 128).
 * An environment value goes through the same rule as the value passed here: a negative B200_VM_TEAM16_MAX means 0, and
 * B200_BLS_SMALL_CTA is the only name of that knob.
 * Unknown knob -> B200_ERR_BAD_ARG; so are the names of the key-range, split-copy and first-wave knobs earlier versions took. */
B200_API int32_t b200_tune(const char* knob, int64_t value);
/* Replaces the scheduled Miller-loop / final-exponentiation programs of one team size (8 or 16 lanes) of the lane-parallel
 * pairing kernels with another SCHEDULE of the same formulas: `blob` is what `tools/gen_pairing_vm.py <team> ... --blob F`
 * writes after executing the schedule numerically against the direct evaluation.  Opcodes and slot indices are validated;
 * a malformed blob -> B200_ERR_BAD_ARG and the programs in use stay.  Schedule tuning only: results never depend on it. */
B200_API int32_t b200_vm_load_programs(const uint32_t* blob, size_t n_words);
/* On-device self-test of the field arithmetic over `n` pseudo-random triples; *mismatches must come back 0. */
B200_API int32_t b200_fp_selftest(uint32_t n, uint32_t seed, uint32_t* mismatches);
/* On-device self-test of single field operations, for comparison with big integers: `op` (bls_kernels.cuh, FP_EVAL_* /
 * FP2_EVAL_* / FPD_EVAL_*) is applied to `n` operand pairs.  a, b: n x 24 raw little-endian 32-bit limbs (Fp in the first
 * 12, Fp2 as c0 then c1); out: n x 25 (the result's limbs, then a carry / borrow / square / on-curve / sign flag).  An
 * FpD value (the FP64 field of the per-key kernel's square root) is words 0..15 of a slot: 8 little-endian IEEE binary64
 * limbs, limb k an integer multiple of 2^(48k), so that a record read as float64[n, 12] holds them in columns 0..7.
 * Test use only. */
B200_API int32_t b200_fp_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out);
/* On-device self-test of single curve stages, for comparison with a big-integer oracle: `op` (bls_kernels.cuh,
 * CURVE_G1L_* on the per-key kernel's lazily reduced field, CURVE_G1_IN_SUBGROUP_ISO on X alone as the role-split per-key
 * kernel checks it, CURVE_G2_* in the signature / hash unit) is applied to `n`
 * operand pairs.  a, b, out: n x 73 words: X, Y, Z as 24-word slots of raw little-endian 32-bit Montgomery limbs (Fp in
 * the first 12 words of a slot, Fp2 as c0 then c1), then a flag word (in: the affine infinity flag; out: the subgroup
 * verdict, or the infinity flag of an affine result).  Test use only. */
B200_API int32_t b200_curve_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out);
/* On-device self-test of the pairing, for comparison with a big-integer oracle: `op` (bls_kernels.cuh, PAIRING_EVAL_*) runs
 * in the unit whose production kernel runs it: Fp6 / Fp12 operations, Miller steps and loop, the final exponentiation
 * (one thread per record), the lane-parallel Miller and final programs at teams of 8 or 16 lanes, the RLC folds, and the
 * segmented product of the aggregate_verify batches (a: the values; b: the word T, then T + 1 segment offsets).
 * a, b, out: n x 145 words: twelve 12-word Fp slots in Fp12 memory order of raw little-endian 32-bit Montgomery limbs,
 * then a flag word (in: the infinity flag of a point; out: the final exponentiation's verdict, or the infinity flag of the
 * G2 fold's affine sum).  n = 0 .. 2^24.  Test use only. */
B200_API int32_t b200_pairing_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out);

#ifdef __cplusplus
}
#endif
#endif /* B200_CONSENSUS_H */
