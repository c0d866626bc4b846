"""Proposer and sync-committee duties on a device-resident deneb `BeaconState` (`ssz.DeviceBeaconState`).

`get_seed`                        — ethereum-consensus/src/deneb/spec/mod.rs:2713-2748
`proposer_indices`                — get_beacon_proposer_index (:2822-2856) for every slot of an epoch
`next_sync_committee`             — get_next_sync_committee (:1973-2060)
`process_sync_committee_updates`  — :1263-1297, on the resident state
`sync_committee_indices`          — the committee-key -> validator-index map of process_sync_aggregate (:463-473)
`committee_count_per_slot`        — get_committee_count_per_slot (phase0/helpers.rs:741-773)
`beacon_committees`               — every get_beacon_committee (:775-806) of an epoch, from one cached shuffle
`beacon_committee`                — one of them
`attester_duties`                 — the validator guide's get_committee_assignment, as beacon-API AttestationDuty rows
`attesting_indices`               — get_indexed_attestation(...).attesting_indices (:896-974) of attestation batches, with
                                    deneb process_attestation's checks (deneb/block_processing.rs:53-100)
No CPU fallback: every function launches kernels through the C ABI (include/b200_consensus.h); the Validator records
never leave HBM.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

# DomainType::as_bytes (domains.rs:19-30)
DOMAIN_BEACON_PROPOSER = bytes([0, 0, 0, 0])
DOMAIN_BEACON_ATTESTER = bytes([1, 0, 0, 0])
DOMAIN_SYNC_COMMITTEE = bytes([7, 0, 0, 0])
SLOTS_PER_EPOCH = {"mainnet": 32, "minimal": 8}
SYNC_COMMITTEE_SIZE = {"mainnet": 512, "minimal": 32}
MISSING = (1 << 64) - 1   # sync_committee_indices' code for a key no validator holds
NOT_ACTIVE = (1 << 64) - 1   # every field of an attester_duties row of a validator not active at the epoch
# beacon-api-client AttestationDuty (types.rs:416-432), without the public key
ATTESTATION_DUTY = np.dtype([("slot", "<u8"), ("committee_index", "<u8"), ("committee_length", "<u8"),
                             ("committees_at_slot", "<u8"), ("validator_committee_index", "<u8")])
# attesting_indices' codes (include/b200_consensus.h), named after InvalidAttestation (error.rs:119-134)
ATTESTATION_INVALID_TARGET_EPOCH = 0x201
ATTESTATION_INVALID_SLOT = 0x202
ATTESTATION_NO_DELAY = 0x203
ATTESTATION_INVALID_INDEX = 0x204
ATTESTATION_BITFIELD = 0x205
ATTESTATION_INDICES_EMPTY = 0x206   # InvalidIndexedAttestation::AttestingIndicesEmpty
ATTESTATION_MALFORMED_BITS = 0x207  # the Bitlist does not decode


def get_seed(dev_state, epoch: int, domain: bytes) -> bytes:
    if len(domain) != 4:
        raise ValueError("domain must be the 4 bytes of a DomainType")
    out = (C.c_uint8 * 32)()
    _lib.check(_lib.lib().b200_state_get_seed(dev_state._h, epoch, bytes(domain), out), "state_get_seed")
    return bytes(out)


def proposer_indices(dev_state, epoch: int) -> np.ndarray:
    """uint64[SLOTS_PER_EPOCH]: the proposer of each slot of `epoch`."""
    out = np.zeros(SLOTS_PER_EPOCH[dev_state.preset], dtype=np.uint64)
    _lib.check(_lib.lib().b200_state_proposer_indices(dev_state._h, epoch, _lib.ptr(out)), "state_proposer_indices")
    return out


def next_sync_committee(dev_state):
    """-> (uint64[SIZE] member indices, SyncCommittee SSZ bytes (SIZE x 48 keys, then the aggregate), aggregation code);
    on a non-zero code the bytes are zero."""
    size = SYNC_COMMITTEE_SIZE[dev_state.preset]
    idx = np.zeros(size, dtype=np.uint64)
    committee = np.zeros(size * 48 + 48, dtype=np.uint8)
    code = C.c_int32(0)
    _lib.check(_lib.lib().b200_state_next_sync_committee(dev_state._h, _lib.ptr(idx), _lib.ptr(committee), C.byref(code)),
               "state_next_sync_committee")
    return idx, committee.tobytes(), code.value


def process_sync_committee_updates(dev_state) -> bool:
    """Rotate the sync committees when the next epoch starts a period; True when they rotated.  A committee whose
    aggregation fails raises crypto.BLSTError (the reference's `?`) and leaves the state unchanged."""
    rotated, code = C.c_int32(0), C.c_int32(0)
    _lib.check(_lib.lib().b200_state_sync_committee_updates(dev_state._h, C.byref(rotated), C.byref(code)),
               "state_sync_committee_updates")
    if code.value:
        from .crypto import BLSTError
        raise BLSTError(code.value)
    return bool(rotated.value)


def sync_committee_indices(dev_state, which: str = "current", missing_ok: bool = False) -> np.ndarray:
    """uint64[SIZE]: for each key of the current or next sync committee, the largest validator index holding it.  A key
    no validator holds raises KeyError (the reference's `expect`), or is MISSING with `missing_ok`."""
    w = {"current": 0, "next": 1}[which]
    out = np.zeros(SYNC_COMMITTEE_SIZE[dev_state.preset], dtype=np.uint64)
    _lib.check(_lib.lib().b200_state_sync_committee_indices(dev_state._h, w, _lib.ptr(out)), "state_sync_committee_indices")
    if not missing_ok and (out == MISSING).any():
        raise KeyError(f"validator public_key should exist: {which} sync committee position {int(np.argmax(out == MISSING))}")
    return out


def committee_count_per_slot(dev_state, epoch: int) -> int:
    """get_committee_count_per_slot (phase0/helpers.rs:741-773): max(1, min(MAX_COMMITTEES_PER_SLOT,
    active / SLOTS_PER_EPOCH / TARGET_COMMITTEE_SIZE))."""
    out = C.c_uint64(0)
    _lib.check(_lib.lib().b200_state_committee_count_per_slot(dev_state._h, epoch, C.byref(out)), "state_committee_count_per_slot")
    return out.value


def beacon_committees(dev_state, epoch: int):
    """-> (uint64[n_active] shuffled active indices, uint32[SLOTS_PER_EPOCH * cps + 1] offsets, cps): committee
    k = (slot % SLOTS_PER_EPOCH) * cps + index is indices[offsets[k]:offsets[k + 1]], i.e. get_beacon_committee
    (phase0/helpers.rs:775-806) through compute_committee (:459-483).  No active validator raises B200Error."""
    idx = np.zeros(max(1, dev_state.n_validators), dtype=np.uint64)
    offsets = np.zeros(SLOTS_PER_EPOCH[dev_state.preset] * 64 + 1, dtype=np.uint32)
    cps, n = C.c_uint64(0), C.c_size_t(0)
    _lib.check(_lib.lib().b200_state_beacon_committees(dev_state._h, epoch, _lib.ptr(idx), _lib.ptr(offsets), C.byref(cps),
                                                       C.byref(n)), "state_beacon_committees")
    return idx[:n.value].copy(), offsets[:SLOTS_PER_EPOCH[dev_state.preset] * cps.value + 1].copy(), cps.value


def beacon_committee(dev_state, slot: int, index: int) -> np.ndarray:
    """get_beacon_committee(state, slot, index) (phase0/helpers.rs:775-806): uint64 validator indices in committee order."""
    spe = SLOTS_PER_EPOCH[dev_state.preset]
    idx, offsets, cps = beacon_committees(dev_state, slot // spe)
    if index >= cps:
        raise IndexError(f"committee index {index} >= committees per slot {cps}")
    k = (slot % spe) * cps + index
    return idx[offsets[k]:offsets[k + 1]]


def attester_duties(dev_state, epoch: int, validators=None) -> np.ndarray:
    """get_committee_assignment for each validator (all when None) as an ATTESTATION_DUTY structured array: slot,
    committee_index, committee_length, committees_at_slot, validator_committee_index (beacon-api-client
    types.rs:416-432).  A validator not active at `epoch` gets NOT_ACTIVE in every field.  `epoch` is at most the state's
    next epoch."""
    if validators is None:
        n, vp = dev_state.n_validators, None
    else:
        v = np.ascontiguousarray(validators, dtype=np.uint64)
        n, vp = v.size, _lib.ptr(v)
    out = np.zeros(n, dtype=ATTESTATION_DUTY)
    _lib.check(_lib.lib().b200_state_attester_duties(dev_state._h, epoch, vp, n, _lib.ptr(out) if n else None),
               "state_attester_duties")
    return out


def attesting_indices(dev_state, attestations):
    """`attestations`: (AttestationData SSZ (128 bytes), aggregation_bits SSZ Bitlist) pairs ->
    (list of uint64 arrays, int32 codes): get_indexed_attestation(...).attesting_indices (phase0/helpers.rs:896-974),
    sorted ascending, and each attestation's code (0, or an ATTESTATION_* code with an empty array) from deneb
    process_attestation's checks (deneb/block_processing.rs:53-100).  The arrays go to SignatureSet.add_indexed_attestation
    or Registry.verify_batch as they are."""
    n = len(attestations)
    data = np.zeros(max(1, n) * 128, dtype=np.uint8)
    offsets = np.zeros(n + 1, dtype=np.uint32)
    for a, (d, bits) in enumerate(attestations):
        if len(d) != 128:
            raise ValueError(f"attestation {a}: AttestationData is 128 bytes, got {len(d)}")
        data[128 * a:128 * a + 128] = np.frombuffer(bytes(d), np.uint8)
        offsets[a + 1] = offsets[a] + len(bits)
    bits = np.frombuffer(b"".join(bytes(b) for _, b in attestations) or bytes(1), np.uint8)
    out = np.zeros(max(1, 8 * int(offsets[-1])), dtype=np.uint64)
    out_off = np.zeros(n + 1, dtype=np.uint32)
    codes = np.zeros(max(1, n), dtype=np.int32)
    _lib.check(_lib.lib().b200_state_attesting_indices(dev_state._h, n, _lib.ptr(data), _lib.ptr(bits), _lib.ptr(offsets),
                                                       _lib.ptr(out), _lib.ptr(out_off), _lib.ptr(codes)), "state_attesting_indices")
    return [out[out_off[a]:out_off[a + 1]].copy() for a in range(n)], codes[:n]
