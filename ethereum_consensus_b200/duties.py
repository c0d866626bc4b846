"""Proposer and sync-committee duties on a device-resident deneb `BeaconState` (`ssz.DeviceBeaconState`).

`get_seed`                        — ethereum-consensus/src/deneb/spec/mod.rs:2713-2748
`proposer_indices`                — get_beacon_proposer_index (:2822-2856) for every slot of an epoch
`next_sync_committee`             — get_next_sync_committee (:1973-2060)
`process_sync_committee_updates`  — :1263-1297, on the resident state
`sync_committee_indices`          — the committee-key -> validator-index map of process_sync_aggregate (:463-473)
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
