"""Mirror of the reference's signing helpers, hashing on the device.

`compute_signing_root` / `verify_signed_data`  — ethereum-consensus/src/signing.rs:14-41
`compute_domain` / `compute_fork_data_root`    — ethereum-consensus/src/phase0/helpers.rs:506-529
`get_domain` (previous / current fork version)  — ethereum-consensus/src/phase0/helpers.rs:190-222
`compute_epoch_at_slot`                        — ethereum-consensus/src/phase0/helpers.rs (slot / SLOTS_PER_EPOCH)
`DomainType`                                   — ethereum-consensus/src/domains.rs:1-30
"""
from __future__ import annotations

import enum
from dataclasses import dataclass

from . import crypto, ssz


class DomainType(enum.IntEnum):
    BeaconProposer = 0
    BeaconAttester = 1
    Randao = 2
    Deposit = 3
    VoluntaryExit = 4
    SelectionProof = 5
    AggregateAndProof = 6
    SyncCommittee = 7
    SyncCommitteeSelectionProof = 8
    ContributionAndProof = 9
    BlsToExecutionChange = 10

    def as_bytes(self) -> bytes:
        return int(self).to_bytes(4, "little")


def compute_fork_data_root(current_version: bytes, genesis_validators_root: bytes) -> bytes:
    """hash_tree_root(ForkData{current_version, genesis_validators_root}) — two leaves."""
    return ssz.merkleize(bytes(current_version).ljust(32, b"\x00") + bytes(genesis_validators_root), 2)


def compute_domain(domain_type: DomainType, fork_version: bytes = b"\x00" * 4, genesis_validators_root: bytes = b"\x00" * 32) -> bytes:
    return DomainType(domain_type).as_bytes() + compute_fork_data_root(fork_version, genesis_validators_root)[:28]


@dataclass(frozen=True)
class Fork:
    """`Fork{previous_version, current_version, epoch}` (phase0/beacon_state.rs:15-22): what `get_domain` reads of the state."""
    previous_version: bytes
    current_version: bytes
    epoch: int


def compute_epoch_at_slot(slot: int, slots_per_epoch: int = 32) -> int:
    return slot // slots_per_epoch


def get_domain(fork: Fork, genesis_validators_root: bytes, domain_type: DomainType, epoch: int = None, current_epoch: int = None) -> bytes:
    """phase0/helpers.rs:190-222: `epoch` defaults to the state's current epoch; a message from before the fork boundary
    (`epoch < state.fork.epoch`) is checked under the PREVIOUS fork version, everything else under the current one."""
    if epoch is None:
        if current_epoch is None:
            raise ValueError("get_domain: need `epoch` or the state's `current_epoch`")
        epoch = current_epoch
    version = fork.previous_version if epoch < fork.epoch else fork.current_version
    return compute_domain(domain_type, version, genesis_validators_root)


def compute_signing_root(object_root: bytes, domain: bytes) -> bytes:
    """hash_tree_root(SigningData{object_root, domain}); `object_root` is the signed object's hash_tree_root."""
    return ssz.merkleize(bytes(object_root) + bytes(domain), 2)


def verify_signed_data(object_root: bytes, signature: bytes, public_key: bytes, domain: bytes) -> None:
    crypto.verify_signature(public_key, compute_signing_root(object_root, domain), signature)
