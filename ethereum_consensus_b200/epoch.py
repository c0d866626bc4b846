"""Epoch processing on a device-resident deneb `BeaconState` (`ssz.DeviceBeaconState`): `process_epoch`
(ethereum-consensus/src/deneb/spec/mod.rs:965-1003) in one call, its sub-steps selectable by name.

The per-validator sub-steps run as CUDA kernels over the records, balances, inactivity scores and participation lists in
HBM (csrc/epoch.cu); the small fields go through the state's update and reshape paths.  Rules the reference leaves to its
build (wrapping u64 arithmetic, refusals before any write) are stated in include/b200_consensus.h.
"""
from __future__ import annotations

import ctypes as C

from . import _lib

# sub-step bits, named as the spec-test handlers of epoch_processing (include/b200_consensus.h: B200_EPOCH_*)
STEPS = ("justification_and_finalization", "inactivity_updates", "rewards_and_penalties", "registry_updates", "slashings",
         "eth1_data_reset", "effective_balance_updates", "slashings_reset", "randao_mixes_reset",
         "historical_summaries_update", "participation_flag_updates", "sync_committee_updates")
STEP = {name: 1 << k for k, name in enumerate(STEPS)}
ALL = (1 << len(STEPS)) - 1


def mask(steps) -> int:
    """A B200_EPOCH_* mask from an int, one step name, or an iterable of names."""
    if isinstance(steps, int):
        return steps
    if isinstance(steps, str):
        return STEP[steps]
    m = 0
    for s in steps:
        m |= STEP[s]
    return m


def process_epoch(dev_state, steps=ALL) -> None:
    """Apply the selected sub-steps of process_epoch to the resident state.  A refused call (_lib.EngineError carrying the
    library's code) leaves the state unchanged; a failed sync-committee aggregation raises
    crypto.BLSTError after every earlier sub-step has been applied, as the reference's `?` leaves its `&mut state`."""
    code = C.c_int32(0)
    _lib.check(_lib.lib().b200_state_process_epoch(dev_state._h, mask(steps), C.byref(code)), "state_process_epoch")
    if code.value:
        from .crypto import BLSTError
        raise BLSTError(code.value)
