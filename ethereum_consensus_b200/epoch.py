"""Epoch processing on a device-resident deneb `BeaconState` (`ssz.DeviceBeaconState`): `process_epoch`
(ethereum-consensus/src/deneb/spec/mod.rs:965-1003) in one call, its sub-steps selectable by name, and the reward and
penalty deltas of `process_rewards_and_penalties` read without applying them (`deltas`).

The per-validator sub-steps run as CUDA kernels over the records, balances, inactivity scores and participation lists in
HBM (csrc/epoch.cu); the small fields go through the state's update and reshape paths.  Rules the reference leaves to its
build (wrapping u64 arithmetic, refusals before any write) are stated in include/b200_consensus.h.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

# sub-step bits, named as the spec-test handlers of epoch_processing (include/b200_consensus.h: B200_EPOCH_*)
STEPS = ("justification_and_finalization", "inactivity_updates", "rewards_and_penalties", "registry_updates", "slashings",
         "eth1_data_reset", "effective_balance_updates", "slashings_reset", "randao_mixes_reset",
         "historical_summaries_update", "participation_flag_updates", "sync_committee_updates")
STEP = {name: 1 << k for k, name in enumerate(STEPS)}
ALL = (1 << len(STEPS)) - 1
# the (reward, penalty) pairs of `deltas`, in the order process_rewards_and_penalties applies them (the spec-test
# `rewards` handler's source, target, head and inactivity-penalty Deltas)
DELTAS = ("source", "target", "head", "inactivity_penalty")


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


def deltas(dev_state) -> np.ndarray:
    """get_flag_index_deltas for flags 0, 1, 2 and get_inactivity_penalty_deltas on the resident state as it is, as a
    uint64 array of shape (4, 2, n): [k, 0] the rewards and [k, 1] the penalties of pair DELTAS[k].  Reads the state and
    never writes it; a refusal raises _lib.EngineError carrying the library's code."""
    n = dev_state.n_validators
    out = np.zeros((len(DELTAS), 2, n), dtype=np.uint64)
    _lib.check(_lib.lib().b200_state_epoch_deltas(dev_state._h, out.ctypes.data if n else None, n), "state_epoch_deltas")
    return out
