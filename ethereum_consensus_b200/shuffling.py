"""Host-side mirror of the reference's committee-shuffling helpers, computed on the device (SURVEY.md §8f-3).

`compute_shuffled_indices`      — ethereum-consensus/src/phase0/helpers.rs:287-360
`compute_shuffled_index`        — :249-283 (one position of the same permutation)
`get_active_validator_indices`  — :646-676
`compute_committee`             — :459-483   (slice of the shuffled list)
No CPU fallback: every function launches kernels through the C ABI (include/b200_consensus.h).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

SHUFFLE_ROUND_COUNT = {"mainnet": 90, "minimal": 10}   # phase0/presets/{mainnet,minimal}.rs


def compute_shuffled_indices(indices, seed: bytes, rounds: int = 90) -> np.ndarray:
    """out[i] = indices[compute_shuffled_index(i, len(indices), seed)]; `indices` may be an int n for the identity list."""
    if len(seed) != 32:
        raise ValueError("seed must be 32 bytes")
    if isinstance(indices, (int, np.integer)):
        n, idx = int(indices), None
    else:
        idx = np.ascontiguousarray(indices, dtype=np.uint64)
        n = len(idx)
    out = np.empty(max(n, 1), dtype=np.uint64)
    sd = np.frombuffer(bytes(seed), dtype=np.uint8)
    _lib.check(_lib.lib().b200_compute_shuffled_indices(_lib.ptr(idx) if idx is not None else 0, n, _lib.ptr(sd), rounds, _lib.ptr(out)),
               "compute_shuffled_indices")
    return out[:n]


def compute_shuffled_index(index: int, index_count: int, seed: bytes, rounds: int = 90) -> int:
    if index >= index_count:
        raise ValueError(f"InvalidShufflingIndex {{ index: {index}, total: {index_count} }}")   # phase0/helpers.rs:255-257
    return int(compute_shuffled_indices(index_count, seed, rounds)[index])


def get_active_validator_indices(validators_ssz, epoch: int) -> np.ndarray:
    """`validators_ssz`: N x 121 bytes of SSZ Validator records (state.validators serialized)."""
    buf = np.frombuffer(validators_ssz, dtype=np.uint8) if not isinstance(validators_ssz, np.ndarray) else validators_ssz.reshape(-1).view(np.uint8)
    if buf.size % 121:
        raise ValueError("validators must be N x 121 bytes")
    n = buf.size // 121
    out = np.empty(max(n, 1), dtype=np.uint64)
    cnt = C.c_size_t(0)
    _lib.check(_lib.lib().b200_get_active_validator_indices(_lib.ptr(buf), n, epoch, _lib.ptr(out), C.byref(cnt)), "get_active_validator_indices")
    return out[:cnt.value]


def state_shuffled_active_indices(dev_state, epoch: int, seed: bytes, rounds: int = 90) -> np.ndarray:
    """Both steps on a `ssz.DeviceBeaconState`: the registry stays in HBM, only the shuffled index list returns."""
    sd = np.frombuffer(bytes(seed), dtype=np.uint8)
    n = dev_state.n_validators
    out = np.empty(max(n, 1), dtype=np.uint64)
    cnt = C.c_size_t(0)
    _lib.check(_lib.lib().b200_state_shuffled_active_indices(dev_state._h, epoch, _lib.ptr(sd), rounds, _lib.ptr(out), C.byref(cnt)),
               "state_shuffled_active_indices")
    return out[:cnt.value]


def compute_committee(shuffled: np.ndarray, index: int, count: int) -> np.ndarray:
    """phase0/helpers.rs:459-483 with the `shuffling` feature: slice `index` of `count` of the shuffled list."""
    n = len(shuffled)
    return shuffled[n * index // count: n * (index + 1) // count]
