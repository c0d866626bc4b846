"""CPU oracle for committee shuffling — TEST INFRASTRUCTURE ONLY (tests/, smoke, bench's cpu_baseline may import it).

Two independent restatements of the reference's two formulations, pinned against each other:
  * `compute_shuffled_index`   — the per-index swap-or-not map, ethereum-consensus/src/phase0/helpers.rs:249-283
  * `compute_shuffled_indices` — the whole-list walk,            ethereum-consensus/src/phase0/helpers.rs:287-360
    (the reference's own runner asserts both equal the spec vector `mapping`, spec-tests/runners/shuffling.rs:35-45)
plus a numpy-vectorised form of the first for 2**20-size checks, and `get_active_validator_indices` (:646-676).
Parity pin: the `consensus-spec-tests` shuffling vectors are absent offline, and the reference tree holds no shuffling
KAT; the pin is (a) the two formulations above agreeing on every size 0..300 and on random sizes, (b) the hand-checkable
n = 1, 2 cases, (c) tests/test_spec_vectors.py consuming `shuffling/core/*/mapping.yaml` when the tarball is present.
"""
from __future__ import annotations

import hashlib
from typing import List, Sequence

import numpy as np


def _h(b: bytes) -> bytes:
    return hashlib.sha256(b).digest()


def compute_shuffled_index(index: int, index_count: int, seed: bytes, rounds: int = 90) -> int:
    if index >= index_count:
        raise ValueError("InvalidShufflingIndex")
    for r in range(rounds):
        pivot = int.from_bytes(_h(seed + bytes([r]))[:8], "little") % index_count
        flip = (pivot + index_count - index) % index_count
        position = max(index, flip)
        source = _h(seed + bytes([r]) + (position // 256).to_bytes(4, "little"))
        byte = source[(position % 256) // 8]
        if (byte >> (position % 8)) & 1:
            index = flip
    return index


def compute_shuffled_indices(indices: Sequence[int], seed: bytes, rounds: int = 90) -> List[int]:
    """The list walk of phase0/helpers.rs:287-360: rounds in reverse, two mirrored sweeps around the pivot."""
    out = list(indices)
    n = len(out)
    if n == 0:
        return out
    for r in range(rounds - 1, -1, -1):
        pivot = int.from_bytes(_h(seed + bytes([r]))[:8], "little") % n

        def src(pos_block: int) -> bytes:
            return _h(seed + bytes([r]) + (pos_block & 0xffffffff).to_bytes(4, "little"))

        source = src(pivot >> 8)
        byte_source = source[(pivot & 0xff) >> 3]
        mirror = (pivot + 1) >> 1
        for i in range(mirror):
            j = pivot - i
            if j & 0xff == 0xff:
                source = src(j >> 8)
            if j & 0x07 == 0x07:
                byte_source = source[(j & 0xff) >> 3]
            if (byte_source >> (j & 0x07)) & 1:
                out[i], out[j] = out[j], out[i]
        end = n - 1
        source = src(end >> 8)
        byte_source = source[(end & 0xff) >> 3]
        mirror = (pivot + n + 1) >> 1
        for k, i in enumerate(range(pivot + 1, mirror)):
            j = end - k
            if j & 0xff == 0xff:
                source = src(j >> 8)
            if j & 0x07 == 0x07:
                byte_source = source[(j & 0xff) >> 3]
            if (byte_source >> (j & 0x07)) & 1:
                out[i], out[j] = out[j], out[i]
    return out


def shuffled_indices_numpy(indices, seed: bytes, rounds: int = 90) -> np.ndarray:
    """Vectorised per-index map: out[i] = indices[compute_shuffled_index(i)] (seconds at n = 2**20)."""
    idx_in = np.arange(indices, dtype=np.uint64) if isinstance(indices, (int, np.integer)) else np.asarray(indices, dtype=np.uint64)
    n = len(idx_in)
    if n == 0:
        return idx_in.copy()
    cur = np.arange(n, dtype=np.int64)
    nblk = (n + 255) // 256
    for r in range(rounds):
        pivot = int.from_bytes(_h(seed + bytes([r]))[:8], "little") % n
        flip = (pivot + n - cur) % n
        pos = np.maximum(cur, flip)
        table = np.frombuffer(b"".join(_h(seed + bytes([r]) + b.to_bytes(4, "little")) for b in range(nblk)), dtype=np.uint8)
        byte = table[(pos >> 8) * 32 + ((pos & 255) >> 3)]
        bit = (byte >> (pos & 7).astype(np.uint8)) & 1
        cur = np.where(bit == 1, flip, cur)
    return idx_in[cur]


def get_active_validator_indices(validators_ssz: bytes, epoch: int) -> List[int]:
    """phase0/helpers.rs:646-676 over 121-byte SSZ Validator records (activation_epoch at 97, exit_epoch at 105)."""
    b = bytes(validators_ssz)
    out = []
    for i in range(len(b) // 121):
        r = b[121 * i: 121 * (i + 1)]
        act, ext = int.from_bytes(r[97:105], "little"), int.from_bytes(r[105:113], "little")
        if act <= epoch < ext:
            out.append(i)
    return out
