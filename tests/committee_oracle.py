"""CPU oracle for beacon committees and attesting indices — test infrastructure for the committee calls of
ethereum_consensus_b200.duties, over a `state.SynthState` (builds on oracle/duties_oracle.py's get_seed and active set).

Restated from the behaviour of ethereum-consensus (phase0/helpers.rs, deneb/block_processing.rs):
  * `committee_count_per_slot`  — get_committee_count_per_slot (:741-773)
  * `beacon_committee`          — get_beacon_committee (:775-806) via compute_committee (:459-483), in both of the
                                  reference's formulations: "index" runs compute_shuffled_index for every member (the
                                  build without the `shuffling` feature), "list" slices the whole-list shuffle
  * `committee_assignment`      — the validator guide's get_committee_assignment, by brute force over the epoch's
                                  committees (row order of beacon-api-client's AttestationDuty, types.rs:416-432)
  * `attesting_indices`         — get_attesting_indices / get_indexed_attestation (:896-974) with the checks of deneb
                                  process_attestation (block_processing.rs:53-100) in order, then the emptiness test of
                                  is_valid_indexed_attestation; a Bitlist that does not decode fails first.
"""
from __future__ import annotations

import numpy as np

from oracle import duties_oracle as do
from oracle import shuffle_oracle as sh

COMMITTEE = {
    "mainnet": dict(TARGET_COMMITTEE_SIZE=128, MAX_COMMITTEES_PER_SLOT=64, MAX_VALIDATORS_PER_COMMITTEE=2048,
                    MIN_ATTESTATION_INCLUSION_DELAY=1),
    "minimal": dict(TARGET_COMMITTEE_SIZE=4, MAX_COMMITTEES_PER_SLOT=4, MAX_VALIDATORS_PER_COMMITTEE=2048,
                    MIN_ATTESTATION_INCLUSION_DELAY=1),
}
DOMAIN_BEACON_ATTESTER = bytes([1, 0, 0, 0])
U64 = (1 << 64) - 1
NOT_ACTIVE = U64

# codes (include/b200_consensus.h B200_ATTESTATION_*)
OK = 0
INVALID_TARGET_EPOCH = 0x201
INVALID_SLOT = 0x202
NO_DELAY = 0x203
INVALID_INDEX = 0x204
BITFIELD = 0x205
INDICES_EMPTY = 0x206
MALFORMED_BITS = 0x207
CODES = {OK: "ok", INVALID_TARGET_EPOCH: "invalid_target_epoch", INVALID_SLOT: "invalid_slot", NO_DELAY: "no_delay",
         INVALID_INDEX: "invalid_index", BITFIELD: "bitfield", INDICES_EMPTY: "indices_empty", MALFORMED_BITS: "malformed_bits"}


def spe(st) -> int:
    return do.PRESET[st.preset]["SLOTS_PER_EPOCH"]


def committee_count_per_slot(st, epoch: int) -> int:
    P = COMMITTEE[st.preset]
    n = len(do.active_indices(st, epoch))
    return max(1, min(P["MAX_COMMITTEES_PER_SLOT"], n // spe(st) // P["TARGET_COMMITTEE_SIZE"]))


def compute_committee(indices: np.ndarray, seed: bytes, index: int, count: int, rounds: int, formulation: str,
                      shuffled: np.ndarray | None = None) -> list:
    n = len(indices)
    start, end = n * index // count, n * (index + 1) // count
    if formulation == "index":
        return [int(indices[sh.compute_shuffled_index(i, n, seed, rounds)]) for i in range(start, end)]
    if formulation == "list":
        if shuffled is None:
            shuffled = sh.shuffled_indices_numpy(indices, seed, rounds) if n else np.zeros(0, np.uint64)
        return [int(x) for x in shuffled[start:end]]
    raise ValueError(formulation)


def beacon_committee(st, slot: int, index: int, formulation: str = "list") -> list:
    epoch = slot // spe(st)
    cps = committee_count_per_slot(st, epoch)
    active = do.active_indices(st, epoch)
    seed = do.get_seed(st, epoch, DOMAIN_BEACON_ATTESTER)
    rounds = do.PRESET[st.preset]["SHUFFLE_ROUND_COUNT"]
    return compute_committee(active, seed, (slot % spe(st)) * cps + index, cps * spe(st), rounds, formulation)


def beacon_committees(st, epoch: int, formulation: str = "list") -> list:
    """Every committee of `epoch`, k = (slot % SLOTS_PER_EPOCH) * cps + index order (one shuffle for "list")."""
    cps = committee_count_per_slot(st, epoch)
    active = do.active_indices(st, epoch)
    seed = do.get_seed(st, epoch, DOMAIN_BEACON_ATTESTER)
    rounds = do.PRESET[st.preset]["SHUFFLE_ROUND_COUNT"]
    count = cps * spe(st)
    shuffled = None
    if formulation == "list" and len(active):
        shuffled = sh.shuffled_indices_numpy(active, seed, rounds)
    return [compute_committee(active, seed, k, count, rounds, formulation, shuffled) for k in range(count)]


def committee_assignment(st, epoch: int, validators=None, committees=None) -> dict:
    """{validator: (slot, committee_index, committee_length, committees_at_slot, validator_committee_index)} for every
    validator that sits on a committee of `epoch` (all of the epoch's committees walked in slot, index order)."""
    committees = committees if committees is not None else beacon_committees(st, epoch)
    cps = len(committees) // spe(st)
    want = None if validators is None else set(int(v) for v in validators)
    out = {}
    for k, members in enumerate(committees):
        slot = epoch * spe(st) + k // cps
        for j, v in enumerate(members):
            if (want is None or v in want) and v not in out:
                out[v] = (slot, k % cps, len(members), cps, j)
    return out


def duty_rows(st, epoch: int, validators) -> np.ndarray:
    """uint64[n, 5]: committee_assignment rows for `validators`, NOT_ACTIVE rows for those on no committee."""
    a = committee_assignment(st, epoch, validators)
    return np.array([a.get(int(v), (NOT_ACTIVE,) * 5) for v in validators], dtype=np.uint64).reshape(-1, 5)


def bitlist_len(b: bytes, max_bits: int = 2048):
    """Length in bits of an SSZ Bitlist[max_bits], None when it does not decode."""
    if len(b) == 0 or b[-1] == 0:
        return None
    n = 8 * (len(b) - 1) + b[-1].bit_length() - 1
    return n if n <= max_bits else None


def attestation_data(slot: int, index: int, target_epoch: int, source_epoch: int = 0, root: bytes = bytes(32)) -> bytes:
    """SSZ AttestationData: slot, index, beacon_block_root, source (epoch, root), target (epoch, root)."""
    le = lambda v: int(v).to_bytes(8, "little")  # noqa: E731
    return le(slot) + le(index) + root + le(source_epoch) + bytes(32) + le(target_epoch) + root


def bitlist(bits) -> bytes:
    """SSZ Bitlist of a bool sequence: the bits little-endian in each byte, then the delimiter bit."""
    n = len(bits)
    out = bytearray(n // 8 + 1)
    for i, b in enumerate(bits):
        if b:
            out[i // 8] |= 1 << (i % 8)
    out[n // 8] |= 1 << (n % 8)
    return bytes(out)


def attesting_indices(st, data: bytes, bits: bytes, formulation: str = "list", committees=None):
    """-> (code, sorted attesting indices, [] unless code == OK).  `committees`: {epoch: beacon_committees(st, epoch)}
    cache (optional)."""
    P = COMMITTEE[st.preset]
    slot = int.from_bytes(data[0:8], "little")
    index = int.from_bytes(data[8:16], "little")
    target = int.from_bytes(data[88:96], "little")
    n_bits = bitlist_len(bits, P["MAX_VALIDATORS_PER_COMMITTEE"])
    if n_bits is None:
        return MALFORMED_BITS, []
    state_slot = do.slot(st)
    cur = state_slot // spe(st)
    prev = cur - 1 if cur else 0
    if target not in (prev, cur):
        return INVALID_TARGET_EPOCH, []
    if slot // spe(st) != target:
        return INVALID_SLOT, []
    if (slot + P["MIN_ATTESTATION_INCLUSION_DELAY"]) & U64 > state_slot:
        return NO_DELAY, []
    cps = committee_count_per_slot(st, target)
    if index >= cps:
        return INVALID_INDEX, []
    if committees is not None:
        if target not in committees:
            committees[target] = beacon_committees(st, target, formulation)
        committee = committees[target][(slot % spe(st)) * cps + index]
    else:
        committee = beacon_committee(st, slot, index, formulation)
    if n_bits != len(committee):
        return BITFIELD, []
    got = sorted({v for i, v in enumerate(committee) if bits[i // 8] >> (i % 8) & 1})
    if not got:
        return INDICES_EMPTY, []
    return OK, got
