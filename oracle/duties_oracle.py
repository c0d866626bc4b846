"""CPU oracle for proposer and sync-committee duties — TEST INFRASTRUCTURE ONLY (tests/ and tools/ import it).

Restates, over a `state.SynthState`, the five selection functions of ethereum-consensus/src/deneb/spec/mod.rs:
  * `get_seed`                         — :2713-2748
  * `proposer_indices`                 — get_beacon_proposer_index (:2822-2856) for each slot of an epoch
  * `next_sync_committee_indices`      — get_next_sync_committee_indices (:1973-2013)
  * `next_sync_committee`              — get_next_sync_committee (:2014-2060), the aggregate by `bls_oracle`
  * `process_sync_committee_updates`   — :1263-1297 (returns the rotated state; the input is not changed)
  * `sync_committee_indices`           — the HashMap lookup of process_sync_aggregate (:463-473)
The two sampling loops (compute_proposer_index :2460-2518, and the committee loop) are each written in both of the
reference's formulations, which tests pin against each other:
  * "index": compute_shuffled_index(i mod n) per candidate (shuffle_oracle.compute_shuffled_index);
  * "list":  the `shuffling` feature's whole shuffled active list indexed by i mod n (:2495-2505), here
             shuffle_oracle.shuffled_indices_numpy.
Rules the reference leaves implicit: effective_balance * 255 wraps in u64 (a release build); the loops, unbounded in the
reference, stop at `cap` candidates (the library's 2^26) and raise SamplingCapReached; an empty active set raises
NoActiveValidator (the reference's CollectionCannotBeEmpty, or its `i % 0` panic in the committee loop).
"""
from __future__ import annotations

import hashlib
from functools import lru_cache

import numpy as np

from oracle import shuffle_oracle as sh

PRESET = {
    "mainnet": dict(SLOTS_PER_EPOCH=32, SHUFFLE_ROUND_COUNT=90, EPOCHS_PER_HISTORICAL_VECTOR=65536, SYNC_COMMITTEE_SIZE=512,
                    EPOCHS_PER_SYNC_COMMITTEE_PERIOD=256),
    "minimal": dict(SLOTS_PER_EPOCH=8, SHUFFLE_ROUND_COUNT=10, EPOCHS_PER_HISTORICAL_VECTOR=64, SYNC_COMMITTEE_SIZE=32,
                    EPOCHS_PER_SYNC_COMMITTEE_PERIOD=8),
}
MIN_SEED_LOOKAHEAD = 1
MAX_EFFECTIVE_BALANCE = 32 * 10**9
MAX_RANDOM_BYTE = 255
DOMAIN_BEACON_PROPOSER = bytes([0, 0, 0, 0])
DOMAIN_SYNC_COMMITTEE = bytes([7, 0, 0, 0])
CAP = 1 << 26
U64 = (1 << 64) - 1
MISSING = U64


class NoActiveValidator(ValueError):
    pass


class SamplingCapReached(RuntimeError):
    pass


def _h(b: bytes) -> bytes:
    return hashlib.sha256(b).digest()


def slot(st) -> int:
    return int.from_bytes(st.fixed["slot"], "little")


def get_seed(st, epoch: int, domain: bytes) -> bytes:
    P = PRESET[st.preset]
    ephv = P["EPOCHS_PER_HISTORICAL_VECTOR"]
    mix_epoch = (epoch + (ephv - MIN_SEED_LOOKAHEAD) - 1) & U64
    return _h(bytes(domain) + (epoch & U64).to_bytes(8, "little") + st.randao_mixes[mix_epoch % ephv].tobytes())


def active_indices(st, epoch: int) -> np.ndarray:
    v = st.validators
    return np.nonzero((v["activation_epoch"] <= np.uint64(epoch)) & (np.uint64(epoch) < v["exit_epoch"]))[0].astype(np.uint64)


def accepts(effective_balance: int, random_byte: int, wrap: bool = True) -> bool:
    lhs = effective_balance * MAX_RANDOM_BYTE
    return ((lhs & U64) if wrap else lhs) >= MAX_EFFECTIVE_BALANCE * random_byte


class _Sampler:
    """Candidates i = 0, 1, ... of one seed over one active list, in either formulation."""

    def __init__(self, st, active: np.ndarray, seed: bytes, formulation: str, wrap: bool = True):
        if len(active) == 0:
            raise NoActiveValidator()
        self.st, self.active, self.seed, self.wrap = st, active, seed, wrap
        self.rounds = PRESET[st.preset]["SHUFFLE_ROUND_COUNT"]
        self.n = len(active)
        if formulation == "list":
            self.shuffled = sh.shuffled_indices_numpy(active, seed, self.rounds)
            self.candidate = lambda i: int(self.shuffled[i % self.n])
        elif formulation == "index":
            f = lru_cache(maxsize=None)(lambda k: int(active[sh.compute_shuffled_index(k, self.n, seed, self.rounds)]))
            self.candidate = lambda i: f(i % self.n)
        else:
            raise ValueError(formulation)
        self.random_block = lru_cache(maxsize=64)(lambda w: _h(seed + w.to_bytes(8, "little")))

    def __iter__(self):
        """(i, candidate, accepted) for i = 0 .. CAP - 1."""
        eff = self.st.validators["effective_balance"]
        for i in range(CAP):
            c = self.candidate(i)
            yield i, c, accepts(int(eff[c]), self.random_block(i // 32)[i % 32], self.wrap)


def compute_proposer_index(st, active: np.ndarray, seed: bytes, formulation: str = "index", wrap: bool = True) -> int:
    for _, c, ok in _Sampler(st, active, seed, formulation, wrap):
        if ok:
            return c
    raise SamplingCapReached()


def proposer_indices(st, epoch: int, formulation: str = "index", wrap: bool = True) -> list:
    """get_beacon_proposer_index with state.slot = epoch * SLOTS_PER_EPOCH + j, for j in 0 .. SLOTS_PER_EPOCH - 1."""
    spe = PRESET[st.preset]["SLOTS_PER_EPOCH"]
    if epoch * spe > U64:
        raise OverflowError("epoch * SLOTS_PER_EPOCH overflows u64")
    base = get_seed(st, epoch, DOMAIN_BEACON_PROPOSER)
    active = active_indices(st, epoch)
    return [compute_proposer_index(st, active, _h(base + (epoch * spe + j).to_bytes(8, "little")), formulation, wrap)
            for j in range(spe)]


def next_sync_committee_indices(st, formulation: str = "index", wrap: bool = True) -> list:
    P = PRESET[st.preset]
    epoch = slot(st) // P["SLOTS_PER_EPOCH"] + 1
    seed = get_seed(st, epoch, DOMAIN_SYNC_COMMITTEE)
    out = []
    for _, c, ok in _Sampler(st, active_indices(st, epoch), seed, formulation, wrap):
        if ok:
            out.append(c)
            if len(out) == P["SYNC_COMMITTEE_SIZE"]:
                return out
    raise SamplingCapReached()


def candidates_drawn(st, formulation: str = "index") -> int:
    """How many candidates the committee loop draws (the regime a case is built for)."""
    P = PRESET[st.preset]
    epoch = slot(st) // P["SLOTS_PER_EPOCH"] + 1
    have = 0
    for i, _, ok in _Sampler(st, active_indices(st, epoch), get_seed(st, epoch, DOMAIN_SYNC_COMMITTEE), formulation):
        have += ok
        if have == P["SYNC_COMMITTEE_SIZE"]:
            return i + 1
    raise SamplingCapReached()


def next_sync_committee(st, aggregate=None, formulation: str = "index"):
    """-> (indices, SyncCommittee bytes, code); `aggregate(keys) -> (code, 48 bytes | None)` is eth_aggregate_public_keys
    (default: bls_oracle's); on a non-zero code the bytes are zero."""
    from oracle import bls_oracle as bo
    aggregate = aggregate or bo.eth_aggregate_public_keys
    idx = next_sync_committee_indices(st, formulation)
    keys = [st.validators["public_key"][i].tobytes() for i in idx]
    code, agg = aggregate(keys)
    if code:
        return idx, bytes(48 * (len(keys) + 1)), code
    return idx, b"".join(keys) + agg, 0


def process_sync_committee_updates(st, aggregate=None):
    """-> (rotated, code, new state): a rotated copy at a period boundary, `st` itself otherwise or on a failed aggregate."""
    import copy
    P = PRESET[st.preset]
    if (slot(st) // P["SLOTS_PER_EPOCH"] + 1) % P["EPOCHS_PER_SYNC_COMMITTEE_PERIOD"]:
        return False, 0, st
    _, committee, code = next_sync_committee(st, aggregate)
    if code:
        return False, code, st
    out = copy.copy(st)
    out.current_sync_committee, out.next_sync_committee = st.next_sync_committee, committee
    return True, 0, out


def sync_committee_indices(st, which: str = "current") -> list:
    """For each committee key: the last validator index holding it (HashMap built in registry order), MISSING if none."""
    size = PRESET[st.preset]["SYNC_COMMITTEE_SIZE"]
    blob = st.current_sync_committee if which == "current" else st.next_sync_committee
    last = {}
    for i, k in enumerate(st.validators["public_key"]):
        last[k.tobytes()] = i
    return [last.get(blob[48 * j:48 * j + 48], MISSING) for j in range(size)]
