"""Seeded deneb states and attestations for the beacon-committee calls of ethereum_consensus_b200.duties, each built for
one regime of the committee arithmetic or one outcome of the attestation checks.  Shared by test_committee_cases.py (CPU:
the oracle's two formulations, the assignment inverse, each case's regime and codes) and test_committees_gpu.py (the device
against the oracle)."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from ethereum_consensus_b200 import state as S
from oracle import duties_oracle as do
from tests import committee_oracle as co

ETH = 10**9
FAR = S.FAR_FUTURE_EPOCH
EPOCH = 1000   # the states' current epoch


@dataclass
class Case:
    name: str
    st: S.SynthState
    cps: dict                                  # epoch -> the committees per slot the case is built for
    attestations: list = field(default_factory=list)   # (AttestationData bytes, Bitlist bytes, intended code)
    small: bool = True                         # the per-member ("index") formulation is cheap enough to run


def step(preset: str) -> int:
    """Active validators per committee-per-slot step: SLOTS_PER_EPOCH x TARGET_COMMITTEE_SIZE."""
    return do.PRESET[preset]["SLOTS_PER_EPOCH"] * co.COMMITTEE[preset]["TARGET_COMMITTEE_SIZE"]


def state(n_active: int, preset: str = "mainnet", seed: int = 1, edges: bool = True, slot_in_epoch: int | None = None):
    """n_active validators active at EPOCH - 1, EPOCH and EPOCH + 1; with `edges`, eight more at the epoch's edges:
    activating exactly at EPOCH (active from EPOCH), at EPOCH + 1 (not yet), exiting exactly at EPOCH (no longer active)
    and at EPOCH + 1 (still active at EPOCH), two of each, interleaved with the others; four of them are active at each of
    the three epochs, so n_active counts them.  Slot: mid-epoch by default."""
    spe = do.PRESET[preset]["SLOTS_PER_EPOCH"]
    n = n_active + (4 if edges else 0)
    st = S.synth_state(n, preset, seed=seed, n_eth1_votes=1, n_historical_summaries=1)
    v = st.validators
    v["activation_epoch"] = 0
    v["exit_epoch"] = FAR
    v["effective_balance"] = 32 * ETH
    if edges:
        rng = np.random.default_rng(seed)
        at = rng.choice(n, 8, replace=False)
        v["activation_epoch"][at[0:2]] = EPOCH       # active at EPOCH and EPOCH + 1, not at EPOCH - 1
        v["activation_epoch"][at[2:4]] = EPOCH + 1   # active at EPOCH + 1 only
        v["exit_epoch"][at[4:6]] = EPOCH             # active at EPOCH - 1 only
        v["exit_epoch"][at[6:8]] = EPOCH + 1         # active at EPOCH - 1 and EPOCH
    st.fixed["slot"] = int(EPOCH * spe + (spe // 2 if slot_in_epoch is None else slot_in_epoch)).to_bytes(8, "little")
    return st


def expected_cps(preset: str, n_active: int) -> int:
    P = co.COMMITTEE[preset]
    return max(1, min(P["MAX_COMMITTEES_PER_SLOT"], n_active // do.PRESET[preset]["SLOTS_PER_EPOCH"] // P["TARGET_COMMITTEE_SIZE"]))


def _attestations(st, rng, full: bool) -> list:
    """One attestation of every code against `st`, and with `full` a spread of valid ones over both epochs' committees:
    all bits, one bit, random bits (bitlist lengths are the committee lengths: 0, 8m, 8m +- 1 come with the states)."""
    spe = co.spe(st)
    slot = do.slot(st)
    cur = slot // spe
    prev = cur - 1
    out = []
    committees = {e: co.beacon_committees(st, e) for e in (prev, cur)}
    cps = {e: len(committees[e]) // spe for e in (prev, cur)}

    def att(e, k, bits, code):
        s = e * spe + k // cps[e]
        out.append((co.attestation_data(s, k % cps[e], e), co.bitlist(bits), code))

    nonempty = {e: [k for k, c in enumerate(committees[e]) if c and e * spe + k // cps[e] + 1 <= slot] for e in (prev, cur)}
    ks = {e: [k for k in range(len(committees[e])) if e * spe + k // cps[e] + 1 <= slot] for e in (prev, cur)}
    e_any = prev if nonempty[prev] else cur
    k0 = nonempty[e_any][0]
    L = len(committees[e_any][k0])
    # valid
    att(e_any, k0, [True] * L, co.OK)
    if full:
        for e in (prev, cur):
            pick = list(rng.choice(nonempty[e], min(6, len(nonempty[e])), replace=False)) if nonempty[e] else []
            for j, k in enumerate(pick):
                n = len(committees[e][k])
                bits = [True] * n if j == 0 else ([i == n - 1 for i in range(n)] if j == 1 else list(rng.random(n) < 0.5))
                if not any(bits):
                    bits[int(rng.integers(0, n))] = True
                att(e, k, bits, co.OK)
    # no bit set
    att(e_any, k0, [False] * L, co.INDICES_EMPTY)
    # an empty committee: a zero-length Bitlist (the delimiter byte alone) has no attesting validator
    empty = [(e, k) for e in (prev, cur) for k in ks[e] if not committees[e][k]]
    if empty:
        att(*empty[0], [], co.INDICES_EMPTY)
        att(*empty[0], [True], co.BITFIELD)
    # wrong length, both ways
    att(e_any, k0, [True] * (L + 1), co.BITFIELD)
    if L:
        att(e_any, k0, [True] * (L - 1), co.BITFIELD)
    # target neither previous nor current
    for e in (cur + 1, prev - 1):
        out.append((co.attestation_data(e * spe, 0, e), co.bitlist([True] * L), co.INVALID_TARGET_EPOCH))
    # target epoch != the slot's epoch
    out.append((co.attestation_data(prev * spe + 1, 0, cur), co.bitlist([True] * L), co.INVALID_SLOT))
    # not timely: the state's own slot
    out.append((co.attestation_data(slot, 0, cur), co.bitlist([True] * L), co.NO_DELAY))
    # index == cps
    out.append((co.attestation_data(e_any * spe, cps[e_any], e_any), co.bitlist([True] * L), co.INVALID_INDEX))
    # malformed Bitlists: no bytes, a zero last byte, 2049 bits
    d = co.attestation_data(e_any * spe + k0 // cps[e_any], k0 % cps[e_any], e_any)
    out.append((d, b"", co.MALFORMED_BITS))
    out.append((d, co.bitlist([True] * L) + b"\x00", co.MALFORMED_BITS))
    out.append((d, co.bitlist([True] * 2049), co.MALFORMED_BITS))
    # malformed before any other check: a bad target with no delimiter is MALFORMED_BITS
    out.append((co.attestation_data(0, 0, 0), b"\x00", co.MALFORMED_BITS))
    return out


def cases() -> list:
    out = []
    for preset in ("mainnet", "minimal"):
        S_ = step(preset)
        spe = do.PRESET[preset]["SLOTS_PER_EPOCH"]
        max_cps = co.COMMITTEE[preset]["MAX_COMMITTEES_PER_SLOT"]
        counts = {
            "below_C": spe - 3,                           # n_active < C = SLOTS_PER_EPOCH: empty committees
            "one": 1,
            "step1_minus": S_ - 1, "step1": S_, "step1_plus": S_ + 1,
            "step2_minus": 2 * S_ - 1, "step2": 2 * S_, "step2_plus": 2 * S_ + 1,
            "clamp_minus": max_cps * S_ - 1, "clamp": max_cps * S_, "clamp_plus": (max_cps + 1) * S_ + 1,
        }
        for j, (name, n) in enumerate(counts.items()):
            st = state(n, preset, seed=100 + 20 * (preset == "minimal") + j, edges=n >= 4)
            want = {e: expected_cps(preset, n) for e in (EPOCH - 1, EPOCH, EPOCH + 1)}
            rng = np.random.default_rng(j)
            out.append(Case(f"{preset}_{name}", st, want, _attestations(st, rng, full=n < 20000), small=n <= 5000))
        # exact cps steps at EPOCH (no edge validators): n_active = k x step - 1, k x step
        for k in (1, 2):
            for d in (-1, 0):
                n = k * S_ + d
                st = state(n, preset, seed=300 + k * 2 + d, edges=False)
                out.append(Case(f"{preset}_exact_{k}step{d:+d}", st, {e: expected_cps(preset, n) for e in (EPOCH - 1, EPOCH, EPOCH + 1)},
                                _attestations(st, np.random.default_rng(k), full=True), small=n <= 5000))
    # committee lengths 7, 8, 9, 15, 16, 17 (the Bitlist's delimiter in the last bit of a byte, alone in a new byte, ...):
    # minimal, cps = 4, C = 32 committees of exactly n / 32 members
    for L in (7, 8, 9, 15, 16, 17):
        st = state(32 * L, "minimal", seed=400 + L, edges=False)
        out.append(Case(f"minimal_len{L}", st, {e: 4 for e in (EPOCH - 1, EPOCH, EPOCH + 1)},
                        _attestations(st, np.random.default_rng(L), full=True)))
    # the first epochs: at epoch 0 previous == current
    st = state(300, "minimal", seed=500, edges=False, slot_in_epoch=5)
    st.fixed["slot"] = (5).to_bytes(8, "little")
    out.append(Case("minimal_genesis", st, {0: 4, 1: 4}, _attestations_genesis(st)))
    return out


def _attestations_genesis(st) -> list:
    """At slot 5 of epoch 0 previous == current == 0: slots 0..4 are attestable."""
    committees = co.beacon_committees(st, 0)
    out = []
    for s in range(5):
        members = committees[s * 4]
        out.append((co.attestation_data(s, 0, 0), co.bitlist([True] * len(members)), co.OK))
    out.append((co.attestation_data(5, 0, 0), co.bitlist([True] * len(committees[20])), co.NO_DELAY))
    out.append((co.attestation_data(8, 0, 1), co.bitlist([True] * len(committees[0])), co.INVALID_TARGET_EPOCH))
    return out
