"""Seeded deneb states for process_epoch on the device-resident state (ethereum_consensus_b200.epoch), each built for one
regime of the twelve sub-steps.  Shared by test_epoch_cases.py (CPU: the oracle's two formulations agree and each case
hits its regime) and test_epoch_gpu.py (the device against the oracle)."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from ethereum_consensus_b200 import state as S
from oracle import bls_oracle as bo
from oracle import epoch_oracle as eo

ETH = 10**9
FAR = S.FAR_FUTURE_EPOCH
U64 = (1 << 64) - 1


@dataclass
class Case:
    name: str
    st: S.SynthState
    regime: str
    refusal: str | None = None   # "bad_arg" / "limit": process_epoch(ALL) is refused


def _cp(epoch: int, tag: bytes) -> bytes:
    return int(epoch).to_bytes(8, "little") + (tag * 32)[:32]


def valid_pubkeys(n: int) -> np.ndarray:
    return np.frombuffer(b"".join(bo.sk_to_pk(0x5eed + 7 * i) for i in range(n)), np.uint8).reshape(n, 48)


def base(n: int, epoch: int, preset: str = "mainnet", seed: int = 1, keys: bool = False, first_slot: bool = False) -> S.SynthState:
    """n validators active since epoch 0, 32 ETH effective, balances 31.5..32.5 ETH, random flags and small scores; the slot
    is the last of `epoch` (where a state transition runs process_epoch); nothing justified recently."""
    rng = np.random.default_rng(seed)
    st = S.synth_state(n, preset, seed=seed, n_eth1_votes=3, n_historical_summaries=2,
                       pubkeys=valid_pubkeys(n) if keys else None)
    v = st.validators
    v["slashed"] = 0
    v["activation_eligibility_epoch"] = 0
    v["activation_epoch"] = 0
    v["exit_epoch"] = FAR
    v["withdrawable_epoch"] = FAR
    v["effective_balance"] = 32 * ETH
    st.balances = (31_500_000_000 + rng.integers(0, ETH, n, dtype=np.uint64)).astype("<u8")
    st.previous_epoch_participation = rng.integers(0, 8, n, dtype=np.uint8)
    st.current_epoch_participation = rng.integers(0, 8, n, dtype=np.uint8)
    st.inactivity_scores = rng.integers(0, 40, n, dtype=np.uint64).astype("<u8")
    st.slashings[:] = 0
    st.slashings[::7] = rng.integers(0, 2 * ETH, len(st.slashings[::7]), dtype=np.uint64)
    spe = eo.PRESET[preset]["SLOTS_PER_EPOCH"]
    st.fixed["slot"] = int(epoch * spe + (0 if first_slot else spe - 1)).to_bytes(8, "little")
    back = lambda k: max(epoch - k, 0)  # noqa: E731
    st.fixed["justification_bits"] = bytes([0])
    st.fixed["previous_justified_checkpoint"] = _cp(back(6), b"p")
    st.fixed["current_justified_checkpoint"] = _cp(back(5), b"c")
    st.fixed["finalized_checkpoint"] = _cp(back(3), b"f")
    return st


def _flags(st, which: str, bit: int, on: bool) -> None:
    a = getattr(st, which)
    setattr(st, which, (np.where(on, a | (1 << bit), a & ~np.uint8(1 << bit))).astype(np.uint8))


def finality(rule: int, preset: str = "mainnet") -> S.SynthState:
    """A state at which exactly finalization rule `rule` (1: bits 1-3 and old previous + 3; 2: bits 1-2 and old previous
    + 2; 3: bits 0-2 and old current + 2; 4: bits 0-1 and old current + 1) fires."""
    cur = 1000
    st = base(200, cur, preset, seed=10 + rule)
    old_bits, pj, cj, prev_hi, cur_hi = {1: (0b0111, cur - 3, cur - 2, True, False), 2: (0b0011, cur - 2, cur - 4, False, False),
                                         3: (0b0011, cur - 5, cur - 2, False, True), 4: (0b0001, cur - 6, cur - 1, False, True)}[rule]
    st.fixed["justification_bits"] = bytes([old_bits])
    st.fixed["previous_justified_checkpoint"] = _cp(pj, b"P")
    st.fixed["current_justified_checkpoint"] = _cp(cj, b"C")
    st.fixed["finalized_checkpoint"] = _cp(cur - 9, b"F")
    _flags(st, "previous_epoch_participation", 1, prev_hi)
    _flags(st, "current_epoch_participation", 1, cur_hi)
    return st


def cases() -> list:
    out = []
    add = lambda name, st, regime, refusal=None: out.append(Case(name, st, regime, refusal))  # noqa: E731

    add("epoch0", base(100, 0, seed=2), "epoch0")
    add("epoch1", base(100, 1, seed=3), "epoch1")
    for r in (1, 2, 3, 4):
        add(f"finality_rule{r}", finality(r), f"finality{r}")
    st = base(200, 1000, seed=4)
    st.fixed["finalized_checkpoint"] = _cp(990, b"f")
    st.inactivity_scores[:] = np.arange(200, dtype=np.uint64) * 3
    add("inactivity_leak", st, "leak")
    st = base(200, 1000, seed=5)
    st.inactivity_scores[:] = 50 + np.arange(200, dtype=np.uint64)
    add("leak_recovery", st, "recovery")
    st = base(150, 1000, seed=6)
    st.previous_epoch_participation[:] = 7
    st.current_epoch_participation[:] = 7
    add("all_participating", st, "all_participating")
    st = base(150, 1000, seed=7)
    st.previous_epoch_participation[:] = 0
    st.current_epoch_participation[:] = 0
    add("none_participating", st, "none_participating")
    for capped in (True, False):
        st = base(120, 1000, seed=8 + capped)
        P = eo.PRESET["mainnet"]
        v = st.validators
        v["slashed"][::5] = 1
        v["withdrawable_epoch"][::10] = 1000 + P["EPOCHS_PER_SLASHINGS_VECTOR"] // 2
        v["withdrawable_epoch"][5::10] = 1000 + P["EPOCHS_PER_SLASHINGS_VECTOR"] // 2 + 1
        v["exit_epoch"][::5] = 1010
        st.slashings[:] = 0
        st.slashings[3] = 10**15 if capped else 300 * ETH
        st.slashings[4] = 10**15 if capped else 0
        add("slashings_" + ("capped" if capped else "partial"), st, "slashings_capped" if capped else "slashings_partial")
    # ejections: E0 below, at and above compute_activation_exit_epoch (1005), and c0 >= L (L = 4)
    for name, exits in (("below", [990, 1001, 1004]), ("at", [1005, 1005]), ("above", [1020]), ("c0_ge_L", [1007] * 6)):
        st = base(150, 1000, seed=20 + len(name))
        v = st.validators
        v["exit_epoch"][140:140 + len(exits)] = exits
        v["withdrawable_epoch"][140:140 + len(exits)] = np.array(exits, np.uint64) + 256
        v["effective_balance"][3:130:12] = 16 * ETH        # 11 ejections
        v["effective_balance"][7] = 16 * ETH + 1           # just above EJECTION_BALANCE: stays
        add(f"eject_{name}", st, f"eject_{name}")
    # activation queue: ties in eligibility, gated by the finalized epoch (995), longer than the churn limit
    st = base(200, 1000, seed=30)
    v = st.validators
    v["activation_epoch"][20:60] = FAR
    v["activation_eligibility_epoch"][20:60] = np.array([994, 990, 995, 996, 990] * 8, np.uint64)
    v["activation_eligibility_epoch"][60:64] = FAR       # become eligible at 1001: not yet in the queue
    v["activation_epoch"][60:64] = FAR
    st.fixed["finalized_checkpoint"] = _cp(995, b"f")
    add("activation_queue", st, "activation_queue")
    st = base(40, 1000, "minimal", seed=31)
    v = st.validators
    v["activation_epoch"][5:25] = FAR
    v["activation_eligibility_epoch"][5:25] = 990
    add("activation_queue_minimal", st, "activation_queue")
    # hysteresis exactly at its thresholds and one gwei around them
    st = base(120, 1000, seed=32)
    eb = np.array([32, 20, 17] * 40, np.uint64)[:120] * ETH
    st.validators["effective_balance"] = eb
    d = np.array([-250_000_000, -250_000_001, -249_999_999, 1_250_000_000, 1_250_000_001, 1_249_999_999] * 20, np.int64)
    st.balances = (eb.astype(np.int64) + d).astype("<u8")
    add("hysteresis", st, "hysteresis")
    st = base(100, 1000, seed=33)
    st.balances[:] = np.arange(100, dtype=np.uint64) * 10_000
    st.previous_epoch_participation[:] = 0
    st.inactivity_scores[:] = 10**6
    add("saturating_penalties", st, "saturate")
    st = base(100, 1000, seed=34)
    st.balances[:] = (40 + np.arange(100, dtype=np.uint64)) * ETH
    add("balances_above_max", st, "above_max")
    st = base(100, 1000, seed=35)
    st.inactivity_scores[:] = (1 << 40) + np.arange(100, dtype=np.uint64)     # eb * score wraps
    st.balances[:20] = U64 - np.arange(20, dtype=np.uint64)                   # increase_balance wraps
    st.previous_epoch_participation[:20] = 7
    st.validators["effective_balance"][50] = 1 << 62                          # base reward products wrap
    st.fixed["finalized_checkpoint"] = _cp(998, b"f")
    add("wrapping", st, "wrapping")
    add("one_validator", base(1, 1000, seed=36), "one_validator")
    st = base(100, 1000, seed=37)
    st.validators["activation_epoch"][:] = 1000
    add("none_active_previous", st, "none_active_previous")
    add("minimal", base(64, 1000, "minimal", seed=38), "minimal")
    # period boundaries (next epoch 8: eth1 voting, historical root and sync committee periods of the minimal preset)
    add("minimal_boundaries", base(64, 7, "minimal", seed=39, keys=True), "boundaries")
    add("randao_wrap", base(48, 63, "minimal", seed=40, keys=True), "randao_wrap")
    add("mainnet_eth1_boundary", base(100, 63, seed=41), "eth1_boundary")
    # mainnet: every period ends at next epoch 256; random keys fail the aggregation after the other writes
    add("mainnet_boundaries_bad_keys", base(600, 255, seed=42), "aggregation_fails")
    # refusals
    st = base(100, 1000, seed=50, first_slot=True)
    st.current_epoch_participation[:] = 7
    add("refuse_block_root", st, "refusal", "bad_arg")
    st = base(100, 1000, seed=51)
    st.validators["effective_balance"][:10] = 1 << 62
    add("refuse_total_overflow", st, "refusal", "limit")
    st = base(100, 1000, seed=52)
    st.validators["exit_epoch"][99] = U64 - 100
    st.validators["effective_balance"][4] = 10 * ETH
    add("refuse_withdrawable_overflow", st, "refusal", "limit")
    st = base(40, 7, "minimal", seed=53)
    st.validators["exit_epoch"][:] = 8
    add("refuse_no_active_next", st, "refusal", "bad_arg")
    return out
