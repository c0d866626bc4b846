"""Seeded deneb states for the proposer / sync-committee duty functions (ethereum_consensus_b200.duties), each built for
one regime of the sampling loops or of the committee-key lookup.  Shared by test_duties_cases.py (CPU: the oracle's two
formulations and each case's regime) and test_duties_gpu.py (the device against the oracle)."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from ethereum_consensus_b200 import state as S
from oracle import duties_oracle as do

ETH = 10**9
FAR = S.FAR_FUTURE_EPOCH
OVERFLOW_BALANCE = -(-(1 << 64) // 255)   # ceil(2^64 / 255): * 255 wraps to 254 in u64


@dataclass
class Case:
    name: str
    st: S.SynthState
    epochs: list                        # proposer-lookahead epochs to check
    regime: str                         # what test_duties_cases checks the case hits
    seed_epochs: list = field(default_factory=list)   # extra get_seed epochs (no proposer call)
    committee: bool = True              # next_sync_committee is defined (an active validator at the next epoch)


def base(n: int, preset: str = "mainnet", seed: int = 1, eff=32 * ETH, slot_epoch: int = 1000) -> S.SynthState:
    """n validators, all active from epoch 0, every effective balance `eff`; slot at the start of `slot_epoch`."""
    st = S.synth_state(n, preset, seed=seed, n_eth1_votes=2, n_historical_summaries=2)
    v = st.validators
    v["activation_epoch"] = 0
    v["exit_epoch"] = FAR
    v["effective_balance"] = eff
    spe = do.PRESET[preset]["SLOTS_PER_EPOCH"]
    st.fixed["slot"] = int(slot_epoch * spe).to_bytes(8, "little")
    return st


def only_active(st: S.SynthState, keep) -> S.SynthState:
    """Every validator outside `keep` is made inactive (half not yet activated, half exited)."""
    v = st.validators
    off = np.ones(len(v), bool)
    off[np.asarray(keep, dtype=np.int64)] = False
    late = off & (np.arange(len(v)) % 2 == 0)
    v["activation_epoch"][late] = FAR - 1
    v["exit_epoch"][off & ~late] = 0
    return st


def set_committees(st: S.SynthState, cur_idx, nxt_idx) -> S.SynthState:
    """current / next sync committees made of the keys of the given validator indices (aggregates: placeholders)."""
    pk = st.validators["public_key"]
    blob = lambda idx: b"".join(pk[int(i)].tobytes() for i in idx) + bytes(48)  # noqa: E731
    st.current_sync_committee, st.next_sync_committee = blob(cur_idx), blob(nxt_idx)
    return st


def cases() -> list:
    out = []
    spe_m = 32
    st = only_active(base(40, seed=2), [17])
    out.append(Case("one_active", st, [1000, 1001], "one_active"))
    out.append(Case("all_32eth", base(1000, seed=3), [1000, 1001, 77], "all_32eth"))
    st = base(2000, seed=4)
    rng = np.random.default_rng(4)
    st.validators["effective_balance"] = rng.choice(np.array([0, 1, 16, 31, 32], np.uint64) * ETH, size=2000)
    out.append(Case("mixed_balances", st, [1000, 1001], "mixed"))
    out.append(Case("all_1eth", base(3000, seed=5, eff=1 * ETH), [1000], "several_windows"))
    out.append(Case("all_0eth", base(600, seed=6, eff=0), [1000], "all_0eth"))
    for k in (1, 2, 3, 255, 256, 257):
        st = only_active(base(k + 50, seed=10 + k), np.arange(25, 25 + k))
        st.validators["effective_balance"][25:25 + k] = np.resize(np.array([32, 31, 16, 0], np.uint64) * ETH, k)
        st.validators["effective_balance"][25] = 32 * ETH
        out.append(Case(f"active_{k}", st, [1000], f"active_{k}"))
    st = base(4000, seed=7)
    rng = np.random.default_rng(7)
    out.append(Case("inactive_majority", only_active(st, np.sort(rng.choice(4000, 300, replace=False))), [1000, 1001],
                    "inactive_majority"))
    st = base(500, "minimal", seed=8)
    st.validators["effective_balance"] = np.random.default_rng(8).choice(np.array([0, 16, 32], np.uint64) * ETH, size=500)
    out.append(Case("minimal", st, [1000, 5], "minimal"))
    # get_seed's mix index (epoch + EPHV - 2) mod EPHV at its wrap: epochs 0 and 1 read the last two mixes, 2 the first;
    # the largest epoch whose slots fit in u64; u64 wrap of the index itself
    st = base(700, seed=9, slot_epoch=0)
    out.append(Case("randao_wrap", st, [0, 1, 2, 65535, 65536, (2**64 - 1) // spe_m], "randao_wrap",
                    seed_epochs=[2**64 - 1, 2**64 - 2, 2**64 - 65536]))
    st = base(700, "minimal", seed=9, slot_epoch=63)
    out.append(Case("randao_wrap_minimal", st, [0, 1, 2, 63, 64, (2**64 - 1) // 8], "randao_wrap", seed_epochs=[2**64 - 1]))
    # one record whose effective_balance * 255 wraps in u64 (accepted only on a random byte of 0), among 0-ETH records
    st = only_active(base(30, seed=11, eff=0), np.arange(4, 12))
    st.validators["effective_balance"][6] = OVERFLOW_BALANCE
    out.append(Case("overflow_record", st, [1000, 1001], "overflow"))
    # registry with repeated keys (7 distinct, tiled): the lookup returns the largest holder; committees of those keys
    st = base(300, seed=12)
    pk = st.validators["public_key"].copy()
    st.validators["public_key"] = pk[np.arange(300) % 7]
    rng = np.random.default_rng(12)
    out.append(Case("repeated_keys", set_committees(st, rng.integers(0, 300, 512), rng.integers(0, 300, 512)), [1000],
                    "repeated_keys"))
    # a committee key no validator holds (current: position 5; next: the last position)
    st = set_committees(base(300, seed=13), np.arange(512) % 300, (np.arange(512) * 7) % 300)
    b = bytearray(st.current_sync_committee); b[5 * 48:6 * 48] = bytes(range(48)); st.current_sync_committee = bytes(b)
    b = bytearray(st.next_sync_committee); b[511 * 48:512 * 48] = bytes(range(1, 49)); st.next_sync_committee = bytes(b)
    out.append(Case("missing_key", st, [1000], "missing_key"))
    return out


def rotation_state(n: int = 300, preset: str = "mainnet", seed: int = 14, boundary: bool = True) -> S.SynthState:
    """A state one epoch before a sync-committee period boundary (or one epoch off it)."""
    P = do.PRESET[preset]
    e = 4 * P["EPOCHS_PER_SYNC_COMMITTEE_PERIOD"] - 1 - (0 if boundary else 1)
    return base(n, preset, seed=seed, slot_epoch=e)
