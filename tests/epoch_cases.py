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


# the launch shape of csrc/epoch.cu: k_epoch_totals / k_epoch_apply run one thread per validator in CTAs of THREADS;
# k_epoch_reduce's REDUCE_THREADS threads fold ranges of `per` consecutive CTAs; a changed-record count above
# max(REHASH_MIN, n / 16) re-hashes the whole Validator list (capi_ssz.cu)
THREADS, REDUCE_THREADS, REHASH_MIN = 256, 512, 4096


@dataclass
class Grid:
    """Where a state's exit queue, ejections, activations and sums fall in the device's launch shape."""
    n: int
    nb: int             # CTAs
    per: int            # CTAs per k_epoch_reduce thread
    act_exit: int       # compute_activation_exit_epoch(current epoch)
    e0: int
    c0: int
    L: int              # churn limit
    limit: int          # activation churn limit
    head: np.ndarray    # indices whose exit epoch is E0 (the c0 validators the exit-queue head counts)
    eject: np.ndarray   # ejected indices in rank order
    eject_epoch: np.ndarray
    offered: np.ndarray  # activation candidates per CTA (after the eligibility update)
    winners: np.ndarray  # activated indices
    sums: list           # the five k_epoch_totals sums, each per CTA (Python ints)
    pushes: int          # records k_epoch_apply and k_activation_select append to the changed list under ALL
    threshold: int

    def cta(self, i):
        return np.asarray(i) // THREADS

    def warp(self, i):   # warp inside its CTA
        return np.asarray(i) % THREADS // 32

    def lane(self, i):
        return np.asarray(i) % 32

    def rthread(self, i):   # the k_epoch_reduce thread whose range holds i's CTA
        return self.cta(i) // self.per

    def overflow(self, k):
        """(the whole sum, the largest CTA partial, the largest k_epoch_reduce range) reach 2^64."""
        s = self.sums[k]
        ranges = [sum(s[t:t + self.per]) for t in range(0, self.nb, self.per)]
        return sum(s) > U64, max(s) > U64, max(ranges) > U64

    def ranks_cross(self):
        """Ranks k (k >= 1) where the exit epoch steps up between ejection k - 1 and k."""
        return np.nonzero(np.diff(self.eject_epoch.astype(np.int64)))[0] + 1


def grid(st: S.SynthState) -> Grid:
    st = eo.clone(st)
    n = len(st.validators)
    nb = -(-n // THREADS)
    per = -(-nb // REDUCE_THREADS)
    v = eo._Vector(st)
    cur, prev = v.cur(), v.prev()
    e0, c0, L = v.exit_queue()
    vv = st.validators
    eb = vv["effective_balance"].astype(np.uint64)
    exit_ = vv["exit_epoch"].astype(np.uint64)
    head = np.nonzero(exit_ == np.uint64(e0))[0]
    eject = np.nonzero(v.active(cur) & (eb <= np.uint64(eo.EJECTION_BALANCE)) & (exit_ == np.uint64(FAR)))[0]
    limit = min(eo.PRESET[st.preset]["MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT"], L)
    slashed = vv["slashed"] != 0
    pf, cf = st.previous_epoch_participation, st.current_epoch_participation
    a_cur, a_prev = v.active(cur), v.active(prev)
    masks = [a_cur] + [a_prev & ~slashed & (((pf >> f) & 1) != 0) for f in range(3)] + [a_cur & ~slashed & ((cf & 2) != 0)]
    ebo = eb.astype(object)
    sums = [[int(ebo[b * THREADS:(b + 1) * THREADS][m[b * THREADS:(b + 1) * THREADS]].sum()) for b in range(nb)] for m in masks]
    reg = eo.clone(st)
    eo._Vector(reg).registry_updates()
    ru = reg.validators
    elig = ru["activation_eligibility_epoch"]
    fin = int.from_bytes(st.fixed["finalized_checkpoint"][:8], "little")
    cand = (elig <= np.uint64(fin)) & (vv["activation_epoch"] == np.uint64(FAR))
    offered = np.bincount(np.nonzero(cand)[0] // THREADS, minlength=nb)
    winners = np.nonzero(ru["activation_epoch"] != vv["activation_epoch"])[0]
    try:
        post, _ = eo.process_epoch(st, eo.ALL)
        pv = post.validators
        rec = ((pv["activation_eligibility_epoch"] != vv["activation_eligibility_epoch"]) | (pv["exit_epoch"] != vv["exit_epoch"])
               | (pv["effective_balance"] != vv["effective_balance"]))
        pushes = int(rec.sum()) + int((pv["activation_epoch"] != vv["activation_epoch"]).sum())
    except eo.Refused:
        pushes = -1
    return Grid(n, nb, per, eo.compute_activation_exit_epoch(cur), e0, c0, L, limit, head, eject, ru["exit_epoch"][eject].astype(np.uint64), offered, winners, sums,
                pushes, max(REHASH_MIN, n // 16))


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


def exits(st, idx, epoch) -> None:
    """Validators `idx` exit at `epoch` (withdrawable MIN_VALIDATOR_WITHDRAWABILITY_DELAY later)."""
    st.validators["exit_epoch"][idx] = epoch
    st.validators["withdrawable_epoch"][idx] = epoch + eo.MIN_VALIDATOR_WITHDRAWABILITY_DELAY


def ejects(st, idx) -> None:
    st.validators["effective_balance"][idx] = eo.EJECTION_BALANCE


def pending(st, idx, elig) -> None:
    """Validators `idx` wait in the activation queue, eligible since `elig`."""
    st.validators["activation_epoch"][idx] = FAR
    st.validators["activation_eligibility_epoch"][idx] = elig


def grid_cases() -> list:
    """Small states whose exit-queue head, ejections, sums, activation candidates and changed-record counts sit where
    the device's kernels pass values between lanes, warps and CTAs (csrc/epoch.cu); every one at most 4 097 validators.
    Regime "grid:<name>"; test_epoch_cases.py asserts each shape from `grid()`."""
    out = []
    add = lambda name, st, refusal=None: out.append(Case(name, st, "grid:" + name, refusal))  # noqa: E731
    # the exit-queue head with c0 < L, merged across warps and CTAs; ejection ranks stepping over a multiple of L between
    # two CTAs.  mainnet n = 600 / 1000 / 520: L = 4, 3 / 4 / 3 CTAs (the last ragged: 88 / 232 / 8 threads)
    st = base(600, 1000, seed=60)
    exits(st, [33, 100, 230], 1012)                         # E0 = the largest exit, c0 = 3, warps 1, 3, 7 of CTA 0
    exits(st, [7, 300], 990)
    ejects(st, [255, 256, 420, 599])                        # (3 + k) / 4 steps at k = 1: thread 255 of CTA 0, 0 of CTA 1
    add("head_c0_3_warps", st)
    st = base(1000, 1000, seed=61)
    exits(st, [0, 999], 1005)                               # E0 = compute_activation_exit_epoch, c0 = 2, first and last CTA
    ejects(st, [31, 767, 768, 998])                         # (2 + k) / 4 steps at k = 2: CTA 2's last thread, CTA 3's first
    add("head_c0_2_first_last_cta", st)
    st = base(520, 1000, seed=62)
    exits(st, [519], 1009)                                  # c0 = 1 at the last valid thread of the ragged CTA
    ejects(st, [100, 200, 255, 256, 511, 512])              # (1 + k) / 4 steps at k = 3: thread 0 of CTA 1
    add("head_c0_1_ragged", st)
    # minimal n = 600: L = 18, c0 = 17 holders in every CTA; ranks step at k = 1 (CTA 0 -> 1) and k = 19 (CTA 1 -> 2)
    st = base(600, 1000, "minimal", seed=63)
    exits(st, [0, 31, 32, 63, 64, 200, 255, 256, 287, 288, 400, 511, 512, 543, 544, 598, 599], 1010)
    ejects(st, [254] + list(range(257, 500, 14)) + [513, 514, 597])
    add("head_c0_17_minimal", st)
    # ejections at lanes 0 and 31, threads 0 and 255, all in the ragged last CTA, one per CTA
    st = base(1000, 1000, seed=64)
    ejects(st, [32, 63, 160, 191, 256, 511, 767])           # c0 = 0: E0 = compute_activation_exit_epoch
    add("eject_lanes_threads", st)
    st = base(1000, 1000, seed=65)
    exits(st, [5], 1005)
    ejects(st, [768, 769, 799, 800, 900, 999])              # c0 = 1; all in CTA 3 (232 threads), its first and last
    add("eject_ragged_last_cta", st)
    st = base(4096, 1000, "minimal", seed=66)                # L = 128, c0 = 126: (126 + k) / 128 steps at k = 2
    exits(st, np.arange(126) * 32 + 7, 1011)
    ejects(st, np.arange(16) * 256 + np.array([0, 255, 31, 32, 128, 1, 254, 63, 64, 100, 200, 17, 96, 33, 250, 255]))
    add("eject_one_per_cta", st)
    # get_total_balance's 128-bit sums: every CTA partial below 2^64, the fold across CTAs at 2^64 (refused) and 2^64 - 1
    for name, total, refusal in (("sum_2p64_across_ctas", 1 << 64, "limit"), ("sum_2p64_minus_1_across_ctas", U64, None)):
        st = base(600, 1000, seed=67)
        eb = st.validators["effective_balance"]
        rest = int(eb.astype(object).sum()) - 3 * int(eb[0])
        eb[[10, 300, 590]] = [1 << 62, 1 << 63, total - rest - (1 << 62) - (1 << 63)]
        add(name, st, refusal)
    # previous-epoch-only overflow: validators exiting at the current epoch count in the previous-epoch flag sums only
    st = base(600, 1000, seed=68)
    exits(st, [20, 21, 400, 401], 1000)
    st.validators["effective_balance"][[20, 21, 400, 401]] = [1 << 62, 1 << 62, 1 << 62, (1 << 62) + 5]
    st.previous_epoch_participation[[20, 21, 400, 401]] = 7
    add("overflow_previous_only", st, "limit")
    # activation candidates (mainnet, limit 4)
    st = base(600, 1000, seed=69)
    pending(st, np.arange(260, 270), 990)                   # CTA 1 offers 10 at the earliest eligibility
    pending(st, [3, 520], 992)
    st.fixed["finalized_checkpoint"] = _cp(995, b"f")
    add("activation_many_in_one_cta", st)
    st = base(1000, 1000, seed=70)
    pending(st, [900, 600, 300, 10, 257, 520], 990)         # ties across CTAs, broken by index
    pending(st, [5, 6], 994)
    st.fixed["finalized_checkpoint"] = _cp(995, b"f")
    add("activation_ties_across_ctas", st)
    st = base(1000, 1000, seed=71)
    pending(st, [768, 999, 850, 851, 852], 985)             # the winners: all in the ragged last CTA
    pending(st, [0, 1, 300, 700], 986)
    st.fixed["finalized_checkpoint"] = _cp(995, b"f")
    add("activation_last_cta_only", st)
    st = base(600, 1000, "minimal", seed=72)
    pending(st, [40, 599], 990)                             # a queue of 2 under limit 4
    add("activation_short_queue", st)
    # changed-record counts at the re-hash threshold (max(4096, n / 16) = 4096 at n = 4097): eligibility set on records
    # with activation_eligibility_epoch = FAR and effective_balance = MAX, plus one activated record whose effective
    # balance also changes (two pushes)
    for count in (4096, 4097):
        st = base(4097, 1000, seed=73)
        st.balances[:] = 32 * ETH
        st.validators["activation_eligibility_epoch"][1:count - 1] = FAR
        pending(st, [4096], 990)
        st.balances[4096] = 40 * ETH
        st.validators["effective_balance"][4096] = 30 * ETH
        add(f"changed_{count}", st)
    return out


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
    return out + grid_cases()
