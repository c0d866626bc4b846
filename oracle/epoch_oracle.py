"""CPU oracle for deneb `process_epoch` — TEST INFRASTRUCTURE ONLY (tests/ and tools/ import it).

Restates the twelve sub-steps of ethereum-consensus/src/deneb/spec/mod.rs:991-1002 over a `state.SynthState`, in two
formulations that tests pin against each other:
  * "literal": the reference loop for loop — membership sets from get_unslashed_participating_indices, the deltas as
    whole vectors applied pair by pair, `initiate_validator_exit` recomputing the exit queue for every ejection, the
    activation queue sorted.  get_total_active_balance is evaluated once per delta function instead of once per
    validator (it cannot change inside one), which keeps the literal form linear.
  * "vector": numpy over whole columns, the exit queue in closed form (the rule include/b200_consensus.h states).
The per-validator sub-steps differ between the two; the small fields (checkpoints, resets, the historical summary, the
participation rotation, the sync committees) are shared.
Rules the reference leaves to its build, as the library states them: arithmetic wraps in u64 (a release build) except
decrease_balance, which saturates; where the reference returns Err the oracle raises `Refused` ("bad_arg" or "limit") and
the input is untouched; a failed sync-committee aggregation comes back as a code with every earlier sub-step applied.
"""
from __future__ import annotations

import copy

import numpy as np

from ethereum_consensus_b200 import state as S
from oracle import duties_oracle as do
from oracle import ssz_oracle as so

U64 = (1 << 64) - 1
FAR = U64
STEPS = ("justification_and_finalization", "inactivity_updates", "rewards_and_penalties", "registry_updates", "slashings",
         "eth1_data_reset", "effective_balance_updates", "slashings_reset", "randao_mixes_reset",
         "historical_summaries_update", "participation_flag_updates", "sync_committee_updates")
STEP = {name: 1 << k for k, name in enumerate(STEPS)}
ALL = (1 << len(STEPS)) - 1

# phase0/presets, altair/presets, bellatrix/presets, configs/{mainnet,minimal}.rs
PRESET = {
    "mainnet": dict(SLOTS_PER_EPOCH=32, SLOTS_PER_HISTORICAL_ROOT=8192, EPOCHS_PER_HISTORICAL_VECTOR=65536,
                    EPOCHS_PER_SLASHINGS_VECTOR=8192, EPOCHS_PER_ETH1_VOTING_PERIOD=64, EPOCHS_PER_SYNC_COMMITTEE_PERIOD=256,
                    MIN_PER_EPOCH_CHURN_LIMIT=4, MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT=8, CHURN_LIMIT_QUOTIENT=65536),
    "minimal": dict(SLOTS_PER_EPOCH=8, SLOTS_PER_HISTORICAL_ROOT=64, EPOCHS_PER_HISTORICAL_VECTOR=64,
                    EPOCHS_PER_SLASHINGS_VECTOR=64, EPOCHS_PER_ETH1_VOTING_PERIOD=4, EPOCHS_PER_SYNC_COMMITTEE_PERIOD=8,
                    MIN_PER_EPOCH_CHURN_LIMIT=2, MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT=4, CHURN_LIMIT_QUOTIENT=32),
}
HISTORICAL_ROOTS_LIMIT = 1 << 24
INC = 10**9                     # EFFECTIVE_BALANCE_INCREMENT
MAX_EFFECTIVE_BALANCE = 32 * INC
EJECTION_BALANCE = 16 * INC
HYSTERESIS_QUOTIENT, HYSTERESIS_DOWNWARD_MULTIPLIER, HYSTERESIS_UPWARD_MULTIPLIER = 4, 1, 5
INACTIVITY_SCORE_BIAS, INACTIVITY_SCORE_RECOVERY_RATE = 4, 16
INACTIVITY_PENALTY_QUOTIENT_BELLATRIX = 1 << 24
PROPORTIONAL_SLASHING_MULTIPLIER_BELLATRIX = 3
BASE_REWARD_FACTOR = 64
MIN_EPOCHS_TO_INACTIVITY_PENALTY = 4
MAX_SEED_LOOKAHEAD = 4
MIN_VALIDATOR_WITHDRAWABILITY_DELAY = 256
PARTICIPATION_FLAG_WEIGHTS = (14, 26, 14)
WEIGHT_DENOMINATOR = 64
TIMELY_TARGET_FLAG_INDEX, TIMELY_HEAD_FLAG_INDEX = 1, 2


class Refused(Exception):
    """The reference's Err: the library refuses with B200_ERR_BAD_ARG ("bad_arg") or B200_ERR_LIMIT ("limit")."""

    def __init__(self, kind: str, msg: str):
        super().__init__(msg)
        self.kind = kind


def mask(steps) -> int:
    if isinstance(steps, int):
        return steps
    if isinstance(steps, str):
        return STEP[steps]
    m = 0
    for s in steps:
        m |= STEP[s]
    return m


def current_epoch(st) -> int:
    return do.slot(st) // PRESET[st.preset]["SLOTS_PER_EPOCH"]


def clone(st: S.SynthState) -> S.SynthState:
    out = copy.copy(st)
    out.fixed = dict(st.fixed)
    for f in ("block_roots", "state_roots", "historical_roots", "eth1_data_votes", "validators", "balances", "randao_mixes",
              "slashings", "previous_epoch_participation", "current_epoch_participation", "inactivity_scores",
              "historical_summaries"):
        setattr(out, f, getattr(st, f).copy())
    return out


def integer_sqrt(x: int) -> int:
    import math
    return math.isqrt(x)


def compute_activation_exit_epoch(epoch: int) -> int:
    return (epoch + 1 + MAX_SEED_LOOKAHEAD) & U64


def churn_limit(st, n_active: int) -> int:
    P = PRESET[st.preset]
    return max(P["MIN_PER_EPOCH_CHURN_LIMIT"], n_active // P["CHURN_LIMIT_QUOTIENT"])


# ---- justification and finalization: the sums differ by formulation, the weighing is shared ----
def get_block_root(st, epoch: int) -> bytes:
    P = PRESET[st.preset]
    at = (epoch * P["SLOTS_PER_EPOCH"]) & U64
    slot = do.slot(st)
    if at >= slot or slot > ((at + P["SLOTS_PER_HISTORICAL_ROOT"]) & U64):
        raise Refused("bad_arg", f"get_block_root: slot {at} out of range at state slot {slot}")
    return st.block_roots[at % P["SLOTS_PER_HISTORICAL_ROOT"]].tobytes()


def weigh_justification_and_finalization(st, total_active: int, previous_target: int, current_target: int) -> None:
    """:1469-1520 on st.fixed (the caller's copy)."""
    cur = current_epoch(st)
    prev = cur - 1 if cur else 0
    f = st.fixed
    old_pj, old_cj = f["previous_justified_checkpoint"], f["current_justified_checkpoint"]
    f["previous_justified_checkpoint"] = old_cj
    b = f["justification_bits"][0]
    bits = ((b << 1) & 0x0e) | (b & 0xf0)
    if (previous_target * 3) & U64 >= (total_active * 2) & U64:
        f["current_justified_checkpoint"] = prev.to_bytes(8, "little") + get_block_root(st, prev)
        bits |= 2
    if (current_target * 3) & U64 >= (total_active * 2) & U64:
        f["current_justified_checkpoint"] = cur.to_bytes(8, "little") + get_block_root(st, cur)
        bits |= 1
    f["justification_bits"] = bytes([bits])
    pj, cj = int.from_bytes(old_pj[:8], "little"), int.from_bytes(old_cj[:8], "little")
    if bits & 0x0e == 0x0e and (pj + 3) & U64 == cur:
        f["finalized_checkpoint"] = old_pj
    if bits & 0x06 == 0x06 and (pj + 2) & U64 == cur:
        f["finalized_checkpoint"] = old_pj
    if bits & 0x07 == 0x07 and (cj + 2) & U64 == cur:
        f["finalized_checkpoint"] = old_cj
    if bits & 0x03 == 0x03 and (cj + 1) & U64 == cur:
        f["finalized_checkpoint"] = old_cj


def is_in_inactivity_leak(st) -> bool:
    cur = current_epoch(st)
    prev = cur - 1 if cur else 0
    fin = int.from_bytes(st.fixed["finalized_checkpoint"][:8], "little")
    return ((prev - fin) & U64) > MIN_EPOCHS_TO_INACTIVITY_PENALTY


# ---- the literal formulation of the per-validator sub-steps ----
class _Literal:
    """Python lists of ints and dicts, mutated in place like the reference's `&mut state`."""

    def __init__(self, st):
        self.st = st
        self.v = [{k: int(r[k]) for k in ("effective_balance", "slashed", "activation_eligibility_epoch", "activation_epoch",
                                           "exit_epoch", "withdrawable_epoch")} for r in st.validators]
        self.bal = [int(x) for x in st.balances]
        self.scores = [int(x) for x in st.inactivity_scores]
        self.prev_part = [int(x) for x in st.previous_epoch_participation]
        self.cur_part = [int(x) for x in st.current_epoch_participation]

    def write_back(self):
        st = self.st
        for k in self.v[0] if self.v else ():
            st.validators[k] = np.array([r[k] for r in self.v], dtype=st.validators.dtype[k])
        st.balances = np.array(self.bal, dtype="<u8")
        st.inactivity_scores = np.array(self.scores, dtype="<u8")

    def cur(self):
        return current_epoch(self.st)

    def prev(self):
        c = self.cur()
        return c - 1 if c else 0

    @staticmethod
    def is_active(v, epoch):
        return v["activation_epoch"] <= epoch < v["exit_epoch"]

    def active_indices(self, epoch):
        return [i for i, v in enumerate(self.v) if self.is_active(v, epoch)]

    def get_total_balance(self, indices):
        acc = 0
        for i in indices:
            acc += self.v[i]["effective_balance"]
            if acc > U64:
                raise Refused("limit", "get_total_balance: checked_add overflow")
        return max(acc, INC)

    def get_total_active_balance(self):
        return self.get_total_balance(set(self.active_indices(self.cur())))

    def get_unslashed_participating_indices(self, flag, epoch):
        part = self.cur_part if epoch == self.cur() else self.prev_part
        return {i for i in self.active_indices(epoch) if (part[i] >> flag) & 1 and not self.v[i]["slashed"]}

    def eligible(self):
        prev = self.prev()
        return [i for i, v in enumerate(self.v) if self.is_active(v, prev) or (v["slashed"] and prev + 1 < v["withdrawable_epoch"])]

    def justification_and_finalization(self):
        cur = self.cur()
        if cur <= 1:
            return
        previous_indices = self.get_unslashed_participating_indices(TIMELY_TARGET_FLAG_INDEX, self.prev())
        current_indices = self.get_unslashed_participating_indices(TIMELY_TARGET_FLAG_INDEX, cur)
        total = self.get_total_active_balance()
        weigh_justification_and_finalization(self.st, total, self.get_total_balance(previous_indices),
                                             self.get_total_balance(current_indices))

    def inactivity_updates(self):
        if self.cur() == 0:
            return
        eligible = self.eligible()
        participating = self.get_unslashed_participating_indices(TIMELY_TARGET_FLAG_INDEX, self.prev())
        not_leaking = not is_in_inactivity_leak(self.st)
        for i in eligible:
            if i in participating:
                self.scores[i] -= min(1, self.scores[i])
            else:
                self.scores[i] = (self.scores[i] + INACTIVITY_SCORE_BIAS) & U64
            if not_leaking:
                self.scores[i] -= min(INACTIVITY_SCORE_RECOVERY_RATE, self.scores[i])

    def flag_index_deltas(self, flag):
        n = len(self.v)
        rewards, penalties = [0] * n, [0] * n
        participating = self.get_unslashed_participating_indices(flag, self.prev())
        weight = PARTICIPATION_FLAG_WEIGHTS[flag]
        participating_increments = self.get_total_balance(participating) // INC
        total = self.get_total_active_balance()
        active_increments = total // INC
        base_per_increment = INC * BASE_REWARD_FACTOR // integer_sqrt(total)
        not_leaking = not is_in_inactivity_leak(self.st)
        for i in self.eligible():
            base = (self.v[i]["effective_balance"] // INC * base_per_increment) & U64
            if i in participating:
                if not_leaking:
                    num = (base * weight * participating_increments) & U64
                    rewards[i] += num // (active_increments * WEIGHT_DENOMINATOR)
            elif flag != TIMELY_HEAD_FLAG_INDEX:
                penalties[i] += ((base * weight) & U64) // WEIGHT_DENOMINATOR
        return rewards, penalties

    def inactivity_penalty_deltas(self):
        n = len(self.v)
        penalties = [0] * n
        matching = self.get_unslashed_participating_indices(TIMELY_TARGET_FLAG_INDEX, self.prev())
        for i in self.eligible():
            if i not in matching:
                num = (self.v[i]["effective_balance"] * self.scores[i]) & U64
                penalties[i] += num // (INACTIVITY_SCORE_BIAS * INACTIVITY_PENALTY_QUOTIENT_BELLATRIX)
        return [0] * n, penalties

    def decrease(self, i, delta):
        self.bal[i] = 0 if delta > self.bal[i] else self.bal[i] - delta

    def rewards_and_penalties(self):
        if self.cur() == 0:
            return
        deltas = [self.flag_index_deltas(f) for f in range(3)]
        deltas.append(self.inactivity_penalty_deltas())
        for rewards, penalties in deltas:
            for i in range(len(self.v)):
                self.bal[i] = (self.bal[i] + rewards[i]) & U64
                self.decrease(i, penalties[i])

    def initiate_validator_exit(self, i):
        if self.v[i]["exit_epoch"] != FAR:
            return
        exit_epochs = [v["exit_epoch"] for v in self.v if v["exit_epoch"] != FAR]
        exit_epochs.append(compute_activation_exit_epoch(self.cur()))
        q = max(exit_epochs)
        churn = sum(1 for v in self.v if v["exit_epoch"] == q)
        if churn >= churn_limit(self.st, len(self.active_indices(self.cur()))):
            q = (q + 1) & U64
        self.v[i]["exit_epoch"] = q
        wd = q + MIN_VALIDATOR_WITHDRAWABILITY_DELAY
        if wd > U64:
            raise Refused("limit", "initiate_validator_exit: withdrawable_epoch overflows")
        self.v[i]["withdrawable_epoch"] = wd

    def registry_updates(self):
        cur = self.cur()
        fin = int.from_bytes(self.st.fixed["finalized_checkpoint"][:8], "little")
        for i, v in enumerate(self.v):
            if v["activation_eligibility_epoch"] == FAR and v["effective_balance"] == MAX_EFFECTIVE_BALANCE:
                v["activation_eligibility_epoch"] = (cur + 1) & U64
            if self.is_active(v, cur) and v["effective_balance"] <= EJECTION_BALANCE:
                self.initiate_validator_exit(i)
        queue = [i for i, v in enumerate(self.v) if v["activation_eligibility_epoch"] <= fin and v["activation_epoch"] == FAR]
        queue.sort(key=lambda i: (self.v[i]["activation_eligibility_epoch"], i))
        P = PRESET[self.st.preset]
        limit = min(P["MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT"], churn_limit(self.st, len(self.active_indices(cur))))
        for i in queue[:limit]:
            self.v[i]["activation_epoch"] = compute_activation_exit_epoch(cur)

    def slashings(self):
        P = PRESET[self.st.preset]
        epoch = self.cur()
        total = self.get_total_active_balance()
        s = 0
        for x in self.st.slashings:
            s = (s + int(x)) & U64
        adjusted = min((s * PROPORTIONAL_SLASHING_MULTIPLIER_BELLATRIX) & U64, total)
        for i, v in enumerate(self.v):
            if v["slashed"] and epoch + P["EPOCHS_PER_SLASHINGS_VECTOR"] // 2 == v["withdrawable_epoch"]:
                num = (v["effective_balance"] // INC * adjusted) & U64
                self.decrease(i, (num // total * INC) & U64)

    def effective_balance_updates(self):
        h = INC // HYSTERESIS_QUOTIENT
        down, up = h * HYSTERESIS_DOWNWARD_MULTIPLIER, h * HYSTERESIS_UPWARD_MULTIPLIER
        for i, v in enumerate(self.v):
            b = self.bal[i]
            if (b + down) & U64 < v["effective_balance"] or (v["effective_balance"] + up) & U64 < b:
                v["effective_balance"] = min(b - b % INC, MAX_EFFECTIVE_BALANCE)


# ---- the vectorised formulation ----
class _Vector:
    def __init__(self, st):
        self.st = st

    def _cols(self):
        v = self.st.validators
        return (v["effective_balance"].astype(np.uint64), v["slashed"] != 0, v["activation_epoch"].astype(np.uint64),
                v["exit_epoch"].astype(np.uint64), v["withdrawable_epoch"].astype(np.uint64))

    def cur(self):
        return current_epoch(self.st)

    def prev(self):
        c = self.cur()
        return c - 1 if c else 0

    def active(self, epoch):
        _, _, act, exit_, _ = self._cols()
        return (act <= np.uint64(epoch)) & (np.uint64(epoch) < exit_)

    @staticmethod
    def total(eb, m):
        s = int(eb[m].astype(object).sum()) if m.any() else 0
        if s > U64:
            raise Refused("limit", "get_total_balance: checked_add overflow")
        return max(s, INC)

    def participating(self, flag, epoch):
        part = self.st.current_epoch_participation if epoch == self.cur() else self.st.previous_epoch_participation
        _, slashed, _, _, _ = self._cols()
        return self.active(epoch) & ~slashed & (((part >> flag) & 1) != 0)

    def total_active(self):
        return self.total(self._cols()[0], self.active(self.cur()))

    def eligible(self):
        _, slashed, _, _, wd = self._cols()
        prev = self.prev()
        return self.active(prev) | (slashed & (np.uint64(prev + 1) < wd))

    def justification_and_finalization(self):
        cur = self.cur()
        if cur <= 1:
            return
        eb = self._cols()[0]
        prev_t = self.total(eb, self.participating(TIMELY_TARGET_FLAG_INDEX, self.prev()))
        cur_t = self.total(eb, self.participating(TIMELY_TARGET_FLAG_INDEX, cur))
        weigh_justification_and_finalization(self.st, self.total_active(), prev_t, cur_t)

    def inactivity_updates(self):
        if self.cur() == 0:
            return
        el = self.eligible()
        tgt = self.participating(TIMELY_TARGET_FLAG_INDEX, self.prev())
        s = self.st.inactivity_scores.astype(np.uint64)
        with np.errstate(over="ignore"):
            s = np.where(el & tgt, s - np.minimum(s, np.uint64(1)), np.where(el, s + np.uint64(INACTIVITY_SCORE_BIAS), s))
        if not is_in_inactivity_leak(self.st):
            s = np.where(el, s - np.minimum(s, np.uint64(INACTIVITY_SCORE_RECOVERY_RATE)), s)
        self.st.inactivity_scores = s.astype("<u8")

    def rewards_and_penalties(self):
        if self.cur() == 0:
            return
        eb = self._cols()[0]
        el = self.eligible()
        total = self.total_active()
        active_inc = total // INC
        bpi = np.uint64(INC * BASE_REWARD_FACTOR // integer_sqrt(total))
        leak = is_in_inactivity_leak(self.st)
        bal = self.st.balances.astype(np.uint64)
        zero = np.zeros_like(bal)
        with np.errstate(over="ignore"):
            base = eb // np.uint64(INC) * bpi
            pairs = []
            for f in range(3):
                part = self.participating(f, self.prev())
                inc = np.uint64(self.total(eb, part) // INC)
                w = np.uint64(PARTICIPATION_FLAG_WEIGHTS[f])
                rew = np.where(el & part & (not leak), base * w * inc // np.uint64(active_inc * WEIGHT_DENOMINATOR), zero)
                pen = np.where(el & ~part, base * w // np.uint64(WEIGHT_DENOMINATOR), zero) if f != TIMELY_HEAD_FLAG_INDEX else zero
                pairs.append((rew, pen))
            tgt = self.participating(TIMELY_TARGET_FLAG_INDEX, self.prev())
            s = self.st.inactivity_scores.astype(np.uint64)
            pairs.append((zero, np.where(el & ~tgt, eb * s // np.uint64(INACTIVITY_SCORE_BIAS * INACTIVITY_PENALTY_QUOTIENT_BELLATRIX), zero)))
            for rew, pen in pairs:
                bal = bal + rew
                bal = np.where(pen > bal, zero, bal - np.minimum(pen, bal))
        self.st.balances = bal.astype("<u8")

    def exit_queue(self):
        """(E0, c0, L) of the closed form."""
        _, _, _, exit_, _ = self._cols()
        cur = self.cur()
        e0 = compute_activation_exit_epoch(cur)
        real = exit_[exit_ != np.uint64(FAR)]
        if real.size:
            e0 = max(e0, int(real.max()))
        c0 = int((exit_ == np.uint64(e0)).sum())
        return e0, c0, churn_limit(self.st, int(self.active(cur).sum()))

    def registry_updates(self):
        v = self.st.validators
        cur = self.cur()
        eb, _, act, exit_, _ = self._cols()
        elig = v["activation_eligibility_epoch"].astype(np.uint64)
        elig = np.where((elig == np.uint64(FAR)) & (eb == np.uint64(MAX_EFFECTIVE_BALANCE)), np.uint64((cur + 1) & U64), elig)
        e0, c0, L = self.exit_queue()
        ej = np.nonzero(self.active(cur) & (eb <= np.uint64(EJECTION_BALANCE)) & (exit_ == np.uint64(FAR)))[0]
        k = np.arange(ej.size, dtype=object)
        epochs = [e0 + (c0 + int(x)) // L if c0 < L else e0 + 1 + int(x) // L for x in k]
        if epochs and epochs[-1] + MIN_VALIDATOR_WITHDRAWABILITY_DELAY > U64:
            raise Refused("limit", "initiate_validator_exit: withdrawable_epoch overflows")
        new_exit = exit_.copy()
        new_wd = v["withdrawable_epoch"].astype(np.uint64)
        if ej.size:
            ep = np.array(epochs, dtype=np.uint64)
            new_exit[ej] = ep
            new_wd[ej] = ep + np.uint64(MIN_VALIDATOR_WITHDRAWABILITY_DELAY)
        fin = int.from_bytes(self.st.fixed["finalized_checkpoint"][:8], "little")
        cand = np.nonzero((elig <= np.uint64(fin)) & (act == np.uint64(FAR)))[0]
        order = cand[np.lexsort((cand, elig[cand]))]
        limit = min(PRESET[self.st.preset]["MAX_PER_EPOCH_ACTIVATION_CHURN_LIMIT"], L)
        new_act = act.copy()
        new_act[order[:limit]] = np.uint64(compute_activation_exit_epoch(cur))
        v["activation_eligibility_epoch"] = elig
        v["exit_epoch"] = new_exit
        v["withdrawable_epoch"] = new_wd
        v["activation_epoch"] = new_act

    def slashings(self):
        P = PRESET[self.st.preset]
        eb, slashed, _, _, wd = self._cols()
        total = self.total_active()
        s = int(self.st.slashings.astype(object).sum()) & U64
        adjusted = min((s * PROPORTIONAL_SLASHING_MULTIPLIER_BELLATRIX) & U64, total)
        hit = slashed & (wd == np.uint64(self.cur() + P["EPOCHS_PER_SLASHINGS_VECTOR"] // 2))
        bal = self.st.balances.astype(np.uint64)
        with np.errstate(over="ignore"):
            pen = eb // np.uint64(INC) * np.uint64(adjusted) // np.uint64(total) * np.uint64(INC)
        self.st.balances = np.where(hit, np.where(pen > bal, np.uint64(0), bal - np.minimum(pen, bal)), bal).astype("<u8")

    def effective_balance_updates(self):
        h = INC // HYSTERESIS_QUOTIENT
        eb = self._cols()[0]
        b = self.st.balances.astype(np.uint64)
        with np.errstate(over="ignore"):
            move = (b + np.uint64(h * HYSTERESIS_DOWNWARD_MULTIPLIER) < eb) | (eb + np.uint64(h * HYSTERESIS_UPWARD_MULTIPLIER) < b)
        new = np.minimum(b - b % np.uint64(INC), np.uint64(MAX_EFFECTIVE_BALANCE))
        self.st.validators["effective_balance"] = np.where(move, new, eb)


# ---- the small fields (shared) ----
def eth1_data_reset(st):
    if (current_epoch(st) + 1) % PRESET[st.preset]["EPOCHS_PER_ETH1_VOTING_PERIOD"] == 0:
        st.eth1_data_votes = st.eth1_data_votes[:0].copy()


def slashings_reset(st):
    st.slashings[(current_epoch(st) + 1) % PRESET[st.preset]["EPOCHS_PER_SLASHINGS_VECTOR"]] = 0


def randao_mixes_reset(st):
    ephv = PRESET[st.preset]["EPOCHS_PER_HISTORICAL_VECTOR"]
    cur = current_epoch(st)
    st.randao_mixes[(cur + 1) % ephv] = st.randao_mixes[cur % ephv]


def historical_summaries_update(st):
    P = PRESET[st.preset]
    if (current_epoch(st) + 1) % (P["SLOTS_PER_HISTORICAL_ROOT"] // P["SLOTS_PER_EPOCH"]) == 0:
        if len(st.historical_summaries) + 1 > HISTORICAL_ROOTS_LIMIT:
            raise Refused("limit", "historical_summaries is full")
        sphr = P["SLOTS_PER_HISTORICAL_ROOT"]
        summary = so.merkleize_bytes(st.block_roots.tobytes(), sphr) + so.merkleize_bytes(st.state_roots.tobytes(), sphr)
        st.historical_summaries = np.concatenate([st.historical_summaries, np.frombuffer(summary, np.uint8).reshape(1, 64)])


def participation_flag_updates(st):
    st.previous_epoch_participation = st.current_epoch_participation.copy()
    st.current_epoch_participation = np.zeros(len(st.validators), np.uint8)


def sync_committee_due(st) -> bool:
    return (current_epoch(st) + 1) % PRESET[st.preset]["EPOCHS_PER_SYNC_COMMITTEE_PERIOD"] == 0


def process_epoch(st: S.SynthState, steps=ALL, formulation: str = "vector", aggregate=None):
    """-> (post-state, aggregation code).  `st` is not changed; Refused is raised where the library refuses.
    `aggregate(keys) -> (code, 48 bytes | None)` is eth_aggregate_public_keys (default: bls_oracle's)."""
    m = mask(steps)
    if m & ~ALL:
        raise Refused("bad_arg", "mask bit above bit 11")
    n = len(st.validators)
    if any(len(x) != n for x in (st.balances, st.previous_epoch_participation, st.current_epoch_participation,
                                 st.inactivity_scores)):
        raise Refused("bad_arg", "the five big lists differ in length")
    out = clone(st)
    impl = {"literal": _Literal, "vector": _Vector}[formulation](out)
    for name in ("justification_and_finalization", "inactivity_updates", "rewards_and_penalties", "registry_updates",
                 "slashings"):
        if m & STEP[name]:
            getattr(impl, name)()
    if m & STEP["effective_balance_updates"] and formulation == "literal":
        impl.effective_balance_updates()
    if formulation == "literal":
        impl.write_back()
    if m & STEP["eth1_data_reset"]:
        eth1_data_reset(out)
    if m & STEP["effective_balance_updates"] and formulation == "vector":
        impl.effective_balance_updates()
    if m & STEP["slashings_reset"]:
        slashings_reset(out)
    if m & STEP["randao_mixes_reset"]:
        randao_mixes_reset(out)
    if m & STEP["historical_summaries_update"]:
        historical_summaries_update(out)
    if m & STEP["participation_flag_updates"]:
        participation_flag_updates(out)
    code = 0
    if m & STEP["sync_committee_updates"] and sync_committee_due(out):
        try:
            _, code, rotated = do.process_sync_committee_updates(out, aggregate)
        except do.NoActiveValidator:
            raise Refused("bad_arg", "no active validator for the next sync committee")
        if not code:
            out = rotated
    return out, code
