"""Seeded states and attestation batches that put the beacon-committee kernels of csrc/shuffle.cu and the host step of
b200_state_attesting_indices on their launch edges: `k_attesting_indices`' 256-bit gather chunks and warp ballots, its
power-of-two bitonic sort up to 2 048 entries, committees one member past MAX_VALIDATORS_PER_COMMITTEE,
`k_attester_duties`' committee cuts and launch tails, a batch of exactly 2^20 attestations, and the four-entry committee
cache.  Shared by test_committee_grid_cases.py (CPU: every case sits on the edge it claims, by the oracle) and
test_committee_grid_gpu.py (the device against the oracle, with launch counts)."""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass, field

import numpy as np

from ethereum_consensus_b200 import state as S
from oracle import duties_oracle as do
from tests import committee_cases as cc
from tests import committee_oracle as co

E = cc.EPOCH
ATT_THREADS = 256          # k_attesting_indices: one CTA of 256 threads per attestation, the gather in chunks of 256 bits
WARP = 32
ROW_THREADS = 256          # k_attester_duties / k_committee_positions: one thread per row / position
MAX_BITS = 2048            # MAX_VALIDATORS_PER_COMMITTEE, kMaxCommitteeBits
MAX_ATTESTATIONS = 1 << 20
MISS = 3 + 2               # an epoch not cached: active-set count, scan and scatter, then the shuffle's sources and map
DEAD_EXIT = 10             # exit epoch of the inactive validators at the ends of the index range
FAILS = (co.INVALID_TARGET_EPOCH, co.INVALID_SLOT, co.NO_DELAY, co.INVALID_INDEX, co.BITFIELD, co.INDICES_EMPTY,
         co.MALFORMED_BITS)


def grid_state(n_active: int, preset: str = "minimal", seed: int = 1, dead: int = 4, slot_in_epoch: int | None = None):
    """n_active validators active at every epoch near E, and `dead` more (half at the front of the index range, half at
    the back) that exited at epoch 10.  Slot: the last slot of E + 1 by default, so every slot of E (previous) and all
    but the last of E + 1 (current) are attestable, and the last one is NO_DELAY."""
    spe = do.PRESET[preset]["SLOTS_PER_EPOCH"]
    st = cc.state(n_active + dead, preset, seed=seed, edges=False,
                  slot_in_epoch=2 * spe - 1 if slot_in_epoch is None else slot_in_epoch)
    v = st.validators
    front = dead // 2
    v["exit_epoch"][:front] = DEAD_EXIT
    v["exit_epoch"][len(v) - (dead - front):] = DEAD_EXIT
    return st


def sort_size(n: int) -> int:
    """The bitonic sort's padded size: the least power of two >= n (1 for n <= 1)."""
    s = 1
    while s < n:
        s <<= 1
    return s


def chunk_lane(i: int):
    """(256-bit gather chunk, warp in the CTA, lane) of committee position i."""
    return i // ATT_THREADS, (i % ATT_THREADS) // WARP, i % WARP


@dataclass
class Att:
    data: bytes
    bits: bytes
    code: int              # the intended code
    tag: str               # the pattern (or failure) it was built for
    length: int = -1       # the committee's length (for attestations that reach the committee)
    epoch: int = -1


@dataclass
class GatherCase:
    name: str
    st: S.SynthState
    lengths: tuple         # the committee lengths the state holds
    attestations: list = field(default_factory=list)


def _bits_of(length: int, on) -> list:
    b = [False] * length
    for i in on:
        b[int(i)] = True
    return b


def patterns(length: int, rng) -> list:
    """(tag, bools) Bitlists of one committee length: every gather chunk and sort-size edge that length reaches."""
    out = [("all", [True] * length), ("bit0", _bits_of(length, [0])), ("last", _bits_of(length, [length - 1]))]
    if length > 256:
        out.append(("cut255_256", _bits_of(length, [255, 256])))
    edges = [i for i in range(length) if i % WARP == WARP - 1 or (i % WARP == 0 and i)]
    if edges:
        out.append(("warp_31_32", _bits_of(length, edges)))
    drop = int(rng.integers(0, length))
    out.append(("all_but_one", [i != drop for i in range(length)]))
    k = 0
    while (1 << k) + 1 <= length:
        for c in ((1 << k), (1 << k) + 1):
            out.append((f"count{c}", _bits_of(length, rng.choice(length, c, replace=False))))
        k += 1
    for d in (0.5, 0.99):
        b = list(rng.random(length) < d)
        if not any(b):
            b[0] = True
        out.append((f"density{d}", b))
    return out


def _epoch_views(st):
    spe = co.spe(st)
    slot = do.slot(st)
    cur = slot // spe
    views = {}
    for e in (cur - 1, cur):
        committees = co.beacon_committees(st, e)
        cps = len(committees) // spe
        ks = [k for k in range(len(committees)) if e * spe + k // cps + 1 <= slot]
        views[e] = (committees, cps, ks)
    return views, cur


def _att(st, views, e, k, bits, code, tag) -> Att:
    committees, cps, _ = views[e]
    s = e * co.spe(st) + k // cps
    return Att(co.attestation_data(s, k % cps, e), co.bitlist(bits), code, tag, len(committees[k]), e)


def failures(st, views, cur, rng) -> dict:
    """One attestation of every failure code against `st` (the state's slot is the last of `cur`)."""
    spe = co.spe(st)
    slot = do.slot(st)
    prev = cur - 1
    committees, cps, ks = views[prev]
    k = int(rng.choice(ks))
    L = len(committees[k])
    d = co.attestation_data(prev * spe + k // cps, k % cps, prev)
    return {
        co.MALFORMED_BITS: Att(d, co.bitlist([True] * L) + b"\x00", co.MALFORMED_BITS, "fail_malformed"),
        co.INVALID_TARGET_EPOCH: Att(co.attestation_data((cur + 1) * spe, 0, cur + 1), co.bitlist([True] * L),
                                     co.INVALID_TARGET_EPOCH, "fail_target"),
        co.INVALID_SLOT: Att(co.attestation_data(prev * spe + 1, 0, cur), co.bitlist([True] * L), co.INVALID_SLOT, "fail_slot"),
        co.NO_DELAY: Att(co.attestation_data(slot, 0, cur), co.bitlist([True] * L), co.NO_DELAY, "fail_no_delay"),
        co.INVALID_INDEX: Att(co.attestation_data(prev * spe, cps, prev), co.bitlist([True] * L), co.INVALID_INDEX, "fail_index"),
        # one bit too many, or one too few where L + 1 bits would not decode
        co.BITFIELD: Att(d, co.bitlist([True] * (L + 1 if L < MAX_BITS else L - 1)), co.BITFIELD, "fail_bitfield", L, prev),
        co.INDICES_EMPTY: Att(d, co.bitlist([False] * L), co.INDICES_EMPTY, "fail_empty", L, prev),
    }


def interleave(ok: list, fails: dict) -> list:
    """`ok` with one failure of every code spread through it: MALFORMED_BITS first, INDICES_EMPTY last, two failures next
    to each other in the middle, the others between passing attestations."""
    mid = [fails[c] for c in (co.INVALID_TARGET_EPOCH, co.INVALID_SLOT, co.NO_DELAY, co.INVALID_INDEX, co.BITFIELD)]
    out = [fails[co.MALFORMED_BITS]]
    step = max(1, len(ok) // (len(mid) + 1))
    j = 0
    for i, a in enumerate(ok):
        out.append(a)
        if j < len(mid) and (i + 1) % step == 0:
            out.append(mid[j])
            j += 1
            if j == 2:                     # the middle pair: two failures in a row
                out.append(mid[j])
                j += 1
    out.extend(mid[j:])
    out.append(fails[co.INDICES_EMPTY])
    return out


def gather_cases() -> list:
    """Minimal preset, n = 32 L + 16 for L in {31, 255, 511, 1023, 2047} (committees of L and L + 1 members), and
    n = 32 x 2048 (every committee 2 048); each length attested with every pattern, alternating the previous and the
    current epoch, in one batch with one failure of every code."""
    out = []
    for j, (name, n) in enumerate([(f"L{L}", 32 * L + 16) for L in (31, 255, 511, 1023, 2047)] + [("L2048", 32 * 2048)]):
        st = grid_state(n, "minimal", seed=700 + j)
        rng = np.random.default_rng(700 + j)
        views, cur = _epoch_views(st)
        lengths = sorted({len(views[cur - 1][0][k]) for k in views[cur - 1][2]})
        ok = []
        for length in lengths:
            for p, (tag, bits) in enumerate(patterns(length, rng)):
                e = cur - 1 if p % 2 == 0 else cur
                committees, cps, ks = views[e]
                k = int(rng.choice([k for k in ks if len(committees[k]) == length]))
                ok.append(_att(st, views, e, k, bits, co.OK, tag))
        out.append(GatherCase(f"gather_{name}", st, tuple(lengths), interleave(ok, failures(st, views, cur, rng))))
    return out


def over_limit_cases() -> list:
    """n = 32 x 2048 + 1 (committee 31 of each epoch has 2 049 members) and 32 x 2049 (every committee 2 049): a
    2 048-bit Bitlist on a 2 049-member committee (BITFIELD) and a 2 049-bit one (MALFORMED_BITS), in every epoch where
    such a committee is attestable."""
    out = []
    for j, (name, n) in enumerate((("over_one", 32 * 2048 + 1), ("over_all", 32 * 2049))):
        st = grid_state(n, "minimal", seed=800 + j)
        views, cur = _epoch_views(st)
        rng = np.random.default_rng(800 + j)
        atts = []
        for e in (cur - 1, cur):
            committees, cps, ks = views[e]
            over = [k for k in ks if len(committees[k]) == 2049]
            if not over:                   # over_one: committee 31 is the last slot's, which is not yet attestable in E + 1
                continue
            k = int(rng.choice(over))
            atts.append(_att(st, views, e, k, [True] * 2048, co.BITFIELD, "bits2048"))
            atts.append(_att(st, views, e, k, [True] * 2049, co.MALFORMED_BITS, "bits2049"))
        out.append(GatherCase(f"{name}", st, (2048, 2049) if n % 32 else (2049,), atts))
    return out


def over_one_ok(case: GatherCase) -> Att:
    """A full 2 048-member committee of `case` (over_one), attested with every bit."""
    views, cur = _epoch_views(case.st)
    committees, cps, ks = views[cur - 1]
    k = next(k for k in ks if len(committees[k]) == 2048)
    return _att(case.st, views, cur - 1, k, [True] * 2048, co.OK, "all")


@dataclass
class DutyCase:
    name: str
    st: S.SynthState
    C: int                 # committees per epoch
    lists: dict            # rows -> uint64 validator list (repeats, inactive validators, N - 1)


def duty_cases() -> list:
    """Both presets with n_active = 0, 1, C - 1 (mod C) and n_active < C; the inactive count makes N = 0, 1 or 255
    (mod 256), so the all-validator call's last CTA is full, holds one row, or misses one."""
    spec = [("minimal", 32 * 40, 0), ("minimal", 32 * 40 + 1, 1), ("minimal", 32 * 41 - 1, 255), ("minimal", 5, 0),
            ("mainnet", 8192, 255), ("mainnet", 8193, 0), ("mainnet", 8192 + 63, 1), ("mainnet", 20, 1)]
    out = []
    for j, (preset, n, r) in enumerate(spec):
        dead = (r - n) % 256
        dead += 256 if dead < 2 else 0
        st = grid_state(n, preset, seed=900 + j, dead=dead)
        N = len(st.validators)
        C = do.PRESET[preset]["SLOTS_PER_EPOCH"] * cc.expected_cps(preset, n)
        rng = np.random.default_rng(900 + j)
        lists = {}
        for rows in (1, 255, 256, 257):
            v = rng.integers(0, N, rows, dtype=np.uint64)
            v[0] = N - 1                       # inactive (back)
            if rows > 1:
                v[1] = 0                       # inactive (front)
                v[2] = N - 1                   # a repeat of an inactive one
                v[-1] = v[rows // 2]           # a repeat at the last row
                v[rows // 2 + 1:rows // 2 + 9] = v[rows // 2]
            lists[rows] = v
        out.append(DutyCase(f"{preset}_n{n}_N{N}", st, C, lists))
    return out


def appended(st, n_new: int, seed: int):
    """Validator records to append to `st` (copies of its own with new keys): a third active at E and E + 1, a third
    activating at E + 5 (not active at either), a third exiting at E + 1 (active at E only)."""
    rng = np.random.default_rng(seed)
    v = st.validators[rng.integers(0, len(st.validators), n_new)].copy()
    v["public_key"] = rng.integers(0, 256, (n_new, 48), dtype=np.uint8).view("V48").reshape(n_new)
    v["activation_epoch"] = 0
    v["exit_epoch"] = S.FAR_FUTURE_EPOCH
    v["activation_epoch"][1::3] = E + 5
    v["exit_epoch"][2::3] = E + 1
    return v, np.full(n_new, 32 * cc.ETH, np.uint64)


# ---- the 2^20-attestation batch ----
BOUND_L = 33               # minimal, n = 32 x 33: every committee 33 members, a 5-byte Bitlist


@dataclass
class BoundBatch:
    st: S.SynthState
    data: np.ndarray       # uint8[A, 128]
    bits: np.ndarray       # uint8[A, 5]
    codes: np.ndarray      # int32[A], the intended codes
    committee: np.ndarray  # int64[A]: row of `members` (passing and INDICES_EMPTY attestations), -1 for the others
    members: np.ndarray    # uint64[K, 33]: the attestable committees, committee order
    mask: np.ndarray       # bool[A, 33]: the Bitlist's bits


def bound_batch(n_att: int = MAX_ATTESTATIONS, seed: int = 1000) -> BoundBatch:
    """n_att attestations over the 60 attestable 33-member committees of E (previous) and E + 1 (current), random bits,
    every 4 099th Bitlist all zero, and every 65 537th attestation a failure (cycling BITFIELD, NO_DELAY, INVALID_INDEX,
    MALFORMED_BITS), the last one included."""
    st = grid_state(32 * BOUND_L, "minimal", seed=seed)
    views, cur = _epoch_views(st)
    spe = co.spe(st)
    keys = [(e, k) for e in (cur - 1, cur) for k in views[e][2]]
    members = np.array([views[e][0][k] for e, k in keys], np.uint64)
    rng = np.random.default_rng(seed)
    which = rng.integers(0, len(keys), n_att)
    mask = rng.random((n_att, BOUND_L)) < 0.5
    mask[::4099] = False
    ep = np.array([e for e, _ in keys], np.uint64)[which]
    kk = np.array([k for _, k in keys], np.uint64)[which]
    cps = 4
    data = np.zeros((n_att, 128), np.uint8)
    for col, vals in ((0, ep * spe + kk // cps), (8, kk % cps), (88, ep)):   # slot, index, target epoch
        data[:, col:col + 8] = vals.astype("<u8").view(np.uint8).reshape(-1, 8)
    # Bitlist of 33 bits: 4 bytes of bits, then byte 4 holds bit 32 and the delimiter (bit 1)
    packed = np.packbits(np.concatenate([mask, np.ones((n_att, 1), bool), np.zeros((n_att, 6), bool)], 1), axis=1,
                         bitorder="little")
    codes = np.where(mask.any(1), co.OK, co.INDICES_EMPTY).astype(np.int32)
    committee = which.astype(np.int64)
    fail = np.arange(n_att)[::65537].tolist() + [n_att - 1]
    for j, a in enumerate(fail):
        kind = (co.BITFIELD, co.NO_DELAY, co.INVALID_INDEX, co.MALFORMED_BITS)[j % 4]
        if kind == co.BITFIELD:            # 34 bits: the delimiter one bit higher, still 5 bytes
            packed[a, 4] = (packed[a, 4] & 1) | 4
        elif kind == co.NO_DELAY:
            data[a, 0:8] = np.frombuffer(int(do.slot(st)).to_bytes(8, "little"), np.uint8)
            data[a, 88:96] = np.frombuffer(int(cur).to_bytes(8, "little"), np.uint8)
        elif kind == co.INVALID_INDEX:
            data[a, 8:16] = np.frombuffer(int(cps).to_bytes(8, "little"), np.uint8)
        else:                              # no delimiter
            packed[a, 4] = 0
        codes[a] = kind
        committee[a] = -1
    return BoundBatch(st, data, packed, codes, committee, members, mask)


def bound_expected(b: BoundBatch):
    """-> (uint32 offsets, uint64 indices) of the batch, vectorised: each committee's members sorted once, each passing
    attestation's mask permuted into that order."""
    order = np.argsort(b.members, axis=1, kind="stable")
    sorted_members = np.take_along_axis(b.members, order, 1)
    ok = b.codes == co.OK
    rows = b.committee[ok]
    pmask = np.take_along_axis(b.mask[ok], order[rows], 1)
    idx = sorted_members[rows][pmask]
    counts = np.zeros(len(b.codes), np.int64)
    counts[ok] = pmask.sum(1)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    return off, idx


def some_attestations(st, seed: int, per_epoch: int = 3) -> list:
    """`per_epoch` passing attestations (random bits) on committees of both of `st`'s attestable epochs."""
    views, cur = _epoch_views(st)
    rng = np.random.default_rng(seed)
    out = []
    for e in (cur - 1, cur):
        committees, cps, ks = views[e]
        for k in rng.choice([k for k in ks if committees[k]], per_epoch, replace=False):
            bits = list(rng.random(len(committees[k])) < 0.5)
            bits[0] = True
            out.append(_att(st, views, e, int(k), bits, co.OK, "random"))
    return out


# ---- the committee cache ----
class LRU:
    """The per-handle committee cache as a launch-count model: four entries, least recently used evicted; an epoch not
    held costs MISS launches, an inverse map not built one more."""

    def __init__(self, size: int = 4):
        self.size = size
        self.entries = OrderedDict()        # epoch -> inverse map built

    def use(self, epoch: int, positions: bool = False) -> int:
        k = 0
        if epoch in self.entries:
            self.entries.move_to_end(epoch)
        else:
            if len(self.entries) == self.size:
                self.entries.popitem(last=False)
            self.entries[epoch] = False
            k += MISS
        if positions and not self.entries[epoch]:
            self.entries[epoch] = True
            k += 1
        return k

    def duties(self, epoch: int) -> int:
        return self.use(epoch, positions=True) + 1


LRU_WALK = [E - 1, E, E + 1, E + 2, E - 1, E + 3, E, E + 1, E + 4, E - 1, E + 2, E + 3, E + 3, E + 5, E - 1, E]
