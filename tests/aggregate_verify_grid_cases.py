"""aggregate_verify batches where the device splits them, shared by the CPU check (tests/test_aggregate_verify_grid_cases.py)
and the device run (tests/test_aggregate_verify_grid_gpu.py).  No device code here.

A batch of T tuples is laid out by the host (capi_bls.cu `stage_small`) as one run of Miller pairs: a tuple with a valid
shape (n > 0 keys and n messages) gets its n key pairs and then (-g1, signature), n + 1 pairs whatever its key and
signature codes; a tuple with another shape gets none.  `k_vm_miller` runs one team of 16 lanes (n_pairs <= vm_team16_max)
or 8 lanes per pair, so a warp holds 2 or 4 consecutive pairs; a pair of a failed tuple is dead and a pair with a point at
infinity is trivial (it writes Fp12 one without running the program), and a warp without a live non-trivial pair leaves
`vm_run` at once.  `plan_fold` then folds each tuple's values in levels of `k_fold_segments` (64-thread CTAs, 32-value
chunks, a segment in k chunks becomes k pieces) until every tuple is in at most two pieces, and plans no level when every
tuple already has two values or none; `k_vm_final` runs one team per tuple (16 lanes when T <= vm_team16_max).  `Layout`
restates all of this, so every case below names the edge it was built for and the CPU file checks that it lands there.

Valid tuples are closed forms over one shared message list: message j is msg(j mod PERIOD), H_j its hash, and tuple k of
size n has keys sk_j = a_n + k + j d (orc_pk_sequence) and signature (a_n + k) A_n + d B_n with A_n = sum_{j<n} H_j and
B_n = sum_{j<n} j H_j.  With period P, n = qP + r: A_n = q A_P + A_r and B_n = P q(q-1)/2 A_P + q B_P + qP A_r + B_r, and
B_r = (r - 1) A_r - C_r with C_r = sum_{1<=k<r} A_k, so one pass over the P hashes serves every size; consecutive k
differ by A_n, one G2 addition each.  Messages repeat past P (aggregate_verify does not ask for distinct messages).
Tuples that must fail take the next k's signature.  Dead tuples (an invalid key, a signature decode error, a signature
outside G2) and shape failures use keys of one pool; tuples whose signature pair is trivial use the infinity signature
over keys that cancel (pk, -pk or three keys summing to zero) on one repeated message, valid under the IETF
CoreAggregateVerify, which both oracles follow."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import re
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field
from functools import lru_cache
from pathlib import Path

from oracle import bls_oracle as bo
from tests import aggregate_batch_cases as ac
from tests import aggregate_grid_cases as gc
from tests import aggregate_verify_cases as av

R = bo.R
SUCCESS, BAD_ENCODING, NOT_ON_CURVE, NOT_IN_GROUP, VERIFY_FAIL, PK_IS_INFINITY = 0, 1, 2, 3, 5, 6
INF_SIG = ac.INF_SIG
PERIOD = 1024                       # distinct messages; message j is msg(j % PERIOD)
POOL = 2100                         # valid keys shared by dead tuples and shape failures
TEAM16_MAX = 2048                   # bls_vm.cu g_team16_max's default
VM_CTAS = (32, 64, 128)
TEAM16_MAXES = (0, TEAM16_MAX, 1 << 30)
CSRC = Path(__file__).resolve().parent.parent / "ethereum_consensus_b200" / "csrc"
THREADS = max(1, min(32, os.cpu_count() or 1))


# ------------------------------------------------------------------------------------------------ tuple specs
LIVE = ("valid", "fail", "triv2", "triv3", "inf1", "trivfail")
DEAD = ("badkey", "badsig", "noc", "nig")
TRIVIAL_LAST = ("triv2", "triv3", "inf1", "trivfail")   # infinity signature: the (-g1, sig) pair is trivial


@dataclass(frozen=True)
class Spec:
    """One tuple: kind, n keys, m messages (None: n).  `bad`: ((position, key code), ...) for "badkey"; k: which closed
    form of size n ("valid", "fail")."""
    kind: str
    n: int
    m: int = None
    bad: tuple = ()
    k: int = 0

    @property
    def msgs(self) -> int:
        return self.n if self.m is None else self.m

    @property
    def shape_ok(self) -> bool:
        return self.n > 0 and self.n == self.msgs

    @property
    def pairs(self) -> int:
        return self.n + 1 if self.shape_ok else 0

    @property
    def live(self) -> bool:
        return self.kind in LIVE and self.shape_ok

    @property
    def trivial_last(self) -> bool:
        return self.kind in TRIVIAL_LAST

    @property
    def want(self) -> int:
        if self.kind == "badkey":
            return min(self.bad)[1]
        if self.kind == "badsig":
            return BAD_ENCODING
        if self.kind == "noc":
            return NOT_ON_CURVE
        if self.kind in ("valid", "triv2", "triv3") and self.shape_ok:
            return SUCCESS
        return VERIFY_FAIL


def pad_spec(kind: str, pairs: int, j: int = 0) -> Spec:
    """A tuple of exactly `pairs` (>= 2) Miller pairs of the given kind; a "badkey" pad's invalid key rotates with j."""
    n = pairs - 1
    assert n >= 1
    if kind == "badkey":
        return Spec("badkey", n, bad=((j % n, KEY_CODES[j % 4]),))
    if kind in ("valid", "fail"):
        return Spec(kind, n, k=j)
    return Spec(kind, n)


KEY_CODES = (PK_IS_INFINITY, NOT_ON_CURVE, NOT_IN_GROUP, BAD_ENCODING)
DEAD_PADS = ("badkey", "badsig", "nig", "noc")


# ------------------------------------------------------------------------------------------------ layout model
def fold_plan(lengths):
    """plan_fold(skip_pairs = true): [] when every segment has 2 values or none, else av.fold_levels."""
    if all(L in (0, 2) for L in lengths):
        return []
    return av.fold_levels(lengths)


@lru_cache(maxsize=None)
def vm_slots():
    """(Miller, final) register-file slots of the 8- and 16-lane programs, read from pairing_vm_prog*.cuh."""
    def grab(path, name):
        return int(re.search(rf"constexpr int {name} = (\d+);", path.read_text()).group(1))
    p8, p16 = CSRC / "pairing_vm_prog.cuh", CSRC / "pairing_vm_prog16.cuh"
    return {8: (grab(p8, "kMillerSlots"), grab(p8, "kFinalSlots")), 16: (grab(p16, "kMillerSlots16"), grab(p16, "kFinalSlots16"))}


@lru_cache(maxsize=None)
def vm_smem_limits():
    """(kVmSlotWords, kVmMaxSmemBytes) from pairing_vm.cuh."""
    t = (CSRC / "pairing_vm.cuh").read_text()
    words = int(re.search(r"constexpr int kVmSlotWords = (\d+);", t).group(1))
    kb = int(re.search(r"constexpr int kVmMaxSmemBytes = (\d+) \* 1024;", t).group(1))
    return words, kb * 1024


def cta_threads(team: int, vm_cta: int, final: bool) -> int:
    """launch_vm_*_t: vm_cta threads, halved while the CTA's register files exceed kVmMaxSmemBytes."""
    slots = vm_slots()[team][1 if final else 0]
    words, limit = vm_smem_limits()
    threads = vm_cta
    while threads > 32 and (threads // team) * slots * words * 4 > limit:
        threads //= 2
    return threads


@dataclass
class Layout:
    """How one aggregate_verify batch call lays out its tuples, at the knobs (vm_cta, vm_team16_max)."""
    specs: list
    vm_cta: int = 32
    team16_max: int = TEAM16_MAX
    registry: bool = False

    def __post_init__(self):
        s = self.specs
        self.T = len(s)
        self.pairs = [x.pairs for x in s]
        self.poff = [0]
        for c in self.pairs:
            self.poff.append(self.poff[-1] + c)
        self.n_pairs = self.poff[-1]
        self.levels = fold_plan(self.pairs)
        self.miller_team = 16 if self.n_pairs <= self.team16_max else 8
        self.final_team = 16 if self.T <= self.team16_max else 8
        self.miller_threads = cta_threads(self.miller_team, self.vm_cta, False)
        self.final_threads = cta_threads(self.final_team, self.vm_cta, True)
        self.pair_tuple = [t for t, c in enumerate(self.pairs) for _ in range(c)]

    # level 0 = the Miller values; level k >= 1 = the pieces level k - 1 wrote
    def level_offsets(self, k: int):
        if k == 0:
            return list(self.poff)
        off = [0]
        for p in self.levels[k - 1][1]:
            off.append(off[-1] + p)
        return off

    def start_lane(self, t: int, level: int = 0) -> int:
        return self.level_offsets(level)[t] % 32

    def pieces(self, t: int):
        """Tuple t's pieces per level (the values it enters each level with at index 0, then what each level leaves)."""
        return [self.pairs[t]] + [lv[1][t] for lv in self.levels]

    def crosses_cta(self, t: int, level: int = 0) -> bool:
        """Does tuple t's segment cross a 64-value (k_fold_segments CTA) edge at this level?"""
        off = self.level_offsets(level)
        lo, hi = off[t], off[t + 1]
        return hi - lo >= 2 and (hi - 1) // 64 != lo // 64

    # Miller warps: 32 / team pairs each
    @property
    def miller_per_warp(self) -> int:
        return 32 // self.miller_team

    def pair_runs(self, i: int) -> bool:
        """Does pair i run the Miller program (a live tuple's pair without a point at infinity)?"""
        t = self.pair_tuple[i]
        sp = self.specs[t]
        return sp.live and not (sp.trivial_last and i == self.poff[t + 1] - 1)

    def pair_live(self, i: int) -> bool:
        return self.specs[self.pair_tuple[i]].live

    def miller_warps(self):
        """Per warp: (positions that run the program, positions of live pairs)."""
        w = self.miller_per_warp
        out = []
        for base in range(0, self.n_pairs, w):
            idx = range(base, min(base + w, self.n_pairs))
            out.append(({i - base for i in idx if self.pair_runs(i)}, {i - base for i in idx if self.pair_live(i)}))
        return out

    def miller_where(self, i: int):
        """Pair i -> (CTA, warp, team position in the warp)."""
        teams = self.miller_threads // self.miller_team
        return i // teams, i // self.miller_per_warp, i % self.miller_per_warp

    def miller_ctas(self):
        teams = self.miller_threads // self.miller_team
        return -(-self.n_pairs // teams)

    def last_miller_cta(self):
        """(pairs in the last Miller CTA, how many of them are live, CTA capacity in pairs)."""
        teams = self.miller_threads // self.miller_team
        lo = (self.miller_ctas() - 1) * teams
        return self.n_pairs - lo, sum(self.pair_live(i) for i in range(lo, self.n_pairs)), teams

    # final-exponentiation warps: 32 / team tuples each
    @property
    def final_per_warp(self) -> int:
        return 32 // self.final_team

    def final_warps(self):
        """Per warp: positions of live tuples."""
        w = self.final_per_warp
        return [{t - base for t in range(base, min(base + w, self.T)) if self.specs[t].live} for base in range(0, self.T, w)]

    @property
    def launches(self) -> int:
        """Launches per call: K1 (strict, keys), K3 (T > 0), K4's two (messages), K2, the pair operands (keys), the Miller
        launch (pairs), one per fold level with inputs, the final exponentiation (T > 0)."""
        n_keys = sum(x.n for x in self.specs)
        n_msgs = sum(x.msgs for x in self.specs)
        k = (0 if self.registry or not n_keys else 1) + (1 if self.T else 0) + (2 if n_msgs else 0) + 1
        k += (1 if n_keys else 0) + (1 if self.n_pairs else 0) + sum(1 for lv in self.levels if lv[0]) + (1 if self.T else 0)
        return k


def layout(case, vm_cta=32, team16_max=TEAM16_MAX, registry=False) -> Layout:
    return Layout(list(case.specs), vm_cta, team16_max, registry)


# ------------------------------------------------------------------------------------------------ cases
@dataclass
class Case:
    name: str
    section: str         # "align", "depth", "skip", "warps", "switch", "keys"
    specs: list
    claim: dict = field(default_factory=dict)


ALIGN_C = (2, 3, 31, 32, 33, 63, 64, 65, 1024, 1025, 2048, 2049)
ALIGN_LANES = (0, 1, 30, 31)
PAD_KINDS = ("badkey", "badsig", "nig", "valid")


def align_cases():
    """Pair count c at start lanes 0, 1, 30, 31, four targets per call: valid targets in one call, failing ones in another.
    Padding in front of each target rotates through dead-with-pairs kinds and valid tuples; from the third target on the
    target starts in an odd chunk, so that lanes 30 / 31 cross a 64-value CTA edge.  Shape failures sit in front of the
    second target and shift nothing."""
    out = []
    for ci, c in enumerate(ALIGN_C):
        for kind in ("valid", "fail"):
            specs, targets, lanes = [], [], {}
            for j, s in enumerate(ALIGN_LANES):
                pk = PAD_KINDS[(ci + j + (kind == "fail")) % 4]
                cur = sum(x.pairs for x in specs)
                p = (s - cur) % 32
                while p == 1 or (j >= 2 and ((cur + p) // 32) % 2 == 0):
                    p += 32
                if p:
                    specs.append(pad_spec(pk, p, j + ci))
                if j == 1:
                    specs += [Spec("valid", 3, m=2), Spec("valid", 0, m=0), Spec("badkey", 2, m=5, bad=((1, NOT_IN_GROUP),))]
                targets.append(len(specs))
                lanes[len(specs)] = s
                specs.append(Spec(kind, c - 1, k=j))
            specs.append(Spec("fail" if kind == "valid" else "valid", 1, k=7))
            out.append(Case(f"c={c} {kind} targets at lanes 0 1 30 31", "align", specs,
                            {"start": lanes, "c": c, "shape_before": targets[1]}))
    return out


def depth_bounds(prefix, L: int):
    """(smallest, largest) pair count c of a tuple behind `prefix` whose call plans exactly L levels (largest None when
    unbounded), by bisection on the level count (monotone in c)."""
    def lv(c):
        return len(fold_plan([x.pairs for x in prefix] + [c]))
    lo_c = 2
    if lv(lo_c) > L:
        return None
    def first_at_least(k):
        a, b = 2, 1 << 20
        while a < b:
            mid = (a + b) // 2
            if lv(mid) >= k:
                b = mid
            else:
                a = mid + 1
        return a
    cmin = first_at_least(L)
    if lv(cmin) != L:
        return None
    nxt = first_at_least(L + 1)
    return cmin, (nxt - 1 if lv(nxt) == L + 1 else None)


DEPTH_PREFIX = {0: [], 31: [Spec("badkey", 30, bad=((29, BAD_ENCODING),))]}


def depth_cases():
    """For 1 to 4 levels the smallest and largest pair count, at start lane 0 and behind a 31-pair dead tuple (lane 31),
    each followed by a failing and a dead short tuple that go through levels they do not need; plus 32 769 values at
    lane 0 (three levels)."""
    out = []
    for lane, prefix in DEPTH_PREFIX.items():
        for L in (1, 2, 3, 4):
            b = depth_bounds(prefix, L)
            for which, c in (("smallest", b[0]), ("largest", b[1])):
                if c is None:
                    continue
                specs = list(prefix) + [Spec("valid", c - 1), Spec("fail", 1, k=3), Spec("nig", 1)]
                out.append(Case(f"{L} levels, {which} c = {c} at lane {lane}", "depth", specs,
                                {"levels": L, "target": len(prefix), "lane": lane, "bound": which, "c": c}))
    out.append(Case("3 levels, c = 32 769 at lane 0", "depth", [Spec("valid", 32768), Spec("fail", 2, k=1), Spec("badsig", 1)],
                    {"levels": 3, "target": 0, "lane": 0, "c": 32769}))
    return out


def skip_cases():
    base = ([Spec("valid", 1, k=k) for k in range(5)] + [Spec("valid", 2, m=1), Spec("valid", 0, m=0), Spec("valid", 1, m=3)]
            + [Spec("fail", 1, k=5), Spec("fail", 1, k=6), Spec("badkey", 1, bad=((0, NOT_ON_CURVE),)), Spec("badsig", 1), Spec("nig", 1)])
    shapes = [Spec("valid", 0, m=0), Spec("valid", 2, m=1), Spec("valid", 1, m=0), Spec("badkey", 3, m=1, bad=((2, PK_IS_INFINITY),)),
              Spec("badsig", 0, m=2), Spec("nig", 2, m=3), Spec("noc", 1, m=2)]
    return [Case("n = 1 tuples and shape failures: no level", "skip", base, {"levels": 0}),
            Case("the same plus one n = 2 tuple: one level for every tuple", "skip", base + [Spec("valid", 2, k=1)], {"levels": 1}),
            Case("only shape failures: no Miller launch, no level", "skip", shapes, {"levels": 0, "n_pairs": 0})]


def _dead(pairs, j):
    return pad_spec(DEAD_PADS[j % 4], pairs, j)


def _fill_to(specs, index: int, j: int):
    """Dead tuples until the next pair index is `index` (which must be 0 or >= 2 pairs away)."""
    cur = sum(x.pairs for x in specs)
    gap = index - cur
    assert gap == 0 or gap >= 2, (cur, index)
    if gap:
        specs.append(_dead(gap, j))


def warp_cases():
    """Miller warps for each team size (w pairs per warp): exactly one pair that runs the program at every team position
    (the last pair of a live tuple at position 0, the first at w - 1, and between them the key pair of an n = 1 tuple
    with the infinity signature, whose trivial pair follows); a live tuple whose only pair in a warp is its trivial one
    (pk, -pk and three keys summing to zero, each SUCCESS); warps of dead pairs only at the front, in the middle and at the
    end, and a last CTA of dead pairs that is ragged at every vm_cta."""
    out = []
    for team in (8, 16):
        w = 32 // team
        specs, lone, trivial = [], {}, {}
        j = 0
        _fill_to(specs, 2 * w, j)                              # warps 0 and 1: dead
        for pos in range(w):
            j += 1
            base = sum(x.pairs for x in specs)
            wbase = -(-(base + 8) // w) * w + w                 # a warp well ahead
            if pos == 0:                                       # a live tuple ending at position 0
                sp = Spec("valid", 3, k=j)
                _fill_to(specs, wbase - 3, j)
                lone[wbase] = 0
            elif pos == w - 1:                                 # a live tuple starting at position w - 1
                sp = Spec("valid", 4, k=j)
                _fill_to(specs, wbase + w - 1, j)
                lone[wbase + w - 1] = w - 1
            else:                                              # key pair at pos, trivial pair at pos + 1
                sp = Spec("inf1", 1, k=j)
                _fill_to(specs, wbase + pos, j)
                lone[wbase + pos] = pos
            specs.append(sp)
            after = sum(x.pairs for x in specs)
            _fill_to(specs, -(-after // w) * w + w if after % w else after + w, j + 7)   # the rest of that warp and one more: dead
        for kind, n in (("triv2", 2), ("triv3", 3)):           # trivial pair alone at position 0 beside dead pairs
            j += 1
            base = sum(x.pairs for x in specs)
            wbase = -(-(base + 2 + n) // w) * w + w
            _fill_to(specs, wbase - n, j)
            specs.append(Spec(kind, n, k=j))
            trivial[wbase] = kind
            _fill_to(specs, wbase + w + w, j + 3)              # the rest of that warp and the next one: dead
        specs.append(Spec("valid", 2, k=9))                    # a live tuple in the middle of the run, then the dead end
        cur = sum(x.pairs for x in specs)
        end = -(-(cur + 2) // 128) * 128 + 128 + 5              # 5 past a multiple of 128: a ragged last CTA at every vm_cta
        _fill_to(specs, end, j + 11)
        out.append(Case(f"Miller warps of {team}-lane teams", "warps", specs,
                        {"team": team, "lone": lone, "trivial_alone": trivial, "dead_front": True, "dead_end": True}))
    # final-exponentiation warps: one live tuple at each team position, the others dead; whole warps of dead tuples
    for team in (8, 16):
        w = 32 // team
        specs, live_at = [], {}
        dead_kinds = [Spec("badkey", 2, bad=((1, NOT_ON_CURVE),)), Spec("badsig", 1), Spec("nig", 2), Spec("valid", 2, m=1),
                      Spec("noc", 3), Spec("badkey", 1, bad=((0, PK_IS_INFINITY),))]
        live_kinds = [Spec("valid", 1, k=20), Spec("triv2", 2, k=21), Spec("fail", 2, k=22), Spec("triv3", 3, k=23),
                      Spec("inf1", 1, k=24), Spec("trivfail", 2, k=25), Spec("valid", 3, k=26), Spec("fail", 1, k=27)]
        specs += [dead_kinds[i % 6] for i in range(w)]         # a dead warp at the front
        q = 0
        for rep in range(2):
            for pos in range(w):
                for i in range(w):
                    if i == pos:
                        live_at[len(specs)] = pos
                        specs.append(live_kinds[q % len(live_kinds)])
                        q += 1
                    else:
                        specs.append(dead_kinds[(q + i) % 6])
            if rep == 0:
                specs += [dead_kinds[(i + 1) % 6] for i in range(w)]   # a dead warp in the middle
        specs += [dead_kinds[(i + 2) % 6] for i in range(w + 1)]     # a dead warp at the end, and one tuple more
        out.append(Case(f"final warps of {team}-lane teams", "warps", specs, {"final_team": team, "final_lone": live_at}))
    return out


def switch_cases():
    """Team-size switches: n_pairs = 2 048 | 2 049 (Miller), T = 2 048 | 2 049 (final), and T = 2 049 tuples of mostly
    shape failures with fewer than 2 048 pairs (16-lane Miller teams, 8-lane final teams)."""
    out = []
    for n_pairs in (2048, 2049):
        specs = [Spec("valid", 999, k=0), Spec("fail", 499, k=0), Spec("triv2", 2, k=1), Spec("valid", 0, m=2)]
        specs += [Spec("valid", 1, k=k) for k in range(40)]
        cur = sum(x.pairs for x in specs)
        specs.append(_dead(n_pairs - cur - 31, 1))
        specs.append(Spec("valid", 30, k=1))
        out.append(Case(f"n_pairs = {n_pairs}", "switch", specs, {"n_pairs": n_pairs, "miller_team": 16 if n_pairs <= 2048 else 8}))
    for T in (2048, 2049):
        specs = []
        for t in range(T):
            r = t % 16
            specs.append(Spec("fail", 1, k=t) if r == 5 else _dead(2, t) if r == 9 else Spec("valid", 0, m=1) if r == 12
                         else Spec("valid", 1, k=t))
        out.append(Case(f"T = {T}", "switch", specs, {"T": T, "final_team": 16 if T <= 2048 else 8}))
    specs = []
    for t in range(2049):
        r = t % 16
        specs.append(Spec("valid", 1, k=t) if r == 0 else Spec("fail", 1, k=t) if r == 7 else _dead(3, t) if r == 11
                     else Spec("valid", t % 3, m=(t % 3) + 1))
    out.append(Case("T = 2 049, mostly shape failures", "switch", specs, {"T": 2049, "miller_team": 16, "final_team": 8}))
    return out


def key_scan_cases():
    """k_g1_aggregate's code-only scan (lane l reads keys l, l + 32, ..): tuples of 33 or more keys whose first invalid key
    is on a lane's second or third pass, and two invalid keys of different codes on one lane in every order, between live
    tuples and shape failures."""
    specs, firsts = [], {}
    def add(n, bad):
        firsts[len(specs)] = min(bad)[0]
        specs.append(Spec("badkey", n, bad=tuple(bad)))
    add(33, [(32, NOT_IN_GROUP)])
    add(41, [(40, BAD_ENCODING)])
    add(70, [(33, NOT_ON_CURVE), (66, PK_IS_INFINITY)])
    add(100, [(70, PK_IS_INFINITY), (71, BAD_ENCODING)])
    specs.append(Spec("valid", 33, k=1))
    specs.append(Spec("valid", 1, m=2))
    for p, gap in ((5, 32), (31, 32), (0, 64)):
        for c1 in KEY_CODES:
            for c2 in KEY_CODES:
                if c1 != c2:
                    add(p + gap + 3, [(p, c1), (p + gap, c2)])
        specs.append(Spec("fail", 40, k=p))
        specs.append(Spec("valid", 34, m=33))
    specs.append(Spec("badkey", 40, m=39, bad=((35, NOT_IN_GROUP),)))   # shape failure behind an invalid key: its code
    return [Case("key scan on later passes", "keys", specs, {"first_bad": firsts})]


@lru_cache(maxsize=None)
def all_cases():
    return align_cases() + depth_cases() + skip_cases() + warp_cases() + switch_cases() + key_scan_cases()


def poison(case) -> Case:
    """The same layout with every tuple valid: after it the device buffers hold passing Miller values, passing fold pieces
    and SUCCESS codes at every index the case uses (a shape failure's slot becomes an n = 1 tuple).  When that changes the
    parity of the level count, one more valid tuple behind them adds a level, so that the final level writes the buffer
    the case's final level reads."""
    specs = [Spec("valid", x.n if x.shape_ok else 1) for x in case.specs]
    want = len(fold_plan([x.pairs for x in case.specs])) % 2
    for c in (0, 65, 2049, 65537):
        extra = [Spec("valid", c - 1)] if c else []
        if len(fold_plan([x.pairs for x in specs + extra])) % 2 == want:
            return Case("poison for " + case.name, case.section, specs + extra)
    raise AssertionError(case.name)


# ------------------------------------------------------------------------------------------------ material
_O = None


def bind(O):
    global _O
    _O = av.bind(O)
    return _O


def _pool_map(fn, items):
    with ThreadPoolExecutor(THREADS) as ex:
        return list(ex.map(fn, items))


def msg(j: int) -> bytes:
    return hashlib.sha256(b"av grid msg %d" % (j % PERIOD)).digest()


@lru_cache(maxsize=None)
def msgs(n: int):
    return [msg(j) for j in range(n)]


@lru_cache(maxsize=None)
def _prefix():
    """A_r and C_r for r <= PERIOD (one pass over the hashes)."""
    hs = _pool_map(lambda j: av._h2g2(_O, msg(j)), range(PERIOD))
    A, Cs = [None], [None]
    for r in range(1, PERIOD + 1):
        A.append(ac.G2.add(A[-1], hs[r - 1]))
        Cs.append(ac.G2.add(Cs[-1], A[r - 1]) if r >= 2 else None)
    return A, Cs


def _lin(*terms):
    acc = None
    for k, pt in terms:
        if pt is not None and k % R:
            acc = ac.G2.add(acc, ac.G2.mul(pt, k))
    return acc


def size_params(n: int):
    return 1 + av._sk(b"av grid a %d" % n) % (R // 2), 1 + av._sk(b"av grid d %d" % n) % 1000


@lru_cache(maxsize=None)
def _A_sig0(n: int):
    """(A_n, signature of k = 0) of size n (module docstring)."""
    A, Cs = _prefix()
    P = PERIOD
    q, r = divmod(n, P)
    a, d = size_params(n)
    An = _lin((q, A[P]), (1, A[r]))
    # sig = a A_n + d B_n,  B_n = P q(q-1)/2 A_P + q B_P + qP A_r + B_r,  B_x = (x - 1) A_x - C_x
    coef_AP = a * q + d * (P * q * (q - 1) // 2 + q * (P - 1))
    coef_Ar = a + d * (q * P + (r - 1 if r else 0))
    sig = _lin((coef_AP, A[P]), (-d * q, Cs[P]), (coef_Ar, A[r]), (-d, Cs[r] if r else None))
    return An, sig


_sigs = {}


def valid_sig(n: int, k: int):
    """The closed-form signature point of tuple k of size n (consecutive k: one addition each)."""
    lst = _sigs.setdefault(n, [])
    if not lst:
        lst.append(_A_sig0(n)[1])
    while len(lst) <= k:
        lst.append(ac.G2.add(lst[-1], _A_sig0(n)[0]))
    return lst[k]


@lru_cache(maxsize=None)
def valid_keys(n: int, k: int):
    a, d = size_params(n)
    out = C.create_string_buffer(48 * n)
    _O.orc_pk_sequence(av._b32(a + k), av._b32(d), n, out)
    raw = out.raw
    return tuple(raw[48 * j:48 * j + 48] for j in range(n))


@lru_cache(maxsize=None)
def key_pool():
    out = C.create_string_buffer(48 * POOL)
    _O.orc_pk_sequence(av._b32(av._sk(b"av grid pool")), av._b32(3), POOL, out)
    raw = out.raw
    return tuple(raw[48 * j:48 * j + 48] for j in range(POOL))


@lru_cache(maxsize=None)
def bad_material():
    """Invalid key encodings by code, and invalid signatures: a bad encoding, one off the curve, one outside G2."""
    inv = gc.key_material()[4]
    s = gc.sig_invalid()
    return {c: inv[c][0] for c in KEY_CODES}, s["bad"][0], s["noc"][0], s["nig"][0]


@lru_cache(maxsize=None)
def cancel_keys(n: int, k: int):
    """n keys (as points) that sum to zero."""
    sks = [av._sk(b"av grid cancel %d %d %d" % (n, k, j)) for j in range(n - 1)]
    sks.append(-sum(sks))
    return tuple(bo.g1_compress(ac.G1.mul(bo.G1_GEN, s)) for s in sks)


def material(sp: Spec) -> dict:
    """The tuple as aggregate_verify_cases' dict (name, pks, msgs, sig, want, why)."""
    kind, n, m = sp.kind, sp.n, sp.msgs
    good_sig = bo.g2_compress(valid_sig(1, 0))
    if kind in ("valid", "fail"):
        if not sp.shape_ok:
            pks, sig = list(key_pool()[:n]), good_sig
        else:
            pks, sig = list(valid_keys(n, sp.k)), bo.g2_compress(valid_sig(n, sp.k + (kind == "fail")))
        ms = msgs(m)
    elif kind in DEAD:
        keys, bad_sig, noc_sig, nig_sig = bad_material()
        pks = list(key_pool()[sp.k % 7:sp.k % 7 + n])
        assert len(pks) == n
        for pos, code in sp.bad:
            pks[pos] = keys[code]
        sig = {"badkey": good_sig, "badsig": bad_sig, "noc": noc_sig, "nig": nig_sig}[kind]
        ms = msgs(m)
    else:   # infinity signature over keys that cancel (or, for inf1, one key)
        sig = INF_SIG
        if kind == "inf1":
            pks, ms = [key_pool()[sp.k % POOL]], [b"av grid lone %d" % sp.k]
        else:
            pks = list(cancel_keys(2 if kind in ("triv2", "trivfail") else 3, sp.k))
            one = b"av grid cancel msg %d" % sp.k
            ms = [one] * len(pks)
            if kind == "trivfail":
                ms[-1] = one + b" changed"
    return {"name": f"{kind} n={n} m={m}", "pks": pks, "msgs": list(ms), "sig": sig, "want": sp.want, "why": kind}


def materials(specs):
    """Material for many specs: the key sequences first, on a thread pool (ctypes releases the GIL)."""
    need = sorted({(x.n, x.k) for x in specs if x.kind in ("valid", "fail") and x.shape_ok})
    _pool_map(lambda nk: valid_keys(*nk), need)
    return [material(x) for x in specs]
