"""Proposer and sync-committee states built to land on the launch shape of the device's sampling and key-matching kernels
(csrc/shuffle.cu): where the SYNC_COMMITTEE_SIZE-th accept falls among k_select_accepted's windows, chunks, scan warps,
ballots and lanes; proposer warps of one CTA that stop after very different numbers of windows; 31 to 65 active validators,
where i mod n wraps inside one ballot; committee keys with equal 8-byte prefixes and holders on k_match_committee_keys'
grid-stride passes.  No device code: shared by test_duties_grid_cases.py (CPU: every case lands where it was built) and
test_duties_grid_gpu.py (the device against oracle/duties_oracle.py).

Cases are placed by balance.  The seeds and the shuffle do not read balances, so for a fixed randao mix the candidate
sequence and its random bytes are fixed; a case gives 32 ETH to the validators at chosen candidate positions and 0 ETH to
the rest.  A 0-ETH candidate is still accepted on a random byte of 0: those background accepts are counted, not avoided.
The randao mixes and the proposer epoch below were found by the `search_*` functions and are stored as constants."""
from __future__ import annotations

import bisect
import hashlib
from collections import namedtuple
from dataclasses import dataclass, field
from functools import lru_cache

import numpy as np

from oracle import duties_oracle as do
from oracle import shuffle_oracle as sh
from tests import duties_cases as dc

ETH = dc.ETH
CHUNK = 1024          # ballots per pass of k_select_accepted (one per thread of its 1 024-thread CTA)
SCAN = 32             # ballots per scan warp of that CTA
SAMPLE_WARPS = 4      # warps per CTA of k_sample_windows and k_sample_proposers
MATCH_THREADS = 256   # threads per CTA of k_match_committee_keys
CAP_WORDS = do.CAP // 32

N_COMMITTEE = (1 << 17) + 5   # late window-8 candidates wrap i mod n
N_PROPOSER = (1 << 16) + 3
N_MINIMAL = 8200
SLOT_EPOCH = 1000             # the committee is drawn for epoch SLOT_EPOCH + 1

# found by search_committee_mix / search_zero_eth_mix / search_proposer_epoch (tags of `mix(tag, k)`)
COMMITTEE_MIX = 3
ZERO_ETH_MIX = {"w7_chunk1": 1, "w8_wrapped": 0}
PROPOSER_EPOCH = 5779


# ---- the device's schedule -------------------------------------------------------------------------------------------

Where = namedtuple("Where", "window chunk warp ballot lane")


class WindowMap:
    """The committee sampler's windows (sample_committee_on_device): window k holds ceil(SIZE / 32) * 2^k ballots of 32
    candidates, capped so that all windows hold at most 2^26 candidates.  k_select_accepted walks a window in chunks of
    1 024 ballots, each split into 32 scan warps of 32 ballots.  `where(i)` places candidate i: its window, the chunk and
    scan warp within that window, the ballot within the scan warp and the lane within the ballot."""

    def __init__(self, preset: str):
        self.preset = preset
        self.size = do.PRESET[preset]["SYNC_COMMITTEE_SIZE"]
        self.start, self.words = [], []
        done, w = 0, -(-self.size // 32)
        while done < CAP_WORDS:
            w = min(w, CAP_WORDS - done)
            self.start.append(done)
            self.words.append(w)
            done += w
            w = min(2 * w, CAP_WORDS)

    def where(self, i: int) -> Where:
        b = i // 32
        k = bisect.bisect_right(self.start, b) - 1
        r = b - self.start[k]
        return Where(k, r // CHUNK, (r % CHUNK) // SCAN, r % SCAN, i % 32)

    def candidate(self, window: int, chunk: int = 0, warp: int = 0, ballot: int = 0, lane: int = 0) -> int:
        r = chunk * CHUNK + warp * SCAN + ballot
        assert r < self.words[window] and 0 <= lane < 32
        return 32 * (self.start[window] + r) + lane

    def chunks(self, window: int) -> int:
        return -(-self.words[window] // CHUNK)

    def launches(self, cut: int) -> int:
        """Launches of one next_sync_committee call whose SIZE-th accept is candidate `cut`: 3 for the active indices, 2 per
        window (k_sample_windows, k_select_accepted), then the key gather, K1, the aggregate and the compression."""
        return 3 + 2 * (self.where(cut).window + 1) + 4


@lru_cache(maxsize=None)
def window_map(preset: str) -> WindowMap:
    return WindowMap(preset)


def match_stride(n: int, sms: int) -> int:
    """k_match_committee_keys' grid stride: min(ceil(n / 256), 4 SMs) CTAs of 256 threads."""
    return min(-(-n // MATCH_THREADS), 4 * sms) * MATCH_THREADS


# ---- candidate streams -----------------------------------------------------------------------------------------------

def mix(tag: str, k: int) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(f"duties-grid {tag} {k}".encode()).digest(), np.uint8)


def random_bytes(seed: bytes, count: int) -> np.ndarray:
    """random_byte of candidates 0 .. count - 1: SHA-256(seed || le64(i / 32))[i % 32]."""
    blocks = -(-count // 32)
    return np.frombuffer(b"".join(hashlib.sha256(seed + w.to_bytes(8, "little")).digest() for w in range(blocks)),
                         np.uint8)[:count]


def accepted(eff: np.ndarray, rb: np.ndarray) -> np.ndarray:
    """effective_balance * 255 >= MAX_EFFECTIVE_BALANCE * random_byte, the product wrapping in u64."""
    with np.errstate(over="ignore"):
        return eff.astype(np.uint64) * np.uint64(255) >= np.uint64(do.MAX_EFFECTIVE_BALANCE) * rb.astype(np.uint64)


def committee_epoch(st) -> int:
    return do.slot(st) // do.PRESET[st.preset]["SLOTS_PER_EPOCH"] + 1


def set_mix(st, epoch: int, m: np.ndarray):
    """randao mix read by get_seed(st, epoch, .)"""
    ephv = do.PRESET[st.preset]["EPOCHS_PER_HISTORICAL_VECTOR"]
    st.randao_mixes[(epoch + ephv - 2) % ephv] = m
    return st


class Stream:
    """The committee loop's candidates 0 .. count - 1 for `st` (list formulation: one shuffle of the active list)."""

    def __init__(self, st, count: int):
        P = do.PRESET[st.preset]
        epoch = committee_epoch(st)
        self.seed = do.get_seed(st, epoch, do.DOMAIN_SYNC_COMMITTEE)
        self.active = do.active_indices(st, epoch)
        self.n = len(self.active)
        self.shuffled = sh.shuffled_indices_numpy(self.active, self.seed, P["SHUFFLE_ROUND_COUNT"])
        self.count = count
        self.rb = random_bytes(self.seed, count)
        self.cand = self.shuffled[np.arange(count) % self.n]

    def accepts(self, st) -> np.ndarray:
        return accepted(st.validators["effective_balance"][self.cand], self.rb)

    def cut(self, st, size: int):
        """The candidate index of the size-th accept, None past `count`."""
        acc = np.flatnonzero(self.accepts(st))
        return int(acc[size - 1]) if len(acc) >= size else None


# ---- committee cases -------------------------------------------------------------------------------------------------

@dataclass
class CommitteeCase:
    name: str
    st: object
    preset: str
    cut: int                                     # the candidate index of the SIZE-th accept, as built
    shape: dict = field(default_factory=dict)    # fields of Where the cut was built to have
    after: tuple = ()                            # accepts placed after the cut
    zero_eth: bool = False


def committee_base(n: int, preset: str, m: np.ndarray, seed: int) -> object:
    st = dc.base(n, preset, seed=seed, eff=0, slot_epoch=SLOT_EPOCH)
    return set_mix(st, SLOT_EPOCH + 1, m)


def place(stream: Stream, st, size: int, cut: int, rng, must=(), after=()):
    """32 ETH at the candidates `must`, `cut`, `after` and at random other candidates before `cut`, so that the cut is
    the size-th accept; the background accepts (random byte 0) before it are counted.  Every position is below n, so no
    validator is drawn twice up to the cut."""
    assert cut < stream.n and all(p < stream.n for p in after)
    zero = stream.rb[:cut] == 0
    must = np.array(sorted(set(must)), dtype=np.int64)
    assert (must < cut).all()
    free = np.flatnonzero(~zero)
    free = free[~np.isin(free, must)]
    need = size - 1 - int(zero.sum()) - int((~zero[must]).sum())
    assert need >= 0, (cut, need)
    chosen = np.concatenate([rng.choice(free, need, replace=False), must, [cut], np.asarray(after, np.int64)])
    eff = st.validators["effective_balance"]
    eff[:] = 0
    eff[stream.cand[chosen.astype(np.int64)]] = 32 * ETH
    return st


def mainnet_stream(m: np.ndarray) -> Stream:
    wm = window_map("mainnet")
    st = committee_base(N_COMMITTEE, "mainnet", m, seed=31)
    return Stream(st, wm.candidate(8) + 64)


def search_committee_mix(start: int = 0) -> int:
    """A mix with at most 500 background accepts before window 8, so that every placed mainnet cut up to the first
    candidate of window 8 can be built."""
    wm = window_map("mainnet")
    end = wm.candidate(8)
    st = committee_base(64, "mainnet", mix("committee", 0), seed=31)
    for k in range(start, start + 1000):
        set_mix(st, SLOT_EPOCH + 1, mix("committee", k))
        seed = do.get_seed(st, SLOT_EPOCH + 1, do.DOMAIN_SYNC_COMMITTEE)
        rb = random_bytes(seed, end + 1)
        if (rb[:end] == 0).sum() <= 500 and rb[end] != 0:
            return k
    raise AssertionError("no mix")


def zero_eth_cut(k: int, count: int):
    """The 512th zero random byte of mix k of the all-0-ETH mainnet state (its committee cut)."""
    st = committee_base(64, "mainnet", mix("zero_eth", k), seed=33)
    seed = do.get_seed(st, SLOT_EPOCH + 1, do.DOMAIN_SYNC_COMMITTEE)
    z = np.flatnonzero(random_bytes(seed, count) == 0)
    return int(z[511]) if len(z) >= 512 else None


def zero_eth_goal(name: str):
    wm = window_map("mainnet")
    if name == "w7_chunk1":
        return lambda c: c is not None and wm.where(c)[:2] == (7, 1)
    return lambda c: c is not None and wm.where(c)[:2] == (8, 0) and c >= N_COMMITTEE + 32 * 64


def search_zero_eth_mix(name: str, start: int = 0) -> int:
    goal, count = zero_eth_goal(name), window_map("mainnet").candidate(8, 1)
    for k in range(start, start + 1000):
        if goal(zero_eth_cut(k, count)):
            return k
    raise AssertionError("no mix")


# (name, window, chunk, warp, ballot, lane, accepts placed before the cut (offsets from the start of its ballot),
#  accepts placed after it (offsets from the cut))
MAINNET_CUTS = [
    ("lane0", 3, 0, 2, 5, 0, (), (1, 7, 31)),
    ("lane31", 5, 0, 9, 13, 31, (0, 3, 17, 30), (1, 9)),
    ("warp_last_ballot", 6, 0, 11, 31, 12, (2, 5), (1, 5, 20, 44)),
    ("warp_first_ballot", 6, 0, 12, 0, 3, (-20, -1, 0, 1, 2), (4, 30, 32)),
    ("window3_first", 3, 0, 0, 0, 0, (), (1, 2, 3)),
    ("window8_first", 8, 0, 0, 0, 0, (), (1, 2, 31, 32)),
    ("w6_chunk0_last", 6, 0, 31, 31, 20, (19,), (1, 11, 40)),
    ("w7_first_ballot", 7, 0, 0, 0, 9, (0, 8), (10, 32)),
    ("w7_chunk0_last", 7, 0, 31, 31, 20, (1, 19), (21, 31, 32, 40)),
    ("w7_chunk1_first", 7, 1, 0, 0, 6, (0, 5), (7, 31, 32)),
]
MINIMAL_CUTS = [
    ("minimal_w0_lane31", 0, 0, 0, 0, 31, tuple(range(31)), ()),
    ("minimal_w5", 5, 0, 0, 17, 4, (1,), (5, 9, 31)),
    ("minimal_w6", 6, 0, 1, 2, 31, (0, 30), (32, 33)),
]


def _placed(name, preset, stream, base_st, spec, rng):
    _, k, c, w, b, lane, before, after = spec
    wm = window_map(preset)
    cut = wm.candidate(k, c, w, b, lane)
    must = [cut - lane + j for j in before]
    if k > 0:   # something accepted in every earlier window and in every earlier chunk of this one
        must += [wm.candidate(j, 0, 0, 0, 7) for j in range(k) if wm.candidate(j, 0, 0, 0, 7) < cut]
        must += [wm.candidate(k, j, 0, 1, 3) for j in range(c)]
    st = base_st.copy_for_case()
    place(stream, st, wm.size, cut, rng, must, [cut + a for a in after])
    return CommitteeCase(name, st, preset, cut, dict(window=k, chunk=c, warp=w, ballot=b, lane=lane),
                         tuple(cut + a for a in after))


class _Base:
    """A state and a cheap per-case copy (only the Validator records change between cases)."""

    def __init__(self, st):
        self.st = st

    def copy_for_case(self):
        import copy
        out = copy.copy(self.st)
        out.validators = self.st.validators.copy()
        return out


@lru_cache(maxsize=None)
def committee_cases() -> tuple:
    out = []
    rng = np.random.default_rng(2024)
    stream = mainnet_stream(mix("committee", COMMITTEE_MIX))
    base = _Base(committee_base(N_COMMITTEE, "mainnet", mix("committee", COMMITTEE_MIX), seed=31))
    for spec in MAINNET_CUTS:
        out.append(_placed(spec[0], "mainnet", stream, base, spec, rng))
    for name, k in ZERO_ETH_MIX.items():
        st = committee_base(N_COMMITTEE, "mainnet", mix("zero_eth", k), seed=33)
        count = window_map("mainnet").candidate(8, 1)
        out.append(CommitteeCase(f"zero_eth_{name}", st, "mainnet", zero_eth_cut(k, count), zero_eth=True))
    mst = committee_base(N_MINIMAL, "minimal", mix("minimal", 0), seed=32)
    stream = Stream(mst, window_map("minimal").candidate(8))
    for spec in MINIMAL_CUTS:
        out.append(_placed(spec[0], "minimal", stream, _Base(mst), spec, rng))
    return tuple(out)


def zero_eth_case(name: str) -> CommitteeCase:
    return next(c for c in committee_cases() if c.name == f"zero_eth_{name}")


# ---- proposer cases --------------------------------------------------------------------------------------------------

# slot -> (window, lane) of its first accept; every other slot's first accept is candidate 0.  Slots 4 * b .. 4 * b + 3
# share CTA b of k_sample_proposers: CTA 1 mixes a 41-window warp with shallow ones, CTA 2 a 9-window warp.
PROPOSER_TARGETS = {0: (0, 0), 1: (0, 31), 2: (1, 0), 3: (0, 5), 4: (2, 17), 5: (0, 0), 6: (40, 13), 7: (0, 1),
                    8: (1, 31), 9: (8, 0), 31: (0, 31)}


def proposer_targets(spe: int = 32) -> list:
    return [32 * PROPOSER_TARGETS.get(s, (0, 0))[0] + PROPOSER_TARGETS.get(s, (0, 0))[1] for s in range(spe)]


def slot_seeds(st, epoch: int) -> list:
    spe = do.PRESET[st.preset]["SLOTS_PER_EPOCH"]
    base = do.get_seed(st, epoch, do.DOMAIN_BEACON_PROPOSER)
    return [hashlib.sha256(base + (epoch * spe + j).to_bytes(8, "little")).digest() for j in range(spe)]


def slot_candidates(st, active: np.ndarray, seed: bytes, count: int) -> np.ndarray:
    """Candidates 0 .. count - 1 of one slot seed: per index when few are needed, else from the list shuffle."""
    rounds = do.PRESET[st.preset]["SHUFFLE_ROUND_COUNT"]
    n = len(active)
    if count <= 200:
        return np.array([active[sh.compute_shuffled_index(i % n, n, seed, rounds)] for i in range(count)], np.uint64)
    return sh.shuffled_indices_numpy(active, seed, rounds)[np.arange(count) % n]


def proposer_base():
    return dc.base(N_PROPOSER, seed=41, eff=0)


def _no_zero_before_targets(seeds, targets) -> bool:
    for s in sorted(range(len(targets)), key=lambda s: -targets[s]):
        t = targets[s]
        if t and (random_bytes(seeds[s], t) == 0).any():
            return False
    return True


def _proposer_placement(st, epoch: int):
    """-> (32-ETH validators, or None when a slot would meet another slot's 32-ETH validator before its target)."""
    targets = proposer_targets()
    active = do.active_indices(st, epoch)
    cands = [slot_candidates(st, active, s, t + 1) for s, t in zip(slot_seeds(st, epoch), targets)]
    rich = {int(c[t]) for c, t in zip(cands, targets)}
    if any(rich & set(c[:t].tolist()) for c, t in zip(cands, targets)):
        return None
    return sorted(rich)


def search_proposer_epoch(start: int = 2000) -> int:
    st, targets = proposer_base(), proposer_targets()
    for e in range(start, start + 100000):
        if _no_zero_before_targets(slot_seeds(st, e), targets) and _proposer_placement(st, e) is not None:
            return e
    raise AssertionError("no epoch")


@dataclass
class ProposerCase:
    name: str
    st: object
    epochs: list
    targets: list = None     # candidate index of each slot's first accept at epochs[0], as built


@lru_cache(maxsize=None)
def proposer_cases() -> tuple:
    st = proposer_base()
    rich = _proposer_placement(st, PROPOSER_EPOCH)
    assert rich is not None
    st.validators["effective_balance"][np.asarray(rich, np.int64)] = 32 * ETH
    out = [ProposerCase("placed_slots", st, [PROPOSER_EPOCH], proposer_targets())]
    for k in (31, 32, 33, 63, 64, 65):
        s = dc.only_active(dc.base(k + 40, seed=50 + k), np.arange(9, 9 + k))
        s.validators["effective_balance"][9:9 + k] = np.resize(np.array([0, 32, 1, 31, 16, 0, 0], np.uint64) * ETH, k)
        out.append(ProposerCase(f"active_{k}", s, [1000, 1001, 4321]))
    return tuple(out)


# ---- key-matcher cases -----------------------------------------------------------------------------------------------

@dataclass
class MatcherCase:
    name: str
    st: object
    stride: int
    holders: dict          # committee -> {position: largest holder} as built (absent: no holder)
    decoys: dict           # committee -> validator indices sharing a committee key's prefix with another tail
    edges: list            # validator indices placed on pass edges


def _key(rng, prefix: bytes) -> np.ndarray:
    k = rng.integers(0, 256, 48, dtype=np.uint8)
    k[:8] = np.frombuffer(prefix, np.uint8)
    return k


def matcher_n(sms: int) -> int:
    return 2 * 4 * sms * MATCH_THREADS + 1000


@lru_cache(maxsize=None)
def matcher_cases(sms: int) -> tuple:
    """One mainnet state of n = 2 * stride + 1 000 validators (three grid-stride passes at `sms` SMs) and arbitrary key
    bytes.  Current committee: 512 keys with one 8-byte prefix.  Next committee: keys that differ only in byte 8 or only
    in byte 47 (both orders), prefixes 0 and 2^64 - 1, repeated committee positions, and keys of random validators."""
    n = matcher_n(sms)
    stride = match_stride(n, sms)
    assert -(-n // stride) == 3
    rng = np.random.default_rng(sms)
    st = dc.base(n, seed=61)
    K = st.validators["public_key"].copy().view(np.uint8).reshape(n, 48)
    edges = [stride - 1, stride, 2 * stride + 1, n - 1]
    used = set()

    def spot(lo=0, hi=n):
        while True:
            i = int(rng.integers(lo, hi))
            if i not in used:
                used.add(i)
                return i

    for e in edges:
        used.add(e)
    # current: one prefix for all 512 keys; holders spread over the passes, the edges among them
    pfx = bytes.fromhex("5a17c0de00ff0102")
    cur = [_key(rng, pfx) for _ in range(512)]
    cur_hold, cur_decoys = {}, []
    for j in range(512):
        if j in (5, 300, 511):        # no holder
            continue
        if j < 4:
            hs = [edges[j]]
        elif j == 4:                  # one key at many positions; the largest in the third pass
            hs = [spot(0, stride) for _ in range(12)] + [spot(stride, 2 * stride) for _ in range(6)] + [spot(2 * stride)]
        else:
            hs = [spot()]
        for h in hs:
            K[h] = cur[j]
        cur_hold[j] = max(hs)
    for j in (6, 7, 300):             # validator keys with the shared prefix and another tail, past the holder
        d = spot(cur_hold.get(j, 0) + 1)
        K[d] = _key(rng, pfx)
        cur_decoys.append(d)

    # next: edge keys at the front, then keys of random validators
    nxt, nxt_hold, nxt_decoys = [], {}, []

    def add(key, holders):
        nxt.append(key)
        for h in holders:
            K[h] = key
        if holders:
            nxt_hold[len(nxt) - 1] = max(holders)

    base = _key(rng, bytes.fromhex("33" * 8))
    for d8 in ((0x10, 0x11), (0x21, 0x20)):   # differ only in byte 8, ascending then descending committee order
        for v in d8:
            k = base.copy(); k[8] = v
            add(k, [spot()])
    base = _key(rng, bytes.fromhex("44" * 8))
    for d47 in ((0x01, 0x02), (0xfe, 0xfd)):  # differ only in byte 47
        for v in d47:
            k = base.copy(); k[47] = v
            add(k, [spot()])
    def fixed(*hs):
        assert not used & set(hs)
        used.update(hs)
        return list(hs)

    add(_key(rng, bytes(8)), fixed(edges[0] - 1, edges[1] + 1))       # prefix 0
    add(_key(rng, b"\xff" * 8), fixed(edges[2] - 1, n - 3))           # prefix 2^64 - 1
    z = _key(rng, bytes(8)); z[47] ^= 1
    add(z, [])                                                         # prefix 0, no holder
    # decoys: another tail under a committee prefix, at a larger index than every holder of that key
    for j, flip in ((0, 8), (2, 47), (4, 47), (8, 47), (9, 20)):
        d = spot(nxt_hold[j] + 1)
        k = nxt[j].copy(); k[flip] ^= 0x80
        K[d] = k
        nxt_decoys.append(d)
    d = spot()
    k = z.copy(); k[47] ^= 1                                           # the unheld key's byte-47 twin is held
    K[d] = k
    nxt_decoys.append(d)
    first = len(nxt)
    rest = rng.choice(np.array(sorted(set(range(n)) - used)), 512 - first - 2, replace=False)
    for h in rest:
        nxt.append(K[h].copy())
        nxt_hold[len(nxt) - 1] = int(h)
    for j in (first, 3):                                               # repeated committee positions
        nxt.append(nxt[j].copy())
        nxt_hold[len(nxt) - 1] = nxt_hold[j]
    assert len(nxt) == 512
    st.validators["public_key"] = K.view("V48").reshape(n)
    st.current_sync_committee = b"".join(k.tobytes() for k in cur) + bytes(48)
    st.next_sync_committee = b"".join(k.tobytes() for k in nxt) + bytes(48)
    return (MatcherCase("matcher", st, stride, {"current": cur_hold, "next": nxt_hold},
                        {"current": cur_decoys, "next": nxt_decoys}, edges),)
