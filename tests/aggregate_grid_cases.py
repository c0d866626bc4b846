"""Batch aggregation where the device splits a group, shared by the CPU check (tests/test_aggregate_grid_cases.py) and the
device run (tests/test_aggregate_grid_gpu.py).  No device code here.

`k_g2_aggregate` (csrc/bls_g2.cu) cuts every group of an `aggregate_batch` call into chunks of `chunk` signatures, one
warp per chunk; lane l of a chunk scans its signatures l, l + 32, ... and stops at its first decode error, and the warp
that completes a group's last chunk combines the chunk codes and sums with a lane-strided loop (chunk k on lane k % 32,
pass k // 32) and a butterfly.  `chunk` = 32 max(1, ceil(n / (256 SMs))) for the call's n signatures, so the shapes here
are built per chunk and each call's n is set by a filler group: a block of distinct valid signatures tiled, n exactly
256 SMs j or one past it (chunk 32 j or 32 (j + 1)).  `k_g1_aggregate` (csrc/bls_g1.cu) runs one warp per tuple (four
per CTA); lane l scans keys l, l + 32, ... and stops at its first invalid key, then a warp-wide min picks the first.

Valid material is the closed-form progression of tests/aggregate_batch_cases.py: pool signature i is (a + i d) H(m), so
every group's expected sum is one scalar multiple of H(m).  Items of a signature group are pool indices (i >= 0), negated
pool signatures (~i for -(a + i d) H(m)) or raw 96-byte encodings (infinity or invalid)."""
from __future__ import annotations

import hashlib
import random
from dataclasses import dataclass, field
from functools import lru_cache

import numpy as np

from oracle import bls_oracle as bo
from tests import aggregate_batch_cases as ac

SMS = (132, 114)           # H100 SXM and PCIe
SUCCESS, BAD_ENCODING, NOT_ON_CURVE, NOT_IN_GROUP, PK_IS_INFINITY, EMPTY = 0, 1, 2, 3, 6, 16
INVALID_SIGNATURE = 5
INF_SIG, INF_PK = ac.INF_SIG, ac.INF_PK
POOL = 1024                # distinct pool signatures
BLOCK = 1000               # the filler's block (not a multiple of 32: block edges fall on every lane)


# ------------------------------------------------------------------------------------------------ launch arithmetic
def g2_chunk(n: int, sms: int) -> int:
    """bls_g2.cu g2_aggregate_chunk: 32 signatures per warp-stride, about eight warps per SM over the call."""
    return 32 * max(1, -(-n // (256 * sms)))


@dataclass
class G2Map:
    """How launch_g2_aggregate lays out one call of groups of `lens` signatures on a device with `sms` SMs."""
    lens: list
    sms: int
    chunk: int = 0
    chunk_off: list = field(default_factory=list)
    chunk_group: list = field(default_factory=list)

    def __post_init__(self):
        self.n = sum(self.lens)
        self.chunk = g2_chunk(self.n, self.sms)
        self.chunk_off = [0]
        for L in self.lens:
            self.chunk_off.append(self.chunk_off[-1] + self.chunks_of(L))
        self.chunk_group = [g for g, L in enumerate(self.lens) for _ in range(self.chunks_of(L))]

    def chunks_of(self, length: int) -> int:
        return max(1, -(-length // self.chunk))

    @property
    def n_chunks(self) -> int:
        return self.chunk_off[-1]

    @property
    def cta(self) -> int:
        """agg_cta: 128-thread CTAs from four warps per SM on."""
        return 128 if self.n_chunks >= 4 * self.sms else 32

    @property
    def launches(self) -> int:
        """k_g2_sig_decode (when there are signatures) + k_g2_aggregate."""
        return (1 if self.n else 0) + 1

    def where(self, g: int, i: int):
        """Signature i of group g -> (global chunk, chunk within the group, lane, pass)."""
        k, o = divmod(i, self.chunk)
        return self.chunk_off[g] + k, k, o % 32, o // 32

    @staticmethod
    def finisher(k: int):
        """Chunk k of a group -> (lane, pass) of the finisher's chunk loop."""
        return k % 32, k // 32


def g2_map(lens, sms: int) -> G2Map:
    return G2Map(list(lens), sms)


def k2_map(t: int, k: int):
    """Key k of tuple t in k_g1_aggregate -> (CTA, warp, lane, pass)."""
    return t // 4, t % 4, k % 32, k // 32


def compress_cta(n_groups: int) -> int:
    """launch_g1_compress_groups: one thread per group, 32-thread CTAs up to 32 groups, else 128."""
    return 32 if n_groups <= 32 else 128


def call_sizes(sms: int):
    """(n, chunk) of the filled calls: n = 256 SMs j and 256 SMs j + 1 for j = 1, 2, 3."""
    return [(256 * sms * j + e, 32 * (j + e)) for j in (1, 2, 3) for e in (0, 1)]


# ------------------------------------------------------------------------------------------------ material
@lru_cache(maxsize=None)
def sig_pool():
    """-> (h, a, d, points, encodings, negated encodings) of the POOL progression signatures."""
    h = bo.hash_to_g2(b"aggregate grid")
    a, d = ac._scalar(b"agg grid a"), 1 + ac._scalar(b"agg grid d") % 1000
    pts = ac.progression(ac.G2, h, a, d, POOL)
    return h, a, d, pts, [bo.g2_compress(p) for p in pts], [bo.g2_compress(ac.G2.neg(p)) for p in pts]


def _g2_on_curve_not_in_group(rnd):
    """A random x on E'(Fp2) (y from the square root): the cofactor leaves it outside G2 except with negligible chance."""
    while True:
        b = bytearray(rnd.randbytes(96))
        b[0] = (b[0] & 0x1F) | 0x80 | (0x20 if rnd.random() < 0.5 else 0)
        if bo.g2_uncompress(bytes(b))[0] == SUCCESS:
            return bytes(b)


@lru_cache(maxsize=None)
def sig_invalid():
    """Invalid signature encodings by name -> (encoding, code): a bad encoding, one off the curve, one outside G2."""
    rnd = random.Random(0x6A6)
    return {"bad": (ac.bad_encodings(96, rnd)[2], BAD_ENCODING),
            "noc": (ac.not_on_curve_g2(rnd), NOT_ON_CURVE), "nig": (_g2_on_curve_not_in_group(rnd), NOT_IN_GROUP)}


def item_bytes(it) -> bytes:
    if isinstance(it, bytes):
        return it
    _, _, _, _, enc, neg = sig_pool()
    return enc[it % POOL] if it >= 0 else neg[(~it) % POOL]


def item_scalar(it) -> int:
    """The discrete log base H(m) of a valid item (0 for infinity)."""
    _, a, d, _, _, _ = sig_pool()
    if isinstance(it, bytes):
        assert it == INF_SIG
        return 0
    return (a + (it % POOL) * d) if it >= 0 else -(a + ((~it) % POOL) * d)


def _inv_code(it):
    for e, c in sig_invalid().values():
        if it == e:
            return c
    return None


def first_failure(items) -> int:
    """aggregate's code by the rule: the first decode error in order, else NOT_IN_GROUP if any, else SUCCESS."""
    codes = [_inv_code(it) if isinstance(it, bytes) else None for it in items]
    dec = [c for c in codes if c in (BAD_ENCODING, NOT_ON_CURVE)]
    if dec:
        return dec[0]
    return NOT_IN_GROUP if NOT_IN_GROUP in codes else (EMPTY if not items else SUCCESS)


def expected(items):
    """(code, 96 bytes or None) of `aggregate` over the items."""
    code = first_failure(items)
    if code != SUCCESS:
        return code, None
    h = sig_pool()[0]
    s = sum(item_scalar(it) for it in items) % bo.R
    return SUCCESS, (INF_SIG if s == 0 else bo.g2_compress(ac.G2.mul(h, s)))


def flat_sigs(groups) -> tuple:
    """-> (uint8 flat encodings, offsets)."""
    off = [0]
    for g in groups:
        off.append(off[-1] + len(g.items))
    flat = b"".join(item_bytes(it) for g in groups for it in g.items)
    return np.frombuffer(flat, dtype=np.uint8) if flat else np.zeros(0, np.uint8), off


# ------------------------------------------------------------------------------------------------ signature groups
@dataclass
class Group:
    name: str
    items: list
    claim: dict = field(default_factory=dict)   # the shape the group was built for (checked by the CPU file)
    _want: tuple = None

    @property
    def want(self):
        if self._want is None:
            self._want = expected(self.items)
        return self._want


def _valid(n, start=0):
    return [(start + i) % POOL for i in range(n)]


def _place(n, marks, start=0):
    items = _valid(n, start)
    for pos, nm in marks:
        items[pos] = sig_invalid()[nm][0]
    return items


# the four orders of two failures on one lane: (first, second)
SAME_LANE_KINDS = (("bad", "nig"), ("nig", "bad"), ("bad", "noc"), ("noc", "bad"))


def sig_cases(C: int):
    """The test groups for calls whose chunk is C."""
    gs = []
    pairs = sorted({(p, p + 32) for p in (0, 5, 31)} | {(p, p + C - 32) for p in (0, 5, 31) if C > 32})
    for p1, p2 in pairs:
        for f, s in SAME_LANE_KINDS:
            gs.append(Group(f"same lane {f}@{p1} {s}@{p2}", _place(p2 + 8, [(p1, f), (p2, s)]),
                            {"same_lane": (p1, p2), "same_chunk": p2 < C}))
    # cuts: chunk - 1 | chunk, and a ragged last chunk
    for f, s in (("nig", "bad"), ("noc", "bad"), ("bad", "noc")):
        gs.append(Group(f"cut {f}@{C - 1} {s}@{C}", _place(C + 9, [(C - 1, f), (C, s)]), {"cut": (C - 1, C)}))
    L = 2 * C + 17
    for marks in ([(L - 1, "nig")], [(2 * C, "bad"), (L - 1, "nig")], [(2 * C, "nig"), (L - 1, "noc")], [(C + 3, "nig"), (L - 1, "bad")]):
        gs.append(Group("ragged " + " ".join(f"{nm}@{p}" for p, nm in marks), _place(L, marks), {"ragged": [p for p, _ in marks]}))
    # more than 32 chunks: two chunks on one finisher lane, a group-check failure long before a decode error, a lone
    # failure in chunk 63 or in the last chunk
    for L, lanes in ((33 * C, (0,)), (64 * C + 1, (0, 31, 32))):
        nck = -(-L // C)
        for l in lanes:
            x = (7 * l + 2) % C
            y = min((11 * l + 3) % C, L - (l + 32) * C - 1)
            for f, s in (("bad", "noc"), ("noc", "bad")):
                gs.append(Group(f"{nck} chunks: {f} in chunk {l}, {s} in chunk {l + 32}",
                                _place(L, [(l * C + x, f), ((l + 32) * C + y, s)]), {"finisher": (l, l + 32), "n_chunks": nck}))
        gs.append(Group(f"{nck} chunks: noc alone in the last chunk", _place(L, [(L - 1, "noc")]), {"chunk_of": {L - 1: nck - 1}}))
    L = 64 * C + 1
    gs.append(Group("65 chunks: nig in chunk 0, bad in chunk 40", _place(L, [(5, "nig"), (40 * C + 9, "bad")]),
                    {"chunk_of": {5: 0, 40 * C + 9: 40}}))
    gs.append(Group("65 chunks: nig alone in chunk 63", _place(L, [(63 * C + C // 2, "nig")]), {"chunk_of": {63 * C + C // 2: 63}}))
    # partial sums that meet in the finisher
    S0 = _valid(C)
    neg0 = [~i for i in S0]
    distinct = lambda k: _valid(C, start=(k * C + 7) % POOL)  # noqa: E731
    gs.append(Group("two equal chunks", S0 + S0, {"equal_chunks": (0, 1)}))
    gs.append(Group("33 chunks, chunk 32 equals chunk 0", sum((distinct(k) for k in range(32)), []) + distinct(0),
                    {"equal_chunks": (0, 32), "finisher": (0, 32)}))
    gs.append(Group("33 chunks, chunk 32 is minus chunk 0", sum((distinct(k) for k in range(32)), []) + [~i for i in distinct(0)],
                    {"opposite_chunks": (0, 32), "finisher": (0, 32)}))
    body = [distinct(k) for k in range(32)]
    body[19] = [~i for i in body[3]]
    gs.append(Group("32 chunks, chunk 19 is minus chunk 3 (butterfly partners at 16)", sum(body, []), {"opposite_chunks": (3, 19)}))
    body = [[INF_SIG] * C for _ in range(32)]
    body[6], body[7] = S0, neg0
    gs.append(Group("32 chunks of infinity but chunks 6 = -7 (partners at 1)", sum(body, []), {"opposite_chunks": (6, 7)}))
    half = C // 2
    gs.append(Group("3 chunks, chunk 1 cancels inside", distinct(0) + _valid(half, 500) + [~i for i in _valid(half, 500)] + distinct(2),
                    {"zero_chunk": 1}))
    gs.append(Group("3 chunks, chunk 1 of infinity signatures", distinct(0) + [INF_SIG] * C + distinct(2), {"zero_chunk": 1}))
    gs.append(Group("64 chunks, a block of chunk tiled", S0 * 64, {"equal_chunks": tuple(range(64))}))
    # CTA-size and group edges: exactly chunk and chunk + 1 signatures, a failure alone in the one-signature chunk
    gs.append(Group("exactly chunk", _valid(C, 3), {"n_chunks": 1}))
    gs.append(Group("chunk + 1", _valid(C + 1, 9), {"n_chunks": 2}))
    gs.append(Group("chunk + 1, noc in the one-signature chunk", _place(C + 1, [(C, "noc")]), {"n_chunks": 2, "chunk_of": {C: 1}}))
    gs.append(Group("empty", []))
    return gs


def filler(length: int) -> "Group":
    """BLOCK distinct pool signatures tiled: sum = (length // BLOCK) x the block sum + the sum of the first length % BLOCK."""
    return Group(f"filler of {length}", [i % BLOCK for i in range(length)], {"filler": True})


def filler_closed_form(length: int) -> int:
    """The filler's discrete log base H(m), from the progression's closed form."""
    _, a, d, _, _, _ = sig_pool()
    m, r = divmod(length, BLOCK)
    blk = lambda n: n * a + d * n * (n - 1) // 2  # noqa: E731
    return (m * blk(BLOCK) + blk(r)) % bo.R


@dataclass
class SigCall:
    name: str
    groups: list
    sms: int
    chunk: int          # the chunk size the call was built for

    @property
    def map(self) -> G2Map:
        return g2_map([len(g.items) for g in self.groups], self.sms)


def _interleave(tests, fill):
    """Test groups on both sides of the filler, an empty group after every fifth and one just before the filler."""
    out = []
    half = len(tests) // 2
    for k, g in enumerate(tests[:half]):
        out.append(g)
        if k % 5 == 4:
            out.append(Group("empty between", []))
    out += [Group("empty before the filler", []), fill]
    out += tests[half:]
    return out


def sig_calls(sms: int):
    """The filled calls: the groups of sig_cases(C) for C = 32, 64, 96, 128 beside fillers, in calls of n = 256 SMs j (+ 1).
    A chunk size that two n reach gets its groups dealt between them; groups that do not fit one call go to another call
    at the same n."""
    sizes = call_sizes(sms)
    calls = []
    for C in sorted({c for _, c in sizes}):
        ns = [n for n, c in sizes if c == C]
        cases = sig_cases(C)
        for r, n in enumerate(ns):
            pending, k = cases[r::len(ns)], 0
            while pending:
                room, take = n - 40 * C, []   # the filler keeps more than 32 chunks
                while pending and (not take or sum(len(g.items) for g in take) + len(pending[0].items) <= room):
                    take.append(pending.pop(0))
                used = sum(len(g.items) for g in take)
                assert used <= room, (C, n, used)
                calls.append(SigCall(f"n={n} chunk={C} #{k}", _interleave(take, filler(n - used)), sms, C))
                k += 1
    return calls


def edge_calls(sms: int):
    """Chunk 32 with n_chunks = 4 SMs - 1 (32-thread CTAs) and 4 SMs (128-thread CTAs): the chunk-32 same-lane and cut groups
    padded with empty groups (one chunk each)."""
    out = []
    base = [g for g in sig_cases(32) if "same_lane" in g.claim or "cut" in g.claim or "ragged" in g.claim]
    for target in (4 * sms - 1, 4 * sms):
        gs = list(base)
        have = g2_map([len(g.items) for g in gs], sms).n_chunks
        pad = target - have
        assert pad > 0
        gs = gs[:len(gs) // 2] + [Group("empty pad", []) for _ in range(pad)] + gs[len(gs) // 2:]
        out.append(SigCall(f"n_chunks={target}", gs, sms, 32))
    return out


# ------------------------------------------------------------------------------------------------ key groups (K2)
KEY_CODES = (PK_IS_INFINITY, NOT_ON_CURVE, NOT_IN_GROUP, BAD_ENCODING)
KEY_T = (31, 32, 33, 127, 128, 129, 255, 256, 257)   # 4k - 1 | 4k | 4k + 1 tuples; 32 | 33 and 128k +- 1 for the compress CTA


def _g1_on_curve_not_in_group(rnd):
    while True:
        b = bytearray(rnd.randbytes(48))
        b[0] = (b[0] & 0x1F) | 0x80
        code, pt = bo.g1_uncompress(bytes(b))
        if code == SUCCESS and pt is not None:
            return bytes(b)


@lru_cache(maxsize=None)
def key_material():
    """-> (valid keys: 160 progression encodings, pts, a, d; invalid: {code: [two distinct encodings]})."""
    enc, pts, a, d = ac.key_pool(77, 160)
    rnd = random.Random(0x6B6)
    bads = ac.bad_encodings(48, rnd)
    inv = {PK_IS_INFINITY: [INF_PK, INF_PK],
           NOT_ON_CURVE: [ac.not_on_curve_g1(rnd), ac.not_on_curve_g1(rnd)],
           NOT_IN_GROUP: [_g1_on_curve_not_in_group(rnd), _g1_on_curve_not_in_group(rnd)],
           BAD_ENCODING: [bads[0], bads[2]]}
    return enc, pts, a, d, inv


@dataclass
class KeyGroup:
    name: str
    slots: list          # per position: int = valid key index, (code, j) = invalid key j of that code
    want: tuple          # (code, 48 bytes or None)
    claim: dict = field(default_factory=dict)


def key_cases():
    """Pairs of invalid keys on one lane at (p, p + 32) and (p, p + 64) for every ordered pair of distinct codes, and valid
    groups (closed-form sums) between them."""
    enc, pts, a, d, inv = key_material()
    gs = []
    for p in (0, 5, 31):
        for gap in (32, 64):
            for c1 in KEY_CODES:
                for c2 in KEY_CODES:
                    if c1 == c2:
                        continue
                    n = p + gap + 1 + (p % 7)
                    slots = [(p * 3 + i) % 160 for i in range(n)]
                    slots[p], slots[p + gap] = (c1, 0), (c2, 1)
                    gs.append(KeyGroup(f"{c1}@{p} {c2}@{p + gap}", slots, (c1, None), {"same_lane": (p, p + gap)}))
        start = 11 * p
        n = 40 + 3 * p
        s = sum(a + ((start + i) % 160) * d for i in range(n))
        gs.append(KeyGroup(f"valid {n} from {start}", [(start + i) % 160 for i in range(n)], (SUCCESS, bo.g1_compress(ac.G1.mul(bo.G1_GEN, s)))))
    return gs


def key_bytes(slot) -> bytes:
    enc, _, _, _, inv = key_material()
    return enc[slot] if isinstance(slot, int) else inv[slot[0]][slot[1]]


def key_call(T: int):
    """T tuples: key_cases() cyclically, started so that the last tuples (the ragged last CTA) are failure cases."""
    cases = key_cases()
    return [cases[(t + 5 * T) % len(cases)] for t in range(T)]


def registry_keys():
    """Registry contents: the 160 valid keys, then the invalid keys (two per code) -> (encodings, {slot: registry index})."""
    enc, _, _, _, inv = key_material()
    keys, where = list(enc), {}
    for c in KEY_CODES:
        for j in range(2):
            where[(c, j)] = len(keys)
            keys.append(inv[c][j])
    return keys, where


def verify_msg(t: int) -> bytes:
    return hashlib.sha256(b"aggregate grid tuple %d" % t).digest()


def verify_sig() -> bytes:
    """A valid signature (of nothing in particular): tuples with valid keys answer INVALID_SIGNATURE."""
    return sig_pool()[4][0]


def verify_want(g: KeyGroup) -> int:
    return g.want[0] if g.want[0] != SUCCESS else INVALID_SIGNATURE


# ------------------------------------------------------------------------------------------------ sync committee
SYNC_GAPS = (32, 480)


def sync_state(n: int = 1024):
    """A mainnet state of n active validators with valid progression keys."""
    from tests import duties_cases as dc
    st = dc.base(n, seed=31)
    enc, _, _, _ = ac.key_pool(131, n)
    st.validators["public_key"] = np.frombuffer(b"".join(enc), dtype="V48")
    return st


def sync_positions(idx, gap: int):
    """Positions p < 32 with p and p + gap held by distinct validators, each at its first occurrence in the committee."""
    first = {}
    for j, v in enumerate(idx):
        first.setdefault(int(v), j)
    return [p for p in range(32) if p + gap < len(idx) and int(idx[p]) != int(idx[p + gap])
            and first[int(idx[p])] == p and first[int(idx[p + gap])] == p + gap]


def sync_cases(idx):
    """(p, q, c1, c2): committee positions p, q = p + gap on one lane get invalid keys of codes c1, c2; want c1."""
    out = []
    for gap in SYNC_GAPS:
        ps = sync_positions(idx, gap)
        for k, (c1, c2) in enumerate((c1, c2) for c1 in KEY_CODES for c2 in KEY_CODES if c1 != c2):
            p = ps[k % len(ps)]
            out.append((p, p + gap, c1, c2))
    return out
