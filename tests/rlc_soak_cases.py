"""Case generators and the exact exponent model of the RLC whole-batch check (bls_rlc.cu), shared by the CPU checks
(tests/test_rlc_soak_cases.py) and the device soak (tests/test_rlc_soak_gpu.py).  No device code.

Every tuple is built from known secrets: its keys are s_i g1, its signature is sigma H(m).  With a_t the sum of the key
secrets, the RLC product prod_t e(r_t agg_t, H_t) e(-g1, sum_t r_t sig_t) is e(g1, H)^(sum r_t (a_t - sigma_t)) per
message H, so its verdict is a function of integers mod R that Python computes exactly for any seed (`model`).  That
makes the soak exact even where every tuple is invalid and the batch must still pass (family A), which only the
documented scalar derivation, carried out exactly, produces.

Families: A. cancelling defects crafted against one seed, with controls the model rejects; B. valid batches whose
scaled signatures meet as equal or opposite points in the G2 fold (and whose sum is infinity); C. one invalid tuple at
every position that matters, with a defect or dead.  `O` is the C oracle (oracle/c/bls_oracle.c) loaded through ctypes."""
from __future__ import annotations

import ctypes
import hashlib
import os
from dataclasses import dataclass, field

import numpy as np

from tests.bls_soak_cases import R, mutate, valid_keys

SEED = hashlib.sha256(b"rlc soak seed").digest()
ZERO_SEED = bytes(32)
MSG = hashlib.sha256(b"rlc soak shared message").digest()
N_POOL = 1024                          # distinct valid tuples of families B and C (batch tuple t is pool tuple t % N_POOL)
INF_G1 = bytes([0xC0]) + bytes(47)
INF_G2 = bytes([0xC0]) + bytes(95)
DEAD_KINDS = ("inf_key", "sig_encoding", "sig_x", "empty")
SMALL_T = (1, 2, 31, 32, 33, 63, 64, 65)
LARGE_T = (1023, 1024, 1025, 1056, 1057, 2047, 2048, 2049, 4096)


def rlc_scalar(seed: bytes, t: int) -> int:
    """bls_rlc.cu rlc_scalar: the first 8 bytes, little-endian, of SHA-256(seed || le64(t)), forced non-zero."""
    r = int.from_bytes(hashlib.sha256(bytes(seed) + t.to_bytes(8, "little")).digest()[:8], "little")
    return r if r else 1


@dataclass(frozen=True)
class Tup:
    """One fast_aggregate_verify tuple: keys s g1 for s in `keys`, signature sigma H(msg), and an optional per-point
    failure ("dead"): inf_key (first key is the point at infinity), sig_encoding (compression bit cleared), sig_x
    (signature x one off: off the curve or outside the subgroup), empty (no keys)."""
    msg: bytes
    keys: tuple
    sigma: int
    dead: str = ""

    @property
    def a(self) -> int:
        return sum(self.keys) % R

    @property
    def defect(self) -> int:
        return (self.sigma - self.a) % R


def model(batch, seed: bytes, t0: int = 0) -> bool:
    """The RLC verdict: no tuple is dead, and for every message group g, sum_{t in g} r_t (sigma_t - a_t) = 0 mod R."""
    if any(t.dead for t in batch):
        return False
    acc = {}
    for i, t in enumerate(batch):
        acc[t.msg] = (acc.get(t.msg, 0) + rlc_scalar(seed, t0 + i) * (t.sigma - t.a)) % R
    return all(v == 0 for v in acc.values())


def expected_code(t: Tup):
    """What the per-tuple path must answer: 0 valid, 5 a defect; a dead tuple only has to be rejected (None)."""
    if t.dead:
        return None
    return 0 if t.defect == 0 else 5


@dataclass
class Case:
    """A batch, the seeds it runs under with the model's verdict for each, and the boundaries it sits on."""
    name: str
    family: str
    batch: list
    runs: list                          # [(seed or None, want)]; None: the library draws the seed (want False)
    tags: set = field(default_factory=set)


def _nz(rng) -> int:
    while True:
        x = int.from_bytes(rng.bytes(32), "big") % R
        if x:
            return x


# ------------------------------------------------------------------------------------------------ keys and secrets
class Keys:
    """The valid_keys sequence s_i = sk0 + i d, plus any other secret's key through orc_sk_to_pk, each made once."""

    def __init__(self, O, n=N_POOL):
        self.O = O
        enc, self.sk0, self.d = valid_keys(O, n, seed=21)
        self.n = n
        self.seq = [(self.sk0 + i * self.d) % R for i in range(n)]
        self.enc = {s: enc[i].tobytes() for i, s in enumerate(self.seq)}

    def get(self, s: int) -> bytes:
        if s not in self.enc:
            buf = ctypes.create_string_buffer(48)
            self.O.orc_sk_to_pk(s.to_bytes(32, "big"), buf)
            self.enc[s] = buf.raw
        return self.enc[s]


def pool(keys: Keys):
    """N_POOL valid K = 1 tuples on one shared message: tuple i has key s_i and sigma = s_i."""
    return [Tup(MSG, (s,), s) for s in keys.seq]


# ------------------------------------------------------------------------------------------------ family A
def _fill_groups(T, groups):
    """The given groups, then the remaining positions in consecutive pairs (a triple at the end if odd)."""
    used = {t for g in groups for t in g}
    rest = [t for t in range(T) if t not in used]
    extra = [rest[i:i + 2] for i in range(0, len(rest), 2)]
    if extra and len(extra[-1]) == 1:
        if len(extra) > 1:
            tail = extra.pop()
            extra[-1] = extra[-1] + tail
        else:
            groups = [list(groups[0]) + extra.pop()] + list(groups[1:])
    return [list(g) for g in groups] + extra


def a_layouts():
    """(name, T, K, groups, tags): every position in a group of tuples that share a message."""
    out = []
    for K in (1, 2, 33, 512):
        out.append((f"ends T 2 K {K}", 2, K, [[0, 1]], {"A:(0,T-1)", f"A:K{K}"}))
    out.append(("ends T 33", 33, 1, _fill_groups(33, [[0, 32]]), {"A:(0,T-1)", "A:across warps", "A:K1"}))
    out.append(("ends T 64 K 33", 64, 33, _fill_groups(64, [[0, 63]]), {"A:(0,T-1)", "A:across warps", "A:K33"}))
    out.append(("(t, t+32) T 64", 64, 1, [[t, t + 32] for t in range(32)], {"A:(t,t+32)", "A:across warps", "A:K1"}))
    out.append(("(t, t+32) T 64 K 2", 64, 2, [[t, t + 32] for t in range(32)], {"A:(t,t+32)", "A:across warps", "A:K2"}))
    out.append(("(t, t+32, t+64) T 96", 96, 1, [[t, t + 32, t + 64] for t in range(32)], {"A:(t,t+32)", "A:across warps", "A:K1"}))
    out.append(("(31, 32), (0, 64) T 65", 65, 1, _fill_groups(65, [[31, 32], [0, 64]]), {"A:(0,T-1)", "A:across warps", "A:K1"}))
    out.append(("one group T 40 K 512", 40, 512, [list(range(40))], {"A:one group", "A:K512"}))
    out.append(("(t, t+1024), (0, T-1) T 1056", 1056, 1, _fill_groups(1056, [[0, 1055]] + [[t, t + 1024] for t in range(1, 31)]),
                {"A:(0,T-1)", "A:(t,t+1024)", "A:across the second fold level", "A:K1"}))
    return out


def craft(keys: Keys, rng, T, K, groups, seed, tag):
    """A batch in which every tuple has a defect e_t != 0 (sigma_t = a_t + e_t) and every group's sum of r_t e_t is
    0 mod R under `seed`: random defects, the last member of each group solved."""
    assert sorted(t for g in groups for t in g) == list(range(T)) and all(len(g) >= 2 for g in groups), tag
    r = [rlc_scalar(seed, t) for t in range(T)]
    tup = [None] * T
    for gi, g in enumerate(groups):
        msg = hashlib.sha256(b"rlc soak A %s %d" % (tag.encode(), gi)).digest()
        ks = {t: tuple(keys.seq[int(i)] for i in rng.integers(0, keys.n, K)) for t in g}
        while True:
            e = {t: _nz(rng) for t in g[:-1]}
            e[g[-1]] = (-sum(r[t] * e[t] for t in g[:-1]) * pow(r[g[-1]], -1, R)) % R
            if e[g[-1]] and all((sum(ks[t]) + e[t]) % R for t in g):   # redraw a zero defect or a zero sigma
                break
        for t in g:
            tup[t] = Tup(msg, ks[t], (sum(ks[t]) + e[t]) % R)
    return tup


def resolve_trunc32(batch, groups, seed):
    """The same batch with each group's last defect solved for r_t mod 2^32 (what a kernel that truncated its scalars
    to 32 bits would accept) instead of r_t."""
    r = [rlc_scalar(seed, t) & 0xFFFFFFFF or 1 for t in range(len(batch))]
    out = list(batch)
    for g in groups:
        j = g[-1]
        ej = (-sum(r[t] * batch[t].defect for t in g[:-1]) * pow(r[j], -1, R)) % R
        out[j] = Tup(batch[j].msg, batch[j].keys, (batch[j].a + ej) % R)
    return out


def _seed_controls(seed):
    flip = bytearray(seed); flip[31] ^= 1
    swap = b"".join(seed[i:i + 4][::-1] for i in range(0, 32, 4))
    others = [hashlib.sha256(b"rlc soak other seed").digest(), bytes(flip)]
    others.append(ZERO_SEED if seed != ZERO_SEED else SEED)
    if swap != seed:
        others.append(swap)
    return others


def family_a(keys: Keys, rng):
    cases = []
    specs = [(n, T, K, g, tags, SEED) for n, T, K, g, tags in a_layouts()]
    specs += [(n + " [zero seed]", T, K, g, tags | {"A:zero seed"}, ZERO_SEED) for n, T, K, g, tags in a_layouts()
              if n in ("ends T 2 K 1", "(t, t+32) T 64")]
    for name, T, K, groups, tags, seed in specs:
        batch = craft(keys, rng, T, K, groups, seed, name)
        tags = set(tags) | {"A:crafted"}
        runs = [(seed, True)] + [(s, model(batch, s)) for s in _seed_controls(seed)] + [(None, False)]
        cases.append(Case(f"A {name}", "A", batch, runs, tags))
        tb = resolve_trunc32(batch, groups, seed)
        cases.append(Case(f"A {name}: crafted with r mod 2^32", "A", tb, [(seed, model(tb, seed))], {"A:control trunc32"}))
        i, j = groups[0][0], (groups[1][0] if len(groups) > 1 else groups[0][-1])
        sw = list(batch); sw[i], sw[j] = sw[j], sw[i]
        cases.append(Case(f"A {name}: tuples {i} and {j} swapped", "A", sw, [(seed, model(sw, seed))], {"A:control swap"}))
        last = groups[0][-1]
        d1 = list(batch); d1[last] = Tup(batch[last].msg, batch[last].keys, (batch[last].sigma + 1) % R)
        cases.append(Case(f"A {name}: one defect + 1", "A", d1, [(seed, model(d1, seed))], {"A:control defect+1"}))
    # an infinity signature (sigma = 0, defect -a) cancelled by its group partner
    k = keys.seq[5]
    r0, r1 = rlc_scalar(SEED, 0), rlc_scalar(SEED, 1)
    e1 = (r0 * k * pow(r1, -1, R)) % R            # r0 (0 - k) + r1 e1 = 0
    msg = hashlib.sha256(b"rlc soak A infinity signature").digest()
    b = [Tup(msg, (k,), 0), Tup(msg, (keys.seq[6],), (keys.seq[6] + e1) % R)]
    cases.append(Case("A infinity signature cancelled", "A", b, [(SEED, True)] + [(s, model(b, s)) for s in _seed_controls(SEED)]
                      + [(None, False)], {"A:crafted", "A:infinity signature"}))
    return cases


# ------------------------------------------------------------------------------------------------ family B
def fold_ops(n):
    """The G2 fold of k_rlc_reduce over n points, launch after launch (warps of 32, lane l adds lane l + s for s = 16 ..
    1), as [(level, warp, s, lane, left tuple indices, right tuple indices)] for every jac_add it performs."""
    cur, ops, level = [[t] for t in range(n)], [], 0
    while True:
        level += 1
        nxt = []
        for w in range((len(cur) + 31) // 32):
            lanes = [list(cur[32 * w + l]) if 32 * w + l < len(cur) else [] for l in range(32)]
            for s in (16, 8, 4, 2, 1):
                for l in range(s):
                    ops.append((level, w, s, l, tuple(lanes[l]), tuple(lanes[l + s])))
                    lanes[l] = lanes[l] + lanes[l + s]
            nxt.append(lanes[0])
        cur = nxt
        if len(cur) <= 1:
            return ops


def _solve(batch, seed, left, right, sign, keys: Keys):
    """Replace the last tuple of `right` (valid, key = sigma) so that the right operand is sign * the left one."""
    c = lambda t: rlc_scalar(seed, t) * batch[t].sigma   # noqa: E731
    j = max(right)
    cj = (sign * sum(c(t) for t in left) - sum(c(t) for t in right if t != j)) % R
    sj = (cj * pow(rlc_scalar(seed, j), -1, R)) % R
    assert sj, "degenerate solve"
    out = list(batch)
    out[j] = Tup(batch[j].msg, (sj,), sj)
    return out


def b_targets():
    """(name, T, level, warp, s, lane, sign, tags); sign +1: equal operands (doubling), -1: opposite (infinity)."""
    out = []
    for sign, what in ((1, "equal"), (-1, "opposite")):
        for s in (16, 8, 4, 2, 1):
            out.append((f"{what} at distance {s}, T {2 * s}", 2 * s, 1, 0, s, 0, sign, {f"B:level1 s{s}", f"B:{what}"}))
            out.append((f"{what} partials at distance {s}, T 32, lane {s - 1}", 32, 1, 0, s, s - 1, sign, {f"B:level1 s{s}", f"B:{what}"}))
        out.append((f"{what} at distance 16 in warp 1, T 64", 64, 1, 1, 16, 5, sign, {"B:level1 s16", f"B:{what}"}))
        out.append((f"{what} warp partials, T 64", 64, 2, 0, 1, 0, sign, {"B:level2", f"B:{what}"}))
        out.append((f"{what} warps 0 and 16, T 1024", 1024, 2, 0, 16, 0, sign, {"B:level2", f"B:{what}"}))
        out.append((f"{what} 1024-blocks, T 2048", 2048, 3, 0, 1, 0, sign, {"B:level3", f"B:{what}"}))
        out.append((f"{what} 1024-block and 32-tail, T 1056", 1056, 3, 0, 1, 0, sign, {"B:level3", f"B:{what}"}))
    return out


def family_b(keys: Keys, base):
    cases = []
    def add(name, batch, tags):
        # the defect rides on the key of a tuple outside the solved one, so the G2 fold (signatures) is unchanged
        cases.append(Case(f"B {name}", "B", batch, [(SEED, model(batch, SEED))], tags | {"B:valid"}))
        d = list(batch); k = d[0]
        d[0] = Tup(k.msg, ((k.a + 1) % R,), k.sigma)
        cases.append(Case(f"B {name} + one defect", "B", d, [(SEED, model(d, SEED))], tags | {"B:defect"}))
    for name, T, level, w, s, lane, sign, tags in b_targets():
        batch = [base[t % N_POOL] for t in range(T)]
        op = next(o for o in fold_ops(T) if o[:4] == (level, w, s, lane))
        assert op[4] and op[5], name
        add(name, _solve(batch, SEED, op[4], op[5], sign, keys), tags)
    for T in (2, 32, 33, 1025, 2048):                     # S = sum r_t sig_t = infinity
        batch = [base[t % N_POOL] for t in range(T)]
        add(f"S = infinity, T {T}", _solve(batch, SEED, tuple(range(T - 1)), (T - 1,), -1, keys), {"B:S=inf"})
    return cases


# ------------------------------------------------------------------------------------------------ family C
def c_positions(T):
    if T in SMALL_T:
        return list(range(T))
    ps = {0, T - 1}
    for w in range((T + 31) // 32):
        ps |= {32 * w, min(32 * w + 31, T - 1)}
    return sorted(ps)


def dead_tuple(keys: Keys, kind):
    s = keys.seq[7]
    return Tup(MSG, () if kind == "empty" else (s,), s, kind)


def family_c(keys: Keys, base, scale=1.0):
    """All-valid batches of every size, and one invalid tuple (a defect, or dead) at every position that matters."""
    cases = []
    bad = Tup(MSG, (keys.seq[3],), (keys.seq[3] + 1) % R)
    for T in SMALL_T + LARGE_T:
        batch = [base[t % N_POOL] for t in range(T)]
        tags = {f"C:T{T}"}
        cases.append(Case(f"C T {T} all valid", "C", batch, [(SEED, True)], tags | {"C:valid"}))
        ps = c_positions(T)
        if scale < 1 and T in LARGE_T:
            ps = sorted({ps[0], ps[-1]} | set(ps[::max(1, int(round(1 / scale)))]))
        for i, p in enumerate(ps):
            for what, tup in (("defect", bad), ("dead", dead_tuple(keys, DEAD_KINDS[i % len(DEAD_KINDS)]))):
                b = list(batch); b[p] = tup
                cases.append(Case(f"C T {T} {what} at {p}", "C", b, [(SEED, False)], tags | {f"C:{what}"}))
    return cases


# ------------------------------------------------------------------------------------------------ bytes
class Material:
    """Encodes distinct tuples once: key bytes (Keys), signatures (one orc_sign_batch over every missing (sigma, msg)),
    per-point failures, and the C oracle's per-tuple code."""

    def __init__(self, O, keys: Keys):
        self.O, self.keys = O, keys
        self.sig = {}
        self.pks = {}
        self.code = {}

    def prepare(self, tuples):
        need = sorted({(t.sigma, t.msg) for t in tuples if (t.sigma, t.msg) not in self.sig and t.sigma})
        if need:
            sks = np.frombuffer(b"".join(s.to_bytes(32, "big") for s, _ in need), dtype=np.uint8).copy()
            ms = np.frombuffer(b"".join(m for _, m in need), dtype=np.uint8).copy()
            out = np.empty((len(need), 96), dtype=np.uint8)
            self.O.orc_sign_batch(sks.ctypes.data, ms.ctypes.data, len(need), out.ctypes.data, os.cpu_count() or 8)
            for k, row in zip(need, out):
                self.sig[k] = row.tobytes()

    def encode(self, t: Tup):
        """(keys bytes, msg, sig bytes) of tuple t."""
        pks = b"".join(self.keys.get(s) for s in t.keys)
        sig = self.sig[(t.sigma, t.msg)] if t.sigma else INF_G2
        if t.dead == "inf_key":
            pks = INF_G1 + pks[48:]
        elif t.dead == "sig_encoding":
            sig = mutate(sig, 96, 2, None)
        elif t.dead == "sig_x":
            sig = mutate(sig, 96, 4, None)
        return pks, t.msg, sig

    def codes(self, tuples):
        """The C oracle's fast_aggregate_verify code of each tuple (computed once per distinct tuple)."""
        todo = list(dict.fromkeys(t for t in tuples if t not in self.code))
        if todo:
            self.prepare(todo)
            enc = [self.encode(t) for t in todo]
            pks = np.frombuffer(b"".join(e[0] for e in enc), dtype=np.uint8).copy()
            off = np.cumsum([0] + [len(e[0]) // 48 for e in enc]).astype(np.uint32)
            ms = np.frombuffer(b"".join(e[1] for e in enc), dtype=np.uint8).copy()
            sg = np.frombuffer(b"".join(e[2] for e in enc), dtype=np.uint8).copy()
            out = np.empty(len(todo), dtype=np.int32)
            self.O.orc_fast_aggregate_verify_batch(pks.ctypes.data if pks.size else 0, off.ctypes.data, ms.ctypes.data, sg.ctypes.data,
                                                   len(todo), out.ctypes.data, os.cpu_count() or 8)
            self.code.update(zip(todo, out.tolist()))
        return [self.code[t] for t in tuples]

    def pack(self, batch):
        """The batch entry points' flat arrays."""
        self.prepare(batch)
        enc = [self.encode(t) for t in batch]
        pks = np.frombuffer(b"".join(e[0] for e in enc), dtype=np.uint8)
        off = np.cumsum([0] + [len(e[0]) // 48 for e in enc]).astype(np.uint32)
        msgs = np.frombuffer(b"".join(e[1] for e in enc), dtype=np.uint8)
        sigs = np.frombuffer(b"".join(e[2] for e in enc), dtype=np.uint8)
        return pks, off, msgs, sigs


def oracle_rlc(O, M: Material, batch, seed, t0=0) -> bool:
    """The RLC restated for the oracle's own pairing: aggregate_verify([sk_to_pk(r_t a_t)], [m_t],
    aggregate([sign(r_t sigma_t, m_t)])).  Dead tuples fail their per-point checks, so the batch is then False."""
    if any(t.dead for t in batch):
        return False
    r = [rlc_scalar(seed, t0 + i) for i in range(len(batch))]
    pks = b"".join(M.keys.get((ri * t.a) % R) for ri, t in zip(r, batch))
    scaled = [Tup(t.msg, (), (ri * t.sigma) % R) for ri, t in zip(r, batch)]
    M.prepare(scaled)
    sigs = b"".join(M.sig[(s.sigma, s.msg)] if s.sigma else INF_G2 for s in scaled)
    agg = ctypes.create_string_buffer(96)
    assert O.orc_aggregate(sigs, len(batch), agg) == 0
    msgs = [t.msg for t in batch]
    arr = (ctypes.c_char_p * len(msgs))(*msgs)
    ln = (ctypes.c_size_t * len(msgs))(*[32] * len(msgs))
    rc = O.orc_aggregate_verify(pks, len(batch), ctypes.cast(arr, ctypes.c_void_p), ctypes.cast(ln, ctypes.c_void_p), len(msgs), agg.raw)
    assert rc in (0, 5), rc
    return rc == 0


def all_cases(O, scale=1.0):
    """(keys, material, cases of A, B, C) for one fixed rng."""
    rng = np.random.default_rng(0x41C)
    keys = Keys(O)
    base = pool(keys)
    return keys, Material(O, keys), {"A": family_a(keys, rng), "B": family_b(keys, base), "C": family_c(keys, base, scale)}
