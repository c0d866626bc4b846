"""Case lists of the sharded entry points at world > 1, shared by the CPU census (tests/test_sharded_cases.py) and the
multi-process device test (tests/test_sharded_loopback_gpu.py, one rank per process in tests/mp_loopback_worker.py).
No device code.

Every case sits on the rank boundaries of the split it exercises:
* strict verify (`b200_fast_aggregate_verify_batch_sharded`): T around world and around the padded block length, ragged
  K with K = 0 tuples and whole zero-key rank blocks, an invalid tuple of every reject class at the first and the last
  position of every rank's block; expected codes from the C oracle;
* RLC (`b200_fast_aggregate_verify_batch_all_sharded`): defects that cancel only across a rank boundary (so two ranks'
  Gt partials are inverse), a rank whose scaled signatures sum to infinity, a dead tuple at every rank's ends; verdicts
  from rlc_soak_cases.model with the GLOBAL tuple index, and every crafted batch False under the per-rank local index;
* states (`b200_htr_beacon_state_deneb_sharded`, `b200_state_upload_deneb_sharded`): lists shorter than world, the
  planner boundaries of ssz_soak_cases, eth1_data_votes and extra_data at both ends; roots from the C oracle;
* refusals every rank must return alike, before any exchange.
`O` is the C BLS oracle and `OS` the C SSZ oracle (oracle/c), loaded through ctypes."""
from __future__ import annotations

import ctypes
import hashlib
import os
import pickle
from pathlib import Path

import numpy as np

from ethereum_consensus_b200 import parallel, state as S
from tests import rlc_soak_cases as rc
from tests import ssz_soak_cases as sc
from tests.bls_soak_cases import R, mutate

WORLDS = (2, 3, 4, 5, 8)
STATE_WORLDS = (2, 4, 8)                 # the state root exists at powers of two only
# loopback file (csrc/comm_loopback.h): 64-byte header, then two generations of world x SLOT_BYTES slots
HEADER_BYTES = 64
SLOT_BYTES = 1 << 20                     # the largest exchange is the 1 MiB b200_comm_all_gather_bytes call
TIMEOUT_MS = 60_000
RLC_PART = 576 + 16                      # one rank's RLC exchange: the Gt partial, then the bad flag (16 bytes)
MAX_TUPLES = 1 << 26                     # kMaxBatchTuples
GATHER_BYTES = (0, 1, 15, 16, 17, 1 << 20)
# the reject classes of the soak: key encoding, key outside the group, infinity key, signature encoding, signature off the
# curve, signature outside the group, a defect, no keys.  fast_aggregate_verify answers VERIFY_FAIL for the last three
# (EMPTY_AGGREGATE is an aggregate-call code), which the census pins.
BAD_KINDS = ("key_encoding", "key_group", "inf_key", "sig_encoding", "sig_curve", "sig_x", "defect", "empty")
KIND_CODE = {"": 0, "key_encoding": 1, "key_group": 3, "inf_key": 6, "sig_encoding": 1, "sig_curve": 2, "sig_x": 5, "defect": 5,
             "empty": 5}
N_STRICT_POOL = 48
ERR_BAD_ARG, ERR_SSZ_MALFORMED = 0x102, 0x103


def c_tuple_shard(n, world, rank):
    """csrc/capi_bls.cu tuple_shard, restated: (lo, cnt)."""
    base, rem = n // world, n % world
    return rank * base + min(rank, rem), base + (1 if rank < rem else 0)


def c_slice_of(n, world, rank):
    """csrc/ssz_plan.cu slice_of, restated: (first, count, k)."""
    per = (n + world - 1) // world
    k = 0
    while (1 << k) < (per if per else 1):
        k += 1
    s = 1 << k
    lo, hi = min(n, s * rank), min(n, s * (rank + 1))
    return lo, hi - lo, k


def blocks(T, world):
    """[(lo, hi)] of every rank (parallel.tuple_shard)."""
    return [parallel.tuple_shard(T, world, r) for r in range(world)]


def rank_ends(T, world):
    """The first and last position of every non-empty rank block, and 0 and T - 1."""
    ps = {0, T - 1}
    for lo, hi in blocks(T, world):
        if hi > lo:
            ps |= {lo, hi - 1}
    return sorted(ps)


# ------------------------------------------------------------------------------------------------ tuples
class Material(rc.Material):
    """rlc_soak_cases.Material with three more reject classes: a bad key encoding, a key outside the group and a
    signature off the curve."""

    def __init__(self, O, keys):
        super().__init__(O, keys)
        self.off_group = _off_group_key(O, keys.get(keys.seq[0]))
        self.off_curve = {}

    def encode(self, t):
        pks, msg, sig = super().encode(t)
        if t.dead == "key_encoding":
            pks = mutate(pks[:48], 48, 2, None) + pks[48:]
        elif t.dead == "key_group":
            pks = self.off_group + pks[48:]
        elif t.dead == "sig_curve":
            if sig not in self.off_curve:
                self.off_curve[sig] = _off_curve_sig(self.O, sig)
            sig = self.off_curve[sig]
        return pks, msg, sig


def _off_group_key(O, valid: bytes) -> bytes:
    """The first x above a valid key's x that is on the curve: a point outside the prime-order subgroup."""
    x = int.from_bytes(valid, "big") & ((1 << 381) - 1)
    for dx in range(1, 200):
        enc = ((0b100 << 381) | (x + dx)).to_bytes(48, "big")
        if O.orc_key_validate(enc) == 3:
            return enc
    raise AssertionError("no on-curve neighbour found")


def _off_curve_sig(O, sig: bytes) -> bytes:
    """The signature with the low byte of x.c0 moved until the point is off the curve (the oracle answers 2)."""
    pk = bytes(48)
    for dx in range(1, 256):
        enc = sig[:95] + bytes([(sig[95] + dx) & 0xff])
        if O.orc_fast_aggregate_verify(pk, 0, bytes(32), 32, enc) == 2:
            return enc
    raise AssertionError("no off-curve neighbour found")


def bad_tuple(keys, kind):
    s = keys.seq[7]
    if kind == "defect":
        return rc.Tup(rc.MSG, (keys.seq[3],), (keys.seq[3] + 1) % R)
    return rc.Tup(rc.MSG, () if kind == "empty" else (s,), s, kind)


def strict_pool(keys):
    """N_STRICT_POOL valid tuples with K = 1 .. 4 keys and their own messages."""
    rng = np.random.default_rng(0x5A7)
    out = []
    for i in range(N_STRICT_POOL):
        ks = tuple(keys.seq[int(j)] for j in rng.integers(0, keys.n, 1 + i % 4))
        out.append(rc.Tup(hashlib.sha256(b"sharded strict %d" % i).digest(), ks, sum(ks) % R))
    return out


def strict_sizes(world):
    return sorted({1, world - 1, world, world + 1, 2 * world - 1, 1023, 1025, 4097} - {0})


def strict_cases(keys, world):
    """[(name, batch, kinds)]: kinds[t] is the reject class placed at t ("" valid)."""
    pool = strict_pool(keys)
    out = []
    for T in strict_sizes(world):
        kinds = ["empty" if t % 53 == 17 else "" for t in range(T)]   # ragged K, with K = 0 tuples inside blocks
        for i, p in enumerate(rank_ends(T, world)):
            kinds[p] = BAD_KINDS[(i + T) % len(BAD_KINDS)]
        out.append((f"w{world} T {T}: a reject at every rank's ends", kinds))
        if T >= world:
            lo, hi = parallel.tuple_shard(T, world, world // 2)
            kz = ["" for _ in range(T)]
            for t in range(lo, hi):
                kz[t] = "empty"
            if lo > 0:
                kz[0] = "defect"
            if hi < T:
                kz[T - 1] = "sig_encoding"
            out.append((f"w{world} T {T}: rank {world // 2}'s block has no keys", kz))
    cases = []
    for name, kinds in out:
        batch = [bad_tuple(keys, k) if k else pool[(7 * t) % N_STRICT_POOL] for t, k in enumerate(kinds)]
        cases.append((name, batch, kinds))
    return cases


# ------------------------------------------------------------------------------------------------ RLC
def model_local(batch, seed, world):
    """The verdict if every rank scaled its block with its LOCAL index (the t0 mutant of k_rlc_scale)."""
    if any(t.dead for t in batch):
        return False
    acc = {}
    for lo, hi in blocks(len(batch), world):
        for i in range(lo, hi):
            t = batch[i]
            acc[t.msg] = (acc.get(t.msg, 0) + rc.rlc_scalar(seed, i - lo) * (t.sigma - t.a)) % R
    return all(v == 0 for v in acc.values())


def _groups(T, pairs):
    """The pairs merged where they share a position, then every other position in groups of two or three."""
    parent = list(range(T))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b in pairs:
        parent[find(a)] = find(b)
    comp = {}
    for a, b in pairs:
        for x in (a, b):
            comp.setdefault(find(x), set()).add(x)
    return rc._fill_groups(T, [sorted(g) for g in comp.values()])


def _cancel_pair(keys, rng, batch, i, j, seed):
    """Defects at i and j (same message) with r_i e_i + r_j e_j = 0 under `seed`."""
    out = list(batch)
    ei = rc._nz(rng)
    ej = (-rc.rlc_scalar(seed, i) * ei * pow(rc.rlc_scalar(seed, j), -1, R)) % R
    for t, e in ((i, ei), (j, ej)):
        out[t] = rc.Tup(batch[t].msg, batch[t].keys, (batch[t].a + e) % R)
    return out


def rlc_cases(keys, world):
    """[rc.Case] with tags naming the rank boundary each case sits on; runs: the crafting seed and four others."""
    rng = np.random.default_rng(0x5A8 + world)
    base = rc.pool(keys)
    seeds = [rc.SEED] + rc._seed_controls(rc.SEED)
    cases = []

    def add(name, batch, tags):
        cases.append(rc.Case(name, "sharded", batch, [(s, rc.model(batch, s)) for s in seeds], set(tags)))

    for T in (world, 2 * world + 1):
        bl = blocks(T, world)
        pairs = [(bl[r][1] - 1, bl[r][1]) for r in range(world - 1)] + [(0, T - 1)]
        batch = rc.craft(keys, rng, T, 1, _groups(T, pairs), rc.SEED, f"sharded w{world} T{T}")
        add(f"w{world} A T {T}: groups across every rank boundary", batch,
            {"crafted"} | {f"straddle {r}" for r in range(world - 1)} | {"straddle 0,last"} | ({"T = world"} if T == world else set()))
    T = 2 * world + 1
    bl = blocks(T, world)
    valid = [base[t] for t in range(T)]
    for r in range(world - 1):
        i, j = bl[r][1] - 1, bl[r + 1][0]
        add(f"w{world} T {T}: partials of ranks {r} and {r + 1} inverse", _cancel_pair(keys, rng, valid, i, j, rc.SEED),
            {"crafted", f"inverse {r},{r + 1}"})
    add(f"w{world} T {T}: partials of ranks 0 and {world - 1} inverse", _cancel_pair(keys, rng, valid, 0, T - 1, rc.SEED),
        {"crafted", "inverse 0,last"})
    for r in (0, world - 1):
        lo, hi = bl[r]
        add(f"w{world} T {T}: rank {r}'s scaled signatures sum to infinity",
            rc._solve(valid, rc.SEED, tuple(range(lo, hi - 1)), (hi - 1,), -1, keys), {"valid", f"S_{r} = inf"})
    for r in range(world):
        lo, hi = bl[r]
        for end, p in (("first", lo), ("last", hi - 1)):
            kind = rc.DEAD_KINDS[(2 * r + (end == "last")) % len(rc.DEAD_KINDS)]
            b = list(valid)
            b[p] = rc.dead_tuple(keys, kind)
            add(f"w{world} T {T}: {kind} tuple at rank {r}'s {end}", b, {"dead", f"dead {r} {end}"})
    return cases


# ------------------------------------------------------------------------------------------------ states
def state_specs():
    """Whole states for the sharded root, both presets."""
    m, M = "minimal", "mainnet"
    mb, Mb = S.PRESETS[m]["ETH1_DATA_VOTES_BOUND"], S.PRESETS[M]["ETH1_DATA_VOTES_BOUND"]
    H, C = sc.HANDOFF, sc.COOP_MAX
    rows = [  # preset, validators, historical_roots, historical_summaries, eth1 votes, extra_data length
        (m, 1, 2, 3, 0, 0), (m, 5, 0, 0, mb, 32), (m, H, 3, 2, 0, 32), (m, H + 1, 65, 64, mb, 0),
        (m, 4 * H, 0, 3, 1, 0), (m, 4 * H + 1, 2, 0, mb, 32), (m, 32 * H, 3, 3, 0, 32), (m, 32 * H + 1, 64, 65, mb, 0),
        (M, 0, 0, 0, 0, 0), (M, 1, 2, 3, Mb, 32), (M, 3, 0, 0, 0, 32), (M, H, 1, 1, Mb, 0), (M, H + 1, 2, 2, 0, 0),
        (M, 70_001, 3, 2, 7, 31), (M, C - 1, 2, 3, Mb, 32), (M, C + 1, 3, 2, 0, 0),
        (M, 4 * C - 4, 2, 2, 0, 32), (M, 4 * C + 4, 1, 1, Mb, 0),
    ]
    return [dict(name=f"{p}:{n}:v{v}:x{x}", preset=p, n=n, hr=hr, hs=hs, votes=v, extra=bytes((5 * j + 1) & 0xff for j in range(x)),
                 seed=0x5AB0 + i) for i, (p, n, hr, hs, v, x) in enumerate(rows)]


def state_list_lengths(spec):
    """Element counts the sharded plan splits: validators, then the chunks of balances, both participations, inactivity."""
    n = spec["n"]
    return [n, (8 * n + 31) // 32, (n + 31) // 32, (n + 31) // 32, (8 * n + 31) // 32]


def oracle_root(OS, ser, preset):
    out = ctypes.create_string_buffer(32)
    assert OS.orc_htr_beacon_state_deneb(ser.ctypes.data, len(ser), {"mainnet": 0, "minimal": 1}[preset], os.cpu_count() or 8, out) == 0
    return out.raw


def malformed_state():
    """One rejected encoding of ssz_soak_cases.malformed_cases (an offset below its predecessor)."""
    name, preset, b, ok = next(c for c in sc.malformed_cases() if c[0] == "minimal: offset 3 below offset 2")
    assert not ok
    return preset, b


# ------------------------------------------------------------------------------------------------ refusals
def refusals(world):
    """(name, expected code) of every refusal the worker makes, in its order."""
    out = [("strict: decreasing offsets", ERR_BAD_ARG), ("strict: n_tuples > 2^26", ERR_BAD_ARG),
           ("rlc: decreasing offsets", ERR_BAD_ARG), ("rlc: n_tuples > 2^26", ERR_BAD_ARG),
           ("rlc: NULL seed", ERR_BAD_ARG), ("rlc: T < world", ERR_BAD_ARG),
           ("htr sharded: malformed state", ERR_SSZ_MALFORMED), ("upload sharded: malformed state", ERR_SSZ_MALFORMED)]
    if world & (world - 1):
        out += [(f"htr sharded: world {world}", ERR_BAD_ARG), (f"upload sharded: world {world}", ERR_BAD_ARG)]
    else:
        out += [("update_bytes on a sharded handle", ERR_BAD_ARG), ("update_elements on a sharded handle", ERR_BAD_ARG),
                ("registry_load_state on a sharded handle", ERR_BAD_ARG),
                ("state_root on a sharded handle after the communicator became world 1", ERR_BAD_ARG)]
    return out


# ------------------------------------------------------------------------------------------------ what a worker reads
def gather_payload(rank, nbytes):
    return hashlib.shake_256(b"gather %d %d" % (rank, nbytes)).digest(nbytes) if nbytes else b""


def gather_codes(rank):
    return np.array([1000 * rank + k for k in range(5)], dtype=np.int32)


def _pack(M, batch):
    return [np.ascontiguousarray(a).copy() for a in M.pack(batch)]


def write_cases(box: Path, world: int, O, OS, shared=None) -> dict:
    """Writes box/cases.pkl (and the serialized states as .npy) for one world and returns the expected values.
    `shared`: a dict kept across calls so keys, signatures, oracle codes and state roots are made once."""
    shared = {} if shared is None else shared
    if "M" not in shared:
        keys = rc.Keys(O)
        shared["keys"], shared["M"] = keys, Material(O, keys)
    keys, M = shared["keys"], shared["M"]
    strict = []
    for name, batch, kinds in strict_cases(keys, world):
        strict.append(dict(name=name, args=_pack(M, batch), want=M.codes(batch)))
    rlc = []
    for c in rlc_cases(keys, world):
        rlc.append(dict(name=c.name, args=_pack(M, c.batch), runs=c.runs))
    states = []
    if world in STATE_WORLDS or world == 1:
        roots = shared.setdefault("roots", {})
        for i, spec in enumerate(state_specs()):
            path = box.parent / f"state_{spec['name'].replace(':', '_')}.npy"
            if spec["name"] not in roots:
                ser = sc.serialized(spec)
                np.save(path, ser)
                roots[spec["name"]] = oracle_root(OS, ser, spec["preset"])
            states.append(dict(name=spec["name"], preset=spec["preset"], path=str(path), want=roots[spec["name"]],
                               resident=i % 3 == 0))
    preset, bad = malformed_state()
    good = sc.serialized(state_specs()[0])
    data = dict(world=world, strict=strict, rlc=rlc, states=states, malformed=(preset, bad), small_state=(state_specs()[0]["preset"], good),
                refusals=refusals(world), gather=list(GATHER_BYTES))
    box.mkdir(parents=True, exist_ok=True)
    (box / "cases.pkl").write_bytes(pickle.dumps(data))
    return data
