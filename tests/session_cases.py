"""A seeded session of one long-lived engine: every entry-point family interleaved (no device code, no torch).

A session is a list of `Step`s.  Each step names one entry point and its arguments, the answer the library must give
(computed here from the oracles: liboracle_bls.so, liboracle_ssz.so, oracle/shuffle_oracle.py, the Python tower of
tests/pairing_cases.py) or the refusal code it must answer, and the resident objects it reads or changes ("state": the
resident BeaconState handle, "registry": the validated-key registry, "knobs": launch-shape knobs and the pairing-VM
schedule).  tests/test_engine_session_gpu.py runs the list through the CUDA library in script order, in a shuffled order
that keeps dependent steps in order, without the pairing VM and from worker threads; tests/test_session_cases.py checks
the list itself on the CPU (its census of transitions, and that the expected answers agree with each other).

What the order is for: the engine's scratch buffers are process-global and grow-only, several families share them, and
some per-call slots sit behind data another call owns.  So the session grows each shared buffer and shrinks it on the
very next call of a family that uses it, crosses the launch-shape thresholds of the strict batch, changes knobs and the
VM schedule in the middle, and follows every refusal kind with a step of the same family.

Sizes scale with B200_SOAK_SCALE (chain length, batch repeats); the thresholds named below are crossed at every scale.
Distinct keys and signatures are few (POOL keys, tiled): the oracle only ever sees the small batches that big ones repeat.
"""
from __future__ import annotations

import copy
import ctypes
import hashlib
import os
import random
import subprocess
import sys
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, List

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import state as S  # noqa: E402
from oracle import bls_oracle as bo  # noqa: E402
from oracle import shuffle_oracle as sh  # noqa: E402
from tests import bls_soak_cases as bsc  # noqa: E402
from tests import ssz_soak_cases as sc  # noqa: E402
from tests import state_reshape_cases as rc  # noqa: E402

SCALE = float(os.environ.get("B200_SOAK_SCALE", "1"))
NT = os.cpu_count() or 1
R = bsc.R

# engine codes (include/b200_consensus.h)
ERR_BAD_ARG, ERR_SSZ_MALFORMED, ERR_LIMIT = 0x102, 0x103, 0x105

# launch-shape thresholds of the strict batch (capi_bls.cu key_phase, bls_g1.cu launch_g1_validate)
VM_TEAM16_MAX = 2048                      # default: Miller launches of up to 2 048 pairs run on 16-lane teams
SMALL_CTA_KEYS = 148 * 384                # n_keys >= 56 832 and T > 1 024: side kernels in 128-thread CTAs
K1_WIDE_KEYS = 170_496                    # above this, K1's first waves go from 128- to 384-thread CTAs
SPLIT_KEYS = 4 * 4 * 148 * 384            # n_keys >= 909 312: the key copy is split in two
REG_EXTRA = 1 << 16                       # registry extra-key tail (kRegistryExtraKeys)
HEADROOM_MIN = rc.HEADROOM_MIN            # reserved entries behind a resident list / the registry

POOL = 2000                               # distinct keys; the chain's validator i carries pool key i % POOL
POOL_INVALID = 400                        # of them rejected by key_validate (every class)
BIG_BLOCK = 80_000                        # one block's deposits: past both the state's and the registry's reserve

REFUSALS = ("offsets decrease", "index past registry + extras", "update_bytes moves an offset", "malformed set_field",
            "sync against a smaller state", "merkleize above its limit", "malformed one-shot state", "unknown curve_eval op")


def refused(code: int) -> tuple:
    return ("refused", int(code))


def digest(a) -> tuple:
    """Compact comparable form of a long answer: its length and SHA-256."""
    b = np.ascontiguousarray(a).tobytes() if not isinstance(a, (bytes, bytearray)) else bytes(a)
    return (len(a), hashlib.sha256(b).hexdigest())


@dataclass
class Step:
    family: str                  # strict | rlc | single | registry | state | ssz | shuffle | eval | settings
    op: str
    args: dict
    want: object                 # the answer, or ("refused", code)
    reads: frozenset = frozenset()
    writes: frozenset = frozenset()
    tags: tuple = ()
    i: int = -1

    def describe(self) -> str:
        def short(v):
            if isinstance(v, (bytes, bytearray)):
                return f"<{len(v)} B>"
            if isinstance(v, np.ndarray):
                return f"<{v.dtype}{list(v.shape)}>"
            if isinstance(v, (list, tuple)) and (len(v) > 6 or any(not isinstance(x, int) for x in v)):
                return f"<{type(v).__name__} of {len(v)}>"
            return repr(v)
        a = ", ".join(f"{k}={short(v)}" for k, v in self.args.items() if not k.startswith("_"))
        w = self.want if not isinstance(self.want, tuple) or len(self.want) <= 6 else f"<{len(self.want)} values>"
        return f"#{self.i} [{self.family}] {self.op}({a}) -> {w}" + (f"  {list(self.tags)}" if self.tags else "")


@dataclass
class Session:
    steps: List[Step]
    init_state: np.ndarray       # serialization the resident handle is uploaded from (minimal preset)
    meta: Dict[str, object] = field(default_factory=dict)


# ---------------------------------------------------------------------------------------------------------- oracles
def oracles():
    """(liboracle_bls.so, liboracle_ssz.so) through ctypes, built by oracle/Makefile if needed."""
    subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True, capture_output=True)
    B = ctypes.CDLL(str(ROOT / "oracle" / "liboracle_bls.so"))
    cp, sz, vp, I = ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int
    B.orc_fast_aggregate_verify.argtypes = [cp, sz, cp, sz, cp]
    B.orc_eth_fast_aggregate_verify.argtypes = [cp, sz, cp, sz, cp]
    B.orc_verify_signature.argtypes = [cp, cp, sz, cp]
    B.orc_aggregate_verify.argtypes = [cp, sz, vp, vp, sz, cp]
    B.orc_aggregate.argtypes = [cp, sz, cp]
    B.orc_eth_aggregate_public_keys.argtypes = [cp, sz, cp]
    B.orc_key_validate.argtypes = [cp]
    B.orc_fast_aggregate_verify_batch.argtypes = [vp, vp, vp, vp, sz, vp, I]
    B.orc_sign_batch.argtypes = [vp, vp, sz, vp, I]
    B.orc_pk_sequence.argtypes = [cp, cp, sz, vp]
    Z = ctypes.CDLL(str(ROOT / "oracle" / "liboracle_ssz.so"))
    Z.orc_merkleize.argtypes = [vp, sz, ctypes.c_uint64, I, vp]
    Z.orc_merkleize.restype = I
    Z.orc_htr_validators.argtypes = [vp, sz, ctypes.c_uint64, I, vp]
    Z.orc_htr_validators.restype = I
    Z.orc_htr_beacon_state_deneb.argtypes = [vp, sz, I, I, vp]
    Z.orc_htr_beacon_state_deneb.restype = I
    return B, Z


def state_root(Z, st: S.SynthState) -> bytes:
    b = S.serialize(st)
    out = ctypes.create_string_buffer(32)
    assert Z.orc_htr_beacon_state_deneb(b.ctypes.data, b.size, 0 if st.preset == "mainnet" else 1, NT, out) == 0
    return out.raw


# ---------------------------------------------------------------------------------------------------------- keys, tuples
class Pool:
    """POOL distinct 48-byte keys (POOL_INVALID of them rejected by key_validate), their codes and the secrets of the
    valid ones; key i of a tiled list is pool key i % POOL."""

    def __init__(self, B, seed=0x5E55):
        keys, sk0, d = bsc.valid_keys(B, POOL, seed)
        self.keys = keys.copy()
        self.sks = [(sk0 + i * d) % R for i in range(POOL)]
        rng = np.random.default_rng(seed)
        enc = [bytes(e) for e in bsc.g1_edge_encodings(keys[:4])] + [r.tobytes() for r in bsc.random_g1_encodings(rng, 600)]
        enc += [bsc.mutate(keys[i % 8].tobytes(), 48, k, rng) for i in range(8) for k in range(bsc.N_MUTATIONS)]
        bad = [e for e in enc if B.orc_key_validate(e) != 0]
        spots = rng.choice(np.arange(1, POOL), POOL_INVALID, replace=False)   # pool key 0 stays valid
        for j, p in enumerate(spots):
            self.keys[p] = np.frombuffer(bad[j % len(bad)], np.uint8)
            self.sks[p] = None
        self.codes = np.array([0 if s is not None else B.orc_key_validate(self.keys[i].tobytes()) for i, s in enumerate(self.sks)],
                              dtype=np.int32)
        assert {1, 2, 3, 6} <= set(self.codes.tolist()), sorted(set(self.codes.tolist()))
        self.valid = [i for i in range(POOL) if self.sks[i] is not None]

    def tiled(self, lo: int, n: int) -> np.ndarray:
        return self.keys[np.arange(lo, lo + n) % POOL]

    def tiled_codes(self, lo: int, n: int) -> np.ndarray:
        return self.codes[np.arange(lo, lo + n) % POOL]


def sign(B, sks, msgs) -> np.ndarray:
    n = len(sks)
    if n == 0:
        return np.zeros((0, 96), np.uint8)
    sk = np.frombuffer(b"".join(int(s if s else 1).to_bytes(32, "big") for s in sks), dtype=np.uint8).copy()
    m = np.frombuffer(b"".join(msgs), dtype=np.uint8).copy()
    out = np.empty((n, 96), dtype=np.uint8)
    B.orc_sign_batch(sk.ctypes.data, m.ctypes.data, n, out.ctypes.data, 8)
    return out


def oracle_codes(B, flat, off, msgs, sigs) -> tuple:
    flat, off = np.ascontiguousarray(flat, np.uint8), np.ascontiguousarray(off, np.uint32)
    msgs, sigs = np.ascontiguousarray(msgs, np.uint8), np.ascontiguousarray(sigs, np.uint8)
    t = len(off) - 1
    out = np.empty(max(t, 1), dtype=np.int32)
    B.orc_fast_aggregate_verify_batch(flat.ctypes.data, off.ctypes.data, msgs.ctypes.data, sigs.ctypes.data, t, out.ctypes.data, 8)
    return tuple(out[:t].tolist())


class Batch:
    """A strict batch (keys, offsets, messages, signatures) and its codes."""

    def __init__(self, flat, off, msgs, sigs, codes):
        self.flat = np.ascontiguousarray(flat, np.uint8).reshape(-1)
        self.off = np.ascontiguousarray(off, np.uint32)
        self.msgs = np.ascontiguousarray(msgs, np.uint8).reshape(-1)
        self.sigs = np.ascontiguousarray(sigs, np.uint8).reshape(-1)
        self.codes = tuple(codes)

    @property
    def T(self):
        return len(self.off) - 1

    @property
    def n_keys(self):
        return int(self.off[-1])

    def args(self):
        return dict(pks=self.flat, off=self.off, msgs=self.msgs, sigs=self.sigs)

    def tile(self, min_keys=0, min_t=0, exact_t=None):
        """Tuples t of the result are this batch's tuples t % T: the codes repeat the same way."""
        K = np.diff(self.off.astype(np.int64))
        if exact_t is not None:
            t = exact_t
        else:
            per = int(K.sum())
            reps = max(-(-min_keys // max(per, 1)), -(-min_t // self.T), 1)
            t = reps * self.T
            while t > self.T and int(np.sum(K[np.arange(t - 1) % self.T])) >= min_keys and t - 1 >= min_t:
                t -= 1
        src = np.arange(t) % self.T
        kk = K[src]
        off = np.concatenate([[0], np.cumsum(kk)]).astype(np.uint32)
        keys = self.flat.reshape(-1, 48)
        kidx = np.concatenate([np.arange(self.off[s], self.off[s + 1]) for s in src]) if off[-1] else np.zeros(0, np.int64)
        return Batch(keys[kidx], off, self.msgs.reshape(-1, 32)[src], self.sigs.reshape(-1, 96)[src],
                     [self.codes[s] for s in src])


def make_batch(B, pool: Pool, Ks, seed: int) -> Batch:
    """Tuples of the BLS soak's eight kinds (tests/bls_soak_cases.py tuple_case) over the pool's valid keys, K keys each
    (K = 0: an empty tuple); codes from the C oracle."""
    rng = np.random.default_rng(seed)
    vk, sk0, d = bsc.valid_keys(B, 256, 700 + seed % 97)
    cases = []
    for t, K in enumerate(Ks):
        if K == 0:
            m = hashlib.sha256(b"session/empty/%d/%d" % (seed, t)).digest()
            cases.append({"kind": -1, "K": 0, "pks": b"", "msg": m, "sk": (1).to_bytes(32, "big"), "sign_msg": m, "sig_mut": None})
        else:
            cases.append(bsc.tuple_case(vk, sk0, d, t + 1000 * seed, rng, K=K))
    sigs = sign(B, [int.from_bytes(c["sk"], "big") for c in cases], [c["sign_msg"] for c in cases])
    sigs = np.stack([np.frombuffer(bsc.finish_tuple(c, s.tobytes()), np.uint8) for c, s in zip(cases, sigs)])
    flat = np.frombuffer(b"".join(c["pks"] for c in cases), np.uint8)
    off = np.concatenate([[0], np.cumsum([len(c["pks"]) // 48 for c in cases])]).astype(np.uint32)
    msgs = np.frombuffer(b"".join(c["msg"] for c in cases), np.uint8)
    return Batch(flat, off, msgs, sigs, oracle_codes(B, flat, off, msgs, sigs))


def valid_batch(B, pool: Pool, T: int, seed: int, kmax=8, bad=()) -> Batch:
    """T tuples of valid pool keys signed correctly; tuples listed in `bad` carry the next tuple's signature."""
    rng = np.random.default_rng(seed)
    tups = [rng.choice(pool.valid, int(rng.integers(1, kmax + 1)), replace=False).tolist() for _ in range(T)]
    msgs = [hashlib.sha256(b"session/valid/%d/%d" % (seed, t)).digest() for t in range(T)]
    sigs = sign(B, [sum(pool.sks[i] for i in tp) % R for tp in tups], msgs)
    for t in bad:
        sigs[t] = sigs[(t + 1) % T]
    flat = pool.keys[np.concatenate([np.asarray(tp) for tp in tups])]
    off = np.concatenate([[0], np.cumsum([len(tp) for tp in tups])]).astype(np.uint32)
    m = np.frombuffer(b"".join(msgs), np.uint8)
    b = Batch(flat, off, m, sigs, oracle_codes(B, flat, off, m, sigs))
    b.tuples = tups
    return b


# ---------------------------------------------------------------------------------------------------------- the generator
class _Builder:
    def __init__(self):
        self.steps: List[Step] = []

    def add(self, family, op, args, want, reads=(), writes=(), tags=()):
        s = Step(family, op, dict(args), want, frozenset(reads), frozenset(writes), tuple(tags), len(self.steps))
        self.steps.append(s)
        return s


def strict(b: _Builder, batch: Batch, tags=()):
    return b.add("strict", "fast_aggregate_verify_batch", batch.args(), batch.codes, tags=tags)


def merkle_branch(rng, depth: int, ok: bool):
    leaf = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    branch = [rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(depth)]
    index = int(rng.integers(0, 1 << min(depth, 62))) | ((1 << 63) if depth == 64 else 0)
    v = leaf
    for i in range(depth):
        v = hashlib.sha256(branch[i] + v).digest() if (index >> i) & 1 else hashlib.sha256(v + branch[i]).digest()
    root = v if ok else bytes([v[0] ^ 1]) + v[1:]
    return dict(leaf=leaf, branch=branch, depth=depth, index=index, root=root)


def vm_blobs():
    """(alternative 8-lane schedule, default 8-lane, default 16-lane) as tools/gen_pairing_vm.py --blob writes them."""
    import tempfile
    out = []
    with tempfile.TemporaryDirectory() as d:
        for args in (("8", "--mix-light", "--heavy-min", "8"), ("8",), ("16",)):
            p = Path(d) / "prog.bin"
            subprocess.run([sys.executable, str(ROOT / "tools" / "gen_pairing_vm.py"), *args, "--blob", str(p)], check=True,
                           capture_output=True, cwd=ROOT)
            out.append(np.fromfile(p, dtype=np.uint32))
    return out


def _eval_rows(seed):
    """A few rows of fp_eval, curve_eval and pairing_eval with their answers (the helpers of the per-op device tests)."""
    from tests import pairing_cases as pc
    from tests import torsion_cases as tc
    rnd = random.Random(seed)
    P, RM = bo.P, 1 << 384
    rinv = pow(RM, -1, P)
    xs = [rnd.randrange(P) for _ in range(6)] + [0, 1, P - 1]
    ys = [rnd.randrange(P) for _ in range(6)] + [P - 1, P - 1, P - 1]
    fp = dict(op="fp_mul", a=xs, b=ys), tuple(x * y * rinv % P for x, y in zip(xs, ys))
    g = bo.G1_GEN
    pts = [bo.pt_to_affine(bo.F1, bo.pt_mul(bo.F1, bo.pt_from_affine(bo.F1, g), k)) for k in (1, 2, 12345)]
    pts += [tc.g1_random(rnd) for _ in range(3)]
    want = tuple(int(tc.mul(bo.F1, a, R) is None) for a in pts)
    cv = dict(op="g1l_in_subgroup", pts=pts), want
    pairs = pc.tower_pairs(seed, n_random=4)[:6]
    a = [x for x, _ in pairs]
    bb = [y for _, y in pairs]
    pw = tuple(tuple(pc.from_oracle(bo.f12_mul(pc.to_oracle(pc.to_real(x)), pc.to_oracle(pc.to_real(y))))) for x, y in zip(a, bb))
    pe = dict(op="fp12_mul", a=a, b=bb), pw
    return fp, cv, pe


def build_session(seed: int = 0x5E55, scale: float = SCALE) -> Session:
    B, Z = oracles()
    pool = Pool(B, seed)
    rng = np.random.default_rng(seed)
    b = _Builder()
    snapshots = []               # (index of a block's incremental-root step, the mirror then; None past the big block)
    n_blocks = max(4, int(round(6 * min(scale, 4))))
    big_at = n_blocks // 2

    # ---- the resident state and its registry
    n0 = 3000
    st = S.synth_state(n0, "minimal", seed=seed, n_eth1_votes=3, n_historical_summaries=2, pubkeys=pool.tiled(0, n0), extra_data=b"")
    init = S.serialize(st)
    b.add("state", "upload", {}, None, writes={"state"})
    b.add("state", "state_root", {}, state_root(Z, st), reads={"state"})
    b.add("registry", "from_state", {}, n0, reads={"state"}, writes={"registry"})
    b.add("registry", "key_codes", {}, digest(pool.tiled_codes(0, n0)), reads={"registry"})
    reg_n = n0

    # ---- strict batch material (every size derives from three small batches)
    ragged = make_batch(B, pool, [t % 65 for t in range(65)], 1)              # K 0..64
    wide = make_batch(B, pool, [48 + (t * 7) % 17 for t in range(32)], 2)    # K 48..64
    one = make_batch(B, pool, [1], 3)
    alt = make_batch(B, pool, [1 + t % 8 for t in range(40)], 4)
    big_side = wide.tile(min_keys=SMALL_CTA_KEYS, min_t=1025)
    big_k1 = wide.tile(min_keys=K1_WIDE_KEYS + 1)
    big_split = wide.tile(min_keys=SPLIT_KEYS)
    pairs_2048 = alt.tile(exact_t=1024)
    pairs_2050 = alt.tile(exact_t=1025)
    rlc_true = [valid_batch(B, pool, T, 30 + T) for T in (200, 17, 1040, 3)]
    rlc_false = [valid_batch(B, pool, T, 40 + T, bad=(T // 2,)) for T in (20, 600, 2)]
    seed_a, seed_b = hashlib.sha256(b"session rlc a").digest(), hashlib.sha256(b"session rlc b").digest()
    fp, cv, pe = _eval_rows(seed)
    alt_blob, def8, def16 = vm_blobs()

    def rlc(batch: Batch, seed32, tags=()):
        b.add("rlc", "fast_aggregate_verify_batch_all", {**batch.args(), "seed": seed32}, all(c == 0 for c in batch.codes), tags=tags)

    def reg_rlc(batch: Batch, seed32):
        # registry indices of the batch's (valid) pool keys: chain validator i carries pool key i % POOL
        idx = np.concatenate([np.asarray(tp) for tp in batch.tuples]).astype(np.uint32)
        b.add("rlc", "registry_verify_batch_all", dict(idx=idx, off=batch.off, msgs=batch.msgs, sigs=batch.sigs, seed=seed32),
              all(c == 0 for c in batch.codes), reads={"registry"})

    def singles(k):
        """The single-call entry points on pool material; answers from the C oracle."""
        r = np.random.default_rng(100 + k)
        i = int(r.choice(pool.valid))
        m = hashlib.sha256(b"session/single/%d" % k).digest()
        sig = sign(B, [pool.sks[i]], [m])[0].tobytes()
        pk = pool.keys[i].tobytes()
        b.add("single", "verify_signature", dict(pk=pk, msg=m, sig=sig), B.orc_verify_signature(pk, m, 32, sig))
        ks = r.choice(pool.valid, 5, replace=False).tolist()
        pks = [pool.keys[j].tobytes() for j in ks]
        fsig = sign(B, [sum(pool.sks[j] for j in ks) % R], [m])[0].tobytes()
        fsig_bad = fsig if k % 2 == 0 else sig
        b.add("single", "fast_aggregate_verify", dict(pks=pks, msg=m, sig=fsig_bad),
              B.orc_fast_aggregate_verify(b"".join(pks), 5, m, 32, fsig_bad))
        inf = bytes([0xC0]) + bytes(95)
        b.add("single", "eth_fast_aggregate_verify", dict(pks=[], msg=m, sig=inf), B.orc_eth_fast_aggregate_verify(b"", 0, m, 32, inf))
        msgs = [hashlib.sha256(b"session/av/%d/%d" % (k, j)).digest() for j in range(3)]
        sg = sign(B, [pool.sks[j] for j in ks[:3]], msgs)
        agg = ctypes.create_string_buffer(96)
        assert B.orc_aggregate(sg.tobytes(), 3, agg) == 0
        apks = b"".join(pks[:3])
        mp = (ctypes.c_char_p * 3)(*msgs)
        ml = (ctypes.c_size_t * 3)(32, 32, 32)
        b.add("single", "aggregate_verify", dict(pks=pks[:3], msgs=msgs, sig=agg.raw),
              B.orc_aggregate_verify(apks, 3, ctypes.cast(mp, ctypes.c_void_p), ctypes.cast(ml, ctypes.c_void_p), 3, agg.raw))
        sigs = [s.tobytes() for s in sg] + ([inf] if k % 2 else [])
        o = ctypes.create_string_buffer(96)
        c = B.orc_aggregate(b"".join(sigs), len(sigs), o)
        b.add("single", "aggregate", dict(sigs=sigs), (c, o.raw if c == 0 else None))
        epks = pks + ([pool.keys[int(np.flatnonzero(pool.codes == 6)[0])].tobytes()] if k % 2 else [])
        o = ctypes.create_string_buffer(48)
        c = B.orc_eth_aggregate_public_keys(b"".join(epks), len(epks), o)
        b.add("single", "eth_aggregate_public_keys", dict(pks=epks), (c, o.raw if c == 0 else None))

    def settings(knob, value, tags=()):
        b.add("settings", "tune", dict(knob=knob, value=value), None, writes={"knobs"}, tags=tags)

    def shuffle(n, seed32, rounds, tags=()):
        want = sh.shuffled_indices_numpy(n, seed32, rounds)
        b.add("shuffle", "compute_shuffled_indices", dict(n=n, seed=seed32, rounds=rounds), digest(want.astype(np.uint64)), tags=tags)

    def active(st_, epoch):
        recs = np.frombuffer(st_.validators.tobytes(), np.uint8)
        b.add("shuffle", "get_active_validator_indices", dict(recs=recs.copy(), epoch=epoch),
              digest(sc.active_numpy(recs, epoch).astype(np.uint64)))

    def state_shuffle(st_, epoch, seed32, rounds=90):
        act = sc.active_numpy(np.frombuffer(st_.validators.tobytes(), np.uint8), epoch)
        b.add("state", "state_shuffled_active_indices", dict(epoch=epoch, seed=seed32, rounds=rounds),
              digest(sh.shuffled_indices_numpy(act, seed32, rounds).astype(np.uint64)), reads={"state"})

    def ssz_hash(n, r_):
        data = r_.integers(0, 256, n, dtype=np.uint8).tobytes()
        b.add("ssz", "hash", dict(data=data), hashlib.sha256(data).digest())

    def merkleize(chunks: np.ndarray, limit=None):
        out = ctypes.create_string_buffer(32)
        n = chunks.size // 32
        rc_ = Z.orc_merkleize(chunks.ctypes.data, n, limit or 0, NT, out)
        b.add("ssz", "merkleize", dict(chunks=chunks, limit=limit), out.raw if rc_ == 0 else refused(ERR_LIMIT),
              tags=(("refusal", REFUSALS[5]),) if rc_ else ())

    def chain_block(k, n_dep, epoch):
        """Block k of the walk: deposits, a vote, a header; sync; one mixed call; the incremental root; the next
        epoch's shuffled active indices."""
        nonlocal reg_n
        r_ = np.random.default_rng(1000 + k)
        recs = rc.validator_records(r_, n_dep, epoch)
        lo = len(st.validators)
        recs["public_key"] = np.ascontiguousarray(pool.tiled(lo, n_dep)).view("V48").reshape(-1)
        bal = (32 * 10**9 + r_.integers(0, 10**6, n_dep, dtype=np.uint64)).astype("<u8")
        step = ("deposits", recs.tobytes(), bal)
        rc.apply(st, step)
        tags = [("block", k)] + ([("relocate", "state"), ("relocate", "registry")] if n_dep >= BIG_BLOCK else [])
        b.add("state", "add_validators", dict(records=step[1], balances=bal), None, writes={"state"}, tags=tags)
        v = rc.vote(r_, 100 + k)
        if len(st.eth1_data_votes) >= S.PRESETS["minimal"]["ETH1_DATA_VOTES_BOUND"]:
            rc.apply(st, ("set", "eth1_data_votes", b""))
            b.add("state", "set_field", dict(field="eth1_data_votes", data=b""), None, writes={"state"})
        rc.apply(st, ("push", "eth1_data_votes", v))
        b.add("state", "append_elements", dict(field="eth1_data_votes", values=v), None, writes={"state"})
        hdr = rc.header(r_, k % 33, 100 + k)
        rc.apply(st, ("set", "latest_execution_payload_header", hdr))
        b.add("state", "set_field", dict(field="latest_execution_payload_header", data=hdr), None, writes={"state"})
        b.add("registry", "sync", {}, len(st.validators), reads={"state"}, writes={"registry"}, tags=tags)
        reg_n = len(st.validators)
        mixed_call(r_, k, tags=[("block", k)])
        b.add("state", "incremental_root", {}, state_root(Z, st), reads={"state"}, writes={"state"}, tags=[("block", k)])
        snapshots.append((len(b.steps) - 1, copy.deepcopy(st) if len(st.validators) < BIG_BLOCK else None))
        state_shuffle(st, epoch + 1, hashlib.sha256(b"session/epoch/%d" % (epoch + 1)).digest())

    def mixed_call(r_, k, tags=()):
        """verify_batch with extra keys: registry indices and extras reg_n + j (pool keys that arrive with the block)."""
        n_x = int(r_.integers(1, 17))
        xlo = int(r_.integers(0, POOL))
        extra = pool.tiled(xlo, n_x)
        keyof = lambda i: pool.keys[i % POOL] if i < reg_n else extra[i - reg_n]   # noqa: E731
        skof = lambda i: pool.sks[i % POOL] if i < reg_n else pool.sks[(xlo + i - reg_n) % POOL]   # noqa: E731
        tups = [[int(x)] for x in r_.integers(0, reg_n, 3)] + [[reg_n + j] for j in range(n_x)]
        tups += [[int(r_.integers(0, reg_n)), reg_n + int(r_.integers(0, n_x)), reg_n - 1] for _ in range(4)]
        tups += [[reg_n - 1 - j for j in range(6)], [int(x) for x in r_.choice(reg_n, 9, replace=False)]]
        msgs = [hashlib.sha256(b"session/mixed/%d/%d" % (k, t)).digest() for t in range(len(tups))]
        sks = [sum(skof(i) for i in tp) % R if all(skof(i) is not None for i in tp) else 1 for tp in tups]
        sigs = sign(B, sks, msgs)
        sigs[0] = sigs[1]                                            # one wrong signature
        idx = np.concatenate([np.asarray(tp) for tp in tups]).astype(np.uint32)
        off = np.concatenate([[0], np.cumsum([len(tp) for tp in tups])]).astype(np.uint32)
        flat = np.stack([keyof(int(i)) for i in idx])
        m = np.frombuffer(b"".join(msgs), np.uint8)
        b.add("registry", "verify_batch", dict(idx=idx, off=off, msgs=m, sigs=sigs.reshape(-1), extra=extra.reshape(-1).copy()),
              oracle_codes(B, flat, off, m, sigs), reads={"registry"}, tags=list(tags) + [("mixed", reg_n)])
        return idx, off, m, sigs, flat

    # ================================================================ the script
    # strict batches: sizes alternate so that every shared buffer is shrunk right after it grew
    strict(b, one)
    strict(b, ragged)
    strict(b, big_side, tags=[("side_cta", 128)])
    strict(b, one, tags=[("shrink",)])
    chain_block(0, 5, 100)
    strict(b, pairs_2048, tags=[("pairs", 2048)])
    strict(b, pairs_2050, tags=[("pairs", 2050)])
    strict(b, one)
    singles(0)
    ssz_hash(1 << 20, rng)
    ssz_hash(0, rng)
    ssz_hash(55, rng)
    rlc(rlc_true[0], seed_a)
    strict(b, ragged)
    rlc(rlc_false[0], seed_a)
    reg_rlc(rlc_true[0], seed_b)
    chain_block(1, 16, 101)
    merkleize(rng.integers(0, 256, 32 << 20, dtype=np.uint8))
    merkleize(rng.integers(0, 256, 32, dtype=np.uint8))
    strict(b, big_k1, tags=[("k1_cta", 384)])
    rlc(rlc_true[1], seed_b)
    reg_rlc(rlc_false[0], seed_a)
    strict(b, one)
    # shuffles of alternating sizes around the resident handle's shuffle: same seed with another n, same n with another seed
    sh_seed, sh_seed2 = hashlib.sha256(b"session shuffle").digest(), hashlib.sha256(b"session shuffle 2").digest()
    shuffle(1 << 20, sh_seed, 10)
    shuffle(5, sh_seed, 10, tags=[("same seed, other n",)])
    active(st, 101)
    state_shuffle(st, 102, sh_seed, 10)
    shuffle(5, sh_seed2, 10, tags=[("same n, other seed",)])
    active(st, 1 << 17)
    b.add("ssz", "htr_validators", dict(ssz=np.frombuffer(st.validators.tobytes(), np.uint8).copy()), _htr_validators(Z, st))
    other = S.synth_state(700, "mainnet", seed=seed + 1)
    b.add("ssz", "htr_beacon_state", dict(ssz=S.serialize(other), preset="mainnet"), state_root(Z, other))
    for d_, ok in ((0, True), (1, True), (40, True), (64, True), (40, False), (64, False)):
        b.add("ssz", "is_valid_merkle_branch", merkle_branch(rng, d_, ok), ok)
    # device self-tests
    b.add("eval", "fp_eval", fp[0], fp[1])
    b.add("eval", "curve_eval", cv[0], cv[1])
    b.add("eval", "pairing_eval", pe[0], pe[1])
    # settings changed mid-session, then restored; the answers do not move
    settings("vm_cta", 64)
    rlc(rlc_true[2], seed_a)
    strict(b, alt)
    settings("vm_cta", 128)
    strict(b, pairs_2050)
    rlc(rlc_false[1], seed_b)
    settings("vm_cta", 32, tags=[("restore",)])
    settings("vm_team16_max", 0)
    strict(b, pairs_2048)
    rlc(rlc_true[0], None)
    settings("vm_team16_max", VM_TEAM16_MAX, tags=[("restore",)])
    settings("bls_small_cta", 128)
    strict(b, ragged)
    settings("bls_small_cta", 0, tags=[("restore",)])
    strict(b, big_side)
    b.add("settings", "vm_load_programs", dict(blob=alt_blob), None, writes={"knobs"})
    strict(b, pairs_2048)
    rlc(rlc_true[3], seed_b)
    b.add("settings", "vm_load_programs", dict(blob=def8), None, writes={"knobs"}, tags=[("restore",)])
    b.add("settings", "vm_load_programs", dict(blob=def16), None, writes={"knobs"}, tags=[("restore",)])
    for k in range(2, big_at):
        chain_block(k, 1 + (k * 5) % 16, 100 + k)
    # the block that moves the state's lists and the registry's arrays; mixed calls before (above) and after it
    chain_block(big_at, BIG_BLOCK, 100 + big_at)
    strict(b, big_split, tags=[("split", SPLIT_KEYS)])
    strict(b, one, tags=[("shrink",)])
    singles(1)
    rlc(rlc_false[2], seed_a)
    rlc(rlc_true[2], seed_b)
    reg_rlc(rlc_true[2], seed_a)
    reg_rlc(rlc_false[1], seed_b)
    strict(b, ragged)
    for k in range(big_at + 1, n_blocks):
        chain_block(k, 1 + (k * 3) % 16, 100 + k)

    # ---- a refusal of every family, each followed by a step of the same family
    root_now = state_root(Z, st)
    codes_now = digest(pool.tiled_codes(0, len(st.validators)))
    bad_off = np.array([0, 2, 1], np.uint32)
    b.add("strict", "fast_aggregate_verify_batch", dict(pks=one.flat, off=bad_off, msgs=np.zeros(64, np.uint8),
                                                        sigs=np.zeros(192, np.uint8)), refused(ERR_BAD_ARG),
          tags=[("refusal", REFUSALS[0])])
    strict(b, ragged, tags=[("after", REFUSALS[0])])
    r_ = np.random.default_rng(77)
    idx, off, m, sigs, _ = mixed_call(r_, 99)
    mixed = b.steps[-1]
    ex = np.asarray(mixed.args["extra"])
    bad = idx.copy()
    bad[-1] = reg_n + ex.size // 48                                        # one past registry + extras
    b.add("registry", "verify_batch", dict(idx=bad, off=off, msgs=m, sigs=sigs.reshape(-1), extra=ex), refused(ERR_BAD_ARG),
          reads={"registry"}, tags=[("refusal", REFUSALS[1])])
    b.add("registry", "verify_batch", mixed.args, mixed.want, reads={"registry"}, tags=[("after", REFUSALS[1])])
    b.add("registry", "key_codes", {}, codes_now, reads={"registry"})
    lay = S.layout(st)
    pos = lay["offset:validators"][0]
    ser = S.serialize(st)
    moved = bytes(ser[pos - 8:pos]) + (int.from_bytes(bytes(ser[pos:pos + 4]), "little") + 121).to_bytes(4, "little")
    try:
        rc.apply(st, ("bytes", pos - 8, moved))
        raise AssertionError("the mirror accepted an update_bytes that moves an offset")
    except S.ReshapeRefused as e:
        assert e.kind == "bad_arg"
    b.add("state", "update_bytes", dict(offset=pos - 8, data=moved), refused(ERR_BAD_ARG), reads={"state"}, writes={"state"},
          tags=[("refusal", REFUSALS[2])])
    b.add("state", "state_root", {}, root_now, reads={"state"}, tags=[("after", REFUSALS[2])])
    hdr = bytearray(rc.header(r_, 3, 999))
    hdr[436:440] = (585).to_bytes(4, "little")
    b.add("state", "set_field", dict(field="latest_execution_payload_header", data=bytes(hdr)), refused(ERR_SSZ_MALFORMED),
          reads={"state"}, writes={"state"}, tags=[("refusal", REFUSALS[3])])
    b.add("state", "incremental_root", {}, root_now, reads={"state"}, writes={"state"}, tags=[("after", REFUSALS[3])])
    small = S.serialize(S.synth_state(n0 - 5, "minimal", seed=seed, pubkeys=pool.tiled(0, n0 - 5)))
    b.add("registry", "sync_smaller", dict(ssz=small), refused(ERR_BAD_ARG), reads={"registry"}, tags=[("refusal", REFUSALS[4])])
    b.add("registry", "key_codes", {}, codes_now, reads={"registry"}, tags=[("after", REFUSALS[4])])
    b.add("registry", "verify_batch", mixed.args, mixed.want, reads={"registry"})
    merkleize(rng.integers(0, 256, 5 * 32, dtype=np.uint8), limit=4)
    merkleize(rng.integers(0, 256, 32, dtype=np.uint8))
    b.steps[-1].tags = (("after", REFUSALS[5]),)
    b.add("ssz", "htr_beacon_state", dict(ssz=S.serialize(other)[:100].copy(), preset="mainnet"), refused(ERR_SSZ_MALFORMED),
          tags=[("refusal", REFUSALS[6])])
    b.add("ssz", "htr_beacon_state", dict(ssz=S.serialize(other), preset="mainnet"), state_root(Z, other), tags=[("after", REFUSALS[6])])
    b.add("eval", "curve_eval", dict(cv[0], op=3), refused(ERR_BAD_ARG), tags=[("refusal", REFUSALS[7])])
    b.add("eval", "curve_eval", cv[0], cv[1], tags=[("after", REFUSALS[7])])
    b.add("state", "state_root", {}, root_now, reads={"state"})
    b.add("registry", "key_codes", {}, codes_now, reads={"registry"})

    for i, s in enumerate(b.steps):
        s.i = i
    return Session(b.steps, init, meta=dict(n0=n0, blocks=n_blocks, big_block=big_at, final_root=root_now,
                                             final_n=len(st.validators), mirror=st, snapshots=snapshots, pool=pool,
                                             batches=dict(ragged=ragged, wide=wide, alt=alt, big_side=big_side, big_k1=big_k1,
                                                          big_split=big_split)))


def _htr_validators(Z, st) -> bytes:
    v = np.frombuffer(st.validators.tobytes(), np.uint8)
    out = ctypes.create_string_buffer(32)
    assert Z.orc_htr_validators(v.ctypes.data, len(st.validators), 1 << 40, NT, out) == 0
    return out.raw


# ---------------------------------------------------------------------------------------------------------- orders
def depends(a: Step, b: Step) -> bool:
    """b (later in script order) must stay after a: one of them writes what the other reads or writes."""
    return bool(a.writes & (b.reads | b.writes)) or bool(b.writes & a.reads)


def shuffled_order(steps: List[Step], seed: int) -> List[int]:
    """A seeded topological shuffle: a random order of the steps that keeps every dependent pair in script order."""
    rnd = random.Random(seed)
    n = len(steps)
    preds = [set() for _ in range(n)]
    for j in range(n):
        for i in range(j):
            if depends(steps[i], steps[j]):
                preds[j].add(i)
    done, order = set(), []
    ready = [j for j in range(n) if not preds[j]]
    while ready:
        j = ready.pop(rnd.randrange(len(ready)))
        order.append(j)
        done.add(j)
        ready += [k for k in range(n) if k not in done and k not in ready and preds[k] <= done]
    assert len(order) == n
    return order


def closure(steps: List[Step], i: int) -> List[int]:
    """Step i and every earlier step it depends on, transitively (what replaying step i alone needs)."""
    need = {i}
    for j in range(i - 1, -1, -1):
        if any(depends(steps[j], steps[k]) and steps[j].writes for k in need):
            need.add(j)
    return sorted(need)
