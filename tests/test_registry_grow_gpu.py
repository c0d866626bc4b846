"""GPU: the validated-key registry follows a growing validator set — `Registry.append`, `Registry.from_state` and
`Registry.sync` (b200_registry_append / _load_state / _sync_state) against a load of the concatenated key list, the strict
batch path and the C oracle.

Sections: append = load of the concatenation (chunk sizes 0, 1, ..., invalid keys on both sides of every boundary);
growth past the reserved capacity (2^18 appended keys); `..._batch_mixed` extra keys around appends; `from_state` on
states of invalid and of valid keys; `sync` over a short chain of deposit blocks, one of which moves the state's validator
list past its reserved region; refusals that leave the registry as it was (a sharded handle in a child process, since the
communicator is process-global).  Valid keys and signatures come from the C oracle; invalid keys from the soak generators
(tests/bls_soak_cases.py).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from tests import bls_soak_cases as bsc  # noqa: E402

pytestmark = pytest.mark.gpu
R = bsc.R


class Keys:
    """A host key list with the secret of every valid key (None for an invalid one)."""

    def __init__(self, keys=None, sks=None):
        self.keys = np.zeros((0, 48), np.uint8) if keys is None else np.ascontiguousarray(keys, dtype=np.uint8).reshape(-1, 48)
        self.sks = [] if sks is None else list(sks)

    def __len__(self):
        return len(self.sks)

    def __add__(self, other):
        return Keys(np.concatenate([self.keys, other.keys]), self.sks + other.sks)

    def __getitem__(self, s):
        return Keys(self.keys[s], self.sks[s])

    def flat(self):
        return np.ascontiguousarray(self.keys).reshape(-1)


def valid_keys(O, n, seed):
    keys, sk0, d = bsc.valid_keys(O, n, seed)
    return Keys(keys, [(sk0 + i * d) % R for i in range(n)])


def invalid_pool(O, seed=1):
    """Keys key_validate rejects, every class: bad encodings (flags, x >= p), infinity, not on the curve, outside G1."""
    rng = np.random.default_rng(seed)
    ok = valid_keys(O, 8, 900 + seed).keys
    enc = list(bsc.g1_edge_encodings(ok[:4]))
    enc += [r.tobytes() for r in bsc.random_g1_encodings(rng, 400)]
    enc += [bsc.mutate(ok[i % 8].tobytes(), 48, k, rng) for i in range(8) for k in range(bsc.N_MUTATIONS)]
    codes = [O.orc_key_validate(e) for e in enc]
    bad = [(e, c) for e, c in zip(enc, codes) if c != 0]
    assert {1, 2, 3, 6} <= {c for _, c in bad}, sorted({c for _, c in bad})
    order = rng.permutation(len(bad))
    return [bad[i][0] for i in order]


def with_invalid(k: Keys, positions, pool) -> Keys:
    out = Keys(k.keys.copy(), k.sks)
    for j, p in enumerate(sorted(set(int(x) for x in positions))):
        out.keys[p] = np.frombuffer(pool[j % len(pool)], np.uint8)
        out.sks[p] = None
    return out


def oracle_codes(O, k: Keys, sample=None):
    idx = range(len(k)) if sample is None else sample
    return [O.orc_key_validate(k.keys[i].tobytes()) for i in idx]


def sign(O, sks, msgs):
    n = len(sks)
    sk_b = np.frombuffer(b"".join(int(s if s else 1).to_bytes(32, "big") for s in sks), dtype=np.uint8).copy()
    m = np.frombuffer(b"".join(msgs), dtype=np.uint8).copy()
    out = np.empty((n, 96), dtype=np.uint8)
    O.orc_sign_batch(sk_b.ctypes.data, m.ctypes.data, n, out.ctypes.data, 8)
    return out


def make_batch(O, k: Keys, tuples, wrong=()):
    """Messages and signatures for tuples of indices into `k`: signed by the sum of the signers' secrets when they are
    all valid; tuples listed in `wrong` carry another tuple's signature."""
    msgs = [hashlib.sha256(b"reg-grow/%d/%s" % (t, ",".join(map(str, tp)).encode())).digest() for t, tp in enumerate(tuples)]
    sks = [sum(k.sks[i] for i in tp) % R if all(k.sks[i] is not None for i in tp) else 1 for tp in tuples]
    sigs = sign(O, sks, msgs)
    for t in wrong:
        sigs[t] = sigs[(t + 1) % len(tuples)]
    return np.frombuffer(b"".join(msgs), dtype=np.uint8), np.ascontiguousarray(sigs).reshape(-1)


def three_way(O, reg, k: Keys, tuples, wrong=(), extra: Keys = None):
    """Registry-mode codes (named by index into `k`; indices >= reg.n are the call's extra keys) == strict batch on the
    same keys == C oracle; returns the codes."""
    from ethereum_consensus_b200 import crypto
    msgs, sigs = make_batch(O, k, tuples, wrong)
    idx = np.concatenate([np.asarray(tp, dtype=np.uint32) for tp in tuples])
    off = np.cumsum([0] + [len(tp) for tp in tuples]).astype(np.uint32)
    got = reg.verify_batch(idx, off, msgs, sigs, extra_keys=None if extra is None else extra.flat())
    flat = np.ascontiguousarray(k.keys[idx]).reshape(-1)
    strict = crypto.fast_aggregate_verify_batch(flat, off, msgs, sigs)
    want = np.empty(len(tuples), dtype=np.int32)
    O.orc_fast_aggregate_verify_batch(flat.ctypes.data, off.ctypes.data, msgs.ctypes.data, sigs.ctypes.data, len(tuples),
                                      want.ctypes.data, 8)
    assert got.tolist() == strict.tolist() == want.tolist()
    return got


def records(rng, pubkeys: np.ndarray) -> np.ndarray:
    """Validator records (as add_validator_to_registry makes them) carrying `pubkeys`."""
    from tests import state_reshape_cases as rc
    recs = rc.validator_records(rng, len(pubkeys), 100)
    recs["public_key"] = np.ascontiguousarray(pubkeys, dtype=np.uint8).view("V48").reshape(-1)
    return recs


def state_pubkeys(st) -> np.ndarray:
    return np.frombuffer(st.validators.tobytes(), np.uint8).reshape(-1, 121)[:, :48].copy()


# ---------------------------------------------------------------------------------------------------------- append
def test_append_equals_load_of_the_concatenation(engine, oracle_bls_c):
    from ethereum_consensus_b200 import crypto
    O = oracle_bls_c
    rng = np.random.default_rng(1)
    chunks = [0, 1, 37, 0, 1, 200, 128, 1, 332]
    n = sum(chunks)
    cuts = np.cumsum(chunks)[:-1]
    bounds = sorted({int(b) for b in cuts if 0 < b < n})
    bad = [p for b in bounds for p in (b - 1, b)] + rng.choice(n, 40, replace=False).tolist()
    k = with_invalid(valid_keys(O, n, 11), bad, invalid_pool(O))
    want = oracle_codes(O, k)
    assert crypto.Registry(k.flat()).key_codes().tolist() == want

    reg = crypto.Registry(k[:chunks[0]].flat())
    lo = chunks[0]
    for c in chunks[1:]:
        reg.append(k[lo:lo + c].flat())
        lo += c
        assert reg.n == lo
        assert reg.key_codes().tolist() == want[:lo]
        if c:
            assert crypto.last_kernel_ms() > 0
    assert reg.n == n

    ok = [i for i in range(n) if k.sks[i] is not None]
    tuples, wrong = [], []
    for b in bounds:
        tuples.append([b - 1, b])                                              # both sides invalid
        left = max((i for i in ok if i < b - 1), default=None)
        right = min(i for i in ok if i > b)
        if left is None:
            continue
        tuples.append([left, right])                                           # valid keys across the boundary
        tuples.append([right, left, b])                                        # ... with an invalid key after them
        tuples.append([left, right])
        wrong.append(len(tuples) - 1)
    for _ in range(30):
        tuples.append(rng.choice(n, int(rng.integers(1, 9)), replace=False).tolist())
    for _ in range(10):
        tuples.append(rng.choice(ok, int(rng.integers(1, 9)), replace=False).tolist())
    codes = three_way(O, reg, k, tuples, wrong)
    assert set(codes.tolist()) >= {0, 5} and len(set(codes.tolist()) - {0, 5}) >= 2


# ---------------------------------------------------------------------------------------------------------- growth
def test_growth_past_the_reserved_capacity(engine, oracle_bls_c):
    """A 1000-key registry reserves headroom (2^16) + the extra-key tail (2^16) + allocation slack, ~150 k entries:
    appending 2^18 keys moves it at least once."""
    from ethereum_consensus_b200 import crypto
    O = oracle_bls_c
    rng = np.random.default_rng(2)
    n0, grow = 1000, 1 << 18
    first = valid_keys(O, n0, 21)
    rest = Keys(bsc.random_g1_encodings(rng, grow), [None] * grow)          # mostly invalid: every class K1 rejects
    spots = np.sort(rng.choice(grow, 1500, replace=False))
    ok = valid_keys(O, len(spots), 22)
    for j, p in enumerate(spots):
        rest.keys[p] = ok.keys[j]
        rest.sks[p] = ok.sks[j]
    k = first + rest

    reg = crypto.Registry(first.flat())
    first_codes = reg.key_codes().tolist()
    assert first_codes == [0] * n0
    lo = n0
    for c in ((1 << 16) - 1, (1 << 16) + 1, 1, (1 << 17) - 1):
        reg.append(k[lo:lo + c].flat())
        lo += c
    assert reg.n == n0 + grow
    codes = reg.key_codes()
    assert codes[:n0].tolist() == first_codes
    sample = np.concatenate([n0 + spots, rng.choice(np.arange(n0, n0 + grow), 600, replace=False)])
    assert codes[sample].tolist() == oracle_codes(O, k, sample)

    good = [int(i) for i in n0 + spots]
    tuples = [[i] for i in range(0, n0, 97)] + [rng.choice(n0, 64, replace=False).tolist() for _ in range(8)]
    tuples += [rng.choice(good, 16, replace=False).tolist() for _ in range(8)]
    tuples += [[int(rng.integers(0, n0)), good[-1], good[0]], [n0 + (1 << 16) - 2, n0 + (1 << 16) - 1, n0 + (1 << 16)]]
    three_way(O, reg, k, tuples, wrong=[3, len(tuples) - 3])
    assert crypto.Registry(k.flat()).key_codes().tolist() == codes.tolist()


# ---------------------------------------------------------------------------------------------------------- mixed
def test_mixed_calls_around_appends(engine, oracle_bls_c):
    from ethereum_consensus_b200 import crypto
    O = oracle_bls_c
    rng = np.random.default_rng(3)
    pool = invalid_pool(O, 3)
    k = valid_keys(O, 3000, 31)
    reg_keys = k[:1000]
    reg = crypto.Registry(reg_keys.flat())

    def mixed(base: Keys, extra: Keys):
        n, m = len(base), len(extra)
        tuples = [[int(i)] for i in rng.choice(n, 10, replace=False)] + [[n + j] for j in range(m)]
        tuples += [[int(rng.integers(0, n)), n + j, int(rng.integers(0, n))] for j in range(m)]
        tuples += [rng.choice(n + m, 12, replace=False).tolist() for _ in range(10)]
        return three_way(O, reg, base + extra, tuples, wrong=[0, 10, 11 + m], extra=extra)

    e1 = with_invalid(k[2000:2016], [3, 9], pool)
    mixed(reg_keys, e1)
    appended = k[1000:1500]
    reg.append(appended.flat())                          # lands where e1 was validated: the tail moves behind it
    reg_keys = reg_keys + appended
    assert reg.n == 1500
    e2 = with_invalid(k[2100:2140], [0, 17, 39], pool)
    mixed(reg_keys, e2)                                   # extra keys named from the new reg_n
    assert reg.key_codes().tolist() == [0] * 1500        # the second tail did not clobber the appended keys
    tuples = [[1000 + i] for i in range(0, 500, 7)] + [list(range(990, 1010)), list(range(1480, 1500))]
    assert three_way(O, reg, reg_keys, tuples).tolist() == [0] * len(tuples)


# ---------------------------------------------------------------------------------------------------------- from_state
def test_from_state_equals_load_of_the_pubkeys(engine, oracle_bls_c):
    from ethereum_consensus_b200 import crypto, ssz, state as S
    O = oracle_bls_c
    rng = np.random.default_rng(4)
    n = 4000
    mix = bsc.random_g1_encodings(rng, n)                # mostly invalid: off the curve or outside G1
    mix[::4] = rng.integers(0, 256, (n // 4, 48), dtype=np.uint8)   # any 48 bytes: mostly bad encodings
    mix[1::8] = valid_keys(O, n // 8, 41).keys
    st = S.synth_state(n, "minimal", pubkeys=mix)
    h = ssz.DeviceBeaconState(S.serialize(st), "minimal")
    reg = crypto.Registry.from_state(h)
    assert reg.n == n and crypto.last_kernel_ms() > 0
    codes = reg.key_codes().tolist()
    assert codes == oracle_codes(O, Keys(state_pubkeys(st), [None] * n))
    assert len(set(codes)) >= 3 and codes.count(0) >= n // 8
    assert crypto.Registry(state_pubkeys(st).reshape(-1)).key_codes().tolist() == codes
    h.close()

    k = valid_keys(O, 3000, 42)
    st = S.synth_state(3000, "mainnet", pubkeys=k.keys)
    h = ssz.DeviceBeaconState(S.serialize(st), "mainnet")
    reg = crypto.Registry.from_state(h)
    assert reg.n == 3000 and reg.key_codes().tolist() == [0] * 3000
    tuples = [rng.choice(3000, int(rng.integers(1, 40)), replace=False).tolist() for _ in range(40)] + [[0], [2999]]
    before = three_way(O, reg, k, tuples, wrong=[5, 6, 30])
    h.close()                                             # the registry holds its own copy of the keys
    assert three_way(O, reg, k, tuples, wrong=[5, 6, 30]).tolist() == before.tolist()
    assert reg.key_codes().tolist() == [0] * 3000


# ---------------------------------------------------------------------------------------------------------- sync
def test_sync_over_a_short_chain(engine, oracle_bls_c):
    from ethereum_consensus_b200 import block, crypto, ssz, state as S
    O = oracle_bls_c
    rng = np.random.default_rng(5)
    n0 = 3000
    pool = valid_keys(O, n0 + 16 + 200, 51)
    st = S.synth_state(n0, "minimal", pubkeys=pool.keys[:n0])
    h = ssz.DeviceBeaconState(S.serialize(st), "minimal")
    reg = crypto.Registry.from_state(h)
    chain = pool[:n0]                                     # the state's keys in validator-index order

    # block 1: 16 deposits decided by verify_deposits, one with a signature by the wrong key
    dep = pool[n0:n0 + 16]
    wcs = [hashlib.sha256(b"wc%d" % j).digest() for j in range(16)]
    roots = [block.deposit_signing_root(dep.keys[j].tobytes(), wcs[j], 32 * 10**9) for j in range(16)]
    sks = [dep.sks[j] if j != 6 else dep.sks[7] for j in range(16)]
    sigs = sign(O, sks, roots)
    verdicts = block.verify_deposits([(dep.keys[j].tobytes(), wcs[j], 32 * 10**9, sigs[j].tobytes()) for j in range(16)])
    assert verdicts == [j != 6 for j in range(16)]
    acc = [j for j in range(16) if verdicts[j]]
    h.add_validators(records(rng, dep.keys[acc]).tobytes(), np.full(len(acc), 32 * 10**9, "<u8"))
    chain = chain + Keys(dep.keys[acc], [dep.sks[j] for j in acc])
    reg.sync(h)
    assert reg.n == h.n_validators == n0 + 15 and crypto.last_kernel_ms() > 0
    assert reg.key_codes().tolist() == [0] * reg.n

    def block_set(new, bad_att=False):
        """A later block's signature set naming validators `new` through an exit and an attestation."""
        s = block.SignatureSet()
        pk = [chain.keys[i].tobytes() for i in range(len(chain))]
        att = sorted(set(rng.choice(n0, 40, replace=False).tolist()) | set(new[:6]))
        plan = [("voluntary_exit", [new[-1]]), ("attestation", att), ("voluntary_exit", [new[0]]), ("attestation", sorted(new))]
        msgs = [hashlib.sha256(b"blk/%d/%s" % (i, site.encode())).digest() for i, (site, _) in enumerate(plan)]
        sg = sign(O, [sum(chain.sks[i] for i in ix) % R for _, ix in plan], msgs)
        if bad_att:
            sg[1] = sg[3]
        for (site, ix), m, sgn in zip(plan, msgs, sg):
            if site == "attestation":
                s.add_indexed_attestation(site, pk, ix, m, sgn.tobytes())
            else:
                s.add_by_index(site, pk, ix, m, sgn.tobytes())
        # a deposit of the block itself rides along as an extra key
        x = n0 + 16 + len(chain) % 100
        xm = hashlib.sha256(b"dep").digest()
        s.add("deposit", [pool.keys[x].tobytes()], xm, sign(O, [pool.sks[x]], [xm])[0].tobytes(), tolerant=True)
        codes = s.verify(registry=reg)
        assert codes.tolist() == s.verify().tolist()
        ent = s.entries
        flat = np.frombuffer(b"".join(p for e in ent for p in e.pubkeys), dtype=np.uint8)
        off = np.cumsum([0] + [len(e.pubkeys) for e in ent]).astype(np.uint32)
        m = np.frombuffer(b"".join(e.signing_root for e in ent), dtype=np.uint8)
        g = np.frombuffer(b"".join(e.signature for e in ent), dtype=np.uint8)
        want = np.empty(len(ent), dtype=np.int32)
        O.orc_fast_aggregate_verify_batch(flat.ctypes.data, off.ctypes.data, m.ctypes.data, g.ctypes.data, len(ent), want.ctypes.data, 8)
        assert codes.tolist() == want.tolist()
        return codes

    new = list(range(n0, n0 + 15))
    assert block_set(new).tolist() == [0] * 5
    assert block_set(new, bad_att=True).tolist() == [0, 5, 0, 0, 0]
    reg.sync(h)                                           # nothing new
    assert reg.n == n0 + 15

    # block 2: more records than the list's reserved region holds (2^16 headroom): the state relocates the list
    big = 70_000
    keys = bsc.random_g1_encodings(rng, big)
    spots = np.sort(rng.choice(big, 150, replace=False))
    ok = pool[n0 + 16:n0 + 16 + 150]
    keys[spots] = ok.keys
    sks = [None] * big
    for j, p in enumerate(spots):
        sks[p] = ok.sks[j]
    base = len(chain)
    h.add_validators(records(rng, keys).tobytes(), np.full(big, 32 * 10**9, "<u8"))
    chain = chain + Keys(keys, sks)
    reg.sync(h)
    assert reg.n == h.n_validators == base + big
    codes = reg.key_codes()
    assert codes[:base].tolist() == [0] * base
    sample = np.concatenate([base + spots, base + rng.choice(big, 400, replace=False)])
    assert codes[sample].tolist() == oracle_codes(O, chain, sample)
    assert block_set([int(base + p) for p in spots[:15]]).tolist() == [0] * 5
    h.close()
    assert crypto.Registry(chain.flat()).key_codes().tolist() == codes.tolist()


# ---------------------------------------------------------------------------------------------------------- refusals
def _assert_unchanged(reg, n, codes, probe, verdicts):
    assert reg.n == n and reg.key_codes().tolist() == codes
    assert probe().tolist() == verdicts


def test_refusals_leave_the_registry_unchanged(engine, oracle_bls_c):
    from ethereum_consensus_b200 import _lib, crypto, ssz, state as S
    O = oracle_bls_c
    L = _lib.lib()
    k = with_invalid(valid_keys(O, 300, 61), [0, 150, 299], invalid_pool(O, 6))
    st = S.synth_state(300, "minimal", pubkeys=k.keys)
    h = ssz.DeviceBeaconState(S.serialize(st), "minimal")
    reg = crypto.Registry.from_state(h)
    codes = reg.key_codes().tolist()
    assert codes == oracle_codes(O, k)
    tuples = [[1, 2], [0], [149, 150, 151], [298, 299]]
    probe = lambda: three_way(O, reg, k, tuples)  # noqa: E731
    first = probe().tolist()

    small = ssz.DeviceBeaconState(S.serialize(S.synth_state(295, "minimal", pubkeys=k.keys[:295])), "minimal")
    with pytest.raises(_lib.EngineError) as e:
        reg.sync(small)
    assert e.value.code == _lib.ERR_BAD_ARG
    _assert_unchanged(reg, 300, codes, probe, first)
    small.close()
    buf = np.zeros(48 * 4, np.uint8)
    assert L.b200_registry_append(None, 3) == _lib.ERR_BAD_ARG
    assert L.b200_registry_append(_lib.ptr(buf), 0x7fffffff - 299) == _lib.ERR_BAD_ARG   # reg_n + n > 0x7fffffff
    assert L.b200_registry_load_state(None) == _lib.ERR_BAD_ARG
    assert L.b200_registry_sync_state(None) == _lib.ERR_BAD_ARG
    _assert_unchanged(reg, 300, codes, probe, first)
    reg.append(b"")                                      # n == 0 and a sync with nothing new: no change
    reg.sync(h)
    assert L.b200_registry_append(None, 0) == 0
    _assert_unchanged(reg, 300, codes, probe, first)
    h.close()


def test_sharded_handle_is_refused_in_a_child_process(engine):
    p = subprocess.run([sys.executable, "-m", "tests.test_registry_grow_gpu"], cwd=str(ROOT), env=dict(os.environ),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    print(p.stdout)
    assert p.returncode == 0, p.stdout
    assert "CHILD_OK" in p.stdout, p.stdout


def _child():
    """A world-1 communicator and a sharded resident state: both registry calls refuse it and leave the registry alone."""
    from ethereum_consensus_b200 import _lib, crypto, parallel, ssz, state as S
    _lib.init(0)
    parallel.comm_init(0, 1)
    rng = np.random.default_rng(7)
    keys = bsc.random_g1_encodings(rng, 200)
    reg = crypto.Registry(keys.reshape(-1))
    codes = reg.key_codes().tolist()
    st = S.synth_state(250, "minimal", pubkeys=bsc.random_g1_encodings(rng, 250))
    h = ssz.DeviceBeaconState(S.serialize(st), "minimal", sharded=True)
    L = _lib.lib()
    assert L.b200_registry_load_state(h._h) == _lib.ERR_BAD_ARG
    assert L.b200_registry_sync_state(h._h) == _lib.ERR_BAD_ARG
    assert reg.n == 200 and reg.key_codes().tolist() == codes
    h.close()
    parallel.comm_destroy()
    print("CHILD_OK")


if __name__ == "__main__":
    _child()
