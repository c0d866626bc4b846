"""GPU: the adversarial SSZ, incremental re-hash and shuffling soak through the CUDA kernels, case by case against the
oracles (the plain-C liboracle_ssz.so on all host threads, oracle/ssz_oracle.py where the state is small, and
oracle/shuffle_oracle.py).

Sections: a. merkleize / packed / Validator lists at the planner's boundary sizes and limits, SHA-256 at every length
0..300; b. whole-state roots (one-shot, resident, shard_roots + combine_roots for world 1..64); c. incremental update
scripts on resident states; d. malformed encodings on every entry point; e. shuffling and active indices, also on a
resident state whose validators changed; f. two resident handles of different presets updated alternately, with one-shot
calls in between.  B200_SSZ_FOLD is read once per process, so sections a, b, c and f run again in a child process
with it off.  The cases come from tests/ssz_soak_cases.py.

    B200_SOAK_SCALE=1 (default) python -m pytest tests/test_ssz_device_soak_gpu.py -m gpu -s
"""
from __future__ import annotations

import ctypes
import hashlib
import os
import pickle
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from tests import ssz_soak_cases as sc  # noqa: E402

pytestmark = pytest.mark.gpu
NT = os.cpu_count() or 1
WORLDS = [1, 2, 4, 8, 16, 32, 64]
ENV_VARIANTS = [{"B200_SSZ_FOLD": "0"}]
REJECT = "reject"


# ---------------------------------------------------------------------------------------------------------- helpers
class Tally:
    """Per-section case and mismatch counts; every mismatch prints what is needed to replay it."""

    def __init__(self, tag=""):
        self.tag, self.n, self.bad = tag, {}, {}

    def check(self, section, want, got, replay):
        self.n[section] = self.n.get(section, 0) + 1
        if want != got:
            self.bad[section] = self.bad.get(section, 0) + 1
            if self.bad[section] <= 5:
                w = want.hex() if isinstance(want, bytes) else want
                g = got.hex() if isinstance(got, bytes) else got
                print(f"  MISMATCH {section}{self.tag}: {replay}: oracle {w!s:.80}, device {g!s:.80}")
                sys.stdout.flush()

    def report(self, minimum=None):
        for s in sorted(self.n):
            print(f"{s + self.tag:60s} cases {self.n[s]:6d}  mismatches {self.bad.get(s, 0)}")
        sys.stdout.flush()
        for s in self.n:
            assert self.bad.get(s, 0) == 0, f"{s}{self.tag}: {self.bad[s]} of {self.n[s]} cases differ from the oracle"
        for s, m in (minimum or {}).items():
            assert self.n.get(s, 0) >= m, (s, self.n.get(s, 0), m)


def dev(fn, *a):
    """A device call's result, or REJECT when it raises MerkleizationError."""
    from ethereum_consensus_b200 import ssz
    try:
        return fn(*a)
    except ssz.MerkleizationError:
        return REJECT


def c_root(O, b, preset):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    out = ctypes.create_string_buffer(32)
    rc = O.orc_htr_beacon_state_deneb(b.ctypes.data, b.size, 0 if preset == "mainnet" else 1, NT, out)
    return out.raw if rc == 0 else REJECT


def small_state(spec):
    return spec["n"] <= 2049 if spec["preset"] == "minimal" else spec["n"] <= 257


def hashlib_root(b, preset):
    from ethereum_consensus_b200 import state as S
    from oracle import ssz_oracle as so
    return so.beacon_state_type(preset).htr(S.to_oracle_value(sc.deserialize(b, preset)))


# ---------------------------------------------------------------------------------------------------------- a. primitives
def prim_cases():
    """(kind, args) for merkleize / hash_tree_root_packed / hash_tree_root_validators / hash; inputs derive from args."""
    out = []
    C17 = sc.COOP_MAX
    for n in [0, 1, 2, 3, 7, 8, 9, 63, 64, 65, 255, 256, 257, 511, 512, 513, 4095, 4096, 4097, C17 - 1, C17, C17 + 1,
              8 * C17 - 1, 8 * C17 + 1, 16 * C17 + 1]:
        lims = [None, 1 << 40] + ([n] if n else []) + ([n - 1] if n > 1 else []) + [1 << max(1, (n - 1).bit_length())]
        for lim in lims:
            out.append(("merkleize", n, lim))
    for nb in [0, 1, 8, 31, 32, 33, 8 * 256, 8 * 257, 2048, 2049, 4 * 8 * C17 - 8, 4 * 8 * C17, 4 * 8 * C17 + 8, 32 * C17 + 1]:
        nch = (nb + 31) // 32
        for lim, is_list in ((1 << 38, True), (1 << 35, True), (max(1, nch), False), (max(1, nch) * 2, True)):
            out.append(("packed", nb, lim, is_list))
        if nch > 1:
            out.append(("packed", nb, nch - 1, True))
    for n in [0, 1, 2, 64, 65, 255, 256, 257, 32768, 65537, C17 - 1, C17, C17 + 1]:
        for lim in (1 << 40, max(1, n), 1 << max(1, (n - 1).bit_length())) + ((n - 1,) if n > 1 else ()):
            out.append(("validators", n, lim))
    for ln in range(0, 301):
        out.append(("hash", ln))
    return out


def prim_input(case):
    rng = np.random.default_rng(case[1] * 7919 + len(case[0]))
    if case[0] == "merkleize":
        return rng.integers(0, 256, 32 * case[1], dtype=np.uint8)
    if case[0] == "packed":
        return rng.integers(0, 256, case[1], dtype=np.uint8)
    if case[0] == "validators":
        from ethereum_consensus_b200 import state as S
        return S.synth_state(case[1], "minimal", seed=case[1]).validators.view(np.uint8).reshape(-1) if case[1] else np.zeros(0, np.uint8)
    return rng.integers(0, 256, case[1], dtype=np.uint8)


def prim_want(O, case):
    d = prim_input(case)
    out = ctypes.create_string_buffer(32)
    p = d.ctypes.data if d.size else None
    if case[0] == "merkleize":
        n, lim = case[1], case[2]
        rc = O.orc_merkleize(p, n, lim or 0, NT, out)
    elif case[0] == "packed":
        nb, lim, is_list = case[1], case[2], case[3]
        rc = 0 if (nb + 31) // 32 <= lim else -1
        if rc == 0:
            O.orc_htr_packed(p, nb, lim, int(is_list), nb // 8, NT, out)
    elif case[0] == "validators":
        rc = 0 if case[1] <= case[2] else -1
        if rc == 0:
            O.orc_htr_validators(p, case[1], case[2], NT, out)
    else:
        return hashlib.sha256(d.tobytes()).digest()
    return out.raw if rc == 0 else REJECT


def prim_got(case):
    from ethereum_consensus_b200 import ssz
    d = prim_input(case)
    if case[0] == "merkleize":
        return dev(ssz.merkleize, d, case[2])
    if case[0] == "packed":
        return dev(ssz.hash_tree_root_packed, d, case[2], case[3], case[1] // 8)
    if case[0] == "validators":
        return dev(ssz.hash_tree_root_validators, d, case[1], case[2])
    return ssz.hash(d.tobytes())


def check_a(T, wants):
    for case, want in zip(prim_cases(), wants):
        T.check(f"a. {case[0]}", want, prim_got(case), f"case {case}")


# ---------------------------------------------------------------------------------------------------------- b. whole states
def check_b(T, wants, worlds=WORLDS):
    from ethereum_consensus_b200 import ssz
    for spec, want in zip(sc.state_specs(), wants):
        b = sc.serialized(spec)
        p = spec["preset"]
        replay = f"state {spec['name']} seed {spec['seed']:#x}"
        T.check("b. one-shot", want, dev(ssz.hash_tree_root_beacon_state, b, p), replay)
        h = ssz.DeviceBeaconState(b, p)
        T.check("b. resident", want, h.hash_tree_root(), replay)
        T.check("b. resident, again", want, h.hash_tree_root(), replay)
        T.check("b. resident, incremental with nothing dirty", want, h.hash_tree_root_incremental(), replay)
        h.close()
        for w in worlds:
            roots = b"".join(ssz.shard_roots(b, p, r, w) for r in range(w))
            T.check(f"b. shard_roots + combine_roots", want, dev(ssz.combine_roots, b, p, w, roots), f"{replay} world {w}")


# ---------------------------------------------------------------------------------------------------------- c. incremental
def script_wants(O, spec, seed):
    """Oracle roots at every root step of the script (C oracle; hashlib too where the state is small)."""
    host = sc.serialized(spec).copy()
    lay = sc.layout_of(host, spec["preset"])
    want = []
    for st in sc.script(spec, seed):
        if st[0] == "root":
            r = c_root(O, host, spec["preset"])
            if small_state(spec) and spec["preset"] == "minimal":
                assert r == hashlib_root(host, spec["preset"]), (spec["name"], st[1])
            want.append(r)
        else:
            sc.apply(host, st, spec["preset"], lay)
    return want


class Resident:
    """A resident state and the host copy its script is applied to, stepping through the script root by root."""

    def __init__(self, spec, seed, wants):
        from ethereum_consensus_b200 import ssz
        self.spec, self.seed, self.wants = spec, seed, wants
        self.host = sc.serialized(spec).copy()
        self.lay = sc.layout_of(self.host, spec["preset"])
        self.steps = sc.script(spec, seed)
        self.pos, self.k = 0, 0
        self.h = ssz.DeviceBeaconState(self.host, spec["preset"])

    def done(self):
        return self.pos >= len(self.steps)

    def advance(self, T, section):
        """Applies the steps up to the next root step, then checks incremental, full and one-shot roots against the oracle."""
        from ethereum_consensus_b200 import ssz
        while not self.done():
            st = self.steps[self.pos]
            self.pos += 1
            if st[0] == "elements":
                self.h.update_elements(st[1], st[2], st[3])
            elif st[0] == "bytes":
                self.h.update_bytes(st[1], st[2])
            if st[0] != "root":
                sc.apply(self.host, st, self.spec["preset"], self.lay)
                continue
            want = self.wants[self.k]
            self.k += 1
            replay = f"state {self.spec['name']} seed {self.spec['seed']:#x} script seed {self.seed} step {self.pos - 1} ({st[1]})"
            T.check(section + ", incremental", want, self.h.hash_tree_root_incremental(), replay)
            T.check(section + ", full", want, self.h.hash_tree_root(), replay)
            T.check(section + ", one-shot of the host copy", want, ssz.hash_tree_root_beacon_state(self.host, self.spec["preset"]), replay)
            return

    def close(self):
        self.h.close()


def check_c(T, wants):
    for k, (spec, want) in enumerate(zip(sc.script_specs(), wants)):
        r = Resident(spec, k, want)
        while not r.done():
            r.advance(T, "c. script")
        r.close()


# ---------------------------------------------------------------------------------------------------------- f. two handles
def check_f(T, wants_c, wants_b):
    """A minimal and a mainnet resident state, stepped alternately, with one-shot hashes and shuffles in between."""
    from ethereum_consensus_b200 import shuffling, ssz
    from oracle import shuffle_oracle as sh
    specs = sc.script_specs()
    pick = [i for i, s in enumerate(specs) if (s["preset"], s["n"]) in (("minimal", 2049), ("mainnet", 65537))]
    hs = [Resident(specs[i], 100 + i, wants_c[len(specs) + j]) for j, i in enumerate(pick)]
    states = sc.state_specs()
    other = next(i for i, s in enumerate(states) if (s["preset"], s["n"]) == ("mainnet", 1000))
    other_b = sc.serialized(states[other])
    seed = hashlib.sha256(b"two handles").digest()
    shuf_want = sh.shuffled_indices_numpy(1000, seed, 90)
    step = 0
    while not all(h.done() for h in hs):
        for h in hs:
            if h.done():
                continue
            h.advance(T, "f. alternating handles")
            T.check("f. one-shot between handles", wants_b[other], ssz.hash_tree_root_beacon_state(other_b, "mainnet"), f"after step {step}")
            T.check("f. shuffle between handles", True, bool(np.array_equal(shuffling.compute_shuffled_indices(1000, seed, 90), shuf_want)),
                    f"after step {step}")
            recs = h.host[h.lay["validators"][0]: h.lay["validators"][0] + h.lay["validators"][1]]
            act = sc.active_numpy(recs, 1 << 17)
            got = shuffling.state_shuffled_active_indices(h.h, 1 << 17, seed, 10)
            T.check("f. resident shuffle between handles", True, bool(np.array_equal(got, sh.shuffled_indices_numpy(act, seed, 10))),
                    f"{h.spec['name']} after step {step}")
            step += 1
    for h in hs:
        h.close()


def f_wants(O):
    specs = sc.script_specs()
    pick = [i for i, s in enumerate(specs) if (s["preset"], s["n"]) in (("minimal", 2049), ("mainnet", 65537))]
    return [script_wants(O, specs[i], 100 + i) for i in pick]


# ---------------------------------------------------------------------------------------------------------- inputs
_CACHE = {}


def wants(O):
    if "w" not in _CACHE:
        t = time.time()
        w = {"a": [prim_want(O, c) for c in prim_cases()]}
        w["b"] = []
        for spec in sc.state_specs():
            b = sc.serialized(spec)
            r = c_root(O, b, spec["preset"])
            if small_state(spec):
                assert r == hashlib_root(b, spec["preset"]), spec["name"]
            w["b"].append(r)
        w["c"] = [script_wants(O, spec, k) for k, spec in enumerate(sc.script_specs())]
        w["c"] += f_wants(O)
        _CACHE["w"] = w
        print(f"oracle side: {time.time() - t:.1f} s")
    return _CACHE["w"]


def minimums():
    n_scripts = len(sc.script_specs())
    return {"a. hash": 301, "a. merkleize": 100, "a. packed": 50, "a. validators": 40,
            "b. one-shot": len(sc.state_specs()), "c. script, incremental": 8 * n_scripts}


def run_abcf(O_wants, tag="", worlds=WORLDS):
    T = Tally(tag)
    t = time.time()
    check_a(T, O_wants["a"])
    print(f"a. wall {time.time() - t:.1f} s"); t = time.time()
    check_b(T, O_wants["b"], worlds)
    print(f"b. wall {time.time() - t:.1f} s"); t = time.time()
    n = len(sc.script_specs())
    check_c(T, O_wants["c"][:n])
    print(f"c. wall {time.time() - t:.1f} s"); t = time.time()
    check_f(T, O_wants["c"], O_wants["b"])
    print(f"f. wall {time.time() - t:.1f} s")
    return T


# ---------------------------------------------------------------------------------------------------------- tests
def test_a_b_c_f_default_kernels(engine, oracle_ssz_c):
    W = wants(oracle_ssz_c)
    T = run_abcf(W)
    T.report(minimums())
    assert any(w == REJECT for w in W["a"]) and any(w != REJECT for w in W["a"])


def test_d_malformed_encodings(engine, oracle_ssz_c):
    """The device rejects (MerkleizationError) exactly the encodings the C oracle rejects, on every entry point, and
    hashes the accepted controls to the oracle's root."""
    from ethereum_consensus_b200 import ssz
    T = Tally()
    cases = sc.malformed_cases()
    for name, preset, b, _ in cases:
        want = c_root(oracle_ssz_c, b, preset)
        T.check("d. one-shot", want, dev(ssz.hash_tree_root_beacon_state, b, preset), name)

        def upload():
            h = ssz.DeviceBeaconState(b, preset)
            r = h.hash_tree_root()
            h.close()
            return r
        T.check("d. resident upload", want, dev(upload), name)
        for w in (1, 4):
            def shard_combine(w=w):
                roots = b"".join(ssz.shard_roots(b, preset, r, w) for r in range(w))
                return ssz.combine_roots(b, preset, w, roots)
            T.check(f"d. shard_roots + combine_roots", want, dev(shard_combine), f"{name} world {w}")
        T.check("d. combine_roots alone", want if want == REJECT else "accepted",
                "accepted" if dev(ssz.combine_roots, b, preset, 1, bytes(160)) != REJECT else REJECT, name)
    T.report({"d. one-shot": len(cases)})
    assert sum(c_root(oracle_ssz_c, b, p) == REJECT for _, p, b, _ in cases) >= 60


def test_e_shuffling_and_active_indices(engine, oracle_ssz_c):
    from ethereum_consensus_b200 import _lib, shuffling, ssz
    from oracle import shuffle_oracle as sh
    T = Tally()
    t = time.time()
    for c in sc.shuffle_cases():
        seed = sc.SEEDS[c["seed"]]
        vals = sc.shuffle_values(c)
        n = c["n"]
        if n <= 64:
            want = sh.compute_shuffled_indices(list(range(n)) if vals is None else vals.tolist(), seed, c["rounds"])
        else:
            want = sh.shuffled_indices_numpy(n if vals is None else vals, seed, c["rounds"]).tolist()
        got = shuffling.compute_shuffled_indices(n if vals is None else vals, seed, c["rounds"]).tolist()
        T.check("e. compute_shuffled_indices", want, got, f"n {n} rounds {c['rounds']} seed {c['seed']} values {c['values']}")
        if 0 < n <= 4097 and c["rounds"] in (1, 255):
            for i in {0, n // 2, n - 1}:
                T.check("e. compute_shuffled_index", sh.compute_shuffled_index(i, n, seed, c["rounds"]),
                        shuffling.compute_shuffled_index(i, n, seed, c["rounds"]), f"i {i} n {n} rounds {c['rounds']}")
    for n in (1, 5, 300):
        try:
            shuffling.compute_shuffled_indices(n, sc.SEEDS["random"], 256)
            got = "accepted"
        except _lib.EngineError:
            got = REJECT
        T.check("e. 256 rounds rejected", REJECT, got, f"n {n}")
    print(f"e. shuffles wall {time.time() - t:.1f} s"); t = time.time()
    for r in sc.registry_cases():
        recs = sc.registry(r["n"], r["pattern"])
        for epoch in r["epochs"]:
            want = sh.get_active_validator_indices(bytes(recs), epoch) if r["n"] <= 1000 else sc.active_numpy(recs, epoch).tolist()
            T.check("e. get_active_validator_indices", want, shuffling.get_active_validator_indices(recs, epoch).tolist(),
                    f"registry {r['name']} epoch {epoch}")
    print(f"e. registries wall {time.time() - t:.1f} s"); t = time.time()
    # resident states whose validators change through update_elements
    E = 1000
    seed = sc.SEEDS["random"]
    for preset, n, pattern in (("minimal", 257, "edges"), ("mainnet", sc.SCAN_CTAS * sc.CTA + 1, "runs")):
        spec = dict(preset=preset, n=n, hr=2, hs=3, votes=3, extra=b"e", seed=0xE0 + n)
        host = sc.serialized(spec).copy()
        lay = sc.layout_of(host, preset)
        vo, vl = lay["validators"]
        h = ssz.DeviceBeaconState(host, preset)
        recs = sc.registry(n, pattern)
        h.update_elements("validators", np.arange(n, dtype=np.uint64), recs)
        host[vo:vo + vl] = recs
        few = np.array(sorted({0, 1, 255, 256, n // 2, n - 2, n - 1}), dtype=np.uint64)
        v = host[vo:vo + vl].reshape(n, 121)
        new = v[few.astype(np.int64)].copy().view(sc.S.VALIDATOR_DTYPE).reshape(-1)
        new["activation_epoch"] = E
        new["exit_epoch"] = [E + 1 if k % 2 else E for k in range(len(few))]
        h.update_elements("validators", few, new.view(np.uint8).tobytes())
        v[few.astype(np.int64)] = new.view(np.uint8).reshape(-1, 121)
        for epoch in (E - 1, E, E + 1):
            act = sc.active_numpy(host[vo:vo + vl], epoch)
            for rounds in ((0, 1, 90, 255) if n < 1000 else (10,)):
                got = shuffling.state_shuffled_active_indices(h, epoch, seed, rounds)
                T.check("e. state_shuffled_active_indices after update_elements", True,
                        bool(np.array_equal(got, sh.shuffled_indices_numpy(act, seed, rounds))), f"{preset} n {n} epoch {epoch} rounds {rounds}")
        try:
            shuffling.state_shuffled_active_indices(h, E, seed, 256)
            got = "accepted"
        except _lib.EngineError:
            got = REJECT
        T.check("e. 256 rounds rejected", REJECT, got, f"resident {preset} n {n}")
        T.check("e. incremental root after the epoch updates", c_root(oracle_ssz_c, host, preset), h.hash_tree_root_incremental(),
                f"{preset} n {n}")
        h.close()
    print(f"e. resident wall {time.time() - t:.1f} s")
    T.report({"e. compute_shuffled_indices": len(sc.shuffle_cases())})


@pytest.mark.parametrize("env", ENV_VARIANTS, ids=lambda e: "-".join(f"{k[5:].lower()}_{v}" for k, v in e.items()))
def test_env_variants_in_child_processes(oracle_ssz_c, tmp_path, env):
    """Sections a, b, c and f with the fold into k_merkle_coop off, which only the environment selects (read once per
    process): one child process per setting, oracle roots from here."""
    t = time.time()
    path = tmp_path / "wants.pkl"
    path.write_bytes(pickle.dumps(wants(oracle_ssz_c)))
    child_env = dict(os.environ, **env)
    p = subprocess.Popen([sys.executable, "-m", "tests.test_ssz_device_soak_gpu", str(path)], cwd=str(ROOT), env=child_env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out = p.communicate(timeout=1200)[0]
    except subprocess.TimeoutExpired:
        p.kill()
        out = p.communicate()[0]
    print(out)
    print(f"child {env} wall {time.time() - t:.1f} s")
    assert p.returncode == 0, out
    assert "CHILD_OK" in out, out


def _child(path):
    from ethereum_consensus_b200 import _lib
    _lib.init(0)
    W = pickle.loads(Path(path).read_bytes())
    tag = " [" + ", ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("B200_SSZ_")) + "]"
    T = run_abcf(W, tag)
    T.report(minimums())
    print("CHILD_OK")


if __name__ == "__main__":
    _child(sys.argv[1])
