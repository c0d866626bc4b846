"""GPU: shape changes of a device-resident deneb BeaconState (append_elements, set_field, add_validators) through the CUDA
library, step by step against the C oracle (liboracle_ssz.so on all host threads) applied to the host mirror.

After every step: the incremental root of one handle, b200_state_root of a second handle given the same steps, and a
one-shot device hash of the mirror's serialization all equal the C oracle's root of the mirror; a refused step is refused
by the library with the mirror's code and leaves both handles' roots where they were.

Sections: a. a minimal-preset chain walk (~200 blocks: eth1 resets, summary appends, 0..16 deposits, indexed writes at
appended validators, update_bytes at shifted offsets); b. boundary scripts (hand-offs, the 2^17 fold, the reserved
capacity, vote bound, headers, malformed encodings, a stale offset); c. 8 mainnet blocks on the 2^20-validator state;
d. shuffled active indices over appended validators; e. the new calls on a sharded handle; f. a and b in a child process
with B200_SSZ_FOLD=0 (read once per process).  Scripts: tests/state_reshape_cases.py.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from ethereum_consensus_b200 import state as S  # noqa: E402
from tests import ssz_soak_cases as sc  # noqa: E402
from tests import state_reshape_cases as rc  # noqa: E402

pytestmark = pytest.mark.gpu
NT = os.cpu_count() or 1


def c_root(O, b, preset):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    out = ctypes.create_string_buffer(32)
    r = O.orc_htr_beacon_state_deneb(b.ctypes.data, b.size, 0 if preset == "mainnet" else 1, NT, out)
    assert r == 0, r
    return out.raw


def dev_apply(h, step):
    """Apply a step to a DeviceBeaconState; None, or the refusal kind (the codes ReshapeRefused names)."""
    from ethereum_consensus_b200 import _lib, ssz
    kind = step[0]
    try:
        if kind == "push":
            if step[1] not in h.RESHAPE_FIELDS:      # an id the library does not take
                _lib.check(_lib.lib().b200_state_append_elements(h._h, 99, _lib.ptr(step[2]), 1), "append")
            else:
                h.append_elements(step[1], step[2])
        elif kind == "set":
            if step[1] not in h.SET_FIELDS:
                buf = np.frombuffer(bytes(step[2]) or b"\0", dtype=np.uint8)
                _lib.check(_lib.lib().b200_state_set_field(h._h, 0, _lib.ptr(buf), len(step[2])), "set_field")
            else:
                h.set_field(step[1], step[2])
        elif kind == "deposits":
            h.add_validators(step[1], step[2])
        elif kind == "elements":
            h.update_elements(step[1], step[2], step[3])
        elif kind == "bytes":
            h.update_bytes(step[1], step[2])
        else:
            raise ValueError(kind)
    except ssz.MerkleizationError as e:
        return "limit" if "limit" in str(e) else "malformed"
    except _lib.EngineError as e:
        assert e.code == _lib.ERR_BAD_ARG, e
        return "bad_arg"
    return None


class Pair:
    """Two handles of the mirror's state: one re-hashed incrementally, one with b200_state_root, after every step."""

    def __init__(self, O, st):
        from ethereum_consensus_b200 import ssz
        self.O, self.st = O, st
        ser = S.serialize(st)
        self.inc = ssz.DeviceBeaconState(ser, st.preset)
        self.full = ssz.DeviceBeaconState(ser, st.preset)
        self.counts = {"steps": 0, "refused": 0}

    def step(self, step, check=True, label=""):
        try:
            rc.apply(self.st, step)
            want = None
        except S.ReshapeRefused as e:
            want = e.kind
        for h in (self.inc, self.full):
            got = dev_apply(h, step)
            assert got == want, (label, step[:2], want, got)
        self.counts["steps"] += 1
        self.counts["refused"] += want is not None
        if check or want is not None:
            self.check(f"{label} after {step[0]} {step[1] if isinstance(step[1], str) else ''}")

    def check(self, where):
        from ethereum_consensus_b200 import ssz
        ser = S.serialize(self.st)
        want = c_root(self.O, ser, self.st.preset)
        assert self.inc.hash_tree_root_incremental() == want, f"incremental root {where}"
        assert self.full.hash_tree_root() == want, f"state_root {where}"
        assert ssz.hash_tree_root_beacon_state(ser, self.st.preset) == want, f"one-shot {where}"
        assert self.inc.n_validators == len(self.st.validators), where

    def close(self):
        self.inc.close()
        self.full.close()


def run_walk(O):
    spec = rc.walk_spec()
    st, steps = rc.walk(spec)
    p = Pair(O, st)
    for s in steps:
        p.step(s, label=spec["name"])
    p.close()
    assert p.counts["refused"] == 0
    return p.counts


def run_boundaries(O):
    n = 0
    for spec in rc.boundary_scripts():
        st, steps = rc.boundary_run(spec)
        p = Pair(O, st)
        for s in steps:
            p.step(s, label=spec["name"])
        n += p.counts["steps"]
        p.close()
    return n


def oracle_lib():
    subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True, capture_output=True)
    lib = ctypes.CDLL(str(ROOT / "oracle" / "liboracle_ssz.so"))
    lib.orc_htr_beacon_state_deneb.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.orc_htr_beacon_state_deneb.restype = ctypes.c_int
    return lib


# ---------------------------------------------------------------------------------------------------------- a, b
def test_a_chain_walk_minimal(engine, oracle_ssz_c):
    t = time.time()
    counts = run_walk(oracle_ssz_c)
    print(f"a. chain walk: {counts['steps']} steps, wall {time.time() - t:.1f} s")


def test_b_boundaries(engine, oracle_ssz_c):
    t = time.time()
    n = run_boundaries(oracle_ssz_c)
    print(f"b. boundaries: {n} steps, wall {time.time() - t:.1f} s")


# ---------------------------------------------------------------------------------------------------------- c
def test_c_mainnet_blocks(engine, oracle_ssz_c):
    """BASELINE config 3 (2^20 validators) through 8 blocks of 16 deposits, one vote, a new header, 513 balances and
    N/32 participation flags; incremental root and one-shot root per block, b200_state_root after the last."""
    from ethereum_consensus_b200 import ssz
    t = time.time()
    st = S.synth_state(1 << 20, "mainnet")
    h = ssz.DeviceBeaconState(S.serialize(st), "mainnet")
    for step in rc.mainnet_blocks(st, 8, seed=0xB10C):
        if step[0] == "root":
            ser = S.serialize(st)
            want = c_root(oracle_ssz_c, ser, "mainnet")
            assert h.hash_tree_root_incremental() == want, f"block {step[1]}"
            assert ssz.hash_tree_root_beacon_state(ser, "mainnet") == want, f"block {step[1]}"
            continue
        rc.apply(st, step)
        assert dev_apply(h, step) is None, step[:2]
    assert h.hash_tree_root() == c_root(oracle_ssz_c, S.serialize(st), "mainnet")
    assert h.n_validators == (1 << 20) + 8 * rc.MAX_DEPOSITS
    h.close()
    print(f"c. mainnet blocks wall {time.time() - t:.1f} s")


# ---------------------------------------------------------------------------------------------------------- d
def test_d_shuffled_active_indices_after_appends(engine):
    from ethereum_consensus_b200 import shuffling, ssz
    from oracle import shuffle_oracle as sh
    rng = np.random.default_rng(4)
    for n0, k in ((0, 5), (63, 3), (1000, 16), (rc.HEADROOM_MIN, 70000)):   # the last one past the reserved capacity
        st = rc.initial_state("minimal", n0, 3)
        h = ssz.DeviceBeaconState(S.serialize(st), "minimal")
        step = rc.deposits(rng, k, 100)
        rc.apply(st, step)
        assert dev_apply(h, step) is None
        recs = np.frombuffer(st.validators.tobytes(), dtype=np.uint8)
        seed = bytes(range(32))
        for epoch in (99, 100, 1 << 17):
            act = sc.active_numpy(recs, epoch)
            new_active = int(np.sum(act >= n0))
            if epoch == 100:
                assert new_active > 0, (n0, k)     # some appended validators are active at epoch 100
            got = shuffling.state_shuffled_active_indices(h, epoch, seed, 10)
            assert np.array_equal(got, sh.shuffled_indices_numpy(act, seed, 10)), (n0, k, epoch)
        h.close()


# ---------------------------------------------------------------------------------------------------------- e
def test_e_sharded_handle_refuses_reshapes(engine):
    from ethereum_consensus_b200 import _lib, parallel, ssz
    parallel.comm_init(0, 1)
    st = rc.initial_state("minimal", 70, 5)
    h = ssz.DeviceBeaconState(S.serialize(st), "minimal", sharded=True)
    root = h.hash_tree_root()
    buf = np.zeros(121 * 2, np.uint8)
    L = _lib.lib()
    for f in range(7):
        assert L.b200_state_append_elements(h._h, f, _lib.ptr(buf), 1) == _lib.ERR_BAD_ARG, f
    hdr = np.frombuffer(st.payload_header(), dtype=np.uint8)
    assert L.b200_state_set_field(h._h, 5, _lib.ptr(buf), 72) == _lib.ERR_BAD_ARG
    assert L.b200_state_set_field(h._h, 7, _lib.ptr(hdr), hdr.size) == _lib.ERR_BAD_ARG
    assert h.hash_tree_root() == root
    h.close()


# ---------------------------------------------------------------------------------------------------------- f
def test_f_fold_off_in_a_child_process(oracle_ssz_c):
    """Sections a and b with the fold into k_merkle_coop off (B200_SSZ_FOLD is read once per process): which jobs fold
    depends on list lengths, so it changes as the lists grow."""
    t = time.time()
    env = dict(os.environ, B200_SSZ_FOLD="0")
    p = subprocess.Popen([sys.executable, "-m", "tests.test_state_reshape_gpu"], cwd=str(ROOT), env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out = p.communicate(timeout=1800)[0]
    except subprocess.TimeoutExpired:
        p.kill()
        out = p.communicate()[0]
    print(out)
    print(f"f. child wall {time.time() - t:.1f} s")
    assert p.returncode == 0, out
    assert "CHILD_OK" in out, out


def _child():
    from ethereum_consensus_b200 import _lib
    _lib.init(0)
    O = oracle_lib()
    counts = run_walk(O)
    n = run_boundaries(O)
    print(f"fold off: walk {counts['steps']} steps, boundaries {n} steps")
    print("CHILD_OK")


if __name__ == "__main__":
    _child()
