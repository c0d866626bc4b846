"""CPU: the SSZ / shuffling soak's case generators (tests/ssz_soak_cases.py) before any of them reaches the device.

The cases must contain every planner boundary they are named for, the C and hashlib oracles must agree on the small
states and on every update script applied on the host, and the C oracle must reject every malformed encoding (and accept
the controls next to them).  tests/test_ssz_device_soak_gpu.py then compares the CUDA library with the same oracles.
"""
import ctypes
import os

import numpy as np
import pytest

from oracle import shuffle_oracle as sh
from oracle import ssz_oracle as so
from ethereum_consensus_b200 import state as S
from tests import ssz_soak_cases as sc

NT = os.cpu_count() or 1


def c_root(O, b, preset):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    out = ctypes.create_string_buffer(32)
    rc = O.orc_htr_beacon_state_deneb(b.ctypes.data, b.size, 0 if preset == "mainnet" else 1, NT, out)
    return out.raw if rc == 0 else rc


def hashlib_root(b, preset):
    return so.beacon_state_type(preset).htr(S.to_oracle_value(sc.deserialize(b, preset)))


def test_state_cases_contain_every_boundary():
    have = {(s["preset"], s["n"]) for s in sc.state_specs()}
    for name, pairs in sc.boundaries().items():
        for p in pairs:
            assert p in have, f"boundary '{name}': no state with {p[1]} validators ({p[0]})"
    assert sc.slices(65535) == [65535]
    assert sc.slices(65536) == [32768, 32768]
    s = sc.slices(65537)
    assert len(s) == 2 and s[-1] < s[0] and s[0] % 256 == 0
    s = sc.slices(4 * sc.COOP_MAX + 4)
    assert len(s) == 16 and s[-1] < s[0]
    assert any(n % 256 for _, n in have if n > 256)
    for preset in ("minimal", "mainnet"):
        specs = [s for s in sc.state_specs() if s["preset"] == preset]
        bound = S.PRESETS[preset]["ETH1_DATA_VOTES_BOUND"]
        assert {0, bound} <= {s["votes"] for s in specs}, preset
        assert {0, 64, 65} <= {s["hr"] for s in specs} and max(s["hr"] for s in specs) >= 300, preset
        assert {0, 64, 65} <= {s["hs"] for s in specs} and max(s["hs"] for s in specs) >= 300, preset
        assert {0, 1, 31, 32} <= {len(s["extra"]) for s in specs}, preset


def test_shuffle_and_registry_cases_cover_their_edges():
    sizes = {c["n"] for c in sc.shuffle_cases()}
    assert set(range(21)) <= sizes
    for k in range(8, 22):
        assert {(1 << k) - 1, 1 << k, (1 << k) + 1} <= sizes, k
    small = [c for c in sc.shuffle_cases() if c["n"] <= 4097]
    assert {(r, s) for c in small for r, s in [(c["rounds"], c["seed"])]} == {(r, s) for r in sc.ROUNDS for s in sc.SEEDS}
    assert any(c["values"] for c in sc.shuffle_cases()) and any(not c["values"] for c in sc.shuffle_cases())
    v = sc.shuffle_values(next(c for c in sc.shuffle_cases() if c["values"] and c["n"] > 100))
    assert int(v.max()) == (1 << 64) - 1 and (v >= np.uint64(1 << 32)).mean() > 0.9    # full 64-bit index values
    regs = {r["n"] for r in sc.registry_cases()}
    assert max(regs) // 256 > sc.SCAN_CTAS and {262_144, 262_145, 1 << 20} <= regs
    assert {"all", "none", "edges", "runs", "random"} <= {r["pattern"] for r in sc.registry_cases()}


def test_registry_patterns_and_numpy_active_indices_match_the_oracle():
    E = 1000
    for n in (1, 31, 32, 33, 255, 256, 257, 1000):
        for pat in ("all", "none", "edges", "runs", "random"):
            recs = sc.registry(n, pat)
            for epoch in (0, E - 1, E, E + 1, sc.FAR - 1, sc.FAR):
                assert sc.active_numpy(recs, epoch).tolist() == sh.get_active_validator_indices(bytes(recs), epoch), (pat, n, epoch)
    recs = sc.registry(600, "edges")
    act = sc.active_numpy(recs, E)
    assert 0 < len(act) < 600          # the boundary epochs split the registry
    assert len(sc.active_numpy(sc.registry(600, "all"), E)) == 600 and len(sc.active_numpy(sc.registry(600, "none"), E)) == 0


def test_oracles_agree_on_small_states(oracle_ssz_c):
    for spec in sc.state_specs():
        if spec["preset"] == "mainnet" and spec["n"] > 257 or spec["n"] > 2049:
            continue
        b = sc.serialized(spec)
        assert np.array_equal(S.serialize(sc.deserialize(b, spec["preset"])), b), spec["name"]
        assert c_root(oracle_ssz_c, b, spec["preset"]) == hashlib_root(b, spec["preset"]), spec["name"]


def test_update_scripts_on_the_host(oracle_ssz_c):
    """Every script touches all 28 fields (each of the nine chains among them), keeps the layout, and the two oracles agree
    on the patched bytes after every root step (hashlib on the small states, C alone on the large ones)."""
    for k, spec in enumerate(sc.script_specs()):
        steps = sc.script(spec, seed=k)
        host = sc.serialized(spec).copy()
        lay = sc.layout_of(host, spec["preset"])
        covered = sc.script_fields_covered(steps, lay)
        want_fields = {f for f in sc.FIELDS_28 if lay[f][1]}
        assert covered == want_fields, (spec["name"], want_fields - covered)
        assert {s[1] for s in steps if s[0] == "elements"} == {f for f in sc.BIG_LISTS if lay[f][1]}
        small = spec["n"] <= 2049 if spec["preset"] == "minimal" else spec["n"] <= 257
        roots = set()
        for i, st in enumerate(steps):
            if st[0] == "root":
                r = c_root(oracle_ssz_c, host, spec["preset"])
                assert isinstance(r, bytes), (spec["name"], i, st[1], r)
                if small:
                    assert hashlib_root(host, spec["preset"]) == r, (spec["name"], i, st[1])
                roots.add(r)
            else:
                sc.apply(host, st, spec["preset"], lay)
        assert sc.layout_of(host, spec["preset"]) == lay
        assert len(roots) == sum(s[0] == "root" for s in steps), spec["name"]   # every root step changed the root


def test_c_oracle_rejects_every_malformed_encoding(oracle_ssz_c):
    cases = sc.malformed_cases()
    assert sum(not ok for _, _, _, ok in cases) >= 60
    for name, preset, b, ok in cases:
        r = c_root(oracle_ssz_c, b, preset)
        if ok:
            assert isinstance(r, bytes), name
            assert r == hashlib_root(b, preset), name
        else:
            assert r == -3, (name, r)
