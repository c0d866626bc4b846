"""GPU: aggregate_verify batches where the device splits them (tests/aggregate_verify_grid_cases.py, shapes checked on the
CPU by tests/test_aggregate_verify_grid_cases.py).  Every case runs through `crypto.aggregate_verify_batch` right after a
poison call of the same or a larger layout whose tuples all pass, so that a kernel that skips a write or a tuple flag
that is lost reads passing Miller values, fold pieces or SUCCESS codes and shows up as a wrong row; codes are compared row
by row and the launch count with the layout model's.  The same cases run through `Registry.aggregate_verify_batch` (some
keys appended after the load), the tuples of at most 64 pairs through the single `b200_aggregate_verify` (after a
passing single call), and the alignment, warp and switch sections again under every vm_cta and both forced team sizes."""
from __future__ import annotations

import time

import pytest

from tests import aggregate_verify_grid_cases as g
from tests.test_aggregate_verify_batch_gpu import _arr, _batch, _registry_batch, _single, _vm_cta_in_effect

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _wall():
    t = time.time()
    yield
    print(f"\ntest_aggregate_verify_grid_gpu.py wall {time.time() - t:.1f} s")


@pytest.fixture(scope="module")
def mats(oracle_bls_c):
    """Material of every tuple of every case and of every poison call, by spec."""
    g.bind(oracle_bls_c)
    specs = []
    for case in g.all_cases():
        specs += case.specs + g.poison(case).specs
    uniq = list(dict.fromkeys(specs))
    return dict(zip(uniq, g.materials(uniq)))


def _launches():
    from ethereum_consensus_b200 import _lib
    return int(_lib.lib().b200_launch_count())


def _rows(case, got, call):
    return [f"{call}: case '{case.name}' tuple {t} ({sp.kind} n={sp.n} m={sp.msgs}): got {c}, want {sp.want}"
            for t, (sp, c) in enumerate(zip(case.specs, got)) if c != sp.want]


def _run(case, mats, call="strict", reg=None, where=None, knobs=(32, g.TEAM16_MAX)):
    """Poison call, then the case; -> mismatch lines."""
    P = g.poison(case)
    ptuples = [mats[x] for x in P.specs]
    pgot = _batch(ptuples)
    bad = [f"{call} {knobs}: poison for '{case.name}' tuple {t} got {c}" for t, c in enumerate(pgot) if c != g.SUCCESS]
    tuples = [mats[x] for x in case.specs]
    n0 = _launches()
    got = _batch(tuples) if reg is None else _registry_batch(reg, where, tuples)
    k = _launches() - n0
    bad += _rows(case, got, f"{call} {knobs}")
    want_k = g.layout(case, *knobs, registry=reg is not None).launches
    if k != want_k:
        bad.append(f"{call} {knobs}: case '{case.name}': {k} launches, want {want_k}")
    return bad


def test_strict_batches(engine, mats):
    from ethereum_consensus_b200 import crypto
    bad = []
    try:
        crypto.tune("vm_cta", 32)
        for case in g.all_cases():
            bad += _run(case, mats)
    finally:
        crypto.tune("vm_cta", _vm_cta_in_effect())
    assert not bad, "\n".join(bad[:30])


def test_registry_equals_strict(engine, mats):
    from ethereum_consensus_b200 import crypto
    keys = list(dict.fromkeys(k for case in g.all_cases() for x in case.specs for k in mats[x]["pks"]))
    where = {k: i for i, k in enumerate(keys)}
    cut = len(keys) * 3 // 5
    reg = crypto.Registry(_arr(b"".join(keys[:cut])))
    reg.append(_arr(b"".join(keys[cut:])))              # keys appended after the load
    assert reg.n == len(keys)
    bad = []
    try:
        crypto.tune("vm_cta", 32)
        for case in g.all_cases():
            bad += _run(case, mats, "registry", reg, where)
            bad += _rows(case, _batch([mats[x] for x in case.specs]), "strict after registry")
    finally:
        crypto.tune("vm_cta", _vm_cta_in_effect())
    assert not bad, "\n".join(bad[:30])


def test_single_calls(engine, mats):
    """Each distinct tuple of at most 64 pairs (shape failures of at most 64 keys included), right after a passing single
    call of a tuple with as many keys."""
    bad, seen = [], set()
    for case in g.all_cases():
        for t, sp in enumerate(case.specs):
            if sp in seen or sp.pairs > 64 or sp.n > 64:
                continue
            seen.add(sp)
            ok = mats[g.Spec("valid", max(sp.n, 1))] if g.Spec("valid", max(sp.n, 1)) in mats else None
            if ok is not None and _single(ok) != g.SUCCESS:
                bad.append(f"single: passing call before '{case.name}' tuple {t} failed")
            c = _single(mats[sp])
            if c != sp.want:
                bad.append(f"single: case '{case.name}' tuple {t} ({sp.kind} n={sp.n} m={sp.msgs}): got {c}, want {sp.want}")
    assert len(seen) > 100
    assert not bad, "\n".join(bad[:30])


@pytest.mark.parametrize("team16_max", [0, 1 << 30])
def test_knobs(engine, mats, team16_max):
    from ethereum_consensus_b200 import crypto
    cases = [c for c in g.all_cases() if c.section in ("align", "warps", "switch")]
    bad = []
    try:
        crypto.tune("vm_team16_max", team16_max)
        for cta in g.VM_CTAS:
            crypto.tune("vm_cta", cta)
            for case in cases:
                bad += _run(case, mats, "strict", knobs=(cta, team16_max))
    finally:
        crypto.tune("vm_team16_max", g.TEAM16_MAX)
        crypto.tune("vm_cta", _vm_cta_in_effect())
    assert not bad, "\n".join(bad[:30])
    # restored: the default knobs give the default launch shapes again
    case = next(c for c in g.all_cases() if c.name == "T = 2 049, mostly shape failures")
    assert not _run(case, mats, knobs=(_vm_cta_in_effect(), g.TEAM16_MAX))
