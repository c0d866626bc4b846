"""CPU: the sharded case lists (tests/sharded_cases.py) sit on every rank boundary they name, the Python mirrors of the
library's splits agree with the C rules, the oracle codes are the ones the cases were built to have, the crafted RLC
batches are accepted with the global tuple index and rejected with the per-rank local one; and the loopback
communicator's file and barrier (csrc/comm_loopback.h, built with g++) gather correctly in 2 .. 8 processes, time out
cleanly when a rank never arrives and refuse a header made for another shape."""
from __future__ import annotations

import ctypes
import hashlib
import multiprocessing as mp
import subprocess
import time
from pathlib import Path

import pytest

from ethereum_consensus_b200 import parallel
from tests import rlc_soak_cases as rc
from tests import ssz_soak_cases as sc
from tests import sharded_cases as sh

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def material(oracle_bls_c):
    keys = rc.Keys(oracle_bls_c)
    return keys, sh.Material(oracle_bls_c, keys)


def test_python_splits_match_the_c_rules():
    sizes = set(range(0, 70))
    for w in sh.WORLDS:
        sizes |= set(sh.strict_sizes(w)) | {w, 2 * w + 1}
    for spec in sh.state_specs():
        sizes |= set(sh.state_list_lengths(spec))
    for w in (1,) + sh.WORLDS:
        for n in sorted(sizes):
            for r in range(w):
                lo, cnt = sh.c_tuple_shard(n, w, r)
                assert parallel.tuple_shard(n, w, r) == (lo, lo + cnt), (n, w, r)
                assert parallel.slice_of(n, w, r) == sh.c_slice_of(n, w, r), (n, w, r)
            assert sum(sh.c_tuple_shard(n, w, r)[1] for r in range(w)) == n
            if not w & (w - 1):
                assert sum(sh.c_slice_of(n, w, r)[1] for r in range(w)) == n


@pytest.mark.parametrize("world", sh.WORLDS)
def test_strict_cases_cover_every_rank_end(world, material):
    keys, M = material
    cases = sh.strict_cases(keys, world)
    sizes = {len(b) for _, b, _ in cases}
    assert sizes == set(sh.strict_sizes(world))
    rems = {T % world for T in sizes}
    assert {0, 1, world - 1} <= rems                         # even splits, and low ranks one tuple longer
    assert any(T < world for T in sizes)                     # ranks with empty blocks
    kinds_seen = set()
    zero_key_block = False
    for name, batch, kinds in cases:
        T = len(batch)
        if "a reject at every rank's ends" in name:
            for lo, hi in sh.blocks(T, world):
                if hi > lo:
                    assert kinds[lo] and kinds[hi - 1], (name, lo, hi)
            assert kinds[0] and kinds[T - 1]
        else:
            lo, hi = parallel.tuple_shard(T, world, world // 2)
            zero_key_block |= hi > lo and all(not batch[t].keys for t in range(lo, hi))
        kinds_seen |= set(kinds)
        assert any(len(t.keys) == 0 for t in batch) or T < 17
        assert M.codes(batch) == [sh.KIND_CODE[k] for k in kinds], name
    assert zero_key_block
    assert set(sh.BAD_KINDS) <= kinds_seen


@pytest.mark.parametrize("world", sh.WORLDS)
def test_rlc_cases_straddle_every_rank_boundary(world, material):
    keys, M = material
    cases = sh.rlc_cases(keys, world)
    tags = set().union(*(c.tags for c in cases))
    for r in range(world - 1):
        assert f"straddle {r}" in tags and f"inverse {r},{r + 1}" in tags, r
    for r in range(world):
        assert f"dead {r} first" in tags and f"dead {r} last" in tags, r
    for t in ("straddle 0,last", "inverse 0,last", "S_0 = inf", f"S_{world - 1} = inf", "T = world"):
        assert t in tags, t
    for c in cases:
        assert len(c.runs) == 5 and c.runs[0][0] == rc.SEED
        assert all(w == rc.model(c.batch, s) for s, w in c.runs)
        if "crafted" in c.tags:
            assert rc.model(c.batch, rc.SEED) and not sh.model_local(c.batch, rc.SEED, world), c.name
            assert all(t.defect for t in c.batch if "groups across" in c.name), c.name     # every tuple invalid
            assert not all(w for _, w in c.runs), c.name
        elif "valid" in c.tags:
            assert rc.model(c.batch, rc.SEED) and sh.model_local(c.batch, rc.SEED, world) and all(w for _, w in c.runs)
            lo, hi = sh.blocks(len(c.batch), world)[0 if "S_0" in " ".join(c.tags) else world - 1]
            assert sum(rc.rlc_scalar(rc.SEED, t) * c.batch[t].sigma for t in range(lo, hi)) % sh.R == 0, c.name
        else:
            assert "dead" in c.tags and not any(w for _, w in c.runs)
    if world == 2:   # the oracle's own pairing agrees with the model on the crafted batches
        for c in cases:
            if "crafted" in c.tags:
                assert rc.oracle_rlc(M.O, M, c.batch, rc.SEED) is True, c.name


def test_state_cases_cover_the_sharded_plan():
    specs = sh.state_specs()
    have = {(s["preset"], s["n"]) for s in specs}
    for p in ("minimal", "mainnet"):
        for n in (1, 64, 65):
            assert (p, n) in have or p == "minimal" and n == 1
        ps = [s for s in specs if s["preset"] == p]
        bound = sh.S.PRESETS[p]["ETH1_DATA_VOTES_BOUND"]
        assert {0, bound} <= {s["votes"] for s in ps} and {0, 32} <= {len(s["extra"]) for s in ps}
    assert ("minimal", 1) in have and ("mainnet", sc.COOP_MAX - 1) in have and ("mainnet", sc.COOP_MAX + 1) in have
    for name, pairs in sc.boundaries().items():
        if name.startswith(("balances", "participation")):
            assert any(p in have for p in pairs), name
    for w in sh.STATE_WORLDS:
        assert any(min(sh.state_list_lengths(s)) < w for s in specs)                   # trailing ranks with empty slices
        assert any(len({sh.c_slice_of(n, w, 0)[2] for n in sh.state_list_lengths(s)}) >= 3 for s in specs)


def test_refusals_per_world():
    for w in sh.WORLDS:
        names = [n for n, _ in sh.refusals(w)]
        assert ("htr sharded: world %d" % w in names) == bool(w & (w - 1))
        assert ("state_root on a sharded handle after the communicator became world 1" in names) == (not w & (w - 1))
        assert len(names) == len(set(names))


# ------------------------------------------------------------------------------------------------ loopback on the host
@pytest.fixture(scope="module")
def loopback_lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("loopback") / "libloopback_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-o", str(out),
                    str(ROOT / "tests" / "host_math" / "loopback_host.cpp")], check=True)
    return str(out)


def _bind(path):
    L = ctypes.CDLL(path)
    L.lb_open.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_ulonglong, ctypes.c_uint]
    L.lb_all_gather.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p]
    L.lb_error.restype = ctypes.c_char_p
    return L


def _payload(gen, rank, n):
    return hashlib.shake_128(b"%d %d" % (gen, rank)).digest(n) if n else b""


def _size(gen, slot):
    if gen % 500 in (0, 1):
        return 0 if gen % 500 == 0 else slot
    return int.from_bytes(hashlib.sha256(b"size %d" % gen).digest()[:4], "little") % (slot + 1)


def _gather_rank(lib, path, rank, world, slot, gens, q):
    L = _bind(lib)
    rc_ = L.lb_open(path.encode(), rank, world, slot, 60_000)
    if rc_:
        q.put((rank, "open", rc_, L.lb_error().decode()))
        return
    recv = ctypes.create_string_buffer(world * slot + 1)
    for g in range(gens):
        n = _size(g, slot)
        rc_ = L.lb_all_gather(_payload(g, rank, n), n, recv)
        if rc_ or recv.raw[: world * n] != b"".join(_payload(g, r, n) for r in range(world)):
            q.put((rank, "gather", g, rc_, L.lb_error().decode()))
            return
    # one byte too many for a slot: refused before this rank arrives
    if L.lb_all_gather(b"x" * (slot + 1), slot + 1, recv) != 0x106:
        q.put((rank, "oversize accepted"))
        return
    q.put((rank, "ok"))


def _run(target, argss, timeout=300):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=(*a, q)) for a in argss]
    try:
        for p in procs:
            p.start()
        out = [q.get(timeout=timeout) for _ in procs]
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
                p.join()
    return sorted(out, key=lambda x: x[0])


@pytest.mark.parametrize("world", range(2, 9))
def test_loopback_gathers_2000_generations(world, loopback_lib, tmp_path):
    slot = 4096
    out = _run(_gather_rank, [(loopback_lib, str(tmp_path / "loop.bin"), r, world, slot, 2000) for r in range(world)])
    assert out == [(r, "ok") for r in range(world)], out


def _late_rank(lib, path, rank, world, timeout_ms, q):
    L = _bind(lib)
    assert L.lb_open(path.encode(), rank, world, 64, timeout_ms) == 0
    if rank == world - 1:          # never arrives
        q.put((rank, "absent"))
        return
    t = time.monotonic()
    rc1 = L.lb_all_gather(b"a" * 8, 8, ctypes.create_string_buffer(64 * world))
    waited = time.monotonic() - t
    err = L.lb_error().decode()
    t = time.monotonic()
    rc2 = L.lb_all_gather(b"a" * 8, 8, ctypes.create_string_buffer(64 * world))   # poisoned: fails at once
    q.put((rank, rc1, waited, err, rc2, time.monotonic() - t))


def test_loopback_times_out_when_a_rank_never_arrives(loopback_lib, tmp_path):
    world, timeout_ms = 3, 1500
    out = _run(_late_rank, [(loopback_lib, str(tmp_path / "loop.bin"), r, world, timeout_ms) for r in range(world)], timeout=120)
    assert out[-1] == (world - 1, "absent")
    for rank, rc1, waited, err, rc2, again in out[:-1]:
        assert rc1 == 0x106 and timeout_ms / 1000 <= waited < timeout_ms / 1000 + 5, (rank, rc1, waited)
        assert "generation 0" in err and f"{world - 1} of {world} ranks arrived" in err, err
        assert rc2 == 0x106 and again < 0.5, (rank, rc2, again)


def _open_only(lib, path, rank, world, slot, q):
    L = _bind(lib)
    rc_ = L.lb_open(path.encode(), rank, world, slot, 5_000)
    q.put((rank, rc_, L.lb_error().decode() if rc_ else ""))


def test_loopback_refuses_a_header_of_another_shape(loopback_lib, tmp_path):
    path = str(tmp_path / "loop.bin")
    assert _run(_open_only, [(loopback_lib, path, 0, 2, 256)]) == [(0, 0, "")]
    out = _run(_open_only, [(loopback_lib, path, 1, 3, 256), (loopback_lib, path, 1, 2, 512), (loopback_lib, path, 1, 2, 128)])
    for _, rc_, err in out:
        assert rc_ == 0x106 and "made for world 2, slot 256 B" in err, err
    assert _run(_open_only, [(loopback_lib, path, 1, 2, 256)]) == [(1, 0, "")]
