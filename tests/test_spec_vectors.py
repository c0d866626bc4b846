"""Runner for the reference's conformance vectors (layout of spec-tests/runners/bls.rs:17-58 and
ssz_static.rs:13-36).  With the `consensus-spec-tests` tarball present (CONSENSUS_SPEC_TESTS=<dir> or
<repo>/consensus-spec-tests) every `bls/*` case runs against the CPU oracle (and, under -m gpu, against the CUDA path),
and every deneb `ssz_static/BeaconState` case against both hash_tree_root implementations.  Offline (this container,
the GPU box) those tests skip; the runner itself is exercised on a synthetic tree in the same layout built from
tests/golden/bls_cases.json, so its YAML handling, malformed-input rules and snappy decoder are covered either way."""
import json
from pathlib import Path

import pytest
import yaml

from tests import spec_vectors as sv

GOLDEN = json.loads((Path(__file__).parent / "golden" / "bls_cases.json").read_text())
REAL = sv.vectors_root()
needs_vectors = pytest.mark.skipif(REAL is None, reason="consensus-spec-tests not present (offline); set CONSENSUS_SPEC_TESTS")


def _hx(b): return "0x" + (b if isinstance(b, str) else b.hex())


def _write_case(base: Path, handler: str, name: str, inp, out):
    d = base / "tests" / "general" / "phase0" / "bls" / handler / "bls" / name
    d.mkdir(parents=True, exist_ok=True)
    (d / "data.yaml").write_text(yaml.safe_dump({"input": inp, "output": out}))


@pytest.fixture(scope="module")
def synthetic_tree(tmp_path_factory):
    """Golden cases re-expressed in the consensus-spec-tests layout (+ the malformed-literal cases of that suite)."""
    base = tmp_path_factory.mktemp("consensus-spec-tests")
    n = 0
    for c in GOLDEN["fast_aggregate_verify"]:
        if len(c["msg"]) != 64:
            continue   # the suite's messages are Bytes32
        inp = {"pubkeys": [_hx(p) for p in c["pks"]], "message": _hx(c["msg"]), "signature": _hx(c["sig"])}
        _write_case(base, "fast_aggregate_verify", f"case_{n}", inp, c["code"] == 0)
        eth_ok = c["code"] == 0 or (not c["pks"] and c["sig"] == "c0" + "00" * 95)
        _write_case(base, "eth_fast_aggregate_verify", f"case_{n}", inp, eth_ok)
        if len(c["pks"]) == 1:
            _write_case(base, "verify", f"case_{n}", {"pubkey": inp["pubkeys"][0], "message": inp["message"], "signature": inp["signature"]},
                        c["code"] == 0)
        n += 1
    for i, c in enumerate(GOLDEN["aggregate_verify"]):
        if any(len(m) != 64 for m in c["msgs"]):
            continue
        _write_case(base, "aggregate_verify", f"case_{i}", {"pubkeys": [_hx(p) for p in c["pks"]], "messages": [_hx(m) for m in c["msgs"]],
                                                            "signature": _hx(c["sig"])}, c["code"] == 0)
    for i, c in enumerate(GOLDEN["aggregate"]):
        _write_case(base, "aggregate", f"case_{i}", [_hx(s) for s in c["sigs"]], _hx(c["out"]) if c["code"] == 0 else None)
    _write_case(base, "aggregate", "case_empty", [], None)
    for i, c in enumerate(GOLDEN["eth_aggregate_public_keys"]):
        _write_case(base, "eth_aggregate_pubkeys", f"case_{i}", [_hx(p) for p in c["pks"]], _hx(c["out"]) if c["code"] == 0 else None)
    # literals that do not even deserialize (the suite has them: "tampered" / wrong-length hex) count as expected failures
    ok = next(c for c in GOLDEN["fast_aggregate_verify"] if c["code"] == 0 and len(c["msg"]) == 64 and c["pks"])
    _write_case(base, "verify", "case_short_sig", {"pubkey": _hx(ok["pks"][0]), "message": _hx(ok["msg"]), "signature": "0x1234"}, False)
    _write_case(base, "fast_aggregate_verify", "case_short_pk", {"pubkeys": ["0x00"], "message": _hx(ok["msg"]), "signature": _hx(ok["sig"])}, False)
    return base


def test_walker_and_runner_on_synthetic_tree(synthetic_tree):
    impl = sv.OracleImpl()
    seen = {}
    for config, fork, handler, case in sv.walk(synthetic_tree, "bls", sv.BLS_HANDLERS):
        assert (config, fork) == ("general", "phase0")
        # the Python oracle is slow on many-key cases: keep the CPU suite to seconds
        d = yaml.safe_load((case / "data.yaml").read_text())
        keys = d["input"].get("pubkeys", []) if isinstance(d["input"], dict) else d["input"]
        if len(keys) > 4:
            continue
        passed, detail = sv.run_bls_case(handler, case, impl)
        assert passed, (handler, case.name, detail)
        seen[handler] = seen.get(handler, 0) + 1
    assert set(seen) == set(sv.BLS_HANDLERS) and sum(seen.values()) >= 40, seen


def test_snappy_raw_decoder():
    data = bytes(range(256)) * 300 + b"tail"
    assert sv.snappy_raw_decompress(sv.snappy_raw_compress_literal(data)) == data
    assert sv.snappy_raw_decompress(sv.snappy_raw_compress_literal(b"")) == b""
    # hand-assembled stream with all three copy forms: "abcd" + copy1(off 4, len 4) + copy2(off 8, len 5) + copy4(off 1, len 3)
    stream = bytes([16, (3 << 2) | 0]) + b"abcd" + bytes([((4 - 4) << 2) | 1, 4]) + bytes([((5 - 1) << 2) | 2, 8, 0]) + \
        bytes([((3 - 1) << 2) | 3, 1, 0, 0, 0])
    assert sv.snappy_raw_decompress(stream) == b"abcdabcd" + b"abcda" + b"aaa"
    with pytest.raises(ValueError):
        sv.snappy_raw_decompress(bytes([4, (3 << 2) | 0]) + b"abcd" + bytes([1, 9]))


def test_ssz_static_layout_roundtrip(tmp_path):
    from ethereum_consensus_b200 import state as S
    from oracle import ssz_oracle as so
    st = S.synth_state(5, "minimal", n_historical_summaries=1, n_historical_roots=1)
    ser = bytes(S.serialize(st))
    root = so.beacon_state_type("minimal").htr(S.to_oracle_value(st))
    case = tmp_path / "tests" / "minimal" / "deneb" / "ssz_static" / "BeaconState" / "ssz_random" / "case_0"
    case.mkdir(parents=True)
    (case / "roots.yaml").write_text(yaml.safe_dump({"root": "0x" + root.hex()}))
    (case / "serialized.ssz_snappy").write_bytes(sv.snappy_raw_compress_literal(ser))
    got = [(c, f, h) for c, f, h, _ in sv.walk(tmp_path, "ssz_static", ("BeaconState",))]
    assert got == [("minimal", "deneb", "BeaconState")]
    assert sv.ssz_static_case(case) == (ser, root)


@pytest.mark.gpu
def test_runner_on_synthetic_tree_gpu(engine, synthetic_tree):
    """The same synthetic tree through the CUDA path (every case, including the many-key ones)."""
    from ethereum_consensus_b200 import crypto
    n = 0
    for _c, _f, handler, case in sv.walk(synthetic_tree, "bls", sv.BLS_HANDLERS):
        passed, detail = sv.run_bls_case(handler, case, crypto)
        assert passed, (handler, case.name, detail)
        n += 1
    assert n >= 60


# ---------------------------------------------------------------- the real vectors (skipped offline)
def _real_bls_cases():
    if REAL is None:
        return []
    return [pytest.param(h, c, id=f"{cfg}/{fork}/{h}/{c.name}") for cfg, fork, h, c in sv.walk(REAL, "bls", sv.BLS_HANDLERS)]


@needs_vectors
@pytest.mark.parametrize("handler,case", _real_bls_cases())
def test_real_bls_vectors_oracle(handler, case):
    passed, detail = sv.run_bls_case(handler, case, sv.OracleImpl())
    assert passed, detail


@needs_vectors
@pytest.mark.gpu
@pytest.mark.parametrize("handler,case", _real_bls_cases())
def test_real_bls_vectors_gpu(engine, handler, case):
    from ethereum_consensus_b200 import crypto
    passed, detail = sv.run_bls_case(handler, case, crypto)
    assert passed, detail


def _real_state_cases():
    if REAL is None:
        return []
    return [pytest.param(cfg, c, id=f"{cfg}/{fork}/{c.parent.name}/{c.name}")
            for cfg, fork, _h, c in sv.walk(REAL, "ssz_static", ("BeaconState",)) if fork == "deneb"]


@needs_vectors
@pytest.mark.parametrize("config,case", _real_state_cases())
def test_real_beacon_state_roots_oracle(oracle_ssz_c, config, case):
    import ctypes
    ser, root = sv.ssz_static_case(case)
    out = ctypes.create_string_buffer(32)
    assert oracle_ssz_c.orc_htr_beacon_state_deneb(ser, len(ser), 0 if config == "mainnet" else 1, 1, out) == 0
    assert out.raw == root


@needs_vectors
@pytest.mark.gpu
@pytest.mark.parametrize("config,case", _real_state_cases())
def test_real_beacon_state_roots_gpu(engine, config, case):
    from ethereum_consensus_b200 import ssz
    ser, root = sv.ssz_static_case(case)
    assert ssz.hash_tree_root_beacon_state(ser, config) == root
