import ctypes
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


def _make_oracles():
    subprocess.run(["make", "-s", "-C", str(ROOT / "oracle")], check=True, capture_output=True)


@pytest.fixture(scope="session")
def oracle_ssz_c():
    """The plain-C SSZ oracle (oracle/c/ssz_oracle.c) loaded through ctypes."""
    _make_oracles()
    lib = ctypes.CDLL(str(ROOT / "oracle" / "liboracle_ssz.so"))
    V, S, U64, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_int
    lib.orc_sha256.argtypes = [V, S, V]
    lib.orc_merkleize.argtypes = [V, S, U64, I, V]
    lib.orc_merkleize.restype = I
    lib.orc_htr_packed.argtypes = [V, S, U64, I, U64, I, V]
    lib.orc_htr_validators.argtypes = [V, S, U64, I, V]
    lib.orc_htr_beacon_state_deneb.argtypes = [V, S, I, I, V]
    lib.orc_htr_beacon_state_deneb.restype = I
    lib.orc_validator_root.argtypes = [V, V]
    lib.orc_mix_in_length.argtypes = [V, U64, V]
    lib.orc_hash_pairs.argtypes = [V, S, I, V]
    return lib


@pytest.fixture(scope="session")
def engine():
    """The CUDA library bound to cuda:0 — fails loudly (no CPU fallback) if it cannot initialise."""
    from ethereum_consensus_b200 import _lib
    return _lib.init(int(os.environ.get("LOCAL_RANK", "0")))


def _host_math_lib(suffix: str, defines):
    src = ROOT / "tests" / "host_math" / "host_math.cpp"
    lib = ROOT / "tests" / "host_math" / f"libhost_math{suffix}.so"
    deps = [src] + list((ROOT / "ethereum_consensus_b200" / "csrc").glob("*.cuh"))
    if not lib.exists() or any(d.stat().st_mtime > lib.stat().st_mtime for d in deps):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", *[f"-D{d}" for d in defines],
                        "-o", str(lib), str(src)], check=True)
    L = ctypes.CDLL(str(lib))
    L.hm_fast_aggregate_verify.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p]
    L.hm_hash_to_g2.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]
    L.hm_hash_to_field.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p]
    return L


@pytest.fixture(scope="session")
def host_math():
    """The product's __host__ __device__ BLS math compiled for the CPU (tests/host_math/host_math.cpp)."""
    return _host_math_lib("", [])


@pytest.fixture(scope="session")
def host_math_sswu_fraction():
    """Same, with the default-off A/B variant of the SSWU map (x kept as a fraction, no Fp2 inversion; h2c.cuh)."""
    return _host_math_lib("_sswu_fraction", ["B200_SSWU_FRACTION"])


@pytest.fixture(scope="session")
def oracle_bls_c():
    """The plain-C BLS oracle (oracle/c/bls_oracle.c) loaded through ctypes."""
    _make_oracles()
    L = ctypes.CDLL(str(ROOT / "oracle" / "liboracle_bls.so"))
    cp, sz, vp = ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p
    L.orc_fast_aggregate_verify.argtypes = [cp, sz, cp, sz, cp]
    L.orc_eth_fast_aggregate_verify.argtypes = [cp, sz, cp, sz, cp]
    L.orc_verify_signature.argtypes = [cp, cp, sz, cp]
    L.orc_aggregate_verify.argtypes = [cp, sz, vp, vp, sz, cp]
    L.orc_aggregate.argtypes = [cp, sz, cp]
    L.orc_eth_aggregate_public_keys.argtypes = [cp, sz, cp]
    L.orc_key_validate.argtypes = [cp]
    L.orc_g1_group_checks_agree.argtypes = [cp]
    L.orc_g2_group_checks_agree.argtypes = [cp]
    L.orc_hash_to_g2.argtypes = [cp, sz, cp]
    L.orc_sk_to_pk.argtypes = [cp, cp]
    L.orc_sign.argtypes = [cp, cp, sz, cp]
    L.orc_fast_aggregate_verify_batch.argtypes = [vp, vp, vp, vp, sz, vp, ctypes.c_int]
    L.orc_sign_batch.argtypes = [vp, vp, sz, vp, ctypes.c_int]
    L.orc_pk_sequence.argtypes = [cp, cp, sz, vp]
    L.orc_fp_mul_count.restype = ctypes.c_uint64
    return L
