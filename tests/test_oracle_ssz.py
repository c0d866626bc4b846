"""CPU: pins the SSZ oracles (oracle/ssz_oracle.py, oracle/c/ssz_oracle.c) to the reference's own KAT and to each other."""
import ctypes
import hashlib
import json
import os
from pathlib import Path

import numpy as np
import pytest

from oracle import ssz_oracle as so
from ethereum_consensus_b200 import state as S

GOLDEN = json.loads((Path(__file__).parent / "golden" / "ssz_roots.json").read_text())

# KAT B-3: ethereum-consensus/src/deneb/blob_sidecar.rs:70-132 (live sepolia blob sidecar)
B3_COMMITMENT = bytes.fromhex("8da04bbe26b2bbc6b042f4db18a36f1b4714123706065ed3946a3c3aeb681f98d3e67a3483b088612cb9b0c5322723a0")
B3_BODY_ROOT = bytes.fromhex("940ebac04b768dab430d21b4b2d7ecd5d3f87e0486293a5612c16b9e8d4c078a")
B3_BRANCH = [bytes.fromhex(x) for x in """
0000000000000000000000000000000000000000000000000000000000000000
f5a5fd42d16a20302798ef6ed309979b43003d2320d9f0e8ea9831a92759fb4b
db56114e00fdd4c1f85c892bf35ac9a89289aaecb1ebd0a96cde606a748b5d71
c78009fdf07fc56a11f122370658a353aaa542ed63e44c4bc15ff4cd105ab33c
536d98837f2dd165a55d5eeae91485954472d56f246df256bf3cae19352a123c
9efde052aa15429fae05bad4d0b1d7c64da64d03d7a1854a588c2cb8430c0d30
d88ddfeed400a8755596b21942c1497e114c302e6118290f91e6772976041fa1
87eb0ddba57e35f6d286673802a4af5975e22506c7cf4c64bb6be5ee11527f2c
26846476fd5fc54a5d43385167c95144f2643f533cc85bb9d16b782f8d7db193
506d86582d252405b840018792cad2bf1259f1ef5aa5f887e13cb2f0094f51e1
ffff0ad7e659772f9534c195c815efc4014ef1e1daed4404c06385d11192e92b
6cf04127db05441cd833107a52be852868890e4317e6a02ab47683aa75964220
0100000000000000000000000000000000000000000000000000000000000000
792930bbd5baac43bcc798ee49aa8185ef76bb3b44ba62b91d86ae569e4bb535
818d8d71c18b108e28500c2bd5bb946069c5877a512a699cdd8a40b90aaf44ca
db56114e00fdd4c1f85c892bf35ac9a89289aaecb1ebd0a96cde606a748b5d71
d130f52a1da1e28d4a38d8f4b89a0f0c3f047e7d9935408aef8efc3bc0930c13""".split()]
# generalized index of blob_kzg_commitments[0] is 221184 (deneb/beacon_block.rs:139-154); subtree index = gindex - 2**17
B3_DEPTH, B3_INDEX = 17, 221184 - (1 << 17)


def test_kat_b3_blob_sidecar_inclusion_proof():
    leaf = so.Bytes48.htr(B3_COMMITMENT)
    assert so.is_valid_merkle_branch(leaf, B3_BRANCH, B3_DEPTH, B3_INDEX, B3_BODY_ROOT)
    assert not so.is_valid_merkle_branch(leaf, B3_BRANCH, B3_DEPTH, B3_INDEX ^ 1, B3_BODY_ROOT)
    # the first 12 siblings of the KAT are the zero-subtree hashes z0..z11 (blob_sidecar.rs:88-99)
    assert B3_BRANCH[:12] == so.ZERO_HASHES[:12]


def test_zero_hashes_and_sha_vectors():
    assert so.ZERO_HASHES[1].hex().startswith("f5a5fd42") and so.ZERO_HASHES[2].hex().startswith("db56114e")
    assert so.sha256(b"abc").hex() == "ba7816bf8f01cfea414140de5dae2223b00361a396177a9cb410ff61f20015ad"


def test_c_oracle_sha256_matches_hashlib(oracle_ssz_c):
    out = ctypes.create_string_buffer(32)
    rng = np.random.default_rng(1)
    for force in (0, 1):
        oracle_ssz_c.orc_force_portable(force)
        for n in [0, 1, 55, 56, 63, 64, 65, 119, 120, 128, 1000]:
            d = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            oracle_ssz_c.orc_sha256(d, n, out)
            assert out.raw == hashlib.sha256(d).digest()
    oracle_ssz_c.orc_force_portable(0)


@pytest.mark.parametrize("n,limit", [(0, 0), (0, 16), (1, 0), (1, 1), (2, 0), (3, 0), (5, 8), (5, 1 << 40), (1000, 0), (1000, 1 << 24), (5000, 0)])
def test_c_oracle_merkleize_matches_python(oracle_ssz_c, n, limit):
    out = ctypes.create_string_buffer(32)
    d = np.random.default_rng(n).integers(0, 256, 32 * n, dtype=np.uint8).tobytes()
    assert oracle_ssz_c.orc_merkleize(d, n, limit, 4, out) == 0
    exp = so.merkleize_chunks([d[32 * i:32 * i + 32] for i in range(n)], limit or None)
    assert out.raw == exp
    assert exp == (so.merkleize_bytes(d, limit or None) if n else exp)


def test_merkleize_over_limit_rejected(oracle_ssz_c):
    out = ctypes.create_string_buffer(32)
    assert oracle_ssz_c.orc_merkleize(bytes(96), 3, 2, 1, out) != 0
    with pytest.raises(ValueError):
        so.merkleize_chunks([bytes(32)] * 3, 2)


@pytest.mark.parametrize("key", sorted(k for k in GOLDEN if k.endswith("hs3:hr2")))
def test_state_roots_python_serializer_c_oracle_agree(oracle_ssz_c, key):
    preset, n = key.split(":")[0], int(key.split(":")[1])
    st = S.synth_state(n, preset, n_historical_summaries=3, n_historical_roots=2)
    ssz = S.serialize(st)
    T = so.beacon_state_type(preset)
    val = S.to_oracle_value(st)
    assert T.serialize(val) == ssz.tobytes()          # product serializer == oracle serializer
    assert T.htr(val).hex() == GOLDEN[key]            # oracle == committed golden
    out = ctypes.create_string_buffer(32)
    for nt in (1, 4):
        assert oracle_ssz_c.orc_htr_beacon_state_deneb(ssz.ctypes.data, len(ssz), 0 if preset == "mainnet" else 1, nt, out) == 0
        assert out.raw.hex() == GOLDEN[key]


def test_c_oracle_rejects_malformed_state(oracle_ssz_c):
    st = S.synth_state(5, "minimal")
    ssz = S.serialize(st)
    out = ctypes.create_string_buffer(32)
    assert oracle_ssz_c.orc_htr_beacon_state_deneb(ssz.ctypes.data, len(ssz) - 1, 1, 1, out) != 0
    assert oracle_ssz_c.orc_htr_beacon_state_deneb(ssz.ctypes.data, 100, 1, 1, out) != 0


@pytest.mark.skipif(os.environ.get("B200_SLOW_TESTS", "1") == "0", reason="slow")
def test_c_oracle_full_mainnet_state_golden(oracle_ssz_c):
    """2**20 validators (BASELINE.json config 3): C oracle == golden produced by the hashlib oracle."""
    st = S.synth_state(1 << 20, "mainnet")
    ssz = S.serialize(st)
    out = ctypes.create_string_buffer(32)
    assert oracle_ssz_c.orc_htr_beacon_state_deneb(ssz.ctypes.data, len(ssz), 0, os.cpu_count() or 1, out) == 0
    assert out.raw.hex() == GOLDEN["mainnet:1048576:default"]


def test_signing_root_shapes():
    # compute_signing_root / compute_domain restated (signing.rs:14-22; phase0/helpers.rs:506-529)
    d = so.compute_domain(bytes.fromhex("01000000"), bytes.fromhex("04000000"), bytes(32))
    assert len(d) == 32 and d[:4] == bytes.fromhex("01000000")
    r = so.compute_signing_root(bytes(32), d)
    assert r == so.hash_pair(bytes(32), d)


@pytest.mark.parametrize("n,preset", [(0, "minimal"), (5, "minimal"), (70, "mainnet"), (1000, "mainnet")])
def test_state_layout_matches_serialization(n, preset):
    """`state.layout` gives the byte coordinates `b200_state_update_bytes` takes: every part must sit where
    `serialize` put it, the offset words must point at the variable-size fields, and the parts must tile the buffer."""
    import numpy as np
    from ethereum_consensus_b200 import state as S
    st = S.synth_state(n, preset, n_historical_summaries=3, n_historical_roots=2)
    b = S.serialize(st)
    lay = S.layout(st)
    spans = sorted(lay.values())
    assert spans[0][0] == 0 and all(a[0] + a[1] == c[0] for a, c in zip(spans, spans[1:])) and spans[-1][0] + spans[-1][1] == len(b)
    for name in ("balances", "inactivity_scores", "previous_epoch_participation", "current_epoch_participation", "validators",
                 "block_roots", "randao_mixes", "slashings", "historical_summaries"):
        o, ln = lay[name]
        assert bytes(b[o:o + ln]) == getattr(st, name).tobytes()
        if "offset:" + name in lay:
            oo, _ = lay["offset:" + name]
            assert int.from_bytes(bytes(b[oo:oo + 4]), "little") == o
    for name in ("slot", "fork", "latest_block_header", "eth1_data", "finalized_checkpoint", "next_withdrawal_index"):
        o, ln = lay[name]
        assert bytes(b[o:o + ln]) == st.fixed[name]
    assert lay["validators"][1] == 121 * n and lay["balances"][1] == 8 * n
