"""SSZ merkleization oracle (TEST INFRASTRUCTURE — never imported by the product path).

CPU restatement, with `hashlib.sha256`, of the SSZ `hash_tree_root` / `merkleize` semantics that the
reference obtains from the un-vendored crate `ssz_rs @ 84ef2b71` (`Cargo.toml:20`,
re-exported at `ethereum-consensus/src/ssz/mod.rs:4-7`).  The algorithm restated is the
consensus-specs `ssz/simple-serialize.md` merkleization; the container shapes follow the reference:

* `deneb::BeaconState`           ethereum-consensus/src/deneb/beacon_state.rs:13-64
* `Validator`                    ethereum-consensus/src/phase0/validator.rs:10-26
* `Fork`, `Checkpoint`, `Eth1Data`, `BeaconBlockHeader`
                                 ethereum-consensus/src/phase0/{beacon_state.rs:15-22,operations.rs:13-17,66-71,beacon_block.rs:83-91}
* `SyncCommittee`                ethereum-consensus/src/altair/sync.rs:17-22
* `ExecutionPayloadHeader`       ethereum-consensus/src/deneb/execution_payload.rs:47-76
* `HistoricalSummary`            ethereum-consensus/src/phase0/beacon_state.rs:42-45
* `SigningData`, `compute_signing_root`  ethereum-consensus/src/signing.rs:9-22
* `is_valid_merkle_branch` use   ethereum-consensus/src/deneb/blob_sidecar.rs:47-64

Pinned by the reference's own KAT B-3 (blob-sidecar inclusion proof, `deneb/blob_sidecar.rs:70-132`) in
`tests/test_oracle_ssz.py`.  Full-state roots are not pinned by any in-tree reference test (the
consensus-spec-tests vectors are absent offline); they follow from SHA-256 + the SSZ spec, which leaves no
implementation freedom.
"""
from __future__ import annotations

import hashlib
from typing import Any, Dict, List as PyList, Sequence, Tuple

BYTES_PER_CHUNK = 32
ZERO_CHUNK = b"\x00" * 32


def sha256(data: bytes) -> bytes:
    """`crypto::hash` — ethereum-consensus/src/crypto/bls.rs:12-20."""
    return hashlib.sha256(data).digest()


def hash_pair(a: bytes, b: bytes) -> bytes:
    return hashlib.sha256(a + b).digest()


# zero-subtree hashes: ZERO_HASHES[d] = root of a depth-d tree of zero chunks
ZERO_HASHES: PyList[bytes] = [ZERO_CHUNK]
for _ in range(64):
    ZERO_HASHES.append(hash_pair(ZERO_HASHES[-1], ZERO_HASHES[-1]))


def _depth_for(n: int) -> int:
    """Smallest d with 2**d >= n (n >= 1)."""
    return 0 if n <= 1 else (n - 1).bit_length()


def merkleize_chunks(chunks: Sequence[bytes], limit: int | None = None) -> bytes:
    """`merkleize(chunks, limit)` of the SSZ spec: pad *virtually* with zero-subtree hashes up to the
    next power of two of `limit` (or of len(chunks) if limit is None)."""
    n = len(chunks)
    if limit is None:
        limit = n
    if n > limit:
        raise ValueError("chunk count exceeds limit")
    depth = _depth_for(max(limit, 1))
    if n == 0:
        return ZERO_HASHES[depth]
    level = list(chunks)
    for d in range(depth):
        if len(level) & 1:
            level.append(ZERO_HASHES[d])
        level = [hash_pair(level[i], level[i + 1]) for i in range(0, len(level), 2)]
    return level[0]


def merkleize_bytes(data: bytes, limit_chunks: int | None = None) -> bytes:
    """Fast path for already-packed chunk data (basic lists/vectors, byte vectors)."""
    if len(data) % 32:
        data = data + b"\x00" * (32 - len(data) % 32)
    n = len(data) // 32
    if limit_chunks is None:
        limit_chunks = n
    depth = _depth_for(max(limit_chunks, 1))
    if n == 0:
        return ZERO_HASHES[depth]
    if n > limit_chunks:
        raise ValueError("chunk count exceeds limit")
    h = hashlib.sha256
    for d in range(depth):
        if (len(data) // 32) & 1:
            data = data + ZERO_HASHES[d]
        data = b"".join(h(data[i:i + 64]).digest() for i in range(0, len(data), 64))
    return data


def mix_in_length(root: bytes, length: int) -> bytes:
    return hash_pair(root, length.to_bytes(32, "little"))


def is_valid_merkle_branch(leaf: bytes, branch: Sequence[bytes], depth: int, index: int, root: bytes) -> bool:
    """ssz_rs `is_valid_merkle_branch` as used at ethereum-consensus/src/deneb/blob_sidecar.rs:58-63
    and ethereum-consensus/src/phase0/block_processing.rs:428-437."""
    value = leaf
    for i in range(depth):
        if (index >> i) & 1:
            value = hash_pair(branch[i], value)
        else:
            value = hash_pair(value, branch[i])
    return value == root


# --------------------------------------------------------------------------------------------------
# A small SSZ type system (serialize + hash_tree_root) sufficient for the deneb BeaconState
# --------------------------------------------------------------------------------------------------
class SszType:
    def is_fixed(self) -> bool: raise NotImplementedError
    def fixed_size(self) -> int: raise NotImplementedError
    def serialize(self, v: Any) -> bytes: raise NotImplementedError
    def htr(self, v: Any) -> bytes: raise NotImplementedError
    def default(self) -> Any: raise NotImplementedError


class UInt(SszType):
    def __init__(self, bits: int): self.n = bits // 8
    def is_fixed(self): return True
    def fixed_size(self): return self.n
    def serialize(self, v): return int(v).to_bytes(self.n, "little")
    def htr(self, v): return int(v).to_bytes(self.n, "little").ljust(32, b"\x00")
    def default(self): return 0


class Boolean(UInt):
    def __init__(self): self.n = 1
    def serialize(self, v): return b"\x01" if v else b"\x00"
    def htr(self, v): return self.serialize(v).ljust(32, b"\x00")
    def default(self): return False


class ByteVector(SszType):
    """`ByteVector<N>` — ethereum-consensus/src/ssz/byte_vector.rs:11-22."""
    def __init__(self, n: int): self.n = n
    def is_fixed(self): return True
    def fixed_size(self): return self.n
    def serialize(self, v):
        assert len(v) == self.n
        return bytes(v)
    def htr(self, v): return merkleize_bytes(bytes(v), (self.n + 31) // 32)
    def default(self): return b"\x00" * self.n


class ByteList(SszType):
    """`ByteList<N>` — ethereum-consensus/src/ssz/byte_list.rs:11-12."""
    def __init__(self, limit: int): self.limit = limit
    def is_fixed(self): return False
    def serialize(self, v): return bytes(v)
    def htr(self, v):
        assert len(v) <= self.limit
        return mix_in_length(merkleize_bytes(bytes(v), (self.limit + 31) // 32), len(v))
    def default(self): return b""


class Bitvector(SszType):
    def __init__(self, n: int): self.n = n
    def is_fixed(self): return True
    def fixed_size(self): return (self.n + 7) // 8
    def serialize(self, v):
        out = bytearray((self.n + 7) // 8)
        for i, b in enumerate(v):
            if b: out[i // 8] |= 1 << (i % 8)
        return bytes(out)
    def htr(self, v): return merkleize_bytes(self.serialize(v), (self.n + 255) // 256)
    def default(self): return [False] * self.n


class Bitlist(SszType):
    def __init__(self, limit: int): self.limit = limit
    def is_fixed(self): return False
    def serialize(self, v):
        n = len(v)
        out = bytearray(n // 8 + 1)
        for i, b in enumerate(v):
            if b: out[i // 8] |= 1 << (i % 8)
        out[n // 8] |= 1 << (n % 8)
        return bytes(out)
    def htr(self, v):
        n = len(v)
        out = bytearray((n + 7) // 8)
        for i, b in enumerate(v):
            if b: out[i // 8] |= 1 << (i % 8)
        return mix_in_length(merkleize_bytes(bytes(out), (self.limit + 255) // 256), n)
    def default(self): return []


def _is_basic(t: SszType) -> bool:
    return isinstance(t, UInt)


def _serialize_seq(elem: SszType, vals: Sequence[Any]) -> bytes:
    if elem.is_fixed():
        return b"".join(elem.serialize(x) for x in vals)
    parts = [elem.serialize(x) for x in vals]
    off = 4 * len(parts)
    head = b""
    for p in parts:
        head += off.to_bytes(4, "little")
        off += len(p)
    return head + b"".join(parts)


class Vector(SszType):
    def __init__(self, elem: SszType, n: int): self.elem, self.n = elem, n
    def is_fixed(self): return self.elem.is_fixed()
    def fixed_size(self): return self.elem.fixed_size() * self.n
    def serialize(self, v):
        assert len(v) == self.n
        return _serialize_seq(self.elem, v)
    def htr(self, v):
        assert len(v) == self.n
        if _is_basic(self.elem):
            return merkleize_bytes(_serialize_seq(self.elem, v), (self.n * self.elem.fixed_size() + 31) // 32)
        return merkleize_chunks([self.elem.htr(x) for x in v], self.n)
    def default(self): return [self.elem.default() for _ in range(self.n)]


class List(SszType):
    def __init__(self, elem: SszType, limit: int): self.elem, self.limit = elem, limit
    def is_fixed(self): return False
    def serialize(self, v): return _serialize_seq(self.elem, v)
    def htr(self, v):
        assert len(v) <= self.limit
        if _is_basic(self.elem):
            root = merkleize_bytes(_serialize_seq(self.elem, v), (self.limit * self.elem.fixed_size() + 31) // 32)
        else:
            root = merkleize_chunks([self.elem.htr(x) for x in v], self.limit)
        return mix_in_length(root, len(v))
    def default(self): return []


class Container(SszType):
    def __init__(self, name: str, fields: Sequence[Tuple[str, SszType]]):
        self.name, self.fields = name, list(fields)
    def is_fixed(self): return all(t.is_fixed() for _, t in self.fields)
    def fixed_size(self): return sum(t.fixed_size() for _, t in self.fields)
    def serialize(self, v: Dict[str, Any]):
        fixed_parts, var_parts = [], []
        for name, t in self.fields:
            if t.is_fixed():
                fixed_parts.append(t.serialize(v[name])); var_parts.append(b"")
            else:
                fixed_parts.append(None); var_parts.append(t.serialize(v[name]))
        fixed_len = sum(4 if p is None else len(p) for p in fixed_parts)
        out, off = b"", fixed_len
        for p, vp in zip(fixed_parts, var_parts):
            if p is None:
                out += off.to_bytes(4, "little"); off += len(vp)
            else:
                out += p
        return out + b"".join(var_parts)
    def htr(self, v: Dict[str, Any]):
        return merkleize_chunks([t.htr(v[name]) for name, t in self.fields])
    def default(self): return {name: t.default() for name, t in self.fields}


# --------------------------------------------------------------------------------------------------
# Containers on the hot path
# --------------------------------------------------------------------------------------------------
u64, u8, u256 = UInt(64), UInt(8), UInt(256)
Bytes4, Bytes20, Bytes32, Bytes48, Bytes96 = ByteVector(4), ByteVector(20), ByteVector(32), ByteVector(48), ByteVector(96)

Fork = Container("Fork", [("previous_version", Bytes4), ("current_version", Bytes4), ("epoch", u64)])
ForkData = Container("ForkData", [("current_version", Bytes4), ("genesis_validators_root", Bytes32)])
Checkpoint = Container("Checkpoint", [("epoch", u64), ("root", Bytes32)])
Eth1Data = Container("Eth1Data", [("deposit_root", Bytes32), ("deposit_count", u64), ("block_hash", Bytes32)])
BeaconBlockHeader = Container("BeaconBlockHeader", [
    ("slot", u64), ("proposer_index", u64), ("parent_root", Bytes32), ("state_root", Bytes32), ("body_root", Bytes32)])
Validator = Container("Validator", [
    ("public_key", Bytes48), ("withdrawal_credentials", Bytes32), ("effective_balance", u64), ("slashed", Boolean()),
    ("activation_eligibility_epoch", u64), ("activation_epoch", u64), ("exit_epoch", u64), ("withdrawable_epoch", u64)])
HistoricalSummary = Container("HistoricalSummary", [("block_summary_root", Bytes32), ("state_summary_root", Bytes32)])
SigningData = Container("SigningData", [("object_root", Bytes32), ("domain", Bytes32)])
AttestationData = Container("AttestationData", [
    ("slot", u64), ("index", u64), ("beacon_block_root", Bytes32), ("source", Checkpoint), ("target", Checkpoint)])


def sync_committee_type(size: int) -> Container:
    return Container("SyncCommittee", [("public_keys", Vector(Bytes48, size)), ("aggregate_public_key", Bytes48)])


def execution_payload_header_type(bytes_per_logs_bloom: int = 256, max_extra_data_bytes: int = 32) -> Container:
    return Container("ExecutionPayloadHeader", [
        ("parent_hash", Bytes32), ("fee_recipient", Bytes20), ("state_root", Bytes32), ("receipts_root", Bytes32),
        ("logs_bloom", ByteVector(bytes_per_logs_bloom)), ("prev_randao", Bytes32), ("block_number", u64),
        ("gas_limit", u64), ("gas_used", u64), ("timestamp", u64), ("extra_data", ByteList(max_extra_data_bytes)),
        ("base_fee_per_gas", u256), ("block_hash", Bytes32), ("transactions_root", Bytes32),
        ("withdrawals_root", Bytes32), ("blob_gas_used", u64), ("excess_blob_gas", u64)])


PRESETS = {
    # ethereum-consensus/src/phase0/presets/mainnet.rs:5-36,82-83; altair/presets/mainnet.rs:19;
    # bellatrix/presets/mainnet.rs:23-24
    "mainnet": dict(SLOTS_PER_HISTORICAL_ROOT=8192, HISTORICAL_ROOTS_LIMIT=1 << 24, ETH1_DATA_VOTES_BOUND=2048,
                    VALIDATOR_REGISTRY_LIMIT=1 << 40, EPOCHS_PER_HISTORICAL_VECTOR=65536,
                    EPOCHS_PER_SLASHINGS_VECTOR=8192, SYNC_COMMITTEE_SIZE=512, BYTES_PER_LOGS_BLOOM=256,
                    MAX_EXTRA_DATA_BYTES=32),
    # ethereum-consensus/src/phase0/presets/minimal.rs:20-25; altair/presets/minimal.rs:19
    "minimal": dict(SLOTS_PER_HISTORICAL_ROOT=64, HISTORICAL_ROOTS_LIMIT=1 << 24, ETH1_DATA_VOTES_BOUND=32,
                    VALIDATOR_REGISTRY_LIMIT=1 << 40, EPOCHS_PER_HISTORICAL_VECTOR=64,
                    EPOCHS_PER_SLASHINGS_VECTOR=64, SYNC_COMMITTEE_SIZE=32, BYTES_PER_LOGS_BLOOM=256,
                    MAX_EXTRA_DATA_BYTES=32),
}


def beacon_state_type(preset: str = "mainnet") -> Container:
    """deneb `BeaconState` — field order = ethereum-consensus/src/deneb/beacon_state.rs:26-63."""
    p = PRESETS[preset]
    return Container("BeaconState", [
        ("genesis_time", u64),
        ("genesis_validators_root", Bytes32),
        ("slot", u64),
        ("fork", Fork),
        ("latest_block_header", BeaconBlockHeader),
        ("block_roots", Vector(Bytes32, p["SLOTS_PER_HISTORICAL_ROOT"])),
        ("state_roots", Vector(Bytes32, p["SLOTS_PER_HISTORICAL_ROOT"])),
        ("historical_roots", List(Bytes32, p["HISTORICAL_ROOTS_LIMIT"])),
        ("eth1_data", Eth1Data),
        ("eth1_data_votes", List(Eth1Data, p["ETH1_DATA_VOTES_BOUND"])),
        ("eth1_deposit_index", u64),
        ("validators", List(Validator, p["VALIDATOR_REGISTRY_LIMIT"])),
        ("balances", List(u64, p["VALIDATOR_REGISTRY_LIMIT"])),
        ("randao_mixes", Vector(Bytes32, p["EPOCHS_PER_HISTORICAL_VECTOR"])),
        ("slashings", Vector(u64, p["EPOCHS_PER_SLASHINGS_VECTOR"])),
        ("previous_epoch_participation", List(u8, p["VALIDATOR_REGISTRY_LIMIT"])),
        ("current_epoch_participation", List(u8, p["VALIDATOR_REGISTRY_LIMIT"])),
        ("justification_bits", Bitvector(4)),
        ("previous_justified_checkpoint", Checkpoint),
        ("current_justified_checkpoint", Checkpoint),
        ("finalized_checkpoint", Checkpoint),
        ("inactivity_scores", List(u64, p["VALIDATOR_REGISTRY_LIMIT"])),
        ("current_sync_committee", sync_committee_type(p["SYNC_COMMITTEE_SIZE"])),
        ("next_sync_committee", sync_committee_type(p["SYNC_COMMITTEE_SIZE"])),
        ("latest_execution_payload_header",
         execution_payload_header_type(p["BYTES_PER_LOGS_BLOOM"], p["MAX_EXTRA_DATA_BYTES"])),
        ("next_withdrawal_index", u64),
        ("next_withdrawal_validator_index", u64),
        ("historical_summaries", List(HistoricalSummary, p["HISTORICAL_ROOTS_LIMIT"])),
    ])


def compute_signing_root(object_root: bytes, domain: bytes) -> bytes:
    """`compute_signing_root` — ethereum-consensus/src/signing.rs:14-22."""
    return SigningData.htr({"object_root": object_root, "domain": domain})


def compute_domain(domain_type: bytes, fork_version: bytes, genesis_validators_root: bytes) -> bytes:
    """`compute_domain` — ethereum-consensus/src/phase0/helpers.rs:506-529."""
    fork_data_root = ForkData.htr({"current_version": fork_version, "genesis_validators_root": genesis_validators_root})
    return domain_type + fork_data_root[:28]
