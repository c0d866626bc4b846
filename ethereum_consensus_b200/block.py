"""Deferred signature-set verification for one block (SURVEY.md §8f-1, Appendix C): the collector that turns the
signature checks `process_block` performs one at a time into ONE batch call, then replays the per-tuple verdicts in
execution order so the observable behaviour is the reference's:

* the first failing check aborts with that check's error,
* except deposits, whose invalid signatures are skipped silently
  (ethereum-consensus/src/phase0/block_processing.rs:389-392),
* `is_valid_indexed_attestation`'s host-side checks (non-empty, sorted, unique, index in range) run before any
  signature work and fail first (ethereum-consensus/src/phase0/helpers.rs:94-131).

Deposits are NOT deferred with the rest (ADVICE round 1): `apply_deposit` returns before `add_validator_to_registry` when
the signature check fails (phase0/block_processing.rs:375-401), so the verdict decides a state mutation that later
operations of the same block — and the state root — depend on.  Their signing root is state-independent
(DOMAIN_DEPOSIT, genesis fork version, zero genesis_validators_root, key taken from the message), so
`verify_deposits()` batches the block's deposit checks BEFORE `process_operations` and hands each verdict to
`apply_deposit`; only the checks whose failure aborts the block are deferred to the end-of-block batch.  (A
`SignatureSet` still accepts `tolerant` entries — the parity tests exercise the whole Appendix C set in one batch —
and reports them through `skipped_deposits`.)

Sites, in the order of deneb `process_block` (deneb/block_processing.rs:402-408, spec/mod.rs:219-230):
block proposer, randao, proposer slashings, attester slashings, attestations, deposits, voluntary exits,
bls-to-execution changes, sync aggregate.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import crypto, signing

SITES = ("block_signature", "randao", "proposer_slashing", "attester_slashing", "attestation", "deposit", "voluntary_exit",
         "bls_to_execution_change", "sync_aggregate")


def deposit_signing_root(pubkey: bytes, withdrawal_credentials: bytes, amount: int, genesis_fork_version: bytes = b"\x00" * 4) -> bytes:
    """Signing root of `DepositMessage{pubkey, withdrawal_credentials, amount}` (phase0/operations.rs:74-80) under
    `compute_domain(DEPOSIT, None, None)` = genesis fork version + zero root (phase0/block_processing.rs:387)."""
    from . import ssz
    pk_root = ssz.merkleize(bytes(pubkey) + bytes(16), 2)                       # ByteVector<48>: two chunks
    leaves = pk_root + bytes(withdrawal_credentials) + int(amount).to_bytes(8, "little").ljust(32, b"\x00")
    obj = ssz.merkleize(leaves, 4)                                              # 3 fields padded to 4 leaves
    return signing.compute_signing_root(obj, signing.compute_domain(signing.DomainType.Deposit, genesis_fork_version, bytes(32)))


def verify_deposits(deposits: Sequence[tuple], genesis_fork_version: bytes = b"\x00" * 4) -> List[bool]:
    """The block's deposit signature checks as ONE batch, before `process_operations`: `deposits` = the
    (pubkey, withdrawal_credentials, amount, signature) of every deposit whose key is not in the registry yet.
    verdict[i] is what `verify_signed_data(...).is_ok()` returns inside `apply_deposit`
    (phase0/block_processing.rs:387-392): False means "skip this deposit, no state change", never a block failure."""
    if not deposits:
        return []
    pks = np.frombuffer(b"".join(bytes(crypto.PublicKey(d[0])) for d in deposits), dtype=np.uint8)
    off = np.arange(len(deposits) + 1, dtype=np.uint32)
    msgs = np.frombuffer(b"".join(deposit_signing_root(d[0], d[1], d[2], genesis_fork_version) for d in deposits), dtype=np.uint8)
    sigs = np.frombuffer(b"".join(bytes(crypto.Signature(d[3])) for d in deposits), dtype=np.uint8)
    return [int(c) == 0 for c in crypto.fast_aggregate_verify_batch(pks, off, msgs, sigs)]


class InvalidIndexedAttestation(ValueError):
    """AttestingIndicesEmpty / AttestingIndicesNotSorted / DuplicateIndices / InvalidIndex (phase0/helpers.rs:94-131)."""


@dataclass
class _Entry:
    site: str
    pubkeys: List[bytes]
    signing_root: bytes
    signature: bytes
    tolerant: bool = False
    eth_variant: bool = False  # eth_fast_aggregate_verify semantics (sync aggregate)
    _indices: Optional[tuple] = None        # validator indices of the signers when they come from state.validators
    _indices_np: Optional[np.ndarray] = None  # the same, packed once at collection time (verify() only concatenates)

    @property
    def indices(self) -> Optional[tuple]:
        """Immutable on purpose: the packed copy verify() uses must not go stale behind an in-place edit."""
        return self._indices

    @indices.setter
    def indices(self, value) -> None:
        if value is None:
            self._indices, self._indices_np = None, None
        else:
            self._indices_np = np.fromiter((int(i) for i in value), dtype=np.uint32)
            self._indices_np.setflags(write=False)
            self._indices = tuple(int(i) for i in self._indices_np)


@dataclass
class SignatureSet:
    entries: List[_Entry] = field(default_factory=list)

    def add(self, site: str, pubkeys: Sequence[bytes], signing_root: bytes, signature: bytes, tolerant: bool = False,
            eth_variant: bool = False) -> None:
        if site not in SITES:
            raise ValueError(f"unknown signature site {site!r}")
        if len(signing_root) != 32:
            raise ValueError("signing root must be 32 bytes")
        # coerce through the byte newtypes (crypto/bls.rs:227-239,287-290): a wrong length would misalign the joined
        # buffers of verify() and every later tuple with it
        pks = [bytes(crypto.PublicKey(p)) for p in pubkeys]
        sig = bytes(crypto.Signature(signature))
        self.entries.append(_Entry(site, pks, bytes(signing_root), sig, tolerant, eth_variant))

    def add_indexed_attestation(self, site: str, validator_pubkeys, attesting_indices: Sequence[int], signing_root: bytes,
                                signature: bytes) -> None:
        """`is_valid_indexed_attestation` up to the BLS call (phase0/helpers.rs:94-131)."""
        idx = list(attesting_indices)
        if not idx:
            raise InvalidIndexedAttestation("AttestingIndicesEmpty")
        dup = set()
        for prev, cur in zip(idx, idx[1:]):
            if cur < prev:
                raise InvalidIndexedAttestation("AttestingIndicesNotSorted")
            if cur == prev:
                dup.add(cur)
        if dup:
            raise InvalidIndexedAttestation(f"DuplicateIndices({sorted(dup)})")
        n = len(validator_pubkeys)
        for i in idx:
            if i >= n:
                raise InvalidIndexedAttestation(f"InvalidIndex({i})")
        self.add(site, [validator_pubkeys[i] for i in idx], signing_root, signature)
        self.entries[-1].indices = idx

    def add_by_index(self, site: str, validator_pubkeys, indices: Sequence[int], signing_root: bytes, signature: bytes) -> None:
        """A check whose signer(s) are named by validator index (proposer, randao, slashings, exits): Appendix C rows
        1-3, 7 draw their keys from `state.validators`, so registry mode applies to them."""
        idx = [int(i) for i in indices]
        self.add(site, [validator_pubkeys[i] for i in idx], signing_root, signature)
        self.entries[-1].indices = idx

    def add_sync_aggregate(self, committee_pubkeys: Sequence[bytes], sync_committee_bits: Sequence[bool], signature: bytes,
                           state_slot: int, block_root_at_previous_slot: bytes, fork: "signing.Fork", genesis_validators_root: bytes,
                           slots_per_epoch: int = 32, committee_indices: Optional[Sequence[int]] = None) -> None:
        """`process_sync_aggregate` up to the BLS call (altair/block_processing.rs:216-243): participants = committee keys
        whose bit is set (duplicates stay: a validator may sit in the committee more than once), message = signing root
        of the block root at `max(slot, 1) - 1` under DOMAIN_SYNC_COMMITTEE at THAT slot's epoch (which `get_domain`
        resolves to the previous fork version right after a fork), checked with `eth_fast_aggregate_verify`."""
        if len(sync_committee_bits) != len(committee_pubkeys):
            raise ValueError("sync_committee_bits and the committee differ in length")
        previous_slot = max(int(state_slot), 1) - 1
        domain = signing.get_domain(fork, genesis_validators_root, signing.DomainType.SyncCommittee,
                                    signing.compute_epoch_at_slot(previous_slot, slots_per_epoch))
        root = signing.compute_signing_root(block_root_at_previous_slot, domain)
        sel = [j for j, b in enumerate(sync_committee_bits) if b]
        self.add("sync_aggregate", [committee_pubkeys[j] for j in sel], root, signature, eth_variant=True)
        if committee_indices is not None:
            self.entries[-1].indices = [int(committee_indices[j]) for j in sel]

    # ---- one batch call for the whole block
    def verify(self, registry: Optional["crypto.Registry"] = None) -> np.ndarray:
        """int32 code per entry, exactly what the per-call reference functions would have returned.
        With a `registry` (validated `state.validators` keys resident in HBM) the whole set is ONE `…_batch_mixed` call:
        entries that name their signers by validator index gather from the registry, keys that come with the message
        itself (deposits, bls-to-execution changes) are validated in the same call.  Same codes either way."""
        t = len(self.entries)
        if t == 0:
            return np.zeros(0, dtype=np.int32)
        if registry is None:
            ent = self.entries
            pks = np.frombuffer(b"".join(p for e in ent for p in e.pubkeys) or b"", dtype=np.uint8)
            off = np.cumsum([0] + [len(e.pubkeys) for e in ent]).astype(np.uint32)
            msgs = np.frombuffer(b"".join(e.signing_root for e in ent), dtype=np.uint8)
            sigs = np.frombuffer(b"".join(e.signature for e in ent), dtype=np.uint8)
            codes = crypto.fast_aggregate_verify_batch(pks, off, msgs, sigs).copy()
        else:
            # ONE call for the whole set: signers named by validator index gather from the resident registry; keys carried
            # by the block (deposits, bls-to-execution changes) ride along as extra keys, validated in the same call
            extra, parts = [], []
            for e in self.entries:
                if e.indices is not None:
                    parts.append(e._indices_np)
                else:
                    parts.append(np.arange(registry.n + len(extra), registry.n + len(extra) + len(e.pubkeys), dtype=np.uint32))
                    extra.extend(e.pubkeys)
            off = np.cumsum([0] + [len(q) for q in parts]).astype(np.uint32)
            idx = np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint32)
            msgs = np.frombuffer(b"".join(e.signing_root for e in self.entries), dtype=np.uint8)
            sigs = np.frombuffer(b"".join(e.signature for e in self.entries), dtype=np.uint8)
            xk = np.frombuffer(b"".join(extra), dtype=np.uint8) if extra else None
            codes = registry.verify_batch(idx, off, msgs, sigs, extra_keys=xk).copy()
        for i, e in enumerate(self.entries):  # eth_fast_aggregate_verify: no participants + infinity signature is Ok
            if e.eth_variant and not e.pubkeys and e.signature == crypto.INFINITY_COMPRESSED_SIGNATURE:
                codes[i] = 0
        return codes

    def first_failure(self, codes: Optional[np.ndarray] = None):
        """(index, site, code) of the first check that aborts the block, or None; tolerant entries never abort."""
        if codes is None:
            codes = self.verify()
        for i, (e, c) in enumerate(zip(self.entries, codes)):
            if c != 0 and not e.tolerant:
                return i, e.site, int(c)
        return None

    def skipped_deposits(self, codes: np.ndarray) -> List[int]:
        return [i for i, (e, c) in enumerate(zip(self.entries, codes)) if e.tolerant and c != 0]
