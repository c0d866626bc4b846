"""Host-side mirror of `ethereum_consensus::crypto` (BLS), backed by the CUDA library — no CPU fallback.

Same names, argument meaning and error behaviour as ethereum-consensus/src/crypto/bls.rs:
`verify_signature` (:64-77), `aggregate` (:79-93), `aggregate_verify` (:95-112), `fast_aggregate_verify` (:114-132),
`eth_aggregate_public_keys` (:135-148), `eth_fast_aggregate_verify` (:150-160), `hash` (:12-20), the byte newtypes
`PublicKey` (:227-239) / `Signature` (:287-290) with their length checks (:257-266, :318-327) and
`Signature.is_infinity` (:343-347); errors mirror `Error` / `BLSTError` (:27-62).
`SecretKey` (key generation, signing) is not on the verification hot path and is not re-implemented here.

Rust `Result<(), Error>` becomes: return None on Ok, raise on Err.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from . import _lib
from .ssz import hash  # noqa: F401,A004  (crypto::hash is the same one-shot SHA-256)

BLS_DST = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_"
BLS_PUBLIC_KEY_BYTES_LEN = 48
BLS_SIGNATURE_BYTES_LEN = 96
INFINITY_COMPRESSED_SIGNATURE = bytes([0xC0]) + bytes(95)

_BLST_TEXT = {1: "bad encoding", 2: "point not on curve", 3: "point not in group", 4: "aggregation type mismatch",
              5: "verification failed", 6: "public key is infinity", 7: "bad scalar input"}

_lib.register_protos({
    "b200_verify_signature": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_fast_aggregate_verify": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_eth_fast_aggregate_verify": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_aggregate_verify": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_aggregate": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_eth_aggregate_public_keys": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_fast_aggregate_verify_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_registry_load": (C.c_int32, [C.c_void_p, C.c_size_t]),
    "b200_registry_append": (C.c_int32, [C.c_void_p, C.c_size_t]),
    "b200_registry_load_state": (C.c_int32, [C.c_void_p]),
    "b200_registry_sync_state": (C.c_int32, [C.c_void_p]),
    "b200_registry_key_codes": (C.c_int32, [C.c_void_p, C.c_size_t]),
    "b200_fast_aggregate_verify_batch_indexed": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_aggregate_verify_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_aggregate_verify_batch_indexed": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                        C.c_void_p]),
    "b200_fast_aggregate_verify_batch_all": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int32)]),
    "b200_fast_aggregate_verify_batch_indexed_all": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int32)]),
    "b200_fast_aggregate_verify_batch_all_sharded": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int32)]),
    "b200_last_dominant_kernel_ms": (C.c_float, []),
    "b200_fp_selftest": (C.c_int32, [C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]),
    "b200_fp_eval": (C.c_int32, [C.c_int32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_curve_eval": (C.c_int32, [C.c_int32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_pairing_eval": (C.c_int32, [C.c_int32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_measure_int_peak": (C.c_int32, [C.c_int32, C.POINTER(C.c_double)]),
})


class Error(Exception):
    """`crypto::Error` (crypto/bls.rs:27-42)."""


class EmptyAggregate(Error):
    def __init__(self):
        super().__init__("inputs required for aggregation but none were provided")


class SimpleSerializeError(Error):
    """Wrong byte length for a `ByteVector<N>` newtype (crypto/bls.rs:257-266, 318-327)."""


class BLSTError(Error):
    """`Error::BLST(BLSTError)` — text from crypto/bls.rs:48-62."""

    def __init__(self, code: int):
        self.code = code
        super().__init__(f"blst error: {_BLST_TEXT.get(code, code)}")


class InvalidSignature(Error):
    def __init__(self):
        super().__init__("invalid signature")


class PublicKey(bytes):
    """`PublicKey(ByteVector<48>)`: any 48 bytes are accepted here; curve checks happen at use (bls.rs:279-285)."""

    def __new__(cls, data=bytes(48)):
        b = bytes(data)
        if len(b) != BLS_PUBLIC_KEY_BYTES_LEN:
            raise SimpleSerializeError(f"expected {BLS_PUBLIC_KEY_BYTES_LEN} bytes, got {len(b)}")
        return super().__new__(cls, b)


class Signature(bytes):
    """`Signature(ByteVector<96>)`."""

    def __new__(cls, data=bytes(96)):
        b = bytes(data)
        if len(b) != BLS_SIGNATURE_BYTES_LEN:
            raise SimpleSerializeError(f"expected {BLS_SIGNATURE_BYTES_LEN} bytes, got {len(b)}")
        return super().__new__(cls, b)

    def is_infinity(self) -> bool:
        return bytes(self) == INFINITY_COMPRESSED_SIGNATURE


def _result(code: int, where: str) -> None:
    _lib.check(code, where)
    if code == _lib.SUCCESS:
        return None
    if code == _lib.VERIFY_FAIL:
        raise InvalidSignature()
    if code == _lib.EMPTY_AGGREGATE:
        raise EmptyAggregate()
    raise BLSTError(code)


def _ptr_array(items: Sequence[bytes]):
    keep = [bytes(x) for x in items]
    arr = (C.c_char_p * max(len(keep), 1))(*keep) if keep else (C.c_char_p * 1)()
    return arr, keep


def verify_signature(public_key: PublicKey, msg: bytes, signature: Signature) -> None:
    pk, sig, m = PublicKey(public_key), Signature(signature), bytes(msg)
    _result(_lib.lib().b200_verify_signature(_lib.ptr(pk), _lib.ptr(m), len(m), _lib.ptr(sig)), "verify_signature")


def fast_aggregate_verify(public_keys: Sequence[PublicKey], msg: bytes, signature: Signature) -> None:
    pks = [PublicKey(p) for p in public_keys]
    sig, m = Signature(signature), bytes(msg)
    arr, _keep = _ptr_array(pks)
    _result(_lib.lib().b200_fast_aggregate_verify(C.cast(arr, C.c_void_p), len(pks), _lib.ptr(m), len(m), _lib.ptr(sig)),
            "fast_aggregate_verify")


def eth_fast_aggregate_verify(public_keys: Sequence[PublicKey], message: bytes, signature: Signature) -> None:
    pks = [PublicKey(p) for p in public_keys]
    sig, m = Signature(signature), bytes(message)
    arr, _keep = _ptr_array(pks)
    _result(_lib.lib().b200_eth_fast_aggregate_verify(C.cast(arr, C.c_void_p), len(pks), _lib.ptr(m), len(m), _lib.ptr(sig)),
            "eth_fast_aggregate_verify")


def aggregate_verify(public_keys: Sequence[PublicKey], msgs: Sequence[bytes], signature: Signature) -> None:
    pks = b"".join(PublicKey(p) for p in public_keys)
    sig = Signature(signature)
    arr, keep = _ptr_array(msgs)
    lens = (C.c_size_t * max(len(keep), 1))(*[len(m) for m in keep])
    _result(_lib.lib().b200_aggregate_verify(_lib.ptr(pks), len(public_keys), C.cast(arr, C.c_void_p),
                                             C.cast(lens, C.c_void_p), len(keep), _lib.ptr(sig)), "aggregate_verify")


def aggregate(signatures: Sequence[Signature]) -> Signature:
    if len(signatures) == 0:
        raise EmptyAggregate()
    flat = b"".join(Signature(s) for s in signatures)
    out = (C.c_uint8 * 96)()
    _result(_lib.lib().b200_aggregate(_lib.ptr(flat), len(signatures), out), "aggregate")
    return Signature(bytes(out))


def eth_aggregate_public_keys(public_keys: Sequence[PublicKey]) -> PublicKey:
    if len(public_keys) == 0:
        raise EmptyAggregate()
    flat = b"".join(PublicKey(p) for p in public_keys)
    out = (C.c_uint8 * 48)()
    _result(_lib.lib().b200_eth_aggregate_public_keys(_lib.ptr(flat), len(public_keys), out), "eth_aggregate_public_keys")
    return PublicKey(bytes(out))


# ---- the throughput path ----------------------------------------------------------------------------------------
def _nbytes(buf) -> int:
    if hasattr(buf, "nbytes"):
        return int(buf.nbytes)
    if hasattr(buf, "numel"):
        return int(buf.numel() * buf.element_size())
    return len(buf)


def _batch_size(off, msgs32, sigs, keys=None, indices=None, seed=None) -> int:
    """T of a batch call.  The C side reads raw pointers: refuse T + 1 offsets whose buffers (48-byte `keys` or uint32
    `indices`, 32-byte messages, 96-byte signatures) disagree with them, and a seed that is not 32 bytes."""
    t = len(off) - 1
    if t < 0:
        raise ValueError("offsets must hold T + 1 entries")
    n = int(off[-1])
    if ((keys is not None and _nbytes(keys) != 48 * n) or (indices is not None and len(indices) != n)
            or _nbytes(msgs32) != 32 * t or _nbytes(sigs) != 96 * t):
        raise ValueError(f"buffer sizes do not match the offsets: {n} keys, msgs {_nbytes(msgs32)} B, sigs {_nbytes(sigs)} B "
                         f"for {t} tuples")
    if seed is not None and len(seed) != 32:
        raise ValueError("seed must be 32 bytes")
    return t


def _groups(offsets, items, item_bytes: int, what: str):
    """uint32 offsets of T groups over `items` (flat `item_bytes`-byte items, or uint32 indices when item_bytes is 0)."""
    off = np.ascontiguousarray(offsets, dtype=np.uint32)
    t = len(off) - 1
    if off.ndim != 1 or t < 0:
        raise ValueError("offsets must hold T + 1 entries")
    if int(off[0]) != 0:
        raise ValueError("offsets must start at 0")
    n = int(off[-1])
    have = len(items) if item_bytes == 0 else _nbytes(items)
    if have != (n if item_bytes == 0 else item_bytes * n):
        raise ValueError(f"buffer sizes do not match the offsets: {n} {what} for {t} groups, got {have}")
    return off, t


def aggregate_batch(sigs_flat, offsets):
    """`aggregate` over T groups: group t is signatures offsets[t] .. offsets[t+1]-1 of sigs_flat (96 bytes each).
    -> (uint8[T, 96] compressed sums, int32[T] codes: 0, a decode code, 3 not in group, 16 empty); failed rows are zero."""
    off, t = _groups(offsets, sigs_flat, 96, "signatures")
    out, codes = np.zeros((max(t, 1), 96), dtype=np.uint8), np.zeros(max(t, 1), dtype=np.int32)
    _lib.check(_lib.lib().b200_aggregate_batch(_lib.ptr(sigs_flat), _lib.ptr(off), t, _lib.ptr(out), _lib.ptr(codes)),
               "aggregate_batch")
    return out[:t], codes[:t]


def eth_aggregate_public_keys_batch(pks_flat, offsets):
    """`eth_aggregate_public_keys` over T groups of 48-byte keys -> (uint8[T, 48], int32[T])."""
    off, t = _groups(offsets, pks_flat, 48, "keys")
    out, codes = np.zeros((max(t, 1), 48), dtype=np.uint8), np.zeros(max(t, 1), dtype=np.int32)
    _lib.check(_lib.lib().b200_eth_aggregate_public_keys_batch(_lib.ptr(pks_flat), _lib.ptr(off), t, _lib.ptr(out), _lib.ptr(codes)),
               "eth_aggregate_public_keys_batch")
    return out[:t], codes[:t]


def fast_aggregate_verify_batch(pks_flat, pk_offsets, msgs32, sigs) -> np.ndarray:
    """T tuples at once -> int32 code per tuple (0 Ok, 5 InvalidSignature, 1/2/3/6 BLST decode errors).
    pks_flat: (sum K) x 48 bytes; pk_offsets: uint32[T+1]; msgs32: T x 32; sigs: T x 96 (host buffers)."""
    off = np.ascontiguousarray(pk_offsets, dtype=np.uint32)
    t = _batch_size(off, msgs32, sigs, keys=pks_flat)
    if int(off[0]) != 0:
        raise ValueError("pk_offsets must start at 0")
    out = np.empty(max(t, 1), dtype=np.int32)
    _lib.check(_lib.lib().b200_fast_aggregate_verify_batch(_lib.ptr(pks_flat), _lib.ptr(off), _lib.ptr(msgs32), _lib.ptr(sigs),
                                                           t, _lib.ptr(out)), "fast_aggregate_verify_batch")
    return out[:t]


def fast_aggregate_verify_batch_all(pks_flat, pk_offsets, msgs32, sigs, seed: bytes = None, sharded: bool = False) -> bool:
    """Optimistic whole-batch check by random linear combination (T Miller loops + ONE final exponentiation): True iff
    every tuple verifies (false accept probability <= 2^-64 over `seed`; None = drawn by the library).  On False ask
    `fast_aggregate_verify_batch` for the per-tuple codes.  `sharded`: all ranks of the library's communicator share the
    batch (same arguments and seed on every rank); the Gt / G2 partials travel in one ncclAllGather."""
    off = np.ascontiguousarray(pk_offsets, dtype=np.uint32)
    t = _batch_size(off, msgs32, sigs, keys=pks_flat, seed=seed)
    if sharded and seed is None:
        raise ValueError("the ranks must share the seed")
    sd = np.frombuffer(bytes(seed), dtype=np.uint8) if seed is not None else None
    ok = C.c_int32(0)
    fn = _lib.lib().b200_fast_aggregate_verify_batch_all_sharded if sharded else _lib.lib().b200_fast_aggregate_verify_batch_all
    _lib.check(fn(_lib.ptr(pks_flat), _lib.ptr(off), _lib.ptr(msgs32), _lib.ptr(sigs), t, _lib.ptr(sd) if sd is not None else 0, C.byref(ok)),
               "fast_aggregate_verify_batch_all")
    return bool(ok.value)


def _messages(msgs, msg_group, t: int):
    """Flat bytes and uint32[n + 1] byte offsets of the messages (a sequence of bytes), and their T + 1 group offsets."""
    grp = np.ascontiguousarray(msg_group, dtype=np.uint32)
    if grp.ndim != 1 or len(grp) != t + 1:
        raise ValueError(f"msg_group must hold T + 1 = {t + 1} entries, got {len(grp)}")
    if int(grp[0]) != 0 or int(grp[-1]) != len(msgs):
        raise ValueError(f"msg_group must run from 0 to the {len(msgs)} messages")
    lens = [len(m) for m in msgs]
    moff = np.zeros(len(msgs) + 1, dtype=np.uint64)
    np.cumsum(lens, out=moff[1:])
    if int(moff[-1]) > 0xFFFFFFFF:
        raise ValueError("messages exceed 4 GiB in total")
    flat = np.frombuffer(b"".join(bytes(m) for m in msgs), dtype=np.uint8)
    return flat, moff.astype(np.uint32), grp


def aggregate_verify_batch(pks_flat, pk_offsets, msgs, msg_group, sigs) -> np.ndarray:
    """`aggregate_verify` over T tuples at once -> int32 code per tuple, as `aggregate_verify` would decide it (0 Ok,
    5 InvalidSignature, 1/2/3/6 BLST decode errors).  Tuple t: keys pk_offsets[t] .. pk_offsets[t+1]-1 of pks_flat (48 bytes
    each), messages msg_group[t] .. msg_group[t+1]-1 of `msgs` (a sequence of bytes, any lengths), signature sigs[96 t ..]."""
    off, t = _groups(pk_offsets, pks_flat, 48, "keys")
    if _nbytes(sigs) != 96 * t:
        raise ValueError(f"sigs must hold {t} x 96 bytes, got {_nbytes(sigs)}")
    flat, moff, grp = _messages(msgs, msg_group, t)
    out = np.empty(max(t, 1), dtype=np.int32)
    _lib.check(_lib.lib().b200_aggregate_verify_batch(_lib.ptr(pks_flat), _lib.ptr(off), _lib.ptr(flat), _lib.ptr(moff), _lib.ptr(grp),
                                                      _lib.ptr(sigs), t, _lib.ptr(out)), "aggregate_verify_batch")
    return out[:t]


class Registry:
    """Validated validator public keys resident in HBM (`state.validators[i].public_key` is immutable,
    phase0/validator.rs:10-13): `load` runs key_validate once per key, `verify_batch` names signers by index.
    The list of keys grows with the validator set: `append` validates only the new keys, `from_state` / `sync` read them
    from a resident `ssz.DeviceBeaconState` in HBM.  The library keeps one registry per process; `n` is its length."""

    def __init__(self, pks_flat):
        n = (pks_flat.nbytes if hasattr(pks_flat, "nbytes") else len(pks_flat)) // 48
        _lib.check(_lib.lib().b200_registry_load(_lib.ptr(pks_flat), n), "registry_load")
        self.n = n

    @classmethod
    def from_state(cls, state) -> "Registry":
        """The registry of every validator's public key of a (single-GPU) resident state, read on the device."""
        reg = cls.__new__(cls)
        _lib.check(_lib.lib().b200_registry_load_state(state._h), "registry_load_state")
        reg.n = state.n_validators
        return reg

    def append(self, pks_flat) -> None:
        """Validate and append 48-byte keys: they become indices n, n + 1, ...; the keys already loaded are not
        validated again."""
        nbytes = _nbytes(pks_flat)
        if nbytes % 48:
            raise ValueError(f"registry keys must be 48 bytes each, got {nbytes} bytes")
        _lib.check(_lib.lib().b200_registry_append(_lib.ptr(pks_flat), nbytes // 48), "registry_append")
        self.n += nbytes // 48

    def sync(self, state) -> None:
        """Append the validators `state` gained since the registry last matched it (`add_validators`); the first n keys
        are taken to be the state's first n public keys."""
        _lib.check(_lib.lib().b200_registry_sync_state(state._h), "registry_sync_state")
        self.n = state.n_validators

    def key_codes(self) -> np.ndarray:
        out = np.empty(max(self.n, 1), dtype=np.int32)
        _lib.check(_lib.lib().b200_registry_key_codes(_lib.ptr(out), self.n), "registry_key_codes")
        return out[:self.n]

    def aggregate_public_keys(self, indices, offsets):
        """`eth_aggregate_public_keys` over T groups of registry indices (group t: indices[offsets[t] .. offsets[t+1]-1])
        -> (uint8[T, 48], int32[T]); each key keeps the code it was validated with."""
        idx = np.ascontiguousarray(indices, dtype=np.uint32)
        off, t = _groups(offsets, idx, 0, "indices")
        out, codes = np.zeros((max(t, 1), 48), dtype=np.uint8), np.zeros(max(t, 1), dtype=np.int32)
        _lib.check(_lib.lib().b200_registry_aggregate_public_keys(_lib.ptr(idx), _lib.ptr(off), t, _lib.ptr(out), _lib.ptr(codes)),
                   "registry_aggregate_public_keys")
        return out[:t], codes[:t]

    def verify_batch(self, indices, offsets, msgs32, sigs, extra_keys=None) -> np.ndarray:
        """`extra_keys` (flat 48-byte keys): keys that arrive with the block (deposits, bls-to-execution changes); index
        self.n + j names extra key j, which this call validates like the strict path would (`..._batch_mixed`)."""
        idx = np.ascontiguousarray(indices, dtype=np.uint32)
        off = np.ascontiguousarray(offsets, dtype=np.uint32)
        t = _batch_size(off, msgs32, sigs, indices=idx)
        out = np.empty(max(t, 1), dtype=np.int32)
        if extra_keys is not None and _nbytes(extra_keys):
            if _nbytes(extra_keys) % 48:
                raise ValueError("extra keys must be 48 bytes each")
            _lib.check(_lib.lib().b200_fast_aggregate_verify_batch_mixed(_lib.ptr(extra_keys), _nbytes(extra_keys) // 48, _lib.ptr(idx), _lib.ptr(off),
                                                                         _lib.ptr(msgs32), _lib.ptr(sigs), t, _lib.ptr(out)), "verify_batch_mixed")
        else:
            _lib.check(_lib.lib().b200_fast_aggregate_verify_batch_indexed(_lib.ptr(idx), _lib.ptr(off), _lib.ptr(msgs32),
                                                                           _lib.ptr(sigs), t, _lib.ptr(out)), "verify_batch_indexed")
        return out[:t]

    def aggregate_verify_batch(self, indices, offsets, msgs, msg_group, sigs) -> np.ndarray:
        """`aggregate_verify_batch` with tuple t's keys named by registry indices indices[offsets[t] .. offsets[t+1]-1]."""
        idx = np.ascontiguousarray(indices, dtype=np.uint32)
        off, t = _groups(offsets, idx, 0, "indices")
        if _nbytes(sigs) != 96 * t:
            raise ValueError(f"sigs must hold {t} x 96 bytes, got {_nbytes(sigs)}")
        flat, moff, grp = _messages(msgs, msg_group, t)
        out = np.empty(max(t, 1), dtype=np.int32)
        _lib.check(_lib.lib().b200_aggregate_verify_batch_indexed(_lib.ptr(idx), _lib.ptr(off), _lib.ptr(flat), _lib.ptr(moff),
                                                                  _lib.ptr(grp), _lib.ptr(sigs), t, _lib.ptr(out)),
                   "aggregate_verify_batch_indexed")
        return out[:t]

    def verify_batch_all(self, indices, offsets, msgs32, sigs, seed: bytes = None) -> bool:
        """`fast_aggregate_verify_batch_all` over registry indices."""
        idx = np.ascontiguousarray(indices, dtype=np.uint32)
        off = np.ascontiguousarray(offsets, dtype=np.uint32)
        t = _batch_size(off, msgs32, sigs, indices=idx, seed=seed)
        sd = np.frombuffer(bytes(seed), dtype=np.uint8) if seed is not None else None
        ok = C.c_int32(0)
        _lib.check(_lib.lib().b200_fast_aggregate_verify_batch_indexed_all(_lib.ptr(idx), _lib.ptr(off), _lib.ptr(msgs32), _lib.ptr(sigs), t,
                                                                           _lib.ptr(sd) if sd is not None else 0, C.byref(ok)), "verify_batch_indexed_all")
        return bool(ok.value)


def last_kernel_ms() -> float:
    return float(_lib.lib().b200_last_kernel_ms())


def last_dominant_kernel_ms() -> float:
    return float(_lib.lib().b200_last_dominant_kernel_ms())


def fp_selftest(n: int = 1 << 16, seed: int = 1) -> int:
    m = C.c_uint32(0)
    _lib.check(_lib.lib().b200_fp_selftest(n, seed, C.byref(m)), "fp_selftest")
    return int(m.value)


# operations of fp_eval (bls_kernels.cuh FP_EVAL_* / FP2_EVAL_*)
FP_EVAL_OPS = {"fp_mul": 0, "fp_sqr": 1, "fpl_mul": 2, "fpl_sqr": 3, "fp_add": 4, "fp_sub": 5, "fp_neg": 6, "fpl_add": 7,
               "fpl_sub": 8, "fpl_neg": 9, "fp_add_raw": 10, "fp_sub_raw": 11, "fp_inv_kaliski": 12, "fp_inv_fermat": 13,
               "fp_sqrt": 14, "fpl_pow_sqrt": 15, "fp_is_lex_largest": 16, "fpl_sqrt_chain": 18,
               "fpl_mul_sub_mul": 19, "fpl_mul_sub_8sqr": 20,
               "fp2_mul": 32, "fp2_sqr": 33, "fp2_inv": 34, "fp2_sqrt": 35, "fp2_sgn0": 36,
               "fpd_mul": 40, "fpd_sqr": 41, "fpd_add": 42, "fpd_from_fp": 43, "fpd_to_fpl": 44, "fpd_sqrt_chain": 45,
               "fpd_y_from_x": 46}


def fp_eval(op: str, a, b=None) -> np.ndarray:
    """Self-test: one device field operation on raw limbs.  a, b: uint32[n, 24] (Fp in columns 0..11, Fp2 c0 | c1, FpD
    as 8 binary64 limbs in columns 0..15, i.e. a.view(np.float64)[:, :8]); returns uint32[n, 25]: the result's limbs,
    then the flag word (carry, borrow, is-square, on-curve, lex-largest or sgn0)."""
    a = np.ascontiguousarray(a, dtype=np.uint32)
    b = np.zeros_like(a) if b is None else np.ascontiguousarray(b, dtype=np.uint32)
    if a.ndim != 2 or a.shape[1] != 24 or b.shape != a.shape:
        raise ValueError("operands must be uint32[n, 24]")
    out = np.zeros((max(a.shape[0], 1), 25), dtype=np.uint32)
    _lib.check(_lib.lib().b200_fp_eval(FP_EVAL_OPS[op], a.shape[0], _lib.ptr(a), _lib.ptr(b), _lib.ptr(out)), f"fp_eval({op})")
    return out[:a.shape[0]]


# operations of curve_eval (bls_kernels.cuh CURVE_G1L_* / CURVE_G2_*)
CURVE_EVAL_OPS = {"g1l_add_mixed": 0, "g1l_add": 1, "g1l_in_subgroup": 2, "g1l_double": 4, "g1_in_subgroup_iso": 6,
                  "g2_add": 32, "g2_add_mixed": 33, "g2_double": 34, "g2_in_subgroup": 35, "g2_psi": 36,
                  "g2_clear_cofactor": 37, "g2_sswu_iso": 38, "g2_h2c_finish": 39}


def curve_eval(op: str, a, b=None) -> np.ndarray:
    """Self-test: one device curve stage on raw limbs.  a, b: uint32[n, 73] (X, Y, Z as 24-word slots, Fp in the first 12
    words, Fp2 c0 | c1, then the affine infinity flag); returns uint32[n, 73]: the result point, then the flag word
    (subgroup verdict, or the infinity flag of an affine result)."""
    a = np.ascontiguousarray(a, dtype=np.uint32)
    b = np.zeros_like(a) if b is None else np.ascontiguousarray(b, dtype=np.uint32)
    if a.ndim != 2 or a.shape[1] != 73 or b.shape != a.shape:
        raise ValueError("operands must be uint32[n, 73]")
    out = np.zeros((max(a.shape[0], 1), 73), dtype=np.uint32)
    _lib.check(_lib.lib().b200_curve_eval(CURVE_EVAL_OPS[op], a.shape[0], _lib.ptr(a), _lib.ptr(b), _lib.ptr(out)),
               f"curve_eval({op})")
    return out[:a.shape[0]]


# operations of pairing_eval (bls_kernels.cuh PAIRING_EVAL_*)
PAIRING_EVAL_OPS = {"fp6_mul": 0, "fp6_inv": 1, "fp12_mul": 2, "fp12_sqr": 3, "fp12_inv": 4, "fp12_mul_by_line": 5,
                    "fp12_frobenius1": 6, "fp12_frobenius2": 7, "fp12_cyclotomic_sqr": 8, "fp12_pow_z": 9,
                    "miller_double_step": 10, "miller_add_step": 11, "miller_loop": 12, "final_exp": 13,
                    "vm_miller8": 32, "vm_miller16": 33, "vm_final8": 34, "vm_final16": 35,
                    "fold_fp12": 48, "fold_g2": 49, "fold_segments": 50}


def pairing_eval(op: str, a, b=None) -> np.ndarray:
    """Self-test: one device pairing operation on raw limbs.  a, b: uint32[n, 145] (twelve 12-word Fp slots in Fp12
    memory order, then the infinity flag of a point); returns uint32[n, 145]: the result's slots, then the flag word (the
    final exponentiation's verdict, or the infinity flag of the G2 fold's sum).  The folds return their one result in row 0;
    fold_segments takes the segment count T and T + 1 offsets as the first words of b and returns rows 2t, 2t + 1."""
    a = np.ascontiguousarray(a, dtype=np.uint32)
    b = np.zeros_like(a) if b is None else np.ascontiguousarray(b, dtype=np.uint32)
    if a.ndim != 2 or a.shape[1] != 145 or b.shape != a.shape:
        raise ValueError("operands must be uint32[n, 145]")
    out = np.zeros((max(a.shape[0], 1), 145), dtype=np.uint32)
    _lib.check(_lib.lib().b200_pairing_eval(PAIRING_EVAL_OPS[op], a.shape[0], _lib.ptr(a), _lib.ptr(b), _lib.ptr(out)),
               f"pairing_eval({op})")
    return out[:a.shape[0]]


def tune(knob: str, value: int) -> None:
    """Launch-shape knobs of the batch pipeline (include/b200_consensus.h, b200_tune): never change a result.

    The knobs are "bls_small_cta", "vm_team16_max" and "vm_cta"; any other name raises EngineError (B200_ERR_BAD_ARG)."""
    _lib.check(_lib.lib().b200_tune(knob.encode(), int(value)), f"tune({knob})")


def vm_load_programs(blob) -> None:
    """Swap in another schedule of the pairing programs (uint32 words written by tools/gen_pairing_vm.py --blob)."""
    a = np.ascontiguousarray(blob, dtype=np.uint32)
    _lib.check(_lib.lib().b200_vm_load_programs(_lib.ptr(a), a.size), "vm_load_programs")


def measure_int_peak(kind: int) -> float:
    """1e9 ops/s of IMAD.WIDE.U32 (0), IMAD.U32 (1) or the LOP3/SHF/IADD3 mix (2) measured on this device."""
    g = C.c_double(0)
    _lib.check(_lib.lib().b200_measure_int_peak(kind, C.byref(g)), "measure_int_peak")
    return float(g.value)
