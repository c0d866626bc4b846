"""Consumer for the reference's REAL parity vectors: the `consensus-spec-tests` tree its `spec-tests` crate walks
(spec-tests/main.rs:20,56-112 — `tests/<config>/<fork>/<runner>/<handler>/<suite>/<case>/`), with the
case semantics of spec-tests/runners/bls.rs:17-58 (per-handler `data.yaml`: `input`, `output`) and
runners/ssz_static.rs:13-36 (`roots.yaml` + `serialized.ssz_snappy`, raw snappy as test_utils.rs:30-37 decodes it).

The vectors are downloaded by the reference's justfile and are absent offline; anyone who has the tarball points
CONSENSUS_SPEC_TESTS at it (or unpacks it as <repo>/consensus-spec-tests) and tests/test_spec_vectors.py closes the
"weakly pinned" gap of DESIGN.md §2 against both the CPU oracle and the CUDA path.  Test infrastructure only.
"""
from __future__ import annotations

import os
from pathlib import Path
from typing import Iterator, Optional, Tuple

import yaml

ROOT = Path(__file__).resolve().parent.parent
BLS_HANDLERS = ("aggregate", "aggregate_verify", "eth_aggregate_pubkeys", "eth_fast_aggregate_verify",
                "fast_aggregate_verify", "verify")   # `sign` needs a SecretKey: not on the verification path


def vectors_root() -> Optional[Path]:
    for cand in (os.environ.get("CONSENSUS_SPEC_TESTS"), ROOT / "consensus-spec-tests"):
        if cand and (Path(cand) / "tests").is_dir():
            return Path(cand)
    return None


def walk(root: Path, runner: str, handlers=None) -> Iterator[Tuple[str, str, str, Path]]:
    """(config, fork, handler, case_dir) for every leaf case of `runner`."""
    base = root / "tests"
    for config in sorted(p for p in base.iterdir() if p.is_dir()):
        for fork in sorted(p for p in config.iterdir() if p.is_dir()):
            r = fork / runner
            if not r.is_dir():
                continue
            for handler in sorted(p for p in r.iterdir() if p.is_dir()):
                if handlers is not None and handler.name not in handlers:
                    continue
                for suite in sorted(p for p in handler.iterdir() if p.is_dir()):
                    for case in sorted(p for p in suite.iterdir() if p.is_dir()):
                        yield config.name, fork.name, handler.name, case


def unhex(s, n=None) -> Optional[bytes]:
    """'0x..' -> bytes; None when the literal is not hex of the expected length (the reference's `DefaultOnError`)."""
    if not isinstance(s, str) or not s.startswith("0x"):
        return None
    try:
        b = bytes.fromhex(s[2:])
    except ValueError:
        return None
    return b if n is None or len(b) == n else None


def snappy_raw_decompress(data: bytes) -> bytes:
    """Raw (unframed) snappy block format: varint length, then literal / copy elements."""
    pos, n, shift = 0, 0, 0
    while True:
        b = data[pos]; pos += 1
        n |= (b & 0x7F) << shift
        if not b & 0x80:
            break
        shift += 7
    out = bytearray()
    while pos < len(data):
        tag = data[pos]; pos += 1
        kind = tag & 3
        if kind == 0:
            ln = tag >> 2
            if ln >= 60:
                nb = ln - 59
                ln = int.from_bytes(data[pos:pos + nb], "little"); pos += nb
            ln += 1
            out += data[pos:pos + ln]; pos += ln
            continue
        if kind == 1:
            ln = ((tag >> 2) & 7) + 4
            off = ((tag >> 5) << 8) | data[pos]; pos += 1
        elif kind == 2:
            ln = (tag >> 2) + 1
            off = int.from_bytes(data[pos:pos + 2], "little"); pos += 2
        else:
            ln = (tag >> 2) + 1
            off = int.from_bytes(data[pos:pos + 4], "little"); pos += 4
        if off == 0 or off > len(out):
            raise ValueError("snappy: bad copy offset")
        for _ in range(ln):   # copies may overlap their own output
            out.append(out[-off])
    if len(out) != n:
        raise ValueError(f"snappy: length {len(out)} != header {n}")
    return bytes(out)


def snappy_raw_compress_literal(data: bytes) -> bytes:
    """Valid raw-snappy stream made of literal elements only (fixtures for the runner's own tests)."""
    out = bytearray()
    n = len(data)
    while True:
        b = n & 0x7F
        n >>= 7
        out.append(b | (0x80 if n else 0))
        if not n:
            break
    pos = 0
    while pos < len(data):
        chunk = data[pos:pos + 65536]
        ln = len(chunk) - 1
        if ln < 60:
            out.append(ln << 2)
        else:
            nb = (ln.bit_length() + 7) // 8
            out.append((59 + nb) << 2)
            out += ln.to_bytes(nb, "little")
        out += chunk
        pos += len(chunk)
    return bytes(out)


# ---- per-handler evaluation: `impl` is any object with the crypto-mirror API (ethereum_consensus_b200.crypto on the GPU,
# tests.spec_vectors.OracleImpl on the CPU).  Returns (passed, detail).
def run_bls_case(handler: str, case_dir: Path, impl) -> Tuple[bool, str]:
    d = yaml.safe_load((case_dir / "data.yaml").read_text())
    inp, want = d["input"], d["output"]

    def ok(fn, *a):
        try:
            fn(*a)
            return True
        except impl.Error:
            return False

    if handler == "aggregate":
        sigs = [unhex(s, 96) for s in inp]
        if any(s is None for s in sigs):
            return want is None, "malformed input"
        try:
            got = bytes(impl.aggregate(sigs))
        except impl.Error:
            return want is None, "aggregate failed"
        return want is not None and got == unhex(want), got.hex()
    if handler == "eth_aggregate_pubkeys":
        pks = [unhex(s, 48) for s in (inp or [])]
        if any(p is None for p in pks):
            return want is None, "malformed input"
        try:
            got = bytes(impl.eth_aggregate_public_keys(pks))
        except impl.Error:
            return want is None, "aggregation failed"
        return want is not None and got == unhex(want), got.hex()
    sig = unhex(inp.get("signature"), 96)
    if handler == "verify":
        pk = unhex(inp.get("pubkey"), 48)
        if sig is None or pk is None:   # undecodable literal: the reference counts the case as a pass when output is false
            return want is False, "malformed input"
        return ok(impl.verify_signature, pk, unhex(inp["message"]), sig) == bool(want), ""
    if handler in ("fast_aggregate_verify", "eth_fast_aggregate_verify"):
        pks = [unhex(s, 48) for s in inp["pubkeys"]]
        if sig is None or any(p is None for p in pks):
            return want is False, "malformed input"
        fn = impl.fast_aggregate_verify if handler == "fast_aggregate_verify" else impl.eth_fast_aggregate_verify
        return ok(fn, pks, unhex(inp["message"]), sig) == bool(want), ""
    if handler == "aggregate_verify":
        pks = [unhex(s, 48) for s in inp["pubkeys"]]
        if sig is None:
            return want is False, "malformed input"
        pks = [p for p in pks if p is not None]   # `.iter().flatten()` in the reference runner
        msgs = [unhex(m) for m in inp["messages"]]
        return ok(impl.aggregate_verify, pks, msgs, sig) == bool(want), ""
    raise ValueError(handler)


class OracleImpl:
    """The Python big-int oracle behind the same call surface (CPU side of the runner)."""

    class Error(Exception):
        pass

    def __init__(self):
        from oracle import bls_oracle as bo
        self.bo = bo

    def _chk(self, code):
        if code != 0:
            raise self.Error(code)

    def verify_signature(self, pk, m, s): self._chk(self.bo.verify_signature(pk, m, s))
    def fast_aggregate_verify(self, pks, m, s): self._chk(self.bo.fast_aggregate_verify(pks, m, s))
    def eth_fast_aggregate_verify(self, pks, m, s): self._chk(self.bo.eth_fast_aggregate_verify(pks, m, s))
    def aggregate_verify(self, pks, ms, s): self._chk(self.bo.aggregate_verify(pks, ms, s))

    def aggregate(self, sigs):
        code, out = self.bo.aggregate(sigs)
        self._chk(code)
        return out

    def eth_aggregate_public_keys(self, pks):
        code, out = self.bo.eth_aggregate_public_keys(pks)
        self._chk(code)
        return out


def ssz_static_case(case_dir: Path) -> Tuple[bytes, bytes]:
    """(serialized bytes, expected root) of one ssz_static case."""
    root = unhex(yaml.safe_load((case_dir / "roots.yaml").read_text())["root"], 32)
    return snappy_raw_decompress((case_dir / "serialized.ssz_snappy").read_bytes()), root
