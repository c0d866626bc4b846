"""Builds the CUDA C-ABI library in-tree: ethereum_consensus_b200/libb200_consensus.so (sm_90a only)."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libb200_consensus.so"
OBJ = PKG / "build"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]   # H100 (Hopper)
FLAGS = [*ARCH, "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr"]
# Per-TU ptxas optimisation level.  The three BLS translation units whose kernels are chains of inline-PTX Montgomery
# products are assembled below the default level: at -O3 ptxas interleaves more carry chains than it has predicate
# registers and spills the carries into a GPR bitmask (LOP3 / P2R / ISETP around every product); at -O1 the same
# IMAD.WIDE remain, four chains stay interleaved and the spill code is gone.  bls_g1.cu, whose per-key kernel has no
# shared-memory table and spills to an L1-resident stack, is fastest at -O2 (DESIGN.md §4, K1's memory).  NVVM still
# runs at -O3.
DEFAULT_PTXAS_OPT = {"bls_g1.cu": 2, "bls_g2.cu": 1, "bls_vm.cu": 1}


def _stale(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compiles every translation unit under csrc/ that is out of date and links the library."""
    srcs = sorted(CSRC.glob("*.cu"))
    hdrs = sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + sorted((PKG.parent / "include").glob("*.h"))
    OBJ.mkdir(exist_ok=True)
    jobs = []
    def command(s, o):
        cmd = [NVCC, *FLAGS, "-c", str(s), "-o", str(o)]
        if s.name in DEFAULT_PTXAS_OPT:
            cmd[1:1] = ["-Xptxas", f"-O{DEFAULT_PTXAS_OPT[s.name]}"]
        return cmd

    for s in srcs:
        o = OBJ / (s.stem + ".o")
        stamp = o.with_suffix(".cmd")   # the object is also stale when its command line changed
        if force or _stale(o, [s] + hdrs) or not stamp.exists() or stamp.read_text() != " ".join(command(s, o)):
            jobs.append((s, o))

    def cc(job):
        s, o = job
        cmd = command(s, o)
        stamp = o.with_suffix(".cmd")
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s.name}:\n{r.stdout}\n{r.stderr}")
        stamp.write_text(" ".join(command(s, o)))
        return r.stderr

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for msg in ex.map(cc, jobs):
            if verbose and msg:
                print(msg, file=sys.stderr)
    objs = [OBJ / (s.stem + ".o") for s in srcs]
    if force or jobs or _stale(LIB, objs):
        cmd = [NVCC, "-shared", "-o", str(LIB), *map(str, objs), *ARCH,
               "-Xcompiler", "-fPIC", "-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
