"""SASS instructions per 64-byte pair hash in the SSZ kernels: the per-unit figure of bench.py's SSZ ALU roofline
(SASS_OPS_PER_PAIR_HASH).  k_validator_roots is straight-line code that computes exactly 8 pair hashes per thread, so
its ALU-class instruction count / 8 is the figure.   python tools/count_sha_sass.py [path/to/ssz_kernels.o]"""
import collections
import re
import subprocess
import sys
from pathlib import Path

obj = sys.argv[1] if len(sys.argv) > 1 else str(Path(__file__).resolve().parent.parent / "ethereum_consensus_b200" / "build" / "ssz_kernels.o")
sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
cur, counts = None, collections.defaultdict(collections.Counter)
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        counts[cur][m.group(1).split(".")[0]] += 1
ALU = {"LOP3", "SHF", "IADD3", "IADD", "PRMT", "VIADD", "LEA", "IMAD", "MOV", "SEL"}
for fn, c in counts.items():
    if "17k_validator_rootsE" not in fn:   # the dense kernel, not k_validator_roots_sparse
        continue
    alu = sum(v for k, v in c.items() if k in ALU)
    core = sum(v for k, v in c.items() if k in ("LOP3", "SHF", "IADD3", "VIADD", "IADD"))
    print(fn[:60])
    print("  total instructions", sum(c.values()), "| LOP3/SHF/IADD3-class", core, "| + PRMT/LEA/IMAD/MOV/SEL", alu)
    print("  per pair hash (8 per thread): LOP3/SHF/IADD3-class", round(core / 8), "| all ALU-class", round(alu / 8))
    print("  mix:", dict(c.most_common(10)))
