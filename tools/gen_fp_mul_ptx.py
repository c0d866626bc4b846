"""Generates ethereum_consensus_b200/csrc/fp_mul_ptx.cuh: the tuned Montgomery product and square for sm_90a, each as
ONE inline-PTX block (a carry chain must never be split across asm statements), plus a C emulation of exactly the
same instruction lists (`fp_mul_emul_core`, `fp_sqr_emul_core`, host-testable) so the sequences are verified against
big-ints on the CPU before the PTX ever runs on a GPU (tests/test_oracle_bls.py::test_fp_mul_ptx_emulation).

12 x 32-bit limbs, R = 2^384.  Everything is organised in even-aligned 64-bit "lanes" (x[2k], x[2k+1]) so that ptxas
fuses each mad.lo.cc / madc.hi.cc pair into one IMAD.WIDE.U32(.X) with carry-in/out predicates:

* product: CIOS with two accumulators, value = sum ev[k] 2^(32k) + sum od[k] 2^(32(k+1)); round i adds a*b_i and m*p
  and divides by 2^32 by swapping the roles of ev and od (no data movement).          288 wide MADs.
* square: off-diagonal products a_i a_j (i<j) into TE (even columns) / TO (odd columns), doubled with funnel shifts,
  diagonal squares added, then 12 reduction rounds that fold one column per round; chain carry-outs are collected
  lazily in a side array (they only affect columns >= 12).                              66 + 12 + 144 = 222 wide MADs.
"""
from pathlib import Path

N = 12
P_INT = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
P_LIMBS = [(P_INT >> (32 * i)) & 0xffffffff for i in range(12)]


def A(j): return f"a{j}"
def B(i): return f"b{i}"
def Pm(j): return f"p{j}"


# ------------------------------------------------------------------------------------------------ product
def build_mul():
    ops = []

    def emit(op, d, a, b=None, c=None):
        ops.append((op, d, a, b, c))

    def cmad_n(acc, src, s0, scalar):
        for j in range(0, N, 2):
            emit("mad.lo.cc" if j == 0 else "madc.lo.cc", acc[j], src(s0 + j), scalar, acc[j])
            emit("madc.hi.cc", acc[j + 1], src(s0 + j), scalar, acc[j + 1])

    def round_(ev, od, bi, first):
        if first:
            for j in range(0, N, 2):
                emit("mul.lo", od[j], A(j + 1), bi); emit("mul.hi", od[j + 1], A(j + 1), bi)
            for j in range(0, N, 2):
                emit("mul.lo", ev[j], A(j), bi); emit("mul.hi", ev[j + 1], A(j), bi)
        else:
            emit("add.cc", ev[0], ev[0], od[1])
            for j in range(0, N - 2, 2):
                emit("madc.lo.cc", od[j], A(j + 1), bi, od[j + 2])
                emit("madc.hi.cc", od[j + 1], A(j + 1), bi, od[j + 3])
            emit("madc.lo.cc", od[N - 2], A(N - 1), bi, "0")
            emit("madc.hi", od[N - 1], A(N - 1), bi, "0")
            cmad_n(ev, A, 0, bi)
            emit("addc", od[N - 1], od[N - 1], "0")
        emit("mul.lo", "m", ev[0], "n0")
        cmad_n(od, Pm, 1, "m")
        cmad_n(ev, Pm, 0, "m")
        emit("addc", od[N - 1], od[N - 1], "0")

    ev = [f"e{k}" for k in range(N)]
    od = [f"o{k}" for k in range(N)]
    for i in range(0, N, 2):
        round_(ev, od, B(i), i == 0)
        round_(od, ev, B(i + 1), False)
    emit("add.cc", ev[0], ev[0], od[1])
    for k in range(1, N - 1):
        emit("addc.cc", ev[k], ev[k], od[k + 1])
    emit("addc", ev[N - 1], ev[N - 1], "0")
    return ops, ev + od + ["m"], ev


# ------------------------------------------------------------------------------------------------ square
def build_sqr():
    ops = []
    live = set()          # registers that hold a defined value

    def emit(op, d, a, b=None, c=None):
        ops.append((op, d, a, b, c))
        live.add(d)

    def val(r):           # operand: register if defined else literal zero
        return r if r in live else "0"

    TE = [f"te{k}" for k in range(26)]   # TE[k] <-> column k
    TO = [f"to{k}" for k in range(26)]   # TO[k] <-> column k + 1
    CY = [f"c{k}" for k in range(26)]    # lazy carries, CY[k] <-> column k

    def lane(col):
        """(array, index) of the even-aligned lane whose low word is column `col`."""
        return (TE, col) if col % 2 == 0 else (TO, col - 1)

    def word(col, arr):
        return arr[col] if arr is TE else arr[col - 1]

    # ---- off-diagonal products
    for i in range(N - 1):
        for parity in (0, 1):  # parity 0: j = i+2, i+4..  (even columns -> TE); parity 1: j = i+1, i+3.. (odd columns -> TO)
            js = list(range(i + 2 - parity, N, 2))
            if not js:
                continue
            for n_, j in enumerate(js):
                arr, idx = lane(i + j)
                lo, hi = arr[idx], arr[idx + 1]
                emit("mad.lo.cc" if n_ == 0 else "madc.lo.cc", lo, A(i), A(j), val(lo))
                emit("madc.hi.cc", hi, A(i), A(j), val(hi))
            arr, idx = lane(i + js[-1])
            top = arr[idx + 2]
            emit("addc", top, val(top), "0")
    # ---- double both arrays with funnel shifts (independent ops, high word first so sources are still intact)
    for arr in (TE, TO):
        for k in range(23, -1, -1):
            hi_w = arr[k]
            lo_w = arr[k - 1] if k > 0 else None
            if hi_w not in live and (lo_w is None or lo_w not in live):
                continue
            emit("shf.l.wrap", hi_w, val(lo_w) if lo_w else "0", val(hi_w), "1")
    # ---- diagonal squares at even columns: one chain over the TE lanes
    for i in range(N):
        lo, hi = TE[2 * i], TE[2 * i + 1]
        emit("mad.lo.cc" if i == 0 else "madc.lo.cc", lo, A(i), A(i), val(lo))
        emit("madc.hi.cc", hi, A(i), A(i), val(hi))
    # ---- 12 reduction rounds; cy = pending carry into the current column
    for i in range(N):
        X, xi = lane(i)                       # lane starting at column i
        Y = TO if X is TE else TE
        xlo = X[xi]
        yw = word(i, Y) if i > 0 or Y is TE else None
        if i == 0:
            yw = None                         # column 0 only exists in TE
        # (h : s) = xlo + yw + cy
        if yw is not None and yw in live:
            emit("add.cc", xlo, val(xlo), yw)
            emit("addc", "h", "0", "0")
            if "cy" in live:
                emit("add.cc", xlo, xlo, "cy")
                emit("addc", "h", "h", "0")
            emit("mov", "cy", "h")
        else:
            if "cy" in live:
                emit("add.cc", xlo, val(xlo), "cy")
                emit("addc", "cy", "0", "0")
        emit("mul.lo", "m", xlo, "n0")
        # even-j products: lanes at columns i, i+2, .., i+10 (array X)
        for j in range(0, N, 2):
            arr, idx = lane(i + j)
            emit("mad.lo.cc" if j == 0 else "madc.lo.cc", arr[idx], Pm(j), "m", val(arr[idx]))
            emit("madc.hi.cc", arr[idx + 1], Pm(j), "m", val(arr[idx + 1]))
        emit("addc", CY[i + 12], val(CY[i + 12]), "0")
        # odd-j products: lanes at columns i+1, .., i+11 (array Y)
        for j in range(1, N, 2):
            arr, idx = lane(i + j)
            emit("mad.lo.cc" if j == 1 else "madc.lo.cc", arr[idx], Pm(j), "m", val(arr[idx]))
            emit("madc.hi.cc", arr[idx + 1], Pm(j), "m", val(arr[idx + 1]))
        emit("addc", CY[i + 13], val(CY[i + 13]), "0")
    # ---- result columns 12..23: r[k] = TE[12+k] + TO-word(12+k) + CY[12+k] (+ cy into column 12)
    res = [f"r{k}" for k in range(N)]
    for k in range(N):
        col = 12 + k
        emit("add.cc" if k == 0 else "addc.cc", res[k], val(TE[col]), val(TO[col - 1]))
    for k in range(N):
        col = 12 + k
        extra = val(CY[col])
        emit("add.cc" if k == 0 else "addc.cc", res[k], res[k], extra)
    if "cy" in live:
        emit("add.cc", res[0], res[0], "cy")
        for k in range(1, N):
            emit("addc.cc", res[k], res[k], "0")
    regs = sorted(live, key=lambda r: (r.rstrip("0123456789"), int("".join(ch for ch in r if ch.isdigit()) or 0)))
    return ops, regs, res


# ------------------------------------------------------------------------------------------------ emitters
def emit_c(name, ops, regs, res, two_inputs):
    c = []
    c.append(f"B200_HD void {name}(uint32_t r[12], const uint32_t a[12]" + (", const uint32_t b[12]" if two_inputs else "") + ") {\n")
    c.append("    const uint32_t n0 = B200_FP_N0;\n")
    c.append("    " + " ".join(f"const uint32_t p{j} = 0x{P_LIMBS[j]:08x}u;" for j in range(12)) + "\n")
    c.append("    " + " ".join(f"const uint32_t a{j} = a[{j}];" for j in range(12)) + "\n")
    if two_inputs:
        c.append("    " + " ".join(f"const uint32_t b{j} = b[{j}];" for j in range(12)) + "\n")
    c.append("    uint32_t cc = 0; uint64_t w; (void)cc; (void)n0;\n")
    c.append("    uint32_t " + ", ".join(f"{r} = 0" for r in regs) + ";\n")
    def lit(x): return "0u" if x == "0" else ("1u" if x == "1" else x)
    for op, d, x, y, z in ops:
        x, y, z = (lit(x) if x is not None else None, lit(y) if y is not None else None, lit(z) if z is not None else None)
        if op == "mul.lo": c.append(f"    {d} = {x} * {y};\n")
        elif op == "mul.hi": c.append(f"    {d} = uint32_t((uint64_t({x}) * {y}) >> 32);\n")
        elif op == "mad.lo.cc": c.append(f"    w = uint64_t(uint32_t({x} * {y})) + {z}; {d} = uint32_t(w); cc = uint32_t(w >> 32);\n")
        elif op == "madc.lo.cc": c.append(f"    w = uint64_t(uint32_t({x} * {y})) + {z} + cc; {d} = uint32_t(w); cc = uint32_t(w >> 32);\n")
        elif op == "madc.hi.cc": c.append(f"    w = ((uint64_t({x}) * {y}) >> 32) + {z} + cc; {d} = uint32_t(w); cc = uint32_t(w >> 32);\n")
        elif op == "madc.hi": c.append(f"    {d} = uint32_t(((uint64_t({x}) * {y}) >> 32) + {z} + cc);\n")
        elif op == "add.cc": c.append(f"    w = uint64_t({x}) + {y}; {d} = uint32_t(w); cc = uint32_t(w >> 32);\n")
        elif op == "addc.cc": c.append(f"    w = uint64_t({x}) + {y} + cc; {d} = uint32_t(w); cc = uint32_t(w >> 32);\n")
        elif op == "addc": c.append(f"    {d} = {x} + {y} + cc;\n")
        elif op == "add": c.append(f"    {d} = {x} + {y};\n")
        elif op == "mov": c.append(f"    {d} = {x};\n")
        elif op == "shf.l.wrap": c.append(f"    {d} = ({y} << 1) | ({x} >> 31);\n")
        else: raise ValueError(op)
    c.append("    " + " ".join(f"r[{k}] = {res[k]};" for k in range(12)) + "\n}\n\n")
    return c


def emit_ptx(name, ops, regs, res, two_inputs):
    names = {}
    temps = [r for r in regs if r not in res]
    for k, nme in enumerate(res): names[nme] = f"%{k}"
    ins = [f"a{j}" for j in range(12)] + ([f"b{j}" for j in range(12)] if two_inputs else [])
    for k, nme in enumerate(ins): names[nme] = f"%{len(res) + k}"
    for k, nme in enumerate(temps): names[nme] = f"t{k}"
    for j in range(12): names[f"p{j}"] = f"0x{P_LIMBS[j]:08x}"
    names["n0"] = "0xfffcfffd"; names["0"] = "0"; names["1"] = "1"
    lines = ["{", f".reg .u32 t<{len(temps)}>;"]
    for op, d, x, y, z in ops:
        args = [names[d], names[x]] + ([names[y]] if y is not None else []) + ([names[z]] if z is not None else [])
        suffix = ".b32" if op in ("shf.l.wrap", "mov") else ".u32"
        lines.append(f"{op}{suffix} {', '.join(args)};")
    lines.append("}")
    c = []
    c.append(f"__device__ __forceinline__ void {name}(uint32_t r[12], const uint32_t a[12]" + (", const uint32_t b[12]" if two_inputs else "") + ") {\n")
    c.append("    uint32_t " + ", ".join(res) + ";\n")
    c.append("    asm(\n")
    for ln in lines:
        c.append(f'        "{ln}\\n\\t"\n')
    c.append("        : " + ", ".join(f'"=&r"({n})' for n in res) + "\n")
    srcs = ["a"] + (["b"] if two_inputs else [])
    c.append("        : " + ", ".join(f'"r"({n}[{j}])' for n in srcs for j in range(12)) + ");\n")
    c.append("    " + " ".join(f"r[{k}] = {res[k]};" for k in range(12)) + "\n}\n\n")
    return c


def split_carry_captures(ops, regs):
    """EXPERIMENT (--split-carry), not used: `x += carry` written as `addc x, x, 0` comes out of ptxas as IMAD.X — on the FMA
    pipe these kernels are bound by (31 per square, 22 per product: ~5 % of the pipe).  Writing it as a capture into a scratch
    register plus a plain add was meant to move both to the ALU pipe; ptxas 12.9 instead materialises the capture as predicated
    IMAD.MOVs (product: 7 -> 59 IMAD.MOV, square: 15 -> 112), still on the FMA pipe and more of them.  Checked in SASS only."""
    out = []
    for op, d, x, y, z in ops:
        if op == "addc" and y == "0" and x != "0":
            out.append(("addc", "ct", "0", "0", None))
            out.append(("add", d, x, "ct", None))
        else:
            out.append((op, d, x, y, z))
    return out, (regs + ["ct"] if "ct" not in regs else regs)


def main():
    import sys
    mul_ops, mul_regs, mul_res = build_mul()
    sqr_ops, sqr_regs, sqr_res = build_sqr()
    if "--split-carry" in sys.argv:
        mul_ops, mul_regs = split_carry_captures(mul_ops, mul_regs)
        sqr_ops, sqr_regs = split_carry_captures(sqr_ops, sqr_regs)
    out = ["// GENERATED by tools/gen_fp_mul_ptx.py — do not edit.  Included from fp.cuh (needs B200_HD, B200_FP_N0).\n#pragma once\n\nnamespace b200 {\n\n"]
    out.append("// C emulations of the PTX instruction lists below (same order, explicit carry flag `cc`).  Results in [0, 2p).\n")
    out += emit_c("fp_mul_emul_core", mul_ops, mul_regs, mul_res, True)
    out += emit_c("fp_sqr_emul_core", sqr_ops, sqr_regs, sqr_res, False)
    out.append("#if defined(__CUDA_ARCH__)\n// r = a*b/R mod p and r = a*a/R mod p, results in [0, 2p); inputs < p.\n")
    out += emit_ptx("fp_mul_ptx_core", mul_ops, mul_regs, mul_res, True)
    out += emit_ptx("fp_sqr_ptx_core", sqr_ops, sqr_regs, sqr_res, False)
    out.append("#endif\n\n}  // namespace b200\n")
    path = Path(__file__).resolve().parent.parent / "ethereum_consensus_b200" / "csrc" / "fp_mul_ptx.cuh"
    path.write_text("".join(out))
    wide = lambda ops: sum(1 for o in ops if o[0] in ("mul.lo", "mad.lo.cc", "madc.lo.cc") and o[3] != "n0")  # noqa: E731
    print("wrote", path, "mul ops:", len(mul_ops), "wide:", wide(mul_ops), "| sqr ops:", len(sqr_ops), "wide:", wide(sqr_ops))


if __name__ == "__main__":
    main()
