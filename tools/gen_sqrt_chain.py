"""Generates ethereum_consensus_b200/csrc/fpl_sqrt_chain.cuh and fpd_sqrt_chain.cuh: y = c^((p+1)/4) on the lazily
reduced field (fpl.cuh) and on the FP64 field (fpd.cuh) as a fixed addition chain, every temporary a named register
variable.

The chain is a sliding-window decomposition of the exponent over a small dictionary of odd powers, chosen with a
shortest-cover dynamic programme.  Besides the small odd powers the dictionary holds c^255: the exponent has runs of 33,
19 and 17 one-bits, which 8-bit windows cover with a quarter of the products of 4-bit windows.  The chain is checked with
Python big integers (evaluate()) before the header is written.  Run from the repo root:  python tools/gen_sqrt_chain.py
(`--check` compares with the committed headers instead of writing them).

An FpD element is 16 registers, so the FP64 chain keeps at most FPD_DICT_CAP odd powers: best_dictionary() picks the
cap-sized dictionary of the cheapest chain, a product weighted FPD_MUL_WEIGHT squarings (the FP64-pipe instructions of
fpd_mul_core over fpd_sqr_core in the sm_90a build).
"""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "ethereum_consensus_b200" / "csrc" / "fpl_sqrt_chain.cuh"
FPD_HEADER = ROOT / "ethereum_consensus_b200" / "csrc" / "fpd_sqrt_chain.cuh"

P = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
EXP = (P + 1) // 4
# odd powers of c kept for the windows, each built from earlier ones (build_dictionary)
DICT = (1, 3, 5, 7, 9, 11, 13, 15, 21, 255)
FPD_DICT_CAP = 5
FPD_MUL_WEIGHT = 1.25


def build_dictionary(dictionary):
    """[(v, j, a, b)]: c^v = (c^a)^(2^j) * c^b, a and b already built (2 stands for c^2)."""
    have, steps = {1, 2}, []
    for v in sorted(dictionary):
        if v in have:
            continue
        step = next(((v, 0, a, v - a) for a in sorted(have, reverse=True) if v - a in have), None)
        for j in range(1, 12):
            if step:
                break
            step = next(((v, j, a, v - (a << j)) for a in sorted(have) if a != 2 and (a << j) < v and v - (a << j) in have), None)
        assert step, f"cannot build c^{v} in one product"
        steps.append(step)
        have.add(v)
    return steps


def windows(e, dictionary):
    """Fewest windows covering the one-bits of e, each window a bit string starting and ending in 1 whose value is in
    the dictionary: [(value, shift)] from the top, shift = the squarings that follow the window's product."""
    bits = bin(e)[2:]
    n, wmax = len(bits), max(dictionary).bit_length()
    best, how = [0] + [None] * n, [None] * (n + 1)
    for i in range(1, n + 1):
        if bits[i - 1] == "0":
            best[i], how[i] = best[i - 1], 0
            continue
        for w in range(1, min(wmax, i) + 1):
            s = bits[i - w:i]
            if s[0] == "1" and int(s, 2) in dictionary and best[i - w] is not None and (best[i] is None or best[i - w] + 1 < best[i]):
                best[i], how[i] = best[i - w] + 1, w
    out, i = [], n
    while i > 0:
        if how[i] == 0:
            i -= 1
            continue
        out.append((int(bits[i - how[i]:i], 2), n - i))
        i -= how[i]
    return out[::-1]


def chain(e=EXP, dictionary=DICT):
    """The program: ("sqr", dst, src) / ("mul", dst, a, b) / ("sqr_n", var, k) on variables named x<v> (c^v) and acc."""
    prog = [("sqr", "x2", "x1")]
    for v, j, a, b in build_dictionary(dictionary):
        if j == 0:
            prog.append(("mul", f"x{v}", f"x{a}", f"x{b}"))
        else:
            prog += [("copy", f"x{v}", f"x{a}"), ("sqr_n", f"x{v}", j), ("mul", f"x{v}", f"x{v}", f"x{b}")]
    wins = windows(e, dictionary)
    prog.append(("copy", "acc", f"x{wins[0][0]}"))
    prev_shift = wins[0][1]
    for v, shift in wins[1:]:
        prog += [("sqr_n", "acc", prev_shift - shift), ("mul", "acc", "acc", f"x{v}")]
        prev_shift = shift
    if prev_shift:
        prog.append(("sqr_n", "acc", prev_shift))
    return prog


def evaluate(prog):
    """Exponent of c that the program leaves in acc."""
    val = {"x1": 1}
    for op in prog:
        if op[0] == "sqr":
            val[op[1]] = 2 * val[op[2]]
        elif op[0] == "copy":
            val[op[1]] = val[op[2]]
        elif op[0] == "sqr_n":
            val[op[1]] <<= op[2]
        else:
            val[op[1]] = val[op[2]] + val[op[3]]
    return val["acc"]


def cost(prog):
    """(squarings, products)"""
    s = sum(1 for op in prog if op[0] == "sqr") + sum(op[2] for op in prog if op[0] == "sqr_n")
    return s, sum(1 for op in prog if op[0] == "mul")


def best_dictionary(cap, mul_weight, e=EXP):
    """The dictionary of at most `cap` odd powers (c^1 among them) whose chain costs least, squarings + mul_weight x
    products; ties go to the first in lexicographic order."""
    from itertools import combinations
    best = None
    candidates = [v for v in range(3, 256, 2)
                  if v < 32 or v in (63, 127, 255)]
    for n in range(cap):
        for rest in combinations(candidates, n):
            d = (1,) + rest
            try:
                prog = chain(e, d)
            except AssertionError:
                continue
            s, m = cost(prog)
            c = s + mul_weight * m
            if best is None or c < best[0]:
                best = (c, d)
    return best[1]


def render(prog, dictionary=DICT):
    s, m = cost(prog)
    names = sorted({op[1] for op in prog if op[1] not in ("x1", "acc")}, key=lambda v: int(v[1:]))
    body = []
    for op in prog:
        if op[0] == "sqr":
            body.append(f"    f_sqr({op[1]}, {op[2]});")
        elif op[0] == "copy":
            body.append(f"    {op[1]} = {op[2]};")
        elif op[0] == "sqr_n":
            body.append(f"    fpl_sqr_n({op[1]}, {op[2]});")
        else:
            body.append(f"    f_mul({op[1]}, {op[2]}, {op[3]});")
    return (
        "// GENERATED by tools/gen_sqrt_chain.py — do not edit.  Included from fpl.cuh.\n"
        f"// r = a^((p+1)/4) by a fixed addition chain: {s} squarings + {m} products, windows over c^{{{', '.join(map(str, dictionary))}}}.\n"
        "#pragma once\n\n"
        "namespace b200 {\n\n"
        "B200_BIG void fpl_sqrt_chain(FpL& r, const FpL& x1) {\n"
        f"    FpL {', '.join(names)}, acc;\n"
        + "\n".join(body) + "\n"
        "    r = acc;\n"
        "}\n\n"
        "}  // namespace b200\n")


def render_fpd(prog, dictionary):
    """The same program on FpD (fpd.cuh): products and squaring runs are calls there."""
    text = render(prog, dictionary)
    for a, b in (("Included from fpl.cuh", "Included from fpd.cuh"), ("fpl_sqrt_chain(FpL& r, const FpL& x1)",
                 "fpd_sqrt_chain(FpD& r, const FpD& x1)"), ("    FpL ", "    FpD "), ("f_sqr(", "fpd_sqr("),
                 ("f_mul(", "fpd_mul("), ("fpl_sqr_n(", "fpd_sqr_n(")):
        text = text.replace(a, b)
    return text


def main(argv):
    fpd_dict = best_dictionary(FPD_DICT_CAP, FPD_MUL_WEIGHT)
    for path, dictionary, rend in ((HEADER, DICT, render), (FPD_HEADER, fpd_dict, render_fpd)):
        prog = chain(EXP, dictionary)
        assert evaluate(prog) == EXP, "the chain does not evaluate to (p+1)/4"
        text = rend(prog, dictionary)
        if "--check" in argv:
            assert path.read_text() == text, f"{path.name} differs from what tools/gen_sqrt_chain.py generates"
            continue
        path.write_text(text)
        print(f"wrote {path.name}: {cost(prog)[0]} squarings + {cost(prog)[1]} products over c^{dictionary}")


if __name__ == "__main__":
    main(sys.argv[1:])
