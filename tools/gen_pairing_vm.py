"""Generates ethereum_consensus_b200/csrc/pairing_vm_prog.cuh: static Fp2-level programs for the Miller loop and the
final exponentiation, list-scheduled into rounds of <= TEAM independent operations, for the lane-parallel "Fp2 VM"
kernels (csrc/pairing_vm.cuh).  One tuple is handled by a TEAM of lanes; every lane executes one Fp2 operation per
round on a shared-memory register file, rounds are separated by __syncwarp().

Why: with one thread per pair / per tuple the pairing kernels expose only T..2T threads (T = 4096) — a latency
floor that no amount of per-thread tuning removes.  The Miller loop and the final exponentiation have no
data-dependent control flow, so they can be *traced once* (symbolic Fp2 values below, mirroring pairing.cuh /
fp12.cuh formula by formula) and replayed with 8-18 way parallelism.

The same formulas run here in two modes: `Sym` (records instructions) and `Num` (big-int arithmetic, from the
oracle's field helpers — generator-time self-check only): the scheduled + register-allocated program is executed
numerically and must reproduce the direct evaluation bit for bit before the header is written.
"""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from oracle import bls_oracle as bo  # noqa: E402  (generator-time checks only)

P = bo.P
Z_ABS = bo.Z_ABS

HEAVY_MIN = 1       # with MIX_LIGHT: a heavy round needs this many ready ops of its class while light ops are also ready (--heavy-min)
MIX_LIGHT = False  # True: ready light ops ride in the idle lanes of heavy rounds (measured offline: halves the rounds but doubles the rounds that pay for a product - a loss)

# opcodes (must match pairing_vm.cuh)
NOP, MUL, SQR, MULFP, INV, ADD, SUB, NEG, DBL, CONJ, MULXI, COPY, LDC = range(13)
HEAVY = {MUL: "mul", SQR: "sqr", MULFP: "mulfp", INV: "inv"}
OPNAME = {MUL: "MUL", SQR: "SQR", MULFP: "MULFP", INV: "INV", ADD: "ADD", SUB: "SUB", NEG: "NEG", DBL: "DBL", CONJ: "CONJ",
          MULXI: "MULXI", COPY: "COPY", LDC: "LDC"}


# ------------------------------------------------------------------------------------------------ value classes
class Tracer:
    def __init__(self):
        self.ins = []          # (op, dst_id, a_id, b_id)
        self.n = 0
        self.inputs = []       # value ids that are program inputs
        self.consts = {}       # const index -> value id

    def new(self):
        self.n += 1
        return self.n - 1

    def input(self):
        v = Sym(self, self.new())
        self.inputs.append(v.id)
        return v

    def const(self, idx):
        if idx not in self.consts:
            v = self.new()
            self.ins.append((LDC, v, idx, 0))
            self.consts[idx] = v
        return Sym(self, self.consts[idx])

    def op(self, code, a, b=None):
        v = self.new()
        self.ins.append((code, v, a.id, b.id if b is not None else a.id))
        return Sym(self, v)


class Sym:
    def __init__(self, tr, vid): self.tr, self.id = tr, vid
    def mul(self, o): return self.tr.op(MUL, self, o)
    def sqr(self): return self.tr.op(SQR, self)
    def mulfp(self, k): return self.tr.op(MULFP, self, k)   # multiply both coefficients by k.c0
    def inv(self): return self.tr.op(INV, self)
    def add(self, o): return self.tr.op(ADD, self, o)
    def sub(self, o): return self.tr.op(SUB, self, o)
    def neg(self): return self.tr.op(NEG, self)
    def dbl(self): return self.tr.op(DBL, self)
    def conj(self): return self.tr.op(CONJ, self)
    def mulxi(self): return self.tr.op(MULXI, self)


class Num:
    def __init__(self, v): self.v = (v[0] % P, v[1] % P)
    def mul(self, o): return Num(bo.f2_mul(self.v, o.v))
    def sqr(self): return Num(bo.f2_sqr(self.v))
    def mulfp(self, k): return Num(bo.f2_muli(self.v, k.v[0]))
    def inv(self): return Num(bo.f2_inv(self.v))
    def add(self, o): return Num(bo.f2_add(self.v, o.v))
    def sub(self, o): return Num(bo.f2_sub(self.v, o.v))
    def neg(self): return Num(bo.f2_neg(self.v))
    def dbl(self): return Num(bo.f2_add(self.v, self.v))
    def conj(self): return Num((self.v[0], -self.v[1]))
    def mulxi(self): return Num((self.v[0] - self.v[1], self.v[0] + self.v[1]))


# constant table (index -> Fp2 value); index 0 = one
XI = (1, 1)
CONSTS = [(1, 0)]
FROB = {}
for k in (1, 2):
    for i in range(1, 6):
        FROB[(k, i)] = len(CONSTS)
        CONSTS.append(bo.f2_pow(XI, i * (P ** k - 1) // 6))


class Ctx:
    """Supplies constants in the active mode."""
    def __init__(self, tracer=None): self.tr = tracer
    def const(self, idx): return self.tr.const(idx) if self.tr else Num(CONSTS[idx])


# ------------------------------------------------------------------------------------------------ tower formulas (mirror fp12.cuh)
def f6_add(a, b): return tuple(x.add(y) for x, y in zip(a, b))
def f6_sub(a, b): return tuple(x.sub(y) for x, y in zip(a, b))
def f6_neg(a): return tuple(x.neg() for x in a)
def f6_dbl(a): return tuple(x.dbl() for x in a)
def f6_mul_v(a): return (a[2].mulxi(), a[0], a[1])


def f6_mul(a, b):
    v0, v1, v2 = a[0].mul(b[0]), a[1].mul(b[1]), a[2].mul(b[2])
    x0 = a[1].add(a[2]).mul(b[1].add(b[2])).sub(v1).sub(v2).mulxi().add(v0)
    x1 = a[0].add(a[1]).mul(b[0].add(b[1])).sub(v0).sub(v1).add(v2.mulxi())
    x2 = a[0].add(a[2]).mul(b[0].add(b[2])).sub(v0).sub(v2).add(v1)
    return (x0, x1, x2)


def f6_mul_by_01(a, b0, b1):
    v0, v1 = a[0].mul(b0), a[1].mul(b1)
    x0 = a[1].add(a[2]).mul(b1).sub(v1).mulxi().add(v0)
    x1 = a[0].add(a[1]).mul(b0.add(b1)).sub(v0).sub(v1)
    x2 = a[0].add(a[2]).mul(b0).sub(v0).add(v1)
    return (x0, x1, x2)


def f6_mul_by_1(a, b1): return (a[2].mul(b1).mulxi(), a[0].mul(b1), a[1].mul(b1))


def f6_inv(a):
    c0 = a[0].sqr().sub(a[1].mul(a[2]).mulxi())
    c1 = a[2].sqr().mulxi().sub(a[0].mul(a[1]))
    c2 = a[1].sqr().sub(a[0].mul(a[2]))
    d = a[2].mul(c1).add(a[1].mul(c2)).mulxi().add(a[0].mul(c0)).inv()
    return (c0.mul(d), c1.mul(d), c2.mul(d))


def f12_mul(a, b):
    v0, v1 = f6_mul(a[0], b[0]), f6_mul(a[1], b[1])
    x1 = f6_sub(f6_sub(f6_mul(f6_add(a[0], a[1]), f6_add(b[0], b[1])), v0), v1)
    return (f6_add(v0, f6_mul_v(v1)), x1)


def f12_sqr(a):
    ab = f6_mul(a[0], a[1])
    x0 = f6_sub(f6_sub(f6_mul(f6_add(a[0], a[1]), f6_add(f6_mul_v(a[1]), a[0])), ab), f6_mul_v(ab))
    return (x0, f6_dbl(ab))


def f12_mul_by_line(f, A, B, C):
    v0 = f6_mul_by_01(f[0], A, B)
    v1 = f6_mul_by_1(f[1], C)
    x1 = f6_sub(f6_sub(f6_mul_by_01(f6_add(f[0], f[1]), A, B.add(C)), v0), v1)
    return (f6_add(v0, f6_mul_v(v1)), x1)


def f12_conj(a): return (a[0], f6_neg(a[1]))


def f12_inv(a):
    t0 = f6_sub(f6_mul(a[0], a[0]), f6_mul_v(f6_mul(a[1], a[1])))
    t0 = f6_inv(t0)
    return (f6_mul(a[0], t0), f6_neg(f6_mul(a[1], t0)))


def f12_frob(cx, a, k):
    slots = [a[0][0], a[1][0], a[0][1], a[1][1], a[0][2], a[1][2]]   # w-power index 0..5
    out = []
    for i, s in enumerate(slots):
        t = s.conj() if k & 1 else s
        out.append(t if i == 0 else t.mul(cx.const(FROB[(k, i)])))
    return ((out[0], out[2], out[4]), (out[1], out[3], out[5]))


def fp4_sqr(a, b):
    t0, t1 = a.sqr(), b.sqr()
    c0 = t1.mulxi().add(t0)
    c1 = a.add(b).sqr().sub(t0).sub(t1)
    return c0, c1


def f12_cyclo_sqr(f):
    z0, z4, z3, z2, z1, z5 = f[0][0], f[0][1], f[0][2], f[1][0], f[1][1], f[1][2]
    t0, t1 = fp4_sqr(z0, z1)
    z0 = t0.sub(z0).dbl().add(t0)
    z1 = t1.add(z1).dbl().add(t1)
    t0, t1 = fp4_sqr(z2, z3)
    t2, t3 = fp4_sqr(z4, z5)
    z4 = t0.sub(z4).dbl().add(t0)
    z5 = t1.add(z5).dbl().add(t1)
    t0 = t3.mulxi()
    z2 = t0.add(z2).dbl().add(t0)
    z3 = t2.sub(z3).dbl().add(t2)
    return ((z0, z4, z3), (z2, z1, z5))


def f12_pow_z(g):
    acc = g
    for bit in range(62, -1, -1):
        acc = f12_cyclo_sqr(acc)
        if (Z_ABS >> bit) & 1:
            acc = f12_mul(acc, g)
    return acc


# ------------------------------------------------------------------------------------------------ pairing formulas (mirror pairing.cuh / curve.cuh)
def jac_double(t):
    X, Y, Zc = t
    A, B = X.sqr(), Y.sqr()
    C = B.sqr()
    D = X.add(B).sqr().sub(A).sub(C).dbl()
    E = A.dbl().add(A)
    F = E.sqr()
    z3 = Y.mul(Zc).dbl()
    x3 = F.sub(D.dbl())
    y3 = E.mul(D.sub(x3)).sub(C.dbl().dbl().dbl())
    return (x3, y3, z3)


def miller_double_step(t, xp, yp, z3p):
    """P enters as (xp, yp, z3p) = (X Z, Y, Z^3) of a Jacobian G1 point: the line is scaled by Z^3 in Fp (killed by the
    final exponentiation), which saves the per-tuple inversion of the aggregate key; affine P: (x, y, 1)."""
    xx, yy, zz = t[0].sqr(), t[1].sqr(), t[2].sqr()
    e = xx.dbl().add(xx)
    A = e.mul(t[0]).sub(yy.dbl()).mulfp(z3p)
    B = e.mul(zz).mulfp(xp).neg()
    t2 = jac_double(t)
    C = t2[2].mul(zz).mulfp(yp)
    return t2, A, B, C


def miller_add_step(t, q, xp, yp, z3p):
    zz = t[2].sqr()
    zzz = zz.mul(t[2])
    h = q[0].mul(zz).sub(t[0])
    rr = q[1].mul(zzz).sub(t[1])
    z3 = t[2].mul(h)
    A = rr.mul(q[0]).sub(q[1].mul(z3)).mulfp(z3p)
    B = rr.mulfp(xp).neg()
    C = z3.mulfp(yp)
    hh = h.sqr()
    hhh = hh.mul(h)
    v = t[0].mul(hh)
    x3 = rr.sqr().sub(hhh).sub(v.dbl())
    y3 = rr.mul(v.sub(x3)).sub(t[1].mul(hhh))
    return (x3, y3, z3), A, B, C


def miller_loop(cx, xp, yp, z3p, qx, qy):
    """f_{z,Q}(P), P, Q not at infinity (the kernels bypass the program for infinite points)."""
    one = cx.const(0)
    t = (qx, qy, one)
    q = (qx, qy)
    f = None
    for bit in range(62, -1, -1):
        t, A, B, C = miller_double_step(t, xp, yp, z3p)
        if f is None:                      # first iteration: f = 1 * line
            zero_free = True
            f = ((A, B, None), (None, C, None))
        else:
            f = f12_mul_by_line(f12_sqr(f), A, B, C)
        if f[0][2] is None:                # materialise the sparse first value as a dense element lazily
            f = _densify(cx, f)
        if (Z_ABS >> bit) & 1:
            t, A, B, C = miller_add_step(t, q, xp, yp, z3p)
            f = f12_mul_by_line(f, A, B, C)
    return f12_conj(f)


def _densify(cx, f):
    one = cx.const(0)
    zero = one.sub(one)
    g = lambda x: x if x is not None else zero  # noqa: E731
    return ((g(f[0][0]), g(f[0][1]), g(f[0][2])), (g(f[1][0]), g(f[1][1]), g(f[1][2])))


def final_exp(cx, f1, f2):
    """(f1*f2)^(3 (p^12-1)/r): the value the kernel compares with one."""
    fin = f12_mul(f1, f2)
    t0 = f12_inv(fin)
    t1 = f12_conj(fin)
    t0 = f12_mul(t1, t0)
    t1 = f12_frob(cx, t0, 2)
    f = f12_mul(t1, t0)
    t0 = f12_conj(f12_mul(f12_pow_z(f), f))
    a = f12_conj(f12_mul(f12_pow_z(t0), t0))
    t0 = f12_conj(f12_pow_z(a))
    b = f12_mul(t0, f12_frob(cx, a, 1))
    t0 = f12_pow_z(f12_pow_z(b))
    c = f12_mul(f12_mul(t0, f12_frob(cx, b, 2)), f12_conj(b))
    return f12_mul(c, f12_mul(f12_sqr(f), f))


# ------------------------------------------------------------------------------------------------ schedule + allocate
def schedule(tr, outputs, team, window=None):
    ins = tr.ins
    producer = {d: i for i, (_, d, _, _) in enumerate(ins)}
    # dead-code elimination from the outputs
    need, stack = set(), [producer[o] for o in outputs if o in producer]
    while stack:
        i = stack.pop()
        if i in need:
            continue
        need.add(i)
        op, d, a, b = ins[i]
        if op != LDC:
            for s in (a, b):
                if s in producer:
                    stack.append(producer[s])
    idx = sorted(need)
    deps = {}
    users = {i: [] for i in idx}
    for i in idx:
        op, d, a, b = ins[i]
        ds = set()
        if op != LDC:
            for s in (a, b):
                if s in producer:
                    ds.add(producer[s])
        deps[i] = ds
        for j in ds:
            users[j].append(i)
    cost = lambda op: {MUL: 3, SQR: 2, MULFP: 2, INV: 600}.get(op, 0.05)  # noqa: E731
    prio = {}
    for i in reversed(idx):
        prio[i] = cost(ins[i][0]) + max((prio[u] for u in users[i]), default=0)
    remaining = {i: len(deps[i]) for i in idx}
    ready = [i for i in idx if remaining[i] == 0]
    rounds = []
    done_round = {}
    pos = {i: k for k, i in enumerate(idx)}          # program order
    unscheduled = set(idx)
    import heapq
    order_heap = list(idx)
    heapq.heapify(order_heap)
    while ready:
        # sliding window over program order: bounds how far ahead of the oldest pending instruction we run,
        # which bounds live ranges (register-file slots = shared memory per team = occupancy)
        while order_heap and order_heap[0] not in unscheduled:
            heapq.heappop(order_heap)
        oldest = pos[order_heap[0]] if order_heap else 0
        cand = [i for i in ready if window is None or pos[i] - oldest < window]
        if not cand:
            cand = [min(ready, key=lambda i: pos[i])]
        classes = {}
        for i in cand:
            op = ins[i][0]
            cl = HEAVY.get(op, "light")
            classes.setdefault(cl, []).append(i)
        heavy_classes = [c for c in classes if c != "light"]
        full_enough = [c for c in heavy_classes if len(classes[c]) >= min(HEAVY_MIN, team) or "light" not in classes]
        if MIX_LIGHT and full_enough:
            # a heavy round whenever one is possible (and full enough); lanes the heavy class leaves idle carry ready light
            # ops (they diverge from the product code, but a light op is a few % of a product and would otherwise cost a round)
            cl = max(full_enough, key=lambda c: max(prio[i] for i in classes[c]))
            pick = sorted(classes[cl], key=lambda i: -prio[i])[:team]
            if len(pick) < team and "light" in classes:
                pick += sorted(classes["light"], key=lambda i: -prio[i])[:team - len(pick)]
        else:
            # light ops are nearly free: flush them first so heavy rounds see the widest ready set
            if "light" in classes:
                cl = "light"
            else:
                cl = max(classes, key=lambda c: max(prio[i] for i in classes[c]))
            pick = sorted(classes[cl], key=lambda i: -prio[i])[:team]
        r = len(rounds)
        rounds.append(pick)
        for i in pick:
            ready.remove(i)
            unscheduled.discard(i)
            done_round[i] = r
        for i in pick:
            for u in users[i]:
                remaining[u] -= 1
                if remaining[u] == 0:
                    ready.append(u)
    # ---- slot allocation (a slot freed by its last reader in round r is reusable from round r + 1)
    last_use = {}
    for i in idx:
        op, d, a, b = ins[i]
        if op != LDC:
            for s in (a, b):
                last_use[s] = max(last_use.get(s, -1), done_round[i])
    for o in outputs:
        last_use[o] = len(rounds) + 1
    slot = {}
    nslots = 0
    free = []
    for v in tr.inputs:                      # inputs occupy the first slots, in declaration order
        slot[v] = nslots; nslots += 1
    release = {}                             # round -> slots to release after it
    for v in tr.inputs:
        if v in last_use:
            release.setdefault(last_use[v], []).append(slot[v])
    out_rounds = []
    for r, pick in enumerate(rounds):
        row = []
        for i in pick:
            op, d, a, b = ins[i]
            if free:
                s = free.pop()
            else:
                s = nslots; nslots += 1
            slot[d] = s
            lu = last_use.get(d, r)
            release.setdefault(lu, []).append(s)
            if op == LDC:
                row.append((op, s, a, 0))
            else:
                row.append((op, s, slot[a], slot[b]))
        out_rounds.append(row)
        free.extend(release.pop(r, []))
    return out_rounds, slot, nslots


def run_program(rounds, nslots, inputs):
    rf = [None] * nslots
    for k, v in enumerate(inputs):
        rf[k] = Num(v)
    for row in rounds:
        res = []
        for op, d, a, b in row:
            if op == LDC: res.append((d, Num(CONSTS[a])))
            elif op == MUL: res.append((d, rf[a].mul(rf[b])))
            elif op == SQR: res.append((d, rf[a].sqr()))
            elif op == MULFP: res.append((d, rf[a].mulfp(rf[b])))
            elif op == INV: res.append((d, rf[a].inv()))
            elif op == ADD: res.append((d, rf[a].add(rf[b])))
            elif op == SUB: res.append((d, rf[a].sub(rf[b])))
            elif op == NEG: res.append((d, rf[a].neg()))
            elif op == DBL: res.append((d, rf[a].dbl()))
            elif op == CONJ: res.append((d, rf[a].conj()))
            elif op == MULXI: res.append((d, rf[a].mulxi()))
            else: raise ValueError(op)
        for d, v in res:                     # all lanes read before any lane of the round writes
            rf[d] = v
    return rf


def flat12(f): return [f[0][0], f[1][0], f[0][1], f[1][1], f[0][2], f[1][2]]


def build(team, window=None, window_final=None):
    # ---- Miller loop: inputs xP, yP (as Fp2 with c1 = 0), Qx, Qy
    tr = Tracer()
    cx = Ctx(tr)
    xp, yp, z3p, qx, qy = tr.input(), tr.input(), tr.input(), tr.input(), tr.input()
    f = miller_loop(cx, xp, yp, z3p, qx, qy)
    outs = [v.id for v in flat12(f)]
    m_rounds, m_slot, m_nslots = schedule(tr, outs, team, window)
    m_out = [m_slot[o] for o in outs]
    # ---- final exponentiation: inputs f1, f2 (w-power order)
    tr2 = Tracer()
    cx2 = Ctx(tr2)
    i1 = [tr2.input() for _ in range(6)]
    i2 = [tr2.input() for _ in range(6)]
    mk = lambda s: ((s[0], s[2], s[4]), (s[1], s[3], s[5]))  # noqa: E731
    c = final_exp(cx2, mk(i1), mk(i2))
    outs2 = [v.id for v in flat12(c)]
    f_rounds, f_slot, f_nslots = schedule(tr2, outs2, team, window_final if window_final is not None else window)
    f_out = [f_slot[o] for o in outs2]
    return (m_rounds, m_nslots, m_out), (f_rounds, f_nslots, f_out)


def selfcheck(team, miller, final):
    """Scheduled programs == direct numeric evaluation; and the whole thing is a correct pairing check."""
    (m_rounds, m_nslots, m_out), (f_rounds, f_nslots, f_out) = miller, final
    F1, F2 = bo.F1, bo.F2
    cxn = Ctx(None)
    def g1(k): return bo.pt_to_affine(F1, bo.pt_mul(F1, bo.pt_from_affine(F1, bo.G1_GEN), k))
    def g2(k): return bo.pt_to_affine(F2, bo.pt_mul(F2, bo.pt_from_affine(F2, bo.G2_GEN), k))
    def mill(pa, qa, z=1):
        # P handed over in Jacobian form (X, Y, Z) = (x z^2, y z^3, z): inputs (X Z, Y, Z^3)
        X, Y = pa[0] * z * z % P, pa[1] * z * z * z % P
        ins = [(X * z % P, 0), (Y, 0), (z * z * z % P, 0)]
        rf = run_program(m_rounds, m_nslots, ins + [qa[0], qa[1]])
        got = [rf[s].v for s in m_out]
        want = [x.v for x in flat12(miller_loop(cxn, Num(ins[0]), Num(ins[1]), Num(ins[2]), Num(qa[0]), Num(qa[1])))]
        assert got == want, "scheduled Miller program != direct evaluation"
        return got
    def fin(fa, fb):
        rf = run_program(f_rounds, f_nslots, fa + fb)
        got = [rf[s].v for s in f_out]
        mk = lambda s: ((Num(s[0]), Num(s[2]), Num(s[4])), (Num(s[1]), Num(s[3]), Num(s[5])))  # noqa: E731
        want = [x.v for x in flat12(final_exp(cxn, mk(fa), mk(fb)))]
        assert got == want, "scheduled final-exp program != direct evaluation"
        return got
    one = [(1, 0)] + [(0, 0)] * 5
    a, b = 0x1234567, 0x7654321
    assert fin(mill(g1(a), g2(b)), mill(g1(bo.R - a * b % bo.R), bo.G2_GEN)) == one, "bilinearity check failed"
    assert fin(mill(g1(a), g2(b), z=0xdeadbeefcafe), mill(g1(bo.R - a * b % bo.R), bo.G2_GEN, z=12345)) == one, "Jacobian-P scaling failed"
    assert fin(mill(g1(a), g2(b)), mill(g1(bo.R - a * b % bo.R + 1), bo.G2_GEN)) != one, "non-degeneracy check failed"


def emit(team, miller, final):
    sfx = "" if team == 8 else str(team)    # the team-8 header owns the unsuffixed names and the shared constant table
    out = ["// GENERATED by tools/gen_pairing_vm.py — do not edit.\n#pragma once\n#include <cstdint>\n\nnamespace b200 {\n\n"]
    out.append(f"constexpr int kVmTeam{sfx} = {team};\n")
    out.append("// instruction word: op | dst << 8 | a << 16 | b << 24 ; rounds are kVmTeam words each (NOP padded)\n")
    def dump(name, prog):
        rounds, nslots, outs = prog
        words = []
        heavy = 0
        for row in rounds:
            if row and any(o[0] in HEAVY for o in row):
                heavy += 1
            for k in range(team):
                if k < len(row):
                    op, d, a, b = row[k]
                    assert max(d, a, b) < 256
                    words.append(op | (d << 8) | (a << 16) | (b << 24))
                else:
                    words.append(NOP)
        out.append(f"constexpr int k{name}Rounds{sfx} = {len(rounds)};   // {heavy} heavy rounds\n")
        out.append(f"constexpr int k{name}Slots{sfx} = {nslots};\n")
        out.append(f"constexpr int k{name}Out{sfx}[6] = {{{', '.join(map(str, outs))}}};\n")
        out.append(f"static const uint32_t h_{name.lower()}_code{sfx}[{len(words)}] = {{\n")
        for i in range(0, len(words), 8):
            out.append("    " + ", ".join(f"0x{w:08x}u" for w in words[i:i + 8]) + ",\n")
        out.append("};\n\n")
    dump("Miller", miller)
    dump("Final", final)
    if team == 8:
        out.append(f"constexpr int kVmConsts = {len(CONSTS)};\n")
        out.append("// constant table in plain integers: 2 x 12 u32 little-endian limbs per Fp2 (converted to Montgomery form at load time)\n")
        out.append(f"static const uint32_t h_vm_consts[{len(CONSTS)}][24] = {{\n")
        for c in CONSTS:
            limbs = [(c[0] >> (32 * i)) & 0xffffffff for i in range(12)] + [(c[1] >> (32 * i)) & 0xffffffff for i in range(12)]
            out.append("    {" + ", ".join(f"0x{v:08x}u" for v in limbs) + "},\n")
        out.append("};\n\n")
    out.append("}  // namespace b200\n")
    path = ROOT / "ethereum_consensus_b200" / "csrc" / ("pairing_vm_prog.cuh" if team == 8 else f"pairing_vm_prog{team}.cuh")
    path.write_text("".join(out))
    return path


def write_blob(path, team, miller, final):
    """Run-time loadable form of one team size's programs (b200_vm_load_programs; layout in csrc/bls_vm.cu)."""
    import struct
    (m_rounds, m_nslots, m_out), (f_rounds, f_nslots, f_out) = miller, final
    def words(rounds):
        out = []
        for row in rounds:
            ws = [(op | (d << 8) | (a << 16) | (b << 24)) for op, d, a, b in row]
            out += ws + [NOP] * (team - len(ws))
        return out
    blob = [0xB200564D, team, len(m_rounds), m_nslots, *m_out, len(f_rounds), f_nslots, *f_out] + words(m_rounds) + words(f_rounds)
    Path(path).write_bytes(struct.pack(f"<{len(blob)}I", *blob))
    return path


def main():
    blob_path = None
    if "--blob" in sys.argv:
        i = sys.argv.index("--blob")
        blob_path = sys.argv[i + 1]
        del sys.argv[i:i + 2]
    global MIX_LIGHT, HEAVY_MIN
    if "--mix-light" in sys.argv:
        sys.argv.remove("--mix-light")
        MIX_LIGHT = True
    if "--heavy-min" in sys.argv:
        i = sys.argv.index("--heavy-min")
        HEAVY_MIN = int(sys.argv[i + 1])
        del sys.argv[i:i + 2]
    team = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    # scheduling windows (Miller, final): trade-off between heavy rounds and register-file slots;
    # defaults: team 16 -> (256, 48), team 8 -> (96, 96).  BOTH headers ship: teams of 8 lanes have the
    # higher throughput (big batches), teams of 16 the shorter critical path (batches too small to fill the machine):
    #   python tools/gen_pairing_vm.py 8 && python tools/gen_pairing_vm.py 16
    window = int(sys.argv[2]) if len(sys.argv) > 2 else (256 if team == 16 else 96)
    window_final = int(sys.argv[3]) if len(sys.argv) > 3 else (48 if team == 16 else 96)
    miller, final = build(team, window, window_final)
    for name, (rounds, nslots, _o) in (("miller", miller), ("final", final)):
        heavy = [r for r in rounds if r and any(o[0] in HEAVY for o in r)]
        util = sum(len(r) for r in heavy) / max(1, len(heavy) * team)
        import collections
        kinds = collections.Counter()
        for r in rounds:
            hv = sorted({HEAVY[o[0]] for o in r if o[0] in HEAVY})
            lt = len({o[0] for o in r if o[0] not in HEAVY})
            kinds[("+".join(hv) or "light") + (f"+{lt}L" if hv and lt else "")] += 1
        print(f"{name}: {len(rounds)} rounds ({len(heavy)} heavy, lane utilisation {util:.2f}), {nslots} slots, "
              f"{sum(len(r) for r in rounds)} instructions; round kinds {dict(kinds)}")
    selfcheck(team, miller, final)
    if blob_path:
        print("self-check ok; wrote", write_blob(blob_path, team, miller, final))
    else:
        print("self-check ok; wrote", emit(team, miller, final))


if __name__ == "__main__":
    main()
