"""Generated witness programs for the interpreter tests (tests/test_witness_programs_cpu.py on the host build of
csrc/witness_core.cuh, tests/test_gpu_witness_programs.py on both device kernels).

The programs are built directly as the `ops` / `lc_ptr` / `lc_slot` / `lc_coef` / `coefs` arrays of a
`WitnessProgram`, not through `compile_block`, so they reach what the circuit compiler never emits: more than 32
externals, no raws or no externals, LCs of 0 to 300 terms with repeated slots, `BIT` at every word boundary,
`INVZ` / `ISZERO` / `SELECT` on zero, `JJ` on the small-order, identity and off-curve points, one-op programs, a
2 000-level chain and levels of 32, 33, 64, 65 and 1 000 ops.  Every case has a fixed seed, and `rows(case, n)`
gives n slots different inputs (canonical ints).  `run_reference` (mpn/witness_program.py) is the ground truth.
Pure Python: no GPU, no compiled code."""
import random
from dataclasses import dataclass, field

import numpy as np

from bazuka_b200.mpn import native as N
from bazuka_b200.mpn import witness_program as W

R = N.R
ONE = W.SLOT_ONE
MONT = [(1 << 256) % R, (1 << 512) % R, pow(1 << 256, -1, R)]   # R, R^2 and R^-1 of the Montgomery form
EDGES = [0, 1, 2, R - 2, R - 1, (R - 1) // 2, (R + 1) // 2] + [1 << k for k in (31, 32, 63, 64, 127, 128, 223, 224, 253, 254)] + MONT
BIT_IMMS = [0, 31, 32, 63, 64, 127, 128, 223, 224, 254, 255]
COEFS = [1, R - 1, 2]
SQRT_M1 = N.fr_sqrt(R - 1)


def _points():
    """named JubJub points: valid ones from the generator, the identity, the small-order points, off-curve pairs."""
    p = N.jj_mul(N.JJ_BASE, 0x1234567)
    q = N.jj_mul(N.JJ_BASE, 0xfedcba98765)
    pts = {"P": p, "-P": ((R - p[0]) % R, p[1]), "Q": q, "2P": N.jj_add(p, p), "id": (0, 1), "ord2": (0, R - 1),
           "ord4+": (SQRT_M1, 0), "ord4-": (R - SQRT_M1, 0), "zero": (0, 0), "off": (p[0], (p[1] + 1) % R), "one-one": (1, 1)}
    assert all(N.jj_on_curve(v) != (k in ("zero", "off", "one-one")) for k, v in pts.items())
    return pts


POINTS = _points()
# a pool of valid points for the per-slot rows: P, P + B, P + 2B, ... (one addition each)
_POOL = [POINTS["P"]]
for _ in range(63):
    _POOL.append(N.jj_add(_POOL[-1], N.JJ_BASE))


class Builder:
    """a WitnessProgram assembled op by op.  Slots: 0 = ONE, 1..n_ext the externals, then one per op; every method
    that adds an op returns the slot it defines.  LC ids are returned by `lc` and are never deduplicated, so two
    distinct LCs may hold the same terms."""

    def __init__(self, n_ext=0, n_raw=0):
        self.n_ext, self.n_raw = n_ext, n_raw
        self.ops = []
        self.lc_ptr, self.lc_slot, self.lc_coef = [0], [], []
        self.coefs, self._ci = [1], {1: 0}

    @property
    def n_slots(self):
        return 1 + self.n_ext + len(self.ops)

    def ext(self, k):
        assert 0 <= k < self.n_ext
        return 1 + k

    def coef(self, c, fresh=False):
        """index of coefficient c; fresh=True adds another entry even when c is already there (1 at an index != 0
        is then multiplied in like any other coefficient)."""
        c %= R
        if fresh or c not in self._ci:
            self._ci.setdefault(c, len(self.coefs))
            self.coefs.append(c)
            return len(self.coefs) - 1
        return self._ci[c]

    def lc(self, *terms):
        """terms: slot, or (slot, coefficient), or (slot, coefficient, "fresh")"""
        for t in terms:
            s, c, fresh = (t, 1, False) if isinstance(t, int) else (t[0], t[1], len(t) > 2)
            assert 0 <= s < self.n_slots, "an LC may only read earlier variables"
            self.lc_slot.append(s)
            self.lc_coef.append(self.coef(c, fresh))
        self.lc_ptr.append(len(self.lc_slot))
        return len(self.lc_ptr) - 2

    def const(self, v):
        return self.lc((ONE, v))

    def _op(self, code, a0=0, a1=0, a2=0, a3=0, imm=0):
        self.ops.append((code, a0, a1, a2, a3, imm))
        return self.n_slots - 1

    def raw(self, imm):
        assert 0 <= imm < self.n_raw
        return self._op(W.OP_RAW, imm=imm)

    def mul(self, a, b):
        return self._op(W.OP_MUL, a, b)

    def bit(self, a, imm):
        return self._op(W.OP_BIT, a, imm=imm)

    def iszero(self, a):
        return self._op(W.OP_ISZERO, a)

    def invz(self, a):
        return self._op(W.OP_INVZ, a)

    def select(self, s, if_zero, if_nonzero):
        return self._op(W.OP_SELECT, s, if_zero, if_nonzero)

    def jj(self, x1, y1, x2, y2):
        x = self._op(W.OP_JJ, x1, y1, x2, y2)
        return x, self._op(W.OP_NOP)

    def build(self):
        i32 = lambda a: np.array(a, dtype=np.int32)
        ops = np.array(self.ops, dtype=np.int32).reshape(-1, 6)
        return W.WitnessProgram(0, 0, ops, i32(self.lc_ptr), i32(self.lc_slot), i32(self.lc_coef), list(self.coefs), self.n_raw, self.n_ext)


def levels(prog):
    """executed ops per level of the kernel's schedule (csrc/witness_core.cuh wit_build_schedule, restated): an op's
    level is 1 + the deepest of its operands; ONE and the externals are at depth 0; NOPs share their JJ's level."""
    depth = [0] * prog.n_slots
    width = {}
    ptr, slots = prog.lc_ptr.tolist(), prog.lc_slot.tolist()
    nlc = {W.OP_JJ: 4, W.OP_SELECT: 3, W.OP_MUL: 2, W.OP_BIT: 1, W.OP_ISZERO: 1, W.OP_INVZ: 1, W.OP_RAW: 0}
    for j, op in enumerate(prog.ops.tolist()):
        if op[0] == W.OP_NOP:
            continue
        d = 1 + max([depth[slots[k]] for a in range(nlc[op[0]]) for k in range(ptr[op[1 + a]], ptr[op[1 + a] + 1])], default=0)
        depth[prog.block0 + j] = d
        if op[0] == W.OP_JJ:
            depth[prog.block0 + j + 1] = d
        width[d] = width.get(d, 0) + 1
    return [width[d] for d in range(1, len(width) + 1)]


@dataclass
class Case:
    name: str
    seed: int
    prog: W.WitnessProgram
    row: callable          # (rng) -> (raws, ext) of one slot, canonical ints
    level_widths: list = field(default=None)   # the schedule the case was built to have, when it is about levels


def edge_or_random(rng):
    return rng.choice(EDGES) if rng.random() < 0.5 else rng.randrange(R)


def _plain_row(prog):
    return lambda rng: ([edge_or_random(rng) for _ in range(prog.n_raw)], [edge_or_random(rng) for _ in range(prog.n_ext)])


def rows(case, n, seed=None):
    """n slots of inputs for `case`, every slot different (seeded by the case unless `seed` is given)."""
    rng = random.Random(case.seed * 7919 + 17 if seed is None else seed)
    out, seen = [], set()
    while len(out) < n:
        raws, ext = case.row(rng)
        key = (tuple(raws), tuple(ext))
        if key in seen and (raws or ext):
            continue
        seen.add(key)
        out.append((raws, ext))
    return out


# ---------------------------------------------------------------------------------------------- the cases
def case_opcodes(seed=101):
    """every opcode on operands from the edge set, raws, externals and random constants; BIT at every word boundary;
    ISZERO / INVZ / SELECT on zero (an empty LC, and x - x); MUL by the same LC (the square path) and by a distinct LC
    of equal value."""
    rng = random.Random(seed)
    b = Builder(n_ext=3, n_raw=6)
    r = [b.raw(k) for k in range(6)]
    x, y, s = b.lc(r[0]), b.lc(r[1]), b.lc(r[2])
    empty = b.lc()
    cancel = b.lc(r[0], (r[0], R - 1))
    operands = [(r[k], None) for k in range(6)] + [(b.ext(k), None) for k in range(3)] + \
               [(None, v) for v in EDGES] + [(None, rng.randrange(R)) for _ in range(4)]
    for slot, v in operands:
        make = (lambda: b.lc(slot)) if slot is not None else (lambda: b.const(v))
        a = make()
        b.mul(a, a)
        b.mul(a, make())
        b.mul(a, y)
        for imm in BIT_IMMS:
            b.bit(a, imm)
        b.iszero(a)
        b.invz(a)
        b.select(a, x, y)
        b.select(s, a, y)
        b.select(s, x, a)
    for z in (empty, cancel):
        b.iszero(z)
        b.invz(z)
        b.select(z, x, y)
        b.select(x, z, y)
        b.select(y, x, z)
        b.mul(z, x)
        b.mul(z, z)
        b.bit(z, 0)
    prog = b.build()

    def row(rng):
        raws = [edge_or_random(rng) for _ in range(6)]
        if rng.random() < 0.4:
            raws[2] = 0                      # the selector
        if rng.random() < 0.2:
            raws[1] = raws[0]
        return raws, [edge_or_random(rng) for _ in range(3)]
    return Case("opcodes", seed, prog, row)


def case_linear_combinations(seed=102):
    """LCs of 0, 1, 9, 64 and 300 terms over ONE, externals, raws, earlier results and the y half of a JJ (a NOP slot),
    with coefficients 1, r-1, 2, a second entry holding 1, and random ones, and a slot repeated inside one LC."""
    rng = random.Random(seed)
    b = Builder(n_ext=33, n_raw=9)
    raws = [b.raw(k) for k in range(9)]
    p, q = POINTS["P"], POINTS["Q"]
    jx, jy = b.jj(b.const(p[0]), b.const(p[1]), b.const(q[0]), b.const(q[1]))
    prod = b.mul(b.lc(raws[0], (b.ext(32), 3)), b.lc(raws[1]))
    readable = [ONE] + [b.ext(k) for k in range(33)] + raws + [jx, jy, prod]
    coefs = COEFS + [rng.randrange(R) for _ in range(5)]
    one = b.lc(ONE)
    for size in (0, 1, 9, 64, 300):
        for rep in range(4):
            terms = []
            for t in range(size):
                c = rng.choice(coefs)
                terms.append((rng.choice(readable), c, "fresh") if c == 1 and rng.random() < 0.2 else (rng.choice(readable), c))
            if size >= 9:
                terms[1] = (terms[0][0], rng.choice(coefs))          # the same slot twice in one LC
                terms[2:6] = [(ONE, 2), (b.ext(rep), R - 1), (jy, 1), (b.ext(32 - rep), 1)]
            elif size == 1:
                terms = [[(jy, 1), (ONE, R - 1), (b.ext(31), 2), (raws[8], 1, "fresh")][rep]]
            a = b.lc(*terms)
            b.mul(a, one)
            b.mul(a, a)
            b.iszero(a)
            b.invz(a)
            b.bit(a, rng.choice(BIT_IMMS))
            b.select(a, b.lc(raws[2]), b.lc(raws[3]))
            readable.append(b.mul(a, b.lc(raws[4])))
    prog = b.build()
    return Case("linear_combinations", seed, prog, _plain_row(prog))


PAIR_KINDS = ("same", "neg", "other", "id", "ord2", "ord4", "off-first", "off-second", "zero")


def _point_pair(rng, kind):
    p = rng.choice(_POOL)
    if kind == "same":
        return p, p
    if kind == "neg":
        return p, ((R - p[0]) % R, p[1])
    if kind == "other":
        return p, rng.choice(_POOL)
    if kind == "id":
        return (p, (0, 1)) if rng.random() < 0.5 else ((0, 1), p)
    if kind == "ord2":
        return p, (0, R - 1)
    if kind == "ord4":
        return rng.choice([POINTS["ord4+"], POINTS["ord4-"]]), rng.choice([p, POINTS["ord4+"], POINTS["ord4-"], POINTS["ord2"]])
    if kind == "off-first":
        return (p[0], (p[1] + rng.randrange(1, R)) % R), p
    if kind == "off-second":
        return p, (rng.randrange(R), rng.randrange(R))
    return (0, 0), p


def case_jubjub(seed=103):
    """JJ on every ordered pair of the named points (valid, P+P, P+(-P), identity, order 2 and 4, off-curve on either
    side) as constants, and on per-slot points from the raws: two JJs in one level, JJs that read the y half of an
    earlier JJ, and JJ operands that are LCs of several terms."""
    b = Builder(n_ext=0, n_raw=8)
    r = [b.raw(k) for k in range(8)]
    c = lambda v: b.const(v)
    for u in POINTS.values():
        for v in POINTS.values():
            b.jj(c(u[0]), c(u[1]), c(v[0]), c(v[1]))
    # per-slot points: (r0,r1) + (r2,r3) and (r4,r5) + (r6,r7) in one level
    a12 = b.jj(b.lc(r[0]), b.lc(r[1]), b.lc(r[2]), b.lc(r[3]))
    a34 = b.jj(b.lc((r[4], 2), (r[4], R - 1)), b.lc(r[5]), b.lc(r[6]), b.lc((r[7], 1, "fresh")))
    s = b.jj(b.lc(a12[0]), b.lc(a12[1]), b.lc(a34[0]), b.lc(a34[1]))            # reads both y halves
    t = b.jj(b.lc(a12[0]), b.lc(a12[1]), b.lc(r[0]), b.lc(r[1]))
    u = b.jj(b.lc(s[0]), b.lc(s[1]), b.lc(s[0]), b.lc(s[1]))                    # doubling of a computed point
    b.jj(b.lc(u[0], (ONE, 0)), b.lc((u[1], R - 1)), b.lc(t[0]), b.lc(t[1]))      # (u.x, -u.y), on the curve as well, plus t
    b.mul(b.lc(s[1]), b.lc(ONE))
    b.iszero(b.lc(u[0]))
    b.select(b.lc(t[1], (ONE, R - 1)), b.lc(s[0]), b.lc(u[1]))

    def row(rng):
        (p1, p2), (p3, p4) = _point_pair(rng, rng.choice(PAIR_KINDS)), _point_pair(rng, rng.choice(PAIR_KINDS))
        return [p1[0], p1[1], p2[0], p2[1], p3[0], p3[1], p4[0], p4[1]], []
    return Case("jubjub", seed, b.build(), row)


def _random_lc(b, rng, pool, max_terms=6, must=None):
    n = rng.randrange(0, max_terms + 1)
    terms = [(rng.choice(pool), rng.choice(COEFS) if rng.random() < 0.7 else rng.randrange(R)) for _ in range(n)]
    if must is not None:
        terms.insert(rng.randrange(len(terms) + 1), (must, rng.choice(COEFS)))
    return b.lc(*terms)


def _random_op(b, rng, pool, must=None, points=(), new_points=None):
    """one op of a random opcode whose operands are random LCs over `pool`; `must` (a slot) is read by the first
    operand, which pins the op's level.  A JJ adds a pool point to one of `points` (slot pairs of valid points) more
    often than not, and its result goes to `new_points`.  Returns the slots the op defines."""
    code = rng.choice([W.OP_MUL, W.OP_MUL, W.OP_BIT, W.OP_ISZERO, W.OP_INVZ, W.OP_SELECT, W.OP_JJ])
    first = _random_lc(b, rng, pool, must=must)
    if code == W.OP_MUL:
        return [b.mul(first, first if rng.random() < 0.3 else _random_lc(b, rng, pool))]
    if code == W.OP_BIT:
        return [b.bit(first, rng.choice(BIT_IMMS) if rng.random() < 0.5 else rng.randrange(256))]
    if code == W.OP_ISZERO:
        return [b.iszero(first)]
    if code == W.OP_INVZ:
        return [b.invz(first)]
    if code == W.OP_SELECT:
        return [b.select(first, _random_lc(b, rng, pool), _random_lc(b, rng, pool))]
    if points and rng.random() < 0.7:
        (ax, ay), (px, py) = rng.choice(points), rng.choice(_POOL)
        # reads `must` with a zero coefficient: the same value, at the level `must` pins
        pt = [b.lc(ax) if must is None else b.lc(ax, (must, 0)), b.lc(ay), b.const(px), b.const(py)]
        out = b.jj(*pt) if rng.random() < 0.5 else b.jj(pt[2], pt[3], pt[0], pt[1])
        new_points.append(out)
        return list(out)
    return list(b.jj(first, _random_lc(b, rng, pool), _random_lc(b, rng, pool), _random_lc(b, rng, pool)))


def _const_jj(b):
    p, q = POINTS["P"], POINTS["Q"]
    return b.jj(b.const(p[0]), b.const(p[1]), b.const(q[0]), b.const(q[1]))


def _layered(b, rng, widths, base, points):
    """levels of exactly the given widths after the ops of `base` (one level): every op of level L reads a variable of
    level L-1 and anything earlier."""
    prev, pool, points = list(base), [ONE] + [b.ext(k) for k in range(b.n_ext)] + list(base), list(points)
    for w in widths:
        cur, new_points = [], []
        for _ in range(w):
            cur += _random_op(b, rng, pool, must=rng.choice(prev), points=points, new_points=new_points)
        points = (new_points + points)[:16]
        pool += cur
        prev = cur
    return b


def case_chain(seed=104):
    """2 000 levels of one op each: op j reads op j-1 (and ONE, an external or a constant)."""
    rng = random.Random(seed)
    b = Builder(n_ext=1, n_raw=1)
    prev = b.raw(0)
    p = POINTS["P"]
    n_exec = 1
    while n_exec < 2000:
        kind = n_exec % 11
        if kind == 10:
            # off-curve unless prev + 1 happens to be a valid x: mostly (0, 0); the next op reads the y half
            _, prev = b.jj(b.lc(prev, (ONE, 1)), b.lc(ONE), b.const(p[0]), b.const(p[1]))
        elif kind in (0, 4, 7):
            prev = b.mul(b.lc(prev, (ONE, rng.randrange(R))), b.lc((b.ext(0), 1), (prev, 2)))
        elif kind in (1, 8):
            prev = b.invz(b.lc(prev, (ONE, rng.choice(EDGES))))
        elif kind == 2:
            prev = b.bit(b.lc(prev, (ONE, rng.randrange(R))), rng.choice(BIT_IMMS))
        elif kind == 3:
            prev = b.select(b.lc(prev), b.lc(b.ext(0)), b.lc((prev, R - 1), (ONE, 5)))
        elif kind == 5:
            prev = b.iszero(b.lc(prev, (ONE, R - 1)))
        elif kind == 6:
            a = b.lc(prev, (ONE, 1))
            prev = b.mul(a, a)
        else:
            prev = b.select(b.lc((prev, 2)), b.lc(prev), b.lc(b.ext(0), (prev, 3)))
        n_exec += 1
    prog = b.build()
    return Case("chain_2000", seed, prog, _plain_row(prog), [1] * 2000)


def case_wide_levels(seed=105):
    """levels of exactly 32, 33, 64, 65 and 1 000 ops (the lanes' `i += 32` loop at and around its boundaries)."""
    rng = random.Random(seed)
    b = Builder(n_ext=2, n_raw=30)
    pq = _const_jj(b)
    base = [b.raw(k) for k in range(30)] + [b.mul(b.lc(b.ext(0)), b.lc(b.ext(1))), *pq]
    widths = [33, 64, 65, 1000]
    _layered(b, rng, widths, base, [pq])
    prog = b.build()
    return Case("wide_levels", seed, prog, _plain_row(prog), [32] + widths)


def case_mixed_levels(seed=106):
    """narrow and wide levels alternating: 1, 33, 1, 65, 2, 32, 64, 1, 5, 100, ten times over."""
    rng = random.Random(seed)
    b = Builder(n_ext=4, n_raw=3)
    pq = _const_jj(b)
    base = [b.raw(k) for k in range(3)] + list(pq)
    widths = [1, 33, 1, 65, 2, 32, 64, 1, 5, 100] * 10
    _layered(b, rng, widths, base, [pq])
    prog = b.build()
    return Case("mixed_levels", seed, prog, _plain_row(prog), [4] + widths)


def case_shape(n_ext, n_raw, n_ops=160, seed=None):
    """a random program of about n_ops ops over n_ext externals and n_raw raws, reading every one of them."""
    seed = seed if seed is not None else 1000 + 100 * n_ext + n_raw
    rng = random.Random(seed)
    b = Builder(n_ext=n_ext, n_raw=n_raw)
    pool = [ONE] + [b.ext(k) for k in range(n_ext)]
    order = list(range(n_raw)) + [rng.randrange(n_raw) for _ in range(min(n_raw, 3))]
    rng.shuffle(order)
    pool += [b.raw(k) for k in order]
    if n_ext:
        # every external, each with its own coefficient: a lane that skips one changes this sum
        s = b.lc(*[(b.ext(k), rng.randrange(1, R)) for k in range(n_ext)])
        pool.append(b.mul(s, s))
        pool.append(b.mul(b.lc(b.ext(n_ext - 1)), b.lc(ONE)))
    points = [_const_jj(b)]
    pool += list(points[0])
    while len(b.ops) < n_ops:
        pool += _random_op(b, rng, pool, points=points, new_points=points)
    prog = b.build()
    return Case(f"shape_e{n_ext}_r{n_raw}", seed, prog, _plain_row(prog))


def case_single_raw(seed=107):
    b = Builder(n_ext=0, n_raw=1)
    b.raw(0)
    prog = b.build()
    return Case("single_raw", seed, prog, _plain_row(prog), [1])


def case_single_op(seed=108):
    b = Builder(n_ext=1, n_raw=0)
    b.invz(b.lc((b.ext(0), 2), (ONE, R - 1)))
    prog = b.build()
    return Case("single_op", seed, prog, _plain_row(prog), [1])


def case_single_op_no_inputs(seed=109):
    b = Builder(n_ext=0, n_raw=0)
    b.iszero(b.lc())
    prog = b.build()
    return Case("single_op_no_inputs", seed, prog, lambda rng: ([], []), [1])


SHAPES = [(e, r) for e in (0, 1, 31, 32, 33, 70) for r in (0, 1, 77)]


def all_cases():
    """every named case, in a fixed order"""
    out = [case_opcodes(), case_linear_combinations(), case_jubjub(), case_chain(), case_wide_levels(), case_mixed_levels(),
           case_single_raw(), case_single_op(), case_single_op_no_inputs()]
    out += [case_shape(e, r) for e, r in SHAPES]
    return out
