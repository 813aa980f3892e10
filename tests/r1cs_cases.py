"""Seeded families of small constraint systems at the edges of the Groth16 driver's bookkeeping (csrc/groth16.cu, the
density lists of csrc/r1cs_blocked.cuh, setup_gpu), shared by test_r1cs_cases_cpu.py and test_gpu_r1cs_cases.py.

Every case carries its rows as `oracle.py.groth16.R1CS`, a witness z (satisfying unless `bad` says how many rows it
breaks), its CSR triple, its blocked form (head-only when the shape has no repeated block), the shape
(log_m, |h|, |l|, |a|, |b|) it must upload to, and fixed toxic waste and (r, s).  Families:
  boundary    ncons + num_inputs in {2^k - 1, 2^k, 2^k + 1}, k = 0..7, num_inputs in {1, 2, 5}; plus 2^12 and 2^16
  degenerate  m = 1, no aux, an empty B side, a zero witness apart from ONE, r = 0 and s = 0
  density     variables missing from A / B / every side, inputs missing from B, stored zero coefficients, duplicate
              entries, cancelling duplicates (v, c), (v, -c)
  value       coefficients 1, r - 1, 2^64 - 1; witness entries 0, 1, r - 1; a 1100-term row; a variable in every row
  unsat       one bad row first, one last, two, every row
  blocked     repeated templates: reps 0 and 1, no template rows, no head, no tail, the last copy naming nv - 1
"""
import random

import numpy as np

from oracle.py import groth16 as G
from oracle.py.field import R_MOD as R

BIG_INT_MAX_LOG_M = 7          # the big-integer restatement is the arbiter up to this domain size


class Case:
    def __init__(self, name, family, ni, na, rows, z, seed, bad=0, blocked=None, expect=None, cancelling=(), rs=None):
        self.name, self.family, self.seed, self.bad = name, family, seed, bad
        self.cs = G.R1CS(ni, na)
        for a, b, c in rows:
            self.cs.enforce(a, b, c)
        self.z = [v % R for v in z]
        assert len(self.z) == ni + na and self.z[0] == 1
        # blocked: (head, tmpl, reps, tail, var_lo, stride, stored rows head | template | tail); default: every row in the head
        self.blocked = blocked or (len(rows), 0, 0, 0, ni + na, 0, list(rows))
        self.expect = expect if expect is not None else presence_shape(ni, na, rows)
        self.cancelling = tuple(cancelling)    # variables whose only terms cancel: an identity column in the key
        g = random.Random(f"toxic-{seed}")
        self.toxic = [g.randrange(1, R) for _ in range(5)]
        self.r, self.s = rs if rs is not None else (g.randrange(R), g.randrange(R))

    ni = property(lambda self: self.cs.num_inputs)
    na = property(lambda self: self.cs.num_aux)
    ncons = property(lambda self: len(self.cs.rows))
    log_m = property(lambda self: self.expect[0])
    big_int = property(lambda self: self.log_m <= BIG_INT_MAX_LOG_M)

    def __repr__(self):
        return self.name


def log2_ceil(n):
    e = 0
    while (1 << e) < n:
        e += 1
    return e


def presence_shape(ni, na, rows):
    """(log_m, |h|, |l|, |a|, |b|) by bellman's presence rule: a term is present when its coefficient is non-zero"""
    in_a = {v for a, _, _ in rows for v, c in a if c % R and v >= ni}
    in_b = {v for _, b, _ in rows for v, c in b if c % R}
    log_m = log2_ceil(len(rows) + ni)
    return log_m, (1 << log_m) - 1, na, ni + len(in_a), len(in_b)


def ev(lc, z):
    return sum(c * z[v] for v, c in lc) % R


def net_vars(rows, side):
    """the variables some row names on `side` with a non-zero net coefficient (duplicates summed): those whose column is
    non-zero at a random tau"""
    out = set()
    for row in rows:
        acc = {}
        for v, c in row[side]:
            acc[v] = (acc.get(v, 0) + c) % R
        out |= {v for v, c in acc.items() if c}
    return out


def bad_rows(case):
    return sum(1 for a, b, c in case.cs.rows if ev(a, case.z) * ev(b, case.z) % R != ev(c, case.z))


# ------------------------------------------------------------------ Montgomery images and CSR
def mont(xs):
    return np.array([list((((x % R) << 256) % R).to_bytes(32, "little")) for x in xs], dtype=np.uint8).view(np.uint64).reshape(-1, 4)


def csr(rows):
    mats = []
    for k in range(3):
        rp, col, val = [0], [], []
        for row in rows:
            for v, c in row[k]:
                col.append(v)
                val.append(c)
            rp.append(len(col))
        mats.append((np.array(rp, np.uint64), np.array(col, np.uint32), mont(val) if val else np.zeros((0, 4), np.uint64)))
    return mats


def case_mats(case):
    return csr(case.cs.rows)


def witness(case):
    """(inputs, aux) as Montgomery images"""
    z = mont(case.z)
    return np.ascontiguousarray(z[:case.ni]), np.ascontiguousarray(z[case.ni:])


def toxic(case):
    return mont(case.toxic)


def rs(case):
    m = mont([case.r, case.s])
    return m[0].copy(), m[1].copy()


def r1cs(case):
    from bazuka_b200.groth16 import R1CS
    return R1CS(case.ni, case.na, *case_mats(case))


def blocked_r1cs(case):
    from bazuka_b200.groth16 import BlockedR1CS
    head, tmpl, reps, tail, var_lo, stride, stored = case.blocked
    return BlockedR1CS(case.ni, case.na, head, tmpl, reps, tail, var_lo, stride, *csr(stored))


# ------------------------------------------------------------------ generators
def _terms(g, vars_, width):
    return [(g.choice(vars_), g.randrange(1, R)) for _ in range(g.randint(1, width))]


def _solved_row(g, vars_, z, width=3, nz=None):
    """random A and B; C's last coefficient solved so that the row holds (its variable, from nz, has z != 0)"""
    a, b = _terms(g, vars_, width), _terms(g, vars_, width)
    c = [(g.choice(vars_), g.randrange(R)) for _ in range(g.randint(0, width - 1))]
    last = g.choice(nz or [v for v in vars_ if z[v]])
    rest = ev(a, z) * ev(b, z) - ev(c, z)
    c.append((last, rest * pow(z[last], -1, R) % R))
    return a, b, c


def _rand_z(g, n):
    return [1] + [g.randrange(R) for _ in range(n - 1)]


def random_case(name, family, ni, na, ncons, seed, width=3, **kw):
    g = random.Random(f"{name}-{seed}")
    z = _rand_z(g, ni + na)
    vars_ = list(range(ni + na))
    nz = [v for v in vars_ if z[v]]
    rows = [_solved_row(g, vars_, z, width, nz) for _ in range(ncons)]
    return Case(name, family, ni, na, rows, z, seed, **kw)


def boundary_cases():
    totals = sorted({t for k in range(8) for t in ((1 << k) - 1, 1 << k, (1 << k) + 1) if t >= 1})
    out = []
    for tot in totals:
        for ni in (1, 2, 5):
            if tot < ni:
                continue
            ncons = tot - ni
            out.append(random_case(f"boundary-{tot}-ni{ni}", "boundary", ni, 1 + ncons // 4, ncons, seed=1000 * tot + ni))
    return out


def large_cases():
    return [random_case("boundary-4096-ni2", "large", 2, 1500, 4094, seed=12),
            random_case("boundary-65536-ni5", "large", 5, 20000, 65531, seed=16)]


def degenerate_cases():
    out = [Case("m1", "degenerate", 1, 0, [], [1], 1, expect=(0, 0, 0, 1, 0)),
           Case("m1-aux-only-in-l", "degenerate", 1, 3, [], [1, 5, 0, R - 1], 2, expect=(0, 0, 3, 1, 0))]
    # no aux: l is empty; inputs only (x1^2 = x2, x2 * x3 = x4 with x4 public)
    x = [1, 3, 9, 7, 63]
    out.append(Case("no-aux", "degenerate", 5, 0, [([(1, 1)], [(1, 1)], [(2, 1)]), ([(2, 1)], [(3, 1)], [(4, 1)]),
                                                   ([(0, 2), (3, 1)], [(0, 1)], [(0, 9)])], x, 3, expect=(3, 7, 0, 5, 3)))
    # every B side empty: every row is a * 0 = 0, so C is empty too
    g = random.Random("empty-b")
    z = _rand_z(g, 8)
    rows = [(_terms(g, list(range(8)), 3), [], []) for _ in range(6)]
    out.append(Case("empty-b", "degenerate", 2, 6, rows, z, 4, expect=(3, 7, 6, 2 + len({v for a, _, _ in rows for v, _ in a if v >= 2}), 0)))
    # a zero witness apart from ONE, and ONE absent from B: the b sums, h and l are the identity
    g = random.Random("zero-witness")
    nv = 9
    rows = [(_terms(g, list(range(nv)), 3), _terms(g, list(range(1, nv)), 3), _terms(g, list(range(1, nv)), 2)) for _ in range(10)]
    out.append(Case("zero-witness", "degenerate", 3, 6, rows, [1] + [0] * (nv - 1), 5))
    for name, rs_ in (("r0", (0, 7)), ("s0", (11, 0)), ("r0-s0", (0, 0))):
        out.append(random_case(name, "degenerate", 2, 6, 9, seed=6, rs=rs_))
    return out


def density_cases():
    out = []
    g = random.Random("density")
    ni, na = 3, 10
    z = _rand_z(g, ni + na)
    # aux 3 + k is absent from A (k = 0), from B (k = 1), from every side (k = 2); aux 3 + 3 only in C
    no_a, no_b, nowhere, c_only = 3, 4, 5, 6
    base = [v for v in range(ni + na) if v not in (no_a, no_b, nowhere, c_only)]
    rows = []
    for _ in range(12):
        a = _terms(g, base + [no_b], 3)
        b = _terms(g, base + [no_a], 3)
        c = _terms(g, base + [no_a, no_b, c_only], 2)
        last = g.choice([v for v in base if z[v]])
        c.append((last, (ev(a, z) * ev(b, z) - ev(c, z)) * pow(z[last], -1, R) % R))
        rows.append((a, b, c))
    rows[0] = (rows[0][0] + [(no_b, 0)], rows[0][1], rows[0][2])
    rows[1] = (rows[1][0] + [(no_a, 0)], rows[1][1] + [(no_b, 0)], rows[1][2])   # stored zeros are not presence
    case = Case("absent-from-a-b-all", "density", ni, na, rows, z, 20)
    a_aux = {v for r in rows for v, c in r[0] if c and v >= ni}
    assert no_a not in a_aux and no_b in a_aux and nowhere not in a_aux and c_only not in a_aux
    out.append(case)
    # inputs (ONE included) absent from B
    g = random.Random("inputs-not-in-b")
    ni, na = 4, 6
    z = _rand_z(g, ni + na)
    rows = []
    for _ in range(7):
        a, b = _terms(g, list(range(ni + na)), 3), _terms(g, list(range(ni, ni + na)), 3)
        last = g.randrange(ni + na)
        rows.append((a, b, [(last, ev(a, z) * ev(b, z) * pow(z[last], -1, R) % R)]))
    out.append(Case("inputs-not-in-b", "density", ni, na, rows, z, 21))
    # a variable present only with stored zero coefficients, on every side
    g = random.Random("zero-coef")
    ni, na = 2, 6
    z = _rand_z(g, ni + na)
    zc = 7
    vars_ = list(range(ni + na - 1))
    rows = [_solved_row(g, vars_, z) for _ in range(5)]
    rows = [(a + [(zc, 0)], b + [(zc, 0)], c + [(zc, 0)]) for a, b, c in rows]
    out.append(Case("zero-coefficient-only", "density", ni, na, rows, z, 22))
    # duplicate (row, col) entries add: 3 v + 5 v in A, -2 w + 2 w + 9 w in B
    g = random.Random("dup")
    ni, na = 2, 5
    z = _rand_z(g, ni + na)
    rows = []
    for _ in range(6):
        v, w = g.randrange(ni + na), g.randrange(ni + na)
        a, b = [(v, 3), (v, 5), (2, 1)], [(w, R - 2), (w, 2), (w, 9)]
        c = [(5, 1), (5, 1)]
        c.append((0, (ev(a, z) * ev(b, z) - ev(c, z)) % R))
        rows.append((a, b, c))
    out.append(Case("duplicates-add", "density", ni, na, rows, z, 23))
    # cancelling duplicates: aux 6 appears only as (6, c), (6, -c) in one A row, aux 7 likewise in one B row
    g = random.Random("cancel")
    ni, na = 2, 6
    z = _rand_z(g, ni + na)
    vars_ = list(range(6))
    rows = [_solved_row(g, vars_, z) for _ in range(7)]
    k = g.randrange(1, R)
    rows[2] = (rows[2][0] + [(6, k), (6, R - k)], rows[2][1], rows[2][2])
    rows[4] = (rows[4][0], rows[4][1] + [(7, 5), (7, R - 5)], rows[4][2])
    out.append(Case("cancelling-duplicates", "density", ni, na, rows, z, 24, cancelling=(6, 7)))
    return out


def value_cases():
    out = []
    g = random.Random("values")
    ni, na = 3, 9
    edges = (1, R - 1, (1 << 64) - 1)
    z = [1, 0, R - 1, 1, 0, R - 1, 1] + [g.randrange(R) for _ in range(ni + na - 7)]
    rows = []
    for i in range(12):
        # two distinct variables per side: 1 and r - 1 on one variable would cancel
        a = [(v, edges[(i + j) % 3]) for j, v in enumerate(g.sample(range(ni + na), 2))]
        b = [(v, edges[(i + j + 1) % 3]) for j, v in enumerate(g.sample(range(ni + na), 2))]
        c = [(g.randrange(ni + na), edges[i % 3])]
        t = (ev(a, z) * ev(b, z) - ev(c, z)) % R
        c.append((0, t))                       # ONE's coefficient closes the row
        rows.append((a, b, c))
    out.append(Case("edge-coefficients-and-witness", "value", ni, na, rows, z, 30))
    # one row of 1100 terms over 64 variables (repeats add), in A and in C
    g = random.Random("wide")
    ni, na = 2, 62
    z = _rand_z(g, ni + na)
    vars_ = list(range(ni + na))
    rows = [_solved_row(g, vars_, z) for _ in range(5)]
    a = [(g.choice(vars_), g.randrange(R)) for _ in range(1100)]
    b = [(3, 1), (0, 2)]
    c = [(g.choice(vars_), g.randrange(R)) for _ in range(1100)]
    c.append((0, (ev(a, z) * ev(b, z) - ev(c, z)) % R))
    rows.insert(2, (a, b, c))
    out.append(Case("row-of-1100-terms", "value", ni, na, rows, z, 31))
    # aux 4 in every row, on every side
    g = random.Random("every-row")
    ni, na = 2, 10
    z = _rand_z(g, ni + na)
    rows = []
    for _ in range(40):
        a = _terms(g, list(range(ni + na)), 2) + [(4, g.randrange(1, R))]
        b = _terms(g, list(range(ni + na)), 2) + [(4, g.randrange(1, R))]
        c = [(4, g.randrange(1, R))]
        c.append((0, (ev(a, z) * ev(b, z) - ev(c, z)) % R))
        rows.append((a, b, c))
    out.append(Case("variable-in-every-row", "value", ni, na, rows, z, 32))
    return out


def unsat_cases():
    """one satisfied system with C coefficients bumped on chosen rows; a row's C always names ONE last, so a bump by 1
    moves c by 1"""
    out = []
    ni, na, ncons = 3, 8, 21
    for name, which in (("unsat-first-row", [0]), ("unsat-last-row", [ncons - 1]), ("unsat-two-rows", [3, 11]),
                        ("unsat-every-row", list(range(ncons)))):
        g = random.Random("unsat")
        z = _rand_z(g, ni + na)
        rows = []
        for j in range(ncons):
            a, b = _terms(g, list(range(ni + na)), 3), _terms(g, list(range(ni + na)), 3)
            c = _terms(g, list(range(1, ni + na)), 2)
            c.append((0, (ev(a, z) * ev(b, z) - ev(c, z) + (j in which)) % R))
            rows.append((a, b, c))
        out.append(Case(name, "unsat", ni, na, rows, z, 40, bad=len(which)))
    return out


def blocked_case(name, ni, head, tmpl, reps, tail, n_pro, stride, n_epi, seed, pad_to=None):
    """a blocked system whose template holds for every copy: template row t is A_t(z) * B_t(z) = out_t with out_t the
    slot's t-th variable, A_t / B_t over shared variables, the slot's inputs and its earlier outputs.  Head and tail
    rows are random rows over every variable (C solved).  The last copy's last slot variable is used by the template,
    so with n_epi = 0 a template column names nv - 1."""
    g = random.Random(f"blocked-{name}-{seed}")
    var_lo = ni + n_pro
    na = n_pro + reps * stride + n_epi
    nv = ni + na
    z = _rand_z(g, nv)
    shared = list(range(var_lo))
    tmpl_rows = []
    for t in range(tmpl):
        ins = list(range(tmpl, stride)) + list(range(t))     # slot-relative: inputs, then earlier outputs
        pick = lambda: [(var_lo + d, g.randrange(1, R)) if d is not None else (g.choice(shared), g.randrange(1, R))
                        for d in [g.choice(ins + [None])]]
        a = pick() + pick() + ([(var_lo + stride - 1, g.randrange(1, R))] if t == 0 else [])
        b = pick() + [(0, g.randrange(1, R))]
        tmpl_rows.append((a, b, [(var_lo + t, 1)]))
    shift = lambda lc, k: [(v + k * stride if v >= var_lo else v, c) for v, c in lc]
    for k in range(reps):
        for t, (a, b, _) in enumerate(tmpl_rows):
            z[var_lo + k * stride + t] = ev(shift(a, k), z) * ev(shift(b, k), z) % R
    ends = list(range(nv))
    head_rows = [_solved_row(g, ends, z) for _ in range(head)]
    tail_rows = [_solved_row(g, ends, z) for _ in range(tail)]
    rows = head_rows + [(shift(a, k), shift(b, k), shift(c, k)) for k in range(reps) for a, b, c in tmpl_rows] + tail_rows
    stored = head_rows + tmpl_rows + tail_rows
    return Case(name, "blocked", ni, na, rows, z, seed, blocked=(head, tmpl, reps, tail, var_lo, stride, stored))


def blocked_cases():
    # the stored template's columns must name variables even when no copy is made: with reps = 0 they name the epilogue
    return [blocked_case("blocked-reps0", 2, 3, 2, 0, 2, 3, 4, 4, 50),
            blocked_case("blocked-reps1", 2, 2, 3, 1, 2, 2, 5, 1, 51),
            blocked_case("blocked-no-template-rows", 3, 4, 0, 4, 2, 2, 3, 1, 52),
            blocked_case("blocked-no-head", 1, 0, 3, 3, 2, 1, 5, 2, 53),
            blocked_case("blocked-no-tail", 2, 2, 2, 5, 0, 2, 4, 1, 54),
            # the last copy's last slot variable is nv - 1; 3 + 2 * 9 + 6 rows and 5 inputs fill a 2^5 domain exactly
            blocked_case("blocked-last-column-nv-1", 5, 3, 2, 9, 6, 2, 4, 0, 55)]


def all_cases(large=False):
    out = boundary_cases() + degenerate_cases() + density_cases() + value_cases() + unsat_cases() + blocked_cases()
    if large:
        out += large_cases()
    names = [c.name for c in out]
    assert len(set(names)) == len(names)
    return out


FAMILIES = ("boundary", "large", "degenerate", "density", "value", "unsat", "blocked")


def oracle_points(params):
    """the C oracle's key (groth16_c.setup) as the big-integer restatement's params dict, with unfiltered a / b columns"""
    from oracle.py import curve as C
    g1 =lambda x: C.g1_from_bytes(bytes(x))
    g2 = lambda x: C.g2_from_bytes(bytes(x))
    vk = {k: (g1(v) if len(v) == 104 else g2(v)) for k, v in params["vk"].items() if k != "ic"}
    vk["ic"] = [g1(x) for x in params["vk"]["ic"]]
    n = params["nv"]
    a_all, b1_all, b2_all = [None] * n, [None] * n, [None] * n
    for i, v in enumerate(params["a_idx"]):
        a_all[v] = g1(params["a"][i])
    for i, v in enumerate(params["b_idx"]):
        b1_all[v], b2_all[v] = g1(params["b_g1"][i]), g2(params["b_g2"][i])
    return {"log_m": params["log_m"], "vk": vk, "h": [g1(x) for x in params["h"]], "l": [g1(x) for x in params["l"]],
            "a_all": a_all, "b1_all": b1_all, "b2_all": b2_all}


def big_int_proof_bytes(case, params=None):
    """G.prove's 387 bytes at the case's (r, s), on the big-integer setup or on `params` (oracle_points)"""
    if params is None:
        params = G.setup(case.cs, *case.toxic)
    return G.proof_to_bytes(G.prove(case.cs, params, case.z, case.r, case.s))
