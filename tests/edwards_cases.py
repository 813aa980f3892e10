"""Edge cases and big-integer reference for the Edwards-curve code (csrc/ed25519.cuh, csrc/jubjub.cuh) in the conformance
harness tests/devshim/edwards.cu (test infrastructure).

The harness has the record layout and the three builds of arith_cases' BLS12-381 harness (sm_90a; g++ over the device text;
g++ over the host fast paths), and this module reuses arith_cases' build, packing and generic field helpers.  It packs the
Ed25519 and JubJub families into records and checks every output against plain Python integers:
`oracle/py/ed25519.py` for Ed25519, `bazuka_b200/mpn/native.py` for JubJub, `hashlib` for SHA-512, and the generic
twisted-Edwards law below (a = -1, complete on both curves) for the group operations.

- the fields mod p = 2^255 - 19 and mod l: arith_cases' generic families, reduce_once above the modulus, and products whose
  first operand is any 256-bit integer (what sc_from_hash multiplies);
- the curve constants as the device and the host hold them;
- both group laws on the identity, (0, -1), (+-sqrt(-1), 0), the order-8 points, the generators, random multiples and
  multiples plus torsion, each given as projective representatives with Z at limb edges; scalars at every edge of the
  windowed and fixed-base multiplications;
- both fixed-base tables, every one of their 8192 entries, read back and through jj_mul_fixed;
- SHA-512 at every length 0-300, 1 KiB and 4 KiB, split into three pieces at the block edges;
- Ed25519's scalar reduction, canonical check, square root, decompression and compression;
- JubJub's Tonelli-Shanks root and decompression, with every order of a^q in one warp.

Everything is seeded and deterministic; counts go to arith_cases.COUNTS and the tests assert them."""
import ctypes as ct
import functools
import hashlib
import itertools
import os
import random

import numpy as np

import arith_cases as A
import ed25519_cases as EC
import eddsa_cases as JC
from arith_cases import Case, rec, words
from bazuka_b200.mpn import native as N
from oracle.py import ed25519 as O

TABLE_ENTRIES = 32 * 256
_count = A._count

SRC = os.path.join(A.SHIM, "edwards.cu")
DEPS = [SRC] + [os.path.join(A.CSRC, h) for h in ("ff.cuh", "jubjub.cuh", "ed25519.cuh")]

# ------------------------------------------------------------------ op table (mirrors the enums of edwards.cu)
FIELDS = {"p25519": (2**255 - 19, 8, 0), "l25519": (2**252 + 27742317777372353535851937790883648493, 8, 1)}
# arith_cases' generic field families look their modulus up by name in its field table
for _name, _spec in FIELDS.items():
    A.FIELDS.setdefault(_name, _spec)
SHA_WORDS = 1040
_FIELD_KINDS = ["add", "sub", "mul", "neg", "dbl", "sqr", "to_mont", "from_mont", "from_u32", "pow", "inv", "inv_gcd", "mul_wide", "reduce_once"]
# (kind, in words, out words); JubJub records carry d (8 words) in front
_EDWARDS_KINDS = [("add", 64, 32), ("add_niels", 56, 32), ("dbl", 32, 32), ("mul", 40, 32), ("mul_fixed", 8, 32), ("equal", 64, 1)]
_ED25519_KINDS = [("sha512", 6 + SHA_WORDS, 16), ("sc_from_hash", 16, 8), ("sc_canonical", 8, 9), ("sqrt_ratio_i", 16, 9),
                  ("decompress", 8, 17), ("compress", 32, 8), ("consts", 1, 24)]
_JUBJUB_KINDS = [("fr_sqrt", 8, 9), ("decompress", 9, 17), ("on_curve", 16, 1), ("consts", 1, 16)]


def _ops():
    ops = {}
    for f, (_, n, t) in FIELDS.items():
        w = {"add": (2 * n, n), "sub": (2 * n, n), "mul": (2 * n, n), "from_u32": (1, n), "pow": (2 * n, n), "mul_wide": (2 * n, 2 * n)}
        for k, name in enumerate(_FIELD_KINDS):
            ops[f"{f}.{name}"] = ((t << 4) | k, *w.get(name, (n, n)))
    for k, (name, i, o) in enumerate(_EDWARDS_KINDS):
        ops[f"ed25519.{name}"] = ((2 << 4) | k, i, o)
        ops[f"jubjub.{name}"] = ((3 << 4) | k, 8 + i, o)
    for k, (name, i, o) in enumerate(_ED25519_KINDS):
        ops[f"ed25519.{name}"] = ((4 << 4) | k, i, o)
    for k, (name, i, o) in enumerate(_JUBJUB_KINDS):
        ops[f"jubjub.{name}"] = ((5 << 4) | k, 8 + i, o)
    return ops


OPS = _ops()


# ------------------------------------------------------------------ builds
def _stale(out):
    return not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in DEPS)


def _compile(cmd, out):
    saved = A.SRC
    A.SRC = SRC     # only used in the error message
    try:
        return A._compile(cmd, out)
    finally:
        A.SRC = saved


def build_host(device_text):
    """g++ build: the device text of the field arithmetic, or the host fast paths"""
    out = os.path.join(A.SHIM, "_edwards_host_dt.so" if device_text else "_edwards_host.so")
    if _stale(out):
        _compile(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++"] + (["-DBZK_HOST_DEVICE_TEXT"] if device_text else []) +
                 ["-I", A.CSRC, SRC], out)
    return out


def build_dev():
    """nvcc build with libbzk's own compiler and flags (sm_90a)"""
    from bazuka_b200 import build as B
    out = os.path.join(A.SHIM, "_edwards_dev.so")
    if _stale(out):
        _compile([B.NVCC] + B.FLAGS + ["-shared", "-I", A.CSRC, SRC], out)
    return out


class HostEdwards:
    """one g++ build; jj_mul_fixed runs over the tables this build's own host code makes"""

    def __init__(self, device_text):
        self.lib = ct.CDLL(build_host(device_text))
        self.lib.edwards_run_host.argtypes = [ct.c_int, ct.c_void_p, ct.c_int, ct.c_void_p, ct.c_int, ct.c_size_t, ct.c_void_p]
        self.tables = {name: read_table(self.lib, name) for name in CURVES}

    def run(self, op, inp):
        code, in_w, out_w = OPS[op]
        inp = np.ascontiguousarray(inp, dtype=np.uint32).reshape(-1, in_w)
        out = np.zeros((len(inp), out_w), dtype=np.uint32)
        tab = self.tables.get(op.split(".")[0])
        self.lib.edwards_run_host(code, inp.ctypes.data, in_w, out.ctypes.data, out_w, len(inp), None if tab is None else tab.ctypes.data)
        return out


class DevEdwards:
    """one thread per record, with a partial last block and a guard record past the end; jj_mul_fixed reads the tables built
    by this library's host code (nvcc's host pass) and uploaded, as libbzk's contexts do"""

    def __init__(self):
        import torch
        self.lib = ct.CDLL(build_dev())
        self.lib.edwards_run_dev.argtypes = [ct.c_int, ct.c_void_p, ct.c_int, ct.c_void_p, ct.c_int, ct.c_size_t, ct.c_int, ct.c_void_p]
        self.blocks = []
        self.tables = {name: torch.from_numpy(read_table(self.lib, name).view(np.int32)).cuda() for name in CURVES}

    def run(self, op, inp):
        import torch
        code, in_w, out_w = OPS[op]
        inp = np.ascontiguousarray(inp, dtype=np.uint32).reshape(-1, in_w)
        n = len(inp)
        block = 127 if n % 127 else 113
        d_in = torch.from_numpy(inp.view(np.int32)).cuda()
        d_out = torch.full((n + 1, out_w), -1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        tab = self.tables.get(op.split(".")[0])
        e = self.lib.edwards_run_dev(code, d_in.data_ptr(), in_w, d_out.data_ptr(), out_w, n, block, None if tab is None else tab.data_ptr())
        assert e == 0, f"{op}: cudaError {e}"
        out = d_out.cpu().numpy().view(np.uint32)
        assert (out[n] == 0xFFFFFFFF).all(), f"{op}: wrote past the last record"
        self.blocks.append((n, block))
        return out[:n]


def read_params(lib, name):
    """p, one, r2, inv (and r3 for l) of a parameter pack as compiled"""
    out = np.zeros(33, np.uint32)
    lib.edwards_params(FIELDS[name][2], out.ctypes.data_as(ct.c_void_p))
    return out


# ------------------------------------------------------------------ the two curves in big integers
class Curve:
    """x^2 (-1) + y^2 = 1 + d x^2 y^2 over F_p; points are affine (x, y) tuples of canonical integers"""

    def __init__(self, name, p, d, gen, field):
        self.name, self.p, self.d, self.gen = name, p, d, gen
        self.f = A._F(field)
        self.jubjub = name == "jubjub"

    def on_curve(self, P):
        x, y = P
        p = self.p
        return (y * y - x * x - 1 - self.d * x * x % p * y * y) % p == 0

    def add(self, P, Q):
        (x1, y1), (x2, y2) = P, Q
        p = self.p
        t = self.d * x1 % p * x2 % p * y1 % p * y2 % p
        return ((x1 * y2 + y1 * x2) * pow(1 + t, -1, p) % p, (y1 * y2 + x1 * x2) * pow(1 - t, -1, p) % p)

    def neg(self, P):
        return ((-P[0]) % self.p, P[1])

    def _ext_add(self, P, Q):
        p, d2 = self.p, 2 * self.d
        x1, y1, z1, t1 = P
        x2, y2, z2, t2 = Q
        a = (y1 - x1) * (y2 - x2) % p
        b = (y1 + x1) * (y2 + x2) % p
        c = d2 * t1 % p * t2 % p
        dd = 2 * z1 * z2 % p
        e, f, g, h = b - a, dd - c, dd + c, b + a
        return (e * f % p, g * h % p, f * g % p, e * h % p)

    def mul(self, P, k):
        """[k] P for any integer k >= 0, not reduced"""
        p = self.p
        acc, q = (0, 1, 1, 0), (P[0], P[1], 1, P[0] * P[1] % p)
        while k:
            if k & 1:
                acc = self._ext_add(acc, q)
            q = self._ext_add(q, q)
            k >>= 1
        zi = pow(acc[2], -1, p)
        return (acc[0] * zi % p, acc[1] * zi % p)

    # ---- packing (Montgomery images, as libbzk stores them)
    def img(self, v):
        return self.f.img(v)

    def d_prefix(self, n):
        """JubJub records start with d"""
        return words([self.img(self.d)] * n, 8) if self.jubjub else np.zeros((n, 0), np.uint32)

    def ext(self, pts, lams):
        """(X, Y, T, Z) = (x l, y l, x y l, l)"""
        p, out = self.p, []
        for (x, y), lam in zip(pts, lams):
            parts = (x * lam, y * lam, x * y % p * lam, lam)
            out.append(sum(self.img(v % p) << (256 * i) for i, v in enumerate(parts)))
        return words(out, 32)

    def niels(self, pts):
        p = self.p
        return words([self.img((y - x) % p) | (self.img((y + x) % p) << 256) | (self.img(2 * self.d * x * y % p) << 512) for x, y in pts], 24)

    def unpack_ext(self, row):
        """output words -> (x, y) or None: canonical limbs, Z != 0 and T Z = X Y (a wrong T only shows at the next addition)"""
        p, f = self.p, self.f
        imgs = A.ints(np.asarray(row).reshape(4, 8))
        if any(v >= p for v in imgs):
            return None
        X, Y, T, Z = (f.val(v) for v in imgs)
        if Z == 0 or T * Z % p != X * Y % p:
            return None
        zi = pow(Z, -1, p)
        return (X * zi % p, Y * zi % p)

    def check_ext(self, want):
        def check(out):
            return [i for i, row in enumerate(np.ascontiguousarray(out)) if self.unpack_ext(row) != want[i]]
        return check

    def lams(self):
        """Z values whose Montgomery images sit at limb edges: 1 (image R mod p), R^-1 (image 1), p - 1, 2^32 - 1, the top limb
        alone, all ones below the top limb, p - 2^32, and one random value"""
        p, f = self.p, self.f
        rnd = random.Random(31 + self.jubjub)
        imgs = [f.Rm, 1, p - 1, 2**32 - 1, 1 << 224, (1 << 224) - 1, p - 2**32, 0xFFFFFFFF << 96, rnd.randrange(1, p)]
        return [f.val(v) for v in imgs]

    def torsion(self):
        return EC.torsion_points() if not self.jubjub else JC.torsion_points()

    def point_order(self, P):
        for k in (1, 2, 4, 8):
            if self.mul(P, k) == (0, 1):
                return k
        return None


ED = Curve("ed25519", O.P, O.D, O.B, "p25519")
JJ = Curve("jubjub", N.R, N.JJ_D, N.JJ_BASE, "fr")
CURVES = {"ed25519": ED, "jubjub": JJ}
L, P25519, R_FR, ORDER = O.L, O.P, N.R, N.JJ_ORDER


@functools.lru_cache(maxsize=None)
def points(name):
    """the identity, (0, -1), (+-sqrt(-1), 0), the order-8 points, the generator, random multiples, and multiples plus each
    torsion point; [(label, point)]"""
    c = CURVES[name]
    p = c.p
    rnd = random.Random(808 + c.jubjub)
    sqrt_m1 = O.SQRT_M1 if not c.jubjub else N.fr_sqrt(p - 1)
    tors = c.torsion()
    out = [("identity", (0, 1)), ("(0,-1)", (0, p - 1)), ("(sqrt-1,0)", (sqrt_m1, 0)), ("(-sqrt-1,0)", (p - sqrt_m1, 0))]
    out += [(f"torsion {j}", t) for j, t in enumerate(tors)]
    out.append(("G", c.gen))
    mults = [c.mul(c.gen, rnd.randrange(1, 2**253)) for _ in range(3)]
    out += [(f"[k]G #{i}", m) for i, m in enumerate(mults)]
    out += [(f"[k]G #0 + torsion {j}", c.add(mults[0], t)) for j, t in enumerate(tors) if j]
    first = {}
    for lab, pt in out:   # distinct points, first label kept
        first.setdefault(pt, lab)
    out = [(lab, pt) for pt, lab in first.items()]
    for lab, pt in out:
        assert c.on_curve(pt), (name, lab)
    for t in tors:
        _count(f"{name} torsion points of order {c.point_order(t)}", 1)
    _count(f"{name} points", len(out))
    return out


def k_edges():
    """the scalar edge list: small windows, both group orders and their neighbours, the Fr modulus, 2^255 and 2^256 - 1"""
    return [0, 1, 15, 16, 255, 256, L - 1, L, L + 1, 8 * L - 1, R_FR - 1, ORDER - 1, ORDER + 1, 2**255, 2**256 - 1]


def k_patterns():
    """nibble and byte patterns: every window 15 or 0, alternating, one window set, the top window alone"""
    rep = lambda unit, bits: int(unit * (256 // bits), 16)
    pats = [rep("f", 4), rep("1", 4), rep("f0", 8), rep("0f", 8), rep("80", 8), rep("01", 8), rep("ff00", 16), rep("00ff", 16),
            rep("5a", 8), rep("a5", 8), 0xF << 252, 0xFF << 248, 0x8 << 252, 1 << 128, (1 << 128) - 1]
    return pats


def k_list(rnd):
    ks = k_edges() + k_patterns() + [rnd.randrange(2**256) for _ in range(6)] + [rnd.randrange(L) for _ in range(2)]
    return ks


# ------------------------------------------------------------------ fields
def fam_field(name):
    """arith_cases' generic families over one of the two 25519 fields"""
    cases = []
    for fn in (A.fam_structured, A.fam_sums, A.fam_mont_boundary, A.fam_inverse, A.fam_pow_u32):
        cases += fn(name)
    return cases


def fam_above_modulus(name):
    """reduce_once above the modulus: p25519 on all of [p, 2^255) (ed_decompress's inputs), l25519 on [l, 2^256) edges and
    random values, where one conditional subtraction gives a - l (sc_canonical's test a == reduce_once(a))"""
    f = A._F(name)
    p = f.p
    rnd = random.Random(5 + f.n)
    if name == "p25519":
        vals = list(range(p, 2**255)) + list(range(0, 40)) + [p - 1, p - 2, 2**255 - 20]
        want = [v % p for v in vals]
    else:
        vals = [p, p + 1, 2 * p - 1, 2 * p, 2 * p + 1, 2**253, 2**255 - 1, 2**255, 2**256 - 1] + [(1 << 256) - (1 << (32 * k)) for k in range(8)]
        vals += [rnd.randrange(p, 2**256) for _ in range(64)] + [rnd.randrange(p, 2 * p) for _ in range(32)] + [0, 1, p - 1]
        want = [v - p if v >= p else v for v in vals]
    _count(f"{name} reduce_once above the modulus", sum(v >= p for v in vals))
    return [Case(f"{name}.reduce_once", words(vals, 8), words(want, 8))]


def fam_wide_l():
    """Montgomery products mod l with a in [l, 2^256) and b < l: a b R^-1 mod l, fully reduced (sc_from_hash multiplies the
    raw digest halves by R^2 and R^3)"""
    f = A._F("l25519")
    l, R = f.p, f.R
    rnd = random.Random(252)
    As = [l, l + 1, 2 * l - 1, 2 * l, 2**253, 2**255 - 1, 2**255, 2**256 - 1, 2**256 - l] + [(1 << 256) - (1 << (32 * k)) for k in range(8)]
    As += [rnd.randrange(l, 2**256) for _ in range(48)]
    r2, r3 = R * R % l, R * R * R % l
    Bs = [0, 1, 2, l - 1, l - 2, r2, r3, f.Rm] + A.structured(f)[::9] + [rnd.randrange(l) for _ in range(8)]
    pairs = list(itertools.product(As, Bs))
    _count("l25519 wide-operand products", len(pairs))
    Ri = f.Rinv
    return [Case("l25519.mul", rec(words([a for a, _ in pairs], 8), words([b for _, b in pairs], 8)), words([a * b * Ri % l for a, b in pairs], 8))]


# ------------------------------------------------------------------ constants
def const_images():
    """the device op's words: ed_d, ed_d2, ed_sqrt_m1 (Montgomery); jubjub: BASE"""
    e = ED.img
    return words([e(O.D) | (e(2 * O.D % P25519) << 256) | (e(O.SQRT_M1) << 512)], 24), words([JJ.img(N.JJ_BASE[0]) | (JJ.img(N.JJ_BASE[1]) << 256)], 16)


def host_const_images():
    """arith_edwards_consts: ed_d, ed_d2, ed_sqrt_m1, B, BASE"""
    e, j = ED.img, JJ.img
    vals = [e(O.D), e(2 * O.D % P25519), e(O.SQRT_M1), e(O.B[0]), e(O.B[1]), j(N.JJ_BASE[0]), j(N.JJ_BASE[1])]
    return words([sum(v << (256 * i) for i, v in enumerate(vals))], 56)[0]


def fam_consts():
    ed, jj = const_images()
    return [Case("ed25519.consts", np.zeros((3, 1), np.uint32), np.repeat(ed, 3, axis=0)),
            Case("jubjub.consts", rec(JJ.d_prefix(3), np.zeros((3, 1), np.uint32)), np.repeat(jj, 3, axis=0))]


def read_consts(lib):
    out = np.zeros(56, np.uint32)
    lib.edwards_consts(out.ctypes.data_as(ct.c_void_p))
    return out


# ------------------------------------------------------------------ group law
def fam_group(name):
    c = CURVES[name]
    p = c.p
    pts = points(name)
    lams = c.lams()
    rnd = random.Random(77 + c.jubjub)
    P = [pt for _, pt in pts]
    cases = []
    # addition (cached form): every ordered pair, the lambdas rotating; plus P + P, P + (-P), P + O and O + P under every pair
    # of lambdas
    ap = [(a, lams[i % len(lams)], b, lams[(i + 3 * j + 1) % len(lams)]) for i, a in enumerate(P) for j, b in enumerate(P)]
    for a in P:
        for l1, l2 in itertools.product(lams[:5], lams[:5]):
            ap += [(a, l1, a, l2), (a, l1, c.neg(a), l2), (a, l1, (0, 1), l2), ((0, 1), l1, a, l2)]
    _count(f"{name} additions", len(ap))
    n = len(ap)
    cases.append(Case(f"{name}.add", rec(c.d_prefix(n), c.ext([x[0] for x in ap], [x[1] for x in ap]), c.ext([x[2] for x in ap], [x[3] for x in ap])),
                      check=c.check_ext([c.add(x[0], x[2]) for x in ap])))
    # addition (Niels form, Z2 = 1: the fixed-base tables' entries)
    npairs = [(a, lams[(i + j) % len(lams)], b) for i, a in enumerate(P) for j, b in enumerate(P)] + [(a, l, c.neg(a)) for a in P for l in lams]
    n = len(npairs)
    cases.append(Case(f"{name}.add_niels", rec(c.d_prefix(n), c.ext([x[0] for x in npairs], [x[1] for x in npairs]), c.niels([x[2] for x in npairs])),
                      check=c.check_ext([c.add(x[0], x[2]) for x in npairs])))
    # doubling
    dp = [(a, l) for a in P for l in lams]
    n = len(dp)
    cases.append(Case(f"{name}.dbl", rec(c.d_prefix(n), c.ext([a for a, _ in dp], [l for _, l in dp])), check=c.check_ext([c.add(a, a) for a, _ in dp])))
    # equality: representatives of one point under two lambdas, P against -P, and distinct points
    eq = [(a, l1, a, l2, 1) for a in P for l1, l2 in ((lams[0], lams[2]), (lams[3], lams[8]), (lams[4], lams[4]))]
    eq += [(a, lams[1], b, lams[5], int(a == b)) for a in P for b in P]
    n = len(eq)
    cases.append(Case(f"{name}.equal", rec(c.d_prefix(n), c.ext([e[0] for e in eq], [e[1] for e in eq]), c.ext([e[2] for e in eq], [e[3] for e in eq])),
                      words([e[4] for e in eq], 1)))
    # windowed multiplication: every point with every scalar of the edge list, the patterns and random values
    ks = k_list(rnd)
    mp = [(a, lams[(i + j) % len(lams)], k) for i, a in enumerate(P) for j, k in enumerate(ks)]
    _count(f"{name} mul records", len(mp))
    n = len(mp)
    cases.append(Case(f"{name}.mul", rec(c.d_prefix(n), c.ext([m[0] for m in mp], [m[1] for m in mp]), words([m[2] for m in mp], 8)),
                      check=c.check_ext([c.mul(m[0], m[2]) for m in mp])))
    # fixed-base multiplication at the same scalars (the table sweep is fam_fixed_sweep)
    n = len(ks)
    cases.append(Case(f"{name}.mul_fixed", rec(c.d_prefix(n), words(ks, 8)), check=c.check_ext([c.mul(c.gen, k) for k in ks])))
    if c.jubjub:
        oc = P + [(x, (y + 1) % p) for x, y in P] + [(0, 0), (1, 1)]
        n = len(oc)
        cases.append(Case("jubjub.on_curve", rec(c.d_prefix(n), words([c.img(x) for x, _ in oc], 8), words([c.img(y) for _, y in oc], 8)),
                          words([int(c.on_curve(q)) for q in oc], 1)))
    else:   # compression of every point under every lambda (Z != 1)
        cp = [(a, l) for a in P for l in lams]
        want = np.frombuffer(b"".join(O.compress(a) for a, _ in cp), np.uint32).reshape(-1, 8)
        cases.append(Case("ed25519.compress", c.ext([a for a, _ in cp], [l for _, l in cp]), want))
    return cases


@functools.lru_cache(maxsize=None)
def table_points(name):
    """[j * 256 + v] -> [v 2^(8j)] G"""
    c = CURVES[name]
    out = []
    row = c.gen
    for _ in range(32):
        cur = (0, 1)
        for _ in range(256):
            out.append(cur)
            cur = c.add(cur, row)
        row = cur
    return out


def table_words(name):
    """the expected table: (y - x, y + x, 2 d x y) of every entry, Montgomery"""
    return CURVES[name].niels(table_points(name))


def read_table(lib, name):
    out = np.zeros((TABLE_ENTRIES, 24), np.uint32)
    d = words([JJ.img(N.JJ_D)], 8)[0]
    lib.edwards_table(0 if name == "ed25519" else 1, d.ctypes.data_as(ct.c_void_p), out.ctypes.data_as(ct.c_void_p))
    return out


def sweep(name, limit=2**256):
    """[(j, v, s, [s] G)] for every table entry (j, v) with s < limit, where s = v 2^(8j) plus, for j > 0, 1: window 0 then
    leaves G in the accumulator, so that adding entry (j, v) reads all three of its coordinates (added to the identity, as
    every window-0 entry is, 2dxy meets T = 0 and drops out)"""
    c = CURVES[name]
    pts = table_points(name)
    out = []
    for i in range(TABLE_ENTRIES):
        j, v = divmod(i, 256)
        s = (v << (8 * j)) + (1 if j else 0)
        if s < limit:
            out.append((j, v, s, c.add(pts[i], c.gen) if j else pts[i]))
    return out


def fam_fixed_sweep(name):
    """jj_mul_fixed over every table entry"""
    c = CURVES[name]
    sw = sweep(name)
    _count(f"{name} fixed-base sweep scalars", len(sw))
    return [Case(f"{name}.mul_fixed", rec(c.d_prefix(len(sw)), words([x[2] for x in sw], 8)), check=c.check_ext([x[3] for x in sw]))]


# ------------------------------------------------------------------ SHA-512
SHA_BYTES = 4 * SHA_WORDS
GAP = 13


def _sha_record(data, split, rnd):
    """data split into three pieces laid out with junk between them and at odd offsets, so that a piece read from the
    wrong base or at the wrong index changes the digest"""
    n0, n1 = split[0], split[1]
    n2 = len(data) - n0 - n1
    o0 = 3
    o1 = o0 + n0 + GAP
    o2 = o1 + n1 + GAP
    assert o2 + n2 <= SHA_BYTES
    buf = bytearray(rnd.randbytes(SHA_BYTES))
    buf[o0:o0 + n0] = data[:n0]
    buf[o1:o1 + n1] = data[n0:n0 + n1]
    buf[o2:o2 + n2] = data[n0 + n1:]
    return np.concatenate([np.array([n0, n1, n2, o0, o1, o2], np.uint32), np.frombuffer(bytes(buf), np.uint32)])


def sha_splits(n):
    s = {(n, 0), (0, 0), (0, n)}
    if n >= 64:
        s.add((32, 32))
    s.add((n // 3, n // 3))
    for e in (111, 112, 127, 128, 239, 240):   # a piece ending on either side of the padding and block edges
        if e <= n:
            s.add((e, 0))
            s.add((0, e))
            s.add((1, e - 1))
    return sorted(s)


def fam_sha512():
    rnd = random.Random(512)
    src = rnd.randbytes(4096)
    recs, want, lens = [], [], set()
    for n in list(range(301)) + [1024, 4096]:
        data = src[:n] if n % 2 else bytes(reversed(src[-n:])) if n else b""
        for sp in sha_splits(n):
            recs.append(_sha_record(data, sp, rnd))
            want.append(hashlib.sha512(data).digest())
            lens.add(n)
    _count("sha512 lengths 0-300", len(lens & set(range(301))))
    _count("sha512 records", len(recs))
    return [Case("ed25519.sha512", np.stack(recs), np.frombuffer(b"".join(want), np.uint32).reshape(-1, 16))]


# ------------------------------------------------------------------ Ed25519 scalars and points
SC_FROM_HASH_VALUES = [0, 1, L - 1, L, L + 1, 2 * L, 2**252, 2**256 - 1, 2**256, 2**256 * (L - 1), 2**512 - 1, L * L, L * 2**256 - 1]


def _le(v, n=32):
    return int(v).to_bytes(n, "little")


def fam_ed25519_scalars():
    rnd = random.Random(25519)
    hs = SC_FROM_HASH_VALUES + [(1 << 512) - (1 << (32 * k)) for k in range(16)] + [(2**256 - 1) << 256 | (2**256 - 1 - k) for k in range(3)]
    hs += [rnd.randrange(2**512) for _ in range(200)] + [int.from_bytes(hashlib.sha512(b"%d" % i).digest(), "little") for i in range(50)]
    _count("ed25519 sc_from_hash values", len(hs))
    cases = [Case("ed25519.sc_from_hash", words(hs, 16), words([h % L for h in hs], 8))]
    ss = [0, 1, L - 2, L - 1, L, L + 1, L + 2, 2 * L - 1, 2 * L, 2 * L + 1, 2**252, 2**253, 2**255 - 1, 2**256 - 1]
    ss += [s | (1 << 255) for s in (0, 1, L - 1, L, 5)] + [rnd.randrange(L) for _ in range(20)] + [rnd.randrange(L, 2**256) for _ in range(20)]
    _count("ed25519 sc_canonical values", len(ss))
    cases.append(Case("ed25519.sc_canonical", words(ss, 8), rec(words([int(s < L) for s in ss], 1), words(ss, 8))))
    return cases


def sqrt_ratio_expected(u, v):
    """dalek's sqrt_ratio_i: (was_square, the even root of u/v, or of i u/v when u/v is not a square; 0 when u or v is 0)"""
    p = P25519
    if u == 0:
        return 1, 0
    if v == 0:
        return 0, 0
    w = u * pow(v, -1, p) % p
    sq = pow(w, (p - 1) // 2, p) == 1
    t = w if sq else O.SQRT_M1 * w % p
    r = pow(t, (p + 3) // 8, p)
    if r * r % p != t:
        r = r * O.SQRT_M1 % p
    assert r * r % p == t
    return int(sq), (p - r if r & 1 else r)


def fam_ed25519_points():
    rnd = random.Random(2552)
    p = P25519
    e = ED.img
    ev = [0, 1, 2, 18, 19, p - 1, p - 2, (p - 1) // 2, O.D, O.SQRT_M1, p - O.SQRT_M1, 2**32 - 1, 2**128, 2**254] + [rnd.randrange(p) for _ in range(40)]
    uv = [(u, v) for u in ev for v in ev[:10]] + [(rnd.randrange(p), rnd.randrange(p)) for _ in range(200)]
    # decompression's own inputs: u = y^2 - 1, v = d y^2 + 1
    for y in range(12):
        uv.append(((y * y - 1) % p, (O.D * y * y + 1) % p))
    want = [sqrt_ratio_expected(u, v) for u, v in uv]
    _count("ed25519 sqrt_ratio_i squares", sum(1 for (u, _), w in zip(uv, want) if w[0] and u))
    _count("ed25519 sqrt_ratio_i non-squares", sum(1 for (_, v), w in zip(uv, want) if not w[0] and v))
    cases = [Case("ed25519.sqrt_ratio_i", rec(words([e(u) for u, _ in uv], 8), words([e(v) for _, v in uv], 8)),
                  rec(words([w[0] for w in want], 1), words([e(w[1]) for w in want], 8)))]
    # decompression: canonical and non-canonical y (y + p for y < 19), "-0", every torsion point and its sign flip, B, random
    encs = [_le(y) for y in list(range(19)) + [p - 1, p - 2, 2**255 - 1]] + [_le(y + p) for y in range(19)]
    encs += [_le(y | (1 << 255)) for y in list(range(19)) + [p - 1]] + [_le((y + p) | (1 << 255)) for y in range(19)]
    for _, pt in points("ed25519"):
        c = O.compress(pt)
        encs += [c, c[:31] + bytes([c[31] ^ 0x80])]
    encs += [rnd.randbytes(32) for _ in range(300)]
    got_none = sum(O.decompress(x) is None for x in encs)
    _count("ed25519 decompress encodings", len(encs))
    _count("ed25519 decompress refusals", got_none)
    dec = [O.decompress(x) for x in encs]

    def check(out):
        bad = []
        for i, (row, d) in enumerate(zip(np.ascontiguousarray(out), dec)):
            if int(row[0]) != int(d is not None):
                bad.append(i)
            elif d is not None and A.ints(row[1:].reshape(2, 8)) != [e(d[0]), e(d[1])]:
                bad.append(i)
        return bad
    cases.append(Case("ed25519.decompress", np.frombuffer(b"".join(encs), np.uint32).reshape(-1, 8).copy(), check=check))
    return cases


# ------------------------------------------------------------------ JubJub roots
def _fr_sqrt_c():
    q = (R_FR - 1) >> 32
    return pow(7, q, R_FR)


def fr_sqrt_inputs():
    """residues with a^q of every order 2^i (i = 0..31; i = 31 runs the full loop), non-residues (a^q of order 2^32), 0, 1, -1,
    interleaved so that neighbouring threads of a warp take different loop counts; [(a, order of a^q or None)]"""
    r = R_FR
    rnd = random.Random(4321)
    c = _fr_sqrt_c()
    out = [(0, 0), (1, 1), (r - 1, 2), (7, 2**32), (5, 2**32)]
    for rep in range(3):
        for i in range(33):
            u = pow(rnd.randrange(2, r), 1 << 32, r)   # a^q = 1
            e = (1 << (32 - i)) * (2 * rnd.randrange(1 << 20) + 1) if i else 0
            out.append((u * pow(c, e, r) % r, 1 << i))
    out += [(rnd.randrange(r), None) for _ in range(64)]
    rnd.shuffle(out)
    return out


def fam_jubjub_roots():
    r = R_FR
    j = JJ.img
    ins = fr_sqrt_inputs()
    for a, o in ins:
        if o is not None:
            _count(f"fr_sqrt a^q of order 2^{o.bit_length() - 1}" if o else "fr_sqrt a = 0", 1)
    roots = [N.fr_sqrt(a) for a, _ in ins]
    n = len(ins)
    cases = [Case("jubjub.fr_sqrt", rec(JJ.d_prefix(n), words([j(a) for a, _ in ins], 8)),
                  rec(words([int(x is not None) for x in roots], 1), words([0 if x is None else j(x) for x in roots], 8)))]
    # decompression: the x of every test point (both parities), x = 0, x with no point, and random x
    rnd = random.Random(99)
    xs = sorted({pt[0] for _, pt in points("jubjub")}) + [0, 1, 2, r - 1] + [rnd.randrange(r) for _ in range(60)]
    rec_in, rec_out = [], []
    for x in xs:
        den = (1 + N.JJ_D * (r - x * x % r)) % r   # 1 - d x^2
        root = N.fr_sqrt((1 + x * x) * pow(den, -1, r) % r) if den else None
        for odd in (0, 1):
            rec_in.append((x, odd))
            if root is None:
                rec_out.append((0, 0, None))
            else:
                y = root if (root & 1) == odd else (r - root) % r
                rec_out.append((1, root, y))
                assert (x, y) == N.jj_decompress_checked((x, bool(odd)))
    _count("jubjub decompress refusals", sum(o[0] == 0 for o in rec_out))
    n = len(rec_in)

    def check(out):
        bad = []
        for i, (row, w) in enumerate(zip(np.ascontiguousarray(out), rec_out)):
            if int(row[0]) != w[0] or (w[0] and A.ints(row[1:].reshape(2, 8)) != [j(w[1]), j(w[2])]):
                bad.append(i)
        return bad
    cases.append(Case("jubjub.decompress", rec(JJ.d_prefix(n), words([j(x) for x, _ in rec_in], 8), words([o for _, o in rec_in], 1)), check=check))
    return cases


# ------------------------------------------------------------------ random bulk records (device against host64)
def bulk_records(seed, n):
    """{op: input words}: random Montgomery products, sums and differences in both 25519 fields, and jj_mul of random curve
    points (random Z) by random 256-bit scalars on both curves"""
    rng = np.random.default_rng(seed)
    out = {}
    for name in ("p25519", "l25519"):
        p = FIELDS[name][0]
        top = p >> 224
        v = rng.integers(0, 1 << 32, size=(2 * n, 8), dtype=np.uint64).astype(np.uint32)
        v[:, 7] = rng.integers(0, top, size=2 * n, dtype=np.uint64).astype(np.uint32)   # below p
        for op in ("mul", "add", "sub"):
            out[f"{name}.{op}"] = v.reshape(n, 16)
    for c in (ED, JJ):
        # points [k] G + T: k from a short seeded list, so that the big-integer side stays cheap; the device and the host
        # build must agree word for word, so Z is random and the scalars are full width
        rnd = random.Random(seed)
        base = [c.add(c.mul(c.gen, rnd.randrange(1, 2**64)), t) for t in c.torsion()]
        idx = rng.integers(0, len(base), n)
        lam = [rnd.randrange(1, c.p) for _ in range(64)]
        li = rng.integers(0, len(lam), n)
        ext = c.ext([base[i] for i in idx], [lam[i] for i in li])
        ks = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
        out[f"{c.name}.mul"] = rec(c.d_prefix(n), ext, ks)
    return out


# ------------------------------------------------------------------ the families, by name
FAMILIES = {}
for _f in ("p25519", "l25519"):
    FAMILIES[f"{_f}.generic"] = functools.partial(fam_field, _f)
    FAMILIES[f"{_f}.above_modulus"] = functools.partial(fam_above_modulus, _f)
FAMILIES["l25519.wide"] = fam_wide_l
FAMILIES["consts"] = fam_consts
for _c in CURVES:
    FAMILIES[f"{_c}.group"] = functools.partial(fam_group, _c)
    FAMILIES[f"{_c}.fixed_sweep"] = functools.partial(fam_fixed_sweep, _c)
FAMILIES["sha512"] = fam_sha512
FAMILIES["ed25519.scalars"] = fam_ed25519_scalars
FAMILIES["ed25519.points"] = fam_ed25519_points
FAMILIES["jubjub.roots"] = fam_jubjub_roots


@functools.lru_cache(maxsize=None)
def family(name):
    return FAMILIES[name]()


def run_family(backend, name):
    fails = {}
    for case in family(name):
        bad = case.bad(backend.run(case.op, case.inp))
        if bad:
            fails[case.op] = (len(bad), len(case.inp), bad[:4])
    return fails
