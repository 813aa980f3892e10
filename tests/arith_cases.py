"""Edge-case generator and big-integer reference for the field and group-law conformance harness (test infrastructure).

`tests/devshim/arith.cu` runs one op per record; this module builds it (host and sm_90a), packs the case families
below into records, and checks what comes back against plain Python integers (`oracle/py/field.py`, `curve.py`,
`bellman_params.py`).

Field cases are limb IMAGES: the words the kernel reads are exactly the integers listed here, so the carry, borrow and
reduction edges are edges of the bits the arithmetic sees.  An image v stands for the field value v / R.  Everything
is seeded and deterministic; `COUNTS` records how many cases of each kind a family holds, and the tests assert them.
"""
import ctypes as ct
import functools
import itertools
import os
import random
import subprocess
import tempfile

import numpy as np

from oracle.py import bellman_params as BP, curve as C, field as Fd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bazuka_b200", "csrc")
SHIM = os.path.join(ROOT, "tests", "devshim")
SRC = os.path.join(SHIM, "arith.cu")
DEPS = [SRC] + [os.path.join(CSRC, h) for h in ("ff.cuh", "ec.cuh")]

# ------------------------------------------------------------------ op table (mirrors the enums of arith.cu)
FIELDS = {"fr": (Fd.R_MOD, 8, 0), "fp": (Fd.P_MOD, 12, 1)}   # name -> (modulus, 32-bit limbs, type code)
DOT_MAX = 17
_FIELD_KINDS = ["add", "sub", "mul", "neg", "dbl", "sqr", "to_mont", "from_mont", "from_u32", "pow", "inv", "inv_gcd",
                "mul_wide", "dot", "redc_wide", "reduce_once"]
_FP2_KINDS = ["add", "sub", "mul", "neg", "dbl", "sqr", "inv"]
_GROUP_KINDS = ["madd", "add", "dbl", "dbl_affine", "to_affine", "scalar_mul", "pair", "on_curve"]


def _ops():
    ops = {}
    for f, (_, n, t) in FIELDS.items():
        w = {"add": (2 * n, n), "sub": (2 * n, n), "mul": (2 * n, n), "from_u32": (1, n), "pow": (2 * n, n),
             "mul_wide": (2 * n, 2 * n), "dot": (1 + 2 * DOT_MAX * n, n), "redc_wide": (2 * n + 1, n)}
        for k, name in enumerate(_FIELD_KINDS):
            ops[f"{f}.{name}"] = ((t << 4) | k, *w.get(name, (n, n)))
    for k, name in enumerate(_FP2_KINDS):
        ops[f"fp2.{name}"] = ((2 << 4) | k, 48 if k <= 2 else 24, 24)
    for g, t, fw in (("g1", 3, 12), ("g2", 4, 24)):
        a, x = 2 * fw, 4 * fw
        w = {"madd": (x + a, x), "add": (2 * x, x), "dbl": (x, x), "dbl_affine": (a, x), "to_affine": (x, a),
             "scalar_mul": (a + 8, x), "pair": (2 * a, fw + a), "on_curve": (a, 1)}
        for k, name in enumerate(_GROUP_KINDS):
            ops[f"{g}.{name}"] = ((t << 4) | k, *w[name])
    return ops


OPS = _ops()


# ------------------------------------------------------------------ builds
def _stale(out):
    return not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in DEPS)


def _compile(cmd_without_out, out):
    """compile to a temporary name and rename, so that a concurrent session never loads a half-written library"""
    fd, tmp = tempfile.mkstemp(suffix=".so", dir=SHIM)
    os.close(fd)
    try:
        r = subprocess.run(cmd_without_out + ["-o", tmp], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"{cmd_without_out[0]} failed on {SRC}:\n{r.stdout}\n{r.stderr}")
        os.replace(tmp, out)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    return out


def build_host(device_text):
    """g++ build: the device text (mul_evenodd, add/sub_limbs32, explicit carries) or the host fast paths"""
    out = os.path.join(SHIM, "_arith_host_dt.so" if device_text else "_arith_host.so")
    if _stale(out):
        _compile(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++"] + (["-DBZK_HOST_DEVICE_TEXT"] if device_text else []) +
                 ["-I", CSRC, SRC], out)
    return out


def build_dev():
    """nvcc build with libbzk's own compiler and flags (sm_90a)"""
    from bazuka_b200 import build as B
    out = os.path.join(SHIM, "_arith_dev.so")
    if _stale(out):
        _compile([B.NVCC] + B.FLAGS + ["-shared", "-I", CSRC, SRC], out)
    return out


class HostArith:
    def __init__(self, device_text):
        self.lib = ct.CDLL(build_host(device_text))
        self.lib.arith_run_host.argtypes = [ct.c_int, ct.c_void_p, ct.c_int, ct.c_void_p, ct.c_int, ct.c_size_t]

    def run(self, op, inp):
        code, in_w, out_w = OPS[op]
        inp = np.ascontiguousarray(inp, dtype=np.uint32).reshape(-1, in_w)
        out = np.zeros((len(inp), out_w), dtype=np.uint32)
        self.lib.arith_run_host(code, inp.ctypes.data, in_w, out.ctypes.data, out_w, len(inp))
        return out


class DevArith:
    """one thread per record; the block size never divides the record count, so every launch has a partial block"""

    def __init__(self):
        self.lib = ct.CDLL(build_dev())
        self.lib.arith_run_dev.argtypes = [ct.c_int, ct.c_void_p, ct.c_int, ct.c_void_p, ct.c_int, ct.c_size_t, ct.c_int]
        self.blocks = []

    def run(self, op, inp):
        import torch
        code, in_w, out_w = OPS[op]
        inp = np.ascontiguousarray(inp, dtype=np.uint32).reshape(-1, in_w)
        n = len(inp)
        block = 127 if n % 127 else 113
        d_in = torch.from_numpy(inp.view(np.int32)).cuda()
        d_out = torch.full((n + 1, out_w), -1, dtype=torch.int32, device="cuda")   # one guard record past the end
        torch.cuda.synchronize()
        e = self.lib.arith_run_dev(code, d_in.data_ptr(), in_w, d_out.data_ptr(), out_w, n, block)
        assert e == 0, f"{op}: cudaError {e}"
        out = d_out.cpu().numpy().view(np.uint32)
        assert (out[n] == 0xFFFFFFFF).all(), f"{op}: wrote past the last record"
        self.blocks.append((n, block))
        return out[:n]


# ------------------------------------------------------------------ packing
def words(vals, nw):
    """integers -> (len, nw) little-endian 32-bit words"""
    return np.frombuffer(b"".join(int(v).to_bytes(4 * nw, "little") for v in vals), dtype=np.uint32).reshape(-1, nw).copy()


def ints(arr):
    """(len, nw) words -> integers"""
    arr = np.ascontiguousarray(arr, dtype=np.uint32)
    return [int.from_bytes(r.tobytes(), "little") for r in arr]


def rec(*cols):
    return np.concatenate([np.asarray(c, dtype=np.uint32).reshape(len(cols[0]), -1) for c in cols], axis=1)


class Case:
    """one op over a batch of records, with the expected output words (exact) or a checker returning bad indices"""

    def __init__(self, op, inp, want=None, check=None):
        self.op, self.inp, self.want, self.check = op, inp, want, check

    def bad(self, out):
        if self.check is not None:
            return self.check(out)
        return [int(i) for i in np.nonzero((out != self.want).any(axis=1))[0]]


COUNTS = {}


def _count(key, n):
    COUNTS[key] = COUNTS.get(key, 0) + n


# ------------------------------------------------------------------ field helpers
class _F:
    def __init__(self, name):
        self.name = name
        self.p, self.n, _ = FIELDS[name]
        self.R = 1 << (32 * self.n)
        self.Rm = self.R % self.p
        self.Rinv = pow(self.Rm, -1, self.p)

    def val(self, img):
        return img * self.Rinv % self.p

    def img(self, v):
        return v % self.p * self.Rm % self.p

    def w(self, vals):
        return words(vals, self.n)


def structured(f):
    """the limb-pattern set: every limb position holding one of ALPHA with the other limbs all 0 or all ones, 2^(32k) - 1,
    p +- 2^(32k), the small and half-way values, and R, R^2, R^-1, p - R (mod p); all reduced mod p"""
    p, n = f.p, f.n
    ones = f.R - 1
    s = {0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, f.Rm, f.Rm * f.Rm % p, f.Rinv, p - f.Rm}
    for k in range(n):
        for a in ALPHA:
            s.add(a << (32 * k))
            s.add(ones ^ ((0xFFFFFFFF ^ a) << (32 * k)))
        s.add((1 << (32 * (k + 1))) - 1)
        s.add(p + (1 << (32 * k)))
        s.add(p - (1 << (32 * k)))
    return sorted({v % p for v in s})


ALPHA = (0, 1, 2, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF)


def _exact(f, op, a_imgs, b_imgs, fn):
    inp = rec(f.w(a_imgs), f.w(b_imgs)) if b_imgs is not None else f.w(a_imgs)
    want = f.w([fn(*ab) for ab in (zip(a_imgs, b_imgs) if b_imgs is not None else ((a,) for a in a_imgs))])
    return Case(f"{f.name}.{op}", inp, want)


def _binops(f, pairs):
    p, Ri = f.p, f.Rinv
    a, b = [x for x, _ in pairs], [y for _, y in pairs]
    return [_exact(f, "add", a, b, lambda x, y: (x + y) % p),
            _exact(f, "sub", a, b, lambda x, y: (x - y) % p),
            _exact(f, "mul", a, b, lambda x, y: x * y * Ri % p),
            Case(f"{f.name}.mul_wide", rec(f.w(a), f.w(b)), words([x * y for x, y in pairs], 2 * f.n))]


# ------------------------------------------------------------------ field families
def fam_structured(name):
    f = _F(name)
    S = structured(f)
    _count(f"{name} structured values", len(S))
    pairs = list(itertools.product(S, S))
    _count(f"{name} structured pairs", len(pairs))
    p, Ri = f.p, f.Rinv
    cases = _binops(f, pairs)
    cases += [_exact(f, "neg", S, None, lambda x: (-x) % p),
              _exact(f, "dbl", S, None, lambda x: 2 * x % p),
              _exact(f, "sqr", S, None, lambda x: x * x * Ri % p),
              _exact(f, "to_mont", S, None, lambda x: x * f.Rm % p),   # S read as canonical values here
              _exact(f, "from_mont", S, None, lambda x: x * Ri % p)]
    # reduce_once over its whole contract (a < 2p): S and S + p
    lifted = S + [x + p for x in S]
    cases.append(_exact(f, "reduce_once", lifted, None, lambda x: x % p))
    return cases


def fam_sums(name):
    """add/sub pairs whose sum is p-1, p, p+1, 2p-2, and carry / borrow runs of every length from every limb"""
    f = _F(name)
    p, n = f.p, f.n
    rnd = random.Random(1000 + n)
    S = structured(f)
    pairs = []
    for target in (p - 1, p, p + 1):
        got = 0
        for a in S + [rnd.randrange(p) for _ in range(64)]:
            b = target - a
            if 0 <= b < p:
                pairs.append((a, b))
                got += 1
        _count(f"{name} sum = {'p' if target == p else ('p-1' if target < p else 'p+1')}", got)
    pairs.append((p - 1, p - 1))
    _count(f"{name} sum = 2p-2", 1)
    ptop = p >> (32 * (n - 1))

    def base():   # random, with a top limb below p's so that the value stays below p
        return rnd.randrange(1 << (32 * (n - 1))) | (rnd.randrange(ptop) << (32 * (n - 1)))
    runs = 0
    for s in range(n - 1):
        for L in range(1, n - s):          # the run occupies limbs s .. s+L-1 and ends in limb s+L <= n-1
            for _ in range(2):
                mask = ((1 << (32 * L)) - 1) << (32 * s)
                lo = rnd.randrange(1, 1 << 32) << (32 * s)
                # carry run: a's run limbs all ones, b's run limbs zero except a nonzero limb s
                a = base() | mask
                b = (base() & ~mask) | lo
                pairs.append((a % p, b % p))
                # borrow run: a's run limbs zero, b's limb s nonzero and the rest of its run zero
                a2 = base() & ~mask
                b2 = (base() & ~mask) | lo
                pairs.append((a2 % p, b2 % p))
                runs += 1
    _count(f"{name} carry/borrow runs", runs)
    cases = _binops(f, pairs + [(b, a) for a, b in pairs])
    return cases


def mont_boundary(f, want=150, seed=7):
    """(a, b) whose unreduced CIOS value t = (ab + mp)/R lies in [p, p + 2^32) ('above') or [p - 2^32, p) ('below'):
    b = c R a^-1 for targets c next to 0 and next to p"""
    p, R = f.p, f.R
    pinv = (-pow(p, -1, R)) % R
    rnd = random.Random(seed + f.n)
    above, below = [], []
    tries = 0
    while (len(above) < want or len(below) < want) and tries < 100000:
        tries += 1
        a = rnd.randrange(1, p)
        small = rnd.randrange(3, 1 << 32)
        c = rnd.choice([0, 1, 2, small, p - 1, p - 2, p - small])
        b = c * R * pow(a, -1, p) % p
        t = (a * b + (a * b * pinv % R) * p) // R
        if p <= t < p + (1 << 32) and len(above) < want:
            above.append((a, b))
        elif p - (1 << 32) <= t < p and len(below) < want:
            below.append((a, b))
    return above, below


def fam_mont_boundary(name):
    f = _F(name)
    above, below = mont_boundary(f)
    _count(f"{name} Montgomery t in [p, p+2^32)", len(above))
    _count(f"{name} Montgomery t in [p-2^32, p)", len(below))
    pairs = above + below
    return _binops(f, pairs + [(b, a) for a, b in pairs])


def fam_lazy_dot(name):
    """mul_wide + wide_accumulate + redc_wide: t = 1..17 terms, all images p-1, all values p-1, all zero, mixed;
    redc_wide alone at the edges of its input bound T < p 2^(32(N+1))"""
    f = _F(name)
    p, n = f.p, f.n
    rnd = random.Random(55 + n)
    S = structured(f)
    recs, want = [], []
    for t in range(1, DOT_MAX + 1):
        for kind in ("img p-1", "val p-1", "zero", "mixed", "random"):
            if kind == "img p-1":
                m = s = [p - 1] * t
            elif kind == "val p-1":
                m = s = [f.img(p - 1)] * t
            elif kind == "zero":
                m = s = [0] * t
            elif kind == "mixed":
                m = [rnd.choice(S) for _ in range(t)]
                s = [rnd.choice(S) for _ in range(t)]
            else:
                m = [rnd.randrange(p) for _ in range(t)]
                s = [rnd.randrange(p) for _ in range(t)]
            pad = [0] * (DOT_MAX - t)
            recs.append(np.concatenate([np.array([t], dtype=np.uint32), f.w(m + pad).ravel(), f.w(s + pad).ravel()]))
            want.append(f.img(sum(f.val(x) * f.val(y) for x, y in zip(m, s))))
    _count(f"{name} lazy inner products", len(recs))
    cases = [Case(f"{name}.dot", np.stack(recs), f.w(want))]
    lim = p << (32 * (n + 1))
    Ts = [0, 1, lim - 1, lim - 2, lim >> 1, p, p * p, (p - 1) * (p - 1) * DOT_MAX, (1 << (32 * 2 * n)) - 1] + [rnd.randrange(lim) for _ in range(64)]
    Ts += [(k << (32 * (n + 1))) - 1 for k in (1, p - 1)] + [k << (32 * (n + 1)) for k in (1, p - 1)]
    Ts = [T for T in Ts if T < lim]
    inv_r1 = pow(1 << (32 * (n + 1)), -1, p)
    cases.append(Case(f"{name}.redc_wide", words(Ts, 2 * n + 1), f.w([T * inv_r1 % p for T in Ts])))
    return cases


def gcd_iterations(a, p):
    """loop trips (halvings + subtractions) of ff.cuh's binary extended Euclid on u = a, v = p"""
    u, v, it = a, p, 0
    while u != 1 and v != 1:
        while not u & 1:
            u >>= 1
            it += 1
        while not v & 1:
            v >>= 1
            it += 1
        if u >= v:
            u -= v
        else:
            v -= u
        it += 1
    return it


def fam_inverse(name):
    f = _F(name)
    p, n = f.p, f.n
    S = structured(f)
    vals = [0, 1, 2, p - 1] + [(1 << k) % p for k in range(32 * n)] + [((1 << k) - 1) % p for k in range(1, 32 * n + 1)] + S
    rnd = random.Random(77 + n)
    cand = sorted(((gcd_iterations(c, p), c) for c in (rnd.randrange(1, p) for _ in range(600))), reverse=True)
    worst = [c for _, c in cand[:16]]
    _count(f"{name} inversion operands", len(vals))
    _count(f"{name} binary-GCD longest (of 600 seeded)", cand[0][0])
    vals += worst
    R2 = f.Rm * f.Rm % p
    inv_img = lambda x: 0 if x == 0 else R2 * pow(x, -1, p) % p   # image of (x/R)^-1
    return [_exact(f, "inv", vals, None, inv_img), _exact(f, "inv_gcd", vals, None, inv_img)]


def fam_pow_u32(name):
    f = _F(name)
    p, n = f.p, f.n
    rnd = random.Random(99 + n)
    S = structured(f)
    base = S[::3] + [0, 1, p - 1]
    exps = [0, 1, 2, 3, p - 1, p - 2, (p - 1) // 2, f.R - 1, rnd.randrange(f.R)]
    pairs = [(a, e) for a in base for e in exps]
    want = [f.img(pow(f.val(a), e, p)) for a, e in pairs]
    u32 = list(ALPHA) + [3, 0x10000, rnd.randrange(1 << 32)]
    return [Case(f"{name}.pow", rec(f.w([a for a, _ in pairs]), f.w([e for _, e in pairs])), f.w(want)),
            Case(f"{name}.from_u32", np.array(u32, dtype=np.uint32).reshape(-1, 1), f.w([f.img(v) for v in u32]))]


# ------------------------------------------------------------------ Fp2
FP = _F("fp")


def fp2_operands():
    """components from the structured Fp set (images), with wrapping Karatsuba sums and c0 < c1, plus the edges"""
    p = FP.p
    S = structured(FP)
    E = [(0, 0), (0, 1), (1, 0), (p - 1, p - 1), (FP.Rm, 0), (0, FP.Rm)]
    sub = S[::4]
    E += [(0, c) for c in sub] + [(c, 0) for c in sub]
    E += [(S[i], S[(7 * i + 3) % len(S)]) for i in range(0, len(S), 2)]
    E = list(dict.fromkeys(E))
    _count("fp2 operands", len(E))
    _count("fp2 c0 + c1 >= p", sum(a + b >= p for a, b in E))
    _count("fp2 c0 < c1", sum(a < b for a, b in E))
    return E


def _f2_img(v):
    return (FP.img(v[0]), FP.img(v[1]))


def _f2_val(e):
    return (FP.val(e[0]), FP.val(e[1]))


def _f2w(es):
    return words([a | (b << 384) for a, b in es], 24)


def fam_fp2():
    p = FP.p
    E = fp2_operands()
    small = E[::3]
    pairs = list(itertools.product(small, small))
    _count("fp2 pairs", len(pairs))
    a, b = [x for x, _ in pairs], [y for _, y in pairs]
    binop = lambda fn: _f2w([_f2_img(fn(_f2_val(x), _f2_val(y))) for x, y in pairs])
    inv = lambda x: (0, 0) if x == (0, 0) else C.f2_inv(x)
    return [Case("fp2.add", rec(_f2w(a), _f2w(b)), binop(C.f2_add)),
            Case("fp2.sub", rec(_f2w(a), _f2w(b)), binop(C.f2_sub)),
            Case("fp2.mul", rec(_f2w(a), _f2w(b)), binop(C.f2_mul)),
            Case("fp2.neg", _f2w(E), _f2w([_f2_img(C.f2_neg(_f2_val(x))) for x in E])),
            Case("fp2.dbl", _f2w(E), _f2w([_f2_img(C.f2_add(_f2_val(x), _f2_val(x))) for x in E])),
            Case("fp2.sqr", _f2w(E), _f2w([_f2_img(C.f2_sqr(_f2_val(x))) for x in E])),
            Case("fp2.inv", _f2w(E), _f2w([_f2_img(inv(_f2_val(x))) for x in E]))]


# ------------------------------------------------------------------ points (canonical values; None = identity)
class _G:
    def __init__(self, name):
        self.name = name
        self.g2 = name == "g2"
        self.F = C.FP2 if self.g2 else C.FP
        self.fw = 24 if self.g2 else 12

    def fimg(self, v):
        return (FP.img(v[0]) | (FP.img(v[1]) << 384)) if self.g2 else FP.img(v)

    def fval(self, word_int):
        if self.g2:
            lo, hi = word_int & ((1 << 384) - 1), word_int >> 384
            return None if lo >= FP.p or hi >= FP.p else (FP.val(lo), FP.val(hi))
        return None if word_int >= FP.p else FP.val(word_int)

    def affine(self, pts):
        """identity -> x = y = 0"""
        z = self.F.zero
        return words([self.fimg(z) | (self.fimg(z) << (32 * self.fw)) if P is None else
                      self.fimg(P[0]) | (self.fimg(P[1]) << (32 * self.fw)) for P in pts], 2 * self.fw)

    def xyzz(self, pts, lams):
        """X = x l^2, Y = y l^3, ZZ = l^2, ZZZ = l^3; identity -> all zero, or 'inf1' -> X = Y = 1, ZZ = ZZZ = 0"""
        F, s = self.F, 32 * self.fw
        out = []
        for P, lam in zip(pts, lams):
            if P is None:
                parts = [F.zero] * 4 if lam != "inf1" else [F.one, F.one, F.zero, F.zero]
            else:
                l2 = F.mul(lam, lam)
                l3 = F.mul(l2, lam)
                parts = [F.mul(P[0], l2), F.mul(P[1], l3), l2, l3]
            out.append(sum(self.fimg(v) << (s * i) for i, v in enumerate(parts)))
        return words(out, 4 * self.fw)

    def check_xyzz(self, want):
        """output words -> bad indices: canonical limbs, ZZ^3 = ZZZ^2 when ZZ != 0, and the same group element as want"""
        F, fw = self.F, self.fw

        def check(out):
            bad = []
            for i, row in enumerate(np.ascontiguousarray(out)):
                X, Y, ZZ, ZZZ = (self.fval(int.from_bytes(row[k * fw:(k + 1) * fw].tobytes(), "little")) for k in range(4))
                if None in (X, Y, ZZ, ZZZ):
                    bad.append(i)
                    continue
                if ZZ == F.zero:
                    got = None
                else:
                    if ZZZ == F.zero or F.mul(F.mul(ZZ, ZZ), ZZ) != F.mul(ZZZ, ZZZ):
                        bad.append(i)
                        continue
                    got = (F.mul(X, F.inv(ZZ)), F.mul(Y, F.inv(ZZZ)))
                if got != want[i]:
                    bad.append(i)
            return bad
        return check


def _lams(F, rnd):
    if F is C.FP:
        return [1, FP.p - 1, 2, rnd.randrange(2, FP.p)]
    return [(1, 0), (FP.p - 1, 0), (2, 0), (rnd.randrange(FP.p), rnd.randrange(FP.p))]


@functools.lru_cache(maxsize=None)
def points(name):
    """random subgroup points, points lifted from edge abscissae (G1: the 3-torsion point (0, 2) among them), their
    negatives and doubles, and the identity"""
    g = _G(name)
    F = g.F
    rnd = random.Random(4242 if g.g2 else 4141)
    gen = C.G2_GEN if g.g2 else C.G1_GEN
    base = [C.mul(F, gen, rnd.randrange(1, Fd.R_MOD)) for _ in range(3)]
    p = FP.p
    if g.g2:
        S = structured(FP)
        xs = [(0, 0), (1, 0), (0, 1), (2, 0), (p - 1, 0), (p - 2, 0), (p - 1, p - 1), (0, p - 1)] + [(c, 0) for c in S[::25]] + [(0, c) for c in S[1::25]]
        lift = BP.g2_lift
    else:
        xs = [0, 1, 2, p - 1, p - 2] + structured(FP)
        lift = BP.g1_lift
    lifted = list(dict.fromkeys(P for P in (lift(x) for x in xs) if P is not None))
    _count(f"{name} lifted edge points", len(lifted))
    core = base + lifted[:6 if g.g2 else 8]
    pts = []
    for P in core:
        pts += [P, C.neg(F, P), C.add(F, P, P)]
    pts = list(dict.fromkeys(pts)) + [None]
    if not g.g2:
        assert (0, 2) in pts and (0, p - 2) in pts
        _count("g1 3-torsion points (0, +-2)", 2)
    _count(f"{name} points", len(pts))
    return pts, lifted


def fam_group(name):
    g = _G(name)
    F = g.F
    rnd = random.Random(9000 + g.fw)
    pts, lifted = points(name)
    lams = _lams(F, rnd)
    cases = []
    # madd: every accumulator (each point under each lambda, both identity encodings) + every affine point
    accs = [(P, lam) for P in pts for lam in (lams if P is not None else [F.zero, "inf1"])]
    mp = [(P, l, Q) for (P, l) in accs for Q in pts] + [(P, lams[3], Q) for P in lifted for Q in (P, C.neg(F, P))]
    cases.append(Case(f"{name}.madd", rec(g.xyzz([m[0] for m in mp], [m[1] for m in mp]), g.affine([m[2] for m in mp])),
                      check=g.check_xyzz([C.add(F, P, Q) for P, _, Q in mp])))
    _count(f"{name} madd records", len(mp))
    # add: both operands in XYZZ form with different lambdas
    ap = [(P, lams[i % 4], Q, lams[(i + j + 1) % 4]) for i, P in enumerate(pts) for j, Q in enumerate(pts)]
    ap = [(P, F.zero if P is None else l1, Q, "inf1" if Q is None else l2) for P, l1, Q, l2 in ap]
    cases.append(Case(f"{name}.add", rec(g.xyzz([a[0] for a in ap], [a[1] for a in ap]), g.xyzz([a[2] for a in ap], [a[3] for a in ap])),
                      check=g.check_xyzz([C.add(F, a[0], a[2]) for a in ap])))
    singles = pts + lifted
    one = [(P, lam) for P in singles for lam in (lams if P is not None else [F.zero, "inf1"])]
    cases.append(Case(f"{name}.dbl", g.xyzz([P for P, _ in one], [l for _, l in one]), check=g.check_xyzz([C.add(F, P, P) for P, _ in one])))
    cases.append(Case(f"{name}.dbl_affine", g.affine(singles), check=g.check_xyzz([C.add(F, P, P) for P in singles])))
    cases.append(Case(f"{name}.to_affine", g.xyzz([P for P, _ in one], [l for _, l in one]), g.affine([P for P, _ in one])))
    # scalar_mul: plain 256-bit scalars, not reduced (the points are not all in the subgroup)
    ks = [0, 1, 2, 3, Fd.R_MOD - 1, Fd.R_MOD, Fd.R_MOD + 1, (1 << 256) - 1, rnd.randrange(1 << 256)]
    if g.g2:   # the big-integer reference is slow on Fp2: every point with three of the scalars
        sm = [(P, k) for i, P in enumerate(pts[::2] + [None]) for k in (ks[i % len(ks)], 3, Fd.R_MOD)]
    else:
        sm = [(P, k) for P in pts for k in ks]
    cases.append(Case(f"{name}.scalar_mul", rec(g.affine([P for P, _ in sm]), words([k for _, k in sm], 8)),
                      check=g.check_xyzz([C.mul(F, P, k) for P, k in sm])))
    _count(f"{name} scalar_mul records", len(sm))
    # pair_denominator + pair_sum over every affine pair
    pp = list(itertools.product(pts, pts))
    den = []
    for P, Q in pp:
        if P is None or Q is None:
            d = F.one
        elif P[0] != Q[0]:
            d = F.sub(Q[0], P[0])
        elif P[1] == Q[1] and P[1] != F.zero:
            d = F.add(P[1], P[1])
        else:
            d = F.one
        den.append(d)
    want = rec(words([g.fimg(d) for d in den], g.fw), g.affine([C.add(F, P, Q) for P, Q in pp]))
    cases.append(Case(f"{name}.pair", rec(g.affine([P for P, _ in pp]), g.affine([Q for _, Q in pp])), want))
    # on_curve: the points, their y + 1 (off the curve), and (0, 0)
    off = [(P[0], F.add(P[1], F.one)) for P in singles if P is not None]
    oc = [P for P in singles if P is not None] + off + [None]
    cases.append(Case(f"{name}.on_curve", g.affine(oc), words([0 if P is None else int(C.on_curve(F, P)) for P in oc], 1)))
    return cases


# ------------------------------------------------------------------ the families, by name
FAMILIES = {}
for _f in FIELDS:
    for _kind, _fn in (("structured", fam_structured), ("sums", fam_sums), ("mont_boundary", fam_mont_boundary),
                       ("lazy_dot", fam_lazy_dot), ("inverse", fam_inverse), ("pow_u32", fam_pow_u32)):
        FAMILIES[f"{_f}.{_kind}"] = functools.partial(_fn, _f)
FAMILIES["fp2"] = fam_fp2
FAMILIES["g1"] = functools.partial(fam_group, "g1")
FAMILIES["g2"] = functools.partial(fam_group, "g2")


@functools.lru_cache(maxsize=None)
def family(name):
    return FAMILIES[name]()


def run_family(backend, name):
    """every case of a family through one backend; returns {op: first bad records} for the ops that disagree"""
    fails = {}
    for case in family(name):
        bad = case.bad(backend.run(case.op, case.inp))
        if bad:
            fails[case.op] = (len(bad), len(case.inp), bad[:4])
    return fails
