"""Seeded input families and big-integer references for the pairing conformance harness (test infrastructure).

`tests/devshim/pairing.cu` runs one op of csrc/pairing.cuh (or one per-proof step of verify.cu's k_verify_miller) per
record; this module builds it three ways (sm_90a, g++ on the device text, g++ on the host fast paths), packs the families
below into records and states what comes back: Fp12 products exactly (a schoolbook product over Fp2[w] / (w^6 - xi) in
Python integers), [r mod 2^127] A as a group element, and the malformed-proof predicate from the encoding contract.  The
Miller loop has no closed form; its builds are compared with each other and, through the final exponentiation, with the
host verifier's multi_miller and with the oracle's pairing.  Everything is seeded and deterministic.
"""
import ctypes as ct
import functools
import os
import random

import numpy as np

import arith_cases as AC
from arith_cases import FP, Case, rec, words
from oracle.py import bellman_params as BP, curve as C, field as Fd

ROOT = AC.ROOT
CSRC = AC.CSRC
SHIM = AC.SHIM
SRC = os.path.join(SHIM, "pairing.cu")
DEPS = [SRC] + [os.path.join(CSRC, h) for h in ("ff.cuh", "ec.cuh", "pairing.cuh")]
P = Fd.P_MOD

F12_W, F2_W, G1A_W, G1X_W, G2A_W = 144, 24, 24, 48, 48
# op -> (code, in words, out words); mirrors the enum of pairing.cu
OPS = {
    "f12_mul": (0, 2 * F12_W, F12_W),
    "f12_sqr": (1, F12_W, F12_W),
    "f12_mul_sparse": (2, F12_W + 3 * F2_W, F12_W),
    "miller_xyzz": (3, G1X_W + G2A_W, F12_W),
    "mul127": (4, G1A_W + 8, G1X_W),
    "proof_check": (5, 97, 1),
    "multi_miller": (6, G1A_W + G2A_W, F12_W),
    "final_exp": (7, F12_W, F12_W),
}
HOST_ONLY = ("multi_miller", "final_exp")


# ------------------------------------------------------------------ builds
def _stale(out):
    return not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in DEPS)


def _compile(cmd, out):
    saved = AC.SRC
    AC.SRC = SRC     # only used in the error message
    try:
        return AC._compile(cmd, out)
    finally:
        AC.SRC = saved


def build_host(device_text):
    out = os.path.join(SHIM, "_pairing_host_dt.so" if device_text else "_pairing_host.so")
    if _stale(out):
        _compile(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++"] + (["-DBZK_HOST_DEVICE_TEXT"] if device_text else []) +
                 ["-I", CSRC, SRC], out)
    return out


def build_dev():
    from bazuka_b200 import build as B
    out = os.path.join(SHIM, "_pairing_dev.so")
    if _stale(out):
        _compile([B.NVCC] + B.FLAGS + ["-shared", "-I", CSRC, SRC], out)
    return out


class HostPairing:
    def __init__(self, device_text):
        self.lib = ct.CDLL(build_host(device_text))
        self.lib.pairing_run_host.argtypes = [ct.c_int, ct.c_void_p, ct.c_int, ct.c_void_p, ct.c_int, ct.c_size_t]

    def run(self, op, inp):
        code, in_w, out_w = OPS[op]
        inp = np.ascontiguousarray(inp, dtype=np.uint32).reshape(-1, in_w)
        out = np.zeros((len(inp), out_w), dtype=np.uint32)
        self.lib.pairing_run_host(code, inp.ctypes.data, in_w, out.ctypes.data, out_w, len(inp))
        return out


class DevPairing:
    """one thread per record, 64-thread blocks as k_verify_miller's, with a guard record past the end"""

    def __init__(self):
        self.lib = ct.CDLL(build_dev())
        self.lib.pairing_run_dev.argtypes = [ct.c_int, ct.c_void_p, ct.c_int, ct.c_void_p, ct.c_int, ct.c_size_t, ct.c_int]

    def run(self, op, inp):
        import torch
        code, in_w, out_w = OPS[op]
        inp = np.ascontiguousarray(inp, dtype=np.uint32).reshape(-1, in_w)
        n = len(inp)
        d_in = torch.from_numpy(inp.view(np.int32)).cuda()
        d_out = torch.full((n + 1, out_w), -1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        e = self.lib.pairing_run_dev(code, d_in.data_ptr(), in_w, d_out.data_ptr(), out_w, n, 64)
        assert e == 0, f"{op}: cudaError {e}"
        out = d_out.cpu().numpy().view(np.uint32)
        assert (out[n] == 0xFFFFFFFF).all(), f"{op}: wrote past the last record"
        return out[:n]


# ------------------------------------------------------------------ Fp12 over Fp2[w] / (w^6 - xi), canonical values
def _xi(a):
    return ((a[0] - a[1]) % P, (a[0] + a[1]) % P)


def f12_mul(a, b):
    t = [(0, 0)] * 11
    for i in range(6):
        for j in range(6):
            t[i + j] = C.f2_add(t[i + j], C.f2_mul(a[i], b[j]))
    return [C.f2_add(t[k], _xi(t[k + 6])) for k in range(5)] + [t[5]]


def sparse(l0, l2, l3):
    return [l0, (0, 0), l2, l3, (0, 0), (0, 0)]


def f12_img(v):
    """6 Fp2 values -> 144 words"""
    return words([sum(FP.img(c) << (384 * i) for i, c in enumerate((x for f2 in v for x in f2)))], F12_W)[0]


def f12_val(w):
    vals = [FP.val(x) for x in AC.ints(np.asarray(w, dtype=np.uint32).reshape(12, 12))]
    return [(vals[2 * k], vals[2 * k + 1]) for k in range(6)]


def f12_to_oracle(w):
    """product Fp12 words -> the oracle's degree-12 polynomial in w (u = w^6 - 1)"""
    v = [0] * 12
    for k, (a, b) in enumerate(f12_val(w)):
        v[k] = (v[k] + a - b) % P
        v[k + 6] = (v[k + 6] + b) % P
    return v


def f2_img(v):
    return words([FP.img(v[0]) | (FP.img(v[1]) << 384)], F2_W)[0]


# ------------------------------------------------------------------ operand families
COUNTS = {}


def _count(key, n):
    COUNTS[key] = COUNTS.get(key, 0) + n


def fp_edges():
    """coefficient values: 0, 1, p-1, and the values whose Montgomery images are p-1, p-2 and 1 (next to p and to 0)"""
    return [0, 1, P - 1, FP.val(P - 1), FP.val(P - 2), FP.val(1)]


@functools.lru_cache(maxsize=None)
def f12_operands():
    rnd = random.Random(1212)
    E = fp_edges()
    ops = [[(0, 0)] * 6, [(1, 0)] + [(0, 0)] * 5]
    for e in E[2:]:
        ops.append([(e, e)] * 6)                                         # every coefficient at the edge
    for k in range(6):                                                  # one coefficient, each position of the fold
        for c in ((P - 1, 0), (0, P - 1), (FP.val(P - 1), FP.val(P - 1))):
            z = [(0, 0)] * 6
            z[k] = c
            ops.append(z)
    for _ in range(14):
        ops.append([(rnd.choice(E), rnd.choice(E)) for _ in range(6)])
    for _ in range(6):
        ops.append([(rnd.randrange(P), rnd.randrange(P)) for _ in range(6)])
    _count("f12 operands", len(ops))
    return ops


@functools.lru_cache(maxsize=None)
def sparse_lines():
    """(l0, l2, l3) with each of them zero in turn, at the edge values and at random"""
    rnd = random.Random(1313)
    E = fp_edges()
    f2 = lambda: (rnd.choice(E), rnd.choice(E)) if rnd.random() < 0.6 else (rnd.randrange(P), rnd.randrange(P))
    out = []
    for zero in (None, 0, 1, 2, (0, 1), (1, 2)):
        for _ in range(4):
            L = [f2(), f2(), f2()]
            for z in (zero if isinstance(zero, tuple) else (zero,)):
                if z is not None:
                    L[z] = (0, 0)
            out.append(tuple(L))
    _count("sparse lines with a zero part", sum(any(x == (0, 0) for x in L) for L in out))
    return out


def fam_f12():
    ops = f12_operands()
    pairs = [(a, b) for i, a in enumerate(ops) for j, b in enumerate(ops) if (i + 2 * j) % 3 == 0 or i < 8 or j < 8]
    _count("f12 product pairs", len(pairs))
    mul = Case("f12_mul", np.stack([np.concatenate([f12_img(a), f12_img(b)]) for a, b in pairs]),
               np.stack([f12_img(f12_mul(a, b)) for a, b in pairs]))
    sqr = Case("f12_sqr", np.stack([f12_img(a) for a in ops]), np.stack([f12_img(f12_mul(a, a)) for a in ops]))
    sp = [(a, L) for a in ops for L in sparse_lines()[::2]] + [(ops[-1], L) for L in sparse_lines()[1::2]]
    _count("f12 sparse products", len(sp))
    msp = Case("f12_mul_sparse", np.stack([np.concatenate([f12_img(a)] + [f2_img(x) for x in L]) for a, L in sp]),
               np.stack([f12_img(f12_mul(a, sparse(*L))) for a, L in sp]))
    return [mul, sqr, msp]


# ------------------------------------------------------------------ points
G1 = AC._G("g1")
G2 = AC._G("g2")


@functools.lru_cache(maxsize=None)
def g1_points():
    """subgroup points: the generator, random multiples and their negatives"""
    rnd = random.Random(4343)
    base = [C.G1_GEN] + [C.mul(C.FP, C.G1_GEN, rnd.randrange(1, Fd.R_MOD)) for _ in range(2)]
    return base + [C.neg(C.FP, base[1])]


@functools.lru_cache(maxsize=None)
def g2_points():
    """(subgroup points, on-curve twist points outside the r-torsion)"""
    rnd = random.Random(4444)
    base = [C.G2_GEN] + [C.mul(C.FP2, C.G2_GEN, rnd.randrange(1, Fd.R_MOD)) for _ in range(2)]
    sub = base + [C.neg(C.FP2, base[1])]
    off = []
    x = 1
    while len(off) < 3:
        Q = BP.g2_lift((x, 7 * x + 3))
        if Q is not None and not BP.in_subgroup(C.FP2, Q):
            off.append(Q)
        x += 1
    _count("g2 twist points outside the r-torsion", len(off))
    return sub, off


def lambdas():
    rnd = random.Random(4545)
    return [1, rnd.randrange(2, P), rnd.randrange(2, P)]


@functools.lru_cache(maxsize=None)
def miller_records():
    """(P or None, lambda, Q or None, in_torsion): P in XYZZ form under lambda = 1 (ZZ = ZZZ = 1) and random lambda"""
    sub, off = g2_points()
    recs = []
    for Pt in g1_points() + [None]:
        for lam in (lambdas() if Pt is not None else [0]):
            for Q in sub + [None]:
                recs.append((Pt, lam, Q, True))
            for Q in off:
                recs.append((Pt, lam, Q, False))
    _count("miller records", len(recs))
    _count("miller records with ZZ*ZZZ != 1", sum(1 for r in recs if r[0] is not None and r[1] != 1))
    return recs


def miller_inputs(recs):
    xs = G1.xyzz([r[0] for r in recs], [r[1] for r in recs])
    return rec(xs, G2.affine([r[2] for r in recs]))


def fam_miller():
    """host-vs-device only: no closed form for the unreduced Miller value"""
    return [Case("miller_xyzz", miller_inputs(miller_records()), check=lambda out: [])]


# multipliers: bit 126 set, small, 0, 1, 2^127 - 1, and values with bits 127.. set (mul127 ignores them)
def multipliers():
    rnd = random.Random(4646)
    ks = [0, 1, 2, 3, (1 << 126), (1 << 127) - 1, (1 << 126) | 1, 0xFFFF, 0x10000, (1 << 127), (1 << 128) + 5, Fd.R_MOD - 1]
    ks += [rnd.randrange(1 << 126, 1 << 127) for _ in range(3)] + [rnd.randrange(1 << 16) for _ in range(2)]
    return ks


@functools.lru_cache(maxsize=None)
def g1_off_subgroup():
    """on-curve G1 points outside the prime-order subgroup: a lifted point of large order and the 3-torsion (0, 2)"""
    out = []
    x = 5
    while len(out) < 2:
        Q = BP.g1_lift(x)
        if Q is not None and not BP.in_subgroup(C.FP, Q):
            out.append(Q)
        x += 1
    return out + [(0, 2)]


def fam_mul127():
    pts = g1_points() + g1_off_subgroup() + [None]
    mp = [(Pt, k) for Pt in pts for k in multipliers()]
    _count("mul127 records", len(mp))
    _count("mul127 multipliers with bit 126 set", sum(1 for _, k in mp if (k >> 126) & 1))
    inp = rec(G1.affine([Pt for Pt, _ in mp]), words([k for _, k in mp], 8))
    return [Case("mul127", inp, check=G1.check_xyzz([C.mul(C.FP, Pt, k % (1 << 127)) for Pt, k in mp]))]


# ------------------------------------------------------------------ proof images (387 bytes) and the encoding contract
def fp_bytes(v_img):
    return int(v_img).to_bytes(48, "little")


def g1_wire(Pt, flag=None):
    if Pt is None:
        return bytes(96) + bytes([1 if flag is None else flag])
    return fp_bytes(FP.img(Pt[0])) + fp_bytes(FP.img(Pt[1])) + bytes([0 if flag is None else flag])


def g2_wire(Q, flag=None):
    if Q is None:
        return bytes(192) + bytes([1 if flag is None else flag])
    (x0, x1), (y0, y1) = Q
    return b"".join(fp_bytes(FP.img(v)) for v in (x0, x1, y0, y1)) + bytes([0 if flag is None else flag])


# (offset of each Fp coordinate in a 387-byte proof, the point it belongs to)
COORDS = {"A.x": 0, "A.y": 48, "B.x0": 97, "B.x1": 145, "B.y0": 193, "B.y1": 241, "C.x": 290, "C.y": 338}
FLAGS = {"A": 96, "B": 289, "C": 386}


def _on_curve_img(F, coords):
    """the point of a list of Fp images (all < p) satisfies its curve equation"""
    v = [FP.val(c) for c in coords]
    if len(v) == 2:
        return C.on_curve(C.FP, (v[0], v[1]))
    return C.on_curve(C.FP2, ((v[0], v[1]), (v[2], v[3])))


def contract_malformed(proof):
    """the encoding contract of every verifier entry point: a point whose flag byte is nonzero is the identity, whatever its
    coordinates; otherwise each coordinate must be a canonical Montgomery image (< p), (0, 0) is the identity, and any
    other point must satisfy its curve equation.  Subgroup membership is not part of it."""
    b = bytes(proof)
    for name, fl, offs in (("A", 96, (0, 48)), ("B", 289, (97, 145, 193, 241)), ("C", 386, (290, 338))):
        if b[fl]:
            continue
        imgs = [int.from_bytes(b[o:o + 48], "little") for o in offs]
        if any(v >= P for v in imgs):
            return True
        if all(v == 0 for v in imgs):
            continue
        if not _on_curve_img(None, imgs):
            return True
    return False


@functools.lru_cache(maxsize=None)
def proof_images():
    """well-formed proofs of random subgroup points, and each encoding edge applied to them: (name, 387 bytes)"""
    rnd = random.Random(4747)
    sub2, off2 = g2_points()
    g1 = g1_points()
    base = [g1_wire(g1[i % 4]) + g2_wire(sub2[(i + 1) % 4]) + g1_wire(g1[(i + 2) % 4]) for i in range(4)]
    out = [("valid", b) for b in base]
    b0 = bytearray(base[1])
    for name, at in COORDS.items():
        v = int.from_bytes(b0[at:at + 48], "little")
        t = bytearray(b0)
        t[at:at + 48] = (v + P).to_bytes(48, "little")
        out.append((f"{name} + p", bytes(t)))
        for word in range(12):
            t = bytearray(b0)
            bit = rnd.randrange(32)
            t[at + 4 * word + bit // 8] ^= 1 << (bit % 8)
            out.append((f"{name} word {word} bit {bit}", bytes(t)))
        t = bytearray(b0)
        t[at:at + 48] = P.to_bytes(48, "little")
        out.append((f"{name} = p", bytes(t)))
    for pt, fl in FLAGS.items():
        lo = {"A": 0, "B": 97, "C": 290}[pt]
        for flag in (1, 2, 0x80, 0xFF):
            t = bytearray(b0)
            t[fl] = flag
            out.append((f"{pt} flag {flag:#x}, coordinates kept", bytes(t)))
            t[lo:fl] = bytes(fl - lo)
            out.append((f"{pt} flag {flag:#x}, coordinates zero", bytes(t)))
            t[lo:lo + 48] = (P + 1).to_bytes(48, "little")
            out.append((f"{pt} flag {flag:#x}, coordinates non-canonical", bytes(t)))
        t = bytearray(b0)
        t[lo:fl + 1] = bytes(fl + 1 - lo)
        out.append((f"{pt} (0, 0) flag clear", bytes(t)))
    g1off = g1_off_subgroup()
    for i, Q in enumerate(g1off):
        t = bytearray(b0)
        t[0:97] = g1_wire(Q)
        out.append((f"A off-subgroup {i}", bytes(t)))
        t = bytearray(b0)
        t[290:387] = g1_wire(Q)
        out.append((f"C off-subgroup {i}", bytes(t)))
    for i, Q in enumerate(off2):
        t = bytearray(b0)
        t[97:290] = g2_wire(Q)
        out.append((f"B off-subgroup {i}", bytes(t)))
    _count("proof images", len(out))
    _count("proof images with a non-canonical coordinate", sum(1 for n, _ in out if "+ p" in n or "= p" in n or "non-canonical" in n))
    return out


def fam_proof_check():
    imgs = proof_images()
    inp = np.stack([np.frombuffer(b + b"\0", dtype=np.uint32) for _, b in imgs])
    want = np.array([[1 if contract_malformed(b) else 0] for _, b in imgs], dtype=np.uint32)
    return [Case("proof_check", inp, want)]


FAMILIES = {"f12": fam_f12, "miller": fam_miller, "mul127": fam_mul127, "proof_check": fam_proof_check}


@functools.lru_cache(maxsize=None)
def family(name):
    return FAMILIES[name]()


def run_family(backend, name):
    """every case of a family through one backend: ({op: first bad records}, {op: output words})"""
    fails, outs = {}, {}
    for case in family(name):
        out = backend.run(case.op, case.inp)
        outs[case.op] = out
        bad = case.bad(out)
        if bad:
            fails[case.op] = (len(bad), len(case.inp), bad[:4])
    return fails, outs
