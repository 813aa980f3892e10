"""Adversarial proof batches for the Groth16 verifier's entry points (test infrastructure).

The circuits (any number of public inputs, each bound into a constraint), the tamper families applied to one proof of
an otherwise valid batch, direct ctypes calls to the five entry points (so that n = 0 inputs and a null `ok_each` can be
passed), and a restatement of verify.cu's SplitMix64 multipliers with seeds chosen to reach their edges.
"""
import ctypes as ct
import functools

import numpy as np

from conftest import fr_arr
from oracle.py import bellman_params as BP, curve as C, field as Fd, groth16 as G
import pairing_cases as PC

P = Fd.P_MOD
M64 = (1 << 64) - 1
GAMMA = 0x9E3779B97F4A7C15
C1, C2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB


# ------------------------------------------------------------------ SplitMix64 multipliers (verify.cu derive_multipliers)
def _mix(z):
    z = ((z ^ (z >> 30)) * C1) & M64
    z = ((z ^ (z >> 27)) * C2) & M64
    return z ^ (z >> 31)


def _unxorshift(z, s):
    x = z
    for _ in range(64 // s + 1):
        x = z ^ (x >> s)
    return x


def _unmix(z):
    z = _unxorshift(z, 31)
    z = (z * pow(C2, -1, 1 << 64)) & M64
    z = _unxorshift(z, 27)
    z = (z * pow(C1, -1, 1 << 64)) & M64
    return _unxorshift(z, 30)


def splitmix_at(seed, k):
    return _mix((seed + (k + 1) * GAMMA) & M64)


def multipliers(seed, m):
    """r_j = a_j + 2^64 (b_j >> 1) for the draws a_j = #2j, b_j = #2j+1 of stream `seed`; zero becomes one"""
    out = []
    for j in range(m):
        v = splitmix_at(seed, 2 * j) | ((splitmix_at(seed, 2 * j + 1) >> 1) << 64)
        out.append(v or 1)
    return out


def seed_with_high_half_zero(j):
    """the seed whose draw #2j+1 is 0, so that r_j = draw #2j < 2^64: 63 leading zero bits in mul127's walk.  (r_j < 2^16
    or r_j = 0 would need two draws fixed at once, about 2^-111 per seed: no search reaches them, so the v == 0
    substitution is not exercised.)"""
    return (_unmix(0) - (2 * j + 2) * GAMMA) & M64


def seed_with_bit(bit, m, start=1):
    """the first seed from `start` at which some r_j of a batch of m has `bit` set (bits 0..126)"""
    s = start
    while not any((r >> bit) & 1 for r in multipliers(s, m)):
        s += 1
    return s


def seed_with_draw_top_bit(m, start=1):
    """a seed at which some draw #2j+1 has bit 63 set: the multiplier would have bit 127 set without the >> 1"""
    s = start
    while not any(splitmix_at(s, 2 * j + 1) >> 63 for j in range(m)):
        s += 1
    return s


# ------------------------------------------------------------------ circuits with n public inputs
def input_circuit(n):
    """public x_1..x_n, each squared into an aux variable, their weighted sum into another, and a cube gadget
    (w^3 + w + 5 = y) so that the aux side is not trivial; returns (cs, witness maker)"""
    cs = G.R1CS(num_inputs=n + 1, num_aux=n + 4)
    X = lambda i: 1 + i
    SQ = lambda i: n + 1 + i
    S, W, U, V = 2 * n + 1, 2 * n + 2, 2 * n + 3, 2 * n + 4
    for i in range(n):
        cs.enforce([(X(i), 1)], [(X(i), 1)], [(SQ(i), 1)])
    cs.enforce([(X(i), i + 1) for i in range(n)] + [(W, 1)], [(0, 1)], [(S, 1)])
    cs.enforce([(W, 1)], [(W, 1)], [(U, 1)])
    cs.enforce([(U, 1)], [(W, 1)], [(V, 1)])

    def witness(xs, w):
        r = Fd.R_MOD
        return [1] + list(xs) + [x * x % r for x in xs] + [(sum((i + 1) * x for i, x in enumerate(xs)) + w) % r, w, w * w % r, w ** 3 % r]
    return cs, witness


# ------------------------------------------------------------------ entry points (ctypes, no reshaping)
def _ptr(a):
    return None if a is None else a.ctypes.data_as(ct.c_void_p)


class Entry:
    """the five entry points on one key; pubs [m, n, 4] Montgomery, proofs [m, 387]"""

    def __init__(self, vk):
        from bazuka_b200 import groth16 as BG, _lib
        self.lib = _lib.load()
        self.vk = vk
        self.blob = np.ascontiguousarray(BG.vk_to_bincode(vk), dtype=np.uint8)
        self.pvk = BG.PreparedVerifyingKey(vk)
        self.ic = np.ascontiguousarray(vk["ic"], dtype=np.uint8).reshape(-1, 104)
        self.wire = [np.ascontiguousarray(vk[k], dtype=np.uint8) for k in ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2")]

    def free(self):
        self.pvk.free()

    @staticmethod
    def _split(proof):
        p = np.ascontiguousarray(proof, dtype=np.uint8).reshape(387)
        a, b, c = np.zeros(104, np.uint8), np.zeros(200, np.uint8), np.zeros(104, np.uint8)
        a[:97], b[:193], c[:97] = p[:97], p[97:290], p[290:]
        return a, b, c

    def plain(self, pub, proof):
        """bzk_groth16_verify"""
        pub = np.ascontiguousarray(pub, dtype=np.uint64).reshape(-1, 4)
        a, b, c = self._split(proof)
        return self.lib.bzk_groth16_verify(*[_ptr(w) for w in self.wire], _ptr(self.ic), len(self.ic), _ptr(pub) if len(pub) else None,
                                           len(pub), _ptr(a), _ptr(b), _ptr(c))

    def prepared(self, pub, proof):
        pub = np.ascontiguousarray(pub, dtype=np.uint64).reshape(-1, 4)
        a, b, c = self._split(proof)
        return self.lib.bzk_groth16_verify_prepared(self.pvk._h, _ptr(pub) if len(pub) else None, len(pub), _ptr(a), _ptr(b), _ptr(c))

    def bytes_(self, pub, proof, blob=None):
        pub = np.ascontiguousarray(pub, dtype=np.uint64).reshape(-1, 4)
        proof = np.ascontiguousarray(proof, dtype=np.uint8).reshape(387)
        blob = self.blob if blob is None else blob
        return self.lib.bzk_groth16_verify_bytes(_ptr(blob), blob.size, _ptr(pub) if len(pub) else None, len(pub), _ptr(proof))

    def batch(self, pubs, proofs, seed, threads, each=True):
        """bzk_groth16_verify_batch -> (status, ok_each or None)"""
        m, n = pubs.shape[0], pubs.shape[1]
        pubs = np.ascontiguousarray(pubs, dtype=np.uint64)
        proofs = np.ascontiguousarray(proofs, dtype=np.uint8)
        ok = np.full(m, 0xA5, np.uint8) if each else None
        st = self.lib.bzk_groth16_verify_batch(self.pvk._h, _ptr(pubs) if n else None, n, _ptr(proofs), m, seed, threads, _ptr(ok))
        return st, ok

    def batch_dev(self, ctx, pubs, proofs, seed, each=True):
        m, n = pubs.shape[0], pubs.shape[1]
        pubs = np.ascontiguousarray(pubs, dtype=np.uint64)
        proofs = np.ascontiguousarray(proofs, dtype=np.uint8)
        ok = np.full(m, 0xA5, np.uint8) if each else None
        st = self.lib.bzk_groth16_verify_batch_dev(ctx._h, self.pvk._h, _ptr(pubs) if n else None, n, _ptr(proofs), m, seed, _ptr(ok))
        return st, ok


# ------------------------------------------------------------------ tamper families
def _g1(b):
    return None if b[96] else (Fd.fp_from_mont_bytes(bytes(b[0:48])), Fd.fp_from_mont_bytes(bytes(b[48:96])))


def _g2(b):
    if b[192]:
        return None
    v = [Fd.fp_from_mont_bytes(bytes(b[48 * k:48 * k + 48])) for k in range(4)]
    return ((v[0], v[1]), (v[2], v[3]))


SPANS = {"A": (0, 97), "B": (97, 290), "C": (290, 387)}


def _put(t, name, Pt):
    lo, hi = SPANS[name]
    t[lo:hi] = np.frombuffer(PC.g2_wire(Pt) if name == "B" else PC.g1_wire(Pt), dtype=np.uint8)


def _points(proof):
    return {"A": _g1(proof[0:97]), "B": _g2(proof[97:290]), "C": _g1(proof[290:387])}


@functools.lru_cache(maxsize=None)
def _off_subgroup():
    g1 = PC.g1_off_subgroup()
    return g1[0], g1[-1], PC.g2_points()[1][0]    # a G1 point of large order, the 3-torsion (0, 2), a twist point


# a valid A or C plus the 3-torsion point (0, 2) is accepted by every entry point: the 3-torsion part pairs to an element of
# order 3 in the order-r target group, that is to one, and [r_j] keeps it in the 3-torsion.  Subgroup membership is not
# checked (DESIGN.md §3.8); these tampers are the ones that stay valid.
ACCEPTED = ("A off the subgroup: A + 3-torsion", "C off the subgroup: C + 3-torsion")


def tampers(proof, other):
    """(name, tampered 387 bytes, swap) for one valid proof; `other` is a valid proof of another statement.  swap = True
    means: keep the proof, exchange its public inputs with another index's.  Every tamper but those named in ACCEPTED
    makes the proof invalid."""
    pts, opts = _points(proof), _points(other)
    out = []
    for k in ("A", "B", "C"):
        F = C.FP2 if k == "B" else C.FP
        for how, Pt in (("other", opts[k]), ("negated", C.neg(F, pts[k])), ("doubled", C.add(F, pts[k], pts[k]))):
            t = proof.copy()
            _put(t, k, Pt)
            out.append((f"{k} {how}", t, False))
    out.append(("inputs swapped", proof.copy(), True))
    for name, at in PC.COORDS.items():
        for word in (0, 5, 11):
            t = proof.copy()
            t[at + 4 * word + (word % 4)] ^= 1 << (word % 8)
            out.append((f"{name} word {word} bit flipped", t, False))
    for k, fl in PC.FLAGS.items():
        lo = SPANS[k][0]
        for flag in (1, 2, 0x80, 0xFF):
            t = proof.copy()
            t[fl] = flag
            out.append((f"{k} flag {flag:#x}, coordinates nonzero", t, False))
        t = proof.copy()
        t[lo:fl] = 0
        t[fl] = 1
        out.append((f"{k} identity, coordinates zero", t, False))
        t = proof.copy()
        t[lo:fl + 1] = 0
        out.append((f"{k} (0, 0) flag clear", t, False))
    g1big, g1t3, g2off = _off_subgroup()
    for k, Pt, tag in (("A", g1big, "large order"), ("C", g1big, "large order"), ("B", g2off, "twist point"),
                       ("A", C.add(C.FP, pts["A"], g1t3), "A + 3-torsion"), ("C", C.add(C.FP, pts["C"], g1t3), "C + 3-torsion")):
        t = proof.copy()
        _put(t, k, Pt)
        out.append((f"{k} off the subgroup: {tag}", t, False))
    for name, at in PC.COORDS.items():
        t = proof.copy()
        v = int.from_bytes(t[at:at + 48].tobytes(), "little")
        t[at:at + 48] = np.frombuffer((v + P).to_bytes(48, "little"), dtype=np.uint8)
        out.append((f"{name} re-encoded as x + p", t, False))
    return out
