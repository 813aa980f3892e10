"""ORACLE (test infrastructure only — never imported by the product path).

bellman 0.14's `Parameters` file format over bls12_381 0.8's uncompressed point encodings, on Python big integers.
Neither crate is vendored and no file they wrote exists here, so the layout below is restated from the crates' source
as remembered *(ext)*, the same footing as SURVEY.md's restatements; bazuka_b200/csrc/params_io.cu cites this module.

  file      = VerifyingKey::write, then for each of h, l, a, b_g1, b_g2: u32 big-endian length + that many points
  vk        = alpha_g1, beta_g1, beta_g2, gamma_g2, delta_g1, delta_g2, u32 big-endian |ic|, ic
  G1 (96 B) = x | y, 48-byte big-endian canonical integers (not Montgomery)
  G2 (192 B)= x.c1 | x.c0 | y.c1 | y.c0
  flags     = byte 0: bit 7 compression (must be 0), bit 6 infinity, bit 5 sort (must be 0); x is read masked;
              the identity is the infinity bit alone
  from_uncompressed_unchecked  refuses a coordinate >= p, the compression or sort bit, the infinity bit with any other
                               bit set; it does not test the curve equation
  from_uncompressed            also requires the curve equation and torsion-freeness
  Parameters::read(checked)    the vk always checked; the five vectors checked or not; the identity refused in ic and
                               in the five vectors ("point at infinity"); nothing after b_g2 is read

Subgroup membership is defined here as [r]P = O.  The endomorphism constants the GPU's faster tests use (beta for
sigma on G1, the psi coefficients on G2) are derived below from their definitions, and `torsion_free_endo` restates
those tests so that the CPU tier can hold them to the definition.
"""
from . import curve as C
from .field import P_MOD as P, R_MOD, fp_from_mont_bytes

G1_BYTES, G2_BYTES = 96, 192
VK_G1 = ("alpha_g1", "beta_g1", "delta_g1")
VK_ORDER = ("alpha_g1", "beta_g1", "beta_g2", "gamma_g2", "delta_g1", "delta_g2")
VECTORS = ("h", "l", "a", "b_g1", "b_g2")
BLS_X = -C.BLS_X


class BadPoint(ValueError):
    """a refused point; `status` is the libbzk code bellman's rule maps to (-8 encoding, -4 curve, -9 subgroup)"""

    def __init__(self, reason, status):
        super().__init__(reason)
        self.reason, self.status = reason, status


BAD_ENCODING, NOT_ON_CURVE, NOT_IN_SUBGROUP = -8, -4, -9


# ------------------------------------------------------------------ square roots (p = 3 mod 4)
def fp_sqrt(a):
    r = pow(a, (P + 1) // 4, P)
    return r if r * r % P == a % P else None


def fp2_sqrt(a):
    """Fp2 = Fp[u]/(u^2 + 1), p = 3 mod 4 (eprint 2012/685, algorithm 9); None when a is not a square."""
    def pw(x, e):
        r = C.F2_ONE
        for bit in bin(e)[2:]:
            r = C.f2_sqr(r)
            if bit == "1":
                r = C.f2_mul(r, x)
        return r
    a1 = pw(a, (P - 3) // 4)
    alpha = C.f2_mul(C.f2_sqr(a1), a)
    x0 = C.f2_mul(a1, a)
    if alpha == (P - 1, 0):
        x = C.f2_mul((0, 1), x0)
    else:
        x = C.f2_mul(pw(C.f2_add(C.F2_ONE, alpha), (P - 1) // 2), x0)
    return x if C.f2_sqr(x) == (a[0] % P, a[1] % P) else None


def g1_lift(x):
    """a point with abscissa x on y^2 = x^3 + 4 (not necessarily in the subgroup), or None"""
    y = fp_sqrt((x * x * x + 4) % P)
    return None if y is None else (x % P, y)


def g2_lift(x):
    y = fp2_sqrt(C.f2_add(C.f2_mul(C.f2_sqr(x), x), C.B2))
    return None if y is None else ((x[0] % P, x[1] % P), y)


# ------------------------------------------------------------------ subgroup: the definition and the endomorphism tests
def in_subgroup(F, pt):
    """[r]P = O"""
    return pt is None or C.mul(F, pt, R_MOD) is None


def _mul_signed(F, pt, k):
    q = C.mul(F, pt, abs(k))
    return C.neg(F, q) if k < 0 else q


def _derive_beta():
    """the primitive cube root of unity with sigma(x, y) = (beta x, y) = [-x^2] on G1"""
    g = 2
    while pow(g, (P - 1) // 3, P) == 1:
        g += 1
    w = pow(g, (P - 1) // 3, P)
    want = _mul_signed(C.FP, C.G1_GEN, -(BLS_X * BLS_X))
    for b in (w, w * w % P):
        if (b * C.G1_GEN[0] % P, C.G1_GEN[1]) == want:
            return b
    raise AssertionError("no cube root of unity acts as [-x^2]")


def _f2_pow(a, e):
    r = C.F2_ONE
    for bit in bin(e)[2:]:
        r = C.f2_sqr(r)
        if bit == "1":
            r = C.f2_mul(r, a)
    return r


BETA = _derive_beta()
PSI_X = C.f2_inv(_f2_pow((1, 1), (P - 1) // 3))   # 1 / (u+1)^((p-1)/3)
PSI_Y = C.f2_inv(_f2_pow((1, 1), (P - 1) // 2))   # 1 / (u+1)^((p-1)/2)


def psi(pt):
    (x0, x1), (y0, y1) = pt
    return (C.f2_mul((x0, (-x1) % P), PSI_X), C.f2_mul((y0, (-y1) % P), PSI_Y))


def torsion_free_endo(F, pt):
    """bls12_381 0.8's tests: G1 sigma(P) == -[x^2] P, G2 psi(P) == [x] P"""
    if pt is None:
        return True
    if F is C.FP:
        return (BETA * pt[0] % P, pt[1]) == _mul_signed(F, pt, -(BLS_X * BLS_X))
    return psi(pt) == _mul_signed(F, pt, BLS_X)


assert psi(C.G2_GEN) == _mul_signed(C.FP2, C.G2_GEN, BLS_X), "psi constants"


# ------------------------------------------------------------------ point codecs
def _be(x):
    return int(x).to_bytes(48, "big")


def g1_to_uncompressed(pt) -> bytes:
    if pt is None:
        return bytes([0x40]) + bytes(95)
    return _be(pt[0]) + _be(pt[1])


def g2_to_uncompressed(pt) -> bytes:
    if pt is None:
        return bytes([0x40]) + bytes(191)
    (x0, x1), (y0, y1) = pt
    return _be(x1) + _be(x0) + _be(y1) + _be(y0)


def _decode(b, ncoord, checked, F):
    b = bytes(b)
    flags = b[0]
    coords = [int.from_bytes(b[48 * i: 48 * i + 48], "big") for i in range(ncoord)]
    coords[0] &= (1 << 381) - 1          # the three flag bits masked off x (x.c1 on G2)
    if flags & 0x80:
        raise BadPoint("compression flag set", BAD_ENCODING)
    if flags & 0x20:
        raise BadPoint("sort flag set", BAD_ENCODING)
    half = ncoord // 2
    if any(c >= P for c in coords[:half]):
        raise BadPoint("x coordinate not below p", BAD_ENCODING)
    if any(c >= P for c in coords[half:]):
        raise BadPoint("y coordinate not below p", BAD_ENCODING)
    if flags & 0x40:
        if any(coords):
            raise BadPoint("infinity flag with coordinate bits set", BAD_ENCODING)
        return None
    pt = (coords[0], coords[1]) if ncoord == 2 else ((coords[1], coords[0]), (coords[3], coords[2]))
    if checked:
        if not C.on_curve(F, pt):
            raise BadPoint("not on the curve", NOT_ON_CURVE)
        if not in_subgroup(F, pt):
            raise BadPoint("not in the prime-order subgroup", NOT_IN_SUBGROUP)
    return pt


def g1_from_uncompressed(b, checked=True):
    """`from_uncompressed` (checked) / `from_uncompressed_unchecked`; raises BadPoint"""
    return _decode(b, 2, checked, C.FP)


def g2_from_uncompressed(b, checked=True):
    return _decode(b, 4, checked, C.FP2)


# ------------------------------------------------------------------ key files
def _point(v, g2):
    """a point as oracle/py/groth16.setup holds it, or a Montgomery wire image (oracle.groth16_c.setup, libbzk)"""
    if v is None or isinstance(v, tuple):
        return v
    b = bytes(memoryview(v).cast("B")) if not isinstance(v, (bytes, bytearray)) else bytes(v)
    return C.g2_from_bytes(b) if g2 else C.g1_from_bytes(b)


def _wire_to_uncompressed(v, g2):
    """fast path for a Montgomery wire image: straight to the big-endian canonical encoding"""
    if v is None or isinstance(v, tuple):
        return (g2_to_uncompressed if g2 else g1_to_uncompressed)(v)
    b = bytes(v) if isinstance(v, (bytes, bytearray)) else bytes(memoryview(v).cast("B"))
    if b[192 if g2 else 96]:
        return (g2_to_uncompressed if g2 else g1_to_uncompressed)(None)
    if g2:
        x0, x1, y0, y1 = (fp_from_mont_bytes(b[48 * i: 48 * i + 48]) for i in range(4))
        return _be(x1) + _be(x0) + _be(y1) + _be(y0)
    return _be(fp_from_mont_bytes(b[:48])) + _be(fp_from_mont_bytes(b[48:96]))


def write(params) -> bytes:
    """`Parameters::write` of a key dict {vk: {...}, h, l, a, b_g1, b_g2}: points or wire images"""
    vk = params["vk"]
    out = [_wire_to_uncompressed(vk[k], k.endswith("g2")) for k in VK_ORDER]
    out.append(len(vk["ic"]).to_bytes(4, "big"))
    out += [_wire_to_uncompressed(p, False) for p in vk["ic"]]
    for k in VECTORS:
        out.append(len(params[k]).to_bytes(4, "big"))
        out += [_wire_to_uncompressed(p, k == "b_g2") for p in params[k]]
    return b"".join(out)


def info(blob):
    """the lengths the image states and the byte count they imply; ValueError when it is shorter"""
    off, n = 96 * 3 + 192 * 3, {}
    for k, size in (("ic", 96), ("h", 96), ("l", 96), ("a", 96), ("b_g1", 96), ("b_g2", 192)):
        if off + 4 > len(blob):
            raise ValueError(f"truncated before the length of {k}")
        n[k] = int.from_bytes(bytes(blob[off: off + 4]), "big")
        off += 4 + n[k] * size
    if off > len(blob):
        raise ValueError("truncated")
    n["bytes"] = off
    return n


def read(blob, checked=True):
    """`Parameters::read(reader, checked)` -> {vk: {...}, h, l, a, b_g1, b_g2} as points.  Raises BadPoint with
    `where` = "vector[index]" for the first refused point in file order."""
    blob = bytes(blob)
    info(blob)
    off = 0

    def take(size, g2, chk, allow_inf, where):
        nonlocal off
        b = blob[off: off + size]
        off += size
        try:
            pt = (g2_from_uncompressed if g2 else g1_from_uncompressed)(b, chk)
            if pt is None and not allow_inf:
                raise BadPoint("point at infinity", BAD_ENCODING)
        except BadPoint as e:
            e.where = where
            raise
        return pt

    def length():
        nonlocal off
        off += 4
        return int.from_bytes(blob[off - 4: off], "big")

    vk = {k: take(192 if k.endswith("g2") else 96, k.endswith("g2"), True, True, f"{k}[0]") for k in VK_ORDER}
    vk["ic"] = [take(96, False, True, False, f"ic[{i}]") for i in range(length())]
    out = {"vk": vk}
    for k in VECTORS:
        g2 = k == "b_g2"
        out[k] = [take(192 if g2 else 96, g2, checked, False, f"{k}[{i}]") for i in range(length())]
    return out
