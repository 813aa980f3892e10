"""ORACLE — Ed25519 verification with the verdict of ed25519-dalek 1.x `PublicKey::verify` (the reference's `Ed25519::verify`,
src/crypto/ed25519.rs:81-83), restated on Python big integers, plus RFC 8032 signing and the reference's `generate_keys`
to make test data.  Test infrastructure only.

The verdict for (pk, sig = R || s, M) is True iff s < L; pk decompresses (y = low 255 bits mod P, non-canonical y accepted,
x^2 = (y^2 - 1) / (d y^2 + 1) solvable, the even root negated when bit 255 is set, "-0" accepted, no torsion check);
k = SHA-512(R || pk || M) mod L; and compress([k](-A) + [s]B) == R as bytes.  No cofactor anywhere."""
import hashlib

P = 2**255 - 19
L = 2**252 + 27742317777372353535851937790883648493
D = (-121665 * pow(121666, -1, P)) % P
SQRT_M1 = pow(2, (P - 1) // 4, P)

IDENTITY = (0, 1)


def on_curve(pt):
    x, y = pt
    return (y * y - x * x - 1 - D * x * x * y * y) % P == 0


def add(p1, p2):
    """affine twisted Edwards addition, a = -1 (complete: d is not a square)"""
    (x1, y1), (x2, y2) = p1, p2
    t = D * x1 * x2 * y1 * y2 % P
    x3 = (x1 * y2 + x2 * y1) * pow(1 + t, -1, P) % P
    y3 = (y1 * y2 + x1 * x2) * pow(1 - t, -1, P) % P
    return (x3, y3)


def neg(pt):
    return ((-pt[0]) % P, pt[1])


# extended coordinates for the multiplications (no inversions in the loop)
def _ext(pt):
    return (pt[0], pt[1], 1, pt[0] * pt[1] % P)


def _ext_add(p, q):
    x1, y1, z1, t1 = p
    x2, y2, z2, t2 = q
    a = (y1 - x1) * (y2 - x2) % P
    b = (y1 + x1) * (y2 + x2) % P
    c = 2 * D * t1 * t2 % P
    d = 2 * z1 * z2 % P
    e, f, g, h = b - a, d - c, d + c, b + a
    return (e * f % P, g * h % P, f * g % P, e * h % P)


def _affine(p):
    x, y, z, _ = p
    zi = pow(z, -1, P)
    return (x * zi % P, y * zi % P)


def mul(pt, k):
    """[k] pt for any integer k >= 0 (no reduction)"""
    acc, q = _ext(IDENTITY), _ext(pt)
    while k:
        if k & 1:
            acc = _ext_add(acc, q)
        q = _ext_add(q, q)
        k >>= 1
    return _affine(acc)


def _recover_x(y, sign):
    """x with x^2 = (y^2 - 1) / (d y^2 + 1): the even root, negated when sign; None when there is none"""
    u, v = (y * y - 1) % P, (D * y * y + 1) % P
    x2 = u * pow(v, -1, P) % P
    if x2 == 0:
        return 0   # "-0" is kept as 0: sign has no effect
    x = pow(x2, (P + 3) // 8, P)
    if (x * x - x2) % P != 0:
        x = x * SQRT_M1 % P
    if (x * x - x2) % P != 0:
        return None
    if x & 1:
        x = P - x
    return (P - x) % P if sign else x


def decompress(b):
    """curve25519-dalek 3.x `CompressedEdwardsY::decompress`: the point or None"""
    b = bytes(b)
    assert len(b) == 32
    n = int.from_bytes(b, "little")
    y = (n & ((1 << 255) - 1)) % P
    x = _recover_x(y, n >> 255)
    return None if x is None else (x, y)


def compress(pt):
    x, y = pt
    return (y | ((x & 1) << 255)).to_bytes(32, "little")


B = (_recover_x(4 * pow(5, -1, P) % P, 0), 4 * pow(5, -1, P) % P)


def k_of(r_bytes, pk, msg):
    return int.from_bytes(hashlib.sha512(bytes(r_bytes) + bytes(pk) + bytes(msg)).digest(), "little") % L


def verify(pk, msg, sig):
    """`ed25519_dalek::PublicKey::verify` (1.x, default features)"""
    pk, sig = bytes(pk), bytes(sig)
    if len(pk) != 32 or len(sig) != 64:
        return False
    s = int.from_bytes(sig[32:], "little")
    if s >= L:
        return False
    a = decompress(pk)
    if a is None:
        return False
    k = k_of(sig[:32], pk, msg)
    return compress(add(mul(neg(a), k), mul(B, s))) == sig[:32]


# ---------------------------------------------------------------------------------------------------------------- signing
def _expand(secret):
    h = hashlib.sha512(bytes(secret)).digest()
    a = int.from_bytes(h[:32], "little")
    a &= (1 << 254) - 8
    a |= 1 << 254
    return a, h[32:]


def public_key(secret):
    """RFC 8032 public key of a 32-byte secret"""
    return compress(mul(B, _expand(secret)[0]))


def sign(secret, msg):
    """RFC 8032 deterministic signature (what ed25519-dalek's `Keypair::sign` computes)"""
    a, prefix = _expand(secret)
    pk = compress(mul(B, a))
    r = int.from_bytes(hashlib.sha512(prefix + bytes(msg)).digest(), "little") % L
    return sign_with(a, r, pk, msg)


def sign_with(a, r, pk, msg):
    """R = [r]B, s = r + k a mod L over the key bytes pk as given (for keys with torsion components or odd encodings)"""
    rb = compress(mul(B, r))
    return rb + ((r + k_of(rb, pk, msg) * a) % L).to_bytes(32, "little")


def generate_keys(seed):
    """the reference's `Ed25519::generate_keys` (src/crypto/ed25519.rs:69-76): secret = sha3_256(seed) with bit 255 cleared
    -> (public key bytes, secret bytes)"""
    x = bytearray(hashlib.sha3_256(bytes(seed)).digest())
    x[31] &= 0x7F
    return public_key(bytes(x)), bytes(x)
