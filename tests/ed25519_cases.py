"""Signature families for the Ed25519 checks (tests/test_ed25519_cpu.py, tests/test_gpu_ed25519_batch.py).

Every case is (name, pk bytes, message bytes, sig bytes) and `expected` is the big-integer restatement of ed25519-dalek 1.x
`PublicKey::verify` (oracle/py/ed25519.py).  Keys without a known secret (small-order, non-canonical encodings) get
signatures R = [r]B, s = r, found by a search over r: then R' = R - [k]A, accepted exactly when [k]A = 0.  Mixed-order keys
A = aB + T get honest signatures: R' = R - [k]T, accepted exactly when [k]T = 0, where a cofactored verifier would accept
either way."""
import functools
import hashlib

from oracle.py import ed25519 as O

P, L, B, IDENTITY = O.P, O.L, O.B, O.IDENTITY


def expected(pk, msg, sig):
    return O.verify(pk, msg, sig)


def point_order(pt):
    for k in (1, 2, 4, 8):
        if O.mul(pt, k) == IDENTITY:
            return k
    return None


@functools.lru_cache(maxsize=1)
def torsion_points():
    """the eight points of order dividing 8: [j] T8 for a generator T8 = [L] Q"""
    y = 2
    while True:
        q = O.decompress(y.to_bytes(32, "little"))
        if q is not None:
            t = O.mul(q, L)
            if point_order(t) == 8:
                return [O.mul(t, j) for j in range(8)]
        y += 1


def _scalar(tag):
    return int.from_bytes(hashlib.sha512(tag).digest(), "little") % L


def _le(v):
    return int(v).to_bytes(32, "little")


def search_no_secret(pk, msg, want, tag):
    """a signature R = [r]B, s = r on a key of order dividing 8, searched over r until the verdict is `want`"""
    for i in range(400):
        r = _scalar(tag + b"-%d" % i)
        sig = O.compress(O.mul(B, r)) + _le(r)
        if O.verify(pk, msg, sig) == want:
            return sig
    raise AssertionError("no signature found")


def search_mixed(a, t, msg, want, tag):
    """an honest signature by A = aB + T, searched over the nonce until the verdict is `want`: (pk, sig)"""
    pk = O.compress(O.add(O.mul(B, a), t))
    for i in range(400):
        sig = O.sign_with(a, _scalar(tag + b"-%d" % i), pk, msg)
        if O.verify(pk, msg, sig) == want:
            return pk, sig
    raise AssertionError("no signature found")


def undecompressable(start=2):
    y = start
    while O.decompress(_le(y)) is not None:
        y += 1
    return _le(y)


def families(seed=b"f", big=True):
    """[(name, pk, msg, sig)]: honest, tampered, s at the l boundary, undecompressable keys, the eight small-order keys (and
    their "-0" and non-canonical encodings), mixed-order keys, non-canonical and "-0" R, empty and (big) 1 MiB messages"""
    pk, sk = O.generate_keys(b"key-" + seed)
    other, _ = O.generate_keys(b"other-" + seed)
    msg = b"message " + seed
    sig = O.sign(sk, msg)
    s = int.from_bytes(sig[32:], "little")
    flip = lambda b, i: b[:i] + bytes([b[i] ^ 1]) + b[i + 1:]
    out = [("honest", pk, msg, sig), ("honest again", pk, msg, sig), ("message tampered", pk, msg + b"!", sig),
           ("message truncated", pk, msg[:-1], sig), ("R tampered", pk, msg, flip(sig, 0)), ("s tampered", pk, msg, flip(sig, 40)),
           ("s + l", pk, msg, sig[:32] + _le(s + L)), ("s with bit 255", pk, msg, sig[:32] + _le(s | (1 << 255))),
           ("another key", other, msg, sig), ("key tampered", flip(pk, 3), msg, sig),
           ("empty message", pk, b"", O.sign(sk, b"")), ("empty message tampered", pk, b"\x00", O.sign(sk, b""))]
    # s at the boundary of the canonical check, on the identity key where [s]B = R is the whole equation
    ident = _le(1)
    for name, sv, ok_expected in (("s = l - 1", L - 1, True), ("s = l", L, False), ("s = l + 1", L + 1, False), ("s = 2^255 + 1", (1 << 255) + 1, False)):
        out.append((name, ident, msg, O.compress(O.mul(B, sv)) + _le(sv)))
    out.append(("s = l - 1 wrong R", pk, msg, sig[:32] + _le(L - 1)))
    # keys that do not decompress
    out.append(("key does not decompress", undecompressable(), msg, sig))
    out.append(("key does not decompress, sign bit", bytes(undecompressable(50)[:31]) + b"\x80", msg, sig))
    # the eight small-order keys, each with an accepted and (order > 1) a rejected signature; identity and (0, -1) also as "-0"
    ts = torsion_points()
    for j, t in enumerate(ts):
        enc = O.compress(t)
        encs = [("", enc)]
        if t[0] == 0:
            encs.append((" -0", enc[:31] + bytes([enc[31] | 0x80])))
        for tag, e in encs:
            out.append((f"small order {point_order(t)} #{j}{tag} acc", e, msg, search_no_secret(e, msg, True, seed + b"so%d" % j)))
            if point_order(t) > 1:
                out.append((f"small order {point_order(t)} #{j}{tag} rej", e, msg, search_no_secret(e, msg, False, seed + b"so%d" % j)))
    # non-canonical key encodings y + p (y < 19: the identity and the order-4 point with y = 0), signed over those bytes
    for y in (1, 0):
        e = _le(y + P)
        assert O.decompress(e) is not None
        out.append((f"non-canonical key y={y}+p acc", e, msg, search_no_secret(e, msg, True, seed + b"nc%d" % y)))
        if y == 0:
            out.append((f"non-canonical key y={y}+p rej", e, msg, search_no_secret(e, msg, False, seed + b"nc%d" % y)))
    # mixed-order keys A = aB + T: honest signatures, accepted iff [k]T = 0, both kinds at each torsion order
    a = _scalar(b"mixed-" + seed)
    for j in (4, 2, 1):
        for want in (True, False):
            mpk, msig = search_mixed(a, ts[j], msg, want, seed + b"mx%d" % j)
            out.append((f"mixed order {point_order(ts[j])} {'acc' if want else 'rej'}", mpk, msg, msig))
    # R encodings: on the identity key with s = 0, R = the identity is accepted; its "-0" and y + p encodings are not
    out.append(("R identity", ident, msg, _le(1) + _le(0)))
    out.append(("R -0", ident, msg, _le(1 | (1 << 255)) + _le(0)))
    out.append(("R non-canonical y+p", ident, msg, _le(1 + P) + _le(0)))
    rp = O.compress(O.mul(B, 5))
    out.append(("R = 5B", ident, msg, rp + _le(5)))
    out.append(("R = 5B non-canonical x sign", ident, msg, rp[:31] + bytes([rp[31] ^ 0x80]) + _le(5)))
    if big:
        m = bytes(hashlib.shake_256(b"big-" + seed).digest(1 << 20))
        out.append(("1 MiB message", pk, m, O.sign(sk, m)))
        out.append(("1 MiB message tampered", pk, m[:-1] + b"\x00", O.sign(sk, m)))
    return out
