"""Signature families for the batch EdDSA checks (tests/test_eddsa_batch_cpu.py, tests/test_gpu_eddsa_batch.py).

Every case is (name, compressed key, message, R, s) with plain Python ints, and `expected` is the Python restatement of
`JubJub::verify` behind the reference's `PublicKey` (src/crypto/jubjub/mod.rs:151-167, curve.rs:78-88): scalars must be
canonical, the key must decompress, then A and R on the curve and [h] A + R == [s] BASE with h and s as full integers."""
import functools

from bazuka_b200.mpn import native as N

R, ORDER, BASE, IDENTITY = N.R, N.JJ_ORDER, N.JJ_BASE, (0, 1)


def expected(pk, msg, r, s):
    if not all(0 <= v < R for v in (pk[0], msg, r[0], r[1], s)):
        return False
    a = N.jj_decompress_checked(pk)
    return a is not None and N.eddsa_verify(a, msg, {"r": r, "s": s})


def jj_neg(p):
    return ((-p[0]) % R, p[1])


def point_order(p):
    for k in (1, 2, 4, 8):
        if N.jj_mul(p, k) == IDENTITY:
            return k
    return None


@functools.lru_cache(maxsize=1)
def torsion8():
    """a generator of the 8-torsion: [ORDER] P for a curve point P whose cofactor part has order 8"""
    x = 3
    while True:
        p = N.jj_decompress_checked((x, False))
        if p is not None:
            t = N.jj_mul(p, ORDER)
            if point_order(t) == 8:
                return t
        x += 1


def torsion_points():
    t = torsion8()
    return [N.jj_mul(t, k) for k in range(8)]   # k = 0: the identity


def sqrt_m1():
    return N.fr_sqrt(R - 1)


def sign_with_torsion(seed, msg, t_key, t_r):
    """A = [a] BASE + t_key and R = [r] BASE + t_r, s = r + h a mod ORDER: (compressed A, R, s, A)"""
    a = N.hash_to_scalar(b"a-" + seed)
    rnd = N.hash_to_scalar(b"r-" + seed)
    A = N.jj_add(N.jj_mul(BASE, a), t_key)
    Rp = N.jj_add(N.jj_mul(BASE, rnd), t_r)
    h = N.poseidon([Rp[0], Rp[1], A[0], A[1], msg])
    return N.jj_compress(A), Rp, (rnd + h * a) % ORDER, A


def families(seed=b"f"):
    """[(name, pk_compressed, msg, R, s)]: valid, tampered, non-canonical, off-curve, undecompressable, torsion cases"""
    pk, sk = N.eddsa_keys(b"key-" + seed)
    other, _ = N.eddsa_keys(b"other-" + seed)
    msg = N.poseidon([int.from_bytes(seed, "big"), 7])
    sig = N.eddsa_sign(sk, msg)
    r, s = sig["r"], sig["s"]
    c, oc = N.jj_compress(pk), N.jj_compress(other)
    bad_x = next(x for x in range(1, 100) if N.jj_decompress_checked((x, False)) is None)
    out = [("valid", c, msg, r, s), ("msg+1", c, msg + 1, r, s), ("s+1", c, msg, r, s + 1), ("s=0", c, msg, r, 0),
           ("s+ORDER", c, msg, r, s + ORDER), ("s>=r", c, msg, r, s + R), ("s=r-1", c, msg, r, R - 1), ("R.x>=r", c, msg, (r[0] + R, r[1]), s),
           ("msg>=r", c, msg + R, r, s), ("pk.x>=r", (c[0] + R, c[1]), msg, r, s), ("R off curve", c, msg, (r[0], r[1] + 1), s),
           ("R=(0,1)", c, msg, IDENTITY, s), ("key does not decompress", (bad_x, c[1]), msg, r, s), ("wrong parity", (c[0], not c[1]), msg, r, s),
           ("another key", oc, msg, r, s), ("valid again", c, msg, r, s)]
    # keys and R with 2-, 4- and 8-torsion components: search T_R so that the restatement accepts, keep some that reject
    ts = torsion_points()
    for k_key in (4, 2, 1):
        accepted = rejected = attempt = 0
        while accepted < 1 or rejected < 2:
            j = (attempt * k_key) % 8   # T_R in the subgroup of the key's torsion, where acceptance is possible
            pkc, Rp, sv, _ = sign_with_torsion(seed + bytes([k_key, attempt]), msg, ts[k_key], ts[j])
            ok = expected(pkc, msg, Rp, sv)
            if (ok and accepted < 1) or (not ok and rejected < 2):
                out.append((f"torsion key {k_key} R {j} {'acc' if ok else 'rej'}", pkc, msg, Rp, sv))
                accepted += ok
                rejected += not ok
            attempt += 1
    # R with a torsion component on a torsion-free key: h drops out of the torsion part, only T_R = 0 accepts
    for j in (0, 4, 1):
        pkc, Rp, sv, _ = sign_with_torsion(seed + b"R", msg, IDENTITY, ts[j])
        out.append((f"torsion R {j}", pkc, msg, Rp, sv))
    return out
