"""CPU tier of the Ed25519 checks: the big-integer oracle (oracle/py/ed25519.py) pinned to libsodium; csrc/ed25519.cuh (the code
the kernels of csrc/ed25519.cu run) compiled with g++ over the device text of the field arithmetic, against big integers and
hashlib; and libbzk's host call bzk_ed25519_verify on every signature family."""
import ctypes as ct
import hashlib
import json
import os
import random
import subprocess

import pytest

import ed25519_cases as E
from oracle.py import ed25519 as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, L = O.P, O.L


@pytest.fixture(scope="module")
def edshim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ed25519_shim") / "_ed25519_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-DBZK_HOST_DEVICE_TEXT", "-I", os.path.join(ROOT, "bazuka_b200", "csrc"),
                           os.path.join(ROOT, "tests", "hostshim", "ed25519_shim.cpp"), "-o", out])
    lib = ct.CDLL(out)
    for f in ("shim_sqrt_ratio_i", "shim_decompress", "shim_verify"):
        getattr(lib, f).restype = ct.c_int
    lib.shim_sha512.argtypes = [ct.c_char_p, ct.c_uint64, ct.c_char_p]
    lib.shim_sha512_parts.argtypes = [ct.c_char_p, ct.c_uint64, ct.c_char_p, ct.c_uint64, ct.c_char_p, ct.c_uint64, ct.c_char_p]
    lib.shim_verify.argtypes = [ct.c_char_p, ct.c_char_p, ct.c_uint64, ct.c_char_p]
    return lib


@pytest.fixture(scope="module")
def fams():
    return E.families(b"f") + E.families(b"g", big=False)


def le(v):
    return int(v).to_bytes(32, "little")


def test_oracle_matches_the_golden_vectors():
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "ed25519_vectors.json")))
    lens = set()
    for v in g["honest"] + g["reference"]:
        secret, pk, msg, sig = (bytes.fromhex(v[k]) for k in ("secret", "pk", "msg", "sig"))
        assert O.public_key(secret) == pk
        assert O.verify(pk, msg, sig) == v["ok"]
        if v["ok"]:
            assert O.sign(secret, msg) == sig
        lens.add(len(msg))
    assert {64 + n for n in lens} >= {111, 112, 127, 128, 239, 240} and {0, 4096} <= lens
    pk, secret = O.generate_keys(b"ABC")
    assert [v["ok"] for v in g["reference"]] == [True, False] and bytes.fromhex(g["reference"][0]["pk"]) == pk
    sig = O.sign(secret, b"salam1")
    assert O.verify(pk, b"salam1", sig) and not O.verify(pk, b"salam2", sig)


def test_oracle_matches_libsodium_on_random_honest_signatures():
    nb = pytest.importorskip("nacl.bindings")
    rng = random.Random(11)
    for i in range(40):
        seed = rng.randbytes(32)
        msg = rng.randbytes(rng.choice([0, 1, 47, 48, 63, 64, 111, 112, 175, 176, 300, 1000]))
        pk, sk = nb.crypto_sign_seed_keypair(seed)
        sig = nb.crypto_sign(msg, sk)[:64]
        assert O.public_key(seed) == pk and O.sign(seed, msg) == sig and O.verify(pk, msg, sig)
        bad = msg + b"x"
        try:
            nb.crypto_sign_open(sig + bad, pk)
            sodium = True
        except Exception:
            sodium = False
        assert O.verify(pk, bad, sig) == sodium == False


_EDGES = [0, 1, 2, 18, 19, 20, P - 1, P, P + 1, P + 18, 2**255 - 1, 2**255, 2**256 - 1, 2**32 - 1, 2**32, 2**64 - 1, 2**128, (P - 1) // 2]


def test_field_arithmetic_at_the_edges(edshim):
    rng = random.Random(3)
    vals = _EDGES + [rng.randrange(2**256) for _ in range(30)]
    out = ct.create_string_buffer(32)
    for a in vals:
        for b in vals[:12] + [rng.randrange(P)]:
            for op, want in ((0, a * b % P), (3, (a + b) % P), (4, (a - b) % P)):
                edshim.shim_fe_op(op, le(a), le(b), out)
                assert int.from_bytes(out.raw, "little") == want, (op, a, b)
        edshim.shim_fe_op(1, le(a), le(0), out)
        assert int.from_bytes(out.raw, "little") == a * a % P, a
        edshim.shim_fe_op(2, le(a), le(0), out)
        assert int.from_bytes(out.raw, "little") == (pow(a, -1, P) if a % P else 0), a


def test_sqrt_ratio_i(edshim):
    rng = random.Random(4)
    out = ct.create_string_buffer(32)
    vals = _EDGES + [rng.randrange(P) for _ in range(60)]
    n_sq = n_non = 0
    for u in vals:
        for v in vals[:8] + [rng.randrange(1, P)]:
            ok = edshim.shim_sqrt_ratio_i(le(u), le(v), out)
            r = int.from_bytes(out.raw, "little")
            assert r < P and r % 2 == 0, (u, v)
            u_, v_ = u % P, v % P
            if u_ == 0:
                assert ok and r == 0
            elif v_ == 0:
                assert not ok and r == 0
            else:
                w = u_ * pow(v_, -1, P) % P
                square = pow(w, (P - 1) // 2, P) == 1
                assert bool(ok) == square, (u, v)
                assert r * r % P == (w if square else O.SQRT_M1 * w % P), (u, v)
                n_sq += square
                n_non += not square
    assert n_sq > 50 and n_non > 50


def test_sha512_at_every_length_and_1_mib(edshim):
    rng = random.Random(5)
    out = ct.create_string_buffer(64)
    data = rng.randbytes(300)
    for n in range(301):
        edshim.shim_sha512(data, n, out)
        assert out.raw == hashlib.sha512(data[:n]).digest(), n
    big = rng.randbytes(1 << 20)
    edshim.shim_sha512(big, len(big), out)
    assert out.raw == hashlib.sha512(big).digest()
    for na, nb, nc in ((32, 32, 0), (32, 32, 47), (32, 32, 64), (0, 0, 5), (5, 0, 200), (100, 100, 100), (127, 1, 0)):
        a, b, c = rng.randbytes(na), rng.randbytes(nb), rng.randbytes(nc)
        edshim.shim_sha512_parts(a, na, b, nb, c, nc, out)
        assert out.raw == hashlib.sha512(a + b + c).digest(), (na, nb, nc)


def test_wide_reduction_mod_l(edshim):
    rng = random.Random(6)
    out = ct.create_string_buffer(32)
    for v in [0, 1, L - 1, L, L + 1, 2 * L, 2**252, 2**256 - 1, 2**256, 2**256 * (L - 1), 2**512 - 1, L * L, L * 2**256 - 1] + [rng.randrange(2**512) for _ in range(200)]:
        edshim.shim_sc_from_hash(v.to_bytes(64, "little"), out)
        assert int.from_bytes(out.raw, "little") == v % L, v


def test_decompression_matches_the_oracle(edshim):
    rng = random.Random(7)
    x, y = ct.create_string_buffer(32), ct.create_string_buffer(32)
    encs = [le(v) for v in (0, 1, 2, P - 1, P, P + 1, 2**255 - 1)] + [le(v | (1 << 255)) for v in (0, 1, P - 1, P, 5)]
    encs += [rng.randbytes(32) for _ in range(400)] + [O.compress(t) for t in E.torsion_points()]
    n_none = 0
    for e in encs:
        want = O.decompress(e)
        got = edshim.shim_decompress(e, x, y)
        assert bool(got) == (want is not None), e.hex()
        if want is not None:
            assert (int.from_bytes(x.raw, "little"), int.from_bytes(y.raw, "little")) == want, e.hex()
        n_none += want is None
    assert n_none > 100


def test_predicate_matches_the_oracle_on_every_family(edshim, fams):
    names = {}
    for name, pk, msg, sig in fams:
        want = E.expected(pk, msg, sig)
        assert bool(edshim.shim_verify(pk, msg, len(msg), sig)) == want, name
        names[name] = want
    assert names["honest"] and names["s = l - 1"] and not names["s = l"] and names["1 MiB message"]


def test_mixed_order_rejections_are_cofactored_acceptances(fams):
    """the 'rej' mixed-order cases are exactly where a cofactored verifier ([8]R' == [8]R) and dalek disagree"""
    for name, pk, msg, sig in fams:
        if name.startswith("mixed order"):
            a = O.decompress(pk)
            k = O.k_of(sig[:32], pk, msg)
            rp = O.add(O.mul(O.neg(a), k), O.mul(O.B, int.from_bytes(sig[32:], "little")))
            assert O.mul(rp, 8) == O.mul(O.decompress(sig[:32]), 8), name
            assert E.expected(pk, msg, sig) == name.endswith("acc"), name


def test_host_call_matches_the_oracle_on_every_family(fams):
    from bazuka_b200 import api
    for name, pk, msg, sig in fams:
        assert api.ed25519_verify(pk, msg, sig) == E.expected(pk, msg, sig), name
    from bazuka_b200 import _lib
    lib = _lib.load()
    pk, msg, sig = fams[0][1:]
    assert lib.bzk_ed25519_verify(pk, msg, len(msg), sig) == 1
    assert lib.bzk_ed25519_verify(None, msg, len(msg), sig) == -1
    assert lib.bzk_ed25519_verify(pk, msg, len(msg), None) == -1
    assert lib.bzk_ed25519_verify(pk, None, 3, sig) == -1
    assert lib.bzk_ed25519_verify(pk, None, 0, sig) == 0
