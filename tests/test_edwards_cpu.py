"""CPU tier: the Ed25519 and JubJub arithmetic of csrc/ed25519.cuh and csrc/jubjub.cuh, element by element, through the
conformance harness (tests/devshim/edwards.cu) built with g++ twice: once over the device text of the field arithmetic, once
over the host fast paths (mul/add/sub_host64, what bzk_ed25519_verify and the table builders run).  Every op is checked
against Python big integers (tests/edwards_cases.py).  Both fixed-base tables are read back entry by entry from each g++ build
and from the host code of the sm_90a build, which builds the tables libbzk uploads.  The GPU tier runs the same families on
sm_90a."""
import ctypes as ct

import numpy as np
import pytest

import arith_cases as A
import edwards_cases as E
from oracle.py import ed25519 as O

BUILDS = ["device_text", "host64"]


@pytest.fixture(scope="module", params=BUILDS)
def host(request):
    return E.HostEdwards(request.param == "device_text")


@pytest.mark.parametrize("family", list(E.FAMILIES))
def test_edwards_host(host, family):
    assert E.run_family(host, family) == {}


def _lib(build):
    if build == "nvcc_host":
        return ct.CDLL(E.build_dev())
    return ct.CDLL(E.build_host(build == "device_text"))


@pytest.mark.parametrize("name", list(E.FIELDS))
def test_edwards_parameter_tables(name):
    """P25519Params / L25519Params as compiled: p, one = R mod p, r2 = R^2 mod p, inv = -p^-1 mod 2^32, and for l the
    r3 = R^3 mod l that sc_from_hash multiplies the digest's upper half by"""
    out = E.read_params(_lib("host64"), name)
    p = E.FIELDS[name][0]
    R = 1 << 256
    assert A.ints(out[:24].reshape(3, 8)) == [p, R % p, R * R % p]
    assert int(out[24]) == (-pow(p, -1, 1 << 32)) % (1 << 32)
    assert p < R >> 1   # the spare top bit add_limbs32 and the products rely on
    assert A.ints(out[25:].reshape(1, 8)) == [R ** 3 % p if name == "l25519" else 0]


def test_edwards_nvcc_build():
    """the sm_90a build of the harness compiles with libbzk's flags (a compile break shows before any GPU run)"""
    assert hasattr(_lib("nvcc_host"), "edwards_run_dev")


@pytest.mark.parametrize("curve", list(E.CURVES))
@pytest.mark.parametrize("build", BUILDS + ["nvcc_host"])
def test_edwards_fixed_base_table_every_entry(build, curve):
    """ed_base_table() / jj_fixed_base_table(d): entry j * 256 + v is (y - x, y + x, 2dxy) of [v 2^(8j)] G, all 8192"""
    got = E.read_table(_lib(build), curve)
    want = E.table_words(curve)
    assert got.shape == want.shape == (E.TABLE_ENTRIES, 24)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert len(bad) == 0, f"{len(bad)} entries differ, first (j, v) = {[divmod(int(i), 256) for i in bad[:4]]}"


@pytest.mark.parametrize("build", BUILDS + ["nvcc_host"])
def test_edwards_constants(build):
    """ed_d, ed_d2, ed_sqrt_m1, ed_base and jj_base as the host code of each build computes them: D, 2D, sqrt(-1) and B of
    the Ed25519 oracle, BASE of the JubJub restatement (Montgomery images)"""
    got = E.read_consts(_lib(build))
    assert (got == E.host_const_images()).all()
    assert O.SQRT_M1 ** 2 % O.P == O.P - 1 and O.B[0] % 2 == 0


def test_edwards_fr_sqrt_roots_pin_the_generator():
    """fr_sqrt keeps c = 7^q in a local, so no op returns it; the jubjub.roots family pins it through the exact roots instead.
    Tonelli-Shanks with any other constant either finds no root for some residues (c' not a primitive 2^32-th root of
    unity) or returns the other root -x for some of the family's inputs (c' an odd power of c)"""
    r = E.R_FR
    q = (r - 1) >> 32
    c = E._fr_sqrt_c()
    assert c == pow(7, q, r) and pow(c, 1 << 31, r) == r - 1

    def ts(a, gen):   # fr_sqrt's loop with the generator as a parameter
        m, t, x = 32, pow(a, q, r), pow(a, (q + 1) // 2, r)
        while t != 1:
            i, t2 = 0, t
            while t2 != 1:
                t2 = t2 * t2 % r
                i += 1
                if i == m:
                    return None
            b = pow(gen, 1 << (m - i - 1), r)
            m, gen = i, b * b % r
            t, x = t * gen % r, x * b % r
        return x if x * x % r == a else None
    ins = [a for a, _ in E.fr_sqrt_inputs() if a]
    assert [ts(a, c) for a in ins] == [E.N.fr_sqrt(a) for a in ins]
    for other in [pow(c, e, r) for e in (3, 5, 7, (1 << 30) + 1, (1 << 31) + 1, (1 << 32) - 1)] + [c + 1, c ^ (1 << 200)]:
        assert any(ts(a, other) != ts(a, c) for a in ins), other


def test_edwards_host_call_table_sweep():
    """bzk_ed25519_verify (the host table) on the identity key, where the verdict is compress([s] B) == R: every 4th entry of
    the table sweep with s < l accepts R = [s] B and refuses R = [s + 1] B"""
    from bazuka_b200 import api
    ident = (1).to_bytes(32, "little")
    sw = E.sweep("ed25519", O.L)[::4]
    for j, v, s, pt in sw:
        sb = s.to_bytes(32, "little")
        assert api.ed25519_verify(ident, b"sweep", O.compress(pt) + sb), (j, v)
        assert not api.ed25519_verify(ident, b"sweep", O.compress(O.add(pt, O.B)) + sb), (j, v)
    assert len(sw) == 1989


def test_edwards_coverage_counts():
    """the families hold the edges they are meant to: printed with -s"""
    for name in E.FAMILIES:
        E.family(name)
    c = A.COUNTS
    print()
    for k in sorted(c):
        if k.split()[0] in ("p25519", "l25519", "ed25519", "jubjub", "sha512", "fr_sqrt"):
            print(f"  {k:48s} {c[k]:7d}")
    for curve in E.CURVES:
        assert c[f"{curve} fixed-base sweep scalars"] == E.TABLE_ENTRIES
        for order, n in ((1, 1), (2, 1), (4, 2), (8, 4)):
            assert c[f"{curve} torsion points of order {order}"] == n, (curve, order)
        assert c[f"{curve} points"] >= 19
        assert c[f"{curve} mul records"] >= 20 * len(E.k_edges())
    assert c["sha512 lengths 0-300"] == 301
    for f in ("p25519", "l25519"):
        assert c[f"{f} Montgomery t in [p, p+2^32)"] >= 100 and c[f"{f} Montgomery t in [p-2^32, p)"] >= 100, f
        assert c[f"{f} inversion operands"] >= 2 * 32 * 8
    assert c["p25519 reduce_once above the modulus"] == 19 and c["l25519 reduce_once above the modulus"] >= 100
    assert c["l25519 wide-operand products"] >= 1000
    ks = E.k_edges()
    L, r, order = E.L, E.R_FR, E.ORDER
    assert ks == [0, 1, 15, 16, 255, 256, L - 1, L, L + 1, 8 * L - 1, r - 1, order - 1, order + 1, 2**255, 2**256 - 1]
    for i in range(32):
        assert c[f"fr_sqrt a^q of order 2^{i}"] >= 3, i
    assert c["fr_sqrt a^q of order 2^32"] >= 2
    assert c["ed25519 sqrt_ratio_i squares"] >= 100 and c["ed25519 sqrt_ratio_i non-squares"] >= 100
    assert c["ed25519 decompress refusals"] >= 100 and c["jubjub decompress refusals"] >= 10
