"""CPU tier: the field and group-law arithmetic of csrc/ff.cuh and csrc/ec.cuh at its carry, reduction and
exceptional-case edges, through the conformance harness (tests/devshim/arith.cu) built with g++ twice — once running
the device text (mul_evenodd, add/sub_limbs32) with an explicit carry variable, once the host fast paths
(mul/add/sub_host64) — and checked against Python big integers.  The GPU tier runs the same families on sm_90a."""
import ctypes as ct
import os

import numpy as np
import pytest

import arith_cases as A


@pytest.fixture(scope="module", params=["device_text", "host64"])
def host(request):
    return A.HostArith(request.param == "device_text")


@pytest.mark.parametrize("family", list(A.FAMILIES))
def test_arith_edges_host(host, family):
    assert A.run_family(host, family) == {}


@pytest.mark.parametrize("name", ["fr", "fp"])
def test_arith_edges_parameter_tables(name):
    """FrParams / FpParams as compiled: p, one = R mod p, r2 = R^2 mod p, inv = -p^-1 mod 2^32"""
    lib = ct.CDLL(A.build_host(False))
    p, n, t = A.FIELDS[name]
    out = np.zeros(3 * n + 1, dtype=np.uint32)
    lib.arith_params(t, out.ctypes.data_as(ct.c_void_p))
    got = A.ints(out[:3 * n].reshape(3, n))
    R = 1 << (32 * n)
    assert got == [p, R % p, R * R % p]
    assert int(out[3 * n]) == (-pow(p, -1, 1 << 32)) % (1 << 32)
    assert p < R >> 1   # the spare top bit add_limbs32 and the products rely on


def test_arith_edges_coverage_counts():
    """the families hold the edges they are meant to: printed with -s"""
    for name in A.FAMILIES:
        A.family(name)
    c = A.COUNTS
    print()
    for k in sorted(c):
        print(f"  {k:44s} {c[k]:7d}")
    for f, n in (("fr", 8), ("fp", 12)):
        assert c[f"{f} structured values"] >= (110 if n == 8 else 170)
        assert c[f"{f} structured pairs"] == c[f"{f} structured values"] ** 2
        for s in ("p-1", "p", "p+1", "2p-2"):
            assert c[f"{f} sum = {s}"] >= 1, s
        assert c[f"{f} carry/borrow runs"] == n * (n - 1)   # two of each (start, length) with start + length <= N - 1
        assert c[f"{f} Montgomery t in [p, p+2^32)"] >= 100 and c[f"{f} Montgomery t in [p-2^32, p)"] >= 100
        assert c[f"{f} lazy inner products"] == 5 * 17
        assert c[f"{f} inversion operands"] >= 2 * 32 * n
    assert c["fp2 c0 + c1 >= p"] >= 10 and c["fp2 c0 < c1"] >= 10
    assert c["g1 3-torsion points (0, +-2)"] == 2
    assert c["g1 lifted edge points"] >= 20 and c["g2 lifted edge points"] >= 5


def test_arith_edges_nvcc_build():
    """the sm_90a build of the harness compiles with libbzk's flags (a compile break shows before any GPU run)"""
    so = A.build_dev()
    assert os.path.getsize(so) > 0
    assert hasattr(ct.CDLL(so), "arith_run_dev")
