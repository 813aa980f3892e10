"""CPU tier of the batch EdDSA checks: csrc/jubjub.cuh (the code the kernels of csrc/jubjub.cu run) compiled with g++ over the
device text of the field arithmetic, against the Python restatement of the reference's JubJub (bazuka_b200/mpn/native.py)."""
import ctypes as ct
import os
import random
import subprocess

import numpy as np
import pytest

import eddsa_cases as E
from bazuka_b200.mpn import native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = N.R


@pytest.fixture(scope="module")
def jjshim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("jubjub_shim") / "_jubjub_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-DBZK_HOST_DEVICE_TEXT", "-I", os.path.join(ROOT, "bazuka_b200", "csrc"),
                           os.path.join(ROOT, "tests", "hostshim", "jubjub_shim.cpp"), "-o", out])
    lib = ct.CDLL(out)
    for f in ("shim_jj_decompress", "shim_eddsa_item"):
        getattr(lib, f).restype = ct.c_int
    return lib


def u256(*vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint64).copy()


def ints(a):
    b = a.tobytes()
    return [int.from_bytes(b[32 * i:32 * i + 32], "little") for i in range(len(b) // 32)]


P = lambda a: a.ctypes.data_as(ct.c_void_p)
D = u256(N.JJ_D)


def test_decompression_matches_the_restatement(jjshim):
    rng = random.Random(5)
    xs = [0, 1, 2, 6, 7, R - 1, R - 2] + list(range(3, 600)) + [rng.randrange(R) for _ in range(1400)]
    y = u256(0)
    n_none = 0
    for x in xs:
        for odd in (False, True) if x in (0, 1, 2, 6, R - 1) or x % 5 == 0 else (bool(x & 1),):
            want = N.jj_decompress_checked((x, odd))
            got = jjshim.shim_jj_decompress(P(D), P(u256(x)), int(odd), P(y))
            assert bool(got) == (want is not None), (x, odd)
            if want is not None:
                assert ints(y)[0] == want[1], (x, odd)
            n_none += want is None
    assert n_none > 100   # non-residues are among the inputs


def _points():
    t = E.torsion_points()
    i = E.sqrt_m1()
    b2 = N.jj_mul(E.BASE, 2)
    return {"BASE": E.BASE, "identity": E.IDENTITY, "(0,-1)": (0, R - 1), "(i,0)": (i, 0), "(-i,0)": (R - i, 0), "order 8": t[1],
            "order 8 (3)": t[3], "BASE + T8": N.jj_add(E.BASE, t[1]), "2 BASE + T4": N.jj_add(b2, t[2]), "key + T2": N.jj_add(N.eddsa_keys(b"k")[0], t[4])}


_SCALARS = [0, 1, 2, E.ORDER - 1, E.ORDER, E.ORDER + 1, 8 * E.ORDER - 1, 1 << 254, R - 1, 15, 16, 255, 256, (1 << 256) - 1]


def test_windowed_multiplication_matches_the_restatement(jjshim):
    rng = random.Random(6)
    out = u256(0, 0)
    for name, p in _points().items():
        assert N.jj_on_curve(p), name
        for k in _SCALARS + [rng.randrange(R) for _ in range(3)]:
            jjshim.shim_jj_mul(P(D), P(u256(p[0])), P(u256(p[1])), P(u256(k)), P(out))
            assert tuple(ints(out)) == N.jj_mul(p, k), (name, k)


def test_fixed_base_table_matches_the_restatement(jjshim):
    rng = random.Random(7)
    out = u256(0, 0)
    for k in _SCALARS + [rng.randrange(R) for _ in range(20)] + [1 << (8 * j) for j in range(32)] + [255 << (8 * j) for j in range(32)]:
        jjshim.shim_jj_mul_fixed(P(D), P(u256(k)), P(out))
        assert tuple(ints(out)) == N.jj_mul(E.BASE, k), k


@pytest.mark.parametrize("seed", [b"f", b"g"])
def test_predicate_matches_the_restatement_on_every_family(jjshim, seed):
    for name, pk, msg, r, s in E.families(seed):
        a = N.jj_decompress_checked(pk) if 0 <= pk[0] < R else None
        h = N.poseidon([r[0], r[1], a[0], a[1], msg]) if a is not None else 0
        got = jjshim.shim_eddsa_item(P(D), P(u256(pk[0])), int(pk[1]), P(u256(msg)), P(u256(r[0])), P(u256(r[1])), P(u256(s)), P(u256(h)))
        assert bool(got) == E.expected(pk, msg, r, s), name


def test_eddsa_item_struct_matches_the_header(tmp_path):
    """signatures.ITEM (what mpn/signatures.py packs) against gcc's view of bzk_eddsa_item in include/bzk.h"""
    from bazuka_b200.mpn import signatures as S
    fs = ["pk_x", "pk_odd", "message", "sig_rx", "sig_ry", "sig_s"]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "bzk.h"', 'int main(void) {', 'printf("%zu", sizeof(bzk_eddsa_item));']
    src += [f'printf(" %zu", offsetof(bzk_eddsa_item, {f}));' for f in fs] + ['printf("\\n");', "return 0;", "}"]
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    size, *offs = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert size == S.ITEM.itemsize == 168
    assert [S.ITEM.fields[f][1] for f in fs] == offs
