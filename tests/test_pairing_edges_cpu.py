"""CPU tier: the device half of csrc/pairing.cuh (f12_mul, f12_sqr, f12_mul_sparse and their fold, miller_one_xyzz) and
k_verify_miller's per-proof steps (mul127, the malformed-proof predicate), through the conformance harness
tests/devshim/pairing.cu built with g++ twice — on the device text and on the host fast paths.  Fp12 products are checked
exactly against Python integers, the Miller loop through the final exponentiation against the host verifier's
multi_miller and the oracle's pairing.  The GPU tier runs the same families on sm_90a."""
import ctypes as ct
import os

import numpy as np
import pytest

import pairing_cases as PC
from oracle.py import curve as C


@pytest.fixture(scope="module")
def hosts():
    return {"device_text": PC.HostPairing(True), "host64": PC.HostPairing(False)}


@pytest.mark.parametrize("build", ["device_text", "host64"])
@pytest.mark.parametrize("family", list(PC.FAMILIES))
def test_pairing_edges_host(hosts, build, family):
    assert PC.run_family(hosts[build], family)[0] == {}


@pytest.mark.parametrize("family", list(PC.FAMILIES))
def test_pairing_edges_host_builds_agree(hosts, family):
    """the device text and the host fast paths give the same words on every record, the Miller loop included"""
    a, b = PC.run_family(hosts["device_text"], family)[1], PC.run_family(hosts["host64"], family)[1]
    for op in a:
        assert (a[op] == b[op]).all(), op


def _final_exp(host, f):
    return host.run("final_exp", f)


def test_miller_xyzz_scaling_vanishes_in_the_final_exponentiation(hosts):
    """final_exp(miller_one_xyzz(P in XYZZ form, Q)) == final_exp(multi_miller(P affine, Q)) for every record: the ZZ*ZZZ
    factor on every line is an Fp scalar, which the final exponentiation removes; identities give one"""
    h = hosts["host64"]
    recs = PC.miller_records()
    f_x = h.run("miller_xyzz", PC.miller_inputs(recs))
    f_a = h.run("multi_miller", PC.rec(PC.G1.affine([r[0] for r in recs]), PC.G2.affine([r[2] for r in recs])))
    e_x, e_a = _final_exp(h, f_x), _final_exp(h, f_a)
    one = PC.f12_img([(1, 0)] + [(0, 0)] * 5)
    for i, (Pt, lam, Q, tors) in enumerate(recs):
        assert (e_x[i] == e_a[i]).all(), (i, lam, tors)
        trivial = Pt is None or Q is None
        assert (e_x[i] == one).all() == trivial, i
        if trivial:
            assert (f_x[i] == one).all(), i
    # the scaled lines really differ before the final exponentiation when ZZ*ZZZ != 1
    scaled = [i for i, r in enumerate(recs) if r[0] is not None and r[2] is not None and r[1] != 1]
    assert scaled and all(not (f_x[i] == f_a[i]).all() for i in scaled)
    unscaled = [i for i, r in enumerate(recs) if r[0] is not None and r[2] is not None and r[1] == 1]
    assert unscaled and all((f_x[i] == f_a[i]).all() for i in unscaled)


def test_miller_xyzz_is_the_oracle_pairing_cubed(hosts):
    """a few pairs (the Python pairing takes seconds): final_exp(miller_one_xyzz(P, Q)) == e(P, Q)^3, with P under a random
    lambda, including -P and -Q"""
    h = hosts["device_text"]
    g1, (g2, _) = PC.g1_points(), PC.g2_points()
    lam = PC.lambdas()[1]
    pairs = [(g1[0], g2[0]), (g1[1], g2[2]), (g1[3], g2[1]), (g1[2], g2[3])]
    recs = [(Pt, lam, Q, True) for Pt, Q in pairs]
    e = _final_exp(h, h.run("miller_xyzz", PC.miller_inputs(recs)))
    for i, (Pt, Q) in enumerate(pairs):
        assert PC.f12_to_oracle(e[i]) == C.f12_pow(C.pairing(Q, Pt), 3), i


def test_pairing_edges_coverage_counts():
    """the families hold the edges they are meant to: printed with -s"""
    for name in PC.FAMILIES:
        PC.family(name)
    c = PC.COUNTS
    print()
    for k in sorted(c):
        print(f"  {k:48s} {c[k]:7d}")
    assert c["f12 operands"] >= 40 and c["f12 product pairs"] >= 500
    assert c["sparse lines with a zero part"] >= 16
    assert c["miller records with ZZ*ZZZ != 1"] >= 40
    assert c["g2 twist points outside the r-torsion"] == 3
    assert c["mul127 multipliers with bit 126 set"] >= 7 * 6
    assert c["proof images with a non-canonical coordinate"] >= 8 + 8 + 12


def test_pairing_harness_nvcc_build():
    """the sm_90a build of the harness compiles with libbzk's flags (a compile break shows before any GPU run)"""
    so = PC.build_dev()
    assert os.path.getsize(so) > 0
    assert hasattr(ct.CDLL(so), "pairing_run_dev")
