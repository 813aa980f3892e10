"""CPU tier: the degenerate and boundary constraint systems of r1cs_cases.py held to their claims in big integers, and the
two oracles held to each other on them.  For every case with m <= 2^7 the C oracle's key (groth16_c.setup) equals the
big-integer restatement's (oracle/py/groth16.setup) point for point, except on cancelling duplicates, where the
difference is exactly one identity per cancelled variable; the C oracle's proof bytes equal the restatement's at the same
(r, s), and the restatement's pairing check accepts them (refuses them for an unsatisfied witness).  The blocked forms
expand to the explicit CSR, and csrc/r1cs_blocked.cuh compiled for the host evaluates, lists densities and transposes
them as the expansion does."""
import multiprocessing as mp
import random

import numpy as np
import pytest

import r1cs_cases as RC
from oracle import groth16_c as GC
from oracle.py import curve as C, groth16 as G
from test_blocked_r1cs_cpu import P, hb, host_columns, host_density, host_spmv, oracle_columns, rand_fr  # noqa: F401 (hb: fixture)

CASES = RC.all_cases()
BY_NAME = {c.name: c for c in CASES}
BIG = [c.name for c in CASES if c.big_int]


def _big_int_reference(name):
    """the restatement's key, proof bytes and verdict for one case (run in a worker process)"""
    case = BY_NAME[name]
    pk = G.setup(case.cs, *case.toxic)
    proof = G.prove(case.cs, pk, case.z, case.r, case.s)
    ok = G.verify(pk["vk"], case.z[1:case.ni], proof)
    keep = {k: pk[k] for k in ("h", "l", "a", "b_g1", "b_g2", "a_all", "b1_all")}
    keep["ic"] = pk["vk"]["ic"]
    return keep, G.proof_to_bytes(proof), ok


@pytest.fixture(scope="module")
def big_int():
    """every case's restatement, computed on all cores at once (the products are pure Python)"""
    with mp.get_context("fork").Pool() as pool:
        return dict(zip(BIG, pool.map(_big_int_reference, BIG, chunksize=1)))


def test_case_counts():
    fam = {f: sum(1 for c in CASES if c.family == f) for f in RC.FAMILIES}
    assert fam == {"boundary": 55, "large": 0, "degenerate": 8, "density": 5, "value": 3, "unsat": 4, "blocked": 6}
    assert [c.expect[0] for c in CASES if c.family == "boundary"].count(8) == 3     # 2^7 + 1 rows: past the big-integer range


@pytest.mark.parametrize("name", [c.name for c in CASES])
def test_case_holds_its_claims_in_big_integers(name):
    from bazuka_b200.groth16 import R1CS
    case = BY_NAME[name]
    assert RC.bad_rows(case) == case.bad
    assert case.cs.is_satisfied(case.z) == (case.bad == 0)
    log_m, h, l, a, b = case.expect
    assert (1 << log_m) >= case.ncons + case.ni and (log_m == 0 or (1 << (log_m - 1)) < case.ncons + case.ni)
    assert log_m == G.domain_log(len(case.cs.with_input_constraints())) and h == (1 << log_m) - 1 and l == case.na
    assert case.expect == RC.presence_shape(case.ni, case.na, case.cs.rows)
    mats = RC.case_mats(case)
    r = R1CS(case.ni, case.na, *mats)
    a_idx, b_idx = r.density()
    ga, gb = GC.density(case.ni, case.na, mats)
    assert r.log_m == log_m and (len(a_idx), len(b_idx)) == (a, b)
    assert (a_idx == ga).all() and (b_idx == gb).all()


@pytest.mark.parametrize("name", BIG)
def test_c_oracle_key_and_proof_equal_the_big_integer_restatement(cref, big_int, name):
    case = BY_NAME[name]
    mats = RC.case_mats(case)
    cpk = GC.setup(case.ni, case.na, mats, RC.toxic(case))
    ref, want, ok = big_int[name]
    pts = lambda imgs, f=C.g1_from_bytes: [f(bytes(x)) for x in imgs]
    assert pts(cpk["h"]) == ref["h"] and len(ref["h"]) == case.expect[1]
    assert pts(cpk["l"]) == ref["l"] and pts(cpk["vk"]["ic"]) == ref["ic"]
    if case.cancelling:
        # the library's presence rule keeps the cancelled variables with an identity column; bellman's generator drops them
        a_i, b_i = GC.density(case.ni, case.na, mats)
        ids_a = [i for i, v in enumerate(a_i) if v in case.cancelling]
        ids_b = [i for i, v in enumerate(b_i) if v in case.cancelling]
        assert len(ids_a) + len(ids_b) == len(case.cancelling) >= 1
        for i in ids_a:
            assert ref["a_all"][a_i[i]] is None and cpk["a"][i][96] == 1
        for i in ids_b:
            assert ref["b1_all"][b_i[i]] is None and cpk["b_g1"][i][96] == 1 and cpk["b_g2"][i][192] == 1
        drop = lambda imgs, ids: np.delete(imgs, ids, axis=0)
        assert pts(drop(cpk["a"], ids_a)) == ref["a"] and pts(drop(cpk["b_g1"], ids_b)) == ref["b_g1"]
        assert pts(drop(cpk["b_g2"], ids_b), C.g2_from_bytes) == ref["b_g2"]
    else:
        assert pts(cpk["a"]) == ref["a"] and pts(cpk["b_g1"]) == ref["b_g1"]
        assert pts(cpk["b_g2"], C.g2_from_bytes) == ref["b_g2"]
        assert len(ref["a"]) == case.expect[3] and len(ref["b_g1"]) == case.expect[4]
    inputs, aux = RC.witness(case)
    r, s = RC.rs(case)
    got = GC.prove(case.ni, case.na, mats, cpk, inputs, aux, r, s)
    assert bytes(GC.proof_bytes(*got)) == want
    assert ok == (case.bad == 0)


@pytest.mark.parametrize("name", [c.name for c in CASES if not c.big_int])
def test_c_oracle_proof_verifies_above_the_big_integer_range(cref, name):
    from bazuka_b200 import groth16 as BG
    case = BY_NAME[name]
    mats = RC.case_mats(case)
    cpk = GC.setup(case.ni, case.na, mats, RC.toxic(case))
    inputs, aux = RC.witness(case)
    proof = GC.prove(case.ni, case.na, mats, cpk, inputs, aux, *RC.rs(case))
    assert BG.verify(cpk["vk"], inputs[1:], proof)


@pytest.mark.parametrize("name", [c.name for c in CASES])
def test_blocked_form_expands_to_the_explicit_csr(hb, name):
    case = BY_NAME[name]
    br = RC.blocked_r1cs(case)
    ex = br.expand()
    assert (ex.num_inputs, ex.num_aux, ex.num_constraints) == (case.ni, case.na, case.ncons)
    for (rp, col, val), (rp2, col2, val2) in zip(ex.mats, RC.case_mats(case)):
        assert (rp == rp2).all() and (col == col2).all() and (val == val2).all()
    for rp, col, val in br.mats:
        assert hb.h_valid(P(np.array(br.blocks, np.uint64)), br.num_vars, P(rp), P(col), P(val))
    for got, w, np_ in zip(host_density(hb, br), ex.density(), br.density()):
        assert (got == w).all() and (np_ == w).all()
    # the header's row mapping evaluates every logical row as the big-integer rows do
    z = np.ascontiguousarray(RC.mont(case.z))
    want = [[RC.ev(row[k], case.z) for row in case.cs.rows] for k in range(3)]
    if case.ncons:
        for got, w in zip(host_spmv(hb, br, z), want):
            assert [int(x) for x in from_mont(got)] == w
        lag = rand_fr(random.Random(case.seed), case.ncons)
        for got, w in zip(host_columns(hb, br, lag), oracle_columns(ex, lag)):
            assert [int.from_bytes(x.tobytes(), "little") for x in got] == w


def from_mont(a):
    rinv = pow(1 << 256, -1, RC.R)
    return [int.from_bytes(x.tobytes(), "little") * rinv % RC.R for x in a]


@pytest.mark.parametrize("image", ["r-1", "r", "r+1", "2^256-1"])
def test_blocked_validation_refuses_coefficient_images_not_below_r(hb, image):
    """an image >= r (r itself is a zero that would count as present) is refused; r - 1 is the largest canonical one"""
    case = BY_NAME["blocked-reps1"]
    br = RC.blocked_r1cs(case)
    rp, col, val = (x.copy() for x in br.mats[1])
    v = {"r-1": RC.R - 1, "r": RC.R, "r+1": RC.R + 1, "2^256-1": (1 << 256) - 1}[image]
    val[len(val) // 2] = np.frombuffer(v.to_bytes(32, "little"), np.uint64)
    ok = bool(hb.h_valid(P(np.array(br.blocks, np.uint64)), br.num_vars, P(rp), P(col), P(val)))
    assert ok == (image == "r-1")
