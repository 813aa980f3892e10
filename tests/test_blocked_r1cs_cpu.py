"""CPU tier: the blocked R1CS.  The blocked compile of the update circuit against the explicit one (expansion, shape,
blocks, witness programs), and the index arithmetic of csrc/r1cs_blocked.cuh compiled for the host against numpy and
big-integer sums over the expanded matrices: row mapping, forward product, density lists, transposed product, and the
upload's validation."""
import ctypes as ct
import os
import random
import subprocess

import numpy as np
import pytest

from conftest import ROOT, fr_arr

R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
RINV = pow(1 << 256, -1, R)

HARNESS = r"""
#include <string.h>
#include "r1cs_blocked.cuh"
using namespace bzk;
static BlockedShape shape_of(const uint64_t s[6]) {
    BlockedShape b;
    b.head_rows = s[0]; b.tmpl_rows = s[1]; b.reps = s[2]; b.tail_rows = s[3]; b.var_lo = s[4]; b.var_stride = s[5];
    return b;
}
extern "C" uint64_t h_row(const uint64_t s[6], uint64_t r, uint64_t *shift) { return blocked_row(shape_of(s), r, shift); }
extern "C" int h_valid(const uint64_t s[6], uint64_t nv, const uint64_t *rp, const uint32_t *col, const void *val) {
    return blocked_valid(shape_of(s), nv, rp, col, val);
}
extern "C" void h_spmv(const uint64_t s[6], const uint64_t *rp, const uint32_t *col, const Fr *val, const Fr *z, Fr *out) {
    const BlockedShape b = shape_of(s);
    for (uint64_t r = 0; r < b.rows(); r++) out[r] = blocked_row_dot(b, rp, col, val, r, z);
}
extern "C" void h_density(const uint64_t s[6], uint64_t ni, uint64_t nv, const uint64_t *rpa, const uint32_t *cola, const Fr *vala,
                          const uint64_t *rpb, const uint32_t *colb, const Fr *valb, uint32_t *a_idx, uint32_t *b_idx, uint64_t lens[2]) {
    const BlockedShape b = shape_of(s);
    std::vector<uint8_t> a_d(nv, 0), b_d(nv, 0);
    blocked_presence(b, rpa, cola, vala, a_d);
    blocked_presence(b, rpb, colb, valb, b_d);
    std::vector<uint32_t> a, bb;
    density_lists(ni, a_d, b_d, a, bb);
    memcpy(a_idx, a.data(), a.size() * 4);
    memcpy(b_idx, bb.data(), bb.size() * 4);
    lens[0] = a.size(); lens[1] = bb.size();
}
// the passes of bzk_r1cs_columns_dev, in order
extern "C" void h_columns(const uint64_t s[6], uint64_t nv, const uint64_t *rp, const uint32_t *col, const Fr *val, const Fr *lag, Fr *out) {
    const BlockedShape b = shape_of(s);
    const HostBlockedT t = blocked_transpose(b, rp, col, val);
    for (uint64_t j = 0; j < nv; j++) out[j] = blocked_slot_column(b, t.span, t.s_ptr.data(), t.s_row.data(), t.s_val.data(), lag, j);
    if (!t.shared.col.empty()) {
        std::vector<Fr> sums(b.tmpl_rows);
        for (uint64_t r = 0; r < b.tmpl_rows; r++) sums[r] = blocked_tmpl_rowsum(b, lag, r);
        for (uint64_t u = 0; u < t.shared.col.size(); u++)
            out[t.shared.col[u]] = out[t.shared.col[u]] + col_list_dot(t.shared.ptr.data(), t.shared.row.data(), t.shared.val.data(), sums.data(), u);
    }
    for (uint64_t u = 0; u < t.fixed.col.size(); u++)
        out[t.fixed.col[u]] = out[t.fixed.col[u]] + col_list_dot(t.fixed.ptr.data(), t.fixed.row.data(), t.fixed.val.data(), lag, u);
}
"""


@pytest.fixture(scope="module")
def hb(tmp_path_factory):
    d = tmp_path_factory.mktemp("r1cs_blocked")
    src, so = d / "harness.cpp", d / "harness.so"
    src.write_text(HARNESS)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(ROOT, "bazuka_b200", "csrc"),
                           str(src), "-o", str(so)])
    lib = ct.CDLL(str(so))
    lib.h_row.restype = ct.c_uint64
    lib.h_row.argtypes = [ct.c_void_p, ct.c_uint64, ct.c_void_p]
    lib.h_valid.argtypes = [ct.c_void_p, ct.c_uint64, ct.c_void_p, ct.c_void_p, ct.c_void_p]
    lib.h_density.argtypes = [ct.c_void_p, ct.c_uint64, ct.c_uint64] + [ct.c_void_p] * 9
    lib.h_columns.argtypes = [ct.c_void_p, ct.c_uint64] + [ct.c_void_p] * 5
    lib.h_spmv.argtypes = [ct.c_void_p] * 6
    return lib


def P(a):
    return ct.c_void_p(a.ctypes.data)


def shape(br):
    return np.array(br.blocks, dtype=np.uint64)


def host_spmv(hb, br, z):
    out = [np.zeros((br.num_constraints, 4), np.uint64) for _ in range(3)]
    for k, (rp, col, val) in enumerate(br.mats):
        hb.h_spmv(P(shape(br)), P(rp), P(col), P(val), P(z), P(out[k]))
    return out


def host_columns(hb, br, lag):
    out = [np.zeros((br.num_vars, 4), np.uint64) for _ in range(3)]
    for k, (rp, col, val) in enumerate(br.mats):
        hb.h_columns(P(shape(br)), br.num_vars, P(rp), P(col), P(val), P(lag), P(out[k]))
    return out


def host_density(hb, br):
    a, b = np.zeros(br.num_vars, np.uint32), np.zeros(br.num_vars, np.uint32)
    lens = np.zeros(2, np.uint64)
    (ra, ca, va), (rb, cb, vb) = br.mats[:2]
    hb.h_density(P(shape(br)), br.num_inputs, br.num_vars, P(ra), P(ca), P(va), P(rb), P(cb), P(vb), P(a), P(b), P(lens))
    return a[:int(lens[0])], b[:int(lens[1])]


def as_explicit(r1cs):
    """an R1CS as a blocked one with every row in the head (no template)"""
    from bazuka_b200.groth16 import BlockedR1CS
    return BlockedR1CS(r1cs.num_inputs, r1cs.num_aux, r1cs.num_constraints, 0, 0, 0, r1cs.num_vars, 0, *r1cs.mats)


def mont_mul(a, b):
    return a * b * RINV % R


def oracle_spmv(r1cs, z):
    """big-integer <M_row, z> over the explicit matrices, Montgomery images in and out"""
    zi = [int.from_bytes(x.tobytes(), "little") for x in z]
    out = []
    for rp, col, val in r1cs.mats:
        vi = [int.from_bytes(x.tobytes(), "little") for x in val]
        rows = []
        for r in range(r1cs.num_constraints):
            rows.append(sum(mont_mul(vi[e], zi[col[e]]) for e in range(int(rp[r]), int(rp[r + 1]))) % R)
        out.append(rows)
    return out


def oracle_columns(r1cs, lag):
    li = [int.from_bytes(x.tobytes(), "little") for x in lag]
    out = []
    for rp, col, val in r1cs.mats:
        vi = [int.from_bytes(x.tobytes(), "little") for x in val]
        cols = [0] * r1cs.num_vars
        for r in range(r1cs.num_constraints):
            for e in range(int(rp[r]), int(rp[r + 1])):
                cols[col[e]] = (cols[col[e]] + mont_mul(vi[e], li[r])) % R
        out.append(cols)
    return out


def as_ints(a):
    return [int.from_bytes(x.tobytes(), "little") for x in a]


def rand_fr(rng, n):
    return np.array([list((rng.randrange(R)).to_bytes(32, "little")) for _ in range(n)], dtype=np.uint8).view(np.uint64).reshape(n, 4)


# ------------------------------------------------------------------ a synthetic blocked R1CS with the edges
NI, NA, VAR_LO, STRIDE = 3, 40, 10, 6


def synthetic(seed, reps):
    """head 4 rows, template 5 rows (slot columns spanning two strides, var_lo - 1 and var_lo both used), tail 4 rows that
    read the last copy and the one variable nothing else names (nv - 1); empty rows in each part; some zero coefficients"""
    from bazuka_b200.groth16 import BlockedR1CS
    rng = random.Random(seed)
    nv = NI + NA
    last = VAR_LO + (reps - 1) * STRIDE
    head = [[0, 1, 5], [], [VAR_LO + 2, 4], [2]]
    tmpl = [[VAR_LO - 1, VAR_LO], [], [VAR_LO + 11, 0, VAR_LO + 6], [VAR_LO + 3, 7], [VAR_LO, VAR_LO + 1, 1]]
    tail = [[last + 11, nv - 1], [], [last, 0], [last + 6, 3]]
    mats = []
    for side in range(3):
        rows = [list(r) for r in head + tmpl + tail]
        for r in rows:
            rng.shuffle(r)
            if side and r:
                r.pop()          # the sides differ
        rp = np.zeros(len(rows) + 1, np.uint64)
        np.cumsum([len(r) for r in rows], out=rp[1:])
        col = np.array([c for r in rows for c in r], dtype=np.uint32)
        val = rand_fr(rng, len(col))
        if len(val) > 3:
            val[3] = 0           # a zero coefficient: not a density entry
        mats.append((rp, col, val))
    return BlockedR1CS(NI, NA, len(head), len(tmpl), reps, len(tail), VAR_LO, STRIDE, *mats)


@pytest.mark.parametrize("reps", [1, 3])
def test_row_mapping(hb, reps):
    br = synthetic(10 + reps, reps)
    shift = np.zeros(1, np.uint64)
    want = list(range(4)) + [4 + t for _ in range(reps) for t in range(5)] + [9 + t for t in range(4)]
    shifts = [0] * 4 + [k * STRIDE for k in range(reps) for _ in range(5)] + [0] * 4
    for r in range(br.num_constraints):
        assert hb.h_row(P(shape(br)), r, P(shift)) == want[r]
        assert int(shift[0]) == shifts[r]


@pytest.mark.parametrize("reps", [1, 3])
def test_forward_product_and_transposed_product_vs_big_integers(hb, reps):
    br = synthetic(20 + reps, reps)
    ex = br.expand()
    # the expansion: slot columns moved by k * stride, var_lo - 1 left in place
    tc = br.mats[0][1][br.mats[0][0][4]:br.mats[0][0][9]]
    assert (VAR_LO - 1 in tc) and (VAR_LO in tc)
    rng = random.Random(reps)
    z, lag = rand_fr(rng, br.num_vars), rand_fr(rng, br.num_constraints)
    for got, want in zip(host_spmv(hb, br, z), oracle_spmv(ex, z)):
        assert as_ints(got) == want
    cols = host_columns(hb, br, lag)
    want = oracle_columns(ex, lag)
    for got, w in zip(cols, want):
        assert as_ints(got) == w
    assert want[0][NI + NA - 1] != 0                    # the tail-only variable has a column


@pytest.mark.parametrize("reps", [1, 3])
def test_density_lists_equal_the_expansions(hb, reps):
    br = synthetic(30 + reps, reps)
    want = br.expand().density()
    for got, w, np_ in zip(host_density(hb, br), want, br.density()):
        assert (got == w).all() and (np_ == w).all()
    assert NI + NA - 1 in want[0]


def test_validation_refuses_what_the_blocked_form_cannot_name(hb):
    br = synthetic(40, 3)
    nv = br.num_vars
    rp, col, val = (x.copy() for x in br.mats[0])
    ok = lambda s, c=col, r=rp: hb.h_valid(P(np.array(s, np.uint64)), nv, P(r), P(c), P(val))
    assert ok(br.blocks)
    # the last copy's largest relative column: VAR_LO + 11 + 2 * STRIDE = 33 < 43; with 6 copies it is 51
    assert not ok((4, 5, 6, 4, VAR_LO, STRIDE))
    assert ok((4, 5, 3, 4, VAR_LO, 0)) == 0                 # a repeated template with a zero stride
    bad = col.copy()
    bad[0] = nv
    assert not ok(br.blocks, c=bad)
    r2 = rp.copy()
    r2[2] = r2[3] + 1                                      # a decreasing rowptr
    assert not ok(br.blocks, r=r2)
    r3 = rp.copy()
    r3[0] = 1
    assert not ok(br.blocks, r=r3)


# ------------------------------------------------------------------ the update circuit
def _pair(A, T, B):
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    return NativeUpdateCircuit(A, T, B), NativeUpdateCircuit(A, T, B, blocked=True)


@pytest.mark.parametrize("A,T,B", [(1, 1, 0), (1, 1, 1), (2, 1, 2), (3, 2, 1)])
def test_blocked_compile_expands_to_the_explicit_compile(A, T, B):
    e, b = _pair(A, T, B)
    ni, na, mats = e.r1cs()
    br = b.blocked_r1cs()
    ex = br.expand()
    assert (ex.num_inputs, ex.num_aux) == (ni, na)
    for (rp, col, val), (rp2, col2, val2) in zip(ex.mats, mats):
        assert (rp == rp2).all() and (col == col2).all() and (val == val2).all()
    # the shape is the expanded system's; the blocks lie where the explicit compile reports them
    for k in ("num_inputs", "num_aux", "num_constraints", "nnz_a", "nnz_b", "nnz_c", "p_aux", "slot_vars", "state_out", "final_fee", "epilogue_vars"):
        assert getattr(e, k) == getattr(b, k), k
    (blocks_e, nnz_e), (blocks_b, nnz_b) = e.blocks(), b.blocks()
    assert blocks_e == blocks_b == br.blocks
    head, tmpl, reps, tail, var_lo, stride = blocks_e
    assert reps == (1 << (2 * B)) - 1 and (tmpl == 0) == (B == 0)
    assert var_lo == ni + e.p_aux and stride == e.slot_vars
    assert nnz_e == (e.nnz_a, e.nnz_b, e.nnz_c)
    for k, (rp, _, _) in enumerate(mats):
        assert int(rp[-1] - rp[head + reps * tmpl]) == int(br.mats[k][0][-1] - br.mats[k][0][head + tmpl])  # the tail
        assert nnz_b[k] == len(br.mats[k][1])
    e.free(); b.free()


@pytest.mark.parametrize("A,T,B", [(1, 1, 0), (2, 1, 2)])
def test_blocked_compile_has_the_same_witness_programs(A, T, B):
    e, b = _pair(A, T, B)
    for which in (0, 1):
        p, q = e.program(which), b.program(which)
        for k in ("ops", "lc_ptr", "lc_slot", "lc_coef"):
            assert (np.asarray(getattr(p, k)) == np.asarray(getattr(q, k))).all(), (which, k)
        assert p.coefs == q.coefs and p.n_raw == q.n_raw and p.n_ext == q.n_ext
    e.free(); b.free()


def test_update_circuit_host_products_equal_the_explicit_ones(hb):
    """the header's passes on the blocked form of a 16-slot batch against the same passes on its expansion"""
    _, b = _pair(1, 1, 2)
    br = b.blocked_r1cs()
    b.free()
    ex = as_explicit(br.expand())
    rng = np.random.default_rng(5)
    z = np.ascontiguousarray(fr_arr([int(x) for x in rng.integers(0, 1 << 62, br.num_vars)]))
    lag = np.ascontiguousarray(fr_arr([int(x) for x in rng.integers(0, 1 << 62, br.num_constraints)]))
    for got, want in zip(host_spmv(hb, br, z), host_spmv(hb, ex, z)):
        assert (got == want).all()
    for got, want in zip(host_columns(hb, br, lag), host_columns(hb, ex, lag)):
        assert (got == want).all()
    for got, want in zip(host_density(hb, br), ex.density()):
        assert (got == want).all()
