"""CPU tier: the witness interpreter's op semantics (csrc/witness_core.cuh, compiled for the host) on generated programs
(tests/witness_program_cases.py) against the big-integer `run_reference`, in program order and in the order of the
kernel's level schedule.  tests/test_gpu_witness_programs.py runs the same cases through both device kernels."""
import ctypes as ct

import numpy as np
import pytest

import witness_program_cases as WC
from bazuka_b200.mpn import witness_program as W
from bazuka_b200.mpn.cs import to_mont
from bazuka_b200.mpn import native as N

CASES = WC.all_cases()


def _canon(values):
    return np.frombuffer(b"".join((v % WC.R).to_bytes(32, "little") for v in values), dtype=np.uint64).reshape(-1, 4).copy() \
        if values else np.zeros((1, 4), dtype=np.uint64)


def _ptr(a):
    return a.ctypes.data_as(ct.c_void_p)


def run_host(shim, prog, raws, ext, levels=False):
    """one slot through shim_witness_run (program order) or shim_witness_run_levels (schedule order, a level backwards)
    -> (Montgomery images [n_ops, 4], level count or None, stats)"""
    ops = np.ascontiguousarray(prog.ops, dtype=np.int32)
    coefs, jj_d = np.ascontiguousarray(prog.coefs_mont()), to_mont([N.JJ_D])
    lc_ptr, lc_slot, lc_coef = (np.ascontiguousarray(a, dtype=np.int32) for a in (prog.lc_ptr, prog.lc_slot, prog.lc_coef))
    if len(lc_slot) == 0:
        lc_slot = lc_coef = np.zeros(1, dtype=np.int32)
    r, e = _canon(raws), _canon(ext)
    out = np.zeros((prog.n_ops, 4), dtype=np.uint64)
    args = [_ptr(ops), ct.c_uint32(prog.n_ops), _ptr(lc_ptr), _ptr(lc_slot), _ptr(lc_coef), _ptr(coefs), ct.c_uint32(prog.n_raw),
            ct.c_uint32(prog.n_ext), _ptr(jj_d), _ptr(r), _ptr(e), _ptr(out)]
    if not levels:
        shim.shim_witness_run(*args)
        return out, None, None
    stats = np.zeros(4, dtype=np.uint64)
    shim.shim_witness_run_levels.restype = ct.c_uint32
    n_levels = shim.shim_witness_run_levels(*args, _ptr(stats))
    return out, n_levels, stats


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_generated_program_on_host_interpreter_equals_reference(hostshim, case):
    """every generated case, a few slots of different inputs: both host orders of the device interpreter's code give
    the reference's witness exactly, and the schedule has the levels the case was built for."""
    prog = case.prog
    widths = WC.levels(prog)
    if case.level_widths is not None:
        assert widths == case.level_widths
    n = 2 if prog.n_ops > 1000 else 4
    for raws, ext in WC.rows(case, n):
        want = to_mont(W.run_reference(prog, raws, ext))
        got, _, _ = run_host(hostshim, prog, raws, ext)
        bad = np.nonzero((got != want).any(axis=1))[0]
        assert len(bad) == 0, (case.name, bad[:8], [prog.ops[j].tolist() for j in bad[:4]])
        got, n_levels, stats = run_host(hostshim, prog, raws, ext, levels=True)
        bad = np.nonzero((got != want).any(axis=1))[0]
        assert len(bad) == 0, (case.name, "levels", bad[:8], [prog.ops[j].tolist() for j in bad[:4]])
        assert n_levels == len(widths) and int(stats[0]) == sum(widths) and int(stats[1]) == max(widths)


def test_generated_cases_cover_what_they_claim():
    """the generator reaches the shapes and values it is there for (a guard against a silently narrowed generator)."""
    by = {c.name: c for c in CASES}
    assert {(c.prog.n_ext, c.prog.n_raw) for c in CASES} >= {(e, r) for e, r in WC.SHAPES}
    assert [c.prog.n_ops for c in CASES if c.name.startswith("single")] == [1, 1, 1]
    assert by["single_raw"].prog.ops[0, 0] == W.OP_RAW
    assert all(c.prog.coefs[0] == 1 for c in CASES)
    codes = set(np.concatenate([c.prog.ops[:, 0] for c in CASES]).tolist())
    assert codes == set(range(8))
    bits = set(by["opcodes"].prog.ops[by["opcodes"].prog.ops[:, 0] == W.OP_BIT, 5].tolist())
    assert bits >= set(WC.BIT_IMMS)
    sizes = set(np.diff(by["linear_combinations"].prog.lc_ptr).tolist())
    assert sizes >= {0, 1, 9, 64, 300}
    # MUL with one LC for both operands (the square path)
    assert any(((c.prog.ops[:, 0] == W.OP_MUL) & (c.prog.ops[:, 1] == c.prog.ops[:, 2])).any() for c in CASES)
    # the JJ case: every kind of sum shows up in the reference's outputs over a few slots
    jc = by["jubjub"]
    jj = np.nonzero(jc.prog.ops[:, 0] == W.OP_JJ)[0]
    outs = set()
    for raws, ext in WC.rows(jc, 16):
        v = W.run_reference(jc.prog, raws, ext)
        outs |= {(v[j], v[j + 1]) for j in jj}
    assert {(0, 0), (0, 1), (0, WC.R - 1), WC.POINTS["2P"]} <= outs
    assert any(p[1] == 0 for p in outs)                 # an order-4 point as a result
    assert sum(1 for p in outs if p != (0, 0) and N.jj_on_curve(p)) > 20
