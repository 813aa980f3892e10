"""GPU tier: both witness kernels of csrc/witness.cu (`k_witness_levels`, a warp per slot level by level, and the serial
`k_witness_run`) on the generated programs of tests/witness_program_cases.py, against the big-integer `run_reference`,
for 1 to 1 025 slots of different inputs; and the upload's refusal of coefficient images it cannot run.  The CPU tier
(tests/test_witness_programs_cpu.py) checks the op semantics on the same cases; what is added here is the device's
memory layout, the lanes over a level and over the externals, and the slot index."""
import ctypes as ct
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import witness_program_cases as WC

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = WC.all_cases()
BY_NAME = {c.name: c for c in CASES}


def _canon(values):
    return np.frombuffer(b"".join((v % WC.R).to_bytes(32, "little") for v in values), dtype=np.uint64).reshape(-1, 4).copy()


def run_device(ctx, handle, prog, rows):
    """rows [(raws, ext)] -> the Montgomery images the kernel wrote, [ntx, n_ops, 4] uint64"""
    import torch
    from bazuka_b200.api import _dev_ptr, _host_ptr
    ntx = len(rows)
    raws = _canon([v for r, _ in rows for v in r]) if prog.n_raw else np.zeros((1, 4), dtype=np.uint64)
    ext = _canon([v for _, e in rows for v in e]) if prog.n_ext else np.zeros((1, 4), dtype=np.uint64)
    d_aux = torch.empty((ntx * prog.n_ops, 4), dtype=torch.int64, device=torch.device("cuda", ctx.device))
    ctx._check(ctx._l.bzk_witness_run_dev(ctx._h, handle, _host_ptr(raws), _host_ptr(ext), ntx, _dev_ptr(d_aux)))
    return d_aux.cpu().numpy().view(np.uint64).reshape(ntx, prog.n_ops, 4)


def reference(prog, rows):
    """run_reference of every slot, as Montgomery images [ntx, n_ops, 4]"""
    from bazuka_b200.mpn import witness_program as W
    from bazuka_b200.mpn.cs import to_mont
    return to_mont([v for raws, ext in rows for v in W.run_reference(prog, raws, ext)]).reshape(len(rows), prog.n_ops, 4)


def _assert_same(case, got, want):
    bad = np.argwhere((got != want).any(axis=2))
    assert len(bad) == 0, (case.name, len(bad), bad[:8].tolist(), [case.prog.ops[j].tolist() for _, j in bad[:4]])


# ntx for every case; the many-slot runs go to programs of about 200 ops so that the reference stays cheap
NTX_ALL = (1, 2)
NTX_SMALL = (31, 32, 33)
NTX_LARGE = {"shape_e70_r77": (257, 1025), "shape_e33_r1": (257, 1025), "opcodes": (257,), "jubjub": (257,)}


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_generated_program_on_device_equals_reference(ctx, case):
    """every slot's output of the level kernel equals the reference bit for bit, for every ntx the case is run at
    (small programs also at 31, 32 and 33 slots, a few at 257 and 1 025); the slots' inputs all differ."""
    from bazuka_b200.mpn.gpu_witness import upload_program
    prog = case.prog
    h = upload_program(ctx, prog)
    try:
        ntxs = NTX_ALL + (NTX_SMALL if prog.n_ops <= 700 else ()) + NTX_LARGE.get(case.name, ())
        for ntx in ntxs:
            rows = WC.rows(case, ntx, seed=case.seed * 31 + ntx)
            _assert_same(case, run_device(ctx, h, prog, rows), reference(prog, rows))
    finally:
        ctx._l.bzk_witness_program_free(ctx._h, h)


SERIAL_CASES = ["chain_2000", "wide_levels", "mixed_levels", "opcodes", "jubjub", "linear_combinations", "shape_e70_r77", "single_op_no_inputs"]
SERIAL_NTX = 3

_SERIAL_SCRIPT = r"""
import hashlib, sys
sys.path[:0] = [{root!r}, {tests!r}]
import bazuka_b200 as B
import witness_program_cases as WC
from bazuka_b200.mpn.gpu_witness import upload_program
from test_gpu_witness_programs import run_device, SERIAL_CASES, SERIAL_NTX
ctx = B.Context(0)
by = {{c.name: c for c in WC.all_cases()}}
for name in SERIAL_CASES:
    c = by[name]
    h = upload_program(ctx, c.prog)
    out = run_device(ctx, h, c.prog, WC.rows(c, SERIAL_NTX))
    ctx._l.bzk_witness_program_free(ctx._h, h)
    print(name, hashlib.sha256(out.tobytes()).hexdigest())
ctx.close()
"""


def test_serial_kernel_equals_level_kernel_and_reference(ctx):
    """BZK_WITNESS_SERIAL=1 (read once per process) selects k_witness_run, one thread per slot in program order: a child
    process runs the level-shape cases and a few others through it and prints digests of the outputs, which equal the
    level kernel's here and the reference's."""
    from bazuka_b200.mpn.gpu_witness import upload_program
    script = _SERIAL_SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    env = dict(os.environ, BZK_WITNESS_SERIAL="1")
    child = subprocess.run([sys.executable, "-c", script], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert child.returncode == 0, child.stderr[-3000:]
    serial = dict(line.split() for line in child.stdout.splitlines() if line.strip())
    assert sorted(serial) == sorted(SERIAL_CASES)
    for name in SERIAL_CASES:
        c = BY_NAME[name]
        rows = WC.rows(c, SERIAL_NTX)
        h = upload_program(ctx, c.prog)
        try:
            levels = run_device(ctx, h, c.prog, rows)
        finally:
            ctx._l.bzk_witness_program_free(ctx._h, h)
        want = reference(c.prog, rows)
        _assert_same(c, levels, want)
        assert serial[name] == hashlib.sha256(want.tobytes()).hexdigest(), name


def test_upload_refuses_coefficient_images_it_cannot_run(ctx):
    """the kernels take coefficient 0 as one without reading coefs[0] and assume reduced operands, so the upload refuses
    coefs[0] != Montgomery one (2, or the canonical 1), a coefficient image >= r, and a curve d image >= r; the same
    program with well-formed images uploads."""
    from bazuka_b200.api import _host_ptr
    from bazuka_b200.mpn import native as N
    from bazuka_b200.mpn.cs import to_mont
    R = WC.R
    ops = np.array([[0, 0, 0, 0, 0, 0], [1, 0, 1, 0, 0, 0]], dtype=np.int32)   # RAW; MUL(ONE, 5 * raw)
    lc_ptr = np.array([0, 1, 2], dtype=np.int32)
    lc_slot = np.array([0, 1], dtype=np.int32)
    lc_coef = np.array([0, 1], dtype=np.int32)
    img = lambda v: np.frombuffer(v.to_bytes(32, "little"), dtype=np.uint64).reshape(1, 4)

    def upload(coefs, jj_d):
        coefs = np.ascontiguousarray(coefs, dtype=np.uint64)
        jj_d = np.ascontiguousarray(jj_d, dtype=np.uint64)
        h = ct.c_void_p()
        st = ctx._l.bzk_witness_program_upload(ctx._h, _host_ptr(ops), len(ops), _host_ptr(lc_ptr), 2, _host_ptr(lc_slot), _host_ptr(lc_coef), 2,
                                               _host_ptr(coefs), len(coefs), 1, 0, _host_ptr(jj_d), ct.byref(h))
        if st == 0:
            ctx._l.bzk_witness_program_free(ctx._h, h)
        return st

    good_d = to_mont([N.JJ_D])
    assert upload(to_mont([1, 5]), good_d) == 0
    assert upload(to_mont([1, R - 1]), good_d) == 0
    assert upload(to_mont([2, 5]), good_d) == -1                                # coefs[0] = 2
    assert upload(np.concatenate([img(1), to_mont([5])]), good_d) == -1         # coefs[0] canonical 1, not its Montgomery image
    assert upload(np.concatenate([to_mont([1]), img(R)]), good_d) == -1         # an image equal to r
    assert upload(np.concatenate([to_mont([1]), img((1 << 256) - 1)]), good_d) == -1
    assert upload(np.concatenate([to_mont([1, 5]), img(R + 7)]), good_d) == -1  # an unused coefficient is checked too
    assert upload(to_mont([1, 5]), img(R)) == -1                                # jj_d = r
    assert upload(to_mont([1, 5]), img(R + N.JJ_D)) == -1
