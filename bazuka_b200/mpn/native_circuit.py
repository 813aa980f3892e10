"""ctypes front-end of the native (C++) update-circuit compiler, csrc/mpn_circuit.cu.

    nc = NativeUpdateCircuit(A, T, B)           # no GPU needed
    ni, na, mats = nc.r1cs()                     # the arrays of groth16.R1CS / bzk_r1cs_upload
    slot, epi = nc.program(0), nc.program(1)     # witness_program.WitnessProgram objects
    NativeUpdateCircuit(A, T, B, blocked=True).blocked_r1cs()
                                                 # groth16.BlockedR1CS: one slot stored, the others are its copies

The Python definition in this package (cs.py, gadgets.py, update.py) stays as the readable restatement and the
test oracle for it: tests compare every emitted array."""
import ctypes as ct
import os

import numpy as np

from . import native as N
from .cs import R
from .witness_program import WitnessProgram

_RINV = pow(1 << 256, -1, R)


def _canon(v):
    return np.frombuffer((v % R).to_bytes(32, "little"), dtype=np.uint64)


class NativeUpdateCircuit:
    """blocked=True: bzk_mpn_update_circuit_compile_blocked — slots 2.. are not stored (blocked_r1cs()); the shape and the
    witness programs are those of the explicit compile"""
    blocked = False

    def __init__(self, A, T, B, blocked=False):
        from .. import _lib
        self._l = _lib.load()
        self.A, self.T, self.B, self.blocked = A, T, B, blocked
        blob = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "data", "poseidon_params.bin"), "rb").read()
        jj = np.ascontiguousarray(np.stack([_canon(N.JJ_D), _canon(N.JJ_BASE_COFACTOR[0]), _canon(N.JJ_BASE_COFACTOR[1])]))
        h = ct.c_void_p()
        name = "bzk_mpn_update_circuit_compile_blocked" if blocked else "bzk_mpn_update_circuit_compile"
        st = getattr(self._l, name)(A, T, B, blob, len(blob), ct.c_void_p(jj.ctypes.data), ct.byref(h))
        if st != 0:
            raise _lib.BzkError(st, name)
        self._h = h
        shape = np.zeros(12, dtype=np.uint64)
        self._l.bzk_mpn_circuit_shape(h, ct.c_void_p(shape.ctypes.data))
        (self.num_inputs, self.num_aux, self.num_constraints, self.nnz_a, self.nnz_b, self.nnz_c, self.p_aux, self.slot_vars,
         self.state_out, self.final_fee, self.epilogue_vars, _) = (int(v) for v in shape)

    def free(self):
        if self._h:
            self._l.bzk_mpn_circuit_free(self._h)
            self._h = None

    def blocks(self):
        """bzk_mpn_circuit_blocks: (head_rows, tmpl_rows, reps, tail_rows, var_lo, var_stride), (stored nnz a, b, c)"""
        out = np.zeros(9, dtype=np.uint64)
        st = self._l.bzk_mpn_circuit_blocks(self._h, ct.c_void_p(out.ctypes.data))
        if st != 0:
            from .._lib import BzkError
            raise BzkError(st, "bzk_mpn_circuit_blocks")
        v = [int(x) for x in out]
        return tuple(v[:6]), tuple(v[6:])

    def _matrices(self, rows, nnzs):
        mats = []
        for side, nnz in enumerate(nnzs):
            rp = np.zeros(rows + 1, dtype=np.uint64)
            col = np.zeros(max(nnz, 1), dtype=np.uint32)
            val = np.zeros((max(nnz, 1), 4), dtype=np.uint64)
            self._l.bzk_mpn_circuit_matrix(self._h, side, ct.c_void_p(rp.ctypes.data), ct.c_void_p(col.ctypes.data), ct.c_void_p(val.ctypes.data))
            mats.append((rp, col[:nnz], val[:nnz]))
        return mats

    def r1cs(self):
        if self.blocked:
            e = self.blocked_r1cs().expand()
            return e.num_inputs, e.num_aux, e.mats
        return self.num_inputs, self.num_aux, self._matrices(self.num_constraints, (self.nnz_a, self.nnz_b, self.nnz_c))

    def blocked_r1cs(self):
        """groth16.BlockedR1CS of a blocked compile (of an explicit one it would hold every slot: use r1cs())"""
        from ..groth16 import BlockedR1CS
        assert self.blocked
        blocks, nnzs = self.blocks()
        head, tmpl, _, tail = blocks[:4]
        return BlockedR1CS(self.num_inputs, self.num_aux, *blocks, *self._matrices(head + tmpl + tail, nnzs))

    def program(self, which) -> WitnessProgram:
        sizes = np.zeros(6, dtype=np.uint64)
        self._l.bzk_mpn_circuit_program(self._h, which, ct.c_void_p(sizes.ctypes.data), None, None, None, None, None)
        n_ops, n_lc, n_terms, n_coefs, n_raw, n_ext = (int(v) for v in sizes)
        ops = np.zeros((n_ops, 6), dtype=np.int32)
        lc_ptr, lc_slot, lc_coef = np.zeros(n_lc + 1, dtype=np.int32), np.zeros(n_terms, dtype=np.int32), np.zeros(n_terms, dtype=np.int32)
        coefs = np.zeros((n_coefs, 4), dtype=np.uint64)
        p = lambda a: ct.c_void_p(a.ctypes.data)
        self._l.bzk_mpn_circuit_program(self._h, which, p(sizes), p(ops), p(lc_ptr), p(lc_slot), p(lc_coef), p(coefs))
        coef_ints = [int.from_bytes(row.tobytes(), "little") * _RINV % R for row in coefs]
        prog = WitnessProgram(self.A, self.T, ops, lc_ptr, lc_slot, lc_coef, coef_ints, n_raw, n_ext)
        if which == 0:
            prog.p_aux, prog.state_out, prog.final_fee = self.p_aux, self.state_out, self.final_fee
        return prog


class NativeTwoPhaseCircuit(NativeUpdateCircuit):
    """DepositCircuit / WithdrawCircuit compiled by libbzk (bzk_mpn_dw_circuit_compile): r1cs() as above,
    program(0) = phase 1, program(1) = phase 2, plus the placement data the witness glue needs
    (n1 / n2 = variables per slot of each phase, reveal_vars, row_local, ext_src, state_out)."""

    def __init__(self, kind, A, T, B):
        from .. import _lib
        self._l = _lib.load()
        self.kind, self.A, self.T, self.B = kind, A, T, B
        blob = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "data", "poseidon_params.bin"), "rb").read()
        jj = np.ascontiguousarray(np.stack([_canon(N.JJ_D), _canon(N.JJ_BASE_COFACTOR[0]), _canon(N.JJ_BASE_COFACTOR[1])]))
        h = ct.c_void_p()
        st = self._l.bzk_mpn_dw_circuit_compile({"deposit": 1, "withdraw": 2}[kind], A, T, B, blob, len(blob), ct.c_void_p(jj.ctypes.data), ct.byref(h))
        if st != 0:
            raise _lib.BzkError(st, "bzk_mpn_dw_circuit_compile")
        self._h = h
        shape = np.zeros(12, dtype=np.uint64)
        self._l.bzk_mpn_circuit_shape(h, ct.c_void_p(shape.ctypes.data))
        (self.num_inputs, self.num_aux, self.num_constraints, self.nnz_a, self.nnz_b, self.nnz_c, self.p_aux, self.n1,
         self.state_out, _, self.n2, self.reveal_vars) = (int(v) for v in shape)
        self.slot_vars, self.final_fee, self.epilogue_vars = self.n1, 0, self.n2
        counts = np.zeros(2, dtype=np.uint64)
        self._l.bzk_mpn_circuit_two_phase_info(h, ct.c_void_p(counts.ctypes.data), None, None)
        self.row_local, ext = np.zeros(int(counts[0]), dtype=np.int32), np.zeros(int(counts[1]), dtype=np.int32)
        self._l.bzk_mpn_circuit_two_phase_info(h, ct.c_void_p(counts.ctypes.data), ct.c_void_p(self.row_local.ctypes.data), ct.c_void_p(ext.ctypes.data))
        self.ext_src = [("state",) if e < 0 else ("raw1", int(e)) for e in ext]

    def program(self, which) -> WitnessProgram:
        prog = super().program(which)
        prog.p_aux = prog.state_out = prog.final_fee = 0
        return prog
