"""CPU tier: the C-ABI library loads, exports every symbol include/bzk.h declares, refuses to run
without a GPU (no CPU fallback), and the host-compiled field/group code agrees with the oracle."""
import ctypes as ct
import os
import re

import numpy as np
import pytest

from oracle.py import curve as C, field as Fd
from conftest import ROOT


def _header_symbols():
    h = open(os.path.join(ROOT, "include", "bzk.h")).read()
    h = re.sub(r"/\*.*?\*/", "", h, flags=re.S)
    return sorted(set(re.findall(r"\b(bzk_[a-z0-9_]+)\s*\(", h)))


def test_library_exports_every_declared_symbol():
    import bazuka_b200 as B
    from bazuka_b200 import _lib
    lib = B.load()
    syms = _header_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(lib, s), f"libbzk.so does not export {s}"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature"
    assert sorted(_lib.SIGNATURES) == syms
    assert lib.bzk_abi_version() >> 16 == 1


def test_struct_sizes_match_reference_images():
    h = open(os.path.join(ROOT, "include", "bzk.h")).read()
    assert "uint64_t l[4]" in h and "uint64_t x[6]" in h and "uint64_t x[12]" in h
    assert len(C.g1_to_bytes(C.G1_GEN)) == 104 and len(C.g2_to_bytes(C.G2_GEN)) == 200


def test_packed_transaction_structs_match_the_header(tmp_path):
    """the numpy record layouts mpn/ledger.py packs (bzk_mpn_tx, bzk_mpn_deposit, bzk_mpn_withdraw) against the C compiler's view
    of include/bzk.h: total size and every field offset."""
    import subprocess
    from bazuka_b200.mpn import ledger as L, works as Wk
    fields = {"bzk_mpn_work_info": (Wk.work_info_dtype(), ["kind", "log4_tree", "log4_token", "log4_batch", "n_transitions", "height", "state", "aux_data",
                                                           "next_state", "new_root_hash", "new_root_size", "reward"]),
              "bzk_mpn_tx": (L._TX, ["nonce", "amount", "fee", "src_pk_odd", "dst_pk_odd", "src_pk_x", "dst_pk_x", "amount_token_id",
                                     "fee_token_id", "sig_rx", "sig_ry", "sig_s"]),
              "bzk_mpn_deposit": (L._DEP, ["pk_x", "pk_odd", "token_id", "amount", "src_id"]),
              "bzk_mpn_withdraw": (L._WD, ["pk_x", "pk_odd", "check_calldata", "nonce", "sig_rx", "sig_ry", "sig_s", "amount_token_id",
                                           "fee_token_id", "fingerprint", "amount", "fee", "calldata"])}
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "bzk.h"', 'int main(void) {']
    for name, (_, fs) in fields.items():
        src.append(f'printf("{name} %zu", sizeof({name}));')
        src += [f'printf(" %zu", offsetof({name}, {f}));' for f in fs]
        src.append('printf("\\n");')
    src += ["return 0;", "}"]
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    for line in subprocess.check_output([str(exe)], text=True).splitlines():
        name, size, *offs = line.split()
        dt, fs = fields[name]
        assert dt.itemsize == int(size), name
        assert [dt.fields[f][1] for f in fs] == [int(o) for o in offs], name


def test_plan_hooks_are_typed_and_refuse_bad_arguments():
    """bzk_ctx_set_msm_table_window / bzk_ctx_last_msm_plan: typed as the header declares them, and a missing context or
    output buffer is refused before anything is touched (the window range is checked on a real context in the gpu tier)."""
    from bazuka_b200 import _lib
    lib = _lib.load()
    h = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bzk.h")).read(), flags=re.S)
    assert "int32_t bzk_ctx_set_msm_table_window(bzk_ctx *ctx, uint32_t c);" in h
    assert "int32_t bzk_ctx_last_msm_plan(const bzk_ctx *ctx, uint32_t out[8]);" in h
    assert _lib.SIGNATURES["bzk_ctx_set_msm_table_window"] == (ct.c_int32, [ct.c_void_p, ct.c_uint32])
    assert _lib.SIGNATURES["bzk_ctx_last_msm_plan"] == (ct.c_int32, [ct.c_void_p, ct.c_void_p])
    out = np.full(8, 7, dtype=np.uint32)
    assert lib.bzk_ctx_last_msm_plan(None, out.ctypes.data_as(ct.c_void_p)) == -1
    assert (out == 7).all()
    for c in (0, 1, 7, 8, 23, 24, 0xFFFFFFFF):
        assert lib.bzk_ctx_set_msm_table_window(None, c) == -1
    assert lib.bzk_abi_version() == (1 << 16) | 1


def test_no_cpu_fallback_without_gpu():
    import torch
    import bazuka_b200 as B
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(B.BzkError) as e:
        B.Context(0)
    assert e.value.status == -6


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "bazuka_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "import oracle" not in txt and "from oracle" not in txt and "bzko_" not in txt, f


def test_host_build_of_device_multiplier(hostshim, cref):
    """the even/odd IMAD.WIDE carry-chain algorithm, compiled with explicit carries, on the CPU."""
    import random
    n = 4000
    a, b = cref.fr_random(21, n), cref.fr_random(22, n)
    r = np.empty_like(a)
    for op, f in ((0, cref.fr_add), (1, cref.fr_sub), (2, cref.fr_mul), (3, cref.fr_mul), (4, cref.fr_add), (5, cref.fr_sub)):
        hostshim.shim_fr(a.ctypes.data_as(ct.c_void_p), b.ctypes.data_as(ct.c_void_p), r.ctypes.data_as(ct.c_void_p), ct.c_size_t(n), op)
        assert (r == f(a, b)).all(), op
    hostshim.shim_fr_inv(a.ctypes.data_as(ct.c_void_p), r.ctypes.data_as(ct.c_void_p), ct.c_size_t(50))
    assert (r[:50] == cref.fr_inv(a[:50])).all()
    # the Euclidean inverse the witness interpreter uses == the Fermat power, edge values included (0 -> 0)
    edge = np.frombuffer(b"".join((v % Fd.R_MOD).to_bytes(32, "little") for v in (0, 1, 2, Fd.R_MOD - 1, Fd.R_MOD - 2, 1 << 254, (1 << 200) + 1)),
                         dtype=np.uint64).reshape(-1, 4)
    ae = np.concatenate([a[:400], edge])
    r1, r2 = np.empty_like(ae), np.empty_like(ae)
    hostshim.shim_fr_inv(ae.ctypes.data_as(ct.c_void_p), r1.ctypes.data_as(ct.c_void_p), ct.c_size_t(len(ae)))
    hostshim.shim_fr_inv_gcd(ae.ctypes.data_as(ct.c_void_p), r2.ctypes.data_as(ct.c_void_p), ct.c_size_t(len(ae)))
    assert (r1 == r2).all() and not r2[400].any()
    rnd = random.Random(1)
    vals = [rnd.randrange(Fd.P_MOD) for _ in range(n - 6)] + [0, 1, 2, Fd.P_MOD - 1, Fd.P_MOD - 2, (1 << 380)]
    x = np.frombuffer(b"".join(v.to_bytes(48, "little") for v in vals), dtype=np.uint64).reshape(-1, 6).copy()
    y = x[::-1].copy()
    r = np.empty_like(x)
    for op, f in ((0, cref.fp_add), (1, cref.fp_sub), (2, cref.fp_mul), (3, cref.fp_mul), (4, cref.fp_add), (5, cref.fp_sub)):
        hostshim.shim_fp(x.ctypes.data_as(ct.c_void_p), y.ctypes.data_as(ct.c_void_p), r.ctypes.data_as(ct.c_void_p), ct.c_size_t(n), op)
        assert (r == f(x, y)).all(), op
    hostshim.shim_fp_inv(x.ctypes.data_as(ct.c_void_p), r.ctypes.data_as(ct.c_void_p), ct.c_size_t(50))
    assert (r[:50] == cref.fp_inv(x[:50])).all()
    xe = np.concatenate([x[:200], x[-6:]])
    r1, r2 = np.empty_like(xe), np.empty_like(xe)
    hostshim.shim_fp_inv(xe.ctypes.data_as(ct.c_void_p), r1.ctypes.data_as(ct.c_void_p), ct.c_size_t(len(xe)))
    hostshim.shim_fp_inv_gcd(xe.ctypes.data_as(ct.c_void_p), r2.ctypes.data_as(ct.c_void_p), ct.c_size_t(len(xe)))
    assert (r1 == r2).all()


def test_host_build_of_lazy_inner_product(hostshim, cref):
    """Poseidon's MDS row product with a single Montgomery reduction (mul_wide/redc_wide), worst-case
    operands included (all r-1)."""
    R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
    from conftest import fr_arr
    for t in (1, 2, 5, 8, 17):
        m, s = cref.fr_random(40 + t, t), cref.fr_random(50 + t, t)
        if t >= 5:
            m[:] = fr_arr([R - 1] * t)
            s[:] = fr_arr([R - 1] * t)
        out = np.zeros(4, dtype=np.uint64)
        hostshim.shim_fr_dot(m.ctypes.data_as(ct.c_void_p), s.ctypes.data_as(ct.c_void_p), ct.c_size_t(t), out.ctypes.data_as(ct.c_void_p))
        want = np.zeros((1, 4), dtype=np.uint64)
        prods = cref.fr_mul(m, s)
        for k in range(t):
            want = cref.fr_add(want, prods[k:k + 1])
        assert (out == want[0]).all(), t


def test_host_build_of_group_law(hostshim, cref):
    """XYZZ madd / add / dbl / to_affine (the device group law) against the Jacobian oracle."""
    g1 = cref.g1_generator()
    k = cref.fr_from_mont(cref.fr_random(5, 2))
    out = np.zeros(96, dtype=np.uint8)
    hostshim.shim_g1_mul(g1[:96].ctypes.data_as(ct.c_void_p), k[0].ctypes.data_as(ct.c_void_p), out.ctypes.data_as(ct.c_void_p))
    want = cref.g1_mul(g1, cref.fr_to_mont(k[:1]))
    assert (out == want[:96]).all()
    g2 = cref.g2_generator()
    out2 = np.zeros(192, dtype=np.uint8)
    hostshim.shim_g2_mul(g2[:192].ctypes.data_as(ct.c_void_p), k[1].ctypes.data_as(ct.c_void_p), out2.ctypes.data_as(ct.c_void_p))
    assert (out2 == cref.g2_mul(g2, cref.fr_to_mont(k[1:2]))[:192]).all()
    # madd / add, including P+P (doubling branch) and P + (-P) (identity -> x=y=0 packed)
    bs = cref.g1_random_bases(3, 2)
    o1, o2 = np.zeros(96, dtype=np.uint8), np.zeros(96, dtype=np.uint8)
    for pa, pb in ((bs[0], bs[1]), (bs[0], bs[0])):
        hostshim.shim_g1_add(pa[:96].ctypes.data_as(ct.c_void_p), pb[:96].ctypes.data_as(ct.c_void_p),
                             o1.ctypes.data_as(ct.c_void_p), o2.ctypes.data_as(ct.c_void_p))
        want = cref.g1_add(pa, pb)[:96]
        assert (o1 == want).all() and (o2 == want).all()
    negp = bs[0].copy()
    y = Fd.fp_from_mont_bytes(bs[0][48:96].tobytes())
    negp[48:96] = np.frombuffer(Fd.fp_to_mont_bytes(Fd.P_MOD - y), dtype=np.uint8)
    hostshim.shim_g1_add(bs[0][:96].ctypes.data_as(ct.c_void_p), negp[:96].ctypes.data_as(ct.c_void_p),
                         o1.ctypes.data_as(ct.c_void_p), o2.ctypes.data_as(ct.c_void_p))
    assert not o1.any() and not o2.any()


def test_host_build_of_witness_interpreter(hostshim):
    """the device interpreter's per-slot loop (csrc/witness_core.cuh) compiled for the host runs the real update-slot
    program on signed transfers and a null slot and reproduces `UpdateCircuit.synthesize`'s aux values — the same
    C++ the kernel executes, checked without a GPU."""
    import ctypes as ct
    from bazuka_b200.mpn import cs as C, native as N, update as U, witness_program as W
    from test_mpn_cpu import make_state, transfer
    st, keys = make_state(3, 3, 3)
    keys.append(N.eddsa_keys(b"newcomer"))
    txs = [transfer(keys, 0, 1, 1), transfer(keys, 0, 3, 2, amount=77, fee=3)]
    pub, trans, _ = U.update(st, txs, 1)
    circ = U.UpdateCircuit(3, 3, 1, commitment=42, height=7, transitions=trans, **pub)
    cs = circ.synthesize(C.ConstraintSystem())
    prog = W.compile_update_block(3, 3)
    roots = W.slot_roots(circ)
    ops = np.ascontiguousarray(prog.ops, dtype=np.int32)
    coefs, jj_d = np.ascontiguousarray(prog.coefs_mont()), C.to_mont([N.JJ_D])
    canon = lambda vals: np.frombuffer(b"".join((v % N.R).to_bytes(32, "little") for v in vals), dtype=np.uint64).copy()
    p = lambda a: a.ctypes.data_as(ct.c_void_p)
    for k in (0, 1, 3):  # two real slots and a null one
        raws, ext = canon(W.raw_values(circ.transitions[k], 3, 3)), canon([circ.fee_token, roots[k]])
        out = np.zeros((prog.n_ops, 4), dtype=np.uint64)
        hostshim.shim_witness_run(p(ops), ct.c_uint32(prog.n_ops), p(prog.lc_ptr), p(prog.lc_slot), p(prog.lc_coef), p(coefs),
                                  ct.c_uint32(prog.n_raw), ct.c_uint32(prog.n_ext), p(jj_d), p(raws), p(ext), p(out))
        want = C.to_mont(cs.aux[prog.p_aux + k * prog.n_ops: prog.p_aux + (k + 1) * prog.n_ops])
        assert (out == want).all(), (k, np.nonzero((out != want).any(axis=1))[0][:5])
        # the order the GPU kernel uses: the upload-time level schedule (wit_build_schedule), a level's ops in any order,
        # variables read from the slot's own output segment
        out2 = np.zeros((prog.n_ops, 4), dtype=np.uint64)
        stats = np.zeros(4, dtype=np.uint64)
        hostshim.shim_witness_run_levels.restype = ct.c_uint32
        n_levels = hostshim.shim_witness_run_levels(p(ops), ct.c_uint32(prog.n_ops), p(prog.lc_ptr), p(prog.lc_slot), p(prog.lc_coef), p(coefs),
                                                    ct.c_uint32(prog.n_raw), ct.c_uint32(prog.n_ext), p(jj_d), p(raws), p(ext), p(out2), p(stats))
        assert (out2 == want).all(), (k, np.nonzero((out2 != want).any(axis=1))[0][:5])
        n_nop = int((ops[:, 0] == 7).sum())
        assert int(stats[0]) == prog.n_ops - n_nop and 1000 < n_levels < prog.n_ops // 8 and int(stats[2]) <= 2 * n_nop


@pytest.mark.parametrize("kind", ["deposit", "withdraw"])
def test_native_programs_through_native_interpreter_on_host(hostshim, kind):
    """all-native on the CPU tier: the deposit / withdraw programs emitted by the C++ circuit compiler (phase 1, reveal,
    phase 2), run by the C++ interpreter core (host build of witness_core.cuh), assemble to `synthesize`'s aux vector."""
    import ctypes as ct
    from bazuka_b200.mpn import cs as C, dw_witness as DW, native as N
    from bazuka_b200.mpn.native_circuit import NativeTwoPhaseCircuit
    from test_mpn_cpu import _dw_scenario
    circ = _dw_scenario(kind)
    cs = circ.synthesize(C.ConstraintSystem())
    nc = NativeTwoPhaseCircuit(kind, 3, 3, 1)
    p1, p2, rv = nc.program(0), nc.program(1), nc.program(2)
    raws_of = DW.KINDS[kind][2]
    roots = DW.slot_roots(circ)
    jj_d = C.to_mont([N.JJ_D])
    canon = lambda vals: np.frombuffer(b"".join((v % N.R).to_bytes(32, "little") for v in vals), dtype=np.uint64).copy() if vals else np.zeros(4, np.uint64)
    ptr = lambda a: a.ctypes.data_as(ct.c_void_p)
    rinv = pow(1 << 256, -1, N.R)

    def run(prog, raws, ext):
        ops, coefs = np.ascontiguousarray(prog.ops, dtype=np.int32), np.ascontiguousarray(prog.coefs_mont())
        r, e, out = canon(raws), canon(ext), np.zeros((prog.n_ops, 4), dtype=np.uint64)
        hostshim.shim_witness_run(ptr(ops), ct.c_uint32(prog.n_ops), ptr(prog.lc_ptr), ptr(prog.lc_slot), ptr(prog.lc_coef), ptr(coefs),
                                  ct.c_uint32(prog.n_raw), ct.c_uint32(prog.n_ext), ptr(jj_d), ptr(r), ptr(e), ptr(out))
        return [int.from_bytes(row.tobytes(), "little") * rinv % N.R for row in out]

    b1, b2, rows = [], [], []
    for k, tr in enumerate(circ.transitions):
        r1, r2 = raws_of(tr, 3, 3)
        out1 = run(p1, r1, [])
        b1 += out1
        rows += [out1[j] for j in nc.row_local]
        ext2 = [roots[k] if s[0] == "state" else r1[s[1]] for s in nc.ext_src]
        b2 += run(p2, r2, ext2)
    assert cs.aux[:nc.p_aux] + b1 + run(rv, [], rows) + b2 == cs.aux
    nc.free()


def test_native_circuit_and_native_interpreter_satisfy_each_other(hostshim):
    """end to end on the CPU tier without the Python circuit definition: the R1CS emitted by the C++ compiler is
    satisfied (a*b == c on every constraint, incl. the Input*0 = 0 convention being absent here) by the witness that
    the C++ interpreter computes from the C++-emitted slot and epilogue programs for a real signed batch."""
    import ctypes as ct
    from bazuka_b200.mpn import native as N, update as U, witness_program as W
    from bazuka_b200.mpn.cs import to_mont
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    from test_mpn_cpu import make_state, transfer
    st, keys = make_state(3, 3, 3)
    txs = [transfer(keys, 0, 1, 1), transfer(keys, 1, 2, 1, amount=5, fee=7), transfer(keys, 2, 0, 1, amount=1)]
    pub, trans, _ = U.update(st, txs, 1)
    circ = U.UpdateCircuit(3, 3, 1, commitment=9, height=4, transitions=trans, **pub)   # only a container of values here
    nc = NativeUpdateCircuit(3, 3, 1)
    ni, na, mats = nc.r1cs()
    slot, epi = nc.program(0), nc.program(1)
    jj_d = to_mont([N.JJ_D])
    canon = lambda vals: np.frombuffer(b"".join((v % N.R).to_bytes(32, "little") for v in vals), dtype=np.uint64).copy() if vals else np.zeros(4, np.uint64)
    ptr = lambda a: a.ctypes.data_as(ct.c_void_p)
    rinv = pow(1 << 256, -1, N.R)

    def run(prog, raws, ext):
        ops, coefs = np.ascontiguousarray(prog.ops, dtype=np.int32), np.ascontiguousarray(prog.coefs_mont())
        r, e, out = canon(raws), canon(ext), np.zeros((prog.n_ops, 4), dtype=np.uint64)
        hostshim.shim_witness_run(ptr(ops), ct.c_uint32(prog.n_ops), ptr(prog.lc_ptr), ptr(prog.lc_slot), ptr(prog.lc_coef), ptr(coefs),
                                  ct.c_uint32(prog.n_raw), ct.c_uint32(prog.n_ext), ptr(jj_d), ptr(r), ptr(e), ptr(out))
        return [int.from_bytes(row.tobytes(), "little") * rinv % N.R for row in out]

    roots = W.slot_roots(circ)
    aux = [circ.commitment, circ.height, circ.state, circ.fee_token, circ.aux_data, circ.next_state]
    fees = []
    for k, tr in enumerate(circ.transitions):
        block = run(slot, W.raw_values(tr, 3, 3), [circ.fee_token, roots[k]])
        fees.append(block[nc.final_fee])
        aux += block
    aux += run(epi, [], [circ.fee_token] + fees)
    z = [1, circ.commitment, circ.height, circ.state, circ.aux_data, circ.next_state] + aux
    assert len(z) == ni + na
    ev = []
    for rp, col, val in mats:
        coef = [int.from_bytes(row.tobytes(), "little") * rinv % N.R for row in val]
        rp = rp.tolist(); col = col.tolist()
        ev.append([sum(coef[i] * z[col[i]] for i in range(rp[j], rp[j + 1])) % N.R for j in range(nc.num_constraints)])
    bad = [j for j in range(nc.num_constraints) if ev[0][j] * ev[1][j] % N.R != ev[2][j]]
    assert not bad, bad[:5]
    # and a wrong claimed next_state breaks exactly the final equality constraint
    z[5] = (z[5] + 1) % N.R
    z[ni + 5] = z[5]
    j = nc.num_constraints - 1
    rp, col, val = mats[0]
    lhs = sum(int.from_bytes(val[i].tobytes(), "little") * rinv % N.R * z[int(col[i])] for i in range(int(rp[j]), int(rp[j + 1]))) % N.R
    rp, col, val = mats[2]
    rhs = sum(int.from_bytes(val[i].tobytes(), "little") * rinv % N.R * z[int(col[i])] for i in range(int(rp[j]), int(rp[j + 1]))) % N.R
    assert lhs != rhs
    nc.free()


def test_host_poseidon_is_the_reference_hash(cref):
    """bzk_poseidon_host_hash (the `ZkHasher` single-hash path, no GPU): the reference's 16 known answers
    (/root/reference/src/zk/poseidon/mod.rs:116-133) and the C oracle on random inputs for every arity."""
    import json, os, time
    from bazuka_b200.api import HostPoseidon
    from conftest import fr_arr, fr_ints
    h = HostPoseidon()
    kats = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "poseidon_kats.json")))["expected_decimal"]
    for n, want in enumerate(kats, 1):
        assert fr_ints(h.hash(fr_arr(list(range(n)))))[0] == int(want), n
    for arity in range(1, 17):
        inp = cref.fr_random(500 + arity, 40 * arity).reshape(40, arity, 4)
        assert (h.hash(inp) == cref.poseidon(inp)).all(), arity
    t0 = time.perf_counter()
    one = cref.fr_random(9, 4)
    for _ in range(200):
        h.hash(one)
    print(f"host Poseidon-4: {(time.perf_counter() - t0) / 200 * 1e6:.0f} us per hash (incl. ctypes)")
    h.free()


def test_host_eddsa_verify_is_the_reference_check():
    """bzk_jubjub_eddsa_verify (host JubJub arithmetic + host Poseidon of libbzk) == the Python restatement of `JubJub::verify`
    (/root/reference/src/crypto/jubjub/mod.rs:151-167) on valid signatures and on every kind of tampering the builders meet."""
    from bazuka_b200.api import HostPoseidon
    from bazuka_b200.mpn import native as N
    hp = HostPoseidon()
    for seed in (b"a", b"b", b"c"):
        pk, sk = N.eddsa_keys(b"key-" + seed)
        other, _ = N.eddsa_keys(b"other-" + seed)
        msg = N.poseidon([int.from_bytes(seed, "big"), 7])
        sig = N.eddsa_sign(sk, msg)
        cases = [(pk, msg, sig["r"], sig["s"]), (pk, msg + 1, sig["r"], sig["s"]), (pk, msg, sig["r"], sig["s"] + 1), (other, msg, sig["r"], sig["s"]),
                 (pk, msg, (sig["r"][0], sig["r"][1] + 1), sig["s"]), ((pk[0] + 1, pk[1]), msg, sig["r"], sig["s"]), (pk, msg, sig["r"], 0),
                 (pk, msg, (0, 1), sig["s"]), (pk, msg, sig["r"], Fd.R_MOD + sig["s"])]
        got = [hp.eddsa_verify(N.JJ_D, *c) for c in cases]
        want = [N.eddsa_verify(c[0], c[1], {"r": c[2], "s": c[3]}) if all(0 <= v < Fd.R_MOD for v in (*c[0], c[1], *c[2], c[3])) else False for c in cases]
        assert got == want and got[0] and not any(got[1:])
    hp.free()
