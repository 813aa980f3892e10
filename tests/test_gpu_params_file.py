"""GPU tier: proving keys through bellman's `Parameters` file format (bzk_groth16_params_read / _write, csrc/params_io.cu)
against the oracle codec (oracle/py/bellman_params.py): oracle-written keys prove byte-equal to the oracle prover, a 2^18
key's image equals the oracle encoder's over the whole file and survives read -> write, every defect kind in every vector is
refused with bellman's status and the exact first bad point, a production verifying key is accepted, and a key written by
an MPN worker proves the worker's block after the round trip."""
import ctypes as ct

import numpy as np
import pytest

from conftest import fr_arr
from oracle.py import bellman_params as BP, curve as C
from test_params_file_cpu import golden_vks, lifts, vk_from_bincode

pytestmark = pytest.mark.gpu
VK_FIELDS = BP.VK_ORDER


def _vk_equal(a, b):
    for k in VK_FIELDS:
        assert (np.asarray(a[k], np.uint8) == np.asarray(b[k], np.uint8)).all(), k
    assert (np.asarray(a["ic"], np.uint8).reshape(-1, 104) == np.asarray(b["ic"], np.uint8).reshape(-1, 104)).all(), "ic"


def test_oracle_written_keys_prove_like_the_oracle(ctx, cref):
    """tiny and synthetic circuits: GC.setup images -> bellman bytes (oracle) -> read_parameters(checked) -> same vk, and the
    proof for fixed (r, s) is byte-equal to GC.prove's"""
    from bazuka_b200 import groth16 as BG, synth
    from oracle import groth16_c as GC
    from test_groth16_cpu import tiny_circuit, to_csr
    cs, z = tiny_circuit()
    zz = fr_arr(z)
    cases = [(cs.num_inputs, cs.num_aux, to_csr(cs), zz[:cs.num_inputs], zz[cs.num_inputs:])]
    ni, na, mats, inputs, aux = synth.build(4, 6, seed=3, ops=GC.CpuOps)
    cases.append((ni, na, mats, inputs, aux))
    for k, (ni, na, mats, inputs, aux) in enumerate(cases):
        cpk = GC.setup(ni, na, mats, cref.fr_random(70 + k, 5))
        blob = BP.write(cpk)
        pk, vk = BG.read_parameters(ctx, blob, checked=True)
        _vk_equal(vk, cpk["vk"])
        r, s = cref.fr_random(80 + k, 2)
        pr = BG.Prover(ctx, BG.R1CS(ni, na, *mats))
        proof, _ = pr.prove(pk, inputs, aux, r, s)
        assert (proof == GC.proof_bytes(*GC.prove(ni, na, mats, cpk, inputs, aux, r, s))).all(), k
        pk.free(); pr.free()


def test_2_18_key_write_read_round_trip(ctx, cref, tmp_path):
    """a 2^18-domain setup_gpu key (every vector crosses 2^16-point chunk boundaries): the written image equals the oracle
    encoder over pk.device_images and the vk, read -> write is byte-identical, the image does not depend on the key's table
    levels, and the read-back key (tabled) proves the same bytes"""
    from bazuka_b200 import groth16 as BG, synth
    ni, na, mats, inputs, aux = synth.build(256, 100, seed=17, ops=synth.GpuOps(ctx))
    pr = BG.Prover(ctx, BG.R1CS(ni, na, *mats))
    assert pr.log_m == 18
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, cref.fr_random(41, 5), cref.g1_generator(), cref.g2_generator())
    img = BG.write_parameters(ctx, pk)
    keys = {k: pk.device_images[k].cpu().numpy() for k in BP.VECTORS}
    assert bytes(img) == BP.write(dict(keys, vk=vk))
    info = BG.parameters_info(img)
    assert info["n_h"] == (1 << 18) - 1 and info["bytes"] == img.size
    assert min(info[f"n_{k}"] for k in ("h", "b_g2")) > 1 << 16, info
    path = tmp_path / "key.params"
    assert BG.write_parameters(ctx, pk, str(path)) == str(path)
    assert open(path, "rb").read() == bytes(img)
    pk2, vk2 = BG.read_parameters(ctx, str(path), checked=True)
    _vk_equal(vk2, vk)
    assert (BG.write_parameters(ctx, pk2) == img).all()
    pk1, _ = BG.read_parameters(ctx, img, checked=False, table_levels=1)
    assert (BG.write_parameters(ctx, pk1) == img).all()
    r, s = cref.fr_random(42, 2)
    want, _ = pr.prove(pk, inputs, aux, r, s)
    got, _ = pr.prove(pk2, inputs, aux, r, s)
    assert (got == want).all()
    got1, _ = pr.prove(pk1, inputs, aux, r, s)
    assert (got1 == want).all()
    for k in (pk, pk1, pk2, pr):
        k.free()


# ------------------------------------------------------------------ corruption matrix
CHUNK = 1 << 16
LEN = {"ic": 3, "h": CHUNK + 2, "l": 3, "a": 3, "b_g1": CHUNK + 2, "b_g2": CHUNK + 2}   # the key needs |b_g1| == |b_g2|


def _matrix_file():
    """a key image with h and b_g2 one chunk and two points long; every point a subgroup point"""
    g1 = [C.mul(C.FP, C.G1_GEN, 5 + 7 * i) for i in range(8)]
    g2 = [C.mul(C.FP2, C.G2_GEN, 11 + 3 * i) for i in range(8)]
    e1 = np.frombuffer(b"".join(BP.g1_to_uncompressed(p) for p in g1), np.uint8).reshape(8, 96)
    e2 = np.frombuffer(b"".join(BP.g2_to_uncompressed(p) for p in g2), np.uint8).reshape(8, 192)
    parts, offs, off = [], {}, 0

    def add(b):
        nonlocal off
        parts.append(np.frombuffer(b, np.uint8) if isinstance(b, bytes) else b.reshape(-1))
        off += parts[-1].size
    for k in VK_FIELDS:
        offs[k] = off
        add(bytes(e2[0]) if k.endswith("g2") else bytes(e1[0]))
    for k in ("ic",) + BP.VECTORS:
        add(LEN[k].to_bytes(4, "big"))
        offs[k] = off
        add(np.resize(e2 if k == "b_g2" else e1, (LEN[k], 192 if k == "b_g2" else 96)))
    return bytearray(np.concatenate(parts).tobytes()), offs


def _defect(kind, g2, good):
    enc = BP.g2_to_uncompressed if g2 else BP.g1_to_uncompressed
    b = bytearray(good)
    yo = 96 if g2 else 48
    if kind == "compression":
        b[0] |= 0x80
    elif kind == "sort":
        b[0] |= 0x20
    elif kind == "infinity_with_bits":
        b[0] |= 0x40
    elif kind == "infinity":
        b = bytearray(enc(None))
    elif kind == "x_eq_p":
        b[0:48] = BP.P.to_bytes(48, "big")
    elif kind == "y_eq_p":
        b[yo:yo + 48] = BP.P.to_bytes(48, "big")
    elif kind == "y_plus_1":
        last = len(b) - 48
        b[last:] = (int.from_bytes(b[last:], "big") + 1).to_bytes(48, "big")
    elif kind == "not_in_subgroup":
        b = bytearray(enc(lifts(99, 1, g2)[0]))
    return bytes(b)


KINDS = ("compression", "sort", "infinity_with_bits", "infinity", "x_eq_p", "y_eq_p", "y_plus_1", "not_in_subgroup")


def _expected(kind, vec, checked):
    vk_point = vec in VK_FIELDS
    if kind == "infinity":
        return 0 if vk_point else -8
    if kind == "y_plus_1":
        return -4 if (checked or vk_point or vec == "ic") else 0
    if kind == "not_in_subgroup":
        return -9 if (checked or vk_point or vec == "ic") else 0
    return -8


def _read_status(ctx, blob, checked):
    import bazuka_b200 as B
    from bazuka_b200 import groth16 as BG
    try:
        pk, _ = BG.read_parameters(ctx, np.frombuffer(blob, np.uint8), checked=checked, table_levels=1)
    except B.BzkError as e:
        return e.status, str(e)
    pk.free()
    return 0, ""


def test_corruption_matrix(ctx, cref):
    """every defect kind in every vector, at index 0, the last index and both sides of a chunk boundary in h and b_g2:
    bellman's status at checked = False / True and the exact first bad point; two defects report the earlier one; after
    the refusals the same context still reads a good key and proves with it"""
    blob, offs = _matrix_file()
    ok, _ = _read_status(ctx, bytes(blob), True)
    assert ok == 0
    places = []
    for vec in VK_FIELDS + ("ic",) + BP.VECTORS:
        n = 1 if vec in VK_FIELDS else LEN[vec]
        idx = {0, n - 1} | ({CHUNK - 1, CHUNK} if vec in ("h", "b_g2") else set())
        places += [(vec, i) for i in sorted(idx)]
    checked_cases = 0
    for vec, i in places:
        g2 = vec.endswith("g2")
        size = 192 if g2 else 96
        at = offs[vec] + i * size
        good = bytes(blob[at:at + size])
        for kind in KINDS:
            blob[at:at + size] = _defect(kind, g2, good)
            for checked in (False, True):
                st, msg = _read_status(ctx, bytes(blob), checked)
                want = _expected(kind, vec, checked)
                assert st == want, (vec, i, kind, checked, st, msg)
                if want:
                    assert f"{vec}[{i}]:" in msg, (vec, i, kind, msg)
                checked_cases += 1
            blob[at:at + size] = good
    # two defects: the one first in file order is reported
    for (v1, i1), (v2, i2) in ((("h", 0), ("l", 2)), (("ic", 2), ("b_g2", CHUNK)), (("h", CHUNK), ("h", CHUNK - 1)), (("beta_g2", 0), ("b_g1", 0))):
        saved = bytes(blob)
        for v, i in ((v1, i1), (v2, i2)):
            g2 = v.endswith("g2")
            size = 192 if g2 else 96
            at = offs[v] + i * size
            blob[at:at + size] = _defect("sort", g2, bytes(blob[at:at + size]))
        st, msg = _read_status(ctx, bytes(blob), True)
        first = min((offs[v1] + i1, v1, i1), (offs[v2] + i2, v2, i2))
        assert st == -8 and f"{first[1]}[{first[2]}]:" in msg, msg
        blob[:] = saved
    print(f"\n{checked_cases} corruption cases")
    # the context is intact: a good key still reads and proves
    test_oracle_written_keys_prove_like_the_oracle(ctx, cref)


def test_golden_vk_file_is_accepted(ctx):
    """a file made of a production verifying key and a few generator multiples reads checked, and the verifying key that
    comes back is the golden image"""
    from bazuka_b200 import groth16 as BG
    g1 = [C.mul(C.FP, C.G1_GEN, k) for k in (1, 2, 3)]
    g2 = [C.mul(C.FP2, C.G2_GEN, k) for k in (1, 2)]
    for name, blob in golden_vks().items():
        vk = vk_from_bincode(blob)
        img = BP.write({"vk": vk, "h": g1, "l": g1[:2], "a": g1, "b_g1": g1[:2], "b_g2": g2})
        pk, vk2 = BG.read_parameters(ctx, img, checked=True, table_levels=1)
        assert bytes(BG.vk_to_bincode(vk2)) == blob, name
        assert (BG.write_parameters(ctx, pk) == np.frombuffer(img, np.uint8)).all()
        pk.free()


def test_worker_key_round_trip_proves_the_block(ctx, cref, tmp_path):
    """the update worker's key (A=3, T=3, B=1) written to a file and read back from the path: the same verifying key image,
    and the native prover with the read key proves the block's update work to the same 391 bytes, which MpnWork::verify
    accepts"""
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn import wire as Wr, works as Wk
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    from bazuka_b200.mpn.worker import MpnUpdateWorker
    from test_wire_cpu import _scenario
    st, keys, deposits, withdraws, wpay, updates = _scenario()
    A, T, B = 3, 3, 1
    wu = MpnUpdateWorker(ctx, A, T, B, cref.fr_random(301, 5))
    path = tmp_path / "update.params"
    BG.write_parameters(ctx, wu.pk, str(path))
    read_pk, read_vk = BG.read_parameters(ctx, str(path), checked=True)
    assert bytes(BG.vk_to_bincode(read_vk)) == bytes(wu.vk_blob)
    config = {"log4_tree_size": A, "log4_token_tree_size": T, "log4_deposit_batch_size": B, "log4_withdraw_batch_size": B, "log4_update_batch_size": B,
              "mpn_contract_id": 0x1234, "mpn_num_update_batches": 1, "mpn_num_deposit_batches": 1, "mpn_num_withdraw_batches": 1,
              "deposit_vk": bytes(wu.vk_blob), "withdraw_vk": bytes(wu.vk_blob), "update_vk": bytes(wu.vk_blob)}
    works, _ = Wk.prepare_works(config, st, deposits, withdraws, updates, {"deposit": 11, "withdraw": 22, "update": 33}, height=9, withdraw_payments=wpay)
    upd = [w for w in works.values() if w["data"][0] == "update"]
    assert upd
    provers = []
    for pk in (wu.pk, read_pk):
        nat = Wk.NativeMpnProver(ctx)
        circ = NativeUpdateCircuit(A, T, B)
        nat.add_circuit("update", circ, pk)
        circ.free()
        provers.append(nat)
    me = bytes(range(32))
    lib = ctx._l
    for k, work in enumerate(upd):
        blob = Wr.work_to_bytes(work)
        r, s = cref.fr_random(600 + k, 2)
        want = provers[0].prove(blob, me, r, s)
        got = provers[1].prove(blob, me, r, s)
        assert len(got) == 391 and got == want
        h = ct.c_void_p()
        assert lib.bzk_mpn_work_decode(blob, len(blob), ct.byref(h), None) == 0
        assert lib.bzk_mpn_work_verify(h, me, got[4:]) == 1
        lib.bzk_mpn_work_free(h)
    for nat in provers:
        nat.free()
    read_pk.free()
    wu.free()
