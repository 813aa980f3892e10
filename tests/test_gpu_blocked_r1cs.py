"""GPU tier: the blocked R1CS (bzk_r1cs_upload_blocked, bzk_r1cs_columns_dev, bzk_g*_bases_fixed_base_mul) against the
explicit path it must equal:

  upload      refuses out-of-range columns (the last copy's included) and inconsistent rowptrs
  synthetic   the edge-case system of tests/test_blocked_r1cs_cpu.py: blocked and explicit proofs byte-equal on a key from
              setup_gpu on the expansion
  update      UpdateCircuit at B = 0, 1, 2 (A=2, T=1): the blocked setup's key file equals the explicit setup's byte for
              byte, proofs are byte-equal over both handles (and to the C oracle prover's at B = 1), a corrupted aux value in
              the last slot is refused as unsatisfied, and sharded proofs over the blocked handle equal the whole one
  configs[3]  UpdateCircuit A=16, T=3, B=5 (1024 signed transfers, 59.9 M constraints, 2^26 domain) on one H100: blocked
              compile and setup, native ledger and witness, checked proof accepted by both verifiers"""
import time

import numpy as np
import pytest

from conftest import fr_arr
from test_blocked_r1cs_cpu import synthetic, rand_fr
from test_gpu_baseline_configs import _ledger_and_transfers

pytestmark = pytest.mark.gpu


def _t():
    import torch
    return torch


def test_upload_refuses_out_of_range_columns_and_bad_rowptrs(ctx):
    import bazuka_b200 as B
    from bazuka_b200 import groth16 as BG
    br = synthetic(40, 3)
    pr = BG.Prover(ctx, br)                    # the valid system uploads
    assert pr.log_m == br.log_m and pr.l_len == br.num_aux
    pr.free()

    def variant(blocks=None, side0=None):
        mats = list(br.mats)
        if side0 is not None:
            mats[0] = side0
        return BG.BlockedR1CS(br.num_inputs, br.num_aux, *(blocks or br.blocks), *mats)

    rp, col, val = br.mats[0]
    h, t, reps, tail, lo, stride = br.blocks
    bad = [variant(blocks=(h, t, 6, tail, lo, stride))]          # copy 5's slot columns pass nv
    c2 = col.copy()
    c2[-1] = br.num_vars                                          # a tail column at nv
    bad.append(variant(side0=(rp, c2, val)))
    r2 = rp.copy()
    r2[2] = r2[3] + 1                                             # a decreasing rowptr
    bad.append(variant(side0=(r2, col, val)))
    bad.append(variant(blocks=(h, t, reps, tail, lo, 0)))          # repeated with a zero stride
    for b in bad:
        with pytest.raises(B.BzkError) as e:
            BG.Prover(ctx, b)
        assert e.value.status == -1
    # the transposed product is for blocked handles only
    ex = BG.Prover(ctx, br.expand())
    d = _t().zeros((br.num_vars, 4), dtype=_t().int64, device="cuda")
    assert ctx._l.bzk_r1cs_columns_dev(ctx._h, ex._h, 0, BG._p(d), BG._p(d)) == -1
    ex.free()


def test_synthetic_blocked_and_explicit_proofs_are_byte_equal(ctx, cref):
    import random
    from bazuka_b200 import groth16 as BG
    for reps in (1, 3):
        br = synthetic(50 + reps, reps)
        ex = br.expand()
        pe, pb = BG.Prover(ctx, ex), BG.Prover(ctx, br)
        assert (pe.log_m, pe.h_len, pe.l_len, pe.a_len, pe.b_len) == (pb.log_m, pb.h_len, pb.l_len, pb.a_len, pb.b_len)
        pk, vk = BG.setup_gpu(ctx, ex, cref.fr_random(60 + reps, 5), cref.g1_generator(), cref.g2_generator())
        z = rand_fr(random.Random(reps), br.num_vars)
        z[0] = fr_arr([1])[0]
        r, s = cref.fr_random(70 + reps, 2)
        inputs, aux = z[:br.num_inputs], z[br.num_inputs:]
        a, _ = pe.prove(pk, inputs, aux, r, s, check_satisfied=False)
        b, _ = pb.prove(pk, inputs, aux, r, s, check_satisfied=False)
        assert (a == b).all()
        pk.free(); pe.free(); pb.free()


def _update_setup(ctx, cref, A, T, B, seed):
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    nc = NativeUpdateCircuit(A, T, B, blocked=True)
    br = nc.blocked_r1cs()
    prog, epi = nc.program(0), nc.program(1)
    nc.free()
    ex = br.expand()
    toxic = cref.fr_random(seed, 5)
    pk_e, vk_e = BG.setup_gpu(ctx, ex, toxic, cref.g1_generator(), cref.g2_generator(), table_levels=1)
    pk_b, vk_b = BG.setup_gpu(ctx, br, toxic, cref.g1_generator(), cref.g2_generator(), table_levels=1)
    assert not hasattr(pk_b, "device_images")
    assert (BG.write_parameters(ctx, pk_e) == BG.write_parameters(ctx, pk_b)).all()
    return br, ex, prog, epi, pk_e, vk_e, pk_b


def _update_witness(ctx, A, T, B, prog, epi):
    from bazuka_b200.mpn.gpu_witness import UpdateWitnessGpu
    from bazuka_b200.mpn import update as U
    wit = UpdateWitnessGpu(ctx, A, T, prog, {B: epi})
    led, txs = _ledger_and_transfers(ctx, A, T, B, nacc=8)
    raws, ext, accepted, pub, n_acc = led.update_build(txs, B)
    assert accepted.all()
    d_in, d_aux = wit.witness_native(raws, ext, [42, 7, pub["state"], U.ZIESHA, pub["aux_data"], pub["next_state"]], B)
    wit.free(); led.free()
    return d_in, d_aux


@pytest.mark.parametrize("B", [0, 1, 2])
def test_update_circuit_blocked_setup_and_proofs_equal_explicit(ctx, cref, B):
    import torch
    import bazuka_b200 as Bz
    from bazuka_b200 import groth16 as BG, dist as bd
    from oracle import groth16_c as GC
    A, T = 2, 1
    br, ex, prog, epi, pk, vk, pk_b = _update_setup(ctx, cref, A, T, B, 800 + B)
    pe, pb = BG.Prover(ctx, ex), BG.Prover(ctx, br)
    d_in, d_aux = _update_witness(ctx, A, T, B, prog, epi)
    r, s = cref.fr_random(810 + B, 2)
    want, pts = pe.prove_dev(pk, d_in, d_aux, r, s)
    got, _ = pb.prove_dev(pk, d_in, d_aux, r, s)
    assert (got == want).all()
    assert (pb.prove_dev(pk_b, d_in, d_aux, r, s)[0] == want).all()
    assert BG.verify(vk, d_in.cpu().numpy().view(np.uint64).reshape(-1, 4)[1:], pts)
    inputs, aux = d_in.cpu().numpy().view(np.uint64).reshape(-1, 4), d_aux.cpu().numpy().view(np.uint64).reshape(-1, 4)
    if B == 1:
        a_idx, b_idx = GC.density(ex.num_inputs, ex.num_aux, ex.mats)
        cpk = {"log_m": pe.log_m, "vk": vk, "a_idx": a_idx, "b_idx": b_idx}
        for k in ("h", "l", "a", "b_g1", "b_g2"):
            cpk[k] = pk.device_images[k].cpu().numpy()
        assert (GC.proof_bytes(*GC.prove(ex.num_inputs, ex.num_aux, ex.mats, cpk, inputs, aux, r, s)) == want).all()
    # one aux value of the last slot corrupted
    head, tmpl, reps, tail, var_lo, stride = br.blocks
    bad = aux.copy()
    j = var_lo - br.num_inputs + reps * stride + stride // 2
    bad[j, 0] ^= 1
    with pytest.raises(Bz.BzkError) as e:
        pb.prove(pk, inputs, bad, r, s, check_satisfied=True)
    assert e.value.status == -7
    # sharded over the blocked handle: 3 base shards, then the split schedule over three contexts
    world = 3
    parts = []
    for rank in range(world):
        spk = BG.shard_proving_key(ctx, pk, pb.log_m, rank, world)
        parts.append(pb.prove_partial(spk, d_in, d_aux))
        spk.free()
    fold = lambda ps: (bd.fold([p[0] for p in ps], "g1"), bd.fold([p[1] for p in ps], "g1"), bd.fold([p[2] for p in ps], "g2"),
                       bd.fold([p[3] for p in ps], "g1"))
    assert (BG.finalize(vk, fold(parts), r, s)[0] == want).all()
    m = 1 << pb.log_m
    ctxs = [Bz.Context(0) for _ in range(world)]
    provers = [BG.Prover(c, br) for c in ctxs]
    spks = [BG.shard_proving_key(c, pk, pb.log_m, k, world) for k, c in enumerate(ctxs)]
    bufs = [torch.empty((m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
    for k in range(world):
        provers[k].shard_begin(spks[k], d_in, d_aux, [bufs[j] if j == k else None for j in range(3)])
    provers[0].h_combine(*bufs)
    ctxs[0].synchronize()
    parts = []
    for k in range(world):
        lo, hi = bd.shard_range(m - 1, k, world)
        parts.append(provers[k].shard_finish(spks[k], bufs[0][lo:hi].contiguous()))
    assert (BG.finalize(vk, fold(parts), r, s)[0] == want).all()
    for x in spks + provers:
        x.free()
    for c in ctxs:
        c.close()
    pk.free(); pk_b.free(); pe.free(); pb.free()
    torch.cuda.empty_cache()


def test_config3_1024_transaction_batch_on_one_gpu(ctx, cref):
    """BASELINE configs[3] at full size: A=16 (the depth-32 tree), T=3, B=5 (1024 signed transfers), 59.9 M constraints, a
    2^26 domain, on one 80 GB H100 — blocked compile, blocked setup without fixed-base tables (table_levels=1), native ledger
    and witness, `prove_dev` with the satisfiability check; the product's byte-image verifier and the oracle's big-integer
    pairing check accept, and both reject a tampered public input.  The C oracle prover is not run at this size (hours of
    CPU time); byte equality with it is pinned at B = 1 above and at 2^24 by test_gpu_baseline_configs.  Prints the stage
    times and the free device memory after setup and after the proof."""
    import torch
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn import update as U
    from bazuka_b200.mpn.cs import to_mont
    from bazuka_b200.mpn.gpu_witness import UpdateWitnessGpu
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    from oracle import groth16_c as GC
    A, T, B = 16, 3, 5
    marks, free_gb = {}, {}
    gb = lambda: round(torch.cuda.mem_get_info()[0] / 1e9, 1)
    t0 = time.time()
    nc = NativeUpdateCircuit(A, T, B, blocked=True)
    br = nc.blocked_r1cs()
    prog, epi = nc.program(0), nc.program(1)
    nc.free()
    marks["compile_s"] = time.time() - t0
    t0 = time.time()
    pk, vk = BG.setup_gpu(ctx, br, cref.fr_random(901, 5), cref.g1_generator(), cref.g2_generator(), table_levels=1)
    pr = BG.Prover(ctx, br)
    torch.cuda.synchronize()
    marks["setup_s"] = time.time() - t0
    free_gb["after_setup"] = gb()
    assert pr.log_m == 26
    wit = UpdateWitnessGpu(ctx, A, T, prog, {B: epi})
    t0 = time.time()
    led, txs = _ledger_and_transfers(ctx, A, T, B, 128)
    marks["ledger_and_signing_s"] = time.time() - t0
    t0 = time.time()
    raws, ext, accepted, pub, n_acc = led.update_build(txs, B)
    assert n_acc == 1024 and accepted.all()
    d_in, d_aux = wit.witness_native(raws, ext, [42, 7, pub["state"], U.ZIESHA, pub["aux_data"], pub["next_state"]], B)
    torch.cuda.synchronize()
    marks["witness_s"] = time.time() - t0
    r, s = cref.fr_random(902, 2)
    t0 = time.time()
    blob, pts = pr.prove_dev(pk, d_in, d_aux, r, s, check_satisfied=True)
    marks["prove_s"] = time.time() - t0
    free_gb["after_proof"] = gb()
    public = to_mont([42, 7, pub["state"], pub["aux_data"], pub["next_state"]])
    assert (d_in.cpu().numpy().view(np.uint64)[1:] == public).all()
    assert BG.verify_bytes(BG.vk_to_bincode(vk), public, blob)
    assert GC.verify_py(vk, public, pts)
    wrong = public.copy()
    wrong[4] = wrong[2]
    assert not BG.verify_bytes(BG.vk_to_bincode(vk), wrong, blob)
    assert not GC.verify_py(vk, wrong, pts)
    print({"A": A, "T": T, "B": B, "log_m": pr.log_m, "constraints": br.num_constraints, "gpu": torch.cuda.get_device_name(),
           **{k: round(v, 1) for k, v in marks.items()}, "free_gb": free_gb})
    wit.free(); led.free(); pk.free(); pr.free()
    del pk, pr, d_in, d_aux
    torch.cuda.empty_cache()
