"""GPU tier: the Groth16 prover (bzk_groth16_prove) against the CPU oracle — identical 387-byte
proof images for identical (parameters, r, s, witness) — plus pairing verification of GPU proofs,
the GPU trusted-setup helper against the oracle generator, and UNSAT detection.  Mirrors the shape
of the reference's own prover tests (setup -> create_random_proof -> verify_proof, negative cases:
/root/reference/src/zk/groth16/gadgets/common/test.rs:46-64, /root/reference/src/mpn/circuits/test.rs:117-229)."""
import numpy as np
import pytest

from conftest import fr_arr
from test_groth16_cpu import tiny_circuit, to_csr

pytestmark = pytest.mark.gpu


def _prover(ctx, ni, na, mats):
    from bazuka_b200 import groth16 as BG
    return BG, BG.Prover(ctx, BG.R1CS(ni, na, *mats))


def test_tiny_circuit_proof_bytes_and_pairing(ctx, cref):
    from oracle import groth16_c as GC
    from oracle.py import groth16 as G, field as Fd
    cs, z = tiny_circuit()
    mats = to_csr(cs)
    g = Fd.SplitMix64(7)
    tox = [g.fr() for _ in range(5)]
    r, s = g.fr(), g.fr()
    cpk = GC.setup(cs.num_inputs, cs.num_aux, mats, fr_arr(tox))
    BG, pr = _prover(ctx, cs.num_inputs, cs.num_aux, mats)
    assert (pr.log_m, pr.h_len, pr.l_len, pr.a_len, pr.b_len) == (3, 7, 3, len(cpk["a"]), len(cpk["b_g1"]))
    pk = BG.proving_key_from_host(ctx, cpk["vk"], cpk["h"], cpk["l"], cpk["a"], cpk["b_g1"], cpk["b_g2"])
    zz = fr_arr(z)
    blob, pts = pr.prove(pk, zz[:2], zz[2:], fr_arr([r])[0], fr_arr([s])[0])
    # == big-integer bellman restatement, == C oracle
    want = G.proof_to_bytes(G.prove(cs, G.setup(cs, *tox), z, r, s))
    assert bytes(blob) == want
    assert (blob == GC.proof_bytes(*GC.prove(cs.num_inputs, cs.num_aux, mats, cpk, zz[:2], zz[2:], fr_arr([r])[0], fr_arr([s])[0]))).all()
    assert GC.verify_py(cpk["vk"], zz[1:2], pts)
    assert len(BG.zkproof_blob(blob)) == 391 and not BG.zkproof_blob(blob)[:4].any()
    # wrong witness: refused when checking, garbage (non-verifying) proof when not — as bellman
    bad = zz.copy()
    bad[2] = fr_arr([4])[0]
    import bazuka_b200 as B
    with pytest.raises(B.BzkError) as e:
        pr.prove(pk, bad[:2], bad[2:], fr_arr([r])[0], fr_arr([s])[0])
    assert e.value.status == -7
    _, pts_bad = pr.prove(pk, bad[:2], bad[2:], fr_arr([r])[0], fr_arr([s])[0], check_satisfied=False)
    assert not GC.verify_py(cpk["vk"], zz[1:2], pts_bad)


@pytest.mark.parametrize("lanes,rounds", [(2, 3), (16, 20)])
def test_synthetic_circuit_vs_oracle_prover(ctx, cref, lanes, rounds):
    from bazuka_b200 import synth
    from oracle import groth16_c as GC
    ni, na, mats, inputs, aux = synth.build(lanes, rounds, seed=9, ops=synth.GpuOps(ctx))
    # the generator gives the same instance on either backend
    ni2, na2, mats2, inputs2, aux2 = synth.build(lanes, rounds, seed=9, ops=GC.CpuOps)
    assert (inputs == inputs2).all() and (aux == aux2).all()
    tox = cref.fr_random(21, 5)
    r, s = cref.fr_random(22, 2)
    cpk = GC.setup(ni, na, mats, tox)
    BG, pr = _prover(ctx, ni, na, mats)
    pk = BG.proving_key_from_host(ctx, cpk["vk"], cpk["h"], cpk["l"], cpk["a"], cpk["b_g1"], cpk["b_g2"])
    blob, pts = pr.prove(pk, inputs, aux, r, s)
    assert (blob == GC.proof_bytes(*GC.prove(ni, na, mats, cpk, inputs, aux, r, s))).all()
    if lanes == 2:
        assert GC.verify_py(cpk["vk"], inputs[1:], pts)


def test_gpu_setup_equals_oracle_generator(ctx, cref):
    from bazuka_b200 import synth
    from oracle import groth16_c as GC
    ni, na, mats, inputs, aux = synth.build(4, 6, seed=3, ops=GC.CpuOps)
    tox = cref.fr_random(31, 5)
    cpk = GC.setup(ni, na, mats, tox)
    BG, pr = _prover(ctx, ni, na, mats)
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, tox, cref.g1_generator(), cref.g2_generator())
    for k in ("alpha_g1", "beta_g1", "delta_g1", "beta_g2", "gamma_g2", "delta_g2", "ic"):
        assert (np.asarray(vk[k]) == cpk["vk"][k]).all(), k
    for k in ("h", "l", "a", "b_g1", "b_g2"):
        assert (pk.device_images[k].cpu().numpy() == cpk[k]).all(), k
    r, s = cref.fr_random(32, 2)
    blob, pts = pr.prove(pk, inputs, aux, r, s)
    assert (blob == GC.proof_bytes(*GC.prove(ni, na, mats, cpk, inputs, aux, r, s))).all()
    assert GC.verify_py(vk, inputs[1:], pts)


def test_prover_2_18_domain_vs_oracle(ctx, cref):
    """a 2^18-point domain (142 k constraints): GPU setup + GPU proof, proof bytes against the
    multi-threaded C prover run on the very same parameters."""
    from bazuka_b200 import synth
    from oracle import groth16_c as GC
    ni, na, mats, inputs, aux = synth.build(256, 100, seed=17, ops=synth.GpuOps(ctx))
    BG, pr = _prover(ctx, ni, na, mats)
    assert pr.log_m == 18
    tox = cref.fr_random(41, 5)
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, tox, cref.g1_generator(), cref.g2_generator())
    r, s = cref.fr_random(42, 2)
    blob, pts = pr.prove(pk, inputs, aux, r, s)
    a_idx, b_idx = GC.density(ni, na, mats)
    cpk = {"log_m": 18, "vk": vk, "a_idx": a_idx, "b_idx": b_idx}
    for k in ("h", "l", "a", "b_g1", "b_g2"):
        cpk[k] = pk.device_images[k].cpu().numpy()
    assert (blob == GC.proof_bytes(*GC.prove(ni, na, mats, cpk, inputs, aux, r, s))).all()


def test_proofs_do_not_depend_on_table_levels(ctx, cref):
    """A key's fixed-base tables get as many levels as fit in the device memory free when it is built, so the same key
    runs different MSM plans on different days.  One 2^16-domain circuit, one oracle proof on the key images, and the GPU
    key built at every level count from 1 to 16: every proof is byte-equal to the oracle's, and the sweep ran at least
    four distinct table plans (read from stand-alone copies of the key's columns tabled at the same level counts)."""
    from bazuka_b200 import synth
    from oracle import groth16_c as GC
    ni, na, mats, inputs, aux = synth.build(64, 100, seed=23, ops=synth.GpuOps(ctx))
    BG, pr = _prover(ctx, ni, na, mats)
    assert pr.log_m == 16
    tox = cref.fr_random(51, 5)
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, tox, cref.g1_generator(), cref.g2_generator(), table_levels=1)
    cols = ("h", "l", "a", "b_g1", "b_g2")
    imgs = {k: pk.device_images[k].cpu().numpy() for k in cols}
    pk.free()
    r, s = cref.fr_random(52, 2)
    a_idx, b_idx = GC.density(ni, na, mats)
    want = GC.proof_bytes(*GC.prove(ni, na, mats, dict(imgs, log_m=16, vk=vk, a_idx=a_idx, b_idx=b_idx), inputs, aux, r, s))
    plans = set()
    for levels in (1, 2, 3, 4, 5, 6, 8, 12, 16):
        pk = BG.proving_key_from_host(ctx, vk, *(imgs[k] for k in cols), table_levels=levels)
        blob, _ = pr.prove(pk, inputs, aux, r, s)
        pk.free()
        assert (blob == want).all(), levels
        for k in cols:
            rb = ctx.g2_bases(imgs[k]) if k == "b_g2" else ctx.g1_bases(imgs[k])
            rb.precompute(levels)
            sc = cref.fr_random(60, len(rb))
            (ctx.msm_g2_resident if k == "b_g2" else ctx.msm_g1_resident)(rb, sc)
            p = ctx.last_msm_plan()
            if p["T"] > 1:
                plans.add((p["c"], p["T"], p["G"]))
            rb.free()
    print(f"\ntable plans run by the key's columns over levels 1..16: {sorted(plans)}")
    assert len(plans) >= 4, plans


def test_base_sharded_partials_fold_to_the_same_proof(ctx, cref):
    """schedule (S) of SURVEY.md §8e on one GPU: the proving key cut into 3 contiguous base shards, each shard's
    four partial sums from `bzk_groth16_prove_partial`, folded with the host group law and finalised —
    byte-equal to the unsharded GPU proof (and so to the oracle's, by the tests above)."""
    import torch
    from bazuka_b200 import groth16 as BG, synth, dist as bd
    ni, na, mats, inputs, aux = synth.build(lanes=16, rounds=6, seed=31, ops=synth.GpuOps(ctx))
    pr = BG.Prover(ctx, BG.R1CS(ni, na, *mats))
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, cref.fr_random(41, 5), cref.g1_generator(), cref.g2_generator())
    r, s = cref.fr_random(42, 2)
    want, _ = pr.prove(pk, inputs, aux, r, s)
    world = 3
    parts = []
    for rank in range(world):
        spk = BG.shard_proving_key(ctx, pk, pr.log_m, rank, world)
        parts.append(pr.prove_partial(spk, inputs, aux))
        with pytest.raises(Exception):
            pr.prove(spk, inputs, aux, r, s)  # a shard cannot finish a proof by itself
        spk.free()
    sums = (bd.fold([p[0] for p in parts], "g1"), bd.fold([p[1] for p in parts], "g1"),
            bd.fold([p[2] for p in parts], "g2"), bd.fold([p[3] for p in parts], "g1"))
    blob, pts = BG.finalize(vk, sums, r, s)
    assert (blob == want).all()
    assert BG.verify(vk, inputs[1:], pts)
    # resident witness through the same entry point
    d_in = torch.from_numpy(inputs.view(np.int64)).cuda()
    d_aux = torch.from_numpy(aux.view(np.int64)).cuda()
    spk = BG.shard_proving_key(ctx, pk, pr.log_m, 0, 1)
    one = pr.prove_partial(spk, d_in, d_aux)
    assert (BG.finalize(vk, one, r, s)[0] == want).all()
    spk.free(); pk.free(); pr.free()


def test_split_sharded_schedule_gives_the_same_proof(ctx, cref):
    """bzk_groth16_shard_begin / _h_combine_dev / _shard_finish: three ranks emulated by three contexts on one GPU — rank s owns
    evaluation vector s (computes it, takes it to the coset), rank 0 combines them into the quotient and deals out slices, every
    rank sums its base shards — folded and finalised to the bytes of the unsharded proof; a finish without a begin is refused."""
    import torch
    import bazuka_b200 as B
    from bazuka_b200 import groth16 as BG, synth, dist as bd
    ni, na, mats, inputs, aux = synth.build(lanes=16, rounds=6, seed=31, ops=synth.GpuOps(ctx))
    pr = BG.Prover(ctx, BG.R1CS(ni, na, *mats))
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, cref.fr_random(41, 5), cref.g1_generator(), cref.g2_generator())
    r, s = cref.fr_random(42, 2)
    want, _ = pr.prove(pk, inputs, aux, r, s)
    d_in = torch.from_numpy(inputs.view(np.int64)).cuda()
    d_aux = torch.from_numpy(aux.view(np.int64)).cuda()
    world, m = 3, 1 << pr.log_m
    ctxs = [B.Context(0) for _ in range(world)]
    provers = [BG.Prover(c, BG.R1CS(ni, na, *mats)) for c in ctxs]
    spks = [BG.shard_proving_key(c, pk, pr.log_m, k, world) for k, c in enumerate(ctxs)]
    with pytest.raises(B.BzkError):
        provers[1].shard_finish(spks[1], torch.zeros((1, 4), dtype=torch.int64, device="cuda"))
    bufs = [torch.empty((m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
    for k in range(world):
        provers[k].shard_begin(spks[k], d_in, d_aux, [bufs[j] if j == k else None for j in range(3)])
    provers[0].h_combine(*bufs)
    ctxs[0].synchronize()
    parts = []
    for k in range(world):
        lo, hi = bd.shard_range(m - 1, k, world)
        parts.append(provers[k].shard_finish(spks[k], bufs[0][lo:hi].contiguous()))
    sums = (bd.fold([p[0] for p in parts], "g1"), bd.fold([p[1] for p in parts], "g1"),
            bd.fold([p[2] for p in parts], "g2"), bd.fold([p[3] for p in parts], "g1"))
    blob, pts = BG.finalize(vk, sums, r, s)
    assert (blob == want).all()
    assert BG.verify(vk, inputs[1:], pts)
    # one rank owning everything (world = 1) through the same entry points
    spk1 = BG.shard_proving_key(ctx, pk, pr.log_m, 0, 1)
    pr.shard_begin(spk1, d_in, d_aux, bufs)
    pr.h_combine(*bufs)
    ctx.synchronize()
    one = pr.shard_finish(spk1, bufs[0][:m - 1].contiguous())
    assert (BG.finalize(vk, one, r, s)[0] == want).all()
    for x in spks + [spk1]:
        x.free()
    for x in provers:
        x.free()
    pk.free(); pr.free()


def test_batch_verifier_on_gpu_equals_host_batch_verifier(ctx, cref):
    """bzk_groth16_verify_batch_dev (one thread per proof: [r_j]A_j, the Jacobian walk of B_j, 68 line evaluations; product,
    key-dependent loops and the single final exponentiation on the host) against the host batch verifier and the oracle's
    pairing check: all-valid batch accepted, a tampered C / a wrong input / a malformed point located."""
    from bazuka_b200 import groth16 as BG, synth
    from oracle import groth16_c as GC
    ni, na, mats, inputs, aux = synth.build(4, 6, seed=3, ops=GC.CpuOps)
    _, pr = _prover(ctx, ni, na, mats)
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, cref.fr_random(31, 5), cref.g1_generator(), cref.g2_generator())
    m = 70
    rs = cref.fr_random(32, 2 * m)
    proofs, pts0 = [], None
    for j in range(m):
        blob, pts = pr.prove(pk, inputs, aux, rs[2 * j], rs[2 * j + 1], check_satisfied=(j == 0))
        proofs.append(blob)
        pts0 = pts0 or pts
    proofs = np.stack(proofs)
    assert GC.verify_py(vk, inputs[1:], pts0)
    pubs = np.repeat(inputs[1:][None], m, axis=0)
    pvk = BG.PreparedVerifyingKey(vk)
    ok_h, each_h = pvk.verify_batch(pubs, proofs, seed=99)
    ok_d, each_d = pvk.verify_batch_gpu(ctx, pubs, proofs, seed=99)
    assert ok_h and ok_d and each_d.all()
    bad = proofs.copy()
    bad[3, 290:387] = proofs[4, 0:97]            # C replaced by another curve point
    wrong = pubs.copy()
    wrong[11, 0] = wrong[11, 1] if wrong.shape[1] > 1 else cref.fr_random(5, 1)[0]
    bad2 = proofs.copy()
    bad2[20, 7] ^= 1                              # not on the curve
    for p_, pub_ in ((bad, pubs), (proofs, wrong), (bad2, pubs)):
        ok_h, each_h = pvk.verify_batch(pub_, p_, seed=7)
        ok_d, each_d = pvk.verify_batch_gpu(ctx, pub_, p_, seed=7)
        assert not ok_h and not ok_d and (each_h == each_d).all() and each_d.sum() == m - 1
    pvk.free(); pk.free(); pr.free()
