"""GPU tier: the Groth16 driver on the degenerate and boundary constraint systems of r1cs_cases.py.  Per case: the upload's
shape, setup_gpu's key and vk images against the C oracle's, and the proof bytes against the big-integer restatement
(m <= 2^7, on the oracle's key) or the C oracle (larger m), from every route: prove, prove_dev, prove_partial +
finalize at world 1..4 (so that some shards are empty), the split schedule shard_begin / h_combine / shard_finish at
world 1..3 (contexts standing in for ranks), the key with all five vectors in host memory, the key with 2-level tables,
the key read back from its bellman file image, and the blocked handle (proved on, and set up from).  Unsatisfied
witnesses are refused with the exact count of bad rows, and prove the oracle's bytes with the check off.  Then one context
interleaving large and small proofs, the refusal of non-canonical coefficient images, and the cancelling duplicates whose
identity column makes the key's file image unreadable."""
import multiprocessing as mp

import numpy as np
import pytest

import r1cs_cases as RC
from oracle import groth16_c as GC

pytestmark = pytest.mark.gpu

CASES = RC.all_cases(large=True)
BY_NAME = {c.name: c for c in CASES}
KEY = ("h", "l", "a", "b_g1", "b_g2")


def _oracle_key(case):
    return GC.setup(case.ni, case.na, RC.case_mats(case), RC.toxic(case))


def _big_int_bytes(name):
    """G.prove on the C oracle's key for one case (a worker process: pure Python)"""
    case = {c.name: c for c in RC.all_cases()}[name]
    cpk = _oracle_key(case)
    cpk["nv"] = case.ni + case.na
    return RC.big_int_proof_bytes(case, RC.oracle_points(cpk))


@pytest.fixture(scope="module")
def big_int(cref):
    """the restatement's proof bytes for every case with m <= 2^7, computed on the host's cores while the GPU works"""
    names = [c.name for c in CASES if c.big_int]
    pool = mp.get_context("spawn").Pool()
    res = pool.map_async(_big_int_bytes, names, chunksize=1)
    got = {}

    def get(name):
        if not got:
            got.update(zip(names, res.get()))
        return got[name]
    yield get
    pool.close()
    pool.join()


@pytest.fixture(scope="module")
def ranks():
    """two more contexts on the same GPU, standing in for ranks 1 and 2 of the split schedule"""
    import bazuka_b200 as B
    cs = [B.Context(0) for _ in range(2)]
    yield cs
    for c in cs:
        c.close()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def _fold(parts):
    from bazuka_b200 import dist as bd
    return (bd.fold([p[0] for p in parts], "g1"), bd.fold([p[1] for p in parts], "g1"),
            bd.fold([p[2] for p in parts], "g2"), bd.fold([p[3] for p in parts], "g1"))


def _want(case, big_int, cpk):
    if case.big_int:
        return np.frombuffer(big_int(case.name), np.uint8)
    inputs, aux = RC.witness(case)
    return GC.proof_bytes(*GC.prove(case.ni, case.na, RC.case_mats(case), cpk, inputs, aux, *RC.rs(case)))


@pytest.mark.parametrize("name", [c.name for c in CASES])
def test_case_on_every_route(ctx, cref, ranks, big_int, name):
    import bazuka_b200 as B
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.dist import shard_range
    case = BY_NAME[name]
    r1 = RC.r1cs(case)
    pr = BG.Prover(ctx, r1)
    assert (pr.log_m, pr.h_len, pr.l_len, pr.a_len, pr.b_len) == case.expect
    cpk = _oracle_key(case)
    pk, vk = BG.setup_gpu(ctx, r1, RC.toxic(case), cref.g1_generator(), cref.g2_generator(), table_levels=1)
    for k in ("alpha_g1", "beta_g1", "delta_g1", "beta_g2", "gamma_g2", "delta_g2", "ic"):
        assert (np.asarray(vk[k]) == cpk["vk"][k]).all(), k
    for k in KEY:
        img = pk.device_images[k].cpu().numpy()
        assert img.shape == cpk[k].shape and (img == cpk[k]).all(), k
    inputs, aux = RC.witness(case)
    r, s = RC.rs(case)
    want = _want(case, big_int, cpk)
    d_in, d_aux = _dev(inputs), _dev(aux)
    check = case.bad == 0
    if case.bad:
        calls = (lambda: pr.prove(pk, inputs, aux, r, s), lambda: pr.prove_dev(pk, d_in, d_aux, r, s),
                 lambda: pr.prove_partial(BG.shard_proving_key(ctx, pk, pr.log_m, 0, 1), inputs, aux))
        for call in calls:
            with pytest.raises(B.BzkError) as e:
                call()
            assert e.value.status == -7 and f": {case.bad} constraints unsatisfied by the witness" in str(e.value)
    blob, pts = pr.prove(pk, inputs, aux, r, s, check_satisfied=check)
    assert (blob == want).all()
    pvk = BG.PreparedVerifyingKey(vk)
    assert BG.verify(vk, inputs[1:], pts) == check
    assert pvk.verify_batch_gpu(ctx, inputs[1:][None], blob[None], seed=case.seed)[0] == check
    pvk.free()
    routes = {"prove_dev": pr.prove_dev(pk, d_in, d_aux, r, s, check_satisfied=check)[0]}
    # base shards: world 1..4, so that short vectors (h at m = 2, b with one entry, l with none) leave ranks empty
    for world in (1, 2, 3, 4):
        parts = []
        for rank in range(world):
            spk = BG.shard_proving_key(ctx, pk, pr.log_m, rank, world)
            parts.append(pr.prove_partial(spk, inputs, aux, check_satisfied=check))
            spk.free()
        routes[f"partial-{world}"] = BG.finalize(vk, _fold(parts), r, s)[0]
    # the split schedule: vector j belongs to rank j mod world; rank 0 combines and deals the quotient out in slices
    import torch
    m = 1 << pr.log_m
    for world in (1, 2, 3):
        ctxs = [ctx] + ranks[:world - 1]
        provers = [pr] + [BG.Prover(c, r1) for c in ctxs[1:]]
        spks = [BG.shard_proving_key(c, pk, pr.log_m, k, world) for k, c in enumerate(ctxs)]
        bufs = [torch.empty((m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
        for k in range(world):
            provers[k].shard_begin(spks[k], d_in, d_aux, [bufs[j] if j % world == k else None for j in range(3)])
        pr.h_combine(*bufs)
        ctx.synchronize()
        parts = []
        for k in range(world):
            lo, hi = shard_range(m - 1, k, world)
            parts.append(provers[k].shard_finish(spks[k], bufs[0][lo:hi].contiguous() if hi > lo else None))
        routes[f"split-{world}"] = BG.finalize(vk, _fold(parts), r, s)[0]
        for x in spks + provers[1:]:
            x.free()
    pk.move(31)
    routes["host-key"] = pr.prove(pk, inputs, aux, r, s, check_satisfied=check)[0]
    pk.move(0)
    pk.precompute(2)
    routes["tables-2"] = pr.prove(pk, inputs, aux, r, s, check_satisfied=check)[0]
    # The key's bellman file image: read back and proved with, or refused when the key holds an identity, as bellman's
    # reader refuses one.  bellman's generator leaves one in l for an aux variable no constraint names, and this library
    # leaves one in a / b for a cancelled variable.
    image = BG.write_parameters(ctx, pk)
    ident = {k: np.nonzero(cpk[k][:, 192 if k == "b_g2" else 96])[0].tolist() for k in KEY}
    net = [RC.net_vars(case.cs.rows, side) for side in range(3)]
    assert ident["a"] == [i for i, v in enumerate(cpk["a_idx"]) if v not in net[0] and v >= case.ni]
    assert ident["b_g1"] == ident["b_g2"] == [i for i, v in enumerate(cpk["b_idx"]) if v not in net[1]]
    assert ident["l"] == [v - case.ni for v in range(case.ni, case.ni + case.na) if v not in net[0] | net[1] | net[2]]
    assert not ident["h"] and bool(ident["a"] or ident["b_g1"]) == bool(case.cancelling)
    first = next((f"{k}[{ident[k][0]}]" for k in KEY if len(ident[k])), None)
    if first:
        with pytest.raises(B.BzkError) as e:
            BG.read_parameters(ctx, image)
        assert e.value.status == -8 and f"{first}: point at infinity" in str(e.value)
    else:
        pk2, _ = BG.read_parameters(ctx, image, table_levels=1)
        routes["file-key"] = pr.prove(pk2, inputs, aux, r, s, check_satisfied=check)[0]
        pk2.free()
    # the blocked handle: the same shape, the same proof, and a key set up from it with the same file image
    br = RC.blocked_r1cs(case)
    prb = BG.Prover(ctx, br)
    assert (prb.log_m, prb.h_len, prb.l_len, prb.a_len, prb.b_len) == case.expect
    routes["blocked"] = prb.prove(pk, inputs, aux, r, s, check_satisfied=check)[0]
    pkb, vkb = BG.setup_gpu(ctx, br, RC.toxic(case), cref.g1_generator(), cref.g2_generator(), table_levels=1)
    assert (BG.write_parameters(ctx, pkb) == image).all()
    routes["blocked-key"] = prb.prove(pkb, inputs, aux, r, s, check_satisfied=check)[0]
    for route, got in routes.items():
        assert (got == want).all(), route
    pkb.free(); prb.free(); pk.free(); pr.free()


def _fresh_proof(case, imgs, vk):
    """the case's proof on a new context with the key built from its images"""
    import bazuka_b200 as B
    from bazuka_b200 import groth16 as BG
    c = B.Context(0)
    try:
        pr = BG.Prover(c, RC.r1cs(case))
        pk = BG.proving_key_from_host(c, vk, *(imgs[k] for k in KEY), table_levels=1)
        inputs, aux = RC.witness(case)
        blob = pr.prove(pk, inputs, aux, *RC.rs(case))[0]
        pk.free(); pr.free()
        return blob
    finally:
        c.close()


def test_one_context_interleaving_large_and_small_proofs(cref):
    """the staging arena only grows: a small proof after a large one runs over the large one's stale evaluations, so only
    the padding memset and the input-row copy keep it right"""
    import bazuka_b200 as B
    from bazuka_b200 import groth16 as BG
    order = ["boundary-65536-ni5", "boundary-9-ni2", "boundary-4096-ni2", "boundary-65536-ni5", "m1", "boundary-2-ni1"]
    keys, fresh = {}, {}
    for name in dict.fromkeys(order):
        case = BY_NAME[name]
        cpk = _oracle_key(case)
        keys[name] = cpk
        fresh[name] = _fresh_proof(case, cpk, cpk["vk"])
        inputs, aux = RC.witness(case)
        want = GC.proof_bytes(*GC.prove(case.ni, case.na, RC.case_mats(case), cpk, inputs, aux, *RC.rs(case)))
        assert (fresh[name] == want).all(), name
    c = B.Context(0)
    try:
        for name in order:
            case = BY_NAME[name]
            pr = BG.Prover(c, RC.r1cs(case))
            pk = BG.proving_key_from_host(c, keys[name]["vk"], *(keys[name][k] for k in KEY), table_levels=1)
            inputs, aux = RC.witness(case)
            assert (pr.prove(pk, inputs, aux, *RC.rs(case))[0] == fresh[name]).all(), name
            pk.free(); pr.free()
    finally:
        c.close()


@pytest.mark.parametrize("image", ["r", "r+1", "2^256-1"])
@pytest.mark.parametrize("form", ["explicit", "blocked"])
def test_upload_refuses_coefficient_images_not_below_r(ctx, cref, form, image):
    """r is a zero whose limbs are not: without the refusal it would count as present and give its variable an identity
    column.  Refused as an argument before any launch; the context then proves the next case."""
    import bazuka_b200 as B
    from bazuka_b200 import groth16 as BG
    case = BY_NAME["blocked-reps1"]
    v = {"r": RC.R, "r+1": RC.R + 1, "2^256-1": (1 << 256) - 1}[image]
    img = np.frombuffer(v.to_bytes(32, "little"), np.uint64)
    r1 = RC.blocked_r1cs(case) if form == "blocked" else RC.r1cs(case)
    for side in range(3):
        rp, col, val = r1.mats[side]
        bad = val.copy()
        bad[len(bad) - 1] = img
        r1.mats[side] = (rp, col, bad)
        before = ctx.launch_count
        with pytest.raises(B.BzkError) as e:
            BG.Prover(ctx, r1)
        assert e.value.status == -1 and ctx.launch_count == before
        r1.mats[side] = (rp, col, val)
    ok = RC.blocked_r1cs(case) if form == "blocked" else RC.r1cs(case)
    pr = BG.Prover(ctx, ok)
    cpk = _oracle_key(case)
    pk = BG.proving_key_from_host(ctx, cpk["vk"], *(cpk[k] for k in KEY), table_levels=1)
    inputs, aux = RC.witness(case)
    want = GC.proof_bytes(*GC.prove(case.ni, case.na, RC.case_mats(case), cpk, inputs, aux, *RC.rs(case)))
    assert (pr.prove(pk, inputs, aux, *RC.rs(case))[0] == want).all()
    pk.free(); pr.free()
