"""GPU tier: the MPN worker (csrc/mpn_worker.cu) — a node's GetMpnWorkResponse bytes in, the PostMpnSolutionRequest bytes out —
on the production block shape (deposit 4^3, withdraw 4^3, update 4^4 at A=15, T=3) with one and two contexts on one GPU, and
on BASELINE configs[3] (1024 signed transfers, A=16, B=5, 2^26) through the blocked update circuit on one H100."""
import ctypes as ct
import time

import numpy as np
import pytest

import mpn_worker_cases as C

pytestmark = pytest.mark.gpu

A, T, BD, BW, BU = 15, 3, 3, 3, 4
ME = bytes(range(32))
SEED = bytes([3]) * 32


def _proof_points(p387):
    return p387[0:97], p387[97:290], p387[290:387]


# first in the file: the 2^26 key needs the device to itself, before the module fixture below holds its keys
def test_config3_1024_transfers_through_the_worker(ctx, cref):
    """BASELINE configs[3]: 1024 signed transfers at A=16, T=3, B=5 through bzk_mpn_prepare_works, then the worker (update only) on
    one 80 GB H100: accepted by bzk_mpn_work_verify and by the oracle's pairing check.  Prints wall times and free memory."""
    import torch
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn import native as N, update as U, works as Wk
    from bazuka_b200.mpn.ledger import NativeLedger
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    from oracle import groth16_c as GC
    A3, T3, B3, nacc = 16, 3, 5, 128
    gb = lambda: round(torch.cuda.mem_get_info()[0] / 1e9, 1)
    marks, free_gb = {}, {"start": gb()}
    t0 = time.time()
    nc = NativeUpdateCircuit(A3, T3, B3, blocked=True)
    br = nc.blocked_r1cs()
    nc.free()
    pk, vk = BG.setup_gpu(ctx, br, cref.fr_random(911, 5), cref.g1_generator(), cref.g2_generator(), table_levels=1)
    del br
    torch.cuda.synchronize()
    marks["setup_s"] = time.time() - t0
    free_gb["after_setup"] = gb()
    cfg = dict(C.config(A3, T3, 1, 1, B3, {"deposit": C.opaque_vk(2), "withdraw": C.opaque_vk(4), "update": bytes(BG.vk_to_bincode(vk))}),
               mpn_num_deposit_batches=0, mpn_num_withdraw_batches=0)
    t0 = time.time()
    led = NativeLedger(ctx, A3, T3)
    keys = []
    for i in range(nacc):
        pkey, sk = N.eddsa_keys(b"acct%d" % i)
        keys.append((pkey, sk))
        led.set_account(i, U.MpnAccount(0, 0, pkey, {0: U.Money(U.ZIESHA, 10 ** 12)}))
    nonces, txs = [0] * nacc, []
    for k in range(1 << (2 * B3)):
        s, d = k % nacc, (k + 1) % nacc
        nonces[s] += 1
        tx = U.MpnTransaction(nonces[s], N.jj_compress(keys[s][0]), N.jj_compress(keys[d][0]), U.Money(U.ZIESHA, 1000 + k), U.Money(U.ZIESHA, 10))
        tx.sign(keys[s][1])
        txs.append(tx)
    resp, n = C.prepare_response(ctx, led, cfg, [], [], txs, {}, {})
    led.free()
    assert n == 1
    marks["ledger_signing_prepare_s"] = time.time() - t0
    t0 = time.time()
    w = Wk.NativeMpnWorker([ctx], C.config_bytes(cfg), [{"update": pk}])
    marks["worker_create_s"] = time.time() - t0
    free_gb["after_worker_create"] = gb()
    t0 = time.time()
    body, status = w.prove_response(resp, ME)
    marks["prove_response_s"] = time.time() - t0
    free_gb["after_proof"] = gb()
    assert status == [0]
    _, proofs = C.solution_proofs(body)
    (wid, h), = C.decode_response(ctx._l, resp)
    proof = bytes(proofs[wid])
    assert ctx._l.bzk_mpn_work_verify(h, ME, proof) == 1
    pub = np.zeros((5, 4), np.uint64)
    assert ctx._l.bzk_mpn_work_public_inputs(h, ME, C._ptr(pub)) == 0
    ctx._l.bzk_mpn_work_free(h)
    assert GC.verify_py(vk, pub, _proof_points(proof))
    print({"config": "A=16 T=3 B=5", "gpu": torch.cuda.get_device_name(), **{k: round(v, 2) for k, v in marks.items()},
           "timing_ms": w.last_timing(), "free_gb": free_gb})
    w.free()
    pk.free()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def block(ctx, cref):
    """keys from setup_gpu (update over the blocked R1CS, deposit and withdraw explicit), the node's config, and the response
    bzk_mpn_prepare_works makes of a block with works of all three kinds"""
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn.native_circuit import NativeTwoPhaseCircuit, NativeUpdateCircuit
    keys, vks = {}, {}
    nc = NativeUpdateCircuit(A, T, BU, blocked=True)
    br = nc.blocked_r1cs()
    nc.free()
    keys["update"], vks["update"] = BG.setup_gpu(ctx, br, cref.fr_random(601, 5), cref.g1_generator(), cref.g2_generator(), table_levels=1)
    for i, (kind, b) in enumerate((("deposit", BD), ("withdraw", BW))):
        c = NativeTwoPhaseCircuit(kind, A, T, b)
        ni, na, mats = c.r1cs()
        c.free()
        keys[kind], vks[kind] = BG.setup_gpu(ctx, BG.R1CS(ni, na, *mats), cref.fr_random(602 + i, 5), cref.g1_generator(), cref.g2_generator(),
                                             table_levels=1)
    cfg = C.config(A, T, BD, BW, BU, {k: bytes(BG.vk_to_bincode(v)) for k, v in vks.items()})
    st, deps, wds, ups, dpay, wpay = C.block(A, T)
    led = C.ledger(ctx, st, A, T)
    resp, n = C.prepare_response(ctx, led, cfg, deps, wds, ups, dpay, wpay)
    led.free()
    assert n == 3
    yield dict(keys=keys, vks=vks, cfg_bytes=C.config_bytes(cfg), resp=resp)
    for k in keys.values():
        k.free()


def _explicit_proof(ctx, kind, pk, work_bytes, r, s):
    from bazuka_b200.mpn import works as Wk
    from bazuka_b200.mpn.native_circuit import NativeTwoPhaseCircuit, NativeUpdateCircuit
    c = NativeUpdateCircuit(A, T, BU) if kind == "update" else NativeTwoPhaseCircuit(kind, A, T, BD if kind == "deposit" else BW)
    p = Wk.NativeMpnProver(ctx)
    p.add_circuit(kind, c, pk)
    c.free()
    out = p.prove(work_bytes, ME, r, s)
    p.free()
    return out[4:]


def test_production_block_one_and_two_contexts(ctx, cref, block):
    import bazuka_b200 as Bz
    from bazuka_b200.mpn import wire as Wr, works as Wk
    from oracle import groth16_c as GC
    keys, lib = block["keys"], ctx._l
    w1 = Wk.NativeMpnWorker([ctx], block["cfg_bytes"], [keys])
    t0 = time.time()
    body1, st1 = w1.prove_response(block["resp"], ME, SEED)
    t1 = time.time() - t0
    ctx2 = Bz.Context(0)
    w2 = Wk.NativeMpnWorker([ctx, ctx2], block["cfg_bytes"], [keys, keys])
    t0 = time.time()
    body2, st2 = w2.prove_response(block["resp"], ME, SEED)
    t2 = time.time() - t0
    print({"one_context_s": round(t1, 2), "two_contexts_s": round(t2, 2), "timing_1": w1.last_timing(), "timing_2": w2.last_timing()})
    assert st1 == st2 == [0, 0, 0] and body1 == body2
    prover, proofs = C.solution_proofs(body1)
    assert prover == ME and sorted(proofs) == [0, 1, 2]
    checked_oracle = False
    for wid, h in C.decode_response(lib, block["resp"]):
        blob = C.encode_work(lib, h)
        kind = Wr.work_from_bytes(blob)["data"][0]
        proof = bytes(proofs[wid])
        r, s = C.seeded_blinding(SEED, wid)
        assert proof == _explicit_proof(ctx, kind, keys[kind], blob, r, s)          # blocked upload == explicit, same r and s
        assert lib.bzk_mpn_work_verify(h, ME, proof) == 1
        if not checked_oracle:
            pub = np.zeros((5, 4), np.uint64)
            assert lib.bzk_mpn_work_public_inputs(h, ME, C._ptr(pub)) == 0
            assert GC.verify_py(block["vks"][kind], pub, _proof_points(proof))
            checked_oracle = True
        lib.bzk_mpn_work_free(h)
    # without a seed: fresh blinding on every call, both accepted
    b_a, s_a = w2.prove_response(block["resp"], ME)
    b_b, s_b = w2.prove_response(block["resp"], ME)
    assert s_a == s_b == [0, 0, 0] and b_a != b_b
    for body in (b_a, b_b):
        _, ps = C.solution_proofs(body)
        for wid, h in C.decode_response(lib, block["resp"]):
            assert lib.bzk_mpn_work_verify(h, ME, bytes(ps[wid])) == 1
            lib.bzk_mpn_work_free(h)
    w1.free(); w2.free()
    ctx2.close()


def test_key_with_a_foreign_h_point_is_rejected_not_proved(ctx, block):
    """the deposit key with h[0] and h[1] swapped: its verifying-key points and lengths match, so creation accepts it; its proof
    fails the self-check and comes back BZK_ERR_REJECTED, left out of the solution, while the other works are proved"""
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn import works as Wk
    img = BG.write_parameters(ctx, block["keys"]["deposit"]).copy()
    info = BG.parameters_info(img)
    off_h = info["bytes"] - (20 + 96 * (info["n_h"] + info["n_l"] + info["n_a"] + info["n_b_g1"]) + 192 * info["n_b_g2"]) + 4
    h0 = img[off_h:off_h + 96].copy()
    img[off_h:off_h + 96] = img[off_h + 96:off_h + 192]
    img[off_h + 96:off_h + 192] = h0
    bad, _ = BG.read_parameters(ctx, img)
    w = Wk.NativeMpnWorker([ctx], block["cfg_bytes"], [{**block["keys"], "deposit": bad}])
    body, status = w.prove_response(block["resp"], ME, SEED)
    assert status == [-10, 0, 0]
    _, proofs = C.solution_proofs(body)
    assert sorted(proofs) == [1, 2]
    w.free()
    bad.free()
