"""GPU tier, BASELINE.json configs at their FULL sizes, bit-exact against the CPU oracle:

  configs[2]  radix-2 NTT/iNTT over Fr, 2^24 coefficients: all four transforms (fft, ifft, coset fft, coset ifft)
              equal the C oracle's output limb for limb
  configs[1]+ G2 multiexp at 2^20 and witness-shaped (0/1-heavy, small-value-heavy) G1/G2 sums at 2^20 — the shapes
              `create_proof` really feeds the MSM (long single-bucket runs -> k_fixup_long / the tree rounds) —
              against the threaded C restatement of bellman's multiexp
  production  UpdateCircuit A=15,T=3,B=4 (256 signed transfers, 14.4 M constraints, 2^24 domain): circuit, ledger,
              witness and prover all native; the 387 proof bytes equal the C oracle prover's on the same key, the
              big-integer pairing check accepts and a tampered public input is rejected
              (shape of /root/reference/src/mpn/circuits/test.rs:117-149 with real transitions)
  configs[3]  UpdateCircuit A=16,T=3,B=4 (the depth-32 tree, 256 transfers, 2^24 domain): proved natively, verified by
              the oracle's pairing verifier, tampered input rejected

The two whole-batch tests cost minutes (key generation for 58 M / 70 M bases, the CPU prover on the host cores); they
print their stage times with `-s`."""
import time

import numpy as np
import pytest

from conftest import fr_ints, fr_arr

pytestmark = pytest.mark.gpu

R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001


def _t():
    import torch
    return torch


def host_u64(tensor):
    return tensor.cpu().numpy().view(np.uint64)


# ------------------------------------------------------------------ configs[2]
def test_ntt_2_24_all_ops_bit_exact_vs_oracle(ctx, cref):
    t = _t()
    log_n, n = 24, 1 << 24
    a = cref.fr_random(3, n)                       # SplitMix64 seed 3 (SURVEY.md §8d config 3)
    d = t.from_numpy(a.view(np.int64)).cuda()
    for op in range(4):
        x = d.clone()
        t.cuda.synchronize()                       # the clone runs on torch's stream, the transform on the context's
        ctx.ntt_dev(x, log_n, op)
        ctx.synchronize()
        got = host_u64(x).reshape(-1, 4)
        want = cref.ntt(a, op)
        assert (got == want).all(), op
        del x


# ------------------------------------------------------------------ MSM shapes of create_proof at 2^20
def _witness_like(cref, seed, n):
    """a Groth16 witness's scalar census (SURVEY.md §8a/§8d): ~45 % booleans, ~10 % small integers (amounts, indices,
    nonces), the rest field-uniform (hash states); plus the edge values r-1, 2^k on window boundaries."""
    rng = np.random.default_rng(seed)
    s = cref.fr_random(seed, n)
    kind = rng.random(n)
    small = np.zeros((n, 4), dtype=np.uint64)
    small[:, 0] = rng.integers(0, 1 << 40, n, dtype=np.uint64)
    bits = np.zeros((n, 4), dtype=np.uint64)
    bits[:, 0] = rng.integers(0, 2, n, dtype=np.uint64)
    canon = np.where((kind < 0.45)[:, None], bits, np.where((kind < 0.55)[:, None], small, 0)).astype(np.uint64)
    mont = cref.fr_to_mont(canon)
    out = np.where((kind < 0.55)[:, None], mont, s)
    edge = fr_arr([R - 1, 1 << 15, 1 << 16, (1 << 16) - 1, 1 << 19, 1 << 20, (1 << 20) - 1, 1 << 254, 0, 1, 2])
    out[: len(edge)] = edge
    return np.ascontiguousarray(out)


def test_msm_g2_2_20_vs_oracle(ctx, cref):
    t = _t()
    n = 1 << 20
    d_img = t.empty((n, 200), dtype=t.uint8, device="cuda")
    ctx.g2_random_bases_dev(7, n, d_img)
    ctx.synchronize()
    bases = d_img.cpu().numpy()
    rb = ctx.g2_bases_from_dev(d_img, n)
    for scalars in (cref.fr_random(8, n), _witness_like(cref, 18, n)):
        got = ctx.msm_g2_resident(rb, scalars)
        assert (got == cref.msm_g2(bases, scalars)).all()
    rb.free()


def test_msm_g1_2_20_witness_shaped_vs_oracle(ctx, cref):
    t = _t()
    n = 1 << 20
    d_img = t.empty((n, 104), dtype=t.uint8, device="cuda")
    ctx.g1_random_bases_dev(2, n, d_img)
    ctx.synchronize()
    bases = d_img.cpu().numpy()
    rb = ctx.g1_bases_from_dev(d_img, n)
    scalars = _witness_like(cref, 28, n)
    assert (ctx.msm_g1_resident(rb, scalars) == cref.msm_g1(bases, scalars)).all()
    # all ones: the whole vector lands in ONE bucket (the longest possible run)
    ones = fr_arr([1]) .repeat(n, axis=0)
    assert (ctx.msm_g1_resident(rb, ones) == cref.msm_g1(bases, ones)).all()
    rb.free()


# ------------------------------------------------------------------ whole update batches, native path
def _ledger_and_transfers(ctx, A, T, B, nacc):
    """synthetic ledger of `nacc` funded accounts at indices 0..nacc-1 and 4^B signed transfers i -> i+1 (SURVEY §8d)."""
    from bazuka_b200.mpn import native as N, update as U
    from bazuka_b200.mpn.ledger import NativeLedger, pack_txs
    ntx = 1 << (2 * B)
    led = NativeLedger(ctx, A, T)
    keys = []
    for i in range(nacc):
        pk, sk = N.eddsa_keys(b"acct%d" % i)
        keys.append((pk, sk))
        led.set_account(i, U.MpnAccount(0, 0, pk, {0: U.Money(U.ZIESHA, 10 ** 12)}))
    nonces, txs = [0] * nacc, []
    for k in range(ntx):
        s, d = k % nacc, (k + 1) % nacc
        nonces[s] += 1
        tx = U.MpnTransaction(nonces[s], N.jj_compress(keys[s][0]), N.jj_compress(keys[d][0]), U.Money(U.ZIESHA, 1000 + k), U.Money(U.ZIESHA, 10))
        tx.sign(keys[s][1])
        txs.append(tx)
    return led, pack_txs(txs)


def _native_batch_proof(ctx, cref, A, T, B, nacc, seed, with_oracle_prover):
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn import update as U
    from bazuka_b200.mpn.cs import to_mont
    from bazuka_b200.mpn.gpu_witness import UpdateWitnessGpu
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    from oracle import groth16_c as GC
    t = _t()
    marks = {}
    t0 = time.time()
    nc = NativeUpdateCircuit(A, T, B)
    ni, na, mats = nc.r1cs()
    prog, epilogues = nc.program(0), {B: nc.program(1)}
    nc.free()
    marks["compile_r1cs_s"] = time.time() - t0
    t0 = time.time()
    pr = BG.Prover(ctx, BG.R1CS(ni, na, *mats))
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, cref.fr_random(seed, 5), cref.g1_generator(), cref.g2_generator())
    marks["key_setup_s"] = time.time() - t0
    wit = UpdateWitnessGpu(ctx, A, T, prog, epilogues)
    t0 = time.time()
    led, txs = _ledger_and_transfers(ctx, A, T, B, nacc)
    marks["ledger_and_signing_s"] = time.time() - t0
    r, s = cref.fr_random(seed + 1, 2)
    t0 = time.time()
    raws, ext, accepted, pub, n_acc = led.update_build(txs, B)
    assert n_acc == 1 << (2 * B) and accepted.all()
    commitment, height = 42, 7
    d_in, d_aux = wit.witness_native(raws, ext, [commitment, height, pub["state"], U.ZIESHA, pub["aux_data"], pub["next_state"]], B)
    blob, pts = pr.prove_dev(pk, d_in, d_aux, r, s, check_satisfied=True)
    marks["build_witness_prove_s"] = time.time() - t0
    public = to_mont([commitment, height, pub["state"], pub["aux_data"], pub["next_state"]])
    assert (d_in.cpu().numpy().view(np.uint64)[1:] == public).all()
    # the product's byte-image verifier, then the oracle's big-integer pairing check (independent code)
    assert BG.verify_bytes(BG.vk_to_bincode(vk), public, blob)
    assert GC.verify_py(vk, public, pts)
    wrong = public.copy()
    wrong[4] = wrong[2]                      # claim next_state = state
    assert not GC.verify_py(vk, wrong, pts)
    assert not BG.verify_bytes(BG.vk_to_bincode(vk), wrong, blob)
    if with_oracle_prover:
        t0 = time.time()
        a_idx, b_idx = GC.density(ni, na, mats)
        cpk = {"log_m": pr.log_m, "vk": vk, "a_idx": a_idx, "b_idx": b_idx}
        for k in ("h", "l", "a", "b_g1", "b_g2"):
            cpk[k] = pk.device_images[k].cpu().numpy()
        inputs, aux = d_in.cpu().numpy().view(np.uint64), d_aux.cpu().numpy().view(np.uint64)
        want = GC.proof_bytes(*GC.prove(ni, na, mats, cpk, inputs, aux, r, s))
        marks["oracle_cpu_prove_s"] = time.time() - t0
        assert (blob == want).all()
    print({"A": A, "T": T, "B": B, "log_m": pr.log_m, "constraints": pr.r1cs.num_constraints, **{k: round(v, 1) for k, v in marks.items()}})
    log_m = pr.log_m
    wit.free(); led.free(); pk.free(); pr.free()
    del pk, pr, d_in, d_aux
    t.cuda.empty_cache()
    return log_m


def test_production_update_batch_proof_bytes_vs_oracle(ctx, cref):
    """A=15,T=3,B=4: /root/reference/src/config/blockchain.rs:22-26 (mpn_log4_tree_size 15, token tree 3, update batch 4)."""
    assert _native_batch_proof(ctx, cref, 15, 3, 4, nacc=64, seed=501, with_oracle_prover=True) == 24


def test_config3_depth32_tree_batch_proves_and_oracle_verifier_accepts(ctx, cref):
    """BASELINE configs[3]'s "Merkle depth 32" tree (A=16) at the 256-tx batch (B=4, 2^24 domain) — native prove, oracle
    pairing verification.  The 1024-tx batch (B=5, 2^26) does not fit an 80 GB H100 even without fixed-base tables: proving
    key 32.1 GB packed + 34.4 GB of wire images kept on the device + 16.9 GB of R1CS = 83 GB before the prover's working set;
    with BZK_TABLE_LEVELS=1 it runs out of memory while the key's bases are allocated."""
    assert _native_batch_proof(ctx, cref, 16, 3, 4, nacc=128, seed=601, with_oracle_prover=False) == 24
