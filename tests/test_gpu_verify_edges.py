"""GPU tier: bzk_groth16_verify_batch_dev (k_verify_miller, one thread per proof) against the host entry points on
adversarial batches of GPU-made proofs: batch sizes around the 64-thread block, 0 / 1 / 5 / 40 public inputs, seeds whose
multipliers reach bit 126 (and bit 127 of the draw the >> 1 drops) or have a zero high half, and every tamper family of
tests/verify_cases.py at indices 0, 63, 64 and m - 1.  The kernel decides the batch verdict alone, so every verdict is
also taken with a null ok_each; with ok_each the per-proof verdicts come from the host re-check and must mark exactly
the tampered indices.  Also the cheap argument refusals, which launch nothing."""
import functools

import numpy as np
import pytest

import verify_cases as V
from conftest import fr_arr
from test_groth16_cpu import to_csr

pytestmark = pytest.mark.gpu

BAD_ARG = -1


@functools.lru_cache(maxsize=None)
def _synth_pool(ctx_id, ctx):
    """the synthetic MPN-like circuit (one public input): key from the GPU setup, 8 GPU proofs of its instance"""
    from bazuka_b200 import groth16 as BG, synth
    from oracle import cref, groth16_c as GC
    ni, na, mats, inputs, aux = synth.build(4, 6, seed=3, ops=GC.CpuOps)
    pr = BG.Prover(ctx, BG.R1CS(ni, na, *mats))
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, cref.fr_random(31, 5), cref.g1_generator(), cref.g2_generator())
    rs = cref.fr_random(33, 16)
    proofs = np.stack([pr.prove(pk, inputs, aux, rs[2 * j], rs[2 * j + 1], check_satisfied=(j == 0))[0] for j in range(8)])
    pk.free(); pr.free()
    pubs = np.repeat(inputs[1:][None], 8, axis=0)
    return vk, pubs, proofs


@functools.lru_cache(maxsize=None)
def _input_pool(ctx_id, ctx, n):
    """the n-input circuit of verify_cases: key from the C oracle's setup, 4 GPU proofs of distinct statements"""
    from bazuka_b200 import groth16 as BG
    from oracle import cref, groth16_c as GC
    cs, wit = V.input_circuit(n)
    mats = to_csr(cs)
    cpk = GC.setup(cs.num_inputs, cs.num_aux, mats, cref.fr_random(70 + n, 5))
    pr = BG.Prover(ctx, BG.R1CS(cs.num_inputs, cs.num_aux, *mats))
    pk = BG.proving_key_from_host(ctx, cpk["vk"], cpk["h"], cpk["l"], cpk["a"], cpk["b_g1"], cpk["b_g2"])
    pubs, proofs = [], []
    for j in range(4):
        zz = fr_arr(wit([(5 * j + 11 * i + 1) for i in range(n)], j + 3))
        r, s = cref.fr_random(80 + 7 * n + j, 2)
        proofs.append(pr.prove(pk, zz[:n + 1], zz[n + 1:], r, s)[0])
        pubs.append(zz[1:n + 1].reshape(n, 4))
    pk.free(); pr.free()
    return cpk["vk"], np.stack(pubs), np.stack(proofs)


def _tile(pubs, proofs, m):
    idx = np.arange(m) % len(proofs)
    return np.ascontiguousarray(pubs[idx]), np.ascontiguousarray(proofs[idx])


def _agree(ctx, e, pubs, proofs, seed, want_bad, threads):
    """every batch path gives the expected verdict; ok_each marks exactly want_bad"""
    m = len(proofs)
    want = [int(j not in want_bad) for j in range(m)]
    st, ok = e.batch_dev(ctx, pubs, proofs, seed)
    assert st == int(not want_bad) and ok.tolist() == want, ("dev", sorted(want_bad), np.nonzero(ok == 0)[0][:8])
    assert e.batch_dev(ctx, pubs, proofs, seed, each=False)[0] == int(not want_bad), "dev, null ok_each"
    for t in threads:
        st, ok = e.batch(pubs, proofs, seed, t)
        assert st == int(not want_bad) and ok.tolist() == want, ("host", t)


def test_gpu_verify_batch_sizes_and_seeds(ctx):
    """m around the 64-thread block and 1000: all-valid accepted, one bad proof at m - 1 located, with multipliers that
    reach bit 126, a draw with bit 63 (bit 127 before the >> 1) and a multiplier below 2^64"""
    from oracle import groth16_c as GC
    vk, pubs0, proofs0 = _synth_pool(id(ctx), ctx)
    assert GC.verify_py(vk, pubs0[0], V.Entry._split(proofs0[0]))
    e = V.Entry(vk)
    try:
        for m in (1, 2, 63, 64, 65, 127, 129, 1000):
            pubs, proofs = _tile(pubs0, proofs0, m)
            seeds = [V.seed_with_bit(126, m), V.seed_with_draw_top_bit(m, start=1000), V.seed_with_high_half_zero(m - 1)]
            assert any(r >> 126 for r in V.multipliers(seeds[0], m))
            assert V.multipliers(seeds[2], m)[m - 1] < 1 << 64
            for seed in seeds:
                _agree(ctx, e, pubs, proofs, seed, set(), threads=(0,) if m > 129 else (1, 0))
            bad = proofs.copy()
            bad[m - 1, 290:387] = np.frombuffer(V.PC.g1_wire(V.C.neg(V.C.FP, V._g1(proofs[m - 1, 290:387]))), dtype=np.uint8)
            _agree(ctx, e, pubs, bad, seeds[1], {m - 1}, threads=(0,) if m > 129 else (3, m))
    finally:
        e.free()


def test_gpu_verify_tamper_families(ctx):
    """every tamper family at indices 0, 63, 64 and 128 of an otherwise valid batch of 129 under the synthetic key: the
    kernel's verdict (null ok_each) at every index, ok_each from the device path and from the host batch at threads 1, 2,
    3 or m at one index per family, rotating, and the single-proof entry points"""
    vk, pubs0, proofs0 = _synth_pool(id(ctx), ctx)
    m = 129
    pubs, proofs = _tile(pubs0, proofs0, m)
    e = V.Entry(vk)
    seed = V.seed_with_bit(126, m)
    try:
        for k, (name, bad, swap) in enumerate(V.tampers(proofs0[1], proofs0[2])):
            if swap:      # one statement only: a swap of inputs is the identity here (the n-input test covers it)
                continue
            want_ok = int(name in V.ACCEPTED)
            for i, at in enumerate((0, 63, 64, m - 1)):
                P = proofs.copy()
                P[at] = bad
                assert e.batch_dev(ctx, pubs, P, seed + at, each=False)[0] == want_ok, (name, at)
                if i != k % 4:
                    continue
                want = [1] * m
                want[at] = want_ok
                st, ok = e.batch_dev(ctx, pubs, P, seed + at)
                assert st == want_ok and ok.tolist() == want, (name, at, "dev")
                t = (1, 2, 3, m)[(k // 4) % 4]
                st, ok = e.batch(pubs, P, seed + at, t, each=t != 1)
                assert st == want_ok and (t == 1 or ok.tolist() == want), (name, at, t)
            got = (e.prepared(pubs[0], bad), e.bytes_(pubs[0], bad), e.plain(pubs[0], bad))
            assert got == (want_ok,) * 3, (name, got)
    finally:
        e.free()


@pytest.mark.parametrize("n", [0, 5, 40])
def test_gpu_verify_public_input_counts(ctx, n):
    """keys with 0, 5 and 40 public inputs: valid batches of 65 accepted, and a family sample (inputs swapped, a
    negated A, a flag byte of 2, a non-canonical coordinate, a 3-torsion addend) at indices 0 and 64"""
    vk, pubs0, proofs0 = _input_pool(id(ctx), ctx, n)
    m = 65
    pubs, proofs = _tile(pubs0, proofs0, m)
    e = V.Entry(vk)
    seed = V.seed_with_bit(126, m)
    try:
        for j in range(4):
            assert (e.prepared(pubs0[j], proofs0[j]), e.bytes_(pubs0[j], proofs0[j]), e.plain(pubs0[j], proofs0[j])) == (1, 1, 1)
        _agree(ctx, e, pubs, proofs, seed, set(), threads=(1, 2, 3, m))
        keep = ("inputs swapped", "A negated", "B flag 0x2, coordinates nonzero", "C.y re-encoded as x + p", "A off the subgroup: A + 3-torsion")
        fams = [f for f in V.tampers(proofs0[1], proofs0[2]) if f[0] in keep]
        assert len(fams) == 5
        for name, bad, swap in fams:
            if swap and n == 0:
                continue
            for at in (0, 64):
                P, Q = proofs.copy(), pubs.copy()
                if swap:
                    other = at + 1 if at + 1 < m else at - 1     # a different statement (the pool cycles through 4)
                    Q[[at, other]] = Q[[other, at]]
                    want_bad = {at, other}
                else:
                    P[at], Q[at] = bad, pubs0[1]
                    want_bad = set() if name in V.ACCEPTED else {at}
                _agree(ctx, e, Q, P, seed, want_bad, threads=(2, 0))
    finally:
        e.free()


def test_gpu_verify_batch_dev_refusals(ctx):
    """m = 0 verifies; m >= 2^24, a null key and an n_inputs that does not match the key are BZK_ERR_BAD_ARG; none of
    them launches a kernel"""
    vk, pubs0, proofs0 = _synth_pool(id(ctx), ctx)
    e = V.Entry(vk)
    lib = e.lib
    try:
        pu, pp = np.ascontiguousarray(pubs0), np.ascontiguousarray(proofs0)
        n0 = ctx.launch_count
        assert lib.bzk_groth16_verify_batch_dev(ctx._h, e.pvk._h, V._ptr(pu), 1, V._ptr(pp), 0, 1, None) == 1
        big = 1 << 24
        huge_p = np.zeros(387 * big, np.uint8)           # the sizes a caller would pass; never read
        huge_i = np.zeros((big, 1, 4), np.uint64)
        assert lib.bzk_groth16_verify_batch_dev(ctx._h, e.pvk._h, V._ptr(huge_i), 1, V._ptr(huge_p), big, 1, None) == BAD_ARG
        del huge_p, huge_i
        assert lib.bzk_groth16_verify_batch_dev(ctx._h, None, V._ptr(pu), 1, V._ptr(pp), 8, 1, None) == BAD_ARG
        assert lib.bzk_groth16_verify_batch_dev(ctx._h, e.pvk._h, V._ptr(pu), 2, V._ptr(pp), 4, 1, None) == BAD_ARG
        assert lib.bzk_groth16_verify_batch_dev(ctx._h, e.pvk._h, None, 0, V._ptr(pp), 8, 1, None) == BAD_ARG
        assert ctx.launch_count == n0
    finally:
        e.free()
