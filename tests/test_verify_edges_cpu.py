"""CPU tier: the host verifier entry points (bzk_groth16_verify, _verify_prepared, _verify_bytes, _verify_batch at several
thread counts) on adversarial proof encodings, with proofs made by the C oracle on circuits with 0, 1 and 5 public inputs;
the prepared-key cache of the plain entry points under evictions; the cheap argument refusals; and the SplitMix64
multiplier restatement the GPU tier chooses its seeds with.  The GPU tier runs the same families through
bzk_groth16_verify_batch_dev."""
import functools

import numpy as np
import pytest

import verify_cases as V
from conftest import fr_arr
from oracle import groth16_c as GC
from test_groth16_cpu import to_csr

BAD_ARG = -1


@functools.lru_cache(maxsize=None)
def _setup(n, tox_seed, count):
    """key and `count` valid proofs of distinct statements for the n-input circuit (C oracle)"""
    from oracle import cref
    cs, wit = V.input_circuit(n)
    mats = to_csr(cs)
    pk = GC.setup(cs.num_inputs, cs.num_aux, mats, cref.fr_random(tox_seed, 5))
    pubs, proofs = [], []
    for j in range(count):
        z = wit([(7 * j + 3 * i + 2) for i in range(n)], j + 2)
        assert cs.is_satisfied(z)
        zz = fr_arr(z)
        r, s = cref.fr_random(1000 + 17 * tox_seed + j, 2)
        proofs.append(GC.proof_bytes(*GC.prove(cs.num_inputs, cs.num_aux, mats, pk, zz[:n + 1], zz[n + 1:], r, s)))
        pubs.append(zz[1:n + 1].reshape(n, 4))
    return pk["vk"], np.stack(pubs), np.stack(proofs)


def test_multiplier_restatement_and_chosen_seeds():
    """the Python SplitMix64 is the C one (spot values), and the chosen seeds reach what they are chosen for"""
    assert V.splitmix_at(0, 0) == 0xE220A8397B1DCDAF          # SplitMix64's first output from state 0
    for z in (0, 1, 0xDEADBEEF, V.M64):
        assert V._mix(V._unmix(z)) == z
    s = V.seed_with_high_half_zero(5)
    r = V.multipliers(s, 8)
    assert r[5] < 1 << 64 and r[5] > 1 << 32
    s126 = V.seed_with_bit(126, 4)
    assert any(x >> 126 for x in V.multipliers(s126, 4))
    assert all(x < 1 << 127 for x in V.multipliers(s126, 64))


@pytest.mark.parametrize("n", [0, 1, 5])
def test_host_entry_points_on_adversarial_proofs(n):
    """every tamper family at the first and the last index of an otherwise valid batch of 4: the batch is refused at
    every thread count, ok_each marks exactly the tampered indices, and the three single-proof entry points refuse them
    (a 3-torsion addend is accepted by all of them alike)"""
    vk, pubs, proofs = _setup(n, 40 + n, 4)
    m = len(proofs)
    e = V.Entry(vk)
    seed = V.seed_with_bit(126, m)
    try:
        for j in range(m):
            assert (e.plain(pubs[j], proofs[j]), e.prepared(pubs[j], proofs[j]), e.bytes_(pubs[j], proofs[j])) == (1, 1, 1)
        for t in (1, 2, 3, m):
            st, ok = e.batch(pubs, proofs, seed, t)
            assert st == 1 and ok.tolist() == [1] * m
            assert e.batch(pubs, proofs, seed, t, each=False)[0] == 1
        seen = set()
        for k, (name, bad, swap) in enumerate(V.tampers(proofs[1], proofs[2])):
            if swap and n == 0:
                continue
            accepted = name in V.ACCEPTED
            for at in (0, m - 1):
                P, Q = proofs.copy(), pubs.copy()
                other = 1 if at == 0 else 0
                if swap:
                    Q[[at, other]] = Q[[other, at]]
                    want_bad = {at, other}
                else:
                    P[at], Q[at] = bad, pubs[1]
                    want_bad = set() if accepted else {at}
                want = [int(j not in want_bad) for j in range(m)]
                t_each = (1, 2, 3, m)[(k + at) % 4]
                st, ok = e.batch(Q, P, seed + at, t_each)
                assert st == int(not want_bad) and ok.tolist() == want, (name, at, t_each, ok)
                for t in (1, 3):
                    assert e.batch(Q, P, seed + at, t, each=False)[0] == int(not want_bad), (name, at, t)
                for j in sorted(want_bad) or [at]:
                    got = (e.plain(Q[j], P[j]), e.prepared(Q[j], P[j]), e.bytes_(Q[j], P[j]))
                    assert got == (want[j],) * 3, (name, at, j, got)
            seen.add(name)
        assert len(seen) >= (50 if n else 49) and set(V.ACCEPTED) <= seen
    finally:
        e.free()


def test_oracle_agrees_on_decodable_tampers():
    """GC.verify_py (the big-integer pairing) on a sample of the tampered proofs it can decode: refused, like every entry
    point; the untampered proof accepted"""
    vk, pubs, proofs = _setup(1, 41, 6)
    e = V.Entry(vk)
    try:
        assert GC.verify_py(vk, pubs[1], V.Entry._split(proofs[1]))
        sample = [f for f in V.tampers(proofs[1], proofs[2]) if f[0] in ("A other", "B negated", "C doubled", "A identity, coordinates zero")]
        assert len(sample) == 4
        for name, bad, _ in sample:
            assert not GC.verify_py(vk, pubs[1], V.Entry._split(bad)), name
            assert e.prepared(pubs[1], bad) == 0, name
    finally:
        e.free()


def test_non_canonical_coordinates_are_refused():
    """the same point under a second byte string (a coordinate's limb image x + p, still below 2^384) is refused by every
    host entry point, alone and in a batch; without the canonical check the curve equation holds and the proof verifies"""
    vk, pubs, proofs = _setup(1, 41, 6)
    e = V.Entry(vk)
    try:
        for name, at in V.PC.COORDS.items():
            t = proofs[2].copy()
            v = int.from_bytes(t[at:at + 48].tobytes(), "little")
            assert v + V.P < 1 << 384
            t[at:at + 48] = np.frombuffer((v + V.P).to_bytes(48, "little"), dtype=np.uint8)
            assert (e.plain(pubs[2], t), e.prepared(pubs[2], t), e.bytes_(pubs[2], t)) == (0, 0, 0), name
            P = proofs.copy()
            P[2] = t
            st, ok = e.batch(pubs, P, 99, 2)
            assert st == 0 and ok.tolist() == [1, 1, 0, 1, 1, 1], name
    finally:
        e.free()


def test_plain_entry_key_cache_under_evictions():
    """bzk_groth16_verify_bytes / bzk_groth16_verify keep the 8 most recently used prepared keys: ten keys visited in an
    order that evicts and re-parses each of them several times, with hits in between; every verdict is the one a fresh
    key gives (own proof accepted, the next key's proof refused)"""
    keys = [_setup(1, 60 + k, 1) for k in range(10)]
    entries = [V.Entry(vk) for vk, _, _ in keys]
    order = list(range(10)) + list(range(10)) + [9, 8, 7, 6, 5, 4, 3, 2] + [0, 9, 1, 8, 2, 7] + list(range(10))[::-1]
    try:
        for k in order:
            e, (_, pub, proof) = entries[k], keys[k]
            _, pub2, proof2 = keys[(k + 1) % 10]
            assert e.bytes_(pub[0], proof[0]) == 1, k
            assert e.bytes_(pub2[0], proof2[0]) == 0, k
            assert e.plain(pub[0], proof[0]) == 1, k
            assert e.plain(pub2[0], proof2[0]) == 0, k
        # a malformed key image is refused, and refusing it does not disturb the cached keys
        short = entries[0].blob[:-1].copy()
        assert entries[0].bytes_(keys[0][1][0], keys[0][2][0], blob=short) == BAD_ARG
        assert entries[0].bytes_(keys[0][1][0], keys[0][2][0]) == 1
    finally:
        for e in entries:
            e.free()


def test_host_batch_refusals():
    """m = 0 verifies; a null key or an n_inputs that does not match the key is BZK_ERR_BAD_ARG"""
    import ctypes as ct
    vk, pubs, proofs = _setup(1, 41, 6)
    e = V.Entry(vk)
    try:
        assert e.batch(pubs[:0], proofs[:0], 1, 1) == (1, pytest.approx(np.zeros(0)))
        lib = e.lib
        pp = np.ascontiguousarray(proofs)
        pu = np.ascontiguousarray(pubs)
        assert lib.bzk_groth16_verify_batch(None, V._ptr(pu), 1, V._ptr(pp), 6, 1, 1, None) == BAD_ARG
        assert lib.bzk_groth16_verify_batch(e.pvk._h, V._ptr(pu), 2, V._ptr(pp), 3, 1, 1, None) == BAD_ARG
        assert lib.bzk_groth16_verify_batch(e.pvk._h, None, 0, V._ptr(pp), 6, 1, 1, None) == BAD_ARG
        assert e.prepared(np.zeros((0, 4), np.uint64), proofs[0]) == BAD_ARG
        assert e.bytes_(np.zeros((2, 4), np.uint64), proofs[0]) == BAD_ARG
    finally:
        e.free()
