"""CPU tier: the closed-form NTT and quotient references of tests/ntt_cases.py against the big-integer restatement of
bellman's `EvaluationDomain` (`oracle/py/ntt.py`: `dft_naive`, `fft`, `coset_fft`, `divide_by_z_on_coset`) at
log n <= 10, so that the references the GPU tier relies on at 2^11-2^28 are themselves checked."""
import random

import pytest

import ntt_cases as NC
from oracle.py import ntt as N

R = NC.R
BIGINT_OPS = (N.fft, N.ifft, N.coset_fft, N.icoset_fft)
SIZES = list(range(11))


def _at(v, js):
    return [v[j] for j in js]


def _rand(seed, n):
    rnd = random.Random(seed)
    return [rnd.randrange(R) for _ in range(n)]


@pytest.mark.parametrize("log_n", SIZES)
def test_ntt_cases_sample_positions_cover_the_edges(log_n):
    n = 1 << log_n
    js = NC.sample_positions(log_n, 1)
    assert js == sorted(set(js)) and all(0 <= j < n for j in js)
    assert {0, n - 1} <= set(js)
    for t in range(log_n):
        assert {(1 << t) - 1, 1 << t, min((1 << t) + 1, n - 1)} <= set(js)
    big = NC.sample_positions(26, 1)
    assert set(range((1 << 14) - 2, (1 << 14) + 3)) <= set(big) and len(big) > 2000
    ks = NC.impulse_positions(log_n, 1)
    assert {0, n - 1, n // 2} <= set(ks) and all(0 <= k < n for k in ks)


@pytest.mark.parametrize("log_n", SIZES)
def test_ntt_cases_impulses_match_the_bigint_transforms(log_n):
    n = 1 << log_n
    js = NC.sample_positions(log_n, 2)
    for k in NC.impulse_positions(log_n, 2):
        delta = [0] * n
        delta[k] = 5
        for op, f in enumerate(BIGINT_OPS):
            assert NC.impulse_expected(log_n, op, k, js, amp=5) == _at(f(delta, log_n), js), (log_n, op, k)


@pytest.mark.parametrize("log_n", range(7))
def test_ntt_cases_impulses_match_the_definition(log_n):
    """fft against the O(n^2) definition, not only against serial_fft"""
    n = 1 << log_n
    for k in NC.impulse_positions(log_n, 3):
        delta = [0] * n
        delta[k] = 1
        assert NC.impulse_expected(log_n, 0, k, range(n)) == N.dft_naive(delta, log_n)


@pytest.mark.parametrize("log_n", SIZES)
def test_ntt_cases_constants_match_the_bigint_transforms(log_n):
    n = 1 << log_n
    js = list(range(n))
    for c in (1, R - 1, _rand(log_n, 1)[0]):
        for op, f in enumerate(BIGINT_OPS):
            assert NC.constant_expected(log_n, op, c, js) == f([c] * n, log_n), (log_n, op, c)


@pytest.mark.parametrize("log_n", SIZES)
def test_ntt_cases_eighth_points_of_random_inputs(cref, log_n):
    n = 1 << log_n
    a = _rand(100 + log_n, n)
    am = NC.to_mont(a)
    js = NC.eighth_points(log_n)
    assert len(js) == min(8, n)
    want = NC.eighth_expected(cref, am)
    for op, f in enumerate(BIGINT_OPS):
        assert want[op] == _at(f(a, log_n), js), (log_n, op)


def test_ntt_cases_powers_and_sums(cref):
    rnd = random.Random(6)
    for bits in (0, 1, 10, 14, 15, 26, 28):
        base = rnd.randrange(R)
        es = {0, (1 << bits) - 1, (1 << 14) - 1, 1 << 14, (1 << 14) + 1} | {rnd.randrange(1 << bits) for _ in range(200)}
        for e in sorted(x for x in es if x < 1 << max(bits, 1)):
            assert NC.fixed_pow(base, e, bits) == pow(base, e, R), (bits, e)
    for count in (1, 2, 3, 7, 8, 1000):
        assert NC.from_mont(NC.powers(cref, 7, count)) == [pow(7, i, R) for i in range(count)]
    v = _rand(5, 1001)
    assert NC.vec_sum(cref, NC.to_mont(v)) == sum(v) % R
    assert NC.strided_sums(cref, NC.to_mont(v[:1000]), 8, 7) == \
        [sum(x * pow(7, i, R) for i, x in enumerate(v[:1000]) if i % 8 == r) % R for r in range(8)]


@pytest.mark.parametrize("log_n", SIZES)
def test_ntt_cases_quotient_closed_forms(log_n):
    n = 1 << log_n
    js = NC.sample_positions(log_n, 4)
    ones, zeros = [1] * n, [0] * n
    b = _rand(200 + log_n, n)
    for k in NC.impulse_positions(log_n, 4)[:4]:
        delta = [0] * n
        delta[k] = 1
        assert NC.quotient_impulse_expected(log_n, k, js) == _at(NC.quotient_bigint(delta, ones, zeros, log_n), js)
        assert NC.quotient_impulse_expected(log_n, k, js, in_c=True) == _at(NC.quotient_bigint(zeros, b, delta, log_n), js)
        # the second half alone: delta_k taken as coset evaluations
        h = N.icoset_fft(N.divide_by_z_on_coset(delta, log_n), log_n)
        assert NC.combine_impulse_expected(log_n, k, js) == _at(h, js)


@pytest.mark.parametrize("log_n", SIZES)
def test_ntt_cases_satisfied_triple_has_top_coefficient_zero(log_n):
    n = 1 << log_n
    a, b = _rand(300 + log_n, n), _rand(400 + log_n, n)
    c = [x * y % R for x, y in zip(a, b)]
    h = NC.quotient_bigint(a, b, c, log_n)
    assert h[n - 1] == 0
    if n >= 2:  # and it is only the top one: an unsatisfied triple does not have it
        c[0] = (c[0] + 1) % R
        assert NC.quotient_bigint(a, b, c, log_n)[n - 1] != 0
