"""Closed-form references for the NTT and the Groth16 quotient pipeline (test infrastructure, no GPU).

Each reference below is independent of the oracle's butterfly algorithm and cheap at any size, so it reaches the
2^25-2^28 domains the C oracle is too slow for.  All of them use bellman's maps (`oracle/py/ntt.py`): omega =
`omega_for(log_n)`, coset generator 7, ifft scaled by n^-1, Z = x^n - 1, which is the constant 7^n - 1 on the coset.

  impulse delta_k    fft: w^(jk)     ifft: n^-1 w^(-jk)     coset_fft: 7^k w^(jk)     icoset_fft: n^-1 7^(-j) w^(-jk)
  constant c         fft: n c delta_0     ifft, icoset_fft: c delta_0     coset_fft: c (7^n - 1) / (7 w^j - 1)
  eighth points      at j = m n/P (P = min(8, n)) w^(jk) depends on k mod P only, so output j is a combination of the
                     P strided partial sums of the input: an exact check of a random transform at any size
  quotient           h(a, b = 1, c = 0) = ifft(a) / (7^n - 1)      h(a = 0, b, c) = -ifft(c) / (7^n - 1)
                     a satisfied triple (c = a*b pointwise) has a quotient of degree <= n - 2: h[n-1] = 0

Values are Python integers; vectors handed to a kernel or to the oracle are [n, 4] uint64 Montgomery images."""
import functools
import random

import numpy as np

from oracle.py import field as Fd, ntt as N

R = Fd.R_MOD
GEN = Fd.FR_GENERATOR
OPS = ("fft", "ifft", "coset_fft", "icoset_fft")      # op codes 0..3 of bzk_ntt* and cref.ntt
GPOW_BITS = 14                                        # coset powers are read as lo[i mod 2^14] * hi[i >> 14]


def to_mont(xs):
    return np.frombuffer(Fd.fr_vec_to_mont([x % R for x in xs]), dtype=np.uint64).reshape(-1, 4).copy()


def from_mont(a):
    return Fd.fr_vec_from_mont(np.ascontiguousarray(a, dtype=np.uint64).tobytes())


def omega(log_n, inverse=False):
    w = N.omega_for(log_n)
    return pow(w, -1, R) if inverse else w


def n_inv(log_n):
    return pow(1 << log_n, -1, R)


def z_inv(log_n):
    """(7^n - 1)^-1: divide_by_z_on_coset's factor"""
    return pow(pow(GEN, 1 << log_n, R) - 1, -1, R)


# ------------------------------------------------------------------ where to look
def impulse_positions(log_n, seed):
    """k in {0, 1, 2, n/2 - 1, n/2, n - 1} and one random k (and 2^14 +- 1 where the coset power table splits)"""
    n = 1 << log_n
    ks = {0, 1, 2, n // 2 - 1, n // 2, n - 1, random.Random(seed * 1000 + log_n).randrange(n)}
    if n > 1 << GPOW_BITS:
        ks |= {(1 << GPOW_BITS) - 1, (1 << GPOW_BITS) + 1}
    return sorted(k for k in ks if 0 <= k < n)


def sample_positions(log_n, seed, n_random=2000):
    """output positions to compare: 0, 1, n-1, every 2^t and 2^t +- 1, the neighbourhood of every multiple of 2^14 up
    to 4 of them (where the coset power lookup changes from the low table alone to low * high), and n_random random j"""
    n = 1 << log_n
    js = {0, 1, n - 1}
    for t in range(log_n + 1):
        js |= {(1 << t) - 1, 1 << t, (1 << t) + 1}
    for m in range(1, 5):
        js |= set(range(m * (1 << GPOW_BITS) - 2, m * (1 << GPOW_BITS) + 3))
    rnd = random.Random(seed * 7919 + log_n)
    js |= {rnd.randrange(n) for _ in range(n_random)}
    return sorted(j for j in js if 0 <= j < n)


def eighth_points(log_n):
    """j = m n/P, m < P = min(8, n): the outputs the eighth-point reference gives exactly"""
    n = 1 << log_n
    p = min(8, n)
    return [m * (n // p) for m in range(p)]


# ------------------------------------------------------------------ closed forms at given output positions
@functools.lru_cache(maxsize=16)
def _pow_table(base, bits):
    lo = [1]
    for _ in range((1 << min(bits, 14)) - 1):
        lo.append(lo[-1] * base % R)
    step, hi = pow(base, 1 << 14, R), [1]
    for _ in range((1 << max(bits - 14, 0)) - 1):
        hi.append(hi[-1] * step % R)
    return lo, hi


def fixed_pow(base, e, bits):
    """base^e for 0 <= e < 2^bits with one product (two tables of up to 2^14 powers, built once per base): the sampled
    references evaluate thousands of powers of the same few bases"""
    assert 0 <= e < 1 << max(bits, 1)
    lo, hi = _pow_table(base % R, max(bits, 1))
    return lo[e & 0x3FFF] * hi[e >> 14] % R


def impulse_expected(log_n, op, k, js, amp=1):
    """op applied to amp * delta_k, at output positions js"""
    n = 1 << log_n
    inverse = op in (1, 3)
    w = omega(log_n, inverse)
    pre = amp * (n_inv(log_n) if inverse else 1) * (pow(GEN, k, R) if op == 2 else 1) % R
    ginv = pow(GEN, -1, R)
    out = []
    for j in js:
        v = pre * fixed_pow(w, j * k % n, log_n)
        if op == 3:
            v = v * fixed_pow(ginv, j, log_n)
        out.append(v % R)
    return out


def constant_expected(log_n, op, c, js):
    """op applied to the constant vector c, at output positions js"""
    n = 1 << log_n
    c %= R
    if op == 0:
        return [n * c % R if j == 0 else 0 for j in js]
    if op in (1, 3):
        return [c if j == 0 else 0 for j in js]
    # coset_fft: sum_i c 7^i w^(ij) = c (7^n - 1) / (7 w^j - 1); 7 w^j != 1 because 7 is not a 2^32-th root of unity
    w = omega(log_n)
    num = c * (pow(GEN, n, R) - 1) % R
    return [num * pow(GEN * fixed_pow(w, j, log_n) - 1, -1, R) % R for j in js]


# ------------------------------------------------------------------ eighth points of an arbitrary input
def powers(cref, base, count):
    """[base^i for i < count] as Montgomery images, by prefix doubling on the oracle"""
    out = to_mont([1])
    while len(out) < count:
        step = np.ascontiguousarray(np.broadcast_to(to_mont([pow(base, len(out), R)]), out.shape))
        out = np.concatenate([out, cref.fr_mul(out, step)])
    return out[:count]


def vec_sum(cref, v):
    """sum of a Montgomery vector (the image of a sum is the sum of the images)"""
    v = np.ascontiguousarray(v, dtype=np.uint64).reshape(-1, 4)
    if len(v) == 0:
        return 0
    while len(v) > 1:
        if len(v) & 1:
            v = np.concatenate([v, np.zeros((1, 4), dtype=np.uint64)])
        h = len(v) // 2
        v = cref.fr_add(v[:h], v[h:])
    return from_mont(v)[0]


def strided_sums(cref, a, p, g=1):
    """S_r = sum over i = r mod p of a_i g^i, for r < p (g = 7 forms the coset input a o 7^i on the way)"""
    a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4)
    n = len(a)
    gp = powers(cref, pow(g, p, R), n // p) if g != 1 else None
    out = []
    for r in range(p):
        col = np.ascontiguousarray(a[r::p])
        if gp is not None:
            col = cref.fr_mul(col, gp)
        out.append(vec_sum(cref, col) * pow(g, r, R) % R)
    return out


def eighth_expected(cref, a, ops=(0, 1, 2, 3)):
    """{op: op applied to the Montgomery vector a, at eighth_points(log_n)}"""
    n = len(np.asarray(a).reshape(-1, 4))
    log_n = n.bit_length() - 1
    p = min(8, n)
    sums = {g: strided_sums(cref, a, p, g) for g in {GEN if op == 2 else 1 for op in ops}}
    res = {}
    for op in ops:
        inverse = op in (1, 3)
        s = sums[GEN if op == 2 else 1]
        wp = pow(omega(log_n, inverse), n // p, R)     # a primitive p-th root of unity
        out = []
        for m, j in enumerate(eighth_points(log_n)):
            v = sum(s[r] * pow(wp, r * m, R) for r in range(p)) % R
            if inverse:
                v = v * n_inv(log_n) % R
            if op == 3:
                v = v * pow(GEN, -j, R) % R
            out.append(v)
        res[op] = out
    return res


# ------------------------------------------------------------------ the quotient pipeline
def quotient_impulse_expected(log_n, k, js, in_c=False):
    """h = coefficients of (a b - c) / Z from evaluations, with a = delta_k, b = 1, c = 0 (in_c False: ifft(a) / Z) or
    a = 0, any b, c = delta_k (in_c True: -ifft(c) / Z)"""
    zi = z_inv(log_n)
    return [(-v if in_c else v) * zi % R for v in impulse_expected(log_n, 1, k, js)]


def combine_impulse_expected(log_n, k, js):
    """h_combine on coset evaluations a = delta_k, b = 1, c = 0: icoset_fft(delta_k) / Z"""
    zi = z_inv(log_n)
    return [v * zi % R for v in impulse_expected(log_n, 3, k, js)]


def quotient_bigint(a, b, c, log_n):
    """the oracle composition in big integers: ifft, coset_fft, a b - c, divide_by_z_on_coset, icoset_fft"""
    ea, eb, ec = (N.coset_fft(N.ifft(v, log_n), log_n) for v in (a, b, c))
    h = N.divide_by_z_on_coset([(x * y - z) % R for x, y, z in zip(ea, eb, ec)], log_n)
    return N.icoset_fft(h, log_n)
