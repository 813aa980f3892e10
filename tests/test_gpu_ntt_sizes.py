"""GPU tier: the NTT (`csrc/ntt.cu`) and the Groth16 quotient pipeline at every domain size.

  sweep          all four transforms at log n = 0..23, limb for limb against the C oracle, through bzk_ntt_dev and the
                 host entry bzk_ntt (2^24 is test_gpu_baseline_configs' all-ops check)
  closed forms   log n = 0..26: impulses, constants, eighth points of random inputs and the quotient closed forms of
                 tests/ntt_cases.py (log n >= 25 on a private context, whose tables go when it is closed); log n = 27
                 and 28 (the largest accepted) impulses only, when the card has room for them
  quotient       bzk_groth16_h_dev, bzk_groth16_h_combine_dev and bzk_divide_by_z_on_coset_dev at log n = 0..22 against
                 the oracle composition ifft -> coset_fft -> a*b - c -> divide_by_z_on_coset -> icoset_fft
  guard bands    every op and entry writes only its own n elements
  table cache    interleaved sizes on one context equal fresh contexts and the oracle
  refusals       bad sizes, ops and null pointers return BZK_ERR_BAD_ARG and launch nothing

`-s` prints the sizes each family covered."""
import contextlib
import ctypes as ct
import time

import numpy as np
import pytest

import ntt_cases as NC

pytestmark = pytest.mark.gpu

BAD_ARG = -1
GUARD = 256
PRIVATE_FROM = 25                 # domains whose twiddle tables (2 x n/2 Fr) would otherwise stay in the session context
R = NC.R


def _t():
    import torch
    return torch


def dev(arr):
    return _t().from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).view(np.int64)).cuda()


def host(d):
    return d.cpu().numpy().view(np.uint64).reshape(-1, 4)


def _ptr(d):
    return ct.c_void_p(d.data_ptr())


def _uploaded():
    _t().cuda.synchronize()       # torch's copies and fills run on torch's stream, the kernels on the context's


@pytest.fixture(scope="module")
def covered():
    cov = {}
    t0 = time.time()
    yield cov
    print(f"\nNTT families and the log n each covered ({time.time() - t0:.0f} s):")
    for fam, sizes in cov.items():
        print(f"  {fam:<34} {sorted(sizes)}")


def _mark(cov, family, log_n):
    cov.setdefault(family, set()).add(log_n)


@contextlib.contextmanager
def _ctx_for(ctx, log_n):
    if log_n < PRIVATE_FROM:
        yield ctx
        return
    import bazuka_b200 as B
    c = B.Context(0, load_poseidon=False)
    try:
        yield c
    finally:
        c.close()
        _t().cuda.empty_cache()


def _h_combine(ctx, a, b, c, log_n):
    ctx._check(ctx._l.bzk_groth16_h_combine_dev(ctx._h, _ptr(a), _ptr(b), _ptr(c), log_n))


def _ntt(ctx, a, log_n, op):
    d = dev(a)
    _uploaded()
    ctx.ntt_dev(d, log_n, op)
    ctx.synchronize()
    return host(d)


# ------------------------------------------------------------------ refusals
def test_ntt_entry_points_refuse_bad_arguments(ctx):
    t = _t()
    l, h = ctx._l, ctx._h
    d = t.zeros((16, 4), dtype=t.int64, device="cuda")
    p = _ptr(d)
    hb = np.zeros((16, 4), dtype=np.uint64)
    hp = hb.ctypes.data_as(ct.c_void_p)
    calls = {
        "ntt_dev log n 29": lambda: l.bzk_ntt_dev(h, p, 29, 0),
        "ntt log n 29": lambda: l.bzk_ntt(h, hp, 29, 0),
        "divide_by_z log n 29": lambda: l.bzk_divide_by_z_on_coset_dev(h, p, 29),
        "groth16_h log n 29": lambda: l.bzk_groth16_h_dev(h, p, p, p, 29),
        "h_combine log n 29": lambda: l.bzk_groth16_h_combine_dev(h, p, p, p, 29),
        "ntt_dev null": lambda: l.bzk_ntt_dev(h, None, 4, 0),
        "ntt null": lambda: l.bzk_ntt(h, None, 4, 0),
        "divide_by_z null": lambda: l.bzk_divide_by_z_on_coset_dev(h, None, 4),
    }
    for op in (-1, 4):
        calls[f"ntt_dev op {op}"] = lambda op=op: l.bzk_ntt_dev(h, p, 4, op)
        calls[f"ntt op {op}"] = lambda op=op: l.bzk_ntt(h, hp, 4, op)
    for name in ("groth16_h", "groth16_h_combine"):
        f = getattr(l, f"bzk_{name}_dev")
        for k in range(3):
            args = [p, p, p]
            args[k] = None
            calls[f"{name} null #{k}"] = lambda f=f, args=args: f(h, *args, 4)
    t.cuda.synchronize()
    before = ctx.launch_count
    for name, call in calls.items():
        assert call() == BAD_ARG, name
    assert ctx.launch_count == before
    assert (hb == 0).all() and (host(d) == 0).all()


# ------------------------------------------------------------------ guard bands
@pytest.mark.parametrize("log_n", [0, 1, 2, 3, 4, 12, 20])
def test_ntt_and_quotient_write_only_their_own_elements(ctx, cref, covered, log_n):
    """each vector sits between two 256-element bands of random values; every entry must leave the bands unchanged"""
    t = _t()
    n = 1 << log_n
    seed = [9000 + 16 * log_n]

    def guarded():
        seed[0] += 1
        full = dev(cref.fr_random(seed[0], n + 2 * GUARD))
        return full, full[GUARD:GUARD + n], full.clone()

    def check(what, *bufs):
        ctx.synchronize()
        for k, (full, _, before) in enumerate(bufs):
            assert t.equal(full[:GUARD], before[:GUARD]), (what, k, "before")
            assert t.equal(full[GUARD + n:], before[GUARD + n:]), (what, k, "after")

    for op in range(4):
        g = guarded()
        want = cref.ntt(host(g[1]), op)
        _uploaded()
        ctx.ntt_dev(g[1], log_n, op)
        check(f"op {op}", g)
        assert (host(g[1]) == want).all(), op
    g = guarded()
    _uploaded()
    ctx.divide_by_z_on_coset_dev(g[1], log_n)
    check("divide_by_z", g)
    for name in ("groth16_h", "h_combine"):
        gs = [guarded() for _ in range(3)]
        _uploaded()
        if name == "groth16_h":
            ctx.groth16_h_dev(gs[0][1], gs[1][1], gs[2][1], log_n)
        else:
            _h_combine(ctx, gs[0][1], gs[1][1], gs[2][1], log_n)
        check(name, *gs)
    _mark(covered, "guard bands", log_n)


# ------------------------------------------------------------------ quotient pipeline vs the oracle composition
@pytest.mark.parametrize("log_n", range(23))
def test_groth16_quotient_pipeline_vs_oracle(ctx, cref, covered, log_n):
    n = 1 << log_n
    a, b, c = (cref.fr_random(500 + 3 * log_n + s, n) for s in range(3))
    ea, eb, ec = (cref.ntt(cref.ntt(v, 1), 2) for v in (a, b, c))

    def oracle_h(ea, eb, ec):
        return cref.ntt(cref.divide_by_z_on_coset(cref.fr_sub(cref.fr_mul(ea, eb), ec)), 3)

    def gpu(entry, a, b, c):
        bufs = [dev(v) for v in (a, b, c)]
        _uploaded()
        if entry == "h":
            ctx.groth16_h_dev(*bufs, log_n)
        else:
            _h_combine(ctx, *bufs, log_n)
        ctx.synchronize()
        return [host(x) for x in bufs]

    # random triple: h, and b, c left on the coset by groth16_to_coset
    h, cb, cc = gpu("h", a, b, c)
    assert (h == oracle_h(ea, eb, ec)).all()
    assert (cb == eb).all() and (cc == ec).all()
    # satisfied triple c = a o b: the quotient has degree <= n - 2
    s = cref.fr_mul(a, b)
    want = oracle_h(ea, eb, cref.ntt(cref.ntt(s, 1), 2))
    assert (want[n - 1] == 0).all()
    assert (gpu("h", a, b, s)[0] == want).all()
    # the second half alone, on random vectors taken as coset evaluations
    assert (gpu("combine", a, b, c)[0] == oracle_h(a, b, c)).all()
    # divide_by_z_on_coset alone
    d = dev(a)
    _uploaded()
    ctx.divide_by_z_on_coset_dev(d, log_n)
    ctx.synchronize()
    assert (host(d) == cref.divide_by_z_on_coset(a)).all()
    for fam in ("groth16_h vs oracle", "h_combine vs oracle", "divide_by_z vs oracle"):
        _mark(covered, fam, log_n)


# ------------------------------------------------------------------ sweep vs the oracle
@pytest.mark.parametrize("log_n", range(24))
def test_ntt_all_ops_vs_oracle(ctx, cref, covered, log_n):
    n = 1 << log_n
    a = cref.fr_random(800 + log_n, n)
    a[0] = NC.to_mont([R - 1])[0]
    for op in range(4):
        want = cref.ntt(a, op)
        assert (_ntt(ctx, a, log_n, op) == want).all(), ("ntt_dev", op)
        assert (ctx.ntt(a, op) == want).all(), ("ntt", op)
    _mark(covered, "all ops vs oracle (dev + host)", log_n)


# ------------------------------------------------------------------ closed forms
def _impulses(ctx, log_n, seed):
    """every op on delta_k at the sampled positions"""
    t = _t()
    n = 1 << log_n
    js = NC.sample_positions(log_n, seed)
    jt = t.tensor(js, dtype=t.int64, device="cuda")
    buf = t.empty((n, 4), dtype=t.int64, device="cuda")
    for k in NC.impulse_positions(log_n, seed):
        for op in range(4):
            buf.zero_()
            buf[k] = dev(NC.to_mont([1]))[0]
            _uploaded()
            ctx.ntt_dev(buf, log_n, op)
            ctx.synchronize()
            assert NC.from_mont(host(buf[jt])) == NC.impulse_expected(log_n, op, k, js), (log_n, op, k)


def _closed_forms(ctx, cref, covered, log_n):
    t = _t()
    n = 1 << log_n
    seed = 11
    js = NC.sample_positions(log_n, seed)
    jt = t.tensor(js, dtype=t.int64, device="cuda")
    ks = NC.impulse_positions(log_n, seed)

    def read(x, idx=jt):
        ctx.synchronize()
        return NC.from_mont(host(x[idx]))

    def filled(v):
        x = t.empty((n, 4), dtype=t.int64, device="cuda")
        x.copy_(dev(NC.to_mont([v])).expand(n, 4))
        return x

    def impulse(k):
        x = t.zeros((n, 4), dtype=t.int64, device="cuda")
        x[k] = dev(NC.to_mont([1]))[0]
        return x

    _impulses(ctx, log_n, seed)
    _mark(covered, "impulses", log_n)

    for cval in (R - 1, pow(3, 100, R)):
        for op in range(4):
            x = filled(cval)
            _uploaded()
            ctx.ntt_dev(x, log_n, op)
            assert read(x) == NC.constant_expected(log_n, op, cval, js), (op, cval)
    _mark(covered, "constants, all (r-1)", log_n)

    rnd = t.empty((n, 4), dtype=t.int64, device="cuda")
    ctx.fr_random_dev(600 + log_n, n, rnd)
    ctx.synchronize()
    want = NC.eighth_expected(cref, host(rnd))
    pts = t.tensor(NC.eighth_points(log_n), dtype=t.int64, device="cuda")
    for op in range(4):
        x = rnd.clone()
        _uploaded()
        ctx.ntt_dev(x, log_n, op)
        assert read(x, pts) == want[op], op
        del x
    _mark(covered, "eighth points of random inputs", log_n)

    for k in ks:
        a, b, c = impulse(k), filled(1), t.zeros((n, 4), dtype=t.int64, device="cuda")
        _uploaded()
        ctx.groth16_h_dev(a, b, c, log_n)
        assert read(a) == NC.quotient_impulse_expected(log_n, k, js), ("h, a = delta", k)
        a, b, c = t.zeros((n, 4), dtype=t.int64, device="cuda"), rnd.clone(), impulse(k)
        _uploaded()
        ctx.groth16_h_dev(a, b, c, log_n)
        assert read(a) == NC.quotient_impulse_expected(log_n, k, js, in_c=True), ("h, c = delta", k)
        a, b, c = impulse(k), filled(1), t.zeros((n, 4), dtype=t.int64, device="cuda")
        _uploaded()
        _h_combine(ctx, a, b, c, log_n)
        assert read(a) == NC.combine_impulse_expected(log_n, k, js), ("h_combine, a = delta", k)
        del a, b, c
    _mark(covered, "quotient closed forms", log_n)

    # a satisfied triple: h[n-1] = 0
    a, b = rnd, t.empty((n, 4), dtype=t.int64, device="cuda")
    ctx.fr_random_dev(700 + log_n, n, b)
    c = t.empty_like(a)
    ctx.fr_binop_dev(2, a, b, c, n)
    ctx.groth16_h_dev(a, b, c, log_n)
    ctx.synchronize()
    assert (host(a[n - 1:]) == 0).all()
    _mark(covered, "satisfied triple h[n-1] = 0", log_n)
    del a, b, c, rnd

    x = filled(1)
    _uploaded()
    ctx.divide_by_z_on_coset_dev(x, log_n)
    assert read(x) == [NC.z_inv(log_n)] * len(js)
    _mark(covered, "divide_by_z closed form", log_n)


@pytest.mark.parametrize("log_n", range(27))
def test_ntt_and_quotient_closed_forms(ctx, cref, covered, log_n):
    with _ctx_for(ctx, log_n) as c:
        _closed_forms(c, cref, covered, log_n)


@pytest.mark.parametrize("log_n", [27, 28])
def test_ntt_impulses_at_the_largest_domains(ctx, covered, log_n):
    """only when the card has about 3x the working set free: the vector plus the two n/2-entry twiddle tables"""
    t = _t()
    t.cuda.empty_cache()
    need = 2 * (1 << log_n) * 32
    free = t.cuda.mem_get_info()[0]
    if free < 3 * need:
        msg = f"log n = {log_n}: {free / 2**30:.1f} GiB free, the impulse checks want {3 * need / 2**30:.0f} GiB"
        print("\n" + msg)
        pytest.skip(msg)
    with _ctx_for(ctx, log_n) as c:
        _impulses(c, log_n, 13)
    _mark(covered, "impulses", log_n)


# ------------------------------------------------------------------ table cache
def test_ntt_tables_cached_across_interleaved_sizes(cref, covered):
    """one context runs sizes 20, 3, 20, 15, 0, 15 with mixed ops, then the quotient pipeline at 15: each result equals
    a fresh context's and the oracle's"""
    import bazuka_b200 as B
    order = [(20, 0), (3, 1), (20, 3), (15, 2), (0, 3), (15, 1)]
    warm = B.Context(0, load_poseidon=False)
    try:
        for i, (log_n, op) in enumerate(order):
            a = cref.fr_random(900 + i, 1 << log_n)
            want = cref.ntt(a, op)
            assert (_ntt(warm, a, log_n, op) == want).all(), (i, log_n, op)
            cold = B.Context(0, load_poseidon=False)
            try:
                assert (_ntt(cold, a, log_n, op) == want).all(), (i, log_n, op)
            finally:
                cold.close()
            _mark(covered, "table cache", log_n)
        a, b, c = (cref.fr_random(950 + s, 1 << 15) for s in range(3))
        ea, eb, ec = (cref.ntt(cref.ntt(v, 1), 2) for v in (a, b, c))
        want = cref.ntt(cref.divide_by_z_on_coset(cref.fr_sub(cref.fr_mul(ea, eb), ec)), 3)
        bufs = [dev(v) for v in (a, b, c)]
        _uploaded()
        warm.groth16_h_dev(*bufs, 15)
        warm.synchronize()
        assert (host(bufs[0]) == want).all()
    finally:
        warm.close()
