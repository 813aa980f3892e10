"""GPU tier: the MSM at every plan geometry it can run, against the C oracle.

The MSM picks a window c, window count W, table levels T, bucket groups G, reduction slice and nbits per call: freely from
n for a plain base vector, from the table for a tabled one (and which table a proving key gets depends on the device memory
free when it is built).  Each case here asserts, through bzk_ctx_last_msm_plan, the plan it means to cover, so that a change
of the cost constants cannot move it silently to another plan, and compares the value with the oracle on uniform scalars
mixed with digit-edge scalars built for that (c, W).  Run with -s for the table of plans covered."""
import numpy as np
import pytest

from conftest import fr_arr
from test_gpu_baseline_configs import _witness_like

pytestmark = pytest.mark.gpu

R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
N_BIG = 1 << 20
N_TAB_G1, N_TAB_G2 = 1 << 16, 4096


# ------------------------------------------------------------------ the planner, restated (csrc/msm_impl.cuh)
def _plan_cost(n, c, T):
    W = -(-256 // c)
    G = -(-W // min(T, W))
    top_bits = 255 - c * (W - 1)
    narrow = 1.5 * n if (W > 1 and top_bits < 10 and n >= 4096) else 0.0
    return float(n) * W + 6.0 * G * float(1 << (c - 1)) + narrow


def _free_c(n):
    """make_plan's window for n terms over plain bases (first minimum wins, as in the C loop)"""
    return min(range(2, 19), key=lambda c: _plan_cost(n, c, 1))


def _first_sizes(n_max):
    """{c: smallest n <= n_max whose free plan has window c}, by bisection (the choice grows with n)"""
    out = {}
    for c in range(2, 19):
        lo, hi = 1, n_max
        if _free_c(hi) < c:
            continue
        while lo < hi:
            mid = (lo + hi) // 2
            if _free_c(mid) >= c:
                hi = mid
            else:
                lo = mid + 1
        if _free_c(lo) == c:
            out[c] = lo
    return out


def _table_shape(c, levels):
    """(W, T, G) of a table built with window c forced and `levels` levels at most (choose_table)"""
    W = -(-256 // c)
    G = -(-W // min(levels, W))
    return W, -(-W // G), G


FREE_SIZES = _first_sizes(N_BIG)
TABLE_CASES = [(c, lv) for c in (8, 9, 10, 11, 12, 13, 14, 16) for lv in (3, 16)] + \
              [(20, 2), (20, 5), (20, 16), (22, 2), (22, 5), (22, 16)]
# c = 22 with 2 levels has 6 groups of 2^21 buckets: 2.4 GB of G1 buckets, 4.8 GB for G2 — G1 only
TABLE_CASES_G2 = [cl for cl in TABLE_CASES if cl != (22, 2)]


# ------------------------------------------------------------------ scalars
def _edge_scalars(c, W, seed):
    """scalars whose c-bit chunks all come from {0, 1, 2^(c-1)-1, 2^(c-1), 2^(c-1)+1, 2^c-1}: every window on one value
    (all 2^(c-1): every digit in bucket NB-1; all 2^(c-1)+1: every digit negative with a carry; all 2^c-1: the carry
    ripples through all W windows), the six values rotating over the windows, random picks, and r-1, r-2 (the top
    window at its narrowest).  Truncated to 254 bits, so every value is below r."""
    half = 1 << (c - 1)
    E = [0, 1, half - 1, half, half + 1, (1 << c) - 1]
    mask = (1 << 254) - 1
    pack = lambda chunks: sum(x << (c * w) for w, x in enumerate(chunks)) & mask
    rng = np.random.default_rng(seed)
    out = [pack([e] * W) for e in E]
    out += [pack([E[(w + k) % 6] for w in range(W)]) for k in range(6)]
    out += [pack([E[j] for j in rng.integers(0, 6, W)]) for _ in range(36)]
    return out + [R - 1, R - 2, mask, 1 << 253]


def _mixed(cref, seed, n, edge):
    """uniform scalars with every third one replaced by the edge set (cycled): each edge value forms runs of equal
    digits in the sorted list and the uniform ones move where the chunk edges fall"""
    s = cref.fr_random(seed, n)
    e = fr_arr(edge)
    idx = np.arange(0, n, 3)
    s[idx] = e[np.arange(len(idx)) % len(e)]
    return s


# ------------------------------------------------------------------ fixtures
_COVERED = []


@pytest.fixture(scope="module", autouse=True)
def _plan_table():
    yield
    if _COVERED:
        print("\n  group   c   W   T   G  slice nbits  long_len  TB > 2^20  case")
        for g, p, case in sorted(_COVERED, key=lambda r: (r[0], r[1]["c"], r[1]["T"], r[1]["G"])):
            print(f"  {g:5} {p['c']:3} {p['W']:3} {p['T']:3} {p['G']:3} {p['slice']:6} {p['nbits']:5} {p['long_len']:9}"
                  f"  {'yes' if p['G'] * p['NB'] > 1 << 20 else '':9}  {case}")


def _record(group, plan, case):
    _COVERED.append((group, plan, case))


@pytest.fixture(scope="module")
def g1_pts(ctx):
    """2^20 random G1 bases: device images and their host copy for the oracle"""
    import torch
    d = torch.empty((N_BIG, 104), dtype=torch.uint8, device="cuda")
    ctx.g1_random_bases_dev(12, N_BIG, d)
    ctx.synchronize()
    return d, d.cpu().numpy()


@pytest.fixture(scope="module")
def g2_pts(ctx):
    import torch
    d = torch.empty((N_TAB_G2, 200), dtype=torch.uint8, device="cuda")
    ctx.g2_random_bases_dev(13, N_TAB_G2, d)
    ctx.synchronize()
    return d, d.cpu().numpy()


def _api(ctx, cref, group):
    if group == "g1":
        return ctx.g1_bases_from_dev, ctx.msm_g1_resident, cref.msm_g1
    return ctx.g2_bases_from_dev, ctx.msm_g2_resident, cref.msm_g2


def _check(ctx, msm, oracle, rb, host_img, scalars, want_plan, offset=0):
    """one MSM over bases[offset : offset + len(scalars)]: its plan has the fields of want_plan, its value is the oracle's"""
    n = len(scalars)
    got = msm(rb, scalars, offset=offset)
    plan = ctx.last_msm_plan()
    assert {k: plan[k] for k in want_plan} == want_plan, (plan, offset, n)
    assert (got == oracle(host_img[offset:offset + n], scalars)).all(), (plan, offset, n)
    return plan


# ------------------------------------------------------------------ free plans
def test_entry_points_refuse_out_of_range_window(ctx):
    import bazuka_b200 as B
    for c in (1, 7, 24, 1 << 31):
        with pytest.raises(B.BzkError) as e:
            ctx.set_msm_table_window(c)
        assert e.value.status == -1
    ctx.set_msm_table_window(0)


def test_free_plans_cover_every_reachable_window():
    """the restated planner reaches the windows the fixed sizes below are for (c = 15 is never the cheapest)"""
    assert set(FREE_SIZES) == set(range(2, 15)) | {16}, FREE_SIZES


@pytest.mark.parametrize("c,n", sorted(FREE_SIZES.items()), ids=[f"c{c}-n{n}" for c, n in sorted(FREE_SIZES.items())])
def test_free_plan_vs_oracle(ctx, cref, g1_pts, c, n):
    """plain bases, n = the first size whose free plan has window c: uniform scalars, then the digit-edge set mixed in
    (sizes below the edge set's length take it in slices of n)"""
    d_img, host = g1_pts
    rb = ctx.g1_bases_from_dev(d_img, n)
    W = -(-256 // c)
    want = {"c": c, "W": W, "T": 1, "G": W}
    plan = _check(ctx, ctx.msm_g1_resident, cref.msm_g1, rb, host, cref.fr_random(100 + c, n), want)
    edge = _edge_scalars(c, W, c)
    if n >= len(edge):
        _check(ctx, ctx.msm_g1_resident, cref.msm_g1, rb, host, _mixed(cref, 200 + c, n, edge), want)
    else:
        e = fr_arr(edge)
        for k in range(0, len(e) - n + 1, n):
            _check(ctx, ctx.msm_g1_resident, cref.msm_g1, rb, host, np.ascontiguousarray(e[k:k + n]), want)
    _record("g1", plan, f"free n={n}")
    rb.free()


# ------------------------------------------------------------------ table plans
def _table_case(ctx, cref, group, pts, n, c, levels, seed):
    from_dev, msm, oracle = _api(ctx, cref, group)
    d_img, host = pts
    W, T, G = _table_shape(c, levels)
    rb = from_dev(d_img, n)
    ctx.set_msm_table_window(c)
    try:
        assert rb.precompute(levels) == T
    finally:
        ctx.set_msm_table_window(0)
    want = {"c": c, "W": W, "T": T, "G": G}
    plan = _check(ctx, msm, oracle, rb, host, cref.fr_random(seed, n), want)
    mixed = _mixed(cref, seed + 1, n, _edge_scalars(c, W, seed))
    _check(ctx, msm, oracle, rb, host, mixed, want)
    # sub-ranges of the table (what the sharded prover runs): a tiny one leaves almost every bucket empty; the last one
    # ends at the table's end
    for off, k in ((777, 1), (n // 2, 2), (5, 17), (n // 3, 1000), (n - 4096, 4096)):
        _check(ctx, msm, oracle, rb, host, np.ascontiguousarray(mixed[off:off + k]), want, offset=off)
    _record(group, plan, f"table n={n} levels<={levels}")
    rb.free()
    return plan


@pytest.mark.parametrize("c,levels", TABLE_CASES, ids=[f"c{c}-L{lv}" for c, lv in TABLE_CASES])
def test_g1_table_plan_vs_oracle(ctx, cref, g1_pts, c, levels):
    plan = _table_case(ctx, cref, "g1", g1_pts, N_TAB_G1, c, levels, 300 + c * 17 + levels)
    if (c, levels) == (22, 2):
        assert plan["G"] * plan["NB"] > 1 << 20  # more than 1024 scan tiles: k_scan_tiles' carried loop


@pytest.mark.parametrize("c,levels", TABLE_CASES_G2, ids=[f"c{c}-L{lv}" for c, lv in TABLE_CASES_G2])
def test_g2_table_plan_vs_oracle(ctx, cref, g2_pts, c, levels):
    _table_case(ctx, cref, "g2", g2_pts, N_TAB_G2, c, levels, 500 + c * 17 + levels)


# ------------------------------------------------------------------ 2^20: long runs, witness shapes
def _long_run_scalars(cref, n):
    """1 + (i mod 8192): 8192 buckets of n/8192 entries in window 0, each cut by more chunk edges than kLongRun"""
    canon = np.zeros((n, 4), dtype=np.uint64)
    canon[:, 0] = 1 + np.arange(n, dtype=np.uint64) % 8192
    return cref.fr_to_mont(canon)


def test_long_run_queue_overflow_free_plan(ctx, cref, g1_pts):
    """more long runs than the CTA-wide queue holds (4096): the rest go through k_fixup's serial fallback"""
    d_img, host = g1_pts
    rb = ctx.g1_bases_from_dev(d_img, N_BIG)
    ctx.set_timing(True)
    try:
        plan = _check(ctx, ctx.msm_g1_resident, cref.msm_g1, rb, host, _long_run_scalars(cref, N_BIG), {"c": 16, "T": 1, "G": 16})
    finally:
        ctx.set_timing(False)
    assert plan["long_len"] > 4096, plan
    _record("g1", plan, "free 2^20, 1 + (i mod 8192)")
    rb.free()


def test_2_20_table_long_runs_witness_shaped_and_ones(ctx, cref, g1_pts):
    """the 2^20 table the planner picks with 16 levels (one bucket set shared by all windows): the long-run overflow,
    a Groth16 witness's scalar census and all ones (one bucket holds the whole vector)"""
    d_img, host = g1_pts
    rb = ctx.g1_bases_from_dev(d_img, N_BIG)
    rb.precompute(16)
    want = {"c": 20, "W": 13, "T": 13, "G": 1}
    ctx.set_timing(True)
    try:
        plan = _check(ctx, ctx.msm_g1_resident, cref.msm_g1, rb, host, _long_run_scalars(cref, N_BIG), want)
    finally:
        ctx.set_timing(False)
    assert plan["long_len"] > 4096, plan
    _record("g1", plan, "table 2^20, 1 + (i mod 8192)")
    _check(ctx, ctx.msm_g1_resident, cref.msm_g1, rb, host, _witness_like(cref, 38, N_BIG), want)
    _check(ctx, ctx.msm_g1_resident, cref.msm_g1, rb, host, fr_arr([1]).repeat(N_BIG, axis=0), want)
    rb.free()
