"""GPU tier: the field and group-law edge families of tests/arith_cases.py through the sm_90a build of the conformance
harness (one thread per record, PTX carry chains), and libbzk's own field entry points (bzk_fr_binop_dev,
bzk_fp_mul_dev) on the same edges, at block-boundary sizes, in place, and on 2^22 random pairs against the C oracle."""
import numpy as np
import pytest

import arith_cases as A

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return A.DevArith()


@pytest.mark.parametrize("family", list(A.FAMILIES))
def test_arith_edges_gpu(dev, family):
    assert A.run_family(dev, family) == {}
    assert all(n % block for n, block in dev.blocks)


# ------------------------------------------------------------------ the production entry points
def _t():
    import torch
    return torch


def _pool(name):
    """the structured, add/sub-boundary and Montgomery-boundary pairs of one field, as (a, b) image words"""
    pairs = []
    for fam in ("structured", "sums", "mont_boundary"):
        for case in A.family(f"{name}.{fam}"):
            if case.op == f"{name}.add":
                n = A.FIELDS[name][1]
                pairs.append(case.inp.reshape(-1, 2, n))
    return np.concatenate(pairs)


def _want(name, op, a, b):
    f = A._F(name)
    p = f.p
    fn = {0: lambda x, y: (x + y) % p, 1: lambda x, y: (x - y) % p, 2: lambda x, y: x * y * f.Rinv % p}[op]
    return f.w([fn(x, y) for x, y in zip(A.ints(a), A.ints(b))])


def _call(ctx, name, op, da, db, out, n):
    if name == "fr":
        ctx.fr_binop_dev(op, da, db, out, n)
    else:
        ctx.fp_mul_dev(da, db, out, n)
    ctx.synchronize()


ENTRY = [("fr", 0), ("fr", 1), ("fr", 2), ("fp", 2)]


@pytest.mark.parametrize("name,op", ENTRY)
def test_arith_edges_entry_points(ctx, name, op):
    t = _t()
    pool = _pool(name)
    a, b = np.ascontiguousarray(pool[:, 0]), np.ascontiguousarray(pool[:, 1])
    da, db = t.from_numpy(a.view(np.int32)).cuda(), t.from_numpy(b.view(np.int32)).cuda()
    out = t.empty_like(da)
    _call(ctx, name, op, da, db, out, len(a))
    assert (out.cpu().numpy().view(np.uint32) == _want(name, op, a, b)).all()


@pytest.mark.parametrize("n", [1, 255, 256, 257, 65537])
@pytest.mark.parametrize("name,op", ENTRY)
def test_arith_edges_entry_sizes_and_in_place(ctx, name, op, n):
    """n records of edge pairs; the record after the last is never written; out == a and out == b give the same result"""
    t = _t()
    pool = _pool(name)
    idx = np.arange(n) % len(pool)
    a, b = np.ascontiguousarray(pool[idx, 0]), np.ascontiguousarray(pool[idx, 1])
    want = _want(name, op, a, b)
    guard = np.full((1, a.shape[1]), 0x5A5A5A5A, dtype=np.uint32)
    da = t.from_numpy(np.concatenate([a, guard]).view(np.int32)).cuda()
    db = t.from_numpy(np.concatenate([b, guard]).view(np.int32)).cuda()
    out = t.full_like(da, 0x3C3C3C3C)
    _call(ctx, name, op, da, db, out, n)
    got = out.cpu().numpy().view(np.uint32)
    assert (got[:n] == want).all() and (got[n] == 0x3C3C3C3C).all()
    for target in ("a", "b"):
        x, y = da.clone(), db.clone()
        dst = x if target == "a" else y
        _call(ctx, name, op, x, y, dst, n)
        got = dst.cpu().numpy().view(np.uint32)
        assert (got[:n] == want).all() and (got[n] == 0x5A5A5A5A).all(), target


def test_arith_edges_entry_bulk_random(ctx, cref):
    """2^22 random pairs per op against the C oracle"""
    t = _t()
    n = 1 << 22
    a, b = cref.fr_random(4101, n), cref.fr_random(4102, n)
    da, db = t.from_numpy(a.view(np.int64)).cuda(), t.from_numpy(b.view(np.int64)).cuda()
    out = t.empty_like(da)
    for op, f in ((0, cref.fr_add), (1, cref.fr_sub), (2, cref.fr_mul)):
        _call(ctx, "fr", op, da, db, out, n)
        assert (out.cpu().numpy().view(np.uint64) == f(a, b)).all(), op
    rng = np.random.default_rng(4103)
    top = A.FIELDS["fp"][0] >> 320   # top 64-bit limb of p: drawing it below that keeps every value < p
    x = rng.integers(0, 1 << 64, size=(n, 6), dtype=np.uint64)
    y = rng.integers(0, 1 << 64, size=(n, 6), dtype=np.uint64)
    x[:, 5] = rng.integers(0, top, size=n, dtype=np.uint64)
    y[:, 5] = rng.integers(0, top, size=n, dtype=np.uint64)
    dx, dy = t.from_numpy(x.view(np.int64)).cuda(), t.from_numpy(y.view(np.int64)).cuda()
    out = t.empty_like(dx)
    _call(ctx, "fp", 2, dx, dy, out, n)
    assert (out.cpu().numpy().view(np.uint64) == cref.fp_mul(x, y)).all()
