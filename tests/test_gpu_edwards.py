"""GPU tier: the Ed25519 and JubJub families of tests/edwards_cases.py through the sm_90a build of the conformance harness
tests/devshim/edwards.cu (one thread per record), with jj_mul_fixed reading the fixed-base tables that the build's host code
made and uploaded, as libbzk's contexts do; random products and jj_mul against the host fast paths; and both fixed-base tables swept entry by entry
through the production batch calls."""
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import edwards_cases as E
from bazuka_b200.mpn import native as N, signatures as S
from oracle.py import ed25519 as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return E.DevEdwards()


@pytest.mark.parametrize("family", list(E.FAMILIES))
def test_edwards_gpu(dev, family):
    assert E.run_family(dev, family) == {}
    assert all(n % block for n, block in dev.blocks)


def test_edwards_bulk_random_against_host64(dev):
    """2^16 random records per op: Montgomery products, sums and differences in both 25519 fields, and jj_mul on both curves
    (random Z, full-width scalars), word for word against the g++ build of the host fast paths"""
    host = E.HostEdwards(False)
    n = 1 << 16
    t0 = time.time()
    with ThreadPoolExecutor(os.cpu_count() or 1) as pool:   # the host runs release the GIL
        for op, inp in E.bulk_records(2026, n).items():
            got = dev.run(op, inp)
            want = np.concatenate(list(pool.map(lambda part: host.run(op, part), np.array_split(inp, 64))))
            assert got.shape == (n, E.OPS[op][2]) and (got == want).all(), op
    print(f"\n  bulk: {time.time() - t0:.1f} s")


def _sweep(curve, limit):
    """(s, [s] G, [s + 1] G) for every table entry of edwards_cases.sweep with s < limit"""
    c = E.CURVES[curve]
    return [(s, p, c.add(p, c.gen)) for _, _, s, p in E.sweep(curve, limit)]


def test_ed25519_table_sweep_through_the_batch_call(ctx):
    """verify_ed25519 on the identity key (y = 1), where [k](-A) vanishes and the verdict is compress([s] B) == R: every
    entry (j, v) of the context's table, with s = v 2^(8j) (+ 1 for j > 0) < l, accepts R = [s] B and refuses R = [s + 1] B"""
    sw = _sweep("ed25519", O.L)
    assert len(sw) == 31 * 256 + 17
    ident = (1).to_bytes(32, "little")
    msg = b"table sweep"
    good = [O.compress(p) + s.to_bytes(32, "little") for s, p, _ in sw]
    bad = [O.compress(q) + s.to_bytes(32, "little") for s, _, q in sw]
    n = len(sw)
    got = S.verify_ed25519(ctx, [ident] * 2 * n, [msg] * 2 * n, good + bad)
    assert got[:n].all(), [divmod(int(i), 256) for i in np.nonzero(~got[:n])[0][:4]]
    assert not got[n:].any()


def test_jubjub_table_sweep_through_the_batch_call(ctx):
    """verify_items on the identity key (x = 0, y = 1), where [h] A vanishes and the verdict is R == [s] BASE: every entry
    (j, v) of the context's table, with s = v 2^(8j) (+ 1 for j > 0) < r, accepts R = [s] BASE and refuses R = [s + 1] BASE"""
    sw = _sweep("jubjub", N.R)
    assert len(sw) == 31 * 256 + (N.R >> 248) + 1
    pk = (0, True)
    sigs = [{"r": p, "s": s} for s, p, _ in sw] + [{"r": q, "s": s} for s, _, q in sw]
    n = len(sw)
    got = S.verify_items(ctx, [pk] * 2 * n, [0] * 2 * n, sigs)
    assert got[:n].all(), [int(i) for i in np.nonzero(~got[:n])[0][:4]]
    assert not got[n:].any()
