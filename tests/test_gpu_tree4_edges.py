"""GPU tier: the 4-ary Poseidon tree kernels at their edges, against plain sequential references.

`k_tree4_versioned_level` (csrc/poseidon.cu) applies an ordered batch of leaf writes to a forest of sparse trees with one
launch per level; every write scans the writes before it, across thread blocks.  Here it meets depth 32 (the top
level's `up >= 64` branch, index 4^32 - 1 = 2^64 - 1), batches of 700 and 4 100 writes whose scans cross 6 and 33
blocks, every write on one leaf or under one parent, two trees written alternately at the same indices, tree ids up
to 2^32 - 1, and n = 1 and 0.  The reference is `sequential_tree_updates` (one write at a time on dictionaries) over
the C oracle's Poseidon-4, and for a few depth-32 writes the plain `SparseTree4`.  The dense-tree kernels
(`merkle4_root_dev` at log4 0, 1 and 32, `merkle4_prove_dev` at log4 0 and 10) and `bzk_poseidon_hash_dev` at every
arity are checked beside it."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MAX64, MAX32 = (1 << 64) - 1, (1 << 32) - 1
R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001


def _mont(values):
    from bazuka_b200.mpn.cs import to_mont
    return to_mont(values)


def _ints(a):
    from bazuka_b200.mpn.batch_update import _from_mont_rows
    return _from_mont_rows(a)


@pytest.fixture(scope="module")
def hash4(cref):
    """Poseidon-4 over Python ints on the C oracle (the pure-Python one is too slow for depth-32 batches)"""
    def h(kids):
        return _ints(cref.poseidon(_mont(kids).reshape(1, 4, 4), threads=1))[0]
    return h


def _device(ctx, depth, tree_ids, indices, leaves, init):
    from bazuka_b200.mpn.batch_update import GpuTreeHasher
    return GpuTreeHasher(ctx).tree_update(depth, tree_ids, indices, leaves, init)


def _check_batch(ctx, hash4, depth, tree_ids, indices, rng, init=None):
    """kernel == sequential reference: every write's path values, root and proof.  Leaf values and pre-batch proofs are
    random field elements unless given, so a sibling taken from the wrong place changes the result."""
    from oracle.py.state import sequential_tree_updates
    n = len(indices)
    leaves = [rng.randrange(R) for _ in range(n)]
    if init is None:
        init = [[[rng.randrange(1 << 254) for _ in range(3)] for _ in range(depth)] for _ in range(n)]
    want_vals, want_proofs = sequential_tree_updates(depth, tree_ids, indices, leaves, init, hash4)
    got_vals, got_proofs = _device(ctx, depth, tree_ids, indices, leaves, init)
    for lvl in range(depth + 1):
        bad = [e for e in range(n) if got_vals[lvl][e] != want_vals[lvl][e]]
        assert not bad, (depth, "level", lvl, bad[:8])
    bad = [e for e in range(n) if got_proofs[e] != want_proofs[e]]
    assert not bad, (depth, "proofs", bad[:8])
    return want_vals


def test_depth32_batch_with_extreme_indices_and_tree_ids(ctx, hash4):
    """700 writes at depth 32: indices 0 and 2^64 - 1, neighbours of both, leaves sharing only their top-level parent,
    repeats, random indices over the whole range; tree ids 0, 1, 2^31 and 2^32 - 1."""
    rng = random.Random(3201)
    depth, n = 32, 700
    special = [0, MAX64, 1, 2, 3, MAX64 - 1, MAX64 - 3, MAX64 - 4, 1 << 62, (1 << 62) - 1, 3 << 62, 1 << 63]
    indices, tree_ids = [], []
    tids = [0, 1, 1 << 31, MAX32]
    for e in range(n):
        r = rng.random()
        if r < 0.3:
            i = rng.choice(special)
        elif r < 0.5 and indices:
            i = rng.choice(indices)                                    # rewrite an earlier leaf
        elif r < 0.7:
            i = (rng.randrange(4) << 62) | rng.randrange(1 << 8)       # share only the top-level parent
        else:
            i = rng.randrange(1 << 64)
        indices.append(i)
        tree_ids.append(rng.choice(tids))
    _check_batch(ctx, hash4, depth, tree_ids, indices, rng)


def test_depth16_batch_of_4100_writes(ctx, hash4):
    """4 100 writes at depth 16 (33 blocks of 128): every backward scan crosses up to 32 earlier blocks; clustered
    indices so that most levels find siblings far back."""
    rng = random.Random(1601)
    depth, n = 16, 4100
    top = 1 << 32
    hot = [rng.randrange(top) for _ in range(40)] + [0, top - 1]
    indices = [(rng.choice(hot) ^ rng.randrange(16)) % top if rng.random() < 0.8 else rng.randrange(top) for _ in range(n)]
    tree_ids = [rng.choice([7, MAX32]) for _ in range(n)]
    _check_batch(ctx, hash4, depth, tree_ids, indices, rng)


@pytest.mark.parametrize("shape", ["one_leaf", "one_parent", "two_trees_alternating"])
def test_batches_that_collide_everywhere(ctx, hash4, shape):
    """every write on one leaf (depth 32, at 2^64 - 1), every write under one parent (depth 32), and two trees written
    alternately at the same indices (depth 8): the scan must pick the latest earlier write of the same tree."""
    rng = random.Random({"one_leaf": 1, "one_parent": 2, "two_trees_alternating": 3}[shape])
    if shape == "one_leaf":
        depth, indices = 32, [MAX64] * 300
        tree_ids = [MAX32] * 300
    elif shape == "one_parent":
        depth = 32
        base = rng.randrange(1 << 62) << 2
        indices = [base + rng.randrange(4) for _ in range(260)]
        tree_ids = [5] * 260
    else:
        depth = 8
        pairs = [rng.randrange(1 << 16) if rng.random() < 0.5 else rng.randrange(8) for _ in range(250)]
        indices = [i for i in pairs for _ in range(2)]
        tree_ids = [(0, MAX32)[e % 2] for e in range(len(indices))]
    _check_batch(ctx, hash4, depth, tree_ids, indices, rng)


def test_single_write_and_empty_batch(ctx, hash4):
    """n = 1 at depth 32 on leaf 2^64 - 1 of tree 2^32 - 1 and on leaf 0 of tree 0; n = 0 is a no-op through the C
    entry point, and depths 0 and 33 are refused."""
    rng = random.Random(11)
    for tid, idx in ((MAX32, MAX64), (0, 0)):
        _check_batch(ctx, hash4, 32, [tid], [idx], rng)
    vals, proofs = ctx.tree4_versioned_update(32, np.zeros(0, np.uint32), np.zeros(0, np.uint64), np.zeros((0, 4), np.uint64), np.zeros((0, 32, 3, 4), np.uint64))
    assert vals.shape == (33, 0, 4) and proofs.shape == (0, 32, 3, 4)
    assert ctx._l.bzk_tree4_versioned_update_dev(ctx._h, 32, None, None, 0, None, None, None) == 0
    for depth in (0, 33):
        assert ctx._l.bzk_tree4_versioned_update_dev(ctx._h, depth, None, None, 0, None, None, None) == -1


def test_depth32_roots_follow_the_sparse_tree_write_by_write(ctx, hash4):
    """a handful of depth-32 writes to two trees with proofs read from real pre-batch trees: every root the kernel
    reports is the SparseTree4 root after that write, and every proof is the tree's proof just before it."""
    from bazuka_b200.mpn import native as N
    rng = random.Random(3202)
    trees = {0: N.SparseTree4(32, 0), MAX32: N.SparseTree4(32, 123)}
    trees[MAX32].set_leaf(MAX64 - 1, 77)
    writes = [(0, 0), (MAX32, MAX64), (0, 1), (MAX32, MAX64 - 1), (0, 0), (MAX32, 3 << 62), (0, MAX64)]
    tree_ids, indices = [t for t, _ in writes], [i for _, i in writes]
    init = [trees[t].prove(i) for t, i in writes]
    leaves = [rng.randrange(N.R) for _ in writes]
    got_vals, got_proofs = _device(ctx, 32, tree_ids, indices, leaves, init)
    for e, (t, i) in enumerate(writes):
        assert got_proofs[e] == trees[t].prove(i), e
        trees[t].set_leaf(i, leaves[e])
        assert got_vals[32][e] == trees[t].root, e


# ---------------------------------------------------------------------------------------------- dense trees, Poseidon
def _fold(hash4, idx, leaf, proof):
    cur = leaf
    for sib in proof:
        kids = list(sib)
        kids.insert(idx & 3, cur)
        cur = hash4(kids)
        idx >>= 2
    return cur


@pytest.mark.parametrize("log4", [0, 1, 32])
def test_merkle4_root_dev_against_a_python_fold(ctx, hash4, log4):
    """root of (index, leaf, proof) for 300 paths (three blocks), indices up to 4^log4 - 1, random siblings."""
    import torch
    rng = random.Random(400 + log4)
    m = 300
    top = 1 << (2 * log4)
    idx = [rng.choice([0, top - 1]) if rng.random() < 0.2 else rng.randrange(top) for _ in range(m)]
    leaves = [rng.randrange(1 << 254) for _ in range(m)]
    proofs = [[[rng.randrange(1 << 254) for _ in range(3)] for _ in range(log4)] for _ in range(m)]
    d_idx = torch.from_numpy(np.array(idx, dtype=np.uint64).view(np.int64)).cuda()
    d_leaves = torch.from_numpy(_mont(leaves).view(np.int64)).cuda()
    flat = [v for p in proofs for lvl in p for v in lvl]
    d_proofs = torch.from_numpy(_mont(flat).view(np.int64).reshape(m, log4, 3, 4)).cuda()
    d_roots = torch.empty((m, 4), dtype=torch.int64, device="cuda")
    ctx.merkle4_root_dev(log4, d_idx, d_leaves, d_proofs, d_roots)
    ctx.synchronize()
    got = _ints(d_roots.cpu().numpy().view(np.uint64))
    want = [_fold(hash4, i, l, p) for i, l, p in zip(idx, leaves, proofs)]
    assert got == want


@pytest.mark.parametrize("log4", [0, 10])
def test_merkle4_prove_then_root_on_a_dense_tree(ctx, cref, hash4, log4):
    """a dense tree built on the device (checked level by level against the C oracle), proofs of 500 leaves read from
    it equal the siblings in the node buffer, and folding them gives the stored root."""
    import torch
    n = 1 << (2 * log4)
    total = (4 ** (log4 + 1) - 1) // 3
    leaves = cref.fr_random(700 + log4, n)
    nodes = torch.zeros((total, 4), dtype=torch.int64, device="cuda")
    nodes[:n] = torch.from_numpy(leaves.view(np.int64)).cuda()
    ctx.merkle4_build_dev(nodes, log4)
    ctx.synchronize()
    host = nodes.cpu().numpy().view(np.uint64)
    off, width = 0, n
    for _ in range(log4):
        assert (host[off + width:off + width + width // 4] == cref.poseidon(host[off:off + width].reshape(width // 4, 4, 4))).all()
        off, width = off + width, width // 4
    rng = random.Random(800 + log4)
    idx = sorted({0, n - 1} | {rng.randrange(n) for _ in range(498)})
    m = len(idx)
    d_idx = torch.from_numpy(np.array(idx, dtype=np.uint64).view(np.int64)).cuda()
    proofs = torch.empty((m, log4, 3, 4), dtype=torch.int64, device="cuda")
    ctx.merkle4_prove_dev(nodes, log4, d_idx, proofs)
    d_leaves = torch.from_numpy(leaves[idx].view(np.int64)).cuda()
    roots = torch.empty((m, 4), dtype=torch.int64, device="cuda")
    ctx.merkle4_root_dev(log4, d_idx, d_leaves, proofs, roots)
    ctx.synchronize()
    hp = proofs.cpu().numpy().view(np.uint64).reshape(m, log4, 3, 4)
    starts = [sum(1 << (2 * (log4 - l)) for l in range(lvl)) for lvl in range(log4 + 1)]
    for k in range(0, m, 7):
        i = idx[k]
        for lvl in range(log4):
            node = i >> (2 * lvl)
            sib = [starts[lvl] + (node & ~3) + c for c in range(4) if (node & ~3) + c != node]
            assert (hp[k, lvl] == host[sib]).all(), (i, lvl)
    assert (roots.cpu().numpy().view(np.uint64) == host[-1]).all()
    ints = _ints(hp.reshape(-1, 4))
    k = m // 2
    proof = [ints[(k * log4 + lvl) * 3:(k * log4 + lvl) * 3 + 3] for lvl in range(log4)]
    assert _fold(hash4, idx[k], _ints(leaves[idx[k]:idx[k] + 1])[0], proof) == _ints(host[-1:])[0]


def test_poseidon_hash_dev_every_arity(ctx, cref):
    """bzk_poseidon_hash_dev (device buffers in and out) equals the C oracle at every arity the parameter table holds,
    for 1 and 300 inputs, edge values among them."""
    import torch
    from bazuka_b200.mpn import native as N
    edges = [0, 1, 2, R - 1, (R - 1) // 2, (1 << 256) % R, 1 << 254]
    for arity in sorted(t - 1 for t in N.poseidon_params()):
        for n in (1, 300):
            inp = cref.fr_random(900 + arity * 10 + n, n * arity).reshape(n, arity, 4)
            inp[0] = _mont([edges[k % len(edges)] for k in range(arity)])
            d_in = torch.from_numpy(np.ascontiguousarray(inp).view(np.int64)).cuda()
            d_out = torch.empty((n, 4), dtype=torch.int64, device="cuda")
            ctx.poseidon_dev(d_in, arity, d_out)
            ctx.synchronize()
            assert (d_out.cpu().numpy().view(np.uint64) == cref.poseidon(inp)).all(), (arity, n)
