"""GPU tier: base vectors in pinned host memory (bzk_g*_bases_move, bzk_groth16_params_move / _read_placed).  Every MSM over
a host vector streams it to the device in chunks; each value here is checked against the C oracle and against the same
vector kept on the device, with chunks forced small (bzk_ctx_set_msm_stream_chunk) so that oracle-sized sums cross many
chunk edges."""
import ctypes as ct

import numpy as np
import pytest

from conftest import fr_arr
from test_gpu_baseline_configs import _witness_like

pytestmark = pytest.mark.gpu

R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
P = 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB
N_PTS = 16384


def _t():
    import torch
    return torch


@pytest.fixture(scope="module")
def vectors(ctx):
    """N_PTS random G1 and G2 bases: host copies of the images for the oracle, and a device and a host vector of each"""
    t = _t()
    out = {}
    for g, w in (("g1", 104), ("g2", 200)):
        d = t.empty((N_PTS, w), dtype=t.uint8, device="cuda")
        getattr(ctx, f"{g}_random_bases_dev")(21 if g == "g1" else 22, N_PTS, d)
        ctx.synchronize()
        dev = getattr(ctx, f"{g}_bases_from_dev")(d, N_PTS)
        host = getattr(ctx, f"{g}_bases_from_dev")(d, N_PTS).move_to_host()
        assert host.on_host and not dev.on_host and len(host) == N_PTS and host.levels == 1
        out[g] = (d.cpu().numpy(), dev, host)
    yield out
    ctx.set_msm_stream_chunk(0)
    for _, dev, host in out.values():
        dev.free(); host.free()


def _msm(ctx, cref, g, vec, scalars, off, chunk):
    imgs, dev, host = vec
    n = len(scalars)
    ctx.set_msm_stream_chunk(chunk)
    msm = getattr(ctx, f"msm_{g}_resident")
    got = msm(host, scalars, offset=off, n=n)
    st = ctx.last_msm_stream()
    cn = min(chunk, n)
    assert st == {"chunks": -(-n // cn), "chunk_points": cn, "bytes_h2d": n * (96 if g == "g1" else 192), "streamed": 1}, (n, chunk, st)
    want = getattr(cref, f"msm_{g}")(imgs[off:off + n], scalars)
    assert (got == want).all(), (g, n, chunk)
    assert (msm(dev, scalars, offset=off, n=n) == want).all()
    assert ctx.last_msm_stream()["streamed"] == 0
    return got


@pytest.mark.parametrize("g", ["g1", "g2"])
@pytest.mark.parametrize("chunk", [256, 4096])
def test_host_vector_msm_geometries(ctx, cref, vectors, g, chunk):
    """n in {1, chunk - 1, chunk, chunk + 1, 3.5 chunks} at a non-zero offset; uniform, witness-shaped (the 45 % booleans put
    window 0's digit-1 bucket into every chunk, through k_fixup_long each time) and all-zero scalars"""
    off = 7
    for n in (1, chunk - 1, chunk, chunk + 1, chunk * 7 // 2):
        witness = _witness_like(cref, 200 + n, max(n, 16))[:n]   # its first 11 entries are edge values
        for k, scalars in enumerate((cref.fr_random(100 + n, n), witness, np.zeros((n, 4), np.uint64))):
            _msm(ctx, cref, g, vectors[g], scalars, off + k, chunk)


def _negate_g1(img):
    """-P for G1 wire images (y -> p - y, Montgomery form is linear)"""
    out = img.copy()
    for row in out:
        y = int.from_bytes(row[48:96].tobytes(), "little")
        row[48:96] = np.frombuffer(((P - y) % P).to_bytes(48, "little"), np.uint8)
    return out


def test_bucket_passes_through_the_identity_across_chunks(ctx, cref):
    """chunk 1 holds the negations of chunk 0's points and every scalar is 1: window 0's digit-1 bucket is exactly the
    identity after chunk 1 and takes chunk 2's points after that"""
    chunk = 256
    t = _t()
    d = t.empty((3 * chunk, 104), dtype=t.uint8, device="cuda")
    ctx.g1_random_bases_dev(31, 3 * chunk, d)
    ctx.synchronize()
    imgs = d.cpu().numpy()
    imgs[chunk:2 * chunk] = _negate_g1(imgs[:chunk])
    host = ctx.g1_bases(imgs).move_to_host()
    dev = ctx.g1_bases(imgs)
    for scalars in (fr_arr([1] * (3 * chunk)), fr_arr([1] * (2 * chunk) + [5] * chunk)):
        _msm(ctx, cref, "g1", (imgs, dev, host), scalars, 0, chunk)
    # only the two cancelling chunks: the sum is the identity
    ctx.set_msm_stream_chunk(chunk)
    got = ctx.msm_g1_resident(host, fr_arr([1] * (2 * chunk)), n=2 * chunk)
    assert got[96] == 1
    ctx.set_msm_stream_chunk(0)
    host.free(); dev.free()


def test_more_long_runs_in_one_chunk_than_the_queue_holds(ctx, cref):
    """2^18 scalars drawn from 300 values, chunks of 2^17 points: every window has 300 buckets of ~440 entries per chunk,
    each cut into more than 6 partial runs, so each chunk has over 4096 long runs and k_fixup sums the excess serially"""
    t = _t()
    n, chunk = 1 << 18, 1 << 17
    d = t.empty((n, 104), dtype=t.uint8, device="cuda")
    ctx.g1_random_bases_dev(41, n, d)
    ctx.synchronize()
    imgs = d.cpu().numpy()
    vals = cref.fr_random(42, 300)
    scalars = np.ascontiguousarray(vals[np.random.default_rng(43).integers(0, 300, n)])
    host = ctx.g1_bases_from_dev(d, n).move_to_host()
    dev = ctx.g1_bases_from_dev(d, n)
    _msm(ctx, cref, "g1", (imgs, dev, host), scalars, 0, chunk)
    ctx.set_timing(True)
    ctx.set_msm_stream_chunk(0)
    ctx.msm_g1_resident(dev, scalars[:chunk], n=chunk)
    assert ctx.last_msm_plan()["long_len"] > 4096   # the same chunk on a device vector overflows the queue
    ctx.set_timing(False)
    host.free(); dev.free()


def test_moves_free_and_refusals(ctx, cref, vectors):
    """device -> host -> device keeps the points; tables are dropped on the way; precompute on a host vector is refused;
    free works in both places; a bad chunk size is refused"""
    import bazuka_b200 as B
    imgs, _, _ = vectors["g1"]
    b = ctx.g1_bases(imgs[:5000])
    s = cref.fr_random(5, 5000)
    want = ctx.msm_g1_resident(b, s)
    assert b.precompute(8) > 1
    b.move_to_host()
    assert b.on_host and b.levels == 1 and len(b) == 5000
    with pytest.raises(B.BzkError) as e:
        b.precompute(8)
    assert e.value.status == -1
    assert (ctx.msm_g1_resident(b, s) == want).all()
    b.move_to_host()   # no-op
    b.move_to_device()
    assert not b.on_host and b.levels == 1
    assert (ctx.msm_g1_resident(b, s) == want).all()
    b.free()
    h2 = ctx.g2_bases(vectors["g2"][0][:10]).move_to_host()
    h2.free()
    for bad in (1, 255):
        with pytest.raises(B.BzkError):
            ctx.set_msm_stream_chunk(bad)
    ctx.set_msm_stream_chunk(256)
    ctx.set_msm_stream_chunk(0)


# ------------------------------------------------------------------ Groth16
@pytest.fixture(scope="module")
def circuit(ctx, cref):
    """a synthetic circuit with its setup_gpu key, the oracle prover's proof for fixed (r, s), and the key's file image"""
    from bazuka_b200 import groth16 as BG, synth
    from oracle import groth16_c as GC
    ni, na, mats, inputs, aux = synth.build(lanes=16, rounds=6, seed=51, ops=synth.GpuOps(ctx))
    pr = BG.Prover(ctx, BG.R1CS(ni, na, *mats))
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, cref.fr_random(52, 5), cref.g1_generator(), cref.g2_generator(), table_levels=1)
    r, s = cref.fr_random(53, 2)
    a_idx, b_idx = GC.density(ni, na, mats)
    cpk = {"log_m": pr.log_m, "vk": vk, "a_idx": a_idx, "b_idx": b_idx}
    for k in BG.KEY_VECTORS:
        cpk[k] = pk.device_images[k].cpu().numpy()
    want = GC.proof_bytes(*GC.prove(ni, na, mats, cpk, inputs, aux, r, s))
    img = BG.write_parameters(ctx, pk)
    yield dict(pr=pr, pk=pk, vk=vk, inputs=inputs, aux=aux, r=r, s=s, want=want, img=img, log_m=pr.log_m)
    pk.free(); pr.free()


def _both_proofs(c, pk):
    t = _t()
    got, _ = c["pr"].prove(pk, c["inputs"], c["aux"], c["r"], c["s"])
    d_in = t.from_numpy(c["inputs"].view(np.int64)).cuda()
    d_aux = t.from_numpy(c["aux"].view(np.int64)).cuda()
    got_dev, _ = c["pr"].prove_dev(pk, d_in, d_aux, c["r"], c["s"])
    return got, got_dev


def test_every_placement_proves_the_oracle_bytes(ctx, circuit):
    """all 32 placements of the five vectors, with 256-point chunks: prove and prove_dev give the device key's bytes, which
    are the oracle prover's; a round trip through the host leaves the key's file image byte-equal"""
    from bazuka_b200 import groth16 as BG
    c, pk = circuit, circuit["pk"]
    assert all(BG.parameters_info(c["img"])[f"n_{k}"] > 256 for k in ("h", "l", "b_g2"))
    assert (_both_proofs(c, pk)[0] == c["want"]).all()
    ctx.set_msm_stream_chunk(256)
    try:
        for mask in range(32):
            pk.move(mask)
            got, got_dev = _both_proofs(c, pk)
            assert (got == c["want"]).all(), mask
            assert (got_dev == c["want"]).all(), mask
            if mask in (0b10101, 31):
                assert (BG.write_parameters(ctx, pk) == c["img"]).all(), mask
    finally:
        ctx.set_msm_stream_chunk(0)
        pk.move(0)
    assert (BG.write_parameters(ctx, pk) == c["img"]).all()


def test_mixed_key_tables_only_its_device_vectors(ctx, circuit):
    """params_precompute on a key with h, a and b_g2 on the host tables l and b_g1 and leaves the host vectors alone; the
    proofs are unchanged, and moving l and b_g1 to the host then frees their tables too"""
    from bazuka_b200 import groth16 as BG
    c = circuit
    info = BG.parameters_info(c["img"])
    pk, _ = BG.read_parameters(ctx, c["img"], checked=False, table_levels=1)
    pk.move(0b10101)
    before = _free_bytes()
    pk.precompute(8)
    tables = before - _free_bytes()
    assert tables > 0
    got, got_dev = _both_proofs(c, pk)
    assert (got == c["want"]).all() and (got_dev == c["want"]).all()
    before = _free_bytes()
    pk.move(31)
    assert _free_bytes() - before > (info["n_l"] + info["n_b_g1"]) * 96
    assert (_both_proofs(c, pk)[0] == c["want"]).all()
    pk.free()


def _free_bytes():
    t = _t()
    t.cuda.synchronize()
    return t.cuda.mem_get_info()[0]


def test_sharded_partials_with_host_shard_keys(ctx, circuit):
    """three ranks' prove_partial with host shard keys give the device shard keys' partial sums"""
    from bazuka_b200 import groth16 as BG
    c = circuit
    ctx.set_msm_stream_chunk(256)
    try:
        for rank in range(3):
            spk = BG.shard_proving_key(ctx, c["pk"], c["log_m"], rank, 3)
            want = c["pr"].prove_partial(spk, c["inputs"], c["aux"])
            spk.move(31)
            got = c["pr"].prove_partial(spk, c["inputs"], c["aux"])
            for w, g in zip(want, got):
                assert (np.asarray(w) == np.asarray(g)).all(), rank
            spk.free()
    finally:
        ctx.set_msm_stream_chunk(0)


def test_key_file_reads_into_host_memory(ctx, circuit):
    """read_parameters with each single vector and with all five in host memory: the same proofs and written images as a
    device read"""
    from bazuka_b200 import groth16 as BG
    c = circuit
    for hv in [(k,) for k in BG.KEY_VECTORS] + ["all"]:
        pk, vk = BG.read_parameters(ctx, c["img"], checked=True, host_vectors=hv)
        assert (BG.write_parameters(ctx, pk) == c["img"]).all(), hv
        got, got_dev = _both_proofs(c, pk)
        assert (got == c["want"]).all() and (got_dev == c["want"]).all(), hv
        pk.free()


def test_corrupt_point_in_a_host_vector_is_refused_as_on_the_device(ctx, circuit):
    import bazuka_b200 as B
    from bazuka_b200 import groth16 as BG
    c = circuit
    info = BG.parameters_info(c["img"])
    # the image's layout: 6 vk points, |ic| + ic, then h, l, ... each behind its u32 length
    off = 96 * 3 + 192 * 3 + 4 + 96 * info["n_ic"] + 4 + 96 * info["n_h"] + 4
    for idx in (0, 300):
        bad = c["img"].copy()
        bad[off + 96 * idx] |= 0x20   # sort flag
        results = []
        for hv in ((), ("l",), "all"):
            with pytest.raises(B.BzkError) as e:
                BG.read_parameters(ctx, bad, checked=True, host_vectors=hv)
            results.append((e.value.status, str(e.value)))
        assert results[0] == results[1] == results[2], results
        assert f"l[{idx}]:" in results[0][1]


def test_host_placed_read_allocates_no_vector_on_the_device(ctx, circuit):
    """a key of 2^20-point vectors (576 MB packed) read with every vector in host memory leaves at least 0.9 x that much
    more device memory free than a device read"""
    from bazuka_b200 import groth16 as BG
    t = _t()
    n = 1 << 20
    g1 = t.empty((n, 104), dtype=t.uint8, device="cuda")
    g2 = t.empty((n, 200), dtype=t.uint8, device="cuda")
    ctx.g1_random_bases_dev(61, n, g1)
    ctx.g2_random_bases_dev(62, n, g2)
    ctx.synchronize()
    vecs = [ctx.g1_bases_from_dev(g1, n) for _ in range(4)] + [ctx.g2_bases_from_dev(g2, n)]
    big = BG._make_pk(ctx, circuit["vk"], *vecs, table_levels=1)
    img = BG.write_parameters(ctx, big)
    big.free()
    del g1, g2
    t.cuda.empty_cache()
    packed = 4 * n * 96 + n * 192
    used = {}
    for hv in ((), "all", ()):
        before = _free_bytes()
        pk, _ = BG.read_parameters(ctx, img, checked=False, table_levels=1, host_vectors=hv)
        used[hv] = before - _free_bytes()
        assert (BG.write_parameters(ctx, pk) == img).all()
        pk.free()
    print(f"\ndevice read {used[()] / 1e6:.0f} MB, host read {used['all'] / 1e6:.0f} MB, packed key {packed / 1e6:.0f} MB")
    assert used[()] - used["all"] >= 0.9 * packed


def test_mpn_work_proves_with_a_host_key(ctx, cref):
    """the one-call MPN prover (bzk_mpn_prover_prove_work) with the update worker's key in host memory: the device key's 391
    bytes, accepted by bzk_mpn_work_verify"""
    from bazuka_b200.mpn import wire as Wr, works as Wk
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    from bazuka_b200.mpn.worker import MpnUpdateWorker
    from test_wire_cpu import _scenario
    st, keys, deposits, withdraws, wpay, updates = _scenario()
    A, T, B = 3, 3, 1
    wu = MpnUpdateWorker(ctx, A, T, B, cref.fr_random(311, 5))
    config = {"log4_tree_size": A, "log4_token_tree_size": T, "log4_deposit_batch_size": B, "log4_withdraw_batch_size": B, "log4_update_batch_size": B,
              "mpn_contract_id": 0x1234, "mpn_num_update_batches": 1, "mpn_num_deposit_batches": 1, "mpn_num_withdraw_batches": 1,
              "deposit_vk": bytes(wu.vk_blob), "withdraw_vk": bytes(wu.vk_blob), "update_vk": bytes(wu.vk_blob)}
    works, _ = Wk.prepare_works(config, st, deposits, withdraws, updates, {"deposit": 11, "withdraw": 22, "update": 33}, height=9, withdraw_payments=wpay)
    work = [w for w in works.values() if w["data"][0] == "update"][0]
    blob = Wr.work_to_bytes(work)
    me = bytes(range(32))
    r, s = cref.fr_random(612, 2)
    nat = Wk.NativeMpnProver(ctx)
    circ = NativeUpdateCircuit(A, T, B)
    nat.add_circuit("update", circ, wu.pk)
    circ.free()
    want = nat.prove(blob, me, r, s)
    wu.pk.move(31)
    ctx.set_msm_stream_chunk(256)
    try:
        got = nat.prove(blob, me, r, s)
    finally:
        ctx.set_msm_stream_chunk(0)
    assert len(got) == 391 and got == want
    lib = ctx._l
    h = ct.c_void_p()
    assert lib.bzk_mpn_work_decode(blob, len(blob), ct.byref(h), None) == 0
    assert lib.bzk_mpn_work_verify(h, me, got[4:]) == 1
    lib.bzk_mpn_work_free(h)
    nat.free()
    wu.free()


def test_production_update_batch_with_a_host_key(ctx, cref):
    """A=15, T=3, B=4 (2^24 domain, as test_gpu_baseline_configs): the proof with every key vector in host memory, at the
    default chunk size, is byte-equal to the tabled device key's, and the move frees at least the packed key on the device"""
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn import update as U
    from bazuka_b200.mpn.gpu_witness import UpdateWitnessGpu
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    from test_gpu_baseline_configs import _ledger_and_transfers
    t = _t()
    A, T, B = 15, 3, 4
    nc = NativeUpdateCircuit(A, T, B)
    ni, na, mats = nc.r1cs()
    prog, epilogues = nc.program(0), {B: nc.program(1)}
    nc.free()
    pr = BG.Prover(ctx, BG.R1CS(ni, na, *mats))
    assert pr.log_m == 24
    pk, vk = BG.setup_gpu(ctx, pr.r1cs, cref.fr_random(521, 5), cref.g1_generator(), cref.g2_generator())
    packed = sum(pk.device_images[k].shape[0] for k in ("h", "l", "a", "b_g1")) * 96 + pk.device_images["b_g2"].shape[0] * 192
    pk.device_images = None
    t.cuda.empty_cache()
    wit = UpdateWitnessGpu(ctx, A, T, prog, epilogues)
    led, txs = _ledger_and_transfers(ctx, A, T, B, 64)
    raws, ext, accepted, pub, n_acc = led.update_build(txs, B)
    d_in, d_aux = wit.witness_native(raws, ext, [42, 7, pub["state"], U.ZIESHA, pub["aux_data"], pub["next_state"]], B)
    r, s = cref.fr_random(522, 2)
    want, _ = pr.prove_dev(pk, d_in, d_aux, r, s)
    before = _free_bytes()
    pk.move(31)
    freed = _free_bytes() - before
    got, _ = pr.prove_dev(pk, d_in, d_aux, r, s)
    assert (got == want).all()
    print(f"\n2^24 key: {packed / 1e9:.2f} GB packed, {freed / 1e9:.2f} GB freed by the move to host memory")
    assert freed >= 0.9 * packed
    wit.free(); led.free(); pk.free(); pr.free()
