"""Groth16 prover front-end over libbzk — the host-side mirror of bellman's
`groth16::{Parameters, create_proof}` as the reference uses them
(/root/reference/src/mpn/circuits/test.rs:133-149: setup -> create_random_proof -> verify_proof;
production boundary: `MpnWork` in, `ZkProof::Groth16` out, /root/reference/src/mpn/mod.rs:264-295).

  R1CS          constraint system in CSR form (what `Circuit::synthesize` emits), numpy arrays
  ProvingKey    `Parameters<Bls12>` resident on one GPU
  setup_gpu     bellman `generate_parameters` with explicit toxic waste, computed with libbzk kernels
                (iNTT for the Lagrange basis, transposed SpMV, fixed-base multiplications); used to
                make keys for synthetic circuits — production keys come from the ceremony
  read_parameters / write_parameters
                bellman's `Parameters::read` / `Parameters::write` file image <-> a resident ProvingKey, every point
                decoded (and, checked, tested for the curve and the prime-order subgroup) on the GPU
  Prover.prove  -> 387-byte `Groth16Proof` bincode image (bit-exact vs the CPU prover for equal
                (params, r, s, witness))
"""
import ctypes as ct
import os

import numpy as np

from . import _lib
from .api import Context, G1_BYTES, G2_BYTES, _dev_ptr, _host_ptr, NTT_IFFT


def _mont_fp_bytes(x):
    P = 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB
    return ((x << 384) % P).to_bytes(48, "little")


# the standard BLS12-381 generators as wire images (what bellman's `generate_random_parameters` would draw
# at random; any generator of the prime-order groups works for setup)
G1_GENERATOR = np.frombuffer(
    _mont_fp_bytes(0x17F1D3A73197D7942695638C4FA9AC0FC3688C4F9774B905A14E3A3F171BAC586C55E83FF97A1AEFFB3AF00ADB22C6BB)
    + _mont_fp_bytes(0x08B3F481E3AAA0F1A09E30ED741D8AE4FCF5E095D5D00AF600DB18CB2C04B3EDD03CC744A2888AE40CAA232946C5E7E1) + bytes(8),
    dtype=np.uint8).copy()
G2_GENERATOR = np.frombuffer(
    _mont_fp_bytes(0x024AA2B2F08F0A91260805272DC51051C6E47AD4FA403B02B4510B647AE3D1770BAC0326A805BBEFD48056C8C121BDB8)
    + _mont_fp_bytes(0x13E02B6052719F607DACD3A088274F65596BD0D09920B61AB5DA61BBDC7F5049334CF11213945D57E5AC7D055D042B7E)
    + _mont_fp_bytes(0x0CE5D527727D6E118CC9CDC6DA2E351AADFD9BAA8CBDD3A76D429A695160D12C923AC9CC3BACA289E193548608B82801)
    + _mont_fp_bytes(0x0606C4A02EA734CC32ACD2B02BC28B99CB3E287E85A763AF267492AB572E99AB3F370D275CEC1DA1AAA9075FF05F79BE) + bytes(8),
    dtype=np.uint8).copy()


class R1CS:
    """A, B, C as CSR (rowptr uint64[n+1], col uint32[nnz], val uint64[nnz,4] Montgomery)."""

    def __init__(self, num_inputs, num_aux, a, b, c):
        self.num_inputs, self.num_aux = int(num_inputs), int(num_aux)
        self.mats = []
        for rp, col, val in (a, b, c):
            rp = np.ascontiguousarray(rp, dtype=np.uint64)
            col = np.ascontiguousarray(col, dtype=np.uint32)
            val = np.ascontiguousarray(val, dtype=np.uint64).reshape(-1, 4)
            assert rp[0] == 0 and rp[-1] == len(col) == len(val)
            self.mats.append((rp, col, val))
        self.num_constraints = len(self.mats[0][0]) - 1
        assert all(len(m[0]) - 1 == self.num_constraints for m in self.mats)

    @property
    def num_vars(self):
        return self.num_inputs + self.num_aux

    @property
    def log_m(self):
        rows, e = self.num_constraints + self.num_inputs, 0
        while (1 << e) < rows:
            e += 1
        return e

    def density(self):
        """bellman's density trackers as index lists into z (zero coefficients skipped):
        a_idx = all inputs ++ aux present in A;  b_idx = inputs present in B ++ aux present in B."""
        nv = self.num_vars
        pres = []
        for rp, col, val in self.mats[:2]:
            d = np.zeros(nv, dtype=bool)
            nz = val.any(axis=1)
            d[col[nz]] = True
            pres.append(d)
        a_idx = np.concatenate([np.arange(self.num_inputs), self.num_inputs + np.nonzero(pres[0][self.num_inputs:])[0]])
        b_idx = np.nonzero(pres[1])[0]
        return a_idx.astype(np.uint32), b_idx.astype(np.uint32)

    def transposed(self, k):
        """matrix k (0/1/2) as CSR over variables (rows = variables, cols = constraints)."""
        rp, col, val = self.mats[k]
        rows = np.repeat(np.arange(self.num_constraints, dtype=np.uint32), np.diff(rp).astype(np.int64))
        order = np.argsort(col, kind="stable")
        counts = np.bincount(col, minlength=self.num_vars).astype(np.uint64)
        trp = np.zeros(self.num_vars + 1, dtype=np.uint64)
        np.cumsum(counts, out=trp[1:])
        return trp, rows[order].astype(np.uint32), val[order]


class BlockedR1CS:
    """A constraint system whose middle is one block of rows repeated `reps` times, stored once (bzk_r1cs_upload_blocked).
    Logical rows: head_rows explicit rows | reps copies of the tmpl_rows template rows | tail_rows explicit rows; each side's
    CSR (rowptr, col, val as in R1CS) holds the stored rows head | template | tail.  A template column c >= var_lo names
    c + k*var_stride in copy k; a smaller one names c in every copy.  An MPN update batch from
    NativeUpdateCircuit(..., blocked=True).blocked_r1cs() is this with one slot as the template."""

    def __init__(self, num_inputs, num_aux, head_rows, tmpl_rows, reps, tail_rows, var_lo, var_stride, a, b, c):
        self.num_inputs, self.num_aux = int(num_inputs), int(num_aux)
        self.head_rows, self.tmpl_rows, self.reps, self.tail_rows = int(head_rows), int(tmpl_rows), int(reps), int(tail_rows)
        self.var_lo, self.var_stride = int(var_lo), int(var_stride)
        stored = self.head_rows + self.tmpl_rows + self.tail_rows
        self.mats = []
        for rp, col, val in (a, b, c):
            rp = np.ascontiguousarray(rp, dtype=np.uint64)
            col = np.ascontiguousarray(col, dtype=np.uint32)
            val = np.ascontiguousarray(val, dtype=np.uint64).reshape(-1, 4)
            assert len(rp) == stored + 1 and rp[0] == 0 and rp[-1] == len(col) == len(val)
            self.mats.append((rp, col, val))
        self.num_constraints = self.head_rows + self.tmpl_rows * self.reps + self.tail_rows

    num_vars = R1CS.num_vars
    log_m = R1CS.log_m

    @property
    def blocks(self):
        return self.head_rows, self.tmpl_rows, self.reps, self.tail_rows, self.var_lo, self.var_stride

    def _parts(self, k):
        """matrix k's stored rows as (head, template, tail), each (row lengths, col, val)"""
        rp, col, val = self.mats[k]
        cut = [0, self.head_rows, self.head_rows + self.tmpl_rows, len(rp) - 1]
        return [(np.diff(rp[a:b + 1]), col[rp[a]:rp[b]], val[rp[a]:rp[b]]) for a, b in zip(cut, cut[1:])]

    def expand(self):
        """the explicit R1CS (numpy; for tests and small sizes: it materialises every copy)"""
        mats = []
        for k in range(3):
            (hl, hc, hv), (tl, tc, tv), (xl, xc, xv) = self._parts(k)
            slot = tc >= self.var_lo
            shifts = np.arange(self.reps, dtype=np.uint64) * np.uint64(self.var_stride)
            tcols = [np.where(slot, tc.astype(np.uint64) + sh, tc.astype(np.uint64)) for sh in shifts]
            lens = np.concatenate([hl] + [tl] * self.reps + [xl]).astype(np.uint64)
            rp = np.zeros(len(lens) + 1, dtype=np.uint64)
            np.cumsum(lens, out=rp[1:])
            col = np.concatenate([hc.astype(np.uint64)] + tcols + [xc.astype(np.uint64)]).astype(np.uint32)
            val = np.concatenate([hv] + [tv] * self.reps + [xv]).reshape(-1, 4)
            mats.append((rp, col, val))
        return R1CS(self.num_inputs, self.num_aux, *mats)

    def density(self):
        """R1CS.density of the expansion, from the blocks (every copy of a template slot column is present)"""
        pres = []
        for k in range(2):
            d = np.zeros(self.num_vars, dtype=bool)
            (hl, hc, hv), (tl, tc, tv), (xl, xc, xv) = self._parts(k)
            for c, v in ((hc, hv), (xc, xv)):
                d[c[v.any(axis=1)]] = True
            if self.reps:
                tc = tc[tv.any(axis=1)]
                d[tc[tc < self.var_lo]] = True
                rel = np.unique(tc[tc >= self.var_lo]).astype(np.int64)
                for k0 in range(0, self.reps, 64):
                    ks = np.arange(k0, min(k0 + 64, self.reps), dtype=np.int64) * self.var_stride
                    d[(rel[None, :] + ks[:, None]).reshape(-1)] = True
            pres.append(d)
        a_idx = np.concatenate([np.arange(self.num_inputs), self.num_inputs + np.nonzero(pres[0][self.num_inputs:])[0]])
        b_idx = np.nonzero(pres[1])[0]
        return a_idx.astype(np.uint32), b_idx.astype(np.uint32)


def _upload_r1cs(ctx, r1cs):
    """a bzk_r1cs handle for an R1CS (bzk_r1cs_upload) or a BlockedR1CS (bzk_r1cs_upload_blocked)"""
    h = ct.c_void_p()
    if isinstance(r1cs, BlockedR1CS):
        arr = lambda i: (ct.c_void_p * 3)(*[m[i].ctypes.data for m in r1cs.mats])
        ctx._check(ctx._l.bzk_r1cs_upload_blocked(ctx._h, r1cs.num_inputs, r1cs.num_aux, *r1cs.blocks, arr(0), arr(1), arr(2), ct.byref(h)))
        return h
    args = []
    for rp, col, val in r1cs.mats:
        args += [_host_ptr(rp), _host_ptr(col), _host_ptr(val)]
    ctx._check(ctx._l.bzk_r1cs_upload(ctx._h, r1cs.num_inputs, r1cs.num_aux, r1cs.num_constraints, *args, ct.byref(h)))
    return h


KEY_VECTORS = ("h", "l", "a", "b_g1", "b_g2")


def host_mask(host_vectors):
    """names from KEY_VECTORS (or "all") -> the bit mask of bzk_groth16_params_move / _read_placed"""
    if isinstance(host_vectors, str):
        host_vectors = KEY_VECTORS if host_vectors == "all" else (host_vectors,)
    mask = 0
    for name in host_vectors or ():
        if name not in KEY_VECTORS:
            raise ValueError(f"unknown key vector {name!r}; expected one of {KEY_VECTORS}")
        mask |= 1 << KEY_VECTORS.index(name)
    return mask


class ProvingKey:
    def __init__(self, ctx, handle, vk):
        self._ctx, self._h, self.vk = ctx, handle, vk

    def move(self, host_mask):
        """place the five vectors: bit v of host_mask (KEY_VECTORS order) set = pinned host memory, clear = device memory
        (bzk_groth16_params_move).  Host vectors are streamed to the device by every proof; proofs are unchanged."""
        self._ctx._check(self._ctx._l.bzk_groth16_params_move(self._ctx._h, self._h, int(host_mask)))
        return self

    def free(self):
        if self._h:
            self._ctx._check(self._ctx._l.bzk_groth16_params_free(self._ctx._h, self._h))
            self._h = None

    def precompute(self, max_levels=0, mem_fraction_percent=60):
        """fixed-base tables for the key's five base vectors (bzk_groth16_params_precompute); max_levels=0: as many
        levels (<= 16) as fit in mem_fraction_percent % of the free device memory.  Proofs are unchanged."""
        self._ctx._check(self._ctx._l.bzk_groth16_params_precompute(self._ctx._h, self._h, int(max_levels), int(mem_fraction_percent)))
        return self

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def proving_key_from_host(ctx, vk, h, l, a, b_g1, b_g2, table_levels=None):
    """vk: dict of wire images (alpha_g1, beta_g1, beta_g2, gamma_g2, delta_g1, delta_g2, ic[]);
    h/l/a/b_g1: [n,104] uint8, b_g2: [n,200] uint8 — bellman `Parameters` vectors.
    table_levels: fixed-base table levels of the key (1 = no tables, 0 = as many as fit in free device memory);
    None = the BZK_TABLE_LEVELS environment value, else 0.  Proofs are the same for every level count."""
    hb, lb, ab, b1b = (ctx.g1_bases(np.ascontiguousarray(x, dtype=np.uint8).reshape(-1, G1_BYTES)) for x in (h, l, a, b_g1))
    b2b = ctx.g2_bases(np.ascontiguousarray(b_g2, dtype=np.uint8).reshape(-1, G2_BYTES))
    return _make_pk(ctx, vk, hb, lb, ab, b1b, b2b, table_levels)


def _make_pk(ctx, vk, hb, lb, ab, b1b, b2b, table_levels=None, host_vectors=()):
    out = ct.c_void_p()
    pts = [np.ascontiguousarray(vk[k], dtype=np.uint8) for k in ("alpha_g1", "beta_g1", "beta_g2", "delta_g1", "delta_g2")]
    ctx._check(ctx._l.bzk_groth16_params_create(ctx._h, *[_host_ptr(p) for p in pts], hb._h, lb._h, ab._h, b1b._h, b2b._h, ct.byref(out)))
    for b in (hb, lb, ab, b1b, b2b):
        b._h = None  # adopted by the params handle
    pk = ProvingKey(ctx, out, vk)
    mask = host_mask(host_vectors)
    if mask:
        pk.move(mask)   # before the tables: host vectors have none
    return _with_tables(pk, table_levels)


def _with_tables(pk, table_levels):
    """the fixed-base table policy of proving_key_from_host"""
    if table_levels is None:
        lv = os.environ.get("BZK_TABLE_LEVELS")   # development override: 1 = no tables
        table_levels = int(lv) if lv else 0
    if table_levels != 1:
        pk.precompute(table_levels)
    return pk


# ------------------------------------------------------------------------------------------------
# bellman `Parameters` files (`Parameters::write` / `Parameters::read`, layout in csrc/params_io.cu)
# ------------------------------------------------------------------------------------------------
def _file_bytes(src):
    """a path (memory-mapped, never loaded whole) or a bytes-like object -> uint8 array"""
    if isinstance(src, (str, os.PathLike)):
        if os.path.getsize(src) == 0:
            return np.zeros(0, dtype=np.uint8)
        return np.memmap(src, dtype=np.uint8, mode="r")
    if isinstance(src, np.ndarray):
        return np.ascontiguousarray(src).reshape(-1).view(np.uint8)
    return np.frombuffer(memoryview(src).cast("B"), dtype=np.uint8)


PARAMS_FILE_INFO = np.dtype([(k, np.uint64) for k in ("n_ic", "n_h", "n_l", "n_a", "n_b_g1", "n_b_g2", "bytes")])


def parameters_info(src):
    """the header of a bellman `Parameters` file (bzk_groth16_params_file_info): point counts and the byte count they imply"""
    lib = _lib.load()
    buf = _file_bytes(src)
    out = np.zeros(1, dtype=PARAMS_FILE_INFO)
    st = lib.bzk_groth16_params_file_info(_host_ptr(buf) if buf.size else None, buf.size, _host_ptr(out))
    if st != 0:
        raise _lib.BzkError(st, "groth16_params_file_info")
    return {k: int(out[0][k]) for k in PARAMS_FILE_INFO.names}


def read_parameters(ctx, src, checked=True, table_levels=None, host_vectors=()):
    """bellman `Parameters::read(src, checked)` onto the GPU -> (ProvingKey, vk dict of wire images).  checked=True tests
    every point for the curve equation and the prime-order subgroup (on the GPU); the verifying key is checked either way.
    table_levels: as in proving_key_from_host (host vectors stay untabled).  host_vectors: names from KEY_VECTORS, or
    "all", read into pinned host memory instead of the device (bzk_groth16_params_read_placed), so a key larger than the
    device can be read.  A refused file raises BzkError naming the first bad point."""
    buf = _file_bytes(src)
    n_ic = parameters_info(buf)["n_ic"]
    g1 = {k: np.zeros(G1_BYTES, np.uint8) for k in ("alpha_g1", "beta_g1", "delta_g1")}
    g2 = {k: np.zeros(G2_BYTES, np.uint8) for k in ("beta_g2", "gamma_g2", "delta_g2")}
    ic = np.zeros((max(n_ic, 1), G1_BYTES), np.uint8)
    out = ct.c_void_p()
    ctx._check(ctx._l.bzk_groth16_params_read_placed(ctx._h, _host_ptr(buf), buf.size, int(bool(checked)), _host_ptr(g1["alpha_g1"]),
                                                     _host_ptr(g1["beta_g1"]), _host_ptr(g2["beta_g2"]), _host_ptr(g2["gamma_g2"]),
                                                     _host_ptr(g1["delta_g1"]), _host_ptr(g2["delta_g2"]), _host_ptr(ic), n_ic,
                                                     host_mask(host_vectors), ct.byref(out)))
    vk = dict(g1, **g2, ic=ic[:n_ic])
    return _with_tables(ProvingKey(ctx, out, vk), table_levels), vk


def write_parameters(ctx, pk, dest=None):
    """bellman `Parameters::write` of a key (level 0 of each vector, whatever its tables) -> a uint8 array, or into the file
    `dest` (memory-mapped at its exact size), returning the path."""
    ic = np.ascontiguousarray(pk.vk["ic"], dtype=np.uint8).reshape(-1, G1_BYTES)
    gamma = np.ascontiguousarray(pk.vk["gamma_g2"], dtype=np.uint8)
    n = ct.c_size_t()
    args = (ctx._h, pk._h, _host_ptr(gamma), _host_ptr(ic), len(ic))
    ctx._check(ctx._l.bzk_groth16_params_write(*args, None, 0, ct.byref(n)))
    if dest is None:
        out = np.empty(n.value, dtype=np.uint8)
        ctx._check(ctx._l.bzk_groth16_params_write(*args, _host_ptr(out), out.size, ct.byref(n)))
        return out
    out = np.memmap(dest, dtype=np.uint8, mode="w+", shape=(n.value,))
    ctx._check(ctx._l.bzk_groth16_params_write(*args, _host_ptr(out), out.size, ct.byref(n)))
    out.flush()
    del out
    return dest


class Prover:
    """One circuit on one GPU: the R1CS (an R1CS or a BlockedR1CS) and (optionally) its proving key resident in HBM."""

    def __init__(self, ctx: Context, r1cs):
        self.ctx, self.r1cs = ctx, r1cs
        self._h = _upload_r1cs(ctx, r1cs)
        shp = np.zeros(5, dtype=np.uint64)
        ctx._check(ctx._l.bzk_r1cs_shape(self._h, _host_ptr(shp)))
        self.log_m, self.h_len, self.l_len, self.a_len, self.b_len = (int(x) for x in shp)

    def free(self):
        if self._h:
            self.ctx._check(self.ctx._l.bzk_r1cs_free(self.ctx._h, self._h))
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def _host_witness(self, inputs, aux):
        inputs = np.ascontiguousarray(inputs, dtype=np.uint64).reshape(-1, 4)
        aux = np.ascontiguousarray(aux, dtype=np.uint64).reshape(-1, 4)
        assert len(inputs) == self.r1cs.num_inputs and len(aux) == self.r1cs.num_aux
        return inputs, aux

    def prove(self, pk: ProvingKey, inputs, aux, r, s, check_satisfied=True):
        """inputs [num_inputs,4] (inputs[0] = R(1)), aux [num_aux,4], r/s [4] — Montgomery.
        Returns (proof_bytes[387], (a[104], b[200], c[104]))."""
        inputs, aux = self._host_witness(inputs, aux)
        return self._prove(self.ctx._l.bzk_groth16_prove, pk, _host_ptr(inputs), _host_ptr(aux), r, s, check_satisfied)

    def prove_dev(self, pk: ProvingKey, d_inputs, d_aux, r, s, check_satisfied=True):
        """`prove` with the witness already resident: d_inputs [num_inputs,4], d_aux [num_aux,4] CUDA int64
        tensors of Montgomery images (e.g. written by mpn.gpu_witness)."""
        assert d_inputs.numel() == 4 * self.r1cs.num_inputs and d_aux.numel() == 4 * self.r1cs.num_aux
        return self._prove(self.ctx._l.bzk_groth16_prove_dev, pk, _dev_ptr(d_inputs), _dev_ptr(d_aux), r, s, check_satisfied)

    def _prove(self, entry, pk, p_inputs, p_aux, r, s, check_satisfied):
        r = np.ascontiguousarray(r, dtype=np.uint64).reshape(4)
        s = np.ascontiguousarray(s, dtype=np.uint64).reshape(4)
        pa, pb, pc = np.zeros(G1_BYTES, np.uint8), np.zeros(G2_BYTES, np.uint8), np.zeros(G1_BYTES, np.uint8)
        c = self.ctx
        c._check(entry(c._h, pk._h, self._h, p_inputs, p_aux, _host_ptr(r), _host_ptr(s), int(check_satisfied),
                       _host_ptr(pa), _host_ptr(pb), _host_ptr(pc)))
        return _proof_blob(c._l, pa, pb, pc), (pa, pb, pc)

    STAGES = ("z_spmv_done", "quotient_ntts_done", "h_msm_done", "l_msm_done", "a_msm_done", "b_g1_msm_done", "b_g2_msm_done")

    def stage_ms(self):
        """CUDA-event marks of the last prove call made with ctx.set_timing(True): ms since the call's first kernel at
        which each stage finished (main stream: z+SpMV, quotient NTTs, h sum; side streams: l, a, b_g1, b_g2 sums)."""
        out = np.zeros(8, dtype=np.float32)
        ok = self.ctx._l.bzk_groth16_stage_ms(self.ctx._h, _host_ptr(out))
        return {k: float(out[i + 1]) for i, k in enumerate(self.STAGES)} if ok == 1 else None

    def _partials(self, entry, spk, *args):
        """entry(ctx, spk, r1cs, *args, a_sum, b1_sum, b2_sum, hl_sum) -> the four partial sums (a, b_g1, b_g2, h+l wire images)"""
        sums = np.zeros(G1_BYTES, np.uint8), np.zeros(G1_BYTES, np.uint8), np.zeros(G2_BYTES, np.uint8), np.zeros(G1_BYTES, np.uint8)
        c = self.ctx
        c._check(entry(c._h, spk._h, self._h, *args, *[_host_ptr(x) for x in sums]))
        return sums

    def prove_partial(self, spk: ProvingKey, inputs, aux, check_satisfied=True):
        """this rank's four partial sums (a, b_g1, b_g2, h+l wire images) under the base-sharded key `spk`
        (shard_proving_key).  inputs/aux: host arrays, or CUDA tensors for a resident witness."""
        on_dev = hasattr(inputs, "is_cuda")
        if on_dev:
            pi, pa_ = _dev_ptr(inputs), _dev_ptr(aux)
        else:
            inputs, aux = self._host_witness(inputs, aux)
            pi, pa_ = _host_ptr(inputs), _host_ptr(aux)
        return self._partials(self.ctx._l.bzk_groth16_prove_partial, spk, pi, pa_, int(on_dev), int(check_satisfied))

    def shard_begin(self, spk: ProvingKey, d_inputs, d_aux, evals):
        """first half of the split sharded schedule: evals = [tensor | None] * 3 — the evaluation vectors (a, b, c) this rank owns,
        as CUDA int64 tensors [2^log_m, 4] that receive them on the coset; the four witness sums start on their streams."""
        c = self.ctx
        ptrs = (ct.c_void_p * 3)(*[_dev_ptr(e) if e is not None else None for e in evals])
        mask = sum(1 << k for k, e in enumerate(evals) if e is not None)
        c._check(c._l.bzk_groth16_shard_begin(c._h, spk._h, self._h, _dev_ptr(d_inputs), _dev_ptr(d_aux), 1, mask, ptrs))

    def h_combine(self, d_a, d_b, d_c):
        """(a*b - c)/Z from the three vectors on the coset, back to coefficients: d_a <- h"""
        c = self.ctx
        c._check(c._l.bzk_groth16_h_combine_dev(c._h, _dev_ptr(d_a), _dev_ptr(d_b), _dev_ptr(d_c), self.log_m))

    def shard_finish(self, spk: ProvingKey, d_h_shard):
        """second half: the h sum over this rank's slice of the quotient -> (a, b_g1, b_g2, h+l) partial sums"""
        return self._partials(self.ctx._l.bzk_groth16_shard_finish, spk, _dev_ptr(d_h_shard) if d_h_shard is not None else None)


def shard_proving_key(ctx, pk: ProvingKey, log_m, rank, world):
    """rank's base-sharded key from a full key produced by `setup_gpu` on this GPU: contiguous ranges
    [len*rank/world, len*(rank+1)/world) of h (first 2^log_m - 1 entries), l, a, b_g1, b_g2 (SURVEY.md §8e)."""
    from .dist import shard_range
    img = pk.device_images

    def sl(t, n):
        lo, hi = shard_range(n, rank, world)
        return t[lo:hi].contiguous(), hi - lo

    m1 = (1 << log_m) - 1
    parts = {k: sl(img[k], m1 if k == "h" else img[k].shape[0]) for k in ("h", "l", "a", "b_g1", "b_g2")}
    hb, lb, ab, b1b = (ctx.g1_bases_from_dev(*parts[k]) for k in ("h", "l", "a", "b_g1"))
    b2b = ctx.g2_bases_from_dev(*parts["b_g2"])
    ctx.synchronize()
    spk = _make_pk(ctx, pk.vk, hb, lb, ab, b1b, b2b)
    ctx._check(ctx._l.bzk_groth16_params_set_shard(spk._h, rank, world))
    spk.rank, spk.world = rank, world
    return spk


def finalize(vk, partials, r, s):
    """tail of bellman `create_proof` from the summed answers (a, b_g1, b_g2, h+l) -> (blob[387], points)."""
    lib = _lib.load()
    pts = [np.ascontiguousarray(vk[k], dtype=np.uint8) for k in ("alpha_g1", "beta_g1", "beta_g2", "delta_g1", "delta_g2")]
    a_sum, b1_sum, b2_sum, hl_sum = (np.ascontiguousarray(x, dtype=np.uint8) for x in partials)
    r = np.ascontiguousarray(r, dtype=np.uint64).reshape(4)
    s = np.ascontiguousarray(s, dtype=np.uint64).reshape(4)
    pa, pb, pc = np.zeros(G1_BYTES, np.uint8), np.zeros(G2_BYTES, np.uint8), np.zeros(G1_BYTES, np.uint8)
    st = lib.bzk_groth16_finalize(*[_host_ptr(p) for p in pts], _host_ptr(a_sum), _host_ptr(b1_sum), _host_ptr(b2_sum), _host_ptr(hl_sum),
                                  _host_ptr(r), _host_ptr(s), _host_ptr(pa), _host_ptr(pb), _host_ptr(pc))
    if st != 0:
        raise _lib.BzkError(st, "groth16_finalize")
    return _proof_blob(lib, pa, pb, pc), (pa, pb, pc)


def _proof_blob(lib, pa, pb, pc):
    """the 387-byte bincode image of `Groth16Proof {a, b, c}` (bzk_groth16_proof_bytes)"""
    blob = np.zeros(387, np.uint8)
    st = lib.bzk_groth16_proof_bytes(_host_ptr(pa), _host_ptr(pb), _host_ptr(pc), _host_ptr(blob))
    if st != 0:
        raise _lib.BzkError(st, "groth16_proof_bytes")
    return blob


def allgather_partials(partials, group=None, device="cpu"):
    """one all-gather of world x 512 B, then the local folds: every rank returns the four summed answers."""
    import torch
    import torch.distributed as dist
    from .dist import fold
    a_sum, b1_sum, b2_sum, hl_sum = (np.ascontiguousarray(x, dtype=np.uint8) for x in partials)
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return a_sum, b1_sum, b2_sum, hl_sum
    world = dist.get_world_size(group)
    mine = torch.from_numpy(np.concatenate([a_sum, b1_sum, hl_sum, b2_sum])).to(device)  # 104*3 + 200 = 512 B
    gathered = torch.empty(world * 512, dtype=torch.uint8, device=device)
    dist.all_gather_into_tensor(gathered, mine, group=group)
    g = gathered.cpu().numpy().reshape(world, 512)
    return (fold(g[:, 0:104], "g1"), fold(g[:, 104:208], "g1"), fold(g[:, 312:512], "g2"), fold(g[:, 208:312], "g1"))


class SplitShardedProver:
    """Schedule (S) with the quotient pipeline split over the ranks (include/bzk.h, bzk_groth16_shard_begin): evaluation vector
    s belongs to rank s mod world, rank 3 mod world combines them and deals the quotient's coefficients out in slices.  The
    vectors move with NCCL point-to-point operations (torch.distributed); buffers are allocated once and reused."""

    def __init__(self, prover, spk, rank, world, device, group=None):
        import torch
        from .dist import shard_range
        self.pr, self.spk, self.rank, self.world, self.dev, self.group = prover, spk, rank, world, device, group
        self.m = 1 << prover.log_m
        self.owner = [s % world for s in range(3)]
        self.comb = 3 % world
        need = [self.owner[s] == rank or self.comb == rank for s in range(3)]
        self.buf = [torch.empty((self.m, 4), dtype=torch.int64, device=device) if n else None for n in need]
        self.ranges = [shard_range(self.m - 1, k, world) for k in range(world)]
        lo, hi = self.ranges[rank]
        self.h_mine = None if self.comb == rank else torch.empty((hi - lo, 4), dtype=torch.int64, device=device)

    def partials(self, d_in, d_aux):
        import torch
        import torch.distributed as dist
        pr, rank, comb = self.pr, self.rank, self.comb
        pr.shard_begin(self.spk, d_in, d_aux, [self.buf[s] if self.owner[s] == rank else None for s in range(3)])
        ops = []
        for s in range(3):
            if self.owner[s] == comb:
                continue
            if rank == self.owner[s]:
                ops.append(dist.P2POp(dist.isend, self.buf[s], comb, self.group))
            elif rank == comb:
                ops.append(dist.P2POp(dist.irecv, self.buf[s], self.owner[s], self.group))
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        ops = []
        if rank == comb:
            torch.cuda.current_stream(self.dev).synchronize()      # the received vectors are complete
            pr.h_combine(*self.buf)                                   # on the context's stream
            pr.ctx.synchronize()
            h = self.buf[0]
            for k, (lo, hi) in enumerate(self.ranges):
                if k != rank and hi > lo:
                    ops.append(dist.P2POp(dist.isend, h[lo:hi], k, self.group))
            lo, hi = self.ranges[rank]
            mine = h[lo:hi]
        else:
            if self.h_mine.shape[0]:
                ops.append(dist.P2POp(dist.irecv, self.h_mine, comb, self.group))
            mine = self.h_mine
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        torch.cuda.current_stream(self.dev).synchronize()
        return pr.shard_finish(self.spk, mine)


def verify(vk, public_inputs, proof_points):
    """`groth16_verify` (/root/reference/src/zk/groth16/mod.rs:67-121): vk = dict of wire images
    (alpha_g1, beta_g2, gamma_g2, delta_g2, ic[n+1]), public_inputs [n,4] Montgomery (without ONE),
    proof_points = (a[104], b[200], c[104]).  Host pairing in libbzk; no GPU needed."""
    lib = _lib.load()
    ic = np.ascontiguousarray(vk["ic"], dtype=np.uint8).reshape(-1, G1_BYTES)
    pub = np.ascontiguousarray(public_inputs, dtype=np.uint64).reshape(-1, 4)
    pts = [np.ascontiguousarray(vk[k], dtype=np.uint8) for k in ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2")]
    a, b, c = (np.ascontiguousarray(x, dtype=np.uint8) for x in proof_points)
    st = lib.bzk_groth16_verify(*[_host_ptr(p) for p in pts], _host_ptr(ic), len(ic), _host_ptr(pub), len(pub),
                                _host_ptr(a), _host_ptr(b), _host_ptr(c))
    if st < 0:
        raise _lib.BzkError(st, "groth16_verify")
    return bool(st)


def vk_to_bincode(vk):
    """1460-byte-style bincode image of `Groth16VerifyingKey` (/root/reference/src/zk/groth16/mod.rs:22-31)."""
    ic = np.ascontiguousarray(vk["ic"], dtype=np.uint8).reshape(-1, G1_BYTES)
    parts = [np.asarray(vk["alpha_g1"])[:97], np.asarray(vk["beta_g1"])[:97], np.asarray(vk["beta_g2"])[:193],
             np.asarray(vk["gamma_g2"])[:193], np.asarray(vk["delta_g1"])[:97], np.asarray(vk["delta_g2"])[:193],
             np.frombuffer(len(ic).to_bytes(8, "little"), dtype=np.uint8)] + [row[:97] for row in ic]
    return np.concatenate([np.asarray(p, dtype=np.uint8) for p in parts])


def verify_bytes(vk_blob, public_inputs, proof387):
    """`check_proof` on the reference's byte images."""
    lib = _lib.load()
    as_u8 = lambda b: np.frombuffer(bytes(b), dtype=np.uint8) if isinstance(b, (bytes, bytearray, memoryview)) else np.ascontiguousarray(b, dtype=np.uint8)
    vk_blob, proof387 = as_u8(vk_blob), as_u8(proof387)
    pub = np.ascontiguousarray(public_inputs, dtype=np.uint64).reshape(-1, 4)
    st = lib.bzk_groth16_verify_bytes(_host_ptr(vk_blob), vk_blob.size, _host_ptr(pub), len(pub), _host_ptr(proof387))
    if st < 0:
        raise _lib.BzkError(st, "groth16_verify_bytes")
    return bool(st)


def zkproof_blob(proof_bytes):
    """391-byte bincode of `ZkProof::Groth16(Box<Groth16Proof>)` — u32 tag 0 + 387 B
    (/root/reference/src/zk/mod.rs:646-651)."""
    return np.concatenate([np.zeros(4, np.uint8), np.asarray(proof_bytes, dtype=np.uint8)])


# ------------------------------------------------------------------------------------------------
# trusted setup on the GPU (bellman `generate_parameters`, explicit toxic waste)
# ------------------------------------------------------------------------------------------------
def setup_gpu(ctx: Context, r1cs, toxic, g1_image, g2_image, table_levels=None, host_vectors=()):
    """toxic = [tau, alpha, beta, gamma, delta] as [5,4] Montgomery; g1/g2: generator wire images.
    Returns (ProvingKey, vk dict).  All field/group work runs in libbzk kernels; numpy only moves
    and reorders data.  table_levels: as in proving_key_from_host.  host_vectors: as in read_parameters; for a
    BlockedR1CS each such vector moves to host memory as soon as it is built, so the device holds one of them at a time.
    r1cs: an R1CS (the key keeps its wire images in pk.device_images), or a BlockedR1CS: the Lagrange columns come from
    bzk_r1cs_columns_dev, each vector is multiplied straight into its resident form and every temporary is dropped before
    the next vector is made, so the device never holds a vector twice; no wire images are kept.  Both give the same key."""
    import torch
    # torch slicing / indexing kernels and libbzk kernels interleave below: put both on one stream
    ctx.use_torch_stream()
    try:
        return _setup_gpu(ctx, r1cs, toxic, g1_image, g2_image, table_levels, host_vectors)
    finally:
        torch.cuda.synchronize()
        ctx.use_own_stream()


def _setup_gpu(ctx, r1cs, toxic, g1_image, g2_image, table_levels, host_vectors):
    import torch
    t = torch
    toxic = np.ascontiguousarray(toxic, dtype=np.uint64).reshape(5, 4)
    ni, na, nc, nv = r1cs.num_inputs, r1cs.num_aux, r1cs.num_constraints, r1cs.num_vars
    log_m = r1cs.log_m
    m = 1 << log_m

    def dev(a):
        return t.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()

    def rep(x, n):  # n copies of one field element on the device
        return dev(np.repeat(np.asarray(x, dtype=np.uint64).reshape(1, 4), n, axis=0))

    def mul(a, b):
        o = t.empty_like(a)
        ctx.fr_binop_dev(2, a, b, o, a.shape[0])
        return o

    def add(a, b):
        o = t.empty_like(a)
        ctx.fr_binop_dev(0, a, b, o, a.shape[0])
        return o

    one = _fr_one()
    # powers of tau by repeated squaring of index halves: pw[i] = tau^i
    pw = np.zeros((m, 4), dtype=np.uint64)
    pw[0] = one
    d_pw = dev(pw)
    cur, step = 1, rep(toxic[0], m)  # step holds tau^(cur) broadcast
    while cur < m:
        n = min(cur, m - cur)
        seg = mul(d_pw[:n].contiguous(), step[:n].contiguous())
        d_pw[cur:cur + n] = seg
        step = mul(step, step)
        cur *= 2
    # scalar helpers on tiny vectors (1 element) — still libbzk arithmetic
    def s_mul(x, y):
        return mul(dev(x.reshape(1, 4)), dev(y.reshape(1, 4))).cpu().numpy().view(np.uint64).reshape(4)

    tau_m = s_mul(d_pw[m - 1:m].cpu().numpy().view(np.uint64).reshape(4), toxic[0])
    o1 = t.empty((1, 4), dtype=t.int64, device="cuda")
    ctx.fr_binop_dev(1, dev(tau_m.reshape(1, 4)), dev(one.reshape(1, 4)), o1, 1)
    zt = o1.cpu().numpy().view(np.uint64).reshape(4)                      # tau^m - 1
    dinv, ginv = _fr_inv_gpu(ctx, toxic[4]), _fr_inv_gpu(ctx, toxic[3])
    zd = s_mul(zt, dinv)
    h_k = mul(d_pw[: m - 1].contiguous(), rep(zd, m - 1))                  # tau^i Z(tau)/delta
    ctx.ntt_dev(d_pw, log_m, NTT_IFFT)                                     # d_pw <- L_j(tau)
    if isinstance(r1cs, BlockedR1CS):
        step = seg = None
        return _setup_blocked(ctx, r1cs, toxic, g1_image, g2_image, table_levels, host_vectors, d_pw, h_k, dinv, ginv, dev, rep, mul, add)
    lag = d_pw
    cols = []
    for k in range(3):
        trp, tcol, tval = r1cs.transposed(k)
        out = t.empty((nv, 4), dtype=t.int64, device="cuda")
        d_trp, d_tcol, d_tval = dev(trp), dev_u32(t, tcol), dev(tval)
        ctx._check(ctx._l.bzk_csr_spmv_dev(ctx._h, _p(d_trp), _p(d_tcol),
                                            _p(d_tval), nv, _p(lag), _p(out)))
        ctx.synchronize()
        cols.append(out)
    at, bt, ctv = cols
    # Input(i) * 0 = 0 rows add L_{nc+i}(tau) to A_i
    at[:ni] = add(at[:ni].contiguous(), lag[nc:nc + ni].contiguous())
    ext = add(add(mul(at, rep(toxic[2], nv)), mul(bt, rep(toxic[1], nv))), ctv)
    ext_ic = mul(ext[:ni].contiguous(), rep(ginv, ni))
    ext_l = mul(ext[ni:].contiguous(), rep(dinv, na)) if na else ext[ni:]
    a_idx, b_idx = r1cs.density()

    def g1_mul(scal):
        n = scal.shape[0]
        out = t.empty((max(n, 1), G1_BYTES), dtype=t.uint8, device="cuda")
        ctx._check(ctx._l.bzk_g1_fixed_base_mul_dev(ctx._h, _host_ptr(g1_image), _p(scal.contiguous()), n, _p(out)))
        return out[:n]

    def g2_mul(scal):
        n = scal.shape[0]
        out = t.empty((max(n, 1), G2_BYTES), dtype=t.uint8, device="cuda")
        ctx._check(ctx._l.bzk_g2_fixed_base_mul_dev(ctx._h, _host_ptr(g2_image), _p(scal.contiguous()), n, _p(out)))
        return out[:n]

    g1_image = np.ascontiguousarray(g1_image, dtype=np.uint8)
    g2_image = np.ascontiguousarray(g2_image, dtype=np.uint8)
    ai = t.from_numpy(a_idx.astype(np.int64)).cuda()
    bi = t.from_numpy(b_idx.astype(np.int64)).cuda()
    h_pts, l_pts = g1_mul(h_k), g1_mul(ext_l)
    a_pts, b1_pts, b2_pts = g1_mul(at[ai]), g1_mul(bt[bi]), g2_mul(bt[bi])
    ic = g1_mul(ext_ic).cpu().numpy()
    tox = dev(toxic)
    vk_g1 = g1_mul(tox[[1, 2, 4]]).cpu().numpy()      # alpha, beta, delta
    vk_g2 = g2_mul(tox[[2, 3, 4]]).cpu().numpy()      # beta, gamma, delta
    ctx.synchronize()
    vk = {"alpha_g1": vk_g1[0], "beta_g1": vk_g1[1], "delta_g1": vk_g1[2],
          "beta_g2": vk_g2[0], "gamma_g2": vk_g2[1], "delta_g2": vk_g2[2], "ic": ic}
    hb = ctx.g1_bases_from_dev(h_pts.contiguous(), m - 1)
    lb = ctx.g1_bases_from_dev(l_pts.contiguous() if na else t.empty((1, G1_BYTES), dtype=t.uint8, device="cuda"), na)
    ab = ctx.g1_bases_from_dev(a_pts.contiguous(), len(a_idx))
    b1b = ctx.g1_bases_from_dev(b1_pts.contiguous() if len(b_idx) else t.empty((1, G1_BYTES), dtype=t.uint8, device="cuda"), len(b_idx))
    b2b = ctx.g2_bases_from_dev(b2_pts.contiguous() if len(b_idx) else t.empty((1, G2_BYTES), dtype=t.uint8, device="cuda"), len(b_idx))
    ctx.synchronize()
    host = {"h": h_pts, "l": l_pts, "a": a_pts, "b_g1": b1_pts, "b_g2": b2_pts}
    pk = _make_pk(ctx, vk, hb, lb, ab, b1b, b2b, table_levels, host_vectors)
    pk.device_images = host  # wire images kept for tests / export
    return pk, vk


def _setup_blocked(ctx, r1cs, toxic, g1_image, g2_image, table_levels, host_vectors, lag, h_k, dinv, ginv, dev, rep, mul, add):
    """the rest of _setup_gpu for a BlockedR1CS (lag = L_j(tau), h_k = tau^i Z(tau)/delta): the same key, built one
    resident vector at a time"""
    import torch
    t = torch
    from .api import G1Bases, G2Bases
    ni, na, nc, nv, m = r1cs.num_inputs, r1cs.num_aux, r1cs.num_constraints, r1cs.num_vars, 1 << r1cs.log_m
    g1_image = np.ascontiguousarray(g1_image, dtype=np.uint8)
    g2_image = np.ascontiguousarray(g2_image, dtype=np.uint8)

    on_host = host_mask(host_vectors)

    def bases(kind, scal, name):
        out = ct.c_void_p()
        n = scal.shape[0]
        fn = ctx._l.bzk_g1_bases_fixed_base_mul if kind == 1 else ctx._l.bzk_g2_bases_fixed_base_mul
        ctx._check(fn(ctx._h, _host_ptr(g1_image if kind == 1 else g2_image), _p(scal.contiguous()) if n else None, n, ct.byref(out)))
        ctx.synchronize()
        b = (G1Bases if kind == 1 else G2Bases)(ctx, out)
        return b.move_to_host() if on_host & host_mask(name) else b

    def drop():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()   # hand freed temporaries back before libbzk allocates the next vector

    hb = bases(1, h_k, "h")
    del h_k
    drop()
    h = _upload_r1cs(ctx, r1cs)
    try:
        cols = []
        for k in range(3):
            out = t.empty((nv, 4), dtype=t.int64, device="cuda")
            ctx._check(ctx._l.bzk_r1cs_columns_dev(ctx._h, h, k, _p(lag), _p(out)))
            cols.append(out)
        ctx.synchronize()
    finally:
        ctx._check(ctx._l.bzk_r1cs_free(ctx._h, h))
    at, bt, ctv = cols
    del cols
    at[:ni] = add(at[:ni].contiguous(), lag[nc:nc + ni].contiguous())   # the Input(i) * 0 = 0 rows
    del lag
    ext = add(add(mul(at, rep(toxic[2], nv)), mul(bt, rep(toxic[1], nv))), ctv)
    del ctv
    ext_ic = mul(ext[:ni].contiguous(), rep(ginv, ni))
    ext_l = mul(ext[ni:].contiguous(), rep(dinv, na)) if na else ext[ni:]
    del ext
    drop()
    lb = bases(1, ext_l, "l")
    del ext_l
    drop()
    a_idx, b_idx = r1cs.density()
    ab = bases(1, at[t.from_numpy(a_idx.astype(np.int64)).cuda()], "a")
    del at
    drop()
    bsc = bt[t.from_numpy(b_idx.astype(np.int64)).cuda()]
    del bt
    drop()
    b1b = bases(1, bsc, "b_g1")
    b2b = bases(2, bsc, "b_g2")
    del bsc
    drop()

    def images(kind, scal):
        n = scal.shape[0]
        w = G1_BYTES if kind == 1 else G2_BYTES
        out = t.empty((max(n, 1), w), dtype=t.uint8, device="cuda")
        fn = ctx._l.bzk_g1_fixed_base_mul_dev if kind == 1 else ctx._l.bzk_g2_fixed_base_mul_dev
        ctx._check(fn(ctx._h, _host_ptr(g1_image if kind == 1 else g2_image), _p(scal.contiguous()), n, _p(out)))
        return out[:n].cpu().numpy()

    tox = dev(toxic)
    ic = images(1, ext_ic)
    vk_g1 = images(1, tox[[1, 2, 4]])      # alpha, beta, delta
    vk_g2 = images(2, tox[[2, 3, 4]])      # beta, gamma, delta
    vk = {"alpha_g1": vk_g1[0], "beta_g1": vk_g1[1], "delta_g1": vk_g1[2],
          "beta_g2": vk_g2[0], "gamma_g2": vk_g2[1], "delta_g2": vk_g2[2], "ic": ic}
    return _make_pk(ctx, vk, hb, lb, ab, b1b, b2b, table_levels, host_vectors), vk


def _p(tensor):
    return ct.c_void_p(tensor.data_ptr())


def dev_u32(t, a):
    return t.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


def _fr_one():
    # R mod r (Montgomery one), little-endian u64 limbs
    return np.array([0x00000001FFFFFFFE, 0x5884B7FA00034802, 0x998C4FEFECBC4FF5, 0x1824B159ACC5056F], dtype=np.uint64)


def _fr_inv_gpu(ctx, x):
    """x^(r-2) by square-and-multiply with libbzk's Fr product (setup only: two inversions)."""
    import torch
    t = torch
    R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
    e = R - 2
    base = t.from_numpy(np.asarray(x, dtype=np.uint64).reshape(1, 4).view(np.int64)).cuda()
    acc = t.from_numpy(_fr_one().reshape(1, 4).view(np.int64)).cuda()
    out = t.empty_like(acc)
    for bit in bin(e)[2:]:
        ctx.fr_binop_dev(2, acc, acc, out, 1)
        acc, out = out, acc
        if bit == "1":
            ctx.fr_binop_dev(2, acc, base, out, 1)
            acc, out = out, acc
    ctx.synchronize()
    return acc.cpu().numpy().view(np.uint64).reshape(4)


class PreparedVerifyingKey:
    """bellman `PreparedVerifyingKey` held across verifications (bzk_groth16_pvk_*): e(alpha,beta) and the line
    coefficients of gamma / delta are computed once.  `vk`: the 878+97n-byte bincode image or a dict of wire images."""

    def __init__(self, vk):
        self._l = _lib.load()
        blob = np.ascontiguousarray(vk_to_bincode(vk) if isinstance(vk, dict) else vk, dtype=np.uint8)
        h = ct.c_void_p()
        st = self._l.bzk_groth16_pvk_from_bytes(_host_ptr(blob), blob.size, ct.byref(h))
        if st != 0:
            raise _lib.BzkError(st, "groth16_pvk_from_bytes")
        self._h = h

    def free(self):
        if self._h:
            self._l.bzk_groth16_pvk_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def verify(self, public_inputs, proof387):
        """one proof as its 387-byte `Groth16Proof` image"""
        p = np.ascontiguousarray(proof387, dtype=np.uint8).reshape(387)
        a, b, c = np.zeros(G1_BYTES, np.uint8), np.zeros(G2_BYTES, np.uint8), np.zeros(G1_BYTES, np.uint8)
        a[:97], b[:193], c[:97] = p[:97], p[97:290], p[290:]
        return self.verify_points(public_inputs, (a, b, c))

    def verify_points(self, public_inputs, proof_points):
        pub = np.ascontiguousarray(public_inputs, dtype=np.uint64).reshape(-1, 4)
        a, b, c = (np.ascontiguousarray(x, dtype=np.uint8) for x in proof_points)
        st = self._l.bzk_groth16_verify_prepared(self._h, _host_ptr(pub), len(pub), _host_ptr(a), _host_ptr(b), _host_ptr(c))
        if st < 0:
            raise _lib.BzkError(st, "groth16_verify_prepared")
        return bool(st)

    def verify_batch_gpu(self, ctx, public_inputs, proofs387, seed=None):
        """verify_batch with the per-proof Miller loops on the GPU (bzk_groth16_verify_batch_dev): same verdicts."""
        proofs = np.ascontiguousarray(proofs387, dtype=np.uint8).reshape(-1, 387)
        m = len(proofs)
        if m == 0:
            return True, np.zeros(0, dtype=bool)
        pub = np.ascontiguousarray(public_inputs, dtype=np.uint64).reshape(m, -1, 4)
        each = np.zeros(m, dtype=np.uint8)
        if seed is None:
            seed = int.from_bytes(os.urandom(8), "little")
        st = self._l.bzk_groth16_verify_batch_dev(ctx._h, self._h, _host_ptr(pub), pub.shape[1], _host_ptr(proofs), m, seed, _host_ptr(each))
        if st < 0:
            raise _lib.BzkError(st, "groth16_verify_batch_dev")
        return bool(st), each.astype(bool)

    def verify_batch(self, public_inputs, proofs387, seed=None, threads=0):
        """public_inputs [m, n, 4] Montgomery, proofs387 [m, 387] -> (all_ok, ok_each[m]).  One final exponentiation for
        the batch (random linear combination with 127-bit multipliers from `seed`, default os.urandom)."""
        pub = np.ascontiguousarray(public_inputs, dtype=np.uint64)
        proofs = np.ascontiguousarray(proofs387, dtype=np.uint8).reshape(-1, 387)
        m = len(proofs)
        if m == 0:
            return True, np.zeros(0, dtype=bool)
        pub = pub.reshape(m, -1, 4)
        each = np.zeros(max(m, 1), dtype=np.uint8)
        if seed is None:
            seed = int.from_bytes(os.urandom(8), "little")
        st = self._l.bzk_groth16_verify_batch(self._h, _host_ptr(pub), pub.shape[1], _host_ptr(proofs), m, seed, int(threads), _host_ptr(each))
        if st < 0:
            raise _lib.BzkError(st, "groth16_verify_batch")
        return bool(st), each[:m].astype(bool)
