"""Python host layer over the libbzk C ABI (see include/bzk.h for the contract of each call)."""
import ctypes as ct

import numpy as np

from . import _lib
from ._lib import BzkError

NTT_FFT, NTT_IFFT, NTT_COSET_FFT, NTT_ICOSET_FFT = 0, 1, 2, 3
FR_ADD, FR_SUB, FR_MUL = 0, 1, 2
G1_BYTES, G2_BYTES = 104, 200


def _host_ptr(a):
    return ct.c_void_p(a.ctypes.data)


def _as_fr(a):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    if a.shape[-1] != 4:
        raise ValueError("Fr arrays are [..., 4] uint64 Montgomery limbs")
    return a


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _any_ptr(x):
    """host numpy array, pinned/unpinned CPU torch tensor -> host pointer."""
    if _is_torch(x):
        if x.is_cuda:
            raise ValueError("expected a host buffer")
        if not x.is_contiguous():
            raise ValueError("expected a contiguous buffer")
        return ct.c_void_p(x.data_ptr())
    return _host_ptr(x)


def _dev_ptr(t):
    if not (_is_torch(t) and t.is_cuda and t.is_contiguous()):
        raise ValueError("expected a contiguous CUDA torch tensor")
    return ct.c_void_p(t.data_ptr())


class _Bases:
    _kind = None

    def __init__(self, ctx, handle):
        self._ctx, self._h = ctx, handle

    def __len__(self):
        return int(getattr(self._ctx._l, f"bzk_{self._kind}_bases_len")(self._h))

    def free(self):
        if self._h:
            self._ctx._check(getattr(self._ctx._l, f"bzk_{self._kind}_bases_free")(self._ctx._h, self._h))
            self._h = None

    def precompute(self, max_levels=16):
        """fixed-base table [2^(c*G*t)] P for t < levels (bzk_g*_bases_precompute): the vector's MSMs then use
        ceil(W/levels) bucket groups.  Same results, levels x the memory.  Returns the level count in use."""
        self._ctx._check(getattr(self._ctx._l, f"bzk_{self._kind}_bases_precompute")(self._ctx._h, self._h, int(max_levels)))
        return self.levels

    @property
    def levels(self):
        return int(getattr(self._ctx._l, f"bzk_{self._kind}_bases_levels")(self._h))

    def move_to_host(self):
        """put the points in pinned host memory and free their device storage, tables included (bzk_g*_bases_move): a
        vector need not fit in device memory; its MSMs stream it to the device in chunks, with the same results."""
        self._ctx._check(getattr(self._ctx._l, f"bzk_{self._kind}_bases_move")(self._ctx._h, self._h, 1))
        return self

    def move_to_device(self):
        """back to device memory, untabled"""
        self._ctx._check(getattr(self._ctx._l, f"bzk_{self._kind}_bases_move")(self._ctx._h, self._h, 0))
        return self

    @property
    def on_host(self):
        return bool(getattr(self._ctx._l, f"bzk_{self._kind}_bases_on_host")(self._h))

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class G1Bases(_Bases):
    """Packed G1 base vector (one `Parameters<Bls12>` column), on the device or in pinned host memory."""
    _kind = "g1"


class G2Bases(_Bases):
    _kind = "g2"


class Context:
    """One per GPU (`bzk_ctx`).  Raises BzkError(BZK_ERR_NO_DEVICE) without a GPU — no CPU path."""

    def __init__(self, device=0, load_poseidon=True):
        self._l = _lib.load()
        h = ct.c_void_p()
        st = self._l.bzk_ctx_create(int(device), ct.byref(h))
        if st != 0:
            raise BzkError(st, self._l.bzk_strerror(st).decode())
        self._h = h
        self.device = int(device)
        if load_poseidon:
            blob = open(_lib.PARAMS_PATH, "rb").read()
            self._check(self._l.bzk_poseidon_load_params(self._h, blob, len(blob)))

    # ---------------------------------------------------------------- plumbing
    def _check(self, st):
        if st != 0:
            raise BzkError(st, self._l.bzk_last_error(self._h).decode() or self._l.bzk_strerror(st).decode())

    def close(self):
        if self._h:
            self._l.bzk_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def use_torch_stream(self):
        """run on torch's current CUDA stream (so torch.cuda.Event timing brackets our kernels)."""
        import torch
        h = torch.cuda.current_stream(self.device).cuda_stream
        # torch reports its default stream as 0; libbzk reserves NULL for "ctx-owned stream", so
        # name the legacy default stream explicitly (cudaStreamLegacy == (cudaStream_t)0x1)
        self._check(self._l.bzk_ctx_set_stream(self._h, ct.c_void_p(h if h else 1)))

    def use_own_stream(self):
        """back to the ctx-owned stream."""
        self.synchronize()
        self._check(self._l.bzk_ctx_set_stream(self._h, None))

    def synchronize(self):
        self._check(self._l.bzk_ctx_synchronize(self._h))

    MSM_STAGES = ("digits_hist", "scan", "scatter", "accumulate", "fixup", "bucket_slices", "window_sum")

    def set_timing(self, on=True):
        self._check(self._l.bzk_ctx_set_timing(self._h, int(on)))

    def set_msm_affine_rounds(self, g1=-1, g2=-1):
        """batched-affine rounds before the XYZZ accumulation (speed knob; results unchanged); -1 = library default"""
        self._check(self._l.bzk_ctx_set_msm_affine_rounds(self._h, int(g1), int(g2)))

    def set_msm_table_window(self, c=0):
        """window of the fixed-base tables built from now on (8..23); 0 = the planner's choice.  Results unchanged."""
        self._check(self._l.bzk_ctx_set_msm_table_window(self._h, int(c)))

    def set_msm_stream_chunk(self, points=0):
        """points per device chunk buffer of the sums over host-resident vectors (>= 256); 0 = the library default.
        Results unchanged."""
        self._check(self._l.bzk_ctx_set_msm_stream_chunk(self._h, int(points)))

    MSM_STREAM_FIELDS = ("chunks", "chunk_points", "bytes_h2d", "streamed")

    def last_msm_stream(self):
        """how the last single MSM on this context used its bases (bzk_ctx_last_msm_stream) as a dict of
        MSM_STREAM_FIELDS; all 0 for a device vector."""
        out = np.zeros(4, dtype=np.uint64)
        self._check(self._l.bzk_ctx_last_msm_stream(self._h, _host_ptr(out)))
        return dict(zip(self.MSM_STREAM_FIELDS, (int(x) for x in out)))

    MSM_PLAN_FIELDS = ("c", "W", "T", "G", "NB", "slice", "nbits", "long_len")

    def last_msm_plan(self):
        """plan of the last single MSM on this context (bzk_ctx_last_msm_plan) as a dict of MSM_PLAN_FIELDS;
        long_len is only read back while set_timing(True) is on."""
        out = np.zeros(8, dtype=np.uint32)
        self._check(self._l.bzk_ctx_last_msm_plan(self._h, _host_ptr(out)))
        return dict(zip(self.MSM_PLAN_FIELDS, (int(x) for x in out)))

    def stage_ms(self):
        """-> (runs, last_ms[16], sum_ms[16]) from the CUDA events the MSM driver records between kernels."""
        last = np.zeros(16, dtype=np.float32)
        tot = np.zeros(16, dtype=np.float64)
        runs = int(self._l.bzk_ctx_stage_ms(self._h, _host_ptr(last), _host_ptr(tot), 16))
        return runs, last, tot

    @property
    def launch_count(self):
        return int(self._l.bzk_ctx_launch_count(self._h))

    # ---------------------------------------------------------------- Poseidon
    def poseidon(self, inputs):
        """inputs [n, arity, 4] (host) -> digests [n, 4].  `poseidon::poseidon` batched."""
        inputs = np.ascontiguousarray(inputs, dtype=np.uint64)
        if inputs.ndim != 3 or inputs.shape[2] != 4:
            raise ValueError("inputs must be [n, arity, 4]")
        n, arity, _ = inputs.shape
        out = np.empty((n, 4), dtype=np.uint64)
        self._check(self._l.bzk_poseidon_hash(self._h, arity, _host_ptr(inputs), n, _host_ptr(out)))
        return out

    def poseidon_dev(self, d_in, arity, d_out):
        n = d_in.numel() * d_in.element_size() // (32 * arity)
        self._check(self._l.bzk_poseidon_hash_dev(self._h, arity, _dev_ptr(d_in), n, _dev_ptr(d_out)))

    # ---------------------------------------------------------------- 4-ary Poseidon Merkle trees
    def merkle4_build_dev(self, d_nodes, log4):
        """d_nodes: CUDA tensor of (4^(log4+1)-1)/3 Fr with the 4^log4 leaves in front; fills the upper levels."""
        self._check(self._l.bzk_merkle4_build_dev(self._h, _dev_ptr(d_nodes), log4))

    def merkle4_prove_dev(self, d_nodes, log4, d_indices, d_proofs):
        m = d_indices.numel()
        self._check(self._l.bzk_merkle4_prove_dev(self._h, _dev_ptr(d_nodes), log4, _dev_ptr(d_indices), m, _dev_ptr(d_proofs)))

    def merkle4_root_dev(self, log4, d_indices, d_leaves, d_proofs, d_roots):
        m = d_indices.numel()
        self._check(self._l.bzk_merkle4_root_dev(self._h, log4, _dev_ptr(d_indices), _dev_ptr(d_leaves), _dev_ptr(d_proofs), m, _dev_ptr(d_roots)))

    def tree4_versioned_update(self, depth, tree_id, indices, leaf_values, init_proofs):
        """ordered batch of leaf writes to a forest of sparse 4-ary Poseidon trees (bzk_tree4_versioned_update_dev).
        Host arrays in: tree_id u32[n], indices u64[n], leaf_values [n,4], init_proofs [n,depth,3,4] (Montgomery).
        -> (vals [depth+1, n, 4]: node values on each write's path after the write, vals[depth] = roots;
            proofs [n, depth, 3, 4]: proof of each leaf just before its write)."""
        import torch
        n = len(indices)
        dev = torch.device("cuda", self.device)
        vals = torch.zeros((depth + 1, n, 4), dtype=torch.int64, device=dev)
        proofs = torch.empty((n, depth, 3, 4), dtype=torch.int64, device=dev)
        if n == 0:
            return vals.cpu().numpy().view(np.uint64), proofs.cpu().numpy().view(np.uint64)
        vals[0] = torch.from_numpy(np.ascontiguousarray(leaf_values, dtype=np.uint64).reshape(n, 4).view(np.int64)).to(dev)
        d_tid = torch.from_numpy(np.ascontiguousarray(tree_id, dtype=np.uint32).view(np.int32)).to(dev)
        d_idx = torch.from_numpy(np.ascontiguousarray(indices, dtype=np.uint64).view(np.int64)).to(dev)
        d_init = torch.from_numpy(np.ascontiguousarray(init_proofs, dtype=np.uint64).reshape(n, depth, 3, 4).view(np.int64)).to(dev)
        torch.cuda.current_stream(dev).synchronize()  # the uploads; not a device-wide sync (other contexts keep running)
        self._check(self._l.bzk_tree4_versioned_update_dev(self._h, depth, _dev_ptr(d_tid), _dev_ptr(d_idx), n, _dev_ptr(vals), _dev_ptr(d_init),
                                                            _dev_ptr(proofs)))
        self.synchronize()
        return vals.cpu().numpy().view(np.uint64), proofs.cpu().numpy().view(np.uint64)

    # ---------------------------------------------------------------- NTT
    def ntt(self, a, op):
        """returns the transformed copy of host array a [2^k, 4]."""
        a = np.array(_as_fr(a), copy=True)
        n = a.size // 4
        log_n = n.bit_length() - 1
        if n == 0 or (1 << log_n) != n:
            raise ValueError("length must be a power of two")
        self._check(self._l.bzk_ntt(self._h, _host_ptr(a), log_n, op))
        return a

    def ntt_host_inplace(self, buf, log_n, op):
        """buf: host buffer (numpy / pinned torch) of 2^log_n Fr, transformed in place."""
        self._check(self._l.bzk_ntt(self._h, _any_ptr(buf), log_n, op))

    def ntt_dev(self, d_a, log_n, op):
        self._check(self._l.bzk_ntt_dev(self._h, _dev_ptr(d_a), log_n, op))

    def divide_by_z_on_coset_dev(self, d_a, log_n):
        self._check(self._l.bzk_divide_by_z_on_coset_dev(self._h, _dev_ptr(d_a), log_n))

    def groth16_h_dev(self, d_a, d_b, d_c, log_n):
        self._check(self._l.bzk_groth16_h_dev(self._h, _dev_ptr(d_a), _dev_ptr(d_b), _dev_ptr(d_c), log_n))

    # ---------------------------------------------------------------- MSM
    def msm_g1(self, bases, scalars):
        """bases [n,104] uint8 host images, scalars [n,4] -> [104] uint8 image of sum [s_i]P_i."""
        bases = np.ascontiguousarray(bases, dtype=np.uint8)
        scalars = _as_fr(scalars)
        n = scalars.size // 4
        if bases.size != n * G1_BYTES:
            raise ValueError("bases/scalars length mismatch")
        out = np.zeros(G1_BYTES, dtype=np.uint8)
        self._check(self._l.bzk_msm_g1(self._h, _host_ptr(bases), _host_ptr(scalars), n, _host_ptr(out)))
        return out

    def msm_g2(self, bases, scalars):
        bases = np.ascontiguousarray(bases, dtype=np.uint8)
        scalars = _as_fr(scalars)
        n = scalars.size // 4
        if bases.size != n * G2_BYTES:
            raise ValueError("bases/scalars length mismatch")
        out = np.zeros(G2_BYTES, dtype=np.uint8)
        self._check(self._l.bzk_msm_g2(self._h, _host_ptr(bases), _host_ptr(scalars), n, _host_ptr(out)))
        return out

    def g1_bases(self, images, check_on_curve=False):
        """upload host images [n,104] (numpy or pinned torch) -> resident G1Bases."""
        n = (images.numel() if _is_torch(images) else images.size) // G1_BYTES
        h = ct.c_void_p()
        self._check(self._l.bzk_g1_bases_upload(self._h, _any_ptr(images), n, int(check_on_curve), ct.byref(h)))
        return G1Bases(self, h)

    def g2_bases(self, images, check_on_curve=False):
        n = (images.numel() if _is_torch(images) else images.size) // G2_BYTES
        h = ct.c_void_p()
        self._check(self._l.bzk_g2_bases_upload(self._h, _any_ptr(images), n, int(check_on_curve), ct.byref(h)))
        return G2Bases(self, h)

    def g1_bases_from_dev(self, d_images, n):
        h = ct.c_void_p()
        self._check(self._l.bzk_g1_bases_from_dev(self._h, _dev_ptr(d_images), n, ct.byref(h)))
        return G1Bases(self, h)

    def g2_bases_from_dev(self, d_images, n):
        h = ct.c_void_p()
        self._check(self._l.bzk_g2_bases_from_dev(self._h, _dev_ptr(d_images), n, ct.byref(h)))
        return G2Bases(self, h)

    def msm_g1_resident(self, bases, scalars, offset=0, n=None):
        """scalars: host buffer (numpy [n,4] / pinned torch) or CUDA torch tensor."""
        return self._msm_resident("g1", G1_BYTES, bases, scalars, offset, n)

    def msm_g2_resident(self, bases, scalars, offset=0, n=None):
        return self._msm_resident("g2", G2_BYTES, bases, scalars, offset, n)

    def _msm_resident(self, kind, nbytes, bases, scalars, offset, n):
        out = np.zeros(nbytes, dtype=np.uint8)
        if _is_torch(scalars) and scalars.is_cuda:
            cnt = scalars.numel() * scalars.element_size() // 32 if n is None else n
            fn = getattr(self._l, f"bzk_msm_{kind}_resident_dev")
            self._check(fn(self._h, bases._h, offset, _dev_ptr(scalars), cnt, _host_ptr(out)))
        else:
            if _is_torch(scalars):
                cnt = scalars.numel() * scalars.element_size() // 32 if n is None else n
            else:
                scalars = _as_fr(scalars)
                cnt = scalars.size // 4 if n is None else n
            fn = getattr(self._l, f"bzk_msm_{kind}_resident")
            self._check(fn(self._h, bases._h, offset, _any_ptr(scalars), cnt, _host_ptr(out)))
        return out

    # ---------------------------------------------------------------- helpers
    def g1_add(self, a, b):
        a = np.ascontiguousarray(a, dtype=np.uint8); b = np.ascontiguousarray(b, dtype=np.uint8)
        out = np.zeros(G1_BYTES, dtype=np.uint8)
        self._check(self._l.bzk_g1_add(_host_ptr(a), _host_ptr(b), _host_ptr(out)))
        return out

    def g2_add(self, a, b):
        a = np.ascontiguousarray(a, dtype=np.uint8); b = np.ascontiguousarray(b, dtype=np.uint8)
        out = np.zeros(G2_BYTES, dtype=np.uint8)
        self._check(self._l.bzk_g2_add(_host_ptr(a), _host_ptr(b), _host_ptr(out)))
        return out

    def g1_random_bases_dev(self, seed, n, d_out):
        self._check(self._l.bzk_g1_random_bases_dev(self._h, seed, n, _dev_ptr(d_out)))

    def g2_random_bases_dev(self, seed, n, d_out):
        self._check(self._l.bzk_g2_random_bases_dev(self._h, seed, n, _dev_ptr(d_out)))

    def fr_random_dev(self, seed, n, d_out):
        self._check(self._l.bzk_fr_random_dev(self._h, seed, n, _dev_ptr(d_out)))

    def fr_binop_dev(self, op, d_a, d_b, d_out, n):
        self._check(self._l.bzk_fr_binop_dev(self._h, op, _dev_ptr(d_a), _dev_ptr(d_b), _dev_ptr(d_out), n))

    def fp_mul_dev(self, d_a, d_b, d_out, n):
        self._check(self._l.bzk_fp_mul_dev(self._h, _dev_ptr(d_a), _dev_ptr(d_b), _dev_ptr(d_out), n))


_FR_MODULUS = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001


class HostPoseidon:
    """`impl ZkHasher for PoseidonHasher` (/root/reference/src/zk/mod.rs:491-511) without a GPU round trip: single hashes on
    the host field arithmetic of libbzk (bzk_poseidon_host_*).  inputs [n, arity, 4] or [arity, 4] Montgomery -> digests."""

    def __init__(self):
        self._l = _lib.load()
        blob = open(_lib.PARAMS_PATH, "rb").read()
        h = ct.c_void_p()
        st = self._l.bzk_poseidon_host_create(blob, len(blob), ct.byref(h))
        if st != 0:
            raise BzkError(st, "poseidon_host_create")
        self._h = h

    def hash(self, inputs):
        a = _as_fr(inputs)
        single = a.ndim == 2
        if single:
            a = a[None]
        n, arity, _ = a.shape
        out = np.zeros((n, 4), dtype=np.uint64)
        st = self._l.bzk_poseidon_host_hash(self._h, arity, _host_ptr(a), n, _host_ptr(out))
        if st != 0:
            raise BzkError(st, "poseidon_host_hash")
        return out[0] if single else out

    def eddsa_verify(self, jubjub_d, pk, message, sig_r, sig_s):
        """`JubJub::verify` (/root/reference/src/crypto/jubjub/mod.rs:151-167) on the host: ints in, bool out"""
        canon = lambda *v: np.frombuffer(b"".join((int(x) % _FR_MODULUS).to_bytes(32, "little") for x in v), dtype=np.uint64).reshape(-1, 4).copy()
        d, a, m, r, s = canon(jubjub_d), canon(*pk), canon(message), canon(*sig_r), canon(sig_s)
        if not all(0 <= int(x) < _FR_MODULUS for x in (*pk, message, *sig_r, sig_s)):
            return False
        st = self._l.bzk_jubjub_eddsa_verify(self._h, _host_ptr(d), _host_ptr(a), _host_ptr(m), _host_ptr(r), _host_ptr(s))
        if st < 0:
            raise BzkError(st, "jubjub_eddsa_verify")
        return bool(st)

    def free(self):
        if self._h:
            self._l.bzk_poseidon_host_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def ed25519_verify(pk, msg, sig):
    """`Ed25519::verify` (src/crypto/ed25519.rs:81-83 of the reference, ed25519-dalek 1.x `PublicKey::verify`) on the host, no
    context and no GPU (include/bzk.h, bzk_ed25519_verify): 32-byte key, message, 64-byte signature in, bool out"""
    pk, msg, sig = bytes(pk), bytes(msg), bytes(sig)
    if len(pk) != 32 or len(sig) != 64:
        raise ValueError("an ed25519 key is 32 bytes and a signature 64")
    st = _lib.load().bzk_ed25519_verify(pk, msg, len(msg), sig)
    if st < 0:
        raise BzkError(st, "ed25519_verify")
    return bool(st)
