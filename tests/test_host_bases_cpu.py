"""CPU tier: the host-resident base vector entry points are typed as include/bzk.h declares them, refuse a missing context
or handle before touching anything, and have their Python front ends (the results are checked in
test_gpu_host_bases.py)."""
import ctypes as ct
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_vp, _i32, _u32, _u64, _sz = ct.c_void_p, ct.c_int32, ct.c_uint32, ct.c_uint64, ct.c_size_t

DECLS = {
    "bzk_ctx_set_msm_stream_chunk": ("int32_t bzk_ctx_set_msm_stream_chunk(bzk_ctx *ctx, uint64_t points);", (_i32, [_vp, _u64])),
    "bzk_ctx_last_msm_stream": ("int32_t bzk_ctx_last_msm_stream(const bzk_ctx *ctx, uint64_t out[4]);", (_i32, [_vp, _vp])),
    "bzk_g1_bases_move": ("int32_t bzk_g1_bases_move(bzk_ctx *ctx, bzk_g1_bases *b, int32_t to_host);", (_i32, [_vp, _vp, _i32])),
    "bzk_g2_bases_move": ("int32_t bzk_g2_bases_move(bzk_ctx *ctx, bzk_g2_bases *b, int32_t to_host);", (_i32, [_vp, _vp, _i32])),
    "bzk_g1_bases_on_host": ("int32_t bzk_g1_bases_on_host(const bzk_g1_bases *b);", (_i32, [_vp])),
    "bzk_g2_bases_on_host": ("int32_t bzk_g2_bases_on_host(const bzk_g2_bases *b);", (_i32, [_vp])),
    "bzk_groth16_params_move": ("int32_t bzk_groth16_params_move(bzk_ctx *ctx, bzk_groth16_params *params, uint32_t host_mask);",
                                (_i32, [_vp, _vp, _u32])),
}


def _header():
    return re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bzk.h")).read(), flags=re.S))


def test_host_bases_entry_points_are_typed_as_declared():
    from bazuka_b200 import _lib
    h = _header()
    for name, (decl, sig) in DECLS.items():
        assert decl in h, name
        assert _lib.SIGNATURES[name] == sig, name
    placed = re.search(r"int32_t bzk_groth16_params_read_placed\((.*?)\);", h).group(1)
    plain = re.search(r"int32_t bzk_groth16_params_read\((.*?)\);", h).group(1)
    # the arguments of bzk_groth16_params_read, with the mask before the output handle
    assert placed.replace(" uint32_t host_mask,", "") == plain
    assert _lib.SIGNATURES["bzk_groth16_params_read_placed"] == (_i32, [_vp, _vp, _sz, _i32] + [_vp] * 7 + [_sz, _u32, ct.POINTER(_vp)])
    assert _lib.load().bzk_abi_version() == (1 << 16) | 1


def test_host_bases_entry_points_refuse_null_before_touching_anything():
    from bazuka_b200 import _lib
    lib = _lib.load()
    out = np.full(4, 7, dtype=np.uint64)
    assert lib.bzk_ctx_last_msm_stream(None, out.ctypes.data_as(_vp)) == -1
    assert (out == 7).all()
    for pts in (0, 1, 255, 256, 1 << 22):
        assert lib.bzk_ctx_set_msm_stream_chunk(None, pts) == -1
    for to_host in (0, 1):
        assert lib.bzk_g1_bases_move(None, None, to_host) == -1
        assert lib.bzk_g2_bases_move(None, None, to_host) == -1
    assert lib.bzk_g1_bases_on_host(None) == 0
    assert lib.bzk_g2_bases_on_host(None) == 0
    assert lib.bzk_groth16_params_move(None, None, 0) == -1
    g1 = [np.zeros(104, np.uint8) for _ in range(4)]
    g2 = [np.zeros(200, np.uint8) for _ in range(3)]
    key = np.zeros(16, np.uint8)
    h = _vp()
    ptr = lambda a: a.ctypes.data_as(_vp)
    args = [ptr(g1[0]), ptr(g1[1]), ptr(g2[0]), ptr(g2[1]), ptr(g1[2]), ptr(g2[2]), ptr(g1[3]), 1]
    assert lib.bzk_groth16_params_read_placed(None, ptr(key), key.size, 1, *args, 0, ct.byref(h)) == -1
    assert h.value is None


def test_host_bases_python_front_ends():
    import inspect
    from bazuka_b200 import api
    from bazuka_b200 import groth16 as BG
    for m in ("move_to_host", "move_to_device"):
        assert callable(getattr(api._Bases, m))
    assert isinstance(api._Bases.on_host, property)
    assert callable(api.Context.set_msm_stream_chunk) and callable(api.Context.last_msm_stream)
    assert api.Context.MSM_STREAM_FIELDS == ("chunks", "chunk_points", "bytes_h2d", "streamed")
    assert callable(BG.ProvingKey.move)
    assert "host_vectors" in inspect.signature(BG.read_parameters).parameters
    assert "host_vectors" in inspect.signature(BG.setup_gpu).parameters
    assert BG.host_mask(()) == 0
    assert BG.host_mask("all") == 31
    assert BG.host_mask(("h", "b_g2")) == 0b10001
    assert BG.host_mask("l") == 0b10
    with pytest.raises(ValueError):
        BG.host_mask(("c",))
