import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with `-m gpu` on an H100)")


@pytest.fixture(scope="session")
def cref():
    """the C oracle (test infrastructure), built on demand."""
    from oracle import cref as c
    c.lib()
    return c


@pytest.fixture(scope="session")
def ctx():
    """one libbzk context on cuda:0 — fails loudly if the extension or the GPU is missing."""
    import bazuka_b200 as B
    c = B.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="session")
def hostshim():
    """ff.cuh/ec.cuh compiled for the host (explicit-carry build of the device algorithm)."""
    import ctypes as ct
    src = os.path.join(ROOT, "tests", "hostshim", "shim.cpp")
    out = os.path.join(ROOT, "tests", "hostshim", "_shim.so")
    deps = [src] + [os.path.join(ROOT, "bazuka_b200", "csrc", h) for h in ("ff.cuh", "ec.cuh", "witness_core.cuh", "pairing.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++",
                               "-I", os.path.join(ROOT, "bazuka_b200", "csrc"), src, "-o", out])
    return ct.CDLL(out)


class _HostMpnCtx:
    """what bazuka_b200's ctypes front-ends need of a Context, over tests/hostshim/_mpn_shim.so: libbzk's HOST sources
    (ledger, builders, wire codec) compiled unmodified with g++, the GPU side replaced by host stand-ins (mpn_shim.cpp)."""
    device = 0

    def __init__(self, lib):
        import ctypes as ct
        self._l = lib
        lib.shim_ctx_create.restype = ct.c_void_p
        self._h = ct.c_void_p(lib.shim_ctx_create())

    def _check(self, status):
        from bazuka_b200._lib import BzkError
        if status != 0:
            raise BzkError(status, "host shim")


@pytest.fixture(scope="session")
def hostmpn():
    """a fake context whose `_l` is the host build of csrc/mpn_host.cu + mpn_wire.cu + poseidon_host.cu (CPU tier only)."""
    import ctypes as ct
    from bazuka_b200 import _lib
    d = os.path.join(ROOT, "tests", "hostshim")
    csrc = os.path.join(ROOT, "bazuka_b200", "csrc")
    srcs = [os.path.join(csrc, f) for f in ("mpn_host.cu", "mpn_wire.cu", "mpn_prover.cu", "mpn_circuit.cu", "poseidon_host.cu") if os.path.exists(os.path.join(csrc, f))]
    srcs.append(os.path.join(d, "mpn_shim.cpp"))
    out = os.path.join(d, "_mpn_shim.so")
    deps = srcs + [os.path.join(d, "fake_cuda_pre.h"), os.path.join(ROOT, "include", "bzk.h")] + \
        [os.path.join(csrc, h) for h in ("ff.cuh", "ec.cuh", "common.cuh", "witness_core.cuh", "mpn_wire.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(x) > os.path.getmtime(out) for x in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-x", "c++", "-include", os.path.join(d, "fake_cuda_pre.h"),
                               "-I", csrc, "-I", "/usr/local/cuda/include"] + srcs +
                              # own definitions win (-Bsymbolic); what the host sources reach in OTHER host parts of the product (the
                              # pairing verifier) comes from the real libbzk.so
                              ["-x", "none", "-Wl,-Bsymbolic", _lib.SO_PATH, "-Wl,-rpath," + os.path.dirname(_lib.SO_PATH), "-o", out])
    lib = ct.CDLL(out)
    for name, (res, args) in _lib.SIGNATURES.items():
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = res, args
    blob = open(_lib.PARAMS_PATH, "rb").read()
    lib.shim_set_poseidon.argtypes = [ct.c_char_p, ct.c_size_t]
    assert lib.shim_set_poseidon(blob, len(blob)) == 0
    return _HostMpnCtx(lib)


def fr_ints(a):
    from oracle.py import field as Fd
    a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4)
    return [Fd.fr_from_mont_bytes(x.tobytes()) for x in a]


def fr_arr(xs):
    from oracle.py import field as Fd
    return np.frombuffer(Fd.fr_vec_to_mont(xs), dtype=np.uint64).reshape(-1, 4).copy()
