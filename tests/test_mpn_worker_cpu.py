"""CPU tier: the MPN worker (csrc/mpn_worker.cu) on the host build of libbzk's MPN sources.  tests/hostshim/worker_shim.cpp adds to
mpn_shim.cpp's stand-ins a "proof" that carries its r and s, the blocked R1CS upload (expanded on the host), bellman's key
lengths, and a batch verifier that accepts (or, on request, rejects) everything: so this tier checks the worker's own logic —
key checks at creation, the config filter, the seeded blinding, the threads, the self-check's verdicts and the solution bytes —
over the real codec, builders, circuits and witness drivers.  The pairing and the MSMs are the GPU tier's."""
import ctypes as ct
import os
import random
import subprocess

import numpy as np
import pytest

from bazuka_b200.mpn import native as N, update as U, wire as Wr, works as Wk
from conftest import ROOT
import mpn_worker_cases as C

A, T, B = 3, 3, 1
KINDS = ("deposit", "withdraw", "update")
ADDR = bytes(range(32))
SEED = bytes([7]) * 32


class _ShimCtx:
    """a context-like object over the worker shim (what bazuka_b200's ctypes front-ends need of a Context)"""

    def __init__(self, lib):
        self._l = lib
        self._h = ct.c_void_p(lib.shim_ctx_create())

    def _check(self, status):
        from bazuka_b200._lib import BzkError
        if status != 0:
            raise BzkError(status, "worker shim")


@pytest.fixture(scope="module")
def shim():
    from bazuka_b200 import _lib
    d = os.path.join(ROOT, "tests", "hostshim")
    csrc = os.path.join(ROOT, "bazuka_b200", "csrc")
    srcs = [os.path.join(csrc, f) for f in ("mpn_host.cu", "mpn_wire.cu", "mpn_prover.cu", "mpn_worker.cu", "mpn_circuit.cu", "poseidon_host.cu")]
    srcs.append(os.path.join(d, "worker_shim.cpp"))
    out = os.path.join(d, "_worker_shim.so")
    deps = srcs + [os.path.join(d, f) for f in ("mpn_shim.cpp", "fake_cuda_pre.h")] + [os.path.join(ROOT, "include", "bzk.h")] + \
        [os.path.join(csrc, h) for h in ("ff.cuh", "ec.cuh", "common.cuh", "witness_core.cuh", "mpn_wire.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(x) > os.path.getmtime(out) for x in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-x", "c++", "-include", os.path.join(d, "fake_cuda_pre.h"),
                               "-I", csrc, "-I", d, "-I", "/usr/local/cuda/include"] + srcs +
                              ["-x", "none", "-Wl,-Bsymbolic", _lib.SO_PATH, "-Wl,-rpath," + os.path.dirname(_lib.SO_PATH), "-o", out])
    lib = ct.CDLL(out)
    for name, (res, args) in _lib.SIGNATURES.items():
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = res, args
    lib.shim_ctx_create.restype = ct.c_void_p
    lib.shim_params_create.restype = ct.c_void_p
    lib.shim_params_create.argtypes = [ct.c_void_p, ct.c_char_p]
    lib.shim_params_free.argtypes = [ct.c_void_p]
    lib.shim_verify_calls.restype = ct.c_uint64
    blob = open(_lib.PARAMS_PATH, "rb").read()
    lib.shim_set_poseidon.argtypes = [ct.c_char_p, ct.c_size_t]
    assert lib.shim_set_poseidon(blob, len(blob)) == 0
    return lib


def _jubjub():
    return np.ascontiguousarray(np.stack([C._canon(N.JJ_D), C._canon(N.JJ_BASE_COFACTOR[0]), C._canon(N.JJ_BASE_COFACTOR[1])]))


def _compile(lib, kind, blocked):
    from bazuka_b200 import _lib
    blob = open(_lib.PARAMS_PATH, "rb").read()
    h = ct.c_void_p()
    jj = _jubjub()
    if kind == "update":
        name = "bzk_mpn_update_circuit_compile_blocked" if blocked else "bzk_mpn_update_circuit_compile"
        assert getattr(lib, name)(A, T, B, blob, len(blob), C._ptr(jj), ct.byref(h)) == 0
    else:
        assert lib.bzk_mpn_dw_circuit_compile(KINDS.index(kind) + 1, A, T, B, blob, len(blob), C._ptr(jj), ct.byref(h)) == 0
    return h


def _key_lens(lib, kind):
    """{h, l, a, b_g1, b_g2} of the kind's circuit, counted from its explicit matrices as bellman counts them"""
    c = _compile(lib, kind, blocked=False)
    shape = np.zeros(12, np.uint64)
    lib.bzk_mpn_circuit_shape(c, C._ptr(shape))
    ni, na, nc = (int(x) for x in shape[:3])
    mats = []
    for s in range(3):
        rp, col, val = np.zeros(nc + 1, np.uint64), np.zeros(int(shape[3 + s]) + 1, np.uint32), np.zeros((int(shape[3 + s]) + 1, 4), np.uint64)
        lib.bzk_mpn_circuit_matrix(c, s, C._ptr(rp), C._ptr(col), C._ptr(val))
        mats.append((rp, col, val))
    lib.bzk_mpn_circuit_free(c)
    a_aux = {int(x) for x, v in zip(mats[0][1][:int(shape[3])], mats[0][2][:int(shape[3])]) if x >= ni and v.any()}
    b_all = {int(x) for x, v in zip(mats[1][1][:int(shape[4])], mats[1][2][:int(shape[4])]) if v.any()}
    m = 1
    while m < nc + ni:
        m *= 2
    return np.array([m - 1, na, ni + len(a_aux), len(b_all), len(b_all)], np.uint64)


@pytest.fixture(scope="module")
def setup(shim):
    vks = {"deposit": C.opaque_vk(2), "withdraw": C.opaque_vk(4), "update": C.opaque_vk(6)}
    cfg = C.config(A, T, B, B, B, vks)
    ctxs = [_ShimCtx(shim) for _ in range(3)]
    lens = {k: _key_lens(shim, k) for k in KINDS}
    keys = {k: ct.c_void_p(shim.shim_params_create(C._ptr(lens[k]), vks[k])) for k in KINDS}
    st, deps, wds, ups, dpay, wpay = C.block(A, T)
    led = C.ledger(ctxs[0], st, A, T)
    resp, n = C.prepare_response(ctxs[0], led, cfg, deps, wds, ups, dpay, wpay)
    assert n == 3
    return dict(cfg=cfg, cfg_bytes=C.config_bytes(cfg), vks=vks, ctxs=ctxs, lens=lens, keys=keys, resp=resp)


def _worker(setup, n_ctx=1, split=None):
    keys = split or [{k: setup["keys"][k] for k in KINDS}] * n_ctx
    return Wk.NativeMpnWorker(setup["ctxs"][:len(keys)], setup["cfg_bytes"], keys)


def _explicit_proof(shim, setup, kind, work_bytes, r, s):
    """bzk_mpn_prover_prove_work on the explicit circuit of the kind"""
    ctx = setup["ctxs"][0]
    c = _compile(shim, kind, blocked=False)
    p = ct.c_void_p()
    jj, fee = _jubjub(), C._canon(U.ZIESHA)
    ctx._check(shim.bzk_mpn_prover_create(ctx._h, c, setup["keys"][kind], C._ptr(jj[0]), C._ptr(fee), ct.byref(p)))
    shim.bzk_mpn_circuit_free(c)
    out = ct.create_string_buffer(391)
    ctx._check(shim.bzk_mpn_prover_prove_work(ctx._h, p, work_bytes, len(work_bytes), ADDR, C._ptr(r), C._ptr(s), 1, out))
    shim.bzk_mpn_prover_free(ctx._h, p)
    return out.raw


def test_response_to_solution_with_seeded_blinding(shim, setup):
    """works of all three kinds from bzk_mpn_prepare_works -> one call -> a PostMpnSolutionRequest for this address with every id;
    each proof is bzk_mpn_prover_prove_work's on the explicit circuit with r, s = SHA3(seed || id || tag) mod r (so the blocked
    update upload gives the explicit one's satisfying witness), and the self-check ran once per kind"""
    calls0 = shim.shim_verify_calls(None)
    w = _worker(setup)
    body, status = w.prove_response(setup["resp"], ADDR, SEED)
    assert status == [0, 0, 0]
    assert shim.shim_verify_calls(None) - calls0 == 3
    prover, proofs = C.solution_proofs(body)
    assert prover == ADDR and sorted(proofs) == [0, 1, 2]
    for wid, h in C.decode_response(shim, setup["resp"]):
        blob = C.encode_work(shim, h)
        kind = Wr.work_from_bytes(blob)["data"][0]
        shim.bzk_mpn_work_free(h)
        r, s = C.seeded_blinding(SEED, wid)
        proof = bytes(proofs[wid])
        assert proof[:32] == r.tobytes() and proof[290:322] == s.tobytes()      # the shim's proof carries its r and s
        assert proof == _explicit_proof(shim, setup, kind, blob, r, s)[4:]
    # without a seed the blinding differs from call to call
    b1, st1 = w.prove_response(setup["resp"], ADDR)
    b2, st2 = w.prove_response(setup["resp"], ADDR)
    assert st1 == st2 == [0, 0, 0] and b1 != b2 and b1 != body
    w.free()


def test_one_two_and_three_threads_give_the_same_bytes(setup):
    outs = []
    for n in (1, 2, 3):
        w = _worker(setup, n)
        outs.append(w.prove_response(setup["resp"], ADDR, SEED))
        w.free()
    keys = setup["keys"]
    w = _worker(setup, split=[{"update": keys["update"]}, {"deposit": keys["deposit"], "withdraw": keys["withdraw"]}])
    outs.append(w.prove_response(setup["resp"], ADDR, SEED))
    w.free()
    assert all(o == outs[0] for o in outs) and outs[0][1] == [0, 0, 0]


def test_foreign_config_and_unsatisfied_works_are_left_out(shim, setup):
    works = Wr.get_mpn_work_response_from_bytes(setup["resp"])
    works[0] = dict(works[0], config=dict(works[0]["config"], deposit_vk=C.opaque_vk(9)))            # another verifying key
    works[1] = dict(works[1], public_inputs=dict(works[1]["public_inputs"], next_state=works[1]["public_inputs"]["next_state"] + 1))
    works[5] = dict(works[2], config=dict(works[2]["config"], log4_tree_size=A + 1))                 # another shape
    resp = Wr.get_mpn_work_response_to_bytes(works)
    w = _worker(setup)
    body, status = w.prove_response(resp, ADDR, SEED)
    assert status == [-1, -7, 0, -1]
    _, proofs = C.solution_proofs(body)
    assert sorted(proofs) == [2]
    want, _ = w.prove_response(setup["resp"], ADDR, SEED)
    assert bytes(proofs[2]) == bytes(C.solution_proofs(want)[1][2])
    # a kind no context serves is foreign too
    w.free()
    w = _worker(setup, split=[{"update": setup["keys"]["update"]}])
    body, status = w.prove_response(setup["resp"], ADDR, SEED)
    assert status == [-1, -1, 0] and sorted(C.solution_proofs(body)[1]) == [2]
    w.free()


def test_rejected_proofs_are_left_out(shim, setup):
    w = _worker(setup)
    shim.shim_reject_all(1)
    try:
        body, status = w.prove_response(setup["resp"], ADDR, SEED)
    finally:
        shim.shim_reject_all(0)
    assert status == [-10, -10, -10]
    assert C.solution_proofs(body) == (ADDR, {})
    w.free()


def test_keys_that_do_not_belong_are_refused_at_create(shim, setup):
    from bazuka_b200._lib import BzkError
    made = []
    for kind in KINDS:
        for k in range(5):                                                    # each vector one point longer
            lens = setup["lens"][kind].copy()
            lens[k] += 1
            made.append(ct.c_void_p(shim.shim_params_create(C._ptr(lens), setup["vks"][kind])))
            with pytest.raises(BzkError) as e:
                Wk.NativeMpnWorker(setup["ctxs"][:1], setup["cfg_bytes"], [{**setup["keys"], kind: made[-1]}])
            assert e.value.status == -1
        vk = bytearray(setup["vks"][kind])
        for off in (0, 97, 194, 580, 677):                                    # alpha_g1, beta_g1, beta_g2, delta_g1, delta_g2
            other = bytearray(vk)
            other[off + 5] ^= 1
            made.append(ct.c_void_p(shim.shim_params_create(C._ptr(setup["lens"][kind]), bytes(other))))
            with pytest.raises(BzkError) as e:
                Wk.NativeMpnWorker(setup["ctxs"][:1], setup["cfg_bytes"], [{**setup["keys"], kind: made[-1]}])
            assert e.value.status == -1
        # gamma_g2 and ic are not the prover's: a key that differs only there passes creation (the self-check catches it)
        other = bytearray(vk)
        other[387 + 5] ^= 1
        made.append(ct.c_void_p(shim.shim_params_create(C._ptr(setup["lens"][kind]), bytes(other))))
        Wk.NativeMpnWorker(setup["ctxs"][:1], setup["cfg_bytes"], [{**setup["keys"], kind: made[-1]}]).free()
    for p in made:
        shim.shim_params_free(p)
    with pytest.raises(BzkError):
        Wk.NativeMpnWorker(setup["ctxs"][:1], setup["cfg_bytes"][:-1], [setup["keys"]])


def test_truncated_and_mutated_responses_never_crash(shim, setup):
    w = _worker(setup)
    resp = setup["resp"]
    lib = shim
    for cut in (0, 1, 7, 8, 9, 100, len(resp) // 2, len(resp) - 1):
        buf, ln, n = ct.c_void_p(), ct.c_size_t(), ct.c_uint64()
        st = np.zeros(4, np.int32)
        assert lib.bzk_mpn_worker_prove_response(w._h, resp[:cut], cut, ADDR, SEED, ct.byref(buf), ct.byref(ln), C._ptr(st), 4, ct.byref(n)) == -1
        assert not buf.value
    rng = random.Random(5)
    outcomes = set()
    for _ in range(60):
        b = bytearray(resp)
        for _ in range(rng.randint(1, 3)):
            b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
        try:
            _, status = w.prove_response(bytes(b), ADDR, SEED)
            outcomes.add(tuple(status))
        except Exception as e:
            outcomes.add(type(e).__name__)
    assert len(outcomes) > 1
    w.free()


def test_worker_client_polls_through_the_native_worker(setup):
    """WorkerClient.run_once with a NativeMpnWorker: one GET, one worker call, one POST of the worker's solution bytes"""
    import struct
    w = _worker(setup)
    log = []

    def opener(method, url, body):
        log.append((method, url.rsplit("/", 1)[-1], body))
        return setup["resp"] if method == "GET" else struct.pack("<Q", len(C.solution_proofs(body)[1]))
    client = Wk.WorkerClient("node:1234", ADDR, w, opener=opener)
    assert client.run_once(None) == (3, 3)
    assert [(m, u) for m, u, _ in log] == [("GET", "work"), ("POST", "solution")]
    prover, proofs = C.solution_proofs(log[1][2])
    assert prover == ADDR and sorted(proofs) == [0, 1, 2]
    w.free()
