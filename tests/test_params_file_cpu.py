"""CPU tier: bellman `Parameters` files.  The oracle codec (oracle/py/bellman_params.py) against itself and the production
verifying keys, its subgroup rules against the definition [r]P = O, the GPU decoder's per-point logic (csrc/params_io.cuh
compiled for the host) against the oracle, and bzk_groth16_params_file_info on the real libbzk.so (no context needed)."""
import ctypes as ct
import json
import os
import random
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle.py import bellman_params as BP, curve as C
from oracle.py.field import R_MOD

GOLDEN = os.path.join(ROOT, "tests", "golden", "mpn_vks.json")


def vk_from_bincode(blob):
    """bincode(Groth16VerifyingKey) -> dict of wire images (97 / 193-byte fields padded to 104 / 200)"""
    off, vk = 0, {}
    for k in BP.VK_ORDER:
        n = 193 if k.endswith("g2") else 97
        vk[k] = np.frombuffer(blob[off:off + n] + bytes(7), dtype=np.uint8)
        off += n
    n_ic = int.from_bytes(blob[off:off + 8], "little")
    off += 8
    vk["ic"] = np.stack([np.frombuffer(blob[off + 97 * i: off + 97 * (i + 1)] + bytes(7), dtype=np.uint8) for i in range(n_ic)])
    return vk


def golden_vks():
    return {k: bytes.fromhex(v) for k, v in json.load(open(GOLDEN))["vks"].items()}


def random_points(seed, n1=4, n2=2):
    rnd = random.Random(seed)
    return ([C.mul(C.FP, C.G1_GEN, rnd.randrange(1, R_MOD)) for _ in range(n1)],
            [C.mul(C.FP2, C.G2_GEN, rnd.randrange(1, R_MOD)) for _ in range(n2)])


def lifts(seed, n, g2):
    rnd, out = random.Random(seed), []
    while len(out) < n:
        p = BP.g2_lift((rnd.randrange(BP.P), rnd.randrange(BP.P))) if g2 else BP.g1_lift(rnd.randrange(BP.P))
        if p is not None:
            out.append(p)
    return out


def test_oracle_codec_round_trips_including_infinity():
    g1s, g2s = random_points(1)
    for p in g1s + [C.G1_GEN, None]:
        b = BP.g1_to_uncompressed(p)
        assert len(b) == 96 and BP.g1_from_uncompressed(b) == p and BP.g1_from_uncompressed(b, checked=False) == p
    for p in g2s + [C.G2_GEN, None]:
        b = BP.g2_to_uncompressed(p)
        assert len(b) == 192 and BP.g2_from_uncompressed(b) == p
    assert BP.g1_to_uncompressed(None) == b"\x40" + bytes(95)
    # G2: x.c1 first
    assert BP.g2_to_uncompressed(C.G2_GEN)[:48] == C.G2_GEN[0][1].to_bytes(48, "big")


def test_production_vks_decode_checked_and_equal():
    """the ceremony's verifying keys, as bellman images: every point passes the curve and subgroup tests and comes back equal"""
    for name, blob in golden_vks().items():
        vk = vk_from_bincode(blob)
        params = {"vk": vk, "h": [], "l": [], "a": [], "b_g1": [], "b_g2": []}
        back = BP.read(BP.write(params), checked=True)
        for k in BP.VK_ORDER:
            assert back["vk"][k] == BP._point(vk[k], k.endswith("g2")), (name, k)
        assert back["vk"]["ic"] == [BP._point(x, False) for x in vk["ic"]], name


def test_swapped_g2_components_are_refused():
    for name, blob in golden_vks().items():
        vk = vk_from_bincode(blob)
        for k in ("beta_g2", "gamma_g2", "delta_g2"):
            b = BP.g2_to_uncompressed(BP._point(vk[k], True))
            swapped = b[48:96] + b[0:48] + b[144:192] + b[96:144]
            with pytest.raises(BP.BadPoint):
                BP.g2_from_uncompressed(swapped)


def test_non_subgroup_points_are_refused_and_the_endomorphism_tests_agree():
    t3 = (0, 2)
    cases1 = [t3, C.add(C.FP, C.G1_GEN, t3)] + lifts(5, 4, False)
    cases2 = lifts(6, 3, True)
    for F, pts, dec, enc in ((C.FP, cases1, BP.g1_from_uncompressed, BP.g1_to_uncompressed),
                             (C.FP2, cases2, BP.g2_from_uncompressed, BP.g2_to_uncompressed)):
        for p in pts:
            assert C.on_curve(F, p) and not BP.in_subgroup(F, p) and not BP.torsion_free_endo(F, p)
            with pytest.raises(BP.BadPoint) as e:
                dec(enc(p))
            assert e.value.status == BP.NOT_IN_SUBGROUP
            assert dec(enc(p), checked=False) == p
    g1s, g2s = random_points(7)
    assert all(BP.torsion_free_endo(C.FP, p) for p in g1s) and all(BP.torsion_free_endo(C.FP2, p) for p in g2s)


# ------------------------------------------------------------------ the GPU decoder's per-point logic, on the host
HARNESS = r"""
#include <string.h>
#include "params_io.cuh"
using namespace bzk;
static EndoConsts k;
extern "C" int h_init(void) { return derive_endo_consts(&k); }
extern "C" void h_beta(uint8_t *out) { Fp b = k.beta.from_mont(); memcpy(out, b.l, 48); }
extern "C" uint32_t h_decode(int g2, const uint8_t *img, int checked, int allow_inf, uint8_t *packed) {
    uint32_t w[48];
    memcpy(w, img, g2 ? 192 : 96);
    if (g2) { G2Affine p = G2Affine::inf(); uint32_t f = decode_point(w, checked, allow_inf, k, p); memcpy(packed, &p, 192); return f; }
    G1Affine p = G1Affine::inf(); uint32_t f = decode_point(w, checked, allow_inf, k, p); memcpy(packed, &p, 96); return f;
}
extern "C" void h_encode(int g2, const uint8_t *packed, uint8_t *img) {
    uint32_t w[48];
    if (g2) { G2Affine p; memcpy(&p, packed, 192); encode_point(p, w); memcpy(img, w, 192); }
    else { G1Affine p; memcpy(&p, packed, 96); encode_point(p, w); memcpy(img, w, 96); }
}
"""
FAULT_STATUS = {0: 0, 1: -8, 2: -8, 3: -8, 4: -8, 5: -8, 6: -8, 7: -4, 8: -9}


@pytest.fixture(scope="module")
def codec(tmp_path_factory):
    d = tmp_path_factory.mktemp("params_codec")
    src, so = d / "harness.cpp", d / "harness.so"
    src.write_text(HARNESS)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(ROOT, "bazuka_b200", "csrc"),
                           str(src), "-o", str(so)])
    lib = ct.CDLL(str(so))
    lib.h_decode.restype = ct.c_uint32
    assert lib.h_init() == 1, "the subgroup-test constants failed their self-check"
    return lib


def _decode(codec, img, g2, checked, allow_inf=0):
    out = ct.create_string_buffer(192 if g2 else 96)
    f = codec.h_decode(int(g2), bytes(img), int(checked), int(allow_inf), out)
    pt = None if not any(out.raw) else (C.g2_from_bytes(out.raw + bytes(8)) if g2 else C.g1_from_bytes(out.raw + bytes(8)))
    return f, pt, out.raw


def test_device_codec_matches_the_oracle(codec):
    """derived beta equals the oracle's; on subgroup points, lifts and the 3-torsion cases the decoder's verdict is the
    definition's; unchecked decode + encode is the identity on images"""
    b = ct.create_string_buffer(48)
    codec.h_beta(b)
    assert int.from_bytes(b.raw, "little") == BP.BETA
    g1s, g2s = random_points(11, 6, 3)
    for g2, pts in ((0, g1s + [(0, 2), C.add(C.FP, C.G1_GEN, (0, 2))] + lifts(12, 6, False)), (1, g2s + lifts(13, 3, True))):
        F, enc = (C.FP2, BP.g2_to_uncompressed) if g2 else (C.FP, BP.g1_to_uncompressed)
        for p in pts:
            img = enc(p)
            f, _, _ = _decode(codec, img, g2, 1)
            assert f == (0 if BP.in_subgroup(F, p) else 8)
            f, q, raw = _decode(codec, img, g2, 0)
            assert f == 0 and q == p
            out = ct.create_string_buffer(len(img))
            codec.h_encode(g2, raw, out)
            assert out.raw == img
        out = ct.create_string_buffer(192 if g2 else 96)
        codec.h_encode(g2, bytes(192 if g2 else 96), out)
        assert out.raw == enc(None)


@pytest.mark.parametrize("g2", [0, 1])
def test_device_codec_defects_follow_bellman_rules(codec, g2):
    F, enc, dec = (C.FP2, BP.g2_to_uncompressed, BP.g2_from_uncompressed) if g2 else (C.FP, BP.g1_to_uncompressed, BP.g1_from_uncompressed)
    p = random_points(21)[g2][0]
    img, yo = bytearray(enc(p)), (96 if g2 else 48)

    def mutated(fn):
        m = bytearray(img)
        fn(m)
        return bytes(m)
    cases = {
        "compression": (mutated(lambda m: m.__setitem__(0, m[0] | 0x80)), -8, -8),
        "sort": (mutated(lambda m: m.__setitem__(0, m[0] | 0x20)), -8, -8),
        "infinity_with_bits": (mutated(lambda m: m.__setitem__(0, m[0] | 0x40)), -8, -8),
        "x_eq_p": (mutated(lambda m: m.__setitem__(slice(0, 48), BP.P.to_bytes(48, "big"))), -8, -8),
        "y_eq_p": (mutated(lambda m: m.__setitem__(slice(yo, yo + 48), BP.P.to_bytes(48, "big"))), -8, -8),
        "off_curve": (mutated(lambda m: m.__setitem__(len(m) - 1, m[-1] ^ 1)), 0, -4),
        "not_in_subgroup": (enc(lifts(22, 1, bool(g2))[0]), 0, -9),
    }
    for name, (m, unchecked, checked) in cases.items():
        for chk, want in ((0, unchecked), (1, checked)):
            f, _, _ = _decode(codec, m, g2, chk)
            assert FAULT_STATUS[f] == want, (name, chk, f)
            try:
                dec(m, bool(chk))
                got = 0
            except BP.BadPoint as e:
                got = e.status
            assert got == want, (name, chk, "oracle")
    inf = enc(None)
    assert _decode(codec, inf, g2, 1, allow_inf=1)[0] == 0
    assert _decode(codec, inf, g2, 0, allow_inf=0)[0] == 6          # point at infinity in a vector


# ------------------------------------------------------------------ bzk_groth16_params_file_info on libbzk.so
def small_params(seed=31):
    g1s, g2s = random_points(seed, 6, 3)
    vk = {"alpha_g1": g1s[0], "beta_g1": g1s[1], "beta_g2": g2s[0], "gamma_g2": g2s[1], "delta_g1": g1s[2], "delta_g2": g2s[2],
          "ic": [g1s[3], g1s[4]]}
    return {"vk": vk, "h": g1s[:3], "l": g1s[3:5], "a": g1s[:4], "b_g1": g1s[1:3], "b_g2": g2s[:2]}


def test_file_info_on_oracle_files_and_truncations():
    from bazuka_b200 import groth16 as BG
    blob = BP.write(small_params())
    want = {"n_ic": 2, "n_h": 3, "n_l": 2, "n_a": 4, "n_b_g1": 2, "n_b_g2": 2, "bytes": len(blob)}
    assert BG.parameters_info(blob) == want
    assert BG.parameters_info(blob + b"trailing bytes are not read") == want
    assert BP.info(blob)["bytes"] == len(blob)
    import bazuka_b200 as B
    # every header boundary (before and after each length prefix) and inside a point
    cuts = [0, 1, 864, 866, 868]
    off = 868 + 2 * 96
    for k, size in (("h", 96), ("l", 96), ("a", 96), ("b_g1", 96), ("b_g2", 192)):
        cuts += [off, off + 2, off + 4, off + 4 + size // 2]
        off += 4 + want["n_" + k] * size
    cuts.append(len(blob) - 1)
    for cut in cuts:
        with pytest.raises(B.BzkError) as e:
            BG.parameters_info(blob[:cut])
        assert e.value.status == -8, cut


def test_file_info_struct_matches_the_header(tmp_path):
    from bazuka_b200 import groth16 as BG
    fs = list(BG.PARAMS_FILE_INFO.names)
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "bzk.h"', 'int main(void) {',
           'printf("%zu", sizeof(bzk_params_file_info));'] + [f'printf(" %zu", offsetof(bzk_params_file_info, {f}));' for f in fs] + \
          ['printf("\\n");', "return 0;", "}"]
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    size, *offs = subprocess.check_output([str(exe)], text=True).split()
    assert BG.PARAMS_FILE_INFO.itemsize == int(size)
    assert [BG.PARAMS_FILE_INFO.fields[f][1] for f in fs] == [int(o) for o in offs]


def test_new_status_codes_have_texts():
    from bazuka_b200 import _lib
    lib = _lib.load()
    assert lib.bzk_strerror(-8) == b"bad key file encoding"
    assert lib.bzk_strerror(-9) == b"point not in the prime-order subgroup"
    assert _lib.ERRORS[-8] == "BZK_ERR_BAD_ENCODING" and _lib.ERRORS[-9] == "BZK_ERR_NOT_IN_SUBGROUP"
