"""GPU tier of the Ed25519 checks (csrc/ed25519.cu, bazuka_b200/mpn/signatures.py): every batch verdict equals the host call
bzk_ed25519_verify and the big-integer restatement of ed25519-dalek 1.x `PublicKey::verify` (oracle/py/ed25519.py), on the
signature families of tests/ed25519_cases.py, at sizes around the warp, the block and the chunk, across the chunks' byte
budget, and on the bincode `Vec<MpnDeposit>` images `prepare_works` takes."""
import ctypes as ct

import numpy as np
import pytest

import ed25519_cases as E
from bazuka_b200 import api
from bazuka_b200._lib import BzkError
from bazuka_b200.mpn import native as N, signatures as S, update as U, wire as Wr
from oracle.py import ed25519 as O

pytestmark = pytest.mark.gpu

CHUNK = 1 << 18          # items per pass through the context's arena (csrc/ed25519.cu)
CHUNK_BYTES = 1 << 26    # message bytes per pass, unless one message alone is longer


def _ptr(a):
    return ct.c_void_p(a.ctypes.data)


@pytest.fixture(scope="module")
def fams():
    cases = E.families(b"f") + E.families(b"g", big=False)
    want = np.array([E.expected(*c[1:]) for c in cases])
    return cases, want


def _run(ctx, pks, msgs, sigs):
    """bzk_ed25519_verify_batch straight from arrays: (ok, n_ok)"""
    n = len(pks)
    offs = np.zeros(n + 1, np.uint64)
    np.cumsum([len(m) for m in msgs], out=offs[1:])
    pk, sg, blob = b"".join(pks), b"".join(sigs), b"".join(msgs)
    ok, n_ok = np.full(max(n, 1), 7, np.uint8), ct.c_uint64(12345)
    assert ctx._l.bzk_ed25519_verify_batch(ctx._h, pk, sg, blob, _ptr(offs), n, _ptr(ok), ct.byref(n_ok)) == 0
    return ok[:n], n_ok.value


def test_signature_families_match_the_host_call_and_the_oracle(ctx, fams):
    cases, want = fams
    got = S.verify_ed25519(ctx, [c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
    for c, g, w in zip(cases, got, want):
        assert g == w, c[0]
        assert api.ed25519_verify(c[1], c[2], c[3]) == w, c[0]
    names = dict(zip((c[0] for c in cases), got))
    assert names["honest"] and names["s = l - 1"] and not names["s = l"] and names["1 MiB message"] and not names["R -0"]
    assert names["mixed order 8 acc"] and not names["mixed order 8 rej"]


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, CHUNK - 1, CHUNK, CHUNK + 1])
def test_verdicts_land_on_their_items_at_every_size(ctx, fams, n):
    cases, want = fams
    small = [k for k, c in enumerate(cases) if len(c[2]) < 4096]
    idx = np.array(small)[np.random.default_rng(n).integers(0, len(small), n)]
    k = min(n, len(small))
    idx[:k] = small[:k]
    ok, n_ok = _run(ctx, [cases[i][1] for i in idx], [cases[i][2] for i in idx], [cases[i][3] for i in idx])
    assert ok.shape == (n,) and (ok == want[idx]).all() and n_ok == int(want[idx].sum())


def test_verdicts_across_the_byte_budget(ctx):
    """70 one-MiB messages (more than one chunk's bytes) between small ones, half of them tampered"""
    pk, sk = O.generate_keys(b"budget")
    base = bytes(np.random.default_rng(1).integers(0, 256, 1 << 20, dtype=np.uint8))
    pks, msgs, sigs, want = [], [], [], []
    for i in range(70):
        m = i.to_bytes(4, "little") + base[4:]
        sig = O.sign(sk, m)
        if i % 2:
            m = m[:-1] + bytes([m[-1] ^ 1])
        for mm, sg in ((m, sig), (b"s%d" % i, O.sign(sk, b"s%d" % i))):
            pks.append(pk); msgs.append(mm); sigs.append(sg); want.append(O.verify(pk, mm, sg))
    assert sum(len(m) for m in msgs) > CHUNK_BYTES and sum(want) == 105
    ok, n_ok = _run(ctx, pks, msgs, sigs)
    assert list(ok.astype(bool)) == want and n_ok == 105


def test_one_message_longer_than_the_byte_budget(ctx):
    pk, sk = O.generate_keys(b"huge")
    m = bytes(np.random.default_rng(2).integers(0, 256, CHUNK_BYTES + 1000, dtype=np.uint8))
    sig = O.sign(sk, m)
    small = [b"", b"a", b"bc"]
    pks = [pk] * 5
    msgs = [small[0], m, small[1], m[:-1], small[2]]
    sigs = [O.sign(sk, small[0]), sig, O.sign(sk, small[1]), sig, b"\x00" * 64]
    want = [True, True, True, False, False]
    ok, n_ok = _run(ctx, pks, msgs, sigs)
    assert list(ok.astype(bool)) == want and n_ok == 3
    assert api.ed25519_verify(pk, m, sig)


def test_verdicts_do_not_depend_on_batching(ctx, fams):
    cases, want = fams
    pks, msgs, sigs = [c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases]
    perm = np.random.default_rng(3).permutation(len(cases))
    shuffled = np.empty(len(cases), bool)
    shuffled[perm] = S.verify_ed25519(ctx, [pks[i] for i in perm], [msgs[i] for i in perm], [sigs[i] for i in perm])
    halves = np.concatenate([S.verify_ed25519(ctx, pks[:17], msgs[:17], sigs[:17]), S.verify_ed25519(ctx, pks[17:], msgs[17:], sigs[17:])])
    one = np.array([S.verify_ed25519(ctx, pks[k:k + 1], msgs[k:k + 1], sigs[k:k + 1])[0] for k in range(0, len(cases), 5)])
    assert (shuffled == want).all() and (halves == want).all() and (one == want[::5]).all()


def test_batch_argument_errors(ctx, fams):
    cases, _ = fams
    lib = ctx._l
    pk, m, sg = cases[0][1:]
    ok, n_ok = np.full(2, 7, np.uint8), ct.c_uint64(9)
    good = np.array([0, len(m), 2 * len(m)], np.uint64)
    pks, sigs, msgs = pk * 2, sg * 2, m * 2
    assert lib.bzk_ed25519_verify_batch(ctx._h, pks, sigs, msgs, _ptr(good), 2, _ptr(ok), ct.byref(n_ok)) == 0 and list(ok) == [1, 1] and n_ok.value == 2
    ok[:] = 7
    for bad in (np.array([1, len(m), 2 * len(m)], np.uint64), np.array([0, 2 * len(m), len(m)], np.uint64)):
        assert lib.bzk_ed25519_verify_batch(ctx._h, pks, sigs, msgs, _ptr(bad), 2, _ptr(ok), None) == -1
    assert lib.bzk_ed25519_verify_batch(ctx._h, None, sigs, msgs, _ptr(good), 2, _ptr(ok), None) == -1
    assert lib.bzk_ed25519_verify_batch(ctx._h, pks, None, msgs, _ptr(good), 2, _ptr(ok), None) == -1
    assert lib.bzk_ed25519_verify_batch(ctx._h, pks, sigs, None, _ptr(good), 2, _ptr(ok), None) == -1
    assert lib.bzk_ed25519_verify_batch(ctx._h, pks, sigs, msgs, None, 2, _ptr(ok), None) == -1
    assert lib.bzk_ed25519_verify_batch(ctx._h, pks, sigs, msgs, _ptr(good), 2, None, None) == -1
    assert lib.bzk_ed25519_verify_batch(None, pks, sigs, msgs, _ptr(good), 2, _ptr(ok), None) == -1
    assert (ok == 7).all()
    zero = np.zeros(3, np.uint64)   # empty messages: msgs may be NULL
    assert lib.bzk_ed25519_verify_batch(ctx._h, pks, sigs, None, _ptr(zero), 2, _ptr(ok), None) == 0 and list(ok) == [0, 0]
    assert lib.bzk_ed25519_verify_batch(ctx._h, None, None, None, None, 0, None, ct.byref(n_ok)) == 0 and n_ok.value == 0


# ---------------------------------------------------------------------------------------------------------------- deposits
def _payment(k, src, nonce=1, memo=None, amount=None):
    return {"memo": memo if memo is not None else "dep %d" % k, "contract_id": 0x1234, "deposit_circuit_id": 0, "calldata": 0, "src": src,
            "amount": {"token_id": "ziesha", "amount": amount if amount is not None else 10 + k}, "fee": {"token_id": "ziesha", "amount": 0},
            "nonce": nonce, "sig": None}


def _unsigned(pay):
    w = Wr.Writer()
    Wr.enc_contract_deposit(w, dict(pay, sig=None))
    return bytes(w.b)


def _signed(pay, sk):
    return dict(pay, sig=O.sign(sk, _unsigned(pay)))


def _dep_expected(pay):
    sig = pay["sig"]
    return sig is not None and len(sig) == 64 and O.verify(pay["src"], _unsigned(pay), sig)


def _image(addrs, pays):
    w = Wr.Writer()
    w.vec([{"mpn_address": tuple(a), "payment": p} for a, p in zip(addrs, pays)], Wr.enc_mpn_deposit)
    return bytes(w.b)


def _deposit_cases():
    pays = []
    for k in range(4):
        pk, sk = O.generate_keys(b"depositor %d" % k)
        pays.append(_signed(_payment(k, pk, nonce=k + 1), sk))
    good = pays[0]
    pays += [dict(good, memo="other memo"), dict(good, amount={"token_id": "ziesha", "amount": 11}), dict(good, nonce=2),
             dict(good, sig=None), dict(good, sig=good["sig"][:63]), dict(good, sig=good["sig"] + b"\x00"), dict(good, src=pays[1]["src"])]
    # small-order and undecompressable sources
    ts = E.torsion_points()
    for j in (0, 2, 1):
        src = O.compress(ts[j])
        pay = _payment(10 + j, src)
        for want in (True, False) if j else (True,):
            pays.append(dict(pay, sig=E.search_no_secret(src, _unsigned(pay), want, b"dep-so%d" % j)))
    pays.append(dict(_payment(20, E.undecompressable()), sig=good["sig"]))
    return pays


def test_deposit_images_match_the_oracle(ctx):
    pays = _deposit_cases()
    want = [_dep_expected(p) for p in pays]
    assert want[:4] == [True] * 4 and not any(want[4:11]) and sum(want) == 4 + 3
    addrs = [N.jj_compress(N.eddsa_keys(b"mpn %d" % k)[0]) for k in range(len(pays))]
    blob = _image(addrs, pays)
    assert list(S.verify_deposits(ctx, blob)) == want
    lib = ctx._l
    n, n_ok = ct.c_uint64(), ct.c_uint64()
    assert lib.bzk_mpn_deposits_verify_bytes(ctx._h, blob, len(blob), None, 0, ct.byref(n), None) == 0 and n.value == len(pays)
    ok = np.full(len(pays), 7, np.uint8)
    assert lib.bzk_mpn_deposits_verify_bytes(ctx._h, blob, len(blob), _ptr(ok), len(pays), ct.byref(n), ct.byref(n_ok)) == 0
    assert list(ok.astype(bool)) == want and n_ok.value == sum(want)
    # cap < n and malformed images: BZK_ERR_BAD_ARG, ok untouched
    bad_tag = _image(addrs[:1], [pays[0]])
    bad_tag = bad_tag[:-(8 + 64 + 1)] + b"\x02" + bad_tag[-(8 + 64):]          # Option tag 2
    for img, cap in ((blob, len(pays) - 1), (blob[:-1], len(pays)), (blob + b"\x00", len(pays)), (bad_tag, len(pays)), (blob[:5], len(pays))):
        ok[:] = 7
        assert lib.bzk_mpn_deposits_verify_bytes(ctx._h, img, len(img), _ptr(ok), cap, ct.byref(n), None) == -1
        assert (ok == 7).all()
    assert lib.bzk_mpn_deposits_verify_bytes(ctx._h, None, 4, _ptr(ok), len(ok), ct.byref(n), None) == -1
    assert lib.bzk_mpn_deposits_verify_bytes(ctx._h, blob, len(blob), _ptr(ok), len(ok), None, None) == -1
    with pytest.raises(BzkError):
        S.verify_deposits(ctx, blob[:-1])
    empty = _image([], [])
    assert len(S.verify_deposits(ctx, empty)) == 0
    # kind 0 stays refused by the JubJub call
    d = np.frombuffer(N.JJ_D.to_bytes(32, "little"), np.uint64).copy()
    assert lib.bzk_mpn_signatures_verify_bytes(ctx._h, _ptr(d), 0, blob, len(blob), _ptr(ok), len(ok), ct.byref(n), None) == -1


def test_filter_then_prepare_works(ctx):
    """forged deposits filtered out by bzk_mpn_deposits_verify_bytes: prepare_works on the survivors gives the same bytes as on
    the honest list alone"""
    from bazuka_b200.mpn.ledger import NativeLedger
    from test_mpn_cpu import make_state
    from test_wire_cpu import _config
    A, T = 3, 3
    st, keys = make_state(A, T, 4)
    honest, addrs = [], []
    for k in range(4):
        pk, sk = O.generate_keys(b"l1 %d" % k)
        honest.append(_signed(_payment(k, pk, nonce=1), sk))
        addrs.append(N.jj_compress(keys[k][0]))
    forged = [dict(honest[1], amount={"token_id": "ziesha", "amount": 1000}), dict(honest[2], sig=None), dict(honest[3], src=honest[0]["src"])]
    mixed_pays = [honest[0], forged[0], honest[1], forged[1], honest[2], forged[2], honest[3]]
    mixed_addrs = [addrs[0], addrs[1], addrs[1], addrs[2], addrs[2], addrs[3], addrs[3]]
    mask = S.verify_deposits(ctx, _image(mixed_addrs, mixed_pays))
    assert list(mask) == [True, False, True, False, True, False, True]
    kept = _image([a for a, m in zip(mixed_addrs, mask) if m], [p for p, m in zip(mixed_pays, mask) if m])
    assert kept == _image(addrs, honest)
    cw = Wr.Writer()
    Wr.enc_config(cw, _config(num=(1, 0, 0)))
    cb = bytes(cw.b)

    def works(db):
        led = NativeLedger(ctx, A, T)
        for i, a in st.accounts.items():
            led.set_account(i, a)
        rw, fee = np.array([11, 22, 33], np.uint64), np.frombuffer(U.ZIESHA.to_bytes(32, "little"), np.uint64).copy()
        fork, buf, ln, n = ct.c_void_p(), ct.c_void_p(), ct.c_size_t(), ct.c_uint64()
        ctx._check(ctx._l.bzk_mpn_prepare_works(ctx._h, led._h, cb, len(cb), db, len(db), None, 0, None, 0, _ptr(rw), 9, _ptr(fee), ct.byref(fork),
                                                ct.byref(buf), ct.byref(ln), ct.byref(n)))
        out = ct.string_at(buf, ln.value)
        ctx._l.bzk_buffer_free(buf)
        ctx._l.bzk_mpn_state_free(fork)
        led.free()
        return out, n.value

    got, n = works(kept)
    want, n_want = works(_image(addrs, honest))
    assert n == n_want == 1 and got == want
    assert len(Wr.get_mpn_work_response_from_bytes(got)[0]["data"][1]) == 4
