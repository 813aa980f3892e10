"""GPU tier of the batch EdDSA checks (csrc/jubjub.cu, bazuka_b200/mpn/signatures.py): every verdict equals the Python
restatement of the reference's `JubJub::verify` (tests/eddsa_cases.py) and, where it applies, libbzk's host call
bzk_jubjub_eddsa_verify — on signature families with tampering, non-canonical scalars, undecompressable keys and small-order
components, at sizes around the warp and the chunk, on transactions and on the bincode images `prepare_works` takes."""
import ctypes as ct

import numpy as np
import pytest

import eddsa_cases as E
from bazuka_b200._lib import BzkError
from bazuka_b200.mpn import dw as DW, native as N, signatures as S, update as U, wire as Wr, works as Wk

pytestmark = pytest.mark.gpu

CHUNK = 1 << 18   # items per pass through the context's arena (csrc/jubjub.cu)
R = N.R


def _ptr(a):
    return ct.c_void_p(a.ctypes.data)


@pytest.fixture(scope="module")
def fams():
    cases = E.families(b"f") + E.families(b"g")
    items = S.pack_items([c[1] for c in cases], [c[2] for c in cases], [{"r": c[3], "s": c[4]} for c in cases])
    want = np.array([E.expected(*c[1:]) for c in cases])
    return cases, items, want


def test_signature_families_match_the_restatement_and_the_host_call(ctx, fams):
    from bazuka_b200.api import HostPoseidon
    cases, items, want = fams
    got = S.verify_items(ctx, [c[1] for c in cases], [c[2] for c in cases], [{"r": c[3], "s": c[4]} for c in cases])
    for c, g, w in zip(cases, got, want):
        assert g == w, c[0]
    names = {c[0]: g for c, g in zip(cases, got)}
    assert names["valid"] and names["s+ORDER"] and not names["s+1"] and not names["key does not decompress"]
    assert 0 < sum(g for c, g in zip(cases, got) if c[0].startswith("torsion")) < sum(c[0].startswith("torsion") for c in cases)
    hp = HostPoseidon()
    for (name, pk, msg, r, s), g in zip(cases, got):
        a = N.jj_decompress_checked(pk)
        if a is not None:
            assert hp.eddsa_verify(N.JJ_D, a, msg, r, s) == g, name
    hp.free()


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, CHUNK + 3])
def test_verdicts_land_on_their_items_at_every_size(ctx, fams, n):
    _, items, want = fams
    idx = np.random.default_rng(n).integers(0, len(items), n)   # every family at known, shuffled positions
    k = min(n, len(items))
    idx[:k] = np.arange(k)
    got = S.verify_items(ctx, items[idx], None, None)
    assert got.shape == (n,) and (got == want[idx]).all()
    ok, n_ok = np.full(n, 7, np.uint8), ct.c_uint64()
    d = np.frombuffer(N.JJ_D.to_bytes(32, "little"), np.uint64).copy()
    sel = np.ascontiguousarray(items[idx])
    assert ctx._l.bzk_jubjub_eddsa_verify_batch(ctx._h, _ptr(d), _ptr(sel), n, _ptr(ok), ct.byref(n_ok)) == 0
    assert n_ok.value == int(want[idx].sum()) and set(np.unique(ok)) <= {0, 1}


def test_verdicts_do_not_depend_on_batching(ctx, fams):
    _, items, want = fams
    one = np.array([S.verify_items(ctx, items[k:k + 1], None, None)[0] for k in range(len(items))])
    perm = np.random.default_rng(3).permutation(len(items))
    shuffled = np.empty(len(items), bool)
    shuffled[perm] = S.verify_items(ctx, items[perm], None, None)
    assert (one == want).all() and (shuffled == want).all() and (S.verify_items(ctx, items, None, None) == want).all()


def _tx(keys, s, d, nonce, amount, fee):
    t = U.MpnTransaction(nonce, N.jj_compress(keys[s][0]), N.jj_compress(keys[d][0]), amount, fee)
    t.sign(keys[s][1])
    return t


def _tx_expected(t):
    if N.jj_decompress_checked(t.dst_pub_key) is None:
        return False
    return E.expected(t.src_pub_key, t.hash(), t.sig["r"], t.sig["s"])


def _transactions():
    from test_mpn_cpu import make_state
    import copy
    _, keys = make_state(3, 3, 4)
    custom = N.poseidon([5, 6])
    txs = [_tx(keys, 0, 1, 1, U.Money(U.ZIESHA, 100), U.Money(U.ZIESHA, 1)), _tx(keys, 1, 2, 7, U.Money(0, 5), U.Money(U.ZIESHA, 2)),
           _tx(keys, 2, 3, 3, U.Money(custom, 9), U.Money(custom, 4)), _tx(keys, 3, 0, 1, U.Money(U.ZIESHA, 1), U.Money(0, 0))]
    out = list(txs)
    for t in txs:
        for field, value in (("nonce", t.nonce + 1), ("amount", U.Money(t.amount.token_id, t.amount.amount + 1)),
                             ("fee", U.Money(t.fee.token_id, t.fee.amount + 1)), ("amount", U.Money(custom if t.amount.token_id != custom else 1, t.amount.amount)),
                             ("fee", U.Money(0 if t.fee.token_id else U.ZIESHA, t.fee.amount))):
            m = copy.deepcopy(t)
            setattr(m, field, value)
            out.append(m)
    bad_x = next(x for x in range(1, 100) if N.jj_decompress_checked((x, False)) is None)
    m = copy.deepcopy(txs[0])
    m.dst_pub_key = (bad_x, False)
    out.append(m)
    m = copy.deepcopy(txs[1])
    m.src_pub_key = txs[2].src_pub_key
    out.append(m)
    return out


def test_transactions_match_the_restatement_on_tx_hash(ctx):
    from bazuka_b200.mpn.ledger import pack_txs
    txs = _transactions()
    want = np.array([_tx_expected(t) for t in txs])
    assert want[:4].all() and not want[4:].any()
    assert (S.verify_transactions(ctx, txs) == want).all()
    assert (S.verify_transactions(ctx, pack_txs(txs)) == want).all()


def _vec(items, enc):
    w = Wr.Writer()
    w.vec(items, enc)
    return bytes(w.b)


def _tx_bytes(txs):
    return _vec([{"nonce": t.nonce, "src_pub_key": tuple(t.src_pub_key), "dst_pub_key": tuple(t.dst_pub_key), "amount": Wk._money_w(t.amount),
                  "fee": Wk._money_w(t.fee), "sig": {"r": tuple(t.sig["r"]), "s": t.sig["s"]}} for t in txs], Wr.enc_mpn_tx)


def _withdrawals():
    from test_mpn_cpu import make_state
    _, keys = make_state(3, 3, 3)
    out = []
    for k in range(6):
        pay = {"memo": "w%d" % k, "contract_id": 0x1234, "withdraw_circuit_id": 0, "calldata": 0, "dst": bytes([k]) * 32,
               "amount": {"token_id": "ziesha", "amount": 10 + k}, "fee": {"token_id": "ziesha", "amount": 1}}
        w = DW.MpnWithdraw(N.jj_compress(keys[k % 3][0]), 1 + k, amount=U.Money(U.ZIESHA, 10 + k), fee=U.Money(U.ZIESHA, 1))
        w.fingerprint = Wk.withdraw_fingerprint(pay)
        w.sign(keys[k % 3][1])
        item = {"mpn_address": tuple(w.mpn_address), "mpn_withdraw_nonce": w.mpn_withdraw_nonce, "mpn_sig": {"r": tuple(w.mpn_sig["r"]), "s": w.mpn_sig["s"]},
                "payment": pay}
        if k == 3:
            item["mpn_withdraw_nonce"] += 1                                   # the signed nonce is part of the message
        if k == 4:
            item["payment"] = dict(pay, amount={"token_id": "ziesha", "amount": 99})   # another payment: another fingerprint
        if k == 5:
            item["mpn_address"] = tuple(N.jj_compress(keys[0][0]))
        out.append(item)
    return out


def _wd_expected(w):
    msg = N.poseidon([Wk.withdraw_fingerprint(w["payment"]), w["mpn_withdraw_nonce"]])
    return E.expected(w["mpn_address"], msg, w["mpn_sig"]["r"], w["mpn_sig"]["s"])


def test_bincode_images_match_the_struct_path_and_the_restatement(ctx):
    txs = _transactions()
    ub = _tx_bytes(txs)
    assert (S.verify_bytes(ctx, S.KIND_TRANSACTIONS, ub) == S.verify_transactions(ctx, txs)).all()
    assert (S.verify_bytes(ctx, S.KIND_TRANSACTIONS, ub) == np.array([_tx_expected(t) for t in txs])).all()
    wds = _withdrawals()
    wb = _vec(wds, Wr.enc_mpn_withdraw)
    want = np.array([_wd_expected(w) for w in wds])
    assert list(want) == [True, True, True, False, False, False]
    assert (S.verify_bytes(ctx, S.KIND_WITHDRAWS, wb) == want).all()
    assert len(S.verify_bytes(ctx, S.KIND_TRANSACTIONS, _vec([], Wr.enc_mpn_tx))) == 0
    # malformed images and kind 0 are refused with ok untouched; ok == NULL gives the count
    lib, d = ctx._l, np.frombuffer(N.JJ_D.to_bytes(32, "little"), np.uint64).copy()
    unreduced = ub[:-32] + b"\xff" * 32                                       # the last transaction's sig.s
    for kind, blob in ((2, ub[:-1]), (2, ub + b"\x00"), (2, unreduced), (1, wb[:-5]), (0, ub), (3, ub)):
        ok, n = np.full(len(txs), 7, np.uint8), ct.c_uint64(12345)
        assert lib.bzk_mpn_signatures_verify_bytes(ctx._h, _ptr(d), kind, blob, len(blob), _ptr(ok), len(ok), ct.byref(n), None) == -1, kind
        assert (ok == 7).all()
    n = ct.c_uint64()
    assert lib.bzk_mpn_signatures_verify_bytes(ctx._h, _ptr(d), 2, ub, len(ub), None, 0, ct.byref(n), None) == 0 and n.value == len(txs)
    ok = np.full(len(txs), 7, np.uint8)
    assert lib.bzk_mpn_signatures_verify_bytes(ctx._h, _ptr(d), 2, ub, len(ub), _ptr(ok), len(txs) - 1, ct.byref(n), None) == -1 and (ok == 7).all()
    with pytest.raises(BzkError):
        S.verify_bytes(ctx, 0, ub)


def test_errors(ctx, fams):
    import bazuka_b200 as B
    _, items, _ = fams
    lib, d = ctx._l, np.frombuffer(N.JJ_D.to_bytes(32, "little"), np.uint64).copy()
    ok, n_ok = np.full(4, 7, np.uint8), ct.c_uint64(9)
    assert lib.bzk_jubjub_eddsa_verify_batch(ctx._h, _ptr(d), _ptr(items), 4, None, None) == -1
    assert lib.bzk_jubjub_eddsa_verify_batch(ctx._h, _ptr(d), None, 4, _ptr(ok), None) == -1
    assert lib.bzk_mpn_tx_verify_batch(ctx._h, _ptr(d), None, 1, _ptr(ok), None) == -1
    bad_d = np.frombuffer((N.JJ_D + R).to_bytes(32, "little"), np.uint64).copy()
    assert lib.bzk_jubjub_eddsa_verify_batch(ctx._h, _ptr(bad_d), _ptr(items), 4, _ptr(ok), None) == -1 and (ok == 7).all()
    assert lib.bzk_jubjub_eddsa_verify_batch(ctx._h, _ptr(d), None, 0, None, ct.byref(n_ok)) == 0 and n_ok.value == 0
    bare = B.Context(0, load_poseidon=False)
    with pytest.raises(BzkError) as e:
        S.verify_items(bare, [(1, False)], [1], [{"r": (0, 1), "s": 0}])
    assert e.value.status == -5
    with pytest.raises(BzkError) as e:
        S.verify_transactions(bare, _transactions()[:1])
    assert e.value.status == -5
    bare.close()


def test_filter_then_prepare_works_then_prove(ctx, cref):
    """transfers with one forged signature: filtered through bzk_mpn_signatures_verify_bytes, the rest go through
    bzk_mpn_prepare_works and the one-call prover, and `MpnWork::verify` accepts the proof"""
    from bazuka_b200.mpn.ledger import NativeLedger
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    from bazuka_b200.mpn.worker import MpnUpdateWorker
    from test_mpn_cpu import make_state, transfer
    from test_wire_cpu import _config
    A, T, B = 3, 3, 1
    st, keys = make_state(A, T, 3)
    forged = transfer(keys, 0, 2, 2)
    forged.sig = dict(forged.sig, s=forged.sig["s"] + 1)
    txs = [transfer(keys, 0, 1, 1), transfer(keys, 1, 2, 1), forged, transfer(keys, 2, 0, 1)]
    mask = S.verify_bytes(ctx, S.KIND_TRANSACTIONS, _tx_bytes(txs))
    assert list(mask) == [True, True, False, True]
    ub = _tx_bytes([t for t, m in zip(txs, mask) if m])
    wu = MpnUpdateWorker(ctx, A, T, B, cref.fr_random(301, 5))
    cw = Wr.Writer()
    Wr.enc_config(cw, dict(_config(num=(0, 0, 1)), update_vk=bytes(wu.vk_blob)))
    cb = bytes(cw.b)
    led = NativeLedger(ctx, A, T)
    for i, a in st.accounts.items():
        led.set_account(i, a)
    rw, fee = np.array([11, 22, 33], np.uint64), np.frombuffer(U.ZIESHA.to_bytes(32, "little"), np.uint64).copy()
    fork, buf, ln, n = ct.c_void_p(), ct.c_void_p(), ct.c_size_t(), ct.c_uint64()
    ctx._check(ctx._l.bzk_mpn_prepare_works(ctx._h, led._h, cb, len(cb), None, 0, None, 0, ub, len(ub), _ptr(rw), 9, _ptr(fee), ct.byref(fork), ct.byref(buf),
                                            ct.byref(ln), ct.byref(n)))
    works = Wr.get_mpn_work_response_from_bytes(ct.string_at(buf, ln.value))
    ctx._l.bzk_buffer_free(buf)
    ctx._l.bzk_mpn_state_free(fork)
    assert n.value == 1 and len(works[0]["data"][1]) == 3
    nat = Wk.NativeMpnProver(ctx)
    circ = NativeUpdateCircuit(A, T, B)
    nat.add_circuit("update", circ, wu.pk)
    circ.free()
    me = bytes(range(32))
    blob = Wr.work_to_bytes(works[0])
    r, s = cref.fr_random(77, 2)
    zk = nat.prove(blob, me, r, s)
    h = ct.c_void_p()
    assert ctx._l.bzk_mpn_work_decode(blob, len(blob), ct.byref(h), None) == 0
    assert ctx._l.bzk_mpn_work_verify(h, me, zk[4:]) == 1
    ctx._l.bzk_mpn_work_free(h)
    nat.free()
    wu.free()
    led.free()
