"""CPU tier: the three native transition builders (csrc/mpn_host.cu, host build) on a ledger whose nonces do not fit in 32 bits,
against the Python restatement; and the rows the builders write equal the rows the work decoder (csrc/mpn_wire.cu) recovers
from the works `bzk_mpn_prepare_works` makes of the same traffic."""
import ctypes as ct

import numpy as np

from bazuka_b200.mpn import dw as D, dw_witness as DW, native as N, update as U, wire as Wr, witness_program as W
from mpn_delta_cases import run_block
from test_mpn_cpu import transfer
from test_native_host_cpu import _canon_rows, _load, _ptr
from test_wire_cpu import _config, _scenario
from test_wire_native_cpu import _canon

A = T = 3
B = 1


def _check_dw(kind, rows, pub, trans):
    circ = (D.DepositCircuit if kind == "deposit" else D.WithdrawCircuit)(A, T, B, commitment=0, height=0, transitions=trans, **pub)
    want = [(DW.deposit_raws if kind == "deposit" else DW.withdraw_raws)(t, A, T) for t in circ.transitions]
    assert rows["public"] == pub and rows["n_accepted"] == len(trans)
    assert (rows["raws1"].reshape(-1, 4) == _canon_rows([v for a, _ in want for v in a])).all()
    assert (rows["raws2"].reshape(-1, 4) == _canon_rows([v for _, b in want for v in b])).all()
    assert (rows["roots"] == _canon_rows(DW.slot_roots(circ))).all()
    assert (rows["reveal"].reshape(-1, 4) == _canon_rows([v for r in DW.reveal_rows_native(kind, circ) for v in r])).all()


def test_builders_write_nonces_of_64_bits(hostmpn):
    """accounts whose tx_nonce / withdraw_nonce are 2^32 or more, and an update whose nonce is above 2^32: every row, entering
    root, revealed row, public value, accepted mask and `state_size` of a deposit, a withdraw and an update batch equal the
    Python restatement's (the rows carry all 64 bits of a nonce)."""
    big = 1 << 32
    st, keys = U.MpnState(A, T), []
    for i, (tn, wn) in enumerate([(big + 5, 3), (7, 2 * big + 1), (big, big + 9)]):
        pk, sk = N.eddsa_keys(b"acct%d" % i)
        keys.append((pk, sk))
        st.set(i, U.MpnAccount(tn, wn, pk, {0: U.Money(U.ZIESHA, 10 ** 12)}))
    keys.append(N.eddsa_keys(b"newcomer"))
    led = _load(hostmpn, st, A, T)

    deps = [D.MpnDeposit(N.jj_compress(keys[1][0]), U.ZIESHA, 50), D.MpnDeposit(N.jj_compress(keys[2][0]), 77, 9),
            D.MpnDeposit(N.jj_compress(keys[3][0]), 77, 4)]
    pub, trans = D.deposit(st, deps, B)
    rows = led.deposit_build(deps, B)
    assert rows["accepted"].tolist() == [True, True, True] and led.root == st.root
    _check_dw("deposit", rows, pub, trans)
    assert led.info()["state_size"] == st.state_size

    w = D.MpnWithdraw(N.jj_compress(keys[0][0]), 4, amount=U.Money(U.ZIESHA, 100), fee=U.Money(U.ZIESHA, 2), fingerprint=4242)
    w.sign(keys[0][1])
    w.calldata = w.expected_calldata()
    stale = D.MpnWithdraw(N.jj_compress(keys[2][0]), 9, amount=U.Money(U.ZIESHA, 1), fee=U.Money(U.ZIESHA, 0), fingerprint=1)
    stale.sign(keys[2][1])
    pub, trans = D.withdraw(st, [w, stale], B)
    rows = led.withdraw_build([w, stale], B)
    assert rows["accepted"].tolist() == [True, False] and led.root == st.root
    _check_dw("withdraw", rows, pub, trans)
    assert led.info()["state_size"] == st.state_size

    txs = [transfer(keys, 2, 1, big + 1), transfer(keys, 0, 2, big + 6, amount=5), transfer(keys, 1, 0, 8, amount=3),
           transfer(keys, 0, 3, 6)]
    pub, trans, rej = U.update(st, txs, B)
    raws, ext, acc, public, n_acc = led.update_build(txs, B)
    assert acc.tolist() == [True, True, True, False] and rej == [txs[3]]
    assert n_acc == len(trans) and public == pub and led.root == st.root
    circ = U.UpdateCircuit(A, T, B, commitment=5, height=1, transitions=trans, **pub)
    assert (raws == np.stack([_canon_rows(W.raw_values(tr, A, T)) for tr in circ.transitions])).all()
    assert (ext == np.stack([_canon_rows([circ.fee_token, r]) for r in W.slot_roots(circ)])).all()
    assert led.info()["state_size"] == st.state_size
    led.free()


def test_builder_rows_equal_the_rows_decoded_from_prepare_works(hostmpn):
    """deposit -> withdraw -> update on one fork, once through the builders' C ABI and once through bzk_mpn_prepare_works and
    the work decoder (bzk_mpn_work_dw_rows, bzk_mpn_work_update_rows): the same rows, entering roots and revealed rows."""
    lib = hostmpn._l
    st, keys, deposits, withdraws, wpay, updates = _scenario()
    dpay = {k: {"memo": "", "contract_id": 0x1234, "deposit_circuit_id": 0, "calldata": 0, "src": bytes([k + 1]) * 32,
                "amount": {"token_id": Wr.scalar_contract_id(d.token_id), "amount": d.amount},
                "fee": {"token_id": "ziesha", "amount": 0}, "nonce": k + 1, "sig": None} for k, d in enumerate(deposits)}
    led = _load(hostmpn, st, A, T)
    image, fork_pw, n = run_block(hostmpn, led, _config(), deposits, withdraws, updates, dpay, wpay)
    assert n == 3
    ids, handles, count = np.zeros(3, np.uint64), np.zeros(3, np.uint64), ct.c_uint64()
    assert lib.bzk_mpn_get_work_response_decode(image, len(image), _ptr(ids), _ptr(handles), 3, ct.byref(count)) == 0 and count.value == 3
    hasher = ct.c_void_p()
    from bazuka_b200 import _lib
    blob = open(_lib.PARAMS_PATH, "rb").read()
    assert lib.bzk_poseidon_host_create(blob, len(blob), ct.byref(hasher)) == 0
    jj_d, fee = _canon(N.JJ_D), _canon(U.ZIESHA)

    direct = led.fork()
    built = {0: direct.deposit_build(deposits, B), 1: direct.withdraw_build(withdraws, B)}
    raws, ext, acc, _, n_acc = direct.update_build(updates, B)
    assert built[0]["n_accepted"] == 2 and built[1]["n_accepted"] == 1 and n_acc == 2
    assert direct.info() == fork_pw.info()
    for i, kind in ((0, "deposit"), (1, "withdraw")):
        rows = built[i]
        got = {k: np.zeros_like(rows[k]) for k in ("raws1", "raws2", "roots", "reveal")}
        assert lib.bzk_mpn_work_dw_rows(ct.c_void_p(int(handles[ids.tolist().index(i)])), hasher, _ptr(jj_d), _ptr(got["raws1"]), _ptr(got["raws2"]),
                                        _ptr(got["roots"]), _ptr(got["reveal"])) == 0
        for k in got:
            assert (got[k] == rows[k]).all(), (kind, k)
    raws2, ext2 = np.zeros_like(raws), np.zeros_like(ext)
    assert lib.bzk_mpn_work_update_rows(ct.c_void_p(int(handles[ids.tolist().index(2)])), hasher, _ptr(jj_d), _ptr(fee), _ptr(raws2), _ptr(ext2)) == 0
    assert (raws2 == raws).all() and (ext2 == ext).all()
    for h in handles:
        lib.bzk_mpn_work_free(ct.c_void_p(int(h)))
    lib.bzk_poseidon_host_free(hasher)
    for l in (direct, fork_pw, led):
        l.free()
