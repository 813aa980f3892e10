"""Blocks for the MPN worker's tests (CPU and GPU tier): a ledger, a block of deposits, withdrawals and transfers, and the
`GetMpnWorkResponse` bytes bzk_mpn_prepare_works makes of it on any context-like object (`_l`, `_h`, `_check`)."""
import ctypes as ct
import hashlib
import struct

import numpy as np

from bazuka_b200.mpn import dw as D, native as N, update as U, wire as Wr, works as Wk

R = N.R


def _ptr(a):
    return ct.c_void_p(a.ctypes.data)


def _canon(v):
    return np.frombuffer((v % R).to_bytes(32, "little"), dtype=np.uint64).copy()


def _vec(items, enc):
    w = Wr.Writer()
    w.vec(items, enc)
    return bytes(w.b)


def config(A, T, Bd, Bw, Bu, vks):
    """vks = {kind: Groth16VerifyingKey image}"""
    return {"log4_tree_size": A, "log4_token_tree_size": T, "log4_deposit_batch_size": Bd, "log4_withdraw_batch_size": Bw,
            "log4_update_batch_size": Bu, "mpn_contract_id": 0x1234, "mpn_num_update_batches": 1, "mpn_num_deposit_batches": 1,
            "mpn_num_withdraw_batches": 1, "deposit_vk": vks["deposit"], "withdraw_vk": vks["withdraw"], "update_vk": vks["update"]}


def config_bytes(cfg):
    w = Wr.Writer()
    Wr.enc_config(w, cfg)
    return bytes(w.b)


def opaque_vk(fill, n_ic=6):
    """a Groth16VerifyingKey image whose points are arbitrary limbs with the infinity flag clear (the CPU tier never pairs)"""
    g1 = bytes([fill]) * 96 + b"\x00"
    g2 = bytes([fill + 1]) * 192 + b"\x00"
    return g1 + g1 + g2 + g2 + g1 + g2 + struct.pack("<Q", n_ic) + g1 * n_ic


def block(A, T, n_acc=3, n_transfers=2):
    """accounts 0..n_acc-1 funded; a newcomer's deposit and a second deposit, one signed withdrawal, the newcomer spending in the
    same block and n_transfers - 1 more transfers.  -> (ledger model, deposits, withdraws, updates, deposit payments, withdraw payments)"""
    st, keys = U.MpnState(A, T), []
    for i in range(n_acc):
        pk, sk = N.eddsa_keys(b"acct%d" % i)
        keys.append((pk, sk))
        st.set(i, U.MpnAccount(0, 0, pk, {0: U.Money(U.ZIESHA, 10 ** 12)}))
    newcomer = N.eddsa_keys(b"dep-new")
    keys.append(newcomer)
    deposits = [D.MpnDeposit(N.jj_compress(newcomer[0]), U.ZIESHA, 5000), D.MpnDeposit(N.jj_compress(keys[0][0]), 77, 9)]
    dpay = {k: {"memo": "d%d" % k, "contract_id": 0x1234, "deposit_circuit_id": 0, "calldata": 0, "src": bytes([k + 1]) * 32,
                "amount": {"token_id": Wr.scalar_contract_id(d.token_id), "amount": d.amount}, "fee": {"token_id": "ziesha", "amount": 0},
                "nonce": k + 1, "sig": None} for k, d in enumerate(deposits)}
    w = D.MpnWithdraw(N.jj_compress(keys[1][0]), 1, amount=U.Money(U.ZIESHA, 100), fee=U.Money(U.ZIESHA, 2))
    pay = {"memo": "rent", "contract_id": 0x1234, "withdraw_circuit_id": 0, "calldata": 0, "dst": bytes(range(32)),
           "amount": {"token_id": "ziesha", "amount": 100}, "fee": {"token_id": "ziesha", "amount": 2}}
    w.fingerprint = Wk.withdraw_fingerprint(pay)
    w.sign(keys[1][1])
    pay["calldata"] = w.expected_calldata()

    def transfer(s, d, nonce, amount=1000, fee=10):
        tx = U.MpnTransaction(nonce, N.jj_compress(keys[s][0]), N.jj_compress(keys[d][0]), U.Money(U.ZIESHA, amount), U.Money(U.ZIESHA, fee))
        tx.sign(keys[s][1])
        return tx
    updates = [transfer(n_acc, 0, 1, amount=40, fee=1)]
    nonces = [0] * n_acc
    for k in range(n_transfers - 1):
        s = k % n_acc
        nonces[s] += 1
        updates.append(transfer(s, (s + 1) % n_acc, nonces[s]))
    return st, deposits, [w], updates, dpay, {0: pay}


def ledger(ctxlike, st, A, T):
    from bazuka_b200.mpn.ledger import NativeLedger
    led = NativeLedger(ctxlike, A, T)
    for i, a in st.accounts.items():
        led.set_account(i, a)
    assert led.root == st.root
    return led


def prepare_response(ctxlike, led, cfg, deposits, withdraws, updates, dpay, wpay, rewards=(11, 22, 33), height=9):
    """bzk_mpn_prepare_works on a fork of `led`: -> (GetMpnWorkResponse bytes, number of works)"""
    lib = ctxlike._l
    cb = config_bytes(cfg)
    db = _vec([{"mpn_address": tuple(d.mpn_address), "payment": dpay[k]} for k, d in enumerate(deposits)], Wr.enc_mpn_deposit)
    wb = _vec([{"mpn_address": tuple(w.mpn_address), "mpn_withdraw_nonce": w.mpn_withdraw_nonce, "mpn_sig": {"r": tuple(w.mpn_sig["r"]), "s": w.mpn_sig["s"]},
                "payment": wpay[k]} for k, w in enumerate(withdraws)], Wr.enc_mpn_withdraw)
    ub = _vec([{"nonce": t.nonce, "src_pub_key": tuple(t.src_pub_key), "dst_pub_key": tuple(t.dst_pub_key), "amount": Wk._money_w(t.amount),
                "fee": Wk._money_w(t.fee), "sig": {"r": tuple(t.sig["r"]), "s": t.sig["s"]}} for t in updates], Wr.enc_mpn_tx)
    rw = np.array(rewards, np.uint64)
    fee = _canon(U.ZIESHA)
    fork, buf, ln, n = ct.c_void_p(), ct.c_void_p(), ct.c_size_t(), ct.c_uint64()
    ctxlike._check(lib.bzk_mpn_prepare_works(ctxlike._h, led._h, cb, len(cb), db, len(db), wb, len(wb), ub, len(ub), _ptr(rw), height, _ptr(fee),
                                             ct.byref(fork), ct.byref(buf), ct.byref(ln), ct.byref(n)))
    out = ct.string_at(buf, ln.value)
    lib.bzk_buffer_free(buf)
    lib.bzk_mpn_state_free(fork)
    return out, n.value


def decode_response(lib, resp):
    """-> [(id, work handle)] (free each with bzk_mpn_work_free)"""
    n = ct.c_uint64()
    ids, hs = np.zeros(64, np.uint64), (ct.c_void_p * 64)()
    assert lib.bzk_mpn_get_work_response_decode(resp, len(resp), _ptr(ids), hs, 64, ct.byref(n)) == 0
    return [(int(ids[i]), ct.c_void_p(hs[i])) for i in range(n.value)]


def encode_work(lib, h):
    n = ct.c_size_t()
    assert lib.bzk_mpn_work_encode(h, None, 0, ct.byref(n)) == 0
    buf = ct.create_string_buffer(n.value)
    assert lib.bzk_mpn_work_encode(h, buf, n.value, ct.byref(n)) == 0
    return buf.raw


def seeded_blinding(seed, wid):
    """the worker's test hook: r, s = SHA3(seed || id || tag) mod r, as Montgomery limbs"""
    out = []
    for tag in b"rs":
        v = int.from_bytes(hashlib.sha3_256(bytes(seed) + struct.pack("<Q", wid) + bytes([tag])).digest(), "little") % R
        out.append(_canon(v * (1 << 256)))
    return out


def solution_proofs(body):
    """PostMpnSolutionRequest bytes -> (prover, {id: 387-byte proof})"""
    return Wr.post_mpn_solution_request_from_bytes(body)
