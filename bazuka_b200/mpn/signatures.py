"""Signature checks of MPN transactions and withdrawals (JubJub EdDSA, csrc/jubjub.cu) and of deposits (Ed25519,
csrc/ed25519.cu) in batches on the GPU.

The reference checks `tx.verify_signature()` one transaction at a time as it enters the mempool (src/blockchain/mempool.rs);
here a whole peer response is checked in one call, with exactly the reference's verdict (include/bzk.h, "EdDSA signature
checks in batches").  Each function returns a bool array, True where the signature is accepted.

    ok = verify_items(ctx, pks, messages, sigs)      # JubJub::verify on (compressed key, message, signature)
    ok = verify_transactions(ctx, txs)               # MpnTransaction::verify_signature
    ok = verify_bytes(ctx, KIND_TRANSACTIONS, blob)  # bincode of Vec<MpnTransaction> (or KIND_WITHDRAWS: Vec<MpnWithdraw>)

Deposits carry the L1 payment's Ed25519 signature (ed25519-dalek 1.x `PublicKey::verify`, include/bzk.h "Ed25519 signature
checks"), checked by the same kind of batch call:

    ok = verify_ed25519(ctx, pks, messages, sigs)    # Ed25519::verify on (32-byte key, message bytes, 64-byte signature)
    ok = verify_deposits(ctx, blob)                  # ContractDeposit::verify_signature of each item of a Vec<MpnDeposit>"""
import ctypes as ct

import numpy as np

from . import native as N
from .ledger import _TX, pack_txs

ITEM = np.dtype([("pk_x", "<u8", 4), ("pk_odd", "u1"), ("pad", "u1", 7), ("message", "<u8", 4), ("sig_rx", "<u8", 4), ("sig_ry", "<u8", 4),
                 ("sig_s", "<u8", 4)])   # bzk_eddsa_item
assert ITEM.itemsize == 168

KIND_WITHDRAWS, KIND_TRANSACTIONS = 1, 2   # as bzk_mpn_work_info.kind (deposits: verify_deposits)


def _u256(v):
    """a 256-bit integer as limbs, not reduced: a scalar >= r reaches the check and is rejected there"""
    return np.frombuffer(int(v).to_bytes(32, "little"), dtype=np.uint64)


def _curve_d():
    return _u256(N.JJ_D).copy()


def pack_items(pks, messages, sigs):
    """compressed keys (x, odd), messages, signatures {"r": (x, y), "s": s} -> array of bzk_eddsa_item"""
    if not len(pks) == len(messages) == len(sigs):
        raise ValueError("pks, messages and sigs differ in length")
    out = np.zeros(len(pks), dtype=ITEM)
    for k, (pk, m, sig) in enumerate(zip(pks, messages, sigs)):
        o = out[k]
        o["pk_x"], o["pk_odd"], o["message"] = _u256(pk[0]), int(bool(pk[1])), _u256(m)
        o["sig_rx"], o["sig_ry"], o["sig_s"] = _u256(sig["r"][0]), _u256(sig["r"][1]), _u256(sig["s"])
    return out


def _run(ctx, fn, arr):
    ok = np.zeros(len(arr), dtype=np.uint8)
    ctx._check(fn(ctx._h, _curve_d().ctypes.data_as(ct.c_void_p), arr.ctypes.data_as(ct.c_void_p), len(arr), ok.ctypes.data_as(ct.c_void_p), None))
    return ok.astype(bool)


def verify_items(ctx, pks, messages, sigs):
    """`JubJub::verify` on each (key, message, signature); `pks`, `messages` and `sigs` may also be given as one packed ITEM
    array in `pks` with the other two None"""
    items = pks if isinstance(pks, np.ndarray) and pks.dtype == ITEM else pack_items(pks, messages, sigs)
    return _run(ctx, ctx._l.bzk_jubjub_eddsa_verify_batch, np.ascontiguousarray(items))


def verify_transactions(ctx, txs):
    """`MpnTransaction::verify_signature` on a list of update.MpnTransaction or a packed ledger._TX array"""
    arr = txs if isinstance(txs, np.ndarray) else pack_txs(txs)
    if arr.dtype != _TX:
        raise ValueError("expected update.MpnTransaction objects or a ledger._TX array")
    return _run(ctx, ctx._l.bzk_mpn_tx_verify_batch, np.ascontiguousarray(arr))


def verify_bytes(ctx, kind, blob):
    """the signature of every item of a bincode `Vec<MpnWithdraw>` (KIND_WITHDRAWS) or `Vec<MpnTransaction>` (KIND_TRANSACTIONS)
    image, as bzk_mpn_prepare_works takes them; a malformed image raises BzkError(BZK_ERR_BAD_ARG)"""
    blob = bytes(blob)
    d, n = _curve_d(), ct.c_uint64()
    fn = ctx._l.bzk_mpn_signatures_verify_bytes
    ctx._check(fn(ctx._h, d.ctypes.data_as(ct.c_void_p), int(kind), blob, len(blob), None, 0, ct.byref(n), None))
    ok = np.zeros(n.value, dtype=np.uint8)
    ctx._check(fn(ctx._h, d.ctypes.data_as(ct.c_void_p), int(kind), blob, len(blob), ok.ctypes.data_as(ct.c_void_p), len(ok), ct.byref(n), None))
    return ok.astype(bool)


def verify_ed25519(ctx, pks, messages, sigs):
    """`Ed25519::verify` on each (32-byte key, message bytes, 64-byte signature), one GPU thread per signature; messages may
    have any length (the TransactionAndDelta arm passes bincode(tx.sig_state_excluded()))"""
    if not len(pks) == len(messages) == len(sigs):
        raise ValueError("pks, messages and sigs differ in length")
    n = len(pks)
    pk = b"".join(bytes(k) for k in pks)
    sg = b"".join(bytes(s) for s in sigs)
    if len(pk) != 32 * n or len(sg) != 64 * n:
        raise ValueError("an ed25519 key is 32 bytes and a signature 64")
    msgs = [bytes(m) for m in messages]
    offs = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum([len(m) for m in msgs], out=offs[1:])
    blob = b"".join(msgs)
    ok = np.zeros(n, dtype=np.uint8)
    ctx._check(ctx._l.bzk_ed25519_verify_batch(ctx._h, pk, sg, blob, offs.ctypes.data_as(ct.c_void_p), n, ok.ctypes.data_as(ct.c_void_p), None))
    return ok.astype(bool)


def verify_deposits(ctx, blob):
    """`ContractDeposit::verify_signature` of every item of a bincode `Vec<MpnDeposit>` image, as bzk_mpn_prepare_works takes
    it (False where the signature is None or not 64 bytes); a malformed image raises BzkError(BZK_ERR_BAD_ARG)"""
    blob = bytes(blob)
    n = ct.c_uint64()
    fn = ctx._l.bzk_mpn_deposits_verify_bytes
    ctx._check(fn(ctx._h, blob, len(blob), None, 0, ct.byref(n), None))
    ok = np.zeros(n.value, dtype=np.uint8)
    ctx._check(fn(ctx._h, blob, len(blob), ok.ctypes.data_as(ct.c_void_p), len(ok), ct.byref(n), None))
    return ok.astype(bool)
