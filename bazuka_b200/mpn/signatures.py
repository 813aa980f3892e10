"""EdDSA signature checks of MPN transactions and withdrawals in batches on the GPU (csrc/jubjub.cu).

The reference checks `tx.verify_signature()` one transaction at a time as it enters the mempool (src/blockchain/mempool.rs);
here a whole peer response is checked in one call, with exactly the reference's verdict (include/bzk.h, "EdDSA signature
checks in batches").  Each function returns a bool array, True where the signature is accepted.

    ok = verify_items(ctx, pks, messages, sigs)      # JubJub::verify on (compressed key, message, signature)
    ok = verify_transactions(ctx, txs)               # MpnTransaction::verify_signature
    ok = verify_bytes(ctx, KIND_TRANSACTIONS, blob)  # bincode of Vec<MpnTransaction> (or KIND_WITHDRAWS: Vec<MpnWithdraw>)"""
import ctypes as ct

import numpy as np

from . import native as N
from .ledger import _TX, pack_txs

ITEM = np.dtype([("pk_x", "<u8", 4), ("pk_odd", "u1"), ("pad", "u1", 7), ("message", "<u8", 4), ("sig_rx", "<u8", 4), ("sig_ry", "<u8", 4),
                 ("sig_s", "<u8", 4)])   # bzk_eddsa_item
assert ITEM.itemsize == 168

KIND_WITHDRAWS, KIND_TRANSACTIONS = 1, 2   # as bzk_mpn_work_info.kind (deposits carry L1 ed25519 signatures: not here)


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
