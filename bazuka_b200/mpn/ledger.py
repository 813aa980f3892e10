"""ctypes front-end of the native MPN ledger and update builder (csrc/mpn_host.cu).

    led = NativeLedger(ctx, A, T)
    led.set_account(index, MpnAccount(...))
    raws, ext, accepted, public = led.update_build(txs, log4_batch)       # rows for the witness program

`raws` [4^B, n_raw, 4] / `ext` [4^B, 2, 4] are canonical uint64 images, exactly what bzk_witness_run_dev consumes
(`UpdateWitnessGpu.witness_rows`); `public` = {"state", "aux_data", "next_state"} as Python ints."""
import ctypes as ct

import numpy as np

from . import native as N
from .cs import R
from .update import ZIESHA, MpnAccount

_TX = np.dtype([("nonce", "<u8"), ("amount", "<u8"), ("fee", "<u8"), ("src_pk_odd", "u1"), ("dst_pk_odd", "u1"), ("pad", "u1", 6),
                ("src_pk_x", "<u8", 4), ("dst_pk_x", "<u8", 4), ("amount_token_id", "<u8", 4), ("fee_token_id", "<u8", 4),
                ("sig_rx", "<u8", 4), ("sig_ry", "<u8", 4), ("sig_s", "<u8", 4)])
assert _TX.itemsize == 32 + 7 * 32


_DEP = np.dtype([("pk_x", "<u8", 4), ("pk_odd", "u1"), ("pad", "u1", 7), ("token_id", "<u8", 4), ("amount", "<u8"), ("src_id", "<u8")])
_WD = np.dtype([("pk_x", "<u8", 4), ("pk_odd", "u1"), ("check_calldata", "u1"), ("pad", "u1", 2), ("nonce", "<u4"), ("sig_rx", "<u8", 4),
                ("sig_ry", "<u8", 4), ("sig_s", "<u8", 4), ("amount_token_id", "<u8", 4), ("fee_token_id", "<u8", 4), ("fingerprint", "<u8", 4),
                ("amount", "<u8"), ("fee", "<u8"), ("calldata", "<u8", 4)])
assert _DEP.itemsize == 88 and _WD.itemsize == 8 * 32 + 24


def _canon(v):
    return np.frombuffer((v % R).to_bytes(32, "little"), dtype=np.uint64)


def _int(a):
    return int.from_bytes(np.ascontiguousarray(a, dtype=np.uint64).tobytes(), "little")


def pack_txs(txs):
    """list of update.MpnTransaction -> array of bzk_mpn_tx"""
    out = np.zeros(len(txs), dtype=_TX)
    for k, tx in enumerate(txs):
        o = out[k]
        o["nonce"], o["amount"], o["fee"] = tx.nonce, tx.amount.amount, tx.fee.amount
        o["src_pk_odd"], o["dst_pk_odd"] = int(tx.src_pub_key[1]), int(tx.dst_pub_key[1])
        o["src_pk_x"], o["dst_pk_x"] = _canon(tx.src_pub_key[0]), _canon(tx.dst_pub_key[0])
        o["amount_token_id"], o["fee_token_id"] = _canon(tx.amount.token_id), _canon(tx.fee.token_id)
        o["sig_rx"], o["sig_ry"], o["sig_s"] = _canon(tx.sig["r"][0]), _canon(tx.sig["r"][1]), _canon(tx.sig["s"])
    return out


def pack_deposits(deps):
    """list of dw.MpnDeposit -> array of bzk_mpn_deposit"""
    out = np.zeros(len(deps), dtype=_DEP)
    src_ids = {}                                   # any hashable `src` -> a non-zero id (0 = not tracked)
    for k, d in enumerate(deps):
        o = out[k]
        o["pk_x"], o["pk_odd"], o["token_id"], o["amount"] = _canon(d.mpn_address[0]), int(d.mpn_address[1]), _canon(d.token_id), d.amount
        o["src_id"] = 0 if d.src is None else src_ids.setdefault(d.src, len(src_ids) + 1)
    return out


def pack_withdraws(ws):
    """list of dw.MpnWithdraw -> array of bzk_mpn_withdraw"""
    out = np.zeros(len(ws), dtype=_WD)
    for k, w in enumerate(ws):
        o = out[k]
        o["pk_x"], o["pk_odd"], o["nonce"] = _canon(w.mpn_address[0]), int(w.mpn_address[1]), w.mpn_withdraw_nonce
        o["sig_rx"], o["sig_ry"], o["sig_s"] = _canon(w.mpn_sig["r"][0]), _canon(w.mpn_sig["r"][1]), _canon(w.mpn_sig["s"])
        o["amount_token_id"], o["fee_token_id"], o["fingerprint"] = _canon(w.amount.token_id), _canon(w.fee.token_id), _canon(w.fingerprint)
        o["amount"], o["fee"] = w.amount.amount, w.fee.amount
        if w.calldata is not None:
            o["check_calldata"], o["calldata"] = 1, _canon(w.calldata)
    return out


class NativeLedger:
    def __init__(self, ctx, A, T):
        from ..api import _host_ptr
        self.ctx, self.A, self.T = ctx, A, T
        h = ct.c_void_p()
        jj_d = np.ascontiguousarray(_canon(N.JJ_D))
        ctx._check(ctx._l.bzk_mpn_state_create(ctx._h, A, T, _host_ptr(jj_d), ct.byref(h)))
        self._h = h
        w = ct.c_uint32()
        ctx._check(ctx._l.bzk_mpn_update_raw_width(A, T, ct.byref(w)))
        self.n_raw = w.value

    def free(self):
        if self._h:
            self.ctx._l.bzk_mpn_state_free(self._h)
            self._h = None

    @property
    def root(self):
        from ..api import _host_ptr
        out = np.zeros(4, dtype=np.uint64)
        self.ctx._check(self.ctx._l.bzk_mpn_state_root(self._h, _host_ptr(out)))
        return _int(out)

    def fork(self):
        """`db.fork_on_ram()` (/root/reference/src/mpn/mod.rs:313): an independent copy to build a block's batches on;
        drop it (free) when the block is not accepted — update_build writes the ledger it is called on."""
        c = NativeLedger.__new__(NativeLedger)
        c.ctx, c.A, c.T, c.n_raw = self.ctx, self.A, self.T, self.n_raw
        h = ct.c_void_p()
        self.ctx._check(self.ctx._l.bzk_mpn_state_clone(self._h, ct.byref(h)))
        c._h = h
        return c

    def info(self):
        """-> dict(state_hash, state_size, account_count, pending_accounts): `ZkCompressedState` for `MpnWork.new_root`,
        the chain-side account count and the accounts created on this fork so far."""
        from ..api import _host_ptr
        root = np.zeros(4, dtype=np.uint64)
        size, count, pend = ct.c_uint64(), ct.c_uint64(), ct.c_uint64()
        self.ctx._check(self.ctx._l.bzk_mpn_state_info(self._h, _host_ptr(root), ct.byref(size), ct.byref(count), ct.byref(pend)))
        return {"state_hash": _int(root), "state_size": size.value, "account_count": count.value, "pending_accounts": pend.value}

    def commit_accounts(self):
        """the block built on this fork was applied: its new accounts enter the chain's address index"""
        self.ctx._check(self.ctx._l.bzk_mpn_state_commit_accounts(self._h))

    def apply_delta(self, delta, expect=None):
        """apply a block's MPN state delta, as a full node does (`update_contract` + `index_mpn_accounts`): `delta` is the dict
        `works.final_delta` returns ({locator: value | None}) or its bincode (`works.enc_delta`, bzk_mpn_state_delta's image);
        `expect` = {"state_hash", "state_size"} (either may be absent), the `ZkCompressedState` the block attested.  All or
        nothing: a refused delta (BzkError) leaves the ledger as it was.  A snapshot is a delta from the empty ledger.
        -> the number of entries applied."""
        from ..api import _host_ptr
        from . import wire as Wr
        from .works import enc_delta
        if isinstance(delta, dict):
            w = Wr.Writer()
            enc_delta(w, delta)
            delta = bytes(w.b)
        expect = expect or {}
        h = expect.get("state_hash")
        hb = np.ascontiguousarray(_canon(h)) if h is not None else None
        size = ct.c_uint64(expect["state_size"]) if expect.get("state_size") is not None else None
        n = ct.c_uint64()
        delta = bytes(delta)
        self.ctx._check(self.ctx._l.bzk_mpn_state_apply_delta(self.ctx._h, self._h, delta, len(delta), _host_ptr(hb) if hb is not None else None,
                                                              ct.byref(size) if size is not None else None, ct.byref(n)))
        return n.value

    def set_account(self, index, acc: MpnAccount):
        from ..api import _host_ptr
        idx = np.array(sorted(acc.tokens), dtype=np.uint32)
        ids = np.ascontiguousarray(np.stack([_canon(acc.tokens[i].token_id) for i in idx]) if len(idx) else np.zeros((0, 4), np.uint64))
        amts = np.array([acc.tokens[i].amount for i in idx], dtype=np.uint64)
        ax, ay = np.ascontiguousarray(_canon(acc.address[0])), np.ascontiguousarray(_canon(acc.address[1]))
        self.ctx._check(self.ctx._l.bzk_mpn_state_set_account(self.ctx._h, self._h, index, acc.tx_nonce, acc.withdraw_nonce, _host_ptr(ax), _host_ptr(ay),
                                                              _host_ptr(idx), _host_ptr(ids), _host_ptr(amts), len(idx)))

    def update_build(self, txs, log4_batch, fee_token=ZIESHA):
        from ..api import _host_ptr
        packed = txs if isinstance(txs, np.ndarray) else pack_txs(txs)
        slots = 1 << (2 * log4_batch)
        raws = np.zeros((slots, self.n_raw, 4), dtype=np.uint64)
        ext = np.zeros((slots, 2, 4), dtype=np.uint64)
        acc = np.zeros(max(len(packed), 1), dtype=np.uint8)
        pub = np.zeros((3, 4), dtype=np.uint64)
        n_acc = ct.c_uint64()
        fee = np.ascontiguousarray(_canon(fee_token))
        self.ctx._check(self.ctx._l.bzk_mpn_update_build(self.ctx._h, self._h, _host_ptr(packed), len(packed), log4_batch, _host_ptr(fee),
                                                         _host_ptr(raws), _host_ptr(ext), _host_ptr(acc), _host_ptr(pub), ct.byref(n_acc)))
        public = {"state": _int(pub[0]), "aux_data": _int(pub[1]), "next_state": _int(pub[2])}
        return raws, ext, acc[:len(packed)].astype(bool), public, n_acc.value

    def _dw_build(self, kind, packed, log4_batch):
        from ..api import _host_ptr
        A, T = self.A, self.T
        w1, w2, wr = (5, 9 + 3 * T + 3 * A, 4) if kind == "deposit" else (12, 12 + 6 * T + 3 * A, 7)
        slots = 1 << (2 * log4_batch)
        raws1, raws2 = np.zeros((slots, w1, 4), dtype=np.uint64), np.zeros((slots, w2, 4), dtype=np.uint64)
        roots, reveal = np.zeros((slots, 4), dtype=np.uint64), np.zeros((slots, wr, 4), dtype=np.uint64)
        acc = np.zeros(max(len(packed), 1), dtype=np.uint8)
        pub = np.zeros((3, 4), dtype=np.uint64)
        n_acc = ct.c_uint64()
        fn = self.ctx._l.bzk_mpn_deposit_build if kind == "deposit" else self.ctx._l.bzk_mpn_withdraw_build
        self.ctx._check(fn(self.ctx._h, self._h, _host_ptr(packed), len(packed), log4_batch, _host_ptr(raws1), _host_ptr(raws2), _host_ptr(roots),
                           _host_ptr(reveal), _host_ptr(acc), _host_ptr(pub), ct.byref(n_acc)))
        public = {"state": _int(pub[0]), "aux_data": _int(pub[1]), "next_state": _int(pub[2])}
        return {"raws1": raws1, "raws2": raws2, "roots": roots, "reveal": reveal, "accepted": acc[:len(packed)].astype(bool), "public": public,
                "n_accepted": n_acc.value}

    def deposit_build(self, deposits, log4_batch):
        """`mpn::deposit::deposit` (/root/reference/src/mpn/deposit.rs:11-233) natively -> dict of the rows
        bzk_mpn_dw_witness consumes (raws1, raws2, roots, reveal), the accepted mask and the three public values."""
        return self._dw_build("deposit", deposits if isinstance(deposits, np.ndarray) else pack_deposits(deposits), log4_batch)

    def withdraw_build(self, withdraws, log4_batch):
        """`mpn::withdraw::withdraw` (/root/reference/src/mpn/withdraw.rs:10-259) natively, signature check included."""
        return self._dw_build("withdraw", withdraws if isinstance(withdraws, np.ndarray) else pack_withdraws(withdraws), log4_batch)
