"""From a block's pending MPN traffic to works, and from a work to a proof — the validator's `prepare_works` and the
external prover's job, around the wire images of mpn/wire.py.

  prepare_works        /root/reference/src/mpn/mod.rs:298-424: on ONE fork of the ledger, `mpn_num_deposit_batches`
                       deposit batches, then the withdraw batches, then the update batches, the map of accounts created
                       on the way (`new_account_indices`) threaded through all of them; every batch becomes an `MpnWork`
                       {config, public_inputs, data, new_root, reward}.  (The validator's own reward deposit and the L1
                       balance bookkeeping of that function are chain state — out of scope, SURVEY §2.)
  MpnWork::verify      :281-295 — commitment from (prover, reward), then `check_proof`
  MpnProver            what the external worker ("zoro") does with a work: witness + Groth16 proof on the GPU
  WorkerClient         `BazukaClient::{get_mpn_works, post_mpn_worker, post_mpn_proof}` (/root/reference/src/client/mod.rs:428-464):
                       GET /bincode/mpn/work, POST /bincode/mpn/solution with bincode bodies (request signing — the node's
                       auth layer — is left to the caller through `headers`)
"""
import hashlib
import urllib.request

from . import dw as D
from . import native as N
from . import update as U
from . import wire as Wr

ZIESHA = U.ZIESHA


# ------------------------------------------------------------------ builder dataclasses <-> wire dicts
def _money_w(m): return {"token_id": Wr.scalar_contract_id(m.token_id), "amount": m.amount}
def _money_b(m): return U.Money(Wr.contract_id_scalar(m["token_id"]), m["amount"])


def _account_w(a):
    return {"tx_nonce": a.tx_nonce, "withdraw_nonce": a.withdraw_nonce, "address": tuple(a.address),
            "tokens": {k: _money_w(m) for k, m in sorted(a.tokens.items())}}


def _account_b(a):
    return U.MpnAccount(a["tx_nonce"], a["withdraw_nonce"], tuple(a["address"]), {k: _money_b(m) for k, m in a["tokens"].items()})


def withdraw_fingerprint(payment):
    """`ContractWithdraw::fingerprint` (/root/reference/src/core/transaction.rs:205-210): hash-to-scalar of the payment's
    bincode image with `calldata` zeroed."""
    w = Wr.Writer()
    Wr.enc_contract_withdraw(w, dict(payment, calldata=0))
    return int.from_bytes(hashlib.sha3_256(bytes(w.b)).digest(), "little") % N.R


def transitions_to_wire(kind, trans, payments=None):
    """builder transitions (update.UpdateTransition / dw.DepositTransition / dw.WithdrawTransition) -> wire dicts.
    `payments` (deposit / withdraw): the L1 `ContractDeposit` / `ContractWithdraw` of each transaction, in order (the builders
    only carry what the circuits consume)."""
    out = []
    for k, t in enumerate(trans):
        if kind == "update":
            tx = t.tx
            out.append({
                "enabled": t.enabled,
                "tx": {"nonce": tx.nonce, "src_pub_key": tuple(tx.src_pub_key), "dst_pub_key": tuple(tx.dst_pub_key), "amount": _money_w(tx.amount),
                       "fee": _money_w(tx.fee), "sig": {"r": tuple(tx.sig["r"]), "s": tx.sig["s"]}},
                "src_before": _account_w(t.src_before), "src_before_balances_hash": t.src_before_balances_hash,
                "src_before_balance": _money_w(t.src_before_balance), "src_before_fee_balance": _money_w(t.src_before_fee_balance),
                "src_proof": t.src_proof, "src_index": t.src_index, "src_token_index": t.src_token_index, "src_balance_proof": t.src_balance_proof,
                "src_fee_token_index": t.src_fee_token_index, "src_fee_balance_proof": t.src_fee_balance_proof,
                "dst_before": _account_w(t.dst_before), "dst_before_balances_hash": t.dst_before_balances_hash,
                "dst_before_balance": _money_w(t.dst_before_balance), "dst_proof": t.dst_proof, "dst_index": t.dst_index,
                "dst_token_index": t.dst_token_index, "dst_balance_proof": t.dst_balance_proof})
        elif kind == "deposit":
            out.append({
                "enabled": t.enabled, "tx": {"mpn_address": tuple(t.tx.mpn_address), "payment": payments[k]},
                "before": _account_w(t.before), "before_balances_hash": t.before_balances_hash, "before_balance": _money_w(t.before_balance),
                "proof": t.proof, "account_index": t.account_index, "token_index": t.token_index, "balance_proof": t.balance_proof})
        else:
            out.append({
                "enabled": t.enabled,
                "tx": {"mpn_address": tuple(t.tx.mpn_address), "mpn_withdraw_nonce": t.tx.mpn_withdraw_nonce,
                       "mpn_sig": {"r": tuple(t.tx.mpn_sig["r"]), "s": t.tx.mpn_sig["s"]}, "payment": payments[k]},
                "before": _account_w(t.before), "before_token_balance": _money_w(t.before_token_balance),
                "before_fee_balance": _money_w(t.before_fee_balance), "proof": t.proof, "account_index": t.account_index,
                "token_index": t.token_index, "token_balance_proof": t.token_balance_proof, "before_token_hash": t.before_token_hash,
                "fee_token_index": t.fee_token_index, "fee_balance_proof": t.fee_balance_proof})
    return out


def _root_from_proof(index, leaf, proof):
    """`calc_root_poseidon4` outside the circuit (/root/reference/src/zk/groth16/gadgets/merkle/mod.rs:53-65)"""
    cur = leaf
    for sib in proof:
        vals = list(sib)
        vals.insert(index & 3, cur)
        cur = N.poseidon(vals)
        index >>= 2
    return cur


def _entering_root(acc, balances_hash, index, proof):
    """the state root a transition was built against — the builders' `pre_root` bookkeeping (the GPU witness path feeds it
    to every slot), which does not travel: recomputed from the transition's own account, proof and index"""
    return _root_from_proof(index, N.poseidon([acc.tx_nonce, acc.withdraw_nonce, acc.address[0], acc.address[1], balances_hash]), proof)


def wire_to_transitions(kind, items):
    """wire dicts -> the builder dataclasses the circuits are synthesised from"""
    out = []
    for t in items:
        if kind == "update":
            x = t["tx"]
            tx = U.MpnTransaction(x["nonce"], tuple(x["src_pub_key"]), tuple(x["dst_pub_key"]), _money_b(x["amount"]), _money_b(x["fee"]),
                                  {"r": tuple(x["sig"]["r"]), "s": x["sig"]["s"]})
            out.append(U.UpdateTransition(
                t["enabled"], tx, _account_b(t["src_before"]), t["src_before_balances_hash"], _money_b(t["src_before_balance"]),
                _money_b(t["src_before_fee_balance"]), t["src_proof"], t["src_index"], t["src_token_index"], t["src_balance_proof"],
                t["src_fee_token_index"], t["src_fee_balance_proof"], _account_b(t["dst_before"]), t["dst_before_balances_hash"],
                _money_b(t["dst_before_balance"]), t["dst_proof"], t["dst_index"], t["dst_token_index"], t["dst_balance_proof"]))
            if t["enabled"]:
                out[-1].pre_root = _entering_root(out[-1].src_before, t["src_before_balances_hash"], t["src_index"], t["src_proof"])
        elif kind == "deposit":
            p = t["tx"]["payment"]
            tx = D.MpnDeposit(tuple(t["tx"]["mpn_address"]), Wr.contract_id_scalar(p["amount"]["token_id"]), p["amount"]["amount"])
            out.append(D.DepositTransition(t["enabled"], tx, _account_b(t["before"]), t["before_balances_hash"], _money_b(t["before_balance"]),
                                           t["proof"], t["account_index"], t["token_index"], t["balance_proof"]))
            if t["enabled"]:
                out[-1].pre_root = _entering_root(out[-1].before, t["before_balances_hash"], t["account_index"], t["proof"])
        else:
            x, p = t["tx"], t["tx"]["payment"]
            tx = D.MpnWithdraw(tuple(x["mpn_address"]), x["mpn_withdraw_nonce"], {"r": tuple(x["mpn_sig"]["r"]), "s": x["mpn_sig"]["s"]},
                               _money_b(p["amount"]), _money_b(p["fee"]), withdraw_fingerprint(p))
            out.append(D.WithdrawTransition(t["enabled"], tx, _account_b(t["before"]), _money_b(t["before_token_balance"]),
                                            _money_b(t["before_fee_balance"]), t["proof"], t["account_index"], t["token_index"],
                                            t["token_balance_proof"], t["before_token_hash"], t["fee_token_index"], t["fee_balance_proof"]))
            if t["enabled"]:
                out[-1].pre_root = _entering_root(out[-1].before, t["before_token_hash"], t["account_index"], t["proof"])
    return out


# ------------------------------------------------------------------ prepare_works
def prepare_works(config, state, deposits, withdraws, updates, rewards, height=0, deposit_payments=None, withdraw_payments=None,
                  builders=None):
    """-> (works: {id: wire work dict}, fork: the ledger after all batches).  `state` is not modified (`fork_on_ram`);
    `rewards` = {"deposit": u64, "withdraw": u64, "update": u64}; `builders` = (deposit_fn, withdraw_fn, update_fn) with the
    signatures of dw.deposit / dw.withdraw / update.update (default) — pass the batched GPU builders of batch_update.py to
    hash on the GPU.  deposit_payments / withdraw_payments: {id(tx) or index -> L1 payment dict} for the wire images."""
    dep_fn, wd_fn, up_fn = builders or (D.deposit, D.withdraw, U.update)
    fork = state.fork()
    works = []
    # what the builders check of the L1 payments (deposit.rs:33,68-83 `rejected_pub_keys`; withdraw.rs:77 `verify_calldata`):
    # entries that come with a payment and do not carry the field yet get it from the payment
    for k, d in enumerate(deposits):
        if d.src is None and k in (deposit_payments or {}):
            d.src = bytes(deposit_payments[k]["src"])
    for k, w in enumerate(withdraws):
        if w.calldata is None and k in (withdraw_payments or {}):
            w.calldata = withdraw_payments[k]["calldata"]

    def payments_of(trans, source, table, default):
        out = []
        for t in trans:
            key = next((i for i, s in enumerate(source) if s is t.tx), None)
            out.append((table or {}).get(key, default(t.tx)))
        return out

    def default_deposit(tx):
        return {"memo": "", "contract_id": None, "deposit_circuit_id": 0, "calldata": 0, "src": bytes(32),
                "amount": {"token_id": Wr.scalar_contract_id(tx.token_id), "amount": tx.amount}, "fee": {"token_id": "ziesha", "amount": 0},
                "nonce": 0, "sig": None}

    def default_withdraw(tx):
        return {"memo": "", "contract_id": None, "withdraw_circuit_id": 0, "calldata": 0, "dst": bytes(32), "amount": _money_w(tx.amount),
                "fee": _money_w(tx.fee)}

    def push(kind, pub, trans, payments=None):
        works.append({"config": config,
                      "public_inputs": {"height": height, "state": pub["state"], "aux_data": pub["aux_data"], "next_state": pub["next_state"]},
                      "data": (kind, transitions_to_wire(kind, trans, payments)),
                      "new_root": {"state_hash": fork.root, "state_size": fork.state_size}, "reward": rewards[kind]})

    for _ in range(config["mpn_num_deposit_batches"]):
        pub, trans = dep_fn(fork, deposits, config["log4_deposit_batch_size"])
        push("deposit", pub, trans, payments_of(trans, deposits, deposit_payments, default_deposit))
    for _ in range(config["mpn_num_withdraw_batches"]):
        pub, trans = wd_fn(fork, withdraws, config["log4_withdraw_batch_size"])
        push("withdraw", pub, trans, payments_of(trans, withdraws, withdraw_payments, default_withdraw))
    for _ in range(config["mpn_num_update_batches"]):
        pub, trans, _ = up_fn(fork, updates, config["log4_update_batch_size"])
        push("update", pub, trans)
    return dict(enumerate(works)), fork


def final_delta(before, after):
    """`MpnWorkPool.final_delta` (/root/reference/src/mpn/mod.rs:17-45,416-417): the scalar leaves the block's batches changed,
    as `ZkDeltaPairs` = {locator: Some(value) | None}; a locator is [account, field] for the four account scalars and
    [account, 4, token slot, 0 | 1] for a token's id / balance (`set_mpn_account`, src/zk/state/mod.rs:140-208); a leaf that
    became zero is a `Remove` (None).  `before` / `after`: the ledger and the fork `prepare_works` returned."""
    def leaves(acc):
        out = {}
        if acc is None:
            return out
        for f, v in enumerate((acc.tx_nonce, acc.withdraw_nonce, acc.address[0], acc.address[1])):
            out[(f,)] = v
        for slot, m in acc.tokens.items():
            out[(4, slot, 0)] = m.token_id
            out[(4, slot, 1)] = m.amount
        return out

    delta = {}
    for idx in sorted(set(before.accounts) | set(after.accounts)):
        old, new = leaves(before.accounts.get(idx)), leaves(after.accounts.get(idx))
        for loc in sorted(set(old) | set(new)):
            o, n = old.get(loc, 0), new.get(loc, 0)
            if o != n:
                delta[(idx,) + loc] = n if n != 0 else None
    return delta


def enc_delta(w, delta):
    """bincode of `ZkDeltaPairs(HashMap<ZkDataLocator(Vec<u64>), Option<ZkScalar>>)`"""
    w.u64(len(delta))
    for loc, v in delta.items():
        w.vec(list(loc), lambda w_, x: w_.u64(x))
        w.option(v, lambda w_, x: w_.fr(x))


def work_public_inputs(work, prover_address):
    """the five Groth16 inputs of `check_proof` for this work and prover (/root/reference/src/mpn/mod.rs:281-295)"""
    p = work["public_inputs"]
    return [Wr.commitment(prover_address, work["reward"]), p["height"], p["state"], p["aux_data"], p["next_state"]]


def work_vk(work):
    kind = work["data"][0]
    return work["config"][kind + "_vk"]


def verify_work(work, prover_address, proof387):
    """`MpnWork::verify`"""
    from .. import groth16 as BG
    from .cs import to_mont
    return BG.verify_bytes(work_vk(work), to_mont(work_public_inputs(work, prover_address)), proof387)


# ------------------------------------------------------------------ the external prover
class MpnProver:
    """one proving context per circuit kind and shape; `prove(work, prover_address)` -> 387-byte Groth16Proof image.
    The keys must be the ones whose verifying keys sit in the node's config (production: the ceremony's; tests: setup_gpu)."""

    def __init__(self, ctx):
        self.ctx, self.kinds = ctx, {}

    def add_circuit(self, kind, prover, pk, witness):
        """prover: groth16.Prover of the circuit's R1CS; pk: its ProvingKey; witness: gpu_witness.UpdateWitnessGpu /
        dw_witness.TwoPhaseWitnessGpu for the shape"""
        self.kinds[kind] = (prover, pk, witness)

    def circuit_of(self, work, prover_address):
        c, (kind, items) = work["config"], work["data"]
        A, T = c["log4_tree_size"], c["log4_token_tree_size"]
        B = c["log4_%s_batch_size" % kind]
        trans = wire_to_transitions(kind, items)
        p = work["public_inputs"]
        common = dict(commitment=Wr.commitment(prover_address, work["reward"]), height=p["height"], state=p["state"], aux_data=p["aux_data"],
                      next_state=p["next_state"], transitions=trans)
        if kind == "update":
            return U.UpdateCircuit(A, T, B, fee_token=ZIESHA, **common)
        return (D.DepositCircuit if kind == "deposit" else D.WithdrawCircuit)(A, T, B, **common)

    def prove(self, work, prover_address, r, s, check_satisfied=True):
        kind = work["data"][0]
        prover, pk, witness = self.kinds[kind]
        d_in, d_aux = witness.witness(self.circuit_of(work, prover_address))
        blob, _ = prover.prove_dev(pk, d_in, d_aux, r, s, check_satisfied=check_satisfied)
        return bytes(blob)


def work_info_dtype():
    """numpy image of `bzk_mpn_work_info` (include/bzk.h); tests/test_abi.py checks it against the C compiler's layout"""
    import numpy as np
    return np.dtype([("kind", "<u4"), ("log4_tree", "<u4"), ("log4_token", "<u4"), ("log4_batch", "<u4"), ("n_transitions", "<u8"), ("height", "<u8"),
                     ("state", "<u8", 4), ("aux_data", "<u8", 4), ("next_state", "<u8", 4), ("new_root_hash", "<u8", 4), ("new_root_size", "<u8"),
                     ("reward", "<u8")])


class NativeMpnProver:
    """the same job with nothing but libbzk between the wire and the proof: `prove(work_bytes, prover_address, r, s)` ->
    391-byte `ZkProof::Groth16` image through bzk_mpn_prover_prove_work (csrc/mpn_prover.cu: bincode decode, rows, GPU witness,
    resident proof).  One circuit per kind, compiled by the C++ definition (mpn/native_circuit.py); `pk` = groth16.ProvingKey of
    that circuit's R1CS (the Python and the C++ definitions emit the same arrays, so a key made for either fits)."""

    def __init__(self, ctx, fee_token=ZIESHA):
        self.ctx, self.fee_token, self._p = ctx, fee_token, {}

    def add_circuit(self, kind, native_circuit, pk):
        import ctypes as ct
        import os
        import numpy as np
        from .. import _lib
        canon = lambda v: np.frombuffer((v % N.R).to_bytes(32, "little"), dtype=np.uint64).copy()
        jj_d, fee = canon(N.JJ_D), canon(self.fee_token)
        h = ct.c_void_p()
        self.ctx._check(self.ctx._l.bzk_mpn_prover_create(self.ctx._h, native_circuit._h, pk._h, ct.c_void_p(jj_d.ctypes.data),
                                                          ct.c_void_p(fee.ctypes.data), ct.byref(h)))
        self._p[kind] = (h, pk)          # the key must outlive the prover

    def prove(self, work_bytes, prover_address, r, s, check_satisfied=True):
        import ctypes as ct
        import numpy as np
        kind = Wr._KINDS[self._kind_of(work_bytes)]
        r, s = (np.ascontiguousarray(x, dtype=np.uint64) for x in (r, s))
        out = ct.create_string_buffer(391)
        self.ctx._check(self.ctx._l.bzk_mpn_prover_prove_work(self.ctx._h, self._p[kind][0], bytes(work_bytes), len(work_bytes), bytes(prover_address),
                                                              ct.c_void_p(r.ctypes.data), ct.c_void_p(s.ctypes.data), 1 if check_satisfied else 0, out))
        return out.raw

    def _kind_of(self, work_bytes):
        import ctypes as ct
        import numpy as np
        h = ct.c_void_p()
        self.ctx._check(self.ctx._l.bzk_mpn_work_decode(bytes(work_bytes), len(work_bytes), ct.byref(h), None))
        info = np.zeros(1, dtype=work_info_dtype())
        self.ctx._l.bzk_mpn_work_get_info(h, ct.c_void_p(info.ctypes.data))
        self.ctx._l.bzk_mpn_work_free(h)
        return int(info[0]["kind"])

    def free(self):
        for h, _ in self._p.values():
            self.ctx._l.bzk_mpn_prover_free(self.ctx._h, h)
        self._p = {}


class NativeMpnWorker:
    """the whole worker in libbzk (csrc/mpn_worker.cu): `prove_response(response_bytes, address, seed=None)` ->
    (PostMpnSolutionRequest bytes, one status per work of the response).  ctxs: the contexts to prove on (several may share a
    GPU); keys_per_ctx[i]: {"deposit" | "withdraw" | "update": proving key} served on ctxs[i] (a key object with `_h`, or a raw
    handle) — the update key over the blocked R1CS, deposit and withdraw explicit, each checked at creation against the verifying
    keys in `config_bytes` (bincode of the node's MpnConfig).  The keys must outlive the worker.  seed (32 bytes) makes the
    blinding reproducible and is for tests only: without it every proof draws r and s from the OS."""

    KINDS = ("deposit", "withdraw", "update")

    def __init__(self, ctxs, config_bytes, keys_per_ctx, fee_token=ZIESHA):
        import ctypes as ct
        import numpy as np
        from .. import _lib
        assert len(ctxs) == len(keys_per_ctx) and ctxs
        self._l, self._ctxs, self._keys = ctxs[0]._l, list(ctxs), [dict(k) for k in keys_per_ctx]
        handle = lambda k: None if k is None else (k._h if hasattr(k, "_h") else k)

        class Dev(ct.Structure):
            _fields_ = [("ctx", ct.c_void_p), ("params", ct.c_void_p * 3)]
        devs = (Dev * len(ctxs))()
        for i, (c, keys) in enumerate(zip(ctxs, self._keys)):
            devs[i].ctx = c._h.value if isinstance(c._h, ct.c_void_p) else c._h
            for k, name in enumerate(self.KINDS):
                h = handle(keys.get(name))
                devs[i].params[k] = h.value if isinstance(h, ct.c_void_p) else h
        canon = lambda v: np.frombuffer((v % N.R).to_bytes(32, "little"), dtype=np.uint64)
        jj = np.ascontiguousarray(np.stack([canon(N.JJ_D), canon(N.JJ_BASE_COFACTOR[0]), canon(N.JJ_BASE_COFACTOR[1])]))
        fee = np.ascontiguousarray(canon(fee_token))
        blob = open(_lib.PARAMS_PATH, "rb").read()
        cfg = bytes(config_bytes)
        h = ct.c_void_p()
        st = self._l.bzk_mpn_worker_create(cfg, len(cfg), ct.byref(devs), len(ctxs), blob, len(blob), ct.c_void_p(jj.ctypes.data),
                                           ct.c_void_p(fee.ctypes.data), ct.byref(h))
        if st != 0:
            raise _lib.BzkError(st, "bzk_mpn_worker_create")
        self._h = h

    def prove_response(self, response_bytes, address, seed=None):
        import ctypes as ct
        import numpy as np
        from .. import _lib
        resp = bytes(response_bytes)
        cap = int.from_bytes(resp[:8], "little") if len(resp) >= 8 else 0
        status = np.zeros(max(min(cap, 1 << 16), 1), dtype=np.int32)
        buf, ln, n = ct.c_void_p(), ct.c_size_t(), ct.c_uint64()
        st = self._l.bzk_mpn_worker_prove_response(self._h, resp, len(resp), bytes(address), None if seed is None else bytes(seed), ct.byref(buf),
                                                   ct.byref(ln), ct.c_void_p(status.ctypes.data), len(status), ct.byref(n))
        if st != 0:
            raise _lib.BzkError(st, "bzk_mpn_worker_prove_response")
        out = ct.string_at(buf, ln.value)
        self._l.bzk_buffer_free(buf)
        return out, [int(x) for x in status[:n.value]]

    def last_timing(self):
        """{call, rows_witness, prove, self_check} in milliseconds (host clock) of the last prove_response"""
        import numpy as np
        ms = np.zeros(4, dtype=np.float64)
        self._l.bzk_mpn_worker_last_timing(self._h, ms.ctypes.data)
        return dict(zip(("call", "rows_witness", "prove", "self_check"), (float(x) for x in ms)))

    def free(self):
        if self._h:
            self._l.bzk_mpn_worker_free(self._h)
            self._h = None


class WorkerClient:
    """the loop of an MPN worker against a node's HTTP API"""

    def __init__(self, peer, address, prover: MpnProver, headers=None, opener=None):
        self.peer, self.address, self.prover = peer, bytes(address), prover
        self.headers = headers or (lambda method, url, body: {})
        self._open = opener or self._urlopen

    def _urlopen(self, method, url, body):
        req = urllib.request.Request(url, data=body, method=method, headers={"content-type": "application/octet-stream", **self.headers(method, url, body)})
        with urllib.request.urlopen(req, timeout=60) as resp:
            return resp.read()

    def register(self):
        return Wr.post_mpn_worker_response_from_bytes(self._open("POST", f"http://{self.peer}/bincode/mpn/worker", Wr.post_mpn_worker_request(self.address)))

    def get_works(self):
        return Wr.get_mpn_work_response_from_bytes(self._open("GET", f"http://{self.peer}/bincode/mpn/work", Wr.get_mpn_work_request(self.address)))

    def post_proofs(self, proofs):
        return Wr.post_mpn_solution_response_from_bytes(
            self._open("POST", f"http://{self.peer}/bincode/mpn/solution", Wr.post_mpn_solution_request(self.address, proofs)))

    def run_once(self, randomness):
        """fetch the works assigned to this address, prove each, post the proofs; -> (n_works, n_accepted).  With a
        NativeMpnWorker the response goes through one call and the worker draws its own blinding (`randomness` is unused)."""
        if isinstance(self.prover, NativeMpnWorker):
            resp = self._open("GET", f"http://{self.peer}/bincode/mpn/work", Wr.get_mpn_work_request(self.address))
            body, status = self.prover.prove_response(resp, self.address)
            n_ok = sum(1 for x in status if x == 0)
            return len(status), (Wr.post_mpn_solution_response_from_bytes(self._open("POST", f"http://{self.peer}/bincode/mpn/solution", body))
                                 if n_ok else 0)
        works = self.get_works()
        proofs = {}
        for wid, work in works.items():
            r, s = randomness()
            if isinstance(self.prover, NativeMpnProver):      # bincode in, 391 bytes out (a decoded work re-encodes to its bytes)
                proofs[wid] = self.prover.prove(Wr.work_to_bytes(work), self.address, r, s)[4:]
            else:
                proofs[wid] = self.prover.prove(work, self.address, r, s)
        return len(works), (self.post_proofs(proofs) if proofs else 0)
