"""GPU tier: bzk_mpn_state_apply_delta over the real plan-step kernel (csrc/poseidon.cu k_poseidon_plan_step): the CPU tier's
scenarios (tests/test_mpn_apply_delta_cpu.py), a production-shape block, a 2^20-account snapshot applied whole, in 16 parts and
(on a 2^12 sample) against set_account, and a tampered delta refused by the root check."""
import random

import pytest

import mpn_delta_cases as C
from bazuka_b200.mpn import dw as D, native as N, update as U, works as Wk
from bazuka_b200.mpn.ledger import NativeLedger
from test_mpn_apply_delta_cpu import run_block_cases
from test_mpn_cpu import make_state, transfer
from test_wire_cpu import _vk_blob

pytestmark = pytest.mark.gpu


def test_gpu_block_deltas_round_trip_to_the_committed_fork(ctx):
    run_block_cases(ctx)


def test_gpu_random_deltas_against_the_leaf_by_leaf_oracle(ctx):
    C.check_random_deltas(ctx, 5, rounds=6)


def test_gpu_every_refusal_leaves_the_ledger_unchanged(ctx):
    st, _ = make_state(3, 2, 3)
    led = C.load(ctx, st, 3, 2)
    C.check_refusals(ctx, led)
    led.free()


def test_gpu_snapshot_rebuilds_a_ledger_built_with_set_account(ctx):
    C.check_snapshot(ctx, 300)


def production_block(n_acc=128):
    """A=15, T=3: 256 transfers, 64 deposits (64 new accounts), 64 withdrawals, one batch of each kind
    -> (state, config, deposits, withdraws, updates, deposit payments, withdraw payments)"""
    st, keys = make_state(15, 3, n_acc)
    config = {"log4_tree_size": 15, "log4_token_tree_size": 3, "log4_deposit_batch_size": 3, "log4_withdraw_batch_size": 3, "log4_update_batch_size": 4,
              "mpn_contract_id": 0x1234, "mpn_num_update_batches": 1, "mpn_num_deposit_batches": 1, "mpn_num_withdraw_batches": 1,
              "deposit_vk": _vk_blob(fill=1), "withdraw_vk": _vk_blob(fill=3), "update_vk": _vk_blob(fill=5)}
    newcomers = [N.eddsa_keys(b"prod-new%d" % k)[0] for k in range(64)]
    deposits = [D.MpnDeposit(N.jj_compress(pk), U.ZIESHA, 1000 + k) for k, pk in enumerate(newcomers)]
    dpay = {k: {"memo": "", "contract_id": 0x1234, "deposit_circuit_id": 0, "calldata": 0, "src": bytes([k + 1]) * 32,
                "amount": {"token_id": "ziesha", "amount": d.amount}, "fee": {"token_id": "ziesha", "amount": 0}, "nonce": 1, "sig": None}
            for k, d in enumerate(deposits)}
    withdraws, wpay = [], {}
    for k in range(64):
        w = D.MpnWithdraw(N.jj_compress(keys[k][0]), 1, amount=U.Money(U.ZIESHA, 50), fee=U.Money(U.ZIESHA, 1))
        pay = {"memo": "", "contract_id": 0x1234, "withdraw_circuit_id": 0, "calldata": 0, "dst": bytes([k]) * 32,
               "amount": {"token_id": "ziesha", "amount": 50}, "fee": {"token_id": "ziesha", "amount": 1}}
        w.fingerprint = Wk.withdraw_fingerprint(pay)
        w.sign(keys[k][1])
        pay["calldata"] = w.expected_calldata()
        withdraws.append(w)
        wpay[k] = pay
    updates = [transfer(keys, k % n_acc, (k * 5 + 1) % n_acc, 1 + k // n_acc, amount=10, fee=1) for k in range(256)]
    return st, keys, (config, deposits, withdraws, updates, dpay, wpay)


def test_gpu_production_block_with_the_root_check_and_a_tampered_delta(ctx):
    st, keys, block = production_block()
    led = C.load(ctx, st, 15, 3)
    _, fork, n = C.run_block(ctx, led, *block)
    assert n == 3
    image, entries = C.delta_bytes(led, fork)
    fork.commit_accounts()
    want = fork.info()
    assert want["account_count"] == 128 + 64 and entries >= 3 * (128 + 64)      # every touched account: a nonce and a balance at least
    applied = led.fork()
    launches = ctx._l.bzk_ctx_launch_count(ctx._h)
    assert applied.apply_delta(image, expect={"state_hash": want["state_hash"], "state_size": want["state_size"]}) == entries
    assert ctx._l.bzk_ctx_launch_count(ctx._h) - launches == 1 + 3 + 1 + 15      # one launch per plan step
    assert applied.info() == want and C.delta_bytes(applied, fork)[1] == 0
    # the next block agrees byte for byte on the applied ledger and on the committed fork
    nxt = (dict(block[0], mpn_num_deposit_batches=0, mpn_num_withdraw_batches=0), [], [],
           [transfer(keys, k, (k + 3) % 128, 3, amount=5) for k in range(0, 128, 2)])
    a, fa, _ = C.run_block(ctx, applied, *nxt)
    b, fb, _ = C.run_block(ctx, fork, *nxt)
    assert a == b and fa.info() == fb.info()
    # one scalar changed: the root check refuses it and the ledger does not move
    entries_ = C.parse(image)
    rng = random.Random(3)
    k = rng.choice([j for j, (loc, v) in enumerate(entries_) if len(loc) == 4 and loc[3] == 1 and v])
    entries_[k] = (entries_[k][0], entries_[k][1] + 1)
    before = led.fork()
    st_, _, err = C.apply_raw(led, C.encode(entries_), want["state_hash"], want["state_size"])
    assert st_ == -1 and "expected" in err and C.same_ledger(led, before)
    for x in (led, fork, applied, fa, fb, before):
        x.free()


def test_gpu_snapshot_of_2_20_accounts_whole_in_parts_and_against_set_account(ctx):
    A, T, n = 15, 3, 1 << 20
    whole = NativeLedger(ctx, A, T)
    image = C.snapshot_image(0, n, T)
    entries = whole.apply_delta(image)
    del image
    info = whole.info()
    assert info["account_count"] == n and entries == info["state_size"] == 9 * n       # 4 scalars + 2.5 tokens of 2 leaves
    parts = NativeLedger(ctx, A, T)
    for p in range(16):
        parts.apply_delta(C.snapshot_image(p * (n // 16), n // 16, T))
    assert parts.info() == info and C.delta_bytes(parts, whole)[1] == 0
    parts.free(); whole.free()
    # a 2^12 sample: the same accounts through set_account, one at a time
    m = 1 << 12
    sample = C.snapshot_mpn_accounts(0, m, T)
    by_set = NativeLedger(ctx, A, T)
    for i, a in sample.items():
        by_set.set_account(i, a)
    by_delta = NativeLedger(ctx, A, T)
    by_delta.apply_delta(C.snapshot_image(0, m, T))
    assert by_delta.info() == by_set.info() and C.delta_bytes(by_delta, by_set)[1] == 0
    by_set.free(); by_delta.free()
