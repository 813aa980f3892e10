"""CPU tier: bzk_mpn_state_apply_delta (csrc/mpn_host.cu, compiled unmodified into tests/hostshim/_mpn_shim.so with the plan
steps run by its host compile: hash_plan.cuh's operand rule over the host Poseidon) against the leaf-by-leaf restatement of `update_contract` /
`index_mpn_accounts` in tests/mpn_delta_cases.py, on the blocks `bzk_mpn_prepare_works` builds, random deltas, every refusal
and snapshots.  tests/test_gpu_mpn_apply_delta.py repeats these over the real kernel."""
import pytest

import mpn_delta_cases as C
from bazuka_b200.mpn import dw as D, native as N, update as U, works as Wk
from test_mpn_cpu import make_state, transfer
from test_wire_cpu import _config, _scenario


def block_scenario():
    """the wire tests' block: the depositor's new account spending in the same block, a deposit refused through its L1 source
    (the next from that source goes with it), a withdrawal with the wrong calldata -> (state, keys, config args)"""
    st, keys, deposits, withdraws, wpay, updates = _scenario()
    deposits = deposits + [D.MpnDeposit((6, False), 77, 1), D.MpnDeposit(N.jj_compress(keys[1][0]), 77, 3)]
    srcs = [bytes([1]) * 32, bytes([2]) * 32, bytes([3]) * 32, bytes([3]) * 32]
    from bazuka_b200.mpn import wire as Wr
    dpay = {k: {"memo": "d%d" % k, "contract_id": 0x1234, "deposit_circuit_id": 0, "calldata": 0, "src": srcs[k],
                "amount": {"token_id": Wr.scalar_contract_id(d.token_id), "amount": d.amount}, "fee": {"token_id": "ziesha", "amount": 0}, "nonce": k + 1,
                "sig": bytes([9]) * 64 if k == 1 else None} for k, d in enumerate(deposits)}
    w2 = D.MpnWithdraw(N.jj_compress(keys[2][0]), 1, amount=U.Money(U.ZIESHA, 7), fee=U.Money(U.ZIESHA, 1))
    pay2 = {"memo": "", "contract_id": None, "withdraw_circuit_id": 0, "calldata": 0, "dst": bytes(32), "amount": {"token_id": "ziesha", "amount": 7},
            "fee": {"token_id": "ziesha", "amount": 1}}
    w2.fingerprint = Wk.withdraw_fingerprint(pay2)
    w2.sign(keys[2][1])
    pay2["calldata"] = w2.expected_calldata() + 1
    return st, keys, (_config(), deposits, withdraws + [w2], updates, dpay, {**wpay, 1: pay2})


def run_block_cases(ctx):
    st, keys, block = block_scenario()
    led = C.load(ctx, st, 3, 3)
    # the next block: the newcomer (index 3, known only through the applied delta's index) and account 0 spend again
    nxt = (_config(num=(0, 0, 1)), [], [], [transfer(keys, 3, 1, 2, amount=5, fee=1), transfer(keys, 0, 3, 2, amount=9)])
    info = C.check_block_round_trip(ctx, led, *block, next_block=nxt)
    assert info["account_count"] == 4
    # the dict form of the same delta (works.final_delta of the Python restatement) gives the same ledger
    _, fork_py = Wk.prepare_works(block[0], st, *block[1:4], {"deposit": 11, "withdraw": 22, "update": 33}, height=9, deposit_payments=block[4],
                                  withdraw_payments=block[5])
    c = led.fork()
    c.apply_delta(Wk.final_delta(st, fork_py))
    assert (c.info()["state_hash"], c.info()["state_size"]) == (fork_py.root, fork_py.state_size) == (info["state_hash"], info["state_size"])
    c.free()
    led.free()
    # two consecutive update batches in one block
    st2, keys2 = make_state(3, 3, 3)
    ups = [transfer(keys2, 0, 1, 1), transfer(keys2, 1, 2, 1), transfer(keys2, 2, 0, 1), transfer(keys2, 0, 2, 2), transfer(keys2, 1, 0, 2),
           transfer(keys2, 2, 1, 2)]
    led2 = C.load(ctx, st2, 3, 3)
    C.check_block_round_trip(ctx, led2, _config(num=(0, 0, 2)), [], [], ups,
                             next_block=(_config(num=(0, 0, 1)), [], [], [transfer(keys2, 0, 1, 3), transfer(keys2, 2, 0, 3)]))
    led2.free()


def test_block_deltas_round_trip_to_the_committed_fork(hostmpn):
    run_block_cases(hostmpn)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_deltas_against_the_leaf_by_leaf_oracle(hostmpn, seed):
    C.check_random_deltas(hostmpn, seed, rounds=6)


def test_every_refusal_leaves_the_ledger_unchanged(hostmpn):
    st, _ = make_state(3, 2, 3)
    led = C.load(hostmpn, st, 3, 2)
    C.check_refusals(hostmpn, led)
    led.free()


def test_snapshot_rebuilds_a_ledger_built_with_set_account(hostmpn):
    C.check_snapshot(hostmpn, 300)


def test_empty_delta_and_the_oracle_itself(hostmpn):
    """an empty delta is a no-op that still checks the expectation; the oracle restates `set_data` (root of MpnState)"""
    st, _ = make_state(3, 2, 2)
    led = C.load(hostmpn, st, 3, 2)
    info = led.info()
    assert led.apply_delta(C.encode([]), expect={"state_hash": info["state_hash"], "state_size": info["state_size"]}) == 0 and led.info() == info
    st_, _, err = C.apply_raw(led, C.encode([]), expect_size=info["state_size"] + 1)
    assert st_ == -1 and "expected" in err
    o = C.oracle_of(st, 3, 2)
    assert (o.root, o.state_size, o.account_count) == (st.root, st.state_size, 2)
    with pytest.raises(C.Inconsistency):
        o.apply([((5, 2), 1), ((5, 3), 1)])
    led.free()
