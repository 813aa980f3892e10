"""The MPN worker (csrc/mpn_worker.cu) from GetMpnWorkResponse bytes to PostMpnSolutionRequest bytes.

    python tools/bench_mpn_worker.py [--reps 3] [--config3] [--out result.json]

production: a block's works — deposit 4^3, withdraw 4^3, update 4^4 at A=15, T=3 — built by bzk_mpn_prepare_works, proved by a
worker on one context and by a worker on two contexts of the same GPU (alternating, after one warm-up call each); per call the
host wall clock of the synchronous call, and the worker's split into rows + witness, the rest of each proof (both summed over
works) and the self-check.  --config3: BASELINE configs[3] (A=16, T=3, B=5, 1024 transfers, 2^26) on one context, with the
device's free memory before and after.  Keys from setup_gpu with table_levels (default 1: no fixed-base tables).  The card's
name, power limit and SM clock are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def _ms(w):
    return {k: round(v, 1) for k, v in w.last_timing().items()}


def production(ctx, reps, table_levels):
    import bazuka_b200 as Bz
    import mpn_worker_cases as C
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn import works as Wk
    from bazuka_b200.mpn.native_circuit import NativeTwoPhaseCircuit, NativeUpdateCircuit
    from oracle import cref
    A, T, BD, BW, BU = 15, 3, 3, 3, 4
    keys, vks = {}, {}
    nc = NativeUpdateCircuit(A, T, BU, blocked=True)
    br = nc.blocked_r1cs()
    nc.free()
    g1, g2 = cref.g1_generator(), cref.g2_generator()
    keys["update"], vks["update"] = BG.setup_gpu(ctx, br, cref.fr_random(601, 5), g1, g2, table_levels=table_levels)
    del br
    for i, (kind, b) in enumerate((("deposit", BD), ("withdraw", BW))):
        c = NativeTwoPhaseCircuit(kind, A, T, b)
        ni, na, mats = c.r1cs()
        c.free()
        keys[kind], vks[kind] = BG.setup_gpu(ctx, BG.R1CS(ni, na, *mats), cref.fr_random(602 + i, 5), g1, g2, table_levels=table_levels)
    cfg = C.config(A, T, BD, BW, BU, {k: bytes(BG.vk_to_bincode(v)) for k, v in vks.items()})
    st, deps, wds, ups, dpay, wpay = C.block(A, T)
    led = C.ledger(ctx, st, A, T)
    resp, n = C.prepare_response(ctx, led, cfg, deps, wds, ups, dpay, wpay)
    led.free()
    ctx2 = Bz.Context(0)
    workers = {"one_context": Wk.NativeMpnWorker([ctx], C.config_bytes(cfg), [keys]),
               "two_contexts": Wk.NativeMpnWorker([ctx, ctx2], C.config_bytes(cfg), [keys, keys])}
    me = bytes(range(32))
    res = {name: {"wall_s": [], "split_ms": []} for name in workers}
    for w in workers.values():
        _, status = w.prove_response(resp, me)
        assert status == [0] * n, status
    for _ in range(reps):
        for name, w in workers.items():
            t0 = time.perf_counter()
            _, status = w.prove_response(resp, me)      # synchronous: returns after the last proof is back on the host
            res[name]["wall_s"].append(round(time.perf_counter() - t0, 3))
            res[name]["split_ms"].append(_ms(w))
            assert status == [0] * n, status
    for name, r in res.items():
        r["mean_s"] = round(sum(r["wall_s"]) / len(r["wall_s"]), 3)
    for w in workers.values():
        w.free()
    ctx2.close()
    for k in keys.values():
        k.free()
    return res


def config3(ctx, reps):
    import torch
    import mpn_worker_cases as C
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn import native as N, update as U, works as Wk
    from bazuka_b200.mpn.ledger import NativeLedger
    from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit
    from oracle import cref
    A, T, B, nacc = 16, 3, 5, 128
    gb = lambda: round(torch.cuda.mem_get_info()[0] / 1e9, 1)
    free = {"start": gb()}
    nc = NativeUpdateCircuit(A, T, B, blocked=True)
    br = nc.blocked_r1cs()
    nc.free()
    t0 = time.perf_counter()
    pk, vk = BG.setup_gpu(ctx, br, cref.fr_random(911, 5), cref.g1_generator(), cref.g2_generator(), table_levels=1)
    del br
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    setup_s = time.perf_counter() - t0
    free["after_setup"] = gb()
    cfg = dict(C.config(A, T, 1, 1, B, {"deposit": C.opaque_vk(2), "withdraw": C.opaque_vk(4), "update": bytes(BG.vk_to_bincode(vk))}),
               mpn_num_deposit_batches=0, mpn_num_withdraw_batches=0)
    led = NativeLedger(ctx, A, T)
    keys = []
    for i in range(nacc):
        pkey, sk = N.eddsa_keys(b"acct%d" % i)
        keys.append((pkey, sk))
        led.set_account(i, U.MpnAccount(0, 0, pkey, {0: U.Money(U.ZIESHA, 10 ** 12)}))
    nonces, txs = [0] * nacc, []
    for k in range(1 << (2 * B)):
        s, d = k % nacc, (k + 1) % nacc
        nonces[s] += 1
        tx = U.MpnTransaction(nonces[s], N.jj_compress(keys[s][0]), N.jj_compress(keys[d][0]), U.Money(U.ZIESHA, 1000 + k), U.Money(U.ZIESHA, 10))
        tx.sign(keys[s][1])
        txs.append(tx)
    resp, _ = C.prepare_response(ctx, led, cfg, [], [], txs, {}, {})
    led.free()
    w = Wk.NativeMpnWorker([ctx], C.config_bytes(cfg), [{"update": pk}])
    free["after_worker_create"] = gb()
    walls, splits = [], []
    for i in range(reps + 1):
        t0 = time.perf_counter()
        _, status = w.prove_response(resp, bytes(range(32)))
        if i:
            walls.append(round(time.perf_counter() - t0, 3))
            splits.append(_ms(w))
        assert status == [0], status
    free["after_proofs"] = gb()
    w.free()
    pk.free()
    return {"setup_s": round(setup_s, 1), "wall_s": walls, "mean_s": round(sum(walls) / len(walls), 3), "split_ms": splits, "free_gb": free}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--table-levels", type=int, default=1)
    ap.add_argument("--config3", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    import bazuka_b200 as Bz
    ctx = Bz.Context(0)
    out = {"gpu": _gpu_info(), "table_levels": a.table_levels, "production": production(ctx, a.reps, a.table_levels)}
    if a.config3:
        out["config3"] = config3(ctx, max(1, a.reps - 1))
    out["gpu_after"] = _gpu_info()
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
