#!/usr/bin/env python3
"""The 1024-transaction update batch of BASELINE configs[3] (A=16, T=3, B=5, 2^26 domain) on one GPU over the blocked R1CS,
and the 256-transaction production batch (A=15, T=3, B=4, 2^24) proved over the explicit and the blocked R1CS in turn.

1024: blocked compile, blocked setup (no fixed-base tables: table_levels=1), native ledger and witness, one warm-up proof,
then --reps timed proofs; the free device memory is read after each stage.  256: one key (the blocked setup), both handles
resident, one warm-up proof each, then --reps rounds that time an explicit and a blocked proof alternately, with the
CUDA-event stage marks of each.  Every timed call ends in a device synchronise.  The GPU's name and power limit are read
in the same run.  One JSON line per batch.

  python tools/bench_mpn_1024.py [--reps 3] [--skip-1024] [--skip-256]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bazuka_b200 as B  # noqa: E402
from bazuka_b200 import groth16 as BG  # noqa: E402
from bazuka_b200.mpn import update as U  # noqa: E402
from bazuka_b200.mpn.gpu_witness import UpdateWitnessGpu  # noqa: E402
from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit  # noqa: E402
from oracle import cref  # noqa: E402
from test_gpu_baseline_configs import _ledger_and_transfers  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or torch.cuda.get_device_name(), "power_limit": limit.strip() or None}


def free_gb():
    return round(torch.cuda.mem_get_info()[0] / 1e9, 2)


def witness(ctx, A, T, B_, prog, epi, nacc):
    wit = UpdateWitnessGpu(ctx, A, T, prog, {B_: epi})
    led, txs = _ledger_and_transfers(ctx, A, T, B_, nacc)
    raws, ext, accepted, pub, n_acc = led.update_build(txs, B_)
    assert accepted.all() and n_acc == 1 << (2 * B_)
    d_in, d_aux = wit.witness_native(raws, ext, [42, 7, pub["state"], U.ZIESHA, pub["aux_data"], pub["next_state"]], B_)
    torch.cuda.synchronize()
    wit.free(); led.free()
    return d_in, d_aux


def timed_prove(ctx, pr, pk, d_in, d_aux, r, s):
    t0 = time.perf_counter()
    blob, _ = pr.prove_dev(pk, d_in, d_aux, r, s, check_satisfied=False)
    ctx.synchronize()
    return time.perf_counter() - t0, blob, pr.stage_ms()


def batch_1024(ctx, reps):
    A, T, B_ = 16, 3, 5
    out = {"batch": "UpdateCircuit A=16 T=3 B=5 (1024 tx)", "r1cs": "blocked", "table_levels": 1, "free_gb": {"start": free_gb()}}
    t0 = time.perf_counter()
    nc = NativeUpdateCircuit(A, T, B_, blocked=True)
    br = nc.blocked_r1cs()
    prog, epi = nc.program(0), nc.program(1)
    nc.free()
    out["compile_s"] = time.perf_counter() - t0
    out.update({"constraints": br.num_constraints, "log_m": br.log_m})
    t0 = time.perf_counter()
    pk, vk = BG.setup_gpu(ctx, br, cref.fr_random(901, 5), cref.g1_generator(), cref.g2_generator(), table_levels=1)
    pr = BG.Prover(ctx, br)
    ctx.synchronize()
    out["setup_s"] = time.perf_counter() - t0
    out["free_gb"]["after_setup"] = free_gb()
    t0 = time.perf_counter()
    d_in, d_aux = witness(ctx, A, T, B_, prog, epi, 128)
    out["ledger_signing_witness_s"] = time.perf_counter() - t0
    out["free_gb"]["after_witness"] = free_gb()
    r, s = cref.fr_random(902, 2)
    ctx.set_timing(True)
    warm, blob, _ = timed_prove(ctx, pr, pk, d_in, d_aux, r, s)
    out["warmup_prove_s"] = warm
    times, stages = [], []
    for _ in range(reps):
        dt, b, st = timed_prove(ctx, pr, pk, d_in, d_aux, r, s)
        assert (b == blob).all()
        times.append(dt)
        stages.append(st)
    ctx.set_timing(False)
    out["free_gb"]["after_proofs"] = free_gb()
    out["prove_s"] = {"mean": float(np.mean(times)), "min": min(times), "max": max(times), "each": times}
    out["stage_ms_last"] = stages[-1]
    out["verify_bytes"] = BG.verify_bytes(BG.vk_to_bincode(vk), d_in.cpu().numpy().view(np.uint64).reshape(-1, 4)[1:], blob)
    pk.free(); pr.free()
    del pk, pr, d_in, d_aux
    torch.cuda.empty_cache()
    return out


def batch_256(ctx, reps):
    A, T, B_ = 15, 3, 4
    out = {"batch": "UpdateCircuit A=15 T=3 B=4 (256 tx)", "table_levels": "default (as many as fit)"}
    nc = NativeUpdateCircuit(A, T, B_, blocked=True)
    br = nc.blocked_r1cs()
    prog, epi = nc.program(0), nc.program(1)
    nc.free()
    ni, na, mats = NativeUpdateCircuit(A, T, B_).r1cs()
    pk, vk = BG.setup_gpu(ctx, br, cref.fr_random(501, 5), cref.g1_generator(), cref.g2_generator())
    prs = {"explicit": BG.Prover(ctx, BG.R1CS(ni, na, *mats)), "blocked": BG.Prover(ctx, br)}
    del mats
    d_in, d_aux = witness(ctx, A, T, B_, prog, epi, 64)
    r, s = cref.fr_random(502, 2)
    ctx.set_timing(True)
    blobs = {k: timed_prove(ctx, p, pk, d_in, d_aux, r, s)[1] for k, p in prs.items()}
    assert (blobs["explicit"] == blobs["blocked"]).all()
    res = {k: {"prove_s": [], "z_spmv_done_ms": []} for k in prs}
    for _ in range(reps):
        for k, p in prs.items():
            dt, b, st = timed_prove(ctx, p, pk, d_in, d_aux, r, s)
            assert (b == blobs[k]).all()
            res[k]["prove_s"].append(dt)
            res[k]["z_spmv_done_ms"].append(st["z_spmv_done"])
    ctx.set_timing(False)
    for k in res:
        res[k]["prove_s_mean"] = float(np.mean(res[k]["prove_s"]))
        res[k]["z_spmv_done_ms_mean"] = float(np.mean(res[k]["z_spmv_done_ms"]))
    out.update(res)
    out["constraints"], out["log_m"] = br.num_constraints, br.log_m
    for p in prs.values():
        p.free()
    pk.free()
    del pk, prs, d_in, d_aux
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-1024", action="store_true")
    ap.add_argument("--skip-256", action="store_true")
    args = ap.parse_args()
    ctx = B.Context(0)
    info = gpu_info()
    if not args.skip_1024:
        print(json.dumps({**info, **batch_1024(ctx, args.reps)}), flush=True)
    if not args.skip_256:
        print(json.dumps({**info, **batch_256(ctx, args.reps)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
