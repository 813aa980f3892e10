#!/usr/bin/env python3
"""Proving keys in host memory: what streaming the bases costs.

1. MSMs: G1 at 2^20 and 2^24, G2 at 2^20, each over a device vector with fixed-base tables, the same vector without tables,
   and the same vector in pinned host memory (streamed in chunks).  Reports scalars/s, and for the streamed runs the
   bytes copied host->device over the call's time and the chunk geometry.
2. The production update proof (A=15, T=3, B=4, 2^24 domain) with three copies of one key: device with tables, device
   without tables, all five vectors in host memory.  Reports proof time and free device memory before and after each key.
3. --big: the 1024-transaction batch (A=16, T=3, B=5, 2^26) with its key built straight into host memory by the blocked
   setup, if the machine has the ~35 GB of host RAM that needs; otherwise says so.

Pinned host->device bandwidth is measured in the same run, and the GPU's name and power limit are read.  Every timed call
ends in a device synchronise; one warm-up per variant, then --reps timed calls with the variants alternated; mean and
min-max.  One JSON line per part.

  python tools/bench_host_key.py [--reps 5] [--skip-msm] [--skip-proof] [--big]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bazuka_b200 as B  # noqa: E402
from bazuka_b200 import groth16 as BG  # noqa: E402
from bazuka_b200.mpn.native_circuit import NativeUpdateCircuit  # noqa: E402
from bench_mpn_1024 import free_gb, gpu_info, timed_prove, witness  # noqa: E402
from oracle import cref  # noqa: E402


def stats(xs):
    return {"mean": float(np.mean(xs)), "min": float(min(xs)), "max": float(max(xs))}


def h2d_gbps(reps):
    """pinned host -> device copies of 1 GiB, CUDA events"""
    n = 1 << 30
    src = torch.empty(n, dtype=torch.uint8).pin_memory()
    dst = torch.empty(n, dtype=torch.uint8, device="cuda")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(src, non_blocking=True)
        b.record()
        b.synchronize()
        out.append(n / (a.elapsed_time(b) / 1e3) / 1e9)
    del src, dst
    torch.cuda.empty_cache()
    return stats(out)


def msm_part(ctx, g, log_n, reps):
    n = 1 << log_n
    w = 104 if g == "g1" else 200
    img = torch.empty((n, w), dtype=torch.uint8, device="cuda")
    getattr(ctx, f"{g}_random_bases_dev")(70 + log_n, n, img)
    d_s = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    ctx.fr_random_dev(80 + log_n, n, d_s)
    ctx.synchronize()
    mk = getattr(ctx, f"{g}_bases_from_dev")
    variants = {"device_tables": mk(img, n), "device": mk(img, n), "host": mk(img, n)}
    del img
    torch.cuda.empty_cache()
    variants["device_tables"].precompute(16)
    variants["host"].move_to_host()
    msm = getattr(ctx, f"msm_{g}_resident")
    res = {k: [] for k in variants}
    want = None
    for k, b in variants.items():   # warm-up, and every variant gives the same sum
        out = msm(b, d_s)
        want = out if want is None else want
        assert (out == want).all(), k
    stream = None
    for _ in range(reps):
        for k, b in variants.items():
            ctx.synchronize()
            t0 = time.perf_counter()
            msm(b, d_s)
            ctx.synchronize()
            res[k].append(time.perf_counter() - t0)
            if k == "host":
                stream = ctx.last_msm_stream()
    out = {"msm": g.upper(), "log_n": log_n, "levels_tabled": variants["device_tables"].levels, "stream": stream}
    for k, ts in res.items():
        out[k] = {"s": stats(ts), "scalars_per_s": n / float(np.mean(ts))}
    out["host"]["h2d_gbps_over_call"] = stream["bytes_h2d"] / float(np.mean(res["host"])) / 1e9
    out["host_vs_device_untabled"] = float(np.mean(res["host"]) / np.mean(res["device"]))
    for b in variants.values():
        b.free()
    del d_s
    torch.cuda.empty_cache()
    return out


def proof_part(ctx, reps):
    A, T, B_ = 15, 3, 4
    nc = NativeUpdateCircuit(A, T, B_, blocked=True)
    br = nc.blocked_r1cs()
    prog, epi = nc.program(0), nc.program(1)
    nc.free()
    pk0, vk = BG.setup_gpu(ctx, br, cref.fr_random(501, 5), cref.g1_generator(), cref.g2_generator(), table_levels=1)
    img = BG.write_parameters(ctx, pk0)
    pk0.free()
    pr = BG.Prover(ctx, br)
    d_in, d_aux = witness(ctx, A, T, B_, prog, epi, 64)
    out = {"batch": "UpdateCircuit A=15 T=3 B=4 (256 tx)", "log_m": br.log_m, "key_packed_gb": img.size / 1e9, "free_gb": {"start": free_gb()}}
    keys = {}
    for k, kw in (("device_tables", {}), ("device", {"table_levels": 1}), ("host", {"host_vectors": "all"})):
        before = free_gb()
        keys[k], _ = BG.read_parameters(ctx, img, checked=False, **kw)
        out["free_gb"][k] = {"before_key": before, "after_key": free_gb()}
    r, s = cref.fr_random(502, 2)
    ctx.set_timing(True)
    blobs = {k: timed_prove(ctx, pr, pk, d_in, d_aux, r, s)[1] for k, pk in keys.items()}
    assert all((b == blobs["device"]).all() for b in blobs.values())
    res = {k: {"prove_s": [], "stage_ms": None} for k in keys}
    for _ in range(reps):
        for k, pk in keys.items():
            dt, b, st = timed_prove(ctx, pr, pk, d_in, d_aux, r, s)
            assert (b == blobs[k]).all()
            res[k]["prove_s"].append(dt)
            res[k]["stage_ms"] = st
    ctx.set_timing(False)
    for k in res:
        res[k]["prove_s"] = stats(res[k]["prove_s"])
    out.update(res)
    out["free_gb"]["after_proofs"] = free_gb()
    for pk in keys.values():
        pk.free()
    pr.free()
    del d_in, d_aux
    torch.cuda.empty_cache()
    return out


def host_ram_gb():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 1e6
    return 0.0


def big_part(ctx, reps):
    A, T, B_ = 16, 3, 5
    out = {"batch": "UpdateCircuit A=16 T=3 B=5 (1024 tx)", "r1cs": "blocked", "key": "host", "host_ram_available_gb": host_ram_gb()}
    if out["host_ram_available_gb"] < 40:
        out["not_measured"] = "less than 40 GB of host RAM available for the 32.1 GB pinned key"
        return out
    out["free_gb"] = {"start": free_gb()}
    nc = NativeUpdateCircuit(A, T, B_, blocked=True)
    br = nc.blocked_r1cs()
    prog, epi = nc.program(0), nc.program(1)
    nc.free()
    t0 = time.perf_counter()
    pk, vk = BG.setup_gpu(ctx, br, cref.fr_random(901, 5), cref.g1_generator(), cref.g2_generator(), table_levels=1, host_vectors="all")
    pr = BG.Prover(ctx, br)
    ctx.synchronize()
    out["setup_s"] = time.perf_counter() - t0
    out["free_gb"]["after_setup"] = free_gb()
    d_in, d_aux = witness(ctx, A, T, B_, prog, epi, 128)
    out["free_gb"]["after_witness"] = free_gb()
    r, s = cref.fr_random(902, 2)
    ctx.set_timing(True)
    out["warmup_prove_s"], blob, _ = timed_prove(ctx, pr, pk, d_in, d_aux, r, s)
    times = []
    for _ in range(reps):
        dt, b, st = timed_prove(ctx, pr, pk, d_in, d_aux, r, s)
        assert (b == blob).all()
        times.append(dt)
    ctx.set_timing(False)
    out["prove_s"] = stats(times)
    out["stage_ms_last"] = st
    out["free_gb"]["after_proofs"] = free_gb()
    out["verify_bytes"] = BG.verify_bytes(BG.vk_to_bincode(vk), d_in.cpu().numpy().view(np.uint64).reshape(-1, 4)[1:], blob)
    pk.free(); pr.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-msm", action="store_true")
    ap.add_argument("--skip-proof", action="store_true")
    ap.add_argument("--big", action="store_true")
    args = ap.parse_args()
    ctx = B.Context(0)
    info = {**gpu_info(), "pinned_h2d_gbps": h2d_gbps(args.reps)}
    print(json.dumps(info), flush=True)
    if not args.skip_msm:
        for g, log_n in (("g1", 20), ("g1", 24), ("g2", 20)):
            print(json.dumps({**info, **msm_part(ctx, g, log_n, args.reps)}), flush=True)
    if not args.skip_proof:
        print(json.dumps({**info, **proof_part(ctx, args.reps)}), flush=True)
    if args.big:
        print(json.dumps({**info, **big_part(ctx, args.reps)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
