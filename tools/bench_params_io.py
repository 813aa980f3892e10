#!/usr/bin/env python3
"""bellman `Parameters` file speed: write, read(checked=False) and read(checked=True) of a resident proving key to / from an
in-memory image (disk speed left out), for the 2^18 and 2^20 synthetic keys and the production update key (A=15, T=3, B=4).
Every timed call returns after a device synchronise; one warm-up call, then --reps timed calls (mean, min, max).  Reports
the image's bytes and point counts, the pinned H2D copy bandwidth measured in the same run, and the GPU's name and power
limit.  One JSON line per key.

  python tools/bench_params_io.py [--keys synth18,synth20,update] [--reps 5]
"""
import argparse
import ctypes as ct
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bazuka_b200 as B  # noqa: E402
from bazuka_b200 import groth16 as BG, synth  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or torch.cuda.get_device_name(), "power_limit": limit.strip() or None}


def pinned_h2d_gbs(nbytes=256 << 20, reps=5):
    src = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = []
    for _ in range(reps):
        e0.record()
        dst.copy_(src, non_blocking=True)
        e1.record()
        e1.synchronize()
        best.append(nbytes / (e0.elapsed_time(e1) * 1e-3) / 1e9)
    return max(best)


def timed(fn, reps):
    """fn may return a key to free after its time is taken"""
    ts = []
    for k in range(reps + 1):
        t0 = time.perf_counter()
        r = fn()
        if k:
            ts.append(time.perf_counter() - t0)
        if r is not None:
            r.free()
    return ts


def synth_key(ctx, lanes, rounds):
    ni, na, mats, _, _ = synth.build(lanes, rounds, seed=17, ops=synth.GpuOps(ctx))
    pr = BG.Prover(ctx, BG.R1CS(ni, na, *mats))
    tox = torch.empty((5, 4), dtype=torch.int64, device="cuda")
    ctx.fr_random_dev(99, 5, tox)
    ctx.synchronize()
    pk, _ = BG.setup_gpu(ctx, pr.r1cs, tox.cpu().numpy().view(np.uint64), BG.G1_GENERATOR, BG.G2_GENERATOR, table_levels=1)
    return f"synthetic {lanes}x{rounds} (2^{pr.log_m} domain)", pk, pr


def update_key(ctx):
    from bazuka_b200.mpn.worker import MpnUpdateWorker
    tox = torch.empty((5, 4), dtype=torch.int64, device="cuda")
    ctx.fr_random_dev(99, 5, tox)
    ctx.synchronize()
    w = MpnUpdateWorker(ctx, 15, 3, 4, tox.cpu().numpy().view(np.uint64), compiler="native")
    return f"UpdateCircuit A=15 T=3 B=4 (2^{w.prover.log_m} domain)", w.pk, w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default="synth18,synth20,update")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    ctx = B.Context(0)
    base = dict(gpu_info(), pinned_h2d_gb_s=round(pinned_h2d_gbs(), 2))
    makers = {"synth18": lambda: synth_key(ctx, 256, 100), "synth20": lambda: synth_key(ctx, 1024, 100), "update": lambda: update_key(ctx)}
    for name in a.keys.split(","):
        label, pk, owner = makers[name]()
        img = BG.write_parameters(ctx, pk)
        info = BG.parameters_info(img)
        points = sum(v for k, v in info.items() if k.startswith("n_"))
        out = dict(base, key=label, bytes=info["bytes"], points=points, counts={k: v for k, v in info.items() if k.startswith("n_")})
        buf = np.zeros_like(img)   # written into a buffer that is already mapped
        ic = np.ascontiguousarray(pk.vk["ic"], dtype=np.uint8).reshape(-1, 104)
        gamma = np.ascontiguousarray(pk.vk["gamma_g2"], dtype=np.uint8)
        n = ct.c_size_t()

        def write():
            ctx._check(ctx._l.bzk_groth16_params_write(ctx._h, pk._h, gamma.ctypes.data, ic.ctypes.data, len(ic), buf.ctypes.data, buf.size,
                                                        ct.byref(n)))
            ctx.synchronize()

        def read(checked):
            k, _ = BG.read_parameters(ctx, img, checked=checked, table_levels=1)
            ctx.synchronize()
            return k
        for tag, fn in (("write", write), ("read_unchecked", lambda: read(False)), ("read_checked", lambda: read(True))):
            ts = timed(fn, a.reps)
            mean = sum(ts) / len(ts)
            out[tag] = {"s_mean": round(mean, 4), "s_min": round(min(ts), 4), "s_max": round(max(ts), 4),
                        "gb_s": round(info["bytes"] / mean / 1e9, 2), "points_per_s": round(points / mean)}
        assert (buf == img).all()
        print(json.dumps(out), flush=True)
        pk.free()
        owner.free()
    ctx.close()


if __name__ == "__main__":
    main()
