"""Signatures per second of the batch Ed25519 checks (csrc/ed25519.cu) against the host call they replace.

GPU: bzk_ed25519_verify_batch on deposit-sized messages (the bincode of an unsigned `ContractDeposit`, about 160 bytes) and on
1 KiB messages, and bzk_mpn_deposits_verify_bytes on the bincode `Vec<MpnDeposit>` image (decoding and re-encoding each payment
on the host included), at each n, the items tiled from a few thousand distinct signatures.  Each timed call is the whole C call
on host arrays (copies in and out included) under a host clock; the call ends in a stream synchronisation.  One warm-up call of
each size runs first; the best of --reps calls is kept.
Host: bzk_ed25519_verify (one signature per call) on deposit-sized messages on one thread and on every usable core (ctypes
releases the GIL), in the same run.  The GPU's name and power limit are read with nvidia-smi.

    python tools/bench_ed25519.py [--log2 10,14,17,20] [--distinct 2048] [--reps 3] [--host-items 2000] [--out results.json]"""
import argparse
import ctypes as ct
import json
import multiprocessing
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np  # noqa: E402

import bazuka_b200 as B  # noqa: E402
from bazuka_b200.mpn import native as N, wire as Wr  # noqa: E402
from oracle.py import ed25519 as O  # noqa: E402   (signing the benchmark's inputs only)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or None, "power_limit": limit.strip() or None}


def _item(i):
    """one signed deposit (its image bytes, key, unsigned message, signature) and one signed 1 KiB message"""
    pk, sk = O.generate_keys(b"bench-%d" % (i % 256))
    pay = {"memo": "deposit %d" % i, "contract_id": 0x1234, "deposit_circuit_id": 0, "calldata": 0, "src": pk,
           "amount": {"token_id": "ziesha", "amount": 1000 + i}, "fee": {"token_id": "ziesha", "amount": 1}, "nonce": 1 + i // 256, "sig": None}
    w = Wr.Writer()
    Wr.enc_contract_deposit(w, pay)
    msg = bytes(w.b)
    sig = O.sign(sk, msg)
    w = Wr.Writer()
    Wr.enc_mpn_deposit(w, {"mpn_address": N.jj_compress(N.eddsa_keys(b"mpn")[0]), "payment": dict(pay, sig=sig)})
    kib = bytes((i * 31 + j) & 0xFF for j in range(1024))
    return bytes(w.b), pk, msg, sig, kib, O.sign(sk, kib)


def time_call(fn, reps):
    best = None
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2", default="10,14,17,20")
    ap.add_argument("--distinct", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-items", type=int, default=2000)
    ap.add_argument("--out", help="also write the results as JSON here")
    a = ap.parse_args()
    t0 = time.perf_counter()
    with multiprocessing.Pool(len(os.sched_getaffinity(0))) as pool:
        items = pool.map(_item, range(a.distinct), chunksize=16)
    print(f"signed {a.distinct} distinct deposits and 1 KiB messages in {time.perf_counter() - t0:.1f} s", flush=True)
    ctx = B.Context(0)
    lib = ctx._l
    out = {**gpu_info(), "distinct": a.distinct, "sizes": {}}
    for lg in (int(v) for v in a.log2.split(",")):
        n = 1 << lg
        sel = [items[i % a.distinct] for i in range(n)]
        pks = b"".join(t[1] for t in sel)
        ok, n_ok, cnt = np.zeros(n, np.uint8), ct.c_uint64(), ct.c_uint64()
        pok = ct.c_void_p(ok.ctypes.data)
        row = {}
        for name, mi, si in (("verify_batch_deposit_msgs", 2, 3), ("verify_batch_1kib_msgs", 4, 5)):
            msgs = b"".join(t[mi] for t in sel)
            sigs = b"".join(t[si] for t in sel)
            offs = np.zeros(n + 1, np.uint64)
            np.cumsum([len(t[mi]) for t in sel], out=offs[1:])
            po = ct.c_void_p(offs.ctypes.data)
            call = lambda: ctx._check(lib.bzk_ed25519_verify_batch(ctx._h, pks, sigs, msgs, po, n, pok, ct.byref(n_ok)))
            call()   # warm-up (the first call of a context also builds the fixed-base table)
            assert n_ok.value == n, (name, n, n_ok.value)
            dt = time_call(call, a.reps)
            row[name] = {"s": round(dt, 5), "sig_per_s": round(n / dt), "msg_bytes": int(offs[-1])}
        blob = n.to_bytes(8, "little") + b"".join(t[0] for t in sel)
        call = lambda: ctx._check(lib.bzk_mpn_deposits_verify_bytes(ctx._h, blob, len(blob), pok, n, ct.byref(cnt), ct.byref(n_ok)))
        call()
        assert cnt.value == n and n_ok.value == n
        dt = time_call(call, a.reps)
        row["deposits_verify_bytes"] = {"s": round(dt, 5), "sig_per_s": round(n / dt), "image_bytes": len(blob)}
        out["sizes"][n] = row
        print(json.dumps({"n": n, **row}), flush=True)
    ctx.close()
    # host: bzk_ed25519_verify on the deposit messages
    m = min(a.host_items, a.distinct)
    cases = [(t[1], t[2], t[3]) for t in items[:m]]

    def host_run(chunk):
        return sum(lib.bzk_ed25519_verify(pk, msg, len(msg), sig) for pk, msg, sig in chunk)

    t0 = time.perf_counter()
    assert host_run(cases) == m
    one = m / (time.perf_counter() - t0)
    cores = len(os.sched_getaffinity(0))
    work = cases * cores
    t0 = time.perf_counter()
    with ThreadPoolExecutor(cores) as ex:
        assert sum(ex.map(host_run, [work[k::cores] for k in range(cores)])) == len(work)
    allc = len(work) / (time.perf_counter() - t0)
    out["host"] = {"one_thread_sig_per_s": round(one), "cores": cores, "all_cores_sig_per_s": round(allc)}
    print(json.dumps({"host": out["host"], "gpu": out["gpu"], "power_limit": out["power_limit"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
