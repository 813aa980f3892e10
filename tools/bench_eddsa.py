"""Signatures per second of the batch EdDSA checks (csrc/jubjub.cu) against the host call they replace.

GPU: bzk_mpn_tx_verify_batch (MpnTransaction::verify_signature: two key decompressions, Poseidon-7, Poseidon-5, the two
scalar multiplications) and bzk_jubjub_eddsa_verify_batch (one decompression, Poseidon-5, the multiplications) at each n, the
items tiled from a few thousand distinct signed transfers.  Each timed call is the whole C call on packed host arrays (copies in
and out included) under a host clock; the call ends in a stream synchronisation.  One warm-up call of each size runs first.
Host: bzk_jubjub_eddsa_verify (libbzk's host arithmetic and host Poseidon, one signature per call) on one thread and on every
usable core (ctypes releases the GIL), in the same run.  The GPU's name and power limit are read with nvidia-smi.

    python tools/bench_eddsa.py [--log2 10,14,17,20] [--distinct 2048] [--reps 3] [--host-items 400]"""
import argparse
import ctypes as ct
import functools
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
from bazuka_b200.api import HostPoseidon  # noqa: E402
from bazuka_b200.mpn import native as N, signatures as S, update as U  # noqa: E402
from bazuka_b200.mpn.ledger import pack_txs  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or None, "power_limit": limit.strip() or None}


@functools.lru_cache(maxsize=None)
def _keys(k):
    return N.eddsa_keys(b"bench-%d" % k)


def _sign(args):
    i, n_keys = args
    s, d = i % n_keys, (i * 7 + 1) % n_keys
    ks, kd = _keys(s), _keys(d)
    t = U.MpnTransaction(1 + i // n_keys, N.jj_compress(ks[0]), N.jj_compress(kd[0]), U.Money(U.ZIESHA, 100 + i), U.Money(U.ZIESHA, 1))
    t.sign(ks[1])
    return t


def signed_transfers(n, n_keys=64):
    """n distinct transfers among n_keys accounts, signed in parallel on the host's cores (Python JubJub arithmetic)"""
    with multiprocessing.Pool(len(os.sched_getaffinity(0))) as pool:
        return pool.map(_sign, [(i, n_keys) for i in range(n)], chunksize=16)


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
    ap.add_argument("--host-items", type=int, default=400)
    a = ap.parse_args()
    t0 = time.perf_counter()
    txs = signed_transfers(a.distinct)
    tx_arr = pack_txs(txs)
    msgs = [t.hash() for t in txs]
    items = S.pack_items([t.src_pub_key for t in txs], msgs, [t.sig for t in txs])
    print(f"signed {a.distinct} distinct transfers in {time.perf_counter() - t0:.1f} s", flush=True)
    ctx = B.Context(0)
    lib = ctx._l
    d = np.frombuffer(N.JJ_D.to_bytes(32, "little"), np.uint64).copy()
    pd = ct.c_void_p(d.ctypes.data)
    out = {**gpu_info(), "distinct": a.distinct, "sizes": {}}
    for lg in (int(v) for v in a.log2.split(",")):
        n = 1 << lg
        idx = np.arange(n) % a.distinct
        tx_n, it_n = np.ascontiguousarray(tx_arr[idx]), np.ascontiguousarray(items[idx])
        ok, n_ok = np.zeros(n, np.uint8), ct.c_uint64()
        row = {}
        for name, fn, arr in (("tx_verify_batch", lib.bzk_mpn_tx_verify_batch, tx_n), ("eddsa_verify_batch", lib.bzk_jubjub_eddsa_verify_batch, it_n)):
            call = lambda: ctx._check(fn(ctx._h, pd, ct.c_void_p(arr.ctypes.data), n, ct.c_void_p(ok.ctypes.data), ct.byref(n_ok)))
            call()   # warm-up (the first call of a context also builds the fixed-base table)
            assert n_ok.value == n, (name, n, n_ok.value)
            dt = time_call(call, a.reps)
            row[name] = {"s": round(dt, 5), "sig_per_s": round(n / dt)}
        out["sizes"][n] = row
        print(json.dumps({"n": n, **row}), flush=True)
    ctx.close()
    # host: bzk_jubjub_eddsa_verify on affine keys (decompressed beforehand, as its callers do)
    m = min(a.host_items, a.distinct)
    cases = [(N.jj_decompress(t.src_pub_key), msgs[i], t.sig["r"], t.sig["s"]) for i, t in enumerate(txs[:m])]

    def host_run(chunk):
        hp = HostPoseidon()
        ok = sum(hp.eddsa_verify(N.JJ_D, *c) for c in chunk)
        hp.free()
        return ok

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
    n17 = 1 << 17
    if n17 in out["sizes"]:
        print(f"n=2^17: tx_verify_batch {out['sizes'][n17]['tx_verify_batch']['sig_per_s']:,} sig/s, eddsa_verify_batch "
              f"{out['sizes'][n17]['eddsa_verify_batch']['sig_per_s']:,} sig/s; host {allc:,.0f} sig/s on {cores} cores, {one:,.0f} on one")


if __name__ == "__main__":
    main()
