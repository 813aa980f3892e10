"""The "MPN Groth16 proofs/s" half of the headline metric, measured on whole update batches through the native path

    bzk_mpn_update_build  ->  bzk_mpn_update_witness  ->  bzk_groth16_prove_dev        (include/bzk.h)

for the production batch (A=15, T=3, B=4: 256 transfers, 14.4 M constraints, 2^24 domain; the reference's
src/config/blockchain.rs:22-26) or BASELINE configs[3]'s depth-32 tree at the same batch (A=16, B=4, 2^24).  The 1024-transfer
batch of configs[3] (B=5, 2^26) does not fit the 80 GB of one H100.
Called by bench.py (default run: production batch at N=1; under torchrun also the (R) replicas and (S) base-sharded
schedules of SURVEY.md §8e) and usable stand-alone:

    python tools/mpn_batch_bench.py 15,3,4 [steps]

Timing: every proof is bracketed by device synchronisation and timed by the host wall clock (the prover drives five
streams, so no single-stream CUDA-event pair covers it); the stage split inside the prover comes from CUDA events
recorded on those streams (bzk_groth16_stage_ms).  N>1: barrier + synchronize on both sides, MAX over ranks."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _ledger_and_batches(ctx, A, T, B, nacc, n_batches):
    from bazuka_b200.mpn import native as N, update as U
    from bazuka_b200.mpn.ledger import NativeLedger, pack_txs
    ntx = 1 << (2 * B)
    led = NativeLedger(ctx, A, T)
    keys = []
    for i in range(nacc):
        pk, sk = N.eddsa_keys(b"acct%d" % i)
        keys.append((pk, sk))
        led.set_account(i, U.MpnAccount(0, 0, pk, {0: U.Money(U.ZIESHA, 10 ** 12)}))
    nonces, batches = [0] * nacc, []
    for _ in range(n_batches):
        txs = []
        for k in range(ntx):
            s, d = k % nacc, (k + 1) % nacc
            nonces[s] += 1
            tx = U.MpnTransaction(nonces[s], N.jj_compress(keys[s][0]), N.jj_compress(keys[d][0]), U.Money(U.ZIESHA, 1000 + k), U.Money(U.ZIESHA, 10))
            tx.sign(keys[s][1])
            txs.append(tx)
        batches.append(pack_txs(txs))
    return led, batches


def algorithmic_bytes(pr):
    """SURVEY.md §8(d): per proof, sum over the MSMs of their true lengths x (32 + 96 | 192) + 7 NTTs x 64 d + SpMV
    nnz x 40 + witness write 32 n_vars."""
    m = 1 << pr.log_m
    nnz = sum(int(mat[0][-1]) for mat in pr.r1cs.mats)
    g1_terms = pr.h_len + pr.l_len + pr.a_len + pr.b_len
    return {"msm_g1": 128 * g1_terms, "msm_g2": 224 * pr.b_len, "ntt": 7 * 64 * m, "spmv": 40 * nnz, "witness": 32 * pr.r1cs.num_vars,
            "g1_terms": g1_terms, "g2_terms": pr.b_len}


def batch_section(ctx, A=15, T=3, B=4, steps=3, dist=None, rank=0, world=1, peak_gbs=None, with_schedules=True):
    import torch
    from bazuka_b200 import groth16 as BG
    from bazuka_b200.mpn import update as U
    from bazuka_b200.mpn.cs import to_mont
    from bazuka_b200.mpn.worker import MpnUpdateWorker
    dev = torch.device("cuda", ctx.device)
    ntx = 1 << (2 * B)
    out = {"circuit": f"UpdateCircuit A={A} T={T} B={B} ({ntx} tx), /root/reference/src/mpn/circuits/update_circuit.rs:49-494",
           "path": "native: bzk_mpn_update_build -> bzk_mpn_update_witness -> bzk_groth16_prove_dev"}
    d = torch.empty((7, 4), dtype=torch.int64, device=dev)
    ctx.fr_random_dev(99, 7, d)
    ctx.synchronize()
    rnd = d.cpu().numpy().view(np.uint64)
    t0 = time.perf_counter()
    worker = MpnUpdateWorker(ctx, A, T, B, rnd[:5], compiler="native")
    pr, pk = worker.prover, worker.pk
    out.update({"constraints": pr.r1cs.num_constraints, "log_m": pr.log_m, "one_off_compile_and_key_s": time.perf_counter() - t0})
    t0 = time.perf_counter()
    led, batches = _ledger_and_batches(ctx, A, T, B, nacc=min(ntx, 64), n_batches=steps + 1)
    out["host_signing_s"] = time.perf_counter() - t0

    def barrier():
        if dist:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        if dist:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # ---- one batch at a time: build -> witness -> prove, each stage between synchronisations
    stage = {"build": [], "witness": [], "prove": []}
    proofs, kernel_marks = [], []
    ctx.set_timing(True)
    for b, txs in enumerate(batches):
        barrier()
        t0 = time.perf_counter()
        raws, ext, acc, pub, n_acc = led.update_build(txs, B)
        ctx.synchronize()
        t1 = time.perf_counter()
        d_in, d_aux = worker.witness.witness_native(raws, ext, [b + 1, b, pub["state"], U.ZIESHA, pub["aux_data"], pub["next_state"]], B)
        ctx.synchronize()
        t2 = time.perf_counter()
        blob, pts = pr.prove_dev(pk, d_in, d_aux, rnd[5], rnd[6], check_satisfied=(b == 0))
        t3 = time.perf_counter()
        assert n_acc == ntx
        if b:   # batch 0 is the warm-up (lazy module load, arena growth)
            stage["build"].append(t1 - t0); stage["witness"].append(t2 - t1); stage["prove"].append(t3 - t2)
            kernel_marks.append(pr.stage_ms())
        proofs.append((blob, to_mont([b + 1, b, pub["state"], pub["aux_data"], pub["next_state"]])))
    ctx.set_timing(False)
    ok = all(BG.verify_bytes(worker.vk_blob, pub_in, blob) for blob, pub_in in proofs)
    med = lambda v: float(np.median(v))
    prove_s = max_over_ranks(med(stage["prove"]))
    total_s = max_over_ranks(med(stage["build"]) + med(stage["witness"]) + med(stage["prove"]))
    out["sequential"] = {"s_per_batch": total_s, "proofs_per_s": 1 / total_s, "tx_per_s": ntx / total_s,
                         "stage_s_median": {k: med(v) for k, v in stage.items()}, "batches_timed": len(stage["prove"]),
                         "all_proofs_verify": bool(ok)}
    out["prove_only"] = {"ms_per_proof": prove_s * 1e3, "proofs_per_s": 1 / prove_s, "tx_per_s": ntx / prove_s,
                         "note": "bzk_groth16_prove_dev from the resident witness, median, host wall clock between synchronisations"}
    if kernel_marks and kernel_marks[0]:
        km = {k: float(np.median([m[k] for m in kernel_marks])) for k in kernel_marks[0]}
        out["prove_only"]["cuda_event_marks_ms"] = km
        ab = algorithmic_bytes(pr)
        total_bytes = ab["msm_g1"] + ab["msm_g2"] + ab["ntt"] + ab["spmv"] + ab["witness"]
        gbs = total_bytes / prove_s / 1e9
        out["prove_only"]["roofline"] = {"bound": "hbm", "algorithmic_bytes_per_proof": total_bytes, "parts": ab, "achieved": gbs, "unit": "GB/s",
                                         "peak": peak_gbs, "frac": gbs / peak_gbs if peak_gbs else None,
                                         "note": "integer-pipe bound in fact (DESIGN.md §3): the HBM fraction is what north_star asks to be reported"}
    # ---- (R) replicas: every GPU proves its own batch, no communication
    if with_schedules:
        reps = max(2, steps)
        d_in, d_aux = worker.witness.witness_native(raws, ext, [len(batches), len(batches) - 1, pub["state"], U.ZIESHA, pub["aux_data"], pub["next_state"]], B)
        ctx.synchronize()
        barrier()
        t0 = time.perf_counter()
        for _ in range(reps):
            pr.prove_dev(pk, d_in, d_aux, rnd[5], rnd[6], check_satisfied=False)
        torch.cuda.synchronize()
        dt = max_over_ranks(time.perf_counter() - t0)
        out["replicas"] = {"schedule": "R: one proof per GPU, independent works (the reference's own axis, /root/reference/src/mpn/mod.rs:79-107)",
                           "n_gpus": world, "proofs": reps * world, "wall_s_max_over_ranks": dt, "proofs_per_s": reps * world / dt,
                           "tx_per_s": ntx * reps * world / dt}
    # ---- (S) one proof base-sharded over all GPUs
    if with_schedules and world > 1:
        try:
            want, _ = pr.prove_dev(pk, d_in, d_aux, rnd[5], rnd[6], check_satisfied=False)
            spk = BG.shard_proving_key(ctx, pk, pr.log_m, rank, world)

            def sharded():
                sums = BG.allgather_partials(pr.prove_partial(spk, d_in, d_aux, check_satisfied=False), device=dev)
                return BG.finalize(worker.vk, sums, rnd[5], rnd[6])

            blob_s, _ = sharded()
            ts = []
            for _ in range(reps):
                barrier()
                t0 = time.perf_counter()
                sharded()
                torch.cuda.synchronize()
                ts.append(max_over_ranks(time.perf_counter() - t0))
            t_one = out["prove_only"]["ms_per_proof"] / 1e3
            out["sharded"] = {"schedule": "S: ONE proof, every MSM's bases sharded over the GPUs, one all-gather of 512 B per rank",
                              "n_gpus": world, "ms_per_proof": min(ts) * 1e3, "ms_per_proof_median": float(np.median(ts)) * 1e3,
                              "single_gpu_ms_per_proof": t_one * 1e3, "speedup_vs_1gpu": t_one / min(ts),
                              "proof_bytes_equal_single_gpu": bool((blob_s == want).all())}
            # (S') the same with the quotient pipeline split over the ranks too (bzk_groth16_shard_begin / _finish)
            try:
                sp = BG.SplitShardedProver(pr, spk, rank, world, dev)

                def sharded_split():
                    return BG.finalize(worker.vk, BG.allgather_partials(sp.partials(d_in, d_aux), device=dev), rnd[5], rnd[6])

                blob_q, _ = sharded_split()
                tq = []
                for _ in range(reps):
                    barrier()
                    t0 = time.perf_counter()
                    sharded_split()
                    torch.cuda.synchronize()
                    tq.append(max_over_ranks(time.perf_counter() - t0))
                out["sharded"]["split_quotient"] = {
                    "schedule": "S': S plus evaluation vector s owned by rank s mod world, combined on rank 3 mod world, quotient slices dealt "
                                "out over NCCL point-to-point (2 x 512 MiB in, (world-1)/world x 512 MiB out at 2^24)",
                    "ms_per_proof": min(tq) * 1e3, "ms_per_proof_median": float(np.median(tq)) * 1e3, "speedup_vs_1gpu": t_one / min(tq),
                    "proof_bytes_equal_single_gpu": bool((blob_q == want).all())}
                del sp
            except Exception as e:
                out["sharded"]["split_quotient"] = {"error": repr(e)}
            spk.free()
        except Exception as e:
            out["sharded"] = {"error": repr(e)}
    led.free()
    worker.free()
    torch.cuda.empty_cache()
    return out


if __name__ == "__main__":
    import bazuka_b200 as Bz
    shape = [int(v) for v in (sys.argv[1] if len(sys.argv) > 1 else "15,3,4").split(",")]
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    ctx = Bz.Context(0)
    print(json.dumps(batch_section(ctx, *shape, steps=steps)), flush=True)
