"""Time bzk_mpn_state_apply_delta: a production-shape block (A=15, T=3: 256 transfers + 64 deposits + 64 withdrawals through
bzk_mpn_prepare_works) and a snapshot of 2^log2 accounts with 1-4 tokens each, applied to a fresh ledger.

Each timed call is the whole C call (decode, plan, every launch, the copy back, the check and the commit) under a host clock;
the call ends in a stream synchronisation.  A warm-up call of the same shape runs first.  Beside the times it reports the plan's
launches (checked against the context's launch counter), Poseidon calls per arity and host-to-device / device-to-host bytes,
computed from the delta and the ledger before it.  For comparison, the leaf-by-leaf host restatement (tests/mpn_delta_cases.py
LeafState, one `set_data` after the other over libbzk's host Poseidon) is timed on a SAMPLE of leaves; its total is an
EXTRAPOLATION from that sample.  The GPU's name and power limit are read in the same run.

    python tools/bench_mpn_apply_delta.py [--log2 20] [--reps 5] [--sample 2000]"""
import argparse
import ctypes as ct
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

import numpy as np  # noqa: E402

import bazuka_b200 as B  # noqa: E402
from bazuka_b200 import _lib  # noqa: E402
from bazuka_b200.mpn.ledger import NativeLedger  # noqa: E402
from bench_mpn_1024 import gpu_info  # noqa: E402
import mpn_delta_cases as C  # noqa: E402
from test_gpu_mpn_apply_delta import production_block  # noqa: E402


def plan_counts(A, T, before_nonempty, touched, slots):
    """the plan bzk_mpn_state_apply_delta builds: touched = sorted account indices, slots = (touched ordinal, token slot) of
    every token the touched accounts hold afterwards, before_nonempty = indices of the non-empty accounts before"""
    touched = np.asarray(touched, np.uint64)
    ords, sl = (np.asarray(x, np.uint64) for x in zip(*slots)) if len(slots) else (np.zeros(0, np.uint64),) * 2
    steps = [("P2", len(sl))]
    for lv in range(1, T + 1):
        steps.append(("P4", len(np.unique(ords * np.uint64(1 << 2 * T) + (sl >> np.uint64(2 * lv))))))
    steps.append(("P5", len(touched)))
    pre = np.asarray(sorted(before_nonempty), np.uint64)
    clean = 0
    for lv in range(1, A + 1):
        steps.append(("P4", len(np.unique(touched >> np.uint64(2 * lv)))))
        parents = np.unique(touched >> np.uint64(2 * lv))
        kids = np.unique(pre >> np.uint64(2 * (lv - 1)))
        dirty = np.unique(touched >> np.uint64(2 * (lv - 1)))
        kids = kids[np.isin(kids >> np.uint64(2), parents)]
        clean += int((~np.isin(kids, dirty)).sum())
    arity = {"P2": 2, "P4": 4, "P5": 5}
    n_ops = sum(arity[k] * n for k, n in steps)
    hv = (T + 1) + (A + 1) + 2 * len(sl) + 4 * len(touched) + clean
    d2h = sum(n for _, n in steps[T + 1:])
    calls = {k: sum(n for kk, n in steps if kk == k) for k in arity}
    return {"launches": sum(1 for _, n in steps if n), "poseidon_calls": calls, "h2d_bytes": 4 * n_ops + 32 * hv, "d2h_bytes": 32 * d2h,
            "clean_siblings_read": clean}


def timed_apply(ctx, make_ledger, image, reps):
    """(seconds per call over `reps` calls after one warm-up, launches of one call)"""
    out, launches = [], 0
    for r in range(reps + 1):
        led = make_ledger()
        l0 = ctx._l.bzk_ctx_launch_count(ctx._h)
        t = time.perf_counter()
        led.apply_delta(image)
        dt = time.perf_counter() - t
        launches = ctx._l.bzk_ctx_launch_count(ctx._h) - l0
        led.free()
        if r:
            out.append(dt)
    return {"mean_s": float(np.mean(out)), "min_s": float(min(out)), "max_s": float(max(out)), "reps": reps}, launches


class HostHasher:
    """libbzk's host Poseidon (bzk_poseidon_host_hash), one hash per call, for the leaf-by-leaf restatement"""
    R2 = pow(2, 512, C.R)

    def __init__(self, lib):
        self.lib, self.h = lib, ct.c_void_p()
        blob = open(_lib.PARAMS_PATH, "rb").read()
        assert lib.bzk_poseidon_host_create(blob, len(blob), ct.byref(self.h)) == 0
        self.buf, self.out = np.zeros((5, 4), np.uint64), np.zeros(4, np.uint64)
        self.rinv = pow(1 << 256, -1, C.R)

    def __call__(self, xs):
        for k, x in enumerate(xs):
            self.buf[k] = np.frombuffer(((x << 256) % C.R).to_bytes(32, "little"), np.uint64)
        assert self.lib.bzk_poseidon_host_hash(self.h, len(xs), C.ptr(self.buf), 1, C.ptr(self.out)) == 0
        return int.from_bytes(self.out.tobytes(), "little") * self.rinv % C.R


def host_sample(lib, A, T, entries, sample):
    """seconds per leaf of the leaf-by-leaf restatement over the first `sample` entries (applied to an empty state)"""
    orc = C.LeafState(A, T, HostHasher(lib))
    part = entries[:sample]
    t = time.perf_counter()
    for loc, v in part:
        orc.set_data(loc, v or 0)
    return (time.perf_counter() - t) / len(part)


def block_part(ctx, reps, sample):
    st, keys, block = production_block()
    led = C.load(ctx, st, 15, 3)
    _, fork, _ = C.run_block(ctx, led, *block)
    image, n = C.delta_bytes(led, fork)
    fork.commit_accounts()
    want = fork.info()
    entries = C.parse(image)
    # the final token slots of every touched account: the old account, then the delta's leaves
    touched = sorted({loc[0] for loc, _ in entries})
    final = {}
    for i in touched:
        a = st.accounts.get(i)
        final[i] = {s: [m.token_id, m.amount] for s, m in (a.tokens.items() if a else [])}
    for loc, v in entries:
        if len(loc) == 4:
            final[loc[0]].setdefault(loc[2], [0, 0])[loc[3]] = v or 0
    slots = [(o, s) for o, i in enumerate(touched) for s, (tid, _) in sorted(final[i].items()) if tid]
    counts = plan_counts(15, 3, [i for i in st.accounts], touched, slots)
    t, launches = timed_apply(ctx, led.fork, image, reps)
    probe = led.fork()
    probe.apply_delta(image, expect={"state_hash": want["state_hash"], "state_size": want["state_size"]})
    probe.free()
    per_leaf = host_sample(ctx._l, 15, 3, entries, min(sample, len(entries)))
    led.free(); fork.free()
    assert launches == counts["launches"], (launches, counts)
    return {"case": "production block A=15 T=3 (256 transfers + 64 deposits + 64 withdrawals)", "entries": n, "touched_accounts": len(touched),
            "apply": t, **counts, "host_restatement_per_leaf_s_sample": per_leaf, "host_restatement_sample_leaves": min(sample, len(entries)),
            "host_restatement_total_s_extrapolated": per_leaf * n}


def snapshot_part(ctx, log2, reps, sample):
    A, T, n = 15, 3, 1 << log2
    image = C.snapshot_image(0, n, T)
    a = C.snapshot_accounts(0, n, T)
    ords = np.repeat(np.arange(n, dtype=np.uint64), a["ntok"].astype(np.int64))
    mask = np.arange(4)[None, :] < a["ntok"][:, None].astype(np.int64)
    counts = plan_counts(A, T, [], np.arange(n, dtype=np.uint64), list(zip(ords, a["slots"][mask])))
    t, launches = timed_apply(ctx, lambda: NativeLedger(ctx, A, T), image, reps)
    entries = C.parse(C.snapshot_image(0, max(1, sample // 9 + 1), T))
    per_leaf = host_sample(ctx._l, A, T, entries, min(sample, len(entries)))
    n_entries = int(np.frombuffer(image[:8], np.uint64)[0])
    assert launches == counts["launches"], (launches, counts)
    return {"case": "snapshot of 2^%d accounts, 1-4 tokens each, A=15 T=3" % log2, "entries": n_entries, "image_bytes": len(image), "apply": t, **counts,
            "host_restatement_per_leaf_s_sample": per_leaf, "host_restatement_sample_leaves": min(sample, len(entries)),
            "host_restatement_total_s_extrapolated": per_leaf * n_entries}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=2000)
    ap.add_argument("--skip-snapshot", action="store_true")
    args = ap.parse_args()
    ctx = B.Context(0)
    info = gpu_info()
    print(json.dumps({**info, **block_part(ctx, args.reps, args.sample)}), flush=True)
    if not args.skip_snapshot:
        print(json.dumps({**info, **snapshot_part(ctx, args.log2, args.reps, args.sample)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
