"""What tracking the transform U costs on the device (B200GSO_TRANSFORM): every integer row operation also updates a row
of U, 8 d bytes on top of the 8 n of the row of b.  Two workloads, each run with and without U, alternating:
  * one tour of BKZ-60 (strategies/default.json, BKZ_NO_LLL | BKZ_MAX_LOOPS = 1, seed 1) on bench.py's dim-200 knapsack
    basis (tests/golden/r200_lll_update_gso.npz), through bkz_reduction(b, param[, u]);
  * device LLL (delta 0.99, eta 0.51) on a batch of 1320 seeded 100 x 100 bases with 30-bit entries (the warp kernel),
    timed from the call to its return (the call ends with a stream synchronise).
Prints one JSON line per run and a summary line; the first line names the GPU and its power limit.

    python tools/transform_bench.py [--rounds 2] [--lll-reps 3] [--arms bkz,lll]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, plim, clk = [s.strip() for s in out.split(",")]
        return dict(gpu=name, power_limit=plim, max_sm_clock=clk)
    except Exception as e:
        return dict(gpu="unknown (%s)" % e)


def bkz_arm(rounds):
    import fplll_b200 as fb
    g = np.load(os.path.join(ROOT, "tests", "golden", "r200_lll_update_gso.npz"))
    par = fb.BKZParam(60, strategies="default", flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS, max_loops=1, seed=1)
    times = {False: [], True: []}
    outs = {}
    for r in range(rounds):
        for with_u in ((False, True) if r % 2 == 0 else (True, False)):
            b = g["b"].copy()
            u = np.zeros((b.shape[0], b.shape[0]), np.int64) if with_u else None
            t0 = time.perf_counter()
            st, stats = fb.bkz_reduction(b, par, u=u)
            sec = time.perf_counter() - t0
            times[with_u].append(sec)
            outs.setdefault(with_u, (b, st, int(stats["enum_nodes"])))
            emit(arm="bkz60_tour", with_u=with_u, round=r, status=int(st), wall_seconds=sec, sec_lll=stats["sec_lll"],
                 sec_enum=stats["sec_enum"], enum_nodes=int(stats["enum_nodes"]))
    same = np.array_equal(outs[False][0], outs[True][0]) and outs[False][1:] == outs[True][1:]
    emit(arm="bkz60_tour", summary=True, same_basis_status_nodes=bool(same),
         median_without_u=float(np.median(times[False])), median_with_u=float(np.median(times[True])),
         min_without_u=min(times[False]), min_with_u=min(times[True]))


def lll_arm(reps):
    import fplll_b200 as fb
    rng = np.random.default_rng(1)
    B, d = 1320, 100
    b = rng.integers(-(1 << 30), 1 << 30, size=(B, d, d), dtype=np.int64)
    times = {False: [], True: []}
    res = {}
    for r in range(reps + 1):  # round 0 warms both up (module load, first launches)
        for with_u in ((False, True) if r % 2 == 0 else (True, False)):
            m = fb.MatGSO(b, fb.GSO_ROW_EXPO | (fb.GSO_TRANSFORM if with_u else 0))
            m.sync()
            t0 = time.perf_counter()
            st, stats = m.lll(0.99, 0.51)
            sec = time.perf_counter() - t0
            res.setdefault(with_u, (m.b, st, stats["n_swaps"].copy()))
            m.close()
            if r:
                times[with_u].append(sec)
                emit(arm="lll_batch", with_u=with_u, round=r, lattices=B, d=d, seconds=sec,
                     swaps=int(stats["n_swaps"].sum()), failures=int((st != 0).sum()))
    same = (np.array_equal(res[False][0], res[True][0]) and np.array_equal(res[False][1], res[True][1]) and
            np.array_equal(res[False][2], res[True][2]))
    emit(arm="lll_batch", summary=True, same_basis_status_swaps=bool(same),
         median_without_u=float(np.median(times[False])), median_with_u=float(np.median(times[True])),
         min_without_u=min(times[False]), min_with_u=min(times[True]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--lll-reps", type=int, default=3)
    ap.add_argument("--arms", default="bkz,lll")
    a = ap.parse_args()
    emit(**gpu_info())
    arms = a.arms.split(",")
    if "lll" in arms:
        lll_arm(a.lll_reps)
    if "bkz" in arms:
        bkz_arm(a.rounds)


if __name__ == "__main__":
    main()
