"""What tracking the transform costs in the device HLLL (b200hh_hlll, B200HH_TRANSFORM / B200HH_INV_TRANSFORM): every
row_addmul_we of size_reduce also updates a row of U (8 d bytes read and written on top of the 8 n_known_cols of the
row of b), and of U^-T; every swap also swaps rows of U and U^-T.  Two workloads, each run without U, with U, and with
U and U^-T, alternating the order from round to round:
  * a batch of 2112 seeded d = n = 100 lattices (30-bit uniform entries; 2112 = 132 SMs x 16 resident warps, one warp
    per lattice), with R_history as hlll needs it (8 MB per lattice);
  * the 120 x 400 sub-lattice of BASELINE config #3 (tests/golden/hlll_q400.npz: q400sub_in), one lattice.
Each call is timed with a host clock from a device synchronise to the return of hlll(), which ends in a stream
synchronise; round 0 warms every arm up and is not timed.  The first line names the GPU and its power limit; one JSON
line per timed call, then a summary per workload that also says whether the three arms ended on the same basis,
status and iteration counts, and the U arms on the same U.

    python tools/hlll_transform_bench.py [--rounds 3] [--batch 2112] [--arms batch100,q400sub]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARMS = ("none", "u", "u_uinvt")


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


def run_workload(name, b, rounds):
    from fplll_b200.householder import MatHouseholder
    d = b.shape[-2]
    eye = np.eye(d, dtype=np.int64)
    kws = {"none": {}, "u": {"u": eye}, "u_uinvt": {"u": eye, "u_inv_t": eye}}
    times = {a: [] for a in ARMS}
    res = {}
    for r in range(rounds + 1):
        order = ARMS[r % 3:] + ARMS[:r % 3]
        for arm in order:
            m = MatHouseholder(b, 5, **kws[arm])
            m.sync()
            t0 = time.perf_counter()
            st, it = m.hlll()
            sec = time.perf_counter() - t0
            res.setdefault(arm, (m.get_basis(), st, it, m.u if arm != "none" else None))
            m.close()
            if r:
                times[arm].append(sec)
                emit(workload=name, arm=arm, round=r, lattices=int(b.shape[0]), d=d, n=int(b.shape[-1]), seconds=sec,
                     iterations=int(it.sum()), failures=int((st != 0).sum()))
    same = all(np.array_equal(res["none"][k], res[a][k]) for a in ARMS[1:] for k in range(3))
    same_u = np.array_equal(res["u"][3], res["u_uinvt"][3])
    med = {a: float(np.median(times[a])) for a in ARMS}
    emit(workload=name, summary=True, same_basis_status_iterations=bool(same), same_u=bool(same_u),
         **{"median_" + a: med[a] for a in ARMS}, **{"min_" + a: min(times[a]) for a in ARMS},
         ratio_u=med["u"] / med["none"], ratio_u_uinvt=med["u_uinvt"] / med["none"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=2112)
    ap.add_argument("--arms", default="batch100,q400sub")
    a = ap.parse_args()
    emit(**gpu_info())
    arms = a.arms.split(",")
    if "batch100" in arms:
        rng = np.random.default_rng(1)
        run_workload("batch100", rng.integers(-(1 << 30), 1 << 30, size=(a.batch, 100, 100), dtype=np.int64), a.rounds)
    if "q400sub" in arms:
        z = np.load(os.path.join(ROOT, "tests", "golden", "hlll_q400.npz"))
        run_workload("q400sub", z["q400sub_in"].astype(np.int64)[None], a.rounds)


if __name__ == "__main__":
    main()
