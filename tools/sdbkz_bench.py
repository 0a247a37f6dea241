"""Measures dual vs primal SVP enumeration (shared-memory walker vs thread-local variant) and one tour of SD-BKZ-60 and
of slide reduction (block 60) on the device, plus the same tours by the reference on the host when oracle/_ref is built.
Prints one JSON line per figure, the first one naming the GPU and its power limit.

    python tools/sdbkz_bench.py [--reps 3] [--arms enum,sd,slide,ref_sd,ref_slide] [--slide-block 60] [--ref-threads N]

The thread-local arm runs in a child process (B200_ENUM_XS=0 is read once per process)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def emit(**kw):
    print(json.dumps(kw), flush=True)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, plim, clk = [s.strip() for s in out.split(",")]
        return dict(gpu=name, power_limit=plim, max_sm_clock=clk)
    except Exception as e:  # the figures below are still the device's; say that the card could not be named
        return dict(gpu="unknown (%s)" % e)


def enum_arm(reps):
    """nodes/s of the pruned BKZ-60 block of bench.py (primal) and of the dual call svp_reduction makes on the same
    rows [140, 200) (beta = 60 pruning, radius delta / r(199, 199)); device time from CUDA events, median of reps."""
    from fplll_b200 import enumeration as en
    xs = os.environ.get("B200_ENUM_XS", "1") != "0"
    p = np.load(os.path.join(GOLD, "enum_r200_b60_pruned_140.npz"))
    g = np.load(os.path.join(GOLD, "bkz_sd_sld.npz"))
    cases = [("primal", p["mut"], p["rdiag"], p["pruning"], float(p["maxdist"]), False),
             ("dual", g["dual60_mut"], g["dual60_rdiag"], g["dual60_pruning"], float(g["dual60_maxdist"]), True)]
    for name, mut, rdiag, prun, R, dual in cases:
        en.enumerate_svp(mut, rdiag, prun, R, dual=dual)  # warm-up: module load, buffers
        rows = []
        for _ in range(reps):
            res = en.enumerate_svp(mut, rdiag, prun, R, dual=dual)
            rows.append((res["stats"]["device_ms"], int(res["nodes"].sum()), res["stats"]["total_us"]))
        rows.sort()
        ms, nodes, us = rows[len(rows) // 2]
        emit(what="enum_%s_d60" % name, walker="shared-memory" if xs else "thread-local", nodes=nodes,
             device_ms=round(ms, 3), call_ms=round(us / 1000, 3), nodes_per_s=nodes / (ms / 1000), reps=reps,
             device_ms_all=[round(r[0], 3) for r in rows])


def tour_arm(which, slide_block):
    """one SD-BKZ-60 tour and one slide tour (block 60), default strategies, dim-200 knapsack basis (LLL-reduced);
    wall time of b200bkz_reduce, which ends in a device synchronise (the basis is read back)"""
    import fplll_b200 as fb
    b0 = np.load(os.path.join(GOLD, "r200_lll_update_gso.npz"))["b"]
    for name, bs, fl in (("sd_bkz60", 60, fb.BKZ_SD_VARIANT), ("slide%d" % slide_block, slide_block, fb.BKZ_SLD_RED)):
        if name.rstrip("0123456789").replace("_bkz", "") not in which:
            continue
        b = b0.copy()
        t0 = time.time()
        st, s = fb.bkz_reduction(b, fb.BKZParam(bs, strategies="default", max_loops=1,
                                                flags=fl | fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS))
        emit(what="tour_%s_dim200" % name, status=st, wall_s=round(time.time() - t0, 3), sec_enum=round(s["sec_enum"], 3),
             sec_lll=round(s["sec_lll"], 3), enum_calls=s["enum_calls"], enum_nodes=s["enum_nodes"],
             r00_before=s["r00_before"], r00_after=s["r00_after"])


def reference_arm(which, threads, slide_block):
    """the same two runs by the reference's bkz_reduction (oracle/_ref/ref_probe, enumlib with `threads` threads)"""
    probe = os.path.join(ROOT, "oracle", "_ref", "ref_probe")
    if not os.path.exists(probe):
        emit(what="reference", skipped="oracle/_ref/ref_probe not built")
        return
    from oracle import oracle as O
    b0 = np.load(os.path.join(GOLD, "r200_lll_update_gso.npz"))["b"]
    with tempfile.TemporaryDirectory() as tmp:
        inp = os.path.join(tmp, "in.txt")
        O.write_matrix(inp, b0)
        for name, bs, fl in (("sd_bkz60", 60, 0x100), ("slide%d" % slide_block, slide_block, 0x200)):
            if "ref_" + name.rstrip("0123456789").replace("_bkz", "") not in which:
                continue
            t0 = time.time()
            o = O.run_ref("load %s\nbkz %d %d 1 default enumlib %d\n" % (inp, bs, fl | 2 | 4, threads), timeout=3600)
            line = [ln for ln in o.splitlines() if ln.startswith("bkz status=")][-1]
            emit(what="reference_tour_%s_dim200" % name, threads=threads, host_cpus=os.cpu_count(),
                 status=int(line.split("status=")[1].split()[0]), sec=float(line.split("sec=")[1].split()[0]),
                 wall_s=round(time.time() - t0, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--arms", default="enum,sd,slide,ref_sd,ref_slide")
    ap.add_argument("--slide-block", type=int, default=60)
    ap.add_argument("--ref-threads", type=int, default=os.cpu_count())
    ap.add_argument("--enum-only", action="store_true", help=argparse.SUPPRESS)  # the child process's arm
    a = ap.parse_args()
    if a.enum_only:
        enum_arm(a.reps)
        return
    import torch
    if not torch.cuda.is_available():
        sys.exit("sdbkz_bench: no CUDA device (this measures the GPU; there is nothing to fall back to)")
    arms = a.arms.split(",")
    emit(what="device", **gpu_info())
    if "enum" in arms:
        enum_arm(a.reps)
        env = dict(os.environ, B200_ENUM_XS="0")
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--enum-only", "--reps", str(a.reps)], env=env,
                           capture_output=True, text=True, timeout=1800)
        sys.stdout.write(p.stdout)
        if p.returncode:
            sys.exit(p.stderr[-2000:])
    tour_arm(arms, a.slide_block)
    reference_arm(arms, a.ref_threads, a.slide_block)


if __name__ == "__main__":
    main()
