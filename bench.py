#!/usr/bin/env python
"""bench.py — GSO-update throughput on H100 (the BASELINE.json metric), one JSON line on stdout.

Step  = what LLLReduction::babai pays per iteration on the GSO state of every lattice of a batch
        (lll.cpp:166-224):  row_op_end(kappa, kappa+1)  [update_bf + Gram/GSO invalidation, gso_interface.cpp:32-53]
        followed by  update_gso_row(kappa, kappa)  [Gram row recompute + forward substitution,
        gso_interface.cpp:131-164], at kappa = d-1 of dim-200 (200 x 201) lattices — the shape of BASELINE
        configs #2/#5.  Independent lattices are the only axis the GSO path shards on (SURVEY §8e: replicas),
        so N GPUs = N independent batches, no data-path collective, scaling "weak".
value = algorithmic bytes of update_gso_row (SURVEY §8a2: 8*[(i+1)*n + i(i-1)/2 + 4(i+1)] per lattice, Gram row
        invalid) * lattices * steps / device time of the timed region (CUDA events on the launching stream,
        max over ranks) — inputs resident in HBM.
e2e   = same metric through the C-ABI with HOST buffers: every step uploads each lattice's refreshed integer row
        kappa from pinned host memory (b200gso_upload_row = write b[kappa] + row_op_end), runs update_gso_row and
        reads rows kappa of mu and r back (b200gso_get_mu_r_row) — the protocol of a host-resident LLL driver.
--impl reference : the UNMODIFIED reference (oracle/_ref/ref_probe over libfplll.so) doing the same step on the
        box's host cores, all threads; bounded sample.
--dump-outputs DIR : after the timed steps, rows kappa of mu and r of every lattice as the device-resident path left
        them (update_row_mu.npy, update_row_r.npy) and as the last end-to-end step read them back (e2e_mu.npy,
        e2e_r.npy), float64; a fixed sample of lattices when the batch would pass 64 MB.  The inputs are seeded, so
        two builds run with the same arguments can be compared array for array.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

D, N_COLS = 200, 201
KAPPA = D - 1
METRIC = "gso_update_row_GBps"


def alg_bytes_update_row(i, n, g=1):
    return 8 * ((i + 1) * n * g + i * (i - 1) // 2 + 4 * (i + 1))


def measure_traffic(batch, local):
    """dram__bytes_read.sum + dram__bytes_write.sum of ONE launch of k_update_row, measured now: `ncu --metrics ...` around
    a child of this script (`--traffic-child`) that builds the same state and launches the kernel a few times.  Hardware
    counters cannot be read from inside an unprofiled run, and nothing timed runs under the profiler.  None if ncu is not
    usable on this box."""
    import csv
    import io
    try:
        env = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", str(local)))
        cmd = ["ncu", "--metrics", "dram__bytes_read.sum,dram__bytes_write.sum", "--clock-control", "none", "--csv",
               "-k", "regex:k_update_row", "--launch-skip", "2", "--launch-count", "1",
               sys.executable, os.path.abspath(__file__), "--traffic-child", str(batch)]
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=240, env=env)
        tot, seen = 0.0, 0
        for row in csv.DictReader(io.StringIO(p.stdout[p.stdout.index('"ID"'):])):
            v = float(row["Metric Value"].replace(",", ""))
            unit = row["Metric Unit"].lower()
            v *= {"byte": 1.0, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9, "tbyte": 1e12}[unit]
            tot += v
            seen += 1
        return tot if seen == 2 else None
    except Exception:
        return None


def traffic_child(batch):
    """`bench.py --traffic-child B`: the bench state, five launches of the update kernel, nothing else (run under ncu)."""
    import ctypes as C
    import torch
    import fplll_b200 as fb
    from fplll_b200.gso import _lib, _ck
    dev_b = torch.randint(-(1 << 20), 1 << 20, (batch, D, N_COLS), dtype=torch.int64, device="cuda")
    m = fb.MatGSO.__new__(fb.MatGSO)
    m.batch, m.d, m.n, m.flags, m.enable_row_expo = batch, D, N_COLS, fb.GSO_ROW_EXPO, True
    m._h = C.c_void_p()
    _ck(_lib().b200gso_create(C.byref(m._h), batch, D, N_COLS, fb.GSO_ROW_EXPO, 0), "create")
    _ck(_lib().b200gso_set_basis_dev(m._h, C.c_void_p(dev_b.data_ptr())), "set_basis_dev")
    assert m.update_gso().all()
    m.time_update_row(KAPPA, 5, True)
    m.sync()
    return 0


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return json.load(open(p)).get("hbm_gbs", 3350.0), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "H100 SXM data sheet HBM3 bandwidth (3.35 TB/s), not measured"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""

    def __init__(self, gpu=0):
        self.gpu, self.rows, self.proc = gpu, [], None

    def start(self):
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.gpu), "--query-gpu=" + q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.th = threading.Thread(target=self._read, daemon=True)
            self.th.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([t.strip() for t in line.split(",")])

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm = sorted(int(r[0]) for r in self.rows if r and r[0].isdigit())
        mx = [int(r[1]) for r in self.rows if len(r) > 1 and r[1].isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for k, n in enumerate(names) if any(len(r) > 2 + k and r[2 + k] == "Active" for r in self.rows)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(sm)}


def host_info():
    """CPU model, online cores and NUMA nodes of the box: the reference arm swings with the host (round 1: 5.9x between
    two boxes), so the ratio can only be read next to this."""
    info = {"cores_online": os.cpu_count()}
    try:
        out = subprocess.run(["lscpu"], capture_output=True, text=True, timeout=10).stdout
        for line in out.splitlines():
            k, _, v = line.partition(":")
            k, v = k.strip(), v.strip()
            if k == "Model name":
                info["cpu_model"] = v
            elif k == "NUMA node(s)":
                info["numa_nodes"] = int(v)
            elif k == "Thread(s) per core":
                info["threads_per_core"] = int(v)
            elif k == "CPU max MHz":
                info["cpu_max_mhz"] = float(v)
        la = os.getloadavg()
        info["loadavg_1m"] = la[0]
    except Exception:
        pass
    return info


def cpu_reference(seconds_target=12.0):
    """Times the reference's own CPU path (oracle/_ref) on all host threads: the same step on dim-200 lattices."""
    import numpy as np
    from oracle import oracle as O
    cores = os.cpu_count() or 1
    if not O.have_ref():
        return None
    rng = np.random.default_rng(12345)
    b = rng.integers(-(1 << 20), 1 << 20, size=(D, N_COLS), dtype=np.int64)
    tmp = tempfile.mkdtemp(prefix="bench_ref_")
    mat = os.path.join(tmp, "b.txt")
    O.write_matrix(mat, b)
    per = 4  # lattices per thread
    # calibrate with a short run, then size reps for ~seconds_target
    def run(reps):
        out = O.run_ref("load %s\ntolong\ngso l 2\ntime_update_row_mt %d %d %d %d\n" % (mat, KAPPA, reps, cores, per))
        tok = dict(t.split("=") for t in out.split("time_update_row_mt")[1].split() if "=" in t)
        return float(tok["timed_sec"]), int(tok["calls"])
    reps = 50
    t, calls = run(reps)
    while t < 0.5 * seconds_target and reps < (1 << 24):
        reps = int(reps * min(8.0, max(1.5, 1.1 * seconds_target / max(t, 1e-3))))
        t, calls = run(reps)
    gbps = calls * alg_bytes_update_row(KAPPA, N_COLS) / t / 1e9
    return {"value": gbps, "unit": "GB/s", "cores": cores, "kind": "reference",
            "sample": "%d calls of {row_op_end(%d,%d); update_gso_row(%d)} on %d private dim-%d MatGSO<long,double> "
                      "objects, %d threads, %.1f s" % (calls, KAPPA, KAPPA + 1, KAPPA, cores * per, D, cores, t),
            "us_per_call_per_thread": t / (calls / cores) * 1e6, "host": host_info()}


def enum_extras(local):
    """Secondary figure of the BASELINE metric's BKZ half: the device enumerator on a full-size BKZ-60 block of the
    dim-200 knapsack basis (tests/golden/enum_r200_b60_pruned_140.npz: 5.6e8 nodes, the reference visits exactly the
    same nodes), next to the reference's own enumerators on the host cores (oracle/_ref, bounded: one run)."""
    import numpy as np
    from fplll_b200 import enumeration as en
    out = {}
    try:
        z = np.load(os.path.join(ROOT, "tests", "golden", "enum_r200_b60_pruned_140.npz"))
        en.enumerate_svp(z["mut"], z["rdiag"], z["pruning"], float(z["maxdist"]), devices=[local])  # warm-up
        t0 = time.perf_counter()
        res = en.enumerate_svp(z["mut"], z["rdiag"], z["pruning"], float(z["maxdist"]), devices=[local])
        dt = time.perf_counter() - t0
        n = int(res["nodes"].sum())
        out = {"workload": "SVP enumeration, block [140,200) of LLL-reduced latticegen r 200 2000, default.json "
                           "beta=60 pruning, radius 1.05*GH", "nodes": n, "nodes_equal_reference": n == int(z["nodes"].sum()),
               "gpu_seconds": dt, "gpu_nodes_per_s": n / dt, "rounds": res["stats"]["n_rounds"]}
        from oracle import oracle as O
        if O.have_ref():
            g = np.load(os.path.join(ROOT, "tests", "golden", "r200_lll_update_gso.npz"))
            tmp = tempfile.mkdtemp(prefix="bench_enum_")
            mat, pr, ob = os.path.join(tmp, "b.txt"), os.path.join(tmp, "p.txt"), os.path.join(tmp, "o.bin")
            O.write_matrix(mat, g["b"])
            open(pr, "w").write(" ".join(repr(float(c)) for c in z["pruning"]))
            factor = float(z["maxdist"]) / float(z["rdiag"][0])
            cores = os.cpu_count() or 1
            o = O.run_ref("load %s\ntolong\ngso l 2\nupdate_gso\nset_threads %d\nenum 140 200 %r %s %s enumlib\n"
                          % (mat, cores, factor, pr, ob), timeout=600)
            tok = dict(t.split("=") for t in o.split("enum d=")[1].split() if "=" in t)
            out["cpu_reference"] = {"kind": "reference enumlib", "threads": cores, "seconds": float(tok["sec"]),
                                    "nodes": int(tok["nodes"]), "nodes_per_s": int(tok["nodes"]) / float(tok["sec"])}
            out["speedup_vs_cpu_reference"] = float(tok["sec"]) / dt
    except Exception as ex:  # never break the headline line
        out["error"] = str(ex)[:300]
    return out


def hh_extras(local):
    """Householder update_R(i) (householder.cpp:151-184) at config #3's shape d = n = 400, i = 399, batched; algorithmic
    bytes per lattice 8*[T(i) + 2n], T(i) = i*n - i(i-1)/2 (V rows streamed once, R_i read+written; history off)."""
    import numpy as np
    out = {}
    try:
        from fplll_b200.householder import MatHouseholder
        d = n = 400
        i = d - 1
        B = int(os.environ.get("B200_BENCH_HH_BATCH", 2640))  # 20 resident warps of hk_update_R<14> x 132 SMs of an H100
        rng = np.random.default_rng(7)
        b = rng.integers(-(1 << 20), 1 << 20, size=(1, d, n), dtype=np.int64)
        m = MatHouseholder(np.broadcast_to(b, (B, d, n)), 5, device=local, keep_history=False)
        for r in range(i):  # a real QR state: V_0 .. V_{i-1} are the reflections of the first i rows
            m.refresh_R_bf(r)
            m.update_R(r)
        m.refresh_R_bf(i)
        m.time_update_R(i, 2)
        ms = m.time_update_R(i, 5)
        T = i * n - i * (i - 1) // 2
        per = 8 * (T + 2 * n)
        peak, _ = peaks()
        out_variant = "hk_update_R_x32" if os.environ.get("B200_HH_X32") == "1" else "hk_update_R"
        out = {"workload": "batched update_R(399, false) on %d lattices of d=n=400 (V = the reflections of rows 0..398)" % B,
               "kernel": out_variant,
               "algorithmic_bytes_per_lattice": per, "ms_per_launch": ms, "GBps": B * per / (ms * 1e-3) / 1e9,
               "frac_of_hbm_peak": B * per / (ms * 1e-3) / 1e9 / peak}
        m.close()
    except Exception as ex:
        out["error"] = str(ex)[:300]
    return out


def bkz_extras(local, devices=None, with_ref=True):
    """The BKZ half of the BASELINE metric: wall-seconds of ONE tour of BKZ-60 (strategies/default.json table, fp64,
    BKZ_NO_LLL | BKZ_MAX_LOOPS=1) on the wrapper-LLL-reduced latticegen r 200 2000 basis (tests/golden), device GSO/LLL +
    device enumeration, next to the reference's bkz_reduction on the same input on the host (1 thread = the CLI default,
    and all threads through set_threads)."""
    import numpy as np
    out = {}
    try:
        import fplll_b200 as fb
        g = np.load(os.path.join(ROOT, "tests", "golden", "r200_lll_update_gso.npz"))
        # fp64 BKZ on this basis is fragile in the reference itself: its own bkz_reduction dies with "infinite loop in
        # babai" (RedStatus 3) for 2 of 5 RNG seeds within one tour (measured with oracle/_ref, DESIGN.md §3.6), so a
        # failed attempt is retried with the next rerandomisation seed, every attempt is reported
        # Every SVP call enumerates the fixed region of its initial radius (include/b200bkz.h: the default), so a tour is a
        # function of (basis, seed) alone: seeds 1 and 3 end with status 8, seed 2 in RED_BABAI_FAILURE near the end of the
        # tour — every time, on any number of devices.
        attempts = []
        for seed in (1, 3, 2):
            b = g["b"].copy()
            t0 = time.perf_counter()
            st, stats = fb.bkz_reduction(b, fb.BKZParam(60, strategies="default",
                                                        flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS, max_loops=1, seed=seed),
                                         devices=devices or [local])
            attempts.append({"seed": seed, "status": int(st), "wall_seconds": time.perf_counter() - t0})
            if st == 8:
                break
        out = {"workload": "BKZ-60, 1 tour, default strategies, dim-200 knapsack (LLL-reduced latticegen r 200 2000)",
               "devices": len(devices or [local]), "attempts": attempts,
               # every attempt counts: the honest cost of one successful tour is the sum (a retry happens only when fp64
               # BKZ ends in RED_BABAI_FAILURE, which the reference's own run does for 2 of 5 seeds on this basis)
               "status": int(st), "wall_seconds": sum(a_["wall_seconds"] for a_ in attempts),
               "wall_seconds_last_attempt": attempts[-1]["wall_seconds"], "sec_lll_sizered": stats["sec_lll"],
               "sec_enum": stats["sec_enum"], "enum_nodes": int(stats["enum_nodes"]), "enum_calls": int(stats["enum_calls"]),
               "r00_before": stats["r00_before"], "r00_after": stats["r00_after"], "slope_after": stats["slope_after"]}
        from oracle import oracle as O
        if with_ref and O.have_ref():
            tmp = tempfile.mkdtemp(prefix="bench_bkz_")
            mat = os.path.join(tmp, "b.txt")
            O.write_matrix(mat, g["b"])
            cores = os.cpu_count() or 1
            ref = {}
            for th in (1, cores):
                o = O.run_ref("load %s\nbkz 60 %d 1 default enumlib %d\n" % (mat, 2 | 4, th), timeout=900)
                tok = dict(t.split("=") for t in o.split("bkz ")[-1].split() if "=" in t)
                ref["threads_%d" % th] = {"status": int(tok["status"]), "wall_seconds": float(tok["sec"])}
            out["cpu_reference"] = ref
    except Exception as ex:
        out["error"] = str(ex)[:300]
    return out


def bkz_child(ndev):
    """`bench.py --bkz-child N`: the N-device BKZ-60 tour in a process of its own (one JSON line on stdout)."""
    print(json.dumps(bkz_extras(0, devices=list(range(ndev)), with_ref=False)))
    return 0


DUMP_LIMIT = 64 << 20


def dump_outputs(path, arrays, rank=0):
    """arrays: name -> (batch, ...) float64.  Rank r > 0 writes <name>_rank<r>.npy.  Over DUMP_LIMIT bytes in all, the
    same seeded sample of lattices is taken from every array."""
    import numpy as np
    os.makedirs(path, exist_ok=True)
    total = sum(v.nbytes for v in arrays.values())
    batch = len(next(iter(arrays.values())))
    keep = None
    if total > DUMP_LIMIT:
        keep = np.sort(np.random.default_rng(0).choice(batch, batch * DUMP_LIMIT // total, replace=False))
    for name, v in arrays.items():
        v = np.asarray(v, dtype=np.float64)
        np.save(os.path.join(path, name + ("_rank%d" % rank if rank else "") + ".npy"), v if keep is None else v[keep])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--batch", type=int, default=0, help="lattices per GPU (0 = two full waves of the update kernel)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip the enumeration / Householder / BKZ figures")
    ap.add_argument("--no-bkz", action="store_true", help="skip the BKZ-60 tour (about 1.5 min GPU + 1-2 min CPU reference)")
    ap.add_argument("--bkz-child", type=int, default=0, help=argparse.SUPPRESS)
    ap.add_argument("--traffic-child", type=int, default=0, help=argparse.SUPPRESS)
    ap.add_argument("--no-traffic", action="store_true", help="skip the live ncu measurement of the kernel's DRAM traffic")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write what the timed steps computed as DIR/<name>.npy")
    a = ap.parse_args()
    if a.bkz_child:
        return bkz_child(a.bkz_child)
    if a.traffic_child:
        return traffic_child(a.traffic_child)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    def workload_str(nb):
        return ("batched {row_op_end(%d,%d); update_gso_row(%d,%d)} on %s independent dim-%d (%dx%d) int64 lattices "
                "per GPU" % (KAPPA, KAPPA + 1, KAPPA, KAPPA, nb, D, D, N_COLS))

    if a.impl == "reference":
        if rank != 0:
            return 0
        steps_v = []
        for _ in range(max(1, min(a.steps, 3))):
            steps_v.append(cpu_reference(seconds_target=8.0))
        ref = max(steps_v, key=lambda r: r["value"])
        line = {"metric": METRIC, "value": ref["value"], "unit": "GB/s", "n_gpus": a.gpus, "steps": a.steps,
                "warmup": a.warmup, "ms_per_step": None, "higher_is_better": True, "scaling": "weak",
                "vs_baseline": None, "dtype": "f64", "data": "synthetic", "impl": "reference",
                "config": {"workload": workload_str("threads*4 private"),
                           "note": "reference fplll 5.5.0 CPU path (oracle/_ref), all host threads"},
                "cpu_baseline": ref,
                "e2e": {"value": ref["value"], "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        print(json.dumps(line))
        return 0

    import ctypes as C
    import numpy as np
    import torch
    import fplll_b200 as fb
    from fplll_b200.gso import _lib, _ck
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device — the product path has no CPU fallback")
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    B = a.batch
    if B <= 0:
        # the resident-slot count depends on d, n (shared memory per warp): ask a handle of the real shape
        hp = C.c_void_p()
        _ck(_lib().b200gso_create(C.byref(hp), 1, D, N_COLS, fb.GSO_ROW_EXPO, local), "create")
        B = 2 * int(_lib().b200gso_resident_lattices(hp))
        _lib().b200gso_destroy(hp)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1234 + rank)
    dev_b = torch.randint(-(1 << 20), 1 << 20, (B, D, N_COLS), dtype=torch.int64, device="cuda", generator=gen)
    m = fb.MatGSO.__new__(fb.MatGSO)
    m.batch, m.d, m.n, m.flags, m.enable_row_expo = B, D, N_COLS, fb.GSO_ROW_EXPO, True
    m._h = C.c_void_p()
    _ck(_lib().b200gso_create(C.byref(m._h), B, D, N_COLS, fb.GSO_ROW_EXPO, local), "create")
    torch.cuda.synchronize()
    _ck(_lib().b200gso_set_basis_dev(m._h, C.c_void_p(dev_b.data_ptr())), "set_basis_dev")
    assert m.update_gso().all()  # all rows valid: the state LLL is in when it revisits kappa
    m.sync()
    del dev_b

    per_lat = alg_bytes_update_row(KAPPA, N_COLS)
    # ---- device-resident timing ---------------------------------------------------------------------------
    m.time_update_row(KAPPA, a.warmup, True)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    if dist:
        dist.barrier()
    torch.cuda.synchronize()
    ms_update, ms_total = m.time_update_row(KAPPA, a.steps, True)
    torch.cuda.synchronize()
    if dist:
        t = torch.tensor([ms_total, ms_update], device="cuda", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms_total, ms_update = float(t[0]), float(t[1])
        dist.barrier()
    value = world * B * per_lat * a.steps / (ms_total * 1e-3) / 1e9
    kern_gbps = B * per_lat / (ms_update * 1e-3) / 1e9
    dumps = {}
    if a.dump_outputs:
        mu, r, _ = m.get_mu_r_row(KAPPA)
        dumps.update(update_row_mu=mu, update_row_r=r)

    # ---- end to end through the C-ABI with host buffers ---------------------------------------------------
    # host buffers are pinned (cudaHostAlloc via torch): the C-ABI takes plain host pointers, pinned ones DMA directly
    rows = torch.randint(-(1 << 20), 1 << 20, (B, N_COLS), dtype=torch.int64,
                         generator=torch.Generator().manual_seed(4321 + rank)).pin_memory().numpy()
    out = (torch.empty((B, D), dtype=torch.float64).pin_memory().numpy(),
           torch.empty((B, D), dtype=torch.float64).pin_memory().numpy(),
           torch.empty((B,), dtype=torch.int32).pin_memory().numpy())
    def e2e_step():
        m.upload_row(KAPPA, rows)                    # H2D B*n*8, then write b[kappa] + row_op_end(kappa,kappa+1)
        m.update_gso_row(KAPPA, want_ok=False)       # stream-ordered
        mu, r, v = m.get_mu_r_row(KAPPA, out=out)    # D2H 2*B*d*8 + B*4, synchronises
        return v
    for _ in range(a.warmup):
        e2e_step()
    if dist:
        dist.barrier()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        v = e2e_step()
    torch.cuda.synchronize()
    e2e_s = time.perf_counter() - t0
    assert (v == KAPPA + 1).all()  # every lattice's row kappa is valid through the diagonal
    if a.dump_outputs:
        dumps.update(e2e_mu=out[0].copy(), e2e_r=out[1].copy())
        dump_outputs(a.dump_outputs, dumps, rank)
    if dist:
        t = torch.tensor([e2e_s], device="cuda", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        e2e_s = float(t[0])
    e2e_val = world * B * per_lat * a.steps / e2e_s / 1e9
    clocks = sampler.stop() if rank == 0 else None  # sampled across both timed regions (device-resident and e2e)
    h2d = B * N_COLS * 8
    d2h = 2 * B * D * 8 + B * 4

    # N > 1: the enumeration is the part of the path that shards — every rank walks its share of the subtree roots of
    # the same BKZ-60 block (roots r with r % world == rank), results merged with NCCL (fplll_b200/dist.py)
    enum_dist = None
    if dist and not a.no_extras:
        try:
            from fplll_b200.dist import enumerate_svp_distributed, attach_peers
            # once per job: the ranks' enumerators reach each other's radius words over NVLink (CUDA IPC handles
            # all-gathered with NCCL) — radius push inside the kernel; the subtree roots are dealt round-robin
            peers = attach_peers(device_index=local)
            z = np.load(os.path.join(ROOT, "tests", "golden", "enum_r200_b60_pruned_140.npz"))
            enumerate_svp_distributed(z["mut"], z["rdiag"], z["pruning"], float(z["maxdist"]), device_index=local)
            dist.barrier()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = enumerate_svp_distributed(z["mut"], z["rdiag"], z["pruning"], float(z["maxdist"]), device_index=local)
            torch.cuda.synchronize()
            dt = torch.tensor([time.perf_counter() - t0], device="cuda", dtype=torch.float64)
            dist.all_reduce(dt, op=dist.ReduceOp.MAX)
            n = int(res["nodes"].sum())
            enum_dist = {"workload": "SVP enumeration of a BKZ-60 block of the dim-200 basis, 8192 subtree roots dealt over "
                                     "%d ranks in order of promise, radius pushed to all peers (NVLink peer atomics over "
                                     "CUDA IPC), results merged with NCCL" % world, "peer_memory": bool(peers), "nodes": n,
                         "nodes_equal_reference": n == int(z["nodes"].sum()), "seconds_max_over_ranks": float(dt[0]),
                         "nodes_per_s": n / float(dt[0])}
        except Exception as ex:
            enum_dist = {"error": str(ex)[:300]}
    # BKZ-60 wall-seconds at N GPUs: one driver (rank 0) with GSO/LLL on its GPU and every enumeration's subtree roots
    # dealt over all N devices of the box (include/b200bkz.h: devices[]).  The other ranks wait on a CPU (gloo) barrier
    # so that no NCCL kernel sits on the GPUs rank 0 launches its cooperative enumeration kernels on.
    bkz_multi = None
    if dist and not a.no_extras and not a.no_bkz:
        cpu_group = None
        try:
            cpu_group = dist.new_group(backend="gloo")
        except Exception as ex:
            bkz_multi = {"error": "gloo group: " + str(ex)[:300]}
        if cpu_group is not None:
            try:
                if rank == 0:
                    # in a child process: a failure of the multi-device path must not take the headline line with it
                    try:
                        env = {k: v for k, v in os.environ.items()
                               if k not in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT")}
                        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--bkz-child", str(world)],
                                           capture_output=True, text=True, timeout=420, env=env)
                        lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
                        bkz_multi = json.loads(lines[-1]) if lines else {"error": "child rc %d: %s" % (
                            p.returncode, p.stderr[-300:])}
                    except Exception as ex:
                        bkz_multi = {"error": str(ex)[:300]}
            finally:
                dist.barrier(group=cpu_group)  # always reached: the other ranks are waiting in it
    traffic, traffic_src = None, None
    if rank == 0 and not a.no_traffic:
        m.close()  # the child needs the memory
        m = None
        traffic = measure_traffic(B, local)
        traffic_src = ("measured in this run: ncu dram__bytes_read.sum + dram__bytes_write.sum of one k_update_row launch "
                       "(child process)" if traffic is not None else "not measured: ncu is not usable here")
    if rank == 0:
        peak, peak_src = peaks()
        line = {"metric": METRIC, "value": value, "unit": "GB/s", "n_gpus": world, "steps": a.steps,
                "warmup": a.warmup, "ms_per_step": ms_total / a.steps, "higher_is_better": True, "scaling": "weak",
                "vs_baseline": None, "dtype": "f64", "data": "synthetic",
                "config": {"workload": workload_str(B), "batch": B, "entries": "uniform int in [-2^20, 2^20)", "flags": "GSO_ROW_EXPO",
                           "state_bytes_per_gpu": int(B * 1.39e6), "l2": "inputs larger than L2 (state >> 50 MB)",
                           "algorithmic_bytes_per_lattice": per_lat},
                "roofline": {"bound": "hbm", "kernel": "k_update_row (update_gso_row, g=1)", "achieved": kern_gbps,
                             "peak": peak, "unit": "GB/s", "frac": kern_gbps / peak, "peak_source": peak_src,
                             "traffic": traffic, "traffic_source": traffic_src,
                             "algorithmic_bytes_per_launch": B * per_lat,
                             "ms_per_launch": ms_update},
                "e2e": {"value": e2e_val, "unit": "GB/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                        "ms_per_step": e2e_s / a.steps * 1e3},
                "gpu_launches": 2 * a.steps, "clocks": clocks}
        if not a.no_extras and world > 1 and enum_dist is not None:
            line["enum"] = enum_dist
            if bkz_multi is not None:
                line["bkz60"] = bkz_multi
        if not a.no_extras and world == 1:
            line["enum"] = enum_extras(local)
            line["householder"] = hh_extras(local)
            if not a.no_bkz:
                line["bkz60"] = bkz_extras(local)
        if not a.no_cpu_baseline:
            try:
                line["cpu_baseline"] = cpu_reference()
            except Exception as ex:  # the reference build did not travel: say so, do not fake it
                line["cpu_baseline"] = {"value": None, "error": str(ex)[:200]}
        print(json.dumps(line))
    if dist:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
