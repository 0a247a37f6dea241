"""SURVEY §8(d) micro-benchmarks M1 / M2 / M3 of the device GSO (run on an H100:  python tools/microbench.py > out.txt).

  M1  per-call update_gso_row(i, i), i in {39, 199, 399}, Gram row invalid (g=1) and valid (g=0): one lattice (the
      latency of a single call, what a per-call forwarder would pay) and a full batch (2 x resident warps).
  M2  whole-matrix update_gso() (all rows, Gram invalid) at d in {200, 400, 768} (the per-warp shared-memory scratch of this layout ends near d = 900), batch sized to fill the GPU.
      Algorithmic bytes = 8 * (d*n + 3*d*(d+1)/2) per lattice (read bf once, write gf, mu, r once).
  M3  batched update_gso() of 64..1024 independent d=60 blocks (the BKZ preprocessing pattern).
All inputs: uniform integers in [-2^20, 2^20) from numpy's seeded generator; timing by CUDA events on the handle's
stream (M1) or wall clock around a synchronising call (M2/M3, milliseconds and up)."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from fplll_b200.gso import MatGSO, GSO_ROW_EXPO  # noqa: E402


def tri(i):
    return i * (i + 1) // 2


def row_bytes(i, n, g):
    # SURVEY §8 (a2): mu rows < i (packed triangle) + r(i,.), mu(i,.) written; g=1 adds bf rows 0..i and gf(i,.)
    return 8 * (tri(i) + 2 * (i + 1)) + (8 * ((i + 1) * n + (i + 1)) if g else 0)


def rand_basis(rng, batch, d, n):
    return rng.integers(-(1 << 20), 1 << 20, size=(batch, d, n), dtype=np.int64)


def main():
    rng = np.random.default_rng(1)
    out = {"M1": [], "M2": [], "M3": []}
    # ---- M1 ----
    for d, i in ((40, 39), (200, 199), (400, 399)):
        n = d + 1 if d == 200 else d
        for batch in (1, None):
            m = MatGSO(rand_basis(rng, 1, d, n), GSO_ROW_EXPO)
            B = 1 if batch == 1 else 2 * m.resident_lattices()
            m.close()
            if B * (d * n * 16 + tri(d) * 24) > 60e9:
                B = int(60e9 // (d * n * 16 + tri(d) * 24))
            m = MatGSO(rand_basis(rng, B, d, n), GSO_ROW_EXPO)
            assert m.update_gso().all()
            for g in (1, 0):
                m.time_update_row(i, 3, bool(g))
                ms, _ = m.time_update_row(i, 20, bool(g))
                rec = dict(d=d, n=n, i=i, g=g, batch=B, us_per_launch=1e3 * ms, algorithmic_bytes_per_lattice=row_bytes(i, n, g),
                           GBps=B * row_bytes(i, n, g) / (ms * 1e-3) / 1e9)
                out["M1"].append(rec)
                print("M1", json.dumps(rec), flush=True)
            m.close()
    # ---- M2 ----
    for d, B in ((200, 5920), (400, 2960), (768, 592)):
        n = d + 1 if d == 200 else d
        m = MatGSO(rand_basis(rng, B, d, n), GSO_ROW_EXPO)
        m.discover_all_rows()
        m.sync()
        t = time.perf_counter()
        ok = m.update_gso()
        dt = time.perf_counter() - t
        assert ok.all()
        by = 8 * (d * n + 3 * tri(d))
        rec = dict(d=d, n=n, batch=B, seconds=dt, algorithmic_bytes_per_lattice=by, GBps=B * by / dt / 1e9,
                   lattices_per_s=B / dt)
        out["M2"].append(rec)
        print("M2", json.dumps(rec), flush=True)
        m.close()
        if True:  # blocked Gram (gso_gram.cuh): 0 = ordered, 1 = DMMA
            for mode in (0, 1):
                m = MatGSO(rand_basis(rng, B, d, n), GSO_ROW_EXPO)
                m.sync()
                t = time.perf_counter()
                ok = m.update_gso_blocked(mode)
                dt = time.perf_counter() - t
                rec = dict(d=d, n=n, batch=B, gram_mode=mode, seconds=dt, GBps=B * by / dt / 1e9, ok=bool(ok.all()))
                print("M2-blocked", json.dumps(rec), flush=True)
                m.close()
    # ---- M3 ----
    for B in (64, 256, 1024, 5920):
        d = n = 60
        m = MatGSO(rand_basis(rng, B, d, n), GSO_ROW_EXPO)
        m.discover_all_rows()
        m.sync()
        t = time.perf_counter()
        ok = m.update_gso()
        dt = time.perf_counter() - t
        assert ok.all()
        by = 8 * (d * n + 3 * tri(d))
        rec = dict(d=d, batch=B, us=1e6 * dt, algorithmic_bytes_per_lattice=by, GBps=B * by / dt / 1e9, blocks_per_s=B / dt)
        out["M3"].append(rec)
        print("M3", json.dumps(rec), flush=True)
        m.close()


if __name__ == "__main__":
    main()
