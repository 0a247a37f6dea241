"""CPU tests (no GPU) for self-dual BKZ / slide reduction: the oracle's dual enumeration on the full-size d = 60 block
against the reference's recorded walk, the flag values of the Python API against include/b200bkz.h, and the driver's
slide potential (slide reduction's termination test) against a restatement of get_slide_potential."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import helpers as H
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_dual_walk_at_d60_pruned_equals_reference():
    """block [140, 200) of the LLL-reduced r200 basis, beta = 60 pruning vector, radius delta / r(199, 199): the oracle's
    dual Schnorr-Euchner walk with a shrinking radius visits the reference's nodes, level by level, and ends on the
    reference's vector (tests/golden/bkz_sd_sld.npz, recorded by make_sdbkz_golden.py)."""
    z = H.gold("bkz_sd_sld.npz")
    assert int(z["dual60_found"]) == 1
    res = O.enum_svp_ex(z["dual60_mut"], z["dual60_rdiag"], z["dual60_pruning"], float(z["dual60_maxdist"]),
                        shrink=True, dual=True)
    assert np.array_equal(res["nodes"], z["dual60_nodes"])
    assert res["best"] * 2.0 ** int(z["dual60_normexp"]) == float(z["dual60_best"])
    assert np.array_equal(res["sol"], z["dual60_sol"]) or np.array_equal(res["sol"], -z["dual60_sol"])


def test_python_flag_values_equal_the_header():
    import fplll_b200 as fb
    hdr = open(os.path.join(ROOT, "include", "b200bkz.h")).read()
    val = lambda name: int(re.search(r"#define B200BKZ_%s (0x[0-9a-fA-F]+|\d+)" % name, hdr).group(1), 0)
    assert fb.BKZ_SD_VARIANT == val("SD_VARIANT") == 0x100  # defs.h:273
    assert fb.BKZ_SLD_RED == val("SLD_RED") == 0x200        # defs.h:274
    for name in ("VERBOSE", "NO_LLL", "MAX_LOOPS", "MAX_TIME", "BOUNDED_LLL", "AUTO_ABORT", "GH_BND"):
        assert getattr(fb, "BKZ_" + name) == val(name), name


def slide_potential(rmant, rexpo, start_row, end_row, block_size):
    """get_slide_potential, gso_interface.cpp:244-258, over get_log_det (:230-242): sum over the first p blocks of
    (p - i) * log det(block i), p the number of blocks less one when block_size divides the range."""
    p = (end_row - start_row) // block_size
    if (end_row - start_row) % block_size == 0:
        p -= 1
    potential = 0.0
    for i in range(p):
        log_det = 0.0
        for k in range(i * block_size, (i + 1) * block_size):
            log_det += math.log(math.ldexp(float(rmant[k]), int(rexpo[k])))
        potential += float(p - i) * log_det
    return potential


def test_driver_slide_potential_equals_the_restatement():
    """b200bkz_slide_potential_of (what slide_tour compares tour to tour) on the stored r diagonal of the LLL-reduced r200
    basis (mantissas with GSO_ROW_EXPO exponents): bit-identical to the restatement, for divisible and ragged block
    counts, and the p / remainder rule itself on a hand-checked case."""
    lp = os.path.join(ROOT, "fplll_b200", "lib", "libb200bkz.so")
    if not os.path.exists(lp):
        pytest.skip("libb200bkz.so not built")
    L = C.CDLL(lp)
    f = L.b200bkz_slide_potential_of
    f.restype = C.c_double
    f.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_long), C.c_int, C.c_int, C.c_int]
    g = H.gold("r200_lll_update_gso.npz")
    d = 200
    R = np.zeros((d, d))
    R[np.tril_indices(d)] = g["r_tril"]
    mant = np.ascontiguousarray(np.diag(R), np.float64)
    expo = np.ascontiguousarray(2 * g["row_expo"].astype(np.int64), np.int64)
    P = C.POINTER
    for bs in (20, 30, 60, 64, 199, 200):
        got = f(mant.ctypes.data_as(P(C.c_double)), expo.ctypes.data_as(P(C.c_long)), 0, d, bs)
        assert got == slide_potential(mant, expo, 0, d, bs), bs
    # 7 rows, blocks of 3: p = 2 (the ragged last block is left out); 6 rows, blocks of 3: p = 1
    m = np.ascontiguousarray(np.exp(np.arange(1.0, 8.0)), np.float64)
    e = np.zeros(7, np.int64)
    want7 = 2 * (1 + 2 + 3) + 1 * (4 + 5 + 6)
    assert abs(f(m.ctypes.data_as(P(C.c_double)), e.ctypes.data_as(P(C.c_long)), 0, 7, 3) - want7) < 1e-12
    assert abs(f(m.ctypes.data_as(P(C.c_double)), e.ctypes.data_as(P(C.c_long)), 0, 6, 3) - 6) < 1e-12
