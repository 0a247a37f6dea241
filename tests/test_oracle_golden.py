"""CPU tests (no GPU): the C restatement (oracle/gso_oracle.c) against the UNMODIFIED reference — committed
golden dumps always, and live through oracle/_ref/ref_probe when that build is present."""
import json

import numpy as np
import pytest

import helpers as H
from oracle import oracle as O


def _state_from_npz(z, prefix=""):
    g = lambda k: z[prefix + k]
    return dict(n_known_rows=int(g("n_known_rows")), n_known_cols=int(g("n_known_cols")),
                n_source_rows=int(g("n_source_rows")), row_expo=g("row_expo"), gso_valid_cols=g("gso_valid_cols"),
                init_row_size=g("init_row_size"), bf=g("bf"), gf=g("gf"), mu=g("mu"), r=g("r"), b=g("b"))


def test_update_gso_u40_bit_exact():
    z = H.gold("u40_update_gso.npz")
    m = O.OracleGSO(z["b"])
    assert m.update_gso()
    H.assert_state_equal(m.state(), _state_from_npz(z), "u40")


def test_ops_trace_u40_bit_exact():
    z = H.gold("u40_ops_trace.npz")
    ops = json.loads(bytes(z["ops_json"]).decode())
    marks = list(z["marks"])
    m = O.OracleGSO(z["b0"])
    t = 0
    for k, op in enumerate(ops):
        H.apply_ops(m, [tuple(op)])
        if t < len(marks) and marks[t] == k:
            H.assert_state_equal(m.state(), _state_from_npz(z, "s%d_" % t), "op %d %s" % (k, op))
            t += 1
    assert t == len(marks)


def test_update_gso_r200_bit_exact():
    z = H.gold("r200_lll_update_gso.npz")
    m = O.OracleGSO(z["b"])
    assert m.update_gso()
    s = m.state()
    tl = np.tril_indices(200)
    assert H.eq_f64(s["mu"][tl] * (tl[0] != tl[1]), z["mu_tril"] * (tl[0] != tl[1]))
    assert H.eq_f64(s["r"][tl], z["r_tril"])
    assert H.eq_f64(s["gf"][tl], z["gf_tril"])
    assert np.array_equal(s["row_expo"], z["row_expo"])


def test_lll_u40_matches_reference_basis():
    z = H.gold("u40_lll_long.npz")
    m = O.OracleGSO(z["b_in"])
    res = m.lll(0.99, 0.51)
    assert res["status"] == int(z["status"]) == 0
    assert res["n_swaps"] == int(z["n_swaps"])
    assert np.array_equal(m.state()["b"], z["b_out"])


@pytest.mark.parametrize("tag", ["lll300", "knap260"])
def test_lll_above_256_rows_matches_reference_basis(tag):
    """d = 300 uniform and a d = 260 knapsack: the reference's LLLReduction<long,double> results are in
    tests/golden/size_classes_ref.npz (make_golden.py --sizes)."""
    z = H.gold("size_classes_ref.npz")
    m = O.OracleGSO(z[tag + "_in"].astype(np.int64))
    res = m.lll(0.99, 0.51)
    assert res["status"] == int(z[tag + "_status"]) == 0
    assert res["n_swaps"] == int(z[tag + "_swaps"])
    assert np.array_equal(m.state()["b"], z[tag + "_out"])


GSO_OPS_CASES = [(1, 12, 12, 20), (2, 33, 40, 30), (3, 64, 65, 12), (4, 7, 9, 50)]


@pytest.mark.parametrize("seed,d,n,bits", GSO_OPS_CASES)
def test_random_ops_live_vs_reference(seed, d, n, bits):
    """a seeded random op script; the reference's state after it is in tests/golden/ref_live.npz (make_golden.py --live)."""
    rng = np.random.default_rng(seed)
    b = rng.integers(-(1 << bits), 1 << bits, size=(d, n), dtype=np.int64)
    ops = H.random_op_script(rng, d, 40)
    m = O.OracleGSO(b)
    H.apply_ops(m, ops)
    H.assert_state_equal(m.state(), _state_from_npz(H.gold("ref_live.npz"), "ops%d_" % seed), "seed %d" % seed)


def test_ragged_and_zero_rows_live():
    """knapsack-style identity tail (n_known_cols grows with discover_row) and an all-zero row (LLL parks it); the
    reference's two states are in tests/golden/ref_live.npz."""
    rng = np.random.default_rng(9)
    d = 10
    b = np.zeros((d, d + 1), np.int64)
    b[:, 0] = rng.integers(1, 1 << 40, size=d)
    b[np.arange(d), np.arange(d) + 1] = 1
    b[4] = 0
    z = H.gold("ref_live.npz")
    m = O.OracleGSO(b)
    for t in range(3):
        m.update_gso_row(t, t)
    H.assert_state_equal(m.state(), _state_from_npz(z, "ragged0_"), "partial")
    m.move_row(1, 9)
    H.assert_state_equal(m.state(), _state_from_npz(z, "ragged1_"), "after move_row beyond known rows")
