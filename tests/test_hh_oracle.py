"""CPU tests (no GPU): the C restatement of MatHouseholder<long,double> (oracle/hh_oracle.c) against the UNMODIFIED
reference driven call by call through oracle/_ref/ref_probe (bit-exact; its results are stored under tests/golden), plus the reference's own test_householder
relation (tests/test_gso.cpp:101-152): mu(i,j) = R(i,j)/R(j,j) and r(i,j) = R(i,j)*R(j,j) against the GSO."""
import numpy as np
import pytest

import helpers as H
from oracle import oracle as O


HH_SEQ_CASES = [(1, 10, 10, 20), (2, 24, 30, 12), (3, 40, 40, 30)]


def hh_call_sequence(seed, d, n, bits):
    """refresh_R_bf / update_R / size_reduce (with integer + float row operations) / swap / recover_R in the order
    HLLLReduction::hlll issues them (hlll.cpp:49-171) on an UNREDUCED random basis; returns (basis, ops, rows of R
    that are defined at every dump)."""
    rng = np.random.default_rng(seed)
    b = rng.integers(-(1 << bits), 1 << bits, size=(d, n), dtype=np.int64)
    ops = [("refresh_R_bf", 0), ("update_R_last", 0), ("refresh_R_bf", 1)]
    k, kmax = 1, 1
    for step in range(3 * d):
        ops += [("update_R", k, 0), ("size_reduce", k, k, 0), ("refresh_R_bf", k), ("update_R", k, 0), ("dump",)]
        if step % 3 != 2 or k == 1:   # "Lovasz holds": finish the row and go up
            ops += [("update_R_last", k)]
            k += 1
            if k >= d:
                break
            ops += [("refresh_R_bf", k)] if k > kmax else [("refresh_R", k)]
            kmax = max(kmax, k)
        else:                           # "Lovasz fails": swap down and recover
            ops += [("swap", k - 1, k)]
            k -= 1
            ops += [("recover_R", k), ("dump",), ("set_updated_R_false",)]
    ops.append(("dump",))
    return b, ops, min(d, kmax + 1)


@pytest.mark.parametrize("seed,d,n,bits", HH_SEQ_CASES)
def test_hlll_like_call_sequence_live_vs_reference(seed, d, n, bits):
    """the call sequence of hh_call_sequence on the oracle, bit-exact against the reference's state at every dump
    (digests of the reference's dumps in tests/golden/ref_live.npz, make_golden.py --live)."""
    b, ops, rows_R = hh_call_sequence(seed, d, n, bits)
    m = O.OracleHouseholder(b, 5)
    states = []
    for op in ops:
        if op[0] == "dump":
            states.append(m.state())
        else:
            getattr(m, op[0])(*op[1:])
    want = H.gold("ref_live.npz")["hh%d_digests" % seed]
    assert len(states) == len(want) > 5
    for t, s in enumerate(states):
        assert H.hh_digest(s, rows_R) == want[t], "seed %d dump %d" % (seed, t)


def test_householder_relation_with_gso():
    """tests/test_gso.cpp:101-152: R(i,j)/R(j,j) = mu(i,j), R(i,j)*R(j,j) = r(i,j), R(i,i) > 0."""
    b = H.gold("bkz_q60.npz")["b_in"]
    d = b.shape[0]
    hh = O.OracleHouseholder(b, 0)
    for i in range(d):
        hh.refresh_R_bf(i)
        hh.update_R(i)
    R = hh.state()["R"]
    g = O.OracleGSO(b, 0)
    assert g.update_gso()
    s = g.state()
    for i in range(d):
        assert R[i, i] > 0
        for j in range(i):
            assert abs(R[i, j] / R[j, j] - s["mu"][i, j]) < 1e-9 * max(1.0, abs(s["mu"][i, j]))
            assert abs(R[i, j] * R[j, j] - s["r"][i, j]) < 1e-9 * max(1.0, abs(s["r"][i, j]))


HLLL_TAGS = ["u40", "r60", "q40", "u100", "q80"]


@pytest.mark.parametrize("tag", HLLL_TAGS)
def test_oracle_hlll_equals_reference_golden(tag):
    """ohh_hlll (the restated HLLLReduction::hlll, hlll.cpp:25-171) ends on the basis the reference's own
    HLLLReduction<long,double> produced (tests/golden/hlll_long.npz, made by make_golden.py --only-hlll)."""
    g = H.gold("hlll_long.npz")
    m = O.OracleHouseholder(g[tag + "_in"])
    st = m.hlll(0.99, 0.51, 0.001, 0.1)
    assert st == int(g[tag + "_status"]) == 0
    assert np.array_equal(m.state()["b"], g[tag + "_out"])


def test_oracle_hlll_n600_matches_reference():
    """rows of 600 columns: the reference's HLLLReduction<long,double> result is in tests/golden/size_classes_ref.npz
    (make_golden.py --sizes)."""
    z = H.gold("size_classes_ref.npz")
    m = O.OracleHouseholder(z["hlll600_in"].astype(np.int64))
    assert m.hlll(0.99, 0.51, 0.001, 0.1) == int(z["hlll600_status"]) == 0
    assert np.array_equal(m.state()["b"], z["hlll600_out"])


HLLL_LIVE_CASES = [(5, 30, 25), (6, 50, 12), (7, 70, 40)]


@pytest.mark.parametrize("seed,d,bits", HLLL_LIVE_CASES)
def test_oracle_hlll_live_vs_reference(seed, d, bits):
    """same, on seeded random bases, against the reference's status and output basis (tests/golden/ref_live.npz)."""
    rng = np.random.default_rng(seed)
    b = rng.integers(-(1 << bits), 1 << bits, size=(d, d), dtype=np.int64)
    z = H.gold("ref_live.npz")
    m = O.OracleHouseholder(b)
    assert m.hlll() == int(z["hlll%d_status" % seed])
    assert np.array_equal(m.state()["b"], z["hlll%d_out" % seed])
