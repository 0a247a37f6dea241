"""GPU tests of the BKZ driver (include/b200bkz.h: host control flow over device GSO/LLL + device enumeration)
against runs of the reference's own bkz_reduction (tests/golden/bkz_q60.npz, made by make_golden.py)."""
import numpy as np
import pytest

import helpers as H
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fb():
    import fplll_b200
    return fplll_b200


def gso_profile(b):
    m = O.OracleGSO(b, 0)
    assert m.update_gso()
    s = m.state()
    return np.array([s["r"][i, i] for i in range(b.shape[0])])


@pytest.mark.parametrize("lll_kernel", ["cta", "warp"])
def test_bkz20_without_pruning_walks_the_reference_trajectory(fb, lll_kernel, monkeypatch):
    """No pruning => no rerandomisation => BKZ is deterministic: device LLL (bit-identical to the reference's) +
    device enumeration (same best vector) must end on the SAME basis as the reference's bkz_reduction."""
    monkeypatch.setenv("B200_LLL_CTA", "1" if lll_kernel == "cta" else "0")
    z = H.gold("bkz_q60.npz")
    b = z["b_in"].copy()
    st, stats = fb.bkz_reduction(b, fb.BKZParam(20, strategies=None, flags=fb.BKZ_NO_LLL))
    assert st == int(z["bkz20_none_status"]) == 0
    assert np.array_equal(b, z["bkz20_none_b"])
    assert stats["enum_calls"] > 0 and stats["enum_nodes"] > 0


@pytest.mark.parametrize("tag,bs", [("bkz30_default", 30), ("bkz40_default", 40)])
def test_bkz_default_strategies_same_status_and_quality(fb, tag, bs):
    """strategies/default.json (pruning + preprocessing + rerandomisation): the RNG differs from the reference's GMP
    state, so compare what the reference's tests compare (status, tests/test_bkz.cpp:42-56) plus reduction quality."""
    z = H.gold("bkz_q60.npz")
    b = z["b_in"].copy()
    st, stats = fb.bkz_reduction(b, fb.BKZParam(bs, strategies="default", flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS,
                                                max_loops=2))
    assert st == int(z[tag + "_status"]) == 8  # RED_BKZ_LOOPS_LIMIT
    ref, got, inp = gso_profile(z[tag + "_b"]), gso_profile(b), gso_profile(z["b_in"])
    # same lattice: determinant preserved exactly (unimodular row operations on an int64 basis)
    assert abs(np.sum(np.log(got)) - np.sum(np.log(inp))) < 1e-6
    # first vector at least as good as LLL's and within a factor 1.5 (squared norm) of the reference's BKZ output:
    # two tours of randomised BKZ have that much run-to-run spread (the reference's own 1 vs 8 thread runs differ
    # by 1.37x, BASELINE.md §3 rows 5a/5b)
    assert got[0] <= inp[0] and got[0] <= 1.5 * ref[0], (got[0], ref[0], inp[0])
    # slope of log r_ii within 10% of the reference's
    ix = np.arange(len(got))
    s_ref, s_got = np.polyfit(ix, np.log(ref), 1)[0], np.polyfit(ix, np.log(got), 1)[0]
    assert abs(s_got - s_ref) < 0.15 * abs(s_ref), (s_got, s_ref)


def test_bkz_output_is_lll_reduced_by_the_reference_checker(fb):
    """is_lll_reduced (lll.cpp:226-258) in exact arithmetic (helpers.py), first checked against the reference's own
    verdicts on fixed bases (tests/golden/ref_islll.json), then on the device BKZ output."""
    u40, z = H.gold("u40_lll_long.npz"), H.gold("bkz_q60.npz")
    swapped = u40["b_out"].copy()
    swapped[[0, 1]] = swapped[[1, 0]]
    verdicts = H.gold_json("ref_islll.json")
    for name, basis in [("u40_b_in", u40["b_in"]), ("u40_b_out", u40["b_out"]), ("u40_b_out_rows_0_1_swapped", swapped),
                        ("q60_b_in", z["b_in"]), ("q60_bkz30_default_b", z["bkz30_default_b"])]:
        assert H.is_lll_reduced(basis, 0.99, 0.51) == bool(verdicts[name]), name
    b = z["b_in"].copy()
    st, _ = fb.bkz_reduction(b, fb.BKZParam(30, strategies="default", flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS,
                                            max_loops=1))
    assert st == 8
    assert H.is_lll_reduced(b, 0.99, 0.51)


def test_bkz_reports_a_failing_preliminary_lll_as_status(fb):
    """ADVICE r1: when the LLL that precedes BKZ (bkz.cpp:869-876) fails in fp64 — 62-bit entries at dimension 50 end in
    RED_BABAI_FAILURE, in the oracle as on the device — b200bkz_reduce must return that status, not let a C++ exception
    cross the C boundary."""
    rng = np.random.default_rng(4)
    b = rng.integers(-(1 << 62), 1 << 62, size=(50, 50), dtype=np.int64)
    assert O.OracleGSO(b).lll(0.99, 0.51)["status"] == 3
    st, stats = fb.bkz_reduction(b.copy(), fb.BKZParam(10, flags=fb.BKZ_MAX_LOOPS, max_loops=1))
    assert st == 3


def test_bkz40_on_dim180_goldstein_mayer_equals_reference(fb):
    """BASELINE config #4 at its stated size: BKZ-40 on the wrapper-LLL-reduced latticegen q 180 1 1800 p basis, one
    tour, no pruning => deterministic: the device driver must end on the reference's own output basis
    (tests/golden/bkz_gm180.npz; 57 s for the reference on one host thread)."""
    z = H.gold("bkz_gm180.npz")
    b = z["b_in"].copy()
    st, stats = fb.bkz_reduction(b, fb.BKZParam(40, flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS, max_loops=1))
    assert st == int(z["bkz40_none_status"]) == 8
    assert np.array_equal(b, z["bkz40_none_b"])


def _profile_quality(b):
    r = gso_profile(b)
    n = len(r)
    x = np.arange(n) - (n - 1) / 2
    slope = float((x * np.log(r)).sum() / (n * (n * n - 1) / 12))
    logpot = float((np.arange(n, 0, -1) * np.log(r)).sum())
    return r[0], slope, logpot


def test_bkz60_default_strategies_on_dim200_one_tour_quality(fb):
    """BASELINE config #5 at its stated size: one tour of BKZ-60 with strategies/default.json on the LLL-reduced
    latticegen r 200 2000 basis.  Pruned BKZ rerandomises (different generators here and in the reference), so the
    gate is the reference's own outcome on the same input (tests/golden/bkz60_r200_ref.npz): same status, GSO slope
    within 1 %, at least 97 % of its drop of the log-potential, and a shorter first vector than before."""
    g = H.gold("r200_lll_update_gso.npz")
    ref = H.gold("bkz60_r200_ref.npz")
    r0_in, slope_in, pot_in = _profile_quality(g["b"])
    r0_ref, slope_ref, pot_ref = _profile_quality(ref["b_out"])
    b = g["b"].copy()
    st, stats = fb.bkz_reduction(b, fb.BKZParam(60, strategies="default", flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS,
                                                max_loops=1))
    assert st == int(ref["status"]) == 8
    r0, slope, pot = _profile_quality(b)
    assert abs(slope - slope_ref) <= 0.01 * abs(slope_ref), (slope, slope_ref)
    assert pot_in - pot >= 0.97 * (pot_in - pot_ref), (pot_in, pot, pot_ref)
    assert r0 < r0_in
    # the output is still a basis of the same lattice: the Gram determinant (sum of log r_ii, ~4400 here) is unchanged up
    # to what an fp64 GSO of a dim-200 basis can resolve (its tail r_ii carry ~1e-4 relative error, SURVEY §8d)
    assert abs(np.log(gso_profile(b)).sum() - np.log(gso_profile(g["b"])).sum()) < 1.0


def test_default_tours_are_reproducible_and_the_shrinking_radius_is_a_flag(fb):
    """include/b200bkz.h: by default every SVP call enumerates the fixed region of its initial radius, so two runs of a
    pruned, rerandomising BKZ with the same seed end on the same basis, bit for bit; B200BKZ_SHRINK_RADIUS (the
    reference's order-dependent evaluator behaviour) is accepted and reduces as well."""
    z = H.gold("bkz_q60.npz")
    outs = []
    for _ in range(2):
        b = z["b_in"].copy()
        st, stats = fb.bkz_reduction(b, fb.BKZParam(30, strategies="default", flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS,
                                                    max_loops=2, seed=5))
        assert st == 8
        outs.append((b, int(stats["enum_nodes"]), int(stats["enum_calls"])))
    assert np.array_equal(outs[0][0], outs[1][0]) and outs[0][1:] == outs[1][1:]
    b = z["b_in"].copy()
    st, stats = fb.bkz_reduction(b, fb.BKZParam(30, strategies="default", max_loops=2, seed=5,
                                                flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS | fb.BKZ_SHRINK_RADIUS))
    assert st == 8 and int(stats["enum_nodes"]) <= outs[0][1]
    assert gso_profile(b)[0] <= gso_profile(z["b_in"])[0]
