"""CPU tests (no GPU): the C restatement of the Schnorr-Euchner walk (oracle/enum_oracle.c) against dumps of the
reference's own enumerator taken through its plugin API (tests/golden/enum_*.npz, made by make_golden.py) and the
Leech-lattice known answer of the reference's tests/test_enum.cpp:55-100."""
import numpy as np

import helpers as H
from oracle import oracle as O


def gso_block(b, first, last):
    """mut / rdiag of a basis block from the oracle GSO (no row_expo: true mu, r)."""
    m = O.OracleGSO(b, 0)
    assert m.update_gso()
    s = m.state()
    d = last - first
    mut = np.zeros((d, d))
    for k in range(d):
        for j in range(k + 1, d):
            mut[k, j] = s["mu"][first + j, first + k]
    rdiag = np.array([s["r"][first + i, first + i] for i in range(d)])
    return mut, rdiag


def test_oracle_matches_reference_unpruned_30():
    z = H.gold("enum_r200_b30_unpruned.npz")
    res = O.enum_svp(z["mut"], z["rdiag"], z["pruning"], float(z["maxdist"]), shrink=True)
    assert np.array_equal(res["nodes"], z["nodes"])  # per level, bit-identical pruning decisions
    assert res["best"] * 2.0 ** int(z["normexp"]) == float(z["best"])
    assert np.array_equal(res["sol"], z["sol"])


def test_leech_kissing_number():
    b = H.gold("leech_lll.npz")["b"]
    mut, rdiag = gso_block(b, 0, 24)
    res = O.enum_svp(mut, rdiag, None, 32.5, shrink=False)
    assert res["nsols"] == 196560 // 2  # +-v counted once (SVP symmetry break, enumerate_base.h:145-171)
    assert abs(res["best"] - 32.0) < 1e-9


def test_reference_svp_known_answer():
    """tests/test_svp.cpp:54-100,373-374: after LLL, the shortest vector of lattices/example_svp_in has the squared norm
    of lattices/example_svp_out.  Oracle LLL + oracle enumeration (radius = |b_0|^2, as shortest_vector does)."""
    z = H.gold("example_svp.npz")
    want = int((z["sv"].astype(object) ** 2).sum())
    m = O.OracleGSO(z["b_in"])
    assert m.lll(0.99, 0.51)["status"] == 0
    b = m.state()["b"]
    d = b.shape[0]
    mut, rdiag = gso_block(b, 0, d)
    res = O.enum_svp(mut, rdiag, None, float(rdiag[0]), shrink=True)
    best = int((b[0].astype(object) ** 2).sum())
    if res["nsols"]:
        v = np.rint(res["sol"]).astype(np.int64) @ b
        best = min(best, int((v.astype(object) ** 2).sum()))
    assert best == want


def test_oracle_dual_and_subsolutions_match_reference():
    """SURVEY §8 f4: the dual SVP walk (chains over alpha, reversed inverted basis, enumerate.cpp:100-124) and the
    per-level sub-solutions (enumerate_base.cpp:36-40) of the reference's own enumerator on block [140,170) of the
    LLL-reduced r200 basis (tests/golden/enum_r200_b30_dual_subsols.npz, made by make_golden.py --dual)."""
    z = H.gold("enum_r200_b30_dual_subsols.npz")
    for name, dual, subs in (("primal", False, False), ("dual", True, False), ("subsols", False, True),
                             ("dual_subsols", True, True)):
        res = O.enum_svp_ex(z["mut"], z["rdiag"], None, float(z[name + "_maxdist"]), dual=dual, findsubsols=subs)
        ne = int(z[name + "_normexp"])
        assert np.array_equal(res["nodes"], z[name + "_nodes"]), name
        assert res["best"] * 2.0 ** ne == float(z[name + "_best"]), name
        assert np.array_equal(res["sol"], z[name + "_sol"]), name
        if subs:
            assert np.array_equal(np.where(res["subdist"] > 0, res["subdist"] * 2.0 ** ne, -1.0), z[name + "_subdist"])
            assert np.array_equal(res["subsol"], z[name + "_subsol"])


ENUM_SIZE_CASES = (("p80", False, False), ("dual80", True, False), ("subsols80", False, True), ("p100", False, False),
                   ("p160", False, False))


def test_oracle_matches_reference_above_64_dimensions():
    """The reference's own enumerator on blocks of 80, 100 and 160 dimensions (tests/golden/enum_size_classes.npz, made
    by make_golden.py --enum-sizes): unpruned primal, dual and sub-solution walks that find a planted shortest vector at
    d = 80, and pruned walks at d = 100 (beta = 100 strategy coefficients) and d = 160 (linear profile)."""
    z = H.gold("enum_size_classes.npz")
    for name, dual, subs in ENUM_SIZE_CASES:
        res = O.enum_svp_ex(z[name + "_mut"], z[name + "_rdiag"], z[name + "_pruning"], float(z[name + "_maxdist"]),
                            dual=dual, findsubsols=subs)
        ne = int(z[name + "_normexp"])
        assert len(res["nodes"]) == len(z[name + "_rdiag"]) > 64, name
        assert np.array_equal(res["nodes"], z[name + "_nodes"]), name
        assert (res["nsols"] > 0) == bool(z[name + "_found"]), name
        if res["nsols"]:
            assert res["best"] * 2.0 ** ne == float(z[name + "_best"]), name
            assert np.array_equal(res["sol"], z[name + "_sol"]), name
        if subs:
            assert np.array_equal(np.where(res["subdist"] > 0, res["subdist"] * 2.0 ** ne, -1.0), z[name + "_subdist"])
            assert np.array_equal(res["subsol"], z[name + "_subsol"])
            assert (z[name + "_subdist"] > 0).sum() > 10
