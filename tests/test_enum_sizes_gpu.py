"""GPU tests of the device enumerator in every size class up to B200ENUM_MAX_DIM = 160 against the oracle and the
reference's own enumerator (tests/golden/enum_size_classes.npz, made by make_golden.py --enum-sizes).

The size classes: the shared-memory walker serves d <= 64 (k_enum<64, true>), the thread-local walker d <= 64 with
sub-solutions (k_enum<64, false>) and every call with 65 <= d <= 160 (k_enum<160, false>).  The host breadth phase
expands the top levels into at most 2^15 subtree roots, each staged with a (d + 3) & ~3 int prefix row.  With a fixed
radius the set of visited nodes does not depend on the walkers' schedule, so the per-level node counts must equal the
oracle's exactly.  The real inputs are blocks [200 - d, 200) of the LLL-reduced r200 basis, with radii chosen so that
each oracle walk visits about 2e5-2e6 nodes."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
from oracle import oracle as O
from test_enum_oracle import gso_block

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def en():
    from fplll_b200 import enumeration as enum
    return enum


def gh2(rdiag):
    """squared Gaussian heuristic of a block with squared GSO norms rdiag"""
    n = len(rdiag)
    return math.exp((2.0 / n) * math.lgamma(n / 2 + 1)) / math.pi * math.exp(np.sum(np.log(rdiag)) / n)


def r200_block(d):
    return gso_block(H.gold("r200_lll_update_gso.npz")["b"], 200 - d, 200)


def strategy_pruning(d):
    """the beta = d coefficients of strategies/default.json for the GH factor 1.0"""
    z = np.load(os.path.join(ROOT, "fplll_b200", "data", "strategies_default.npz"))
    return np.ascontiguousarray(z["coef_%d" % d][int(np.argmin(np.abs(z["ghf_%d" % d] - 1.0)))], np.float64)


# fixed radius = factor * gh2(block) (primal) or factor * gh2(1 / rdiag) (dual); d <= 5: 4 * r(0, 0)
PRIMAL_F = {63: 0.182, 64: 0.182, 65: 0.16, 80: 0.0669, 100: 0.0246, 128: 0.00548, 160: 0.00112}
DUAL_F = {65: 0.164, 100: 0.0202, 160: 0.000865}
PRUNED_F = {65: 0.552, 80: 0.319, 100: 0.128}


def primal_case(d):
    mut, rdiag = r200_block(d)
    return mut, rdiag, (4.0 * rdiag[0] if d <= 5 else PRIMAL_F[d] * gh2(rdiag))


def check_fixed(en, mut, rdiag, prun, R, dual=False, findsubsols=False, min_nodes=0):
    """device vs oracle with a fixed radius: per-level nodes, leaves, best distance; returns both results"""
    ref = O.enum_svp_ex(mut, rdiag, prun, R, shrink=False, dual=dual, findsubsols=findsubsols)
    res = en.enumerate_svp(mut, rdiag, prun, R, fixed_radius=True, dual=dual, findsubsols=findsubsols)
    assert int(ref["nodes"].sum()) >= min_nodes
    assert np.array_equal(res["nodes"], ref["nodes"])
    assert res["stats"]["leaves"] == ref["nsols"]
    if ref["nsols"]:
        assert res["solutions"][-1][0] == ref["best"]
    else:
        assert not res["solutions"]
    return res, ref


@pytest.mark.parametrize("d", [2, 3, 5, 63, 64, 65, 80, 100, 128, 160])
def test_fixed_radius_primal_equals_oracle(en, d):
    mut, rdiag, R = primal_case(d)
    check_fixed(en, mut, rdiag, None, R, min_nodes=2 if d <= 5 else 100000)


@pytest.mark.parametrize("d", [65, 100, 160])
def test_fixed_radius_dual_equals_oracle(en, d):
    mut, rdiag = r200_block(d)
    check_fixed(en, mut, rdiag, None, DUAL_F[d] * gh2(1.0 / rdiag), dual=True, min_nodes=100000)


@pytest.mark.parametrize("d", [65, 160])
def test_subsolutions_equal_oracle(en, d):
    """per level, the shortest partial vector of the full-radius walk: its length and its coefficients"""
    mut, rdiag, R = primal_case(d)
    res, ref = check_fixed(en, mut, rdiag, None, R, findsubsols=True, min_nodes=100000)
    assert (ref["subdist"] > 0).sum() > 10
    for k in range(d):
        if ref["subdist"][k] > 0:
            assert k in res["subsolutions"], k
            dist, x = res["subsolutions"][k]
            assert dist == ref["subdist"][k], k
            assert np.array_equal(x, ref["subsol"][k]), k
        else:
            assert k not in res["subsolutions"], k


@pytest.mark.parametrize("d", [65, 80, 100])
def test_fixed_radius_pruned_equals_oracle(en, d):
    mut, rdiag = r200_block(d)
    check_fixed(en, mut, rdiag, strategy_pruning(d), PRUNED_F[d] * gh2(rdiag), min_nodes=100000)


@pytest.mark.parametrize("name,dual,subs", [("p80", False, False), ("dual80", True, False), ("subsols80", False, True)])
def test_shrinking_radius_best_vector_equals_reference(en, name, dual, subs):
    """unpruned d = 80 with a planted shortest vector: the radius shrinks on the way, and the best vector is the
    oracle's and the reference's (up to sign); the sub-solution walk also gives the reference's per-level lengths"""
    z = H.gold("enum_size_classes.npz")
    mut, rdiag, R, ne = z[name + "_mut"], z[name + "_rdiag"], float(z[name + "_maxdist"]), int(z[name + "_normexp"])
    ref = O.enum_svp_ex(mut, rdiag, None, R, shrink=True, dual=dual, findsubsols=subs)
    res = en.enumerate_svp(mut, rdiag, None, R, dual=dual, findsubsols=subs)
    assert res["solutions"], name
    dist, x = res["solutions"][-1]
    assert dist == ref["best"] and dist * 2.0 ** ne == float(z[name + "_best"]), name
    assert np.array_equal(x, z[name + "_sol"]) or np.array_equal(x, -z[name + "_sol"]), name
    assert np.array_equal(x, ref["sol"]) or np.array_equal(x, -ref["sol"]), name
    if subs:
        # the shrinking radius moved only at the final leaf: every level's shortest partial vector is the reference's
        want = z[name + "_subdist"]
        for k in range(len(rdiag)):
            if want[k] > 0:
                assert res["subsolutions"][k][0] * 2.0 ** ne == want[k], k
                assert np.array_equal(res["subsolutions"][k][1], z[name + "_subsol"][k]), k


@pytest.mark.parametrize("name", ["p100", "p160"])
def test_pruned_fixture_walks_equal_reference(en, name):
    """the reference found nothing in these pruned walks, so its radius never moved: fixed or shrinking, the device
    must visit exactly its nodes"""
    z = H.gold("enum_size_classes.npz")
    assert int(z[name + "_found"]) == 0
    args = (z[name + "_mut"], z[name + "_rdiag"], z[name + "_pruning"], float(z[name + "_maxdist"]))
    for fixed in (True, False):
        res = en.enumerate_svp(*args, fixed_radius=fixed)
        assert np.array_equal(res["nodes"], z[name + "_nodes"]), fixed
        assert not res["solutions"]


@pytest.mark.parametrize("name", ["p100", "p160"])
def test_shards_partition_the_tree_above_64(en, name):
    """r % 3 == rank sharding at d = 100 and 160: the shards' node counts add up to the unsharded run's, the oracle's and
    the reference's"""
    z = H.gold("enum_size_classes.npz")
    args = (z[name + "_mut"], z[name + "_rdiag"], z[name + "_pruning"], float(z[name + "_maxdist"]))
    full = en.enumerate_svp(*args, fixed_radius=True)
    parts = [en.enumerate_svp(*args, fixed_radius=True, shard=(r, 3)) for r in range(3)]
    assert all(p["nodes"].sum() > 0 for p in parts)
    assert np.array_equal(sum(p["nodes"] for p in parts), full["nodes"])
    assert np.array_equal(full["nodes"], O.enum_svp(*args, shrink=False)["nodes"])
    assert np.array_equal(full["nodes"], z[name + "_nodes"])


_CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from fplll_b200 import enumeration as en
z = np.load(sys.argv[2])
res = en.enumerate_svp(z["mut"], z["rdiag"], None, float(z["R"]), fixed_radius=True)
print(json.dumps([int(v) for v in res["nodes"]]))
"""


@pytest.mark.parametrize("d", [63, 64])
def test_both_walkers_at_the_boundary(en, d, tmp_path):
    """d = 63 and 64 take the shared-memory walker; B200_ENUM_XS=0 (read once per process, hence the subprocess) makes
    them take the thread-local one: both must visit the oracle's nodes"""
    mut, rdiag, R = primal_case(d)
    onodes = O.enum_svp(mut, rdiag, None, R, shrink=False)["nodes"]
    assert np.array_equal(en.enumerate_svp(mut, rdiag, None, R, fixed_radius=True)["nodes"], onodes)
    f = str(tmp_path / "in.npz")
    np.savez(f, mut=mut, rdiag=rdiag, R=np.float64(R))
    env = dict(os.environ, B200_ENUM_XS="0")
    p = subprocess.run([sys.executable, "-c", _CHILD, ROOT, f], capture_output=True, text=True, env=env, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    assert np.array_equal(np.array(json.loads(p.stdout.strip().splitlines()[-1]), dtype=np.uint64), onodes)


def wide_top(d, top):
    """mu = 0, r = 1 except r(d-1, d-1) = 1 / top^2, radius 1: level d-1 has `top` candidates x = 1 .. top, and below
    each of them only x = 0 fits, so the walk is about top * d nodes"""
    rdiag = np.ones(d)
    rdiag[-1] = 1.0 / float(top) ** 2
    return np.zeros((d, d)), rdiag


@pytest.mark.parametrize("d,top", [(6, 100000), (100, 40000), (160, 16000)])
def test_wide_top_level_equals_oracle(en, d, top):
    """more top-level candidates than the 2^15 subtree roots the breadth phase stages (d = 6, 100), and 16 000 roots
    with 160-wide prefix rows (d = 160): every candidate is walked"""
    mut, rdiag = wide_top(d, top)
    res, ref = check_fixed(en, mut, rdiag, None, 1.0)
    assert int(ref["nodes"][d - 1]) == top
    assert res["stats"]["n_roots"] >= min(top, 1 << 15)
    # shrinking radius: the shortest vector is x = e_{d-1}
    res = en.enumerate_svp(mut, rdiag, None, 1.0)
    dist, x = res["solutions"][-1]
    assert dist == rdiag[-1] and np.array_equal(np.abs(x), np.eye(d)[d - 1])


def test_wide_second_level_sharded_equals_oracle(en):
    """d = 80: 101 candidates at level 79 and about 27 000 at level 78 — the breadth phase stages level 78 both for an
    unsharded call and for a sharded one (8192 roots wanted); the shards add up to the oracle's nodes"""
    d = 80
    mut, rdiag = np.zeros((d, d)), np.ones(d)
    rdiag[-1], rdiag[-2] = 1e-4, 3.38e-5
    ref = O.enum_svp(mut, rdiag, None, 1.0, shrink=False)
    full = en.enumerate_svp(mut, rdiag, None, 1.0, fixed_radius=True)
    assert full["stats"]["top_levels"] == 2 and full["stats"]["n_roots"] > 25000
    assert np.array_equal(full["nodes"], ref["nodes"]) and full["stats"]["leaves"] == ref["nsols"]
    parts = [en.enumerate_svp(mut, rdiag, None, 1.0, fixed_radius=True, shard=(r, 3)) for r in range(3)]
    assert np.array_equal(sum(p["nodes"] for p in parts), ref["nodes"])
    assert sum(p["stats"]["leaves"] for p in parts) == ref["nsols"]


@pytest.mark.parametrize("d,maxdist", [(1, 1.0), (161, 1.0), (30, 0.0), (30, -1.0), (30, float("nan"))])
def test_refusals(en, d, maxdist):
    from fplll_b200 import B200Error
    mut, rdiag = np.zeros((d, d)), np.ones(d)
    with pytest.raises(B200Error, match="bad arguments"):
        en.enumerate_svp(mut, rdiag, None, maxdist)
