"""GPU parity tests of the device enumerator (through the C-ABI of include/b200enum.h) against the oracle, the
reference dumps (tests/golden/enum_*.npz) and the Leech-lattice known answer."""
import numpy as np
import pytest

import helpers as H
from oracle import oracle as O
from test_enum_oracle import gso_block

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def en():
    from fplll_b200 import enumeration as enum
    return enum


def test_unpruned_30_best_vector_equals_reference(en):
    z = H.gold("enum_r200_b30_unpruned.npz")
    res = en.enumerate_svp(z["mut"], z["rdiag"], z["pruning"], float(z["maxdist"]))
    assert res["solutions"], "no solution found"
    dist, x = res["solutions"][-1]
    assert dist * 2.0 ** int(z["normexp"]) == float(z["best"])  # identical best-vector norm (SURVEY §8d gate 3)
    assert np.array_equal(x, z["sol"]) or np.array_equal(x, -z["sol"])
    dists = [s[0] for s in res["solutions"]]
    assert dists == sorted(dists, reverse=True)  # replayed in order of improvement


def test_fixed_radius_node_counts_equal_oracle(en):
    """with a fixed radius the visited node set is order-independent: per-level counts must be IDENTICAL."""
    z = H.gold("enum_r200_b30_unpruned.npz")
    R = 0.55 * float(z["maxdist"])
    ref = O.enum_svp(z["mut"], z["rdiag"], None, R, shrink=False)
    res = en.enumerate_svp(z["mut"], z["rdiag"], None, R, fixed_radius=True)
    assert np.array_equal(res["nodes"], ref["nodes"])
    assert res["stats"]["leaves"] == ref["nsols"]
    if ref["nsols"]:
        assert res["solutions"][-1][0] == ref["best"]


def test_leech_kissing_number(en):
    """tests/test_enum.cpp:55-100: 196560 vectors of squared norm 32 inside radius 32.5 (each +-pair counted once)."""
    b = H.gold("leech_lll.npz")["b"]
    mut, rdiag = gso_block(b, 0, 24)
    res = en.enumerate_svp(mut, rdiag, None, 32.5, fixed_radius=True)
    assert res["stats"]["leaves"] == 196560 // 2
    assert abs(res["solutions"][-1][0] - 32.0) < 1e-9
    ref = O.enum_svp(mut, rdiag, None, 32.5, shrink=False)
    assert np.array_equal(res["nodes"], ref["nodes"])


def test_bkz60_block_without_solution_same_node_count_as_reference(en):
    """BASELINE config #5 size: block [140,200) of the LLL-reduced r200 basis, strategies/default.json beta=60
    pruning, radius 1.05 GH.  The reference finds nothing, so its radius never moves and its 561 045 742 visited
    nodes (18 s on one core) are a full-size known answer: the device must visit exactly the same nodes."""
    z = H.gold("enum_r200_b60_pruned_140.npz")
    assert int(z["found"]) == 0
    res = en.enumerate_svp(z["mut"], z["rdiag"], z["pruning"], float(z["maxdist"]))
    assert not res["solutions"]
    assert np.array_equal(res["nodes"], z["nodes"])
    assert int(res["nodes"].sum()) == 561045742


def test_bkz60_block_best_vector_equals_reference(en):
    """block [100,160): the reference (3.2e9 nodes, 96 s on one core) finds a vector; same norm and same vector."""
    z = H.gold("enum_r200_b60_pruned_100.npz")
    res = en.enumerate_svp(z["mut"], z["rdiag"], z["pruning"], float(z["maxdist"]))
    dist, x = res["solutions"][-1]
    assert dist * 2.0 ** int(z["normexp"]) == float(z["best"])
    assert np.array_equal(x, z["sol"]) or np.array_equal(x, -z["sol"])


def test_shards_partition_the_tree(en):
    """r % world == rank sharding (one process per GPU): the shards' node counts add up to the unsharded run."""
    z = H.gold("enum_r200_b30_unpruned.npz")
    R = 0.5 * float(z["maxdist"])
    full = en.enumerate_svp(z["mut"], z["rdiag"], None, R, fixed_radius=True)
    parts = [en.enumerate_svp(z["mut"], z["rdiag"], None, R, fixed_radius=True, shard=(r, 3)) for r in range(3)]
    assert np.array_equal(sum(p["nodes"] for p in parts), full["nodes"])
    assert sum(p["stats"]["leaves"] for p in parts) == full["stats"]["leaves"]


def test_reference_bkz_with_the_plugin_installed(tmp_path):
    """INTEGRATION.md end to end: the UNMODIFIED reference library runs its own bkz_reduction with the device
    enumerator installed through set_external_enumerator (tests/plugin_demo.cpp + fplll_extenum_adapter.cpp).
    BKZ-20 without pruning is deterministic, so the output must equal the reference's own (enumlib) output."""
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build", "plugin_demo")
    if not os.path.exists(exe):
        pytest.skip("tests/_build/plugin_demo not built (needs the reference headers)")
    z = H.gold("bkz_q60.npz")
    inp, out = str(tmp_path / "in.txt"), str(tmp_path / "out.txt")
    O.write_matrix(inp, z["b_in"])
    p = subprocess.run([exe, inp, out, "20", "2", "0", "none", "b200"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    assert "status=0" in p.stdout
    assert np.array_equal(np.array(O.read_matrix(out), dtype=np.int64), z["bkz20_none_b"])


@pytest.mark.multigpu
def test_two_devices_in_one_process_visit_the_same_nodes(en):
    """b200enum_run(devices = [0, 1]): subtree roots dealt over two GPUs of the box from ONE process (what the BKZ driver
    does with `devices`); fixed radius, so the per-level node counts must equal the oracle's.  Needs two GPUs (skipped
    on a one-GPU machine, tests/conftest.py)."""
    # a call this small stays on the first device (hand-off threshold B200_ENUM_FAN_NODES, 200 M nodes) ...
    z = H.gold("enum_r200_b30_unpruned.npz")
    R = 0.55 * float(z["maxdist"])
    ref = O.enum_svp(z["mut"], z["rdiag"], None, R, shrink=False)
    for _ in range(2):
        res = en.enumerate_svp(z["mut"], z["rdiag"], None, R, fixed_radius=True, devices=[0, 1])
        assert res["stats"]["n_devices"] == 1
        assert np.array_equal(res["nodes"], ref["nodes"])
    # ... the 5.6e8-node BKZ-60 block is handed off: both devices claim subtrees from one ticket over NVLink and the
    # fleet still visits exactly the reference's nodes
    z = H.gold("enum_r200_b60_pruned_140.npz")
    for _ in range(2):  # second call: both device contexts already exist
        res = en.enumerate_svp(z["mut"], z["rdiag"], z["pruning"], float(z["maxdist"]), devices=[0, 1])
        assert res["stats"]["n_devices"] == 2
        assert np.array_equal(res["nodes"], z["nodes"])


def test_dual_enumeration_and_subsolutions_equal_reference(en):
    """SURVEY §8 f4: the hook's dual / findsubsols requests are served on the device.  Fixed radius: per-level node
    counts equal the oracle's (pinned to the reference in tests/test_enum_oracle.py); shrinking radius: the best vector
    and the per-level sub-solutions are the reference's own (tests/golden/enum_r200_b30_dual_subsols.npz)."""
    z = H.gold("enum_r200_b30_dual_subsols.npz")
    for name, dual, subs in (("dual", True, False), ("subsols", False, True), ("dual_subsols", True, True)):
        R = float(z[name + "_maxdist"])
        ne = int(z[name + "_normexp"])
        ref = O.enum_svp_ex(z["mut"], z["rdiag"], None, 0.7 * R, shrink=False, dual=dual, findsubsols=subs)
        res = en.enumerate_svp(z["mut"], z["rdiag"], None, 0.7 * R, fixed_radius=True, dual=dual, findsubsols=subs)
        assert np.array_equal(res["nodes"], ref["nodes"]), name
        res = en.enumerate_svp(z["mut"], z["rdiag"], None, R, dual=dual, findsubsols=subs)
        dist, x = res["solutions"][-1]
        assert dist * 2.0 ** ne == float(z[name + "_best"]), name
        assert np.array_equal(x, z[name + "_sol"]) or np.array_equal(x, -z[name + "_sol"]), name
        if subs:
            # a shrinking radius changes which nodes exist below a solution, not which partial vectors are shortest
            # above the level where the radius first moved; the full-radius walk (fixed) must reproduce every level
            full = en.enumerate_svp(z["mut"], z["rdiag"], None, R, fixed_radius=True, dual=dual, findsubsols=True)
            oref = O.enum_svp_ex(z["mut"], z["rdiag"], None, R, shrink=False, dual=dual, findsubsols=True)
            for k in range(len(z["rdiag"])):
                if oref["subdist"][k] > 0:
                    assert k in full["subsolutions"], (name, k)
                    assert full["subsolutions"][k][0] == oref["subdist"][k], (name, k)
                else:
                    assert k not in full["subsolutions"], (name, k)


def test_reference_svp_known_answer_on_device(en):
    """tests/test_svp.cpp:373-374 end to end on the device: device LLL, device enumeration with radius |b_0|^2, squared
    norm of the result equals that of lattices/example_svp_out."""
    import fplll_b200 as fb
    z = H.gold("example_svp.npz")
    want = int((z["sv"].astype(object) ** 2).sum())
    b = z["b_in"].copy()
    assert fb.lll_reduction(b, 0.99, 0.51) == 0
    d = b.shape[0]
    mut, rdiag = gso_block(b, 0, d)
    res = en.enumerate_svp(mut, rdiag, None, float(rdiag[0]))
    best = int((b[0].astype(object) ** 2).sum())
    if res["solutions"]:
        v = np.rint(res["solutions"][-1][1]).astype(np.int64) @ b
        best = min(best, int((v.astype(object) ** 2).sum()))
    assert best == want
