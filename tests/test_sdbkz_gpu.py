"""GPU tests of self-dual BKZ (BKZ_SD_VARIANT) and slide reduction (BKZ_SLD_RED) on the device BKZ driver, and of dual
enumeration in the shared-memory enumeration walker, against runs of the reference (tests/golden/bkz_sd_sld.npz, made by
make_sdbkz_golden.py) and the CPU oracle."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
from oracle import oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = os.path.join(ROOT, "tests", "_build", "libb200fplll.so")
REF = os.path.join(ROOT, "oracle", "_ref")


@pytest.fixture(scope="module")
def fb():
    import fplll_b200
    return fplll_b200


@pytest.fixture(scope="module")
def gold():
    return H.gold("bkz_sd_sld.npz")


def _dual_cases(gold):
    """(name, mut, rdiag, pruning, fixed radius, oracle fixed-radius nodes or None, shrinking radius, best, sol, normexp)"""
    z30 = H.gold("enum_r200_b30_dual_subsols.npz")
    R30 = float(z30["dual_maxdist"])
    yield ("d30", z30["mut"], z30["rdiag"], None, 0.7 * R30, None, R30, float(z30["dual_best"]), z30["dual_sol"],
           int(z30["dual_normexp"]))
    g = gold
    yield ("d40", g["dual40_mut"], g["dual40_rdiag"], None, float(g["dual40_fixed_R"]), g["dual40_fixed_nodes"],
           float(g["dual40_maxdist"]), float(g["dual40_best"]), g["dual40_sol"], 0)
    yield ("d60", g["dual60_mut"], g["dual60_rdiag"], g["dual60_pruning"], float(g["dual60_fixed_R"]),
           g["dual60_fixed_nodes"], float(g["dual60_maxdist"]), float(g["dual60_best"]), g["dual60_sol"],
           int(g["dual60_normexp"]))


_CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from fplll_b200 import enumeration as en
z = np.load(sys.argv[2])
pr = z["pruning"] if "pruning" in z.files else None
res = en.enumerate_svp(z["mut"], z["rdiag"], pr, float(z["R"]), fixed_radius=True, dual=True)
print(json.dumps([int(v) for v in res["nodes"]]))
"""


def _thread_local_nodes(tmp_path, name, mut, rdiag, prun, R):
    """fixed-radius dual node counts of the thread-local kernel variant (B200_ENUM_XS=0 is read once per process)"""
    f = str(tmp_path / ("%s.npz" % name))
    extra = {} if prun is None else {"pruning": prun}
    np.savez(f, mut=mut, rdiag=rdiag, R=np.float64(R), **extra)
    env = dict(os.environ, B200_ENUM_XS="0")
    p = subprocess.run([sys.executable, "-c", _CHILD, ROOT, f], capture_output=True, text=True, env=env, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    return np.array(json.loads(p.stdout.strip().splitlines()[-1]), dtype=np.uint64)


def test_dual_enumeration_in_the_shared_memory_walker_equals_reference(gold, tmp_path):
    """d = 30, 40 (unpruned) and 60 (the beta = 60 pruning vector): with a fixed radius, the per-level node counts of the
    shared-memory walker (dim <= 64 takes it) equal the oracle's and the thread-local variant's; with the shrinking
    radius, the best dual vector is the reference's (d = 30, 60) or the oracle's (d = 40), up to sign."""
    from fplll_b200 import enumeration as en
    for name, mut, rdiag, prun, Rf, onodes, Rs, best, sol, ne in _dual_cases(gold):
        if onodes is None:
            onodes = O.enum_svp_ex(mut, rdiag, prun, Rf, shrink=False, dual=True)["nodes"]
        res = en.enumerate_svp(mut, rdiag, prun, Rf, fixed_radius=True, dual=True)
        assert np.array_equal(res["nodes"], onodes), name
        assert int(onodes.sum()) > 1000, name  # a walk big enough to be spread over many walkers
        assert np.array_equal(_thread_local_nodes(tmp_path, name, mut, rdiag, prun, Rf), onodes), name
        res = en.enumerate_svp(mut, rdiag, prun, Rs, dual=True)
        assert res["solutions"], name
        dist, x = res["solutions"][-1]
        assert dist * 2.0 ** ne == best, (name, dist, best)
        assert np.array_equal(x, sol) or np.array_equal(x, -sol), name


@pytest.mark.parametrize("lll_kernel", ["cta", "warp"])
@pytest.mark.parametrize("tag", ["sd20_none", "sld20_none", "sld20_bounded_none"])
def test_unpruned_sd_and_slide_walk_the_reference_trajectory(fb, gold, tag, lll_kernel, monkeypatch):
    """No pruning => no rerandomisation => deterministic: device LLL (bit-identical) + device primal and dual
    enumeration (the reference's vectors) must end on the reference's own output basis, for both LLL kernels."""
    monkeypatch.setenv("B200_LLL_CTA", "1" if lll_kernel == "cta" else "0")
    b = H.gold("bkz_q60.npz")["b_in"].copy()
    st, stats = fb.bkz_reduction(b, fb.BKZParam(20, strategies=None, flags=int(gold[tag + "_flags"]), max_loops=2))
    assert st == int(gold[tag + "_status"])
    assert np.array_equal(b, gold[tag + "_b"])
    assert stats["enum_calls"] > 0
    assert H.is_lll_reduced(b, 0.99, 0.51)


def test_sd_bkz40_on_dim180_equals_reference(fb, gold):
    """one SD-BKZ-40 loop (dual tour + primal tour + the closing hkz of the last window) on the dim-180
    Goldstein-Mayer basis, no pruning: the reference's output basis."""
    b = H.gold("bkz_gm180.npz")["b_in"].copy()
    st, _ = fb.bkz_reduction(b, fb.BKZParam(40, flags=int(gold["gm180_sd40_none_flags"]), max_loops=1))
    assert st == int(gold["gm180_sd40_none_status"])
    assert np.array_equal(b, gold["gm180_sd40_none_b"])


def _quality(b):
    m = O.OracleGSO(b, 0)
    assert m.update_gso()
    s = m.state()
    r = np.array([s["r"][i, i] for i in range(b.shape[0])])
    n = len(r)
    x = np.arange(n) - (n - 1) / 2
    return r, float((x * np.log(r)).sum() / (n * (n * n - 1) / 12)), float((np.arange(n, 0, -1) * np.log(r)).sum())


@pytest.mark.parametrize("tag", ["sd30_default", "sld30_default"])
def test_default_strategies_same_status_and_quality(fb, gold, tag):
    """strategies/default.json (pruning, preprocessing, rerandomisation): the generator differs from the reference's GMP
    state, so the gates are the reference's status, its GSO slope within 10 %, 90 % of its drop of the log-potential, a
    first vector no longer than LLL's, the same lattice, and two runs with one seed ending on the same basis."""
    z = H.gold("bkz_q60.npz")
    outs = []
    for _ in range(2):
        b = z["b_in"].copy()
        st, _ = fb.bkz_reduction(b, fb.BKZParam(30, strategies="default", flags=int(gold[tag + "_flags"]),
                                                max_loops=2, seed=3))
        assert st == int(gold[tag + "_status"])
        outs.append(b)
    assert np.array_equal(outs[0], outs[1])
    r_in, _, pot_in = _quality(z["b_in"])
    _, slope_ref, pot_ref = _quality(gold[tag + "_b"])
    r, slope, pot = _quality(outs[0])
    assert abs(slope - slope_ref) <= 0.1 * abs(slope_ref), (slope, slope_ref)
    assert pot_in - pot >= 0.9 * (pot_in - pot_ref), (pot_in, pot, pot_ref)
    assert r[0] <= r_in[0]
    assert abs(np.log(r).sum() - np.log(r_in).sum()) < 1e-6
    assert H.is_lll_reduced(outs[0], 0.99, 0.51)


def test_sd_and_slide_together_is_the_reference_error_and_sd_alone_terminates(fb, capfd):
    """bkz.cpp:531-534: both flags -> the reference's message; bkz.cpp:548-554: SD-BKZ without a termination condition
    turns auto-abort on (with the reference's warning) and stops."""
    b = H.gold("bkz_q60.npz")["b_in"].copy()
    with pytest.raises(fb.B200Error, match="Invalid flags: SD-BKZ and Slide reduction are mutually exclusive!"):
        fb.bkz_reduction(b.copy(), fb.BKZParam(20, flags=fb.BKZ_SD_VARIANT | fb.BKZ_SLD_RED | fb.BKZ_NO_LLL))
    st, stats = fb.bkz_reduction(b, fb.BKZParam(10, flags=fb.BKZ_SD_VARIANT | fb.BKZ_NO_LLL))
    assert st == 0 and stats["tours"] >= 1
    assert "SD Variant of BKZ requires explicit termination condition. Turning auto abort on!" in capfd.readouterr().err
    assert H.is_lll_reduced(b, 0.99, 0.51)


@pytest.mark.parametrize("algo,tag", [("sdb", "sd"), ("sld", "sld")])
def test_reference_cli_sd_and_slide_with_the_shim_preloaded(tmp_path, algo, tag):
    """`fplll -a sdb|sld -b 20 -f double` (the reference's unmodified program) on the dim-60 q-ary basis, plain and with
    libb200fplll.so preloaded: same printed basis, and the preloaded run took bkz() over to the device driver."""
    cli = os.path.join(REF, "fplll")
    for p in (SHIM, cli):
        if not os.path.exists(p):
            pytest.skip("%s not built (needs the reference headers: built in the development container)" % p)
    inp = str(tmp_path / "in.txt")
    O.write_matrix(inp, H.gold("bkz_q60.npz")["b_in"])
    outs = []
    for preload in (False, True):
        env = dict(os.environ)
        env.pop("LD_PRELOAD", None)
        if preload:
            env["LD_PRELOAD"], env["B200_SHIM_STATS"] = SHIM, "1"
        p = subprocess.run([cli, "-a", algo, "-b", "20", "-f", "double", inp], capture_output=True, text=True,
                           timeout=900, env=env)
        assert p.returncode == 0, p.stderr[-1500:]
        if preload:
            line = [ln for ln in p.stderr.splitlines() if "b200 MatGSO shim" in ln][-1]
            assert int(line.split("device driver ")[1].split()[0]) >= 1, line
        open(str(tmp_path / "o.txt"), "w").write(p.stdout)
        outs.append(np.array(O.read_matrix(str(tmp_path / "o.txt")), dtype=np.int64))
    assert np.array_equal(outs[0], outs[1]), tag
