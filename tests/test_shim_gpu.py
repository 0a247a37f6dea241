"""GPU tests of the MatGSO forwarding shim (fplll_b200/csrc/fplll_matgso_shim.cpp, SURVEY §8 b1 / N2): the UNMODIFIED
reference library and its unmodified callers (LLLReduction, BKZReduction, the reference's own test programs) run
with libb200fplll.so preloaded, so every MatGSO<Z_NR<long>|Z_NR<mpz_t>, FP_NR<double>>::update_gso_row executes on the
GPU.  The device GSO is bit-exact, so results must be byte-identical to the plain runs."""
import os
import subprocess

import numpy as np
import pytest

import helpers as H
from oracle import oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = os.path.join(ROOT, "tests", "_build", "libb200fplll.so")
DEMO = os.path.join(ROOT, "tests", "_build", "shim_demo")
REF = os.path.join(ROOT, "oracle", "_ref")


def _need(*paths):
    for p in paths:
        if not os.path.exists(p):
            pytest.skip("%s not built (needs the reference headers: built in the development container)" % p)


def _run(cmd, preload, timeout=900):
    env = dict(os.environ)
    env.pop("LD_PRELOAD", None)
    if preload:
        env["LD_PRELOAD"] = SHIM
        env["B200_SHIM_STATS"] = "1"
    return subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)


def _stat(text, key):
    return int(text.split(key + "=")[1].split()[0])


@pytest.mark.parametrize("mode", ["long", "mpz", "long_gram", "mpz_gram"])
def test_reference_lll_over_the_device_gso_is_byte_identical(tmp_path, mode):
    """LLLReduction<ZT, FP_NR<double>>::lll() of the unmodified reference over its own MatGSO object, plain and with the
    shim preloaded: same status, same basis, same mu / r / row_expo bits; the preloaded run forwarded its updates.
    long: BASELINE config #1 (latticegen u 40 40-bit basis); mpz: a 400-bit knapsack basis that does not fit int64, the
    regime where B stays in GMP on the host (GSO_ROW_EXPO | GSO_OP_FORCE_LONG, wrapper.cpp:538-553); *_gram: the same two
    integer types with GSO_INT_GRAM (SURVEY §8 f2: the exact integer Gram matrix stays on the host, gso.cpp:140-159, its
    rows travel as doubles through b200gso_set_gram_row)."""
    _need(SHIM, DEMO, os.path.join(REF, "libfplll.so"))
    inp = str(tmp_path / "in.txt")
    if mode == "long":
        O.write_matrix(inp, H.gold("u40_lll_long.npz")["b_in"])
    elif mode == "long_gram":
        open(inp, "w").write(O.latticegen(["u", 30, 12]))   # 12-bit entries: the exact Gram matrix fits Z_NR<long>
    else:
        open(inp, "w").write(O.latticegen(["r", 30, 400]))
    outs = []
    for preload in (False, True):
        out = str(tmp_path / ("out%d.bin" % preload))
        p = _run([DEMO, inp, mode, out], preload)
        assert p.returncode == 0, p.stderr[-2000:]
        assert "status=0" in p.stdout, p.stdout
        fwd = _stat(p.stdout, "forwarded")
        assert (fwd > 0) == preload, p.stdout
        if preload:
            assert _stat(p.stdout, "adopted") >= 1 and (_stat(p.stdout, "uploads") > 0 or mode.endswith("_gram"))
        outs.append((open(out, "rb").read(), open(out + ".basis").read()))
    assert outs[0][1] == outs[1][1], "basis differs"
    assert outs[0][0] == outs[1][0], "mu / r / row_expo differ"


def test_config2_lll_on_r200_2000_in_the_mpz_regime_fails_exactly_like_the_reference(tmp_path):
    """BASELINE config #2 at its stated size and in its stated regime: the reference's LLLReduction<Z_NR<mpz_t>,
    FP_NR<double>> (GSO_ROW_EXPO | GSO_OP_FORCE_LONG, wrapper.cpp:538-553) on latticegen r 200 2000 — 2000-bit entries, B
    stays in GMP on the host — with every update_gso_row forwarded to the device.  The reference's own fp64 stage cannot
    finish this input (RED_BABAI_FAILURE near kappa = 180 after 33 s, BASELINE.md §3 row 2a); the device GSO is bit-exact,
    so the run must fail at the same point: same status, same mu / r / row_expo dump and same basis as the reference's
    own run (tests/golden/lll_r200_mpz_ref.json, hashes)."""
    import hashlib
    import json
    _need(SHIM, DEMO, os.path.join(REF, "libfplll.so"), os.path.join(REF, "latticegen"))
    ref = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lll_r200_mpz_ref.json")))
    inp, out = str(tmp_path / "r200.txt"), str(tmp_path / "out.bin")
    text = O.latticegen(["r", 200, 2000])
    assert hashlib.md5(text.encode()).hexdigest() == ref["input_md5"]
    open(inp, "w").write(text)
    p = _run([DEMO, inp, "mpz", out], True, timeout=1500)
    assert p.returncode == 0, p.stderr[-2000:]
    assert "status=%d gso_ok=%d" % (ref["status"], ref["gso_ok"]) in p.stdout and ref["status"] == 3, p.stdout
    assert _stat(p.stdout, "adopted") >= 1 and _stat(p.stdout, "forwarded") > 100000, p.stdout
    sha = lambda f: hashlib.sha256(open(f, "rb").read()).hexdigest()
    assert sha(out + ".basis") == ref["out_basis_sha256"], "basis after the failing LLL differs"
    assert sha(out) == ref["out_bin_sha256"], "mu / r / row_expo after the failing LLL differ"


# the reference's test_bkz takes minutes per run with every update_gso_row forwarded: deselected unless B200_TEST_SLOW=1
# (tests/conftest.py)
_SLOW = pytest.mark.slow


@pytest.mark.parametrize("prog,bkz_takeover", [("test_gso", 1), ("test_lll", 1),
                                               pytest.param("test_bkz", 0, marks=_SLOW),
                                               pytest.param("test_bkz", 1, marks=_SLOW)])
def test_reference_test_programs_pass_over_the_device_gso(prog, bkz_takeover, monkeypatch):
    """The reference's own tests/test_gso.cpp, test_lll.cpp and test_bkz.cpp (compiled unmodified by oracle/Makefile.ref)
    with the shim preloaded: 'All tests passed.' and at least one MatGSO object ran on the device.  test_bkz runs twice:
    with the reference's BKZ control flow over the forwarded GSO (B200_SHIM_BKZ=0) and with BKZReduction::bkz() taken over
    by the device driver."""
    exe = os.path.join(REF, prog)
    _need(SHIM, exe)
    monkeypatch.setenv("B200_SHIM_BKZ", str(bkz_takeover))
    p = _run([exe], True, timeout=1500)
    assert p.returncode == 0, (p.stdout[-500:], p.stderr[-1500:])
    assert "All tests passed." in p.stderr  # the reference's tests report on stderr (tests/test_lll.cpp:175)
    line = [l for l in p.stderr.splitlines() if "b200 MatGSO shim" in l][-1]
    adopted = int(line.split("adopted ")[1].split()[0])
    forwarded = int(line.split("forwarded ")[1].split(",")[0])
    assert adopted >= 1 and forwarded > 0, line
    if prog == "test_bkz":
        taken = int(line.split("device driver ")[1].split()[0])
        assert (taken > 0) == bool(bkz_takeover), line


def test_reference_cli_bkz_with_the_shim_preloaded(tmp_path):
    """`fplll -a bkz -b 20 -f double` (the reference's unmodified command-line program) on the dim-60 q-ary basis, plain
    and with libb200fplll.so preloaded: without pruning BKZ is deterministic, so both runs must print the same basis —
    the reference's own output (tests/golden/bkz_q60.npz) — and the preloaded one ran bkz() on the device driver."""
    cli = os.path.join(REF, "fplll")
    _need(SHIM, cli)
    z = H.gold("bkz_q60.npz")
    inp = str(tmp_path / "in.txt")
    O.write_matrix(inp, z["b_in"])
    outs = []
    for preload in (False, True):
        p = _run([cli, "-a", "bkz", "-b", "20", "-f", "double", inp], preload)
        assert p.returncode == 0, p.stderr[-1500:]
        if preload:
            line = [l for l in p.stderr.splitlines() if "b200 MatGSO shim" in l][-1]
            assert int(line.split("device driver ")[1].split()[0]) >= 1, line
        open(str(tmp_path / "o.txt"), "w").write(p.stdout)
        outs.append(np.array(O.read_matrix(str(tmp_path / "o.txt")), dtype=np.int64))
    assert np.array_equal(outs[0], outs[1])
    assert np.array_equal(outs[1], z["bkz20_none_b"])
