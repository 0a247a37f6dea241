"""GPU parity tests of the kernel variants only large inputs reach, against the CPU oracle and the reference, bit for bit.

Device LLL (b200gso_lll*): d <= 128 runs k_lll<4> / k_lll_cta<4>, d <= 256 the <8> kernels, d <= 512 the <16> kernels.
The CTA kernel caches as many leading mu panels in shared memory as fit next to its scratch: all of them up to d = 211,
six of them from d = 216 on, so that above that readers pick shared or global memory per panel.  Its UPDATE and BACKSUB
run as streamed wavefronts while the active panel span is below CTA_WARPS = 8 panels and switch to the barrier-per-panel
form, with two panels per warp, from row 257 on (d >= 258).  MatGSO's default GSO_ROW_EXPO is covered with flags 0 too.

Device HLLL (b200hh_hlll, b200hh_update_R): a lane keeps ceil(n/32) + 1 elements of a reflection in 4, 8, 14 or 32
registers (n <= 96, 224, 416, 992); wider rows are refused."""
import numpy as np
import pytest

import helpers as H
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fb():
    import fplll_b200
    return fplll_b200


@pytest.fixture(params=["cta", "warp"])
def lll_mode(request, monkeypatch):
    """Both device LLL kernels: one CTA per lattice (taken for small batches) and one warp per lattice."""
    monkeypatch.setenv("B200_LLL_CTA", "1" if request.param == "cta" else "0")
    return request.param


_oracle_runs = {}


def _oracle_lll(key, b, flags):
    """OracleGSO(b, flags).lll(): (result, final state); both kernels compare against the same run."""
    if key not in _oracle_runs:
        mo = O.OracleGSO(b, flags)
        res = mo.lll(0.99, 0.51)
        _oracle_runs[key] = (res, mo.state())
    return _oracle_runs[key]


def _assert_lll_like_oracle(md, st, stats, b, flags, key):
    s = md.state()
    for l in range(b.shape[0]):
        res, ref = _oracle_lll(key + (l,), b[l], flags)
        what = "%s lattice %d" % (key, l)
        assert st[l] == res["status"], what + " status"
        assert stats["n_swaps"][l] == res["n_swaps"], what + " n_swaps"
        assert stats["zeros"][l] == res["zeros"], what + " zeros"
        assert stats["final_kappa"][l] == res["final_kappa"], what + " final_kappa"
        assert np.array_equal(s["b"][l], ref["b"]), what + " basis"
        H.assert_state_equal(H.lattice_state(s, l), ref, what)


def _uniform(seed, batch, d, bits):
    rng = np.random.default_rng(seed)
    b = rng.integers(-(1 << bits), 1 << bits, size=(batch, d, d + 1), dtype=np.int64)
    b[1, 3] = 0  # a zero vector: parked at the end
    b[1, d - 2] = b[1, d - 3]  # a dependency in the last panel: found as a zero vector during the reduction
    return b


# d = 70 is the control: the <4> kernels with every mu panel cached, the class the rest of the suite covers
@pytest.mark.parametrize("d,batch", [(70, 3), (216, 3), (232, 3), (257, 3), (300, 3), (512, 2)])
def test_device_lll_vs_oracle_by_size(fb, lll_mode, d, batch):
    b = _uniform(d, batch, d, 12)
    md = fb.MatGSO(b)
    st, stats = md.lll(0.99, 0.51)
    _assert_lll_like_oracle(md, st, stats, b, 2, ("uniform", d))


def test_device_lll_without_row_expo_d300(fb, lll_mode):
    b = _uniform(1300, 2, 300, 12)
    md = fb.MatGSO(b, 0)
    st, stats = md.lll(0.99, 0.51)
    _assert_lll_like_oracle(md, st, stats, b, 0, ("flags0", 300))


@pytest.mark.parametrize("tag", ["lll300", "knap260"])
def test_device_lll_vs_reference_size_fixture(fb, lll_mode, tag):
    """the reference's own LLLReduction<long,double> run on the same input (tests/golden/size_classes_ref.npz)."""
    z = H.gold("size_classes_ref.npz")
    b = z[tag + "_in"].astype(np.int64)
    md = fb.MatGSO(b)
    st, stats = md.lll(0.99, 0.51)
    assert st[0] == int(z[tag + "_status"]) == 0
    assert stats["n_swaps"][0] == int(z[tag + "_swaps"])
    assert np.array_equal(md.b[0], z[tag + "_out"])
    _assert_lll_like_oracle(md, st, stats, b[None], 2, ("gold", tag))


def test_ranged_lll_and_size_reduction_resume_d300(fb, lll_mode):
    """lll(0,0,k) / size_reduction(0,k) with prefixes ending on both sides of row 256 and a row above it touched in
    between: the basis must equal a from-scratch oracle run of the same call sequence."""
    import ctypes as C
    from fplll_b200.gso import _lib, _ck, _ptr
    rng = np.random.default_rng(42)
    d = 300
    b = rng.integers(-(1 << 12), 1 << 12, size=(d, d), dtype=np.int64)
    md = fb.MatGSO(b)
    st = np.zeros(1, np.int32)

    def dev_lll(kend):
        _ck(_lib().b200gso_lll_range(md._h, 0.99, 0.51, 0, 0, kend, 0, _ptr(st, C.c_int), None), "lll_range")
        return int(st[0])

    def dev_sr(kend):
        _ck(_lib().b200gso_size_reduction(md._h, 0.51, 0, kend, 0, _ptr(st, C.c_int)), "size_reduction")
        return int(st[0])

    def ora_lll(bb, kend):
        # lll(0, 0, kend) of the reference on the rows < kend: a fresh oracle on those rows
        sub = O.OracleGSO(bb[:kend])
        r = sub.lll(0.99, 0.51)
        out = bb.copy()
        out[:kend] = sub.state()["b"]
        return r["status"], out
    bb = b
    for kend in (240, 280):
        assert dev_lll(kend) == 0
        s, bb = ora_lll(bb, kend)
        assert s == 0 and np.array_equal(md.b[0], bb), "lll(0, 0, %d)" % kend
    md.row_addmul_we(262, 3, 7.0, 0)
    md.row_op_end(262, 263)
    mo = O.OracleGSO(bb)
    mo.row_addmul_we(262, 3, 7.0, 0)
    mo.row_op_end(262, 263)
    assert dev_sr(290) == 0
    assert dev_lll(300) == 0
    s, bb = ora_lll(mo.state()["b"], 300)
    assert s == 0 and np.array_equal(md.b[0], bb)


@pytest.mark.parametrize("flags", [2, 0])
@pytest.mark.parametrize("d", [255, 256, 257, 300, 512])
def test_random_ops_vs_oracle_by_size(fb, d, flags):
    """move_row, row_addmul_we with and without exponents and row updates, mostly on rows in panel 8 and above."""
    rng = np.random.default_rng(7000 + d + flags)
    b = rng.integers(-(1 << 20), 1 << 20, size=(d, d + 1), dtype=np.int64)
    ops = H.random_op_script(rng, d, 40)
    mo = O.OracleGSO(b, flags)
    md = fb.MatGSO(b, flags)
    for k, op in enumerate(ops):
        H.apply_ops(mo, [op])
        H.apply_ops(md, [op])
        if k % 7 == 0 or k == len(ops) - 1:
            H.assert_state_equal(H.lattice_state(md.state(), 0), mo.state(), "d %d op %d %s" % (d, k, op))


def test_device_lll_refuses_d513(fb):
    b = np.random.default_rng(513).integers(-100, 100, size=(1, 513, 514), dtype=np.int64)
    md = fb.MatGSO(b)
    with pytest.raises(fb.B200Error):
        md.lll(0.99, 0.51)


# ---- Householder ----------------------------------------------------------------------------------------------------

def _mixed(seed, batch, d, n):
    """random small combinations of random rows: d random rows of n >> d columns are nearly orthogonal already, these
    make HLLL swap and size-reduce."""
    rng = np.random.default_rng(seed)
    u = rng.integers(-64, 65, size=(batch, d, d), dtype=np.int64)
    return u @ rng.integers(-(1 << 10), 1 << 10, size=(batch, d, n), dtype=np.int64)


@pytest.mark.parametrize("n", [96, 97, 224, 225, 416, 417, 600, 992])
def test_device_hlll_vs_oracle_by_width(n):
    from fplll_b200.householder import hlll_reduction
    b = _mixed(n, 2, 20 if n > 600 else 30, n)
    outs, sts = hlll_reduction(b)
    for l in range(2):
        mo = O.OracleHouseholder(b[l])
        assert mo.hlll() == sts[l], "n %d lattice %d status" % (n, l)
        assert np.array_equal(outs[l], mo.state()["b"]), "n %d lattice %d basis" % (n, l)


def test_device_hlll_vs_reference_size_fixture():
    from fplll_b200.householder import hlll_reduction
    z = H.gold("size_classes_ref.npz")
    out, st = hlll_reduction(z["hlll600_in"].astype(np.int64))
    assert st == int(z["hlll600_status"]) == 0
    assert np.array_equal(out, z["hlll600_out"])


def test_hlll_call_sequence_n500_bit_exact():
    """update_R<32> step by step in HLLLReduction::hlll's call order: R, V, sigma, bf, b after every Lovasz step."""
    from fplll_b200.householder import MatHouseholder
    from test_hh_oracle import hh_call_sequence
    d, n = 30, 500
    b = np.random.default_rng(500).integers(-(1 << 20), 1 << 20, size=(2, d, n), dtype=np.int64)
    _, ops, rows = hh_call_sequence(500, d, n, 20)
    md = MatHouseholder(b, 5)
    mos = [O.OracleHouseholder(b[l], 5) for l in range(2)]
    checks = 0
    for op in ops:
        if op[0] == "dump":
            st = md.state()
            for l, mo in enumerate(mos):
                s = mo.state()
                nk = s["n_known_rows"]
                what = "lattice %d check %d" % (l, checks)
                assert st["n_known_rows"][l] == nk and st["n_known_cols"][l] == s["n_known_cols"], what
                assert np.array_equal(st["b"][l], s["b"]), what + " b"
                for k in ["row_expo", "expo_norm_square_b"]:
                    assert np.array_equal(st[k][l][:rows], s[k][:rows]), what + " " + k
                for k in ["sigma", "norm_square_b"]:
                    assert H.eq_f64(st[k][l][:nk], s[k][:nk]), what + " " + k
                for k in ["bf", "R"]:
                    assert H.eq_f64(st[k][l][:rows], s[k][:rows]), what + " " + k
                assert H.eq_f64(st["V"][l][:nk], s["V"][:nk]), what + " V"
            checks += 1
        else:
            r = getattr(md, op[0])(*op[1:])
            for l, mo in enumerate(mos):
                ro = getattr(mo, op[0])(*op[1:])
                if op[0] == "size_reduce":
                    assert bool(r[l]) == bool(ro)
    assert checks > 5


@pytest.mark.parametrize("n", [993, 1100])
def test_hlll_and_update_R_refuse_rows_wider_than_992(n):
    """a lane holds at most 32 elements of a reflection: wider rows would leave columns >= 1024 of the first
    reflections unapplied, so hlll and update_R refuse them instead of returning a wrong R."""
    from fplll_b200 import B200Error
    from fplll_b200.householder import MatHouseholder, hlll_reduction
    b = np.random.default_rng(n).integers(-(1 << 20), 1 << 20, size=(6, n), dtype=np.int64)
    with pytest.raises(B200Error, match="992"):
        hlll_reduction(b)
    m = MatHouseholder(b, 5)
    m.refresh_R_bf(0)
    with pytest.raises(B200Error, match="992"):
        m.update_R(0)
