"""GPU parity tests: the CUDA GSO path (through the C-ABI of include/b200gso.h) against the CPU oracle and the
committed reference dumps.  Everything is integer / order-preserving fp64, so the bar is BIT-EXACT."""
import json

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
    """Both device LLL kernels: one CTA per lattice with the Babai iteration shared between its warps (gso_cta.cuh,
    taken for small batches) and one warp per lattice (taken for large batches); B200_LLL_CTA selects."""
    monkeypatch.setenv("B200_LLL_CTA", "1" if request.param == "cta" else "0")
    return request.param


def _gold_state(z, prefix=""):
    g = lambda k: z[prefix + k]
    return dict(n_known_rows=int(g("n_known_rows")), n_known_cols=int(g("n_known_cols")),
                n_source_rows=int(g("n_source_rows")), row_expo=g("row_expo"), gso_valid_cols=g("gso_valid_cols"),
                init_row_size=g("init_row_size"), bf=g("bf"), gf=g("gf"), mu=g("mu"), r=g("r"), b=g("b"))


def test_update_gso_u40_vs_reference_dump(fb):
    z = H.gold("u40_update_gso.npz")
    m = fb.MatGSO(z["b"])
    assert m.update_gso().all()
    H.assert_state_equal(H.lattice_state(m.state(), 0), _gold_state(z), "u40")


def test_ops_trace_u40_vs_reference_dump(fb):
    z = H.gold("u40_ops_trace.npz")
    ops = json.loads(bytes(z["ops_json"]).decode())
    marks = list(z["marks"])
    m = fb.MatGSO(z["b0"])
    t = 0
    for k, op in enumerate(ops):
        H.apply_ops(m, [tuple(op)])
        if t < len(marks) and marks[t] == k:
            H.assert_state_equal(H.lattice_state(m.state(), 0), _gold_state(z, "s%d_" % t), "op %d %s" % (k, op))
            t += 1
    assert t == len(marks)


def test_update_gso_r200_vs_reference_dump(fb):
    """BASELINE config #2/#5 state: the wrapper-LLL-reduced latticegen r 200 2000 basis (int64 regime)."""
    z = H.gold("r200_lll_update_gso.npz")
    m = fb.MatGSO(z["b"])
    assert m.update_gso().all()
    s = H.lattice_state(m.state(), 0)
    tl = np.tril_indices(200)
    off = tl[0] != tl[1]
    assert H.eq_f64(s["mu"][tl][off], z["mu_tril"][off])
    assert H.eq_f64(s["r"][tl], z["r_tril"])
    assert H.eq_f64(s["gf"][tl], z["gf_tril"])
    assert np.array_equal(s["row_expo"], z["row_expo"])


@pytest.mark.parametrize("seed,d,n,bits,flags", [(1, 12, 12, 20, 2), (2, 33, 40, 30, 2), (3, 64, 65, 12, 0),
                                                  (4, 7, 9, 50, 2), (5, 97, 97, 25, 2), (6, 130, 131, 10, 2)])
def test_random_ops_vs_oracle(fb, seed, d, n, bits, flags):
    rng = np.random.default_rng(seed)
    b = rng.integers(-(1 << bits), 1 << bits, size=(d, n), dtype=np.int64)
    ops = H.random_op_script(rng, d, 50)
    mo = O.OracleGSO(b, flags)
    md = fb.MatGSO(b, flags)
    for k, op in enumerate(ops):
        H.apply_ops(mo, [op])
        H.apply_ops(md, [op])
        if k % 7 == 0 or k == len(ops) - 1:
            H.assert_state_equal(H.lattice_state(md.state(), 0), mo.state(), "seed %d op %d %s" % (seed, k, op))


def test_batch_lattices_are_independent(fb):
    """a batch of different lattices == each lattice run alone (the replica axis of SURVEY §8e)."""
    rng = np.random.default_rng(11)
    B, d, n = 9, 24, 30
    b = rng.integers(-1000, 1000, size=(B, d, n), dtype=np.int64)
    md = fb.MatGSO(b)
    assert md.update_gso().all()
    x = rng.integers(-5, 6, size=B).astype(np.float64)
    md.row_addmul_we(7, 3, x, 0)
    md.row_op_end(7, 8)
    md.move_row(20, 5)
    md.update_gso()
    st = md.state()
    for l in range(B):
        mo = O.OracleGSO(b[l])
        mo.update_gso()
        mo.row_addmul_we(7, 3, x[l], 0)
        mo.row_op_end(7, 8)
        mo.move_row(20, 5)
        mo.update_gso()
        H.assert_state_equal(H.lattice_state(st, l), mo.state(), "lattice %d" % l)


def test_ragged_knapsack_and_zero_row(fb):
    rng = np.random.default_rng(9)
    d = 10
    b = np.zeros((d, d + 1), np.int64)
    b[:, 0] = rng.integers(1, 1 << 40, size=d)
    b[np.arange(d), np.arange(d) + 1] = 1
    b[4] = 0
    mo, md = O.OracleGSO(b), fb.MatGSO(b)
    for t in range(3):
        # catastrophic cancellation on the raw knapsack basis may make r(1,1) == 0 and the next row fail with a
        # non-finite mu: whatever the reference's arithmetic does, the device must do the same
        assert mo.update_gso_row(t, t) == bool(md.update_gso_row(t, t)[0])
    H.assert_state_equal(H.lattice_state(md.state(), 0), mo.state(), "partial discovery")
    mo.move_row(1, 9)
    md.move_row(1, 9)
    H.assert_state_equal(H.lattice_state(md.state(), 0), mo.state(), "row leaves the known set")


def test_gso_failure_reported_like_reference(fb):
    """duplicate row -> r(j,j) == 0 -> mu = x/0 not finite -> update_gso_row returns false (gso_interface.cpp:156)."""
    b = np.array([[3, 1, 4], [3, 1, 4], [1, 5, 9]], dtype=np.int64)
    mo, md = O.OracleGSO(b), fb.MatGSO(b)
    assert mo.update_gso_row(0) and md.update_gso_row(0).all()
    assert mo.update_gso_row(1) and md.update_gso_row(1).all()
    assert mo.update_gso_row(2) is False
    assert not md.update_gso_row(2).any()


def test_device_lll_u40_equals_reference_basis(fb, lll_mode):
    """BASELINE config #1: LLL delta=0.99 on latticegen u 40 40 — the device LLL must walk the reference's exact
    basis trajectory (same swaps, same output basis as MatGSO<long,double>+LLLReduction of the reference)."""
    z = H.gold("u40_lll_long.npz")
    m = fb.MatGSO(z["b_in"])
    st, stats = m.lll(0.99, 0.51)
    assert st[0] == int(z["status"]) == 0
    assert stats["n_swaps"][0] == int(z["n_swaps"])
    assert np.array_equal(m.b[0], z["b_out"])


@pytest.mark.parametrize("seed,d,bits", [(21, 16, 20), (22, 48, 30), (23, 70, 16)])
def test_device_lll_random_vs_oracle(fb, lll_mode, seed, d, bits):
    rng = np.random.default_rng(seed)
    B = 5
    b = rng.integers(-(1 << bits), 1 << bits, size=(B, d, d), dtype=np.int64)
    b[1, 3] = 0  # a zero vector: parked at the end (lll.cpp:66-69)
    b[2, 5] = b[2, 4]  # a dependency: discovered as a zero vector during reduction (lll.cpp:144-150)
    md = fb.MatGSO(b)
    st, stats = md.lll(0.99, 0.51)
    out = md.b
    for l in range(B):
        mo = O.OracleGSO(b[l])
        res = mo.lll(0.99, 0.51)
        assert st[l] == res["status"], "lattice %d status" % l
        assert stats["n_swaps"][l] == res["n_swaps"]
        assert stats["zeros"][l] == res["zeros"]
        assert np.array_equal(out[l], mo.state()["b"]), "lattice %d basis" % l


def test_device_lll_output_passes_reference_is_lll_reduced(fb, lll_mode):
    """the reference's own acceptance check, is_lll_reduced (lll.cpp:226-258), in exact arithmetic (helpers.py), and
    the reference's verdict on the basis the device must produce (tests/golden/ref_islll.json)."""
    z = H.gold("u40_lll_long.npz")
    b = z["b_in"].copy()
    assert fb.lll_reduction(b, 0.99, 0.51) == 0
    assert H.is_lll_reduced(b, 0.99, 0.51)
    assert np.array_equal(b, z["b_out"]) and H.gold_json("ref_islll.json")["u40_b_out"] == 1


@pytest.mark.parametrize("seed,d,bits", [(31, 140, 10), (32, 200, 8)])
def test_device_lll_wide_vs_oracle(fb, lll_mode, seed, d, bits):
    """d > 128 takes the 8-registers-per-lane Babai path (k_lll<8>) that BKZ on dim-200 uses."""
    rng = np.random.default_rng(seed)
    b = rng.integers(-(1 << bits), 1 << bits, size=(2, d, d + 1), dtype=np.int64)
    md = fb.MatGSO(b)
    st, stats = md.lll(0.99, 0.51)
    out = md.b
    for l in range(2):
        mo = O.OracleGSO(b[l])
        res = mo.lll(0.99, 0.51)
        assert st[l] == res["status"] == 0
        assert stats["n_swaps"][l] == res["n_swaps"]
        assert np.array_equal(out[l], mo.state()["b"]), "lattice %d basis" % l


def test_ranged_lll_and_size_reduction_resume_are_exact(fb, lll_mode):
    """lll(0,0,k) / size_reduction(0,k) resume after the clean prefix (BKZ's pattern: reduce a prefix, touch a row,
    reduce a longer prefix).  Status, n_swaps, zeros, final_kappa and the whole state after every call must equal the
    ranged oracle's on the same continuing object."""
    from test_lll_ranged_gpu import Pair
    rng = np.random.default_rng(41)
    d = 60
    p = Pair(fb, rng.integers(-(1 << 12), 1 << 12, size=(1, d, d), dtype=np.int64))
    p.lll(kend=30)
    p.lll(kend=45)
    p.run([["addmul", 20, 3, 7.0]])
    p.sr(kend=40)
    p.lll(kend=60)


@pytest.mark.parametrize("mode", [0, 1])
def test_blocked_update_gso_small_entries_bit_exact(fb, mode):
    """b200gso_update_gso_blocked: Gram matrix in 32x32 tiles, then the row sweeps.  Entries below 2^20 make every
    partial sum of a Gram entry exact, so the tensor-core (DMMA) mode must agree bit for bit as well."""
    rng = np.random.default_rng(51)
    b = rng.integers(-(1 << 20), 1 << 20, size=(3, 70, 75), dtype=np.int64)
    b[1, :, 60:] = 0  # ragged: fewer known columns
    md = fb.MatGSO(b)
    assert md.update_gso_blocked(mode).all()
    st = md.state()
    for l in range(3):
        mo = O.OracleGSO(b[l])
        assert mo.update_gso()
        H.assert_state_equal(H.lattice_state(st, l), mo.state(), "blocked mode %d lattice %d" % (mode, l))


def test_blocked_update_gso_large_entries(fb):
    """40-bit entries: the ordered mode stays bit-exact, the DMMA mode is within north_star's 1e-9 on mu and r."""
    rng = np.random.default_rng(52)
    b = rng.integers(-(1 << 40), 1 << 40, size=(2, 64, 64), dtype=np.int64)
    for mode in (0, 1):
        md = fb.MatGSO(b)
        assert md.update_gso_blocked(mode).all()
        st = md.state()
        for l in range(2):
            mo = O.OracleGSO(b[l])
            assert mo.update_gso()
            s = mo.state()
            if mode == 0:
                H.assert_state_equal(H.lattice_state(st, l), s, "ordered lattice %d" % l)
            else:
                for i in range(64):
                    for name in ("mu", "r"):
                        a, e = st[name][l][i, :i], s[name][i, :i]
                        assert np.all(np.abs(a - e) <= 1e-9 * np.maximum(1.0, np.abs(e))), (name, l, i)


# ---- direct tests of the remaining C-ABI entry points (SURVEY §8 a7 and the accessors the drop-in class forwards to) ----

def test_row_swap_set_r_negate_direct_vs_oracle(fb):
    """row_swap (gso.cpp:264-287: integer rows only, bracketed by row_op_begin/end as bkz.cpp:221-263 does),
    set_r (gso_interface.h:739-746) and negate_row_of_b (gso.h:291-297), each followed by the state comparison."""
    rng = np.random.default_rng(71)
    b = rng.integers(-(1 << 30), 1 << 30, size=(3, 40, 44), dtype=np.int64)
    md = fb.MatGSO(b)
    mos = [O.OracleGSO(b[l]) for l in range(3)]
    assert md.update_gso().all()
    for mo in mos:
        assert mo.update_gso()
    for (i, j) in ((3, 17), (39, 0), (20, 21)):
        lo, hi = min(i, j), max(i, j)
        md.row_op_begin(lo, hi + 1)
        md.row_swap(i, j)
        md.row_op_end(lo, hi + 1)
        for mo in mos:
            mo.row_swap(i, j)
            mo.row_op_end(lo, hi + 1)
        st = md.state()
        for l, mo in enumerate(mos):
            H.assert_state_equal(H.lattice_state(st, l), mo.state(), "row_swap(%d,%d) lattice %d" % (i, j, l))
        assert md.update_gso().all()
        for mo in mos:
            assert mo.update_gso()
    # set_r on the diagonal of a valid row (what lll.cpp:137-142 does after the Lovasz test)
    vals = np.array([1.5, 2.25, 1e10])
    md.set_r(12, 12, vals)
    for l, mo in enumerate(mos):
        mo.set_r(12, 12, float(vals[l]))
    st = md.state()
    for l, mo in enumerate(mos):
        H.assert_state_equal(H.lattice_state(st, l), mo.state(), "set_r lattice %d" % l)
    # negate_row_of_b inside a row operation
    md.row_op_begin(7, 8)
    md.negate_row_of_b(7)
    md.row_op_end(7, 8)
    st = md.state()
    for l in range(3):
        want = mos[l].state()["b"].copy()
        want[7] = -want[7]
        assert np.array_equal(st["b"][l], want)
        assert int(st["gso_valid_cols"][l][7]) == 0


def test_upload_row_equals_row_rewrite_plus_row_op_end(fb):
    """b200gso_upload_row(i, rows): the host-resident-driver protocol (host rewrites b_i, ships the row): must leave
    exactly the state of `b[i] = row; row_op_end(i, i+1)` on a fresh object."""
    rng = np.random.default_rng(72)
    b = rng.integers(-(1 << 25), 1 << 25, size=(2, 30, 33), dtype=np.int64)
    md = fb.MatGSO(b)
    assert md.update_gso().all()
    newrow = rng.integers(-(1 << 27), 1 << 27, size=(2, 33), dtype=np.int64)
    md.upload_row(11, newrow)
    assert md.update_gso().all()
    st = md.state()
    for l in range(2):
        b2 = b[l].copy()
        b2[11] = newrow[l]
        mo = O.OracleGSO(b2)
        assert mo.update_gso()
        H.assert_state_equal(H.lattice_state(st, l), mo.state(), "upload_row lattice %d" % l)


def test_get_block_and_get_r_diag_vs_oracle(fb):
    """b200gso_get_block / get_r_diag: the block view Enumeration::enumerate builds (enumerate_ext.cpp:91-148) from
    get_mu / get_r_exp, row_expo applied."""
    rng = np.random.default_rng(73)
    b = rng.integers(-(1 << 40), 1 << 40, size=(2, 48, 50), dtype=np.int64)
    md = fb.MatGSO(b)
    assert md.update_gso().all()
    for l in range(2):
        mo = O.OracleGSO(b[l])
        assert mo.update_gso()
        s = mo.state()
        first, beta = 9, 30
        mut, rm, re = md.get_block(first, beta, lattice=l)
        for k in range(beta):
            for j in range(k + 1, beta):
                e = int(s["row_expo"][first + j]) - int(s["row_expo"][first + k])
                assert mut[k, j] == float(np.ldexp(s["mu"][first + j, first + k], e))
            assert rm[k] == s["r"][first + k, first + k] and re[k] == 2 * int(s["row_expo"][first + k])
        rm2, re2 = md.get_r_diag(0, 48, lattice=l)
        assert np.array_equal(rm2, np.diag(s["r"])) and np.array_equal(re2, 2 * s["row_expo"])


def test_two_live_handles_of_different_size(fb):
    """ADVICE r1: a second, smaller handle must not lower the kernels' dynamic shared-memory limit under a larger live
    one (the attribute is process-wide)."""
    rng = np.random.default_rng(74)
    big = rng.integers(-(1 << 20), 1 << 20, size=(1, 200, 201), dtype=np.int64)
    small = rng.integers(-(1 << 20), 1 << 20, size=(1, 40, 40), dtype=np.int64)
    mb = fb.MatGSO(big)
    ms = fb.MatGSO(small)
    assert ms.update_gso().all()
    assert mb.update_gso().all()          # the larger handle, after the smaller one was created and used
    st, _ = ms.lll(0.99, 0.51)
    assert st[0] == 0
    st, _ = mb.lll(0.99, 0.51)
    assert st[0] == 0
    mo = O.OracleGSO(big[0])
    assert mo.lll(0.99, 0.51)["status"] == 0
    assert np.array_equal(mb.b[0], mo.state()["b"])


@pytest.mark.parametrize("d,n,B,bits", [(70, 75, 1600, 20), (200, 201, 800, 20), (96, 96, 777, 30)])
def test_update_row_mixed_states_equal_oracle(fb, d, n, B, bits):
    """The batched update_gso_row kernel against the oracle, bit for bit, on a sample of lattices of a large batch whose
    lattices are in mixed states: full recompute, Gram row partly valid, row already valid, partial update
    (last_j < i)."""
    rng = np.random.default_rng(d)
    base = rng.integers(-(1 << bits), 1 << bits, size=(8, d, n), dtype=np.int64)
    b = base[rng.integers(0, 8, size=B)]
    x = rng.integers(-3, 4, size=B).astype(np.float64)
    rows = [d - 1, 33, 1, 0, d - 9, 64 if d > 64 else 31]
    m = fb.MatGSO(b)
    assert m.update_gso().all()
    for i in rows:
        if i:
            m.row_addmul_we(i, i - 1, x, 0)                      # some lattices get x = 0: still a row_op_end
        m.row_op_end(i, i + 1)
        if i > 40:
            assert m.update_gso_row(i, i - 7).all()              # partial row first, then the rest of it
        assert m.update_gso_row(i, i).all()
        if i + 1 < d:
            assert m.update_gso_row(i + 1, i + 1).all()          # row i + 1: only its Gram entry (i+1, i) is invalid
    st = m.state()
    m.close()
    for l in (0, 1, B // 2, B - 1):
        mo = O.OracleGSO(b[l])
        mo.update_gso()
        for i in rows:
            if i:
                mo.row_addmul_we(i, i - 1, x[l], 0)
            mo.row_op_end(i, i + 1)
            if i > 40:
                mo.update_gso_row(i, i - 7)
            mo.update_gso_row(i, i)
            if i + 1 < d:
                mo.update_gso_row(i + 1, i + 1)
        H.assert_state_equal(H.lattice_state(st, l), mo.state(), "lattice %d" % l)
