"""GPU parity tests of the ranged LLL entry points the BKZ driver calls, against the ranged oracle, bit for bit.

b200gso_lll_range(kappa_min, kappa_start, kappa_end, size_reduction_start) and b200gso_size_reduction are
LLLReduction::lll (lll.cpp:44-164) and LLLReduction::size_reduction (lll.h:106-122) on one continuing object.  The
device keeps a clean prefix per lattice (M_CLEAN_LLL / M_CLEAN_SR, gso_layout.cuh): a repeated lll(0, 0, k) or
size_reduction(0, k) starts at the first row touched since the last such call.  Every mutating entry point must lower
that prefix, and only a call with kappa_min == kappa_start == size_reduction_start == 0 and the same delta and eta may
raise it.  A mistake leaves a stale row on the device that no final basis shows until a later call diverges, so every
test here compares, after every call and for every lattice: the status, n_swaps, zeros, final_kappa and the whole GSO
state.  babai_iterations is not compared: the resume legitimately skips Babai passes that change nothing.

Each case runs on both device LLL kernels (one CTA per lattice, one warp per lattice)."""
import numpy as np
import pytest

import helpers as H
from oracle import oracle as O

pytestmark = pytest.mark.gpu

RED_SUCCESS, RED_GSO_FAILURE, RED_BABAI_FAILURE = 0, 2, 3


@pytest.fixture(scope="module")
def fb():
    import fplll_b200
    return fplll_b200


@pytest.fixture(params=["cta", "warp"])
def lll_mode(request, monkeypatch):
    """Both device LLL kernels: one CTA per lattice (taken for small batches) and one warp per lattice."""
    monkeypatch.setenv("B200_LLL_CTA", "1" if request.param == "cta" else "0")
    return request.param


def device_status(res):
    """The status the device reports for an oracle result.  The reference returns a bool and keeps a status member
    that a fresh LLLReduction starts at RED_SUCCESS.  Where it returns false without setting a status (update_gso_row
    failing at kappa_start, lll.cpp:71-76, or in size_reduction, lll.h:118-119), the device reports RED_GSO_FAILURE."""
    if res["ok"]:
        assert res["status"] == RED_SUCCESS
        return RED_SUCCESS
    return res["status"] if res["status"] != RED_SUCCESS else RED_GSO_FAILURE


class Pair:
    """A device batch and one oracle per lattice, driven call for call; the state is compared after every call."""

    def __init__(self, fb, b, flags=2):
        self.md = fb.MatGSO(b, flags)
        self.mos = [O.OracleGSO(x, flags) for x in b]
        self.k = 0

    def check(self, what):
        st = self.md.state()
        for l, mo in enumerate(self.mos):
            H.assert_state_equal(H.lattice_state(st, l), mo.state(), "call %d %s lattice %d" % (self.k, what, l))
        self.k += 1

    def lll(self, delta=0.99, eta=0.51, kmin=0, kstart=0, kend=-1, srs=0):
        what = "lll(%d, %d, %d, %d) delta %r eta %r" % (kmin, kstart, kend, srs, delta, eta)
        st, stats = self.md.lll(delta, eta, kmin, kstart, kend, srs)
        res = [mo.lll(delta, eta, kmin, kstart, kend, srs) for mo in self.mos]
        for l, r in enumerate(res):
            w = "call %d %s lattice %d" % (self.k, what, l)
            assert st[l] == device_status(r), w + " status"
            assert stats["n_swaps"][l] == r["n_swaps"], w + " n_swaps"
            assert stats["zeros"][l] == r["zeros"], w + " zeros"
            assert stats["final_kappa"][l] == r["final_kappa"], w + " final_kappa"
        self.check(what)
        return res

    def sr(self, eta=0.51, kmin=0, kend=-1, srs=0):
        what = "size_reduction(%d, %d, %d) eta %r" % (kmin, kend, srs, eta)
        st = self.md.size_reduction(eta, kmin, kend, srs)
        res = [mo.size_reduction(eta, kmin, kend, srs) for mo in self.mos]
        for l, r in enumerate(res):
            assert st[l] == device_status(r), "call %d %s lattice %d status" % (self.k, what, l)
        self.check(what)
        return res

    def run(self, ops):
        """entries of helpers.ranged_call_script"""
        for op in ops:
            if op[0] == "lll":
                self.lll(*op[1:])
            elif op[0] == "sr":
                self.sr(*op[1:])
            else:
                for m in [self.md] + self.mos:
                    H.ranged_apply(m, op)
                if op[0] != "update_rows":
                    self.check(str(op))

    def update_rows(self, k):
        self.run([["update_rows", k]])

    def negate(self, i):
        self.md.row_op_begin(i, i + 1)
        self.md.negate_row_of_b(i)
        self.md.row_op_end(i, i + 1)
        for mo in self.mos:
            mo.negate_row_of_b(i)
            mo.row_op_end(i, i + 1)
        self.check("negate_row_of_b(%d)" % i)

    def set_r(self, i, vals):
        self.md.set_r(i, i, vals)
        for l, mo in enumerate(self.mos):
            mo.set_r(i, i, float(vals[l]))
        self.check("set_r(%d, %d)" % (i, i))

    def upload(self, i, rows):
        self.md.upload_row(i, rows)
        for l, mo in enumerate(self.mos):
            mo.upload_row(i, rows[l])
        self.check("upload_row(%d)" % i)

    def apply_ops(self, ops):
        """one b200gso_apply_ops launch on the device, the same calls one by one on the oracle"""
        import fplll_b200.gso as G
        self.md.apply_ops(ops)
        for mo in self.mos:
            for t, a, b, x in ops:
                if t == G.OP_ROW_ADDMUL:
                    mo.row_addmul_we(a, b, x, 0)
                elif t == G.OP_MOVE_ROW:
                    mo.move_row(a, b)
                elif t == G.OP_ROW_SWAP:
                    mo.row_swap(a, b)
                elif t == G.OP_ROW_OP_END:
                    mo.row_op_end(a, b)
                else:
                    mo.negate_row_of_b(a)
        self.check("apply_ops %s" % (ops,))


def _pair(fb, seeds, d, bits=12):
    return Pair(fb, np.stack([H.ranged_inputs(s, d, bits) for s in seeds]))


# ---- ranged shapes ----------------------------------------------------------------------------------------------------

def _edges(d):
    return [e for e in (31, 32, 33, 63, 64, 65, 255, 256, 257) if e < d - 4]


@pytest.mark.parametrize("d", [20, 40, 70, 200, 300])
def test_ranged_shapes(fb, lll_mode, d):
    """BKZ's call shapes, with range ends on the 32-row panel edges: lll(k, k, k+beta) after inserting a row at k
    (BKZ_BOUNDED_LLL, slide reduction), lll(0, 0, k+beta) (svp_preprocessing), size_reduction(m-1, m, m-2) (hkz);
    kappa_start > kappa_min; size_reduction_start at 0, below kappa_min, inside the range and at or above
    kappa_start, in a different panel from the rows it reduces; the smallest ranges and kappa_end = -1.  At d = 300
    the ranges reach the CTA kernel's partly cached mu and its barrier-per-panel UPDATE / BACKSUB with kappa_min > 0."""
    p = _pair(fb, [d, d + 1], d)
    beta = min(24, d // 2)
    edges = _edges(d)
    p.lll(kend=edges[len(edges) // 2] if edges else d // 2)
    p.run([["discover_all"]])  # move_row may only move known rows down (gso.cpp:294)
    if d > 256:  # the edges below 256 are exercised at d = 70 and 200 already
        edges = [32, 64, 255, 256, 257]
    for k in edges + [1, d - beta - 4]:
        kend = min(d, k + beta)
        p.run([["move", d - 1, k]])  # BKZ's insertion: the unreduced last row moves to k
        p.update_rows(k)
        p.lll(kmin=k, kstart=k, kend=kend)
        p.lll(kend=kend)
        p.update_rows(kend - 1)
        p.sr(kmin=kend - 1, kend=kend, srs=kend - 2)
    for k in edges[::2][-3:] + [d // 2]:
        kend = min(d, k + beta + 9)
        lo = max(0, k - 40)
        p.run([["move", d - 1, k - 3], ["addmul", k + 2, lo, 3.0]])
        p.update_rows(k)
        p.lll(kmin=max(0, k - 7), kstart=k, kend=kend)  # kappa_start > kappa_min: the initial babai at kappa_start
        p.run([["addmul", k + 1, lo, -2.0], ["addmul", kend - 1, 1, 5.0]])
        p.update_rows(lo)
        for srs in (0, max(0, lo - 33), min(kend - 1, lo + 33), k):  # 0, below kappa_min, inside, >= kappa_start
            p.lll(kmin=lo, kstart=lo, kend=kend, srs=srs)
        p.run([["addmul", k + 1, 0, 7.0]])
        p.update_rows(lo)
        p.sr(kmin=lo, kend=kend, srs=max(0, lo - 33))
        p.sr(kmin=lo, kend=kend, srs=0)
    k = (edges or [d // 2])[-1]
    p.update_rows(k)
    p.lll(kmin=k, kstart=k, kend=k + 2)  # smallest range
    p.sr(kmin=k, kend=k)  # empty
    p.sr(kmin=0, kend=0)
    p.run([["move", d - 1, k]])
    p.lll(kmin=k, kstart=k, kend=-1)
    p.lll(kend=-1)
    p.sr(kend=-1)


@pytest.mark.parametrize("d", [40, 300])
def test_zero_row_0_quirk(fb, lll_mode, d):
    """lll.cpp:66-69 tests row 0 for zero but moves row kappa_min: with row 0 zero, a call with kappa_min > 0 rotates
    rows [kappa_min, kappa_end) kappa_end - kappa_min times and reduces nothing; lll(0, 0, d) then parks the zero row
    at the end."""
    b = np.stack([H.ranged_inputs(s, d, 10) for s in (7, 8)])
    b[:, 0] = 0
    p = Pair(fb, b)
    p.lll(kmin=5, kstart=5, kend=d - 6)
    p.lll(kmin=3, kstart=9, kend=-1, srs=2)
    p.lll()


@pytest.mark.parametrize("d,kmin", [(70, 33), (300, 257)])
def test_insertion_stops_at_kappa_min(fb, lll_mode, d, kmin):
    """A very short row planted above kappa_min (upload_row, what BKZ's insertion does on the device) fails the Lovasz
    test down to kappa_min: lll(kmin, kmin, kend) must leave it at row kappa_min, not below (lll.cpp:127)."""
    p = _pair(fb, [d + 5, d + 6], d)
    p.lll(kend=d - 3)
    short = np.zeros((2, d + 1), np.int64)
    short[:, 0], short[0, 1], short[1, d] = 1, 1, -1
    i = min(d - 4, kmin + 20)
    p.upload(i, short)
    p.update_rows(kmin)
    p.lll(kmin=kmin, kstart=kmin, kend=i + 3)
    b = p.md.b
    for l in range(2):
        assert np.array_equal(b[l, kmin], short[l]), "lattice %d: the short row is not at kappa_min" % l
    p.lll()


# ---- clean prefix ----------------------------------------------------------------------------------------------------

MUTATIONS = ["addmul", "move_row", "row_swap", "negate", "set_r", "upload_row", "ops_addmul", "ops_move", "ops_swap",
             "ops_row_op_end", "ops_negate"]


def _mutate(p, kind, i):
    """one mutation of row i (inside the clean prefix) through the named entry point"""
    import fplll_b200.gso as G
    if kind == "addmul":
        p.run([["addmul", i, 3, 5.0]])
    elif kind == "move_row":
        p.run([["move", i + 10, i - 20]])
    elif kind == "row_swap":
        p.run([["swap", i - 20, i + 5]])
    elif kind == "negate":
        p.negate(i)
    elif kind == "set_r":
        p.set_r(i, np.array([mo.state()["r"][i, i] * 3.0 for mo in p.mos]))
    elif kind == "upload_row":
        b = p.md.b
        p.upload(i, b[:, i] + 2 * b[:, 3])
    elif kind == "ops_addmul":
        p.apply_ops([(G.OP_ROW_ADDMUL, i, 3, 2.0), (G.OP_ROW_OP_END, i, i + 1, 0.0)])
    elif kind == "ops_move":
        p.apply_ops([(G.OP_MOVE_ROW, i + 10, i - 20, 0.0)])
    elif kind == "ops_swap":
        p.apply_ops([(G.OP_ROW_SWAP, i - 20, i + 5, 0.0), (G.OP_ROW_OP_END, i - 20, i + 6, 0.0)])
    elif kind == "ops_row_op_end":
        p.apply_ops([(G.OP_ROW_ADDMUL, i + 5, 2, -1.0), (G.OP_ROW_ADDMUL, i, 2, 1.0), (G.OP_ROW_OP_END, i, i + 6, 0.0)])
    elif kind == "ops_negate":
        p.apply_ops([(G.OP_NEGATE, i, 0, 0.0), (G.OP_ROW_OP_END, i, i + 1, 0.0)])
    else:
        raise ValueError(kind)


@pytest.mark.parametrize("kind", MUTATIONS)
def test_mutation_lowers_clean_prefix(fb, lll_mode, kind):
    """lll(0,0,d), a mutation of a row inside the clean prefix, size_reduction(0, k); the same mutation again,
    lll(0, 0, d): the device must redo the mutated row as the reference does."""
    d = 70
    p = _pair(fb, [71, 72], d)
    p.lll()
    _mutate(p, kind, 40)
    p.sr(kend=60)
    _mutate(p, kind, 40)
    p.lll()


def test_delta_or_eta_change_between_calls(fb, lll_mode):
    p = _pair(fb, [73, 74], 70)
    p.lll()
    p.lll(delta=0.999)  # a stronger delta: the prefix clean at 0.99 is not clean at 0.999
    p.lll(delta=0.99)
    p.sr(eta=0.501)
    p.lll(eta=0.501)
    p.lll(delta=0.75, eta=0.6)
    p.run([["addmul", 50, 1, 9.0]])
    p.sr(eta=0.6, kend=60)
    p.lll(delta=0.999, eta=0.501)


def test_ranged_call_does_not_clean_rows_below_kappa_min(fb, lll_mode):
    """A mutation below kappa_min, then calls above it that may not raise the clean prefix (kappa_min > 0,
    kappa_start > 0 or size_reduction_start > 0), then lll(0, 0, d): row 10 must still be reduced."""
    p = _pair(fb, [75, 76], 70)
    p.lll()
    p.run([["addmul", 10, 2, 6.0]])
    p.update_rows(40)
    p.lll(kmin=40, kstart=40, kend=70)
    p.lll(kmin=40, kstart=50, kend=70)
    p.lll(kend=70, srs=33)
    p.sr(kend=70, srs=33)
    p.sr(kmin=40, kend=70)
    p.lll()


def test_size_reduction_start_leaves_left_columns_unreduced(fb, lll_mode):
    """size_reduction(0, d, s) with s > 0 reduces row 40 only against rows >= s: mu(40, 3) stays above eta, and the
    prefix may not be marked size-reduced; size_reduction(0, d) then reduces it."""
    p = _pair(fb, [77, 78], 70)
    p.lll()
    p.run([["addmul", 40, 3, 5.0], ["addmul", 45, 38, -4.0]])
    p.sr(srs=33)
    for mo in p.mos:
        s = mo.state()
        assert abs(np.ldexp(s["mu"][40, 3], int(s["row_expo"][40] - s["row_expo"][3]))) > 0.51
    p.sr()
    p.lll()


def test_repeated_lll_is_a_no_op(fb, lll_mode):
    """A second identical lll(0, 0, d) does nothing: 0 swaps, the same state."""
    b = np.random.default_rng(79).integers(-(1 << 12), 1 << 12, size=(2, 200, 201), dtype=np.int64)
    p = Pair(fb, b)
    p.lll()
    before = p.md.state()
    res = p.lll()
    after = p.md.state()
    assert all(r["n_swaps"] == 0 for r in res)
    for l in range(2):
        H.assert_state_equal(H.lattice_state(after, l), H.lattice_state(before, l), "second lll lattice %d" % l)
    p.sr()
    p.lll(kend=150)


# ---- failing calls ---------------------------------------------------------------------------------------------------

def test_ranged_babai_failure_and_next_call(fb, lll_mode):
    """62-bit rows in [20, 40): the ranged lll(20, 20, 40) ends in RED_BABAI_FAILURE; final_kappa, the state left
    behind and the following calls must match."""
    rng = np.random.default_rng(81)
    b = rng.integers(-(1 << 10), 1 << 10, size=(2, 40, 41), dtype=np.int64)
    b[:, 20:] = rng.integers(-(1 << 62), 1 << 62, size=(2, 20, 41), dtype=np.int64)
    p = Pair(fb, b)
    p.lll(kend=20)
    p.update_rows(20)
    res = p.lll(kmin=20, kstart=20, kend=40)
    assert any(r["status"] == RED_BABAI_FAILURE for r in res)
    p.lll(kend=20)
    p.sr(kend=20)
    p.lll()


def test_ranged_gso_failure_at_kappa_start_and_next_call(fb, lll_mode):
    """rows 23 and 24 equal: r(24, 24) = 0, and lll(20, 25, 40) fails in update_gso_row at kappa_start; the next
    lll(0, 0, d) finds the dependency as a zero vector."""
    b = np.stack([H.ranged_inputs(s, 40, 12) for s in (82, 83)])
    b[:, 24] = b[:, 23]
    p = Pair(fb, b)
    p.update_rows(25)
    res = p.lll(kmin=20, kstart=25, kend=40)
    assert all(not r["ok"] and r["final_kappa"] == 25 for r in res)
    p.sr(kmin=10, kend=30)
    res = p.lll()
    assert all(r["zeros"] >= 1 for r in res)


# ---- batches whose lattices diverge ----------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [84, 85])
def test_divergent_batch_random_script(fb, lll_mode, seed):
    """B = 3 lattices of d = 70 driven by one seeded call script (helpers.ranged_call_script): 8-bit entries, a knapsack
    whose column 0 has 30-bit entries, and 16-bit entries with a dependency that a mid-range call finds.  The same
    calls leave each lattice with a different clean prefix."""
    d = 70
    rng = np.random.default_rng(seed)
    b = np.stack([H.ranged_inputs(seed, d, 8), np.zeros((d, d + 1), np.int64), H.ranged_inputs(seed + 1, d, 16)])
    b[1, :, 0] = rng.integers(1, 1 << 30, size=d)
    b[1, np.arange(d), np.arange(d) + 1] = 1
    b[2, 60] = b[2, 38]
    Pair(fb, b).run(H.ranged_call_script(rng, d, 16))


# ---- apply_ops -------------------------------------------------------------------------------------------------------

def _op_list(rng, d, G):
    """A list mixing all five op types in random order: x in {0, +-1, +-7, +-2^40} on rows of small entries, so that
    int64 does not wrap; move_row both ways across panels, including 0 <-> d-1 and 255 -> 257 at d = 300; row_swap,
    row_addmul and negate_row_of_b each closed by the row_op_end that follows it."""
    groups = [[(G.OP_MOVE_ROW, 0, d - 1, 0.0)], [(G.OP_MOVE_ROW, d - 1, 0, 0.0)],
              [(G.OP_MOVE_ROW, 5, min(d - 1, 40), 0.0)], [(G.OP_MOVE_ROW, min(d - 1, 40), 5, 0.0)]]
    if d > 257:
        groups.append([(G.OP_MOVE_ROW, 255, 257, 0.0)])
    i, j = (int(x) for x in rng.choice(d, 2, replace=False))
    groups.append([(G.OP_ROW_SWAP, i, j, 0.0), (G.OP_ROW_OP_END, min(i, j), max(i, j) + 1, 0.0)])
    for x in (0.0, 1.0, -1.0, 7.0, -7.0, float(1 << 40) * (1 if rng.random() < 0.5 else -1)):
        i, j = (int(t) for t in rng.choice(d, 2, replace=False))
        groups.append([(G.OP_ROW_ADDMUL, i, j, x), (G.OP_ROW_OP_END, i, i + 1, 0.0)])
    k = int(rng.integers(0, d))
    groups.append([(G.OP_NEGATE, k, 0, 0.0), (G.OP_ROW_OP_END, k, k + 1, 0.0)])
    return [op for t in rng.permutation(len(groups)) for op in groups[t]]


@pytest.mark.parametrize("d", [40, 65, 200, 300])
def test_apply_ops_equals_individual_calls(fb, lll_mode, d):
    """b200gso_apply_ops (the one launch that carries BKZ's insertions and rerandomisation) against the oracle running
    the same calls one by one, state bit for bit, then lll(0, 0, d) on the result."""
    import fplll_b200.gso as G
    rng = np.random.default_rng(d)
    b = rng.integers(-15, 16, size=(3, d, d + 1), dtype=np.int64)
    p = Pair(fb, b)
    p.lll()
    for _ in range(2):
        p.apply_ops(_op_list(rng, d, G))
        assert np.abs(p.md.b).max() < (1 << 62)
        p.lll()


def test_apply_ops_refuses_bad_ops(fb):
    import fplll_b200.gso as G
    md = fb.MatGSO(H.ranged_inputs(86, 40, 10))
    for ops in ([(0, 1, 2, 0.0)], [(6, 1, 2, 0.0)], [(G.OP_ROW_ADDMUL, 40, 1, 1.0)], [(G.OP_MOVE_ROW, 1, -1, 0.0)],
                [(G.OP_ROW_SWAP, -1, 3, 0.0)], [(G.OP_NEGATE, 40, 0, 0.0)], [(G.OP_ROW_OP_END, 5, 4, 0.0)],
                [(G.OP_ROW_OP_END, 5, 41, 0.0)], [(G.OP_ROW_ADDMUL, 3, 1, 1.0), (0, 0, 0, 0.0)]):
        with pytest.raises(fb.B200Error):
            md.apply_ops(ops)
    assert np.array_equal(md.b[0], H.ranged_inputs(86, 40, 10))  # a refused list runs none of its ops


# ---- refusals --------------------------------------------------------------------------------------------------------

def test_bad_ranges_are_refused(fb):
    md = fb.MatGSO(H.ranged_inputs(87, 40, 10))
    for args in ((5, 4, 20, 0), (5, 20, 20, 0), (5, 25, 20, 0), (0, 0, 41, 0), (0, 0, 20, -1)):
        with pytest.raises(fb.B200Error):
            md.lll(0.99, 0.51, *args)
    for args in ((5, 4, 0), (0, 41, 0), (0, 20, -1)):
        with pytest.raises(fb.B200Error):
            md.size_reduction(0.51, *args)


# ---- the reference's own calls ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", [0, 1, 2])
def test_ranged_scripts_vs_reference_fixture(fb, lll_mode, case):
    """The call scripts of tests/golden/lll_ranged_ref.npz (make_golden.py --ranged): the reference's per-call results
    and state digests, and at d <= 64 its state after every call."""
    import json
    z = H.gold("lll_ranged_ref.npz")
    p = "c%d_" % case
    ops = json.loads(bytes(z[p + "ops_json"]).decode())
    md = fb.MatGSO(z[p + "b"].astype(np.int64))
    t = 0
    for op in ops:
        r = H.ranged_apply(md, op)
        if r is None:
            continue
        ok, status, swaps, final_kappa, zeros = (int(x) for x in z[p + "res"][t])
        what = "case %d call %d %s" % (case, t, op)
        st = r[0] if op[0] == "lll" else r
        assert st[0] == device_status(dict(ok=ok, status=status)), what + " status"
        if op[0] == "lll":
            assert r[1]["n_swaps"][0] == swaps, what + " n_swaps"
            assert r[1]["final_kappa"][0] == final_kappa, what + " final_kappa"
            assert r[1]["zeros"][0] == zeros, what + " zeros"
        s = H.lattice_state(md.state(), 0)
        if p + "s_mu" in z:
            ref = {k: z[p + "s_" + k][t] for k in ["n_known_rows", "n_known_cols", "n_source_rows", "row_expo",
                                                  "gso_valid_cols", "init_row_size", "b", "bf", "gf", "mu", "r"]}
            ref["b"] = ref["b"].astype(np.int64)
            H.assert_state_equal(s, ref, what)
        assert H.gso_digest(s) == z[p + "digest"][t], what + " digest"
        t += 1
    assert t == len(z[p + "res"])
    if p + "b_out" in z:
        assert np.array_equal(md.b[0], z[p + "b_out"])
