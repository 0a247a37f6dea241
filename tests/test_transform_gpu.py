"""GPU tests of the transform U (B200GSO_TRANSFORM, include/b200gso.h): every integer row operation the device applies
to b — single calls, op lists, the warp and CTA LLL kernels, size reduction, the BKZ driver, the interposer's BKZ
take-over — is applied to U as well, and U never changes a decision.

What is checked, against tests/golden/transform_ref.npz (made by make_transform_golden.py from the reference):
  * a transform handle ends every call with the b, GSO state, status and statistics of the same call without U;
  * U is the reference's U bit for bit, except after a negation of a row of b, which the reference does not apply to
    its u and the device does (the one intended divergence);
  * U * B_in == B (mod 2^64 for the op scripts, which wrap; exactly over the integers for the reductions) and
    det U = +-1 modulo a few 31-bit primes."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

import helpers as H

pytestmark = pytest.mark.gpu

PRIMES = (2147483647, 2147483629, 2147483587)


@pytest.fixture(scope="module")
def fb():
    import fplll_b200
    return fplll_b200


@pytest.fixture(scope="module")
def z():
    return H.gold("transform_ref.npz")


def identity_mod64(u, b0, b):
    """U * B0 == B mod 2^64 (numpy's integer matmul wraps)"""
    return np.array_equal(u.astype(np.uint64) @ b0.astype(np.uint64), b.astype(np.uint64))


def identity_exact(u, b0, b):
    """U * B0 == B over the integers (in int64 when no partial sum can overflow, else over Python integers)"""
    if int(np.abs(u).max()) * int(np.abs(b0).max()) * u.shape[1] < 2 ** 62:
        return np.array_equal(u @ b0, b)
    return np.array_equal(np.dot(u.astype(object), b0.astype(object)), b.astype(object))


def det_mod(u, p):
    a = np.mod(u.astype(object), p).astype(np.int64)
    n, det = a.shape[0], 1
    for c in range(n):
        piv = next((r for r in range(c, n) if a[r, c]), None)
        if piv is None:
            return 0
        if piv != c:
            a[[c, piv]] = a[[piv, c]]
            det = -det
        det = det * int(a[c, c]) % p
        inv = pow(int(a[c, c]), p - 2, p)
        f = (a[c + 1:, c] * inv) % p
        a[c + 1:] = (a[c + 1:] - np.outer(f, a[c]) % p) % p
    return det % p


def unimodular(u):
    return all(det_mod(u, p) in (1, p - 1) for p in PRIMES)


def pair(fb, b):
    """the same basis on a plain handle and on a transform handle (U = identity)"""
    return fb.MatGSO(b), fb.MatGSO(b, fb.GSO_ROW_EXPO | fb.GSO_TRANSFORM)


def same_state(m, mt, what):
    s, st = m.state(), mt.state()
    for l in range(m.batch):
        H.assert_state_equal(H.lattice_state(st, l), H.lattice_state(s, l), "%s lattice %d" % (what, l))


# ---- op scripts -------------------------------------------------------------------------------------------------------
def run_group(fb, m, ops, as_list):
    if as_list:
        lst = []
        for k, *a in ops:
            if k == "addmul":  # x * 2^e is what row_addmul_we(i, j, x, e) multiplies by (get_si_exp_we)
                lst += [(fb.OP_ROW_ADDMUL, a[0], a[1], a[2] * 2.0 ** a[3]), (fb.OP_ROW_OP_END, a[0], a[0] + 1, 0)]
            elif k == "swap":
                lst += [(fb.OP_ROW_SWAP, a[0], a[1], 0), (fb.OP_ROW_OP_END, a[0], a[1] + 1, 0)]
            elif k == "move":
                lst.append((fb.OP_MOVE_ROW, a[0], a[1], 0))
            else:
                lst += [(fb.OP_NEGATE, a[0], 0, 0), (fb.OP_ROW_OP_END, a[0], a[0] + 1, 0)]
        m.apply_ops(lst)
    else:
        for k, *a in ops:
            if k == "addmul":
                m.row_addmul_we(a[0], a[1], a[2], a[3])
                m.row_op_end(a[0], a[0] + 1)
            elif k == "swap":
                m.row_swap(a[0], a[1])
                m.row_op_end(a[0], a[1] + 1)
            elif k == "move":
                m.move_row(a[0], a[1])
            else:
                m.negate_row_of_b(a[0])
                m.row_op_end(a[0], a[0] + 1)
    assert m.update_gso().all()


@pytest.mark.parametrize("script", [0, 1])
@pytest.mark.parametrize("as_list", [False, True], ids=["calls", "op_list"])
def test_op_scripts_follow_the_reference_u(fb, z, script, as_list):
    """row_addmul_we (with 2^e shifts, some wrapping), row_swap, move_row both ways and negate_row_of_b on two lattices
    at once: after every group the state equals the plain handle's, U equals the reference's until the first group
    with a negation, and U * B0 == B mod 2^64 throughout."""
    groups = json.loads(bytes(z["ops%d_script" % script]).decode())
    b0 = z["ops%d_b_in" % script]
    b = np.stack([b0, b0])
    m, mt = pair(fb, b)  # the fixture's object has GSO_OP_FORCE_LONG, which the device implies
    assert m.update_gso().all() and mt.update_gso().all()
    assert np.array_equal(mt.u, np.stack([np.eye(40, dtype=np.int64)] * 2))
    negated = False
    for g, ops in enumerate(groups):
        run_group(fb, m, ops, as_list)
        run_group(fb, mt, ops, as_list)
        same_state(m, mt, "group %d" % g)
        negated |= any(o[0] == "negate" for o in ops)
        u, bb = mt.u, mt.b
        for l in range(2):
            assert identity_mod64(u[l], b0, bb[l]), "group %d lattice %d" % (g, l)
            if not negated:
                assert np.array_equal(u[l], z["ops%d_u" % script][g]), "group %d lattice %d" % (g, l)
    assert negated and np.array_equal(mt.b[0], z["ops%d_b_out" % script])


# ---- LLL --------------------------------------------------------------------------------------------------------------
def lll_pair(fb, b):
    m, mt = pair(fb, b)
    st, stats = m.lll(0.99, 0.51)
    stt, statst = mt.lll(0.99, 0.51)
    assert np.array_equal(st, stt)
    for k in stats:
        assert np.array_equal(stats[k], statst[k]), k
    same_state(m, mt, "after lll")
    return stt, mt.b, mt.u


@pytest.mark.parametrize("tag,kernel", [("lll_u40", "cta"), ("lll_u40", "warp"), ("lll_r200", "cta"),
                                        ("lll_rankdef", "cta"), ("lll_rankdef", "warp")])
def test_lll_u_equals_the_reference(fb, z, monkeypatch, tag, kernel):
    """One lattice (the CTA kernel, or the warp kernel with B200_LLL_CTA=0), d = 40, 200 and a rank-deficient 40 x 41
    basis whose ten zero rows leave U undetermined by B: same state as without U, the reference's b and U."""
    monkeypatch.setenv("B200_LLL_CTA", "1" if kernel == "cta" else "0")
    b_in = z[tag + "_b_in"]
    st, b, u = lll_pair(fb, b_in[None])
    assert st[0] == int(z[tag + "_status"]) == 0
    assert np.array_equal(b[0], z[tag + "_b_out"])
    assert bool(z[tag + "_consistent"])
    assert np.array_equal(u[0], z[tag + "_u"])
    assert identity_exact(u[0], b_in, b[0]) and unimodular(u[0])


def test_lll_warp_kernel_on_a_full_batch(fb, z):
    """3 x 132 lattices (the one-warp-per-lattice kernel): u 40 inputs of config #1 and the rank-deficient basis's
    rows in other orders; the lattices that are the fixture's inputs end on the reference's U."""
    rng = np.random.default_rng(3)
    u40, rd = z["lll_u40_b_in"], z["lll_rankdef_b_in"][:, :40]
    b = np.stack([u40 if l % 3 == 0 else (rd[rng.permutation(40)] if l % 3 == 1 else
                                          rng.integers(-(1 << 30), 1 << 30, size=(40, 40), dtype=np.int64))
                  for l in range(396)])
    st, bo, u = lll_pair(fb, b)
    assert (st == 0).all()
    for l in range(396):
        if l % 3 == 0:
            assert np.array_equal(u[l], z["lll_u40_u"]), l
        assert identity_mod64(u[l], b[l], bo[l]), l
    for l in range(0, 396, 37):
        assert identity_exact(u[l], b[l], bo[l]) and unimodular(u[l]), l


def test_cta_lll_above_256_rows(fb):
    """d = 260 (partial mu cache, a barrier per panel in the CTA kernel): a knapsack basis [x | I], whose U is the
    identity part of the reduced basis."""
    rng = np.random.default_rng(8)
    d = 260
    b = np.zeros((d, d + 1), np.int64)
    b[:, 0] = rng.integers(1, 1 << 40, size=d)
    b[:, 1:] = np.eye(d, dtype=np.int64)
    st, bo, u = lll_pair(fb, b[None])
    assert st[0] == 0
    assert np.array_equal(u[0], bo[0][:, 1:])
    assert identity_exact(u[0], b, bo[0]) and unimodular(u[0])


# ---- ranged calls -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,d,kernel", [(1, 70, "cta"), (2, 70, "warp"), (3, 40, "cta")])
def test_ranged_calls_on_one_continuing_handle(fb, monkeypatch, seed, d, kernel):
    """helpers.ranged_call_script (ranged lll, size_reduction, row_addmul / row_swap / move_row insertions): after every
    call the transform handle's status and state equal the plain handle's, and U * B_in == B."""
    monkeypatch.setenv("B200_LLL_CTA", "1" if kernel == "cta" else "0")
    b = H.ranged_inputs(seed, d, 24)
    m, mt = pair(fb, b[None])
    for k, op in enumerate(H.ranged_call_script(np.random.default_rng(seed), d, 30)):
        r, rt = H.ranged_apply(m, op), H.ranged_apply(mt, op)
        if op[0] == "lll":
            assert np.array_equal(r[0], rt[0]) and all(np.array_equal(r[1][q], rt[1][q]) for q in r[1]), k
        elif op[0] == "sr":
            assert np.array_equal(r, rt), k
        same_state(m, mt, "call %d %s" % (k, op[0]))
        assert identity_exact(mt.u[0], b, mt.b[0]), k


def test_apply_ops_list_with_every_op_type(fb):
    """one op list with all five op types on a batch of three different lattices"""
    rng = np.random.default_rng(2)
    b = rng.integers(-(1 << 20), 1 << 20, size=(3, 24, 26), dtype=np.int64)
    m, mt = pair(fb, b)
    assert m.update_gso().all() and mt.update_gso().all()
    ops = [(fb.OP_ROW_ADDMUL, 5, 2, 3.0), (fb.OP_ROW_OP_END, 5, 6, 0), (fb.OP_MOVE_ROW, 20, 3, 0),
           (fb.OP_ROW_SWAP, 1, 7, 0), (fb.OP_ROW_OP_END, 1, 8, 0), (fb.OP_NEGATE, 4, 0, 0), (fb.OP_ROW_OP_END, 4, 5, 0),
           (fb.OP_MOVE_ROW, 2, 22, 0), (fb.OP_ROW_ADDMUL, 0, 23, -5.0 * 2.0 ** 62), (fb.OP_ROW_OP_END, 0, 1, 0)]
    m.apply_ops(ops)
    mt.apply_ops(ops)
    assert m.update_gso().all() and mt.update_gso().all()
    same_state(m, mt, "op list")
    u = mt.u
    for l in range(3):
        assert identity_mod64(u[l], b[l], mt.b[l]), l


# ---- BKZ --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag,golden,key", [("bkz20", "bkz_q60.npz", "bkz20_none"),
                                            ("sd20", "bkz_sd_sld.npz", "sd20_none"),
                                            ("sld20", "bkz_sd_sld.npz", "sld20_none")])
def test_bkz_without_pruning_u_equals_the_reference(fb, z, tag, golden, key):
    """b200bkz_reduce_transform through bkz_reduction(u=...): the golden b, the reference's U where the reference's U is
    consistent, U * B_in == B_out always."""
    g = H.gold(golden)
    b_in = z["q60_b_in"]
    b, u = b_in.copy(), np.zeros((60, 60), np.int64)
    st, _ = fb.bkz_reduction(b, fb.BKZParam(20, flags=int(z[tag + "_flags"]), max_loops=int(z[tag + "_max_loops"])),
                             u=u)
    assert st == int(z[tag + "_status"]) == int(g[key + "_status"])
    assert np.array_equal(b, g[key + "_b"]) and np.array_equal(b, z[tag + "_b_out"])
    if bool(z[tag + "_consistent"]):
        assert np.array_equal(u, z[tag + "_u"])
    assert identity_exact(u, b_in, b) and unimodular(u)


def test_bkz40_on_dim180_with_u(fb):
    """BKZ-40 on the dim-180 Goldstein-Mayer basis, one tour: the reference's output basis, and U * B_in == B_out"""
    g = H.gold("bkz_gm180.npz")
    b, u = g["b_in"].copy(), np.zeros((180, 180), np.int64)
    st, _ = fb.bkz_reduction(b, fb.BKZParam(40, flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS, max_loops=1), u=u)
    assert st == int(g["bkz40_none_status"])
    assert np.array_equal(b, g["bkz40_none_b"])
    assert identity_exact(u, g["b_in"], b) and unimodular(u)


@pytest.mark.parametrize("bs", [30, 40])
def test_pruned_bkz_with_u_takes_the_same_decisions(fb, z, bs):
    """pruned BKZ with default strategies (rerandomisation, preprocessing, negations in the post-processing): b and
    every statistic except the timings equal the run without U, and U * B_in == B_out"""
    b_in = z["q60_b_in"]
    par = fb.BKZParam(bs, strategies="default", flags=fb.BKZ_NO_LLL | fb.BKZ_MAX_LOOPS, max_loops=2)
    b0, b1, u = b_in.copy(), b_in.copy(), np.zeros((60, 60), np.int64)
    st0, s0 = fb.bkz_reduction(b0, par)
    st1, s1 = fb.bkz_reduction(b1, par, u=u)
    assert st0 == st1 == 8
    assert np.array_equal(b0, b1)
    for k in s0:
        if not k.startswith("sec_"):
            assert s0[k] == s1[k], k
    assert identity_exact(u, b_in, b1) and unimodular(u)


# ---- the C-ABI's refusals and the Python surface ----------------------------------------------------------------------
def test_refusals(fb):
    from fplll_b200 import gso
    L = gso._lib()
    h = C.c_void_p()
    assert L.b200gso_create(C.byref(h), 1, 8, 8, fb.GSO_TRANSFORM | 256, 0) == -1  # with B200GSO_HOST_BASIS
    b = np.arange(64, dtype=np.int64).reshape(8, 8) + np.eye(8, dtype=np.int64) * 100
    mt, m = fb.MatGSO(b, fb.GSO_ROW_EXPO, u=np.eye(8, dtype=np.int64)), fb.MatGSO(b)
    row = np.ones(8, np.int64)
    assert L.b200gso_upload_row(mt._h, 0, row.ctypes.data_as(C.POINTER(C.c_int64))) == -1
    assert L.b200gso_upload_row(m._h, 0, row.ctypes.data_as(C.POINTER(C.c_int64))) == 0
    uu = np.zeros((8, 8), np.int64)
    assert L.b200gso_get_transform(m._h, uu.ctypes.data_as(C.POINTER(C.c_int64))) == -1
    assert L.b200gso_set_transform(m._h, uu.ctypes.data_as(C.POINTER(C.c_int64))) == -1
    # set_transform replaces U, set_basis leaves it alone, negate_row_of_b negates the row of U
    u = np.arange(64, dtype=np.int64).reshape(8, 8)
    mt.set_transform(u)
    L.b200gso_set_basis(mt._h, b.ctypes.data_as(C.POINTER(C.c_int64)))
    assert np.array_equal(mt.u[0], u)
    mt.negate_row_of_b(3)
    u[3] = -u[3]
    assert np.array_equal(mt.u[0], u)


def test_lll_reduction_with_u_and_zeros_first(fb, z):
    """lll_reduction(b, u=u): the b of the call without u; zeros_first moves the matching rows of u to the front"""
    b_in = z["lll_rankdef_b_in"]
    b0, b1, u = b_in.copy(), b_in.copy(), np.full((40, 40), 7, np.int64)
    assert fb.lll_reduction(b0) == fb.lll_reduction(b1, u=u) == 0
    assert np.array_equal(b0, b1)
    assert not b1[:10].any() and np.all(np.any(b1[10:] != 0, axis=1))
    assert identity_exact(u, b_in, b1) and unimodular(u)
    ref = z["lll_rankdef_u"]  # LLL parks the zero rows at the end: zeros_first rotates them (and their U rows) first
    assert np.array_equal(u, np.concatenate([ref[30:], ref[:30]]))
    bb, uu = np.stack([b_in, b_in]), np.zeros((2, 40, 40), np.int64)
    assert (fb.lll_reduction(bb, u=uu) == 0).all() and np.array_equal(uu[1], u)


def test_bkz_reduction_with_u_same_b(fb, z):
    b_in = z["q60_b_in"]
    b0, b1, u = b_in.copy(), b_in.copy(), np.zeros((60, 60), np.int64)
    par = fb.BKZParam(10, flags=fb.BKZ_MAX_LOOPS, max_loops=1)
    assert fb.bkz_reduction(b0, par)[0] == fb.bkz_reduction(b1, par, u=u)[0]
    assert np.array_equal(b0, b1) and identity_exact(u, b_in, b1)


# ---- the interposer ---------------------------------------------------------------------------------------------------
def test_cli_bkz_with_u_through_the_shim(tmp_path):
    """`fplll -a bkz -b 20 -f double -of bu` on the dim-60 q-ary basis, plain and with libb200fplll.so preloaded: the same
    b, and the same U (or, where the reference's U is not a transform of its own input, a U that is); the preloaded run
    took bkz() over."""
    import subprocess
    from oracle import oracle as O
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    shim, cli = os.path.join(root, "tests", "_build", "libb200fplll.so"), os.path.join(root, "oracle", "_ref", "fplll")
    for p in (shim, cli):
        if not os.path.exists(p):
            pytest.skip("%s not built (needs the reference headers: built in the development container)" % p)
    b_in = H.gold("bkz_q60.npz")["b_in"]
    inp = str(tmp_path / "in.txt")
    O.write_matrix(inp, b_in)
    outs = []
    for preload in (False, True):
        env = dict(os.environ)
        env.pop("LD_PRELOAD", None)
        if preload:
            env.update(LD_PRELOAD=shim, B200_SHIM_STATS="1")
        p = subprocess.run([cli, "-a", "bkz", "-b", "20", "-f", "double", "-of", "bu", inp], capture_output=True,
                           text=True, timeout=900, env=env)
        assert p.returncode == 0, p.stderr[-1500:]
        if preload:
            line = [l for l in p.stderr.splitlines() if "b200 MatGSO shim" in l][-1]
            assert int(line.split("device driver ")[1].split()[0]) >= 1, line
        mats = []
        for blk in [t for t in re.split(r"(?m)^(?=\[\[)", p.stdout) if t.strip()]:  # "-of bu": b, then u
            f = tmp_path / "m.txt"
            f.write_text(blk)
            mats.append(np.array(O.read_matrix(str(f)), dtype=np.int64))
        assert len(mats) == 2
        outs.append(mats)
    (b_ref, u_ref), (b_dev, u_dev) = outs
    assert np.array_equal(b_ref, b_dev) and np.array_equal(b_dev, H.gold("bkz_q60.npz")["bkz20_none_b"])
    if identity_exact(u_ref, b_in, b_ref):
        assert np.array_equal(u_ref, u_dev)
    assert identity_exact(u_dev, b_in, b_dev) and unimodular(u_dev)
