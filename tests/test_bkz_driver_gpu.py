"""GPU tests of the whole BKZ driver call (fplll_b200.bkz_reduction, include/b200bkz.h) against the reference's own
bkz_reduction (tests/golden/bkz_driver_ref.npz, made by make_bkz_golden.py): the preliminary LLL at both deltas, runs
to convergence, BKZ_AUTO_ABORT at several settings, SD-BKZ's implicit auto-abort, BKZ_GH_BND around block size 30 with
two GH factors, preprocessing strategies without pruning, BKZ_BOUNDED_LLL, block sizes from 2 to past the rank, a
non-square basis, rank-deficient bases (zeros_last, trailing zero rows outside the tours, zeros_first) and U.

No case prunes, so no call rerandomises and every unpruned enumeration returns the shortest vector of its ball: the
device must end on the reference's status, basis and tour count bit for bit, and on its U wherever the reference's U
satisfies U * B_in = B_out.  Strategies are the dict form with no pruning vector (b200bkz_add_strategy with n_prune = 0),
which the driver completes with PruningParams() as load_strategies_json does.

The device's preliminary LLL is one fp64 LLL(delta, 0.51); the reference's is its wrapper (heuristic LLL, then a proved
LLL at the precision the dimension needs).  On every case here both end on the same basis, which each case checks first
(_lll_out), so that a divergence is placed in the LLL or in BKZ."""
import json

import numpy as np
import pytest

import helpers as H

pytestmark = pytest.mark.gpu

Z = H.gold("bkz_driver_ref.npz")
TAGS = json.loads(bytes(Z["tags"]).decode())
NO_LLL = 2
PRIMES = (2147483647, 2147483629, 2147483587)


@pytest.fixture(scope="module")
def fb():
    import fplll_b200
    return fplll_b200


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


def strategies(tag):
    """{block_size: (preprocessing, gh_factor, expectation, coefficients)} with no pruning vector"""
    pre = json.loads(bytes(Z[tag + "_strategies"]).decode())
    if not pre:
        return None
    empty = np.zeros(0)
    return {int(k): (np.array(v, np.int32), empty, empty, empty) for k, v in pre.items()}


def param(fb, tag):
    return fb.BKZParam(int(Z[tag + "_block"]), strategies=strategies(tag), delta=float(Z[tag + "_delta"]),
                       flags=int(Z[tag + "_flags"]), max_loops=int(Z[tag + "_max_loops"]),
                       auto_abort_scale=float(Z[tag + "_aa_scale"]), auto_abort_max_no_dec=int(Z[tag + "_aa_max_no_dec"]),
                       gh_factor=float(Z[tag + "_gh_factor"]))


def zeros_first(b):
    """the reference's lll_reduction output order: zero rows first"""
    z = [i for i, r in enumerate(b) if not r.any()]
    return np.concatenate([b[z], b[[i for i in range(len(b)) if i not in z]]])


def with_lll(tag):
    """cases whose device run starts with the preliminary LLL or holds zero rows: both LLL kernels"""
    return not int(Z[tag + "_flags"]) & NO_LLL or not Z[tag + "_b_out"][0].any()


CASES = [pytest.param(t, k, id="%s-%s" % (t, k)) for t in TAGS for k in (("cta", "warp") if with_lll(t) else ("cta",))]


@pytest.mark.parametrize("tag,lll_kernel", CASES)
def test_driver_call_equals_reference_bkz_reduction(fb, tag, lll_kernel, monkeypatch):
    monkeypatch.setenv("B200_LLL_CTA", "1" if lll_kernel == "cta" else "0")
    b_in = Z[tag + "_b_in"]
    if not int(Z[tag + "_flags"]) & NO_LLL:
        # the preliminary LLL alone: the device's LLL(delta, 0.51) ends where the reference's wrapper LLL does
        m = fb.MatGSO(b_in[None].copy())
        st, _ = m.lll(float(Z[tag + "_delta"]), 0.51)
        assert int(st[0]) == int(Z[tag + "_lll_status"]) == 0
        assert np.array_equal(zeros_first(m.b[0]), Z[tag + "_lll_out"]), "preliminary LLL differs from the wrapper's"
    b = b_in.copy()
    u = np.zeros((b.shape[0], b.shape[0]), np.int64) if bool(Z[tag + "_with_u"]) else None
    st, stats = fb.bkz_reduction(b, param(fb, tag), u=u)
    assert st == int(Z[tag + "_status"])
    assert int(stats["tours"]) == int(Z[tag + "_tours"])
    assert np.array_equal(b, Z[tag + "_b_out"])
    if u is None:
        return
    assert np.array_equal(u.astype(np.uint64) @ b_in.astype(np.uint64), b.astype(np.uint64))
    assert all(det_mod(u, p) in (1, p - 1) for p in PRIMES)
    assert bool(Z[tag + "_consistent"])
    if int(Z[tag + "_flags"]) & NO_LLL:
        assert np.array_equal(u, Z[tag + "_u"])
        return
    # With U, the reference's wrapper LLL runs on mpz integers (wrapper.cpp:287-290).  On a full-rank basis its U is the
    # one the device's LLL tracks; on a rank-deficient one it is not: both end on the same basis, but the row operations
    # that involve the rows which become zero differ, and so does U, by vectors of the kernel (DESIGN.md §3.6).  Pin the
    # BKZ part exactly there: the device's U of the same call run from the wrapper's output under BKZ_NO_LLL, composed
    # with the wrapper's own U, is the reference's U.
    if Z[tag + "_b_out"][0].any():
        assert np.array_equal(u, Z[tag + "_u"])
    b2, u2 = Z[tag + "_lll_out"].copy(), np.zeros_like(u)
    p2 = param(fb, tag)
    p2.flags |= NO_LLL
    st2, stats2 = fb.bkz_reduction(b2, p2, u=u2)
    assert st2 == st and int(stats2["tours"]) == int(stats["tours"]) and np.array_equal(b2, b)
    assert np.array_equal(np.dot(u2.astype(object), Z[tag + "_lll_u"].astype(object)), Z[tag + "_u"].astype(object))
