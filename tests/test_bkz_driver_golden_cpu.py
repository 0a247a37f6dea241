"""CPU checks of tests/golden/bkz_driver_ref.npz (the reference's whole bkz_reduction call, made by make_bkz_golden.py),
which tests/test_bkz_driver_gpu.py compares the device driver against: the recorded outputs are what the fixture says
they are — bases of the input lattice, LLL-reduced, zero rows first — and every case exercises what its name claims."""
import json

import numpy as np
import pytest

import helpers as H

Z = H.gold("bkz_driver_ref.npz")
TAGS = json.loads(bytes(Z["tags"]).decode())
NO_LLL, MAX_LOOPS, BOUNDED_LLL, AUTO_ABORT, SD, SLD = 2, 4, 0x10, 0x20, 0x100, 0x200


def exact(a):
    return a.astype(object)


def gram_det(b):
    """det(B B^T) of the nonzero rows, exactly (fraction-free Gaussian elimination, Bareiss)"""
    rows = [r for r in exact(b) if any(r)]
    g = [[sum(x * y for x, y in zip(r, s)) for s in rows] for r in rows]
    n, prev = len(g), 1
    for k in range(n - 1):
        if g[k][k] == 0:
            piv = next(i for i in range(k + 1, n) if g[i][k] != 0)
            g[k], g[piv] = g[piv], g[k]
        for i in range(k + 1, n):
            for j in range(k + 1, n):
                g[i][j] = (g[i][j] * g[k][k] - g[i][k] * g[k][j]) // prev
        prev = g[k][k]
    return abs(g[n - 1][n - 1]) if n else 1


def zero_rows(b):
    return [i for i, r in enumerate(b) if not r.any()]


def test_fixture_has_every_kind_of_case():
    assert len(TAGS) >= 30
    flags = {t: int(Z[t + "_flags"]) for t in TAGS}
    assert sum(not f & NO_LLL for f in flags.values()) >= 10  # preliminary LLL
    assert {float(Z[t + "_delta"]) for t in TAGS if not flags[t] & NO_LLL} == {0.75, 0.99}
    conv = [t for t in TAGS if not flags[t] & (MAX_LOOPS | AUTO_ABORT)]
    assert any(int(Z[t + "_tours"]) > 20 for t in conv)  # runs to convergence
    aa = {(float(Z[t + "_aa_scale"]), int(Z[t + "_aa_max_no_dec"])) for t in TAGS if flags[t] & AUTO_ABORT}
    assert {(1.0, 5), (1.0, 1), (1.02, 2)} <= aa
    # block sizes 2, 3, d - 1, d, d + 5 of the dim-30 basis, a 40 x 60 basis, SD and SLD on a rank-deficient basis
    assert {int(Z[t + "_block"]) for t in TAGS if Z[t + "_b_in"].shape == (30, 30)} == {2, 3, 29, 30, 35}
    assert any(Z[t + "_b_in"].shape == (40, 60) for t in TAGS)
    rd = [t for t in TAGS if len(zero_rows(Z[t + "_b_out"]))]
    assert any(flags[t] & SD for t in rd) and any(flags[t] & SLD for t in rd)
    assert any(json.loads(bytes(Z[t + "_strategies"]).decode()) for t in TAGS)
    assert sum(bool(Z[t + "_with_u"]) for t in TAGS) >= 5


@pytest.mark.parametrize("tag", TAGS)
def test_output_is_an_lll_reduced_basis_of_the_input_lattice_with_zero_rows_first(tag):
    b_in, b_out, lll_out = Z[tag + "_b_in"], Z[tag + "_b_out"], Z[tag + "_lll_out"]
    assert b_out.shape == b_in.shape == lll_out.shape
    assert int(Z[tag + "_status"]) in (0, 8) and int(Z[tag + "_lll_status"]) == 0
    # zeros_first (bkz.cpp:925) and lll_reduction's own zeros_first: the zero rows are the leading ones
    for b in (b_out, lll_out):
        z = zero_rows(b)
        assert z == list(range(len(z))), z
    nz = len(zero_rows(b_out))
    assert nz == len(zero_rows(lll_out))
    # the same lattice as the wrapper LLL's output (and so as the input): same rank, same Gram determinant, exactly
    det = gram_det(b_out)
    assert det == gram_det(lll_out) and det > 0
    if not nz:
        assert det == gram_det(b_in)
    # BKZ_BOUNDED_LLL ("use at your own risk", bkz_param.h:85) LLL-reduces each block from kappa on, so the rows it
    # changes are not size-reduced against the rows before the block: the reference's output is not LLL-reduced then
    bounded = bool(int(Z[tag + "_flags"]) & BOUNDED_LLL)
    assert H.is_lll_reduced(b_out[nz:], float(Z[tag + "_delta"]), 0.51) != bounded


@pytest.mark.parametrize("tag", [t for t in TAGS if bool(Z[t + "_with_u"])])
def test_reference_u_is_what_the_flag_says(tag):
    b_in, b_out, u = Z[tag + "_b_in"], Z[tag + "_b_out"], Z[tag + "_u"]
    ok = np.array_equal(np.dot(exact(u), exact(b_in)), exact(b_out))
    assert ok == bool(Z[tag + "_consistent"])
    # the same call without U ends on the same basis (the tag without "_u", where the fixture has it)
    twin = tag[:-2]
    if twin in TAGS:
        assert np.array_equal(Z[twin + "_b_out"], b_out) and int(Z[twin + "_tours"]) == int(Z[tag + "_tours"])


def test_tour_counts_follow_the_termination_flags():
    for t in TAGS:
        fl, tours = int(Z[t + "_flags"]), int(Z[t + "_tours"])
        if fl & MAX_LOOPS:
            assert tours <= int(Z[t + "_max_loops"]), t
        if int(Z[t + "_block"]) >= Z[t + "_b_in"].shape[0] - len(zero_rows(Z[t + "_b_out"])):
            assert tours == 1, t  # a block at least as large as the rank: one HKZ pass
        assert tours >= 1, t
