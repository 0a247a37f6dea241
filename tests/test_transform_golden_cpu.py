"""CPU checks of tests/golden/transform_ref.npz (the reference's transform U, made by make_transform_golden.py), which
tests/test_transform_gpu.py compares the device's U against: the recorded consistency flags are what they claim, the
fixture's bases are those of the existing goldens, and the reference's own U breaks U * B_in == B_out exactly where its
negate_row_of_b leaves u alone."""
import json

import numpy as np

import helpers as H

LLL_TAGS, BKZ_TAGS = ("lll_u40", "lll_r200", "lll_rankdef"), ("bkz20", "sd20", "sld20")


def identity_exact(u, b0, b):
    """U * B0 == B over the integers (in int64 when no partial sum can overflow, else over Python integers)"""
    if int(np.abs(u).max()) * int(np.abs(b0).max()) * u.shape[1] < 2 ** 62:
        return np.array_equal(u @ b0, b)
    return np.array_equal(np.dot(u.astype(object), b0.astype(object)), b.astype(object))


def test_consistency_flags_are_what_they_claim():
    z = H.gold("transform_ref.npz")
    for tag in LLL_TAGS:
        assert bool(z[tag + "_consistent"]) == identity_exact(z[tag + "_u"], z[tag + "_b_in"], z[tag + "_b_out"]), tag
        assert bool(z[tag + "_consistent"]), tag
    for tag in BKZ_TAGS:
        assert bool(z[tag + "_consistent"]) == identity_exact(z[tag + "_u"], z["q60_b_in"], z[tag + "_b_out"]), tag
    for k in (0, 1):
        u, b0, b = z["ops%d_u" % k][-1], z["ops%d_b_in" % k], z["ops%d_b_out" % k]
        assert bool(z["ops%d_consistent" % k]) == np.array_equal(u.astype(np.uint64) @ b0.astype(np.uint64),
                                                                 b.astype(np.uint64))


def test_op_scripts_negate_only_in_their_second_half_and_then_break_the_reference_u():
    z = H.gold("transform_ref.npz")
    for k in (0, 1):
        groups = json.loads(bytes(z["ops%d_script" % k]).decode())
        kinds = {o[0] for g in groups for o in g}
        assert kinds == {"addmul", "swap", "move", "negate"}
        first = min(g for g, ops in enumerate(groups) if any(o[0] == "negate" for o in ops))
        assert first >= len(groups) // 2
        assert any(o[0] == "addmul" and o[4] >= 61 for g in groups for o in g)  # shifted (wrapping) products
        assert any(o[0] == "move" and o[1] < o[2] for g in groups for o in g)
        assert any(o[0] == "move" and o[1] > o[2] for g in groups for o in g)
        assert not bool(z["ops%d_consistent" % k])  # the reference's negate_row_of_b does not negate u


def test_fixture_bases_are_the_existing_goldens():
    z = H.gold("transform_ref.npz")
    q60, sd = H.gold("bkz_q60.npz"), H.gold("bkz_sd_sld.npz")
    u40 = H.gold("u40_lll_long.npz")
    assert np.array_equal(z["q60_b_in"], q60["b_in"])
    assert np.array_equal(z["bkz20_b_out"], q60["bkz20_none_b"]) and int(z["bkz20_status"]) == int(q60["bkz20_none_status"])
    for tag in ("sd20", "sld20"):
        assert np.array_equal(z[tag + "_b_out"], sd[tag + "_none_b"]), tag
        assert int(z[tag + "_flags"]) == int(sd[tag + "_none_flags"]) and int(z[tag + "_status"]) == int(sd[tag + "_none_status"])
    assert np.array_equal(z["lll_u40_b_in"], u40["b_in"]) and np.array_equal(z["lll_u40_b_out"], u40["b_out"])
    assert int(z["lll_u40_swaps"]) == int(u40["n_swaps"])
    assert int(z["lll_rankdef_zeros"]) == 10 and not z["lll_rankdef_b_out"][30:].any()
