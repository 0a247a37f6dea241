"""CPU checks of tests/golden/hh_transform_ref.npz (make_hh_transform_golden.py: the reference's U and U^-T next to b in
MatHouseholder<long, double> and HLLLReduction<long, double>) and of the oracle's transform (hh_transform_oracle.py over
oracle/hh_oracle.c):
  * its hlll() over the C primitives ends with the basis and status of the C oracle's own ohh_hlll;
  * its U and U^-T equal the reference's bit for bit, after every whole-HLLL case and at every check point of the call
    script;
  * the reference's U * B_in == B_out and U * (U^-T)^T == I hold over the integers;
  * the fixture's bases are the outputs already pinned by hlll_long.npz, hlll_q400.npz and size_classes_ref.npz."""
import json

import numpy as np
import pytest

import helpers as H
from oracle import oracle as O
from hh_transform_oracle import TransformOracle

Z = H.gold("hh_transform_ref.npz")
CASES = json.loads(bytes(Z["cases"]).decode())
PINNED = {"u40": ("hlll_long.npz", "u40"), "r60": ("hlll_long.npz", "r60"), "q40": ("hlll_long.npz", "q40"),
          "u100": ("hlll_long.npz", "u100"), "q80": ("hlll_long.npz", "q80"), "q400sub": ("hlll_q400.npz", "q400sub"),
          "hlll600": ("size_classes_ref.npz", "hlll600")}


def case_input(tag):
    src = CASES[tag]
    if src == "self":
        return Z[tag + "_in"].astype(np.int64)
    f, k = src.split(":")
    return H.gold(f)[k].astype(np.int64)


def exact(a):
    return np.asarray(a).astype(object)


def test_fixture_has_every_case():
    assert set(CASES) == set(PINNED) | {"mix170"}
    b = case_input("mix170")
    assert b.shape[0] >= 160 and b.shape[0] % 32 != 0


@pytest.mark.parametrize("tag", sorted(PINNED))
def test_fixture_bases_are_the_pinned_outputs(tag):
    f, k = PINNED[tag]
    g = H.gold(f)
    assert np.array_equal(Z[tag + "_out"], g[k + "_out"])
    assert int(Z[tag + "_status"]) == int(g[k + "_status"])


@pytest.mark.parametrize("tag", ["u40", "r60", "q40", "u100", "q80", "q400sub", "hlll600", "mix170"])
def test_reference_u_identities_and_oracle_u(tag):
    b_in = case_input(tag)
    d = b_in.shape[0]
    u, ut, b_out = Z[tag + "_u"], Z[tag + "_uinvt"], Z[tag + "_out"]
    assert np.array_equal(exact(u).dot(exact(b_in)), exact(b_out)), "U * B_in != B_out"
    assert np.array_equal(exact(u).dot(exact(ut).T), exact(np.eye(d, dtype=np.int64))), "U * (U^-T)^T != I"
    eye = np.eye(d, dtype=np.int64)
    mo = TransformOracle(b_in, u=eye, u_inv_t=eye)
    assert mo.hlll() == int(Z[tag + "_status"])
    assert np.array_equal(mo.state()["b"], b_out)
    plain = O.OracleHouseholder(b_in)
    assert plain.hlll() == int(Z[tag + "_status"]) and np.array_equal(plain.state()["b"], b_out), "C ohh_hlll"
    assert np.array_equal(mo.u, u), "oracle U"
    assert np.array_equal(mo.u_inv_t, ut), "oracle U^-T"


def test_oracle_follows_the_reference_script():
    b = Z["script_in"]
    d = b.shape[0]
    ops = json.loads(bytes(Z["script_ops"]).decode())
    eye = np.eye(d, dtype=np.int64)
    mo = TransformOracle(b, 5, u=eye, u_inv_t=eye)
    checks = 0
    for op in ops:
        if op[0] == "check":
            what = "check %d" % checks
            assert np.array_equal(mo.state()["b"], Z["script_b"][checks]), what + " b"
            assert np.array_equal(mo.u, Z["script_u"][checks]), what + " U"
            assert np.array_equal(mo.u_inv_t, Z["script_uinvt"][checks]), what + " U^-T"
            checks += 1
        else:
            getattr(mo, op[0])(*op[1:])
    assert checks == len(Z["script_u"]) > 10
    # the script reduced something: U moved away from the identity
    assert not np.array_equal(Z["script_u"][-1], eye)


@pytest.mark.parametrize("seed,d,n,bits", [(1, 20, 22, 20), (2, 30, 30, 30), (3, 12, 40, 50)])
def test_restated_hlll_follows_the_c_oracle(seed, d, n, bits):
    """the Python hlll() loop over the C primitives against ohh_hlll on random bases: same basis, status and state"""
    b = np.random.default_rng(seed).integers(-(1 << bits), 1 << bits, size=(d, n), dtype=np.int64)
    mo, plain = TransformOracle(b), O.OracleHouseholder(b)
    assert mo.hlll() == plain.hlll()
    for k in ("b", "R", "V", "bf", "sigma", "norm_square_b", "row_expo"):
        assert np.array_equal(mo.state()[k], plain.state()[k]), k
    assert np.array_equal(np.dot(mo.u.astype(object), b.astype(object)), mo.state()["b"].astype(object))


def test_u_inv_t_alone_is_refused():
    b = case_input("u40")
    with pytest.raises(ValueError):
        TransformOracle(b, u_inv_t=np.eye(b.shape[0], dtype=np.int64))
