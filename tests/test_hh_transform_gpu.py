"""GPU tests of the Householder transform (B200HH_TRANSFORM / B200HH_INV_TRANSFORM, include/b200hh.h): U and U^-T take
every integer row operation of size_reduce and swap, on their own and inside the device hlll() loop, and never change a
decision.

What is checked, against the oracle (tests/hh_transform_oracle.py over oracle/hh_oracle.c, pinned to the reference by
test_hh_transform_cpu.py) and
against tests/golden/hh_transform_ref.npz (the reference's own U and U^-T, make_hh_transform_golden.py):
  * a transform handle ends every call with the b, R, V, sigma, bf, status and iteration count of a plain handle;
  * U and U^-T are the reference's bit for bit (HLLL never negates a row, so there is no intended divergence);
  * U * B_in == B and U * (U^-T)^T == I mod 2^64 on every lattice, whatever its status."""
import json

import numpy as np
import pytest

import helpers as H
from oracle import oracle as O
from hh_transform_oracle import TransformOracle

pytestmark = pytest.mark.gpu

FLAGS = 5  # HOUSEHOLDER_ROW_EXPO | HOUSEHOLDER_OP_FORCE_LONG


@pytest.fixture(scope="module")
def hh():
    from fplll_b200 import householder
    return householder


@pytest.fixture(scope="module")
def z():
    return H.gold("hh_transform_ref.npz")


def hlll_like_ops(d):
    """HLLLReduction::hlll's call order (hlll.cpp:49-171) with a swap every third step, as in test_hh_gpu.py"""
    ops = [("refresh_R_bf", 0), ("update_R_last", 0), ("refresh_R_bf", 1)]
    k, kmax = 1, 1
    for step in range(3 * d):
        ops += [("update_R", k, 0), ("size_reduce", k, k, 0), ("refresh_R_bf", k), ("update_R", k, 0), ("check",)]
        if step % 3 != 2 or k == 1:
            ops += [("update_R_last", k)]
            k += 1
            if k >= d:
                break
            ops += [("refresh_R_bf", k)] if k > kmax else [("refresh_R", k)]
            kmax = max(kmax, k)
        else:
            ops += [("swap", k - 1, k)]
            k -= 1
            ops += [("recover_R", k), ("check",), ("set_updated_R_false",)]
    ops.append(("check",))
    return ops


def case_input(z, tag):
    src = json.loads(bytes(z["cases"]).decode())[tag]
    if src == "self":
        return z[tag + "_in"].astype(np.int64)
    f, k = src.split(":")
    return H.gold(f)[k].astype(np.int64)


def mixed(seed, batch, d, n):
    """small random combinations of random rows: HLLL swaps and size-reduces them (test_size_classes_gpu.py)"""
    rng = np.random.default_rng(seed)
    u = rng.integers(-64, 65, size=(batch, d, d), dtype=np.int64)
    return u @ rng.integers(-(1 << 10), 1 << 10, size=(batch, d, n), dtype=np.int64)


def wrap_mul(a, b):
    """a @ b mod 2^64 (numpy's uint64 matmul wraps)"""
    return (a.astype(np.uint64) @ b.astype(np.uint64)).astype(np.int64)


def identities_hold(u, ut, b_in, b_out):
    eye = np.eye(u.shape[0], dtype=np.int64)
    return np.array_equal(wrap_mul(u, b_in), b_out) and np.array_equal(wrap_mul(u, ut.T), eye)


def same_state(s, st, what):
    for k in ("b", "row_expo", "expo_norm_square_b", "n_known_rows", "n_known_cols", "updated_R"):
        assert np.array_equal(s[k], st[k]), what + " " + k
    for k in ("R", "V", "bf", "sigma", "norm_square_b"):
        assert H.eq_f64(s[k], st[k]), what + " " + k


def test_call_script_batch_of_three_against_plain_handle_and_oracle(hh):
    d, n, batch = 30, 34, 3
    b = np.random.default_rng(31).integers(-(1 << 30), 1 << 30, size=(batch, d, n), dtype=np.int64)
    eye = np.eye(d, dtype=np.int64)
    m = hh.MatHouseholder(b, FLAGS)
    mt = hh.MatHouseholder(b, FLAGS, u=eye, u_inv_t=eye)
    mos = [TransformOracle(b[l], FLAGS, u=eye, u_inv_t=eye) for l in range(batch)]
    checks = 0
    for op in hlll_like_ops(d):
        if op[0] == "check":
            what = "check %d" % checks
            same_state(m.state(), mt.state(), what)
            u, ut = mt.u, mt.u_inv_t
            for l, mo in enumerate(mos):
                assert np.array_equal(u[l], mo.u), what + " U lattice %d" % l
                assert np.array_equal(ut[l], mo.u_inv_t), what + " U^-T lattice %d" % l
            checks += 1
        else:
            r, rt = getattr(m, op[0])(*op[1:]), getattr(mt, op[0])(*op[1:])
            for mo in mos:
                getattr(mo, op[0])(*op[1:])
            if op[0] == "size_reduce":
                assert np.array_equal(r, rt)
    assert checks > 10
    assert not np.array_equal(mt.u[0], eye)


def test_reference_call_script_replayed_on_the_device(hh, z):
    b = z["script_in"]
    d = b.shape[0]
    eye = np.eye(d, dtype=np.int64)
    mt = hh.MatHouseholder(b, FLAGS, u=eye, u_inv_t=eye)
    checks = 0
    for op in json.loads(bytes(z["script_ops"]).decode()):
        if op[0] == "check":
            what = "check %d" % checks
            assert np.array_equal(mt.get_basis()[0], z["script_b"][checks]), what + " b"
            assert np.array_equal(mt.u[0], z["script_u"][checks]), what + " U"
            assert np.array_equal(mt.u_inv_t[0], z["script_uinvt"][checks]), what + " U^-T"
            checks += 1
        else:
            getattr(mt, op[0])(*op[1:])
    assert checks == len(z["script_u"])


def hlll_three_ways(hh, b):
    """hlll on a plain handle, a U handle and a U + U^-T handle over the same batch"""
    eye = np.eye(b.shape[-2], dtype=np.int64)
    out = []
    for kw in ({}, {"u": eye}, {"u": eye, "u_inv_t": eye}):
        m = hh.MatHouseholder(b, FLAGS, **kw)
        st, it = m.hlll()
        out.append(dict(b=m.get_basis(), st=st, it=it, u=m.u if kw else None,
                        ut=m.u_inv_t if "u_inv_t" in kw else None, state=m.state()))
        m.close()
    for r in out[1:]:
        assert np.array_equal(r["st"], out[0]["st"]) and np.array_equal(r["it"], out[0]["it"])
        same_state(out[0]["state"], r["state"], "hlll with a transform")
    assert np.array_equal(out[1]["u"], out[2]["u"])
    return out[2]


@pytest.mark.parametrize("tag", ["u40", "r60", "q40", "u100", "q80", "q400sub", "hlll600", "mix170"])
def test_whole_hlll_against_the_reference(hh, z, tag):
    b = case_input(z, tag)
    r = hlll_three_ways(hh, b)
    assert int(r["st"][0]) == int(z[tag + "_status"])
    assert np.array_equal(r["b"][0], z[tag + "_out"])
    assert np.array_equal(r["u"][0], z[tag + "_u"]), "U"
    assert np.array_equal(r["ut"][0], z[tag + "_uinvt"]), "U^-T"


@pytest.mark.parametrize("n", [96, 97, 224, 225, 416, 417, 600, 992])
def test_every_update_R_width_against_the_oracle(hh, n):
    b = mixed(n, 2, 20 if n > 600 else 30, n)
    r = hlll_three_ways(hh, b)
    d = b.shape[1]
    eye = np.eye(d, dtype=np.int64)
    for l in range(2):
        mo = TransformOracle(b[l], u=eye, u_inv_t=eye)
        assert mo.hlll() == r["st"][l], "n %d lattice %d status" % (n, l)
        assert np.array_equal(r["b"][l], mo.state()["b"]), "n %d lattice %d basis" % (n, l)
        assert np.array_equal(r["u"][l], mo.u), "n %d lattice %d U" % (n, l)
        assert np.array_equal(r["ut"][l], mo.u_inv_t), "n %d lattice %d U^-T" % (n, l)


def random_unimodular(rng, d, steps):
    """U0 from random row additions on the identity, and its U0^-T by the same rule the transform follows"""
    u, ut = np.eye(d, dtype=np.int64), np.eye(d, dtype=np.int64)
    for _ in range(steps):
        i, j = (int(t) for t in rng.choice(d, 2, replace=False))
        x = int(rng.integers(-3, 4))
        u[i] += x * u[j]
        ut[j] -= x * ut[i]
    return u, ut


def test_batch_lattices_start_from_their_own_u(hh):
    """set_transform with a different U0 per lattice on the same basis: hlll continues from it, U = U_hlll * U0 and
    U^-T = U_hlll^-T * U0^-T per lattice"""
    d, n, batch = 40, 44, 4
    b0 = mixed(4, 1, d, n)[0]
    rng = np.random.default_rng(44)
    pairs = [random_unimodular(rng, d, 60 * l) for l in range(batch)]   # lattice 0 starts at the identity
    u0, ut0 = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    for l in range(batch):
        assert np.array_equal(wrap_mul(u0[l], ut0[l].T), np.eye(d, dtype=np.int64))
    m = hh.MatHouseholder(np.repeat(b0[None], batch, 0), FLAGS, u=np.eye(d, dtype=np.int64),
                          u_inv_t=np.eye(d, dtype=np.int64))
    m.set_transform(u0, ut0)
    st, _ = m.hlll()
    u, ut, out = m.u, m.u_inv_t, m.get_basis()
    eye = np.eye(d, dtype=np.int64)
    mo = TransformOracle(b0, u=eye, u_inv_t=eye)
    assert mo.hlll() == 0 and list(st) == [0] * batch
    for l in range(batch):
        assert np.array_equal(out[l], mo.state()["b"])
        assert np.array_equal(u[l], wrap_mul(mo.u, u0[l])), "lattice %d U" % l
        assert np.array_equal(ut[l], wrap_mul(mo.u_inv_t, ut0[l])), "lattice %d U^-T" % l


def failing_lattice():
    """the first of a few small random bases with 62-bit entries on which the oracle's HLLLReduction<long, double> ends
    with a non-zero status (RED_HLLL_NORM_FAILURE / RED_HLLL_SR_FAILURE), or None"""
    for seed in range(40):
        b = np.random.default_rng(seed).integers(-(1 << 62), 1 << 62, size=(12, 12), dtype=np.int64)
        if O.OracleHouseholder(b).hlll() != 0:
            return b
    return None


def test_identities_hold_whatever_the_status(hh):
    d, n = 12, 12
    lat = [mixed(s, 1, d, n)[0] for s in (1, 2, 3)]
    fail = failing_lattice()
    if fail is None:
        print("no small lattice with a non-zero HLLL status was found with the oracle; all lattices end in status 0")
    else:
        lat.append(fail)
    b = np.stack(lat)
    eye = np.eye(d, dtype=np.int64)
    m = hh.MatHouseholder(b, FLAGS, u=eye, u_inv_t=eye)
    st, _ = m.hlll()
    u, ut, out = m.u, m.u_inv_t, m.get_basis()
    for l in range(len(lat)):
        mo = TransformOracle(b[l], u=eye, u_inv_t=eye)
        assert mo.hlll() == st[l]
        assert identities_hold(u[l], ut[l], b[l], out[l]), "lattice %d (status %d)" % (l, st[l])
        assert np.array_equal(u[l], mo.u) and np.array_equal(ut[l], mo.u_inv_t)
    if fail is not None:
        assert st[-1] != 0


def test_hlll_reduction_fills_u_and_u_inv_in_place(hh, z):
    b = case_input(z, "q40")
    d = b.shape[0]
    u = np.full((d, d), 7, np.int64)   # overwritten: the call starts from the identity
    ui = np.zeros((d, d), np.int64)
    out, st = hh.hlll_reduction(b, u=u, u_inv=ui)
    assert st == 0 and np.array_equal(out, z["q40_out"])
    assert np.array_equal(u, z["q40_u"]) and np.array_equal(ui, z["q40_uinvt"].T)
    assert np.array_equal(np.dot(u.astype(object), ui.astype(object)), np.eye(d, dtype=np.int64).astype(object))
    # without u_inv, and batched; the plain call is unchanged
    bb = np.stack([b, b])
    ub = np.zeros((2, d, d), np.int64)
    outs, sts = hh.hlll_reduction(bb, u=ub)
    assert list(sts) == [0, 0] and np.array_equal(ub[1], z["q40_u"]) and np.array_equal(outs[0], z["q40_out"])
    out2, st2 = hh.hlll_reduction(b)
    assert st2 == 0 and np.array_equal(out2, out)


def test_refusals(hh):
    from fplll_b200 import B200Error
    b = mixed(5, 1, 10, 12)[0]
    eye = np.eye(10, dtype=np.int64)
    with pytest.raises(B200Error):      # INV_TRANSFORM without TRANSFORM, at the C-ABI
        hh.MatHouseholder(b, FLAGS | hh.HOUSEHOLDER_INV_TRANSFORM)
    with pytest.raises(ValueError):
        hh.MatHouseholder(b, FLAGS, u_inv_t=eye)
    plain = hh.MatHouseholder(b, FLAGS)
    with pytest.raises(B200Error):
        plain.u
    with pytest.raises(B200Error):
        plain.set_transform(eye)
    only_u = hh.MatHouseholder(b, FLAGS, u=eye)
    assert np.array_equal(only_u.u[0], eye)
    with pytest.raises(B200Error):
        only_u.u_inv_t
    with pytest.raises(B200Error):
        only_u.set_transform(eye, eye)
    assert np.array_equal(only_u.u[0], eye)     # a refused set copies nothing
    both = hh.MatHouseholder(b, FLAGS | hh.HOUSEHOLDER_TRANSFORM | hh.HOUSEHOLDER_INV_TRANSFORM)
    assert np.array_equal(both.u[0], eye) and np.array_equal(both.u_inv_t[0], eye)
    with pytest.raises(ValueError):
        both.set_transform(np.eye(9, dtype=np.int64))
    with pytest.raises(ValueError):
        hh.hlll_reduction(b, u=np.zeros((9, 9), np.int64))
    with pytest.raises(ValueError):
        hh.hlll_reduction(b, u_inv=np.zeros((10, 10), np.int64))
