"""Shared test helpers: golden-fixture access, state comparison on the entries the reference defines."""
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gold(name):
    return np.load(os.path.join(GOLD, name), allow_pickle=False)


def gold_json(name):
    import json
    with open(os.path.join(GOLD, name)) as f:
        return json.load(f)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def eq_f64(a, b):
    """bit-exact equality with NaN == NaN (any payload)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(bits(np.nan_to_num(a, nan=0.0)),
                                                                        bits(np.nan_to_num(b, nan=0.0)))


def assert_state_equal(got, ref, what="", check_b=True):
    """Compare two MatGSO states (dicts as produced by OracleGSO.state / MatGSO.state()[l] / ref dumps) on exactly
    the entries the reference defines (SURVEY Appendix A): rows < n_known_rows, mu(i,j) for j < min(valid,i),
    r(i,j) for j < valid, gf(i,j) for j <= i (NaN = invalid), all of bf / row_expo / validity / metadata."""
    d = int(ref["d"]) if "d" in ref else ref["mu"].shape[-1]
    nkr = int(ref["n_known_rows"])
    assert int(got["n_known_rows"]) == nkr, what + " n_known_rows"
    assert int(got["n_known_cols"]) == int(ref["n_known_cols"]), what + " n_known_cols"
    assert int(got["n_source_rows"]) == int(ref["n_source_rows"]), what + " n_source_rows"
    assert np.array_equal(got["gso_valid_cols"][:nkr], ref["gso_valid_cols"][:nkr]), what + " gso_valid_cols"
    assert np.array_equal(got["init_row_size"], ref["init_row_size"]), what + " init_row_size"
    assert np.array_equal(got["row_expo"], ref["row_expo"]), what + " row_expo"
    if check_b and "b" in ref:
        assert np.array_equal(got["b"], ref["b"]), what + " b"
    assert eq_f64(got["bf"], ref["bf"]), what + " bf"
    for i in range(nkr):
        v = int(ref["gso_valid_cols"][i])
        assert eq_f64(got["gf"][i, : i + 1], ref["gf"][i, : i + 1]), "%s gf row %d" % (what, i)
        assert eq_f64(got["mu"][i, : min(v, i)], ref["mu"][i, : min(v, i)]), "%s mu row %d" % (what, i)
        assert eq_f64(got["r"][i, :v], ref["r"][i, :v]), "%s r row %d" % (what, i)


def _f64_bytes(a):
    """float64 bytes with every NaN in one canonical encoding (eq_f64's NaN == NaN, any payload)."""
    a = np.array(a, dtype=np.float64)
    a[np.isnan(a)] = np.nan
    return a.tobytes()


def hh_digest(s, rows_R):
    """sha256 over the MatHouseholder state entries test_hh_oracle compares: metadata, integer arrays, the first rows_R
    rows of sigma / norm_square_b / bf / R and the known rows of V (bit patterns, NaN canonical)."""
    import hashlib
    h = hashlib.sha256()
    nk = int(s["n_known_rows"])
    h.update(np.array([nk, int(s["n_known_cols"])], np.int64).tobytes())
    for k in ["row_expo", "expo_norm_square_b", "b"]:
        h.update(np.ascontiguousarray(s[k], np.int64).tobytes())
    for k in ["sigma", "norm_square_b", "bf", "R"]:
        h.update(_f64_bytes(s[k][:rows_R]))
    h.update(_f64_bytes(s["V"][:nk]))
    return h.hexdigest()


def strategy_digest(entry):
    """sha256 of one block size's (preprocessing, gh_factor, expectation, coefficients) arrays."""
    import hashlib
    h = hashlib.sha256()
    pp, gh, ex, coef = entry
    h.update(np.asarray(pp, np.int32).tobytes())
    for a in (gh, ex, coef):
        h.update(np.array(a.shape, np.int64).tobytes() + _f64_bytes(a))
    return h.hexdigest()


def is_lll_reduced(b, delta=0.99, eta=0.51):
    """The test of is_lll_reduced (lll.cpp:226-258) in exact arithmetic: |mu(i,j)| <= eta for all j < i and
    r(i,i) >= (delta - mu(i,i-1)^2) r(i-1,i-1).  Integral Gram-Schmidt (Cohen, Algorithm 2.6.7): dd[i+1] = r(0,0)
    ... r(i,i) and lam[i][j] = dd[j+1] mu(i,j) are integers.  tests/golden/ref_islll.json pins it to the reference."""
    from fractions import Fraction
    b = [[int(x) for x in row] for row in np.asarray(b)]
    d = len(b)
    dd = [1] + [0] * d
    lam = [[0] * d for _ in range(d)]
    for i in range(d):
        for j in range(i + 1):
            u = sum(x * y for x, y in zip(b[i], b[j]))
            for k in range(j):
                u = (dd[k + 1] * u - lam[i][k] * lam[j][k]) // dd[k]
            if j < i:
                lam[i][j] = u
            else:
                dd[i + 1] = u
        if dd[i + 1] == 0:
            raise ValueError("rows are linearly dependent")
    e, de = Fraction(eta), Fraction(delta)
    for i in range(d):
        for j in range(i):
            if abs(Fraction(lam[i][j], dd[j + 1])) > e:
                return False
    for i in range(1, d):
        mu = Fraction(lam[i][i - 1], dd[i])
        r_prev, r_i = Fraction(dd[i], dd[i - 1]), Fraction(dd[i + 1], dd[i])
        if r_i < (de - mu * mu) * r_prev:
            return False
    return True


def lattice_state(st, l):
    """slice lattice l out of a batched fplll_b200.MatGSO.state()"""
    out = {k: (v[l] if isinstance(v, np.ndarray) and v.ndim >= 1 else v) for k, v in st.items()}
    return out


def random_op_script(rng, d, n_ops, allow_move=True):
    """A random but valid MatGSO call sequence in the style of tests/test_gso.cpp:196-228 (move_row, row_addmul
    inside row_op_begin/end, update_gso_row).  Returns a list of tuples."""
    ops = [("update_gso",)]
    for _ in range(n_ops):
        kind = rng.integers(0, 4 if allow_move else 3)
        if kind == 0:
            i = int(rng.integers(1, d))
            j = int(rng.integers(0, i))
            x = float(rng.integers(-9, 10))
            ops += [("row_op_begin", i, i + 1), ("row_addmul_we", i, j, x, 0), ("row_op_end", i, i + 1)]
        elif kind == 1:
            i = int(rng.integers(1, d))
            j = int(rng.integers(0, i))
            x = float(rng.integers(-3, 4))
            e = int(rng.integers(1, 4))
            ops += [("row_op_begin", i, i + 1), ("row_addmul_we", i, j, x, e), ("row_op_end", i, i + 1)]
        elif kind == 2:
            i = int(rng.integers(0, d))
            ops += [("update_rows_to", i)]
        else:
            a, b = int(rng.integers(0, d)), int(rng.integers(0, d))
            ops += [("move_row", a, b)]
    ops.append(("update_gso",))
    return ops


def apply_ops(m, ops, is_batch=False):
    """Run an op script on an object with the reference method names (OracleGSO or fplll_b200.MatGSO)."""
    for op in ops:
        k = op[0]
        if k == "update_gso":
            m.update_gso()
        elif k == "update_rows_to":
            # the reference requires rows < i to be valid before update_gso_row(i): update them in order
            for t in range(op[1] + 1):
                m.update_gso_row(t, t)
        elif k == "row_op_begin":
            if hasattr(m, "row_op_begin"):
                m.row_op_begin(op[1], op[2])
        elif k == "row_op_end":
            m.row_op_end(op[1], op[2])
        elif k == "row_addmul_we":
            m.row_addmul_we(op[1], op[2], op[3], op[4])
        elif k == "move_row":
            m.move_row(op[1], op[2])
        elif k == "row_swap":
            m.row_swap(op[1], op[2])
        else:
            raise ValueError(k)


def ops_to_ref_script(ops):
    lines = []
    for op in ops:
        k = op[0]
        if k == "update_rows_to":
            for t in range(op[1] + 1):
                lines.append("update_row %d %d" % (t, t))
        elif k == "row_addmul_we":
            lines.append("row_addmul_we %d %d %r %d" % (op[1], op[2], op[3], op[4]))
        else:
            lines.append(" ".join(str(x) for x in op))
    return lines


def gso_digest(s):
    """sha256 over the MatGSO state entries assert_state_equal compares (NaN canonical)."""
    import hashlib
    h = hashlib.sha256()
    nkr = int(s["n_known_rows"])
    h.update(np.array([nkr, int(s["n_known_cols"]), int(s["n_source_rows"])], np.int64).tobytes())
    h.update(np.ascontiguousarray(s["gso_valid_cols"][:nkr], np.int64).tobytes())
    for k in ["init_row_size", "row_expo", "b"]:
        h.update(np.ascontiguousarray(s[k], np.int64).tobytes())
    h.update(_f64_bytes(s["bf"]))
    for i in range(nkr):
        v = int(s["gso_valid_cols"][i])
        h.update(_f64_bytes(s["gf"][i, : i + 1]) + _f64_bytes(s["mu"][i, : min(v, i)]) + _f64_bytes(s["r"][i, :v]))
    return h.hexdigest()


def ranged_inputs(seed, d, bits):
    """A (d, d + 1) basis for ranged_call_script: uniform `bits`-bit rows, the last three of them very short (entries in
    [-2, 2]): the rows that the script's insertions move into the reduced part one after the other."""
    rng = np.random.default_rng(seed)
    b = rng.integers(-(1 << bits), 1 << bits, size=(d, d + 1), dtype=np.int64)
    b[d - 3:] = rng.integers(-2, 3, size=(3, d + 1))
    return b


def _range_edges(d):
    return [e for e in (2, 3, 31, 32, 33, 63, 64, 65, 255, 256, 257) if e < d] + [d]


def ranged_call_script(rng, d, n_calls):
    """A seeded script of LLLReduction calls and row mutations in the style of the BKZ driver (bkz.cpp): ranged
    lll(kappa_min, kappa_start, kappa_end, size_reduction_start) and size_reduction calls with range ends on the
    32-row panel edges, delta / eta changes, and row_addmul, row_swap and move_row insertions of the short rows that
    ranged_inputs plants at the end (while no call has reached them).  The script keeps to what the reference asks of
    its callers: before a call that starts above row 0 the rows below its start get a valid GSO (update_gso_row), and
    a row is discovered before move_row moves it down.  Entries are JSON-friendly lists:
      ["lll", delta, eta, kmin, kstart, kend, srs], ["sr", eta, kmin, kend, srs], ["addmul", i, j, x],
      ["swap", i, j], ["move", old, new], ["discover_all"], ["update_rows", k] (update_gso_row(t, t) for t < k)."""
    edges = _range_edges(d)
    first = [e for e in edges if e < d - 3]  # the planted rows stay out of the first reduction
    ops = [["lll", 0.99, 0.51, 0, 0, int(rng.choice(first[len(first) // 2:])), 0]]
    delta, eta, inserted, reached = 0.99, 0.51, 0, ops[0][5]
    for _ in range(n_calls):
        u = rng.random()
        if u < 0.1:
            delta, eta = [(0.99, 0.51), (0.75, 0.51), (0.99, 0.6), (0.999, 0.501)][int(rng.integers(0, 4))]
        kend = int(rng.choice(edges)) if rng.random() < 0.7 else int(rng.integers(2, d + 1))
        if u < 0.5:
            shape = int(rng.integers(0, 4))
            if shape == 0:  # lll(0, 0, kend): the resuming prefix call of svp_preprocessing
                kmin = kstart = 0
            elif shape == 1:  # lll(k, k, kend): BKZ_BOUNDED_LLL and slide reduction
                kmin = kstart = int(rng.integers(0, kend - 1))
            else:  # kappa_start > kappa_min
                kmin = int(rng.integers(0, kend - 1))
                kstart = int(rng.integers(kmin, kend))
            srs = [0, 0, int(rng.integers(0, kmin + 1)), int(rng.integers(kmin, kend)), kstart][int(rng.integers(0, 5))]
            if kstart:
                ops.append(["update_rows", kstart])
            ops.append(["lll", delta, eta, kmin, kstart, -1 if kend == d and rng.random() < 0.5 else kend, srs])
            reached = max(reached, kend)
        elif u < 0.65:
            kmin = int(rng.integers(0, kend + 1))
            srs = [0, 0, int(rng.integers(0, kmin + 1)), max(0, kmin - 2)][int(rng.integers(0, 4))]
            if kmin:
                ops.append(["update_rows", kmin])
            ops.append(["sr", eta, kmin, kend, srs])
            reached = max(reached, kend)
        elif u < 0.8:
            i = int(rng.integers(1, d - 3))
            ops.append(["addmul", i, int(rng.integers(0, i)), float(rng.choice([-2, -1, 1, 3]))])
        elif u < 0.9 and reached <= d - 3 + inserted:
            # BKZ's insertion (bkz.cpp svp_postprocessing): a new row moved to kappa, then lll(kappa, kappa, kappa + beta)
            k = int(rng.integers(0, reached))
            ops += [["discover_all"], ["move", d - 1, k]]
            inserted += 1
            kend = int(min(d - 3 + inserted, k + rng.integers(2, 40)))
            reached = max(reached, kend)
            if k:
                ops.append(["update_rows", k])
            ops.append(["lll", delta, eta, k, k, kend, 0])
        else:
            i, j = (int(x) for x in rng.choice(d - 3, 2, replace=False))
            ops.append(["swap", i, j])
    ops.append(["lll", 0.99, 0.51, 0, 0, d, 0])
    return ops


def ranged_apply(m, op):
    """Runs one entry of ranged_call_script on an OracleGSO or a fplll_b200.MatGSO; returns what lll / size_reduction
    return, None for the mutations."""
    k, a = op[0], op[1:]
    if k == "lll":
        return m.lll(*a)
    if k == "sr":
        return m.size_reduction(*a)
    if k == "addmul":
        m.row_addmul_we(a[0], a[1], a[2], 0)
        m.row_op_end(a[0], a[0] + 1)
    elif k == "swap":
        m.row_swap(a[0], a[1])
        m.row_op_end(min(a), max(a) + 1)
    elif k == "move":
        m.move_row(a[0], a[1])
    elif k == "discover_all":
        m.discover_all_rows()
    elif k == "update_rows":
        for t in range(a[0]):
            m.update_gso_row(t, t)
    else:
        raise ValueError(k)
    return None


def ranged_ref_lines(op):
    """The ref_probe commands of one ranged_call_script entry (oracle/ref_probe.cpp)."""
    k, a = op[0], op[1:]
    if k == "lll":
        return ["lll_range %r %r %d %d %d %d" % tuple(a)]
    if k == "sr":
        return ["size_reduction %r %d %d %d" % tuple(a)]
    if k == "addmul":
        return ["row_op_begin %d %d" % (a[0], a[0] + 1), "row_addmul_we %d %d %r 0" % tuple(a),
                "row_op_end %d %d" % (a[0], a[0] + 1)]
    if k == "swap":
        lo, hi = min(a), max(a) + 1
        return ["row_op_begin %d %d" % (lo, hi), "row_swap %d %d" % tuple(a), "row_op_end %d %d" % (lo, hi)]
    if k == "move":
        return ["move_row %d %d" % tuple(a)]
    if k == "discover_all":
        return ["discover_all"]
    if k == "update_rows":
        return ["update_row %d %d" % (t, t) for t in range(a[0])]
    raise ValueError(k)
