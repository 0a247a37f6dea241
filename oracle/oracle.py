"""ctypes front-end for the CPU oracle (TEST INFRASTRUCTURE ONLY — see oracle/gso_oracle.c header).

Two checkers live here:
  * `OracleGSO`   — the plain-C restatement (oracle/liboracle.so, built by oracle/build.py)
  * `RefProbe`    — the UNMODIFIED reference library driven through oracle/_ref/ref_probe (when present)
plus `read_dumps`, the parser for ref_probe's binary state records.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this module.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REF_PROBE = os.path.join(REF_DIR, "ref_probe")
LATTICEGEN = os.path.join(REF_DIR, "latticegen")
LIB_PATH = os.path.join(HERE, "liboracle.so")

GSO_ROW_EXPO = 2


def have_ref():
    return os.path.exists(REF_PROBE) and os.path.exists(os.path.join(REF_DIR, "libfplll.so"))


class _OGSO(C.Structure):
    _fields_ = [
        ("d", C.c_int), ("n", C.c_int), ("enable_row_expo", C.c_int),
        ("n_known_rows", C.c_int), ("n_known_cols", C.c_int), ("n_source_rows", C.c_int),
        ("cols_locked", C.c_int),
        ("b", C.POINTER(C.c_int64)), ("bf", C.POINTER(C.c_double)),
        ("gf", C.POINTER(C.c_double)), ("mu", C.POINTER(C.c_double)), ("r", C.POINTER(C.c_double)),
        ("row_expo", C.POINTER(C.c_int64)),
        ("gso_valid_cols", C.POINTER(C.c_int)), ("init_row_size", C.POINTER(C.c_int)),
        ("tmp_col_expo", C.POINTER(C.c_int64)),
    ]


class _OLLL(C.Structure):
    _fields_ = [("delta", C.c_double), ("eta", C.c_double), ("swap_threshold", C.c_double),
                ("status", C.c_int), ("n_swaps", C.c_int), ("final_kappa", C.c_int), ("zeros", C.c_int),
                ("n_babai_iters", C.c_long), ("n_row_ops", C.c_long)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            from . import build as _b  # noqa
            _b.build_oracle()
        L = C.CDLL(LIB_PATH)
        L.ogso_create.restype = C.POINTER(_OGSO)
        L.ogso_create.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int64), C.c_int]
        L.ogso_destroy.argtypes = [C.POINTER(_OGSO)]
        L.ogso_update_gso_row.argtypes = [C.POINTER(_OGSO), C.c_int, C.c_int]
        L.ogso_update_gso.argtypes = [C.POINTER(_OGSO)]
        L.ogso_discover_all_rows.argtypes = [C.POINTER(_OGSO)]
        L.ogso_row_op_end.argtypes = [C.POINTER(_OGSO), C.c_int, C.c_int]
        L.ogso_row_addmul_we.argtypes = [C.POINTER(_OGSO), C.c_int, C.c_int, C.c_double, C.c_long]
        L.ogso_row_swap.argtypes = [C.POINTER(_OGSO), C.c_int, C.c_int]
        L.ogso_move_row.argtypes = [C.POINTER(_OGSO), C.c_int, C.c_int]
        L.ogso_set_r.argtypes = [C.POINTER(_OGSO), C.c_int, C.c_int, C.c_double]
        L.ogso_get_gram.argtypes = [C.POINTER(_OGSO), C.c_int, C.c_int]
        L.ogso_get_gram.restype = C.c_double
        L.ogso_rnd_we.argtypes = [C.c_double, C.c_long]
        L.ogso_rnd_we.restype = C.c_double
        L.ogso_lll_range.argtypes = [C.POINTER(_OGSO), C.POINTER(_OLLL), C.c_int, C.c_int, C.c_int, C.c_int]
        L.ogso_size_reduction.argtypes = [C.POINTER(_OGSO), C.POINTER(_OLLL), C.c_int, C.c_int, C.c_int]
        L.ogso_negate_row_of_b.argtypes = [C.POINTER(_OGSO), C.c_int]
        L.ogso_babai.argtypes = [C.POINTER(_OGSO), C.POINTER(_OLLL), C.c_int, C.c_int, C.c_int,
                                 C.POINTER(C.c_double), C.POINTER(C.c_long)]
        _lib = L
    return _lib


class OracleGSO:
    """MatGSO<Z_NR<long>, FP_NR<double>> restated in C; same method names as the reference class."""

    def __init__(self, b, flags=GSO_ROW_EXPO):
        b = np.ascontiguousarray(b, dtype=np.int64)
        self.d, self.n = b.shape
        self._p = lib().ogso_create(self.d, self.n, b.ctypes.data_as(C.POINTER(C.c_int64)), flags)
        self.flags = flags

    def __del__(self):
        if getattr(self, "_p", None):
            lib().ogso_destroy(self._p)
            self._p = None

    # -- operations ---------------------------------------------------------------------------------------
    def update_gso_row(self, i, last_j=None):
        return bool(lib().ogso_update_gso_row(self._p, i, i if last_j is None else last_j))

    def update_gso(self):
        return bool(lib().ogso_update_gso(self._p))

    def discover_all_rows(self):
        lib().ogso_discover_all_rows(self._p)

    def row_op_end(self, first, last):
        lib().ogso_row_op_end(self._p, first, last)

    def row_addmul_we(self, i, j, x, expo_add=0):
        lib().ogso_row_addmul_we(self._p, i, j, float(x), expo_add)

    def row_swap(self, i, j):
        lib().ogso_row_swap(self._p, i, j)

    def move_row(self, old_r, new_r):
        lib().ogso_move_row(self._p, old_r, new_r)

    def set_r(self, i, j, f):
        lib().ogso_set_r(self._p, i, j, float(f))

    def negate_row_of_b(self, i):
        lib().ogso_negate_row_of_b(self._p, i)

    def upload_row(self, i, row):
        """What b200gso_upload_row does to one lattice: b[i] = row, then row_op_end(i, i+1)."""
        row = np.ascontiguousarray(row, dtype=np.int64)
        assert row.shape == (self.n,)
        C.memmove(C.addressof(self._p.contents.b.contents) + 8 * i * self.n, row.ctypes.data, 8 * self.n)
        self.row_op_end(i, i + 1)

    def get_gram(self, i, j):
        return lib().ogso_get_gram(self._p, i, j)

    def lll(self, delta=0.99, eta=0.51, kappa_min=0, kappa_start=0, kappa_end=-1, size_reduction_start=0):
        """LLLReduction(m, delta, eta, LLL_DEFAULT).lll(kappa_min, kappa_start, kappa_end, size_reduction_start) on a
        fresh LLLReduction object: `ok` is the reference's return value, `status` its status member, which starts at
        RED_SUCCESS (lll.cpp:28-29) and stays there when update_gso_row fails at kappa_start (lll.cpp:71-76)."""
        L = _OLLL(delta=delta, eta=eta)
        ok = lib().ogso_lll_range(self._p, C.byref(L), kappa_min, kappa_start, kappa_end, size_reduction_start)
        return dict(ok=bool(ok), status=L.status, n_swaps=L.n_swaps, final_kappa=L.final_kappa, zeros=L.zeros,
                    n_babai_iters=L.n_babai_iters, n_row_ops=L.n_row_ops)

    def size_reduction(self, eta=0.51, kappa_min=0, kappa_end=-1, size_reduction_start=0):
        """LLLReduction(m, 0.99, eta, LLL_DEFAULT).size_reduction(kappa_min, kappa_end, size_reduction_start) on a fresh
        LLLReduction object (lll.h:106-122): `ok` and `status` as in lll()."""
        L = _OLLL(delta=0.99, eta=eta)
        ok = lib().ogso_size_reduction(self._p, C.byref(L), kappa_min, kappa_end, size_reduction_start)
        return dict(ok=bool(ok), status=L.status)

    # -- state views (copies) -----------------------------------------------------------------------------
    def _arr(self, ptr, shape, dt):
        n = int(np.prod(shape))
        return np.ctypeslib.as_array(ptr, shape=(n,)).astype(dt).reshape(shape).copy()

    def state(self):
        m = self._p.contents
        d, n = self.d, self.n
        return dict(
            d=d, n=n, n_known_rows=m.n_known_rows, n_known_cols=m.n_known_cols,
            n_source_rows=m.n_source_rows,
            row_expo=self._arr(m.row_expo, (d,), np.int64),
            gso_valid_cols=self._arr(m.gso_valid_cols, (d,), np.int32),
            init_row_size=self._arr(m.init_row_size, (d,), np.int32),
            bf=self._arr(m.bf, (d, n), np.float64), gf=self._arr(m.gf, (d, d), np.float64),
            mu=self._arr(m.mu, (d, d), np.float64), r=self._arr(m.r, (d, d), np.float64),
            b=self._arr(m.b, (d, n), np.int64))


# ---- reference (oracle/_ref) ----------------------------------------------------------------------------

def read_dumps(path):
    """Parse the records ref_probe's `dump` appends (layout in oracle/ref_probe.cpp header)."""
    raw = open(path, "rb").read()
    off, out = 0, []
    while off < len(raw):
        hdr = np.frombuffer(raw, np.int32, 8, off)
        off += 32
        assert hdr[0] == 0x4753304F, "bad magic"
        d, n = int(hdr[1]), int(hdr[2])
        rec = dict(d=d, n=n, n_known_rows=int(hdr[3]), n_known_cols=int(hdr[4]), n_source_rows=int(hdr[5]),
                   flags=int(hdr[6]), ztype=int(hdr[7]))

        def take(dt, shape):
            nonlocal off
            cnt = int(np.prod(shape))
            a = np.frombuffer(raw, dt, cnt, off).reshape(shape).copy()
            off += a.nbytes
            return a
        rec["row_expo"] = take(np.int64, (d,))
        rec["gso_valid_cols"] = take(np.int32, (d,))
        rec["init_row_size"] = take(np.int32, (d,))
        rec["bf"] = take(np.float64, (d, n))
        rec["gf"] = take(np.float64, (d, d))
        rec["mu"] = take(np.float64, (d, d))
        rec["r"] = take(np.float64, (d, d))
        if rec["ztype"] == 0:
            rec["b"] = take(np.int64, (d, n))
        out.append(rec)
    return out


def write_matrix(path, b):
    """fplll text matrix format (nr/matrix.cpp:136-203): [[a b c]\\n[d e f]]"""
    with open(path, "w") as f:
        f.write("[")
        for row in b:
            f.write("[" + " ".join(str(int(x)) for x in row) + "]\n")
        f.write("]\n")


def read_matrix(path):
    txt = open(path).read().replace("[", " ").replace("]", "\n")
    rows = [[int(t) for t in line.split()] for line in txt.splitlines() if line.strip()]
    w = max(len(r) for r in rows)
    return [r + [0] * (w - len(r)) for r in rows]


def run_ref(script, timeout=600):
    """Feed a command script to ref_probe; returns its stdout."""
    if not have_ref():
        raise RuntimeError("oracle/_ref is not built (run `python oracle/build.py --ref` where /root/reference exists)")
    p = subprocess.run([REF_PROBE], input=script, capture_output=True, text=True, timeout=timeout)
    if p.returncode != 0:
        raise RuntimeError("ref_probe failed: " + p.stderr[-2000:])
    return p.stdout


def latticegen(args, timeout=600):
    """Run the reference's own latticegen (the only supported input generator, SURVEY §8c)."""
    p = subprocess.run([LATTICEGEN] + [str(a) for a in args], capture_output=True, text=True, timeout=timeout)
    if p.returncode != 0:
        raise RuntimeError(p.stderr)
    return p.stdout


class RefSession:
    """Accumulates a ref_probe script over a long-basis MatGSO and returns the dumped states."""

    def __init__(self, b, flags=GSO_ROW_EXPO):
        self.tmp = tempfile.mkdtemp(prefix="refprobe_")
        self.mat = os.path.join(self.tmp, "in.txt")
        self.dump = os.path.join(self.tmp, "dump.bin")
        write_matrix(self.mat, b)
        self.lines = ["load %s" % self.mat, "tolong", "gso l %d" % flags]

    def cmd(self, *a):
        self.lines.append(" ".join(repr(x) if isinstance(x, float) else str(x) for x in a))

    def dump_state(self):
        self.lines.append("dump %s" % self.dump)

    def run(self):
        out = run_ref("\n".join(self.lines) + "\n")
        recs = read_dumps(self.dump) if os.path.exists(self.dump) else []
        return out, recs


# ---- enumeration ----------------------------------------------------------------------------------------

def enum_svp(mut, rdiag, pruning, maxdist, shrink=True):
    """oracle/enum_oracle.c::oenum_svp.  Returns dict(nsols, best, sol, nodes)."""
    L = lib()
    d = len(rdiag)
    mut = np.ascontiguousarray(mut, np.float64).reshape(d, d)
    rdiag = np.ascontiguousarray(rdiag, np.float64)
    pr = None if pruning is None else np.ascontiguousarray(pruning, np.float64)
    sol = np.zeros(d)
    best = C.c_double()
    nodes = np.zeros(d, np.uint64)
    L.oenum_svp.restype = C.c_long
    L.oenum_svp.argtypes = [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double),
                            C.c_double, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double),
                            C.POINTER(C.c_uint64)]
    n = L.oenum_svp(d, mut.ctypes.data_as(C.POINTER(C.c_double)), rdiag.ctypes.data_as(C.POINTER(C.c_double)),
                    pr.ctypes.data_as(C.POINTER(C.c_double)) if pr is not None else None, float(maxdist),
                    1 if shrink else 0, sol.ctypes.data_as(C.POINTER(C.c_double)), C.byref(best),
                    nodes.ctypes.data_as(C.POINTER(C.c_uint64)))
    return dict(nsols=int(n), best=best.value, sol=sol, nodes=nodes)


def enum_svp_ex(mut, rdiag, pruning, maxdist, shrink=True, dual=False, findsubsols=False):
    """oracle/enum_oracle.c::oenum_svp_ex: dual enumeration and sub-solutions.  mut / rdiag: the primal block's."""
    L = lib()
    d = len(rdiag)
    mut = np.ascontiguousarray(mut, np.float64).reshape(d, d)
    rdiag = np.ascontiguousarray(rdiag, np.float64)
    pr = None if pruning is None else np.ascontiguousarray(pruning, np.float64)
    sol = np.zeros(d)
    best = C.c_double()
    nodes = np.zeros(d, np.uint64)
    subdist = np.full(d, -1.0)
    subsol = np.zeros((d, d))
    P = C.POINTER
    L.oenum_svp_ex.restype = C.c_long
    L.oenum_svp_ex.argtypes = [C.c_int, P(C.c_double), P(C.c_double), P(C.c_double), C.c_double, C.c_int, C.c_int,
                               C.c_int, P(C.c_double), P(C.c_double), P(C.c_uint64), P(C.c_double), P(C.c_double)]
    n = L.oenum_svp_ex(d, mut.ctypes.data_as(P(C.c_double)), rdiag.ctypes.data_as(P(C.c_double)),
                       pr.ctypes.data_as(P(C.c_double)) if pr is not None else None, float(maxdist),
                       1 if shrink else 0, 1 if dual else 0, 1 if findsubsols else 0,
                       sol.ctypes.data_as(P(C.c_double)), C.byref(best), nodes.ctypes.data_as(P(C.c_uint64)),
                       subdist.ctypes.data_as(P(C.c_double)), subsol.ctypes.data_as(P(C.c_double)))
    return dict(nsols=int(n), best=best.value, sol=sol, nodes=nodes, subdist=subdist, subsol=subsol)


def read_enum_records(path):
    """Parse the records ref_probe's `enum` appends (layout in oracle/ref_probe.cpp)."""
    raw = open(path, "rb").read()
    off, out = 0, []
    while off < len(raw):
        hdr = np.frombuffer(raw, np.int32, 4, off)
        off += 16
        assert hdr[0] == 0x454E554D
        d, found, mode = int(hdr[1]), int(hdr[2]), int(hdr[3]) & 15
        dual, subsols = bool(int(hdr[3]) & 16), bool(int(hdr[3]) & 32)
        md, best = np.frombuffer(raw, np.float64, 2, off)
        off += 16
        normexp = int(np.frombuffer(raw, np.int64, 1, off)[0])
        off += 8
        sol = np.frombuffer(raw, np.float64, d, off).copy()
        off += 8 * d
        nodes = np.frombuffer(raw, np.uint64, d, off).copy()
        off += 8 * d
        rec = dict(d=d, found=found, mode=mode, maxdist=float(md), best=float(best), normexp=normexp, sol=sol,
                   nodes=nodes, dual=dual, subsols=subsols)
        if mode == 2:
            rec["mut"] = np.frombuffer(raw, np.float64, d * d, off).reshape(d, d).copy()
            off += 8 * d * d
            rec["rdiag"] = np.frombuffer(raw, np.float64, d, off).copy()
            off += 8 * d
            rec["pruning"] = np.frombuffer(raw, np.float64, d, off).copy()
            off += 8 * d
        if subsols:
            rec["subdist"] = np.frombuffer(raw, np.float64, d, off).copy()
            off += 8 * d
            rec["subsol"] = np.frombuffer(raw, np.float64, d * d, off).reshape(d, d).copy()
            off += 8 * d * d
        out.append(rec)
    return out


# ---- Householder ----------------------------------------------------------------------------------------

class _OHH(C.Structure):
    _fields_ = [("d", C.c_int), ("n", C.c_int), ("enable_row_expo", C.c_int), ("n_known_rows", C.c_int),
                ("n_known_cols", C.c_int), ("updated_R", C.c_int),
                ("b", C.POINTER(C.c_int64)), ("bf", C.POINTER(C.c_double)), ("R", C.POINTER(C.c_double)),
                ("V", C.POINTER(C.c_double)), ("sigma", C.POINTER(C.c_double)), ("hist", C.POINTER(C.c_double)),
                ("row_expo", C.POINTER(C.c_int64)), ("init_row_size", C.POINTER(C.c_int)),
                ("norm_square_b", C.POINTER(C.c_double)), ("expo_norm_square_b", C.POINTER(C.c_int64))]


HOUSEHOLDER_ROW_EXPO, HOUSEHOLDER_OP_FORCE_LONG = 1, 4  # householder.h:26-32


class OracleHouseholder:
    """MatHouseholder<Z_NR<long>, FP_NR<double>> restated in C (oracle/hh_oracle.c); reference method names."""

    def __init__(self, b, flags=HOUSEHOLDER_ROW_EXPO | HOUSEHOLDER_OP_FORCE_LONG):
        L = lib()
        b = np.ascontiguousarray(b, dtype=np.int64)
        self.d, self.n = b.shape
        L.ohh_create.restype = C.POINTER(_OHH)
        L.ohh_create.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int64), C.c_int]
        for f, at in [("ohh_destroy", [C.POINTER(_OHH)]), ("ohh_refresh_R_bf", [C.POINTER(_OHH), C.c_int]),
                      ("ohh_refresh_R", [C.POINTER(_OHH), C.c_int]),
                      ("ohh_update_R", [C.POINTER(_OHH), C.c_int, C.c_int]),
                      ("ohh_update_R_last", [C.POINTER(_OHH), C.c_int]),
                      ("ohh_size_reduce", [C.POINTER(_OHH), C.c_int, C.c_int, C.c_int]),
                      ("ohh_swap", [C.POINTER(_OHH), C.c_int, C.c_int]),
                      ("ohh_recover_R", [C.POINTER(_OHH), C.c_int]),
                      ("ohh_set_updated_R_false", [C.POINTER(_OHH)]),
                      ("ohh_hlll", [C.POINTER(_OHH), C.c_double, C.c_double, C.c_double, C.c_double])]:
            getattr(L, f).argtypes = at
        self._p = L.ohh_create(self.d, self.n, b.ctypes.data_as(C.POINTER(C.c_int64)), flags)

    def __del__(self):
        if getattr(self, "_p", None):
            lib().ohh_destroy(self._p)
            self._p = None

    def refresh_R_bf(self, i):
        lib().ohh_refresh_R_bf(self._p, i)

    def refresh_R(self, i):
        lib().ohh_refresh_R(self._p, i)

    def update_R(self, i, last_j=True):
        lib().ohh_update_R(self._p, i, 1 if last_j else 0)

    def update_R_last(self, i):
        lib().ohh_update_R_last(self._p, i)

    def size_reduce(self, k, end, start=0):
        return bool(lib().ohh_size_reduce(self._p, k, end, start))

    def swap(self, i, j):
        lib().ohh_swap(self._p, i, j)

    def recover_R(self, i):
        lib().ohh_recover_R(self._p, i)

    def set_updated_R_false(self):
        lib().ohh_set_updated_R_false(self._p)

    def hlll(self, delta=0.99, eta=0.51, theta=0.001, c=0.1):
        """HLLLReduction::hlll() (hlll.cpp:25-171) on this object; returns the RedStatus."""
        return int(lib().ohh_hlll(self._p, delta, eta, theta, c))

    def state(self):
        m = self._p.contents
        d, n = self.d, self.n

        def arr(ptr, shape, dt):
            cnt = int(np.prod(shape))
            return np.ctypeslib.as_array(ptr, shape=(cnt,)).astype(dt).reshape(shape).copy()
        return dict(d=d, n=n, n_known_rows=m.n_known_rows, n_known_cols=m.n_known_cols, updated_R=m.updated_R,
                    row_expo=arr(m.row_expo, (d,), np.int64), sigma=arr(m.sigma, (d,), np.float64),
                    norm_square_b=arr(m.norm_square_b, (d,), np.float64),
                    expo_norm_square_b=arr(m.expo_norm_square_b, (d,), np.int64),
                    bf=arr(m.bf, (d, n), np.float64), R=arr(m.R, (d, n), np.float64),
                    V=arr(m.V, (d, n), np.float64), b=arr(m.b, (d, n), np.int64))


def read_hh_dumps(path):
    raw = open(path, "rb").read()
    off, out = 0, []
    while off < len(raw):
        hdr = np.frombuffer(raw, np.int32, 6, off)
        off += 24
        assert hdr[0] == 0x48483030
        d, n = int(hdr[1]), int(hdr[2])
        rec = dict(d=d, n=n, n_known_rows=int(hdr[3]), n_known_cols=int(hdr[4]), updated_R=int(hdr[5]))

        def take(dt, shape):
            nonlocal off
            a = np.frombuffer(raw, dt, int(np.prod(shape)), off).reshape(shape).copy()
            off += a.nbytes
            return a
        rec["row_expo"] = take(np.int64, (d,))
        rec["sigma"] = take(np.float64, (d,))
        rec["norm_square_b"] = take(np.float64, (d,))
        rec["expo_norm_square_b"] = take(np.int64, (d,))
        rec["bf"] = take(np.float64, (d, n))
        rec["R"] = take(np.float64, (d, n))
        rec["V"] = take(np.float64, (d, n))
        rec["b"] = take(np.int64, (d, n))
        out.append(rec)
    return out
