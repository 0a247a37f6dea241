"""Host-side mirror of MatGSO<Z_NR<long>, FP_NR<double>> (fplll/gso.h:33, fplll/gso_interface.h:59) over the
C-ABI of include/b200gso.h.  A MatGSO here is a BATCH of independent lattices (batch=1 == the reference object);
method names / argument order follow the reference so the parity tests read like tests/test_gso.cpp."""
import ctypes as C

import numpy as np

from ._lib import B200Error, load

GSO_DEFAULT, GSO_INT_GRAM, GSO_ROW_EXPO, GSO_OP_FORCE_LONG = 0, 1, 2, 4  # gso_interface.h:26-32
GSO_TRANSFORM = 512  # include/b200gso.h B200GSO_TRANSFORM (not a reference value): the handle keeps U
RED_SUCCESS, RED_GSO_FAILURE, RED_BABAI_FAILURE, RED_LLL_FAILURE = 0, 2, 3, 4  # defs.h:153-169
# b200gso_op types (include/b200gso.h)
OP_ROW_ADDMUL, OP_MOVE_ROW, OP_ROW_SWAP, OP_ROW_OP_END, OP_NEGATE = 1, 2, 3, 4, 5
_OP_DTYPE = np.dtype([("type", np.int32), ("a", np.int32), ("b", np.int32), ("pad", np.int32), ("x", np.float64)])

_P = C.POINTER
_sig_done = False


def _lib():
    global _sig_done
    L = load("libb200gso.so")
    if not _sig_done:
        vp, i, dp, ip, lp = C.c_void_p, C.c_int, _P(C.c_double), _P(C.c_int), _P(C.c_long)
        i64p = _P(C.c_int64)
        L.b200gso_version.restype = C.c_char_p
        L.b200gso_last_error.restype = C.c_char_p
        L.b200gso_create.argtypes = [_P(vp), i, i, i, i, i]
        L.b200gso_destroy.argtypes = [vp]
        L.b200gso_destroy.restype = None
        L.b200gso_set_basis.argtypes = [vp, i64p]
        L.b200gso_set_basis_dev.argtypes = [vp, vp]
        L.b200gso_get_basis.argtypes = [vp, i64p]
        L.b200gso_upload_row.argtypes = [vp, i, i64p]
        L.b200gso_set_transform.argtypes = [vp, i64p]
        L.b200gso_get_transform.argtypes = [vp, i64p]
        L.b200gso_discover_all_rows.argtypes = [vp]
        L.b200gso_update_gso_row.argtypes = [vp, i, i, ip]
        L.b200gso_update_gso.argtypes = [vp, ip]
        L.b200gso_update_gso_blocked.argtypes = [vp, i, ip]
        L.b200gso_row_addmul_we.argtypes = [vp, i, i, dp, lp]
        L.b200gso_row_op_begin.argtypes = [vp, i, i]
        L.b200gso_row_op_end.argtypes = [vp, i, i]
        L.b200gso_row_swap.argtypes = [vp, i, i]
        L.b200gso_move_row.argtypes = [vp, i, i]
        L.b200gso_set_r.argtypes = [vp, i, i, dp]
        L.b200gso_get_state.argtypes = [vp, dp, dp, dp, dp, i64p, ip, ip, ip]
        L.b200gso_get_mu_r_row.argtypes = [vp, i, dp, dp, ip]
        L.b200gso_lll.argtypes = [vp, C.c_double, C.c_double, ip, lp]
        L.b200gso_lll_range.argtypes = [vp, C.c_double, C.c_double, i, i, i, i, ip, lp]
        L.b200gso_size_reduction.argtypes = [vp, C.c_double, i, i, i, ip]
        L.b200gso_negate_row_of_b.argtypes = [vp, i]
        L.b200gso_get_block.argtypes = [vp, i, i, i, dp, dp, lp]
        L.b200gso_get_r_diag.argtypes = [vp, i, i, i, dp, lp]
        L.b200gso_apply_ops.argtypes = [vp, C.c_void_p, i]
        L.b200gso_time_update_row.argtypes = [vp, i, i, i, _P(C.c_float), _P(C.c_float)]
        L.b200gso_sync.argtypes = [vp]
        L.b200gso_resident_lattices.argtypes = [vp]
        _sig_done = True
    return L


def _ck(rc, what):
    if rc != 0:
        raise B200Error("%s failed (%d): %s" % (what, rc, _lib().b200gso_last_error().decode()))


def _ptr(a, ct):
    return a.ctypes.data_as(_P(ct))


class MatGSO:
    """MatGSO(b, flags, device, u): b is (d, n) or (batch, d, n) int64.  u (d, d) or (batch, d, d) int64 makes it a
    transform object like the reference's MatGSO(b, u, u_inv_t = {}, flags) with a non-empty u (enable_transform): U
    starts as u and takes every integer row operation applied to b (.u reads it back).  GSO_TRANSFORM in flags without
    u starts U at the identity.  One intended divergence from the reference: negate_row_of_b / OP_NEGATE negate the row
    of U too, so that U * B_in == B always holds (include/b200gso.h).  u_inv_t is not supported; GSO_INT_GRAM raises
    like an unsupported template instantiation."""

    def __init__(self, b, flags=GSO_ROW_EXPO, device=0, u=None):
        b = np.ascontiguousarray(b, dtype=np.int64)
        if b.ndim == 2:
            b = b[None]
        self.batch, self.d, self.n = b.shape
        if u is not None:
            flags |= GSO_TRANSFORM
        self.flags = flags
        self.enable_row_expo = bool(flags & GSO_ROW_EXPO)
        self.enable_transform = bool(flags & GSO_TRANSFORM)
        self._h = C.c_void_p()
        _ck(_lib().b200gso_create(C.byref(self._h), self.batch, self.d, self.n, flags, device), "b200gso_create")
        _ck(_lib().b200gso_set_basis(self._h, _ptr(b, C.c_int64)), "b200gso_set_basis")
        if u is not None:
            self.set_transform(u)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            _lib().b200gso_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    # ---- reference API -------------------------------------------------------------------------------
    def discover_all_rows(self):
        _ck(_lib().b200gso_discover_all_rows(self._h), "discover_all_rows")

    def update_gso_row(self, i, last_j=None, want_ok=True):
        """update_gso_row(i, last_j) -> bool per lattice.  want_ok=False skips the read-back (stream-ordered, no sync)."""
        lj = i if last_j is None else last_j
        if not want_ok:
            _ck(_lib().b200gso_update_gso_row(self._h, i, lj, None), "update_gso_row")
            return None
        ok = np.zeros(self.batch, np.int32)
        _ck(_lib().b200gso_update_gso_row(self._h, i, lj, _ptr(ok, C.c_int)), "update_gso_row")
        return ok.astype(bool)

    def update_gso(self):
        ok = np.zeros(self.batch, np.int32)
        _ck(_lib().b200gso_update_gso(self._h, _ptr(ok, C.c_int)), "update_gso")
        return ok.astype(bool)

    def update_gso_blocked(self, gram_mode=0):
        """update_gso() with the Gram matrix recomputed in 32x32 tiles first (0: reference-order dot
        products, 1: fp64 tensor-core DMMA) — include/b200gso.h."""
        ok = np.zeros(self.batch, np.int32)
        _ck(_lib().b200gso_update_gso_blocked(self._h, gram_mode, _ptr(ok, C.c_int)), "update_gso_blocked")
        return ok.astype(bool)

    def row_addmul_we(self, i, j, x, expo_add=0):
        x = np.ascontiguousarray(np.broadcast_to(np.asarray(x, np.float64), (self.batch,)))
        e = np.ascontiguousarray(np.broadcast_to(np.asarray(expo_add, np.int64), (self.batch,)))
        _ck(_lib().b200gso_row_addmul_we(self._h, i, j, _ptr(x, C.c_double), _ptr(e, C.c_long)), "row_addmul_we")

    def row_addmul(self, i, j, x):
        self.row_addmul_we(i, j, x, 0)

    def row_op_begin(self, first, last):
        _ck(_lib().b200gso_row_op_begin(self._h, first, last), "row_op_begin")

    def row_op_end(self, first, last):
        _ck(_lib().b200gso_row_op_end(self._h, first, last), "row_op_end")

    def row_swap(self, i, j):
        _ck(_lib().b200gso_row_swap(self._h, i, j), "row_swap")

    def move_row(self, old_r, new_r):
        _ck(_lib().b200gso_move_row(self._h, old_r, new_r), "move_row")

    def set_r(self, i, j, f):
        f = np.ascontiguousarray(np.broadcast_to(np.asarray(f, np.float64), (self.batch,)))
        _ck(_lib().b200gso_set_r(self._h, i, j, _ptr(f, C.c_double)), "set_r")

    def negate_row_of_b(self, i):
        """MatGSO::negate_row_of_b (gso.h:291-297): integer row only; the caller brackets it with row_op_begin/end."""
        _ck(_lib().b200gso_negate_row_of_b(self._h, i), "negate_row_of_b")

    def get_block(self, first, beta, lattice=0):
        """What Enumeration::enumerate pulls out of the GSO for block [first, first+beta) (enumerate_ext.cpp:91-148):
        mut[k, j] = get_mu(first+j, first+k) for j > k (row_expo applied) and get_r_exp(first+i, first+i) as
        (mantissa[beta], exponent[beta])."""
        mut = np.empty((beta, beta))
        rm = np.empty(beta)
        re = np.empty(beta, np.int64)
        _ck(_lib().b200gso_get_block(self._h, lattice, first, beta, _ptr(mut, C.c_double), _ptr(rm, C.c_double),
                                     _ptr(re, C.c_long)), "get_block")
        return mut, rm, re

    def get_r_diag(self, first, count, lattice=0):
        """get_r_exp(first+i, first+i), i < count (gso_interface.h:704-722): (mantissa, exponent)."""
        rm = np.empty(count)
        re = np.empty(count, np.int64)
        _ck(_lib().b200gso_get_r_diag(self._h, lattice, first, count, _ptr(rm, C.c_double), _ptr(re, C.c_long)),
            "get_r_diag")
        return rm, re

    def upload_row(self, i, rows):
        rows = np.ascontiguousarray(rows, dtype=np.int64).reshape(self.batch, self.n)
        _ck(_lib().b200gso_upload_row(self._h, i, _ptr(rows, C.c_int64)), "upload_row")

    def set_transform(self, u):
        """replaces U: (d, d) (every lattice) or (batch, d, d) int64"""
        u = np.ascontiguousarray(np.broadcast_to(np.asarray(u, np.int64), (self.batch, self.d, self.d)))
        _ck(_lib().b200gso_set_transform(self._h, _ptr(u, C.c_int64)), "set_transform")

    # ---- state ---------------------------------------------------------------------------------------
    @property
    def u(self):
        """U of a transform object, (batch, d, d) int64"""
        out = np.empty((self.batch, self.d, self.d), np.int64)
        _ck(_lib().b200gso_get_transform(self._h, _ptr(out, C.c_int64)), "get_transform")
        return out

    @property
    def b(self):
        out = np.empty((self.batch, self.d, self.n), np.int64)
        _ck(_lib().b200gso_get_basis(self._h, _ptr(out, C.c_int64)), "get_basis")
        return out

    def state(self):
        B, d, n = self.batch, self.d, self.n
        mu, r, gf = (np.empty((B, d, d)) for _ in range(3))
        bf = np.empty((B, d, n))
        re = np.empty((B, d), np.int64)
        vc, irs = np.empty((B, d), np.int32), np.empty((B, d), np.int32)
        meta = np.empty((B, 4), np.int32)
        _ck(_lib().b200gso_get_state(self._h, _ptr(mu, C.c_double), _ptr(r, C.c_double), _ptr(gf, C.c_double),
                                     _ptr(bf, C.c_double), _ptr(re, C.c_int64), _ptr(vc, C.c_int),
                                     _ptr(irs, C.c_int), _ptr(meta, C.c_int)), "get_state")
        return dict(mu=mu, r=r, gf=gf, bf=bf, row_expo=re, gso_valid_cols=vc, init_row_size=irs,
                    n_known_rows=meta[:, 0].copy(), n_known_cols=meta[:, 1].copy(),
                    n_source_rows=meta[:, 2].copy(), b=self.b)

    def get_mu_r_row(self, i, out=None):
        """rows i of mu and r and gso_valid_cols[i] for every lattice.  out=(mu, r, valid) reuses caller buffers
        (pinned host memory makes the copies asynchronous DMA)."""
        if out is None:
            out = (np.empty((self.batch, self.d)), np.empty((self.batch, self.d)), np.empty(self.batch, np.int32))
        mu, r, v = out
        _ck(_lib().b200gso_get_mu_r_row(self._h, i, _ptr(mu, C.c_double), _ptr(r, C.c_double), _ptr(v, C.c_int)),
            "get_mu_r_row")
        return mu, r, v

    def get_mu_matrix(self):
        return self.state()["mu"]

    def get_r_matrix(self):
        return self.state()["r"]

    # ---- device LLL ----------------------------------------------------------------------------------
    def lll(self, delta=0.99, eta=0.51, kappa_min=0, kappa_start=0, kappa_end=-1, size_reduction_start=0):
        """LLLReduction(m, delta, eta, LLL_DEFAULT).lll(kappa_min, kappa_start, kappa_end, size_reduction_start) on every
        lattice; returns (status[batch], stats)."""
        st = np.zeros(self.batch, np.int32)
        stats = np.zeros((self.batch, 4), np.int64)
        if (kappa_min, kappa_start, kappa_end, size_reduction_start) == (0, 0, -1, 0):
            _ck(_lib().b200gso_lll(self._h, delta, eta, _ptr(st, C.c_int), _ptr(stats, C.c_long)), "lll")
        else:
            _ck(_lib().b200gso_lll_range(self._h, delta, eta, kappa_min, kappa_start, kappa_end, size_reduction_start,
                                         _ptr(st, C.c_int), _ptr(stats, C.c_long)), "lll")
        return st, dict(n_swaps=stats[:, 0], final_kappa=stats[:, 1], zeros=stats[:, 2], babai_iters=stats[:, 3])

    def size_reduction(self, eta=0.51, kappa_min=0, kappa_end=-1, size_reduction_start=0):
        """LLLReduction(m, 0.99, eta, LLL_DEFAULT).size_reduction(kappa_min, kappa_end, size_reduction_start) on every
        lattice; returns status[batch] (RED_GSO_FAILURE where the reference returns false without a status)."""
        st = np.zeros(self.batch, np.int32)
        _ck(_lib().b200gso_size_reduction(self._h, eta, kappa_min, kappa_end, size_reduction_start, _ptr(st, C.c_int)),
            "size_reduction")
        return st

    def apply_ops(self, ops):
        """Runs a list of (type, a, b, x) in one launch on every lattice (b200gso_apply_ops): OP_ROW_ADDMUL
        row_addmul(a, b, x), OP_MOVE_ROW move_row(a, b), OP_ROW_SWAP row_swap(a, b), OP_ROW_OP_END row_op_end(a, b),
        OP_NEGATE negate_row_of_b(a)."""
        arr = np.zeros(len(ops), _OP_DTYPE)
        for k, (t, a, b, x) in enumerate(ops):
            arr[k] = (t, a, b, 0, x)
        _ck(_lib().b200gso_apply_ops(self._h, arr.ctypes.data_as(C.c_void_p), len(ops)), "apply_ops")

    def time_update_row(self, i, reps, invalidate=True):
        """returns (mean ms of one update_gso_row launch, total ms of the `reps` steps), CUDA events on the handle's stream"""
        ms, tot = C.c_float(), C.c_float()
        _ck(_lib().b200gso_time_update_row(self._h, i, reps, 1 if invalidate else 0, C.byref(ms), C.byref(tot)),
            "time_update_row")
        return ms.value, tot.value

    def resident_lattices(self):
        return int(_lib().b200gso_resident_lattices(self._h))

    def sync(self):
        _ck(_lib().b200gso_sync(self._h), "sync")


def lll_reduction(b, delta=0.99, eta=0.51, device=0, u=None):
    """lll_reduction(ZZ_mat<long>& b, [u,] delta, eta, LM_FAST, FT_DOUBLE) (wrapper.h:136-157, wrapper.cpp:538-553):
    reduces b IN PLACE (numpy int64 array (d,n) or (batch,d,n)); returns RedStatus (int or array).  u ((d,d) or
    (batch,d,d) int64) is overwritten with the transform of the whole call, U * b_in == b_out (the reference starts it
    at the identity, u.gen_identity(d) in FPLLL_DEFINE_LLL)."""
    arr = np.asarray(b)
    d = arr.shape[-2]
    m = MatGSO(arr, GSO_ROW_EXPO | GSO_OP_FORCE_LONG, device, u=None if u is None else np.eye(d, dtype=np.int64))
    st, _ = m.lll(delta, eta)
    out = m.b
    uo = m.u if u is not None else None
    m.close()
    # zeros_first (wrapper.cpp:732, util.cpp:257-287): zero rows parked at the end by LLL move to the front, and the
    # rows of u move with them
    for l in range(out.shape[0]):
        nz = np.any(out[l] != 0, axis=1)
        perm = np.concatenate([np.flatnonzero(~nz), np.flatnonzero(nz)])
        out[l] = out[l][perm]
        if uo is not None:
            uo[l] = uo[l][perm]
    if arr.ndim == 2:
        b[...] = out[0]
        if u is not None:
            u[...] = uo[0]
        return int(st[0])
    b[...] = out
    if u is not None:
        u[...] = uo
    return st
