"""Host-side mirror of MatHouseholder<Z_NR<long>, FP_NR<double>> (fplll/householder.h:38) over include/b200hh.h."""
import ctypes as C

import numpy as np

from ._lib import B200Error, load

HOUSEHOLDER_DEFAULT, HOUSEHOLDER_ROW_EXPO, HOUSEHOLDER_OP_FORCE_LONG = 0, 1, 4  # householder.h:26-32
# include/b200hh.h (not reference values): the handle keeps U / also U^-T
HOUSEHOLDER_TRANSFORM, HOUSEHOLDER_INV_TRANSFORM = 512, 1024
_P = C.POINTER
_done = False


def _lib():
    global _done
    L = load("libb200hh.so")
    if not _done:
        vp, i = C.c_void_p, C.c_int
        L.b200hh_last_error.restype = C.c_char_p
        L.b200hh_create.argtypes = [_P(vp), i, i, i, i, i, i]
        L.b200hh_destroy.argtypes = [vp]
        L.b200hh_destroy.restype = None
        L.b200hh_set_basis.argtypes = [vp, _P(C.c_int64)]
        L.b200hh_get_basis.argtypes = [vp, _P(C.c_int64)]
        L.b200hh_set_transform.argtypes = [vp, _P(C.c_int64), _P(C.c_int64)]
        L.b200hh_get_transform.argtypes = [vp, _P(C.c_int64), _P(C.c_int64)]
        for f in ("refresh_R_bf", "refresh_R", "update_R_last", "recover_R"):
            getattr(L, "b200hh_" + f).argtypes = [vp, i]
        L.b200hh_update_R.argtypes = [vp, i, i]
        L.b200hh_swap.argtypes = [vp, i, i]
        L.b200hh_size_reduce.argtypes = [vp, i, i, i, _P(C.c_int)]
        L.b200hh_set_updated_R_false.argtypes = [vp]
        L.b200hh_get_state.argtypes = [vp] + [_P(C.c_double)] * 5 + [_P(C.c_int64)] * 2 + [_P(C.c_int)]
        L.b200hh_time_update_R.argtypes = [vp, i, i, _P(C.c_float)]
        L.b200hh_sync.argtypes = [vp]
        L.b200hh_hlll.argtypes = [vp, C.c_double, C.c_double, C.c_double, C.c_double, _P(C.c_int), _P(C.c_uint64)]
        _done = True
    return L


def _ck(rc, what):
    if rc != 0:
        raise B200Error("%s failed (%d): %s" % (what, rc, _lib().b200hh_last_error().decode()))


class MatHouseholder:
    """MatHouseholder(b, flags, device, keep_history, u, u_inv_t): b (d, n) or (batch, d, n) int64; reference method
    names (householder.h).  u ((d, d) or (batch, d, d) int64) makes it the reference's MatHouseholder(b, u, u_inv_t,
    flags) with a non-empty u: U starts as u and takes every integer row operation applied to b (.u reads it back);
    u_inv_t likewise keeps U^-T (.u_inv_t) and needs u.  HOUSEHOLDER_TRANSFORM / HOUSEHOLDER_INV_TRANSFORM in flags
    without the arrays start them at the identity."""

    def __init__(self, b, flags=HOUSEHOLDER_ROW_EXPO | HOUSEHOLDER_OP_FORCE_LONG, device=0, keep_history=True, u=None,
                 u_inv_t=None):
        b = np.ascontiguousarray(b, dtype=np.int64)
        if b.ndim == 2:
            b = b[None]
        self.batch, self.d, self.n = b.shape
        if u_inv_t is not None and u is None:
            raise ValueError("u_inv_t needs u (the reference updates u_inv_t only when u is enabled)")
        if u is not None:
            flags |= HOUSEHOLDER_TRANSFORM
        if u_inv_t is not None:
            flags |= HOUSEHOLDER_INV_TRANSFORM
        self.flags = flags
        self.enable_transform = bool(flags & HOUSEHOLDER_TRANSFORM)
        self.enable_inverse_transform = bool(flags & HOUSEHOLDER_INV_TRANSFORM)
        self._h = C.c_void_p()
        _ck(_lib().b200hh_create(C.byref(self._h), self.batch, self.d, self.n, flags, device, 1 if keep_history else 0),
            "b200hh_create")
        _ck(_lib().b200hh_set_basis(self._h, b.ctypes.data_as(_P(C.c_int64))), "set_basis")
        if u is not None:
            self.set_transform(u, u_inv_t)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            _lib().b200hh_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def refresh_R_bf(self, i):
        _ck(_lib().b200hh_refresh_R_bf(self._h, i), "refresh_R_bf")

    def refresh_R(self, i):
        _ck(_lib().b200hh_refresh_R(self._h, i), "refresh_R")

    def update_R(self, i, last_j=True):
        _ck(_lib().b200hh_update_R(self._h, i, 1 if last_j else 0), "update_R")

    def update_R_last(self, i):
        _ck(_lib().b200hh_update_R_last(self._h, i), "update_R_last")

    def size_reduce(self, k, end, start=0):
        red = np.zeros(self.batch, np.int32)
        _ck(_lib().b200hh_size_reduce(self._h, k, end, start, red.ctypes.data_as(_P(C.c_int))), "size_reduce")
        return red.astype(bool)

    def swap(self, i, j):
        _ck(_lib().b200hh_swap(self._h, i, j), "swap")

    def recover_R(self, i):
        _ck(_lib().b200hh_recover_R(self._h, i), "recover_R")

    def set_updated_R_false(self):
        _ck(_lib().b200hh_set_updated_R_false(self._h), "set_updated_R_false")

    def state(self):
        B, d, n = self.batch, self.d, self.n
        R, V, bf = (np.empty((B, d, n)) for _ in range(3))
        sg, nsb = np.empty((B, d)), np.empty((B, d))
        re, en = np.empty((B, d), np.int64), np.empty((B, d), np.int64)
        meta = np.empty((B, 3), np.int32)
        b = np.empty((B, d, n), np.int64)
        dp = lambda a: a.ctypes.data_as(_P(C.c_double))
        _ck(_lib().b200hh_get_state(self._h, dp(R), dp(V), dp(bf), dp(sg), dp(nsb), re.ctypes.data_as(_P(C.c_int64)),
                                    en.ctypes.data_as(_P(C.c_int64)), meta.ctypes.data_as(_P(C.c_int))), "get_state")
        _ck(_lib().b200hh_get_basis(self._h, b.ctypes.data_as(_P(C.c_int64))), "get_basis")
        return dict(R=R, V=V, bf=bf, sigma=sg, norm_square_b=nsb, row_expo=re, expo_norm_square_b=en, b=b,
                    n_known_rows=meta[:, 0].copy(), n_known_cols=meta[:, 1].copy(), updated_R=meta[:, 2].copy())

    def hlll(self, delta=0.99, eta=0.51, theta=0.001, c=0.1):
        """HLLLReduction(m, delta, eta, theta, c, flags).hlll() (hlll.cpp:25-171), whole loop on the device.
        Returns (status per lattice, main-loop iterations per lattice)."""
        st = np.zeros(self.batch, np.int32)
        it = np.zeros(self.batch, np.uint64)
        _ck(_lib().b200hh_hlll(self._h, delta, eta, theta, c, st.ctypes.data_as(_P(C.c_int)),
                               it.ctypes.data_as(_P(C.c_uint64))), "hlll")
        return st, it

    def get_basis(self):
        b = np.empty((self.batch, self.d, self.n), np.int64)
        _ck(_lib().b200hh_get_basis(self._h, b.ctypes.data_as(_P(C.c_int64))), "get_basis")
        return b

    def _mats(self, a):
        """(d, d) broadcast to every lattice, or (batch, d, d); None stays None"""
        if a is None:
            return None
        a = np.asarray(a, np.int64)
        if a.shape not in ((self.d, self.d), (self.batch, self.d, self.d)):
            raise ValueError("expected shape (%d, %d) or (%d, %d, %d), got %s"
                             % (self.d, self.d, self.batch, self.d, self.d, a.shape))
        return np.ascontiguousarray(np.broadcast_to(a, (self.batch, self.d, self.d)))

    def set_transform(self, u=None, u_inv_t=None):
        """replaces U and / or U^-T: (d, d) (every lattice) or (batch, d, d) int64; None leaves that matrix alone"""
        u, ut = self._mats(u), self._mats(u_inv_t)
        p = lambda a: None if a is None else a.ctypes.data_as(_P(C.c_int64))
        _ck(_lib().b200hh_set_transform(self._h, p(u), p(ut)), "set_transform")

    def _get(self, inverse):
        out = np.empty((self.batch, self.d, self.d), np.int64)
        p = out.ctypes.data_as(_P(C.c_int64))
        _ck(_lib().b200hh_get_transform(self._h, None if inverse else p, p if inverse else None), "get_transform")
        return out

    @property
    def u(self):
        """U of a transform object, (batch, d, d) int64"""
        return self._get(False)

    @property
    def u_inv_t(self):
        """U^-T of an inverse-transform object, (batch, d, d) int64"""
        return self._get(True)

    def sync(self):
        _ck(_lib().b200hh_sync(self._h), "sync")

    def time_update_R(self, i, reps):
        ms = C.c_float()
        _ck(_lib().b200hh_time_update_R(self._h, i, reps, C.byref(ms)), "time_update_R")
        return ms.value


RED_HLLL_FAILURE, RED_HLLL_NORM_FAILURE, RED_HLLL_SR_FAILURE = 9, 10, 11  # defs.h:164-166


def hlll_reduction(b, delta=0.99, eta=0.51, theta=0.001, c=0.1, device=0, u=None, u_inv=None):
    """hlll_reduction(ZZ_mat<long>& b, [u, [u_inv,]] delta, eta, theta, c, HM_FAST, FT_DOUBLE) — fplll/wrapper.cpp:789-806
    and :1055-1087 with defaults LLL_DEF_DELTA / LLL_DEF_ETA / HLLL_DEF_THETA / HLLL_DEF_C (defs.h:143-151).  b: (d, n)
    or (batch, d, n) int64.  Returns (reduced basis, status) — per lattice for a batch; the input array is not
    modified.  u and u_inv (int64 arrays of b's leading shape with (d, d) last) are overwritten IN PLACE with the
    transform of the call, starting from the identity as the reference does (gen_identity): u * b_in == b_out, and
    u_inv = U^-1 (the reference runs with u_inv transposed and transposes it back).  u_inv needs u."""
    a = np.ascontiguousarray(b, dtype=np.int64)
    single = a.ndim == 2
    if u_inv is not None and u is None:
        raise ValueError("u_inv needs u (the reference updates u_inv only when u is enabled)")
    for name, t in (("u", u), ("u_inv", u_inv)):
        if t is not None and (not isinstance(t, np.ndarray) or t.dtype != np.int64 or
                              t.shape != a.shape[:-2] + (a.shape[-2], a.shape[-2])):
            raise ValueError("%s must be an int64 array of shape %s" % (name, a.shape[:-2] + (a.shape[-2],) * 2))
    eye = np.eye(a.shape[-2], dtype=np.int64)
    m = MatHouseholder(a, HOUSEHOLDER_ROW_EXPO | HOUSEHOLDER_OP_FORCE_LONG, device=device, keep_history=True,
                       u=None if u is None else eye, u_inv_t=None if u_inv is None else eye)
    try:
        st, _ = m.hlll(delta, eta, theta, c)
        out = m.get_basis()
        uo = m.u if u is not None else None
        ui = m.u_inv_t.transpose(0, 2, 1) if u_inv is not None else None
    finally:
        m.close()
    if u is not None:
        u[...] = uo[0] if single else uo
    if u_inv is not None:
        u_inv[...] = ui[0] if single else ui
    return (out[0], int(st[0])) if single else (out, st)
