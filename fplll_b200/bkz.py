"""Host-side mirror of fplll's BKZ entry point over the C-ABI of include/b200bkz.h:
bkz_reduction(ZZ_mat&, BKZParam) — fplll/bkz.h:357-426, fplll/bkz_param.h:68-176."""
import ctypes as C
import os

import numpy as np

from ._lib import B200Error, load

BKZ_DEFAULT, BKZ_VERBOSE, BKZ_NO_LLL, BKZ_MAX_LOOPS, BKZ_MAX_TIME = 0, 1, 2, 4, 8  # defs.h:264-274
BKZ_BOUNDED_LLL, BKZ_AUTO_ABORT, BKZ_GH_BND = 0x10, 0x20, 0x80
BKZ_SD_VARIANT, BKZ_SLD_RED = 0x100, 0x200  # self-dual BKZ, slide reduction (mutually exclusive)
BKZ_SHRINK_RADIUS = 0x10000  # include/b200bkz.h: not a reference flag (order-dependent enumeration like the reference's)
RED_BKZ_FAILURE, RED_BKZ_TIME_LIMIT, RED_BKZ_LOOPS_LIMIT = 6, 7, 8
_P = C.POINTER
DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "strategies_default.npz")


class _Param(C.Structure):
    _fields_ = [("block_size", C.c_int), ("delta", C.c_double), ("flags", C.c_int), ("max_loops", C.c_int),
                ("max_time", C.c_double), ("auto_abort_scale", C.c_double), ("auto_abort_max_no_dec", C.c_int),
                ("gh_factor", C.c_double), ("min_success_probability", C.c_double),
                ("rerandomization_density", C.c_int), ("seed", C.c_uint64)]


class _Stats(C.Structure):
    _fields_ = [("status", C.c_int), ("tours", C.c_int), ("enum_nodes", C.c_uint64), ("enum_calls", C.c_long),
                ("lll_calls", C.c_long), ("sizered_calls", C.c_long), ("sec_total", C.c_double),
                ("sec_enum", C.c_double), ("sec_lll", C.c_double), ("sec_other", C.c_double),
                ("sec_ops", C.c_double), ("sec_get", C.c_double), ("op_calls", C.c_long), ("ops_total", C.c_long),
                ("get_calls", C.c_long),
                ("r00_before", C.c_double), ("r00_after", C.c_double), ("slope_before", C.c_double),
                ("slope_after", C.c_double)]


_done = False


def _lib():
    global _done
    L = load(os.environ.get("B200_BKZ_LIB", "libb200bkz.so"))  # B200_BKZ_LIB: profiling build (see csrc/gso_lll.cuh)
    if not _done:
        L.b200bkz_last_error.restype = C.c_char_p
        L.b200bkz_default_param.argtypes = [_P(_Param), C.c_int]
        L.b200bkz_default_param.restype = None
        L.b200bkz_create.argtypes = [_P(C.c_void_p), _P(C.c_int), C.c_int]
        L.b200bkz_destroy.argtypes = [C.c_void_p]
        L.b200bkz_destroy.restype = None
        L.b200bkz_add_strategy.argtypes = [C.c_void_p, C.c_int, _P(C.c_int), C.c_int, _P(C.c_double), _P(C.c_double),
                                           _P(C.c_double), C.c_int]
        L.b200bkz_reduce.argtypes = [C.c_void_p, C.c_int, C.c_int, _P(C.c_int64), _P(_Param), _P(_Stats)]
        L.b200bkz_reduce_transform.argtypes = [C.c_void_p, C.c_int, C.c_int, _P(C.c_int64), _P(C.c_int64),
                                               _P(_Param), _P(_Stats)]
        _done = True
    return L


def load_strategies(path=DATA):
    """the table of strategies/default.json (bkz_param.cpp:82-157) in array form: {block_size: (pre, ghf, exp, coef)}"""
    z = np.load(path)
    return {int(bs): (z["pre_%d" % bs], z["ghf_%d" % bs], z["exp_%d" % bs], z["coef_%d" % bs])
            for bs in z["block_sizes"]}


class BKZParam:
    """BKZParam(block_size, strategies, delta, flags, max_loops, ...) — bkz_param.h:68-176, same defaults."""

    def __init__(self, block_size, strategies=None, delta=0.99, flags=BKZ_DEFAULT, max_loops=0, max_time=0.0,
                 auto_abort_scale=1.0, auto_abort_max_no_dec=5, gh_factor=1.1, min_success_probability=0.5,
                 rerandomization_density=3, seed=0):
        self.block_size, self.strategies, self.delta, self.flags = block_size, strategies, delta, flags
        self.max_loops, self.max_time = max_loops, max_time
        self.auto_abort_scale, self.auto_abort_max_no_dec = auto_abort_scale, auto_abort_max_no_dec
        self.gh_factor, self.min_success_probability = gh_factor, min_success_probability
        self.rerandomization_density, self.seed = rerandomization_density, seed


def bkz_reduction(b, param, devices=None, u=None):
    """bkz_reduction(ZZ_mat<long>& b, BKZParam) in the int64 regime (bkz.cpp:812-836): reduces the (d, n) int64 numpy
    array IN PLACE.  BKZ 2.0 by default, self-dual BKZ with BKZ_SD_VARIANT, slide reduction with BKZ_SLD_RED.  Returns (RedStatus, stats dict).  param.strategies: None (EmptyStrategy for every block size),
    "default" (the reference's strategies/default.json table) or a dict as returned by load_strategies.
    u: a (d, d) int64 array overwritten with the transform of the whole call, U * b_in == b_out (bkz_reduction(b, u,
    param), which starts u at the identity, bkz.cpp:857-859); b, status and stats are those of the call without u."""
    L = _lib()
    arr = np.ascontiguousarray(b, dtype=np.int64)
    d, n = arr.shape
    h = C.c_void_p()
    dv = np.ascontiguousarray(devices if devices is not None else [0], np.int32)
    rc = L.b200bkz_create(C.byref(h), dv.ctypes.data_as(_P(C.c_int)), len(dv))
    if rc:
        raise B200Error("b200bkz_create failed (%d): %s" % (rc, L.b200bkz_last_error().decode()))
    try:
        strat = param.strategies
        if strat == "default":
            strat = load_strategies()
        for bs, (pre, ghf, ex, coef) in (strat or {}).items():
            pre = np.ascontiguousarray(pre, np.int32)
            ghf, ex = np.ascontiguousarray(ghf, np.float64), np.ascontiguousarray(ex, np.float64)
            coef = np.ascontiguousarray(coef, np.float64)
            L.b200bkz_add_strategy(h, int(bs), pre.ctypes.data_as(_P(C.c_int)), len(pre),
                                   ghf.ctypes.data_as(_P(C.c_double)), ex.ctypes.data_as(_P(C.c_double)),
                                   coef.ctypes.data_as(_P(C.c_double)), len(ghf))
        p = _Param()
        L.b200bkz_default_param(C.byref(p), param.block_size)
        p.delta, p.flags, p.max_loops, p.max_time = param.delta, param.flags, param.max_loops, param.max_time
        p.auto_abort_scale, p.auto_abort_max_no_dec = param.auto_abort_scale, param.auto_abort_max_no_dec
        p.gh_factor, p.min_success_probability = param.gh_factor, param.min_success_probability
        p.rerandomization_density, p.seed = param.rerandomization_density, param.seed
        st = _Stats()
        if u is None:
            rc = L.b200bkz_reduce(h, d, n, arr.ctypes.data_as(_P(C.c_int64)), C.byref(p), C.byref(st))
        else:
            ua = np.eye(d, dtype=np.int64)
            rc = L.b200bkz_reduce_transform(h, d, n, arr.ctypes.data_as(_P(C.c_int64)), ua.ctypes.data_as(_P(C.c_int64)),
                                            C.byref(p), C.byref(st))
        if rc:
            raise B200Error("b200bkz_reduce failed (%d): %s" % (rc, L.b200bkz_last_error().decode()))
    finally:
        L.b200bkz_destroy(h)
    b[...] = arr
    if u is not None:
        u[...] = ua
    return st.status, {f: getattr(st, f) for f, _ in _Stats._fields_}
