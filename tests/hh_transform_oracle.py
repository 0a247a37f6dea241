"""The transform U and U^-T next to the CPU oracle's MatHouseholder (oracle/hh_oracle.c, OracleHouseholder), TEST
INFRASTRUCTURE ONLY.

The reference's MatHouseholder(b, u, u_inv_t, flags) applies each integer row operation on b to u and u_inv_t as well
(householder.cpp:372-398, :455-559): size_reduce's row_addmul_we(k, i, x, expo_add) adds lx * 2^expo * u[i] to u[k] over
all d columns and (-lx) * 2^expo * u_inv_t[k] to u_inv_t[i], with the lx and expo of b's update and Z_NR<long>'s
wrapping arithmetic; swap(i, j) swaps rows i and j of both.  The C oracle does not keep them, so this wrapper does:
  * size_reduce recomputes, from the C oracle's R and row exponents before the call, the coefficients
    row_addmul_we receives (householder.cpp:403-451, rnd_we nr_FP_d.inl:226-233, get_si_exp_we :46-53), replaying the
    float update of R[k] between them as hh_oracle.c does.  After the C call it checks that R[k] and b[k] came out as
    that replay says: the (i, lx, expo) sequence is the one the C oracle applied to b, and it is applied to U and U^-T.
  * swap swaps their rows after the C call.
  * hlll restates HLLLReduction::hlll() (hlll.cpp:25-171, as ohh_hlll) over these primitives; its basis and status
    are checked against the C oracle's own ohh_hlll (tests/test_hh_transform_cpu.py)."""
import math

import numpy as np

from oracle import oracle as O

ROW_EXPO, FORCE_LONG = O.HOUSEHOLDER_ROW_EXPO, O.HOUSEHOLDER_OP_FORCE_LONG


def _fexpo(x):
    """ilogb(x) + 1 (hh_oracle.c fexpo); 0 has no exponent: ilogb gives INT_MIN there"""
    if x == 0:
        return -(1 << 31) + 1
    return math.frexp(float(x))[1]


def _addmul(mat, a, c, lx, expo):
    """row a += (lx * 2^expo) * row c, wrapping mod 2^64; a shift by 64 or more gives 0 (as hh_oracle.c does on b)"""
    with np.errstate(over="ignore"):
        t = mat[c].astype(np.uint64) * np.uint64(lx % (1 << 64))
        if expo:
            t = np.zeros_like(t) if expo >= 64 else t << np.uint64(expo)
        mat[a] = (mat[a].astype(np.uint64) + t).astype(np.int64)


class TransformOracle:
    """OracleHouseholder(b, flags) with U (u, or the identity) and, when u_inv_t is given, U^-T.  The reference's
    method names; .u / .u_inv_t are (d, d) int64 (u_inv_t None when it is not kept)."""

    def __init__(self, b, flags=ROW_EXPO | FORCE_LONG, u=None, u_inv_t=None):
        if u_inv_t is not None and u is None:
            raise ValueError("u_inv_t needs u (the reference updates u_inv_t only when u is enabled)")
        self.m = O.OracleHouseholder(b, flags)
        self.d, self.n = self.m.d, self.m.n
        self.row_expo_en = bool(flags & ROW_EXPO)
        eye = np.eye(self.d, dtype=np.int64)
        self.u = (eye if u is None else np.array(u, dtype=np.int64)).reshape(self.d, self.d).copy()
        self.u_inv_t = None if u_inv_t is None else np.array(u_inv_t, dtype=np.int64).reshape(self.d, self.d).copy()
        c = self.m._p.contents
        d, n = self.d, self.n
        # views of the C object's arrays (allocated once in ohh_create)
        self._R = np.ctypeslib.as_array(c.R, shape=(d, n))
        self._b = np.ctypeslib.as_array(c.b, shape=(d, n))
        self._re = np.ctypeslib.as_array(c.row_expo, shape=(d,))
        self._nsb = np.ctypeslib.as_array(c.norm_square_b, shape=(d,))
        self._ensb = np.ctypeslib.as_array(c.expo_norm_square_b, shape=(d,))

    # ---- the primitives that do not touch the integer basis ----
    def refresh_R_bf(self, i):
        self.m.refresh_R_bf(i)

    def refresh_R(self, i):
        self.m.refresh_R(i)

    def update_R(self, i, last_j=True):
        self.m.update_R(i, last_j)

    def update_R_last(self, i):
        self.m.update_R_last(i)

    def recover_R(self, i):
        self.m.recover_R(i)

    def set_updated_R_false(self):
        self.m.set_updated_R_false()

    def state(self):
        return self.m.state()

    # ---- the two that do ----
    def size_reduce(self, k, end, start=0):
        R, re = self._R, self._re
        rk = R[k].copy()
        ops = []
        for i in range(end - 1, start - 1, -1):
            f = rk[i] / R[i, i]
            de = int(re[k] - re[i])
            if not (_fexpo(f) + de >= 53):
                f = math.ldexp(float(np.rint(math.ldexp(f, de))), -de)
            f = -f
            if f != 0:
                e = _fexpo(f) + de - 63
                expo = e if e > 0 else 0
                ops.append((i, int(math.ldexp(f, de - expo)), expo))
                # R[k] += x R[i] over columns [0, k) (R[i].addmul(R[j], x, i) in householder.cpp:553-558)
                if f == 1.0:
                    rk[:k] = rk[:k] + R[i, :k]
                elif f == -1.0:
                    rk[:k] = rk[:k] - R[i, :k]
                else:
                    rk[:k] = rk[:k] + R[i, :k] * f
        bk = self._b.copy()
        nc = self.m._p.contents.n_known_cols
        reduced = self.m.size_reduce(k, end, start)
        assert reduced == bool(ops), "size_reduce(%d): reduced" % k
        assert np.array_equal(R[k].view(np.int64), rk.view(np.int64)), "size_reduce(%d): R[k] replay" % k
        for i, lx, expo in ops:
            _addmul(bk[:, :nc], k, i, lx, expo)
            _addmul(self.u, k, i, lx, expo)
            if self.u_inv_t is not None:
                _addmul(self.u_inv_t, i, k, -lx, expo)
        assert np.array_equal(self._b, bk), "size_reduce(%d): b replay" % k
        return reduced

    def swap(self, i, j):
        self.m.swap(i, j)
        for mat in (self.u, self.u_inv_t):
            if mat is not None:
                mat[[i, j]] = mat[[j, i]]

    # ---- HLLLReduction::hlll(), hlll.cpp:25-171, as ohh_hlll in hh_oracle.c ----
    def _dot_asc(self, a, beg, end):
        """numvect.h:385-395: products rounded one by one, added in ascending order (cumsum adds sequentially)"""
        return float(np.cumsum(a[beg:end] * a[beg:end])[-1])

    def _size_reduction(self, kappa):
        prev_not_stop = True
        self.update_R(kappa, False)
        self.set_updated_R_false()
        while True:
            if not self.size_reduce(kappa, kappa, 0):
                return
            t, expo0 = self._nsb[kappa], int(self._ensb[kappa])
            self.refresh_R_bf(kappa)
            f1, expo1 = self._nsb[kappa], int(self._ensb[kappa])
            f0 = math.ldexp(0.1 * t, expo0 - expo1)
            not_stop = f1 <= f0
            self.update_R(kappa, False)
            if prev_not_stop or not_stop:
                prev_not_stop = not_stop
            else:
                return

    def hlll(self, delta=0.99, eta=0.51, theta=0.001, c=0.1):
        """returns the RedStatus (0, 10 RED_HLLL_NORM_FAILURE, 11 RED_HLLL_SR_FAILURE); eta and c are not read on this
        path (hlll.h:147-159, hlll.cpp:296-312)"""
        d, n, R, re = self.d, self.n, self._R, self._re
        dR, eR, prev_R, prev_expo = [0.0] * d, [0.0] * d, [0.0] * d, [0] * d

        def compute_dR_eR(k):
            f = R[k, k]
            dR[k] = delta * (f * f)
            eR[k] = delta * R[k, k]

        self.refresh_R_bf(0)
        self.update_R_last(0)
        compute_dR_eR(0)
        if d < 2:
            return 0
        k, k_max, prev_k = 1, 1, -1
        self.refresh_R_bf(1)
        while True:
            self._size_reduction(k)
            # verify_size_reduction(k)
            f1 = math.sqrt(self._dot_asc(R[k], k, n)) if n > k else 0.0
            f1 = f1 * theta
            for i in range(k):
                if abs(R[k, i]) > f1 + math.ldexp(eR[i], int(re[i] - re[k])):
                    return 11
            # lovasz_test(k)
            f1 = self._dot_asc(R[k], 0, k - 1) if k - 1 > 0 else 0.0
            f1 = self._nsb[k] - f1
            expo1 = 2 * int(re[k]) if self.row_expo_en else 0
            f1 = math.ldexp(f1, expo1 - 2 * int(re[k - 1]))
            if dR[k - 1] <= f1:
                self.update_R_last(k)
                compute_dR_eR(k)
                if prev_k == k + 1 and R[k, k] > math.ldexp(prev_R[k], prev_expo[k] - int(re[k])):
                    return 10
                prev_k = k
                prev_R[k], prev_expo[k] = R[k, k], int(re[k])
                k += 1
                if k >= d:
                    return 0
                if k > k_max:
                    k_max = k
                    self.refresh_R_bf(k)
                else:
                    self.refresh_R(k)
            else:
                self.swap(k - 1, k)
                prev_k = k
                if k - 1 == 0:
                    self.refresh_R(0)
                    self.update_R_last(0)
                    compute_dR_eR(0)
                    self.refresh_R(1)
                    k = 1
                else:
                    k -= 1
                    self.recover_R(k)
