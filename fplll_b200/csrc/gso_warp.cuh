// gso_warp.cuh — warp-cooperative device implementation of the MatGSO<long,double> state machine.
//
// One warp owns one lattice.  Every routine is the reference routine named in its comment with the SAME
// per-accumulator operation order (separately rounded multiply then add/sub, ascending index), so results are
// bit-identical to the reference's fp64 GSO — see SURVEY.md §0.8 / §7 "order-preserving schedules".
// All 32 lanes must call these functions together (they contain __syncwarp / shuffles).
#pragma once
#include "gso_layout.cuh"
#include <cuda_runtime.h>
#include <math_constants.h>

namespace b200 {

constexpr unsigned FULL = 0xffffffffu;

// per-warp shared-memory scratch (doubles).  full: vb[n] | rrow | murow | aux | xs  (LLL / Babai);
// compact (update_gso_row only): vb[n] | rrow | murow, aux aliases murow (the diagonal product is formed in place).
struct WarpSmem
{
  double *vb, *rrow, *murow, *aux, *xs;
  __host__ __device__ static size_t doubles(int d, int n, bool full = true)
  {
    int dpad = (d + 32 + 1) & ~1, npad = (n + 1) & ~1;
    return (size_t)npad + (full ? 4 : 2) * (size_t)dpad;
  }
  __device__ void carve(double *base, int d, int n, bool full = true)
  {
    int dpad = (d + 32 + 1) & ~1, npad = (n + 1) & ~1;
    vb = base, rrow = vb + npad, murow = rrow + dpad;
    aux = full ? murow + dpad : murow;
    xs  = full ? aux + dpad : nullptr;
  }
};

// Row `idx` (and possibly everything after it) has been modified: the "already reduced" prefix ends there.
__device__ inline void lower_clean(const View &v, int idx, int lane)
{
  if (lane == 0)
  {
    v.meta[M_CLEAN_SR]  = min(v.meta[M_CLEAN_SR], idx);
    v.meta[M_CLEAN_LLL] = min(v.meta[M_CLEAN_LLL], idx);
  }
}

// FP_NR<double>::exponent, nr_FP_d.inl:44 (out of line: ilogb is a 30-instruction routine, and the callers on the hot
// paths only need it for zeros, subnormals and non-finite values)
static __device__ __noinline__ long fexponent(double x) { return (long)ilogb(x) + 1; }

// ---- exact power-of-two arithmetic without the math library --------------------------------------------------------
// ldexp / frexp / ilogb are 10-20 instruction library routines; on the one-lattice critical paths (Babai's rounding,
// update_bf, the staging of bf_i) they were a large part of every serial step.  For the operand ranges of this code
// they reduce to exponent-field arithmetic: multiplying a double by 2^e (|e| < 1000) is exact whenever the result is a
// normal number and rounds exactly like ldexp when it is not, and the exponent of a normal number is a bit field.
__device__ inline double pow2d(int e)  // 2^e, |e| <= 1022
{
  return __longlong_as_double((long long)(e + 1023) << 52);
}
static __device__ __noinline__ double ldexp_slow(double x, long e) { return ldexp(x, (int)e); }
__device__ inline double scale2(double x, long e)  // == ldexp(x, e)
{
  if (e > -1000 && e < 1000)
    return __dmul_rn(x, pow2d((int)e));
  return ldexp_slow(x, e);
}
// exponent of FP_NR<double>::exponent() for a NORMAL non-zero x (ilogb(x) + 1); callers handle 0 / subnormals
__device__ inline int fexp_normal(double x) { return (int)((__double_as_longlong(x) >> 52) & 0x7ff) - 1022; }
__device__ inline bool is_normal_nz(double x)
{
  const int be = (int)((__double_as_longlong(x) >> 52) & 0x7ff);
  return be != 0 && be != 0x7ff;
}
__device__ inline long fexponent_fast(double x) { return is_normal_nz(x) ? (long)fexp_normal(x) : fexponent(x); }

// FP_NR<double>::get_si_exp_we, nr_FP_d.inl:46-53
__device__ inline long get_si_exp_we(double x, long &expo, long expo_add)
{
  if (x == 0)
    expo = 0;
  else
  {
    long e = fexponent_fast(x) + expo_add - 63;
    expo   = e > 0 ? e : 0;
  }
  return (long)scale2(x, expo_add - expo);
}

// FP_NR<double>::rnd_we, nr_FP_d.inl:226-233 (rint = round-half-even).  The library form lives out of line: inlined
// into every unrolled step of the back-substitution it made those loops ~370 instructions per step, and a lone warp
// streaming 200 KB of straight-line code through the instruction caches per call was what the single-lattice LLL spent
// most of its time on.
static __device__ __noinline__ double rnd_we_slow(double x, long expo_add)
{
  if (fexponent(x) + expo_add >= 53)
    return x;
  return ldexp(rint(ldexp(x, (int)expo_add)), (int)-expo_add);
}
__device__ inline double rnd_we(double x, long expo_add)
{
  if (expo_add == 0 && fabs(x) < 4503599627370496.0)  // |x| < 2^52: both branches below reduce to rint(x)
    return rint(x);
  if (is_normal_nz(x) && expo_add > -1000 && expo_add < 1000)
  {
    if (fexp_normal(x) + expo_add >= 53)
      return x;
    // x * 2^e is exact (or, far below 1, rounds to something rint sends to zero exactly as ldexp's result would be);
    // an integer times 2^-e is exact
    return __dmul_rn(rint(__dmul_rn(x, pow2d((int)expo_add))), pow2d((int)-expo_add));
  }
  return rnd_we_slow(x, expo_add);
}

// One thread's ordered chain  a = a (+|-) x[0] (+|-) x[1] ... over n shared-memory values, optionally recording every
// prefix (out[t + 1] = value after x[t]).  The adds are a dependent chain (8 cycles each); the loads are not — they are
// fetched 8 at a time ahead of the adds, so a step costs the add latency instead of a shared-memory round trip (29
// cycles) it would cost in a plain loop where the compiler cannot move the loads across the prefix stores.
template <bool SUB, bool PREFIX> __device__ inline double serial_chain(double a, const double *x, int n, double *out)
{
  int t = 0;
  double cur[8], nxt[8];
  if (n >= 8)
  {
#pragma unroll
    for (int u = 0; u < 8; u++)
      cur[u] = x[u];
  }
  for (; t + 8 <= n; t += 8)
  {
    const bool more = t + 16 <= n;
    if (more)
    {
#pragma unroll
      for (int u = 0; u < 8; u++)
        nxt[u] = x[t + 8 + u];
    }
#pragma unroll
    for (int u = 0; u < 8; u++)
    {
      a = SUB ? __dsub_rn(a, cur[u]) : __dadd_rn(a, cur[u]);
      if (PREFIX)
        out[t + u + 1] = a;
    }
    if (more)
    {
#pragma unroll
      for (int u = 0; u < 8; u++)
        cur[u] = nxt[u];
    }
  }
  for (; t < n; t++)
  {
    a = SUB ? __dsub_rn(a, x[t]) : __dadd_rn(a, x[t]);
    if (PREFIX)
      out[t + 1] = a;
  }
  return a;
}

// MatGSO::update_bf(i), gso.cpp:24-48 for Z_NR<long> (get_f_exp = frexp((double)x), nr_Z_misc.inl:17-22)
__device__ inline void warp_update_bf(const View &v, int i, int lane)
{
  const int n = max(v.meta[M_NKC], v.irs[i]);
  const int64_t *brow = v.b + (size_t)i * v.ldb;
  if (v.row_expo_en)
  {
    // frexp((double)x) = (f, e) with e = 0 for x = 0, else the exponent field; ldexp(f, e - mx) = (double)x * 2^-mx
    // exactly (|x| < 2^63, mx <= 64: never near the ends of the exponent range)
    int mx = INT_MIN;
    for (int c = lane; c < n; c += 32)
    {
      const double f = (double)brow[c];
      mx = max(mx, f == 0.0 ? 0 : fexp_normal(f));
    }
    for (int o = 16; o; o >>= 1)
      mx = max(mx, __shfl_xor_sync(FULL, mx, o));
    const double sc = pow2d(-mx);
    for (int c = lane; c < n; c += 32)
      v.bf[bf_off(i, c, v.n)] = __dmul_rn((double)brow[c], sc);
    if (lane == 0)
      v.row_expo[i] = mx;
  }
  else
  {
    for (int c = lane; c < n; c += 32)
      v.bf[bf_off(i, c, v.n)] = (double)brow[c];
  }
  __syncwarp();
}

// invalidate_gram_row, gso.cpp:50-54
__device__ inline void warp_invalidate_gram_row(const View &v, int i, int lane)
{
  double *g = v.gf + tri_off(i);
  for (int j = lane; j <= i; j += 32)
    g[j] = CUDART_NAN;
}

// discover_row, gso.cpp:56-82 (float Gram)
__device__ inline void warp_discover_row(const View &v, int lane)
{
  const int i = v.meta[M_NKR];
  __syncwarp();
  if (lane == 0)
  {
    v.meta[M_NKR] = i + 1;
    if (!v.meta[M_LOCKED])
    {
      v.meta[M_NSR] = i + 1;
      v.meta[M_NKC] = max(v.meta[M_NKC], v.irs[i]);
    }
    v.valid[i] = 0;
  }
  warp_invalidate_gram_row(v, i, lane);
  __syncwarp();
}

// Stage bf(i, 0..ncols) in shared memory.  Row i of bf is a 256-byte-strided gather in the panel layout, so it is
// re-derived from the contiguous int64 row instead: update_bf (gso.cpp:24-48) stores frexp/ldexp of (double)b(i,c),
// which is exactly (double)b(i,c) * 2^-row_expo[i] (power-of-two scaling is exact), hence bit-identical.
// Precondition (the reference's !in_row_op_range(i) assert, gso.h:316): row_op_end has run since b[i] last changed.
__device__ inline void stage_bf_row(const View &v, int i, int ncols, double *vb, int first, int step)
{
  if (v.host_basis)
  {
    // no integer mirror on the device: gather the row from the panel layout (one 256-byte-strided load per column)
    const double *bfrow = v.bf + bf_off(i, 0, v.n);
    for (int c = first; c < ncols; c += step)
      vb[c] = bfrow[(size_t)c * 32];
    return;
  }
  const int64_t *brow = v.b + (size_t)i * v.ldb;
  const double sc     = v.row_expo_en ? pow2d(-v.row_expo[i]) : 1.0;  // row_expo in [0, 64]: exact scaling
  for (int c = first; c < ncols; c += step)
    vb[c] = __dmul_rn((double)brow[c], sc);
}
__device__ inline void warp_stage_bf_row(const View &v, int i, int ncols, double *vb, int lane)
{
  stage_bf_row(v, i, ncols, vb, lane, 32);
}

// One lane's ordered chain  acc = acc (+|-) col[k] * vec[k]  for k = k0 .. k1-1 (ascending, two roundings per step):
// the inner loop of both dot_product (numvect.h:385-395, SUB=false) and update_gso_row (gso_interface.cpp:147-151,
// SUB=true).  col points at this lane's row inside a panel (consecutive k are 32 doubles apart, so a warp-wide load
// is one 256-byte line); vec lives in shared memory.  Loads are double-buffered 8 deep: the kernel is bound by HBM
// latency x bytes in flight, so the next group is always requested before the current one is consumed.
template <bool SUB>
__device__ inline double lane_chain(double acc, const double *__restrict__ col, const double *vec, int k0, int k1,
                                    const int cs = 32 /* column stride of the panel: 32 in HBM */)
{
  const int ng = (k1 - k0) >> 3;
  double x[8], y[8];
  if (ng > 0)
  {
#pragma unroll
    for (int u = 0; u < 8; u++)
      x[u] = col[(size_t)(k0 + u) * cs];
  }
  for (int g = 0; g < ng; g += 2)
  {
    const int k = k0 + 8 * g;
    if (g + 1 < ng)
    {
#pragma unroll
      for (int u = 0; u < 8; u++)
        y[u] = col[(size_t)(k + 8 + u) * cs];
    }
#pragma unroll
    for (int u = 0; u < 8; u++)
    {
      const double t = __dmul_rn(x[u], vec[k + u]);
      acc            = SUB ? __dsub_rn(acc, t) : __dadd_rn(acc, t);
    }
    if (g + 2 < ng)
    {
#pragma unroll
      for (int u = 0; u < 8; u++)
        x[u] = col[(size_t)(k + 16 + u) * cs];
    }
    if (g + 1 < ng)
    {
#pragma unroll
      for (int u = 0; u < 8; u++)
      {
        const double t = __dmul_rn(y[u], vec[k + 8 + u]);
        acc            = SUB ? __dsub_rn(acc, t) : __dadd_rn(acc, t);
      }
    }
  }
  for (int k = k0 + 8 * ng; k < k1; k++)
  {
    const double t = __dmul_rn(col[(size_t)k * cs], vec[k]);
    acc            = SUB ? __dsub_rn(acc, t) : __dadd_rn(acc, t);
  }
  return acc;
}

// dot_product(bf_i, bf_j) over [0,ncols), numvect.h:385-395: first term a bare product, then the ordered chain.
__device__ inline double lane_dot(const double *__restrict__ bfcol /* &bf(j,0) */, const double *vb, int ncols)
{
  return lane_chain<false>(__dmul_rn(bfcol[0], vb[0]), bfcol, vb, 1, ncols);
}

// MatGSOInterface::update_gso_row(i, last_j), gso_interface.cpp:131-164, with get_gram (gso.h:314-331) inlined.
// Lane l of panel p owns column j = 32p + l of row i:
//   acc_j = g(i,j);  for k = 0..j-1 (ascending): acc_j -= mu(j,k) * r(i,k)      [two roundings per step]
// r(i,k) for k outside the panel comes from shared memory (rrow), inside the panel by shuffle from the lane that
// has just finished its own chain — the "right-looking" schedule that keeps every chain in reference order.
// Returns false (warp-uniform) if some mu(i,j) is not finite; gso_valid_cols[i] is then left unchanged.
__device__ inline bool warp_update_gso_row(const View &v, int i, int last_j, WarpSmem &s, int lane)
{
  if (i >= v.meta[M_NKR])
    warp_discover_row(v, lane);
  const int j0 = max(0, v.valid[i]);
  if (j0 > last_j)
    return true;
  const int ncols = v.meta[M_NKC], n = v.n;
  double *gfrow = v.gf + tri_off(i), *rrow_g = v.r + tri_off(i);

  int anyn = 0;
  for (int j = j0 + lane; j <= last_j; j += 32)
    anyn |= (gfrow[j] != gfrow[j]);
  anyn = __any_sync(FULL, anyn);
  if (anyn)
    warp_stage_bf_row(v, i, ncols, s.vb, lane);
  for (int k = lane; k < j0; k += 32)
    s.rrow[k] = rrow_g[k];
  __syncwarp();

  bool ok      = true;
  const int jl = min(last_j, i - 1);  // last off-diagonal column to produce
  for (int p = j0 >> 5; 32 * p <= jl; ++p)
  {
    const int j     = 32 * p + lane;
    const bool act  = (j >= j0) && (j <= jl);
    double acc      = 0.0;
    if (act)
    {
      double g = gfrow[j];
      if (g != g)
      {
        g        = lane_dot(v.bf + bf_off(j, 0, n), s.vb, ncols);
        gfrow[j] = g;
      }
      acc = g;
    }
    else if (j < j0)
      acc = s.rrow[j];  // already-valid r(i,j): only broadcast in the triangle below
    const double *mup = v.mu + mu_panel_base(p) + lane;
    double rd         = 1.0;  // r(j,j), read from the mu(j,j) slot of the diagonal tile (see gso_layout.cuh)
    // rectangular part: columns k < 32p, all r(i,k) already in shared memory
    if (act)
      acc = lane_chain<true>(acc, mup, s.rrow, 0, 32 * p);
    // triangular part: column 32p+t is final in lane t once steps 0..t-1 are applied.  4 chunks of 8 columns,
    // the next chunk's tile entries are requested while the current chunk's shuffle chain runs.
    {
      const double *tile = mup + (size_t)(32 * p) * 32;
      double m[8], mn[8];
#pragma unroll
      for (int u = 0; u < 8; u++)
        m[u] = (act && lane >= u) ? tile[(size_t)u * 32] : 0.0;  // lane == u picks up its diagonal r(j,j) mirror
#pragma unroll
      for (int q = 0; q < 4; q++)
      {
        if (q < 3)
        {
#pragma unroll
          for (int u = 0; u < 8; u++)
            mn[u] = (act && lane >= 8 * (q + 1) + u) ? tile[(size_t)(8 * (q + 1) + u) * 32] : 0.0;
        }
#pragma unroll
        for (int u = 0; u < 8; u++)
        {
          const int t = 8 * q + u;
          if (lane == t)
            rd = m[u];
          if (t < 31)
          {
            const double rk = __shfl_sync(FULL, acc, t);
            if (act && lane > t)
              acc = __dsub_rn(acc, __dmul_rn(m[u], rk));
          }
        }
#pragma unroll
        for (int u = 0; u < 8; u++)
          m[u] = mn[u];
      }
    }
    if (act)
    {
      rrow_g[j]       = acc;
      s.rrow[j]       = acc;
      const double mm = __ddiv_rn(acc, rd);
      v.mu[mu_off(i, j)] = mm;
      s.murow[j]      = mm;
      if (!isfinite(mm))
        ok = false;
    }
    __syncwarp();
  }
  ok = __all_sync(FULL, ok);
  if (!ok)
    return false;

  if (last_j >= i)
  {
    // diagonal r(i,i) = g(i,i) - sum_{k<i} mu(i,k) r(i,k): products in parallel, one ordered subtraction chain
    for (int k = lane; k < min(j0, i); k += 32)
      s.murow[k] = v.mu[mu_off(i, k)];
    __syncwarp();
    for (int k = lane; k < i; k += 32)
      s.aux[k] = __dmul_rn(s.murow[k], s.rrow[k]);
    __syncwarp();
    if (lane == 0)
    {
      double g = gfrow[i];
      if (g != g)
      {
        g = __dmul_rn(s.vb[0], s.vb[0]);
        for (int c = 1; c < ncols; c++)
          g = __dadd_rn(g, __dmul_rn(s.vb[c], s.vb[c]));
        gfrow[i] = g;
      }
      const double acc   = serial_chain<true, false>(g, s.aux, i, nullptr);
      rrow_g[i]          = acc;
      v.mu[mu_off(i, i)] = acc;  // diagonal mirror
    }
    __syncwarp();
  }
  if (lane == 0)
    v.valid[i] = last_j + 1;
  __syncwarp();
  return true;
}

// row_op_end(first,last), gso_interface.cpp:32-53
__device__ inline void warp_row_op_end(const View &v, int first, int last, int lane)
{
  const int nkr = v.meta[M_NKR];
  for (int i = first; i < last; i++)
  {
    if (!v.host_basis)  // host-basis handles: bf(i,.) and row_expo[i] were uploaded (b200gso_upload_row_fp)
      warp_update_bf(v, i, lane);
    warp_invalidate_gram_row(v, i, lane);
    for (int j = i + 1 + lane; j < nkr; j += 32)
      v.gf[tri_off(j) + i] = CUDART_NAN;
    if (lane == 0)
      v.valid[i] = 0;
  }
  for (int i = last + lane; i < nkr; i += 32)
    v.valid[i] = min(v.valid[i], first);
  lower_clean(v, first, lane);
  __syncwarp();
}

// row_addmul_we(i, j, x, expo_add), gso.cpp:236-262 -> row_add/row_sub/row_addmul_si/row_addmul_si_2exp
// (gso.cpp:84-195, numvect.h:268-341) on b only (u, u_inv_t empty in the BKZ regime).  int64 wraps like Z_NR<long>.
__device__ inline void warp_row_addmul_we(const View &v, int i, int j, double x, long expo_add, int lane)
{
  long expo;
  const long lx = get_si_exp_we(x, expo, expo_add);
  if (expo == 0 && lx == 0)
    return;
  lower_clean(v, i, lane);
  const int nc           = v.meta[M_NKC];
  unsigned long long *bi = (unsigned long long *)(v.b + (size_t)i * v.ldb);
  const unsigned long long *bj = (const unsigned long long *)(v.b + (size_t)j * v.ldb);
  const unsigned long long ux  = (unsigned long long)lx;
  if (expo == 0)
    for (int c = lane; c < nc; c += 32)
      bi[c] += bj[c] * ux;
  else
    for (int c = lane; c < nc; c += 32)
    {
      unsigned long long t = bj[c] * ux;
      bi[c] += (expo >= 64 ? 0ull : (t << expo));
    }
  __syncwarp();
}

// row_swap(i,j), gso.cpp:264-287: integer rows only
__device__ inline void warp_row_swap(const View &v, int i, int j, int lane)
{
  int64_t *a = v.b + (size_t)i * v.ldb, *b = v.b + (size_t)j * v.ldb;
  lower_clean(v, min(i, j), lane);
  for (int c = lane; c < v.n; c += 32)
  {
    int64_t t = a[c];
    a[c]      = b[c];
    b[c]      = t;
  }
  __syncwarp();
}

__device__ inline int size_nz_warp(const int64_t *row, int n, int lane)
{
  int last = 0;
  for (int c = lane; c < n; c += 32)
    if (row[c] != 0)
      last = c + 1;
  for (int o = 16; o; o >>= 1)
    last = max(last, __shfl_xor_sync(FULL, last, o));
  return last;
}

// Rotate the sequence e(lo), ..., e(hi) by one position (right: e(hi) -> lo, the rest shift up; left: e(lo) -> hi).
// `at(i)` returns a reference to element i.  Elements are moved in chunks of 8 held in registers so that 8 loads are in
// flight at a time: written as a one-by-one shift, every load would wait for the previous store (same array) and a
// rotation over D rows would cost D dependent memory round trips.
template <class T, class At> __device__ inline void rotate_seq(At at, int lo, int hi, bool right)
{
  if (hi <= lo)
    return;
  if (right)
  {
    const T t = at(hi);
    int i     = hi;
    for (; i - 8 >= lo; i -= 8)
    {
      T v[8];
#pragma unroll
      for (int u = 0; u < 8; u++)
        v[u] = at(i - 1 - u);
#pragma unroll
      for (int u = 0; u < 8; u++)
        at(i - u) = v[u];
    }
    for (; i > lo; --i)
      at(i) = at(i - 1);
    at(lo) = t;
  }
  else
  {
    const T t = at(lo);
    int i     = lo;
    for (; i + 8 <= hi; i += 8)
    {
      T v[8];
#pragma unroll
      for (int u = 0; u < 8; u++)
        v[u] = at(i + 1 + u);
#pragma unroll
      for (int u = 0; u < 8; u++)
        at(i + u) = v[u];
    }
    for (; i < hi; ++i)
      at(i) = at(i + 1);
    at(hi) = t;
  }
}

// move_row(old_r, new_r), gso.cpp:289-366 (float Gram, no transforms).  Rotations of mu, r, b, bf, row_expo,
// gso_valid_cols are done column-by-column (each lane carries one column through the rotated rows, no scratch);
// only the entries that can still be valid after the call (columns < min(old,new), SURVEY Appendix A) are moved
// for mu and r.  The symmetric row+column rotation of gf (matrix.cpp:65-93) goes through v.scratch.
__device__ inline void warp_move_row(const View &v, int old_r, int new_r, int lane)
{
  if (old_r == new_r)
    return;
  const int nkr   = v.meta[M_NKR];
  const bool right = new_r < old_r;  // rows [lo..hi]: right: row hi -> lo; left: row lo -> hi
  const int lo = right ? new_r : old_r, hi = right ? old_r : new_r;
  for (int i = lo + lane; i < nkr; i += 32)
    v.valid[i] = min(v.valid[i], lo);
  lower_clean(v, lo, lane);
  __syncwarp();
  // mu and r (columns k < lo), b and bf rows (all n columns): one column per lane, rows rotated in register chunks
  for (int k = lane; k < lo; k += 32)
  {
    rotate_seq<double>([&](int i) -> double & { return v.mu[mu_off(i, k)]; }, lo, hi, right);
    rotate_seq<double>([&](int i) -> double & { return v.r[tri_off(i) + k]; }, lo, hi, right);
  }
  for (int c = lane; c < v.n; c += 32)
  {
    rotate_seq<int64_t>([&](int i) -> int64_t & { return v.b[(size_t)i * v.ldb + c]; }, lo, hi, right);
    rotate_seq<double>([&](int i) -> double & { return v.bf[bf_off(i, c, v.n)]; }, lo, hi, right);
  }
  // gf: new(i,j) = old_sym(s(i), s(j)) on the known rows; rotate_gram_left only when old_r < nkr-1 and up to
  // min(new_r, nkr-1) (gso.cpp:338-341).  Rows below the rotated range only permute their columns [lo, ghi] (done in
  // place, one row per lane); the rotated rows themselves are rebuilt from a scratch copy of just those rows.
  {
    const int ghi = right ? hi : min(hi, nkr - 1);
    if (right || lo < nkr - 1)
    {
      for (int i = ghi + 1 + lane; i < nkr; i += 32)
      {
        double *row = v.gf + tri_off(i);
        rotate_seq<double>([&](int j) -> double & { return row[j]; }, lo, ghi, right);
      }
      const size_t beg = tri_off(lo), end = tri_off(ghi + 1);
      for (size_t t = beg + lane; t < end; t += 32)
        v.scratch[t - beg] = v.gf[t];
      __syncwarp();
      for (int i = lo; i <= ghi; i++)
      {
        const int si = right ? (i == lo ? ghi : i - 1) : (i == ghi ? lo : i + 1);
        for (int j = lane; j <= i; j += 32)
        {
          int sj = j;
          if (j >= lo)
            sj = right ? (j == lo ? ghi : j - 1) : (j == ghi ? lo : j + 1);
          const int a = max(si, sj), b = min(si, sj);
          v.gf[tri_off(i) + j] = v.scratch[tri_off(a) + b - beg];
        }
      }
    }
  }
  __syncwarp();
  // row_expo, gso_valid_cols (and init_row_size when the row leaves the known set): three lanes, one array each
  if (lane == 0)
    rotate_seq<int>([&](int i) -> int & { return v.valid[i]; }, lo, hi, right);
  else if (lane == 1)
    rotate_seq<int>([&](int i) -> int & { return v.row_expo[i]; }, lo, hi, right);
  else if (lane == 2 && !right && new_r >= nkr)
    rotate_seq<int>([&](int i) -> int & { return v.irs[i]; }, lo, hi, false);
  __syncwarp();
  if (!right && new_r >= nkr && old_r < nkr)
  {
    const int nz = v.host_basis ? v.n : size_nz_warp(v.b + (size_t)new_r * v.ldb, v.n, lane);
    if (lane == 0)
    {
      v.meta[M_NKR] = nkr - 1;
      v.meta[M_NSR] = nkr - 1;
      v.irs[new_r]  = max(nz, 1);
    }
  }
  __syncwarp();
}

// set_r(i,j,f), gso_interface.h:739-746
__device__ inline void warp_set_r(const View &v, int i, int j, double f, int lane)
{
  if (lane == 0)
  {
    v.r[tri_off(i) + j] = f;
    if (i == j)
      v.mu[mu_off(i, i)] = f;  // diagonal mirror
    if (v.valid[i] == j)
      v.valid[i] = j + 1;
  }
  __syncwarp();
}

}  // namespace b200
