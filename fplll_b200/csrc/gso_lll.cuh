// gso_lll.cuh — device-resident LLL inner loop (one warp per lattice).
//
// LLLReduction<Z_NR<long>, FP_NR<double>>::lll / babai (fplll/lll.cpp:44-224) run entirely on the device against
// the HBM-resident GSO state: no host round trip per update_gso_row / row_addmul_we (SURVEY §7 "hard parts":
// the CPU spends ~1 us per such call, less than one kernel launch).  Control flow is warp-uniform; every
// floating-point chain keeps the reference's operation order so the basis trajectory is the reference's.
#pragma once
#include "gso_cta.cuh"
#include "gso_warp.cuh"

namespace b200 {

enum { RED_SUCCESS = 0, RED_GSO_FAILURE = 2, RED_BABAI_FAILURE = 3, RED_LLL_FAILURE = 4 };  // defs.h:153-169
constexpr long SIZE_RED_FAILURE_THRESH = 5;                                                    // defs.h:146

struct LLLStats
{
  long n_swaps, final_kappa, zeros, babai_iters;
  // device-clock breakdown (SM cycles of the owning warp): update_gso_row, rest of babai (scan, back-substitution,
  // integer row operations, row_op_end), Lovasz test, move_row
  long long cyc_update, cyc_babai, cyc_lovasz, cyc_move;
  long long cyc_gather, cyc_backsub, cyc_igemv, cyc_ropend;  // inside cyc_babai
};

#ifdef B200_LLL_PROFILE
#define LLL_PT(var) const long long var = clock64()
#define LLL_PACC(field, t0) \
  do                        \
  {                         \
    if (pst)                \
      pst->field += clock64() - (t0); \
  } while (0)
#else
#define LLL_PT(var)
#define LLL_PACC(field, t0)
#endif

// LLLReduction::babai(kappa, size_reduction_end, size_reduction_start), lll.cpp:166-224.
// MAXQ*32 >= d.  Returns RED_SUCCESS or the failing status (warp-uniform).  XF: the handle tracks U, whose row kappa
// takes the same integer row operations as b's.
template <int MAXQ, bool COOP, bool XF>
__device__ inline int warp_babai(const LLLView<XF> &v, WarpSmem &s, int kappa, int sr_end, int sr_start, double eta, int lane,
                                 long &iters, LLLStats *pst = nullptr, CoopShared *C = nullptr)
{
  long max_expo = LONG_MAX;
  for (int iter = 0;; iter++)
  {
    LLL_PT(tu_);
    const bool upd_ok = lll_update_gso_row<COOP>(v, kappa, sr_end - 1, s, lane, C);
    LLL_PACC(cyc_update, tu_);
    LLL_PT(tg_);
    if (!upd_ok)
      return RED_GSO_FAILURE;
    // gather row kappa of mu (stride-32 in the panel layout) + exponent differences
    const int ek = v.row_expo[kappa];
    int loop_needed = 0;
    long new_max    = LONG_MIN;
    double bm[MAXQ];
#pragma unroll
    for (int q = 0; q < MAXQ; q++)
    {
      const int k = 32 * q + lane;
      bm[q]       = 0.0;
      if (k < sr_end)
      {
        bm[q]          = lll_mu_load<COOP>(v, C, kappa, k);
        const long de  = v.row_expo_en ? (long)(ek - v.row_expo[k]) : 0;
        s.xs[k]        = 0.0;
        if (k >= sr_start)
          loop_needed |= (fabs(scale2(bm[q], de)) > eta);  // get_mu, gso_interface.h:694-701
        new_max = max(new_max, de + fexponent_fast(bm[q]));         // get_max_mu_exp, gso_interface.cpp:88-98
      }
    }
    if (!__any_sync(FULL, loop_needed))
      break;
    if (iter >= 2)
    {
      for (int o = 16; o; o >>= 1)
        new_max = max(new_max, __shfl_xor_sync(FULL, new_max, o));
      if (new_max > max_expo - SIZE_RED_FAILURE_THRESH)
        return RED_BABAI_FAILURE;
      max_expo = new_max;
    }
    iters++;
    __syncwarp();
    unsigned *xmask = (unsigned *)(s.xs + ((v.d + 1) & ~1));  // per-panel bit masks of the non-zero X_j (padding of xs)
    if (lane < MAXQ)
      xmask[lane] = 0;
    __syncwarp();
    LLL_PACC(cyc_gather, tg_);
    LLL_PT(tb_);
    // back-substitution, j descending (lll.cpp:202-214): X_j = rnd_we(babai_mu[j]); babai_mu[k] -= X_j*mu(j,k), k<j
    const bool coop_bs = COOP && sr_end > 32;  // more than one panel: wavefront over the CTA's warps (gso_cta.cuh)
    if (coop_bs)
    {
#pragma unroll
      for (int q = 0; q < MAXQ; q++)
      {
        const int k = 32 * q + lane;
        if (k < sr_end)
          C->bm[k] = bm[q];
      }
      coop_post(C, COOP_BACKSUB, kappa, sr_end, sr_start, lane);
      cta_backsub(*C, kappa, sr_end, sr_start, 0, lane);
    }
    for (int p = coop_bs ? -1 : ((sr_end - 1) >> 5); p >= (sr_start >> 5); --p)
    {
      // in-panel triangle: lane l owns column k = 32p+l
      double val = 0.0;
#pragma unroll
      for (int q = 0; q < MAXQ; q++)
        if (q == p)
          val = bm[q];
      const int kcol        = 32 * p + lane;
      const double *tilecol = v.mu + mu_panel_base(p) + (size_t)kcol * 32;  // mu(32p+t, kcol) at [t]
      unsigned nzmask       = 0;  // rows of this panel with X != 0 (warp-uniform)
      // this lane's column of the diagonal tile, requested up front: inside the serial t-loop every load would be a
      // ~0.3 us round trip on the critical path (the device profile showed Babai dominated by exactly that)
      double tc[32];
#pragma unroll
      for (int t = 0; t < 32; t++)
        tc[t] = (t > lane && 32 * p + t < sr_end) ? tilecol[t] : 0.0;
#pragma unroll
      for (int t = 31; t >= 0; --t)
      {
        const int j = 32 * p + t;
        if (j >= sr_end || j < sr_start)
          continue;
        const double bj = __shfl_sync(FULL, val, t);
        const long de   = v.row_expo_en ? (long)(ek - v.row_expo[j]) : 0;
        const double X  = rnd_we(bj, de);
        if (X == 0.0)
          continue;
        nzmask |= 1u << t;
        if (lane == 0)
          s.xs[j] = X;
        if (lane < t && kcol >= sr_start)
          val = __dsub_rn(val, __dmul_rn(X, tc[t]));
      }
      if (lane == 0)
        xmask[p] = nzmask;
      __syncwarp();
      // rectangular part: columns k < 32p (lanes over k), rows of this panel descending
#pragma unroll
      for (int q = 0; q < MAXQ; q++)
      {
        if (q < p && nzmask)
        {
          const int k = 32 * q + lane;
          if (k >= sr_start)
          {
            const double *col = v.mu + mu_panel_base(p) + (size_t)k * 32;
            double a          = bm[q];
            double cv[32];  // mu(32p + t, k), t = 0..31: 32 independent loads in flight
#pragma unroll
            for (int t = 0; t < 32; t++)
              cv[t] = ((nzmask >> t) & 1u) ? col[t] : 0.0;
#pragma unroll
            for (int t = 31; t >= 0; --t)  // rows with X != 0 only, still in descending order
              if ((nzmask >> t) & 1u)
                a = __dsub_rn(a, __dmul_rn(s.xs[32 * p + t], cv[t]));
            bm[q] = a;
          }
        }
      }
    }
    __syncwarp();
    LLL_PACC(cyc_backsub, tb_);
    LLL_PT(ti_);
    // integer row operations b_kappa += (-X_j) * 2^expo_j * b_j, fused over j (row_addmul_we, gso.cpp:236-262).
    // Integer additions commute exactly (mod 2^64), so one pass over the columns applies all j.  Only the rows with
    // X_j != 0 are visited (typically a handful): compact them first — lx -> aux[t], shift -> murow[t], row -> xs'[t].
    int nnz = 0;
    {
      const int p_hi = (sr_end - 1) >> 5, p_lo = sr_start >> 5;
      for (int p = p_hi; p >= p_lo; --p)
      {
        const unsigned m = xmask[p];
        if ((m >> lane) & 1u)
        {
          const int j    = 32 * p + lane;
          const int slot = nnz + (lane == 31 ? 0 : __popc(m >> (lane + 1)));  // descending j within the panel
          const double X = s.xs[j];
          long expo      = 0;
          const long lx  = get_si_exp_we(-X, expo, v.row_expo_en ? (long)(ek - v.row_expo[j]) : 0);
          s.aux[slot]    = __longlong_as_double((long long)lx);
          s.murow[slot]  = __longlong_as_double(((long long)expo << 32) | (unsigned)j);
        }
        nnz += __popc(m);
      }
    }
    __syncwarp();
    if (COOP && nnz)
    {
      coop_post(C, COOP_IGEMV, kappa, nnz, 0, lane);
      cta_igemv<XF>(*C, kappa, nnz, 0, lane);
    }
    else if (nnz)
    {
      // lane l owns columns l, l+32, ... of a group of up to 8*32 columns: 4 source rows x 8 column chunks = 32 loads in
      // flight per round (the source rows are contiguous, every load is a 256-byte coalesced line).  XF: b's nc columns
      // are followed by U's d columns (column c >= nc is U's column c - nc: U rows are updated over all d columns).
      const int nc           = v.meta[M_NKC];
      const int ncx          = XF ? nc + v.d : nc;
      unsigned long long *bk = (unsigned long long *)(v.b + (size_t)kappa * v.ldb);
      unsigned long long *uk = nullptr;
      if constexpr (XF)
        uk = (unsigned long long *)u_row(v, kappa);
      for (int cg0 = 0; cg0 < ncx; cg0 += 256)
      {
        unsigned long long acc[8];
#pragma unroll
        for (int w = 0; w < 8; w++)
        {
          const int c = cg0 + 32 * w + lane;
          acc[w]      = (c < nc) ? bk[c] : (XF && c < ncx) ? uk[c - nc] : 0ull;
        }
        for (int t0 = 0; t0 < nnz; t0 += 4)
        {
          unsigned long long bv[4][8], lxv[4];
          int ev[4];
#pragma unroll
          for (int u = 0; u < 4; u++)
          {
            const int t = t0 + u;
            lxv[u] = 0ull, ev[u] = 0;
            const unsigned long long *src = bk, *usrc = uk;
            if (t < nnz)
            {
              lxv[u]             = (unsigned long long)__double_as_longlong(s.aux[t]);
              const long long pk = __double_as_longlong(s.murow[t]);
              ev[u]              = (int)(pk >> 32);
              src = (const unsigned long long *)(v.b + (size_t)(int)(pk & 0xffffffffll) * v.ldb);
              if constexpr (XF)
                usrc = (const unsigned long long *)u_row(v, (int)(pk & 0xffffffffll));
            }
#pragma unroll
            for (int w = 0; w < 8; w++)
            {
              const int c = cg0 + 32 * w + lane;
              bv[u][w]    = (t < nnz && c < nc) ? src[c] : (XF && t < nnz && c < ncx) ? usrc[c - nc] : 0ull;
            }
          }
#pragma unroll
          for (int u = 0; u < 4; u++)
#pragma unroll
            for (int w = 0; w < 8; w++)
            {
              const unsigned long long tt = bv[u][w] * lxv[u];
              acc[w] += (ev[u] >= 64 ? 0ull : (tt << ev[u]));
            }
        }
#pragma unroll
        for (int w = 0; w < 8; w++)
        {
          const int c = cg0 + 32 * w + lane;
          if (c < nc)
            bk[c] = acc[w];
          else if (XF && c < ncx)
            uk[c - nc] = acc[w];
        }
      }
    }
    __syncwarp();
    LLL_PACC(cyc_igemv, ti_);
    LLL_PT(tr_);
    warp_row_op_end(v, kappa, kappa + 1, lane);
    LLL_PACC(cyc_ropend, tr_);
  }
  return RED_SUCCESS;
}

// Matrix::get_max_exp over b with Z_NR<long>::exponent (nr_Z_l.inl:40-48)
__device__ inline long warp_max_exp_of_b(const ViewCore &v, int lane)
{
  long mx = 0;
  for (int i = 0; i < v.d; i++)
    for (int c = lane; c < v.n; c += 32)
    {
      const long x = v.b[(size_t)i * v.ldb + c];
      int e;
      const double f = frexp((double)x, &e);
      long ex        = e;
      if (x > ((1L << 52) - 1) && fabs(f) == 0.5)
      {
        unsigned long long y = (unsigned long long)x;
        for (ex = 0; y; ex++, y >>= 1)
          ;
      }
      mx = max(mx, ex);
    }
  for (int o = 16; o; o >>= 1)
    mx = max(mx, __shfl_xor_sync(FULL, mx, o));
  return mx;
}

__device__ inline bool warp_b_row_is_zero(const ViewCore &v, int i, int lane)
{
  int nz = 0;
  for (int c = lane; c < v.n; c += 32)
    nz |= (v.b[(size_t)i * v.ldb + c] != 0);
  return !__any_sync(FULL, nz);
}

// get_gram(kappa,kappa) (gso.h:314-331) for the Lovasz test; computes the dot product if the entry is invalid.
__device__ inline double warp_get_gram_diag(const ViewCore &v, WarpSmem &s, int i, int lane)
{
  double *g  = v.gf + tri_off(i) + i;
  double val = *g;
  if (val != val)
  {
    const int ncols = v.meta[M_NKC];
    // stage bf_i squared (one correctly rounded product per element, in parallel): the ordered chain only adds
    const int64_t *brow = v.b + (size_t)i * v.ldb;
    const double sc     = v.row_expo_en ? pow2d(-v.row_expo[i]) : 1.0;
    for (int c = lane; c < ncols; c += 32)
    {
      const double f = __dmul_rn((double)brow[c], sc);
      s.vb[c]        = __dmul_rn(f, f);
    }
    __syncwarp();
    if (lane == 0)
      *g = serial_chain<false, false>(s.vb[0], s.vb + 1, ncols - 1, nullptr);
    __syncwarp();
    val = *g;
  }
  return val;
}

// LLLReduction::size_reduction(kappa_min, kappa_end, size_reduction_start), lll.h:106-122
template <int MAXQ, bool COOP, bool XF>
__device__ inline int warp_size_reduction(const LLLView<XF> &v, WarpSmem &s, int kappa_min, int kappa_end, int sr_start,
                                          double eta, int lane, long &iters, CoopShared *C = nullptr)
{
  // Rows below the clean prefix are size-reduced with a valid GSO and untouched since: on them the reference's loop
  // body (babai finds nothing to reduce, update_gso_row finds the row valid) changes no state, so start after them.
  const bool eta_same = (v.meta[M_ETA_LO] == __double2loint(eta)) && (v.meta[M_ETA_HI] == __double2hiint(eta));
  const int clean     = (eta_same && sr_start == 0) ? v.meta[M_CLEAN_SR] : 0;
  const int k_first   = (kappa_min <= clean) ? max(kappa_min, min(clean, kappa_end)) : kappa_min;
  __syncwarp();
  for (int k = k_first; k < kappa_end; k++)
  {
    if (k > 0)
    {
      const int st = warp_babai<MAXQ, COOP, XF>(v, s, k, k, sr_start, eta, lane, iters, nullptr, C);
      if (st != RED_SUCCESS)
        return st;
    }
    if (!lll_update_gso_row<COOP>(v, k, k, s, lane, C))
      return RED_GSO_FAILURE;  // the reference returns false here without touching status (lll.h:118-119)
  }
  if (sr_start == 0 && kappa_min <= clean && lane == 0)
  {
    // rows [0, k_first) were clean, rows [k_first, kappa_end) have just been size-reduced (row operations inside
    // this loop only lowered the marker to rows >= k_first, which were then redone)
    if (!eta_same)
    {
      v.meta[M_ETA_LO]    = __double2loint(eta);
      v.meta[M_ETA_HI]    = __double2hiint(eta);
      v.meta[M_CLEAN_LLL] = 0;
      v.meta[M_CLEAN_SR]  = kappa_end;
    }
    else
      v.meta[M_CLEAN_SR] = max(v.meta[M_CLEAN_SR], kappa_end);
  }
  __syncwarp();
  return RED_SUCCESS;
}

// LLLReduction::lll(kappa_min, kappa_start, kappa_end, size_reduction_start), lll.cpp:44-164; LLL_DEFAULT flags
// (no siegel, no early reduction, not verbose).  lov = shared array of d+1 doubles.  XF: U follows every row operation
// (only integer rows change; no decision reads U).
template <int MAXQ, bool COOP, bool XF>
__device__ inline int warp_lll(const LLLView<XF> &v, WarpSmem &s, double *lov, double delta, double eta, int kappa_min,
                               int kappa_start, int kappa_end, int sr_start, int lane, LLLStats &st,
                               CoopShared *C = nullptr)
{
  const int d = kappa_end - kappa_min;
  int kappa = kappa_start + 1, zeros = 0;
  st.n_swaps = st.final_kappa = st.zeros = st.babai_iters = 0;
  st.cyc_update = st.cyc_babai = st.cyc_lovasz = st.cyc_move = 0;
  st.cyc_gather = st.cyc_backsub = st.cyc_igemv = st.cyc_ropend = 0;
  const double swap_threshold = delta;
  // Clean prefix: rows [0, c) are (delta, eta)-LLL-reduced with a valid GSO and untouched since the call that made
  // them so.  On such rows every iteration of the reference's loop is a no-op on the state (babai finds |mu| <= eta,
  // Lovasz holds, set_r re-writes the value the same chain produced before), so the loop may start at row c.
  const bool par_same = v.meta[M_ETA_LO] == __double2loint(eta) && v.meta[M_ETA_HI] == __double2hiint(eta) &&
                        v.meta[M_DELTA_LO] == __double2loint(delta) && v.meta[M_DELTA_HI] == __double2hiint(delta);
  const bool track    = (kappa_min == 0 && kappa_start == 0 && sr_start == 0);
  if (track && par_same)
    kappa = max(kappa, min(v.meta[M_CLEAN_LLL], kappa_end));
  __syncwarp();
  for (; zeros < d && warp_b_row_is_zero(v, 0, lane); zeros++)
  {
    lll_move_row<COOP, XF>(v, kappa_min, kappa_end - 1 - zeros, lane, C);
    lll_mu_reload<COOP>(C, kappa_min, kappa_end - 1 - zeros, lane);
  }
  if (zeros < d)
  {
    if (kappa_start > 0)
    {
      const int bst =
          warp_babai<MAXQ, COOP, XF>(v, s, kappa_start, kappa_start, sr_start, eta, lane, st.babai_iters, nullptr, C);
      if (bst != RED_SUCCESS)
      {
        st.final_kappa = kappa_start, st.zeros = zeros;
        return bst;
      }
    }
    if (!lll_update_gso_row<COOP>(v, kappa_start, kappa_start, s, lane, C))
    {
      st.final_kappa = kappa_start, st.zeros = zeros;
      return RED_GSO_FAILURE;
    }
  }
  // max_iter = d - 2d(d+1)((max_exp_of_b + 3)/log delta)  (lll.cpp:78-82) needs a scan of the whole basis; it is only a
  // safety cap, so start from its smallest possible value (max_exp_of_b = 0) and pay for the exact one only if the
  // loop ever gets that far — same termination behaviour, no d*n scan per call.
  long long max_iter = (long long)((double)d - (double)(2 * d * (d + 1)) * (3.0 / log(delta)));
  bool max_iter_exact = false;
  long long iter;
  for (iter = 0; kappa < kappa_end - zeros; iter++)
  {
    if (iter >= max_iter)
    {
      if (max_iter_exact)
        break;
      const long maxe = warp_max_exp_of_b(v, lane);
      max_iter        = (long long)((double)d - (double)(2 * d * (d + 1)) * ((double)(maxe + 3) / log(delta)));
      max_iter_exact  = true;
      if (iter >= max_iter)
        break;
    }
#ifdef B200_LLL_PROFILE
    const long long tb_ = clock64();
    const long long cu_ = st.cyc_update;
#endif
    const int bst =
        warp_babai<MAXQ, COOP, XF>(v, s, kappa, kappa, sr_start, eta, lane, st.babai_iters, &st, C);
#ifdef B200_LLL_PROFILE
    st.cyc_babai += (clock64() - tb_) - (st.cyc_update - cu_);
    const long long tl_ = clock64();
#endif
    if (bst != RED_SUCCESS)
    {
      st.final_kappa = kappa, st.zeros = zeros;
      return bst;
    }
    // Lovasz test (lll.cpp:110-122): prefix chain lov[i] = lov[i-1] - mu(kappa,i-1) * r(kappa,i-1)
    const double g = warp_get_gram_diag(v, s, kappa, lane);
    for (int k = lane; k < kappa; k += 32)
      s.aux[k] = __dmul_rn(lll_mu_load<COOP>(v, C, kappa, k), v.r[tri_off(kappa) + k]);
    __syncwarp();
    int new_kappa = kappa, action = 0;  // 0: accept, 1: move_row(old_k,new_kappa), 2: zero vector
    if (lane == 0)
    {
      lov[0] = g;
      (void)serial_chain<true, true>(g, s.aux, kappa, lov);
      // r(k-1,k-1): the diagonal mirror in mu's unused slot (gso_layout.cuh) — shared memory when that panel is cached
      double thr = __dmul_rn(lll_mu_load<COOP>(v, C, kappa - 1, kappa - 1), swap_threshold);
      if (v.row_expo_en)
        thr = scale2(thr, 2 * (v.row_expo[kappa - 1] - v.row_expo[kappa]));
      if (thr > lov[kappa - 1])
      {
        int kk = kappa;
        for (kk--; kk > kappa_min; kk--)
        {
          double t2 = __dmul_rn(lll_mu_load<COOP>(v, C, kk - 1, kk - 1), swap_threshold);
          if (v.row_expo_en)
            t2 = scale2(t2, 2 * (v.row_expo[kk - 1] - v.row_expo[kappa]));
          if (t2 < lov[kk - 1])
            break;
        }
        new_kappa = kk;
        action    = (lov[kk] > 0) ? 1 : 2;
      }
    }
    action    = __shfl_sync(FULL, action, 0);
    new_kappa = __shfl_sync(FULL, new_kappa, 0);
#ifdef B200_LLL_PROFILE
    st.cyc_lovasz += clock64() - tl_;
    const long long tm_ = clock64();
#endif
    if (action)
    {
      st.n_swaps++;
      const int old_k = kappa;
      if (action == 1)
      {
        lll_move_row<COOP, XF>(v, old_k, new_kappa, lane, C);
        lll_mu_reload<COOP>(C, new_kappa, old_k, lane);
        kappa = new_kappa;
      }
      else
      {
        zeros++;
        lll_move_row<COOP, XF>(v, old_k, kappa_end - zeros, lane, C);
        lll_mu_reload<COOP>(C, old_k, kappa_end - zeros, lane);
        kappa = old_k;
        continue;
      }
    }
    __syncwarp();
    warp_set_r(v, kappa, kappa, lov[kappa], lane);
    lll_mu_refresh_diag<COOP>(C, kappa, lane);
    kappa++;
#ifdef B200_LLL_PROFILE
    st.cyc_move += clock64() - tm_;
#endif
  }
  st.zeros = zeros;
  if (kappa < kappa_end - zeros)
    return RED_LLL_FAILURE;
  if (track && lane == 0)
  {
    const int upto = kappa_end - zeros;
    if (!par_same)
    {
      v.meta[M_ETA_LO] = __double2loint(eta), v.meta[M_ETA_HI] = __double2hiint(eta);
      v.meta[M_DELTA_LO] = __double2loint(delta), v.meta[M_DELTA_HI] = __double2hiint(delta);
      v.meta[M_CLEAN_LLL] = upto;
      v.meta[M_CLEAN_SR]  = upto;
    }
    else
    {
      v.meta[M_CLEAN_LLL] = max(v.meta[M_CLEAN_LLL], upto);
      v.meta[M_CLEAN_SR]  = max(v.meta[M_CLEAN_SR], upto);
    }
  }
  __syncwarp();
  return RED_SUCCESS;
}

}  // namespace b200
