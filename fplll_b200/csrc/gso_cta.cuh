// gso_cta.cuh — CTA-cooperative pieces of the device LLL for the single-lattice (BKZ) regime.
//
// With one warp per lattice (gso_lll.cuh) a Babai iteration on a dim-200 basis is latency-bound: every load is an exposed
// L2 round trip and every dependent instruction an exposed pipeline latency.  A batch hides that behind
// other lattices; BKZ on ONE lattice cannot.  Here one CTA of CTA_WARPS warps serves one lattice: warp 0 (the master)
// runs the LLL control flow of gso_lll.cuh unchanged, and the three O(kappa * d) pieces of an iteration are executed by
// all warps as SPMD "cooperative operations", one 32-column panel per warp:
//
//   UPDATE   update_gso_row(i, last_j): Gram entries of different panels in parallel, then the forward substitution
//            as a WAVEFRONT over panels — panel p applies the tiles (p, q) in ascending q as soon as panel q's
//            r(i, .) are final, so the critical path is P (triangle + one tile) instead of P^2/2 tiles.
//   BACKSUB  Babai's back-substitution (lll.cpp:202-214) as the mirrored wavefront, panels descending.
//   IGEMV    the fused integer row update b_kappa += sum_j (-X_j 2^e_j) b_j, columns split over the warps.
//
// Every output element is still produced by exactly the reference's sequence of correctly rounded operations (the
// per-lane chains are the ones of gso_warp.cuh / gso_lll.cuh, cut at panel boundaries), so results are bit-identical to
// the one-warp kernels — tests/test_gso_gpu.py runs both against the same reference trajectories.
//
// Synchronisation: named barrier 1 dispatches a command (master posts it in shared memory, all warps arrive), named
// barrier 2 separates the steps inside an operation (all warps execute the same operation with warp-uniform control
// flow).  No spin-waits.
#pragma once
#include "gso_warp.cuh"

namespace b200 {

// -DB200_LLL_PROFILE: device-clock counters of the cooperative operations (thread 0 of the one CTA BKZ runs), read back
// by b200gso_lll_cta_prof: [0] update calls [1] wavefront steps [2] Gram+prefix cycles [3] wavefront cycles [4] diagonal
// cycles [5] back-substitution calls [6] its steps [7] its cycles [9] integer-row calls [10] rows [11] cycles
// [12] sum of i over update calls [13] Gram entries recomputed
#ifdef B200_LLL_PROFILE
static __device__ long long g_cta_prof[32];
#define CTA_PT(var) const long long var = clock64()
#define CTA_PADD(slot, t0)                      \
  do                                            \
  {                                             \
    if (threadIdx.x == 0)                       \
      g_cta_prof[slot] += clock64() - (t0);     \
  } while (0)
#define CTA_PCNT(slot, val)                     \
  do                                            \
  {                                             \
    if (threadIdx.x == 0)                       \
      g_cta_prof[slot] += (val);                \
  } while (0)
// same, from whichever single thread `cond` selects (one writer per slot per operation)
#define CTA_PADD_IF(cond, slot, t0)             \
  do                                            \
  {                                             \
    if (cond)                                   \
      g_cta_prof[slot] += clock64() - (t0);     \
  } while (0)
#define CTA_PCNT_IF(cond, slot, val)            \
  do                                            \
  {                                             \
    if (cond)                                   \
      g_cta_prof[slot] += (val);                \
  } while (0)
#else
#define CTA_PT(var)
#define CTA_PADD(slot, t0)
#define CTA_PCNT(slot, val)
#define CTA_PADD_IF(cond, slot, t0)
#define CTA_PCNT_IF(cond, slot, val)
#endif

constexpr int CTA_WARPS = 8;
constexpr int CTA_OWN   = 2;  // panels a warp can own: 16 panels = d <= 512

enum { COOP_EXIT = 0, COOP_UPDATE = 1, COOP_BACKSUB = 2, COOP_IGEMV = 3, COOP_MULOAD = 4, COOP_MOVE = 5 };

struct CoopShared
{
  View v;      // the master's view (its metadata pointers point into the master's shared-memory cache)
  WarpSmem s;  // the master's scratch rows (vb, rrow, murow, aux, xs)
  double *bm;  // babai_mu row handed to BACKSUB
  // Shared-memory cache of the leading mu panels, as many as fit next to the rest of the CTA's shared memory (none at
  // large d): global memory stays authoritative — every writer of mu in the LLL path writes through or refreshes the
  // cached copy — and the readers of the cooperative operations take panels < mu_s_panels from here, so that the
  // kappa-deep serial chains pay shared-memory instead of L2 latency per tile.
  double *mu_s;
  int mu_s_panels;
  // the last panel of the lattice has only d - 32 (P-1) rows: cached with a column stride just above that (odd), so that
  // at d = 200 (8 rows: stride 9, 16 KB instead of 59 KB) the WHOLE of mu is resident in shared memory
  int mu_last_p, mu_last_stride;
  // Streamed wavefronts (the pl - p0 < CTA_WARPS branch of cta_update_gso_row, cta_backsub_stream): pub[2k] = value of
  // column (row) k, pub[2k+1] = its tag (epoch + k), written with ONE 16-byte store so a reader sees both or neither.
  // The owner of a panel publishes every value the moment it is final; the warps of the later panels consume them in
  // order while the owner is still in its 32-step triangle, instead of waiting at a barrier for the whole triangle and
  // then applying 32 columns at once — the critical path becomes the chain of dependent steps itself.
  double *pub;
  double epoch;
  int cmd, a0, a1, a2;
  int flag;
};

__device__ inline void pub_store(double *slot, double val, double tag)
{
  asm volatile("st.volatile.shared.v2.f64 [%0], {%1, %2};" ::"r"((unsigned)__cvta_generic_to_shared(slot)), "d"(val),
               "d"(tag)
               : "memory");
}
// spin until the slot carries this operation's tag (all lanes read the same address: one broadcast load per poll)
__device__ inline double pub_wait(const double *slot, double tag)
{
  double val, t;
  const unsigned a = (unsigned)__cvta_generic_to_shared(slot);
  for (;;)
  {
    asm volatile("ld.volatile.shared.v2.f64 {%0, %1}, [%2];" : "=d"(val), "=d"(t) : "r"(a) : "memory");
    if (t == tag)
      break;
  }
  return val;
}

// The cached copy uses a column stride of 33 doubles instead of the global layout's 32: the forward substitution walks a
// panel by columns (lanes = 32 rows of one column: consecutive addresses either way), Babai's back-substitution walks it
// by ROWS (lanes = 32 columns of one row) — with stride 32 that is a 32-way bank conflict on every shared-memory load,
// with 33 both directions are conflict-free.
constexpr int MU_SS = 33;
__host__ __device__ inline size_t mu_s_panel_base(int p) { return (size_t)(16 * MU_SS) * p * (p + 1); }
__host__ __device__ inline int mu_s_last_stride(int d)
{
  const int rows = d - 32 * (n_panels(d) - 1);
  return rows >= 32 ? MU_SS : (rows | 1);
}
struct MuRef  // the (cached | global) mu panels as seen by one operation: copied out of CoopShared once, into registers
{
  const double *mu_s, *mu_g;
  int panels, last_p, last_stride;
  __device__ inline const double *panel(int p) const
  {
    return (p < panels) ? mu_s + mu_s_panel_base(p) : mu_g + mu_panel_base(p);
  }
  __device__ inline int stride(int p) const { return (p < panels) ? (p == last_p ? last_stride : MU_SS) : 32; }
  __device__ inline double load(int i, int k) const { return panel(i >> 5)[(size_t)k * stride(i >> 5) + (i & 31)]; }
};
__device__ inline MuRef mu_ref(const CoopShared &C)
{
  MuRef m;
  m.mu_s = C.mu_s, m.mu_g = C.v.mu, m.panels = C.mu_s_panels, m.last_p = C.mu_last_p, m.last_stride = C.mu_last_stride;
  return m;
}
__device__ inline const double *coop_mu_panel(const CoopShared &C, int p)
{
  return (p < C.mu_s_panels) ? C.mu_s + mu_s_panel_base(p) : C.v.mu + mu_panel_base(p);
}
__device__ inline int coop_mu_stride(const CoopShared &C, int p)
{
  return (p < C.mu_s_panels) ? (p == C.mu_last_p ? C.mu_last_stride : MU_SS) : 32;
}
__device__ inline void coop_mu_store(CoopShared &C, int i, int k, double val)
{
  C.v.mu[mu_off(i, k)] = val;
  if ((i >> 5) < C.mu_s_panels)
    C.mu_s[mu_s_panel_base(i >> 5) + (size_t)k * coop_mu_stride(C, i >> 5) + (i & 31)] = val;
}
__device__ inline double coop_mu_load(const CoopShared &C, int i, int k)
{
  return coop_mu_panel(C, i >> 5)[(size_t)k * coop_mu_stride(C, i >> 5) + (i & 31)];
}

__device__ inline void cta_bar(int id)
{
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(CTA_WARPS * 32) : "memory");
}

// master: publish a command and release the helpers (they wait in barrier 1)
__device__ inline void coop_post(CoopShared *C, int cmd, int a0, int a1, int a2, int lane)
{
  __syncwarp();
  if (lane == 0)
  {
    C->cmd = cmd;
    C->a0 = a0, C->a1 = a1, C->a2 = a2;
    C->epoch += 4096.0;  // a fresh tag range for the values this operation publishes
  }
  __syncwarp();
  cta_bar(1);
}

// The Gram dot product for a lone warp: same ordered chain as lane_dot (gso_warp.cuh), but 16 loads per group,
// double-buffered (32 in flight) — with nobody to hide an L2 round trip behind, the 8-deep form spends 25 trips on a
// 201-column row — and the tail fetched as one predicated group.
__device__ inline double lane_dot_deep(const double *__restrict__ col, const double *vec, int ncols)
{
  constexpr int DEPTH = 16;
  double acc   = __dmul_rn(col[0], vec[0]);
  const int k0 = 1, ng = (ncols - k0) / DEPTH;
  double x[DEPTH], y[DEPTH];
  if (ng > 0)
  {
#pragma unroll
    for (int u = 0; u < DEPTH; u++)
      x[u] = col[(size_t)(k0 + u) * 32];
  }
  for (int g = 0; g < ng; g += 2)
  {
    const int k = k0 + DEPTH * g;
    if (g + 1 < ng)
    {
#pragma unroll
      for (int u = 0; u < DEPTH; u++)
        y[u] = col[(size_t)(k + DEPTH + u) * 32];
    }
#pragma unroll
    for (int u = 0; u < DEPTH; u++)
      acc = __dadd_rn(acc, __dmul_rn(x[u], vec[k + u]));
    if (g + 2 < ng)
    {
#pragma unroll
      for (int u = 0; u < DEPTH; u++)
        x[u] = col[(size_t)(k + 2 * DEPTH + u) * 32];
    }
    if (g + 1 < ng)
    {
#pragma unroll
      for (int u = 0; u < DEPTH; u++)
        acc = __dadd_rn(acc, __dmul_rn(y[u], vec[k + DEPTH + u]));
    }
  }
  const int kt = k0 + DEPTH * ng, rem = ncols - kt;
  if (rem > 0)
  {
#pragma unroll
    for (int u = 0; u < DEPTH; u++)
      x[u] = (u < rem) ? col[(size_t)(kt + u) * 32] : 0.0;
#pragma unroll
    for (int u = 0; u < DEPTH; u++)
      if (u < rem)
        acc = __dadd_rn(acc, __dmul_rn(x[u], vec[kt + u]));
  }
  return acc;
}

// The closing part of update_gso_row(i, last_j) for the CTA: the diagonal r(i,i) = g(i,i) - sum_{k<i} mu(i,k) r(i,k)
// (products in parallel, one ordered subtraction chain) when it is asked for, then gso_valid_cols[i].
__device__ inline bool cta_update_diag(CoopShared &C, int i, int last_j, int j0, int ncols, int tid)
{
  const View v     = C.v;  // by value: registers, not a reload from shared memory after every store
  const WarpSmem s = C.s;
  double *gfrow = v.gf + tri_off(i), *rrow_g = v.r + tri_off(i);
  CTA_PT(tp2_);
  if (last_j >= i)
  {
    for (int k = tid; k < min(j0, i); k += CTA_WARPS * 32)
      s.murow[k] = coop_mu_load(C, i, k);
    cta_bar(2);
    for (int k = tid; k < i; k += CTA_WARPS * 32)
      s.aux[k] = __dmul_rn(s.murow[k], s.rrow[k]);
    const bool gnan = (gfrow[i] != gfrow[i]);  // then s.vb holds bf_i: square it in place, the chain below only adds
    if (gnan)
      for (int c = tid; c < ncols; c += CTA_WARPS * 32)
        s.vb[c] = __dmul_rn(s.vb[c], s.vb[c]);
    cta_bar(2);
    if (tid == 0)
    {
      double g = gfrow[i];
      if (gnan)
      {
        g        = serial_chain<false, false>(s.vb[0], s.vb + 1, ncols - 1, nullptr);
        gfrow[i] = g;
      }
      const double a     = serial_chain<true, false>(g, s.aux, i, nullptr);
      rrow_g[i]          = a;
      coop_mu_store(C, i, i, a);  // diagonal mirror
    }
  }
  if (tid == 0)
    v.valid[i] = last_j + 1;
  cta_bar(2);
  CTA_PADD(4, tp2_);
  return true;
}

// ---- UPDATE ---------------------------------------------------------------------------------------------------------
// update_gso_row(i, last_j) for a row that is already discovered and has valid[i] <= last_j (the master checks both).
// Same arithmetic as warp_update_gso_row: lane l of panel p owns column j = 32p + l,
//   acc_j = g(i,j); acc_j -= mu(j,k) r(i,k) for k = 0 .. j-1 ascending.
__device__ inline bool cta_update_gso_row(CoopShared &C, int i, int last_j, int w, int lane)
{
  const View v     = C.v;  // by value: registers, not a reload from shared memory after every store
  const WarpSmem s = C.s;
  const int tid = threadIdx.x;
  const int j0  = max(0, v.valid[i]);
  const int ncols = v.meta[M_NKC], n = v.n;
  double *gfrow = v.gf + tri_off(i), *rrow_g = v.r + tri_off(i);
  const int jl = min(last_j, i - 1);  // last off-diagonal column to produce
  const int p0 = j0 >> 5;
  const int pl = (jl >= j0) ? (jl >> 5) : p0 - 1;  // panels p0..pl carry work (none if only the diagonal is asked for)
  CTA_PT(tp0_);
  CTA_PCNT(0, 1);
  CTA_PCNT(1, pl - p0 + 1);
  CTA_PCNT(12, i);

  {
    // bf_i is needed if any Gram entry of the row is invalid: every warp looks (the same few loads, in parallel) and the
    // whole CTA stages the row — one element per thread instead of one warp walking it alone before everybody's barrier
    int anyn = 0;
    for (int j = j0 + lane; j <= last_j; j += 32)
      anyn |= (gfrow[j] != gfrow[j]);
    if (__any_sync(FULL, anyn))
      stage_bf_row(v, i, ncols, s.vb, tid, CTA_WARPS * 32);
    if (tid == 0)
      C.flag = 1;
  }
  for (int k = tid; k < j0; k += CTA_WARPS * 32)
    s.rrow[k] = rrow_g[k];
  cta_bar(2);

  if (pl - p0 < CTA_WARPS)
  {
    // ---- streamed wavefront: one panel per warp, values handed on through C.pub as they become final ----
    const int p    = p0 + w;
    const int j    = 32 * p + lane;
    const bool own = p <= pl;
    const bool a_  = own && j >= j0 && j <= jl;
    const MuRef M  = mu_ref(C);
    double *pub    = C.pub;
    const int cs   = own ? M.stride(p) : 32;
    const double *mup = own ? M.panel(p) + lane : v.mu;
    double a = 0.0;
    CTA_PT(tgd_);
    if (a_)
    {
      double g = gfrow[j];
      if (g != g)
      {
        g        = lane_dot_deep(v.bf + bf_off(j, 0, n), s.vb, ncols);
        gfrow[j] = g;
        if (threadIdx.x == 0)
          CTA_PCNT(13, 32);
      }
      CTA_PADD(21, tgd_);
      CTA_PT(tgp_);
      a = lane_chain<true>(g, mup, s.rrow, 0, 32 * p0, cs);
      CTA_PADD(22, tgp_);
    }
    else if (own && j < j0)
      a = s.rrow[j];  // already-valid r(i,j): published for the later panels, broadcast in the triangle
    CTA_PADD(2, tp0_);
    CTA_PT(tps_);
    bool ok = true;
    if (own)
    {
      const double tb = C.epoch;
      // columns of the earlier panels, in order, as their owners publish them
      CTA_PT(tuc_);
      for (int k = 32 * p0; k < 32 * p; k += 8)
      {
        double m[8];
#pragma unroll
        for (int u = 0; u < 8; u++)
          m[u] = a_ ? mup[(size_t)(k + u) * cs] : 0.0;
#pragma unroll
        for (int u = 0; u < 8; u++)
        {
          const double rk = pub_wait(pub + 2 * (k + u), tb + (double)(k + u));
          if (a_)
            a = __dsub_rn(a, __dmul_rn(m[u], rk));
        }
      }
      CTA_PADD_IF(lane == 0 && p == pl && p != p0, 19, tuc_);
      CTA_PT(tut_);
      // my triangle: column 32 p + t is final in lane t once steps 0..t-1 are applied — published at once.  A ROLLED loop
      // (the step stays in the instruction cache); the tile entry of the next column is requested one step ahead.
      const double *tile = mup + (size_t)(32 * p) * cs;
      double rd          = 1.0;
      double m           = a_ ? tile[0] : 0.0;  // lane >= 0
#pragma unroll 1
      for (int t = 0; t < 32; ++t)
      {
        const double mn = (a_ && lane >= t + 1 && t < 31) ? tile[(size_t)(t + 1) * cs] : 0.0;
        if (lane == t)
        {
          rd = m;  // r(j,j), mirrored in the mu(j,j) slot of the diagonal tile
          pub_store(pub + 2 * (32 * p + t), a, tb + (double)(32 * p + t));
        }
        const double rk = __shfl_sync(FULL, a, t);
        if (a_ && lane > t)
          a = __dsub_rn(a, __dmul_rn(m, rk));
        m = mn;
      }
      CTA_PADD_IF(lane == 0 && p == p0, 18, tut_);
      CTA_PADD_IF(lane == 0 && p == pl && p != p0, 20, tut_);
      if (a_)
      {
        rrow_g[j]       = a;
        s.rrow[j]       = a;
        const double mm = __ddiv_rn(a, rd);
        coop_mu_store(C, i, j, mm);
        s.murow[j]      = mm;
        if (!isfinite(mm))
          ok = false;
      }
    }
    if (!ok)
      C.flag = 0;
    cta_bar(2);
    CTA_PADD(3, tps_);
    if (!C.flag)
      return false;
    return cta_update_diag(C, i, last_j, j0, ncols, tid);
  }

  // Gram entries + the part of every chain that only needs the already-valid r(i, k), k < 32 p0
  double acc[CTA_OWN];
  bool act[CTA_OWN];
#pragma unroll
  for (int u = 0; u < CTA_OWN; u++)
  {
    const int p = p0 + w + CTA_WARPS * u;
    const int j = 32 * p + lane;
    act[u]      = (p <= pl) && (j >= j0) && (j <= jl);
    double a    = 0.0;
    if (act[u])
    {
      double g = gfrow[j];
      if (g != g)
      {
        g        = lane_dot_deep(v.bf + bf_off(j, 0, n), s.vb, ncols);
        gfrow[j] = g;
        if (threadIdx.x == 0)
          CTA_PCNT(13, 32);
      }
      a = lane_chain<true>(g, coop_mu_panel(C, p) + lane, s.rrow, 0, 32 * p0, coop_mu_stride(C, p));
    }
    else if (p <= pl && j < j0)
      a = s.rrow[j];  // already-valid r(i,j): only broadcast in the triangle below
    acc[u] = a;
  }

  bool ok = true;
  CTA_PADD(2, tp0_);
  CTA_PT(tp1_);
  for (int sp = p0; sp <= pl; ++sp)
  {
    const int ow = (sp - p0) % CTA_WARPS, ou = (sp - p0) / CTA_WARPS;
    if (ow == w)
    {
      // triangular part of panel sp: column 32 sp + t is final in lane t once steps 0..t-1 are applied
#pragma unroll
      for (int u = 0; u < CTA_OWN; u++)
        if (u == ou)
        {
          const int j        = 32 * sp + lane;
          const bool a_      = act[u];
          double a           = acc[u];
          const int cs       = coop_mu_stride(C, sp);
          const double *tile = coop_mu_panel(C, sp) + lane + (size_t)(32 * sp) * cs;
          double rd          = 1.0;
          double m[8], mn[8];
#pragma unroll
          for (int x = 0; x < 8; x++)
            m[x] = (a_ && lane >= x) ? tile[(size_t)x * cs] : 0.0;
#pragma unroll
          for (int q = 0; q < 4; q++)
          {
            if (q < 3)
            {
#pragma unroll
              for (int x = 0; x < 8; x++)
                mn[x] = (a_ && lane >= 8 * (q + 1) + x) ? tile[(size_t)(8 * (q + 1) + x) * cs] : 0.0;
            }
#pragma unroll
            for (int x = 0; x < 8; x++)
            {
              const int t = 8 * q + x;
              if (lane == t)
                rd = m[x];
              if (t < 31)
              {
                const double rk = __shfl_sync(FULL, a, t);
                if (a_ && lane > t)
                  a = __dsub_rn(a, __dmul_rn(m[x], rk));
              }
            }
#pragma unroll
            for (int x = 0; x < 8; x++)
              m[x] = mn[x];
          }
          if (a_)
          {
            rrow_g[j]          = a;
            s.rrow[j]          = a;
            const double mm    = __ddiv_rn(a, rd);
            coop_mu_store(C, i, j, mm);
            s.murow[j]         = mm;
            if (!isfinite(mm))
              ok = false;
          }
          acc[u] = a;
        }
    }
    cta_bar(2);
    // everybody below: apply the tile (p, sp) now that r(i, 32 sp .. 32 sp + 31) are final
#pragma unroll
    for (int u = 0; u < CTA_OWN; u++)
    {
      const int p = p0 + w + CTA_WARPS * u;
      if (p > sp && act[u])
        acc[u] = lane_chain<true>(acc[u], coop_mu_panel(C, p) + lane, s.rrow, 32 * sp, 32 * sp + 32, coop_mu_stride(C, p));
    }
  }
  if (!ok)
    C.flag = 0;
  cta_bar(2);
  CTA_PADD(3, tp1_);
  if (!C.flag)
    return false;
  return cta_update_diag(C, i, last_j, j0, ncols, tid);
}

// ---- BACKSUB --------------------------------------------------------------------------------------------------------
// X_j = rnd_we(babai_mu[j]); babai_mu[k] -= X_j * mu(j,k) for k < j, j descending (lll.cpp:202-214).  C.bm holds
// babai_mu (columns < sr_end); the X_j land in s.xs[j], the per-panel masks of the non-zero ones in xmask[].
__device__ inline void cta_backsub(CoopShared &C, int kappa, int sr_end, int sr_start, int w, int lane)
{
  const View v     = C.v;  // by value: registers, not a reload from shared memory after every store
  const WarpSmem s = C.s;
  const int ek  = v.row_expo[kappa];
  unsigned *xmask = (unsigned *)(s.xs + ((v.d + 1) & ~1));
  const int p_hi = (sr_end - 1) >> 5, p_lo = sr_start >> 5;
  CTA_PT(tb0_);
  CTA_PCNT(5, 1);
  CTA_PCNT(6, p_hi - p_lo + 1);
  if (p_hi - p_lo < CTA_WARPS)
  {
    // ---- streamed: warp w owns panel q = p_hi - w; every X_j is published the moment it is rounded and the lower panels
    // apply row j while the owner goes on to row j-1 (see CoopShared::pub) ----
    const int q    = p_hi - w;
    const bool own = q >= p_lo;
    if (own)
    {
      const MuRef M     = mu_ref(C);
      double *pub       = C.pub;
      const double tb   = C.epoch;
      const int k       = 32 * q + lane;
      const bool colact = k >= sr_start && k < sr_end;
      double a          = (k < sr_end) ? C.bm[k] : 0.0;
      // rows of the panels above mine, descending, as their owners publish X_j
      CTA_PT(tcons_);
      for (int pj = p_hi; pj > q; --pj)
      {
        const double *rowp = M.panel(pj) + (size_t)k * M.stride(pj);  // mu(32 pj + t, k) at [t]
        for (int t = min(31, sr_end - 1 - 32 * pj); t >= 0; --t)
        {
          const double m = colact ? rowp[t] : 0.0;
          const double X = pub_wait(pub + 2 * (32 * pj + t), tb + (double)(32 * pj + t));
          if (X != 0.0 && colact)
            a = __dsub_rn(a, __dmul_rn(X, m));
        }
      }
      CTA_PADD_IF(lane == 0 && q == p_lo && q != p_hi, 16, tcons_);
      CTA_PT(ttri_);
      // my triangle.  Lane l holds the constants of ROW 32q + l: rnd_we(x, de) = rint(x * 2^de) * 2^-de for every finite
      // x once |de| is moderate (de = 0: rint(x); |x * 2^de| >= 2^52: already an integer, the product is undone
      // exactly = the reference's "return x" branch; tiny: rounds to zero like ldexp's result would), so every lane
      // rounds its own value each step and the owner of row t broadcasts the result — no branches, no library calls.
      const int jl_     = 32 * q + lane;
      const bool rowin  = jl_ >= sr_start && jl_ < sr_end;
      const long de_l   = (rowin && v.row_expo_en) ? (long)(ek - v.row_expo[jl_]) : 0;
      const bool fast   = !__any_sync(FULL, rowin && (de_l <= -900 || de_l >= 900));
      const double sc   = fast ? pow2d((int)de_l) : 1.0, isc = fast ? pow2d((int)-de_l) : 1.0;
      const double *tilecol = M.panel(q) + (size_t)k * M.stride(q);  // mu(32q+t, k) at [t]
      const int t_hi = min(31, sr_end - 1 - 32 * q), t_lo = max(0, sr_start - 32 * q);
      const bool upd = k >= sr_start;
      unsigned nzmask = 0;
      // A ROLLED loop: the step is ~20 instructions that stay in the instruction cache; the tile entry of the next row
      // is requested one step ahead (a shared-memory load when the panel is cached, and every panel of a d <= 200 lattice
      // is), so it is off the critical path  round -> shuffle -> multiply -> subtract.
      double m = (t_hi > lane && t_hi >= t_lo) ? tilecol[t_hi] : 0.0;
#pragma unroll 1
      for (int t = t_hi; t >= t_lo; --t)
      {
        const double mn = (t - 1 > lane && t - 1 >= t_lo) ? tilecol[t - 1] : 0.0;
        double X;
        if (fast)
        {
          const double y = __dmul_rn(a, sc);
          double xl      = __dmul_rn(rint(y), isc);
          if (!(fabs(y) < 1e300))  // overflowed product / non-finite input: the reference's own branches
            xl = rnd_we_slow(a, de_l);
          X = __shfl_sync(FULL, xl, t);
        }
        else
        {
          const double bj = __shfl_sync(FULL, a, t);
          X               = rnd_we(bj, __shfl_sync(FULL, (int)de_l, t));
        }
        if (lane == 0)
          pub_store(pub + 2 * (32 * q + t), X, tb + (double)(32 * q + t));
        if (X != 0.0)
        {
          nzmask |= 1u << t;
          if (lane == 0)
            s.xs[32 * q + t] = X;
          if (lane < t && upd)
            a = __dsub_rn(a, __dmul_rn(X, m));
        }
        m = mn;
      }
      if (lane == 0)
        xmask[q] = nzmask;
      CTA_PADD_IF(lane == 0 && q == p_hi, 8, ttri_);
      CTA_PCNT_IF(lane == 0 && q == p_hi, 14, t_hi - t_lo + 1);
      CTA_PADD_IF(lane == 0 && q == p_lo && q != p_hi, 17, ttri_);
      CTA_PCNT_IF(lane == 0 && q == p_lo && q != p_hi, 15, t_hi - t_lo + 1);
    }
    cta_bar(2);
    CTA_PADD(7, tb0_);
    return;
  }
  // panel q is owned by warp (p_hi - q) % CTA_WARPS, slot (p_hi - q) / CTA_WARPS
  double val[CTA_OWN];
#pragma unroll
  for (int u = 0; u < CTA_OWN; u++)
  {
    const int q = p_hi - w - CTA_WARPS * u;
    const int k = 32 * q + lane;
    val[u]      = (q >= p_lo && k < sr_end) ? C.bm[k] : 0.0;
  }
  for (int p = p_hi; p >= p_lo; --p)
  {
    const int ow = (p_hi - p) % CTA_WARPS, ou = (p_hi - p) / CTA_WARPS;
    if (ow == w)
    {
#pragma unroll
      for (int u = 0; u < CTA_OWN; u++)
        if (u == ou)
        {
          double a              = val[u];
          const int kcol        = 32 * p + lane;
          const double *tilecol = coop_mu_panel(C, p) + (size_t)kcol * coop_mu_stride(C, p);  // mu(32p+t, kcol) at [t]
          unsigned nzmask       = 0;
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
            const double bj = __shfl_sync(FULL, a, t);
            const long de   = v.row_expo_en ? (long)(ek - v.row_expo[j]) : 0;
            const double X  = rnd_we(bj, de);
            if (X == 0.0)
              continue;
            nzmask |= 1u << t;
            if (lane == 0)
              s.xs[j] = X;
            if (lane < t && kcol >= sr_start)
              a = __dsub_rn(a, __dmul_rn(X, tc[t]));
          }
          if (lane == 0)
            xmask[p] = nzmask;
          val[u] = a;
        }
    }
    cta_bar(2);
    const unsigned nzmask = xmask[p];
    if (nzmask)
    {
#pragma unroll
      for (int u = 0; u < CTA_OWN; u++)
      {
        const int q = p_hi - w - CTA_WARPS * u;
        const int k = 32 * q + lane;
        if (q < p && q >= p_lo && k >= sr_start)
        {
          const double *col = coop_mu_panel(C, p) + (size_t)k * coop_mu_stride(C, p);
          double a          = val[u];
          double cv[32];  // mu(32p + t, k), t = 0..31: 32 independent loads in flight
#pragma unroll
          for (int t = 0; t < 32; t++)
            cv[t] = ((nzmask >> t) & 1u) ? col[t] : 0.0;
#pragma unroll
          for (int t = 31; t >= 0; --t)  // rows with X != 0 only, still in descending order
            if ((nzmask >> t) & 1u)
              a = __dsub_rn(a, __dmul_rn(s.xs[32 * p + t], cv[t]));
          val[u] = a;
        }
      }
    }
  }
  CTA_PADD(7, tb0_);
}

// ---- IGEMV ----------------------------------------------------------------------------------------------------------
// b_kappa += sum_t lx_t * 2^e_t * b_{row_t} over the nnz compacted rows (lx in s.aux[t], (e << 32 | row) in s.murow[t]):
// row_addmul_we (gso.cpp:236-262) fused over j; int64 arithmetic wraps, so the order of the additions is immaterial.
// Warp w takes the column groups w, w + CTA_WARPS, ... of 32 columns.
__device__ inline void cta_igemv(CoopShared &C, int kappa, int nnz, int w, int lane)
{
  const View v     = C.v;  // by value: registers, not a reload from shared memory after every store
  const WarpSmem s = C.s;
  const int nc  = v.meta[M_NKC];
  CTA_PT(ti0_);
  CTA_PCNT(9, 1);
  CTA_PCNT(10, nnz);
  unsigned long long *bk = (unsigned long long *)(v.b + (size_t)kappa * v.ldb);
  for (int c0 = 32 * w; c0 < nc; c0 += 32 * CTA_WARPS)
  {
    const int c = c0 + lane;
    unsigned long long acc = (c < nc) ? bk[c] : 0ull;
    for (int t0 = 0; t0 < nnz; t0 += 16)
    {
      unsigned long long bv[16], lxv[16];
      int ev[16];
#pragma unroll
      for (int x = 0; x < 16; x++)
      {
        const int t = t0 + x;
        bv[x] = 0ull, lxv[x] = 0ull, ev[x] = 0;
        if (t < nnz)
        {
          lxv[x]             = (unsigned long long)__double_as_longlong(s.aux[t]);
          const long long pk = __double_as_longlong(s.murow[t]);
          ev[x]              = (int)(pk >> 32);
          const unsigned long long *src = (const unsigned long long *)(v.b + (size_t)(int)(pk & 0xffffffffll) * v.ldb);
          if (c < nc)
            bv[x] = src[c];
        }
      }
#pragma unroll
      for (int x = 0; x < 16; x++)
      {
        const unsigned long long tt = bv[x] * lxv[x];
        acc += (ev[x] >= 64 ? 0ull : (tt << ev[x]));
      }
    }
    if (c < nc)
      bk[c] = acc;
  }
  cta_bar(2);
  CTA_PADD(11, ti0_);
}

// ---- MULOAD --------------------------------------------------------------------------------------------------------
// (re)fill the shared-memory copies of the mu panels pa..pb (those that are cached) from global memory
__device__ inline void cta_mu_load(CoopShared &C, int pa, int pb, int w, int lane)
{
  const int tid = threadIdx.x;
  const int hi  = min(pb, C.mu_s_panels - 1);
  for (int p = max(pa, 0); p <= hi; ++p)
  {
    // global panel [column][32 rows] -> cached panel [column][stride]: both sides walk the rows of one column; the
    // partial last panel keeps only its real rows
    const double *src = C.v.mu + mu_panel_base(p);
    double *dst       = C.mu_s + mu_s_panel_base(p);
    const int cs      = coop_mu_stride(C, p);
    const int rows    = (p == C.mu_last_p) ? C.v.d - 32 * p : 32;
    const int cnt     = 32 * 32 * (p + 1);
    int t = tid;
    for (; t + 7 * CTA_WARPS * 32 < cnt; t += 8 * CTA_WARPS * 32)
    {
      double x[8];
#pragma unroll
      for (int u = 0; u < 8; u++)
        x[u] = ((t & 31) < rows) ? src[t + u * CTA_WARPS * 32] : 0.0;  // (t + u * 256) & 31 == t & 31
#pragma unroll
      for (int u = 0; u < 8; u++)
      {
        const int q = t + u * CTA_WARPS * 32;
        if ((q & 31) < rows)
          dst[(q >> 5) * cs + (q & 31)] = x[u];
      }
    }
    for (; t < cnt; t += CTA_WARPS * 32)
      if ((t & 31) < rows)
        dst[(t >> 5) * cs + (t & 31)] = src[t];
  }
  cta_bar(2);
}

// ---- MOVE -----------------------------------------------------------------------------------------------------------
// move_row(old_r, new_r) (gso.cpp:289-366) by the whole CTA: warp_move_row (gso_warp.cuh) with its lane-strided passes
// (one column of mu / r / b / bf per lane, one Gram row per lane) strided over all CTA_WARPS * 32 threads instead; the
// data movement per element is the same, only who carries it differs.
__device__ inline void cta_move_row(CoopShared &C, int old_r, int new_r, int w, int lane)
{
  const View v  = C.v;
  const int tid = threadIdx.x, NT = CTA_WARPS * 32;
  if (old_r == new_r)
  {
    cta_bar(2);
    return;
  }
  const int nkr    = v.meta[M_NKR];
  const bool right = new_r < old_r;
  const int lo = right ? new_r : old_r, hi = right ? old_r : new_r;
  cta_bar(2);  // everybody has read nkr and the old validity before anybody lowers it
  for (int i = lo + tid; i < nkr; i += NT)
    v.valid[i] = min(v.valid[i], lo);
  if (tid == 0)
  {
    v.meta[M_CLEAN_SR]  = min(v.meta[M_CLEAN_SR], lo);
    v.meta[M_CLEAN_LLL] = min(v.meta[M_CLEAN_LLL], lo);
  }
  for (int k = tid; k < lo; k += NT)
  {
    rotate_seq<double>([&](int i) -> double & { return v.mu[mu_off(i, k)]; }, lo, hi, right);
    rotate_seq<double>([&](int i) -> double & { return v.r[tri_off(i) + k]; }, lo, hi, right);
  }
  for (int c = tid; c < v.n; c += NT)
  {
    rotate_seq<int64_t>([&](int i) -> int64_t & { return v.b[(size_t)i * v.ldb + c]; }, lo, hi, right);
    rotate_seq<double>([&](int i) -> double & { return v.bf[bf_off(i, c, v.n)]; }, lo, hi, right);
  }
  const int ghi      = right ? hi : min(hi, nkr - 1);
  const bool do_gram = right || lo < nkr - 1;
  const size_t beg   = tri_off(lo), end = do_gram ? tri_off(ghi + 1) : beg;
  if (do_gram)
  {
    for (int i = ghi + 1 + tid; i < nkr; i += NT)
    {
      double *row = v.gf + tri_off(i);
      rotate_seq<double>([&](int j) -> double & { return row[j]; }, lo, ghi, right);
    }
    for (size_t t = beg + tid; t < end; t += NT)
      v.scratch[t - beg] = v.gf[t];
  }
  cta_bar(2);  // scratch copy complete
  if (do_gram)
  {
    // the rotated rows, rebuilt from the scratch copy: new(i,j) = old_sym(s(i), s(j)); (row, column) pairs over the CTA
    for (int i = lo + w; i <= ghi; i += CTA_WARPS)
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
  cta_bar(2);  // validity minima above are complete before the per-row metadata rotates
  if (tid == 0)
    rotate_seq<int>([&](int i) -> int & { return v.valid[i]; }, lo, hi, right);
  else if (tid == 32)
    rotate_seq<int>([&](int i) -> int & { return v.row_expo[i]; }, lo, hi, right);
  else if (tid == 64 && !right && new_r >= nkr)
    rotate_seq<int>([&](int i) -> int & { return v.irs[i]; }, lo, hi, false);
  cta_bar(2);
  if (!right && new_r >= nkr && old_r < nkr && w == 0)
  {
    const int nz = v.host_basis ? v.n : size_nz_warp(v.b + (size_t)new_r * v.ldb, v.n, lane);
    if (lane == 0)
    {
      v.meta[M_NKR] = nkr - 1;
      v.meta[M_NSR] = nkr - 1;
      v.irs[new_r]  = max(nz, 1);
    }
  }
  cta_bar(2);
}

// helper warps: wait for commands until the master says EXIT
__device__ inline void coop_helper_loop(CoopShared &C, int w, int lane)
{
  for (;;)
  {
    cta_bar(1);
    const int cmd = C.cmd, a0 = C.a0, a1 = C.a1, a2 = C.a2;
    if (cmd == COOP_EXIT)
      break;
    if (cmd == COOP_UPDATE)
      (void)cta_update_gso_row(C, a0, a1, w, lane);
    else if (cmd == COOP_BACKSUB)
      cta_backsub(C, a0, a1, a2, w, lane);
    else if (cmd == COOP_IGEMV)
      cta_igemv(C, a0, a1, w, lane);
    else if (cmd == COOP_MULOAD)
      cta_mu_load(C, a0, a1, w, lane);
    else if (cmd == COOP_MOVE)
      cta_move_row(C, a0, a1, w, lane);
  }
}

// master side of update_gso_row: the reference's early exits, then the cooperative operation
template <bool COOP>
__device__ inline bool lll_update_gso_row(const View &v, int i, int last_j, WarpSmem &s, int lane, CoopShared *C)
{
  if (!COOP)
    return warp_update_gso_row(v, i, last_j, s, lane);
  if (i >= v.meta[M_NKR])
    warp_discover_row(v, lane);
  const int j0 = max(0, v.valid[i]);
  if (j0 > last_j)
    return true;
  if (i < 32)
  {
    // a single panel: nothing to share.  The one-warp routine writes mu(i, .) to global memory only: refresh the
    // cached copy of that row (mu_off(i, k) = 32 k + i in panel 0)
    const bool ok = warp_update_gso_row(v, i, last_j, s, lane);
    if (C->mu_s_panels > 0)
    {
      __syncwarp();
      C->mu_s[coop_mu_stride(*C, 0) * lane + i] = v.mu[32 * lane + i];
      __syncwarp();
    }
    return ok;
  }
  coop_post(C, COOP_UPDATE, i, last_j, 0, lane);
  return cta_update_gso_row(*C, i, last_j, 0, lane);
}

// mu(i,k) as the LLL loop reads it: the one-CTA kernel through its cached panels
template <bool COOP> __device__ inline double lll_mu_load(const View &v, const CoopShared *C, int i, int k)
{
  return COOP ? coop_mu_load(*C, i, k) : v.mu[mu_off(i, k)];
}

// master: after a one-warp routine rewrote parts of mu in global memory (move_row: rows lo..hi rotate; set_r: the
// diagonal mirror), bring the cached panels back in line
template <bool COOP> __device__ inline void lll_mu_reload(CoopShared *C, int row_lo, int row_hi, int lane)
{
  if (!COOP || C->mu_s_panels == 0 || (row_lo >> 5) >= C->mu_s_panels)
    return;
  coop_post(C, COOP_MULOAD, row_lo >> 5, row_hi >> 5, 0, lane);
  cta_mu_load(*C, row_lo >> 5, row_hi >> 5, 0, lane);
}
template <bool COOP> __device__ inline void lll_mu_refresh_diag(CoopShared *C, int i, int lane)
{
  if (!COOP || (i >> 5) >= C->mu_s_panels)
    return;
  __syncwarp();
  if (lane == 0)
    C->mu_s[mu_s_panel_base(i >> 5) + (size_t)i * coop_mu_stride(*C, i >> 5) + (i & 31)] = C->v.mu[mu_off(i, i)];
  __syncwarp();
}

template <bool COOP> __device__ inline void lll_move_row(const View &v, int old_r, int new_r, int lane, CoopShared *C)
{
  if (!COOP)
  {
    warp_move_row(v, old_r, new_r, lane);
    return;
  }
  coop_post(C, COOP_MOVE, old_r, new_r, 0, lane);
  cta_move_row(*C, old_r, new_r, 0, lane);
}

}  // namespace b200
