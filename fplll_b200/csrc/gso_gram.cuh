// gso_gram.cuh — blocked recomputation of the whole float Gram matrix gf = bf * bf^T (lower triangle) for a batch.
//
// update_gso() row by row (k_update_gso) recomputes g(i, j) inside update_gso_row: row i re-streams the bf panels of
// all rows j <= i, d^2 n / 64 panel-column loads per lattice (32 MB at d = 200) — HBM-bound on its own re-reads.  Here
// one warp produces a 32 x 32 TILE of Gram entries
// per pass over the columns, so a bf panel column is loaded once per 32 results: this is the one piece of the path
// that is a dense contraction (SURVEY §8 a3).
//
//   ORDERED  every entry is the reference's left-to-right dot product (numvect.h:385-395: first term a bare product,
//            then acc = acc + x*y with two roundings, ascending column) — lane j keeps 32 accumulators, the 32 row values of
//            a column arrive by shuffle.  Bit-identical to get_gram (gso.h:314-331).
//   DMMA     fp64 tensor-core mma.sync.m8n8k4 (16 per 32 x 32 tile and 4 columns).  The hardware's summation order is
//            not the reference's: results are bit-identical only where every partial sum is exact (|bf|^2 n < 2^53, e.g.
//            the 2^20-entry benchmark bases), otherwise equal to ~1 ulp per term — inside north_star's 1e-9 on mu, r
//            for well-conditioned rows, NOT trajectory-exact; never used by the LLL/BKZ path.
//
// STATUS: written at the end of round 1 with no GPU time left — compiled, exported (b200gso_update_gso_blocked) and
// covered by tests that only run with B200_TEST_EXPERIMENTAL=1; not yet exercised on hardware, not called by anything
// else.
#pragma once
#include "gso_warp.cuh"

namespace b200 {

enum { GRAM_ORDERED = 0, GRAM_DMMA = 1 };

// tile pair t -> (pi >= pj)
__device__ inline void gram_pair(int t, int &pi, int &pj)
{
  int p = (int)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
  while ((p + 1) * (p + 2) / 2 <= t)
    ++p;
  while (p * (p + 1) / 2 > t)
    --p;
  pi = p;
  pj = t - p * (p + 1) / 2;
}

// One warp: Gram tile (rows 32 pi .. +31) x (columns 32 pj .. +31), reference order.
__device__ inline void warp_gram_tile_ordered(const View &v, int pi, int pj, int ncols, int lane)
{
  const int n = v.n, d = v.d;
  const double *bj = v.bf + (size_t)pj * 32 * n + lane;  // bf(32 pj + lane, c) at bj[32 c]
  const double *bi = v.bf + (size_t)pi * 32 * n + lane;  // bf(32 pi + lane, c) at bi[32 c]
  double acc[32];
  {
    const double x = bj[0], y = bi[0];
#pragma unroll
    for (int r = 0; r < 32; r++)
      acc[r] = __dmul_rn(__shfl_sync(FULL, y, r), x);
  }
  constexpr int G = 4;  // columns requested ahead
  double xs[G], ys[G];
  int c = 1;
#pragma unroll
  for (int u = 0; u < G; u++)
  {
    xs[u] = (c + u < ncols) ? bj[(size_t)(c + u) * 32] : 0.0;
    ys[u] = (c + u < ncols) ? bi[(size_t)(c + u) * 32] : 0.0;
  }
  for (; c < ncols; c += G)
  {
    double xn[G], yn[G];
#pragma unroll
    for (int u = 0; u < G; u++)
    {
      xn[u] = (c + G + u < ncols) ? bj[(size_t)(c + G + u) * 32] : 0.0;
      yn[u] = (c + G + u < ncols) ? bi[(size_t)(c + G + u) * 32] : 0.0;
    }
#pragma unroll
    for (int u = 0; u < G; u++)
      if (c + u < ncols)
      {
#pragma unroll
        for (int r = 0; r < 32; r++)
          acc[r] = __dadd_rn(acc[r], __dmul_rn(__shfl_sync(FULL, ys[u], r), xs[u]));
      }
#pragma unroll
    for (int u = 0; u < G; u++)
      xs[u] = xn[u], ys[u] = yn[u];
  }
  const int j = 32 * pj + lane;
#pragma unroll
  for (int r = 0; r < 32; r++)
  {
    const int i = 32 * pi + r;
    if (i < d && j <= i)
      v.gf[tri_off(i) + j] = acc[r];
  }
}

__device__ inline void dmma_8x8x4(double &c0, double &c1, double a, double b)
{
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// The same tile on the fp64 tensor cores: 4 x 4 blocks of 8 x 8, k = 4 columns per step.
// Fragment layout (PTX ISA, mma.m8n8k4 .f64): lane t holds A[t>>2][t&3], B[t&3][t>>2], C[t>>2][2(t&3)], C[t>>2][2(t&3)+1].
// With A = bf rows of panel pi and B^T = bf rows of panel pj both operands are read as bf(row0 + (t>>2), c0 + (t&3)).
__device__ inline void warp_gram_tile_dmma(const View &v, int pi, int pj, int ncols, int lane)
{
  const int n = v.n, d = v.d;
  const int fr = lane >> 2, fk = lane & 3;
  const double *pa = v.bf + (size_t)pi * 32 * n + fr;  // + 8 ib + 32 (c0 + fk)
  const double *pb = v.bf + (size_t)pj * 32 * n + fr;
  double c0[4][4], c1[4][4];
#pragma unroll
  for (int ib = 0; ib < 4; ib++)
#pragma unroll
    for (int jb = 0; jb < 4; jb++)
      c0[ib][jb] = c1[ib][jb] = 0.0;
  for (int cb = 0; cb < ncols; cb += 4)
  {
    const int c   = cb + fk;
    const bool in = c < ncols;  // zero-padded last step
    double a[4], b[4];
#pragma unroll
    for (int q = 0; q < 4; q++)
    {
      a[q] = in ? pa[(size_t)c * 32 + 8 * q] : 0.0;
      b[q] = in ? pb[(size_t)c * 32 + 8 * q] : 0.0;
    }
#pragma unroll
    for (int ib = 0; ib < 4; ib++)
#pragma unroll
      for (int jb = 0; jb < 4; jb++)
        dmma_8x8x4(c0[ib][jb], c1[ib][jb], a[ib], b[jb]);
  }
#pragma unroll
  for (int ib = 0; ib < 4; ib++)
#pragma unroll
    for (int jb = 0; jb < 4; jb++)
    {
      const int i = 32 * pi + 8 * ib + fr;
      const int j = 32 * pj + 8 * jb + 2 * fk;
      if (i < d)
      {
        if (j <= i)
          v.gf[tri_off(i) + j] = c0[ib][jb];
        if (j + 1 <= i)
          v.gf[tri_off(i) + j + 1] = c1[ib][jb];
      }
    }
}

}  // namespace b200
