// hh_api.cu — GPU-native MatHouseholder<long,double> (HLLL data plane) behind include/b200hh.h.
//
// One warp per lattice (batches are the replica axis, SURVEY §8e).  HBM layout per lattice: b (int64), bf, R, V
// row-major d x n — update_R streams V_j[j..n) row by row (contiguous, 256-byte coalesced warp loads) against R_i held
// in shared memory; the reference's R_history trace (householder.h:103-109) is kept in full when requested, addressed
// through a per-row slot table so that swap() is the O(1) pointer swap it is in the reference.
// Bit parity: a dot product is formed as element products in parallel (each correctly rounded, as the reference's
// mul) followed by ONE lane adding them in ascending index order — the reference's exact chain (numvect.h:385-395).
// In a batch the serial chain of one warp hides behind the other resident warps' HBM streaming (update_R moves
// 16*T(i) bytes per lattice, 1.3 MB at i = 399, n = 400).
#include "../../include/b200hh.h"
#include "tma.cuh"
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <algorithm>
#include <math_constants.h>
#include <string>
#include <utility>
#include <vector>

namespace {

constexpr unsigned FULLM = 0xffffffffu;
constexpr int HW = 4;  // warps per CTA
thread_local std::string g_err;
#define CKH(call)                                                                                  \
  do                                                                                               \
  {                                                                                                \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
    {                                                                                              \
      g_err = std::string(#call) + ": " + cudaGetErrorString(e_);                                  \
      return B200HH_ECUDA;                                                                         \
    }                                                                                              \
  } while (0)

enum { HM_NKR = 0, HM_NKC = 1, HM_UPDATED = 2, HM_STRIDE = 4 };

struct HBatch
{
  int B, d, n, ldb, row_expo_en, keep_hist;
  int64_t *b;
  double *bf, *R, *V, *sigma, *nsb, *hist;
  int *row_expo, *irs, *meta, *hslot;
  long *ensb;
};

// which matrices a kernel instantiation updates next to b (a template parameter, chosen at launch from the handle)
enum { HT_NONE = 0, HT_U = 1, HT_UINV = 2 };

struct HView
{
  int d, n, ldb, row_expo_en, keep_hist;
  int64_t *b;
  double *bf, *R, *V, *sigma, *nsb, *hist;
  int *row_expo, *irs, *meta, *hslot;
  long *ensb;
};

// B200HH_TRANSFORM / B200HH_INV_TRANSFORM: U and U^-T, dense d x d per lattice (nullptr unless the flags ask).  They are
// the LAST kernel argument of hk_size_reduce, hk_swap and hk_hlll rather than fields of HBatch: a bigger HBatch moves
// the arguments behind it and changes how the compiler reads the struct (past 128 bytes it is no longer taken apart into
// registers), so the instantiations without a transform would no longer compile to the code they had before U existed.
// It travels down by value (a reference to it also changed their code).
struct HTr
{
  int64_t *u, *uinvt;
};

// U and U^-T of the calling warp's lattice (both nullptr when TR == HT_NONE)
template <int TR> __device__ inline HTr htr(const HBatch &S, HTr T)
{
  HTr t{nullptr, nullptr};
  if (TR != HT_NONE)
  {
    const size_t l = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), dd = (size_t)S.d * S.d;
    t.u = T.u + l * dd;
    if (TR == HT_UINV)
      t.uinvt = T.uinvt + l * dd;
  }
  return t;
}

__device__ inline HView hview(const HBatch &S, int l)
{
  HView v;
  v.d = S.d, v.n = S.n, v.ldb = S.ldb, v.row_expo_en = S.row_expo_en, v.keep_hist = S.keep_hist;
  const size_t dn = (size_t)S.d * S.n;
  v.b        = S.b + (size_t)l * S.d * S.ldb;
  v.bf       = S.bf + l * dn;
  v.R        = S.R + l * dn;
  v.V        = S.V + l * dn;
  v.sigma    = S.sigma + (size_t)l * S.d;
  v.nsb      = S.nsb + (size_t)l * S.d;
  v.ensb     = S.ensb + (size_t)l * S.d;
  v.hist     = S.keep_hist ? S.hist + (size_t)l * dn * S.n : nullptr;
  v.row_expo = S.row_expo + (size_t)l * S.d;
  v.irs      = S.irs + (size_t)l * S.d;
  v.hslot    = S.hslot + (size_t)l * S.d;
  v.meta     = S.meta + (size_t)l * HM_STRIDE;
  return v;
}

__device__ inline bool hsetup(const HBatch &S, HView &v, double *&sR, double *&sP, int &lane)
{
  extern __shared__ __align__(16) double smem[];
  const int w = threadIdx.x >> 5;
  lane        = threadIdx.x & 31;
  const int l = blockIdx.x * (blockDim.x >> 5) + w;
  const size_t npad = (size_t)(S.n + 1) & ~(size_t)1;
  sR = smem + (size_t)w * 2 * npad;
  sP = sR + npad;
  if (l >= S.B)
    return false;
  v = hview(S, l);
  return true;
}

// ascending chain over products already in shared memory: r = p[beg]; r += p[k] ... (numvect.h:385-395), lane 0, result
// broadcast.  The products themselves were formed one per lane (each a correctly rounded multiply).
__device__ inline double chain_sum(const double *p, int beg, int end, int lane)
{
  // (a register-chunked variant — loads fetched 8 ahead of the dependent adds — was slower: the kernel is bound by how
  // many warps fit an SM, and the extra registers halved that)
  double r = 0.0;
  if (lane == 0)
  {
    r = p[beg];
    for (int k = beg + 1; k < end; k++)
      r = __dadd_rn(r, p[k]);
  }
  return __shfl_sync(FULLM, r, 0);
}

// refresh_R_bf(i), householder.cpp:186-245
__device__ inline void w_refresh_R_bf(const HView &v, int i, double *sP, int lane)
{
  const int n = v.n;
  int nc      = max(v.meta[HM_NKC], v.irs[i]);
  __syncwarp();
  if (lane == 0)
    v.meta[HM_NKC] = nc;
  const int64_t *brow = v.b + (size_t)i * v.ldb;
  double *bfr = v.bf + (size_t)i * n, *Rr = v.R + (size_t)i * n;
  int mx = 0;
  if (v.row_expo_en)
  {
    mx = INT_MIN;
    for (int c = lane; c < nc; c += 32)
    {
      int e;
      (void)frexp((double)brow[c], &e);
      mx = max(mx, e);
    }
    for (int o = 16; o; o >>= 1)
      mx = max(mx, __shfl_xor_sync(FULLM, mx, o));
  }
  for (int c = lane; c < n; c += 32)
  {
    double f = 0.0;
    if (c < nc)
    {
      if (v.row_expo_en)
      {
        int e;
        const double m = frexp((double)brow[c], &e);
        f              = ldexp(m, e - mx);
      }
      else
        f = (double)brow[c];
    }
    bfr[c] = f;
    Rr[c]  = f;
    if (c < nc)
      sP[c] = __dmul_rn(f, f);
  }
  __syncwarp();
  const double ns = chain_sum(sP, 0, nc, lane);  // norm_square_b_row, householder.h:538-551
  if (lane == 0)
  {
    if (v.row_expo_en)
      v.row_expo[i] = mx;
    v.nsb[i]  = ns;
    v.ensb[i] = v.row_expo_en ? 2L * mx : 0L;
  }
  __syncwarp();
}

// refresh_R(i), householder.cpp:247-261
__device__ inline void w_refresh_R(const HView &v, int i, int lane)
{
  const int n = v.n, nc = v.meta[HM_NKC];
  const double *bfr = v.bf + (size_t)i * n;
  double *Rr        = v.R + (size_t)i * n;
  for (int c = lane; c < n; c += 32)
    Rr[c] = (c < nc) ? bfr[c] : 0.0;
  __syncwarp();
}

// update_R_last(i), householder.cpp:27-146 (default branch, no precomputed inverse)
__device__ inline void w_update_R_last(const HView &v, int i, double *sP, int lane)
{
  const int n = v.n;
  double *Rr = v.R + (size_t)i * n, *Vr = v.V + (size_t)i * n;
  const double rii = Rr[i];
  const double sg  = (rii < 0) ? -1.0 : 1.0;
  double f3        = 0.0;
  if (i + 1 < n)
  {
    for (int k = i + 1 + lane; k < n; k += 32)
      sP[k] = __dmul_rn(Rr[k], Rr[k]);
    __syncwarp();
    f3 = chain_sum(sP, i + 1, n, lane);
  }
  double f1 = __dadd_rn(__dmul_rn(rii, rii), f3);
  if (f1 != 0.0)
  {
    const double f2 = sqrt(f1);  // IEEE sqrt (correctly rounded, as ::sqrt)
    double f0       = __dmul_rn(sg, f2);
    f1              = __dadd_rn(rii, f0);
    f3              = -f3;
    f3              = __ddiv_rn(f3, f1);
    if (f3 != 0.0)
    {
      f0 = -f0;
      f0 = __dmul_rn(f0, f3);
      f0 = sqrt(f0);
      for (int k = i + 1 + lane; k < n; k += 32)
        Vr[k] = __ddiv_rn(Rr[k], f0);
      if (lane == 0)
      {
        Vr[i] = __ddiv_rn(f3, f0);
        Rr[i] = f2;
      }
    }
    else
    {
      for (int k = i + 1 + lane; k < n; k += 32)
        Vr[k] = 0.0;
      if (lane == 0)
      {
        Vr[i] = 0.0;
        if (rii < 0)
          Rr[i] = -rii;
      }
    }
  }
  else
  {
    for (int k = i + 1 + lane; k < n; k += 32)
      Vr[k] = 0.0;
    if (lane == 0)
    {
      Rr[i] = 0.0;
      Vr[i] = 0.0;
    }
  }
  if (lane == 0)
  {
    v.sigma[i] = sg;
    v.meta[HM_NKR] += 1;
  }
  __syncwarp();
}

// update_R(i, last_j), householder.cpp:151-184.  NPL = elements of a row each lane owns (n <= 32*NPL): the lane's
// slice of V_j lives in registers, and the slice of V_{j+1} is requested BEFORE the serial summation of reflection j,
// so the HBM latency of the next row hides behind the ordered chain of the current one.
template <int NPL>
__device__ inline void w_update_R(const HView &v, int i, int last_j, double *sR, double *sP, int lane)
{
  const int n = v.n;
  if (!v.meta[HM_UPDATED])
  {
    double *Rr = v.R + (size_t)i * n;
    for (int k = lane; k < n; k += 32)
      sR[k] = Rr[k];
    __syncwarp();
    double *hrow = v.keep_hist ? v.hist + (size_t)v.hslot[i] * n * n : nullptr;
    double vk[NPL], vn[NPL];
    if (i > 0)
    {
#pragma unroll
      for (int u = 0; u < NPL; u++)
      {
        const int k = 32 * u + lane;  // row 0 starts at column 0
        vk[u]       = (k < n) ? v.V[k] : 0.0;
      }
    }
    for (int j = 0; j < i; j++)
    {
      // lane's columns of reflection j: k = kb + 32u + lane, kb = j rounded down to a multiple of 32
      const int kb = j & ~31;
      if (j + 1 < i)
      {
        const double *Vn = v.V + (size_t)(j + 1) * n;
        const int kbn    = (j + 1) & ~31;
#pragma unroll
        for (int u = 0; u < NPL; u++)
        {
          const int k = kbn + 32 * u + lane;
          vn[u]       = (k >= j + 1 && k < n) ? Vn[k] : 0.0;
        }
      }
#pragma unroll
      for (int u = 0; u < NPL; u++)
      {
        const int k = kb + 32 * u + lane;
        if (k >= j && k < n)
          sP[k] = __dmul_rn(vk[u], sR[k]);
      }
      __syncwarp();
      double f0 = chain_sum(sP, j, n, lane);
      f0        = -f0;
#pragma unroll
      for (int u = 0; u < NPL; u++)
      {
        const int k = kb + 32 * u + lane;
        if (k >= j && k < n)
        {
          double r = __dadd_rn(sR[k], __dmul_rn(vk[u], f0));
          if (k == j)
            r = __dmul_rn(v.sigma[j], r);
          sR[k] = r;
          if (hrow)
            hrow[(size_t)j * n + k] = r;  // R_history[i][j][k] = R(i,k), k >= j
        }
      }
      __syncwarp();
#pragma unroll
      for (int u = 0; u < NPL; u++)
        vk[u] = vn[u];
    }
    for (int k = lane; k < n; k += 32)
      Rr[k] = sR[k];
    __syncwarp();
    if (last_j)
      w_update_R_last(v, i, sP, lane);
  }
}

__device__ inline long hfexpo(double x) { return (long)ilogb(x) + 1; }

// row a += (x * 2^expo) * row c of a dense d x d int64 matrix, all d columns, wrapping: Z_NR<long>'s addmul_si and
// addmul_si_2exp as row_add / row_sub / row_addmul_si / row_addmul_si_2exp apply them to u and u_inv_t
// (householder.cpp:455-520: no n_known_cols bound there)
__device__ inline void w_mat_addmul(int64_t *m, int d, int a, int c, unsigned long long x, long expo, int lane)
{
  unsigned long long *ra = (unsigned long long *)(m + (size_t)a * d);
  const unsigned long long *rc = (const unsigned long long *)(m + (size_t)c * d);
  for (int col = lane; col < d; col += 32)
  {
    unsigned long long t = rc[col] * x;
    if (expo)
      t = expo >= 64 ? 0ull : (t << expo);
    ra[col] += t;
  }
}

// size_reduce(k, end, start), householder.cpp:403-451 with row_addmul_we, :522-559.  TR >= HT_U: U[k] += lx 2^expo U[i];
// TR == HT_UINV also U^-T[i] -= lx 2^expo U^-T[k], with the lx and expo of b's update.
template <int TR>
__device__ inline bool w_size_reduce(const HView &v, HTr t, int k, int sr_end, int sr_start, int lane)
{
  const int n = v.n, nc = v.meta[HM_NKC];
  double *Rk          = v.R + (size_t)k * n;
  unsigned long long *bk = (unsigned long long *)(v.b + (size_t)k * v.ldb);
  bool reduced = false;
  for (int i = sr_end - 1; i >= sr_start; i--)
  {
    const double *Ri = v.R + (size_t)i * n;
    double f         = __ddiv_rn(Rk[i], Ri[i]);
    const long de    = (long)(v.row_expo[k] - v.row_expo[i]);
    if (!(hfexpo(f) + de >= 53))
      f = ldexp(rint(ldexp(f, (int)de)), (int)-de);  // rnd_we, nr_FP_d.inl:226-233
    f = -f;
    if (f != 0.0)
    {
      long expo = 0;
      const long e = hfexpo(f) + de - 63;  // get_si_exp_we, nr_FP_d.inl:46-53
      expo         = e > 0 ? e : 0;
      const unsigned long long lx = (unsigned long long)(long)ldexp(f, (int)(de - expo));
      const unsigned long long *bi = (const unsigned long long *)(v.b + (size_t)i * v.ldb);
      for (int c = lane; c < nc; c += 32)
      {
        unsigned long long t = bi[c] * lx;
        if (expo)
          t = expo >= 64 ? 0ull : (t << expo);
        bk[c] += t;
      }
      if (TR >= HT_U)
        w_mat_addmul(t.u, v.d, k, i, lx, expo, lane);
      if (TR == HT_UINV)
        w_mat_addmul(t.uinvt, v.d, i, k, 0ull - lx, expo, lane);
      for (int c = lane; c < i; c += 32)
      {
        if (f == 1.0)
          Rk[c] = __dadd_rn(Rk[c], Ri[c]);
        else if (f == -1.0)
          Rk[c] = __dsub_rn(Rk[c], Ri[c]);
        else
          Rk[c] = __dadd_rn(Rk[c], __dmul_rn(Ri[c], f));
      }
      reduced = true;
      __syncwarp();
    }
  }
  if (reduced && lane == 0 && k < v.meta[HM_NKR])
    v.meta[HM_NKR] = k;  // invalidate_row(k)
  __syncwarp();
  return reduced;
}

// ---- kernels ---------------------------------------------------------------------------------------------------
__global__ void hk_init(HBatch S)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (!hsetup(S, v, sR, sP, lane))
    return;
  if (lane < HM_STRIDE)
    v.meta[lane] = 0;
  for (int i = 0; i < v.d; i++)
  {
    int last = 0;
    for (int c = lane; c < v.n; c += 32)
      if (v.b[(size_t)i * v.ldb + c] != 0)
        last = c + 1;
    for (int o = 16; o; o >>= 1)
      last = max(last, __shfl_xor_sync(FULLM, last, o));
    if (lane == 0)
    {
      v.irs[i]      = max(last, 1);
      v.row_expo[i] = 0;
      v.hslot[i]    = i;
      v.sigma[i]    = 0.0;
      v.nsb[i]      = 0.0;
      v.ensb[i]     = 0;
    }
  }
}

__global__ void hk_pack_b(HBatch S, const int64_t *src, int dir)
{
  const int l      = blockIdx.y;
  int64_t *b       = S.b + (size_t)l * S.d * S.ldb;
  const size_t tot = (size_t)S.d * S.n;
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < tot; t += (size_t)gridDim.x * blockDim.x)
  {
    const int i = (int)(t / S.n), c = (int)(t % S.n);
    if (dir == 0)
      b[(size_t)i * S.ldb + c] = src[(size_t)l * tot + t];
    else
      ((int64_t *)src)[(size_t)l * tot + t] = b[(size_t)i * S.ldb + c];
  }
}

__global__ void hk_refresh_R_bf(HBatch S, int i)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (hsetup(S, v, sR, sP, lane))
    w_refresh_R_bf(v, i, sP, lane);
}
__global__ void hk_refresh_R(HBatch S, int i)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (hsetup(S, v, sR, sP, lane))
    w_refresh_R(v, i, lane);
}
template <int NPL> __global__ void hk_update_R(HBatch S, int i, int last_j)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (hsetup(S, v, sR, sP, lane))
    w_update_R<NPL>(v, i, last_j, sR, sP, lane);
}

// the widest NPL instantiation bounds the row width update_R and hlll accept
static_assert((B200HH_MAX_N + 31) / 32 + 1 <= 32, "B200HH_MAX_N needs more than 32 elements per lane");

static void launch_update_R(const HBatch &S, int grid, size_t smem, cudaStream_t st, int i, int last_j)
{
  // a lane's slice of a row must fit NPL registers even when the row starts in the middle of a 32-column group
  const int need = (S.n + 31) / 32 + 1;
  if (need <= 4)
    hk_update_R<4><<<grid, HW * 32, smem, st>>>(S, i, last_j);
  else if (need <= 8)
    hk_update_R<8><<<grid, HW * 32, smem, st>>>(S, i, last_j);
  else if (need <= 14)
    hk_update_R<14><<<grid, HW * 32, smem, st>>>(S, i, last_j);
  else
    hk_update_R<32><<<grid, HW * 32, smem, st>>>(S, i, last_j);
}
__global__ void hk_update_R_last(HBatch S, int i)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (hsetup(S, v, sR, sP, lane))
    w_update_R_last(v, i, sP, lane);
}
template <int TR> __global__ void hk_size_reduce(HBatch S, int k, int e, int st, int *reduced, HTr T)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (!hsetup(S, v, sR, sP, lane))
    return;
  const bool r = w_size_reduce<TR>(v, htr<TR>(S, T), k, e, st, lane);
  if (reduced && lane == 0)
    reduced[blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)] = r ? 1 : 0;
}
// rows i and j of a dense d x d int64 matrix
__device__ inline void w_mat_swap(int64_t *m, int d, int i, int j, int lane)
{
  for (int c = lane; c < d; c += 32)
  {
    const int64_t t    = m[(size_t)i * d + c];
    m[(size_t)i * d + c] = m[(size_t)j * d + c];
    m[(size_t)j * d + c] = t;
  }
}

// swap(i, j), householder.cpp:372-398, with rows i and j of U (TR >= HT_U) and of U^-T (TR == HT_UINV)
template <int TR>
__device__ inline void w_swap(const HView &v, HTr t, int i, int j, int lane)
{
  if (lane == 0 && i < v.meta[HM_NKR])
    v.meta[HM_NKR] = i;  // invalidate_row(i)
  for (int c = lane; c < v.n; c += 32)
  {
    const int64_t t = v.b[(size_t)i * v.ldb + c];
    v.b[(size_t)i * v.ldb + c] = v.b[(size_t)j * v.ldb + c];
    v.b[(size_t)j * v.ldb + c] = t;
    const double f = v.bf[(size_t)i * v.n + c];
    v.bf[(size_t)i * v.n + c] = v.bf[(size_t)j * v.n + c];
    v.bf[(size_t)j * v.n + c] = f;
  }
  if (TR >= HT_U)
    w_mat_swap(t.u, v.d, i, j, lane);
  if (TR == HT_UINV)
    w_mat_swap(t.uinvt, v.d, i, j, lane);
  if (lane == 0)
  {
    double t = v.sigma[i];
    v.sigma[i] = v.sigma[j], v.sigma[j] = t;
    if (v.row_expo_en)
    {
      int e = v.row_expo[i];
      v.row_expo[i] = v.row_expo[j], v.row_expo[j] = e;
    }
    int q = v.irs[i];
    v.irs[i] = v.irs[j], v.irs[j] = q;
    q = v.hslot[i];
    v.hslot[i] = v.hslot[j], v.hslot[j] = q;  // iter_swap(R_history.begin()+i, +j): pointer swap
    t = v.nsb[i];
    v.nsb[i] = v.nsb[j], v.nsb[j] = t;
    long le = v.ensb[i];
    v.ensb[i] = v.ensb[j], v.ensb[j] = le;
  }
  __syncwarp();
}
template <int TR> __global__ void hk_swap(HBatch S, int i, int j, HTr T)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (hsetup(S, v, sR, sP, lane))
    w_swap<TR>(v, htr<TR>(S, T), i, j, lane);
}
// recover_R(i), householder.h:597-608
__device__ inline void w_recover_R(const HView &v, int i, int lane)
{
  const int n = v.n;
  const double *hrow = v.hist + (size_t)v.hslot[i] * n * n;
  double *Rr = v.R + (size_t)i * n;
  for (int k = lane; k < n; k += 32)
    Rr[k] = (k < i - 1) ? hrow[(size_t)k * n + k] : hrow[(size_t)(i - 1) * n + k];
  if (lane == 0)
    v.meta[HM_UPDATED] = 1;
  __syncwarp();
}
__global__ void hk_recover_R(HBatch S, int i)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (hsetup(S, v, sR, sP, lane))
    w_recover_R(v, i, lane);
}

// ---- HLLLReduction::hlll(), hlll.cpp:25-171, whole loop on the device: one warp per lattice -------------------------
struct HlllArgs
{
  double delta, theta;
  double *dR, *eR, *prevR;  // B x d each
  int *prevE;               // B x d
  int *status;              // B
  unsigned long long *iters;  // B (loop iterations, diagnostics)
  unsigned long long max_iter;
};

// size_reduction(kappa, kappa, 0), hlll.cpp:262-354 (default branch: approx = 0.1)
template <int NPL, int TR>
__device__ inline void w_hlll_size_reduction(const HView &v, HTr t, int kappa, double *sR, double *sP, int lane)
{
  bool prev_not_stop = true;
  w_update_R<NPL>(v, kappa, 0, sR, sP, lane);
  __syncwarp();
  if (lane == 0)
    v.meta[HM_UPDATED] = 0;  // set_updated_R_false(), hlll.cpp:322
  __syncwarp();
  for (;;)
  {
    if (!w_size_reduce<TR>(v, t, kappa, kappa, 0, lane))
      return;
    const double t    = v.nsb[kappa];
    const long expo0  = v.ensb[kappa];
    __syncwarp();
    w_refresh_R_bf(v, kappa, sP, lane);
    const double f1   = v.nsb[kappa];
    const long expo1  = v.ensb[kappa];
    double f0         = __dmul_rn(0.1, t);
    f0                = ldexp(f0, (int)(expo0 - expo1));
    const bool not_stop = (f1 <= f0);
    w_update_R<NPL>(v, kappa, 0, sR, sP, lane);
    if (prev_not_stop || not_stop)
      prev_not_stop = not_stop;
    else
      return;
  }
}

template <int NPL, int TR>
__device__ inline int w_hlll(const HView &v, HTr t, const HlllArgs &A, int l, double *sR, double *sP, int lane)
{
  const int d = v.d, n = v.n;
  double *dR = A.dR + (size_t)l * d, *eR = A.eR + (size_t)l * d, *pR = A.prevR + (size_t)l * d;
  int *pE = A.prevE + (size_t)l * d;
  // compute_dR / compute_eR, hlll.h:147-159 (eR is delta * R(k,k) in the reference, and here)
  auto compute_dR_eR = [&](int k) {
    const double rkk = v.R[(size_t)k * n + k];
    if (lane == 0)
    {
      dR[k] = __dmul_rn(A.delta, __dmul_rn(rkk, rkk));
      eR[k] = __dmul_rn(A.delta, rkk);
    }
    __syncwarp();
  };
  w_refresh_R_bf(v, 0, sP, lane);
  w_update_R_last(v, 0, sP, lane);
  compute_dR_eR(0);
  if (d < 2)
    return 0;
  int k = 1, k_max = 1, prev_k = -1;
  w_refresh_R_bf(v, 1, sP, lane);
  unsigned long long it = 0;
  int status = -1;
  for (;;)
  {
    if (++it > A.max_iter)
    {
      status = 9;  // RED_HLLL_FAILURE: iteration guard (the reference has none; protects the device from a livelock)
      break;
    }
    w_hlll_size_reduction<NPL, TR>(v, t, k, sR, sP, lane);
    // verify_size_reduction(k), hlll.cpp:373-478 (default branch)
    const double *Rk = v.R + (size_t)k * n;
    {
      for (int c = k + lane; c < n; c += 32)
        sP[c] = __dmul_rn(Rk[c], Rk[c]);
      __syncwarp();
      double f1 = (n > k) ? sqrt(chain_sum(sP, k, n, lane)) : 0.0;  // norm_R_row(k, k, n), householder.h:572-588
      f1        = __dmul_rn(f1, A.theta);
      const int expo0 = v.row_expo[k];
      bool bad = false;
      for (int i = lane; i < k; i += 32)
      {
        const double f0 = fabs(Rk[i]);
        const double f2 = __dadd_rn(f1, ldexp(eR[i], v.row_expo[i] - expo0));
        bad |= (f0 > f2);
      }
      __syncwarp();
      if (__any_sync(FULLM, bad))
      {
        status = 11;  // RED_HLLL_SR_FAILURE
        break;
      }
    }
    // lovasz_test(k), hlll.cpp:173-236
    bool lov;
    {
      double f1 = 0.0;
      if (k - 1 > 0)
      {
        for (int c = lane; c < k - 1; c += 32)
          sP[c] = __dmul_rn(Rk[c], Rk[c]);
        __syncwarp();
        f1 = chain_sum(sP, 0, k - 1, lane);  // norm_square_R_row(k, 0, k-1), householder.h:554-568
      }
      f1 = __dsub_rn(v.nsb[k], f1);
      const long expo1 = v.row_expo_en ? 2L * v.row_expo[k] : 0L;
      f1  = ldexp(f1, (int)(expo1 - 2L * v.row_expo[k - 1]));
      lov = (dR[k - 1] <= f1);
      __syncwarp();
    }
    if (lov)
    {
      w_update_R_last(v, k, sP, lane);
      compute_dR_eR(k);
      const double rkk = Rk[k];
      const int ek     = v.row_expo[k];
      if (prev_k == k + 1)
      {
        const double f1 = ldexp(pR[k], pE[k] - ek);
        if (rkk > f1)
        {
          status = 10;  // RED_HLLL_NORM_FAILURE
          break;
        }
      }
      prev_k = k;
      __syncwarp();
      if (lane == 0)
        pR[k] = rkk, pE[k] = ek;
      __syncwarp();
      k++;
      if (k < d)
      {
        if (k > k_max)
        {
          k_max = k;
          w_refresh_R_bf(v, k, sP, lane);
        }
        else
          w_refresh_R(v, k, lane);
      }
      else
      {
        status = 0;
        break;
      }
    }
    else
    {
      w_swap<TR>(v, t, k - 1, k, lane);
      prev_k = k;
      if (k - 1 == 0)
      {
        w_refresh_R(v, 0, lane);
        w_update_R_last(v, 0, sP, lane);
        compute_dR_eR(0);
        w_refresh_R(v, 1, lane);
        k = 1;
      }
      else
      {
        k--;
        w_recover_R(v, k, lane);
      }
    }
  }
  if (lane == 0)
    A.iters[l] = it;
  return status;
}

template <int NPL, int TR> __global__ void hk_hlll(HBatch S, HlllArgs A, HTr T)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (!hsetup(S, v, sR, sP, lane))
    return;
  const int l  = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int st = w_hlll<NPL, TR>(v, htr<TR>(S, T), A, l, sR, sP, lane);
  if (lane == 0)
    A.status[l] = st;
}
// U (and U^-T) = identity on every lattice (the buffers were zeroed)
__global__ void hk_identity(int64_t *m, int d)
{
  int64_t *ml = m + (size_t)blockIdx.x * d * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x)
    ml[(size_t)i * d + i] = 1;
}

__global__ void hk_set_updated(HBatch S, int val)
{
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l < S.B)
    S.meta[(size_t)l * HM_STRIDE + HM_UPDATED] = val;
}

}  // namespace

// =====================================================================================================================
// update_R with 32 lattices per warp: lane = lattice (batched calls, history off).
//
// hk_update_R (one warp per lattice) forms every dot product V_j . R_i as per-lane products followed by ONE lane adding
// them in the reference's order: that single-lane chain takes a full warp issue slot per add and the kernel is issue-bound
// far below the HBM peak.  With one LATTICE per lane the 32 chains of a group of
// lattices advance in one instruction.  The state stays row-major per lattice (hview): the transposition is done by the
// TMA unit — a tensor map over V (and R) seen as {flat d*n elements} x {lattice} delivers boxes of 16 consecutive elements
// x 32 lattices (128-byte segments of 32 different rows of HBM) into shared memory with the 128-byte swizzle, which lane r
// reads back as 8 conflict-free LDS.128 of its own row.  R_i of the 32 lattices lives in shared memory as [k][lane].
// Reflection j's update  R[k] += V_j[k] * f_j  and reflection j+1's dot product  sum_k V_{j+1}[k] * R[k]  run fused in one
// sweep over k (the dot product of j+1 only needs R[k] after the update of j at the same k), so V is streamed once from
// HBM and once more from L2, and every element costs one dependent DADD (8 cycles) instead of two passes.
// Operation order per lattice is exactly w_update_R's (householder.cpp:151-184): bit-identical R.
constexpr int X_K       = 16;                 // elements of a row per chunk
constexpr int X_HALF_DBL = 32 * X_K;          // one box: 32 lattices x 16 doubles (4 KB)
constexpr int X_STAGE_DBL = 2 * X_HALF_DBL;   // A (V_j) + B (V_{j+1})

struct XMaps
{
  CUtensorMap V, R;  // {d*n, B}, box {16, 32}, SWIZZLE_128B
};

// lane r's 16 elements of a swizzled box: element k at row r, 16-byte column (k >> 1) ^ (r & 7).  (Dense 256-byte rows
// read back with a per-lane skew were tried too — half the TMA row requests — and were slower.)
__device__ inline void x_read_box(const double *box, int lane, double (&v)[X_K])
{
  const char *row = (const char *)box + lane * 128;
#pragma unroll
  for (int c = 0; c < 8; c++)
  {
    const double2 t = *(const double2 *)(row + ((c ^ (lane & 7)) << 4));
    v[2 * c] = t.x, v[2 * c + 1] = t.y;
  }
}

// ---- one CTA per group of 32 lattices = 1 producer warp + XM_NA update warps + 1 chain warp ----
// A single warp doing the whole sweep is bound by its own issue rate.  Here the sweep over k of pass q (reflection j = q - 2) is a pipeline of three
// roles connected by mbarriers:
//   producer  lane 0 of warp 0 walks the chunk sequence and issues the TMA boxes of chunk g into stage g % XM_S as soon
//             as the stage is empty;
//   update    warp 1 + (g % XM_NA) takes chunk g: R[k] += V_j[k] * f_j (times sigma_j at k = j), writes R back to shared
//             memory and the products  p[k] = V_{j+1}[k] * R[k]  into slot g % XM_PR of a product ring;
//   chain     the last warp consumes the product slots IN ORDER and adds them — one dependent DADD per element, the only
//             serial work left — and at the end of a pass publishes f_{j+1} = -sum for the update warps of the next pass.
// Every lattice (lane) sees exactly w_update_R's operation order (householder.cpp:151-184): bit-identical R.
constexpr int XM_NA = 6;   // update warps
constexpr int XM_S  = 8;   // TMA stages (A | B boxes, 8 KB each)
constexpr int XM_PR = 8;   // product slots (4 KB each)
constexpr int XM_WARPS = XM_NA + 2;
static_assert(XM_S == XM_PR, "an update warp relies on 'product slot free' implying 'TMA stage consumed'");
// ... and the product ring must not be shorter than the number of update warps: a warp's previous chunk is XM_NA behind
// its current one, so with XM_PR >= XM_NA the chain warp is never two rounds of a slot behind a waiting warp — a parity
// wait can only tell adjacent phases apart.  (XM_S = 13 / XM_PR = 4 — more bytes in flight, what bounds this kernel —
// passed the small parity tests and hung at n = 400 for exactly this reason; growing the ring needs XM_NA <= XM_PR <= XM_S and the shared memory for it.)
static_assert(XM_PR >= XM_NA, "product ring shorter than the number of update warps");

struct XmCtl
{
  unsigned long long full[XM_S], empty[XM_S], pready[XM_PR], pfree[XM_PR];
  // number of passes the chain warp has closed.  A plain counter, not an mbarrier: an update warp without a chunk in some
  // passes (late passes have fewer chunks than there are update warps) would have to skip phases, and a parity wait can
  // only tell adjacent phases apart.
  int pass_done;
  int pad;
};
__device__ inline void xm_store_release(int *p, int v)
{
  asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"(tma_smem_u32(p)), "r"(v) : "memory");
}
__device__ inline int xm_load_acquire(const int *p)
{
  int v;
  asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(v) : "r"(tma_smem_u32(p)) : "memory");
  return v;
}

// chunk sequence in pass-major order: pass q = 0 loads R_i (k0 = 0, 16, ...); pass q >= 1 is reflection j = q - 2 (j = -1:
// only the dot product of reflection 0), k0 from (max(j,0) & ~15) in steps of 16.  Passes 0 .. i + 1.
struct XmIter
{
  int q, k0;
  __device__ void start() { q = 0, k0 = 0; }
  __device__ bool done(int i) const { return q > i + 1; }
  __device__ bool last_of_pass(int n) const { return k0 + X_K >= n; }
  __device__ void next(int n)
  {
    k0 += X_K;
    if (k0 >= n)
    {
      q++;
      k0 = max(q - 2, 0) & ~(X_K - 1);
    }
  }
};

__global__ void __launch_bounds__(XM_WARPS * 32, 1) hk_update_R_x32(HBatch S, int i, const __grid_constant__ XMaps M)
{
  extern __shared__ unsigned char x_raw[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, n = S.n;
  const int l0 = blockIdx.x * 32, l = l0 + lane, lc = min(l, S.B - 1);
  double *ring = (double *)(((size_t)x_raw + 1023) & ~(size_t)1023);   // XM_S stages of A | B boxes
  double *prod = ring + (size_t)XM_S * X_STAGE_DBL;                    // XM_PR slots of [u][lane]
  double *Rk   = prod + (size_t)XM_PR * X_HALF_DBL;                    // [k][lane]
  const int npad = (n + X_K - 1) & ~(X_K - 1);
  double *fbuf = Rk + (size_t)npad * 32;                               // [2][lane]
  XmCtl *C     = (XmCtl *)(fbuf + 64);
  unsigned *sigbits = (unsigned *)(C + 1);                             // [j]: bit l set <=> sigma_j of lattice l is -1
  // sigma_j is a sign (householder.cpp:40: +-1.0): all reflections' signs of the 32 lattices fit 4 i bytes, so no pass
  // waits on a global load for it
  for (int j = w; j < i; j += XM_WARPS)
  {
    const unsigned neg = __ballot_sync(FULLM, S.sigma[(size_t)lc * S.d + j] < 0.0);
    if (lane == 0)
      sigbits[j] = neg;
  }
  if (threadIdx.x == 0)
  {
    for (int q = 0; q < XM_S; q++)
    {
      tma_mbar_init<1>(&C->full[q]);
      tma_mbar_init<1>(&C->empty[q]);
    }
    for (int q = 0; q < XM_PR; q++)
    {
      tma_mbar_init<1>(&C->pready[q]);
      tma_mbar_init<1>(&C->pfree[q]);
    }
    C->pass_done = 0;
    tma_fence_mbar_init();
  }
  __syncthreads();

  if (w == 0)
  {
    // ---- producer: lane p < XM_S owns stage p and issues the chunks g = p, p + XM_S, ... (one thread walking the whole
    // sequence is slowed by the address arithmetic and barrier operations of a lone thread and starved the pipeline;
    // eight lanes do it eight wide) ----
    if (lane < XM_S)
    {
      XmIter it;
      it.start();
      for (int q = 0; q < lane && !it.done(i); q++)
        it.next(n);
      unsigned g  = lane;
      bool active = !it.done(i);
      while (__any_sync((1u << XM_S) - 1u, active))
      {
        if (active && tma_mbar_test(&C->empty[lane], ((g / XM_S) & 1u) ^ 1u))
        {
          double *dst             = ring + (size_t)lane * X_STAGE_DBL;
          unsigned long long *bar = &C->full[lane];
          const int j             = it.q - 2;
          if (it.q == 0)
          {
            tma_mbar_expect_tx(bar, X_HALF_DBL * 8);
            tma_load_2d(dst, &M.R, i * n + it.k0, l0, bar);
          }
          else
          {
            const bool hasA = j >= 0, hasB = j + 1 < i;
            tma_mbar_expect_tx(bar, (int)(hasA + hasB) * X_HALF_DBL * 8);
            if (hasA)
              tma_load_2d(dst, &M.V, j * n + it.k0, l0, bar);
            if (hasB)
              tma_load_2d(dst + X_HALF_DBL, &M.V, (j + 1) * n + it.k0, l0, bar);
          }
          for (int q = 0; q < XM_S && !it.done(i); q++)
            it.next(n);
          g += XM_S;
          active = !it.done(i);
        }
      }
    }
  }
  else if (w <= XM_NA)
  {
    // ---- update warps ----
    const int me = w - 1;
    XmIter it;
    it.start();
    unsigned g = 0;
    int fq = 0;          // passes up to fq have had their f / their predecessor's completion observed
    double f0 = 0.0, sg = 1.0;
    for (; !it.done(i); g++, it.next(n))
    {
      if ((int)(g % XM_NA) != me)
        continue;
      const int q = it.q, j = q - 2, k0 = it.k0;
      if (q >= 1 && fq < q)
      {
        // pass q may start once the chain warp has closed pass q - 1: that orders every R[k] write of the earlier passes
        // before this warp's reads, and carries f_j (j >= 0)
        while (xm_load_acquire(&C->pass_done) < q)
          ;
        f0 = fbuf[(q & 1) * 32 + lane];
        fq = q;
        if (j >= 0)
          sg = ((sigbits[j] >> lane) & 1u) ? -1.0 : 1.0;
      }
      // the product slot first: the chain warp consumes in order, so "slot g % 8 is free" also means chunk g - 8 — the
      // previous user of this TMA stage — has landed and been consumed, and the parity wait below cannot see a stale phase
      tma_mbar_wait(&C->pfree[g % XM_PR], ((g / XM_PR) & 1u) ^ 1u);
      tma_mbar_wait(&C->full[g % XM_S], (g / XM_S) & 1u);
      const double *st = ring + (size_t)(g % XM_S) * X_STAGE_DBL;
      double *rp = Rk + (size_t)k0 * 32 + lane;
      if (q == 0)
      {
        double a[X_K];
        x_read_box(st, lane, a);
#pragma unroll
        for (int u = 0; u < X_K; u++)
          rp[u * 32] = a[u];
      }
      else
      {
        const bool hasA = j >= 0, hasB = j + 1 < i;
        double a[X_K], b[X_K], r[X_K];
        if (hasA)
          x_read_box(st, lane, a);
        if (hasB)
          x_read_box(st + X_HALF_DBL, lane, b);
        if (hasA && k0 > j && k0 + X_K <= n)
        {
#pragma unroll
          for (int u = 0; u < X_K; u++)
            r[u] = __dadd_rn(rp[u * 32], __dmul_rn(a[u], f0));
#pragma unroll
          for (int u = 0; u < X_K; u++)
            rp[u * 32] = r[u];
        }
        else
        {
#pragma unroll
          for (int u = 0; u < X_K; u++)
          {
            const int k = k0 + u;
            double t    = rp[u * 32];
            if (hasA && k >= j && k < n)
            {
              t = __dadd_rn(t, __dmul_rn(a[u], f0));
              if (k == j)
                t = __dmul_rn(sg, t);
              rp[u * 32] = t;
            }
            r[u] = t;
          }
        }
        if (hasB)
        {
          double *ps = prod + (size_t)(g % XM_PR) * X_HALF_DBL + lane;
#pragma unroll
          for (int u = 0; u < X_K; u++)
            ps[u * 32] = __dmul_rn(b[u], r[u]);
        }
      }
      __syncwarp();
      if (lane == 0)
      {
        tma_mbar_arrive(&C->pready[g % XM_PR]);
        tma_mbar_arrive(&C->empty[g % XM_S]);
      }
    }
  }
  else
  {
    // ---- chain warp ----
    XmIter it;
    it.start();
    double acc = 0.0;
    for (unsigned g = 0; !it.done(i); g++, it.next(n))
    {
      const int q = it.q, j = q - 2, k0 = it.k0;
      tma_mbar_wait(&C->pready[g % XM_PR], (g / XM_PR) & 1u);
      if (q >= 1 && j + 1 < i)
      {
        const double *ps = prod + (size_t)(g % XM_PR) * X_HALF_DBL + lane;
        double t[X_K];
#pragma unroll
        for (int u = 0; u < X_K; u++)
          t[u] = ps[u * 32];
        if (k0 > j + 1 && k0 + X_K <= n)
        {
#pragma unroll
          for (int u = 0; u < X_K; u++)
            acc = __dadd_rn(acc, t[u]);
        }
        else
        {
#pragma unroll
          for (int u = 0; u < X_K; u++)
          {
            const int k = k0 + u;
            if (k >= j + 1 && k < n)
              acc = (k == j + 1) ? t[u] : __dadd_rn(acc, t[u]);
          }
        }
      }
      __syncwarp();
      if (lane == 0)
        tma_mbar_arrive(&C->pfree[g % XM_PR]);
      if (it.last_of_pass(n))
      {
        // pass q is closed: f of reflection j + 1 (the factor of pass q + 1) is minus the dot product just accumulated
        fbuf[((q + 1) & 1) * 32 + lane] = -acc;
        __syncwarp();
        if (lane == 0)
          xm_store_release(&C->pass_done, q + 1);
      }
    }
  }
  __syncthreads();
  const bool live = l < S.B && !S.meta[(size_t)lc * HM_STRIDE + HM_UPDATED];
  if (live)
  {
    double *Rr = S.R + (size_t)l * S.d * n + (size_t)i * n;
    for (int k = w; k < n; k += XM_WARPS)
      Rr[k] = Rk[(size_t)k * 32 + lane];
  }
}

__global__ void hk_update_R_last_cond(HBatch S, int i)
{
  HView v;
  double *sR, *sP;
  int lane;
  if (hsetup(S, v, sR, sP, lane) && !v.meta[HM_UPDATED])
    w_update_R_last(v, i, sP, lane);
}

struct b200hh
{
  HBatch S;
  int device;
  cudaStream_t stream;
  size_t smem;
  int *d_red;
  double *d_hlll = nullptr;  // dR, eR, prevR: 3 x B x d
  int *d_hlll_i = nullptr;   // prevE: B x d, status: B
  unsigned long long *d_hlll_it = nullptr;
  XMaps xmaps;
  int x_state = 0;  // tensor maps of hk_update_R_x32: 0 not built, 1 ready, -1 unavailable
  int tr = HT_NONE;  // the transform template parameter of hk_size_reduce, hk_swap and hk_hlll
  HTr T{nullptr, nullptr};  // batch x d x d each
  std::vector<void *> allocs;
};

template <class T> static int hh_alloc(b200hh *h, T **p, size_t count)
{
  void *q = nullptr;
  if (cudaMalloc(&q, count * sizeof(T) + 256) != cudaSuccess)
  {
    g_err = "cudaMalloc failed";
    cudaGetLastError();
    return B200HH_ENOMEM;
  }
  h->allocs.push_back(q);
  *p = (T *)q;
  return 0;
}
static int hgrid(const b200hh *h) { return (h->S.B + HW - 1) / HW; }

// tensor maps of the lane-per-lattice kernel
static bool x_maps(b200hh *h)
{
  if (h->x_state)
    return h->x_state > 0;
  h->x_state = -1;
  const HBatch &S = h->S;
  const size_t dn = (size_t)S.d * S.n;
  if (dn % 2)
    return false;  // lattice stride must be a multiple of 16 bytes
  const cuuint64_t dims[2] = {(cuuint64_t)dn, (cuuint64_t)S.B}, str[1] = {(cuuint64_t)dn * 8};
  const cuuint32_t box[2] = {X_K, 32};
  for (int w = 0; w < 2; w++)
    if (!tma_encode_f64(w ? &h->xmaps.R : &h->xmaps.V, w ? (void *)S.R : (void *)S.V, 2, dims, str, box,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B))
      return false;
  h->x_state = 1;
  return true;
}

// the transform instantiations of the kernels that change b
template <int TR> static cudaError_t hh_kernel_attrs()
{
  const void *fns[] = {(const void *)hk_size_reduce<TR>, (const void *)hk_swap<TR>, (const void *)hk_hlll<4, TR>,
                       (const void *)hk_hlll<8, TR>, (const void *)hk_hlll<14, TR>, (const void *)hk_hlll<32, TR>};
  for (const void *f : fns)
  {
    const cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess)
      return e;
  }
  return cudaSuccess;
}

static void launch_size_reduce(const b200hh *h, int k, int e, int st)
{
  switch (h->tr)
  {
  case HT_NONE: hk_size_reduce<HT_NONE><<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, k, e, st, h->d_red, h->T); break;
  case HT_U: hk_size_reduce<HT_U><<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, k, e, st, h->d_red, h->T); break;
  default: hk_size_reduce<HT_UINV><<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, k, e, st, h->d_red, h->T); break;
  }
}

static void launch_swap(const b200hh *h, int i, int j)
{
  switch (h->tr)
  {
  case HT_NONE: hk_swap<HT_NONE><<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, i, j, h->T); break;
  case HT_U: hk_swap<HT_U><<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, i, j, h->T); break;
  default: hk_swap<HT_UINV><<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, i, j, h->T); break;
  }
}

template <int TR> static void launch_hlll_tr(const b200hh *h, const HlllArgs &A)
{
  const HBatch &S = h->S;
  const int need  = (S.n + 31) / 32 + 1;
  if (need <= 4)
    hk_hlll<4, TR><<<hgrid(h), HW * 32, h->smem, h->stream>>>(S, A, h->T);
  else if (need <= 8)
    hk_hlll<8, TR><<<hgrid(h), HW * 32, h->smem, h->stream>>>(S, A, h->T);
  else if (need <= 14)
    hk_hlll<14, TR><<<hgrid(h), HW * 32, h->smem, h->stream>>>(S, A, h->T);
  else
    hk_hlll<32, TR><<<hgrid(h), HW * 32, h->smem, h->stream>>>(S, A, h->T);
}

static void launch_update_R_h(b200hh *h, int i, int last_j)
{
  const HBatch &S = h->S;
  // B200_HH_X32=1 selects the lane-per-lattice kernel (default: one warp per lattice).  It needs a batch (32 lattices per
  // CTA), no R_history (its scattered per-lattice writes would cost more than the V stream) and R_i of 32 lattices in
  // shared memory.  It is faster than hk_update_R at one group per SM but slower at the batch bench.py times (bound by
  // the per-reflection hand-off), so it is not the default.
  const char *e     = getenv("B200_HH_X32");
  const int use_x32 = e ? atoi(e) : 0;
  const size_t npad = ((size_t)S.n + X_K - 1) & ~(size_t)(X_K - 1);
  const size_t smx  = 1024 + ((size_t)XM_S * X_STAGE_DBL + (size_t)XM_PR * X_HALF_DBL + npad * 32 + 64) * 8 + sizeof(XmCtl) + (size_t)S.d * 4;
  if (use_x32 && S.B >= 64 && !S.keep_hist && i > 0 && smx <= 227 * 1024 && (size_t)S.d * S.n < (1ull << 31) && x_maps(h))
  {
    hk_update_R_x32<<<(S.B + 31) / 32, XM_WARPS * 32, smx, h->stream>>>(S, i, h->xmaps);
    if (last_j)
      hk_update_R_last_cond<<<hgrid(h), HW * 32, h->smem, h->stream>>>(S, i);
    return;
  }
  launch_update_R(S, hgrid(h), h->smem, h->stream, i, last_j);
}

extern "C" {

const char *b200hh_last_error(void) { return g_err.c_str(); }

int b200hh_create(b200hh_t **out, int batch, int d, int n, int flags, int device, int keep_history)
{
  if (!out || batch <= 0 || d <= 0 || n <= 0)
    return B200HH_EINVAL;
  if ((flags & B200HH_INV_TRANSFORM) && !(flags & B200HH_TRANSFORM))
  {
    g_err = "b200hh_create: B200HH_INV_TRANSFORM needs B200HH_TRANSFORM (the reference updates u_inv_t only with u)";
    return B200HH_EINVAL;
  }
  int nd = 0;
  if (cudaGetDeviceCount(&nd) != cudaSuccess || nd <= device)
  {
    cudaGetLastError();
    g_err = "b200hh_create: no CUDA device (this library has no CPU fallback)";
    return B200HH_ENODEV;
  }
  CKH(cudaSetDevice(device));
  b200hh *h = new b200hh();
  h->device = device;
  HBatch &S = h->S;
  S.B = batch, S.d = d, S.n = n, S.ldb = (n + 1) & ~1, S.row_expo_en = (flags & B200HH_ROW_EXPO) ? 1 : 0;
  S.keep_hist     = keep_history ? 1 : 0;
  const size_t dn = (size_t)d * n;
  int rc          = 0;
  rc |= hh_alloc(h, &S.b, (size_t)batch * d * S.ldb);
  rc |= hh_alloc(h, &S.bf, batch * dn);
  rc |= hh_alloc(h, &S.R, batch * dn);
  rc |= hh_alloc(h, &S.V, batch * dn);
  rc |= hh_alloc(h, &S.sigma, (size_t)batch * d);
  rc |= hh_alloc(h, &S.nsb, (size_t)batch * d);
  rc |= hh_alloc(h, &S.ensb, (size_t)batch * d);
  rc |= hh_alloc(h, &S.row_expo, (size_t)batch * d);
  rc |= hh_alloc(h, &S.irs, (size_t)batch * d);
  rc |= hh_alloc(h, &S.hslot, (size_t)batch * d);
  rc |= hh_alloc(h, &S.meta, (size_t)batch * HM_STRIDE);
  rc |= hh_alloc(h, &h->d_red, (size_t)batch);
  S.hist = nullptr;
  if (!rc && keep_history)
    rc |= hh_alloc(h, &S.hist, batch * dn * n);
  const size_t dd = (size_t)batch * d * d;
  h->tr           = (flags & B200HH_INV_TRANSFORM) ? HT_UINV : (flags & B200HH_TRANSFORM) ? HT_U : HT_NONE;
  if (!rc && h->tr >= HT_U)
    rc |= hh_alloc(h, &h->T.u, dd);
  if (!rc && h->tr == HT_UINV)
    rc |= hh_alloc(h, &h->T.uinvt, dd);
  if (rc)
  {
    for (void *p : h->allocs)
      cudaFree(p);
    delete h;
    return B200HH_ENOMEM;
  }
  CKH(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  h->smem = (size_t)HW * 2 * ((n + 1) & ~1) * sizeof(double);
  const void *fns[] = {(const void *)hk_init,        (const void *)hk_refresh_R_bf, (const void *)hk_refresh_R,
                       (const void *)hk_update_R<4>, (const void *)hk_update_R<8>, (const void *)hk_update_R<14>,
                       (const void *)hk_update_R<32>, (const void *)hk_update_R_last,
                       (const void *)hk_update_R_x32, (const void *)hk_update_R_last_cond,
                       (const void *)hk_recover_R};
  for (const void *f : fns)
    CKH(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));  // process-wide: opt-in maximum, never lowered
  switch (h->tr)
  {
  case HT_NONE: CKH(hh_kernel_attrs<HT_NONE>()); break;
  case HT_U: CKH(hh_kernel_attrs<HT_U>()); break;
  default: CKH(hh_kernel_attrs<HT_UINV>()); break;
  }
  CKH(cudaMemsetAsync(S.b, 0, (size_t)batch * d * S.ldb * 8, h->stream));
  CKH(cudaMemsetAsync(S.bf, 0, batch * dn * 8, h->stream));
  CKH(cudaMemsetAsync(S.R, 0, batch * dn * 8, h->stream));
  CKH(cudaMemsetAsync(S.V, 0, batch * dn * 8, h->stream));
  CKH(cudaMemsetAsync(S.meta, 0, (size_t)batch * HM_STRIDE * 4, h->stream));
  for (int64_t *m : {h->T.u, h->T.uinvt})
    if (m)
    {
      CKH(cudaMemsetAsync(m, 0, dd * 8, h->stream));
      hk_identity<<<batch, 128, 0, h->stream>>>(m, d);
      CKH(cudaGetLastError());
    }
  CKH(cudaStreamSynchronize(h->stream));
  *out = h;
  return 0;
}

void b200hh_destroy(b200hh_t *h)
{
  if (!h)
    return;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  cudaStreamDestroy(h->stream);
  for (void *p : h->allocs)
    cudaFree(p);
  delete h;
}

int b200hh_set_basis(b200hh_t *h, const int64_t *b)
{
  if (!h || !b)
    return B200HH_EINVAL;
  CKH(cudaSetDevice(h->device));
  const size_t cnt = (size_t)h->S.B * h->S.d * h->S.n;
  int64_t *tmp     = nullptr;
  CKH(cudaMalloc(&tmp, cnt * 8));
  CKH(cudaMemcpyAsync(tmp, b, cnt * 8, cudaMemcpyHostToDevice, h->stream));
  dim3 g(32, h->S.B);
  hk_pack_b<<<g, 256, 0, h->stream>>>(h->S, tmp, 0);
  hk_init<<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S);
  CKH(cudaStreamSynchronize(h->stream));
  cudaFree(tmp);
  CKH(cudaGetLastError());
  return 0;
}

int b200hh_get_basis(b200hh_t *h, int64_t *b)
{
  if (!h || !b)
    return B200HH_EINVAL;
  CKH(cudaSetDevice(h->device));
  const size_t cnt = (size_t)h->S.B * h->S.d * h->S.n;
  int64_t *tmp     = nullptr;
  CKH(cudaMalloc(&tmp, cnt * 8));
  dim3 g(32, h->S.B);
  hk_pack_b<<<g, 256, 0, h->stream>>>(h->S, tmp, 1);
  CKH(cudaMemcpyAsync(b, tmp, cnt * 8, cudaMemcpyDeviceToHost, h->stream));
  CKH(cudaStreamSynchronize(h->stream));
  cudaFree(tmp);
  CKH(cudaGetLastError());
  return 0;
}

#define HH_CALL(cond, launch)                    \
  if (!h || !(cond))                             \
    return B200HH_EINVAL;                        \
  CKH(cudaSetDevice(h->device));                 \
  launch;                                        \
  CKH(cudaGetLastError());                       \
  return 0;

int b200hh_refresh_R_bf(b200hh_t *h, int i)
{
  HH_CALL(i >= 0 && i < h->S.d, (hk_refresh_R_bf<<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, i)))
}
int b200hh_refresh_R(b200hh_t *h, int i)
{
  HH_CALL(i >= 0 && i < h->S.d, (hk_refresh_R<<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, i)))
}
// update_R and hlll keep a lane's share of a reflection in registers: rows wider than B200HH_MAX_N do not fit
static bool width_ok(const b200hh *h, const char *fn)
{
  if (h->S.n <= B200HH_MAX_N)
    return true;
  g_err = std::string(fn) + ": n = " + std::to_string(h->S.n) + " exceeds B200HH_MAX_N = " + std::to_string(B200HH_MAX_N);
  return false;
}

int b200hh_update_R(b200hh_t *h, int i, int last_j)
{
  HH_CALL(i >= 0 && i < h->S.d && width_ok(h, "b200hh_update_R"), launch_update_R_h(h, i, last_j))
}
int b200hh_update_R_last(b200hh_t *h, int i)
{
  HH_CALL(i >= 0 && i < h->S.d, (hk_update_R_last<<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, i)))
}
int b200hh_swap(b200hh_t *h, int i, int j)
{
  HH_CALL(i >= 0 && i < j && j < h->S.d, launch_swap(h, i, j))
}
int b200hh_recover_R(b200hh_t *h, int i)
{
  HH_CALL(i >= 1 && i < h->S.d && h->S.keep_hist, (hk_recover_R<<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, i)))
}
int b200hh_set_updated_R_false(b200hh_t *h)
{
  HH_CALL(true, (hk_set_updated<<<(h->S.B + 127) / 128, 128, 0, h->stream>>>(h->S, 0)))
}

int b200hh_size_reduce(b200hh_t *h, int k, int e, int st, int *reduced)
{
  if (!h || k <= 0 || k >= h->S.d || e > k || st < 0 || st > e)
    return B200HH_EINVAL;
  CKH(cudaSetDevice(h->device));
  launch_size_reduce(h, k, e, st);
  if (reduced)
  {
    CKH(cudaMemcpyAsync(reduced, h->d_red, sizeof(int) * h->S.B, cudaMemcpyDeviceToHost, h->stream));
    CKH(cudaStreamSynchronize(h->stream));
  }
  CKH(cudaGetLastError());
  return 0;
}

// U / U^-T (batch x d x d, dense on both sides) to or from the host; a NULL pointer skips that matrix, a non-NULL one for
// a matrix the handle does not keep is refused before anything is copied
static int copy_transform(b200hh_t *h, int64_t *u, int64_t *uinvt, bool to_device)
{
  if (!h)
    return B200HH_EINVAL;
  if ((u && !h->T.u) || (uinvt && !h->T.uinvt))
  {
    g_err = u && !h->T.u ? "b200hh_set/get_transform: the handle was created without B200HH_TRANSFORM"
                         : "b200hh_set/get_transform: the handle was created without B200HH_INV_TRANSFORM";
    return B200HH_EINVAL;
  }
  CKH(cudaSetDevice(h->device));
  const size_t bytes = (size_t)h->S.B * h->S.d * h->S.d * sizeof(int64_t);
  const std::pair<int64_t *, int64_t *> mats[] = {{u, h->T.u}, {uinvt, h->T.uinvt}};
  for (const auto &m : mats)
    if (m.first)
    {
      if (to_device)
        CKH(cudaMemcpyAsync(m.second, m.first, bytes, cudaMemcpyHostToDevice, h->stream));
      else
        CKH(cudaMemcpyAsync(m.first, m.second, bytes, cudaMemcpyDeviceToHost, h->stream));
    }
  CKH(cudaStreamSynchronize(h->stream));
  CKH(cudaGetLastError());
  return 0;
}

int b200hh_set_transform(b200hh_t *h, const int64_t *u, const int64_t *u_inv_t)
{
  return copy_transform(h, (int64_t *)u, (int64_t *)u_inv_t, true);
}

int b200hh_get_transform(b200hh_t *h, int64_t *u, int64_t *u_inv_t) { return copy_transform(h, u, u_inv_t, false); }

int b200hh_get_state(b200hh_t *h, double *R, double *V, double *bf, double *sigma, double *norm_square_b,
                     int64_t *row_expo, int64_t *expo_norm_square_b, int *meta)
{
  if (!h)
    return B200HH_EINVAL;
  CKH(cudaSetDevice(h->device));
  const HBatch &S = h->S;
  const size_t dn = (size_t)S.B * S.d * S.n, bd = (size_t)S.B * S.d;
  if (R)
    CKH(cudaMemcpyAsync(R, S.R, dn * 8, cudaMemcpyDeviceToHost, h->stream));
  if (V)
    CKH(cudaMemcpyAsync(V, S.V, dn * 8, cudaMemcpyDeviceToHost, h->stream));
  if (bf)
    CKH(cudaMemcpyAsync(bf, S.bf, dn * 8, cudaMemcpyDeviceToHost, h->stream));
  if (sigma)
    CKH(cudaMemcpyAsync(sigma, S.sigma, bd * 8, cudaMemcpyDeviceToHost, h->stream));
  if (norm_square_b)
    CKH(cudaMemcpyAsync(norm_square_b, S.nsb, bd * 8, cudaMemcpyDeviceToHost, h->stream));
  if (expo_norm_square_b)
    CKH(cudaMemcpyAsync(expo_norm_square_b, S.ensb, bd * 8, cudaMemcpyDeviceToHost, h->stream));
  std::vector<int> re, m;
  if (row_expo)
  {
    re.resize(bd);
    CKH(cudaMemcpyAsync(re.data(), S.row_expo, bd * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  if (meta)
  {
    m.resize((size_t)S.B * HM_STRIDE);
    CKH(cudaMemcpyAsync(m.data(), S.meta, m.size() * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  CKH(cudaStreamSynchronize(h->stream));
  if (row_expo)
    for (size_t t = 0; t < bd; t++)
      row_expo[t] = re[t];
  if (meta)
    for (int l = 0; l < S.B; l++)
      for (int q = 0; q < 3; q++)
        meta[3 * l + q] = m[(size_t)l * HM_STRIDE + q];
  CKH(cudaGetLastError());
  return 0;
}

int b200hh_time_update_R(b200hh_t *h, int i, int reps, float *ms_update_mean)
{
  if (!h || !ms_update_mean || reps <= 0 || i < 0 || i >= h->S.d || !width_ok(h, "b200hh_time_update_R"))
    return B200HH_EINVAL;
  CKH(cudaSetDevice(h->device));
  std::vector<cudaEvent_t> ev(2 * (size_t)reps);
  for (auto &e : ev)
    CKH(cudaEventCreate(&e));
  for (int r = 0; r < reps; r++)
  {
    hk_refresh_R<<<hgrid(h), HW * 32, h->smem, h->stream>>>(h->S, i);
    CKH(cudaEventRecord(ev[2 * r], h->stream));
    launch_update_R_h(h, i, 0);
    CKH(cudaEventRecord(ev[2 * r + 1], h->stream));
  }
  CKH(cudaStreamSynchronize(h->stream));
  double tot = 0;
  for (int r = 0; r < reps; r++)
  {
    float ms = 0;
    CKH(cudaEventElapsedTime(&ms, ev[2 * r], ev[2 * r + 1]));
    tot += ms;
  }
  for (auto &e : ev)
    cudaEventDestroy(e);
  *ms_update_mean = (float)(tot / reps);
  CKH(cudaGetLastError());
  return 0;
}

int b200hh_hlll(b200hh_t *h, double delta, double eta, double theta, double c, int *status, uint64_t *iterations)
{
  (void)eta;  // hlll.h:155-159: eR is formed with delta in the reference; eta is not read on this code path
  (void)c;    // sr = 2^(-c d) is read only under HOUSEHOLDER_USE_SIZE_REDUCTION_TEST (hlll.cpp:296-312)
  if (!h || !status)
    return B200HH_EINVAL;
  if (!h->S.keep_hist)
  {
    g_err = "b200hh_hlll: the handle was created without keep_history (recover_R needs R_history)";
    return B200HH_EINVAL;
  }
  if (!width_ok(h, "b200hh_hlll"))
    return B200HH_EINVAL;
  CKH(cudaSetDevice(h->device));
  const HBatch &S = h->S;
  const size_t bd = (size_t)S.B * S.d;
  if (!h->d_hlll)
  {
    int rc = hh_alloc(h, &h->d_hlll, 3 * bd);
    rc |= hh_alloc(h, &h->d_hlll_i, bd + S.B);
    rc |= hh_alloc(h, &h->d_hlll_it, (size_t)S.B);
    if (rc)
      return B200HH_ENOMEM;
  }
  CKH(cudaMemsetAsync(h->d_hlll, 0, 3 * bd * 8, h->stream));
  CKH(cudaMemsetAsync(h->d_hlll_i, 0, (bd + S.B) * 4, h->stream));
  CKH(cudaMemsetAsync(h->d_hlll_it, 0, (size_t)S.B * 8, h->stream));
  hk_init<<<hgrid(h), HW * 32, h->smem, h->stream>>>(S);  // a fresh MatHouseholder over the current b
  HlllArgs A;
  A.delta = delta, A.theta = theta;
  A.dR = h->d_hlll, A.eR = h->d_hlll + bd, A.prevR = h->d_hlll + 2 * bd;
  A.prevE = h->d_hlll_i, A.status = h->d_hlll_i + bd, A.iters = h->d_hlll_it;
  A.max_iter = 1000000ull + 64ull * S.d * S.d;
  switch (h->tr)
  {
  case HT_NONE: launch_hlll_tr<HT_NONE>(h, A); break;
  case HT_U: launch_hlll_tr<HT_U>(h, A); break;
  default: launch_hlll_tr<HT_UINV>(h, A); break;
  }
  CKH(cudaMemcpyAsync(status, A.status, (size_t)S.B * 4, cudaMemcpyDeviceToHost, h->stream));
  if (iterations)
    CKH(cudaMemcpyAsync(iterations, A.iters, (size_t)S.B * 8, cudaMemcpyDeviceToHost, h->stream));
  CKH(cudaStreamSynchronize(h->stream));
  CKH(cudaGetLastError());
  return 0;
}

int b200hh_sync(b200hh_t *h)
{
  if (!h)
    return B200HH_EINVAL;
  CKH(cudaSetDevice(h->device));
  CKH(cudaStreamSynchronize(h->stream));
  CKH(cudaGetLastError());
  return 0;
}

}  // extern "C"
