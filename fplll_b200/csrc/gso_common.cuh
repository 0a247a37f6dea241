// gso_common.cuh — what the translation units behind include/b200gso.h share: error string, launch geometry, the
// shared-memory metadata cache, the handle.  The library is compiled as three units (gso_api.cu: everything but the LLL
// kernels; gso_lll_api.cu: one-warp-per-lattice LLL kernels; gso_lll_cta_api.cu: one-CTA-per-lattice LLL kernels) so
// that nvcc processes run in parallel and the build stays deterministic (no --split-compile, whose code generation
// differs from run to run).
#pragma once
#include "../../include/b200gso.h"
#include "gso_lll.cuh"
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

using namespace b200;

extern thread_local std::string b200gso_g_err;  // defined in gso_api.cu
#define g_err b200gso_g_err

constexpr int WARPS_PER_CTA = 4;
// opt-in maximum of dynamic shared memory per CTA on sm_90: what every kernel's MaxDynamicSharedMemorySize is set to
constexpr int SMEM_OPTIN_MAX = 227 * 1024;
// -DB200_LLL_PROFILE builds: device-clock phase counters of the last LLL call (b200gso_lll_profile reads them)
extern long b200gso_g_prof[8];

#define CK(call)                                                                                   \
  do                                                                                               \
  {                                                                                                \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
    {                                                                                              \
      g_err = std::string(#call) + ": " + cudaGetErrorString(e_);                                  \
      return B200GSO_ECUDA;                                                                        \
    }                                                                                              \
  } while (0)

namespace {

// The LLL-family kernels (k_lll, k_size_reduction, k_apply_ops) are chains of short dependent steps on ONE lattice per
// warp; every read of gso_valid_cols / row_expo / init_row_size / n_known_* from global memory is a ~0.5 us round trip
// on the critical path.  MetaCache stages those arrays in shared memory for the lifetime of the kernel (the View's
// pointers are simply re-pointed, every device routine keeps working unchanged) and writes them back at the end.
struct MetaCache
{
  int *g_valid, *g_expo, *g_irs, *g_meta;
  int d;
  __host__ __device__ static size_t ints(int d) { return 3 * (size_t)((d + 3) & ~3) + M_STRIDE; }
  __device__ void load(ViewCore &v, int *sm, int lane)
  {
    d = v.d;
    const int dp = (d + 3) & ~3;
    g_valid = v.valid, g_expo = v.row_expo, g_irs = v.irs, g_meta = v.meta;
    int *s_valid = sm, *s_expo = sm + dp, *s_irs = sm + 2 * dp, *s_meta = sm + 3 * dp;
    for (int i = lane; i < d; i += 32)
    {
      s_valid[i] = g_valid[i];
      s_expo[i]  = g_expo[i];
      s_irs[i]   = g_irs[i];
    }
    if (lane < M_STRIDE)
      s_meta[lane] = g_meta[lane];
    v.valid = s_valid, v.row_expo = s_expo, v.irs = s_irs, v.meta = s_meta;
    __syncwarp();
  }
  __device__ void store(const ViewCore &v, int lane)
  {
    __syncwarp();
    for (int i = lane; i < d; i += 32)
    {
      g_valid[i] = v.valid[i];
      g_expo[i]  = v.row_expo[i];
      g_irs[i]   = v.irs[i];
    }
    if (lane < M_STRIDE)
      g_meta[lane] = v.meta[lane];
  }
};

template <bool FULL_SMEM = true>
__device__ inline bool warp_setup(const Batch &S, View &v, WarpSmem &s, double *&lov, int &lane)
{
  extern __shared__ __align__(16) double smem[];
  const int w = threadIdx.x >> 5;
  lane        = threadIdx.x & 31;
  const int l = blockIdx.x * (blockDim.x >> 5) + w;
  const size_t base = WarpSmem::doubles(S.d, S.n, FULL_SMEM);
  const size_t per  = base + (FULL_SMEM ? (size_t)((S.d + 2 + 1) & ~1) + ((MetaCache::ints(S.d) + 1) >> 1) : 0);
  s.carve(smem + (size_t)w * per, S.d, S.n, FULL_SMEM);
  lov = FULL_SMEM ? smem + (size_t)w * per + base : nullptr;
  if (l >= S.B)
    return false;
  v = S.view(l);
  return true;
}

__device__ inline int *meta_scratch(const Batch &S, double *lov) { return (int *)(lov + ((S.d + 2 + 1) & ~1)); }

// Single-lattice regime (BKZ): one CTA of CTA_WARPS warps per lattice, warp 0 runs the LLL / size-reduction control
// flow and shares the O(kappa d) pieces of every Babai iteration with the other warps (gso_cta.cuh).
// mode 0: lll(kmin, kstart, kend, sr_start); mode 1: size_reduction(kmin, kend, sr_start).
__host__ __device__ inline size_t cta_smem_doubles(int d, int n)
{
  const size_t per = WarpSmem::doubles(d, n) + (size_t)((d + 2 + 1) & ~1) + ((((MetaCache::ints(d) + 1) >> 1) + 1) & ~(size_t)1);
  // scratch | CoopShared | bm[d+32] | pub[2 (d+32)]  (the mu cache follows, gso_lll_cta_api.cu)
  return per + ((sizeof(CoopShared) + 15) / 16) * 2 + 3 * (size_t)((d + 32 + 1) & ~1);
}

}  // namespace

struct b200gso
{
  Batch S;
  int device;
  cudaStream_t stream;
  size_t smem_bytes, smem_compact;
  int *d_ok;      // batch ints
  double *d_tmp;  // batch doubles
  long *d_ltmp;   // batch longs
  int64_t *d_rows;    // batch*n   (upload_row staging)
  double *d_rowbuf;   // 2*batch*d (get_mu_r_row staging)
  int *d_valid_i;     // batch
  long *d_stats;      // 4*batch (LLL statistics)
  double *d_blk;      // d*d + 2*d doubles + d longs (get_block / get_r_diag staging)
  b200gso_op *d_ops;  // op-list staging (grown on demand)
  size_t ops_cap;
  // pinned host staging for the single-lattice driver calls (BKZ: ~10^5 small synchronous calls per tour — every
  // pageable copy costs a driver-side bounce, so results travel in ONE copy into pinned memory and are scattered here)
  unsigned char *h_pin;
  size_t pin_bytes;
  b200gso_op *h_ops;
  size_t h_ops_cap;
  std::vector<void *> allocs;
  int sm_count = 0;  // SMs of the device: the LLL launcher picks the CTA or the warp kernel by batch size against it
};

inline int grid_warps(const b200gso *h) { return (h->S.B + WARPS_PER_CTA - 1) / WARPS_PER_CTA; }

// launchers living next to their kernels (internal, not part of the C-ABI)
int b200gso_lll_warp_attrs(size_t smem_bytes);
int b200gso_lll_warp_launch(b200gso *h, int mode, double delta, double eta, int kmin, int kstart, int kend,
                            int sr_start, int *d_st, long *d_stats);
int b200gso_lll_cta_attrs(int d, int n);
int b200gso_lll_cta_prof(long long *out32);
int b200gso_lll_cta_launch(b200gso *h, int mode, double delta, double eta, int kmin, int kstart, int kend, int sr_start,
                           int *d_st, long *d_stats);
