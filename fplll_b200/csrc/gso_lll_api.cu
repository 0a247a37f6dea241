// gso_lll_api.cu — the one-warp-per-lattice LLL / size-reduction kernels (gso_lll.cuh) and their launcher.
#include "gso_common.cuh"

namespace {

// XF: the handle tracks the transform U (B200GSO_TRANSFORM); the untransformed instantiations never touch it
template <int MAXQ, bool XF>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32)
    k_lll(Batch S, double delta, double eta, int kmin, int kstart, int kend, int sr_start, int *status, long *stats)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  const int l = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  LLLStats st;
  MetaCache mc;
  mc.load(v, meta_scratch(S, lov), lane);
  const int r = warp_lll<MAXQ, false, XF>(v, s, lov, delta, eta, kmin, kstart, kend, sr_start, lane, st);
  mc.store(v, lane);
  if (lane == 0)
  {
    status[l] = r;
    if (stats)
    {
      stats[4 * l + 0] = st.n_swaps, stats[4 * l + 1] = st.final_kappa;
      stats[4 * l + 2] = st.zeros, stats[4 * l + 3] = st.babai_iters;
#ifdef B200_LLL_PROFILE
      // profiling builds (batch 1 only): overwrite final_kappa/zeros/babai_iters slots?  no — append after the batch block
      long *px = stats + 4 * S.B;
      px[0] = st.cyc_update, px[1] = st.cyc_babai, px[2] = st.cyc_lovasz, px[3] = st.cyc_move;
#endif
    }
  }
}

template <int MAXQ, bool XF>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32)
    k_size_reduction(Batch S, double eta, int kmin, int kend, int sr_start, int *status)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  const int l = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  long iters  = 0;
  MetaCache mc;
  mc.load(v, meta_scratch(S, lov), lane);
  const int r = warp_size_reduction<MAXQ, false, XF>(v, s, kmin, kend, sr_start, eta, lane, iters);
  mc.store(v, lane);
  if (lane == 0)
    status[l] = r;
}

}  // namespace

int b200gso_lll_warp_attrs(size_t smem_bytes)
{
  (void)smem_bytes;  // process-wide kernels: always the opt-in maximum (a smaller handle must not lower it)
  const void *fns[] = {(const void *)k_lll<4, false>,  (const void *)k_lll<8, false>,  (const void *)k_lll<16, false>,
                       (const void *)k_lll<4, true>,   (const void *)k_lll<8, true>,   (const void *)k_lll<16, true>,
                       (const void *)k_size_reduction<4, false>, (const void *)k_size_reduction<8, false>,
                       (const void *)k_size_reduction<16, false>, (const void *)k_size_reduction<4, true>,
                       (const void *)k_size_reduction<8, true>,  (const void *)k_size_reduction<16, true>};
  for (const void *f : fns)
    CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_OPTIN_MAX));
  return 0;
}

int b200gso_lll_warp_launch(b200gso *h, int mode, double delta, double eta, int kmin, int kstart, int kend,
                            int sr_start, int *d_st, long *d_stats)
{
  const Batch &S = h->S;
  const int g = grid_warps(h), t = WARPS_PER_CTA * 32;
#define LLL_LAUNCH(Q, XF)                                                                                          \
  do                                                                                                               \
  {                                                                                                                \
    if (mode == 0)                                                                                                 \
      k_lll<Q, XF><<<g, t, h->smem_bytes, h->stream>>>(S, delta, eta, kmin, kstart, kend, sr_start, d_st, d_stats); \
    else                                                                                                           \
      k_size_reduction<Q, XF><<<g, t, h->smem_bytes, h->stream>>>(S, eta, kmin, kend, sr_start, d_st);             \
  } while (0)
  const bool xf = S.u != nullptr;
  if (S.d <= 128)
  {
    if (xf) LLL_LAUNCH(4, true); else LLL_LAUNCH(4, false);
  }
  else if (S.d <= 256)
  {
    if (xf) LLL_LAUNCH(8, true); else LLL_LAUNCH(8, false);
  }
  else
  {
    if (xf) LLL_LAUNCH(16, true); else LLL_LAUNCH(16, false);
  }
#undef LLL_LAUNCH
  return 0;
}
