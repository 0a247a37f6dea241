// gso_lll_cta_api.cu — the one-CTA-per-lattice LLL / size-reduction kernel (gso_cta.cuh) and its launcher.
#include "gso_common.cuh"

namespace {

// XF: the handle tracks the transform U (B200GSO_TRANSFORM); the untransformed instantiations never touch it
template <int MAXQ, bool XF>
__global__ void __launch_bounds__(CTA_WARPS * 32)
    k_lll_cta(Batch S, int mode, double delta, double eta, int kmin, int kstart, int kend, int sr_start, int *status,
              long *stats, int mu_panels)
{
  extern __shared__ __align__(16) double smem[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, l = blockIdx.x;
  const size_t base = WarpSmem::doubles(S.d, S.n);
  const size_t lovn = (size_t)((S.d + 2 + 1) & ~1);
  const size_t per  = base + lovn + ((((MetaCache::ints(S.d) + 1) >> 1) + 1) & ~(size_t)1);
  CoopShared *C     = reinterpret_cast<CoopShared *>(smem + per);
  double *bm        = smem + per + ((sizeof(CoopShared) + 15) / 16) * 2;
  if (w != 0)
  {
    coop_helper_loop<XF>(*C, w, lane);
    return;
  }
  LLLView<XF> v = S.view(l);
  WarpSmem s;
  s.carve(smem, S.d, S.n, true);
  double *lov = smem + base;
  MetaCache mc;
  mc.load(v, (int *)(lov + lovn), lane);
  if (lane == 0)
  {
    C->v = v;
    if constexpr (XF)
      C->u = v.u;
    C->s = s;
    C->bm = bm;
    C->pub = bm + (size_t)((S.d + 32 + 1) & ~1);
    C->epoch = 4096.0;
    C->mu_s = bm + 3 * (size_t)((S.d + 32 + 1) & ~1);
    C->mu_s_panels = mu_panels;
    C->mu_last_p = n_panels(S.d) - 1, C->mu_last_stride = mu_s_last_stride(S.d);
    C->cmd = COOP_EXIT, C->flag = 1;
  }
  // no slot of the publish array may look like a published value: tags start at 4096
  for (int t = lane; t < 2 * ((S.d + 32 + 1) & ~1); t += 32)
    bm[(size_t)((S.d + 32 + 1) & ~1) + t] = -1.0;
  __syncwarp();
  if (mu_panels > 0)
  {
    // shared-memory cache of the leading mu panels: every row the call can touch is < kend
    coop_post(C, COOP_MULOAD, 0, (kend - 1) >> 5, 0, lane);
    cta_mu_load(*C, 0, (kend - 1) >> 5, 0, lane);
  }
  LLLStats st;
  st.n_swaps = st.final_kappa = st.zeros = st.babai_iters = 0;
  int r;
  if (mode == 0)
    r = warp_lll<MAXQ, true, XF>(v, s, lov, delta, eta, kmin, kstart, kend, sr_start, lane, st, C);
  else
    r = warp_size_reduction<MAXQ, true, XF>(v, s, kmin, kend, sr_start, eta, lane, st.babai_iters, C);
  coop_post(C, COOP_EXIT, 0, 0, 0, lane);
  mc.store(v, lane);
  if (lane == 0)
  {
    status[l] = r;
    if (stats)
    {
      stats[4 * l + 0] = st.n_swaps, stats[4 * l + 1] = st.final_kappa;
      stats[4 * l + 2] = st.zeros, stats[4 * l + 3] = st.babai_iters;
#ifdef B200_LLL_PROFILE
      if (mode == 0)
      {
        long *px = stats + 4 * S.B;
        px[0] = st.cyc_update, px[1] = st.cyc_babai, px[2] = st.cyc_lovasz, px[3] = st.cyc_move;
        px[4] = st.cyc_gather, px[5] = st.cyc_backsub, px[6] = st.cyc_igemv, px[7] = st.cyc_ropend;
      }
#endif
    }
  }
}

}  // namespace

// profile builds: the cooperative operations' device-clock counters (gso_cta.cuh); zeros otherwise
int b200gso_lll_cta_prof(long long *out32)
{
  memset(out32, 0, 32 * sizeof(long long));
#ifdef B200_LLL_PROFILE
  CK(cudaMemcpyFromSymbol(out32, g_cta_prof, 32 * sizeof(long long)));
#endif
  return 0;
}

int b200gso_lll_cta_attrs(int d, int n)
{
  (void)d, (void)n;  // process-wide kernels: always the opt-in maximum (a smaller handle must not lower it)
  const int sm = SMEM_OPTIN_MAX;
  const void *fns[] = {(const void *)k_lll_cta<4, false>, (const void *)k_lll_cta<8, false>,
                       (const void *)k_lll_cta<16, false>, (const void *)k_lll_cta<4, true>,
                       (const void *)k_lll_cta<8, true>,  (const void *)k_lll_cta<16, true>};
  for (const void *f : fns)
    CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
  return 0;
}

int b200gso_lll_cta_launch(b200gso *h, int mode, double delta, double eta, int kmin, int kstart, int kend, int sr_start,
                           int *d_st, long *d_stats)
{
  const Batch &S = h->S;
  size_t sm = cta_smem_doubles(S.d, S.n) * sizeof(double);
  // cache as many leading mu panels as fit into the 227 KB of the CTA
  // full panels take 32 (p+1) columns of 33 doubles; the last panel of the lattice only its real rows (gso_cta.cuh)
  const int P   = n_panels(S.d);
  int mu_panels = 0;
  size_t used   = 0;
  while (mu_panels < P)
  {
    const size_t cols = 32 * (size_t)(mu_panels + 1);
    const size_t need = cols * (mu_panels == P - 1 ? mu_s_last_stride(S.d) : MU_SS);
    if (sm + (used + need) * sizeof(double) > (size_t)227 * 1024)
      break;
    used += need;
    mu_panels++;
  }
  sm += used * sizeof(double);
#define CTA_LAUNCH(Q, XF) \
  k_lll_cta<Q, XF><<<S.B, CTA_WARPS * 32, sm, h->stream>>>(S, mode, delta, eta, kmin, kstart, kend, sr_start, d_st, d_stats, mu_panels)
  const bool xf = S.u != nullptr;
  if (S.d <= 128)
  {
    if (xf) CTA_LAUNCH(4, true); else CTA_LAUNCH(4, false);
  }
  else if (S.d <= 256)
  {
    if (xf) CTA_LAUNCH(8, true); else CTA_LAUNCH(8, false);
  }
  else
  {
    if (xf) CTA_LAUNCH(16, true); else CTA_LAUNCH(16, false);
  }
#undef CTA_LAUNCH
  return 0;
}
