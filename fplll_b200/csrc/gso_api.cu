// gso_api.cu — kernels + extern "C" entry points declared in include/b200gso.h.
//
// Launch geometry: one warp per lattice, WARPS_PER_CTA lattices per CTA, grid = ceil(batch / WARPS_PER_CTA).
// With the panel-packed layout (gso_layout.cuh) every hot global access is a 256-byte coalesced warp load, so the
// kernels are HBM-streaming: occupancy (16+ resident warps per SM, 8 independent loads in flight per lane in the
// sweep loops) is what hides DRAM latency, not shared-memory tiling.  There is no CPU fallback anywhere.
#include "gso_common.cuh"
#include "gso_gram.cuh"

thread_local std::string b200gso_g_err;
long b200gso_g_prof[8] = {0, 0, 0, 0, 0, 0, 0, 0};

namespace {

// size_increased(), gso.cpp:368-403: init_row_size, zero-filled bf, update_bf for every row; fresh metadata.
__global__ void k_init(Batch S)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  if (lane < M_STRIDE)
    v.meta[lane] = 0;
  const size_t nbf = bf_size(v.d, v.n);
  for (size_t t = lane; t < nbf; t += 32)
    v.bf[t] = 0.0;
  __syncwarp();
  for (int i = 0; i < v.d; i++)
  {
    const int nz = size_nz_warp(v.b + (size_t)i * v.ldb, v.n, lane);
    if (lane == 0)
    {
      v.irs[i]      = max(nz, 1);
      v.valid[i]    = 0;
      v.row_expo[i] = 0;
    }
    __syncwarp();
    warp_update_bf(v, i, lane);
  }
}

__global__ void k_init_host_basis(Batch S)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  if (lane < M_STRIDE)
    v.meta[lane] = 0;
  const size_t nbf = bf_size(v.d, v.n);
  for (size_t t = lane; t < nbf; t += 32)
    v.bf[t] = 0.0;
  for (int i = lane; i < v.d; i += 32)
  {
    v.irs[i]      = v.n;
    v.valid[i]    = 0;
    v.row_expo[i] = 0;
  }
}

// repack a plain row-major batch*d*n int64 buffer into the ldb-strided device basis
__global__ void k_pack_b(Batch S, const int64_t *src)
{
  const int l = blockIdx.y;
  View v      = S.view(l);
  const size_t tot = (size_t)S.d * S.n;
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < tot; t += (size_t)gridDim.x * blockDim.x)
  {
    const int i = (int)(t / S.n), c = (int)(t % S.n);
    v.b[(size_t)i * S.ldb + c] = src[(size_t)l * tot + t];
  }
}
__global__ void k_unpack_b(Batch S, int64_t *dst)
{
  const int l = blockIdx.y;
  View v      = S.view(l);
  const size_t tot = (size_t)S.d * S.n;
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < tot; t += (size_t)gridDim.x * blockDim.x)
  {
    const int i = (int)(t / S.n), c = (int)(t % S.n);
    dst[(size_t)l * tot + t] = v.b[(size_t)i * S.ldb + c];
  }
}

__global__ void k_discover_all(Batch S, int upto)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  while (v.meta[M_NKR] < upto)
    warp_discover_row(v, lane);
}

__global__ void __launch_bounds__(WARPS_PER_CTA * 32, 5) k_update_row(Batch S, int i, int last_j, int *ok)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup<false>(S, v, s, lov, lane))
    return;
  const bool r = warp_update_gso_row(v, i, last_j, s, lane);
  if (ok && lane == 0)
    ok[blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)] = r ? 1 : 0;
}

__global__ void __launch_bounds__(WARPS_PER_CTA * 32) k_update_gso(Batch S, int *ok)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup<false>(S, v, s, lov, lane))
    return;
  bool r = true;
  for (int i = 0; i < v.d && r; i++)
    r = warp_update_gso_row(v, i, i, s, lane);
  if (ok && lane == 0)
    ok[blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)] = r ? 1 : 0;
}

// Whole Gram matrix in 32 x 32 tiles (gso_gram.cuh): warp w of CTA (x, l) takes tile pair 4 x + w of lattice l.
__global__ void __launch_bounds__(128) k_gram_tiles(Batch S, int mode)
{
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  View v      = S.view(blockIdx.y);
  const int P = n_panels(v.d), t = blockIdx.x * 4 + w;
  if (t >= P * (P + 1) / 2)
    return;
  int pi, pj;
  gram_pair(t, pi, pj);
  const int ncols = v.meta[M_NKC];
  if (mode == GRAM_DMMA)
    warp_gram_tile_dmma(v, pi, pj, ncols, lane);
  else
    warp_gram_tile_ordered(v, pi, pj, ncols, lane);
}

__global__ void k_row_addmul_we(Batch S, int i, int j, const double *x, const long *expo_add)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  const int l = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  warp_row_addmul_we(v, i, j, x[l], expo_add ? expo_add[l] : 0, lane);
}

__global__ void k_row_op_end(Batch S, int first, int last)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  warp_row_op_end(v, first, last, lane);
}

// invalidate_gso_row(i, 0) only (gso_interface.cpp:24-30) — used by the g=0 timing mode
__global__ void k_invalidate_gso_row(Batch S, int i)
{
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l < S.B)
    S.view(l).valid[i] = 0;
}

__global__ void k_row_swap(Batch S, int i, int j)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  warp_row_swap(v, i, j, lane);
}

__global__ void k_move_row(Batch S, int old_r, int new_r)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  warp_move_row(v, old_r, new_r, lane);
  if (v.u && old_r != new_r)
    warp_move_u_row(v, old_r, new_r, lane);
}

__global__ void k_set_r(Batch S, int i, int j, const double *f)
{
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l < S.B)
  {
    View v              = S.view(l);
    v.r[tri_off(i) + j] = f[l];
    if (i == j)
      v.mu[mu_off(i, i)] = f[l];  // diagonal mirror (gso_layout.cuh)
    v.meta[M_CLEAN_SR]  = min(v.meta[M_CLEAN_SR], i);
    v.meta[M_CLEAN_LLL] = min(v.meta[M_CLEAN_LLL], i);
    if (v.valid[i] == j)
      v.valid[i] = j + 1;
  }
}

__global__ void k_upload_row(Batch S, int i, const int64_t *rows)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  const int l = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  for (int c = lane; c < v.n; c += 32)
    v.b[(size_t)i * v.ldb + c] = rows[(size_t)l * v.n + c];
  __syncwarp();
  warp_row_op_end(v, i, i + 1, lane);
}

// host-basis handles: store the uploaded floating-point row, then the invalidation half of row_op_end(i, i+1)
__global__ void k_upload_row_fp(Batch S, int i, const double *rows, const long *expo)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  const int l = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  for (int c = lane; c < v.n; c += 32)
    v.bf[bf_off(i, c, v.n)] = rows[(size_t)l * v.n + c];
  if (lane == 0)
    v.row_expo[i] = v.row_expo_en ? (int)expo[l] : 0;
  __syncwarp();
  if (i < v.meta[M_NKR])
    warp_row_op_end(v, i, i + 1, lane);
}

// dense read-back (the reference's Matrix<FT> view of the state)
__global__ void k_unpack_state(Batch S, double *mu, double *r, double *gf, double *bf)
{
  const int l = blockIdx.y;
  View v      = S.view(l);
  const int d = S.d, n = S.n;
  const size_t dd = (size_t)d * d, dn = (size_t)d * n;
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < dd; t += (size_t)gridDim.x * blockDim.x)
  {
    const int i = (int)(t / d), j = (int)(t % d);
    if (mu)
      mu[l * dd + t] = (j < i) ? v.mu[mu_off(i, j)] : 0.0;
    if (r)
      r[l * dd + t] = (j <= i) ? v.r[tri_off(i) + j] : 0.0;
    if (gf)
      gf[l * dd + t] = (j <= i) ? v.gf[tri_off(i) + j] : 0.0;
  }
  if (bf)
    for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < dn; t += (size_t)gridDim.x * blockDim.x)
    {
      const int i = (int)(t / n), c = (int)(t % n);
      bf[l * dn + t] = v.bf[bf_off(i, c, n)];
    }
}

__global__ void k_get_row(Batch S, int i, double *mu_row, double *r_row, int *valid)
{
  const int l = blockIdx.x;
  View v      = S.view(l);
  for (int j = threadIdx.x; j < S.d; j += blockDim.x)
  {
    if (mu_row)
      mu_row[(size_t)l * S.d + j] = (j < i) ? v.mu[mu_off(i, j)] : 0.0;
    if (r_row)
      r_row[(size_t)l * S.d + j] = (j <= i) ? v.r[tri_off(i) + j] : 0.0;
  }
  if (valid && threadIdx.x == 0)
    valid[l] = v.valid[i];
}

__global__ void k_apply_ops(Batch S, const b200gso_op *ops, int n)
{
  View v;
  WarpSmem s;
  double *lov;
  int lane;
  if (!warp_setup(S, v, s, lov, lane))
    return;
  MetaCache mc;
  mc.load(v, meta_scratch(S, lov), lane);
  for (int t = 0; t < n; t++)
  {
    const b200gso_op op = ops[t];
    switch (op.type)
    {
    case B200GSO_OP_ROW_ADDMUL: warp_row_addmul_we(v, op.a, op.b, op.x, 0, lane); break;
    case B200GSO_OP_MOVE_ROW:
      warp_move_row(v, op.a, op.b, lane);
      if (v.u && op.a != op.b)
        warp_move_u_row(v, op.a, op.b, lane);
      break;
    case B200GSO_OP_ROW_SWAP: warp_row_swap(v, op.a, op.b, lane); break;
    case B200GSO_OP_ROW_OP_END: warp_row_op_end(v, op.a, op.b, lane); break;
    case B200GSO_OP_NEGATE: warp_negate_row(v, op.a, lane); break;
    }
    __syncwarp();
  }
  mc.store(v, lane);
}

// MatGSO::negate_row_of_b(i), gso.h:291-297 (integer row only), and row i of U on a transform handle (warp_negate_row)
__global__ void k_negate_row(Batch S, int i)
{
  const int l = blockIdx.y;
  View v      = S.view(l);
  if (blockIdx.x == 0 && threadIdx.x == 0)
  {
    v.meta[M_CLEAN_SR]  = min(v.meta[M_CLEAN_SR], i);
    v.meta[M_CLEAN_LLL] = min(v.meta[M_CLEAN_LLL], i);
  }
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < S.n; c += gridDim.x * blockDim.x)
    v.b[(size_t)i * S.ldb + c] = -v.b[(size_t)i * S.ldb + c];
  if (v.u)
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < S.d; c += gridDim.x * blockDim.x)
      u_row(v, i)[c] = -u_row(v, i)[c];
}

// U = identity on every lattice (the buffer was zeroed)
__global__ void k_u_identity(Batch S)
{
  View v = S.view(blockIdx.x);
  for (int i = threadIdx.x; i < S.d; i += blockDim.x)
    u_row(v, i)[i] = 1;
}

__global__ void k_get_r_diag(Batch S, int l, int first, int count, double *rmant, long *rexpo)
{
  View v = S.view(l);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x)
  {
    rmant[i] = v.r[tri_off(first + i) + first + i];
    rexpo[i] = v.row_expo_en ? 2L * v.row_expo[first + i] : 0L;
  }
}

// What Enumeration::enumerate pulls out of the GSO for a block (enumerate.cpp:91-141, enumerate_ext.cpp:91-148):
// mut[k*beta+j] = get_mu(first+j, first+k) for j > k (true value, row_expo applied), and r(first+i,first+i) as
// (mantissa, exponent) = get_r_exp.  Lattice l only.
__global__ void k_get_block(Batch S, int l, int first, int beta, double *mut, double *rmant, long *rexpo)
{
  View v = S.view(l);
  for (int t = threadIdx.x; t < beta * beta; t += blockDim.x)
  {
    const int k = t / beta, j = t % beta;
    double val = 0.0;
    if (j > k)
    {
      val = v.mu[mu_off(first + j, first + k)];
      if (v.row_expo_en)
        val = ldexp(val, v.row_expo[first + j] - v.row_expo[first + k]);
    }
    mut[t] = val;
  }
  for (int i = threadIdx.x; i < beta; i += blockDim.x)
  {
    rmant[i] = v.r[tri_off(first + i) + first + i];
    rexpo[i] = v.row_expo_en ? 2L * v.row_expo[first + i] : 0L;
  }
}

}  // namespace

static void launch_update_row(b200gso *h, int i, int last_j)
{
  k_update_row<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_compact, h->stream>>>(h->S, i, last_j, h->d_ok);
}

template <class T> static int dev_alloc(b200gso *h, T **p, size_t count)
{
  void *q = nullptr;
  cudaError_t e = cudaMalloc(&q, count * sizeof(T) + 256);
  if (e != cudaSuccess)
  {
    g_err = std::string("cudaMalloc: ") + cudaGetErrorString(e);
    return B200GSO_ENOMEM;
  }
  h->allocs.push_back(q);
  *p = (T *)q;
  return 0;
}

extern "C" {

const char *b200gso_version(void) { return "b200gso 0.1 (sm_90a)"; }
const char *b200gso_last_error(void) { return g_err.c_str(); }

int b200gso_device_count(void)
{
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess)
  {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int b200gso_create(b200gso_t **out, int batch, int d, int n, int flags, int device)
{
  if (!out || batch <= 0 || d <= 0 || n <= 0 || (flags & 1) ||
      (flags & ~(1 | 2 | 4 | B200GSO_HOST_BASIS | B200GSO_TRANSFORM)))
  {
    g_err = "b200gso_create: bad arguments (GSO_INT_GRAM is not supported on the device)";
    return B200GSO_EINVAL;
  }
  if ((flags & B200GSO_TRANSFORM) && (flags & B200GSO_HOST_BASIS))
  {
    g_err = "b200gso_create: B200GSO_TRANSFORM needs the int64 basis on the device (not B200GSO_HOST_BASIS)";
    return B200GSO_EINVAL;
  }
  if (b200gso_device_count() <= device)
  {
    g_err = "b200gso_create: no CUDA device (this library has no CPU fallback)";
    return B200GSO_ENODEV;
  }
  CK(cudaSetDevice(device));
  // L2 -> DRAM fetch granularity hint.  The panel sweeps issue whole 256-byte lines, but the partial last panel, the
  // diagonal tiles and the scattered mu(i,.) row write touch single 32-byte sectors; at the default (128 B) those cost
  // extra DRAM traffic.
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
  b200gso *h = new b200gso();
  h->device  = device;
  cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, device);
  Batch &S   = h->S;
  S.B = batch, S.d = d, S.n = n, S.ldb = ld_b(n), S.row_expo_en = (flags & B200GSO_ROW_EXPO) ? 1 : 0;
  S.host_basis = (flags & B200GSO_HOST_BASIS) ? 1 : 0;
  S.b_stride       = (size_t)d * S.ldb;
  S.bf_stride      = bf_size(d, n);
  S.mu_stride      = mu_size(d);
  S.tri_stride     = tri_size(d);
  S.scratch_stride = tri_size(d);
  S.u              = nullptr;
  S.u_stride       = (flags & B200GSO_TRANSFORM) ? (size_t)d * ld_b(d) : 0;
  int rc = 0;
  if (flags & B200GSO_TRANSFORM)
    rc |= dev_alloc(h, &S.u, S.u_stride * batch);
  rc |= dev_alloc(h, &S.b, S.b_stride * batch);
  rc |= dev_alloc(h, &S.bf, S.bf_stride * batch);
  rc |= dev_alloc(h, &S.mu, S.mu_stride * batch);
  rc |= dev_alloc(h, &S.r, S.tri_stride * batch);
  rc |= dev_alloc(h, &S.gf, S.tri_stride * batch);
  rc |= dev_alloc(h, &S.scratch, S.scratch_stride * batch);
  rc |= dev_alloc(h, &S.row_expo, (size_t)d * batch);
  rc |= dev_alloc(h, &S.valid, (size_t)d * batch);
  rc |= dev_alloc(h, &S.irs, (size_t)d * batch);
  rc |= dev_alloc(h, &S.meta, (size_t)M_STRIDE * batch);
  rc |= dev_alloc(h, &h->d_ok, (size_t)batch);
  rc |= dev_alloc(h, &h->d_tmp, (size_t)batch);
  rc |= dev_alloc(h, &h->d_ltmp, (size_t)batch * 4);
  rc |= dev_alloc(h, &h->d_rows, (size_t)batch * n);
  rc |= dev_alloc(h, &h->d_rowbuf, (size_t)2 * batch * d);
  rc |= dev_alloc(h, &h->d_valid_i, (size_t)batch);
  rc |= dev_alloc(h, &h->d_stats, (size_t)batch * 4 + 8 + ((size_t)batch + 1) / 2);  // + status ints behind the longs
  rc |= dev_alloc(h, &h->d_blk, (size_t)d * d + 4 * (size_t)d + 16);
  h->d_ops = nullptr, h->ops_cap = 0;
  h->h_pin = nullptr, h->pin_bytes = 0, h->h_ops = nullptr, h->h_ops_cap = 0;
  h->stream = nullptr;
  if (rc)
  {
    for (void *p : h->allocs)
      cudaFree(p);
    delete h;
    return B200GSO_ENOMEM;
  }
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess)
  {
    g_err = "b200gso_create: cudaStreamCreate failed";
    h->stream = nullptr;
    b200gso_destroy(h);
    return B200GSO_ECUDA;
  }
  h->pin_bytes = ((size_t)d * d + 4 * (size_t)d + 64) * sizeof(double) + ((size_t)batch * 4 + 8) * sizeof(long) +
                 (size_t)batch * sizeof(int);
  if (cudaMallocHost(&h->h_pin, h->pin_bytes) != cudaSuccess)
  {
    g_err = "b200gso_create: cudaMallocHost failed";
    h->h_pin = nullptr;
    b200gso_destroy(h);
    return B200GSO_ENOMEM;
  }
  h->smem_bytes = WARPS_PER_CTA * (WarpSmem::doubles(d, n) + (size_t)((d + 2 + 1) & ~1) + ((MetaCache::ints(d) + 1) >> 1)) *
                  sizeof(double);
  h->smem_compact = WARPS_PER_CTA * WarpSmem::doubles(d, n, false) * sizeof(double);
  if (h->smem_bytes > 227 * 1024)
  {
    g_err = "b200gso_create: d/n too large for the per-warp shared-memory scratch";
    b200gso_destroy(h);
    return B200GSO_EINVAL;
  }
  const void *fns[] = {(const void *)k_init,         (const void *)k_discover_all, (const void *)k_update_row,
                       (const void *)k_update_gso,   (const void *)k_row_addmul_we, (const void *)k_row_op_end,
                       (const void *)k_row_swap,     (const void *)k_move_row,     (const void *)k_upload_row,
                       (const void *)k_apply_ops,    (const void *)k_upload_row_fp, (const void *)k_init_host_basis};
  // The kernels are process-wide: the attribute is the opt-in maximum (227 KB), never this handle's own size — a
  // second, smaller handle must not lower the limit under a larger live one.
  for (const void *f : fns)
  {
    const cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_OPTIN_MAX);
    if (e != cudaSuccess)
    {
      g_err = std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e);
      b200gso_destroy(h);
      return B200GSO_ECUDA;
    }
  }
  if (b200gso_lll_warp_attrs(h->smem_bytes) || b200gso_lll_cta_attrs(d, n))
  {
    b200gso_destroy(h);
    return B200GSO_ECUDA;
  }
  cudaError_t me = cudaMemsetAsync(S.b, 0, S.b_stride * batch * sizeof(int64_t), h->stream);
  if (me == cudaSuccess) me = cudaMemsetAsync(S.mu, 0, S.mu_stride * batch * sizeof(double), h->stream);
  if (me == cudaSuccess) me = cudaMemsetAsync(S.r, 0, S.tri_stride * batch * sizeof(double), h->stream);
  if (me == cudaSuccess) me = cudaMemsetAsync(S.gf, 0, S.tri_stride * batch * sizeof(double), h->stream);
  if (me == cudaSuccess) me = cudaMemsetAsync(S.meta, 0, (size_t)M_STRIDE * batch * sizeof(int), h->stream);
  if (me == cudaSuccess && S.u)
  {
    me = cudaMemsetAsync(S.u, 0, S.u_stride * batch * sizeof(int64_t), h->stream);
    if (me == cudaSuccess)
    {
      k_u_identity<<<batch, 128, 0, h->stream>>>(S);
      me = cudaGetLastError();
    }
  }
  if (me == cudaSuccess) me = cudaStreamSynchronize(h->stream);
  if (me != cudaSuccess)
  {
    g_err = std::string("b200gso_create: ") + cudaGetErrorString(me);
    b200gso_destroy(h);
    return B200GSO_ECUDA;
  }
  if (S.host_basis)
  {
    // size_increased() without an integer basis: every row spans all n columns, bf zero until uploaded
    k_init_host_basis<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S);
    me = cudaStreamSynchronize(h->stream);
    if (me != cudaSuccess)
    {
      g_err = std::string("b200gso_create: ") + cudaGetErrorString(me);
      b200gso_destroy(h);
      return B200GSO_ECUDA;
    }
  }
  *out = h;
  return 0;
}

void b200gso_destroy(b200gso_t *h)
{
  if (!h)
    return;
  cudaSetDevice(h->device);
  if (h->stream)
  {
    cudaStreamSynchronize(h->stream);
    cudaStreamDestroy(h->stream);
  }
  for (void *p : h->allocs)
    cudaFree(p);
  if (h->d_ops)
    cudaFree(h->d_ops);
  if (h->h_pin)
    cudaFreeHost(h->h_pin);
  if (h->h_ops)
    cudaFreeHost(h->h_ops);
  delete h;
}

#define NO_HOST_BASIS(h_)                                                                        \
  do                                                                                             \
  {                                                                                              \
    if ((h_)->S.host_basis)                                                                      \
    {                                                                                            \
      g_err = "this entry point needs the int64 basis on the device (handle is B200GSO_HOST_BASIS)"; \
      return B200GSO_EINVAL;                                                                     \
    }                                                                                            \
  } while (0)

int b200gso_set_basis_dev(b200gso_t *h, const int64_t *dev_b)
{
  if (!h || !dev_b)
    return B200GSO_EINVAL;
  NO_HOST_BASIS(h);
  CK(cudaSetDevice(h->device));
  dim3 g(64, h->S.B);
  k_pack_b<<<g, 256, 0, h->stream>>>(h->S, dev_b);
  k_init<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S);
  CK(cudaGetLastError());
  return 0;
}

int b200gso_set_basis(b200gso_t *h, const int64_t *b)
{
  if (!h || !b)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  const size_t cnt = (size_t)h->S.B * h->S.d * h->S.n;
  int64_t *tmp     = nullptr;
  CK(cudaMalloc(&tmp, cnt * sizeof(int64_t)));
  cudaError_t e = cudaMemcpyAsync(tmp, b, cnt * sizeof(int64_t), cudaMemcpyHostToDevice, h->stream);
  int rc        = (e == cudaSuccess) ? b200gso_set_basis_dev(h, tmp) : B200GSO_ECUDA;
  cudaStreamSynchronize(h->stream);
  cudaFree(tmp);
  if (e != cudaSuccess)
    g_err = cudaGetErrorString(e);
  return rc;
}

int b200gso_get_basis(b200gso_t *h, int64_t *b)
{
  if (!h || !b)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  const size_t cnt = (size_t)h->S.B * h->S.d * h->S.n;
  int64_t *tmp     = nullptr;
  CK(cudaMalloc(&tmp, cnt * sizeof(int64_t)));
  dim3 g(64, h->S.B);
  k_unpack_b<<<g, 256, 0, h->stream>>>(h->S, tmp);
  cudaError_t e = cudaMemcpyAsync(b, tmp, cnt * sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream);
  cudaStreamSynchronize(h->stream);
  cudaFree(tmp);
  if (e != cudaSuccess)
  {
    g_err = cudaGetErrorString(e);
    return B200GSO_ECUDA;
  }
  CK(cudaGetLastError());
  return 0;
}

int b200gso_upload_row_fp(b200gso_t *h, int i, const double *bf_rows, const long *expo)
{
  if (!h || !bf_rows || i < 0 || i >= h->S.d || !h->S.host_basis || (h->S.row_expo_en && !expo))
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  // d_rows (batch*n int64) doubles as the staging area: same element size
  CK(cudaMemcpyAsync(h->d_rows, bf_rows, (size_t)h->S.B * h->S.n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  if (expo)
    CK(cudaMemcpyAsync(h->d_ltmp, expo, (size_t)h->S.B * sizeof(long), cudaMemcpyHostToDevice, h->stream));
  k_upload_row_fp<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, i, (const double *)h->d_rows,
                                                                                   expo ? h->d_ltmp : nullptr);
  CK(cudaStreamSynchronize(h->stream));  // host arrays may be reused by the caller
  CK(cudaGetLastError());
  return 0;
}

// U (batch x d x d, dense) <-> the device's ld_b(d)-strided rows: one 2D copy, every lattice's rows share the pitch
static int copy_transform(b200gso_t *h, int64_t *dst, const int64_t *src, bool to_device)
{
  if (!h || (to_device ? !src : !dst))
    return B200GSO_EINVAL;
  if (!h->S.u)
  {
    g_err = "b200gso_set/get_transform: the handle was created without B200GSO_TRANSFORM";
    return B200GSO_EINVAL;
  }
  CK(cudaSetDevice(h->device));
  const size_t d = h->S.d, dev_pitch = ld_b(h->S.d) * sizeof(int64_t), rows = (size_t)h->S.B * d;
  if (to_device)
    CK(cudaMemcpy2DAsync(h->S.u, dev_pitch, src, d * sizeof(int64_t), d * sizeof(int64_t), rows,
                         cudaMemcpyHostToDevice, h->stream));
  else
    CK(cudaMemcpy2DAsync(dst, d * sizeof(int64_t), h->S.u, dev_pitch, d * sizeof(int64_t), rows,
                         cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  return 0;
}

int b200gso_set_transform(b200gso_t *h, const int64_t *u) { return copy_transform(h, nullptr, u, true); }

int b200gso_get_transform(b200gso_t *h, int64_t *u) { return copy_transform(h, u, nullptr, false); }

int b200gso_upload_row(b200gso_t *h, int i, const int64_t *rows)
{
  if (!h || !rows || i < 0 || i >= h->S.d)
    return B200GSO_EINVAL;
  NO_HOST_BASIS(h);
  if (h->S.u)
  {
    g_err = "b200gso_upload_row: a row rewritten on the host leaves U unknown (handle is B200GSO_TRANSFORM)";
    return B200GSO_EINVAL;
  }
  CK(cudaSetDevice(h->device));
  // stream-ordered: with pinned `rows` this returns without waiting (the caller must not reuse `rows` before the
  // next synchronising call); pageable memory makes cudaMemcpyAsync stage synchronously, which is also correct.
  CK(cudaMemcpyAsync(h->d_rows, rows, (size_t)h->S.B * h->S.n * sizeof(int64_t), cudaMemcpyHostToDevice, h->stream));
  k_upload_row<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, i, h->d_rows);
  CK(cudaGetLastError());
  return 0;
}

int b200gso_discover_all_rows(b200gso_t *h)
{
  if (!h)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  k_discover_all<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, h->S.d);
  CK(cudaGetLastError());
  return 0;
}

int b200gso_discover_rows(b200gso_t *h, int upto)
{
  if (!h || upto < 0 || upto > h->S.d)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  k_discover_all<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, upto);
  CK(cudaGetLastError());
  return 0;
}

static int fetch_ok(b200gso_t *h, int *ok)
{
  if (ok)
  {
    CK(cudaMemcpyAsync(ok, h->d_ok, sizeof(int) * h->S.B, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  CK(cudaGetLastError());
  return 0;
}

int b200gso_update_gso_row(b200gso_t *h, int i, int last_j, int *ok)
{
  if (!h || i < 0 || i >= h->S.d || last_j < 0 || last_j > i)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  launch_update_row(h, i, last_j);
  return fetch_ok(h, ok);
}

int b200gso_update_gso(b200gso_t *h, int *ok)
{
  if (!h)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  k_update_gso<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_compact, h->stream>>>(h->S, h->d_ok);
  return fetch_ok(h, ok);
}

int b200gso_update_gso_blocked(b200gso_t *h, int gram_mode, int *ok)
{
  if (!h || (gram_mode != B200GSO_GRAM_ORDERED && gram_mode != B200GSO_GRAM_DMMA) || h->S.B > 65535)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  k_discover_all<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, h->S.d);
  const int P = n_panels(h->S.d), pairs = P * (P + 1) / 2;
  k_gram_tiles<<<dim3((pairs + 3) / 4, h->S.B), 128, 0, h->stream>>>(h->S, gram_mode);
  k_update_gso<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_compact, h->stream>>>(h->S, h->d_ok);
  return fetch_ok(h, ok);
}

int b200gso_row_addmul_we(b200gso_t *h, int i, int j, const double *x, const long *expo_add)
{
  if (!h || !x || i < 0 || j < 0 || i >= h->S.d || j >= h->S.d)
    return B200GSO_EINVAL;
  NO_HOST_BASIS(h);
  CK(cudaSetDevice(h->device));
  CK(cudaMemcpyAsync(h->d_tmp, x, sizeof(double) * h->S.B, cudaMemcpyHostToDevice, h->stream));
  if (expo_add)
    CK(cudaMemcpyAsync(h->d_ltmp, expo_add, sizeof(long) * h->S.B, cudaMemcpyHostToDevice, h->stream));
  k_row_addmul_we<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, i, j, h->d_tmp,
                                                                                   expo_add ? h->d_ltmp : nullptr);
  CK(cudaStreamSynchronize(h->stream));  // host arrays may be reused by the caller
  CK(cudaGetLastError());
  return 0;
}

int b200gso_row_op_begin(b200gso_t *h, int first, int last)
{
  (void)first, (void)last;  // no-op in release builds of the reference too (gso_interface.h:785-788)
  return h ? 0 : B200GSO_EINVAL;
}

int b200gso_row_op_end(b200gso_t *h, int first, int last)
{
  if (!h || first < 0 || last > h->S.d || first > last)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  k_row_op_end<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, first, last);
  CK(cudaGetLastError());
  return 0;
}

int b200gso_row_swap(b200gso_t *h, int i, int j)
{
  if (!h || i < 0 || j < 0 || i >= h->S.d || j >= h->S.d)
    return B200GSO_EINVAL;
  if (h->S.host_basis)
    return 0;  // row_swap touches the integer rows only (gso.cpp:264-287): they live on the host
  CK(cudaSetDevice(h->device));
  k_row_swap<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, i, j);
  CK(cudaGetLastError());
  return 0;
}

int b200gso_move_row(b200gso_t *h, int old_r, int new_r)
{
  if (!h || old_r < 0 || new_r < 0 || old_r >= h->S.d || new_r >= h->S.d)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  k_move_row<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, old_r, new_r);
  CK(cudaGetLastError());
  return 0;
}

int b200gso_set_r(b200gso_t *h, int i, int j, const double *f)
{
  if (!h || !f || i < 0 || i >= h->S.d || j < 0 || j > i)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  CK(cudaMemcpyAsync(h->d_tmp, f, sizeof(double) * h->S.B, cudaMemcpyHostToDevice, h->stream));
  k_set_r<<<(h->S.B + 127) / 128, 128, 0, h->stream>>>(h->S, i, j, h->d_tmp);
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  return 0;
}

// gf(i, 0..count-1) <- vals: the Gram row of a GSO_INT_GRAM object, computed exactly on the host (gso.h:314-331, int branch)
__global__ void k_set_gram_row(Batch S, int i, int count, const double *vals)
{
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= S.B * count)
    return;
  const int l = t / count, j = t - l * count;
  S.gf[(size_t)l * S.tri_stride + tri_off(i) + j] = vals[t];
}

int b200gso_set_gram_row(b200gso_t *h, int i, int count, const double *vals)
{
  if (!h || !vals || i < 0 || i >= h->S.d || count < 1 || count > i + 1)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  // staging: d_rowbuf holds 2 * batch * d doubles
  CK(cudaMemcpyAsync(h->d_rowbuf, vals, sizeof(double) * (size_t)h->S.B * count, cudaMemcpyHostToDevice, h->stream));
  k_set_gram_row<<<(h->S.B * count + 127) / 128, 128, 0, h->stream>>>(h->S, i, count, h->d_rowbuf);
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  return 0;
}

int b200gso_get_state(b200gso_t *h, double *mu, double *r, double *gf, double *bf, int64_t *row_expo,
                      int *gso_valid_cols, int *init_row_size, int *meta)
{
  if (!h)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  const Batch &S  = h->S;
  const size_t dd = (size_t)S.B * S.d * S.d, dn = (size_t)S.B * S.d * S.n;
  double *t_mu = nullptr, *t_r = nullptr, *t_gf = nullptr, *t_bf = nullptr;
  if (mu)
    CK(cudaMalloc(&t_mu, dd * 8));
  if (r)
    CK(cudaMalloc(&t_r, dd * 8));
  if (gf)
    CK(cudaMalloc(&t_gf, dd * 8));
  if (bf)
    CK(cudaMalloc(&t_bf, dn * 8));
  dim3 g(32, S.B);
  k_unpack_state<<<g, 256, 0, h->stream>>>(S, t_mu, t_r, t_gf, t_bf);
  if (mu)
    cudaMemcpyAsync(mu, t_mu, dd * 8, cudaMemcpyDeviceToHost, h->stream);
  if (r)
    cudaMemcpyAsync(r, t_r, dd * 8, cudaMemcpyDeviceToHost, h->stream);
  if (gf)
    cudaMemcpyAsync(gf, t_gf, dd * 8, cudaMemcpyDeviceToHost, h->stream);
  if (bf)
    cudaMemcpyAsync(bf, t_bf, dn * 8, cudaMemcpyDeviceToHost, h->stream);
  std::vector<int> tmp;
  if (row_expo)
  {
    tmp.resize((size_t)S.B * S.d);
    cudaMemcpyAsync(tmp.data(), S.row_expo, tmp.size() * 4, cudaMemcpyDeviceToHost, h->stream);
  }
  if (gso_valid_cols)
    cudaMemcpyAsync(gso_valid_cols, S.valid, (size_t)S.B * S.d * 4, cudaMemcpyDeviceToHost, h->stream);
  if (init_row_size)
    cudaMemcpyAsync(init_row_size, S.irs, (size_t)S.B * S.d * 4, cudaMemcpyDeviceToHost, h->stream);
  std::vector<int> m;
  if (meta)
  {
    m.resize((size_t)S.B * M_STRIDE);
    cudaMemcpyAsync(m.data(), S.meta, m.size() * 4, cudaMemcpyDeviceToHost, h->stream);
  }
  cudaError_t e = cudaStreamSynchronize(h->stream);
  cudaFree(t_mu), cudaFree(t_r), cudaFree(t_gf), cudaFree(t_bf);
  if (e != cudaSuccess)
  {
    g_err = cudaGetErrorString(e);
    return B200GSO_ECUDA;
  }
  if (row_expo)
    for (size_t t = 0; t < tmp.size(); t++)
      row_expo[t] = tmp[t];
  if (meta)
    for (int l = 0; l < S.B; l++)
      for (int q = 0; q < 4; q++)
        meta[4 * l + q] = m[(size_t)l * M_STRIDE + q];
  CK(cudaGetLastError());
  return 0;
}

int b200gso_get_mu_r_row(b200gso_t *h, int i, double *mu_row, double *r_row, int *valid)
{
  if (!h || i < 0 || i >= h->S.d)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  const Batch &S   = h->S;
  const size_t cnt = (size_t)S.B * S.d;
  double *t        = h->d_rowbuf;
  k_get_row<<<S.B, 128, 0, h->stream>>>(S, i, mu_row ? t : nullptr, r_row ? t + cnt : nullptr,
                                        valid ? h->d_valid_i : nullptr);
  if (mu_row)
    CK(cudaMemcpyAsync(mu_row, t, cnt * 8, cudaMemcpyDeviceToHost, h->stream));
  if (r_row)
    CK(cudaMemcpyAsync(r_row, t + cnt, cnt * 8, cudaMemcpyDeviceToHost, h->stream));
  if (valid)
    CK(cudaMemcpyAsync(valid, h->d_valid_i, sizeof(int) * S.B, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  return 0;
}

static int lll_dispatch(b200gso_t *h, int mode, double delta, double eta, int kmin, int kstart, int kend, int sr_start,
                        int *status, long *stats)
{
  if (!h || !status)
    return B200GSO_EINVAL;
  NO_HOST_BASIS(h);  // the device LLL does the integer row operations itself
  CK(cudaSetDevice(h->device));
  const Batch &S = h->S;
  if (kend < 0)
    kend = S.d;
  if (S.d > 512 || kmin < 0 || kstart < kmin || kend > S.d || kstart >= kend + (mode ? 1 : 0) || sr_start < 0)
  {
    g_err = "b200gso_lll/size_reduction: bad range (or d > 512)";
    return B200GSO_EINVAL;
  }
  // status ints live right behind the statistics longs: one D2H copy into pinned memory brings back both
  long *d_stats = h->d_stats;
  int *d_st     = (int *)(h->d_stats + 4 * (size_t)S.B + 8);
  // few lattices (BKZ works on one): a whole CTA per lattice (k_lll_cta); many: one warp per lattice, the batch hides
  // the latencies; the switch-over is two CTAs per SM.  B200_LLL_CTA=0 forces the one-warp kernels.
  const int cta_on = getenv("B200_LLL_CTA") ? atoi(getenv("B200_LLL_CTA")) : 1;  // read per call: tests switch kernels
  const bool cta   = cta_on && S.B <= 2 * h->sm_count && S.d > 32;
  if (cta)
  {
    if (b200gso_lll_cta_launch(h, mode, delta, eta, kmin, kstart, kend, sr_start, d_st, (stats && mode == 0) ? d_stats : nullptr))
      return B200GSO_ECUDA;
  }
  else if (b200gso_lll_warp_launch(h, mode, delta, eta, kmin, kstart, kend, sr_start, d_st, stats ? d_stats : nullptr))
    return B200GSO_ECUDA;
  const size_t nl = 4 * (size_t)S.B + 8, bytes = nl * sizeof(long) + (size_t)S.B * sizeof(int);
  CK(cudaMemcpyAsync(h->h_pin, d_stats, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  memcpy(status, h->h_pin + nl * sizeof(long), (size_t)S.B * sizeof(int));
  if (stats)
    memcpy(stats, h->h_pin, 4 * (size_t)S.B * sizeof(long));  // `stats` is batch*4 longs for the caller, always
#ifdef B200_LLL_PROFILE
  memcpy(b200gso_g_prof, h->h_pin + 4 * (size_t)S.B * sizeof(long), 8 * sizeof(long));
#endif
  return 0;
}

int b200gso_lll(b200gso_t *h, double delta, double eta, int *status, long *stats)
{
  return lll_dispatch(h, 0, delta, eta, 0, 0, -1, 0, status, stats);
}

int b200gso_lll_range(b200gso_t *h, double delta, double eta, int kappa_min, int kappa_start, int kappa_end,
                      int size_reduction_start, int *status, long *stats)
{
  return lll_dispatch(h, 0, delta, eta, kappa_min, kappa_start, kappa_end, size_reduction_start, status, stats);
}

int b200gso_size_reduction(b200gso_t *h, double eta, int kappa_min, int kappa_end, int size_reduction_start,
                           int *status)
{
  return lll_dispatch(h, 1, 0.99, eta, kappa_min, kappa_min, kappa_end, size_reduction_start, status, nullptr);
}

int b200gso_negate_row_of_b(b200gso_t *h, int i)
{
  if (!h || i < 0 || i >= h->S.d)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  dim3 g(1, h->S.B);
  k_negate_row<<<g, 256, 0, h->stream>>>(h->S, i);
  CK(cudaGetLastError());
  return 0;
}

int b200gso_apply_ops(b200gso_t *h, const b200gso_op *ops, int n)
{
  if (!h || (n > 0 && !ops) || n < 0)
    return B200GSO_EINVAL;
  if (n == 0)
    return 0;
  for (int t = 0; t < n; t++)
  {
    const b200gso_op &o = ops[t];
    const bool two = o.type == B200GSO_OP_ROW_ADDMUL || o.type == B200GSO_OP_MOVE_ROW || o.type == B200GSO_OP_ROW_SWAP;
    if (o.type < 1 || o.type > 5 || o.a < 0 || o.a >= h->S.d || (two && (o.b < 0 || o.b >= h->S.d)) ||
        (o.type == B200GSO_OP_ROW_OP_END && (o.b < o.a || o.b > h->S.d)))
    {
      g_err = "b200gso_apply_ops: bad op";
      return B200GSO_EINVAL;
    }
  }
  CK(cudaSetDevice(h->device));
  if ((size_t)n > h->ops_cap)
  {
    if (h->d_ops)
      cudaFree(h->d_ops);
    h->ops_cap = std::max<size_t>(1024, (size_t)n * 2);
    CK(cudaMalloc(&h->d_ops, sizeof(b200gso_op) * h->ops_cap));
  }
  if ((size_t)n > h->h_ops_cap)
  {
    if (h->h_ops)
      cudaFreeHost(h->h_ops);
    h->h_ops     = nullptr;
    h->h_ops_cap = 0;
    CK(cudaMallocHost(&h->h_ops, sizeof(b200gso_op) * std::max<size_t>(1024, (size_t)n * 2)));
    h->h_ops_cap = std::max<size_t>(1024, (size_t)n * 2);
  }
  memcpy(h->h_ops, ops, sizeof(b200gso_op) * n);  // pinned copy: the caller's array is free on return
  b200gso_op *d_ops = h->d_ops;
  CK(cudaMemcpyAsync(d_ops, h->h_ops, sizeof(b200gso_op) * n, cudaMemcpyHostToDevice, h->stream));
  k_apply_ops<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, d_ops, n);
  CK(cudaStreamSynchronize(h->stream));  // the next call reuses the staging buffer
  CK(cudaGetLastError());
  return 0;
}

int b200gso_get_r_diag(b200gso_t *h, int lattice, int first, int count, double *r_mant, long *r_expo)
{
  if (!h || lattice < 0 || lattice >= h->S.B || first < 0 || count < 1 || first + count > h->S.d || !r_mant || !r_expo)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  double *t = h->d_blk;
  long *te  = (long *)(t + count);
  k_get_r_diag<<<(count + 127) / 128, 128, 0, h->stream>>>(h->S, lattice, first, count, t, te);
  CK(cudaMemcpyAsync(r_mant, t, (size_t)count * 8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(r_expo, te, (size_t)count * sizeof(long), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  return 0;
}

int b200gso_get_block(b200gso_t *h, int lattice, int first, int beta, double *mut, double *r_mant, long *r_expo)
{
  if (!h || lattice < 0 || lattice >= h->S.B || first < 0 || beta < 1 || first + beta > h->S.d || !mut || !r_mant ||
      !r_expo)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  double *t       = h->d_blk;
  const size_t nd = (size_t)beta * beta + beta;
  long *te        = (long *)(t + nd);
  k_get_block<<<1, 256, 0, h->stream>>>(h->S, lattice, first, beta, t, t + (size_t)beta * beta, te);
  // mut | r_mant | r_expo are contiguous on the device: one copy into pinned memory, scattered on the host
  const size_t bytes = nd * 8 + (size_t)beta * sizeof(long);
  CK(cudaMemcpyAsync(h->h_pin, t, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  memcpy(mut, h->h_pin, (size_t)beta * beta * 8);
  memcpy(r_mant, h->h_pin + (size_t)beta * beta * 8, (size_t)beta * 8);
  memcpy(r_expo, h->h_pin + nd * 8, (size_t)beta * sizeof(long));
  return 0;
}

int b200gso_time_update_row(b200gso_t *h, int i, int reps, int invalidate, float *ms_update_mean, float *ms_total)
{
  if (!h || reps <= 0 || i < 0 || i >= h->S.d)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  struct Events  // released on every exit path
  {
    std::vector<cudaEvent_t> v;
    ~Events()
    {
      for (cudaEvent_t e : v)
        if (e)
          cudaEventDestroy(e);
    }
  } evs;
  evs.v.assign(2 * (size_t)reps + 2, nullptr);
  std::vector<cudaEvent_t> &ev = evs.v;
  for (auto &e : ev)
    CK(cudaEventCreate(&e));
  CK(cudaEventRecord(ev[2 * reps], h->stream));
  for (int r = 0; r < reps; r++)
  {
    if (invalidate)
      k_row_op_end<<<grid_warps(h), WARPS_PER_CTA * 32, h->smem_bytes, h->stream>>>(h->S, i, i + 1);
    else
      k_invalidate_gso_row<<<(h->S.B + 127) / 128, 128, 0, h->stream>>>(h->S, i);
    CK(cudaEventRecord(ev[2 * r], h->stream));
    launch_update_row(h, i, i);
    CK(cudaEventRecord(ev[2 * r + 1], h->stream));
  }
  CK(cudaEventRecord(ev[2 * reps + 1], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  double tot = 0;
  for (int r = 0; r < reps; r++)
  {
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, ev[2 * r], ev[2 * r + 1]));
    tot += ms;
  }
  float all = 0;
  CK(cudaEventElapsedTime(&all, ev[2 * reps], ev[2 * reps + 1]));
  if (ms_update_mean)
    *ms_update_mean = (float)(tot / reps);
  if (ms_total)
    *ms_total = all;
  CK(cudaGetLastError());
  return 0;
}

int b200gso_resident_lattices(b200gso_t *h)
{
  if (!h)
    return B200GSO_EINVAL;
  cudaSetDevice(h->device);
  int nb = 0, sms = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_update_row, WARPS_PER_CTA * 32, h->smem_compact) != cudaSuccess)
    return B200GSO_ECUDA;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
  return nb * sms * WARPS_PER_CTA;
}

int b200gso_lll_profile(long *out8)
{
  if (!out8)
    return B200GSO_EINVAL;
  for (int q = 0; q < 8; q++)
    out8[q] = b200gso_g_prof[q];
  return 0;
}

int b200gso_lll_cta_profile(long long *out32)
{
  if (!out32)
    return B200GSO_EINVAL;
  return b200gso_lll_cta_prof(out32);
}

int b200gso_sync(b200gso_t *h)
{
  if (!h)
    return B200GSO_EINVAL;
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  return 0;
}

}  // extern "C"
