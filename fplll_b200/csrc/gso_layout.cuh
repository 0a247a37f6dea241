// gso_layout.cuh — HBM layout of the fp64 Gram-Schmidt state (one lattice; a batch is an array of these).
//
// Reference layout (fplll/gso_interface.h:548-618, nr/matrix.h:223): bf d x n, gf/mu/r d x d as
// vector<NumVect<FP_NR<double>>> — full rectangles, one heap allocation per row.
//
// Device layout, chosen for the one access pattern every hot loop shares — "lane j owns output j and walks
// its own row of an operand matrix in ascending column order" (update_gso_row's k-loop over mu(j,.),
// gso_interface.cpp:147-151; get_gram's dot product over bf(j,.), numvect.h:385-395).  A plain row-major (or
// row-packed) triangle makes that walk a 32-way strided gather.  So the two swept operands are stored as
//
//   PANEL-PACKED: rows are grouped in panels of 32; inside a panel the storage is column-major
//                 [column][lane] so that, for a fixed column, the 32 rows of a panel are one contiguous,
//                 256-byte, fully coalesced warp load.
//
//   mu  : packed LOWER TRIANGLE of panels — panel p keeps columns 0 .. 32(p+1)-1 only
//         (base 512*p*(p+1) doubles, element (j,k) at base + 32*k + (j & 31)); the upper halves of the diagonal
//         32x32 tiles are never read (loads are predicated) so DRAM traffic stays at the packed-triangle bytes.
//         The otherwise unused slot mu(j,j) mirrors r(j,j): update_gso_row divides by it (gso_interface.cpp:155), and
//         this way the divisor arrives with the diagonal tile's own lines instead of a 256-byte-strided gather.
//   bf  : panel p keeps all n columns (base 32*n*p, element (j,c) at base + 32*c + (j & 31)).
//
//   r, gf : row-packed lower triangle including the diagonal, rows padded to an even length so every row
//           starts 16-byte aligned: row i starts at ((i+1)^2)>>1 and holds i+1 (+pad) doubles.  These are only
//           ever touched as whole rows (read r(i,0..), write r(i,.), gf(i,.)), which row-packed makes coalesced.
//   b   : int64, row-major, row stride ldb = n rounded up to even (16-byte aligned rows for 128-bit row ops).
//   u   : int64, row-major d x d, row stride ld_b(d) — the transform U of a B200GSO_TRANSFORM handle (null otherwise).
//         Every integer row operation on b is applied to the row of u with the same index, over all d columns.
//
// NaN in gf marks an invalid Gram entry exactly as in the reference (gso.cpp:50-54, gso.h:324).
#pragma once
#include <cstddef>
#include <cstdint>

namespace b200 {

constexpr int PANEL = 32;

__host__ __device__ inline size_t tri_off(int i) { return ((size_t)(i + 1) * (size_t)(i + 1)) >> 1; }
__host__ __device__ inline size_t tri_size(int d) { return (tri_off(d) + 1) & ~(size_t)1; }
__host__ __device__ inline int n_panels(int d) { return (d + PANEL - 1) / PANEL; }
__host__ __device__ inline size_t mu_panel_base(int p) { return (size_t)512 * p * (p + 1); }
__host__ __device__ inline size_t mu_off(int j, int k) { return mu_panel_base(j >> 5) + (size_t)k * 32 + (j & 31); }
__host__ __device__ inline size_t mu_size(int d) { return mu_panel_base(n_panels(d)); }
__host__ __device__ inline size_t bf_off(int j, int c, int n) { return (size_t)(j >> 5) * 32 * n + (size_t)c * 32 + (j & 31); }
__host__ __device__ inline size_t bf_size(int d, int n) { return (size_t)n_panels(d) * 32 * n; }
__host__ __device__ inline int ld_b(int n) { return (n + 1) & ~1; }

// meta[] slots (per lattice)
// M_CLEAN_SR / M_CLEAN_LLL: number of leading rows known to be size-reduced (eta) / LLL-reduced (delta, eta) with a
// valid GSO — maintained so that a repeated lll(0,0,k) / size_reduction(0,k) call resumes at the first row that was
// touched since, instead of re-walking rows on which the reference's loop is a proven no-op (gso_lll.cuh).
enum
{
  M_NKR = 0, M_NKC = 1, M_NSR = 2, M_LOCKED = 3, M_CLEAN_SR = 4, M_CLEAN_LLL = 5,
  M_DELTA_LO = 6, M_DELTA_HI = 7, M_ETA_LO = 8, M_ETA_HI = 9, M_STRIDE = 16
};

// One lattice's state (device pointers) without the transform.  The CTA LLL keeps a copy of it in shared memory
// (CoopShared, gso_cta.cuh) and carries u next to it, so that adding u changed neither that layout nor the code of the
// kernels that never touch u.
struct ViewCore
{
  int d, n, ldb, row_expo_en;
  int host_basis;  // B200GSO_HOST_BASIS: b is not on the device, bf rows are uploaded by the host
  int64_t *b;
  double *bf, *mu, *r, *gf;
  int *row_expo, *valid, *irs, *meta;
  double *scratch;  // >= tri_size(d) + 2*d*ld + ... doubles, see gso_api
};
struct View : ViewCore
{
  int64_t *u;  // B200GSO_TRANSFORM: d x d, row stride ld_b(d); nullptr otherwise
};

// A batch: base pointers + per-lattice strides.
struct Batch
{
  int B, d, n, ldb, row_expo_en;
  int host_basis;
  int64_t *b;
  double *bf, *mu, *r, *gf, *scratch;
  int *row_expo, *valid, *irs, *meta;
  size_t b_stride, bf_stride, mu_stride, tri_stride, scratch_stride;
  int64_t *u;  // B200GSO_TRANSFORM handles only (nullptr otherwise), u_stride = d * ld_b(d) per lattice
  size_t u_stride;

  __host__ __device__ View view(int l) const
  {
    View v;
    v.d = d, v.n = n, v.ldb = ldb, v.row_expo_en = row_expo_en, v.host_basis = host_basis;
    v.b        = b + (size_t)l * b_stride;
    v.bf       = bf + (size_t)l * bf_stride;
    v.mu       = mu + (size_t)l * mu_stride;
    v.r        = r + (size_t)l * tri_stride;
    v.gf       = gf + (size_t)l * tri_stride;
    v.scratch  = scratch + (size_t)l * scratch_stride;
    v.row_expo = row_expo + (size_t)l * d;
    v.valid    = valid + (size_t)l * d;
    v.irs      = irs + (size_t)l * d;
    v.meta     = meta + (size_t)l * M_STRIDE;
    v.u        = u ? u + (size_t)l * u_stride : nullptr;
    return v;
  }
};

}  // namespace b200
