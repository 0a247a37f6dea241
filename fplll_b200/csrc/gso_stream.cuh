// gso_stream.cuh — the batched update_gso_row sweep (gso_interface.cpp:131-164) as a TMA-fed streaming kernel.
//
// Same algorithm, same operation order and therefore the same bits as warp_update_gso_row (gso_warp.cuh); what changes
// is how the two swept operands reach the SM.  The register-staged kernel (k_update_row) keeps 16 x 256 B in flight per
// warp and is limited to 20 resident warps per SM by its staging registers: ~80 KB in flight per SM.  Here the bytes in flight live in shared memory and the TMA unit puts
// them there:
//
//   * one persistent CTA per SM of NW warps; warp c walks its own lattices (c, c + stride, ...) with the arithmetic of
//     warp_update_gso_row, reading its operands from a private ring of ST_STAGES x 4 KB.  A stage holds one CHUNK — 16
//     consecutive columns of one 32-row panel of bf or mu, which the panel-packed layout (gso_layout.cuh) makes one
//     dense box — delivered by one cp.async.bulk.tensor (SASS UTMALDG) that completes on the stage's mbarrier;
//   * the chunk sequence of a row update is the same for every lattice of the launch, so the CTA builds it ONCE as a
//     table of descriptors in shared memory (map, byte count, coordinates relative to the lattice).  After consuming a
//     chunk, lane 0 of the warp re-arms the stage with the chunk ST_STAGES further down the table — a 16-byte load, a few
//     integer adds, one TMA instruction; no staging registers, no address arithmetic in the consumer loops — and the
//     table index simply runs on into the warp's NEXT lattice, so the ring stays full while the warp is inside the
//     serial parts of a row (the 32-step triangles, the r(i,i) chain);
//   * tensor maps with different boxes fetch only what the row needs: {32 x 16} for full panels, {R x 16} for the last
//     panel when only R of its rows are < i (at d = 200 that is 8 rows: 64 B instead of 256 B per column), {16 x 16} for
//     the second half of a diagonal tile (its upper-right quarter is never read);
//   * the int64 row b_i the Gram recompute needs as bf_i travels as a 1-D bulk copy (UBLKCP) at the head of the
//     lattice's chunk sequence.
//
// Scope: the full recompute LLL's babai pays after every row_op_end (lll.cpp:166-224): gso_valid_cols[i] == 0 and the
// whole Gram row invalid, all n columns known.  A warp classifies its next lattice one lattice ahead; a lattice in any
// other state takes warp_update_gso_row (out of line) and the stream skips it.
#pragma once
#include "gso_warp.cuh"
#include "tma.cuh"

namespace b200 {

constexpr int ST_STAGES    = 4;
constexpr int ST_COLS      = 16;            // columns per chunk
constexpr int ST_STAGE_DBL = ST_COLS * 32;  // doubles per stage (4 KB)
constexpr int ST_MAX_CONS  = 12;            // warps per CTA (384 threads: 168 registers)

// 3-D tensor maps {row, column, slab}: bf — slab = lattice * P + panel, n columns each; mu — one slab, the columns of the
// whole allocation.  [0] bf {32 x 16}  [1] bf {R x 16}  [2] mu {32 x 16}  [3] mu {R x 16}  [4] mu {16 x 16}
struct StreamMaps
{
  CUtensorMap m[5];
};
enum { SM_BF_FULL = 0, SM_BF_PART = 1, SM_MU_FULL = 2, SM_MU_PART = 3, SM_MU_B = 4, SM_BROW = 5 };

// per warp: vb | rrow | murow (compact WarpSmem) | ring | mbarriers (128 bytes)
__host__ __device__ inline size_t stream_warp_doubles(int d, int n)
{
  return ((WarpSmem::doubles(d, n, false) + 15) & ~(size_t)15) + (size_t)ST_STAGES * ST_STAGE_DBL + 16;
}

// What the row update of ONE lattice looks like to the stream; the same for every streamed lattice of a launch except
// for ncols (n_known_cols), which is read per lattice.
struct StreamShape
{
  int i, last_j, jl;  // jl = min(last_j, i - 1): last off-diagonal column
  int P;              // panels that carry work: 0 .. P-1
  int rows_last;      // rows of panel P-1 that are fetched: (jl & 31) + 1 rounded up to 2 (32: a full panel)
};

__host__ __device__ inline StreamShape stream_shape(int i, int last_j)
{
  StreamShape sh;
  sh.i = i, sh.last_j = last_j;
  sh.jl        = min(last_j, i - 1);
  sh.P         = sh.jl >= 0 ? (sh.jl >> 5) + 1 : 0;
  sh.rows_last = sh.jl >= 0 ? (((sh.jl & 31) + 1 + 1) & ~1) : 32;
  return sh;
}
// columns of panel p's diagonal tile that carry a row (32 for a full panel)
__host__ __device__ inline int stream_tile_cols(const StreamShape &sh, int p) { return min(32, sh.jl - 32 * p + 1); }

// ---- the chunk table -------------------------------------------------------------------------------------------------
// The chunk sequence of one lattice:  b_i | for p < P: bf panel p (ceil(n / 16) chunks), mu panel p rectangular part
// (2 p chunks), diagonal tile columns 0..15, diagonal tile columns 16..31 (if they carry rows).
struct StreamDesc
{
  int map;    // SM_* : which copy
  int bytes;  // what lands in the stage
  int c1;     // column coordinate relative to the lattice (mu) / inside the panel (bf)
  int c2;     // panel (bf); row coordinate (mu: 0, or 16 for the second half of a full diagonal tile)
};
__host__ __device__ inline int stream_panel_chunks(const StreamShape &sh, int p, int n)
{
  return (n + ST_COLS - 1) / ST_COLS + 2 * p + 1 + (stream_tile_cols(sh, p) > 16 ? 1 : 0);
}
__host__ __device__ inline int stream_num_chunks(const StreamShape &sh, int n)
{
  int c = 1;
  for (int p = 0; p < sh.P; p++)
    c += stream_panel_chunks(sh, p, n);
  return c;
}
__host__ __device__ inline StreamDesc stream_desc(const StreamShape &sh, int n, int ldb, int e)
{
  StreamDesc d;
  if (e == 0)
  {
    d.map = SM_BROW, d.bytes = ldb * 8, d.c1 = 0, d.c2 = 0;
    return d;
  }
  e -= 1;
  int p = 0;
  for (; p < sh.P; p++)
  {
    const int c = stream_panel_chunks(sh, p, n);
    if (e < c)
      break;
    e -= c;
  }
  const bool part = (p == sh.P - 1) && sh.rows_last < 32;
  const int rows  = part ? sh.rows_last : 32;
  const int nbf   = (n + ST_COLS - 1) / ST_COLS;
  d.bytes         = rows * ST_COLS * 8;
  if (e < nbf)
  {
    d.map = part ? SM_BF_PART : SM_BF_FULL, d.c1 = ST_COLS * e, d.c2 = p;
    return d;
  }
  e -= nbf;
  const int col = (int)(mu_panel_base(p) >> 5);
  d.map = part ? SM_MU_PART : SM_MU_FULL, d.c2 = 0;
  if (e < 2 * p)
    d.c1 = col + ST_COLS * e;
  else if (e == 2 * p)
    d.c1 = col + 32 * p;
  else
  {
    d.c1 = col + 32 * p + 16;
    if (!part)
      d.map = SM_MU_B, d.c2 = 16, d.bytes = 16 * 16 * 8;  // rows 16..31 of columns 16..31
  }
  return d;
}

// lane 0: start the copy of chunk e of lattice l into `dst`, completing on `bar`
__device__ inline void stream_issue(const Batch &S, const StreamMaps &M, const StreamDesc *tab, int row_i, int l, int e,
                                    double *dst, unsigned long long *bar)
{
  const StreamDesc d = tab[e];
  tma_mbar_expect_tx(bar, (unsigned)d.bytes);
  if (d.map == SM_BROW)
  {
    tma_bulk_1d(dst, S.b + (size_t)l * S.b_stride + (size_t)row_i * S.ldb, (unsigned)d.bytes, bar);
    return;
  }
  const bool bf = d.map <= SM_BF_PART;
  const int c1  = bf ? d.c1 : d.c1 + l * (int)(S.mu_stride >> 5);
  const int c2  = bf ? d.c2 + l * n_panels(S.d) : 0;
  tma_load_3d(dst, &M.m[d.map], bf ? 0 : d.c2, c1, c2, bar);
}

// ---- consumer ----------------------------------------------------------------------------------------------------------
// A warp's ring and its position in the stream.  `issued`/`consumed` count chunks over the life of the warp (stage =
// count % ST_STAGES, mbarrier parity = (count / ST_STAGES) & 1); (iss_l, iss_e) = the next chunk to issue: entry iss_e of
// lattice iss_l's table walk.
struct StreamRing
{
  double *ring;
  unsigned long long *bars;
  const StreamDesc *tab;
  int NC;        // chunks per lattice
  int row_i;     // the row being updated
  int stride;    // distance between a warp's lattices
  unsigned issued, consumed;
  int iss_l, iss_e;
  int cur_l;     // the lattice being consumed
  bool next_ok;  // the warp's next lattice (cur_l + stride) takes the stream: the table walk may run on into it
  __device__ const double *head() const { return ring + (size_t)(consumed % ST_STAGES) * ST_STAGE_DBL; }
  __device__ void wait() const { tma_mbar_wait(bars + (consumed % ST_STAGES), (consumed / ST_STAGES) & 1u); }
  __device__ void issue_one(const Batch &S, const StreamMaps &M, int lane)
  {
    if (iss_e == NC)
    {
      if (iss_l != cur_l || !next_ok)
        return;  // one lattice of lookahead at most
      iss_l = cur_l + stride, iss_e = 0;
    }
    if (lane == 0)
      stream_issue(S, M, tab, row_i, iss_l, iss_e, ring + (size_t)(issued % ST_STAGES) * ST_STAGE_DBL,
                   bars + (issued % ST_STAGES));
    issued++, iss_e++;
  }
  // every lane is done with the head stage: re-arm it with the next chunk of the stream
  __device__ void release(const Batch &S, const StreamMaps &M, int lane)
  {
    __syncwarp();
    consumed++;
    issue_one(S, M, lane);
  }
};

// ordered chain over one staged chunk: acc (+|-)= tile[u * rs] * vec[u], u = 0 .. nc-1 ascending (two roundings per
// step); tile = this lane's row in the stage (consecutive columns rs doubles apart), vec in shared memory.  All 16
// products are formed first (independent; columns >= nc read stale but mapped shared memory and are dropped), the
// chain only adds.  FIRST: the chain starts with the bare product of column 0 (dot_product, numvect.h:385-395).
template <bool SUB, bool FIRST>
__device__ inline double chunk_chain(double acc, const double *tile, const double *vec, int nc, int rs)
{
  double t[ST_COLS];
#pragma unroll
  for (int u = 0; u < ST_COLS; u++)
    t[u] = __dmul_rn(tile[u * rs], vec[u]);
  if (FIRST)
    acc = t[0];
  if (nc == ST_COLS)
  {
#pragma unroll
    for (int u = FIRST ? 1 : 0; u < ST_COLS; u++)
      acc = SUB ? __dsub_rn(acc, t[u]) : __dadd_rn(acc, t[u]);
    return acc;
  }
#pragma unroll
  for (int u = FIRST ? 1 : 0; u < ST_COLS; u++)
    if (u < nc)
      acc = SUB ? __dsub_rn(acc, t[u]) : __dadd_rn(acc, t[u]);
  return acc;
}

// 16 steps of the in-panel triangle: column 32 p + t (t = t0 .. t0 + 15) is final in lane t once steps < t are applied.
// tile(t) = mu(32 p + lane, 32 p + t) for lane >= t (the diagonal slot mirrors r(j,j), gso_layout.cuh), read from the
// staged half tile  st[(t - t0) * rs + lane - roff].
__device__ inline void tile_half(double &acc, double &rd, const double *st, int t0, int tmax, int rs, int roff, int rows,
                                 bool act, int lane)
{
  double m[16];
#pragma unroll
  for (int u = 0; u < 16; u++)
  {
    const int t = t0 + u;
    m[u]        = (t <= tmax && lane >= t && lane < rows) ? st[u * rs + lane - roff] : 0.0;
  }
#pragma unroll
  for (int u = 0; u < 16; u++)
  {
    const int t = t0 + u;
    if (lane == t)
      rd = m[u];
    if (t < 31)
    {
      const double rk = __shfl_sync(FULL, acc, t);
      if (act && lane > t)
        acc = __dsub_rn(acc, __dmul_rn(m[u], rk));
    }
  }
}

static __device__ __noinline__ bool stream_fallback(const Batch &S, int l, int i, int last_j, WarpSmem s, int lane)
{
  const View v = S.view(l);
  return warp_update_gso_row(v, i, last_j, s, lane);
}

// n_known_cols of lattice l if it takes the stream (row discovered, nothing of it valid, every Gram entry the call needs
// invalid), else 0; row_expo[i] on the side
__device__ inline int stream_classify(const Batch &S, int l, int i, int glast, int lane, int &expo)
{
  const int *meta = S.meta + (size_t)l * M_STRIDE;
  const int valid = S.valid[(size_t)l * S.d + i], nkr = meta[M_NKR], nkc = meta[M_NKC];
  expo            = S.row_expo_en ? S.row_expo[(size_t)l * S.d + i] : 0;
  const double *g = S.gf + (size_t)l * S.tri_stride + tri_off(i);
  int notnan      = 0;
  for (int j = lane; j <= glast; j += 32)
    notnan |= (g[j] == g[j]);
  const bool el = !S.host_basis && i < nkr && valid <= 0 && nkc == S.n && !__any_sync(FULL, notnan);
  return el ? nkc : 0;
}

// What a consumer warp keeps of its lattice: four row pointers and its scratch rows (no View, no address arithmetic for
// the streams — registers are what bounds the number of consumer warps per SM).
struct StreamRow
{
  double *gfrow, *rrow_g, *mu_i;  // gf(i, .), r(i, .), &mu(i, 0): mu(i, j) at mu_i[32 j] inside panel i >> 5
  double *vb, *rrow, *murow;      // shared memory: bf_i, r(i, .), mu(i, .)
};

// One panel of the forward substitution.  ROWS = 32: a full panel (strides are compile-time); ROWS = 0: the partial last
// panel, `rows` rows staged per column.
template <int ROWS>
__device__ inline bool stream_panel(const Batch &S, const StreamMaps &M, const StreamShape &sh, const StreamRow &row,
                                    StreamRing &R, int p, int ncols, int rows, bool live, int lane)
{
  const int rs     = ROWS ? ROWS : rows;
  const int j      = 32 * p + lane;
  const bool act   = live && j <= sh.jl;
  const bool inbox = live && lane < rs;
  double acc       = 0.0;
  // Gram entry g(i, j): dot_product over bf (numvect.h:385-395), first term a bare product
  {
    R.wait();
    if (inbox)
      acc = chunk_chain<false, true>(acc, R.head() + lane, row.vb, min(ST_COLS, ncols), rs);
    R.release(S, M, lane);
  }
#pragma unroll 1
  for (int c0 = ST_COLS; c0 < ncols; c0 += ST_COLS)
  {
    R.wait();
    if (inbox)
      acc = chunk_chain<false, false>(acc, R.head() + lane, row.vb + c0, min(ST_COLS, ncols - c0), rs);
    R.release(S, M, lane);
  }
  if (act)
    row.gfrow[j] = acc;  // get_gram caches the entry (gso.h:324-327)
  // rectangular part of the forward substitution: columns k < 32 p, r(i, k) in shared memory
#pragma unroll 1
  for (int c0 = 0; c0 < 32 * p; c0 += ST_COLS)
  {
    R.wait();
    if (inbox)
      acc = chunk_chain<true, false>(acc, R.head() + lane, row.rrow + c0, ST_COLS, rs);
    R.release(S, M, lane);
  }
  // diagonal tile, two halves of 16 columns
  double rd      = 1.0;
  const int tmax = stream_tile_cols(sh, p) - 1;
  R.wait();
  tile_half(acc, rd, R.head(), 0, tmax, rs, 0, rs, act, lane);
  R.release(S, M, lane);
  if (tmax >= 16)
  {
    R.wait();
    if (ROWS)
      tile_half(acc, rd, R.head(), 16, tmax, 16, 16, 32, act, lane);
    else
      tile_half(acc, rd, R.head(), 16, tmax, rs, 0, rs, act, lane);
    R.release(S, M, lane);
  }
  bool okp = true;
  if (act)
  {
    row.rrow_g[j]    = acc;
    row.rrow[j]      = acc;
    const double mm  = __ddiv_rn(acc, rd);
    row.mu_i[32 * j] = mm;
    row.murow[j]     = mm;
    okp              = isfinite(mm);
  }
  __syncwarp();
  return __all_sync(FULL, okp);
}

__device__ inline void stream_consumer(const Batch &S, const StreamMaps &M, const StreamShape &sh, int l, int stride,
                                       int *ok_out, double *base, const StreamDesc *tab, int NC, int lane)
{
  const int i = sh.i, last_j = sh.last_j;
  WarpSmem s;
  s.carve(base, S.d, S.n, false);
  StreamRing R;
  R.ring   = base + ((WarpSmem::doubles(S.d, S.n, false) + 15) & ~(size_t)15);
  R.bars   = (unsigned long long *)(R.ring + (size_t)ST_STAGES * ST_STAGE_DBL);
  R.tab    = tab, R.NC = NC, R.row_i = i, R.stride = stride;
  R.issued = R.consumed = 0;
  R.iss_l = -1, R.iss_e = NC;
  StreamRow row;
  row.vb = s.vb, row.rrow = s.rrow, row.murow = s.murow;
  const int glast = min(last_j, i);
  int expo = 0, expo_next = 0;
  int ncols = stream_classify(S, l, i, glast, lane, expo);
#pragma unroll 1
  for (; l < S.B; l += stride)
  {
    int ncols_next = 0;
    if (l + stride < S.B)
      ncols_next = stream_classify(S, l + stride, i, glast, lane, expo_next);
    R.cur_l = l, R.next_ok = ncols_next != 0;
    if (ncols == 0)
    {
      const bool r = stream_fallback(S, l, i, last_j, s, lane);
      if (ok_out && lane == 0)
        ok_out[l] = r ? 1 : 0;
      ncols = ncols_next, expo = expo_next;
      continue;
    }
    if (R.iss_l != l)
    {
      // no lookahead reached this lattice (first of the warp, or its predecessor took the fallback): fill the ring
      R.iss_l = l, R.iss_e = 0;
      for (int q = 0; q < ST_STAGES; q++)
        R.issue_one(S, M, lane);
    }
    row.gfrow  = S.gf + (size_t)l * S.tri_stride + tri_off(i);
    row.rrow_g = S.r + (size_t)l * S.tri_stride + tri_off(i);
    row.mu_i   = S.mu + (size_t)l * S.mu_stride + mu_off(i, 0);
    // ---- b_i -> bf_i (update_bf, gso.cpp:24-48: (double) b * 2^-row_expo exactly) ----
    {
      R.wait();
      const long long *brow = (const long long *)R.head();
      const double sc       = pow2d(-expo);
      for (int c = lane; c < ncols; c += 32)
        row.vb[c] = __dmul_rn((double)brow[c], sc);
      R.release(S, M, lane);
    }
    bool live = true;  // false once a mu(i, j) came out non-finite: the reference returns false there, the rest of this
                       // lattice's chunks are only drained
#pragma unroll 1
    for (int p = 0; p < sh.P; ++p)
    {
      const bool part = (p == sh.P - 1) && sh.rows_last < 32;
      const bool okp  = part ? stream_panel<0>(S, M, sh, row, R, p, ncols, sh.rows_last, live, lane)
                             : stream_panel<32>(S, M, sh, row, R, p, ncols, 32, live, lane);
      live            = live && okp;
    }
    if (live)
    {
      if (last_j >= i)
      {
        // diagonal r(i,i) = g(i,i) - sum_{k<i} mu(i,k) r(i,k): products in parallel, one ordered subtraction chain
        for (int kk = lane; kk < i; kk += 32)
          row.murow[kk] = __dmul_rn(row.murow[kk], row.rrow[kk]);
        for (int c = lane; c < ncols; c += 32)
          row.vb[c] = __dmul_rn(row.vb[c], row.vb[c]);
        __syncwarp();
        if (lane == 0)
        {
          const double g = serial_chain<false, false>(row.vb[0], row.vb + 1, ncols - 1, nullptr);
          row.gfrow[i]   = g;
          const double a = serial_chain<true, false>(g, row.murow, i, nullptr);
          row.rrow_g[i]  = a;
          row.mu_i[32 * i] = a;  // diagonal mirror
        }
      }
      if (lane == 0)
        S.valid[(size_t)l * S.d + i] = last_j + 1;
      __syncwarp();
    }
    if (ok_out && lane == 0)
      ok_out[l] = live ? 1 : 0;
    ncols = ncols_next, expo = expo_next;
  }
}

// The kernel body.  blockDim.x = 32 * NW; warp c of CTA x owns the lattices (x * NW + c) + k * (gridDim.x * NW).
// Dynamic shared memory: NW x (scratch | ring | mbarriers), then the chunk table (NC descriptors).
__device__ inline void stream_update_rows(const Batch &S, const StreamMaps &M, int i, int last_j, int *ok_out,
                                          double *smem_base)
{
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, NW = blockDim.x >> 5;
  const size_t per     = stream_warp_doubles(S.d, S.n);
  const StreamShape sh = stream_shape(i, last_j);
  const int NC         = stream_num_chunks(sh, S.n);
  StreamDesc *tab      = (StreamDesc *)(smem_base + (size_t)NW * per);
  for (int e = threadIdx.x; e < NC; e += blockDim.x)
    tab[e] = stream_desc(sh, S.n, S.ldb, e);
  if (lane == 0)
  {
    unsigned long long *bars = (unsigned long long *)(smem_base + (size_t)w * per + (per - 16));
    for (int q = 0; q < ST_STAGES; q++)
      tma_mbar_init<1>(bars + q);
    tma_fence_mbar_init();
  }
  __syncthreads();
  const int l = blockIdx.x * NW + w;
  if (l < S.B)
    stream_consumer(S, M, sh, l, gridDim.x * NW, ok_out, smem_base + (size_t)w * per, tab, NC, lane);
}

}  // namespace b200
