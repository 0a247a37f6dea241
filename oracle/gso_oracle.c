/* gso_oracle.c — CPU ORACLE, TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C restatement of the reference's fp64 Gram-Schmidt hot path for the
 * <Z_NR<long>, FP_NR<double>> instantiation (the BKZ regime, bkz.cpp:826-836), written from the
 * algorithm, one function per reference routine, each citing the reference file:line it follows.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this; nothing under
 * fplll_b200/ does.  Parity of this restatement against the real reference is pinned by
 * tests/test_oracle_vs_ref.py (live, through oracle/_ref/ref_probe) and tests/golden/ (committed dumps).
 *
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared (no FMA contraction: the reference is built without -march,
 * configure.ac:25, so FP_NR<double>::addmul is a separately rounded multiply and add, nr_FP_d.inl:177-181).
 *
 * Storage is dense d x d / d x n row-major like the reference's Matrix<FT> (nr/matrix.h:223); entries the
 * reference leaves undefined are undefined here too.  NaN in gf marks an invalid Gram entry (gso.cpp:50-54).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define OGSO_ROW_EXPO 2 /* GSO_ROW_EXPO, gso_interface.h:26-32 */

typedef struct
{
  int d, n, enable_row_expo;
  int n_known_rows, n_known_cols, n_source_rows, cols_locked;
  int64_t *b;        /* d*n  integer basis (int64 wraps silently like Z_NR<long>, nr_Z_l.inl:175) */
  double *bf;        /* d*n  */
  double *gf, *mu, *r; /* d*d */
  int64_t *row_expo; /* d */
  int *gso_valid_cols, *init_row_size; /* d */
  int64_t *tmp_col_expo; /* n */
} ogso_t;

#define B(i, j) m->b[(size_t)(i) * m->n + (j)]
#define BF(i, j) m->bf[(size_t)(i) * m->n + (j)]
#define GF(i, j) m->gf[(size_t)(i) * m->d + (j)]
#define MU(i, j) m->mu[(size_t)(i) * m->d + (j)]
#define R(i, j) m->r[(size_t)(i) * m->d + (j)]

static int imax(int a, int b) { return a > b ? a : b; }
static int imin(int a, int b) { return a < b ? a : b; }

/* NumVect::size_nz (nr/numvect.h): 1 + index of the last non-zero coefficient */
static int size_nz(const int64_t *v, int n)
{
  int i = n;
  while (i > 0 && v[i - 1] == 0)
    i--;
  return i;
}

/* MatGSO::update_bf, gso.cpp:24-48; Z_NR<long>::get_f_exp = frexp((double)x), nr_Z_misc.inl:17-22;
 * FP_NR<double>::mul_2si = ldexp, nr_FP_d.inl:166-169 */
void ogso_update_bf(ogso_t *m, int i)
{
  int n = imax(m->n_known_cols, m->init_row_size[i]);
  if (m->enable_row_expo)
  {
    int64_t max_expo = INT64_MIN;
    for (int j = 0; j < n; j++)
    {
      int e;
      BF(i, j)           = frexp((double)B(i, j), &e);
      m->tmp_col_expo[j] = e;
      if (e > max_expo)
        max_expo = e;
    }
    for (int j = 0; j < n; j++)
      BF(i, j) = ldexp(BF(i, j), (int)(m->tmp_col_expo[j] - max_expo));
    m->row_expo[i] = max_expo;
  }
  else
  {
    for (int j = 0; j < n; j++)
      BF(i, j) = (double)B(i, j);
  }
}

/* MatGSO ctor + size_increased, gso.h:113-130, gso.cpp:368-403 */
ogso_t *ogso_create(int d, int n, const int64_t *b, int flags)
{
  ogso_t *m           = (ogso_t *)calloc(1, sizeof(ogso_t));
  m->d                = d;
  m->n                = n;
  m->enable_row_expo  = (flags & OGSO_ROW_EXPO) ? 1 : 0;
  m->b                = (int64_t *)malloc(sizeof(int64_t) * d * n);
  m->bf               = (double *)calloc((size_t)d * n, sizeof(double));
  m->gf               = (double *)calloc((size_t)d * d, sizeof(double));
  m->mu               = (double *)calloc((size_t)d * d, sizeof(double));
  m->r                = (double *)calloc((size_t)d * d, sizeof(double));
  m->row_expo         = (int64_t *)calloc(d, sizeof(int64_t));
  m->gso_valid_cols   = (int *)calloc(d, sizeof(int));
  m->init_row_size    = (int *)calloc(d, sizeof(int));
  m->tmp_col_expo     = (int64_t *)calloc(n, sizeof(int64_t));
  memcpy(m->b, b, sizeof(int64_t) * d * n);
  for (int i = 0; i < d; i++)
  {
    m->init_row_size[i] = imax(size_nz(&B(i, 0), n), 1);
    ogso_update_bf(m, i); /* bf row was zero-filled first, gso.cpp:399 */
  }
  return m;
}

void ogso_destroy(ogso_t *m)
{
  free(m->b), free(m->bf), free(m->gf), free(m->mu), free(m->r);
  free(m->row_expo), free(m->gso_valid_cols), free(m->init_row_size), free(m->tmp_col_expo);
  free(m);
}

/* invalidate_gram_row, gso.cpp:50-54 */
static void invalidate_gram_row(ogso_t *m, int i)
{
  for (int j = 0; j <= i; j++)
    GF(i, j) = NAN;
}

/* discover_row, gso.cpp:56-82 (float-Gram branch) */
void ogso_discover_row(ogso_t *m)
{
  int i = m->n_known_rows++;
  if (!m->cols_locked)
  {
    m->n_source_rows = m->n_known_rows;
    m->n_known_cols  = imax(m->n_known_cols, m->init_row_size[i]);
  }
  invalidate_gram_row(m, i);
  m->gso_valid_cols[i] = 0;
}

void ogso_discover_all_rows(ogso_t *m) /* gso_interface.h:761-765 */
{
  while (m->n_known_rows < m->d)
    ogso_discover_row(m);
}

/* get_gram, gso.h:314-331, with dot_product of numvect.h:385-395: first term a product, then
 * left-to-right `acc = acc + x*y` with two roundings per term */
double ogso_get_gram(ogso_t *m, int i, int j)
{
  if (GF(i, j) != GF(i, j))
  {
    int n      = m->n_known_cols;
    double acc = BF(i, 0) * BF(j, 0);
    for (int c = 1; c < n; c++)
    {
      double t = BF(i, c) * BF(j, c);
      acc      = acc + t;
    }
    GF(i, j) = acc;
  }
  return GF(i, j);
}

/* update_gso_row, gso_interface.cpp:131-164.  Returns 1 on success, 0 when a mu(i,j) is not finite. */
int ogso_update_gso_row(ogso_t *m, int i, int last_j)
{
  if (i >= m->n_known_rows)
    ogso_discover_row(m);
  int j = imax(0, m->gso_valid_cols[i]);
  for (; j <= last_j; j++)
  {
    double acc = ogso_get_gram(m, i, j);
    for (int k = 0; k < j; k++)
    {
      double t = MU(j, k) * R(i, k);
      acc      = acc - t;
    }
    R(i, j) = acc;
    if (i > j)
    {
      MU(i, j) = acc / R(j, j);
      if (!isfinite(MU(i, j)))
        return 0;
    }
  }
  m->gso_valid_cols[i] = j;
  return 1;
}

int ogso_update_gso(ogso_t *m) /* gso_interface.h:767-775 */
{
  for (int i = 0; i < m->d; i++)
    if (!ogso_update_gso_row(m, i, i))
      return 0;
  return 1;
}

/* row_op_end, gso_interface.cpp:32-53 (float-Gram branch) */
void ogso_row_op_end(ogso_t *m, int first, int last)
{
  for (int i = first; i < last; i++)
  {
    ogso_update_bf(m, i);
    invalidate_gram_row(m, i);
    for (int j = i + 1; j < m->n_known_rows; j++)
      GF(j, i) = NAN;
    m->gso_valid_cols[i] = 0;
  }
  for (int i = last; i < m->n_known_rows; i++)
    m->gso_valid_cols[i] = imin(m->gso_valid_cols[i], first);
}

/* FP_NR<double>::exponent, nr_FP_d.inl:44 */
static long fexponent(double x) { return (long)ilogb(x) + 1; }

/* FP_NR<double>::get_si_exp_we, nr_FP_d.inl:46-53 */
long ogso_get_si_exp_we(double x, long *expo, long expo_add)
{
  if (x == 0)
    *expo = 0;
  else
  {
    long e = fexponent(x) + expo_add - 63;
    *expo  = e > 0 ? e : 0;
  }
  return (long)ldexp(x, (int)(expo_add - *expo));
}

/* FP_NR<double>::rnd_we, nr_FP_d.inl:226-233 */
double ogso_rnd_we(double x, long expo_add)
{
  if (fexponent(x) + expo_add >= 53)
    return x;
  return ldexp(rint(ldexp(x, (int)expo_add)), (int)-expo_add);
}

/* row_addmul_we, gso.cpp:236-262, on b only (u/u_inv_t are empty in the BKZ regime, bkz.cpp:826-836):
 * row_add / row_sub / row_addmul_si / row_addmul_si_2exp, gso.cpp:84-195 via numvect.h:268-341.
 * Z_NR<long> arithmetic wraps (two's complement), so do the math in uint64_t. */
void ogso_row_addmul_we(ogso_t *m, int i, int j, double x, long expo_add)
{
  long expo;
  long lx = ogso_get_si_exp_we(x, &expo, expo_add);
  int n   = m->n_known_cols;
  if (expo == 0)
  {
    if (lx == 0)
      return;
    for (int c = n - 1; c >= 0; c--)
      B(i, c) = (int64_t)((uint64_t)B(i, c) + (uint64_t)B(j, c) * (uint64_t)lx);
  }
  else
  {
    /* row_addmul_si_2exp: tmp = b_j*x; tmp <<= expo (Z_NR<long>::mul_2si, nr_Z_l.inl); b_i += tmp */
    for (int c = n - 1; c >= 0; c--)
    {
      uint64_t t = (uint64_t)B(j, c) * (uint64_t)lx;
      t          = expo >= 64 ? 0 : (t << expo);
      B(i, c)    = (int64_t)((uint64_t)B(i, c) + t);
    }
  }
}

/* row_swap, gso.cpp:264-287: integer rows only */
void ogso_row_swap(ogso_t *m, int i, int j)
{
  for (int c = 0; c < m->n; c++)
  {
    int64_t t = B(i, c);
    B(i, c)   = B(j, c);
    B(j, c)   = t;
  }
}

static void rot_rows_d(double *a, int w, int first, int last, int right)
{ /* Matrix::rotate_right/left on whole rows, nr/matrix.h:186-189 */
  double *tmp = (double *)malloc(sizeof(double) * w);
  if (right)
  {
    memcpy(tmp, a + (size_t)last * w, sizeof(double) * w);
    memmove(a + (size_t)(first + 1) * w, a + (size_t)first * w, sizeof(double) * w * (last - first));
    memcpy(a + (size_t)first * w, tmp, sizeof(double) * w);
  }
  else
  {
    memcpy(tmp, a + (size_t)first * w, sizeof(double) * w);
    memmove(a + (size_t)first * w, a + (size_t)(first + 1) * w, sizeof(double) * w * (last - first));
    memcpy(a + (size_t)last * w, tmp, sizeof(double) * w);
  }
  free(tmp);
}

/* Symmetric row+column rotation of the lower-triangular Gram matrix, Matrix::rotate_gram_{left,right},
 * nr/matrix.cpp:65-93, stated as the permutation it implements: new(i,j) = old_sym(s(i), s(j)), j<=i<nv. */
static void rot_gram(ogso_t *m, int first, int last, int nv, int right)
{
  int d       = m->d;
  double *old = (double *)malloc(sizeof(double) * d * d);
  memcpy(old, m->gf, sizeof(double) * d * d);
  for (int i = first; i < nv; i++)
    for (int j = 0; j <= i; j++)
    {
      int si = i, sj = j;
      if (right)
      {
        if (i >= first && i <= last)
          si = (i == first) ? last : i - 1;
        if (j >= first && j <= last)
          sj = (j == first) ? last : j - 1;
      }
      else
      {
        if (i >= first && i <= last)
          si = (i == last) ? first : i + 1;
        if (j >= first && j <= last)
          sj = (j == last) ? first : j + 1;
      }
      GF(i, j) = si >= sj ? old[(size_t)si * d + sj] : old[(size_t)sj * d + si];
    }
  free(old);
}

static void rot_i64(int64_t *v, int first, int last, int right)
{
  if (right)
  {
    int64_t t = v[last];
    memmove(v + first + 1, v + first, sizeof(int64_t) * (last - first));
    v[first] = t;
  }
  else
  {
    int64_t t = v[first];
    memmove(v + first, v + first + 1, sizeof(int64_t) * (last - first));
    v[last] = t;
  }
}
static void rot_int(int *v, int first, int last, int right)
{
  if (right)
  {
    int t = v[last];
    memmove(v + first + 1, v + first, sizeof(int) * (last - first));
    v[first] = t;
  }
  else
  {
    int t = v[first];
    memmove(v + first, v + first + 1, sizeof(int) * (last - first));
    v[last] = t;
  }
}

/* move_row, gso.cpp:289-366 (float-Gram, no transform) */
void ogso_move_row(ogso_t *m, int old_r, int new_r)
{
  int d = m->d, n = m->n;
  if (new_r < old_r)
  {
    for (int i = new_r; i < m->n_known_rows; i++)
      m->gso_valid_cols[i] = imin(m->gso_valid_cols[i], new_r);
    rot_int(m->gso_valid_cols, new_r, old_r, 1);
    rot_rows_d(m->mu, d, new_r, old_r, 1);
    rot_rows_d(m->r, d, new_r, old_r, 1);
    rot_rows_d((double *)m->b, n, new_r, old_r, 1); /* int64 rows: same width, bit copy */
    rot_gram(m, new_r, old_r, m->n_known_rows, 1);
    rot_rows_d(m->bf, n, new_r, old_r, 1);
    if (m->enable_row_expo)
      rot_i64(m->row_expo, new_r, old_r, 1);
  }
  else if (new_r > old_r)
  {
    for (int i = old_r; i < m->n_known_rows; i++)
      m->gso_valid_cols[i] = imin(m->gso_valid_cols[i], old_r);
    rot_int(m->gso_valid_cols, old_r, new_r, 0);
    rot_rows_d(m->mu, d, old_r, new_r, 0);
    rot_rows_d(m->r, d, old_r, new_r, 0);
    rot_rows_d((double *)m->b, n, old_r, new_r, 0);
    if (old_r < m->n_known_rows - 1)
      rot_gram(m, old_r, imin(new_r, m->n_known_rows - 1), m->n_known_rows, 0);
    rot_rows_d(m->bf, n, old_r, new_r, 0);
    if (m->enable_row_expo)
      rot_i64(m->row_expo, old_r, new_r, 0);
    if (new_r >= m->n_known_rows)
    {
      rot_int(m->init_row_size, old_r, new_r, 0);
      if (old_r < m->n_known_rows)
      {
        m->n_known_rows--;
        m->n_source_rows        = m->n_known_rows;
        m->init_row_size[new_r] = imax(size_nz(&B(new_r, 0), n), 1);
      }
    }
  }
}

/* set_r, gso_interface.h:739-746 */
void ogso_set_r(ogso_t *m, int i, int j, double f)
{
  R(i, j) = f;
  if (m->gso_valid_cols[i] == j)
    m->gso_valid_cols[i]++;
}

/* get_max_mu_exp, gso_interface.cpp:88-98 */
long ogso_get_max_mu_exp(ogso_t *m, int i, int n_columns)
{
  long max_expo = INT64_MIN;
  for (int j = 0; j < n_columns; j++)
  {
    long expo = m->enable_row_expo ? (long)(m->row_expo[i] - m->row_expo[j]) : 0;
    long e2   = fexponent(MU(i, j));
    if (expo + e2 > max_expo)
      max_expo = expo + e2;
  }
  return max_expo;
}

/* ---- LLL driver (lll.cpp), restated so device LLL can be checked call-for-call ---------------------------- */

enum
{
  ORED_SUCCESS       = 0,
  ORED_GSO_FAILURE   = 2,
  ORED_BABAI_FAILURE = 3,
  ORED_LLL_FAILURE   = 4
}; /* defs.h:153-169 */

typedef struct
{
  double delta, eta, swap_threshold;
  int status, n_swaps, final_kappa, zeros;
  long n_babai_iters, n_row_ops;
} olll_t;

/* LLLReduction::babai, lll.cpp:166-224.  X values of the last pass are written to xs (may be NULL). */
int ogso_babai(ogso_t *m, olll_t *L, int kappa, int sr_end, int sr_start, double *babai_mu, long *babai_expo)
{
  long max_expo = INT64_MAX;
  for (int iter = 0;; iter++)
  {
    if (!ogso_update_gso_row(m, kappa, sr_end - 1))
    {
      L->status = ORED_GSO_FAILURE;
      return 0;
    }
    int loop_needed = 0;
    for (int j = sr_end - 1; j >= sr_start && !loop_needed; j--)
    {
      double v = MU(kappa, j);
      if (m->enable_row_expo)
        v = ldexp(v, (int)(m->row_expo[kappa] - m->row_expo[j])); /* get_mu, gso_interface.h:694-701 */
      loop_needed |= (fabs(v) > L->eta);
    }
    if (!loop_needed)
      break;
    if (iter >= 2)
    {
      long nm = ogso_get_max_mu_exp(m, kappa, sr_end);
      if (nm > max_expo - 5) /* SIZE_RED_FAILURE_THRESH, defs.h:146 */
      {
        L->status = ORED_BABAI_FAILURE;
        return 0;
      }
      max_expo = nm;
    }
    for (int j = sr_start; j < sr_end; j++)
    {
      babai_mu[j]   = MU(kappa, j);
      babai_expo[j] = m->enable_row_expo ? (long)(m->row_expo[kappa] - m->row_expo[j]) : 0;
    }
    L->n_babai_iters++;
    for (int j = sr_end - 1; j >= sr_start; j--)
    {
      double x = ogso_rnd_we(babai_mu[j], babai_expo[j]);
      if (x == 0)
        continue;
      for (int k = sr_start; k < j; k++)
      {
        double t    = x * MU(j, k);
        babai_mu[k] = babai_mu[k] - t;
      }
      ogso_row_addmul_we(m, kappa, j, -x, babai_expo[j]);
      L->n_row_ops++;
    }
    ogso_row_op_end(m, kappa, kappa + 1);
  }
  return 1;
}

static int b_row_is_zero(ogso_t *m, int i)
{
  for (int c = 0; c < m->n; c++)
    if (B(i, c))
      return 0;
  return 1;
}

static long get_max_exp_of_b(ogso_t *m) /* Matrix::get_max_exp, Z_NR<long>::exponent nr_Z_l.inl:40-48 */
{
  long mx = 0;
  for (int i = 0; i < m->d; i++)
    for (int c = 0; c < m->n; c++)
    {
      int e;
      int64_t v = B(i, c);
      double f  = frexp((double)v, &e);
      long ex   = e;
      if (v > ((1L << 52) - 1) && fabs(f) == 0.5) /* MAX_LONG_FAST fix-up */
      {
        uint64_t y = (uint64_t)(v < 0 ? -v : v);
        for (ex = 0; y; ex++, y >>= 1)
          ;
      }
      if (ex > mx)
        mx = ex;
    }
  return mx;
}

/* LLLReduction::lll(kappa_min, kappa_start, kappa_end, size_reduction_start), lll.cpp:44-164, with LLL_DEFAULT flags
 * (no early reduction, no siegel).  kappa_end = -1 stands for d (lll.cpp:48-49).  Returns the reference's bool; L->status
 * is only written where the reference calls set_status, so a caller starts it at ORED_SUCCESS like the constructor
 * (lll.cpp:28-29) and the one early `return false` that sets no status (update_gso_row failing at kappa_start,
 * lll.cpp:71-76) leaves it there. */
int ogso_lll_range(ogso_t *m, olll_t *L, int kappa_min, int kappa_start, int kappa_end, int sr_start)
{
  if (kappa_end == -1)
    kappa_end = m->d;
  int d = kappa_end - kappa_min, kappa = kappa_start + 1, ok = 0;
  double *lov = (double *)calloc(kappa_end + 1, sizeof(double));
  double *bmu = (double *)calloc(kappa_end + 1, sizeof(double));
  long *bex   = (long *)calloc(kappa_end + 1, sizeof(long));
  L->swap_threshold = L->delta;
  L->zeros = L->n_swaps = L->final_kappa = 0;
  L->n_babai_iters = L->n_row_ops = 0;
  /* row 0 is tested, row kappa_min is moved: the reference's own loop (lll.cpp:66-69) */
  for (; L->zeros < d && b_row_is_zero(m, 0); L->zeros++)
    ogso_move_row(m, kappa_min, kappa_end - 1 - L->zeros);
  if (L->zeros < d && ((kappa_start > 0 && !ogso_babai(m, L, kappa_start, kappa_start, sr_start, bmu, bex)) ||
                       !ogso_update_gso_row(m, kappa_start, kappa_start)))
  {
    L->final_kappa = kappa_start;
    goto out;
  }
  {
    long long max_iter =
        (long long)(d - 2.0 * d * (d + 1) * ((get_max_exp_of_b(m) + 3) / log(L->delta)));
    long long iter;
    for (iter = 0; iter < max_iter && kappa < kappa_end - L->zeros; iter++)
    {
      if (!ogso_babai(m, L, kappa, kappa, sr_start, bmu, bex))
      {
        L->final_kappa = kappa;
        goto out;
      }
      lov[0] = ogso_get_gram(m, kappa, kappa);
      for (int i = 1; i <= kappa; i++)
      {
        double t = MU(kappa, i - 1) * R(kappa, i - 1);
        lov[i]   = lov[i - 1] - t;
      }
      double thr = R(kappa - 1, kappa - 1) * L->swap_threshold;
      if (m->enable_row_expo)
        thr = ldexp(thr, (int)(2 * (m->row_expo[kappa - 1] - m->row_expo[kappa])));
      if (thr > lov[kappa - 1])
      {
        L->n_swaps++;
        int old_k = kappa;
        for (kappa--; kappa > kappa_min; kappa--)
        {
          double t2 = R(kappa - 1, kappa - 1) * L->swap_threshold;
          if (m->enable_row_expo)
            t2 = ldexp(t2, (int)(2 * (m->row_expo[kappa - 1] - m->row_expo[old_k])));
          if (t2 < lov[kappa - 1])
            break;
        }
        if (lov[kappa] > 0)
          ogso_move_row(m, old_k, kappa);
        else
        {
          L->zeros++;
          ogso_move_row(m, old_k, kappa_end - L->zeros);
          kappa = old_k;
          continue;
        }
      }
      ogso_set_r(m, kappa, kappa, lov[kappa]);
      kappa++;
    }
    L->status = (kappa < kappa_end - L->zeros) ? ORED_LLL_FAILURE : ORED_SUCCESS;
    ok        = L->status == ORED_SUCCESS;
  }
out:
  free(lov), free(bmu), free(bex);
  return ok;
}

/* LLLReduction::size_reduction(kappa_min, kappa_end, size_reduction_start), lll.h:106-122.  Returns the reference's
 * bool; L->status as in ogso_lll_range (a failing update_gso_row returns false without a status, lll.h:118-119). */
int ogso_size_reduction(ogso_t *m, olll_t *L, int kappa_min, int kappa_end, int sr_start)
{
  if (kappa_end == -1)
    kappa_end = m->d;
  double *bmu = (double *)calloc(kappa_end + 1, sizeof(double));
  long *bex   = (long *)calloc(kappa_end + 1, sizeof(long));
  int ok      = 1;
  for (int k = kappa_min; k < kappa_end && ok; k++)
    if ((k > 0 && !ogso_babai(m, L, k, k, sr_start, bmu, bex)) || !ogso_update_gso_row(m, k, k))
      ok = 0;
  if (ok)
    L->status = ORED_SUCCESS;
  free(bmu), free(bex);
  return ok;
}

/* MatGSO::negate_row_of_b, gso.h:291-297 (no integer Gram matrix: the integer row only) */
void ogso_negate_row_of_b(ogso_t *m, int i)
{
  for (int c = 0; c < m->n; c++)
    B(i, c) = (int64_t)(0 - (uint64_t)B(i, c));
}
