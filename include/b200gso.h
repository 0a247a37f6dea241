/* b200gso.h — C-ABI of the GPU-native Gram-Schmidt (GSO) state.
 *
 * Drop-in boundary for fplll's fp64 GSO hot path (SURVEY.md §8b).  The reference has no FFI: its boundary is the
 * C++ class MatGSO<Z_NR<long>, FP_NR<double>> (fplll/gso.h:33, fplll/gso_interface.h:59) whose non-virtual
 * accessors read mu/r directly, so a drop-in replaces the translation units gso.cpp / gso_interface.cpp with a
 * thin class that forwards every method to one entry point below (see INTEGRATION.md for that adapter).
 * Every function cites the reference method it stands in for.
 *
 * A handle owns the state of a BATCH of `batch` independent lattices of identical shape d x n, all resident in
 * HBM (batch = 1 is the reference's single MatGSO object; the batch axis is the replica axis of SURVEY §8e).
 * Batched calls apply the same reference call to every lattice of the batch; arguments that the reference takes
 * per object (x of row_addmul_we, results of update_gso_row) are arrays of length `batch`.
 *
 * All functions return 0 on success or a negative B200GSO_E* code; reduction outcomes use the reference's own
 * RedStatus values (fplll/defs.h:153-169).  No function falls back to the CPU: without a CUDA device
 * b200gso_create fails with B200GSO_ENODEV.
 *
 * Plain C: pointers are HOST pointers unless named dev_*; no torch/STL types.
 */
#ifndef B200GSO_H
#define B200GSO_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200gso b200gso_t;

/* MatGSOInterfaceFlags, fplll/gso_interface.h:26-32.  GSO_INT_GRAM is not supported on the device (SURVEY §2 #3:
 * out of scope); GSO_OP_FORCE_LONG is implied (the device integer mirror is int64, like Z_NR<long>). */
#define B200GSO_DEFAULT 0
#define B200GSO_ROW_EXPO 2
#define B200GSO_OP_FORCE_LONG 4
/* The integer basis stays on the HOST in GMP (MatGSO<Z_NR<mpz_t>, FP_NR<double>>, the LLL stage-1 regime of
 * wrapper.cpp:538-553): the device holds bf / row_expo and the fp64 state only.  The host does every integer row
 * operation itself and ships the refreshed floating-point row with b200gso_upload_row_fp; the int64 entry points
 * (set_basis, row_addmul_we, upload_row, device LLL) are rejected on such a handle. */
#define B200GSO_HOST_BASIS 256

/* RedStatus, fplll/defs.h:153-169 */
#define B200_RED_SUCCESS 0
#define B200_RED_GSO_FAILURE 2
#define B200_RED_BABAI_FAILURE 3
#define B200_RED_LLL_FAILURE 4

#define B200GSO_EINVAL (-1)
#define B200GSO_ENODEV (-2)
#define B200GSO_ECUDA (-3)
#define B200GSO_ENOMEM (-4)

/* Library / device probes (no reference counterpart). */
const char *b200gso_version(void);
int b200gso_device_count(void);
const char *b200gso_last_error(void);

/* MatGSO::MatGSO(b, u={}, u_inv_t={}, flags) + size_increased(): gso.h:113-130, gso.cpp:368-403.
 * b: batch*d*n int64, row-major, lattice-major.  Converts every row to bf (update_bf, gso.cpp:24-48). */
int b200gso_create(b200gso_t **out, int batch, int d, int n, int flags, int device);
void b200gso_destroy(b200gso_t *h);
int b200gso_set_basis(b200gso_t *h, const int64_t *b);
/* Same, from a device-resident int64 buffer (batch*d*n, row-major). */
int b200gso_set_basis_dev(b200gso_t *h, const int64_t *dev_b);
/* The integer basis back to the host (the caller-owned `Matrix<ZT>& b` of gso.h:136). */
int b200gso_get_basis(b200gso_t *h, int64_t *b);

/* Uploads replacement contents for row i of every lattice (batch*n int64) — the protocol of SURVEY §7 for a host
 * that performs the integer row operation itself: equivalent to writing b[i] then row_op_end(i, i+1). */
int b200gso_upload_row(b200gso_t *h, int i, const int64_t *rows);

/* MatGSOInterface::discover_all_rows, gso_interface.h:761-765 */
int b200gso_discover_all_rows(b200gso_t *h);
/* discover_row() (gso.cpp:56-82) until n_known_rows == upto: what a host driver that discovers rows itself (the
 * MatGSO forwarding shim, INTEGRATION.md) uses to keep the device in step. */
int b200gso_discover_rows(b200gso_t *h, int upto);

/* MatGSOInterface::update_gso_row(i, last_j), gso_interface.cpp:131-164.  ok[l] = 1/0 as the reference's bool
 * (0: a mu(i,j) is not finite -> caller reports RED_GSO_FAILURE).  ok may be NULL. */
int b200gso_update_gso_row(b200gso_t *h, int i, int last_j, int *ok);
/* MatGSOInterface::update_gso, gso_interface.h:767-775 */
int b200gso_update_gso(b200gso_t *h, int *ok);
/* update_gso() with the whole float Gram matrix recomputed first in 32 x 32 tiles — the blocked form of get_gram
 * (gso.h:314-331) — then the row sweeps (bit-exact with B200GSO_GRAM_ORDERED, within 1e-9 otherwise).  B200GSO_GRAM_ORDERED keeps the reference's left-to-right dot products (bit-identical state);
 * B200GSO_GRAM_DMMA uses fp64 tensor-core mma.m8n8k4 (identical only where every partial sum is exact). */
#define B200GSO_GRAM_ORDERED 0
#define B200GSO_GRAM_DMMA 1
int b200gso_update_gso_blocked(b200gso_t *h, int gram_mode, int *ok);

/* GSO_INT_GRAM objects (exact integer Gram matrix kept on the host, gso.cpp:140-159, gso_gram.cpp): get_gram(i, j) for
 * j < count (gso.h:314-331, integer branch: the exact entry converted to double) written as row i of the float Gram
 * matrix, so that the next update_gso_row(i, .) finds its Gram entries valid and only does the forward substitution.
 * vals: batch * count doubles.  The handle is a B200GSO_HOST_BASIS one without row exponents (the reference forbids
 * GSO_ROW_EXPO together with GSO_INT_GRAM, gso.h:116). */
int b200gso_set_gram_row(b200gso_t *h, int i, int count, const double *vals);

/* MatGSO::row_addmul_we(i, j, x, expo_add), gso.cpp:236-262: b_i += x * 2^expo_add * b_j with x an integer-valued
 * double converted by get_si_exp_we (nr_FP_d.inl:46-53).  x, expo_add: arrays of length batch. */
int b200gso_row_addmul_we(b200gso_t *h, int i, int j, const double *x, const long *expo_add);
/* MatGSOInterface::row_op_begin / row_op_end, gso_interface.h:172-178, gso_interface.cpp:32-53 */
int b200gso_row_op_begin(b200gso_t *h, int first, int last);
int b200gso_row_op_end(b200gso_t *h, int first, int last);
/* MatGSO::row_swap(i, j), gso.cpp:264-287 (integer rows only; bracket with row_op_begin/end) */
int b200gso_row_swap(b200gso_t *h, int i, int j);
/* MatGSO::move_row(old_r, new_r), gso.cpp:289-366 */
int b200gso_move_row(b200gso_t *h, int old_r, int new_r);
/* MatGSOInterface::set_r(i, j, f), gso_interface.h:739-746; f: array of length batch */
int b200gso_set_r(b200gso_t *h, int i, int j, const double *f);

/* State read-back, dense like the reference's Matrix<FT> (get_mu_matrix / get_r_matrix, gso_interface.h:207-214):
 * mu, r, gf: batch*d*d (row-major, entries the reference leaves undefined are 0 / NaN for invalid Gram);
 * bf: batch*d*n; row_expo: batch*d; gso_valid_cols, init_row_size: batch*d;
 * meta: batch*4 = {n_known_rows, n_known_cols, n_source_rows, cols_locked}.  Any pointer may be NULL. */
int b200gso_get_state(b200gso_t *h, double *mu, double *r, double *gf, double *bf, int64_t *row_expo,
                      int *gso_valid_cols, int *init_row_size, int *meta);

/* Rows i of mu and r for every lattice (batch*d each; entries j >= gso_valid_cols are unspecified) and
 * gso_valid_cols[i] (batch) — what LLLReduction::babai reads after update_gso_row (lll.cpp:166-224). */
int b200gso_get_mu_r_row(b200gso_t *h, int i, double *mu_row, double *r_row, int *valid);

/* Device LLL over every lattice of the batch: LLLReduction<Z_NR<long>,FP_NR<double>>::lll(0,0,d) with
 * LLL_DEFAULT flags, lll.cpp:44-164, including babai (lll.cpp:166-224).  status[l] = RedStatus.
 * stats (may be NULL): batch*4 = {n_swaps, final_kappa, zeros, babai_iterations}. */
int b200gso_lll(b200gso_t *h, double delta, double eta, int *status, long *stats);

/* LLLReduction::lll(kappa_min, kappa_start, kappa_end, size_reduction_start), lll.cpp:44-164 (kappa_end = -1: d). */
int b200gso_lll_range(b200gso_t *h, double delta, double eta, int kappa_min, int kappa_start, int kappa_end,
                      int size_reduction_start, int *status, long *stats);
/* LLLReduction::size_reduction(kappa_min, kappa_end, size_reduction_start), lll.h:106-122.  status[l] = RedStatus. */
int b200gso_size_reduction(b200gso_t *h, double eta, int kappa_min, int kappa_end, int size_reduction_start,
                           int *status);
/* MatGSO::negate_row_of_b(i), gso.h:291-297 (bracket with row_op_begin/end like the reference's callers). */
int b200gso_negate_row_of_b(b200gso_t *h, int i);
/* What Enumeration pulls out of the GSO for block [first, first+beta) of lattice `lattice` (enumerate.cpp:91-141,
 * enumerate_ext.cpp:91-148): mut[k*beta+j] = get_mu(first+j, first+k) for j > k (true value, row exponents applied)
 * and get_r_exp(first+i, first+i) as mantissa r_mant[i] and exponent r_expo[i]. */
int b200gso_get_block(b200gso_t *h, int lattice, int first, int beta, double *mut, double *r_mant, long *r_expo);

/* A recorded sequence of the calls above, executed in order by ONE kernel launch on every lattice of the batch —
 * what BKZ's svp_postprocessing / rerandomize_block issue as dozens of individual calls (bkz.cpp:43-80,128-272). */
typedef struct
{
  int type, a, b, pad; /* ROW_ADDMUL: row_addmul(a, b, x); MOVE_ROW: move_row(a, b); ROW_SWAP: row_swap(a, b); */
  double x;            /* ROW_OP_END: row_op_end(a, b); NEGATE: negate_row_of_b(a) */
} b200gso_op;
#define B200GSO_OP_ROW_ADDMUL 1
#define B200GSO_OP_MOVE_ROW 2
#define B200GSO_OP_ROW_SWAP 3
#define B200GSO_OP_ROW_OP_END 4
#define B200GSO_OP_NEGATE 5
int b200gso_apply_ops(b200gso_t *h, const b200gso_op *ops, int n);

/* get_r_exp(first+i, first+i) for i < count of lattice `lattice` (gso_interface.h:704-722): mantissa and exponent. */
int b200gso_get_r_diag(b200gso_t *h, int lattice, int first, int count, double *r_mant, long *r_expo);

/* Timing helper for bench.py: runs `reps` back-to-back steps { row_op_end(i,i+1); update_gso_row(i,i) }
 * (invalidate != 0) or { invalidate_gso_row(i,0); update_gso_row(i,i) } on the handle's stream, timed with CUDA
 * events ON THAT STREAM: *ms_update_mean = mean device time of ONE update_gso_row launch (events around each
 * launch), *ms_total = device time of the whole region (all 2*reps launches).  Either pointer may be NULL. */
int b200gso_time_update_row(b200gso_t *h, int i, int reps, int invalidate, float *ms_update_mean, float *ms_total);

/* Number of lattices the update_gso_row kernel keeps resident at once on this device (SMs x CTAs/SM x warps/CTA):
 * batches that are a multiple of it run in full waves.  Negative on error. */
int b200gso_resident_lattices(b200gso_t *h);

/* Host-basis handles (B200GSO_HOST_BASIS): row i of every lattice was rewritten on the host (row_addmul_we on the
 * mpz rows, gso.cpp:236-262) and converted there exactly as update_bf does for Z_NR<mpz_t> (mpz_get_d_2exp,
 * gso.cpp:24-48, nr_Z_misc.inl:114-147): bf_rows[l*n + c] = mantissa of b(i,c) scaled by 2^-row_expo, expo[l] = the
 * row's exponent (0 without GSO_ROW_EXPO).  The device stores the row and does the rest of row_op_end(i, i+1)
 * (gso_interface.cpp:32-53): Gram row / column and GSO row invalidated, validity of later rows lowered.
 * A never-seen row (i >= n_known_rows) may be uploaded before it is discovered. */
int b200gso_upload_row_fp(b200gso_t *h, int i, const double *bf_rows, const long *expo);

/* Profiling builds only (-DB200_LLL_PROFILE): device-clock phase counters of the last LLL call of this process
 * (update_gso_row, Babai rest, Lovasz, move_row+set_r, gather/scan, back-substitution, integer rows, row_op_end).
 * All zero in release builds.  `stats` of b200gso_lll is always batch*4 longs. */
int b200gso_lll_profile(long *out8);
/* ... and the counters of the CTA-cooperative operations, accumulated over the process (slots: csrc/gso_cta.cuh). */
int b200gso_lll_cta_profile(long long *out32);

/* Synchronise the handle's stream (all calls above are stream-ordered on one stream per handle). */
int b200gso_sync(b200gso_t *h);

#ifdef __cplusplus
}
#endif
#endif
