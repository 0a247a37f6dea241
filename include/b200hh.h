/* b200hh.h — C-ABI of the GPU-native Householder QR state (the HLLL inner loop's data plane).
 *
 * Stands in for MatHouseholder<Z_NR<long>, FP_NR<double>> (fplll/householder.h:38, fplll/householder.cpp) with
 * HOUSEHOLDER_ROW_EXPO | HOUSEHOLDER_OP_FORCE_LONG — the object HLLLReduction drives (fplll/hlll.h:36,
 * fplll/hlll.cpp:26-173).  Like b200gso.h, a handle is a BATCH of independent d x n lattices resident in HBM and every
 * call applies the same reference call to each lattice.  SURVEY.md §8 rows a11-a17.
 *
 * Arithmetic: each entry point performs the reference's floating-point operations in the reference's order (ascending
 * dot products numvect.h:385-395, separately rounded multiply/add), so R, V, sigma are bit-identical to the
 * reference's.  No CPU fallback: without a device b200hh_create returns B200HH_ENODEV.
 */
#ifndef B200HH_H
#define B200HH_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200hh b200hh_t;

/* MatHouseholderFlags, householder.h:26-32 */
#define B200HH_DEFAULT 0
#define B200HH_ROW_EXPO 1
#define B200HH_OP_FORCE_LONG 4
/* Not a reference value.  The handle also keeps the transform U of MatHouseholder(b, u, u_inv_t, flags) with a
 * non-empty u (householder.h:41-135, enable_transform): int64, d x d per lattice, starting as the identity.  Both
 * integer row operations of HLLL are applied to U with the same index: size_reduce's row_addmul_we(k, i, x, expo_add)
 * adds lx * 2^expo * U[i] to U[k] with the lx and expo it uses for b (householder.cpp:455-559) and the same wrapping
 * int64 arithmetic as Z_NR<long> (a shift by 64 or more gives 0, as on b), over all d columns of U (the reference's
 * u[i].addmul_si(u[j], x) has no n_known_cols bound); swap(i, j) swaps rows i and j of U (householder.cpp:372-398).
 * HLLL never negates a row, so U equals the reference's bit for bit.  No decision reads U: a transform handle ends every
 * call with the same b, R, V, sigma, bf, status and iteration count as a handle without it. */
#define B200HH_TRANSFORM 512
/* Not a reference value.  With B200HH_TRANSFORM only (B200HH_EINVAL otherwise: the reference updates u_inv_t only when
 * u is enabled): the handle also keeps U^-T, the reference's u_inv_t, starting as the identity.  row_addmul_we(k, i, ...)
 * adds (-lx) * 2^expo * U^-T[k] to U^-T[i]; swap(i, j) swaps its rows i and j.  U * (U^-T)^T = I holds mod 2^64. */
#define B200HH_INV_TRANSFORM 1024

#define B200HH_EINVAL (-1)
#define B200HH_ENODEV (-2)
#define B200HH_ECUDA (-3)
#define B200HH_ENOMEM (-4)

/* Widest row update_R and hlll accept: a lane keeps its share of a reflection (ceil(n/32) + 1 elements, the row may
 * start inside a 32-column group) in at most 32 registers.  Wider handles can be created and use the other entry
 * points; b200hh_update_R, b200hh_time_update_R and b200hh_hlll return B200HH_EINVAL for them. */
#define B200HH_MAX_N (32 * 31)

const char *b200hh_last_error(void);

/* MatHouseholder ctor, householder.h:41-135.  b: batch*d*n int64 row-major.  keep_history != 0 allocates the
 * reference's R_history (d*n*n doubles per lattice, householder.h:103-109) so recover_R works; 0 saves the memory
 * (recover_R then fails with B200HH_EINVAL). */
int b200hh_create(b200hh_t **out, int batch, int d, int n, int flags, int device, int keep_history);
void b200hh_destroy(b200hh_t *h);
int b200hh_set_basis(b200hh_t *h, const int64_t *b);
int b200hh_get_basis(b200hh_t *h, int64_t *b);

/* Replace / read back U and U^-T: batch*d*d int64 each, row-major, lattice-major.  Either pointer may be NULL (that matrix
 * is left alone); a non-NULL pointer for a matrix the handle does not keep (no B200HH_TRANSFORM, no
 * B200HH_INV_TRANSFORM) gives B200HH_EINVAL and nothing is copied.  set_basis and hlll leave U and U^-T where they are:
 * hlll continues from the current U. */
int b200hh_set_transform(b200hh_t *h, const int64_t *u, const int64_t *u_inv_t);
int b200hh_get_transform(b200hh_t *h, int64_t *u, int64_t *u_inv_t);

/* refresh_R_bf(i) householder.cpp:186-245; refresh_R(i) :247-261 */
int b200hh_refresh_R_bf(b200hh_t *h, int i);
int b200hh_refresh_R(b200hh_t *h, int i);
/* update_R(i, last_j) householder.cpp:151-184; update_R_last(i) :27-146 */
int b200hh_update_R(b200hh_t *h, int i, int last_j);
int b200hh_update_R_last(b200hh_t *h, int i);
/* size_reduce(k, size_reduction_end, size_reduction_start) householder.cpp:403-451 with row_addmul_we :522-559.
 * reduced[l] (may be NULL) = the reference's bool per lattice. */
int b200hh_size_reduce(b200hh_t *h, int k, int size_reduction_end, int size_reduction_start, int *reduced);
/* swap(i, j) householder.cpp:372-398; recover_R(i) householder.h:597-608; set_updated_R_false householder.h:267 */
int b200hh_swap(b200hh_t *h, int i, int j);
int b200hh_recover_R(b200hh_t *h, int i);
int b200hh_set_updated_R_false(b200hh_t *h);

/* State read-back (any pointer may be NULL): R, V, bf: batch*d*n; sigma, norm_square_b: batch*d; row_expo,
 * expo_norm_square_b: batch*d; meta: batch*3 = {n_known_rows, n_known_cols, updated_R}. */
int b200hh_get_state(b200hh_t *h, double *R, double *V, double *bf, double *sigma, double *norm_square_b,
                     int64_t *row_expo, int64_t *expo_norm_square_b, int *meta);

/* bench helper: `reps` launches of { refresh_R(i); update_R(i, 0) } timed with CUDA events on the handle's stream;
 * *ms_update_mean = mean time of one update_R launch. */
int b200hh_time_update_R(b200hh_t *h, int i, int reps, float *ms_update_mean);

/* HLLLReduction<Z_NR<long>, FP_NR<double>>::hlll() (fplll/hlll.cpp:25-171, with size_reduction :262-354,
 * verify_size_reduction :373-478 and lovasz_test :173-236, all default compile-time branches) over a FRESH
 * MatHouseholder built on the handle's current basis — what hlll_reduction(ZZ_mat<long>&, delta, eta, theta, c,
 * HM_FAST, FT_DOUBLE) runs (fplll/wrapper.cpp:789-806).  The whole loop runs on the device, one warp per lattice of
 * the batch; the handle must have been created with keep_history (recover_R reads R_history).
 * status[batch]: RedStatus per lattice (0 RED_SUCCESS, 10 RED_HLLL_NORM_FAILURE, 11 RED_HLLL_SR_FAILURE; 9 if the
 * device-side iteration guard trips — the reference has no such guard).  iterations[batch] (optional): main-loop
 * trips.  The reduced bases are read back with b200hh_get_basis; on a B200HH_TRANSFORM handle U (and U^-T) have taken
 * every row operation of the call, starting from what they held (b200hh_get_transform). */
int b200hh_hlll(b200hh_t *h, double delta, double eta, double theta, double c, int *status, uint64_t *iterations);
int b200hh_sync(b200hh_t *h);

#ifdef __cplusplus
}
#endif
#endif
