/* b200bkz.h — C-ABI of the BKZ driver that runs over the device GSO (b200gso.h) and the device enumerator
 * (b200enum.h): the reference's  bkz_reduction(ZZ_mat<long>-regime, FT_DOUBLE)  — fplll/bkz.h:357-426,
 * fplll/bkz.cpp:522-672 (bkz), :274-358 (svp_reduction, primal and dual), :100-126 (svp_preprocessing), :128-272
 * (svp_postprocessing), :43-80 (rerandomize_block), :360-441 (tour / trunc_tour / hkz), :405-520 (trunc_dtour / sd_tour /
 * slide_tour), :800-809 (BKZAutoAbort).  All three algorithms of the reference's bkz(): BKZ 2.0, self-dual BKZ and slide
 * reduction; only BKZ_DUMP_GSO (0x40) is not supported (B200BKZ_EINVAL).
 *
 * Host C++ keeps only the control flow (which block, which radius, which pruning vector, when to stop); every
 * floating-point GSO update, every LLL / size-reduction call and the enumeration run on the GPU(s).
 * Flags and defaults carry the reference's numeric values (fplll/defs.h:256-274).
 */
#ifndef B200BKZ_H
#define B200BKZ_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200bkz b200bkz_t;

/* BKZFlags, defs.h:264-274 */
#define B200BKZ_DEFAULT 0
#define B200BKZ_VERBOSE 1
#define B200BKZ_NO_LLL 2
#define B200BKZ_MAX_LOOPS 4
#define B200BKZ_MAX_TIME 8
#define B200BKZ_BOUNDED_LLL 0x10
#define B200BKZ_AUTO_ABORT 0x20
#define B200BKZ_GH_BND 0x80
#define B200BKZ_SD_VARIANT 0x100 /* self-dual BKZ: dual tour backwards + primal tour forwards (bkz.cpp:443-463) */
#define B200BKZ_SLD_RED 0x200    /* slide reduction (bkz.cpp:465-520); exclusive with B200BKZ_SD_VARIANT */
/* the error both flags together give, word for word the reference's (bkz.cpp:531-534) */
#define B200BKZ_SD_SLD_MSG "Invalid flags: SD-BKZ and Slide reduction are mutually exclusive!"
/* Not a reference flag.  By default every PRUNED SVP call enumerates the FIXED region of its initial radius and pruning bounds and
 * takes the shortest vector inside it (ties: smallest coefficient vector): a function of the block alone, so a tour is
 * reproducible run to run and across device counts, and never worse than what the reference's walk returns.  With this
 * flag the radius shrinks the moment a walker meets an admissible vector, like the reference's evaluator
 * (enum/evaluator.h:122-156): fewer nodes, but which vector is met first — hence the whole trajectory of a pruned tour —
 * depends on the schedule of thousands of walkers (the reference has the same property with set_threads > 1). */
#define B200BKZ_SHRINK_RADIUS 0x10000

/* RedStatus values this driver can return (defs.h:153-169) */
#define B200_RED_BKZ_FAILURE 6
#define B200_RED_BKZ_TIME_LIMIT 7
#define B200_RED_BKZ_LOOPS_LIMIT 8

#define B200BKZ_EINVAL (-1)
#define B200BKZ_ENODEV (-2)
#define B200BKZ_ECUDA (-3)

typedef struct
{
  int block_size;
  double delta;                   /* LLL_DEF_DELTA 0.99 */
  int flags;
  int max_loops;
  double max_time;                /* seconds */
  double auto_abort_scale;        /* 1.0 */
  int auto_abort_max_no_dec;      /* 5 */
  double gh_factor;               /* 1.1 */
  double min_success_probability; /* 0.5 */
  int rerandomization_density;    /* 3 */
  uint64_t seed;                  /* rerandomisation RNG (the reference uses the GMP global state) */
} b200bkz_param;

typedef struct
{
  int status; /* RedStatus */
  int tours;
  uint64_t enum_nodes;
  long enum_calls, lll_calls, sizered_calls;
  double sec_total, sec_enum, sec_lll, sec_other;
  double sec_ops, sec_get; /* inside sec_other: op-list launches (post-processing, rerandomisation), block read-backs */
  long op_calls, ops_total, get_calls;
  double r00_before, r00_after; /* squared norm of b_0 */
  double slope_before, slope_after;
} b200bkz_stats;

void b200bkz_default_param(b200bkz_param *p, int block_size);

/* devices: CUDA ordinals; the GSO lives on devices[0], enumeration subtrees are dealt over all of them. */
int b200bkz_create(b200bkz_t **out, const int *devices, int ndev);
void b200bkz_destroy(b200bkz_t *h);
/* One Strategy (bkz_param.h:34-66) per block size: preprocessing block sizes and n_prune pruning vectors
 * (gh_factor, expectation, block_size coefficients each) — the content of strategies/default.json for that size.
 * Block sizes without a strategy use the reference's EmptyStrategy (no preprocessing, no pruning). */
int b200bkz_add_strategy(b200bkz_t *h, int block_size, const int *preproc, int n_preproc, const double *gh_factor,
                         const double *expectation, const double *coefficients, int n_prune);
/* bkz_reduction on a d x n int64 basis, in place.  Returns 0 or a negative error; RedStatus in stats->status. */
int b200bkz_reduce(b200bkz_t *h, int d, int n, int64_t *b, const b200bkz_param *param, b200bkz_stats *stats);
/* bkz_reduction(b, u, param) (bkz.h:357-426, BKZReduction with a transform, bkz.cpp:822-836): the same call, and u
 * (d x d int64, row-major, in/out) takes every integer row operation applied to b.  The caller initialises u as for
 * BKZReduction (bkz_reduction itself starts it at the identity, bkz.cpp:857-859).  Same b, status and statistics as
 * b200bkz_reduce; u differs from the reference's where the reference negates a row of b without u (B200GSO_TRANSFORM in
 * b200gso.h), so that U * B_in = B_out always holds here. */
int b200bkz_reduce_transform(b200bkz_t *h, int d, int n, int64_t *b, int64_t *u, const b200bkz_param *param,
                             b200bkz_stats *stats);
const char *b200bkz_last_error(void);
/* get_slide_potential(start_row, end_row, block_size) (gso_interface.cpp:244-258) of an r diagonal given as mantissa /
 * exponent pairs (rows 0 .. end_row - 1): what slide reduction's termination test compares tour to tour. */
double b200bkz_slide_potential_of(const double *rmant, const long *rexpo, int start_row, int end_row, int block_size);

#ifdef __cplusplus
}
#endif
#endif
