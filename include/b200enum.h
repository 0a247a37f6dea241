/* b200enum.h — C-ABI of the GPU-native lattice enumerator (the BKZ SVP subtree search).
 *
 * Drop-in boundary: fplll's external-enumerator hook.  The reference calls a process-wide
 *   std::function<extenum_fc_enumerate>  (fplll/enum/enumerate_ext_api.h:88-92, installed with
 *   set_external_enumerator(), fplll/enum/enumerate_ext.h:100) from Enumeration::enumerate (enum/enumerate.h:87-111)
 * handing it `dim`, the normalised `maxdist`, and three callbacks (set_config / process_sol / process_subsol).
 * std::function cannot cross a C ABI, so b200enum_run below is the C core with exactly that information flattened to
 * plain pointers, and INTEGRATION.md shows the 30-line C++ adapter with the typedef'd signature that a maintainer
 * registers through set_external_enumerator (fplll_b200/csrc/fplll_extenum_adapter.cpp).
 *
 * Scope (SURVEY.md §8 a18/a19, f4): SVP enumeration, primal (what BKZ's svp_reduction asks for, bkz.cpp:329-331 with
 * FastEvaluator(1) — bkz.h:324) and dual (SD-BKZ / slide reduction, bkz.cpp:443-520), with or without sub-solutions:
 * the plugin never has to decline a request of the hook (the bundled enumlib declines dual,
 * enum-parallel/enumlib.cpp:98-104).
 */
#ifndef B200ENUM_H
#define B200ENUM_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200ENUM_MAX_DIM 160

#define B200ENUM_OK 0
#define B200ENUM_EINVAL (-1)
#define B200ENUM_ENODEV (-2)
#define B200ENUM_ECUDA (-3)
#define B200ENUM_UNSUPPORTED (-5)
#define B200ENUM_EOVERFLOW (-6) /* more improving solutions in one wave than the device buffer holds */

/* flags */
#define B200ENUM_FIXED_RADIUS 1 /* never shrink the radius: counts every leaf inside it (known-answer tests) */
#define B200ENUM_DUAL 2         /* dual SVP enumeration (enumerate.cpp:100-124): mut/rdiag are the PRIMAL block's; the
                                 * enumerator forms the reversed dual basis itself and returns coefficients in the
                                 * block's own order */
#define B200ENUM_FINDSUBSOLS 4  /* report the best partial vector per level (enumerate_base.cpp:36-40): b200enum_run_ex */
#define B200ENUM_IPC_HANDLE_BYTES 64

/* extenum_cb_process_sol (enumerate_ext_api.h:62-63): gets the squared length and the coefficient vector of a new
 * solution, returns the new enumeration bound. */
typedef double (*b200enum_sol_cb)(void *ctx, double dist, const double *sol);

/* extenum_cb_process_subsol (enumerate_ext_api.h:70-71): squared length of the partial vector, its coefficients
 * (zero below `offset`) and the level it starts at. */
typedef void (*b200enum_subsol_cb)(void *ctx, double dist, const double *subsol, int offset);

typedef struct
{
  uint64_t host_nodes;   /* nodes visited by the host breadth phase (top levels) */
  uint64_t device_nodes; /* nodes visited by the GPU subtree walkers */
  uint64_t leaves;       /* FIXED_RADIUS: number of non-zero leaves inside the radius (this shard) */
  int top_levels;        /* T: levels expanded on the host */
  int n_roots;           /* subtree roots handed to the GPU(s) (all shards) */
  int n_solutions;       /* improving solutions replayed through the callback */
  int n_devices;
  int n_rounds;          /* kernel rounds (budgeted walk + work split) */
  double final_maxdist;
  float device_ms; /* max over devices of the kernel time (CUDA events on the launching streams) */
  float host_breadth_us; /* wall time of the host breadth phase */
  float total_us;        /* wall time of the whole call */
} b200enum_stats;

/* Enumerate { x in Z^dim, x != 0 :  sum_k rdiag[k] * (x_k + sum_{j>k} mut[k*dim+j] * x_j)^2  <=  pruning[k]-bounded
 * partial sums of maxdist }  in Schnorr-Euchner order (enum/enumerate_base.cpp:152-254).
 *   mut      dim*dim, row-major, mut[k*dim+j] = mu(j,k) for j > k — the `mutranspose=true` layout the hook's set_config
 *            callback fills (enumerate_ext.cpp:108-121); rdiag, pruning: dim each (pruning may be NULL = all ones);
 *            all normalised by 2^-normexp by the caller, as ExternalEnumeration::enumerate does (enumerate_ext.cpp:64-79)
 *   devices  ndev CUDA ordinals driven from this process (NULL = {0}); subtree roots are dealt round-robin
 *   shard_rank/shard_world  additionally restrict this call to roots r with r % shard_world == shard_rank — used when
 *            one process per GPU cooperates (torch.distributed): every rank calls with the same inputs and exchanges
 *            (dist, sol) afterwards.  Use 0/1 otherwise.
 *   cb       called on the host, in order of improvement, for every solution that lowered the radius (FastEvaluator
 *            "best 1" semantics, enum/evaluator.h:122-156); may be NULL
 *   nodes    dim counters (per level, like the array the hook returns), may be NULL
 * Returns B200ENUM_OK or a negative code.  There is no CPU fallback: without a device -> B200ENUM_ENODEV. */
int b200enum_run(int dim, double maxdist, const double *mut, const double *rdiag, const double *pruning, int flags,
                 const int *devices, int ndev, int shard_rank, int shard_world, b200enum_sol_cb cb, void *ctx,
                 uint64_t *nodes, b200enum_stats *stats);

/* Same, plus the sub-solution callback (required with B200ENUM_FINDSUBSOLS): called once per level that has a partial
 * vector shorter than rdiag[level], with the shortest one found (what Evaluator::eval_sub_sol keeps, evaluator.h:191-205). */
int b200enum_run_ex(int dim, double maxdist, const double *mut, const double *rdiag, const double *pruning, int flags,
                    const int *devices, int ndev, int shard_rank, int shard_world, b200enum_sol_cb cb,
                    b200enum_subsol_cb subcb, void *ctx, uint64_t *nodes, b200enum_stats *stats);

/* One process per GPU (torch.distributed): let the ranks' enumerators reach each other's radius words over NVLink (CUDA
 * IPC).  Every rank exports a handle for its device, the job all-gathers the world*64 bytes (NCCL / gloo), every rank
 * attaches.  After that, sharded calls (shard_world == world) push every radius improvement to all peers — enumlib's
 * one shared radius (enum-parallel/enumeration.h:62-81) — instead of running with private radii; the subtree roots are
 * dealt round-robin in order of promise either way.  Ranks must not start call k+1 before every rank has finished call
 * k (the result exchange after each call guarantees that). */
int b200enum_ipc_export(int device, unsigned char *handle64);
int b200enum_ipc_attach(int device, int world, int rank, const unsigned char *handles);
int b200enum_ipc_detach(int device);

const char *b200enum_last_error(void);
int b200enum_device_count(void);

#ifdef __cplusplus
}
#endif
#endif
