// enum_api.cu — GPU-native Schnorr-Euchner enumeration (BKZ's SVP subtree search) behind include/b200enum.h.
//
// Reference algorithm: EnumerationBase::enumerate_loop (fplll/enum/enumerate_base.cpp:152-254) + next_pos_up
// (enumerate_base.h:145-171); the only parallel strategy in the reference is enumlib's subtree fan-out over
// std::threads with one shared radius and a shared subtree counter (fplll/enum-parallel/enumeration.h:62-81,
// 382-510).  Device design:
//   1. HOST BREADTH PHASE  — the top T levels (d-1 .. d-T) are expanded level by level, each level in exact
//      Schnorr-Euchner order, into subtree roots (x[d-T..d-1], partial length).  T grows until there are enough roots
//      to seed the machine.  Roots are sorted by partial length so the most promising subtrees run first (enumlib does
//      the same, enumeration.h:417-422).
//   2. DEVICE DEPTH PHASE  — one THREAD per task ("walk the remaining siblings of level l under a fixed prefix"), tasks
//      handed out by an atomic ticket; walkers that exhaust a node budget (or notice that the round ran dry) turn the
//      unvisited parts of their subtree into tasks of the next round.  All rounds run inside one persistent cooperative
//      launch (k_enum), separated by grid barriers.
//   3. RADIUS — one 8-byte word per device, lowered with atomicMin on the bit pattern of the (positive) squared length;
//      walkers re-read it between tasks and every 64 steps: FastEvaluator "best 1" semantics (enum/evaluator.h:122-156),
//      which is what BKZ uses (bkz.h:324).  With several devices the finder of a shorter vector PUSHES the new radius
//      into every peer's word with a system-scope atomicMin over NVLink (peer-mapped memory: cudaDeviceEnablePeerAccess
//      inside one process, CUDA IPC between the processes of a torch.distributed job) — the reference's one shared
//      atomic radius (enumeration.h:62-81), without anybody polling remote memory.
//   4. HAND-OFF — small enumerations (all but a handful of the ~18 k calls of a BKZ-60 tour) never leave device 0.  A
//      call that is still busy after `fan_nodes` nodes SUSPENDS at a round boundary; its pending task queue is copied to
//      every other device over NVLink (cudaMemcpyPeer) and all devices — the first one included — resume from it,
//      claiming tasks from ONE shared ticket in device 0's memory (system-scope atomicAdd), the device-side form of
//      enumlib's shared subtree counter (enumeration.h:460-475).  One-process-per-GPU jobs (sharded calls) deal the host's
//      subtree roots round-robin in order of promise — 8192 roots, so the deal balances a heavy-tailed tree — and push
//      radius improvements into each other's words, reached through CUDA IPC (b200enum_ipc_*).
// Arithmetic: every centre is the chain ((0 - x[d-1] mu) - x[d-2] mu) - ... in descending j with separately rounded
// multiply and subtract (--fmad=false), the order of the reference's center_partsums, so with a fixed radius the set
// of visited nodes — and therefore the node count — is identical to the reference's own enumerator.
// Dual enumeration (enumerate_base.cpp:64-68: the chain runs over alpha_j = x_j - c_j instead of x_j, on the reversed
// inverted basis, enumerate.cpp:100-124) runs in both kernel variants: the shared-memory one keeps alpha next to x.
// Sub-solutions (enumerate_base.cpp:36-40) are served by the thread-local variant only.
#include "../../include/b200enum.h"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <deque>
#include <mutex>
#include <string>
#include <vector>

namespace {

thread_local std::string g_err;
#define CKE(call)                                                                                  \
  do                                                                                               \
  {                                                                                                \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
    {                                                                                              \
      g_err = std::string(#call) + ": " + cudaGetErrorString(e_);                                  \
      return B200ENUM_ECUDA;                                                                       \
    }                                                                                              \
  } while (0)

constexpr int SOL_CAP    = 4096;     // improving solutions of one call (device list)
constexpr int SOL_FAST   = 8;        // ... of which this many travel with the result block (one D2H copy per call)
constexpr int SUB_CAP    = 1 << 14;  // improving sub-solutions of one call (findsubsols)
constexpr int THREADS    = 128;
constexpr int THREADS_XS = 512;      // upper bound of the CTA size of the x-in-shared-memory variant (one CTA per SM)
constexpr int MIN_ROOTS  = 128;      // host breadth phase: grow T until at least this many roots (the device multiplies
                                     // them by work splitting, a round costs one grid barrier) ...
constexpr int MAX_ROOTS  = 1 << 15;  // ... but never beyond this (the pinned staging block is sized for it)
constexpr int SMEM_XS_MAX = 227 * 1024;  // opt-in dynamic shared memory per CTA on sm_90
constexpr unsigned TASK_CAP = 1u << 21;  // device task queue capacity (tasks of one round)
constexpr int MAX_PEERS = 8;
constexpr unsigned long long INF_BITS = 0x7ff0000000000000ull;

// device words (one block of 16 per device context)
enum
{
  W_A = 0,      // radius (bit pattern of a positive double)
  W_BEST = 1,   // best-so-far in fixed-radius mode
  W_LEAVES = 2,
  W_SOLC = 3,   // unsigned[2]: improving solutions, improving sub-solutions
  W_CTR = 4,    // unsigned[4]: ticket, tail, tasks of the next round, rounds done
  W_FLAGS = 6,  // unsigned[2]: round 0 of a shared-ticket run has run dry, call suspended
  W_NODES = 7,  // nodes visited so far (all rounds, this device)
  W_GTICKET = 8,  // the SHARED ticket (device 0 / rank 0 owns the word everybody claims from): epoch << 32 | count
  W_COUNT = 16
};

struct SolRec
{
  double dist;
  int lvl, pad;  // sub-solutions: the level (offset) the partial vector starts at
  int x[B200ENUM_MAX_DIM];
};

// A unit of work: "at level lvl, with x[lvl+1..d-1] fixed, walk the remaining siblings starting at x[lvl] = xs (in
// Schnorr-Euchner order around cen) and everything below them".  The host's subtree roots are tasks; a walker that
// has used up its node budget turns the unvisited siblings of every ancestor on its path into new tasks (the classic
// depth-first work split), so the heavy-tailed subtree sizes of pruned enumeration get re-balanced between rounds.
struct TaskHdr
{
  double pd, cen, xs;
  int lvl, pad;
};

struct EnumArgs
{
  int d, dstride;              // dim; task prefix row stride (d rounded up to a multiple of 4 ints)
  const double *mut, *rdiag, *prun;
  const TaskHdr *hdr_first;    // round 0 reads its tasks here (the staged roots, or a handed-off queue) ...
  const int *tx_first;
  TaskHdr *hdrq[2];            // ... and round r >= 0 appends to half (out0 + r) & 1, which round r + 1 reads
  int *txq[2];                 // [TASK_CAP * dstride] coefficients by absolute level (entries > lvl are meaningful)
  int out0;
  unsigned n_first;            // number of tasks of round 0
  unsigned long long *words;   // W_* above
  unsigned long long *gticket; // shared ticket for round 0 (peer memory), or null: the local ticket
  unsigned gepoch;             // ... its epoch for this call
  int share_div;               // devices sharing round 0 (sizes the warp spreading)
  unsigned long long *A_peer[MAX_PEERS];  // the other devices' radius words
  int n_peer;
  unsigned long long node_cap; // suspend at a round boundary once this many nodes are visited (0 = never)
  unsigned yield_nodes;          // a walker re-checks the split / yield conditions every this many nodes ...
  unsigned yield_small;          // ... or this many, in a round with fewer tasks than warps
  unsigned budget0, budget_mul;  // nodes a walker may visit before it must split: budget0 * mul^round (capped)
  unsigned long long *nodes;   // [d]
  SolRec *sols_fast, *sols_more;
  SolRec *subs;                // findsubsols records
  unsigned long long *sub_bits;  // [d] best sub-solution length per level
  int fixed_radius, dual, findsubsols;
};

__device__ inline double next_sibling(double x, double c, double pdk)
{
  // next_pos_up's coefficient update (enumerate_base.h:145-171) with the zig-zag state (dx, ddx) re-derived from
  // (x, centre): x0 = round(c), s = +1 if c >= x0 else -1, sequence x0, x0+s, x0-s, x0+2s, ...
  if (pdk == 0.0)
    return x + 1.0;  // SVP: only the positive half at the top non-zero coefficient
  const double x0 = round(c), s = (c >= x0) ? 1.0 : -1.0, t = x - x0;
  return (t == 0.0) ? x0 + s : ((t * s > 0.0) ? x0 - t : x0 - t + s);
}

__device__ inline unsigned long long atomic_min_sys(unsigned long long *p, unsigned long long v)
{
  unsigned long long old;
  asm volatile("atom.global.sys.min.u64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(v) : "memory");
  return old;
}
__device__ inline void red_min_sys(unsigned long long *p, unsigned long long v)
{
  asm volatile("red.global.sys.min.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ inline unsigned long long atomic_add_sys(unsigned long long *p, unsigned long long v)
{
  unsigned long long old;
  asm volatile("atom.global.sys.add.u64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(v) : "memory");
  return old;
}

// ------------------------------------------------------------------------------------------------------------
// device depth phase
// Persistent cooperative kernel: ALL rounds of one enumeration run inside one launch, separated by grid-wide barriers
// (a round = every walker works off the current half of the task queue, walkers that split or yield append to the other
// half).  One launch per Enumeration::enumerate call instead of one launch + host synchronisation per round.
//
// XS = true (dim <= 64, every BKZ block size in use; no sub-solutions): the coefficient vectors x[] of all
// walkers of the CTA live in SHARED memory ([level][thread], conflict-free) — the centre chain reads x[j] d-k times per
// node, and with x[] in thread-local memory that traffic (L1 misses for 3/4 of it, ~1.6 KB of L2 reads per node) was
// what bounded the first version.  One CTA per SM then shares a single copy of mu^T.  XDUAL = true is the dual
// instantiation: the chains read alpha_j, kept in a second [level][thread] array right after x[] (two d-vectors per
// walker, so the CTA has fewer walkers: launch_shape).  The primal instantiation is compiled without it.
// Both variants also keep pre[k] = the part of level k's centre chain that only involves the task's FIXED coefficients
// (j > top0): it is computed the first time the walker reaches level k inside a task and is the exact prefix of the
// reference's descending chain, so the remaining chain is top0-k long instead of d-1-k.
template <int ML, bool XS, bool XDUAL = false>
__global__ void __launch_bounds__(XS ? THREADS_XS : THREADS) k_enum(EnumArgs a)
{
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  extern __shared__ __align__(16) double sm[];
  const int d  = a.d;
  const int ds = XS ? (d | 1) : d;  // odd row stride: walkers on different levels read different rows of mu^T
  double *s_mut = sm, *s_r = sm + (size_t)d * ds, *s_p = s_r + d;
  double *s_x = s_p + d + threadIdx.x;  // XS: x[j] of this thread at s_x[j * blockDim.x]
  const int xstr = blockDim.x;
  double *s_al = s_x + (size_t)d * xstr;  // XS dual: alpha[j] of this thread at s_al[j * blockDim.x]
  for (int t = threadIdx.x; t < d * d; t += blockDim.x)
    s_mut[(t / d) * ds + (t % d)] = a.mut[t];
  for (int t = threadIdx.x; t < d; t += blockDim.x)
  {
    s_r[t] = a.rdiag[t];
    s_p[t] = a.prun[t];
  }
  __syncthreads();
  const bool DUAL = XS ? XDUAL : (a.dual != 0), SUBS = !XS && a.findsubsols;

  double xl[XS ? 1 : ML], al[XS ? 1 : ML], cen[ML], pd[ML], pre[ML];
  unsigned cnt[ML];
  auto getx = [&](int j) -> double { return XS ? s_x[(size_t)j * xstr] : xl[XS ? 0 : j]; };
  auto setx = [&](int j, double val) {
    if (XS)
      s_x[(size_t)j * xstr] = val;
    else
      xl[XS ? 0 : j] = val;
  };
  auto getal = [&](int j) -> double { return XS ? s_al[(size_t)j * xstr] : al[XS ? 0 : j]; };
  auto setal = [&](int j, double val) {
    if (XS)
      s_al[(size_t)j * xstr] = val;
    else
      al[XS ? 0 : j] = val;
  };
  // what the centre chains multiply mu with: x_j, or alpha_j = x_j - c_j in a dual enumeration
  auto chainv = [&](int j) -> double { return DUAL ? getal(j) : getx(j); };
  int top0 = 0, pvalid = 0;
#pragma unroll 1
  for (int k = 0; k < d; k++)
    cnt[k] = 0;
  unsigned long long my_leaves = 0;
  unsigned long long *A_bits = a.words + W_A;
  unsigned *ctr = (unsigned *)(a.words + W_CTR), *flags = (unsigned *)(a.words + W_FLAGS);
  unsigned *sol_count = (unsigned *)(a.words + W_SOLC);
  double A     = __longlong_as_double(*(volatile unsigned long long *)A_bits);
  int steps    = 0;
  unsigned end = a.n_first, budget = a.budget0;

  for (unsigned rno = 0;; ++rno)
  {
  const TaskHdr *hdr_in = rno == 0 ? a.hdr_first : a.hdrq[(a.out0 + rno - 1) & 1];
  const int *tx_in      = rno == 0 ? a.tx_first : a.txq[(a.out0 + rno - 1) & 1];
  TaskHdr *hdr_out      = a.hdrq[(a.out0 + rno) & 1];
  int *tx_out           = a.txq[(a.out0 + rno) & 1];
  unsigned *ticket = ctr, *tail = ctr + 1;
  const bool shared_round     = (rno == 0 && a.gticket != nullptr);
  const unsigned total_warps  = gridDim.x * (blockDim.x >> 5);
  const unsigned my_share     = shared_round ? (end + a.share_div - 1) / a.share_div : end;
  const unsigned lanes_allowed = min(32u, max(1u, (my_share + total_warps - 1) / total_warps));
  int k        = -2;  // -2: idle (needs a task)
  int top      = 0;   // highest level this walker still owns
  unsigned n   = 0;   // nodes since the last split
  unsigned nr  = 0;   // nodes of this round
  const unsigned ynodes = (my_share < total_warps) ? a.yield_small : a.yield_nodes;
  unsigned next_check = ynodes;
  for (;;)
  {
    if (k == -2)
    {
      // a round with fewer tasks than lanes is spread over WARPS first: 32 walkers of one warp sit on different
      // levels and serialise each other (SIMT divergence), a lone walker in a warp runs at full single-thread speed
      if ((threadIdx.x & 31u) >= lanes_allowed)
        break;
      unsigned t;
      if (shared_round)
      {
        if (*(volatile unsigned *)flags)  // somebody on this device already saw the shared ticket run out
          break;
        const unsigned long long w = atomic_add_sys(a.gticket, 1ull);
        t = ((unsigned)(w >> 32) == a.gepoch) ? (unsigned)w : 0xffffffffu;
        if (t >= end)
          *(volatile unsigned *)flags = 1u;
      }
      else
        t = atomicAdd(ticket, 1u);
      if (t >= end)
        break;
      const TaskHdr h = hdr_in[t];
      const int4 *tx4 = (const int4 *)(tx_in + (size_t)t * a.dstride);
      A               = __longlong_as_double(*(volatile unsigned long long *)A_bits);
      top = k = h.lvl;
      top0 = pvalid = k;
      // prefix x[lvl+1 .. d-1]: 128-bit loads, 4 in flight (a walker that starts a task stalls its whole warp, so
      // this must cost one memory latency, not d of them)
#pragma unroll 4
      for (int j4 = (k + 1) >> 2; j4 < (a.dstride >> 2); j4++)
      {
        const int4 q = tx4[j4];
        const int j  = 4 * j4;
        if (j > k && j < d)
          setx(j, (double)q.x);
        if (j + 1 > k && j + 1 < d)
          setx(j + 1, (double)q.y);
        if (j + 2 > k && j + 2 < d)
          setx(j + 2, (double)q.z);
        if (j + 3 > k && j + 3 < d)
          setx(j + 3, (double)q.w);
      }
      if (DUAL)
      {
        // alpha_j of the fixed prefix, top down: c_j is the descending chain over alpha_i, i > j (the values the
        // walker that created the task had)
#pragma unroll 1
        for (int j = d - 1; j > k; --j)
        {
          double c = 0.0;
          const double *mr = s_mut + (size_t)j * ds;
#pragma unroll 1
          for (int i = d - 1; i > j; --i)
            c = __dsub_rn(c, __dmul_rn(getal(i), mr[i]));
          setal(j, __dsub_rn(getx(j), c));
        }
      }
      pd[k]  = h.pd;
      cen[k] = h.cen;
      setx(k, h.xs);
      n      = 0;
      next_check = ynodes;
    }

    // ---- one step of enumerate_loop (enumerate_base.cpp:193-254) ----
    const double xk      = getx(k);
    const double alphak  = __dsub_rn(xk, cen[k]);
    const double newdist = __dadd_rn(pd[k], __dmul_rn(__dmul_rn(alphak, alphak), s_r[k]));
    bool up              = true;
    if (newdist <= __dmul_rn(s_p[k], A))
    {
      cnt[k]++;
      n++;
      nr++;
      if (DUAL)
        setal(k, alphak);
      if (SUBS && newdist != 0.0 && newdist < __longlong_as_double(*(volatile unsigned long long *)(a.sub_bits + k)))
      {
        // sub-solution (enumerate_base.cpp:36-40): best partial vector per level; the host keeps the per-level minimum
        const unsigned long long nb = (unsigned long long)__double_as_longlong(newdist);
        if (nb < atomicMin(a.sub_bits + k, nb))
        {
          const unsigned slot = atomicAdd(sol_count + 1, 1u);
          if (slot < SUB_CAP)
          {
            SolRec *s = a.subs + slot;
            s->dist = newdist, s->lvl = k;
#pragma unroll 1
            for (int j = k; j < d; j++)
              s->x[j] = (int)getx(j);
          }
        }
      }
      if (k == 0)
      {
        if (newdist > 0.0)
        {
          my_leaves++;
          const unsigned long long nb  = (unsigned long long)__double_as_longlong(newdist);
          const unsigned long long old = atomicMin(a.words + (a.fixed_radius ? W_BEST : W_A), nb);
          // (fixed radius: ties with the best so far are recorded too — the host picks among equally short vectors by
          // their coefficients, so the result does not depend on which walker got there first)
          if (nb < old || (a.fixed_radius && nb == old))
          {
            const unsigned slot = atomicAdd(sol_count, 1u);
            if (slot < SOL_CAP)
            {
              SolRec *s = slot < SOL_FAST ? a.sols_fast + slot : a.sols_more + slot;
              s->dist   = newdist;
              s->lvl    = 0;
#pragma unroll 1
              for (int j = 0; j < d; j++)
                s->x[j] = (int)getx(j);
            }
            if (!a.fixed_radius)
              for (int q = 0; q < a.n_peer; q++)  // push the new radius to every peer (NVLink, fire and forget)
                red_min_sys(a.A_peer[q], nb);
          }
          if (!a.fixed_radius)
            A = fmin(A, newdist);
        }
        k = -1;  // the reference decrements first and lets next_pos_up come back to level 0
      }
      else
      {
        --k;
        // centre: the reference's chain ((0 - x[d-1] mu) - x[d-2] mu) - ... - x[k+1] mu, descending j
        double nc;
        const double *mrow = s_mut + (size_t)k * ds;
        if (k < pvalid)
        {
          // first visit of level k inside this task (k == pvalid - 1): the fixed part of the chain, j = d-1 .. top0+1
          nc = 0.0;
#pragma unroll 4
          for (int j = d - 1; j > top0; --j)
            nc = __dsub_rn(nc, __dmul_rn(chainv(j), mrow[j]));
          pre[k] = nc;
          pvalid = k;
        }
        else
          nc = pre[k];
#pragma unroll 4
        for (int j = top0; j > k; --j)
          nc = __dsub_rn(nc, __dmul_rn(chainv(j), mrow[j]));
        cen[k] = nc;
        pd[k]  = newdist;
        setx(k, round(nc));
        up     = false;
      }
    }
    if (up)
    {
      ++k;
      if (k > top)
        k = -2;  // everything this walker owned is done
      else
        setx(k, next_sibling(getx(k), cen[k], pd[k]));
    }
    else if (n >= next_check)
    {
      // Work split (we are at a just-created node: level k holds its first, not yet tested, candidate x[k]).
      //  * the round still has unclaimed tasks: a walker that used up its budget donates the unvisited siblings of
      //    its two top-most ancestor levels (the biggest chunks) and goes on;
      //  * the round has run dry (idle lanes are waiting): after only 64 more nodes the walker YIELDS — every
      //    ancestor's remaining siblings plus its current position become tasks of the next round — so the tail of
      //    a round is bounded by ~64 nodes instead of by the largest subtree.
      const bool dry = shared_round ? (*(volatile unsigned *)flags != 0u) : (*(volatile unsigned *)ticket >= end);
      next_check     = n + ynodes;
      if (dry || n >= budget)
      {
        int jj = top, given = 0;
        bool full = false;
        for (; jj > k && (dry || given < 2); --jj)
        {
          // siblings come in order of increasing distance from the centre: if the next one is already outside the
          // bound there is nothing left at this level
          const double nx = next_sibling(getx(jj), cen[jj], pd[jj]);
          const double alj = __dsub_rn(nx, cen[jj]);
          const double nd = __dadd_rn(pd[jj], __dmul_rn(__dmul_rn(alj, alj), s_r[jj]));
          if (!(nd <= __dmul_rn(s_p[jj], A)))
            continue;
          const unsigned slot = atomicAdd(tail, 1u);
          if (slot >= TASK_CAP)
          {
            full = true;
            break;  // queue full: keep levels <= jj ourselves
          }
          TaskHdr h;
          h.pd = pd[jj], h.cen = cen[jj], h.xs = nx, h.lvl = jj, h.pad = 0;
          hdr_out[slot] = h;
          int *tx       = tx_out + (size_t)slot * a.dstride;
#pragma unroll 4
          for (int j = jj + 1; j < d; j++)
            tx[j] = (int)getx(j);
          given++;
        }
        top = jj;  // levels above jj are donated or exhausted; the walker keeps the siblings of levels <= jj
        if (dry && !full && top == k)
        {
          const unsigned slot = atomicAdd(tail, 1u);
          if (slot < TASK_CAP)
          {
            TaskHdr h;
            h.pd = pd[k], h.cen = cen[k], h.xs = getx(k), h.lvl = k, h.pad = 0;
            hdr_out[slot] = h;
            int *tx       = tx_out + (size_t)slot * a.dstride;
#pragma unroll 4
            for (int j = k + 1; j < d; j++)
              tx[j] = (int)getx(j);
            k = -2;  // yielded: this walker is idle (and the round is dry, so it will leave the loop)
          }
        }
        n          = 0;
        next_check = ynodes;
      }
    }
    if (((++steps) & 63) == 0 && !a.fixed_radius)
      A = __longlong_as_double(*(volatile unsigned long long *)A_bits);
  }
  // ---- end of round: everybody has left the walker loop; publish the next round's task count ----
  if (nr && a.node_cap)
    atomicAdd(a.words + W_NODES, (unsigned long long)nr);
  __threadfence();
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x == 0)
  {
    const unsigned produced = *(volatile unsigned *)tail;
    ctr[2] = produced < TASK_CAP ? produced : TASK_CAP;
    ctr[0] = 0;
    ctr[1] = 0;
    ctr[3] = rno + 1;
    // hand-off: still work left after node_cap nodes -> stop here, the host spreads the pending queue over all devices
    if (a.node_cap && produced > 0 && *(volatile unsigned long long *)(a.words + W_NODES) >= a.node_cap)
      flags[1] = 1u;
    __threadfence();
  }
  grid.sync();
  end = *(volatile unsigned *)(ctr + 2);
  if (end == 0 || *(volatile unsigned *)(flags + 1))
    break;
  const unsigned long long nb = (unsigned long long)budget * a.budget_mul;
  budget = nb > 16384ull ? 16384u : (unsigned)nb;
  }
#pragma unroll 1
  for (int kk = 0; kk < d; kk++)
    if (cnt[kk])
      atomicAdd(a.nodes + kk, (unsigned long long)cnt[kk]);
  if (my_leaves)
    atomicAdd(a.words + W_LEAVES, my_leaves);
}

// ------------------------------------------------------------------------------------------------------------
// host breadth phase: the top levels, level by level, each level in exact Schnorr-Euchner order (the children of one
// node in zig-zag order around its centre, the nodes of a level in depth-first order — what a depth-first walk cut off
// at that level would emit).  Arithmetic as in enumerate_loop: centre = descending chain, newdist = pd + alpha^2 r.
struct BNode
{
  double pd, alpha;  // partial length including this node; alpha = x - centre at this node (dual chains)
  int parent, x;
};
struct Breadth
{
  std::vector<std::vector<BNode>> lev;  // lev[t] = accepted nodes of tree level d-1-t; lev[t][0] is the all-zero prefix
  std::vector<uint64_t> nodes;          // d: counted nodes per tree level
  // level d-1 alone had more candidates than fit: lev[0] holds the first `cap` of them (x = 0 .. cap-1) and the rest,
  // x = top_rest, top_rest + 1, ..., is left to the device as one task at level d-1 (0: nothing left)
  int top_rest = 0;
};

// children of node `pi` of level t-1 at tree level k = d-1-t; stops once `out` holds more than `cap` nodes
static void expand_children(int d, int k, const double *mut, const double *rdiag, const double *prun, double A, bool dual,
                            const Breadth &br, int t, int pi, std::vector<BNode> &out, std::vector<double> &chain,
                            size_t cap)
{
  // values the chain multiplies with: x_j (primal) or alpha_j (dual) of the ancestors, levels d-1 .. k+1
  int q = pi;
  for (int tt = t - 1; tt >= 0; --tt)
  {
    const BNode &b = br.lev[tt][q];
    chain[d - 1 - tt] = dual ? b.alpha : (double)b.x;
    q = b.parent;
  }
  double nc = 0.0;
  for (int j = d - 1; j > k; --j)
    nc = nc - chain[j] * mut[(size_t)k * d + j];
  const double pdk = (t == 0) ? 0.0 : br.lev[t - 1][pi].pd;
  const bool zero_prefix = (t == 0) || (pi == 0);
  if (zero_prefix)
  {
    // the all-zero prefix continues (never counted), then x = 1, 2, ... (SVP: positive half only; pd == 0, centre 0)
    BNode z;
    z.pd = 0.0, z.alpha = 0.0, z.parent = pi, z.x = 0;
    out.push_back(z);
    for (double x = 1.0; out.size() <= cap; x += 1.0)
    {
      const double alphak = x - nc, newdist = pdk + alphak * alphak * rdiag[k];
      if (!(newdist <= prun[k] * A))
        break;
      BNode b;
      b.pd = newdist, b.alpha = alphak, b.parent = pi, b.x = (int)x;
      out.push_back(b);
    }
    return;
  }
  const double x0 = std::round(nc), s = (nc >= x0) ? 1.0 : -1.0;
  double x = x0;
  while (out.size() <= cap)
  {
    const double alphak = x - nc, newdist = pdk + alphak * alphak * rdiag[k];
    if (!(newdist <= prun[k] * A))
      break;
    BNode b;
    b.pd = newdist, b.alpha = alphak, b.parent = pi, b.x = (int)x;
    out.push_back(b);
    // x0, x0+s, x0-s, x0+2s, ...
    const double tq = x - x0;
    x = (tq == 0.0) ? x0 + s : ((tq * s > 0.0) ? x0 - tq : x0 - tq + s);
  }
}

// grows the expansion until there are >= want roots (keeps the last level that fits into `cap`); T >= 1 levels
static void breadth_phase(int d, const double *mut, const double *rdiag, const double *prun, double A, bool dual,
                          size_t want, size_t cap, Breadth &br)
{
  br.lev.clear();
  br.nodes.assign(d, 0);
  br.top_rest = 0;
  std::vector<double> chain(d + 1, 0.0);
  for (int t = 0; t < d - 1; ++t)
  {
    const int k = d - 1 - t;
    std::vector<BNode> cur;
    const size_t np = (t == 0) ? 1 : br.lev[t - 1].size();
    bool over = false;
    for (size_t pi = 0; pi < np && !over; ++pi)
    {
      expand_children(d, k, mut, rdiag, prun, A, dual, br, t, (int)pi, cur, chain, cap);
      over = cur.size() > cap;
    }
    if (over && t > 0)
      break;  // too many: keep the previous depth
    if (over)
    {
      // level d-1 alone has more than `cap` candidates (a tiny r(d-1, d-1)): its children of the all-zero root are
      // x = 0, 1, 2, ... in this order, so the first `cap` become roots and the device walks the rest from one task
      cur.resize(cap);
      br.top_rest = cur.back().x + 1;
    }
    br.nodes[k] = cur.size() - 1;  // the all-zero prefix is not a node
    br.lev.push_back(std::move(cur));
    if (br.lev.back().size() >= want || br.top_rest)
      break;
  }
}

// ------------------------------------------------------------------------------------------------------------
// per-device persistent buffers
struct DevCtx
{
  int device = -1, sms = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  // result block  [SolRec x SOL_FAST | words | nodes | sub_bits]  — one D2H copy per call —
  // followed by the staging area  [cfg | round-0 task headers | round-0 task prefixes]  — one H2D copy per call
  unsigned char *d_blk = nullptr, *h_up = nullptr, *h_down = nullptr;
  size_t blk_bytes = 0;
  TaskHdr *d_hdr = nullptr;  // 2 x TASK_CAP
  int *d_tx = nullptr;
  size_t tx_cap = 0;  // ints
  SolRec *d_sols_more = nullptr, *d_subs = nullptr;
  SolRec *h_more = nullptr;  // pinned, SOL_CAP (also receives the sub-solution records)
  unsigned epoch = 0;
  int occ_xs_threads = 0, occ_xs = 0;
  // one-process-per-GPU cooperation (b200enum_ipc_*): the other ranks' word blocks, mapped through CUDA IPC
  int ipc_world = 0, ipc_rank = 0;
  unsigned long long *ipc_words[MAX_PEERS] = {nullptr};
  unsigned long long *words() const { return (unsigned long long *)(d_blk + OFF_WORDS); }
  static constexpr size_t OFF_WORDS = sizeof(SolRec) * SOL_FAST;
  static constexpr size_t OFF_NODES = OFF_WORDS + W_COUNT * 8;
  static constexpr size_t OFF_SUBB  = OFF_NODES + B200ENUM_MAX_DIM * 8;
  static constexpr size_t OFF_STAGE = OFF_SUBB + B200ENUM_MAX_DIM * 8;  // multiple of 16
};
std::mutex g_mu;
std::deque<DevCtx> g_ctx;  // deque: get_ctx hands out pointers that must survive later push_backs
bool g_peer_on[16][16];

int get_ctx(int device, DevCtx **out)
{
  for (auto &c : g_ctx)
    if (c.device == device)
    {
      *out = &c;
      return 0;
    }
  DevCtx c;
  c.device = device;
  CKE(cudaSetDevice(device));
  CKE(cudaDeviceGetAttribute(&c.sms, cudaDevAttrMultiProcessorCount, device));
  CKE(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
  CKE(cudaEventCreate(&c.e0));
  CKE(cudaEventCreate(&c.e1));
  // staging: cfg (16-byte aligned), then up to MAX_ROOTS roots plus the task for the rest of a wide level d-1, each
  // with a prefix row of (d + 3) & ~3 ints — sized for B200ENUM_MAX_DIM (22 MB), so any call's roots fit
  const size_t cfg_max = (((size_t)B200ENUM_MAX_DIM * B200ENUM_MAX_DIM + 2 * B200ENUM_MAX_DIM) * 8 + 15) & ~(size_t)15;
  const size_t row_max = (size_t)((B200ENUM_MAX_DIM + 3) & ~3) * sizeof(int);
  c.blk_bytes = DevCtx::OFF_STAGE + cfg_max + (size_t)(MAX_ROOTS + 1) * (sizeof(TaskHdr) + row_max);
  CKE(cudaMalloc(&c.d_blk, c.blk_bytes));
  CKE(cudaMemset(c.d_blk, 0, DevCtx::OFF_STAGE));
  CKE(cudaMallocHost(&c.h_up, c.blk_bytes));
  CKE(cudaMallocHost(&c.h_down, DevCtx::OFF_STAGE));
  CKE(cudaMalloc(&c.d_sols_more, SOL_CAP * sizeof(SolRec)));
  CKE(cudaMalloc(&c.d_subs, SUB_CAP * sizeof(SolRec)));
  CKE(cudaMalloc(&c.d_hdr, (size_t)2 * TASK_CAP * sizeof(TaskHdr)));
  CKE(cudaMallocHost(&c.h_more, (size_t)std::max(SOL_CAP, SUB_CAP) * sizeof(SolRec)));
  CKE(cudaFuncSetAttribute((const void *)k_enum<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  CKE(cudaFuncSetAttribute((const void *)k_enum<160, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  CKE(cudaFuncSetAttribute((const void *)k_enum<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_XS_MAX));
  CKE(cudaFuncSetAttribute((const void *)k_enum<64, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_XS_MAX));
  g_ctx.push_back(c);
  *out = &g_ctx.back();
  return 0;
}

template <class T> int ensure(T **p, size_t *cap, size_t need)
{
  if (*cap >= need)
    return 0;
  if (*p)
  {
    CKE(cudaFree(*p));
    *p = nullptr, *cap = 0;
  }
  CKE(cudaMalloc(p, need * sizeof(T)));
  *cap = need;
  return 0;
}

int enable_peers(const std::vector<DevCtx *> &ctxs)
{
  for (DevCtx *a : ctxs)
    for (DevCtx *b : ctxs)
      if (a != b && a->device < 16 && b->device < 16 && !g_peer_on[a->device][b->device])
      {
        int can = 0;
        CKE(cudaDeviceCanAccessPeer(&can, a->device, b->device));
        if (!can)
        {
          g_err = "b200enum_run: devices cannot access each other's memory (no NVLink / P2P)";
          return B200ENUM_ECUDA;
        }
        CKE(cudaSetDevice(a->device));
        const cudaError_t e = cudaDeviceEnablePeerAccess(b->device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
        {
          g_err = std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e);
          return B200ENUM_ECUDA;
        }
        cudaGetLastError();
        g_peer_on[a->device][b->device] = true;
      }
  return 0;
}

struct Tuning
{
  unsigned budget0, budget_mul, yield_nodes;
  int bpsm, use_xs, xs_threads_cap;
  unsigned long long fan_nodes;
  int min_roots;
  unsigned yield_small;
  int shard_roots;
  const char *trace;
};
const Tuning &tuning()
{
  static const Tuning t = [] {
    Tuning q;
    auto geti = [](const char *n, long dflt) { return getenv(n) ? atol(getenv(n)) : dflt; };
    q.budget0        = (unsigned)geti("B200_ENUM_BUDGET0", 64);
    q.budget_mul     = (unsigned)geti("B200_ENUM_BUDGET_MUL", 4);
    q.yield_nodes    = (unsigned)geti("B200_ENUM_YIELD", 64);
    q.bpsm           = (int)geti("B200_ENUM_BLOCKS_PER_SM", 4);
    q.use_xs         = (int)geti("B200_ENUM_XS", 1);
    q.xs_threads_cap = (int)geti("B200_ENUM_XS_THREADS", 320);
    // hand-off threshold: a call that has visited this many nodes on the first device and still has work pending is
    // spread over all devices.  A low threshold makes a BKZ-60 tour on two devices slower than on one (fixed-region
    // calls of 30-100 M nodes are common, and suspending at a round boundary + peer copies + a cooperative launch and a
    // read-back per device cost more than half such a call saves): a tour must never pay for devices it cannot use.
    q.fan_nodes = (unsigned long long)geti("B200_ENUM_FAN_NODES", 200000000);
    q.min_roots   = (int)geti("B200_ENUM_MIN_ROOTS", MIN_ROOTS);
    q.shard_roots = (int)geti("B200_ENUM_SHARD_ROOTS", 8192);
    // rounds with fewer tasks than warps are bound by the latency of a lone walker: yield sooner
    q.yield_small = (unsigned)geti("B200_ENUM_YIELD_SMALL", 8);
    q.trace     = getenv("B200_ENUM_TRACE");  // append one line per call to this file
    return q;
  }();
  return t;
}

struct LaunchShape
{
  const void *fn;
  int threads, blocks;
  size_t smem;
};

int launch_shape(DevCtx *c, int d, bool xs, bool dual, LaunchShape &ls)
{
  const Tuning &tn      = tuning();
  const size_t cfg_n    = (size_t)d * d + 2 * d;
  const size_t cfg_smem = xs ? ((size_t)d * (d | 1) + 2 * d) * sizeof(double) : cfg_n * sizeof(double);
  // XS: every walker keeps one d-vector in shared memory (x), two in a dual call (x and alpha) — at d = 64 that is 320
  // walkers per CTA primal (the thread cap) and 192 dual
  const size_t per_walker = (xs && dual ? 2 : 1) * (size_t)d * sizeof(double);
  int threads = THREADS;
  if (xs)
  {
    threads = (int)((SMEM_XS_MAX - cfg_smem) / per_walker);
    threads = std::min(std::min(threads, tn.xs_threads_cap), THREADS_XS) & ~31;
    if (threads < 32)
      threads = 32;
  }
  ls.smem    = cfg_smem + (xs ? (size_t)threads * per_walker : 0);
  ls.threads = threads;
  ls.fn = xs ? (dual ? (const void *)k_enum<64, true, true> : (const void *)k_enum<64, true>)
             : (d <= 64 ? (const void *)k_enum<64, false> : (const void *)k_enum<160, false>);
  if (xs)
  {
    ls.blocks = c->sms;  // one CTA per SM by construction (shared memory); every CTA must be resident (grid barrier)
    return 0;
  }
  int occ = 0;
  CKE(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, ls.fn, threads, ls.smem));
  if (occ < 1)
  {
    g_err = "b200enum_run: kernel does not fit on an SM";
    return B200ENUM_ECUDA;
  }
  ls.blocks = c->sms * std::min(occ, tn.bpsm);
  return 0;
}

int run_impl(int dim, double maxdist, const double *mut_in, const double *rdiag_in, const double *pruning, int flags,
             const int *devices, int ndev, int shard_rank, int shard_world, b200enum_sol_cb cb,
             b200enum_subsol_cb subcb, void *ctx, uint64_t *nodes, b200enum_stats *stats)
{
  if (dim < 2 || dim > B200ENUM_MAX_DIM || !mut_in || !rdiag_in || !(maxdist > 0) || shard_world < 1 || shard_rank < 0 ||
      shard_rank >= shard_world || ndev > MAX_PEERS || shard_world > MAX_PEERS ||
      ((flags & B200ENUM_FINDSUBSOLS) && !subcb))
  {
    g_err = "b200enum_run: bad arguments";
    return B200ENUM_EINVAL;
  }
  const int navail = b200enum_device_count();
  if (navail == 0)
  {
    g_err = "b200enum_run: no CUDA device (this library has no CPU fallback)";
    return B200ENUM_ENODEV;
  }
  int dev0 = 0;
  if (!devices || ndev <= 0)
  {
    devices = &dev0;
    ndev    = 1;
  }
  for (int i = 0; i < ndev; i++)
    if (devices[i] < 0 || devices[i] >= navail)
    {
      g_err = "b200enum_run: bad device ordinal";
      return B200ENUM_EINVAL;
    }
  if (shard_world > 1 && ndev != 1)
  {
    g_err = "b200enum_run: a sharded call (shard_world > 1) drives exactly one device per process";
    return B200ENUM_EINVAL;
  }
  std::lock_guard<std::mutex> lock(g_mu);
  const Tuning &tn   = tuning();
  const auto t_begin = std::chrono::steady_clock::now();
  const int d        = dim;
  const bool fixed = (flags & B200ENUM_FIXED_RADIUS) != 0, dual = (flags & B200ENUM_DUAL) != 0,
             subs  = (flags & B200ENUM_FINDSUBSOLS) != 0;
  std::vector<double> prun(d, 1.0), mutv, rdv;
  if (pruning)
    std::copy(pruning, pruning + d, prun.begin());
  const double *mut = mut_in, *rdiag = rdiag_in;
  if (dual)
  {
    // enumerate.cpp:100-113: the dual basis of the block, reversed: r'_{d-1-i} = 1 / r_i, mu'^T[d-1-j][d-1-i] = -mu(j,i)
    mutv.assign((size_t)d * d, 0.0), rdv.resize(d);
    for (int i = 0; i < d; i++)
      rdv[d - 1 - i] = 1.0 / rdiag_in[i];
    for (int i = 0; i < d; i++)
      for (int j = i + 1; j < d; j++)
        mutv[(size_t)(d - 1 - j) * d + (d - 1 - i)] = -mut_in[(size_t)i * d + j];
    mut = mutv.data(), rdiag = rdv.data();
  }

  // ---- host breadth phase ----
  Breadth br;
  // A sharded call (one process per GPU) shares only its ROOTS between the ranks — the tasks a walker splits off later
  // stay in its own device's queue — so the roots must be fine-grained enough to balance a heavy-tailed tree on their
  // own: with 128 roots per rank two GPUs finished the 5.6e8-node BKZ-60 block no sooner than one.
  size_t want = (size_t)tn.min_roots * (size_t)shard_world;
  if (shard_world > 1)
    want = std::max(want, (size_t)tn.shard_roots);
  breadth_phase(d, mut, rdiag, prun.data(), maxdist, dual, std::min<size_t>(want, MAX_ROOTS), MAX_ROOTS, br);
  const int T = (int)br.lev.size(), L = d - T;
  const std::vector<BNode> &leaf = br.lev[T - 1];
  const size_t nroots = leaf.size();
  // round-0 tasks: the roots, plus (index nroots) the rest of a level d-1 that had more candidates than MAX_ROOTS
  const size_t ntask = nroots + (br.top_rest ? 1 : 0);
  // roots sorted by partial length (ascending; the all-zero prefix first): most promising subtrees first.  The rest of
  // level d-1 goes last: its nodes are longer than every root's.
  std::vector<unsigned> order(ntask);
  for (size_t i = 0; i < ntask; i++)
    order[i] = (unsigned)i;
  std::stable_sort(order.begin(), order.begin() + nroots,
                   [&](unsigned a, unsigned b) { return leaf[a].pd < leaf[b].pd; });
  const auto t_host = std::chrono::steady_clock::now();

  // ---- contexts ----
  // Only the first device is touched here: the others are set up when (and if) a call is handed off to them — a BKZ tour
  // issues ~18 k calls of which a handful fan out, and two cudaSetDevice round trips per call were 0.6 s of a tour.
  std::vector<DevCtx *> ctxs(ndev, nullptr);
  auto prepare_ctx = [&](int q) -> int {
    if (ctxs[q])
      return 0;
    int rc = get_ctx(devices[q], &ctxs[q]);
    if (rc)
      return rc;
    CKE(cudaSetDevice(ctxs[q]->device));
    // sized for dim <= 64 up front (BKZ calls with every block size from 2 to beta: growing would re-allocate ~1 GB
    // a dozen times), re-allocated once if a larger dimension ever shows up
    return ensure(&ctxs[q]->d_tx, &ctxs[q]->tx_cap, (size_t)2 * TASK_CAP * (d <= 64 ? 64 : B200ENUM_MAX_DIM));
  };
  {
    const int rc = prepare_ctx(0);
    if (rc)
      return rc;
  }
  DevCtx *home      = ctxs[0];
  const int dstride = (d + 3) & ~3;
  const size_t cfg_n = (size_t)d * d + 2 * d;
  const size_t off_cfg = DevCtx::OFF_STAGE, off_hdr = off_cfg + ((cfg_n * 8 + 15) & ~(size_t)15);
  // ipc mode: ranks attached to each other push radius improvements into each other's words over NVLink.  The roots are
  // dealt round-robin in order of promise in either case: a shared ticket over the ROOTS was measured and dropped — a root
  // is split into its device's own queue after 64 nodes, so the 47 k walkers of whichever rank starts a few microseconds
  // earlier claim every root before the other one arrives (two ranks were no faster than one).
  const bool ipc = shard_world > 1 && home->ipc_world == shard_world && home->ipc_rank == shard_rank;
  // the staged round-0 tasks of this process: its share of the roots
  std::vector<unsigned> mine;
  if (shard_world > 1)
    for (size_t g = (size_t)shard_rank; g < ntask; g += (size_t)shard_world)
      mine.push_back(order[g]);
  else
    mine = order;
  const size_t nmine = mine.size();
  const size_t off_tx = off_hdr + nmine * sizeof(TaskHdr);
  const size_t up_end = off_tx + nmine * (size_t)dstride * sizeof(int);
  if (up_end > home->blk_bytes)
  {
    g_err = "b200enum_run: staging block overflow";
    return B200ENUM_EINVAL;
  }
  {
    // fill the pinned staging block: words | nodes | sub_bits | cfg | hdr | tx
    unsigned char *u = home->h_up;
    memset(u + DevCtx::OFF_WORDS, 0, DevCtx::OFF_STAGE - DevCtx::OFF_WORDS);
    unsigned long long *w = (unsigned long long *)(u + DevCtx::OFF_WORDS);
    memcpy(&w[W_A], &maxdist, 8);
    w[W_BEST] = ~0ull;
    if (subs)
    {
      unsigned long long *sb = (unsigned long long *)(u + DevCtx::OFF_SUBB);
      for (int k = 0; k < d; k++)
        memcpy(&sb[k], &rdiag[k], 8);  // subsoldists = rdiag (enumerate.cpp:141)
    }
    double *cfg = (double *)(u + off_cfg);
    std::copy(mut, mut + (size_t)d * d, cfg);
    std::copy(rdiag, rdiag + d, cfg + (size_t)d * d);
    std::copy(prun.begin(), prun.end(), cfg + (size_t)d * d + d);
    TaskHdr *hdr = (TaskHdr *)(u + off_hdr);
    int *tx      = (int *)(u + off_tx);
    memset(tx, 0, nmine * (size_t)dstride * sizeof(int));
    std::vector<double> chain(d + 1, 0.0);
    for (size_t g = 0; g < nmine; g++)
    {
      if (mine[g] == nroots)
      {
        // the rest of level d-1: x = top_rest, top_rest + 1, ... under the all-zero prefix (centre 0, and pd = 0 makes
        // next_sibling step x + 1), each with everything below it
        TaskHdr h;
        h.lvl = d - 1, h.pad = 0, h.pd = 0.0, h.cen = 0.0, h.xs = (double)br.top_rest;
        hdr[g] = h;
        continue;
      }
      // the task "level L-1 under this root": prefix x[L..d-1], centre of level L-1 (same chain as the device)
      int q = (int)mine[g];
      int *row = tx + g * (size_t)dstride;
      for (int tt = T - 1; tt >= 0; --tt)
      {
        const BNode &b = br.lev[tt][q];
        row[d - 1 - tt]   = b.x;
        chain[d - 1 - tt] = dual ? b.alpha : (double)b.x;
        q = b.parent;
      }
      double nc = 0.0;
      for (int j = d - 1; j >= L; --j)
        nc = nc - chain[j] * mut[(size_t)(L - 1) * d + j];
      TaskHdr h;
      h.lvl = L - 1, h.pad = 0, h.pd = leaf[mine[g]].pd, h.cen = nc, h.xs = std::round(nc);
      hdr[g] = h;
    }
  }

  const bool xs = tn.use_xs && d <= 64 && !subs;  // B200_ENUM_XS=0: the thread-local variant for every call
  auto make_args = [&](DevCtx *c, EnumArgs &a) {
    memset(&a, 0, sizeof(a));
    a.d = d, a.dstride = dstride;
    a.mut = (const double *)(c->d_blk + off_cfg), a.rdiag = a.mut + (size_t)d * d, a.prun = a.rdiag + d;
    a.hdrq[0] = c->d_hdr, a.hdrq[1] = c->d_hdr + TASK_CAP;
    a.txq[0] = c->d_tx, a.txq[1] = c->d_tx + (size_t)TASK_CAP * dstride;
    a.words = c->words();
    a.nodes = (unsigned long long *)(c->d_blk + DevCtx::OFF_NODES);
    a.sub_bits = (unsigned long long *)(c->d_blk + DevCtx::OFF_SUBB);
    a.sols_fast = (SolRec *)c->d_blk, a.sols_more = c->d_sols_more, a.subs = c->d_subs;
    a.budget0 = tn.budget0, a.budget_mul = tn.budget_mul, a.yield_nodes = tn.yield_nodes;
    a.yield_small = tn.yield_small;
    a.fixed_radius = fixed ? 1 : 0, a.dual = dual ? 1 : 0, a.findsubsols = subs ? 1 : 0;
    a.share_div = 1;
  };
  auto launch = [&](DevCtx *c, EnumArgs &a) -> int {
    LaunchShape ls;
    int rc = launch_shape(c, d, xs, dual, ls);
    if (rc)
      return rc;
    void *params[] = {(void *)&a};
    CKE(cudaLaunchCooperativeKernel(ls.fn, dim3(ls.blocks), dim3(ls.threads), params, ls.smem, c->stream));
    return 0;
  };
  auto download = [&](DevCtx *c) -> int {  // result block -> pinned, one copy
    CKE(cudaMemcpyAsync(c->h_down, c->d_blk, DevCtx::OFF_STAGE, cudaMemcpyDeviceToHost, c->stream));
    return 0;
  };

  // ---- phase A: the first device ----
  CKE(cudaSetDevice(home->device));
  CKE(cudaMemcpyAsync(home->d_blk + DevCtx::OFF_WORDS, home->h_up + DevCtx::OFF_WORDS, up_end - DevCtx::OFF_WORDS,
                      cudaMemcpyHostToDevice, home->stream));
  CKE(cudaEventRecord(home->e0, home->stream));
  EnumArgs a0;
  make_args(home, a0);
  a0.hdr_first = (const TaskHdr *)(home->d_blk + off_hdr), a0.tx_first = (const int *)(home->d_blk + off_tx);
  a0.out0 = 0, a0.n_first = (unsigned)nmine;
  if (ipc)
    for (int r = 0; r < shard_world; r++)
      if (r != shard_rank)
        a0.A_peer[a0.n_peer++] = home->ipc_words[r] + W_A;
  a0.node_cap = (ndev > 1) ? tn.fan_nodes : 0;
  bool fanned = false;
  if (nmine > 0)
  {
    int rc = launch(home, a0);
    if (rc)
      return rc;
  }
  CKE(cudaEventRecord(home->e1, home->stream));
  int rc = download(home);
  if (rc)
    return rc;
  CKE(cudaStreamSynchronize(home->stream));
  CKE(cudaGetLastError());
  float ms_total = 0;
  {
    float ms = 0;
    cudaEventElapsedTime(&ms, home->e0, home->e1);
    ms_total += ms;
  }
  int used_dev = 1;
  // ---- phase B: hand the pending queue to every device (only calls that are still busy after fan_nodes nodes) ----
  {
    const unsigned long long *hw = (const unsigned long long *)(home->h_down + DevCtx::OFF_WORDS);
    const unsigned *hflags = (const unsigned *)(hw + W_FLAGS), *hctr = (const unsigned *)(hw + W_CTR);
    if (ndev > 1 && hflags[1])
    {
      fanned = true;
      used_dev = ndev;
      for (int q = 1; q < ndev; q++)
      {
        rc = prepare_ctx(q);
        if (rc)
          return rc;
      }
      rc = enable_peers(ctxs);
      if (rc)
        return rc;
      const unsigned pending = hctr[2], rounds = hctr[3];
      const int half = (int)((a0.out0 + rounds - 1) & 1u);
      // the shared ticket lives on the first device: clear it, the suspended flag and the local counters
      unsigned long long *hu = (unsigned long long *)(home->h_up + DevCtx::OFF_WORDS);
      memcpy(hu, hw, W_COUNT * 8);
      ((unsigned *)(hu + W_FLAGS))[0] = 0, ((unsigned *)(hu + W_FLAGS))[1] = 0;
      ((unsigned *)(hu + W_CTR))[0] = 0, ((unsigned *)(hu + W_CTR))[1] = 0, ((unsigned *)(hu + W_CTR))[2] = 0;
      home->epoch++;
      hu[W_GTICKET] = (unsigned long long)home->epoch << 32;
      CKE(cudaMemcpyAsync(home->d_blk + DevCtx::OFF_WORDS, hu, W_COUNT * 8, cudaMemcpyHostToDevice, home->stream));
      CKE(cudaEventRecord(home->e0, home->stream));
      for (int q = 1; q < ndev; q++)
      {
        DevCtx *c = ctxs[q];
        CKE(cudaSetDevice(c->device));
        // peer words: the current radius, everything else zero; cfg from the host staging block; the queue over NVLink
        unsigned char *u = c->h_up;
        memset(u + DevCtx::OFF_WORDS, 0, DevCtx::OFF_STAGE - DevCtx::OFF_WORDS);
        unsigned long long *w = (unsigned long long *)(u + DevCtx::OFF_WORDS);
        w[W_A] = hw[W_A], w[W_BEST] = ~0ull;
        memcpy(u + DevCtx::OFF_SUBB, home->h_down + DevCtx::OFF_SUBB, B200ENUM_MAX_DIM * 8);
        memcpy(u + off_cfg, home->h_up + off_cfg, cfg_n * 8);
        CKE(cudaStreamWaitEvent(c->stream, home->e0, 0));
        CKE(cudaMemcpyAsync(c->d_blk + DevCtx::OFF_WORDS, u + DevCtx::OFF_WORDS, off_cfg + cfg_n * 8 - DevCtx::OFF_WORDS,
                            cudaMemcpyHostToDevice, c->stream));
        CKE(cudaMemcpyPeerAsync(c->d_hdr, c->device, home->d_hdr + (size_t)half * TASK_CAP, home->device,
                                (size_t)pending * sizeof(TaskHdr), c->stream));
        CKE(cudaMemcpyPeerAsync(c->d_tx, c->device, home->d_tx + (size_t)half * TASK_CAP * dstride, home->device,
                                (size_t)pending * dstride * sizeof(int), c->stream));
        CKE(cudaEventRecord(c->e0, c->stream));
      }
      for (int q = 0; q < ndev; q++)
      {
        DevCtx *c = ctxs[q];
        CKE(cudaSetDevice(c->device));
        EnumArgs a;
        make_args(c, a);
        const int myhalf = (q == 0) ? half : 0;
        a.hdr_first = c->d_hdr + (size_t)myhalf * TASK_CAP, a.tx_first = c->d_tx + (size_t)myhalf * TASK_CAP * dstride;
        a.out0 = myhalf ^ 1, a.n_first = pending;
        a.gticket = home->words() + W_GTICKET, a.gepoch = home->epoch, a.share_div = ndev;
        for (int p = 0; p < ndev; p++)
          if (p != q)
            a.A_peer[a.n_peer++] = ctxs[p]->words() + W_A;
        rc = launch(c, a);
        if (rc)
          return rc;
        CKE(cudaEventRecord(c->e1, c->stream));
        rc = download(c);
        if (rc)
          return rc;
      }
      float ms_b = 0;
      for (int q = 0; q < ndev; q++)
      {
        DevCtx *c = ctxs[q];
        CKE(cudaSetDevice(c->device));
        CKE(cudaStreamSynchronize(c->stream));
        CKE(cudaGetLastError());
        float ms = 0;
        cudaEventElapsedTime(&ms, ctxs[q]->e0, c->e1);
        ms_b = std::max(ms_b, ms);
      }
      ms_total += ms_b;
    }
  }

  // ---- collect ----
  int rounds = 0;
  std::vector<uint64_t> tot(d, 0);
  uint64_t host_nodes = 0, dev_nodes = 0, leaves = 0;
  if (shard_rank == 0)
    for (int k = 0; k < d; k++)
    {
      tot[k] += br.nodes[k];
      host_nodes += br.nodes[k];
    }
  std::vector<SolRec> found, subfound;
  bool overflow = false;
  for (int q = 0; q < used_dev; q++)
  {
    DevCtx *c = ctxs[q];
    const unsigned long long *hw = (const unsigned long long *)(c->h_down + DevCtx::OFF_WORDS);
    const unsigned long long *hn = (const unsigned long long *)(c->h_down + DevCtx::OFF_NODES);
    const unsigned nsol = ((const unsigned *)(hw + W_SOLC))[0], nsub = ((const unsigned *)(hw + W_SOLC))[1];
    for (int k = 0; k < d; k++)
    {
      tot[k] += hn[k];
      dev_nodes += hn[k];
    }
    leaves += hw[W_LEAVES];
    rounds = std::max(rounds, (int)((const unsigned *)(hw + W_CTR))[3]);
    if (nsol > SOL_CAP || nsub > SUB_CAP)
      overflow = true;
    const SolRec *fast = (const SolRec *)c->h_down;
    for (unsigned s = 0; s < std::min<unsigned>(nsol, SOL_FAST); s++)
      found.push_back(fast[s]);
    if (nsol > SOL_FAST)
    {
      const unsigned n2 = std::min<unsigned>(nsol, SOL_CAP);
      CKE(cudaSetDevice(c->device));
      CKE(cudaMemcpyAsync(c->h_more + SOL_FAST, c->d_sols_more + SOL_FAST, (size_t)(n2 - SOL_FAST) * sizeof(SolRec),
                          cudaMemcpyDeviceToHost, c->stream));
      CKE(cudaStreamSynchronize(c->stream));
      for (unsigned s = SOL_FAST; s < n2; s++)
        found.push_back(c->h_more[s]);
    }
    if (nsub)
    {
      const unsigned n2 = std::min<unsigned>(nsub, SUB_CAP);
      CKE(cudaSetDevice(c->device));
      CKE(cudaMemcpyAsync(c->h_more, c->d_subs, (size_t)n2 * sizeof(SolRec), cudaMemcpyDeviceToHost, c->stream));
      CKE(cudaStreamSynchronize(c->stream));
      for (unsigned s = 0; s < n2; s++)
        subfound.push_back(c->h_more[s]);
    }
  }
  // the all-zero prefix is walked by the device from level L-1 down; the reference does not count it on levels >= 1
  // (initial-descent compensation, enumerate_base.cpp:165-183) — only its level-0 node
  if (shard_rank == 0)
    for (int k = 1; k < L; k++)
    {
      tot[k]--;
      dev_nodes--;
    }
  // sub-solutions: the per-level minimum (what Evaluator::eval_sub_sol keeps, evaluator.h:191-205)
  if (subs && subcb)
  {
    std::vector<int> bestrec(d, -1);
    for (size_t s = 0; s < subfound.size(); s++)
    {
      const int k = subfound[s].lvl;
      if (k >= 0 && k < d && (bestrec[k] < 0 || subfound[s].dist < subfound[bestrec[k]].dist))
        bestrec[k] = (int)s;
    }
    // the host's top levels can hold sub-solutions too
    std::vector<double> sub(d);
    for (int k = d - 1; k >= 0; --k)
    {
      double bd    = bestrec[k] >= 0 ? subfound[bestrec[k]].dist : INFINITY;
      const int tt = d - 1 - k;
      int hb = -1;
      if (tt < T)
        for (size_t q = 1; q < br.lev[tt].size(); q++)
          if (br.lev[tt][q].pd != 0.0 && br.lev[tt][q].pd < rdiag[k] && br.lev[tt][q].pd < bd)
            bd = br.lev[tt][q].pd, hb = (int)q;
      if (hb < 0 && bestrec[k] < 0)
        continue;
      std::fill(sub.begin(), sub.end(), 0.0);
      if (hb >= 0)
      {
        int q = hb;
        for (int t2 = tt; t2 >= 0; --t2)
        {
          sub[d - 1 - t2] = br.lev[t2][q].x;
          q = br.lev[t2][q].parent;
        }
      }
      else
        for (int j = k; j < d; j++)
          sub[j] = subfound[bestrec[k]].x[j];
      subcb(ctx, bd, sub.data(), k);
    }
  }
  // replay the improving solutions in order of improvement through the evaluator callback
  std::sort(found.begin(), found.end(), [](const SolRec &x, const SolRec &y) { return x.dist > y.dist; });
  double cur = maxdist;
  int nrep   = 0;
  std::vector<double> sol(d);
  auto deliver = [&](const SolRec &s) -> double {
    // a dual enumeration walks the reversed dual basis: hand the coefficients back in the block's own order
    // (what EnumerationDyn does with reverse_by_swap, enumerate.cpp:150-154)
    for (int j = 0; j < d; j++)
      sol[dual ? d - 1 - j : j] = s.x[j];
    return cb ? cb(ctx, s.dist, sol.data()) : s.dist;
  };
  if (fixed)
  {
    if (!found.empty())
    {
      // the shortest vector inside the fixed region; among equally short ones the lexicographically smallest coefficient
      // vector — a function of the input alone, whatever the schedule of the walkers and the number of devices was
      const SolRec *best = &found.back();
      for (const SolRec &s : found)
        if (s.dist == best->dist && std::lexicographical_compare(s.x, s.x + d, best->x, best->x + d))
          best = &s;
      deliver(*best);
      nrep = 1;
    }
  }
  else
    for (const SolRec &s : found)
    {
      if (!(s.dist < cur))
        continue;
      cur = deliver(s);
      nrep++;
    }
  if (nodes)
    for (int k = 0; k < d; k++)
      nodes[k] = tot[k];
  const double total_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_begin).count();
  const double host_us  = std::chrono::duration<double, std::micro>(t_host - t_begin).count();
  if (stats)
  {
    stats->host_nodes = host_nodes, stats->device_nodes = dev_nodes, stats->leaves = leaves;
    stats->top_levels = T, stats->n_roots = (int)ntask, stats->n_solutions = nrep, stats->n_devices = used_dev;
    stats->n_rounds = rounds;
    stats->final_maxdist = cur, stats->device_ms = ms_total;
    stats->host_breadth_us = (float)host_us;
    stats->total_us = (float)total_us;
  }
  if (tn.trace)
  {
    static FILE *tf = fopen(tn.trace, "a");
    if (tf)
      fprintf(tf, "d=%d roots=%zu T=%d host_us=%.1f dev_ms=%.4f total_us=%.1f host_nodes=%llu dev_nodes=%llu rounds=%d "
                  "fanned=%d sols=%d\n",
              d, nroots, T, host_us, ms_total, total_us, (unsigned long long)host_nodes, (unsigned long long)dev_nodes,
              rounds, fanned ? 1 : 0, nrep);
  }
  if (overflow)
  {
    g_err = "b200enum_run: solution buffer overflow";
    return B200ENUM_EOVERFLOW;
  }
  return B200ENUM_OK;
}

}  // namespace

extern "C" {

const char *b200enum_last_error(void) { return g_err.c_str(); }

int b200enum_device_count(void)
{
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess)
  {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int b200enum_run(int dim, double maxdist, const double *mut, const double *rdiag, const double *pruning, int flags,
                 const int *devices, int ndev, int shard_rank, int shard_world, b200enum_sol_cb cb, void *ctx,
                 uint64_t *nodes, b200enum_stats *stats)
{
  if (flags & B200ENUM_FINDSUBSOLS)
    return B200ENUM_UNSUPPORTED;  // needs the sub-solution callback: b200enum_run_ex
  return b200enum_run_ex(dim, maxdist, mut, rdiag, pruning, flags, devices, ndev, shard_rank, shard_world, cb, nullptr,
                         ctx, nodes, stats);
}

int b200enum_run_ex(int dim, double maxdist, const double *mut, const double *rdiag, const double *pruning, int flags,
                    const int *devices, int ndev, int shard_rank, int shard_world, b200enum_sol_cb cb,
                    b200enum_subsol_cb subcb, void *ctx, uint64_t *nodes, b200enum_stats *stats)
{
  try
  {
    return run_impl(dim, maxdist, mut, rdiag, pruning, flags, devices, ndev, shard_rank, shard_world, cb, subcb, ctx,
                    nodes, stats);
  }
  catch (std::exception &ex)  // std::bad_alloc of the host vectors: nothing may cross the C boundary
  {
    g_err = std::string("b200enum_run: ") + ex.what();
    return B200ENUM_ECUDA;
  }
}

int b200enum_ipc_export(int device, unsigned char *handle64)
{
  if (!handle64)
    return B200ENUM_EINVAL;
  std::lock_guard<std::mutex> lock(g_mu);
  DevCtx *c;
  int rc = get_ctx(device, &c);
  if (rc)
    return rc;
  static_assert(sizeof(cudaIpcMemHandle_t) == B200ENUM_IPC_HANDLE_BYTES, "handle size");
  cudaIpcMemHandle_t h;
  CKE(cudaSetDevice(c->device));
  CKE(cudaIpcGetMemHandle(&h, c->d_blk));
  memcpy(handle64, &h, sizeof(h));
  return 0;
}

int b200enum_ipc_attach(int device, int world, int rank, const unsigned char *handles)
{
  if (!handles || world < 2 || world > MAX_PEERS || rank < 0 || rank >= world)
    return B200ENUM_EINVAL;
  std::lock_guard<std::mutex> lock(g_mu);
  DevCtx *c;
  int rc = get_ctx(device, &c);
  if (rc)
    return rc;
  CKE(cudaSetDevice(c->device));
  for (int r = 0; r < world; r++)
  {
    if (r == rank)
    {
      c->ipc_words[r] = c->words();
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)r * B200ENUM_IPC_HANDLE_BYTES, sizeof(h));
    void *p = nullptr;
    CKE(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->ipc_words[r] = (unsigned long long *)((unsigned char *)p + DevCtx::OFF_WORDS);
  }
  c->ipc_world = world, c->ipc_rank = rank;
  return 0;
}

int b200enum_ipc_detach(int device)
{
  std::lock_guard<std::mutex> lock(g_mu);
  for (auto &c : g_ctx)
    if (c.device == device && c.ipc_world)
    {
      cudaSetDevice(c.device);
      cudaStreamSynchronize(c.stream);
      for (int r = 0; r < c.ipc_world; r++)
        if (r != c.ipc_rank && c.ipc_words[r])
          cudaIpcCloseMemHandle((unsigned char *)c.ipc_words[r] - DevCtx::OFF_WORDS);
      c.ipc_world = 0;
      for (auto &p : c.ipc_words)
        p = nullptr;
    }
  return 0;
}

}  // extern "C"
