// bkz_api.cu — host control flow of BKZ 2.0, SD-BKZ and slide reduction over the device GSO / LLL (b200gso.h) and the device enumerator
// (b200enum.h).  Mirrors BKZReduction<Z_NR<long>, FP_NR<double>> (fplll/bkz.cpp) method for method; every method
// names the reference lines it restates.  Nothing here computes a Gram-Schmidt coefficient on the CPU: the host only
// decides which block, which radius and which pruning vector, and replays the enumeration result as row operations.
#include "../../include/b200bkz.h"
#include "../../include/b200enum.h"
#include "../../include/b200gso.h"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <map>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

namespace {

thread_local std::string g_bkz_err;

double now_s()
{
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

struct Pruning
{
  double gh_factor = 1.0, expectation = 1.0;  // PruningParams(), pruner/pruner.h:47
  std::vector<double> coeff;                  // empty = no pruning
};
struct Strategy
{
  std::vector<int> preproc;
  std::vector<Pruning> prune;
};

struct RedFailure
{
  int status;
};

}  // namespace

struct b200bkz
{
  std::vector<int> devs;
  std::map<int, Strategy> strat;
};

namespace {

#define GCK(call)                                                                         \
  do                                                                                      \
  {                                                                                       \
    int rc_ = (call);                                                                     \
    if (rc_ != 0)                                                                         \
      throw std::runtime_error(std::string(#call) + ": " + b200gso_last_error());         \
  } while (0)

struct SolCatch
{
  int d;
  std::vector<double> sol;
  double dist = -1;
};
double sol_cb(void *ctx, double dist, const double *sol)
{
  SolCatch *c = (SolCatch *)ctx;
  c->dist     = dist;
  c->sol.assign(sol, sol + c->d);
  return dist;  // FastEvaluator(1): the new bound is this solution (evaluator.h:122-156)
}

class Driver
{
public:
  Driver(b200bkz *ctx, b200gso_t *g, int d, const b200bkz_param &top, b200bkz_stats *st)
      : ctx(ctx), g(g), num_rows(d), top(top), st(st), rng(top.seed ? top.seed : 0x9e3779b97f4a7c15ull)
  {
    lll_delta = top.delta < 1 ? top.delta : 0.99;  // bkz.cpp:862
    // the fixed region unless the caller asks for the shrinking radius (only pruned calls: without pruning the shrinking
    // walk returns the shortest vector of the ball whatever the order, and the fixed ball would cost an unpruned BKZ-40
    // tour on dim 180 24 s instead of 1.7 s)
    enum_flags = (top.flags & B200BKZ_SHRINK_RADIUS) ? 0 : B200ENUM_FIXED_RADIUS;
  }
  int enum_flags = 0;

  // ---- thin wrappers over the device GSO -------------------------------------------------------------
  void lll(int kmin, int kstart, int kend, long *n_swaps, bool check = true)
  {
    const double t0 = now_s();
    int status      = 0;
    long stats[12]  = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    GCK(b200gso_lll_range(g, lll_delta, 0.51, kmin, kstart, kend, 0, &status, stats));
    const double dt = now_s() - t0;
    st->sec_lll += dt;
    st->lll_calls++;
#ifdef B200_LLL_PROFILE
    long pc[8];
    b200gso_lll_profile(pc);
    for (int q = 0; q < 8; q++)
      prof_cyc[q] += pc[q];
    prof_lll_sec += dt;
    prof_swaps += stats[0], prof_iters += stats[3];
#endif
    if (n_swaps)
      *n_swaps = stats[0];
    if (status != 0 && check)
      throw RedFailure{status};  // the reference throws runtime_error(RED_STATUS_STR[status]), bkz.cpp:109-112
  }
  void size_reduction(int kmin, int kend, int sr_start = 0)
  {
    const double t0 = now_s();
    int status      = 0;
    GCK(b200gso_size_reduction(g, 0.51, kmin, kend, sr_start, &status));
    st->sec_lll += now_s() - t0;
    prof_sr_sec += now_s() - t0;
    st->sizered_calls++;
    if (status != 0)
      throw RedFailure{status};  // bkz.cpp:289-292
  }
  void r_exp(int i, double &mant, long &expo)
  {
    double mu;
    const double t0 = now_s();
    GCK(b200gso_get_block(g, 0, i, 1, &mu, &mant, &expo));
    st->sec_get += now_s() - t0;
    st->get_calls++;
  }
  long long prof_cyc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  double prof_lll_sec = 0, prof_sr_sec = 0;
  long prof_swaps = 0, prof_iters = 0;
  // recorded GSO calls, flushed as one kernel launch (b200gso_apply_ops)
  std::vector<b200gso_op> ops;
  void op(int type, int a, int b, double x = 0.0)
  {
    b200gso_op o;
    o.type = type, o.a = a, o.b = b, o.pad = 0, o.x = x;
    ops.push_back(o);
  }
  void row_addmul(int i, int j, double x) { op(B200GSO_OP_ROW_ADDMUL, i, j, x); }
  void move_row(int a, int b) { op(B200GSO_OP_MOVE_ROW, a, b); }
  void row_swap(int a, int b) { op(B200GSO_OP_ROW_SWAP, a, b); }
  void row_op_end(int a, int b) { op(B200GSO_OP_ROW_OP_END, a, b); }
  void negate_row(int a) { op(B200GSO_OP_NEGATE, a, 0); }
  void flush()
  {
    if (ops.empty())
      return;
    const double t0 = now_s();
    GCK(b200gso_apply_ops(g, ops.data(), (int)ops.size()));
    st->sec_ops += now_s() - t0;
    st->op_calls++;
    st->ops_total += (long)ops.size();
    ops.clear();
  }

  // adjust_radius_to_gh_bound, gso_interface.cpp:260-276
  static void adjust_radius_to_gh_bound(double &max_dist, long max_dist_expo, int block_size, double root_det,
                                        double gh_factor)
  {
    double t = (double)block_size / 2.0 + 1;
    t        = lgamma(t);
    t        = pow(M_E, t * 2.0 / (double)block_size);
    t        = t / M_PI;
    double f = t * root_det;
    f        = ldexp(f, (int)-max_dist_expo);
    f        = f * gh_factor;
    if (f < max_dist)
      max_dist = f;
  }

  const Strategy &strategy(int block_size)
  {
    static const Strategy empty_with_default = [] {
      Strategy s;
      s.prune.emplace_back();  // Strategy::EmptyStrategy, bkz_param.h:46-52
      return s;
    }();
    auto it = ctx->strat.find(block_size);
    if (it == ctx->strat.end() || it->second.prune.empty())
    {
      if (it != ctx->strat.end())
      {
        tmp      = it->second;
        tmp.prune.emplace_back();
        return tmp;
      }
      return empty_with_default;
    }
    return it->second;
  }

  // rerandomize_block, bkz.cpp:43-80 (std::mt19937_64 instead of the GMP global state)
  void rerandomize_block(int min_row, int max_row, int density)
  {
    if (max_row - min_row < 2)
      return;
    auto below = [&](unsigned long n) { return (unsigned long)(rng() % n); };
    // 1. permute rows.  The reference issues 4*(max_row-min_row) move_row calls; the block is re-converted and
    // invalidated by the row_op_end below, so of all those rotations only the NET permutation of the integer rows
    // is observable (SURVEY Appendix A: everything a move_row leaves valid lies in columns < min_row or in rows
    // >= max_row, which a rotation inside the block does not touch).  Simulate the moves on an index vector and
    // apply the result as at most max_row-min_row-1 integer row swaps.
    const size_t niter = 4 * (size_t)(max_row - min_row);
    const int m        = max_row - min_row;
    std::vector<int> cur(m);
    for (int i = 0; i < m; i++)
      cur[i] = i;
    for (size_t i = 0; i < niter; ++i)
    {
      size_t a = below(max_row - min_row - 1), b = a;
      while (b == a)
        b = below(max_row - min_row - 1);
      const int t = cur[b];  // move_row(b, a): row b lands at a, rows between shift by one
      cur.erase(cur.begin() + b);
      cur.insert(cur.begin() + a, t);
    }
    {
      std::vector<int> at(m), where(m);  // at[p] = original row now at position p, where[o] = position of row o
      for (int i = 0; i < m; i++)
        at[i] = where[i] = i;
      for (int p = 0; p < m; p++)
      {
        const int q = where[cur[p]];
        if (q != p)
        {
          row_swap(min_row + p, min_row + q);
          const int op_ = at[p], oq = at[q];
          at[p] = oq, at[q] = op_;
          where[oq] = p, where[op_] = q;
        }
      }
    }
    for (long a = min_row; a < max_row - 2; ++a)
      for (long i = 0; i < density; i++)
      {
        size_t b = below(max_row - (a + 1) - 1) + a + 1;
        row_addmul((int)a, (int)b, below(2) ? 1.0 : -1.0);  // row_add / row_sub
      }
    row_op_end(min_row, max_row);
    flush();
  }

  // svp_preprocessing, bkz.cpp:100-126
  bool svp_preprocessing(int kappa, int block_size, const b200bkz_param &par)
  {
    bool clean          = true;
    const int lll_start = (par.flags & B200BKZ_BOUNDED_LLL) ? kappa : 0;
    long swaps          = 0;
    lll(lll_start, lll_start, kappa + block_size, &swaps);
    if (swaps > 0)
      clean = false;
    const std::vector<int> preproc = strategy(block_size).preproc;
    for (int pb : preproc)
    {
      int dummy_kappa_max = num_rows;
      b200bkz_param prepar;
      b200bkz_default_param(&prepar, pb);
      prepar.flags = B200BKZ_GH_BND;
      clean &= tour(0, dummy_kappa_max, prepar, kappa, kappa + block_size);
    }
    return clean;
  }

  // svp_postprocessing, bkz.cpp:128-203.  Dual: the solution is a dual vector; the row operations are the transposed
  // inverses of the primal ones and the new vector lands at the END of the block (pos = kappa + block_size - 1).
  void svp_postprocessing(int kappa, int block_size, const std::vector<double> &solution, bool dual)
  {
    int nz_vectors = 0, i_vector = -1;
    for (int i = block_size - 1; i >= 0; i--)
      if (solution[i] != 0)
      {
        nz_vectors++;
        if (i_vector == -1 && fabs(solution[i]) == 1)
          i_vector = i;
      }
    const int pos = dual ? kappa + block_size - 1 : kappa;
    if (nz_vectors == 1)
      move_row(kappa + i_vector, pos);
    else if (i_vector != -1)
    {
      int sol_i = (int)solution[i_vector];
      if (dual)
        sol_i *= -1;
      for (int i = 0; i < block_size; ++i)
        if (solution[i] != 0 && i != i_vector)
        {
          if (dual)
            row_addmul(kappa + i, kappa + i_vector, sol_i * solution[i]);
          else
            row_addmul(kappa + i_vector, kappa + i, sol_i * solution[i]);
        }
      if (dual)
        row_op_end(kappa, kappa + block_size);
      else
        row_op_end(kappa + i_vector, kappa + i_vector + 1);
      move_row(kappa + i_vector, pos);
    }
    else
      svp_postprocessing_generic(kappa, block_size, solution, dual);
    flush();
  }

  // svp_postprocessing_generic, bkz.cpp:205-272: tree-based gcd on the coefficient vector (dual: row_sub in the other
  // direction, and the vector is already where it belongs, at the end of the block)
  void svp_postprocessing_generic(int kappa, int block_size, const std::vector<double> &solution, bool dual)
  {
    std::vector<double> x = solution;
    const int dd          = block_size;
    for (int i = 0; i < dd; i++)
      if (x[i] < 0)
      {
        x[i] = -x[i];
        negate_row(i + kappa);
      }
    int off = 1, k;
    while (off < dd)
    {
      k = dd - 1;
      while (k - off >= 0)
      {
        if (!(x[k] == 0 && x[k - off] == 0))
        {
          if (x[k] < x[k - off])
          {
            std::swap(x[k], x[k - off]);
            row_swap(kappa + k - off, kappa + k);
          }
          while (x[k - off] != 0)
          {
            while (x[k - off] <= x[k])
            {
              x[k] = x[k] - x[k - off];
              if (dual)
                row_addmul(kappa + k, kappa + k - off, -1.0);  // row_sub(kappa + k, kappa + k - off)
              else
                row_addmul(kappa + k - off, kappa + k, 1.0);  // row_add(kappa + k - off, kappa + k)
            }
            std::swap(x[k], x[k - off]);
            row_swap(kappa + k - off, kappa + k);
          }
        }
        k -= 2 * off;
      }
      off *= 2;
    }
    row_op_end(kappa, kappa + dd);
    if (!dual)
      move_row(kappa + dd - 1, kappa);
  }

  // svp_reduction, bkz.cpp:274-358.  Dual: the block's LAST Gram-Schmidt vector is the one to shorten; the radius is
  // delta / r(first, first) (exponent negated), while the GH bound and get_pruning still read the primal block.
  bool svp_reduction(int kappa, int block_size, const b200bkz_param &par, bool dual = false)
  {
    const int first = dual ? kappa + block_size - 1 : kappa;
    size_reduction(0, first + 1, 0);
    double old_first;
    long old_first_expo;
    r_exp(first, old_first, old_first_expo);
    bool rerandomize             = false;
    double remaining_probability = 1.0;
    std::vector<double> mut((size_t)block_size * block_size), rmant(block_size), rdiag(block_size);
    std::vector<long> rexpo(block_size);
    while (remaining_probability > 1. - par.min_success_probability)
    {
      if (rerandomize)
        rerandomize_block(kappa + 1, kappa + block_size, par.rerandomization_density);
      svp_preprocessing(kappa, block_size, par);

      {
        const double tg = now_s();
        GCK(b200gso_get_block(g, 0, kappa, block_size, mut.data(), rmant.data(), rexpo.data()));
        st->sec_get += now_s() - tg;
        st->get_calls++;
      }
      // a zero r(i, i) (a dependent row inside the reduced range) has no place in the enumerator: its normalisation and
      // radius would be meaningless and the walk need not end
      for (int i = 0; i < block_size; i++)
        if (!(rmant[i] > 0))
          throw std::runtime_error("BKZ block [" + std::to_string(kappa) + ", " + std::to_string(kappa + block_size) +
                                   ") has r(" + std::to_string(kappa + i) + ", " + std::to_string(kappa + i) +
                                   ") = 0: the rows are linearly dependent");
      long max_dist_expo = rexpo[first - kappa];
      double max_dist    = rmant[first - kappa];
      if (dual)
      {
        max_dist      = pow(max_dist, -1.0);  // FP_NR<double>::pow_si(max_dist, -1), nr_FP_d.inl:189-192
        max_dist_expo = -max_dist_expo;
      }
      max_dist *= delta();
      double log_det = 0;  // get_root_det / get_log_det, gso_interface.cpp:220-242 (the primal block in both cases)
      for (int i = 0; i < block_size; i++)
        log_det += log(ldexp(rmant[i], (int)rexpo[i]));
      const double root_det = exp(log_det / block_size);
      if ((par.flags & B200BKZ_GH_BND) && block_size > 30)
        adjust_radius_to_gh_bound(max_dist, max_dist_expo, block_size, root_det, par.gh_factor);

      // get_pruning, bkz.cpp:82-98 + Strategy::get_pruning, bkz_param.cpp:62-78: reads the primal r(kappa, kappa) even
      // in a dual call, as the reference does
      const Strategy &strat = strategy(block_size);
      const long kexpo      = rexpo[0];
      double gh_max_dist    = rmant[0];
      adjust_radius_to_gh_bound(gh_max_dist, kexpo, block_size, root_det, 1.0);
      const double radius = rmant[0] * pow(2, kexpo), gh = gh_max_dist * pow(2, kexpo);
      const double ghf    = radius / gh;
      const Pruning *pr   = &strat.prune[0];
      double closest      = pow(2, 80);
      for (const Pruning &p : strat.prune)
        if (fabs(p.gh_factor - ghf) < closest)
        {
          closest = fabs(p.gh_factor - ghf);
          pr      = &p;
        }

      // normalisation as the enumerators do it: primal rdiag scaled by 2^-normexp (enumerate_ext.cpp:64-79,100-106);
      // a dual radius is a bound on 1/r, so it scales by 2^+normexp (enumerate.cpp:98-105)
      long normexp = -1;
      for (int i = 0; i < block_size; i++)
        normexp = std::max(normexp, rexpo[i] + (long)ilogb(rmant[i]) + 1);
      const double maxdist_norm = ldexp(max_dist, (int)(dual ? max_dist_expo + normexp : max_dist_expo - normexp));
      for (int i = 0; i < block_size; i++)
        rdiag[i] = ldexp(rmant[i], (int)(rexpo[i] - normexp));
      SolCatch sc;
      sc.d = block_size;
      if (block_size >= 2)
      {
        // (a block of one row, the tail of a slide tour, has no vector shorter than delta times its own)
        b200enum_stats es;
        std::vector<uint64_t> nodes(block_size);
        const int eflags = (pr->coeff.empty() ? 0 : enum_flags) | (dual ? B200ENUM_DUAL : 0);
        const double t0  = now_s();
        const int rc     = b200enum_run(block_size, maxdist_norm, mut.data(), rdiag.data(),
                                        pr->coeff.empty() ? nullptr : pr->coeff.data(), eflags, ctx->devs.data(),
                                        (int)ctx->devs.size(), 0, 1, sol_cb, &sc, nodes.data(), &es);
        st->sec_enum += now_s() - t0;
        st->enum_calls++;
        if (rc != 0)
          throw std::runtime_error(std::string("b200enum_run: ") + b200enum_last_error());
        for (uint64_t v : nodes)
          st->enum_nodes += v;
      }

      if (sc.dist > 0)
      {
        svp_postprocessing(kappa, block_size, sc.sol, dual);
        rerandomize = false;
      }
      else
        rerandomize = true;
      remaining_probability *= (1 - pr->expectation);
    }
    size_reduction(0, first + 1, 0);
    double new_first;
    long new_first_expo;
    r_exp(first, new_first, new_first_expo);
    new_first = ldexp(new_first, (int)(new_first_expo - old_first_expo));
    return dual ? old_first >= new_first : old_first <= new_first;
  }

  // tour / trunc_tour / hkz, bkz.cpp:360-441
  bool tour(int loop, int &kappa_max, const b200bkz_param &par, int min_row, int max_row)
  {
    (void)loop;
    bool clean = true;
    clean &= trunc_tour(kappa_max, par, min_row, max_row);
    clean &= hkz(kappa_max, par, std::max(max_row - par.block_size, 0), max_row);
    return clean;
  }
  bool trunc_tour(int &kappa_max, const b200bkz_param &par, int min_row, int max_row)
  {
    bool clean = true;
    for (int kappa = min_row; kappa < max_row - par.block_size; ++kappa)
    {
      clean &= svp_reduction(kappa, par.block_size, par);
      if (kappa_max < kappa && clean)
        kappa_max = kappa;
    }
    return clean;
  }
  bool hkz(int &kappa_max, const b200bkz_param &par, int min_row, int max_row)
  {
    bool clean = true;
    for (int kappa = min_row; kappa < max_row - 1; ++kappa)
    {
      clean &= svp_reduction(kappa, max_row - kappa, par);
      if (kappa_max < kappa && clean)
        kappa_max = kappa;
    }
    {
      // bkz.cpp:436-438: the reference calls lll_obj.size_reduction here and IGNORES its return value (a Babai failure
      // at this point does not abort the tour)
      const double t0 = now_s();
      int status      = 0;
      GCK(b200gso_size_reduction(g, 0.51, max_row - 1, max_row, max_row - 2, &status));
      st->sec_lll += now_s() - t0;
      st->sizered_calls++;
    }
    return clean;
  }

  // trunc_dtour, bkz.cpp:405-417: dual SVP reduction of the blocks ending at max_row - 1, max_row - 2, ..., min_row + block_size
  bool trunc_dtour(const b200bkz_param &par, int min_row, int max_row)
  {
    bool clean = true;
    for (int kappa = max_row - par.block_size; kappa > min_row; --kappa)
      clean &= svp_reduction(kappa, par.block_size, par, true);
    return clean;
  }

  // sd_tour, bkz.cpp:443-463: a dual tour backwards, then a truncated primal tour forwards
  bool sd_tour(const b200bkz_param &par, int min_row, int max_row)
  {
    int dummy_kappa_max = num_rows;
    bool clean          = true;
    clean &= trunc_dtour(par, min_row, max_row);
    clean &= trunc_tour(dummy_kappa_max, par, min_row, max_row);
    return clean;
  }

  // slide_tour, bkz.cpp:465-520: SVP-reduce the disjoint blocks until nothing changes, then dual-SVP-reduce the blocks
  // shifted by one; progress is measured by the slide potential
  bool slide_tour(const b200bkz_param &par, int min_row, int max_row)
  {
    int p = (max_row - min_row) / par.block_size;
    if ((max_row - min_row) % par.block_size)
      ++p;
    bool clean;  // only for the inner loop
    do
    {
      clean = true;
      for (int i = 0; i < p; ++i)
      {
        const int kappa      = min_row + i * par.block_size;
        const int block_size = std::min(max_row - kappa, par.block_size);
        clean &= svp_reduction(kappa, block_size, par);
      }
      if (par.flags & B200BKZ_BOUNDED_LLL)  // otherwise svp_preprocessing's LLL from row 0 covers it
      {
        long swaps = 0;
        lll(min_row, min_row, max_row, &swaps);
        if (swaps > 0)
          clean = false;
      }
    } while (!clean);
    for (int i = 0; i < p - 1; ++i)
      svp_reduction(min_row + i * par.block_size + 1, par.block_size, par, true);
    const double new_potential = slide_potential(min_row, max_row, par.block_size);
    if (new_potential >= sld_potential)
      return true;
    sld_potential = new_potential;
    return false;
  }

  // get_slide_potential, gso_interface.cpp:244-258, over get_log_det (:230-242) of the STORED r diagonal (get_r, no
  // update_gso: the reference reads whatever the last reduction left, and so must the termination test here)
  double slide_potential(int start_row, int end_row, int block_size)
  {
    int p = (end_row - start_row) / block_size;
    if ((end_row - start_row) % block_size == 0)
      --p;
    if (p <= 0)
      return 0.0;
    const int n = p * block_size;
    std::vector<double> mant(n);
    std::vector<long> expo(n);
    GCK(b200gso_get_r_diag(g, 0, 0, n, mant.data(), expo.data()));
    return b200bkz_slide_potential_of(mant.data(), expo.data(), start_row, end_row, block_size);
  }
  double sld_potential = 0;

  // get_current_slope, gso_interface.cpp:198-218 (requires valid rows: callers run after LLL / a tour)
  double current_slope(int start_row, int stop_row)
  {
    const int n = stop_row - start_row;
    std::vector<double> mant(n);
    std::vector<long> expo(n);
    int ok = 1;
    GCK(b200gso_update_gso(g, &ok));
    GCK(b200gso_get_r_diag(g, 0, start_row, n, mant.data(), expo.data()));
    double v1 = 0, v2 = (double)(n + 1) * n * (n - 1) / 12.0, weight = (1.0 - n) / 2.0;
    for (int i = 0; i < n; i++)
    {
      v1 += weight * (log(mant[i]) + expo[i] * log(2.0));
      weight++;
    }
    return v1 / v2;
  }

  // bkz(), bkz.cpp:522-672: plain BKZ, SD-BKZ (B200BKZ_SD_VARIANT) or slide reduction (B200BKZ_SLD_RED)
  int bkz()
  {
    int flags        = top.flags;
    int final_status = 0;
    const bool sd = (flags & B200BKZ_SD_VARIANT) != 0, sld = (flags & B200BKZ_SLD_RED) != 0;
    const char *algorithm = sd ? "SD-BKZ" : sld ? "SLD" : "BKZ";
    if (sd && sld)
      throw std::runtime_error(B200BKZ_SD_SLD_MSG);
    if (top.block_size < 2)
      return 0;
    if (sd && !(flags & (B200BKZ_MAX_LOOPS | B200BKZ_MAX_TIME | B200BKZ_AUTO_ABORT)))
    {
      fprintf(stderr, "Warning: SD Variant of BKZ requires explicit termination condition. Turning auto abort on!\n");
      flags |= B200BKZ_AUTO_ABORT;
    }
    if (flags & B200BKZ_VERBOSE)
      fprintf(stderr, "Entering %s: block size %d\n", algorithm, top.block_size);
    GCK(b200gso_discover_all_rows(g));
    const double t_start = now_s();
    if (sld)
    {
      int ok = 1;
      GCK(b200gso_update_gso(g, &ok));
      sld_potential = slide_potential(0, num_rows, top.block_size);
    }
    if (sd)  // sd-bkz starts with a dual tour, whose size reductions need LLL-reduced lower blocks (bkz.cpp:573-577; the
      lll(0, 0, num_rows, nullptr, false);  // reference ignores this call's status)
    int no_dec           = -1;
    double old_slope     = std::numeric_limits<double>::max();
    int kappa_max        = -1;
    bool clean           = true;
    int i                = 0;
    for (i = 0;; ++i)
    {
      if ((flags & B200BKZ_MAX_LOOPS) && i >= top.max_loops)
      {
        final_status = B200_RED_BKZ_LOOPS_LIMIT;
        break;
      }
      if ((flags & B200BKZ_MAX_TIME) && now_s() - t_start >= top.max_time)
      {
        final_status = B200_RED_BKZ_TIME_LIMIT;
        break;
      }
      if (flags & B200BKZ_AUTO_ABORT)
      {
        // BKZAutoAbort::test_abort, bkz.cpp:800-809
        const double new_slope = -current_slope(0, num_rows);
        if (no_dec == -1 || new_slope < top.auto_abort_scale * old_slope)
          no_dec = 0;
        else
          no_dec++;
        old_slope = std::min(old_slope, new_slope);
        if (no_dec >= top.auto_abort_max_no_dec)
          break;
      }
      if (sd)
        clean = sd_tour(top, 0, num_rows);
      else if (sld)
        clean = slide_tour(top, 0, num_rows);
      else
        clean = tour(i, kappa_max, top, 0, num_rows);
      st->tours = i + 1;
      if (flags & B200BKZ_VERBOSE)
      {
        double m;
        long e;
        r_exp(0, m, e);
        fprintf(stderr, "End of %s loop %d, time = %.3fs, r_0 = %.6g, enum nodes = 2^%.2f\n", algorithm, i,
                now_s() - t_start, ldexp(m, (int)e), log2((double)st->enum_nodes + 1));
      }
      if (clean || top.block_size >= num_rows)
        break;
    }
    int dummy_kappa_max = num_rows;
    if (sd)  // hkz-reduce the last window, which SD-BKZ leaves unreduced (bkz.cpp:626-641)
      hkz(dummy_kappa_max, top, std::max(num_rows - top.block_size, 0), num_rows);
    if (sld)
    {
      // hkz-reduce the blocks, which slide reduction leaves only SVP- and dual-SVP-reduced (bkz.cpp:642-665)
      int p = num_rows / top.block_size;
      if (num_rows % top.block_size)
        ++p;
      for (int j = 0; j < p; ++j)
      {
        const int kappa = j * top.block_size + 1;
        hkz(dummy_kappa_max, top, kappa, std::min(num_rows, kappa + top.block_size - 1));
      }
    }
    return final_status;
  }

  double delta() const { return top.delta; }
  // BKZReduction's constructor, bkz.cpp:35: the rows the tours reduce end before the trailing zero rows
  void set_num_rows(int rows) { num_rows = rows; }

private:
  b200bkz *ctx;
  b200gso_t *g;
  int num_rows;  // rows 0..num_rows-1: the basis without its trailing zero rows (bkz.cpp:35)
  const b200bkz_param &top;
  b200bkz_stats *st;
  std::mt19937_64 rng;
  double lll_delta;
  Strategy tmp;
};

// zeros_last / zeros_first (util.cpp:257-287) on the host arrays: rotate the rows so that row mid comes first, in b
// (d x n) and, when given, u (d x d)
void rotate_rows(int64_t *b, int d, int n, int64_t *u, int mid)
{
  if (mid <= 0 || mid >= d)
    return;
  std::rotate(b, b + (size_t)mid * n, b + (size_t)d * n);
  if (u)
    std::rotate(u, u + (size_t)mid * d, u + (size_t)d * d);
}
bool row_is_zero(const int64_t *b, int n, int i)
{
  for (int j = 0; j < n; j++)
    if (b[(size_t)i * n + j] != 0)
      return false;
  return true;
}
// the leading zero rows to the end (bkz.cpp:869-870 under BKZ_NO_LLL)
void zeros_last(int64_t *b, int d, int n, int64_t *u)
{
  int i = 0;
  while (i < d && row_is_zero(b, n, i))
    i++;
  rotate_rows(b, d, n, u, i);
}
// the number of rows before the trailing zero rows (BKZReduction::num_rows, bkz.cpp:35)
int nonzero_prefix(const int64_t *b, int d, int n)
{
  int i = d;
  while (i > 0 && row_is_zero(b, n, i - 1))
    i--;
  return i;
}
// the trailing zero rows to the front (bkz.cpp:925)
void zeros_first(int64_t *b, int d, int n, int64_t *u) { rotate_rows(b, d, n, u, nonzero_prefix(b, d, n)); }

}  // namespace

extern "C" {

const char *b200bkz_last_error(void) { return g_bkz_err.c_str(); }

double b200bkz_slide_potential_of(const double *rmant, const long *rexpo, int start_row, int end_row, int block_size)
{
  // get_slide_potential / get_log_det, gso_interface.cpp:230-258, in the reference's order of operations
  double potential = 0.0;
  int p            = (end_row - start_row) / block_size;
  if ((end_row - start_row) % block_size == 0)
    --p;
  for (int i = 0; i < p; ++i)
  {
    double log_det = 0.0;
    for (int k = i * block_size; k < (i + 1) * block_size; ++k)
      log_det += log(ldexp(rmant[k], (int)rexpo[k]));
    potential += (double)(p - i) * log_det;
  }
  return potential;
}

void b200bkz_default_param(b200bkz_param *p, int block_size)
{
  memset(p, 0, sizeof(*p));
  p->block_size              = block_size;
  p->delta                   = 0.99;  // LLL_DEF_DELTA
  p->flags                   = B200BKZ_DEFAULT;
  p->auto_abort_scale        = 1.0;   // BKZ_DEF_AUTO_ABORT_SCALE
  p->auto_abort_max_no_dec   = 5;     // BKZ_DEF_AUTO_ABORT_MAX_NO_DEC
  p->gh_factor               = 1.1;   // BKZ_DEF_GH_FACTOR
  p->min_success_probability = 0.5;   // BKZ_DEF_MIN_SUCCESS_PROBABILITY
  p->rerandomization_density = 3;     // BKZ_DEF_RERANDOMIZATION_DENSITY
}

int b200bkz_create(b200bkz_t **out, const int *devices, int ndev)
{
  if (!out)
    return B200BKZ_EINVAL;
  if (b200gso_device_count() == 0)
  {
    g_bkz_err = "b200bkz_create: no CUDA device (no CPU fallback)";
    return B200BKZ_ENODEV;
  }
  b200bkz *h = new b200bkz();
  if (devices && ndev > 0)
    h->devs.assign(devices, devices + ndev);
  else
    h->devs.push_back(0);
  *out = h;
  return 0;
}

void b200bkz_destroy(b200bkz_t *h) { delete h; }

int b200bkz_add_strategy(b200bkz_t *h, int block_size, const int *preproc, int n_preproc, const double *gh_factor,
                         const double *expectation, const double *coefficients, int n_prune)
{
  if (!h || block_size < 0 || n_preproc < 0 || n_prune < 0)
    return B200BKZ_EINVAL;
  Strategy s;
  for (int i = 0; i < n_preproc; i++)
    s.preproc.push_back(preproc[i]);
  for (int i = 0; i < n_prune; i++)
  {
    Pruning p;
    p.gh_factor   = gh_factor[i];
    p.expectation = expectation[i];
    p.coeff.assign(coefficients + (size_t)i * block_size, coefficients + (size_t)(i + 1) * block_size);
    s.prune.push_back(p);
  }
  h->strat[block_size] = s;
  return 0;
}

}  // extern "C"

// b200bkz_reduce (u == nullptr) and b200bkz_reduce_transform: u rides along on a B200GSO_TRANSFORM handle, which takes
// every decision exactly as an untransformed one would.
static int bkz_reduce(b200bkz_t *h, int d, int n, int64_t *b, int64_t *u, const b200bkz_param *param,
                      b200bkz_stats *stats)
{
  if (!h || !b || !param || d < 1 || n < 1)
  {
    g_bkz_err = "b200bkz_reduce: bad arguments";
    return B200BKZ_EINVAL;
  }
  if ((param->flags & B200BKZ_SD_VARIANT) && (param->flags & B200BKZ_SLD_RED))
  {
    g_bkz_err = B200BKZ_SD_SLD_MSG;  // bkz.cpp:531-534
    return B200BKZ_EINVAL;
  }
  b200bkz_stats local;
  if (!stats)
    stats = &local;
  memset(stats, 0, sizeof(*stats));
  if (param->flags & B200BKZ_NO_LLL)
    zeros_last(b, d, n, u);  // bkz.cpp:869-870; with the wrapper LLL, LLL itself moves zero rows to the end
  b200gso_t *g = nullptr;
  int rc       = b200gso_create(&g, 1, d, n, B200GSO_ROW_EXPO | (u ? B200GSO_TRANSFORM : 0), h->devs[0]);  // bkz.cpp:819-820
  if (rc)
  {
    g_bkz_err = b200gso_last_error();
    return rc == B200GSO_ENODEV ? B200BKZ_ENODEV : B200BKZ_ECUDA;
  }
  const double t0 = now_s();
  int ret         = 0;
  try
  {
    GCK(b200gso_set_basis(g, b));
    if (u)
      GCK(b200gso_set_transform(g, u));  // the caller's U (bkz.cpp:857-859 starts it at the identity)
    Driver drv(h, g, d, *param, stats);
    double tb         = now_s();
    int num_rows      = d;
    bool wrapper_fail = false;
    try
    {
      if (!(param->flags & B200BKZ_NO_LLL))
      {
        // the reference runs its wrapper LLL here (bkz.cpp:869-876); in the int64 regime that is LLL(delta, 0.51).
        // A failure of this LLL (RED_BABAI_FAILURE on an fp64-fragile basis) is the call's status, not an exception.
        long swaps;
        wrapper_fail = true;
        drv.lll(0, 0, d, &swaps);
        wrapper_fail = false;
      }
      else
      {
        int ok = 1;
        GCK(b200gso_update_gso(g, &ok));
      }
      {
        // the tours reduce the rows before the trailing zero rows only (bkz.cpp:35): no block ever holds a zero row
        std::vector<int64_t> cur((size_t)d * n);
        GCK(b200gso_get_basis(g, cur.data()));
        num_rows = nonzero_prefix(cur.data(), d, n);
        drv.set_num_rows(num_rows);
      }
      if (num_rows > 0)
      {
        stats->slope_before = drv.current_slope(0, num_rows);
        double m;
        long e;
        drv.r_exp(0, m, e);
        stats->r00_before = ldexp(m, (int)e);
      }
      stats->sec_lll = 0, stats->lll_calls = 0;
      tb            = now_s();
      stats->status = num_rows > 0 ? drv.bkz() : 0;  // a zero basis has nothing to reduce
    }
    catch (RedFailure &f)
    {
      stats->status = f.status;  // the reference lets this escape as runtime_error (SURVEY §0.8); report the status
    }
    stats->sec_total = now_s() - tb;
#ifdef B200_LLL_PROFILE
    fprintf(stderr, "LLL profile (lll calls only): %.1f s wall; device cycles update_gso_row %.3g, babai-rest %.3g, "
                    "lovasz %.3g, move_row+set_r %.3g; swaps %ld, babai iterations %ld\n",
            drv.prof_lll_sec, (double)drv.prof_cyc[0], (double)drv.prof_cyc[1], (double)drv.prof_cyc[2],
            (double)drv.prof_cyc[3], drv.prof_swaps, drv.prof_iters);
    fprintf(stderr, "  inside babai-rest: gather/scan %.3g, back-substitution %.3g, compaction+integer rows %.3g, row_op_end "
                    "%.3g cycles; size_reduction calls %.1f s wall\n",
            (double)drv.prof_cyc[4], (double)drv.prof_cyc[5], (double)drv.prof_cyc[6], (double)drv.prof_cyc[7],
            drv.prof_sr_sec);
    {
      long long cp[32];
      b200gso_lll_cta_profile(cp);
      fprintf(stderr, "  CTA ops (all LLL + size-reduction calls): update calls %lld (mean i %.1f, wavefront steps %lld, Gram entries "
                      "%lld): Gram+prefix %.3g, wavefront %.3g, diagonal %.3g cycles; back-substitutions %lld (steps %lld) %.3g "
                      "cycles; integer-row calls %lld (rows %lld) %.3g cycles\n",
              cp[0], cp[0] ? (double)cp[12] / cp[0] : 0.0, cp[1], cp[13], (double)cp[2], (double)cp[3], (double)cp[4], cp[5],
              cp[6], (double)cp[7], cp[9], cp[10], (double)cp[11]);
      fprintf(stderr, "  streamed ops: back-substitution top-panel triangle %.3g cycles over %lld rows, bottom panel: consumer "
                      "%.3g + triangle %.3g cycles over %lld rows; update: first-panel triangle %.3g, last panel consumer %.3g "
                      "+ triangle %.3g; master Gram dot %.3g, prefix chain %.3g cycles\n",
              (double)cp[8], cp[14], (double)cp[16], (double)cp[17], cp[15], (double)cp[18], (double)cp[19], (double)cp[20],
              (double)cp[21], (double)cp[22]);
    }
#endif
    stats->sec_other = stats->sec_total - stats->sec_enum - stats->sec_lll;
    if (num_rows > 0 &&
        (stats->status == 0 || stats->status == B200_RED_BKZ_LOOPS_LIMIT || stats->status == B200_RED_BKZ_TIME_LIMIT))
    {
      stats->slope_after = drv.current_slope(0, num_rows);
      double m;
      long e;
      drv.r_exp(0, m, e);
      stats->r00_after = ldexp(m, (int)e);
    }
    GCK(b200gso_get_basis(g, b));
    if (u)
      GCK(b200gso_get_transform(g, u));
    if (!wrapper_fail)
      zeros_first(b, d, n, u);  // bkz.cpp:925 (a failed wrapper LLL returns before it, bkz.cpp:874-875)
  }
  catch (std::exception &ex)
  {
    g_bkz_err = ex.what();
    ret       = B200BKZ_ECUDA;
  }
  catch (...)  // nothing may cross the C boundary
  {
    g_bkz_err = "b200bkz_reduce: unknown C++ exception";
    ret       = B200BKZ_ECUDA;
  }
  (void)t0;
  b200gso_destroy(g);
  return ret;
}

extern "C" {

int b200bkz_reduce(b200bkz_t *h, int d, int n, int64_t *b, const b200bkz_param *param, b200bkz_stats *stats)
{
  return bkz_reduce(h, d, n, b, nullptr, param, stats);
}

int b200bkz_reduce_transform(b200bkz_t *h, int d, int n, int64_t *b, int64_t *u, const b200bkz_param *param,
                             b200bkz_stats *stats)
{
  if (!u)
  {
    g_bkz_err = "b200bkz_reduce_transform: u is NULL";
    return B200BKZ_EINVAL;
  }
  return bkz_reduce(h, d, n, b, u, param, stats);
}

}  // extern "C"
