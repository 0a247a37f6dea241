/* ref_probe — TEST INFRASTRUCTURE (oracle side), not product code.
 *
 * A command interpreter over the UNMODIFIED reference library (oracle/_ref/libfplll.so, built from
 * /root/reference by oracle/Makefile.ref).  It lets the parity tests drive the reference's own
 * MatGSO<Z_NR<long|mpz_t>, FP_NR<double>> / MatHouseholder / LLL / BKZ / Enumeration objects one call at
 * a time and dump their complete floating-point state as raw binary, and it is the `cpu_baseline`
 * ("kind": "reference") timer of bench.py.  Nothing under fplll_b200/ links or executes it.
 *
 * Commands are read from stdin, one per line (see `help`).  Dump record layout (little endian):
 *   int32 magic=0x4753304f, d, n, n_known_rows, n_known_cols, n_source_rows, flags, ztype(0=long,1=mpz)
 *   int64 row_expo[d]; int32 gso_valid_cols[d]; int32 init_row_size[d]
 *   f64 bf[d*n]; f64 gf[d*d]; f64 mu[d*d]; f64 r[d*d]; int64 b[d*n] (ztype long only, else absent)
 */
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <functional>
#include <iostream>
#include <map>
#include <memory>
#include <numeric>
#include <set>
#include <sstream>
#include <string>
#include <thread>
#include <vector>
/* the probe reads private state of the reference classes (MatHouseholder::R, V, sigma ...): same object layout,
   access checks off — standard headers are already included above so only fplll's own declarations are affected */
#define private public
#define protected public
#include <fplll.h>
#undef private
#undef protected

using namespace fplll;
using namespace std;

typedef MatGSO<Z_NR<long>, FP_NR<double>> GsoL;
typedef MatGSO<Z_NR<mpz_t>, FP_NR<double>> GsoM;

static ZZ_mat<mpz_t> Bm, Um, UTm;
static ZZ_mat<long> Bl, Ul, UTl;
static unique_ptr<GsoL> gl;
static unique_ptr<GsoM> gm;
static int gflags = 0;

static double now()
{
  return chrono::duration<double>(chrono::steady_clock::now().time_since_epoch()).count();
}

template <class T> static void wr(FILE *f, const T *p, size_t n) { fwrite(p, sizeof(T), n, f); }

template <class G> static void dump_state(G &m, const char *path, int ztype)
{
  FILE *f = fopen(path, "ab");
  if (!f)
  {
    perror(path);
    exit(2);
  }
  int d = m.d, n = m.b.get_cols();
  int32_t hdr[8] = {0x4753304f, d, n, m.n_known_rows, m.n_known_cols, m.n_source_rows, gflags, ztype};
  wr(f, hdr, 8);
  vector<int64_t> re(d, 0);
  if (m.enable_row_expo)
    for (int i = 0; i < d; i++)
      re[i] = m.row_expo[i];
  wr(f, re.data(), d);
  vector<int32_t> vc(d), irs(d);
  for (int i = 0; i < d; i++)
  {
    vc[i]  = m.gso_valid_cols[i];
    irs[i] = m.init_row_size[i];
  }
  wr(f, vc.data(), d);
  wr(f, irs.data(), d);
  vector<double> buf((size_t)d * n);
  for (int i = 0; i < d; i++)
    for (int j = 0; j < n; j++)
      buf[(size_t)i * n + j] = m.bf(i, j).get_d();
  wr(f, buf.data(), buf.size());
  buf.assign((size_t)d * d, 0.0);
  for (int i = 0; i < d; i++)
    for (int j = 0; j < d; j++)
      buf[(size_t)i * d + j] = m.gf(i, j).get_d();
  wr(f, buf.data(), buf.size());
  for (int i = 0; i < d; i++)
    for (int j = 0; j < d; j++)
      buf[(size_t)i * d + j] = m.mu(i, j).get_d();
  wr(f, buf.data(), buf.size());
  for (int i = 0; i < d; i++)
    for (int j = 0; j < d; j++)
      buf[(size_t)i * d + j] = m.r(i, j).get_d();
  wr(f, buf.data(), buf.size());
  fclose(f);
}

static void dump_b_long(const char *path)
{
  FILE *f = fopen(path, "ab");
  int d = Bl.get_rows(), n = Bl.get_cols();
  vector<int64_t> buf((size_t)d * n);
  for (int i = 0; i < d; i++)
    for (int j = 0; j < n; j++)
      buf[(size_t)i * n + j] = Bl(i, j).get_si();
  wr(f, buf.data(), buf.size());
  fclose(f);
}

template <class G> static void time_update_row(G &m, int i, int reps, int invalidate)
{
  /* times what LLL's babai() pays per iteration on row i: row_op_end(i,i+1) [update_bf + invalidation]
     followed by update_gso_row(i, i)  (gso_interface.cpp:32-53,131-164).  invalidate=0 keeps gf valid (g=0) */
  m.update_gso();
  double t0 = now();
  for (int rep = 0; rep < reps; rep++)
  {
    if (invalidate)
    {
      m.row_op_begin(i, i + 1);
      m.row_op_end(i, i + 1);
    }
    else
      m.invalidate_gso_row(i, 0);
    m.update_gso_row(i, i);
  }
  double t1 = now();
  printf("time_update_row i=%d reps=%d invalidate=%d sec=%.9f per_call_us=%.4f\n", i, reps, invalidate,
         t1 - t0, (t1 - t0) / reps * 1e6);
}

/* Multi-threaded CPU baseline: T threads, each owning `per` private copies of the current long basis, run
 * `reps` x { row_op_end(i,i+1); update_gso_row(i,i) } on every copy (distinct objects may run concurrently,
 * README.md:310).  Prints the aggregate wall time. */
static void time_update_row_mt(int i, int reps, int threads, int per)
{
  vector<thread> th;
  vector<double> secs(threads);
  double t0 = now();
  for (int t = 0; t < threads; t++)
    th.emplace_back([&, t]() {
      vector<ZZ_mat<long>> bs(per, Bl);
      ZZ_mat<long> eu, eut;
      vector<unique_ptr<GsoL>> gs;
      for (int p = 0; p < per; p++)
      {
        gs.emplace_back(new GsoL(bs[p], eu, eut, gflags));
        gs.back()->update_gso();
      }
      double a = now();
      for (int rep = 0; rep < reps; rep++)
        for (int p = 0; p < per; p++)
        {
          gs[p]->row_op_begin(i, i + 1);
          gs[p]->row_op_end(i, i + 1);
          gs[p]->update_gso_row(i, i);
        }
      secs[t] = now() - a;
    });
  for (auto &x : th)
    x.join();
  double t1 = now(), mx = 0;
  for (double s : secs)
    mx = max(mx, s);
  printf("time_update_row_mt i=%d reps=%d threads=%d per=%d calls=%ld timed_sec=%.9f wall_sec=%.6f\n", i, reps,
         threads, per, (long)reps * threads * per, mx, t1 - t0);
}

static void time_update_gso_mt(int reps, int threads, int per)
{
  vector<thread> th;
  vector<double> secs(threads);
  for (int t = 0; t < threads; t++)
    th.emplace_back([&, t]() {
      vector<ZZ_mat<long>> bs(per, Bl);
      ZZ_mat<long> eu, eut;
      vector<unique_ptr<GsoL>> gs;
      for (int p = 0; p < per; p++)
        gs.emplace_back(new GsoL(bs[p], eu, eut, gflags));
      double a = now();
      for (int rep = 0; rep < reps; rep++)
        for (int p = 0; p < per; p++)
        {
          gs[p]->row_op_begin(0, gs[p]->d);
          gs[p]->row_op_end(0, gs[p]->d);
          gs[p]->update_gso();
        }
      secs[t] = now() - a;
    });
  for (auto &x : th)
    x.join();
  double mx = 0;
  for (double s : secs)
    mx = max(mx, s);
  printf("time_update_gso_mt reps=%d threads=%d per=%d calls=%ld timed_sec=%.9f\n", reps, threads, per,
         (long)reps * threads * per, mx);
}

/* ---- enumeration probes -------------------------------------------------------------------------------
 * enum FIRST LAST FACTOR PRUNEFILE OUT MODE : Enumeration<Z_NR<long>,FP_NR<double>>::enumerate on block
 *   [FIRST,LAST) of the current long GSO with max_dist = FACTOR * r(FIRST,FIRST), pruning coefficients read from
 *   PRUNEFILE ("-" = none).  MODE = internal (EnumerationDyn, enumerate.cpp:58) | enumlib (the bundled parallel
 *   enumerator through the extenum hook) | capture (a hook that records exactly what the plugin API hands an
 *   external enumerator — enumerate_ext.cpp:48-148 — and declines, so the internal enumerator then runs).
 *   A suffix of the mode adds the other two cases of the hook: internal_dual (dual SVP of the block as svp_reduction
 *   asks for it, bkz.cpp:277-318: max_dist = FACTOR / r(LAST-1,LAST-1)), internal_subsols, internal_dual_subsols
 *   (evaluator with find_subsolutions; the record then ends with f64 subdist[d] (-1 = none), f64 subsol[d*d]).
 * OUT (binary, appended): int32 magic 0x454e554d, d, found, mode; f64 maxdist_norm (capture mode: as handed to the
 *   hook, else -1), f64 best_dist (evaluator's, denormalised), int64 normexp; f64 sol[d]; u64 nodes[d];
 *   capture mode only: f64 mut[d*d] (transposed layout of enumerate_ext.cpp:108-121), f64 rdiag[d], f64 pruning[d]
 */
struct EnumCapture
{
  int d         = 0;
  double maxdist = -1;
  vector<double> mut, rdiag, pruning;
};
static EnumCapture g_cap;

static std::array<uint64_t, FPLLL_EXTENUM_MAX_EXTENUM_DIM>
capture_enumerator(const int dim, fplll_extenum_enumf maxdist, std::function<extenum_cb_set_config> cbfunc,
                   std::function<extenum_cb_process_sol>, std::function<extenum_cb_process_subsol>, bool, bool)
{
  g_cap.d       = dim;
  g_cap.maxdist = maxdist;
  g_cap.mut.assign((size_t)dim * dim, 0.0);
  g_cap.rdiag.assign(dim, 0.0);
  g_cap.pruning.assign(dim, 0.0);
  cbfunc(g_cap.mut.data(), dim, true, g_cap.rdiag.data(), g_cap.pruning.data());
  std::array<uint64_t, FPLLL_EXTENUM_MAX_EXTENUM_DIM> ret{};
  ret[0] = ~uint64_t(0);  // "unsupported": fplll falls back to its own enumerator (enumerate_ext.cpp:88)
  return ret;
}

static void run_enum(GsoL &m, int first, int last, double factor, const string &prunefile, const string &out,
                     const string &mode)
{
  static std::function<extenum_fc_enumerate> bundled = get_external_enumerator();
  int d = last - first;
  vector<double> pr;
  if (prunefile != "-")
  {
    ifstream f(prunefile);
    double x;
    while (f >> x)
      pr.push_back(x);
    if ((int)pr.size() != d)
    {
      fprintf(stderr, "pruning file has %d entries, need %d\n", (int)pr.size(), d);
      exit(2);
    }
  }
  int imode = 0;
  const bool dual = mode.find("dual") != string::npos, subsols = mode.find("subsols") != string::npos;
  if (mode.rfind("internal", 0) == 0)
    set_external_enumerator(nullptr);
  else if (mode == "enumlib")
  {
    set_external_enumerator(bundled);
    imode = 1;
  }
  else
  {
    set_external_enumerator(capture_enumerator);
    imode   = 2;
    g_cap   = EnumCapture();
  }
  FastEvaluator<FP_NR<double>> ev(1, EVALSTRATEGY_BEST_N_SOLUTIONS, subsols);
  Enumeration<Z_NR<long>, FP_NR<double>> en(m, ev);
  long expo;
  FP_NR<double> maxd = m.get_r_exp(dual ? last - 1 : first, dual ? last - 1 : first, expo);
  if (dual)
  {
    maxd.pow_si(maxd, -1, GMP_RNDU);  // bkz.cpp:312-316
    expo *= -1;
  }
  maxd.mul(maxd, factor);
  double t0 = now();
  en.enumerate(first, last, maxd, expo, vector<FP_NR<double>>(), vector<enumxt>(), pr, dual);
  double sec = now() - t0;
  set_external_enumerator(bundled);
  FILE *f        = fopen(out.c_str(), "ab");
  int found      = ev.empty() ? 0 : 1;
  int32_t hdr[4] = {0x454e554d, d, found, imode | (dual ? 16 : 0) | (subsols ? 32 : 0)};
  wr(f, hdr, 4);
  double md = imode == 2 ? g_cap.maxdist : -1.0;
  if (dual)
  {
    // The hook's own normalisation of a DUAL radius (enumerate_ext.cpp:72: mul_2si(fmaxdist, _normexp - fmaxdistexpo))
    // differs from EnumerationDyn's (enumerate.cpp:92-98: normexp negated, fmaxdistexpo - normexp) by 2^(2 * expo of
    // r(last-1)) whenever GSO_ROW_EXPO is on, so what the capture hook saw is not the radius the reference's own dual
    // enumeration (whose nodes / solution this record holds) ran with.  Record the latter, restated:
    long rexpo, normexp = -1;
    for (int i = 0; i < d; ++i)
    {
      FP_NR<double> fr = m.get_r_exp(i + first, i + first, rexpo);
      normexp          = std::max(normexp, rexpo + fr.exponent());
    }
    normexp *= -1;
    long e2;
    FP_NR<double> md2 = m.get_r_exp(last - 1, last - 1, e2);
    md2.pow_si(md2, -1, GMP_RNDU);
    e2 *= -1;
    md2.mul(md2, factor);
    FP_NR<double> nrm;
    nrm.mul_2si(md2, e2 - normexp);
    md = nrm.get_d(GMP_RNDU);
  }
  wr(f, &md, 1);
  double best = found ? ev.begin()->first.get_d() : -1.0;
  wr(f, &best, 1);
  int64_t ne = ev.normExp;
  wr(f, &ne, 1);
  vector<double> sol(d, 0.0);
  if (found)
    for (int i = 0; i < d; i++)
      sol[i] = ev.begin()->second[i].get_d();
  wr(f, sol.data(), d);
  vector<uint64_t> nodes(d);
  uint64_t tot = 0;
  for (int i = 0; i < d; i++)
  {
    nodes[i] = en.get_nodes(i);
    tot += nodes[i];
  }
  wr(f, nodes.data(), d);
  if (imode == 2)
  {
    wr(f, g_cap.mut.data(), g_cap.mut.size());
    wr(f, g_cap.rdiag.data(), d);
    wr(f, g_cap.pruning.data(), d);
  }
  if (subsols)
  {
    vector<double> sd(d, -1.0), ss((size_t)d * d, 0.0);
    for (size_t k = 0; k < ev.sub_solutions.size() && (int)k < d; k++)
      if (!ev.sub_solutions[k].second.empty())
      {
        sd[k] = ev.sub_solutions[k].first.get_d();
        for (int i = 0; i < d; i++)
          ss[k * d + i] = ev.sub_solutions[k].second[i].get_d();
      }
    wr(f, sd.data(), d);
    wr(f, ss.data(), ss.size());
  }
  fclose(f);
  printf("enum d=%d mode=%s found=%d best=%.17g nodes=%llu sec=%.6f\n", d, mode.c_str(), found, best,
         (unsigned long long)tot, sec);
}

/* ---- Householder probes: MatHouseholder<Z_NR<long>, FP_NR<double>> over the current long matrix --------------
 * hh FLAGS | hh_refresh_R_bf I | hh_refresh_R I | hh_update_R I LASTJ | hh_update_R_last I | hh_size_reduce K END START
 * | hh_swap I J | hh_recover_R I | hh_set_updated_R_false | hh_dump FILE
 * dump (appended): int32 magic 0x48483030, d, n, n_known_rows, n_known_cols, updated_R; int64 row_expo[d];
 *   f64 sigma[d]; f64 norm_square_b[d]; int64 expo_norm_square_b[d]; f64 bf[d*n]; f64 R[d*n]; f64 V[d*n]; int64 b[d*n]
 */
typedef MatHouseholder<Z_NR<long>, FP_NR<double>> HhL;
static unique_ptr<HhL> hh;
static void hh_dump(const char *path)
{
  FILE *f = fopen(path, "ab");
  int d = hh->d, n = hh->n;
  int32_t hdr[6] = {0x48483030, d, n, hh->n_known_rows, hh->n_known_cols, (int)hh->updated_R};
  wr(f, hdr, 6);
  vector<int64_t> re(d), en(d);
  vector<double> sg(d), nb(d);
  for (int i = 0; i < d; i++)
  {
    re[i] = hh->row_expo[i];
    sg[i] = hh->sigma[i].get_d();
    nb[i] = hh->norm_square_b[i].get_d();
    en[i] = hh->expo_norm_square_b[i];
  }
  wr(f, re.data(), d), wr(f, sg.data(), d), wr(f, nb.data(), d), wr(f, en.data(), d);
  vector<double> buf((size_t)d * n);
  for (int i = 0; i < d; i++)
    for (int j = 0; j < n; j++)
      buf[(size_t)i * n + j] = hh->bf(i, j).get_d();
  wr(f, buf.data(), buf.size());
  for (int i = 0; i < d; i++)
    for (int j = 0; j < n; j++)
      buf[(size_t)i * n + j] = hh->R(i, j).get_d();
  wr(f, buf.data(), buf.size());
  for (int i = 0; i < d; i++)
    for (int j = 0; j < n; j++)
      buf[(size_t)i * n + j] = hh->V(i, j).get_d();
  wr(f, buf.data(), buf.size());
  fclose(f);
  dump_b_long(path);
}

int main(int argc, char **argv)
{
  string line;
  while (getline(cin, line))
  {
    istringstream is(line);
    string c;
    if (!(is >> c) || c[0] == '#')
      continue;
    if (c == "help")
    {
      puts("load P | save P | tolong | gso l|m FLAGS | update_gso | update_row I J | discover_all | "
           "row_addmul_we I J X E | row_op_begin F L | row_op_end F L | move_row O N | row_swap I J | "
           "set_r I J V | dump P | dumpb P | lll DELTA ETA METHOD FLOAT FLAGS | lll_range DELTA ETA KMIN KSTART KEND SRSTART | "
           "size_reduction ETA KMIN KEND SRSTART | islll DELTA ETA | "
           "bkz BLOCK FLAGS MAXLOOPS default|none internal|enumlib THREADS | enum FIRST LAST FACTOR PRUNEFILE OUT internal|enumlib|capture | set_threads T | time_update_row I REPS INV | time_update_row_mt I REPS T PER | time_update_gso_mt REPS T PER");
    }
    else if (c == "load")
    {
      string p;
      is >> p;
      ifstream f(p);
      if (!f)
      {
        fprintf(stderr, "cannot open %s\n", p.c_str());
        return 2;
      }
      f >> Bm;
      gl.reset();
      gm.reset();
      printf("load %d %d\n", Bm.get_rows(), Bm.get_cols());
    }
    else if (c == "save")
    {
      string p;
      is >> p;
      ofstream f(p);
      if (gl)
        f << Bl << endl;
      else
        f << Bm << endl;
    }
    else if (c == "save_long")
    {
      string p;
      is >> p;
      ofstream f(p);
      f << Bl << endl;
    }
    else if (c == "tolong")
    {
      int d = Bm.get_rows(), n = Bm.get_cols();
      Bl.resize(d, n);
      for (int i = 0; i < d; i++)
        for (int j = 0; j < n; j++)
          Bl(i, j) = Bm(i, j).get_si();
      printf("tolong ok\n");
    }
    else if (c == "gso")
    {
      string t;
      is >> t >> gflags;
      if (t == "l")
      {
        gm.reset();
        gl.reset(new GsoL(Bl, Ul, UTl, gflags));
      }
      else
      {
        gl.reset();
        gm.reset(new GsoM(Bm, Um, UTm, gflags));
      }
    }
    else if (c == "update_gso")
    {
      bool ok = gl ? gl->update_gso() : gm->update_gso();
      printf("update_gso %d\n", (int)ok);
    }
    else if (c == "discover_all")
    {
      if (gl)
        gl->discover_all_rows();
      else
        gm->discover_all_rows();
    }
    else if (c == "update_row")
    {
      int i, j;
      is >> i >> j;
      bool ok = gl ? gl->update_gso_row(i, j) : gm->update_gso_row(i, j);
      printf("update_row %d %d %d\n", i, j, (int)ok);
    }
    else if (c == "row_addmul_we")
    {
      int i, j;
      double x;
      long e;
      is >> i >> j >> x >> e;
      FP_NR<double> fx = x;
      if (gl)
        gl->row_addmul_we(i, j, fx, e);
      else
        gm->row_addmul_we(i, j, fx, e);
    }
    else if (c == "row_op_begin")
    {
      int a, b;
      is >> a >> b;
      if (gl)
        gl->row_op_begin(a, b);
      else
        gm->row_op_begin(a, b);
    }
    else if (c == "row_op_end")
    {
      int a, b;
      is >> a >> b;
      if (gl)
        gl->row_op_end(a, b);
      else
        gm->row_op_end(a, b);
    }
    else if (c == "move_row")
    {
      int a, b;
      is >> a >> b;
      if (gl)
        gl->move_row(a, b);
      else
        gm->move_row(a, b);
    }
    else if (c == "row_swap")
    {
      int a, b;
      is >> a >> b;
      if (gl)
        gl->row_swap(a, b);
      else
        gm->row_swap(a, b);
    }
    else if (c == "set_r")
    {
      int i, j;
      double v;
      is >> i >> j >> v;
      FP_NR<double> f = v;
      if (gl)
        gl->set_r(i, j, f);
      else
        gm->set_r(i, j, f);
    }
    else if (c == "dump")
    {
      string p;
      is >> p;
      if (gl)
      {
        dump_state(*gl, p.c_str(), 0);
        dump_b_long(p.c_str());
      }
      else
        dump_state(*gm, p.c_str(), 1);
    }
    else if (c == "lll")
    {
      /* lll DELTA ETA METHOD(wrapper|proved|heuristic|fast) FLOAT(default|double|...) FLAGS ; on the mpz matrix */
      double delta, eta;
      string ms, fs;
      int fl;
      is >> delta >> eta >> ms >> fs >> fl;
      LLLMethod me = ms == "wrapper" ? LM_WRAPPER : ms == "proved" ? LM_PROVED : ms == "fast" ? LM_FAST : LM_HEURISTIC;
      FloatType ft = fs == "double" ? FT_DOUBLE : fs == "mpfr" ? FT_MPFR : fs == "ld" ? FT_LONG_DOUBLE : FT_DEFAULT;
      double t0 = now();
      int st    = lll_reduction(Bm, delta, eta, me, ft, 0, fl);
      printf("lll status=%d sec=%.6f\n", st, now() - t0);
    }
    else if (c == "lll_long")
    {
      /* LLL on the long matrix through the same code path bkz.cpp:826-836 uses: MatGSO<long,double>, GSO_ROW_EXPO */
      double delta, eta;
      is >> delta >> eta;
      ZZ_mat<long> eu, eut;
      GsoL m(Bl, eu, eut, GSO_ROW_EXPO);
      LLLReduction<Z_NR<long>, FP_NR<double>> lll(m, delta, eta, LLL_DEFAULT);
      double t0 = now();
      lll.lll();
      printf("lll_long status=%d sec=%.6f swaps=%d\n", lll.status, now() - t0, lll.n_swaps);
    }
    else if (c == "lll_range" || c == "size_reduction")
    {
      /* lll_range DELTA ETA KMIN KSTART KEND SRSTART | size_reduction ETA KMIN KEND SRSTART : a fresh
         LLLReduction<Z_NR<long>, FP_NR<double>> (LLL_DEFAULT) on the current long GSO object, so that its status starts
         at RED_SUCCESS (lll.cpp:28-29); prints the return value, status, swaps, final_kappa and zeros */
      double delta = 0.99, eta;
      int kmin, kstart = 0, kend, srs;
      if (c == "lll_range")
        is >> delta >> eta >> kmin >> kstart >> kend >> srs;
      else
        is >> eta >> kmin >> kend >> srs;
      if (!gl)
      {
        fprintf(stderr, "%s needs a long GSO\n", c.c_str());
        return 2;
      }
      LLLReduction<Z_NR<long>, FP_NR<double>> red(*gl, delta, eta, LLL_DEFAULT);
      bool ok = c == "lll_range" ? red.lll(kmin, kstart, kend, srs) : red.size_reduction(kmin, kend, srs);
      printf("%s ok=%d status=%d swaps=%d final_kappa=%d zeros=%d\n", c.c_str(), (int)ok, red.status, red.n_swaps,
             red.final_kappa, red.zeros);
    }
    else if (c == "islll")
    {
      double delta, eta;
      is >> delta >> eta;
      ZZ_mat<mpz_t> B2;
      if (Bl.get_rows() > 0 && gl)
      {
        B2.resize(Bl.get_rows(), Bl.get_cols());
        for (int i = 0; i < Bl.get_rows(); i++)
          for (int j = 0; j < Bl.get_cols(); j++)
            B2(i, j) = Bl(i, j).get_si();
      }
      else
        B2 = Bm;
      int old = FP_NR<mpfr_t>::set_prec(512);
      ZZ_mat<mpz_t> eu, eut;
      MatGSO<Z_NR<mpz_t>, FP_NR<mpfr_t>> M(B2, eu, eut, GSO_INT_GRAM);
      int ok = is_lll_reduced<Z_NR<mpz_t>, FP_NR<mpfr_t>>(M, delta, eta);
      FP_NR<mpfr_t>::set_prec(old);
      printf("islll %d\n", ok);
    }
    else if (c == "enum")
    {
      int first, last;
      double factor;
      string pf, out, mode;
      is >> first >> last >> factor >> pf >> out >> mode;
      if (!gl)
      {
        fprintf(stderr, "enum needs a long GSO\n");
        return 2;
      }
      run_enum(*gl, first, last, factor, pf, out, mode);
    }
    else if (c == "set_threads")
    {
      int t;
      is >> t;
      printf("set_threads %d\n", set_threads(t));
    }
    else if (c == "bkz")
    {
      /* bkz BLOCK FLAGS MAXLOOPS STRATEGIES(default|none) ENUM(internal|enumlib) THREADS : bkz_reduction(&Bm, NULL, param,
         FT_DOUBLE) — bkz.cpp:849-927 — on the mpz matrix (converted to long inside when entries fit, bkz.cpp:826) */
      int bs, fl, ml, th;
      string strat, em;
      is >> bs >> fl >> ml >> strat >> em >> th;
      static std::function<extenum_fc_enumerate> bundled = get_external_enumerator();
      set_external_enumerator(em == "internal" ? std::function<extenum_fc_enumerate>(nullptr) : bundled);
      set_threads(th);
      vector<Strategy> strategies;
      if (strat == "default")
        strategies = load_strategies_json(strategy_full_path("default.json"));
      BKZParam param(bs, strategies);
      param.flags     = fl;
      param.max_loops = ml;
      double t0       = now();
      int st          = -100;
      try
      {
        st = bkz_reduction(&Bm, NULL, param, FT_DOUBLE, 0);
      }
      catch (std::exception &e)
      {
        printf("bkz exception %s\n", e.what());
      }
      set_external_enumerator(bundled);
      printf("bkz status=%d sec=%.6f\n", st, now() - t0);
    }
    else if (c == "hh")
    {
      int fl;
      is >> fl;
      hh.reset(new HhL(Bl, Ul, UTl, fl));
    }
    else if (c == "hh_refresh_R_bf") { int i; is >> i; hh->refresh_R_bf(i); }
    else if (c == "hh_refresh_R") { int i; is >> i; hh->refresh_R(i); }
    else if (c == "hh_update_R") { int i, l; is >> i >> l; hh->update_R(i, l != 0); }
    else if (c == "hh_update_R_last") { int i; is >> i; hh->update_R_last(i); }
    else if (c == "hh_size_reduce") { int k, e, st; is >> k >> e >> st; printf("hh_size_reduce %d\n", (int)hh->size_reduce(k, e, st)); }
    else if (c == "hh_swap") { int i, j; is >> i >> j; hh->swap(i, j); }
    else if (c == "hh_recover_R") { int i; is >> i; hh->recover_R(i); }
    else if (c == "hh_set_updated_R_false") { hh->set_updated_R_false(); }
    else if (c == "hh_dump") { string p; is >> p; hh_dump(p.c_str()); }
    else if (c == "hlll_long")
    {
      /* hlll_reduction on the long matrix: HLLLReduction<Z_NR<long>,FP_NR<double>> with ROW_EXPO|OP_FORCE_LONG
         (wrapper.cpp:789-806 for the mpz type) */
      double delta, eta, theta, cc;
      is >> delta >> eta >> theta >> cc;
      HhL m(Bl, Ul, UTl, HOUSEHOLDER_ROW_EXPO | HOUSEHOLDER_OP_FORCE_LONG);
      HLLLReduction<Z_NR<long>, FP_NR<double>> red(m, delta, eta, theta, cc, LLL_DEFAULT);
      double t0 = now();
      red.hlll();
      printf("hlll_long status=%d sec=%.6f\n", red.get_status(), now() - t0);
    }
    else if (c == "seed")
    {
      unsigned long sd;
      is >> sd;
      RandGen::init_with_seed(sd);
    }
    else if (c == "time_update_row")
    {
      int i, reps, inv;
      is >> i >> reps >> inv;
      if (gl)
        time_update_row(*gl, i, reps, inv);
      else
        time_update_row(*gm, i, reps, inv);
    }
    else if (c == "time_update_row_mt")
    {
      int i, reps, t, per;
      is >> i >> reps >> t >> per;
      time_update_row_mt(i, reps, t, per);
    }
    else if (c == "time_update_gso_mt")
    {
      int reps, t, per;
      is >> reps >> t >> per;
      time_update_gso_mt(reps, t, per);
    }
    else
    {
      fprintf(stderr, "unknown command: %s\n", c.c_str());
      return 2;
    }
    fflush(stdout);
  }
  return 0;
}
