// fplll_matgso_shim.cpp — the reference-side binding of the device GSO: every
//     fplll::MatGSO<Z_NR<long>,  FP_NR<double>>   (BKZ regime, bkz.cpp:812-836; wrapper small-entry stage)  and
//     fplll::MatGSO<Z_NR<mpz_t>, FP_NR<double>>   (LLL stage 1, wrapper.cpp:538-553; the basis stays in GMP on the host)
// object of a process runs its update_gso_row on the GPU, with the UNMODIFIED libfplll and unmodified callers
// (lll.cpp, bkz.cpp, enumerate.cpp, hlll excluded, user code).
//
// How: fplll has no FFI for the GSO — callers hold MatGSOInterface<ZT,FT>& and read mu / r through inline accessors
// (gso_interface.h:674-746).  The heavy member functions, however, are ordinary out-of-line template instantiations with
// WEAK dynamic symbols in libfplll.so (gso_interface.cpp:313-360, gso.cpp:511-529), so a library that is linked (or
// LD_PRELOADed) before libfplll and defines them as explicit specialisations — strong symbols — takes their place for
// every caller, inside and outside libfplll.  This file specialises exactly four of them per type:
//     update_gso_row(i, last_j)   gso_interface.cpp:131-164   -> b200gso_update_gso_row, row i of mu / r mirrored back
//     row_op_end(first, last)     gso_interface.cpp:32-53     -> the rows rewritten on the host travel to the device
//     move_row(old_r, new_r)      gso.cpp:289-366             -> b200gso_move_row
//     size_increased()            gso.cpp:368-403             -> (called by the constructor, gso.h:113-130) marks a new object
// and calls the reference's own implementations (dlsym RTLD_NEXT) for the host-side bookkeeping, so row_expo, bf, the
// validity state machine, the integer basis and the transforms u / u_inv stay exactly what the reference computes —
// only the O(d^2) floating-point work of update_gso_row leaves the host.  The host's integer basis is authoritative:
// the reference's contract (gso_interface.h:172-178) is that every modification of b happens between row_op_begin and
// row_op_end, so the touched rows are shipped at row_op_end — int64 rows for Z_NR<long> (b200gso_upload_row), the
// freshly converted floating-point rows + exponents for Z_NR<mpz_t> (b200gso_upload_row_fp; update_bf itself,
// mpz_get_d_2exp, stays on the host next to GMP).
// An object is adopted the first time one of the first three functions sees it (constructors are inline in gso.h, but
// they call size_increased(), which is how a new object at a recycled address is told from the old one); objects
// the device cannot hold (MatGSOGram, d > 512) keep the reference's path untouched.  GSO_INT_GRAM objects (exact integer
// Gram matrix, gso.cpp:140-159) are adopted too: b and g stay on the host, update_gso_row ships row i of g converted as
// get_gram does (b200gso_set_gram_row) and the device does the forward substitution.  There is no CPU
// fallback for an adopted object: a CUDA failure throws.
//
// On top of that, BKZReduction<Z_NR<long>, FP_NR<double>>::bkz() (bkz.cpp:522-672) — what bkz_reduction() / `fplll -a bkz`
// run after their wrapper-LLL when the basis fits long (bkz.cpp:812-836) — is taken over whole by the device driver
// (b200bkz_reduce: device-resident LLL loops, device enumeration, no per-call forwarding) whenever the request is one
// that driver implements (plain BKZ, no transformation matrices, no GSO dump); SD-BKZ / slide reduction keep the
// reference's control flow over the forwarded GSO.  B200_SHIM_BKZ=0 turns the take-over off.
//
// Build (where fplll's headers are installed):  g++ -shared -fPIC fplll_matgso_shim.cpp -lb200bkz -ldl  -> libb200fplll.so
// Use:  LD_PRELOAD=libb200fplll.so fplll -a bkz -b 40 ...   or link it before -lfplll.   B200_SHIM_STATS=1 prints the
// forwarded-call counters at exit; B200_SHIM_DISABLE=1 turns the forwarding off.
#include <fplll/fplll.h>

#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200bkz.h"
#include "../../include/b200gso.h"

extern "C" long b200_matgso_shim_bkz_taken(void);

namespace b200shim {

struct Entry
{
  b200gso_t *h = nullptr;  // null: declined (the reference's path)
  int d = 0, n = 0;
  bool host_basis = false;
  bool int_gram   = false;     // GSO_INT_GRAM object: the exact Gram matrix stays on the host, its rows travel as doubles
  int dev_nkr = 0;             // rows the device has discovered
  std::vector<int> dev_valid;  // the device's gso_valid_cols as of the last call (detects the inlined set_r)
  std::vector<double> row_mu, row_r;
  std::vector<int64_t> irow;
  std::vector<double> frow, frow_g;
};

static std::mutex g_mu;
static std::unordered_map<const void *, Entry> g_tab;
static long g_adopted = 0, g_declined = 0, g_updates = 0, g_uploads = 0, g_moves = 0, g_setr = 0;

static bool enabled()
{
  static const bool on = !getenv("B200_SHIM_DISABLE");
  return on;
}

static void ck(int rc, const char *what)
{
  if (rc != 0)
    throw std::runtime_error(std::string("b200 MatGSO shim: ") + what + ": " + b200gso_last_error());
}

struct AtExit
{
  ~AtExit()
  {
    if (getenv("B200_SHIM_STATS"))
      fprintf(stderr, "b200 MatGSO shim: adopted %ld objects (declined %ld), update_gso_row forwarded %ld, rows uploaded %ld, "
                      "move_row %ld, set_r %ld, bkz() on the device driver %ld\n",
              g_adopted, g_declined, g_updates, g_uploads, g_moves, g_setr, b200_matgso_shim_bkz_taken());
    for (auto &kv : g_tab)
      if (kv.second.h)
        b200gso_destroy(kv.second.h);
  }
} g_at_exit;

template <class F> static F next_symbol(const char *name)
{
  void *p = dlsym(RTLD_NEXT, name);
  if (!p)
    throw std::runtime_error(std::string("b200 MatGSO shim: libfplll does not export ") + name);
  return reinterpret_cast<F>(p);
}

}  // namespace b200shim

FPLLL_BEGIN_NAMESPACE

// ---- what differs between the two integer types -------------------------------------------------------------------
template <class ZT> struct B200ShimTraits;
template <> struct B200ShimTraits<Z_NR<long>>
{
  static constexpr bool host_basis = false;
  static const char *sym_update() { return "_ZN5fplll15MatGSOInterfaceINS_4Z_NRIlEENS_5FP_NRIdEEE14update_gso_rowEii"; }
  static const char *sym_row_op_end() { return "_ZN5fplll15MatGSOInterfaceINS_4Z_NRIlEENS_5FP_NRIdEEE10row_op_endEii"; }
  static const char *sym_move_row() { return "_ZN5fplll6MatGSOINS_4Z_NRIlEENS_5FP_NRIdEEE8move_rowEii"; }
  static const char *sym_size_increased() { return "_ZN5fplll6MatGSOINS_4Z_NRIlEENS_5FP_NRIdEEE14size_increasedEv"; }
};
template <> struct B200ShimTraits<Z_NR<mpz_t>>
{
  static constexpr bool host_basis = true;
  static const char *sym_update()
  {
    return "_ZN5fplll15MatGSOInterfaceINS_4Z_NRIA1_12__mpz_structEENS_5FP_NRIdEEE14update_gso_rowEii";
  }
  static const char *sym_row_op_end()
  {
    return "_ZN5fplll15MatGSOInterfaceINS_4Z_NRIA1_12__mpz_structEENS_5FP_NRIdEEE10row_op_endEii";
  }
  static const char *sym_move_row() { return "_ZN5fplll6MatGSOINS_4Z_NRIA1_12__mpz_structEENS_5FP_NRIdEEE8move_rowEii"; }
  static const char *sym_size_increased()
  {
    return "_ZN5fplll6MatGSOINS_4Z_NRIA1_12__mpz_structEENS_5FP_NRIdEEE14size_increasedEv";
  }
};

namespace {

using b200shim::Entry;

// The specialisations below are MEMBER functions, so they see the protected state of the object they run on; they hand
// the helpers references to what those need.
template <class ZT> struct Guts
{
  MatGSOInterface<ZT, FP_NR<double>> *self;
  Matrix<FP_NR<double>> &mu, &r, &bf;
  std::vector<int> &valid;
  std::vector<long> &row_expo;
  int &nkr;
  int d;
  bool int_gram, row_expo_en;
};

// ship row i as the host has it: the integer row (long) or the converted floating-point row and its exponent (mpz)
inline void shim_upload_row(Entry &e, int i, MatGSO<Z_NR<long>, FP_NR<double>> &m, Guts<Z_NR<long>> &)
{
  for (int c = 0; c < e.n; c++)
    e.irow[c] = m.b(i, c).get_si();
  b200shim::ck(b200gso_upload_row(e.h, i, e.irow.data()), "upload_row");
  b200shim::g_uploads++;
}
inline void shim_upload_row(Entry &e, int i, MatGSO<Z_NR<mpz_t>, FP_NR<double>> &, Guts<Z_NR<mpz_t>> &g)
{
  for (int c = 0; c < e.n; c++)
    e.frow[c] = c < g.bf.get_cols() ? g.bf(i, c).get_d() : 0.0;
  long ex = g.row_expo_en ? g.row_expo[i] : 0;
  b200shim::ck(b200gso_upload_row_fp(e.h, i, e.frow.data(), &ex), "upload_row_fp");
  b200shim::g_uploads++;
}

// adoption: the whole basis.  long: b200gso_set_basis = size_increased() on the device (init_row_size, bf, metadata);
// mpz: the floating-point rows size_increased() converted on the host, one by one.
inline void shim_initial_basis(Entry &e, MatGSO<Z_NR<long>, FP_NR<double>> &m, Guts<Z_NR<long>> &)
{
  std::vector<int64_t> flat((size_t)e.d * e.n);
  for (int i = 0; i < e.d; i++)
    for (int c = 0; c < e.n; c++)
      flat[(size_t)i * e.n + c] = m.b(i, c).get_si();
  b200shim::ck(b200gso_set_basis(e.h, flat.data()), "set_basis");
  b200shim::g_uploads += e.d;
}
inline void shim_initial_basis(Entry &e, MatGSO<Z_NR<mpz_t>, FP_NR<double>> &m, Guts<Z_NR<mpz_t>> &g)
{
  for (int i = 0; i < e.d; i++)
    shim_upload_row(e, i, m, g);
}

template <class ZT> Entry *shim_entry(Guts<ZT> &g)
{
  if (!b200shim::enabled())
    return nullptr;
  std::lock_guard<std::mutex> lock(b200shim::g_mu);
  auto it = b200shim::g_tab.find(g.self);
  if (it != b200shim::g_tab.end())
  {
    Entry &e = it->second;
    if (e.h == nullptr)
      return nullptr;  // declined earlier (a new object at this address announces itself through size_increased())
    // Destructors and copy constructors are inline: an object that died without a word may have been replaced by a copy
    // of another one.  The entry is trusted only while the host's validity vector is what the device's was after the
    // last call (or one ahead on the diagonal: the inlined set_r).
    bool same = e.d == g.d && e.dev_nkr <= g.d;
    for (int i = 0; same && i < g.nkr && i < e.d; i++)
      same = std::max(g.valid[i], 0) == e.dev_valid[i] || (g.valid[i] == i + 1 && e.dev_valid[i] == i) ||
             i >= e.dev_nkr;
    if (same)
      return &e;
    b200gso_destroy(e.h);
    b200shim::g_tab.erase(it);
  }
  Entry e;
  auto *m = dynamic_cast<MatGSO<ZT, FP_NR<double>> *>(g.self);
  bool ok = m != nullptr && g.d >= 1 && g.d <= 512 && b200gso_device_count() > 0;
  for (int i = 0; ok && i < g.nkr; i++)
    ok = g.valid[i] <= 0;  // adoption needs a GSO with nothing computed yet (true at the first update_gso_row / row_op_end)
  if (ok)
  {
    e.d = g.d, e.n = m->b.get_cols();
    // GSO_INT_GRAM (gso.cpp:140-159): b and the exact Gram matrix g stay on the host (row operations update g
    // incrementally there); the device needs neither b nor bf, only the rows of g as doubles (b200gso_set_gram_row)
    e.int_gram   = g.int_gram;
    e.host_basis = B200ShimTraits<ZT>::host_basis || e.int_gram;
    const int flags = (g.row_expo_en ? B200GSO_ROW_EXPO : 0) | (e.host_basis ? B200GSO_HOST_BASIS : 0);
    if (b200gso_create(&e.h, 1, e.d, e.n, flags, 0) != 0)
      ok = false, e.h = nullptr;
  }
  if (!ok)
  {
    b200shim::g_declined++;
    b200shim::g_tab[g.self] = Entry();
    return nullptr;
  }
  e.dev_valid.assign(e.d, 0);
  e.row_mu.resize(e.d), e.row_r.resize(e.d), e.irow.resize(e.n), e.frow.resize(e.n), e.frow_g.resize(e.d);
  if (!e.int_gram)
    shim_initial_basis(e, *m, g);  // the basis as the host has it now
  b200shim::g_adopted++;
  Entry &slot = b200shim::g_tab[g.self] = e;
  return &slot;
}

// update_gso_row(i, last_j), gso_interface.cpp:131-164: bookkeeping as the reference, arithmetic on the device
template <class ZT> bool shim_update_gso_row(Guts<ZT> &g, Entry &e, int i, int last_j)
{
  // rows the host discovered (update_gso_row's own discover_row, discover_all_rows, ...) become known on the device
  if (e.dev_nkr < g.nkr)
  {
    b200shim::ck(b200gso_discover_rows(e.h, g.nkr), "discover_rows");
    e.dev_nkr = g.nkr;
  }
  const int j0 = std::max(0, g.valid[i]);
  if (j0 > last_j)
    return true;
  // the inlined set_r (gso_interface.h:739-746; lll.cpp:137-142 stores the Lovasz value as r(k,k)) only reached the
  // host copy: rows whose host validity ran ahead of the device's get their diagonal pushed before anybody divides by it
  for (int j = 0; j <= std::min(i, last_j); j++)
    if (g.valid[j] == j + 1 && e.dev_valid[j] == j)
    {
      const double f = g.r(j, j).get_d();
      b200shim::ck(b200gso_set_r(e.h, j, j, &f), "set_r");
      e.dev_valid[j] = j + 1;
      b200shim::g_setr++;
    }
  if (e.int_gram)
  {
    // the Gram entries the update will read, exactly as the reference's get_gram converts them (gso.h:318-322)
    const int cnt = std::min(i, last_j) + 1;
    FP_NR<double> f;
    for (int j = 0; j < cnt; j++)
      e.frow_g[j] = g.self->get_gram(f, i, j).get_d();
    b200shim::ck(b200gso_set_gram_row(e.h, i, cnt, e.frow_g.data()), "set_gram_row");
  }
  int ok = 1;
  b200shim::ck(b200gso_update_gso_row(e.h, i, last_j, &ok), "update_gso_row");
  b200shim::g_updates++;
  if (!ok)
    return false;  // non-finite mu: like the reference, gso_valid_cols[i] stays (gso_interface.cpp:155-157)
  int v = 0;
  b200shim::ck(b200gso_get_mu_r_row(e.h, i, e.row_mu.data(), e.row_r.data(), &v), "get_mu_r_row");
  for (int j = j0; j <= last_j; j++)
  {
    g.r(i, j) = e.row_r[j];
    if (j < i)
      g.mu(i, j) = e.row_mu[j];
  }
  g.valid[i]     = last_j + 1;
  e.dev_valid[i] = v;
  return true;
}

}  // namespace

#define B200_SHIM_GUTS(ZT) Guts<ZT> g{this, mu, r, bf, gso_valid_cols, row_expo, n_known_rows, d, enable_int_gram, enable_row_expo}

#define B200_SHIM_FOR(ZT)                                                                                           \
  template <> bool MatGSOInterface<ZT, FP_NR<double>>::update_gso_row(int i, int last_j)                            \
  {                                                                                                                 \
    typedef bool (*fn_t)(MatGSOInterface<ZT, FP_NR<double>> *, int, int);                                           \
    static fn_t orig = b200shim::next_symbol<fn_t>(B200ShimTraits<ZT>::sym_update());                               \
    B200_SHIM_GUTS(ZT);                                                                                             \
    Entry *e = shim_entry<ZT>(g);                                                                                   \
    if (!e)                                                                                                         \
      return orig(this, i, last_j);                                                                                 \
    if (i >= n_known_rows)                                                                                          \
      discover_row(); /* the reference's own (host bookkeeping: n_known_rows, n_known_cols, Gram row) */            \
    return shim_update_gso_row<ZT>(g, *e, i, last_j);                                                               \
  }                                                                                                                 \
  template <> void MatGSOInterface<ZT, FP_NR<double>>::row_op_end(int first, int last)                              \
  {                                                                                                                 \
    typedef void (*fn_t)(MatGSOInterface<ZT, FP_NR<double>> *, int, int);                                           \
    static fn_t orig = b200shim::next_symbol<fn_t>(B200ShimTraits<ZT>::sym_row_op_end());                           \
    B200_SHIM_GUTS(ZT);                                                                                             \
    Entry *e = shim_entry<ZT>(g); /* before the host's invalidation: adoption looks at the validity */              \
    orig(this, first, last);       /* host: update_bf, Gram / GSO invalidation (gso_interface.cpp:32-53) */          \
    if (!e)                                                                                                         \
      return;                                                                                                       \
    auto *m = static_cast<MatGSO<ZT, FP_NR<double>> *>(this);                                                       \
    if (e->int_gram) /* nothing to ship (no bf): the device only invalidates; Gram rows travel with update_gso_row */    \
      b200shim::ck(b200gso_row_op_end(e->h, first, last), "row_op_end");                                            \
    for (int i = first; i < last; i++) /* row i + row_op_end(i, i+1) on the device; the union is row_op_end(first, last) */ \
    {                                                                                                               \
      if (!e->int_gram)                                                                                             \
        shim_upload_row(*e, i, *m, g);                                                                              \
      e->dev_valid[i] = 0;                                                                                          \
    }                                                                                                               \
    for (int i = last; i < d; i++)                                                                                  \
      e->dev_valid[i] = std::min(e->dev_valid[i], first);                                                           \
  }                                                                                                                 \
  template <> void MatGSO<ZT, FP_NR<double>>::move_row(int old_r, int new_r)                                        \
  {                                                                                                                 \
    typedef void (*fn_t)(MatGSO<ZT, FP_NR<double>> *, int, int);                                                    \
    static fn_t orig = b200shim::next_symbol<fn_t>(B200ShimTraits<ZT>::sym_move_row());                             \
    B200_SHIM_GUTS(ZT);                                                                                             \
    Entry *e = shim_entry<ZT>(g);                                                                                   \
    if (e && e->dev_nkr < n_known_rows)                                                                             \
    {                                                                                                               \
      b200shim::ck(b200gso_discover_rows(e->h, n_known_rows), "discover_rows");                                     \
      e->dev_nkr = n_known_rows;                                                                                    \
    }                                                                                                               \
    orig(this, old_r, new_r); /* host: b, u, bf, mu, r, gf, validity (gso.cpp:289-366) */                           \
    if (!e || old_r == new_r)                                                                                       \
      return;                                                                                                       \
    b200shim::ck(b200gso_move_row(e->h, old_r, new_r), "move_row");                                                 \
    b200shim::g_moves++;                                                                                            \
    e->dev_nkr = n_known_rows; /* a row moved past the known set leaves it on both sides (gso.cpp:352-364) */       \
    const int lo = std::min(old_r, new_r), hi = std::max(old_r, new_r);                                             \
    for (int i = lo; i < d; i++)                                                                                    \
      e->dev_valid[i] = std::min(e->dev_valid[i], lo);                                                              \
    (void)hi;                                                                                                       \
  }

static void shim_forget(const void *self)
{
  std::lock_guard<std::mutex> lock(b200shim::g_mu);
  auto it = b200shim::g_tab.find(self);
  if (it != b200shim::g_tab.end())
  {
    if (it->second.h)
      b200gso_destroy(it->second.h);
    b200shim::g_tab.erase(it);
  }
}

#define B200_SHIM_CTOR_FOR(ZT)                                                                                     \
  template <> void MatGSO<ZT, FP_NR<double>>::size_increased()                                                     \
  {                                                                                                                 \
    typedef void (*fn_t)(MatGSO<ZT, FP_NR<double>> *);                                                              \
    static fn_t orig = b200shim::next_symbol<fn_t>(B200ShimTraits<ZT>::sym_size_increased());                       \
    /* constructor (gso.h:113-130) or create_rows / remove_last_rows: whatever the device held for this address is  \
       gone; the object is adopted again at its next update_gso_row if nothing of its GSO is valid */                \
    shim_forget(static_cast<MatGSOInterface<ZT, FP_NR<double>> *>(this));                                           \
    orig(this);                                                                                                     \
  }

B200_SHIM_FOR(Z_NR<long>)
B200_SHIM_FOR(Z_NR<mpz_t>)
B200_SHIM_CTOR_FOR(Z_NR<long>)
B200_SHIM_CTOR_FOR(Z_NR<mpz_t>)

FPLLL_END_NAMESPACE

// ---- BKZReduction<Z_NR<long>, FP_NR<double>>::bkz() on the device driver -------------------------------------------------
FPLLL_BEGIN_NAMESPACE
namespace {
long g_bkz_taken = 0;
}
template <> bool BKZReduction<Z_NR<long>, FP_NR<double>>::bkz()
{
  typedef bool (*fn_t)(BKZReduction<Z_NR<long>, FP_NR<double>> *);
  static fn_t orig = b200shim::next_symbol<fn_t>("_ZN5fplll12BKZReductionINS_4Z_NRIlEENS_5FP_NRIdEEE3bkzEv");
  static const bool takeover = b200shim::enabled() && !(getenv("B200_SHIM_BKZ") && atoi(getenv("B200_SHIM_BKZ")) == 0);
  auto *mg = dynamic_cast<MatGSO<Z_NR<long>, FP_NR<double>> *>(&m);
  const int unsupported = BKZ_SD_VARIANT | BKZ_SLD_RED | BKZ_DUMP_GSO;
  if (!takeover || !mg || (param.flags & unsupported) || mg->enable_int_gram || mg->enable_transform ||
      param.block_size < 2 || num_rows != mg->b.get_rows() || num_rows > 512 || b200gso_device_count() == 0)
    return orig(this);
  const int d = mg->b.get_rows(), n = mg->b.get_cols();
  b200bkz_t *h = nullptr;
  int dev0     = 0;
  if (b200bkz_create(&h, &dev0, 1) != 0)
    throw std::runtime_error(std::string("b200 shim: b200bkz_create: ") + b200bkz_last_error());
  // Strategy table (bkz_param.h:34-66): preprocessing block sizes and pruning vectors per block size
  for (size_t bs = 0; bs < param.strategies.size(); bs++)
  {
    const Strategy &st = param.strategies[bs];
    if (st.pruning_parameters.empty() && st.preprocessing_block_sizes.empty())
      continue;
    std::vector<int> pre(st.preprocessing_block_sizes.begin(), st.preprocessing_block_sizes.end());
    std::vector<double> gh, ex, co;
    for (const PruningParams &pp : st.pruning_parameters)
    {
      if (pp.coefficients.size() != bs)
        continue;  // the default PruningParams() of an EmptyStrategy carries no vector: "no pruning"
      gh.push_back(pp.gh_factor), ex.push_back(pp.expectation);
      co.insert(co.end(), pp.coefficients.begin(), pp.coefficients.end());
    }
    b200bkz_add_strategy(h, (int)bs, pre.data(), (int)pre.size(), gh.data(), ex.data(), co.data(), (int)gh.size());
  }
  b200bkz_param p;
  b200bkz_default_param(&p, param.block_size);
  p.delta = param.delta, p.flags = (param.flags & (BKZ_VERBOSE | BKZ_MAX_LOOPS | BKZ_MAX_TIME | BKZ_BOUNDED_LLL |
                                                   BKZ_AUTO_ABORT | BKZ_GH_BND)) | B200BKZ_NO_LLL;
  p.max_loops = param.max_loops, p.max_time = param.max_time;
  p.auto_abort_scale = param.auto_abort_scale, p.auto_abort_max_no_dec = param.auto_abort_max_no_dec;
  p.gh_factor = param.gh_factor, p.min_success_probability = param.min_success_probability;
  p.rerandomization_density = param.rerandomization_density;
  std::vector<int64_t> flat((size_t)d * n);
  for (int i = 0; i < d; i++)
    for (int j = 0; j < n; j++)
      flat[(size_t)i * n + j] = mg->b(i, j).get_si();
  b200bkz_stats stt;
  const int rc = b200bkz_reduce(h, d, n, flat.data(), &p, &stt);
  b200bkz_destroy(h);
  if (rc != 0)
    throw std::runtime_error(std::string("b200 shim: b200bkz_reduce: ") + b200bkz_last_error());
  // the reduced basis back into the caller's matrix; its GSO object is told through the reference's own protocol
  m.row_op_begin(0, d);
  for (int i = 0; i < d; i++)
    for (int j = 0; j < n; j++)
      mg->b(i, j) = (long)flat[(size_t)i * n + j];
  m.row_op_end(0, d);
  nodes = (long)stt.enum_nodes;
  g_bkz_taken++;
  return set_status(stt.status);
}
FPLLL_END_NAMESPACE

extern "C" long b200_matgso_shim_bkz_taken(void) { return fplll::g_bkz_taken; }

extern "C" void b200_matgso_shim_stats(long *out6)
{
  out6[0] = b200shim::g_adopted, out6[1] = b200shim::g_declined, out6[2] = b200shim::g_updates;
  out6[3] = b200shim::g_uploads, out6[4] = b200shim::g_moves, out6[5] = b200shim::g_setr;
}
