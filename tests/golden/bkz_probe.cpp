// bkz_probe.cpp — records what the reference library's whole bkz_reduction call computes, for
// tests/golden/bkz_driver_ref.npz.  Built and run by make_bkz_golden.py against the reference build in oracle/_ref; the
// test suite only reads the fixture it writes.
//
//   bkz_probe IN OUT BLOCK DELTA FLAGS MAX_LOOPS AA_SCALE AA_MAX_NO_DEC GH_FACTOR STRATEGIES WITH_U
//
// IN: the input basis (fplll text format).  STRATEGIES: a JSON file read by load_strategies_json, or "-" for none (the
// EmptyStrategy of every block size).  WITH_U: 1 runs bkz_reduction with a non-empty U (the reference then starts it at
// the identity, bkz.cpp:857-859, and its wrapper LLL takes the mpz path, wrapper.cpp:287-290).
// Writes OUT.b (B after bkz_reduction), OUT.u (U, with WITH_U), OUT.lll (the wrapper LLL alone on IN, lll_reduction with
// the same delta, and with a U when WITH_U, so that it takes the same path), OUT.lllu (that U); prints "status=S lll_status=L" on stdout.
// The call runs with BKZ_VERBOSE added, which only prints: the caller counts the per-tour lines on stderr.  The bundled
// enumerator runs on one thread.
#include <fplll.h>

#include <cstdlib>
#include <fstream>
#include <iostream>
#include <string>

using namespace std;
using namespace fplll;

int main(int argc, char **argv)
{
  if (argc != 12)
  {
    fprintf(stderr, "usage: bkz_probe IN OUT BLOCK DELTA FLAGS MAX_LOOPS AA_SCALE AA_MAX_NO_DEC GH_FACTOR STRATEGIES "
                    "WITH_U\n");
    return 2;
  }
  const string in = argv[1], out = argv[2], strat_path = argv[10];
  const int block_size = atoi(argv[3]), flags = atoi(argv[5]), max_loops = atoi(argv[6]);
  const double delta = atof(argv[4]), aa_scale = atof(argv[7]), gh_factor = atof(argv[9]);
  const int aa_max_no_dec = atoi(argv[8]);
  const bool with_u       = atoi(argv[11]) != 0;

  ZZ_mat<mpz_t> B, L, U, UL;
  {
    ifstream f(in);
    f >> B;
  }
  L = B;

  // the wrapper LLL alone, as bkz_reduction runs it before BKZ (same delta: bkz.cpp:862)
  const double lll_delta = delta < 1 ? delta : LLL_DEF_DELTA;
  int lll_status;
  if (with_u)
  {
    UL.gen_identity(L.get_rows());
    lll_status = lll_reduction(L, UL, lll_delta, LLL_DEF_ETA, LM_WRAPPER, FT_DEFAULT, 0, LLL_DEFAULT);
  }
  else
    lll_status = lll_reduction(L, lll_delta, LLL_DEF_ETA, LM_WRAPPER, FT_DEFAULT, 0, LLL_DEFAULT);

  set_threads(1);  // the bundled enumerator on one thread, as the other BKZ goldens were made
  vector<Strategy> strategies;
  if (strat_path != "-")
    strategies = load_strategies_json(strat_path);
  BKZParam param(block_size, strategies, delta, flags | BKZ_VERBOSE, max_loops, 0.0, aa_scale, aa_max_no_dec,
                 gh_factor);
  if (with_u)
    U.resize(1, 1);  // non-empty: bkz_reduction starts it at the identity
  const int status = bkz_reduction(&B, with_u ? &U : nullptr, param, FT_DOUBLE, 0);

  {
    ofstream f(out + ".b");
    f << B << endl;
  }
  if (with_u)
  {
    ofstream f(out + ".u");
    f << U << endl;
  }
  {
    ofstream f(out + ".lll");
    f << L << endl;
  }
  if (with_u)
  {
    ofstream f(out + ".lllu");
    f << UL << endl;
  }
  printf("status=%d lll_status=%d\n", status, lll_status);
  return 0;
}
