// hh_transform_probe.cpp — records what the reference library computes for the transform U and U^-T of
// MatHouseholder<Z_NR<long>, FP_NR<double>> (u and u_inv_t non-empty) and of HLLLReduction over it, for
// tests/golden/hh_transform_ref.npz.  Built and run by make_hh_transform_golden.py against the reference build in
// oracle/_ref; the test suite only reads the fixture it writes.
//
// Commands on stdin, one per line:
//   load P                       basis (fplll text format) -> the long matrix B
//   hh FLAGS                     MatHouseholder<Z_NR<long>, FP_NR<double>>(B, U, UT, FLAGS) with U = UT = identity
//                                (non-empty: the reference tracks u only then, and u_inv_t only with u)
//   hh_refresh_R_bf I | hh_refresh_R I | hh_update_R I LASTJ | hh_update_R_last I | hh_size_reduce K END START |
//   hh_swap I J | hh_recover_R I | hh_set_updated_R_false      the MatHouseholder calls of the same names
//   hlll DELTA ETA THETA C       HLLLReduction<Z_NR<long>, FP_NR<double>>(MatHouseholder(B, U, UT, ROW_EXPO |
//                                OP_FORCE_LONG), DELTA, ETA, THETA, C, LLL_DEFAULT).hlll() with U = UT = identity, the
//                                object hlll_reduction(b, u, u_inv, ...) builds (wrapper.cpp:790-806, :1075-1087)
//   save_b P | save_u P | save_uinvt P    the long B, U and UT (UT is u_inv_t as the object holds it: U^-T)
#include <fplll.h>

#include <fstream>
#include <iostream>
#include <memory>
#include <sstream>
#include <string>

using namespace std;
using namespace fplll;

typedef MatHouseholder<Z_NR<long>, FP_NR<double>> HhL;

static void read_long(const string &p, ZZ_mat<long> &B)
{
  ZZ_mat<mpz_t> Bm;
  ifstream f(p);
  f >> Bm;
  B.resize(Bm.get_rows(), Bm.get_cols());
  for (int i = 0; i < Bm.get_rows(); i++)
    for (int j = 0; j < Bm.get_cols(); j++)
      B(i, j) = Bm(i, j).get_si();
}

int main()
{
  ZZ_mat<long> B, U, UT;
  unique_ptr<HhL> hh;
  string line;
  while (getline(cin, line))
  {
    istringstream is(line);
    string c;
    if (!(is >> c) || c[0] == '#')
      continue;
    if (c == "load")
    {
      string p;
      is >> p;
      hh.reset();
      read_long(p, B);
    }
    else if (c == "hh")
    {
      int fl;
      is >> fl;
      U.gen_identity(B.get_rows());
      UT.gen_identity(B.get_rows());
      hh.reset(new HhL(B, U, UT, fl));
    }
    else if (c == "hh_refresh_R_bf") { int i; is >> i; hh->refresh_R_bf(i); }
    else if (c == "hh_refresh_R") { int i; is >> i; hh->refresh_R(i); }
    else if (c == "hh_update_R") { int i, l; is >> i >> l; hh->update_R(i, l != 0); }
    else if (c == "hh_update_R_last") { int i; is >> i; hh->update_R_last(i); }
    else if (c == "hh_size_reduce")
    {
      int k, e, st;
      is >> k >> e >> st;
      printf("hh_size_reduce %d\n", (int)hh->size_reduce(k, e, st));
    }
    else if (c == "hh_swap") { int i, j; is >> i >> j; hh->swap(i, j); }
    else if (c == "hh_recover_R") { int i; is >> i; hh->recover_R(i); }
    else if (c == "hh_set_updated_R_false") { hh->set_updated_R_false(); }
    else if (c == "hlll")
    {
      double delta, eta, theta, cc;
      is >> delta >> eta >> theta >> cc;
      hh.reset();
      U.gen_identity(B.get_rows());
      UT.gen_identity(B.get_rows());
      HhL m(B, U, UT, HOUSEHOLDER_ROW_EXPO | HOUSEHOLDER_OP_FORCE_LONG);
      HLLLReduction<Z_NR<long>, FP_NR<double>> red(m, delta, eta, theta, cc, LLL_DEFAULT);
      red.hlll();
      printf("hlll status=%d\n", red.get_status());
    }
    else if (c == "save_b" || c == "save_u" || c == "save_uinvt")
    {
      string p;
      is >> p;
      ofstream f(p);
      f << (c == "save_b" ? B : c == "save_u" ? U : UT) << endl;
    }
    else
    {
      fprintf(stderr, "unknown command %s\n", c.c_str());
      return 2;
    }
    fflush(stdout);
  }
  return 0;
}
