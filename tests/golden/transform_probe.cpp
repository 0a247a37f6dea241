// transform_probe.cpp — records what the reference library computes for the transform U (MatGSO with a non-empty u,
// BKZ with a non-empty U), for tests/golden/transform_ref.npz.  Built and run by make_transform_golden.py against the
// reference build in oracle/_ref; the test suite only reads the fixture it writes.
//
// Commands on stdin, one per line:
//   load P                       basis (fplll text format) -> the long matrix B and the mpz matrix Bm
//   gso FLAGS                    MatGSO<Z_NR<long>, FP_NR<double>>(B, U, {}, FLAGS) with U = identity (non-empty: the
//                                reference tracks U only then)
//   update_gso | update_row I J | row_op_begin F L | row_op_end F L | row_addmul_we I J X E | row_swap I J |
//   move_row O N | negate I      the MatGSO calls of the same names (negate = negate_row_of_b)
//   lll DELTA ETA                LLLReduction<Z_NR<long>, FP_NR<double>>(gso, DELTA, ETA, LLL_DEFAULT).lll()
//   bkz BLOCK FLAGS MAXLOOPS     bkz_reduction(&Bm, &Um, BKZParam(BLOCK, no strategies), FT_DOUBLE) with Um non-empty
//   save_b P | save_u P          the long B / U, or after bkz the mpz Bm / Um
#include <fplll.h>

#include <fstream>
#include <iostream>
#include <memory>
#include <sstream>
#include <string>

using namespace std;
using namespace fplll;

typedef MatGSO<Z_NR<long>, FP_NR<double>> GsoL;

int main()
{
  ZZ_mat<mpz_t> Bm, Um;
  ZZ_mat<long> B, U, UT;
  unique_ptr<GsoL> g;
  bool after_bkz = false;
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
      ifstream f(p);
      f >> Bm;
      B.resize(Bm.get_rows(), Bm.get_cols());
      for (int i = 0; i < Bm.get_rows(); i++)
        for (int j = 0; j < Bm.get_cols(); j++)
          B(i, j) = Bm(i, j).get_si();
      g.reset();
      after_bkz = false;
    }
    else if (c == "gso")
    {
      int fl;
      is >> fl;
      U.gen_identity(B.get_rows());
      g.reset(new GsoL(B, U, UT, fl));
    }
    else if (c == "update_gso")
      printf("update_gso %d\n", (int)g->update_gso());
    else if (c == "update_row")
    {
      int i, j;
      is >> i >> j;
      printf("update_row %d %d %d\n", i, j, (int)g->update_gso_row(i, j));
    }
    else if (c == "row_op_begin" || c == "row_op_end")
    {
      int a, b;
      is >> a >> b;
      if (c == "row_op_begin")
        g->row_op_begin(a, b);
      else
        g->row_op_end(a, b);
    }
    else if (c == "row_addmul_we")
    {
      int i, j;
      double x;
      long e;
      is >> i >> j >> x >> e;
      FP_NR<double> fx = x;
      g->row_addmul_we(i, j, fx, e);
    }
    else if (c == "row_swap")
    {
      int a, b;
      is >> a >> b;
      g->row_swap(a, b);
    }
    else if (c == "move_row")
    {
      int a, b;
      is >> a >> b;
      g->move_row(a, b);
    }
    else if (c == "negate")
    {
      int i;
      is >> i;
      g->negate_row_of_b(i);
    }
    else if (c == "lll")
    {
      double delta, eta;
      is >> delta >> eta;
      LLLReduction<Z_NR<long>, FP_NR<double>> lll(*g, delta, eta, LLL_DEFAULT);
      lll.lll();
      printf("lll status=%d swaps=%d zeros=%d\n", lll.status, lll.n_swaps, lll.zeros);
    }
    else if (c == "bkz")
    {
      int bs, fl, ml;
      is >> bs >> fl >> ml;
      vector<Strategy> strategies;
      BKZParam param(bs, strategies);
      param.flags     = fl;
      param.max_loops = ml;
      Um.resize(1, 1);  // non-empty: bkz_reduction then starts it at the identity (bkz.cpp:857-859), like fplll -of u
      int st = bkz_reduction(&Bm, &Um, param, FT_DOUBLE, 0);
      after_bkz = true;
      printf("bkz status=%d\n", st);
    }
    else if (c == "save_b" || c == "save_u")
    {
      string p;
      is >> p;
      ofstream f(p);
      if (after_bkz)
        f << (c == "save_b" ? Bm : Um) << endl;
      else
        f << (c == "save_b" ? B : U) << endl;
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
