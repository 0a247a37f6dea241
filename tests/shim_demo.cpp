// shim_demo — TEST PROGRAM: the reference's own LLLReduction over its own MatGSO, compiled against the unmodified
// reference headers and linked with the unmodified libfplll.so.  Run once plainly and once with
// LD_PRELOAD=libb200fplll.so (fplll_b200/csrc/fplll_matgso_shim.cpp): the second run executes every update_gso_row on
// the GPU and must print byte-identical results (the device GSO is bit-exact, so LLL walks the same trajectory).
// usage: shim_demo IN.txt long|mpz|long_gram|mpz_gram OUT.bin     (_gram: GSO_INT_GRAM, the exact integer Gram matrix)
#include <fplll/fplll.h>
#include <cstdio>
#include <fstream>
#include <iostream>
using namespace fplll;
extern "C" void b200_matgso_shim_stats(long *out6) __attribute__((weak));

template <class ZT> static int run(ZZ_mat<ZT> &b, int flags, const char *out)
{
  ZZ_mat<ZT> u, ui;
  MatGSO<Z_NR<ZT>, FP_NR<double>> M(b, u, ui, flags);
  LLLReduction<Z_NR<ZT>, FP_NR<double>> lll(M, 0.99, 0.51, LLL_DEFAULT);
  lll.lll();
  const int st = lll.status;
  bool ok = M.update_gso();
  FILE *f = fopen(out, "wb");
  const int d = b.get_rows(), n = b.get_cols();
  int hdr[4] = {d, n, st, ok ? 1 : 0};
  fwrite(hdr, sizeof(int), 4, f);
  for (int i = 0; i < d; i++)
    for (int j = 0; j <= i; j++)
    {
      double m = j < i ? M.get_mu_matrix()(i, j).get_d() : 0.0, r = M.get_r_matrix()(i, j).get_d();
      fwrite(&m, 8, 1, f);
      fwrite(&r, 8, 1, f);
    }
  for (int i = 0; i < d; i++)
  {
    long e = M.row_expo.empty() ? 0 : M.row_expo[i];
    fwrite(&e, 8, 1, f);
  }
  std::ofstream o(std::string(out) + ".basis");
  o << b << std::endl;
  fclose(f);
  // the reference's own checker on the result (is_lll_reduced over an mpfr GSO, lll.cpp:226-258)
  printf("shim_demo status=%d gso_ok=%d", st, ok ? 1 : 0);
  return st;
}

int main(int argc, char **argv)
{
  if (argc < 4)
    return 2;
  ZZ_mat<mpz_t> B;
  std::ifstream f(argv[1]);
  f >> B;
  const std::string mode = argv[2];
  if (mode == "long" || mode == "long_gram")
  {
    ZZ_mat<long> b(B.get_rows(), B.get_cols());
    for (int i = 0; i < B.get_rows(); i++)
      for (int j = 0; j < B.get_cols(); j++)
        b(i, j) = B(i, j).get_si();
    run<long>(b, mode == "long" ? GSO_ROW_EXPO : GSO_INT_GRAM, argv[3]);
  }
  else if (mode == "mpz_gram")
    run<mpz_t>(B, GSO_INT_GRAM, argv[3]);  // the flavour the wrapper's proved stage uses (wrapper.cpp:354-356)
  else
    run<mpz_t>(B, GSO_ROW_EXPO | GSO_OP_FORCE_LONG, argv[3]);  // wrapper.cpp:538-553
  long s[6] = {0, 0, 0, 0, 0, 0};
  if (b200_matgso_shim_stats)
    b200_matgso_shim_stats(s);
  printf(" adopted=%ld declined=%ld forwarded=%ld uploads=%ld moves=%ld set_r=%ld\n", s[0], s[1], s[2], s[3], s[4], s[5]);
  return 0;
}
