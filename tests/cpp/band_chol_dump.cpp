// band_chol_dump.cpp — runs the compiled glio::detail::cholesky_solve_scalar on band systems read from stdin and writes what it
// returns to stdout, so tests/test_band_solve_reference.py can hold it to tests/band_solve_reference.py bit for bit.
// Per case, in: int32 n, int32 hb, n*(hb+1) doubles of band (glio_batch_solve's layout), n doubles of b.
// Per case, out: int32 ok, n*(hb+1) doubles of the factored band, n doubles of x.  The band is used as given (no BandMat::reset
// clamp), so slots with j < 0 are passed through untouched.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../glio_b200/csrc/solver.h"

int main() {
  int32_t hdr[2];
  while (fread(hdr, sizeof(int32_t), 2, stdin) == 2) {
    const int n = hdr[0], hb = hdr[1];
    if (n <= 0 || hb < 0) return 2;
    glio::BandMat A;
    A.n = n; A.hb = hb; A.a.resize((size_t)n * (hb + 1));
    std::vector<double> b(n), x(n, 0.0);
    if (fread(A.a.data(), sizeof(double), A.a.size(), stdin) != A.a.size() || fread(b.data(), sizeof(double), n, stdin) != (size_t)n) return 3;
    const int32_t ok = glio::detail::cholesky_solve_scalar(A, b.data(), x.data()) ? 1 : 0;
    fwrite(&ok, sizeof(int32_t), 1, stdout);
    fwrite(A.a.data(), sizeof(double), A.a.size(), stdout);
    fwrite(x.data(), sizeof(double), n, stdout);
  }
  return 0;
}
