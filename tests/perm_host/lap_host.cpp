// Host build of the assignment solver the matching kernel runs (sgdml_b200/csrc/perm_solve.cuh), with a team of one
// thread, for tests/test_perm_oracle.py: index and loop-bound mistakes show up here, under a CPU debugger if need be.
#include <vector>

#include "perm_solve.cuh"

extern "C" int lap_host(int n, const double* cost, int ldc, double penalty, const int* z, int* col4row) {
  std::vector<double> u(n), v(n), spc(n);
  std::vector<int> path(n), row4col(n);
  std::vector<unsigned char> sc(n);
  sgdml::perm::SerialTeam tm;
  sgdml::perm::lap_solve(tm, n, cost, ldc, penalty, z, u.data(), v.data(), spc.data(), path.data(), row4col.data(),
                         col4row, sc.data());
  for (int j = 0; j < n; ++j)
    if (row4col[j] < 0 || col4row[row4col[j]] != j) return 1;
  return 0;
}
