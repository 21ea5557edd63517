// Linear assignment by shortest augmenting paths (Jonker-Volgenant; the algorithm behind
// scipy.optimize.linear_sum_assignment, which utils/perm.py:73 calls once per pair of geometries), written once for a
// "team" of cooperating threads: a warp or a CTA on the device (csrc/perm.cu), a single thread on the host (the CPU test
// builds this header with a host compiler and checks it against SciPy).
//
// A team provides
//   tid, size      this thread's rank and the number of threads; column j belongs to thread j % size
//   sync()         barrier + memory fence over the team
//   argmin(a)      the smallest (val, idx) pair over the team's threads, ties to the lowest idx, idx < 0 = "none";
//                  every thread gets the same answer
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define SG_PERM_HD __host__ __device__ __forceinline__
#else
#define SG_PERM_HD inline
#endif

namespace sgdml {
namespace perm {

struct ArgMin {
  double val;
  int idx;
};

// a, unless b is a candidate and smaller (lower index on equal values).  Written so that a NaN never displaces a
// candidate and the result always has idx >= 0 when either side has.
SG_PERM_HD ArgMin argmin2(const ArgMin& a, const ArgMin& b) {
  if (b.idx < 0) return a;
  if (a.idx < 0) return b;
  if (b.val < a.val || (b.val == a.val && b.idx < a.idx)) return b;
  return a;
}

struct SerialTeam {
  static constexpr int tid = 0;
  static constexpr int size = 1;
  void sync() const {}
  ArgMin argmin(const ArgMin& a) const { return a; }
};

// Minimum-cost assignment of the n rows of c(i, j) = cost[i * ldc + j] + (z[i] != z[j] ? penalty : 0) to its n columns:
// on return col4row[i] is the column of row i and row4col its inverse.  Rows are inserted in index order; the column that
// closes each scan is the arg-min with the lowest index, so the result depends on the input only, not on the team.
// Work arrays: u, v, spc (n doubles each), path, row4col, col4row (n ints each), sc (n bytes).
// Every loop is bounded by n: each scan step moves one column into the scanned set, and since row `cur` is not assigned
// yet one of the n columns is free, so a sink is reached after at most n steps whatever the values are (NaN included);
// every column outside the scanned set has a predecessor after the first step, so the result is always a permutation.
template <class Team>
SG_PERM_HD void lap_solve(const Team& tm, int n, const double* cost, int ldc, double penalty, const int* z, double* u,
                          double* v, double* spc, int* path, int* row4col, int* col4row, unsigned char* sc) {
  const int tid = tm.tid, nt = tm.size;
  for (int j = tid; j < n; j += nt) {
    u[j] = 0.0;
    v[j] = 0.0;
    row4col[j] = -1;
    col4row[j] = -1;
    path[j] = -1;
  }
  tm.sync();
  for (int cur = 0; cur < n; ++cur) {
    for (int j = tid; j < n; j += nt) {  // own columns only: no barrier needed before the scan reads them
      spc[j] = (double)INFINITY;
      path[j] = -1;
      sc[j] = 0;
    }
    double min_val = 0.0;
    int i = cur, sink = -1;
    for (int step = 0; step < n && sink < 0; ++step) {
      const double ui = u[i];
      const int zi = z[i];
      const double* ci = cost + (int64_t)i * ldc;
      ArgMin best;
      best.val = 0.0;
      best.idx = -1;
      for (int j = tid; j < n; j += nt) {
        if (sc[j]) continue;
        const double c = ci[j] + (z[j] != zi ? penalty : 0.0);
        const double r = min_val + c - ui - v[j];
        if (path[j] < 0 || r < spc[j]) {  // the first visit always records a predecessor, whatever r is
          spc[j] = r;
          path[j] = i;
        }
        ArgMin cand;
        cand.val = spc[j];
        cand.idx = j;
        best = argmin2(best, cand);
      }
      best = tm.argmin(best);
      const int jm = best.idx;
      if (jm < 0) break;  // unreachable: a column outside the scanned set exists at every step
      min_val = best.val;
      if (jm % nt == tid) sc[jm] = 1;
      const int r4 = row4col[jm];
      if (r4 < 0)
        sink = jm;
      else
        i = r4;
    }
    // dual update: the scanned rows are `cur` and the rows assigned to the scanned columns.  Nobody reads u or v
    // between the last arg-min and the barrier below.
    for (int j = tid; j < n; j += nt) {
      if (!sc[j]) continue;
      const double d = min_val - spc[j];
      v[j] -= d;
      const int r = row4col[j];
      if (r >= 0) u[r] += d;
    }
    if (tid == 0) u[cur] += min_val;
    tm.sync();
    // augment along the predecessor chain from the sink back to `cur`
    if (tid == 0 && sink >= 0) {
      int j = sink;
      for (int hop = 0; hop < n; ++hop) {
        const int r = path[j];
        if (r < 0) break;
        row4col[j] = r;
        const int prev = col4row[r];
        col4row[r] = j;
        j = prev;
        if (r == cur || j < 0) break;
      }
    }
    tm.sync();
  }
}

}  // namespace perm
}  // namespace sgdml
