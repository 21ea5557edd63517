// Gaussian-process posterior covariance blocks of an analytic-solver model (sgdml_b200_posterior_blocks,
// sgdml_b200/posterior.py).  With C = -K_ref over [training; queries], L the Cholesky factor of C_XX + lam I over the
// training columns X and V = C(z, X) L^-T the solved cross rows of a chunk of queries, every query q gets
//   Sigma_q = scale * sgn * (P_q - V_q V_q^T),   sgn = -1 on the E-F entries, +1 elsewhere,
// where V_q gathers the 3N force rows and the one energy row of q and P_q = C(z_q, z_q) is its prior block.
//
// The length-n reduction V_q V_q^T runs in two launches with no atomics:
//   k_posterior_partial  grid (lower-triangle 32 x 32 tiles, column slices of POST_SLICE, queries): each CTA sums
//                        one tile over one slice, in increasing column order, into its own slot of a workspace;
//   k_posterior_blocks   grid (tiles, queries): adds the slices' partial sums in slice order, subtracts from the prior,
//                        scales, flips the E-F sign and writes each lower-triangle entry and its mirror.
// Slice bounds are multiples of POST_SLICE from column 0, and no sum depends on the query's position in V or on how
// many queries V holds, so every Sigma_q is bit-identical for every chunking of a batch.
#include <algorithm>

#include "common.cuh"

namespace sgdml {

constexpr int POST_T = 32;         // tile edge (entries of Sigma_q)
constexpr int POST_KB = 32;        // columns per shared-memory stage
constexpr int POST_SLICE = 4096;   // columns per CTA of the first stage (a multiple of POST_KB)

// Row of V holding output component i (< d = 3N + 1) of query q: force rows q 3N + r, then the energy rows.
__device__ __forceinline__ int64_t post_row(int i, int q, int n3, int n_query) {
  return i < n3 ? (int64_t)q * n3 + i : (int64_t)n_query * n3 + q;
}

// tile t of the lower block triangle -> (tile row I, tile column J), J <= I
__device__ __forceinline__ void post_tile(int t, int& I, int& J) {
  I = 0;
  while ((I + 1) * (I + 2) / 2 <= t) ++I;
  J = t - I * (I + 1) / 2;
}

// part[((q * n_slices + s) * n_tiles + t) * 1024 + r * 32 + c] = sum over the columns of slice s of V[row_i] V[row_j],
// i = 32 I + r, j = 32 J + c (zero outside d).  256 threads: column c = threadIdx.x & 31, rows r = threadIdx.x / 32 + 8 k.
__global__ void __launch_bounds__(256) k_posterior_partial(const double* __restrict__ V, int64_t ldv, int64_t n,
                                                           int n_atoms, int n_query, int n_tiles, int n_slices,
                                                           double* __restrict__ part) {
  __shared__ double A[POST_T][POST_KB + 1], B[POST_T][POST_KB + 1];
  const int t = blockIdx.x, s = blockIdx.y, q = blockIdx.z;
  const int n3 = 3 * n_atoms, d = n3 + 1;
  int I, J;
  post_tile(t, I, J);
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t k0 = (int64_t)s * POST_SLICE, k1 = min(k0 + POST_SLICE, n);
  // rows 32 I + ty + 8 u (A) and 32 J + ty + 8 u (B) that this thread stages, nullptr outside d
  const double* ra[4];
  const double* rb[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int i = I * POST_T + ty + 8 * u, j = J * POST_T + ty + 8 * u;
    ra[u] = i < d ? V + post_row(i, q, n3, n_query) * ldv : nullptr;
    rb[u] = j < d ? V + post_row(j, q, n3, n_query) * ldv : nullptr;
  }
  double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
  for (int64_t kb = k0; kb < k1; kb += POST_KB) {
    const int64_t k = kb + tx;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      A[ty + 8 * u][tx] = (ra[u] != nullptr && k < k1) ? ra[u][k] : 0.0;
      B[ty + 8 * u][tx] = (rb[u] != nullptr && k < k1) ? rb[u][k] : 0.0;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < POST_KB; ++k) {
      const double b = B[tx][k];
      a0 = fma(A[ty][k], b, a0);
      a1 = fma(A[ty + 8][k], b, a1);
      a2 = fma(A[ty + 16][k], b, a2);
      a3 = fma(A[ty + 24][k], b, a3);
    }
    __syncthreads();
  }
  double* __restrict__ out = part + (((int64_t)q * n_slices + s) * n_tiles + t) * (POST_T * POST_T);
  out[ty * POST_T + tx] = a0;
  out[(ty + 8) * POST_T + tx] = a1;
  out[(ty + 16) * POST_T + tx] = a2;
  out[(ty + 24) * POST_T + tx] = a3;
}

// Sigma_q[i][j] = Sigma_q[j][i] = scale * sgn * (P_q[i][j] - sum_s part[q][s][t][.]) for i >= j, slices in order.
__global__ void __launch_bounds__(256) k_posterior_blocks(const double* __restrict__ part, const double* __restrict__ prior,
                                                          int n_atoms, int n_tiles, int n_slices, double scale,
                                                          double* __restrict__ out) {
  const int t = blockIdx.x, q = blockIdx.y;
  const int d = 3 * n_atoms + 1;
  int I, J;
  post_tile(t, I, J);
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int j = J * POST_T + tx;
  const double* __restrict__ P = prior + (int64_t)q * d * d;
  double* __restrict__ S = out + (int64_t)q * d * d;
  for (int u = 0; u < 4; ++u) {
    const int r = ty + 8 * u, i = I * POST_T + r;
    if (i >= d || j >= d || j > i) continue;
    const double* __restrict__ p = part + ((int64_t)q * n_slices * n_tiles + t) * (POST_T * POST_T) + r * POST_T + tx;
    double g = p[0];
    for (int s = 1; s < n_slices; ++s) g += p[(int64_t)s * n_tiles * (POST_T * POST_T)];
    const double sgn = ((i == d - 1) != (j == d - 1)) ? -scale : scale;
    const double v = sgn * (P[(int64_t)i * d + j] - g);
    S[(int64_t)i * d + j] = v;
    S[(int64_t)j * d + i] = v;
  }
}

}  // namespace sgdml

using namespace sgdml;

extern "C" int sgdml_b200_posterior_blocks(const double* V, int64_t ldv, int64_t n, int64_t n_query, int64_t n_atoms,
                                           const double* prior, double scale, double* out, void* stream) {
  SG_TRY(require_device());
  SG_ARG(V != nullptr && prior != nullptr && out != nullptr && is_device_ptr(V));
  SG_ARG(n >= 1 && ldv >= n && n_query >= 1 && n_query <= 65535 && n_atoms >= 1 && n_atoms <= 1023);
  const int64_t d = 3 * n_atoms + 1;
  const int nT = ceil_div(d, POST_T);
  const int n_tiles = nT * (nT + 1) / 2;
  const int64_t n_slices = (n + POST_SLICE - 1) / POST_SLICE;
  SG_ARG(n_slices <= 65535);
  cudaStream_t s = (cudaStream_t)stream;
  Staged sP, sO;
  SG_TRY(sP.init(prior, sizeof(double) * (size_t)(n_query * d * d), true, s));
  SG_TRY(sO.init(out, sizeof(double) * (size_t)(n_query * d * d), false, s));
  double* part = nullptr;
  const size_t part_bytes = sizeof(double) * (size_t)n_query * n_slices * n_tiles * POST_T * POST_T;
  SG_CUDA(cached_malloc(&part, part_bytes));
  auto body = [&]() -> int {
    k_posterior_partial<<<dim3((unsigned)n_tiles, (unsigned)n_slices, (unsigned)n_query), 256, 0, s>>>(
        V, ldv, n, (int)n_atoms, (int)n_query, n_tiles, (int)n_slices, part);
    SG_CUDA(cudaGetLastError());
    k_posterior_blocks<<<dim3((unsigned)n_tiles, (unsigned)n_query), 256, 0, s>>>(
        part, (const double*)sP.dev(), (int)n_atoms, n_tiles, (int)n_slices, scale, (double*)sO.dev());
    SG_CUDA(cudaGetLastError());
    count_launch(KID_MISC, 2);
    SG_TRY(sO.finish(s));
    SG_CUDA(cudaStreamSynchronize(s));
    return 0;
  };
  const int rc = body();
  cudaStreamSynchronize(s);  // the workspace goes back to the cache only once no kernel reads it
  cached_free(part);
  return rc;
}
