// The BAOAB Langevin integrator step of sgdml_b200_md_run (driver: md_run in predict.cu).
//
// A step from (r, v, F(r)) with h = dt/2, c1 = exp(-gamma dt), s_i = inverse mass of the atom of coordinate i and
// sigma_i = sqrt((1 - c1^2) kT s_i):
//   B  v += h (F s)    A  r += h v    O  v = c1 v + sigma xi    A  r += h v    F = F(r)    B  v += h (F s)
// The last B needs the new forces, so it runs at the start of the next step's kernel (or in the completing launch
// at the end of a run): one kernel per step.  The B and A updates round exactly as written (__dmul_rn / __dadd_rn,
// never contracted into an FMA), so a NumPy restatement fed the same forces reproduces them bit for bit.
//
// Noise: Philox4x32-10 (Salmon et al., SC'11), key (seed mod 2^32, seed >> 32), counter (j, replica, step mod 2^32,
// step >> 32) for the coordinate pair (2j, 2j + 1), Box-Muller on the two 53-bit uniforms of its four output words.
// The step index comes from the handle's counter in device memory, so a replayed graph draws fresh noise each step
// and a run continued over several calls draws exactly the noise of one long run.
#include <cmath>

#include "common.cuh"
#include "md.cuh"

namespace sgdml {

namespace {

__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c[0], hi0 = __umulhi(0xD2511F53u, c[0]);
    const uint32_t lo1 = 0xCD9E8D57u * c[2], hi1 = __umulhi(0xCD9E8D57u, c[2]);
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0;
    c[1] = lo1;
    c[2] = n2;
    c[3] = lo0;
  }
}

// uniform in (0, 1) from the 53 high bits of (hi:lo)
__device__ __forceinline__ double uniform53(uint32_t hi, uint32_t lo) {
  const uint64_t u = ((uint64_t)hi << 32) | lo;
  return ((double)(u >> 11) + 0.5) * 0x1p-53;
}

__global__ void __launch_bounds__(MD_THREADS) k_md_step(const MdParams* __restrict__ P, const double* __restrict__ s,
                                                       const double* __restrict__ sigma, double* __restrict__ R,
                                                       double* __restrict__ V, const double* __restrict__ F,
                                                       const double* __restrict__ E, uint64_t* __restrict__ step,
                                                       int dimi, int advance) {
  __shared__ double red[MD_THREADS];
  const int64_t rep = blockIdx.x, n_rep = gridDim.x;
  const MdParams p = *P;
  const uint64_t n = step[rep];
  const uint64_t done = n - p.run_start;  // steps of this run taken so far
  const bool pending = done != 0;         // the last of them still needs its second half-kick
  const bool sample = pending && p.stride > 0 && done % (uint64_t)p.stride == 0;
  const int64_t frame = sample ? (int64_t)(done / (uint64_t)p.stride) - 1 : 0;
  double* r = R + rep * dimi;
  double* v = V + rep * dimi;
  const double* f = F + rep * dimi;
  const int64_t fo = (frame * n_rep + rep) * dimi;
  double ke = 0.0;
  const int n_pairs = (dimi + 1) / 2;
  for (int j = threadIdx.x; j < n_pairs; j += MD_THREADS) {
    double xi[2] = {0.0, 0.0};
    if (advance && p.use_O) {
      uint32_t c[4] = {(uint32_t)j, (uint32_t)rep, (uint32_t)n, (uint32_t)(n >> 32)};
      philox4x32_10(c, p.key[0], p.key[1]);
      const double ua = uniform53(c[0], c[1]), ub = uniform53(c[2], c[3]);
      const double rad = sqrt(-2.0 * log(ua));
      double sn, cs;
      sincos(2.0 * M_PI * ub, &sn, &cs);
      xi[0] = rad * cs;
      xi[1] = rad * sn;
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = 2 * j + q;
      if (i >= dimi) break;
      double vi = v[i], ri = r[i];
      const double kick = __dmul_rn(p.h, __dmul_rn(f[i], s[i]));
      if (pending) {
        vi = __dadd_rn(vi, kick);
        if (sample) {
          if (p.R_f) p.R_f[fo + i] = ri;
          if (p.V_f) p.V_f[fo + i] = vi;
          ke = __dadd_rn(ke, __ddiv_rn(__dmul_rn(vi, vi), s[i]));
        }
      }
      if (advance) {
        vi = __dadd_rn(vi, kick);
        ri = __dadd_rn(ri, __dmul_rn(p.h, vi));
        if (p.use_O) vi = __dadd_rn(__dmul_rn(p.c1, vi), __dmul_rn(sigma[i], xi[q]));
        ri = __dadd_rn(ri, __dmul_rn(p.h, vi));
        r[i] = ri;
      }
      v[i] = vi;
    }
  }
  if (sample) {  // fixed-order tree: the same sum on every run
    red[threadIdx.x] = ke;
    __syncthreads();
    for (int w = MD_THREADS / 2; w > 0; w >>= 1) {
      if ((int)threadIdx.x < w) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + w]);
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      if (p.Ek_f) p.Ek_f[frame * n_rep + rep] = 0.5 * red[0];
      if (p.Ep_f) p.Ep_f[frame * n_rep + rep] = E[rep];
    }
  }
  __syncthreads();  // every thread has read the counter
  if (advance && threadIdx.x == 0) step[rep] = n + 1;
}

}  // namespace

int launch_md_step(const MdParams* P, const double* s, const double* sigma, double* R, double* V, const double* F,
                   const double* E, uint64_t* step, int64_t n_rep, int dimi, int advance, cudaStream_t st) {
  k_md_step<<<(unsigned)n_rep, MD_THREADS, 0, st>>>(P, s, sigma, R, V, F, E, step, dimi, advance);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

}  // namespace sgdml
