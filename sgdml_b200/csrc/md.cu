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

// k_md_step's fixed-order tree over the CTA; every thread gets the sum
__device__ __forceinline__ double block_sum(double x, double* red) {
  red[threadIdx.x] = x;
  __syncthreads();
  for (int w = MD_THREADS / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + w]);
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();  // red is free again
  return r;
}

// The ring-polymer step (launch_pimd_step in md.cuh).  Each tile holds TI coordinates of all nb beads in shared memory
// (TI = PIMD_TILE / nb rounded down to even, so a Philox coordinate pair never straddles two tiles); every thread owns
// at most PIMD_TILE / MD_THREADS = 4 elements of it in each transform, whatever nb.  Sums over beads and modes run in
// index order from the first product, and every update rounds as written.  At nb = 1 (C = 1, cos = 1, sin/w = h,
// -w sin = 0) each update is k_md_step's, bit for bit.
__global__ void __launch_bounds__(MD_THREADS) k_pimd_step(const PimdParams* __restrict__ P,
                                                         const double* __restrict__ tab, const double* __restrict__ s,
                                                         const double* __restrict__ sigma, double* __restrict__ R,
                                                         double* __restrict__ V, const double* __restrict__ F,
                                                         const double* __restrict__ E, uint64_t* __restrict__ step,
                                                         int dimi, int nb, int advance) {
  __shared__ double sC[PIMD_MAX_BEADS * PIMD_MAX_BEADS];
  __shared__ double sM[4 * PIMD_MAX_BEADS];  // cos, sin/w, -w sin, c1 per mode
  __shared__ double sX[PIMD_TILE], sU[PIMD_TILE];
  __shared__ double red[MD_THREADS];
  constexpr int PER_THREAD = PIMD_TILE / MD_THREADS;
  const int tid = threadIdx.x;
  const int64_t poly = blockIdx.x, n_poly = gridDim.x;
  const int64_t n_rep = n_poly * nb, rep0 = poly * nb;
  const PimdParams p = *P;
  const uint64_t n = step[rep0];
  const uint64_t done = n - p.run_start;
  const bool pending = done != 0;
  const bool sample = pending && p.stride > 0 && done % (uint64_t)p.stride == 0;
  const int64_t frame = sample ? (int64_t)(done / (uint64_t)p.stride) - 1 : 0;
  const int n_pairs = (dimi + 1) / 2;

  if (sample) {
    // per bead: R, full-step V and E_kin exactly as k_md_step writes them
    for (int j = 0; j < nb; ++j) {
      const int64_t rep = rep0 + j;
      const double *r = R + rep * dimi, *v = V + rep * dimi, *f = F + rep * dimi;
      const int64_t fo = (frame * n_rep + rep) * dimi;
      double ke = 0.0;
      for (int jp = tid; jp < n_pairs; jp += MD_THREADS) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int i = 2 * jp + q;
          if (i >= dimi) break;
          const double vi = __dadd_rn(v[i], __dmul_rn(p.h, __dmul_rn(f[i], s[i])));
          if (p.R_f) p.R_f[fo + i] = r[i];
          if (p.V_f) p.V_f[fo + i] = vi;
          ke = __dadd_rn(ke, __ddiv_rn(__dmul_rn(vi, vi), s[i]));
        }
      }
      ke = block_sum(ke, red);
      if (tid == 0) {
        if (p.Ek_f) p.Ek_f[frame * n_rep + rep] = 0.5 * ke;
        if (p.Ep_f) p.Ep_f[frame * n_rep + rep] = E[rep];
      }
    }
    // per polymer: the spring sum (x_j - x_j+1)^2 / s and the centroid virial (x_j - xbar) F_j, each thread over its
    // coordinates i = tid, tid + MD_THREADS, ..., beads in order, then the tree
    const double* x = R + rep0 * dimi;
    const double* fx = F + rep0 * dimi;
    double spr = 0.0, vir = 0.0;
    for (int i = tid; i < dimi; i += MD_THREADS) {
      double xb = x[i];
      for (int j = 1; j < nb; ++j) xb = __dadd_rn(xb, x[(int64_t)j * dimi + i]);
      xb = __ddiv_rn(xb, (double)nb);
      double si = 0.0, vi = 0.0;
      for (int j = 0; j < nb; ++j) {
        const double xj = x[(int64_t)j * dimi + i];
        const double d = __dsub_rn(xj, x[(int64_t)(j + 1 == nb ? 0 : j + 1) * dimi + i]);
        si = __dadd_rn(si, __dmul_rn(d, d));
        vi = __dadd_rn(vi, __dmul_rn(__dsub_rn(xj, xb), fx[(int64_t)j * dimi + i]));
      }
      spr = __dadd_rn(spr, __ddiv_rn(si, s[i]));
      vir = __dadd_rn(vir, vi);
    }
    spr = block_sum(spr, red);
    vir = block_sum(vir, red);
    if (tid == 0) {
      if (p.Kp_f) p.Kp_f[frame * n_poly + poly] = __dsub_rn(p.kprim0, __dmul_rn(p.kspring, spr));
      if (p.Kcv_f) p.Kcv_f[frame * n_poly + poly] = __dsub_rn(p.kcv0, __dmul_rn(p.kvir, vir));
    }
  }
  __syncthreads();  // the frame has read R and V before they change

  double* r0 = R + rep0 * dimi;
  double* v0 = V + rep0 * dimi;
  const double* f0 = F + rep0 * dimi;
  if (!advance) {  // complete the last step of a run
    if (pending)
      for (int64_t e = tid; e < (int64_t)nb * dimi; e += MD_THREADS) {
        const int i = (int)(e % dimi);
        v0[e] = __dadd_rn(v0[e], __dmul_rn(p.h, __dmul_rn(f0[e], s[i])));
      }
    return;
  }

  for (int e = tid; e < nb * nb; e += MD_THREADS) sC[e] = tab[e];
  for (int e = tid; e < 4 * nb; e += MD_THREADS) sM[e] = tab[nb * nb + e];
  const double *m_cos = sM, *m_sow = sM + nb, *m_msin = sM + 2 * nb, *m_c1 = sM + 3 * nb;
  const int TI = (PIMD_TILE / nb) & ~1;
  const int ne = nb * TI;
  for (int i0 = 0; i0 < dimi; i0 += TI) {
    const int w = min(TI, dimi - i0);
    // B (after the pending half-kick) into the tile: element e = (bead e / TI, coordinate i0 + e % TI)
    for (int e = tid; e < ne; e += MD_THREADS) {
      const int j = e / TI, c = e % TI;
      if (c >= w) continue;
      const int64_t o = (int64_t)j * dimi + i0 + c;
      double vi = v0[o];
      const double kick = __dmul_rn(p.h, __dmul_rn(f0[o], s[i0 + c]));
      if (pending) vi = __dadd_rn(vi, kick);
      sX[e] = r0[o];
      sU[e] = __dadd_rn(vi, kick);
    }
    __syncthreads();
    // to normal modes: q_k = sum_j C_jk x_j, u_k likewise
    double q[PER_THREAD], u[PER_THREAD];
#pragma unroll
    for (int m = 0; m < PER_THREAD; ++m) {
      const int e = tid + m * MD_THREADS, k = e / TI, c = e % TI;
      if (e < ne && c < w) {
        double a = __dmul_rn(sC[k], sX[c]), b = __dmul_rn(sC[k], sU[c]);
        for (int j = 1; j < nb; ++j) {
          const double cjk = sC[j * nb + k];
          a = __dadd_rn(a, __dmul_rn(cjk, sX[j * TI + c]));
          b = __dadd_rn(b, __dmul_rn(cjk, sU[j * TI + c]));
        }
        q[m] = a;
        u[m] = b;
      }
    }
    __syncthreads();
#pragma unroll
    for (int m = 0; m < PER_THREAD; ++m) {
      const int e = tid + m * MD_THREADS;
      if (e < ne && e % TI < w) {
        sX[e] = q[m];
        sU[e] = u[m];
      }
    }
    __syncthreads();
    // A, O, A per (mode, coordinate pair); the pair's normals are those of replica rep0 + k
    const int tp = TI / 2;
    for (int t = tid; t < nb * tp; t += MD_THREADS) {
      const int k = t / tp, c = 2 * (t % tp);
      if (c >= w) continue;
      double xi[2] = {0.0, 0.0};
      if (p.use_O) {
        const int64_t rep = rep0 + k;
        uint32_t ct[4] = {(uint32_t)((i0 + c) / 2), (uint32_t)rep, (uint32_t)n, (uint32_t)(n >> 32)};
        philox4x32_10(ct, p.key[0], p.key[1]);
        const double ua = uniform53(ct[0], ct[1]), ub = uniform53(ct[2], ct[3]);
        const double rad = sqrt(-2.0 * log(ua));
        double sn, cs;
        sincos(2.0 * M_PI * ub, &sn, &cs);
        xi[0] = rad * cs;
        xi[1] = rad * sn;
      }
      const double cs = m_cos[k], so = m_sow[k], ms = m_msin[k], c1 = m_c1[k];
#pragma unroll
      for (int qq = 0; qq < 2; ++qq) {
        if (c + qq >= w) break;
        const int e = k * TI + c + qq;
        double x = sX[e], y = sU[e];
        double x1 = __dadd_rn(__dmul_rn(cs, x), __dmul_rn(so, y));
        y = __dadd_rn(__dmul_rn(ms, x), __dmul_rn(cs, y));
        if (p.use_O) y = __dadd_rn(__dmul_rn(c1, y), __dmul_rn(sigma[(int64_t)k * dimi + i0 + c + qq], xi[qq]));
        x = __dadd_rn(__dmul_rn(cs, x1), __dmul_rn(so, y));
        y = __dadd_rn(__dmul_rn(ms, x1), __dmul_rn(cs, y));
        sX[e] = x;
        sU[e] = y;
      }
    }
    __syncthreads();
    // back to beads: x_j = sum_k C_jk q_k, straight into the state
#pragma unroll
    for (int m = 0; m < PER_THREAD; ++m) {
      const int e = tid + m * MD_THREADS, j = e / TI, c = e % TI;
      if (e < ne && c < w) {
        double a = __dmul_rn(sC[j * nb], sX[c]), b = __dmul_rn(sC[j * nb], sU[c]);
        for (int k = 1; k < nb; ++k) {
          const double cjk = sC[j * nb + k];
          a = __dadd_rn(a, __dmul_rn(cjk, sX[k * TI + c]));
          b = __dadd_rn(b, __dmul_rn(cjk, sU[k * TI + c]));
        }
        const int64_t o = (int64_t)j * dimi + i0 + c;
        r0[o] = a;
        v0[o] = b;
      }
    }
    __syncthreads();  // the next tile overwrites sX, sU
  }
  if (tid < nb) step[rep0 + tid] = n + 1;  // every thread read the counter before the first barrier
}

}  // namespace

int launch_md_step(const MdParams* P, const double* s, const double* sigma, double* R, double* V, const double* F,
                   const double* E, uint64_t* step, int64_t n_rep, int dimi, int advance, cudaStream_t st) {
  k_md_step<<<(unsigned)n_rep, MD_THREADS, 0, st>>>(P, s, sigma, R, V, F, E, step, dimi, advance);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

int launch_pimd_step(const PimdParams* P, const double* tab, const double* s, const double* sigma, double* R, double* V,
                     const double* F, const double* E, uint64_t* step, int64_t n_poly, int dimi, int nb, int advance,
                     cudaStream_t st) {
  if (nb < 1 || nb > PIMD_MAX_BEADS) return fail_arg("launch_pimd_step: n_beads outside [1, PIMD_MAX_BEADS]");
  k_pimd_step<<<(unsigned)n_poly, MD_THREADS, 0, st>>>(P, tab, s, sigma, R, V, F, E, step, dimi, nb, advance);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

}  // namespace sgdml
