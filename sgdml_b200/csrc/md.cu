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

// ---------------------------------------------------------------------------------- geometry optimisation
// The FIRE and L-BFGS steps of sgdml_b200_relax_* (driver: relax_impl in predict.cu); the exact sums and updates are
// in md.cuh.  Every thread holds the replica's RelaxState and every CTA-wide sum, so branches on them are uniform;
// thread 0 writes the state back at the end.  Each thread updates only its own coordinates, except where the per-atom
// maximum reads three of them (a barrier precedes it).

constexpr double FIRE_FINC = 1.1, FIRE_FDEC = 0.5, FIRE_ALPHA0 = 0.1, FIRE_FALPHA = 0.99;
constexpr int FIRE_NMIN = 5;

// the maximum over the CTA, NaN if any thread holds NaN (max is exact: the order does not matter)
__device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }

__device__ __forceinline__ double block_max(double x, double* red) {
  red[threadIdx.x] = x;
  __syncthreads();
  for (int w = MD_THREADS / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] = nan_max(red[threadIdx.x], red[threadIdx.x + w]);
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// max over atoms of |x_a|^2 = (x_a0^2 + x_a1^2) + x_a2^2 of one replica's (3N) vector
__device__ __forceinline__ double atom_max2(const double* x, int dimi, double* red) {
  double m = 0.0;
  for (int a = threadIdx.x; 3 * a < dimi; a += MD_THREADS) {
    const double* xa = x + 3 * a;
    m = nan_max(m, __dadd_rn(__dadd_rn(__dmul_rn(xa[0], xa[0]), __dmul_rn(xa[1], xa[1])), __dmul_rn(xa[2], xa[2])));
  }
  return block_max(m, red);
}

// the convergence test on F at the current positions; true: the replica is frozen (now or earlier)
__device__ __forceinline__ bool relax_test(RelaxState& z, const double* f, int dimi, double fmax2, double* red) {
  if (z.conv) return true;
  z.fmax2 = atom_max2(f, dimi, red);
  z.conv = z.fmax2 < fmax2 ? 1 : 0;
  return z.conv != 0;
}

__device__ __forceinline__ void relax_store(RelaxState* st, const RelaxState& z) {
  __syncthreads();  // every thread has read the state
  if (threadIdx.x == 0) *st = z;
}

__global__ void __launch_bounds__(MD_THREADS) k_fire_step(const RelaxParams* __restrict__ P, RelaxState* st,
                                                         double* __restrict__ R, double* __restrict__ V,
                                                         const double* __restrict__ F, int dimi, int advance) {
  __shared__ double red[MD_THREADS];
  const int64_t rep = blockIdx.x;
  const RelaxParams p = *P;
  RelaxState z = st[rep];
  double* r = R + rep * dimi;
  double* v = V + rep * dimi;
  const double* f = F + rep * dimi;
  if (relax_test(z, f, dimi, p.fmax2, red) || !advance) return relax_store(st + rep, z);

  if (z.n_steps == 0) {  // ASE's first step: no mixing, dt kept
    z.dt = p.dt0;
    z.alpha = FIRE_ALPHA0;
    z.n_pos = 0;
  } else {
    double fv = 0.0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) fv = __dadd_rn(fv, __dmul_rn(f[i], v[i]));
    fv = block_sum(fv, red);
    if (fv > 0.0) {
      double vv = 0.0, ff = 0.0;
      for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
        vv = __dadd_rn(vv, __dmul_rn(v[i], v[i]));
        ff = __dadd_rn(ff, __dmul_rn(f[i], f[i]));
      }
      vv = block_sum(vv, red);
      ff = block_sum(ff, red);
      const double c = __dmul_rn(z.alpha, __ddiv_rn(sqrt(vv), sqrt(ff)));
      const double om = __dsub_rn(1.0, z.alpha);
      for (int i = threadIdx.x; i < dimi; i += MD_THREADS) v[i] = __dadd_rn(__dmul_rn(om, v[i]), __dmul_rn(c, f[i]));
      if (z.n_pos > FIRE_NMIN) {
        z.dt = fmin(__dmul_rn(z.dt, FIRE_FINC), p.dtmax);
        z.alpha = __dmul_rn(z.alpha, FIRE_FALPHA);
      }
      ++z.n_pos;
    } else {
      for (int i = threadIdx.x; i < dimi; i += MD_THREADS) v[i] = 0.0;
      z.alpha = FIRE_ALPHA0;
      z.dt = __dmul_rn(z.dt, FIRE_FDEC);
      z.n_pos = 0;
    }
  }
  double nn = 0.0;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    const double vi = __dadd_rn(v[i], __dmul_rn(z.dt, f[i]));
    v[i] = vi;
    const double dr = __dmul_rn(z.dt, vi);
    nn = __dadd_rn(nn, __dmul_rn(dr, dr));
  }
  const double nrm = sqrt(block_sum(nn, red));
  const bool cap = nrm > p.maxstep;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    double dr = __dmul_rn(z.dt, v[i]);
    if (cap) dr = __ddiv_rn(__dmul_rn(p.maxstep, dr), nrm);
    r[i] = __dadd_rn(r[i], dr);
  }
  ++z.n_steps;
  relax_store(st + rep, z);
}

__global__ void __launch_bounds__(MD_THREADS) k_lbfgs_step(const RelaxParams* __restrict__ P, RelaxState* st,
                                                          double* __restrict__ R, double* __restrict__ D,
                                                          const double* __restrict__ F,
                                                          const double* __restrict__ E, int dimi, int advance) {
  __shared__ double red[MD_THREADS];
  __shared__ double sa[LBFGS_MAX_MEMORY];  // a_k of the first loop, k = 0 the newest pair
  const int64_t rep = blockIdx.x;
  const RelaxParams p = *P;
  RelaxState z = st[rep];
  double* r = R + rep * dimi;
  double* d = D + rep * dimi;
  const double* f = F + rep * dimi;
  if (relax_test(z, f, dimi, p.fmax2, red) || !advance) return relax_store(st + rep, z);

  const int m = p.memory;
  double* S = p.S + rep * p.m_cap * dimi;
  double* Y = p.Y + rep * p.m_cap * dimi;
  double* rho = p.rho + rep * p.m_cap;
  double* rp = p.r_prev + rep * dimi;
  double* gp = p.g_prev + rep * dimi;
  const double e = E[rep];
  if (z.n_steps != 0) {
    // the new pair goes into the slot after the newest; if it is rejected the history is cleared anyway
    const int slot = (z.head + 1) % m;
    double* sk = S + (int64_t)slot * dimi;
    double* yk = Y + (int64_t)slot * dimi;
    double sy = 0.0, yy = 0.0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
      const double si = __dsub_rn(r[i], rp[i]), yi = __dsub_rn(-f[i], gp[i]);
      sk[i] = si;
      yk[i] = yi;
      sy = __dadd_rn(sy, __dmul_rn(si, yi));
      yy = __dadd_rn(yy, __dmul_rn(yi, yi));
    }
    sy = block_sum(sy, red);
    yy = block_sum(yy, red);
    if (sy > 0.0) {
      z.head = slot;
      z.n_hist = min(z.n_hist + 1, m);
      z.gamma = __ddiv_rn(sy, yy);
      if (threadIdx.x == 0) rho[slot] = __ddiv_rn(1.0, sy);
    } else {
      z.n_hist = 0;
    }
    if (e > z.E_prev) z.n_hist = 0;
    __syncthreads();  // rho[slot] is stored before any thread reads it
  }
  // two-loop recursion on d, which holds q, then z, then the direction
  const int nh = z.n_hist;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) d[i] = -f[i];
  for (int k = 0; k < nh; ++k) {
    const int sl = (z.head - k + m) % m;
    const double* sk = S + (int64_t)sl * dimi;
    const double* yk = Y + (int64_t)sl * dimi;
    double t = 0.0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) t = __dadd_rn(t, __dmul_rn(sk[i], d[i]));
    t = block_sum(t, red);  // a statement of its own: rho[sl] is read after its barriers
    const double a = __dmul_rn(rho[sl], t);
    if (threadIdx.x == 0) sa[k] = a;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) d[i] = __dsub_rn(d[i], __dmul_rn(a, yk[i]));
  }
  const double gam = nh > 0 ? z.gamma : p.h0;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) d[i] = __dmul_rn(gam, d[i]);
  for (int k = nh - 1; k >= 0; --k) {
    const int sl = (z.head - k + m) % m;
    const double* sk = S + (int64_t)sl * dimi;
    const double* yk = Y + (int64_t)sl * dimi;
    double t = 0.0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) t = __dadd_rn(t, __dmul_rn(yk[i], d[i]));
    t = block_sum(t, red);
    const double b = __dmul_rn(rho[sl], t);
    const double c = __dsub_rn(sa[k], b);
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) d[i] = __dadd_rn(d[i], __dmul_rn(sk[i], c));
  }
  double dg = 0.0;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    const double di = -d[i];
    d[i] = di;
    dg = __dadd_rn(dg, __dmul_rn(di, -f[i]));
  }
  dg = block_sum(dg, red);
  if (!(dg < 0.0)) {  // not a descent direction: steepest descent from a fresh history
    z.n_hist = 0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) d[i] = __dmul_rn(p.h0, f[i]);
  }
  __syncthreads();  // d is complete: the per-atom maximum reads other threads' coordinates
  const double L = sqrt(atom_max2(d, dimi, red));
  const bool cap = L > p.maxstep;
  const double sc = __ddiv_rn(p.maxstep, L);
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    double di = d[i];
    if (cap) di = __dmul_rn(di, sc);
    const double ri = r[i];
    rp[i] = ri;
    gp[i] = -f[i];
    r[i] = __dadd_rn(ri, di);
  }
  z.E_prev = e;
  ++z.n_steps;
  relax_store(st + rep, z);
}

__global__ void __launch_bounds__(MD_THREADS) k_relax_count(const RelaxState* __restrict__ st, int64_t n_rep,
                                                           int* n_active) {
  __shared__ int red[MD_THREADS];
  int c = 0;
  for (int64_t r = threadIdx.x; r < n_rep; r += MD_THREADS) c += st[r].conv == 0;
  red[threadIdx.x] = c;
  __syncthreads();
  for (int w = MD_THREADS / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *n_active = red[0];
}

__global__ void k_relax_report(const RelaxState* __restrict__ st, int64_t n_rep, int64_t* n_steps, int* conv,
                               double* fmax) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rep) return;
  if (n_steps) n_steps[r] = st[r].n_steps;
  if (conv) conv[r] = st[r].conv;
  if (fmax) fmax[r] = sqrt(st[r].fmax2);
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

int launch_fire_step(const RelaxParams* P, RelaxState* st, double* R, double* V, const double* F, int64_t n_rep,
                     int dimi, int advance, cudaStream_t s) {
  k_fire_step<<<(unsigned)n_rep, MD_THREADS, 0, s>>>(P, st, R, V, F, dimi, advance);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

int launch_lbfgs_step(const RelaxParams* P, RelaxState* st, double* R, double* D, const double* F, const double* E,
                      int64_t n_rep, int dimi, int advance, cudaStream_t s) {
  k_lbfgs_step<<<(unsigned)n_rep, MD_THREADS, 0, s>>>(P, st, R, D, F, E, dimi, advance);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

int launch_relax_count(const RelaxState* st, int64_t n_rep, int* n_active, cudaStream_t s) {
  k_relax_count<<<1, MD_THREADS, 0, s>>>(st, n_rep, n_active);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

int launch_relax_report(const RelaxState* st, int64_t n_rep, int64_t* n_steps, int* conv, double* fmax,
                        cudaStream_t s) {
  k_relax_report<<<(unsigned)((n_rep + 255) / 256), 256, 0, s>>>(st, n_rep, n_steps, conv, fmax);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

}  // namespace sgdml
