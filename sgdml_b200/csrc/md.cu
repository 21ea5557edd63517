// Molecular dynamics, replica exchange, metadynamics, umbrella sampling, path-integral MD, geometry optimisation and
// saddle searches on the device: the integrator, exchange, bias, optimiser and dimer kernels (contract in md.cuh), then
// the driver of sgdml_b200_md_*, sgdml_b200_remd_run, sgdml_b200_npt_*, sgdml_b200_metad_*, sgdml_b200_umbrella_*
// (but _mbar, in mbar.cu), sgdml_b200_pimd_*, sgdml_b200_relax_*, sgdml_b200_neb_fire and sgdml_b200_dimer_fire, which
// evaluates forces through the predictor interface of predict.cuh.
//
// The BAOAB Langevin integrator step of sgdml_b200_md_run.
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
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstring>
#include <functional>
#include <initializer_list>
#include <vector>

#include "common.cuh"
#include "md.cuh"
#include "predict.cuh"

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

// the normals of coordinate pair j of replica rep at step n: Philox4x32-10 under key (k0, k1), then Box-Muller
__device__ __forceinline__ void normal_pair(double xi[2], uint32_t j, uint32_t rep, uint64_t n, uint32_t k0,
                                            uint32_t k1) {
  uint32_t c[4] = {j, rep, (uint32_t)n, (uint32_t)(n >> 32)};
  philox4x32_10(c, k0, k1);
  const double ua = uniform53(c[0], c[1]), ub = uniform53(c[2], c[3]);
  const double rad = sqrt(-2.0 * log(ua));
  double sn, cs;
  sincos(2.0 * M_PI * ub, &sn, &cs);
  xi[0] = rad * cs;
  xi[1] = rad * sn;
}

// The fixed-order tree over the CTA (the same result on every run): red[t] = op(red[t], red[t + w]) for
// w = MD_THREADS / 2, ..., 1, each level after a barrier; returns red[0]
template <class T, class Op>
__device__ __forceinline__ T block_tree(T x, T* red, Op op) {
  red[threadIdx.x] = x;
  __syncthreads();
  for (int w = MD_THREADS / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] = op(red[threadIdx.x], red[threadIdx.x + w]);
    __syncthreads();
  }
  return red[0];
}

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }

// B, A, O, A of coordinate i from (ri, vi), vi after the pending half-kick: the one copy of the update of k_md_step and
// k_npt_step (kick = h (F s), sg the replica's sigma row, xi the coordinate's normal)
__device__ __forceinline__ void baoab(const MdParams& p, double kick, const double* __restrict__ sg, int i, double xi,
                                      double& ri, double& vi) {
  vi = __dadd_rn(vi, kick);
  ri = __dadd_rn(ri, __dmul_rn(p.h, vi));
  if (p.use_O) vi = __dadd_rn(__dmul_rn(p.c1, vi), __dmul_rn(sg[i], xi));
  ri = __dadd_rn(ri, __dmul_rn(p.h, vi));
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
  const double* sg = sigma + (rep % p.n_temps) * dimi;
  const int64_t fo = (frame * n_rep + rep) * dimi;
  double ke = 0.0;
  const int n_pairs = (dimi + 1) / 2;
  for (int j = threadIdx.x; j < n_pairs; j += MD_THREADS) {
    double xi[2] = {0.0, 0.0};
    if (advance && p.use_O) normal_pair(xi, (uint32_t)j, (uint32_t)rep, n, p.key[0], p.key[1]);
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
        baoab(p, kick, sg, i, xi[q], ri, vi);
        r[i] = ri;
      }
      v[i] = vi;
    }
  }
  if (sample) {
    ke = block_tree(ke, red, dadd);
    if (threadIdx.x == 0) {
      if (p.Ek_f) p.Ek_f[frame * n_rep + rep] = 0.5 * ke;
      if (p.Ep_f) p.Ep_f[frame * n_rep + rep] = E[rep];
    }
  }
  __syncthreads();  // every thread has read the counter
  if (advance && threadIdx.x == 0) step[rep] = n + 1;
}

// The NPT step of sgdml_b200_npt_run (contract in md.cuh): k_md_step's pending half-kick and frame, the instantaneous
// pressure, the barostat's volume move, then k_md_step's B, A, O, A followed by the isotropic rescaling.  The first
// pass leaves the full-step velocities in V; each thread reads back only its own coordinates in the second.
__global__ void __launch_bounds__(MD_THREADS) k_npt_step(const MdParams* __restrict__ P, const NptParams* __restrict__ Q,
                                                        const double* __restrict__ s, const double* __restrict__ sigma,
                                                        double* __restrict__ R, double* __restrict__ V,
                                                        const double* __restrict__ F, const double* __restrict__ E,
                                                        const double* __restrict__ W, NptCell* __restrict__ cell,
                                                        Lattice* __restrict__ lat, uint64_t* __restrict__ step,
                                                        int dimi, int advance) {
  __shared__ double red[MD_THREADS];
  const int64_t rep = blockIdx.x, n_rep = gridDim.x;
  const MdParams p = *P;
  const NptParams q = *Q;
  const uint64_t n = step[rep];
  const uint64_t done = n - p.run_start;
  const bool pending = done != 0;
  const bool sample = pending && p.stride > 0 && done % (uint64_t)p.stride == 0;
  const int64_t frame = sample ? (int64_t)(done / (uint64_t)p.stride) - 1 : 0;
  double* r = R + rep * dimi;
  double* v = V + rep * dimi;
  const double* f = F + rep * dimi;
  const int64_t fo = (frame * n_rep + rep) * dimi;
  const int n_pairs = (dimi + 1) / 2;
  double ke = 0.0;
  for (int j = threadIdx.x; j < n_pairs; j += MD_THREADS) {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int i = 2 * j + c;
      if (i >= dimi) break;
      double vi = v[i];
      if (pending) vi = __dadd_rn(vi, __dmul_rn(p.h, __dmul_rn(f[i], s[i])));
      if (sample) {
        if (p.R_f) p.R_f[fo + i] = r[i];
        if (p.V_f) p.V_f[fo + i] = vi;
      }
      ke = __dadd_rn(ke, __ddiv_rn(__dmul_rn(vi, vi), s[i]));
      v[i] = vi;
    }
  }
  const double K = 0.5 * block_tree(ke, red, dadd);
  NptCell* cl = cell + rep;
  const double eps0 = cl->eps;
  const double* w = W + rep * 9;
  const double vol = __dmul_rn(cl->V0, exp(eps0));
  const double pint = __ddiv_rn(__dadd_rn(__dmul_rn(2.0, K), __dadd_rn(__dadd_rn(w[0], w[4]), w[8])),
                                __dmul_rn(3.0, vol));
  if (sample) {
    const int64_t fr = frame * n_rep + rep;
    if (threadIdx.x == 0) {
      if (p.Ek_f) p.Ek_f[fr] = K;
      if (p.Ep_f) p.Ep_f[fr] = E[rep];
      if (q.P_f) q.P_f[fr] = pint;
    }
    if (q.cell_f && threadIdx.x < 9) q.cell_f[fr * 9 + threadIdx.x] = lat[rep].vec[threadIdx.x];
  }
  if (advance) {
    double de = __dmul_rn(-q.c_a, __dsub_rn(q.P0, pint));
    if (q.c_b != 0.0) {
      double eta[2];
      normal_pair(eta, 0xFFFFFFFFu, (uint32_t)rep, n, p.key[0], p.key[1]);
      de = __dadd_rn(de, __dmul_rn(sqrt(__ddiv_rn(q.c_b, vol)), eta[0]));
    }
    const double mu = exp(__ddiv_rn(de, 3.0));
    for (int j = threadIdx.x; j < n_pairs; j += MD_THREADS) {
      double xi[2] = {0.0, 0.0};
      if (p.use_O) normal_pair(xi, (uint32_t)j, (uint32_t)rep, n, p.key[0], p.key[1]);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int i = 2 * j + c;
        if (i >= dimi) break;
        double vi = v[i], ri = r[i];
        baoab(p, __dmul_rn(p.h, __dmul_rn(f[i], s[i])), sigma, i, xi[c], ri, vi);
        r[i] = __dmul_rn(ri, mu);
        v[i] = __ddiv_rn(vi, mu);
      }
    }
    const double eps = __dadd_rn(eps0, de);
    const double a = exp(__ddiv_rn(eps, 3.0));
    if (threadIdx.x < 9) {
      lat[rep].vec[threadIdx.x] = __dmul_rn(a, cl->L0[threadIdx.x]);
      lat[rep].inv[threadIdx.x] = __ddiv_rn(cl->L0inv[threadIdx.x], a);
    }
    __syncthreads();  // every thread has read the counter and the cell
    if (threadIdx.x == 0) {
      cl->eps = eps;
      step[rep] = n + 1;
    }
  }
}

// The replica exchange of sgdml_b200_remd_run (contract in md.cuh).  Thread t decides the pairs t, t + MD_THREADS, ...
// of its ladder and swaps their energies, walker labels and counts; then every thread swaps its coordinates of the
// accepted pairs' R, V and F rows.  The pairs are disjoint, so no two threads touch the same entry.
__global__ void __launch_bounds__(MD_THREADS) k_remd_exchange(const RemdParams* __restrict__ X,
                                                             const MdParams* __restrict__ P,
                                                             const double* __restrict__ s, double* __restrict__ R,
                                                             double* __restrict__ V, double* __restrict__ F,
                                                             double* __restrict__ E, int* __restrict__ walker,
                                                             const uint64_t* __restrict__ step, int dimi) {
  __shared__ int acc[MD_THREADS];
  const RemdParams x = *X;
  const int nt = x.n_temps;
  const int64_t lad = blockIdx.x, n_rep = (int64_t)gridDim.x * nt, base = lad * nt;
  const uint64_t c = step[base];
  const uint64_t done = c - x.run_start;
  const bool sample = done != 0 && x.stride > 0 && done % (uint64_t)x.stride == 0 && x.W_f != nullptr;
  const bool exchange = x.every > 0 && done != 0 && c % (uint64_t)x.every == 0;
  if (!exchange && !sample) return;
  if (exchange) {
    const double h = P->h;
    const int par = (int)((c / (uint64_t)x.every) & 1);
    const int n_pairs = (nt - par) / 2;  // k = 2 j + par for j < n_pairs
    for (int j0 = 0; j0 < n_pairs; j0 += MD_THREADS) {
      const int j = j0 + (int)threadIdx.x;
      if (j < n_pairs) {
        const int k = 2 * j + par;
        const int64_t a = base + k, b = a + 1;
        const double ea = E[a], eb = E[b];
        const double d = __dmul_rn(__dsub_rn(x.beta[k], x.beta[k + 1]), __dsub_rn(ea, eb));
        bool ok = d >= 0.0;
        if (!ok) {
          uint32_t ct[4] = {0x80000000u | (uint32_t)k, (uint32_t)lad, (uint32_t)c, (uint32_t)(c >> 32)};
          philox4x32_10(ct, x.key[0], x.key[1]);
          ok = uniform53(ct[0], ct[1]) < exp(d);
        }
        acc[threadIdx.x] = ok ? 1 : 0;
        const int64_t q = lad * (nt - 1) + k;
        x.n_att[q] += 1;
        if (ok) {
          x.n_acc[q] += 1;
          E[a] = eb;
          E[b] = ea;
          const int w = walker[a];
          walker[a] = walker[b];
          walker[b] = w;
        }
      }
      __syncthreads();  // the decisions are in acc
      const int nj = min(MD_THREADS, n_pairs - j0);
      for (int t = 0; t < nj; ++t) {
        if (!acc[t]) continue;
        const int k = 2 * (j0 + t) + par;
        const int64_t o = (base + k) * dimi;
        double *ra = R + o, *va = V + o, *fa = F + o;
        double *rb = ra + dimi, *vb = va + dimi, *fb = fa + dimi;
        const double lu = x.lam_up[k], ld = x.lam_dn[k];
        for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
          const double ka = __dmul_rn(h, __dmul_rn(fa[i], s[i])), kb = __dmul_rn(h, __dmul_rn(fb[i], s[i]));
          const double wa = __dadd_rn(va[i], ka), wb = __dadd_rn(vb[i], kb);
          va[i] = __dsub_rn(__dmul_rn(ld, wb), kb);  // configuration b moves down to slot k
          vb[i] = __dsub_rn(__dmul_rn(lu, wa), ka);  // configuration a moves up to slot k + 1
          const double r = ra[i], f = fa[i];
          ra[i] = rb[i];
          rb[i] = r;
          fa[i] = fb[i];
          fb[i] = f;
        }
      }
      __syncthreads();  // acc is free again, and the walker labels are swapped
    }
  }
  if (sample) {
    const int64_t frame = (int64_t)(done / (uint64_t)x.stride) - 1;
    for (int k = threadIdx.x; k < nt; k += MD_THREADS) x.W_f[frame * n_rep + base + k] = walker[base + k];
  }
}

// sets the walker labels of the n_rep slots to the identity
__global__ void k_remd_identity(int* walker, int64_t n_rep) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n_rep) walker[r] = (int)r;
}

// k_md_step's sum over the CTA; every thread gets it
__device__ __forceinline__ double block_sum(double x, double* red) {
  const double r = block_tree(x, red, dadd);
  __syncthreads();  // red is free again
  return r;
}

// The ring-polymer step (contract in md.cuh).  Each tile holds TI coordinates of all nb beads in shared memory
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
      if (p.use_O) normal_pair(xi, (uint32_t)((i0 + c) / 2), (uint32_t)(rep0 + k), n, p.key[0], p.key[1]);
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
// The FIRE and L-BFGS steps of sgdml_b200_relax_* (driver: relax_impl below); the exact sums and updates are in
// md.cuh.  Every thread holds the replica's RelaxState and every CTA-wide sum, so branches on them are uniform;
// thread 0 writes the state back at the end.  Each thread updates only its own coordinates, except where the per-atom
// maximum reads three of them (a barrier precedes it).

constexpr double FIRE_FINC = 1.1, FIRE_FDEC = 0.5, FIRE_ALPHA0 = 0.1, FIRE_FALPHA = 0.99;
constexpr int FIRE_NMIN = 5;

// the maximum over the CTA, NaN if any thread holds NaN (max is exact: the order does not matter)
__device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }

__device__ __forceinline__ double block_max(double x, double* red) {
  const double r = block_tree(x, red, nan_max);
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

// One FIRE step (md.cuh) of the n coordinates r, v, f after the convergence test: the arithmetic of k_fire_step (n the
// replica's 3N) and of k_neb_fire_step (n a band's (P - 2) 3N).
__device__ __forceinline__ void fire_update(RelaxState& z, double dt0, double dtmax, double maxstep, double* r,
                                            double* v, const double* f, int n, double* red) {
  if (z.n_steps == 0) {  // ASE's first step: no mixing, dt kept
    z.dt = dt0;
    z.alpha = FIRE_ALPHA0;
    z.n_pos = 0;
  } else {
    double fv = 0.0;
    for (int i = threadIdx.x; i < n; i += MD_THREADS) fv = __dadd_rn(fv, __dmul_rn(f[i], v[i]));
    fv = block_sum(fv, red);
    if (fv > 0.0) {
      double vv = 0.0, ff = 0.0;
      for (int i = threadIdx.x; i < n; i += MD_THREADS) {
        vv = __dadd_rn(vv, __dmul_rn(v[i], v[i]));
        ff = __dadd_rn(ff, __dmul_rn(f[i], f[i]));
      }
      vv = block_sum(vv, red);
      ff = block_sum(ff, red);
      const double c = __dmul_rn(z.alpha, __ddiv_rn(sqrt(vv), sqrt(ff)));
      const double om = __dsub_rn(1.0, z.alpha);
      for (int i = threadIdx.x; i < n; i += MD_THREADS) v[i] = __dadd_rn(__dmul_rn(om, v[i]), __dmul_rn(c, f[i]));
      if (z.n_pos > FIRE_NMIN) {
        z.dt = fmin(__dmul_rn(z.dt, FIRE_FINC), dtmax);
        z.alpha = __dmul_rn(z.alpha, FIRE_FALPHA);
      }
      ++z.n_pos;
    } else {
      for (int i = threadIdx.x; i < n; i += MD_THREADS) v[i] = 0.0;
      z.alpha = FIRE_ALPHA0;
      z.dt = __dmul_rn(z.dt, FIRE_FDEC);
      z.n_pos = 0;
    }
  }
  double nn = 0.0;
  for (int i = threadIdx.x; i < n; i += MD_THREADS) {
    const double vi = __dadd_rn(v[i], __dmul_rn(z.dt, f[i]));
    v[i] = vi;
    const double dr = __dmul_rn(z.dt, vi);
    nn = __dadd_rn(nn, __dmul_rn(dr, dr));
  }
  const double nrm = sqrt(block_sum(nn, red));
  const bool cap = nrm > maxstep;
  for (int i = threadIdx.x; i < n; i += MD_THREADS) {
    double dr = __dmul_rn(z.dt, v[i]);
    if (cap) dr = __ddiv_rn(__dmul_rn(maxstep, dr), nrm);
    r[i] = __dadd_rn(r[i], dr);
  }
  ++z.n_steps;
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
  fire_update(z, p.dt0, p.dtmax, p.maxstep, r, v, f, dimi, red);
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

// The NEB force of one interior image (md.cuh).  Each thread keeps its coordinates of tau, then of th, in its own
// entries of Fn before overwriting them with F_neb, so no barrier beyond block_sum's is needed.
__global__ void __launch_bounds__(MD_THREADS) k_neb_force(const NebParams* __restrict__ Q, const double* __restrict__ R,
                                                         const double* __restrict__ F, const double* __restrict__ E,
                                                         double* __restrict__ Fn, int* __restrict__ climb_idx,
                                                         int dimi) {
  __shared__ double red[MD_THREADS];
  const NebParams p = *Q;
  const int ni = p.P - 2;
  const int64_t band = blockIdx.x / ni;
  const int i = (int)(blockIdx.x % ni) + 1;
  const double* eb = E + band * p.P;
  int top = 1;  // the highest interior image, the lowest index on ties
  for (int j = 2; j <= ni; ++j)
    if (eb[j] > eb[top]) top = j;
  if (i == 1 && threadIdx.x == 0) climb_idx[band] = top;

  const int64_t rep = band * p.P + i;
  const double* r = R + rep * dimi;
  const double* f = F + rep * dimi;
  double* fn = Fn + rep * dimi;
  const double e = eb[i], ep = eb[i + 1], em = eb[i - 1];
  const int mode = ep > e && e > em ? 1 : (ep < e && e < em ? 2 : 0);  // 1: tau = t+, 2: tau = t-, 0: the mixture
  const double dp = fabs(__dsub_rn(ep, e)), dm = fabs(__dsub_rn(em, e));
  const double dmax = dp > dm ? dp : dm, dmin = dp > dm ? dm : dp;
  const double wp = ep > em ? dmax : dmin, wm = ep > em ? dmin : dmax;
  double tt = 0.0, pp = 0.0, mm = 0.0;
  for (int c = threadIdx.x; c < dimi; c += MD_THREADS) {
    const double x = r[c];
    const double tp = __dsub_rn(r[c + dimi], x), tm = __dsub_rn(x, r[c - dimi]);
    const double t = mode == 1 ? tp : (mode == 2 ? tm : __dadd_rn(__dmul_rn(tp, wp), __dmul_rn(tm, wm)));
    fn[c] = t;
    tt = __dadd_rn(tt, __dmul_rn(t, t));
    pp = __dadd_rn(pp, __dmul_rn(tp, tp));
    mm = __dadd_rn(mm, __dmul_rn(tm, tm));
  }
  const double nt = sqrt(block_sum(tt, red));
  const double np = sqrt(block_sum(pp, red));
  const double nm = sqrt(block_sum(mm, red));
  double fd = 0.0;
  for (int c = threadIdx.x; c < dimi; c += MD_THREADS) {
    const double th = nt == 0.0 ? 0.0 : __ddiv_rn(fn[c], nt);
    fn[c] = th;
    fd = __dadd_rn(fd, __dmul_rn(f[c], th));
  }
  fd = block_sum(fd, red);
  const bool climbing = p.climb && i == top;
  const double spring = __dmul_rn(p.k, __dsub_rn(np, nm));
  const double fd2 = __dmul_rn(2.0, fd);
  for (int c = threadIdx.x; c < dimi; c += MD_THREADS) {
    const double th = fn[c];
    fn[c] = climbing ? __dsub_rn(f[c], __dmul_rn(fd2, th))
                     : __dadd_rn(__dsub_rn(f[c], __dmul_rn(fd, th)), __dmul_rn(spring, th));
  }
}

// FIRE on one band's interior images with the NEB forces Fn (one RelaxState per band)
__global__ void __launch_bounds__(MD_THREADS) k_neb_fire_step(const NebParams* __restrict__ Q, RelaxState* st,
                                                             double* __restrict__ R, double* __restrict__ V,
                                                             const double* __restrict__ Fn, int dimi, int advance) {
  __shared__ double red[MD_THREADS];
  const int64_t band = blockIdx.x;
  const NebParams p = *Q;
  RelaxState z = st[band];
  // The L-BFGS fields are zero already (the driver zeroes the state and FIRE never writes them).  Storing the constant
  // lets the compiler drop the two loaded values instead of carrying them through the step to relax_store, which
  // otherwise costs 16 bytes of spills.
  z.gamma = z.E_prev = 0.0;
  const int64_t o = (band * p.P + 1) * dimi;  // image 1 of the band: the interior images are contiguous
  const int n = (p.P - 2) * dimi;
  if (relax_test(z, Fn + o, n, p.fmax2, red) || !advance) return relax_store(st + band, z);
  fire_update(z, p.dt0, p.dtmax, p.maxstep, R + o, V + o, Fn + o, n, red);
  relax_store(st + band, z);
}

__global__ void __launch_bounds__(MD_THREADS) k_relax_count(const RelaxState* __restrict__ st, int64_t n_rep,
                                                           int* n_active) {
  __shared__ int red[MD_THREADS];
  int c = 0;
  for (int64_t r = threadIdx.x; r < n_rep; r += MD_THREADS) c += st[r].conv == 0;
  c = block_tree(c, red, [](int a, int b) { return a + b; });
  if (threadIdx.x == 0) *n_active = c;
}

__global__ void k_relax_report(const RelaxState* __restrict__ st, int64_t n_rep, int64_t* n_steps, int* conv,
                               double* fmax) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rep) return;
  if (n_steps) n_steps[r] = st[r].n_steps;
  if (conv) conv[r] = st[r].conv;
  if (fmax) fmax[r] = sqrt(st[r].fmax2);
}

// ---------------------------------------------------------------------------------- metadynamics
// The CVs, the hill sum and the deposit of sgdml_b200_metad_run (contract in md.cuh).  Every operation rounds as
// written there.

__device__ __forceinline__ void sub3(double o[3], const double* a, const double* b) {
  for (int x = 0; x < 3; ++x) o[x] = __dsub_rn(a[x], b[x]);
}
__device__ __forceinline__ double dot3(const double* a, const double* b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}
__device__ __forceinline__ void cross3(double o[3], const double* a, const double* b) {
  o[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  o[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  o[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}

// CV of `type` on atoms at of the replica's positions r: its value, and g (4 x 3) its gradient per atom slot
__device__ void cv_eval(int type, const int* at, const double* r, double* sv, double g[4][3]) {
  for (int p = 0; p < 4; ++p)
    for (int x = 0; x < 3; ++x) g[p][x] = 0.0;
  const double *ri = r + 3 * at[0], *rj = r + 3 * at[1], *rk = r + 3 * at[2], *rl = r + 3 * at[3];
  if (type == CV_DISTANCE) {
    double d[3];
    sub3(d, rj, ri);
    const double s = sqrt(dot3(d, d));
    *sv = s;
    if (s != 0.0)
      for (int x = 0; x < 3; ++x) {
        g[1][x] = __ddiv_rn(d[x], s);
        g[0][x] = -g[1][x];
      }
  } else if (type == CV_ANGLE) {
    double a[3], b[3], c[3];
    sub3(a, ri, rj);
    sub3(b, rk, rj);
    cross3(c, a, b);
    const double cn = sqrt(dot3(c, c));
    *sv = atan2(cn, dot3(a, b));
    if (cn != 0.0) {
      double ac[3], cb[3];
      cross3(ac, a, c);
      cross3(cb, c, b);
      const double da = __dmul_rn(dot3(a, a), cn), db = __dmul_rn(dot3(b, b), cn);
      for (int x = 0; x < 3; ++x) {
        g[0][x] = __ddiv_rn(ac[x], da);
        g[2][x] = __ddiv_rn(cb[x], db);
        g[1][x] = -__dadd_rn(g[0][x], g[2][x]);
      }
    }
  } else {
    double b1[3], b2[3], b3[3], m[3], n[3];
    sub3(b1, rj, ri);
    sub3(b2, rk, rj);
    sub3(b3, rl, rk);
    cross3(m, b1, b2);
    cross3(n, b2, b3);
    const double nb = sqrt(dot3(b2, b2));
    *sv = atan2(__dmul_rn(nb, dot3(b1, n)), dot3(m, n));
    const double mm = dot3(m, m), nn = dot3(n, n), bb = dot3(b2, b2);
    if (mm != 0.0 && nn != 0.0) {
      const double fi = __ddiv_rn(nb, mm), fl = __ddiv_rn(nb, nn);
      const double p = __ddiv_rn(dot3(b1, b2), bb), q = __ddiv_rn(dot3(b3, b2), bb);
      for (int x = 0; x < 3; ++x) {
        const double gi = -__dmul_rn(fi, m[x]), gl = __dmul_rn(fl, n[x]);
        const double t = __dsub_rn(__dmul_rn(p, gi), __dmul_rn(q, gl));
        g[0][x] = gi;
        g[1][x] = -__dadd_rn(gi, t);
        g[2][x] = __dsub_rn(t, gl);
        g[3][x] = gl;
      }
    }
  }
}

// The CTA stages the CVs of the replica's positions r and their gradients in shared memory: thread j < n_cv
// evaluates CV j, then a barrier
__device__ __forceinline__ void stage_cvs(int n_cv, const int* type, const int (*atoms)[4], const double* r,
                                          double* s_cv, double (*s_g)[4][3]) {
  const int tid = threadIdx.x;
  if (tid < n_cv) cv_eval(type[tid], atoms[tid], r, &s_cv[tid], s_g[tid]);
  __syncthreads();
}

// The CTA's bias force of one replica from dV/ds (s_dv, written before the call by any thread) and the staged
// gradients s_g: f = fm, then on the touched atoms f = fm + fb and fb_out = fb (md.cuh).  Starts with a barrier.
__device__ __forceinline__ void bias_force(int n_cv, const int* type, const int (*atoms)[4], const double* s_dv,
                                           const double (*s_g)[4][3], const double* fm, double* f, double* fb_out,
                                           int dimi) {
  const int tid = threadIdx.x;
  // F = Fm everywhere, then the touched atoms: thread j 4 + p owns atom slot p of CV j if it is that atom's first
  // appearance in (j, p) order
  for (int i = tid; i < dimi; i += MD_THREADS) f[i] = fm[i];
  __syncthreads();  // s_dv is complete, and every plain F is written
  if (tid < 4 * n_cv) {  // CV type t holds t + 2 atoms
    const int j0 = tid / 4, p0 = tid % 4;
    const int at = atoms[j0][p0];
    bool first = p0 < type[j0] + 2;
    for (int j = 0; j <= j0 && first; ++j)
      for (int p = 0; p < (j == j0 ? p0 : type[j] + 2); ++p)
        if (atoms[j][p] == at) first = false;
    if (first) {
      double fb[3] = {0.0, 0.0, 0.0};
      for (int j = j0; j < n_cv; ++j)
        for (int p = 0; p < type[j] + 2; ++p)
          if (atoms[j][p] == at)
            for (int x = 0; x < 3; ++x) fb[x] = __dsub_rn(fb[x], __dmul_rn(s_dv[j], s_g[j][p][x]));
      for (int x = 0; x < 3; ++x) {
        f[3 * at + x] = __dadd_rn(fm[3 * at + x], fb[x]);
        fb_out[3 * at + x] = fb[x];
      }
    }
  }
}

__global__ void __launch_bounds__(MD_THREADS) k_metad_bias(const MetadParams* __restrict__ Q,
                                                          const MdParams* __restrict__ P,
                                                          const double* __restrict__ R, const double* __restrict__ Fm,
                                                          double* __restrict__ F, const uint64_t* __restrict__ step,
                                                          int dimi, int deposit) {
  __shared__ double red[MD_THREADS];
  __shared__ double s_cv[MD_MAX_CV], s_dv[MD_MAX_CV];
  __shared__ double s_g[MD_MAX_CV][4][3];
  const MetadParams& q = *Q;
  const int n_cv = q.n_cv, nw = q.n_walkers;
  const int64_t rep = blockIdx.x, n_rep = gridDim.x, grp = rep / nw, w = rep % nw;
  const uint64_t c = step[rep];
  const uint64_t run_start = P->run_start;
  const int tid = threadIdx.x;
  stage_cvs(n_cv, q.type, q.atoms, R + rep * dimi, s_cv, s_g);
  const uint64_t pace = (uint64_t)q.pace;
  const int64_t n_g = q.count[grp] + (deposit ? (int64_t)nw * (int64_t)((c - 1) / pace - run_start / pace) : 0);
  const double* C = q.centers + grp * q.cap * n_cv;
  const double* W = q.widths + grp * q.cap * n_cv;
  const double* H = q.heights + grp * q.cap;
  double v = 0.0, dv[MD_MAX_CV] = {0.0, 0.0, 0.0, 0.0};
  for (int64_t k = tid; k < n_g; k += MD_THREADS) {
    double u[MD_MAX_CV], wk[MD_MAX_CV], a = 0.0;
#pragma unroll
    for (int j = 0; j < MD_MAX_CV; ++j) {
      if (j >= n_cv) break;
      double e = __dsub_rn(s_cv[j], C[k * n_cv + j]);
      if (q.type[j] == CV_DIHEDRAL) {
        if (e >= M_PI)
          e = __dsub_rn(e, 2.0 * M_PI);
        else if (e < -M_PI)
          e = __dadd_rn(e, 2.0 * M_PI);
      }
      wk[j] = W[k * n_cv + j];
      u[j] = __ddiv_rn(e, wk[j]);
      a = __dadd_rn(a, __dmul_rn(u[j], u[j]));
    }
    const double x = __dmul_rn(H[k], exp(__dmul_rn(-0.5, a)));
    v = __dadd_rn(v, x);
#pragma unroll
    for (int j = 0; j < MD_MAX_CV; ++j) {
      if (j >= n_cv) break;
      dv[j] = __dsub_rn(dv[j], __dmul_rn(x, __ddiv_rn(u[j], wk[j])));
    }
  }
  const double V = block_sum(v, red);
#pragma unroll
  for (int j = 0; j < MD_MAX_CV; ++j) {
    if (j >= n_cv) break;
    const double d = block_sum(dv[j], red);
    if (tid == 0) s_dv[j] = d;
  }
  bias_force(n_cv, q.type, q.atoms, s_dv, s_g, Fm + rep * dimi, F + rep * dimi, q.Fb + rep * dimi, dimi);
  if (tid < n_cv) q.cv[rep * n_cv + tid] = s_cv[tid];
  if (tid == 0) q.Vb[rep] = V;
  if (!deposit) return;
  const MdParams& p = *P;
  const uint64_t done = c - run_start;
  if (p.stride > 0 && done % (uint64_t)p.stride == 0) {
    const int64_t fr = (int64_t)(done / (uint64_t)p.stride) - 1;
    if (q.cv_f != nullptr && tid < n_cv) q.cv_f[(fr * n_rep + rep) * n_cv + tid] = s_cv[tid];
    if (q.bias_f != nullptr && tid == 0) q.bias_f[fr * n_rep + rep] = V;
  }
  if (c % pace == 0) {
    const int64_t slot = grp * q.cap + n_g + w;
    if (tid < n_cv) {
      q.centers[slot * n_cv + tid] = s_cv[tid];
      q.widths[slot * n_cv + tid] = q.width[tid];
    }
    if (tid == 0) q.heights[slot] = __dmul_rn(q.w0, exp(__ddiv_rn(-V, q.dkT)));
  }
}

// the commit after a run: count[g] += add for every group
__global__ void k_metad_commit(int64_t* count, int64_t n_groups, int64_t add) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_groups) count[g] += add;
}

// ---------------------------------------------------------------------------------- umbrella sampling
// The restraint, its bias force and the Hamiltonian exchange of sgdml_b200_umbrella_run (contract in md.cuh).

struct UmbrellaSmem {
  double cv[MD_MAX_CV], dv[MD_MAX_CV];
  double g[MD_MAX_CV][4][3];
};

// The CTA evaluates the configuration in slot rep under window k: its CVs and gradients, b and u, F = Fm + Fb, and the
// state's s, b and Fb.  Shared memory is free again only after a barrier.
__device__ __forceinline__ void umbrella_slot(const UmbrellaParams& q, int64_t rep, int k, const double* R,
                                              const double* Fm, double* F, int dimi, UmbrellaSmem& sm) {
  const int n_cv = q.n_cv;
  stage_cvs(n_cv, q.type, q.atoms, R + rep * dimi, sm.cv, sm.g);
  if (threadIdx.x == 0)
    q.Vb[rep] = umbrella_restraint(n_cv, q.type, sm.cv, q.win + k * n_cv, q.win + (q.n_windows + k) * n_cv, sm.dv);
  bias_force(n_cv, q.type, q.atoms, sm.dv, sm.g, Fm + rep * dimi, F + rep * dimi, q.Fb + rep * dimi, dimi);
  if ((int)threadIdx.x < n_cv) q.cv[rep * n_cv + threadIdx.x] = sm.cv[threadIdx.x];
}

__global__ void __launch_bounds__(MD_THREADS) k_umbrella_bias(const UmbrellaParams* __restrict__ Q,
                                                             const double* __restrict__ R,
                                                             const double* __restrict__ Fm, double* __restrict__ F,
                                                             int dimi) {
  __shared__ UmbrellaSmem sm;
  const UmbrellaParams& q = *Q;
  umbrella_slot(q, blockIdx.x, (int)(blockIdx.x % (unsigned)q.n_windows), R, Fm, F, dimi, sm);
}

// Thread t decides the pairs t, t + MD_THREADS, ... of its ladder and swaps their energies, CVs, walker labels and
// counts; then, pair by pair, every thread carries its coordinates of the two configurations' full-step velocities,
// swaps R and Fm, the CTA re-evaluates both slots, and the velocities are stored against the new forces.
__global__ void __launch_bounds__(MD_THREADS) k_umbrella_exchange(const RemdParams* __restrict__ X,
                                                                 const UmbrellaParams* __restrict__ Q,
                                                                 const MdParams* __restrict__ P,
                                                                 const double* __restrict__ s, double* __restrict__ R,
                                                                 double* __restrict__ V, double* __restrict__ F,
                                                                 double* __restrict__ Fm, double* __restrict__ E,
                                                                 int* __restrict__ walker,
                                                                 const uint64_t* __restrict__ step, int dimi) {
  __shared__ int acc[MD_THREADS];
  __shared__ UmbrellaSmem sm;
  const RemdParams& x = *X;
  const UmbrellaParams& q = *Q;
  const int nw = x.n_temps, n_cv = q.n_cv;
  const int64_t lad = blockIdx.x, n_rep = (int64_t)gridDim.x * nw, base = lad * nw;
  const uint64_t c = step[base];
  const uint64_t done = c - x.run_start;
  const bool sample = done != 0 && x.stride > 0 && done % (uint64_t)x.stride == 0;
  const bool exchange = x.every > 0 && done != 0 && c % (uint64_t)x.every == 0;
  if (!exchange && !sample) return;
  if (exchange) {
    const double h = P->h;
    const int par = (int)((c / (uint64_t)x.every) & 1);
    const int n_pairs = (nw - par) / 2;  // k = 2 j + par for j < n_pairs
    for (int j0 = 0; j0 < n_pairs; j0 += MD_THREADS) {
      const int j = j0 + (int)threadIdx.x;
      if (j < n_pairs) {
        const int k = 2 * j + par;
        const int64_t a = base + k, b = a + 1;
        double* ca = q.cv + a * n_cv;
        double* cb = q.cv + b * n_cv;
        const double *c0 = q.win + k * n_cv, *c1 = c0 + n_cv;
        const double *k0 = q.win + (nw + k) * n_cv, *k1 = k0 + n_cv;
        const double od = __dadd_rn(umbrella_restraint(n_cv, q.type, ca, c0, k0, nullptr),
                                    umbrella_restraint(n_cv, q.type, cb, c1, k1, nullptr));
        const double nd = __dadd_rn(umbrella_restraint(n_cv, q.type, cb, c0, k0, nullptr),
                                    umbrella_restraint(n_cv, q.type, ca, c1, k1, nullptr));
        const double d = -__dmul_rn(q.beta, __dsub_rn(nd, od));
        bool ok = d >= 0.0;
        if (!ok) {
          uint32_t ct[4] = {0x80000000u | (uint32_t)k, (uint32_t)lad, (uint32_t)c, (uint32_t)(c >> 32)};
          philox4x32_10(ct, x.key[0], x.key[1]);
          ok = uniform53(ct[0], ct[1]) < exp(d);
        }
        acc[threadIdx.x] = ok ? 1 : 0;
        const int64_t pq = lad * (nw - 1) + k;
        x.n_att[pq] += 1;
        if (ok) {
          x.n_acc[pq] += 1;
          const double e = E[a];
          E[a] = E[b];
          E[b] = e;
          const int w = walker[a];
          walker[a] = walker[b];
          walker[b] = w;
          for (int i = 0; i < n_cv; ++i) {
            const double t = ca[i];
            ca[i] = cb[i];
            cb[i] = t;
          }
        }
      }
      __syncthreads();  // the decisions are in acc
      const int nj = min(MD_THREADS, n_pairs - j0);
      for (int t = 0; t < nj; ++t) {
        if (!acc[t]) continue;
        const int k = 2 * (j0 + t) + par;
        const int64_t a = base + k, o = a * dimi;
        for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {  // V holds w until the new forces are known
          const int64_t ia = o + i, ib = ia + dimi;
          const double wa = __dadd_rn(V[ia], __dmul_rn(h, __dmul_rn(F[ia], s[i])));
          const double wb = __dadd_rn(V[ib], __dmul_rn(h, __dmul_rn(F[ib], s[i])));
          V[ia] = wb;
          V[ib] = wa;
          const double r = R[ia], m = Fm[ia];
          R[ia] = R[ib];
          R[ib] = r;
          Fm[ia] = Fm[ib];
          Fm[ib] = m;
        }
        __syncthreads();  // the swapped rows are complete
        umbrella_slot(q, a, k, R, Fm, F, dimi, sm);
        __syncthreads();  // sm is free again
        umbrella_slot(q, a + 1, k + 1, R, Fm, F, dimi, sm);
        __syncthreads();  // both slots' F are complete
        for (int i = threadIdx.x; i < 2 * dimi; i += MD_THREADS) {
          const int64_t ia = o + i;
          V[ia] = __dsub_rn(V[ia], __dmul_rn(h, __dmul_rn(F[ia], s[i % dimi])));
        }
      }
      __syncthreads();  // acc is free again, and the labels, CVs and biases are final
    }
  }
  if (sample) {
    const int64_t fr = (int64_t)(done / (uint64_t)x.stride) - 1;
    for (int k = threadIdx.x; k < nw; k += MD_THREADS) {
      const int64_t r = base + k, o = fr * n_rep + r;
      if (x.W_f) x.W_f[o] = walker[r];
      if (q.bias_f) q.bias_f[o] = q.Vb[r];
      if (q.cv_f)
        for (int j = 0; j < n_cv; ++j) q.cv_f[o * n_cv + j] = q.cv[r * n_cv + j];
    }
  }
}

// ---------------------------------------------------------------------------------- dimer search
// The dimer kernels of sgdml_b200_dimer_fire (contract in md.cuh).  As in the optimiser kernels, every thread holds the
// dimer's state and every CTA-wide sum, and each thread writes only its own coordinates i = t, t + MD_THREADS, ...; the
// rigid projection's atom sums read other threads' coordinates of N, after a barrier.

constexpr int DIMER_SUMS = 9;  // the most values one reduction carries: L (3) and I (6)

// K sums over the CTA at once, each by block_sum's tree (the same bits as K block_sum calls); every thread gets them
template <int K>
__device__ __forceinline__ void block_sums(double (&x)[K], double* red) {
#pragma unroll
  for (int k = 0; k < K; ++k) red[k * MD_THREADS + threadIdx.x] = x[k];
  __syncthreads();
  for (int w = MD_THREADS / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w)
#pragma unroll
      for (int k = 0; k < K; ++k)
        red[k * MD_THREADS + threadIdx.x] = __dadd_rn(red[k * MD_THREADS + threadIdx.x],
                                                      red[k * MD_THREADS + threadIdx.x + w]);
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < K; ++k) x[k] = red[k * MD_THREADS];
  __syncthreads();  // red is free again
}

// x if coordinate i belongs to component c, else 0.0 (the masked terms of the component sums)
__device__ __forceinline__ double comp(int i, int c, double x) { return i % 3 == c ? x : 0.0; }

// The rigid projection and normalisation (md.cuh, 5) of the mode n at centre r (n_atoms = dimi / 3), in place; the
// caller's writes of n are its own coordinates.  Returns n.n before the normalisation.
__device__ __forceinline__ double dimer_project(double* n, const double* r, int dimi, int periodic, double* red) {
  const double na = (double)(dimi / 3);
  double s[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // component sums of n (0..2) and of r (3..5)
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    const double ni = n[i], ri = r[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      s[c] = __dadd_rn(s[c], comp(i, c, ni));
      s[3 + c] = __dadd_rn(s[3 + c], comp(i, c, ri));
    }
  }
  block_sums(s, red);
  double m[3], rb[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    m[c] = __ddiv_rn(s[c], na);
    rb[c] = __ddiv_rn(s[3 + c], na);
  }
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    const int c = i % 3;
    n[i] = __dsub_rn(n[i], c == 0 ? m[0] : (c == 1 ? m[1] : m[2]));
  }
  if (!periodic) {
    __syncthreads();  // the atom sums read the other threads' coordinates of n
    double q[DIMER_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // L0..2, I00, I11, I22, P01, P02, P12
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
      if (i % 3 != 0) continue;  // the other coordinates add 0.0
      double x[3], na3[3], l[3];
      sub3(x, r + i, rb);
      for (int c = 0; c < 3; ++c) na3[c] = n[i + c];
      cross3(l, x, na3);
      const double x00 = __dmul_rn(x[0], x[0]), x11 = __dmul_rn(x[1], x[1]), x22 = __dmul_rn(x[2], x[2]);
      const double t[DIMER_SUMS] = {l[0], l[1], l[2], __dadd_rn(x11, x22), __dadd_rn(x00, x22), __dadd_rn(x00, x11),
                                    __dmul_rn(x[0], x[1]), __dmul_rn(x[0], x[2]), __dmul_rn(x[1], x[2])};
#pragma unroll
      for (int k = 0; k < DIMER_SUMS; ++k) q[k] = __dadd_rn(q[k], t[k]);
    }
    block_sums(q, red);
    const double I00 = q[3], I11 = q[4], I22 = q[5], I01 = -q[6], I02 = -q[7], I12 = -q[8];
    const double A00 = __dsub_rn(__dmul_rn(I11, I22), __dmul_rn(I12, I12));
    const double A01 = __dsub_rn(__dmul_rn(I02, I12), __dmul_rn(I01, I22));
    const double A02 = __dsub_rn(__dmul_rn(I01, I12), __dmul_rn(I11, I02));
    const double A11 = __dsub_rn(__dmul_rn(I00, I22), __dmul_rn(I02, I02));
    const double A12 = __dsub_rn(__dmul_rn(I01, I02), __dmul_rn(I00, I12));
    const double A22 = __dsub_rn(__dmul_rn(I00, I11), __dmul_rn(I01, I01));
    const double det = __dadd_rn(__dadd_rn(__dmul_rn(I00, A00), __dmul_rn(I01, A01)), __dmul_rn(I02, A02));
    const double tr = __ddiv_rn(__dadd_rn(__dadd_rn(I00, I11), I22), 3.0);
    if (det > __dmul_rn(1e-10, __dmul_rn(__dmul_rn(tr, tr), tr))) {
      const double L0 = q[0], L1 = q[1], L2 = q[2];
      const double w[3] = {
          __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(A00, L0), __dmul_rn(A01, L1)), __dmul_rn(A02, L2)), det),
          __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(A01, L0), __dmul_rn(A11, L1)), __dmul_rn(A12, L2)), det),
          __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(A02, L0), __dmul_rn(A12, L1)), __dmul_rn(A22, L2)), det)};
      for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
        const int c = i % 3;
        double x[3], wx[3];
        sub3(x, r + (i - c), rb);
        cross3(wx, w, x);
        n[i] = __dsub_rn(n[i], c == 0 ? wx[0] : (c == 1 ? wx[1] : wx[2]));
      }
    }
  }
  double nn = 0.0;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) nn = __dadd_rn(nn, __dmul_rn(n[i], n[i]));
  nn = block_sum(nn, red);
  const double nrm = sqrt(nn);
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) n[i] = __ddiv_rn(n[i], nrm);
  return nn;
}

// The initial modes of a call: src (n_dimers, 3N) projected at each centre into the scratch modes nd, the images
// R0 + D N into the scratch rows img (n_dimers, 3N), bad[d] as md.cuh says.  Nothing of the handle changes.
__global__ void __launch_bounds__(MD_THREADS) k_dimer_init(const DimerParams* __restrict__ Q,
                                                          const double* __restrict__ R, const double* __restrict__ src,
                                                          double* __restrict__ nd, double* __restrict__ img,
                                                          int* __restrict__ bad, int dimi) {
  __shared__ double red[DIMER_SUMS * MD_THREADS];
  const int64_t d = blockIdx.x;
  const double* r0 = R + 2 * d * dimi;
  const double* s = src + d * dimi;
  double* n = nd + d * dimi;
  double n0 = 0.0;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    const double x = s[i];
    n[i] = x;
    n0 = __dadd_rn(n0, __dmul_rn(x, x));
  }
  n0 = block_sum(n0, red);
  const double n1 = dimer_project(n, r0, dimi, Q->periodic, red);
  if (threadIdx.x == 0) bad[d] = !(isfinite(n0) && n1 > __dmul_rn(1e-12, n0));
  const double D = Q->D;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) img[d * dimi + i] = __dadd_rn(r0[i], __dmul_rn(D, n[i]));
}

__device__ __forceinline__ void dimer_store(RelaxState* st, DimerState* ds, const RelaxState& z, const DimerState& y) {
  __syncthreads();  // every thread has read the state
  if (threadIdx.x == 0) {
    *st = z;
    *ds = y;
  }
}

// The test and one step of dimer d (md.cuh): R rows 2d (centre) and 2d + 1 (image), the mode and T rows d, and the
// translation force Fd into Fn row 2d.
__global__ void __launch_bounds__(MD_THREADS) k_dimer_step(const DimerParams* __restrict__ Q, RelaxState* st,
                                                          DimerState* ds, double* __restrict__ R,
                                                          double* __restrict__ V, const double* __restrict__ F,
                                                          double* __restrict__ Fn, double* __restrict__ Nm,
                                                          double* __restrict__ Th, int dimi, int advance) {
  __shared__ double red[DIMER_SUMS * MD_THREADS];
  const int64_t d = blockIdx.x;
  const DimerParams p = *Q;
  RelaxState z = st[d];
  DimerState y = ds[d];
  z.gamma = z.E_prev = 0.0;  // (L-BFGS fields: zero already, as in k_neb_fire_step)
  double* r0 = R + 2 * d * dimi;
  double* r1 = r0 + dimi;
  const double* f0 = F + 2 * d * dimi;
  const double* f1 = f0 + dimi;
  double* n = Nm + d * dimi;
  double* th = Th + d * dimi;
  if (z.conv) return dimer_store(st + d, ds + d, z, y);
  if (y.phase == DIMER_EVAL_N) {
    double c = 0.0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) c = __dadd_rn(c, __dmul_rn(__dsub_rn(f0[i], f1[i]), n[i]));
    y.C_N = __ddiv_rn(block_sum(c, red), p.D);
  }
  z.fmax2 = atom_max2(f0, dimi, red);
  z.conv = z.fmax2 < p.fmax2 && y.C_N < 0.0 ? 1 : 0;
  if (z.conv || !advance) return dimer_store(st + d, ds + d, z, y);

  double cu;  // C_use
  if (y.phase == DIMER_EVAL_N) {
    double g = 0.0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS)
      g = __dadd_rn(g, __dmul_rn(__ddiv_rn(__dsub_rn(f1[i], f0[i]), p.D), n[i]));
    g = block_sum(g, red);
    double pp = 0.0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
      const double pi = __dsub_rn(__ddiv_rn(__dsub_rn(f1[i], f0[i]), p.D), __dmul_rn(g, n[i]));
      th[i] = pi;
      pp = __dadd_rn(pp, __dmul_rn(pi, pi));
    }
    const double f = sqrt(block_sum(pp, red));
    if (!(f < p.rot_min) && f != 0.0) {  // rotate: place the image on the trial direction
      for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
        const double t = __ddiv_rn(th[i], f);
        th[i] = t;
        r1[i] = __dadd_rn(r0[i], __dmul_rn(p.D, __dadd_rn(__dmul_rn(p.c_t, n[i]), __dmul_rn(p.s_t, t))));
      }
      y.C0 = y.C_N;
      y.b1 = -f;
      y.phase = DIMER_TRIAL;
      return dimer_store(st + d, ds + d, z, y);
    }
    cu = y.C_N;
  } else {
    double c = 0.0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
      const double nt = __dadd_rn(__dmul_rn(p.c_t, n[i]), __dmul_rn(p.s_t, th[i]));
      c = __dadd_rn(c, __dmul_rn(__dsub_rn(f0[i], f1[i]), nt));
    }
    const double ct = __ddiv_rn(block_sum(c, red), p.D);
    const double a1 = __ddiv_rn(__dadd_rn(__dsub_rn(y.C0, ct), __dmul_rn(y.b1, p.s2_t)), p.omc2_t);
    const double rr = sqrt(__dadd_rn(__dmul_rn(a1, a1), __dmul_rn(y.b1, y.b1)));
    const double c2 = __ddiv_rn(-a1, rr), s2 = __ddiv_rn(-y.b1, rr);
    double cs, sn;
    if (c2 >= 0.0) {
      cs = sqrt(__ddiv_rn(__dadd_rn(1.0, c2), 2.0));
      sn = __ddiv_rn(s2, __dmul_rn(2.0, cs));
    } else {
      sn = sqrt(__ddiv_rn(__dsub_rn(1.0, c2), 2.0));
      cs = __ddiv_rn(s2, __dmul_rn(2.0, sn));
    }
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) n[i] = __dadd_rn(__dmul_rn(cs, n[i]), __dmul_rn(sn, th[i]));
    dimer_project(n, r0, dimi, p.periodic, red);
    cu = __dsub_rn(__dsub_rn(y.C0, a1), rr);
    ++y.n_rot;
  }
  double* fd = Fn + 2 * d * dimi;
  double pf = 0.0;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) pf = __dadd_rn(pf, __dmul_rn(f0[i], n[i]));
  pf = block_sum(pf, red);
  const double pf2 = __dmul_rn(2.0, pf);
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS)
    fd[i] = cu < 0.0 ? __dsub_rn(f0[i], __dmul_rn(pf2, n[i])) : -__dmul_rn(pf, n[i]);
  fire_update(z, p.dt0, p.dtmax, p.maxstep, r0, V + 2 * d * dimi, fd, dimi, red);
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) r1[i] = __dadd_rn(r0[i], __dmul_rn(p.D, n[i]));
  y.phase = DIMER_EVAL_N;
  dimer_store(st + d, ds + d, z, y);
}

// the curvature, rotation count and mode of every dimer into the call's outputs (each may be null)
__global__ void k_dimer_report(const DimerState* __restrict__ ds, int64_t n_dimers, double* curv, int64_t* n_rot) {
  const int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n_dimers) return;
  if (curv) curv[d] = ds[d].C_N;
  if (n_rot) n_rot[d] = ds[d].n_rot;
}

// ---------------------------------------------------------------------------------- reaction path
// The IRC kernels of sgdml_b200_irc_rk4 (contract in md.cuh).  As in the optimiser kernels, every thread holds the
// branch's state and every CTA-wide sum, and each thread writes only its own coordinates i = t, t + MD_THREADS, ...

// The check (commit == 0) or the commit (commit == 1) of pair k's start, V (n_pairs, 3N) the caller's modes in transit.
__global__ void __launch_bounds__(MD_THREADS) k_irc_init(const IrcParams* __restrict__ Q, const double* __restrict__ s,
                                                        double* __restrict__ R, const double* __restrict__ F,
                                                        const double* __restrict__ E, double* __restrict__ V,
                                                        int* __restrict__ bad, double* __restrict__ Rn,
                                                        double* __restrict__ Fn, IrcState* __restrict__ is, int dimi,
                                                        int commit) {
  __shared__ double red[MD_THREADS];
  const int64_t k = blockIdx.x;
  double* v = V + k * dimi;
  if (!commit) {
    double q = 0.0;
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
      const double x = __ddiv_rn(v[i], sqrt(s[i]));
      v[i] = x;
      q = __dadd_rn(q, __dmul_rn(x, x));
    }
    q = block_sum(q, red);
    const double nrm = sqrt(q);
    for (int i = threadIdx.x; i < dimi; i += MD_THREADS) v[i] = __ddiv_rn(v[i], nrm);
    if (threadIdx.x == 0) bad[k] = !(isfinite(q) && q > 0.0);
    return;
  }
  const IrcParams p = *Q;
  const int64_t mp = p.max_points;
  const double e0 = E[2 * k];
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    const double r0 = R[2 * k * dimi + i], f0 = F[2 * k * dimi + i], ri = sqrt(s[i]);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int64_t b = 2 * k + j;
      Rn[b * dimi + i] = r0;
      Fn[b * dimi + i] = f0;
      R[b * dimi + i] = __dadd_rn(r0, __dmul_rn(ri, __dmul_rn(j ? -p.h : p.h, v[i])));
      if (p.R_path) p.R_path[b * mp * dimi + i] = r0;
    }
  }
  for (int j = 0; j < 2; ++j) {
    const int64_t b = 2 * k + j;
    if (p.R_path)
      for (int64_t o = dimi + threadIdx.x; o < mp * dimi; o += MD_THREADS) p.R_path[b * mp * dimi + o] = nan;
    if (p.E_path)
      for (int64_t o = threadIdx.x; o < mp; o += MD_THREADS) p.E_path[b * mp + o] = o == 0 ? e0 : nan;
    if (threadIdx.x == 0) {
      is[b].phase = IRC_POINT;
      is[b].end = 0;
      is[b].n_points = 1;
      is[b].E_n = e0;
    }
  }
}

// The test and one stage of branch b (md.cuh): R, F, E rows b, the point buffers Rn, Fn and the running sum K rows b.
__global__ void __launch_bounds__(MD_THREADS) k_irc_step(const IrcParams* __restrict__ Q, RelaxState* st,
                                                        IrcState* is, const double* __restrict__ s,
                                                        double* __restrict__ R, double* __restrict__ F,
                                                        double* __restrict__ E, double* __restrict__ Rn,
                                                        double* __restrict__ Fn, double* __restrict__ K, int dimi,
                                                        int advance) {
  __shared__ double red[MD_THREADS];
  const int64_t b = blockIdx.x;
  const IrcParams p = *Q;
  RelaxState z = st[b];
  IrcState y = is[b];
  double* r = R + b * dimi;
  double* f = F + b * dimi;
  double* rn = Rn + b * dimi;
  double* fn = Fn + b * dimi;
  double* k = K + b * dimi;
  if (y.end) return relax_store(st + b, z);
  if (y.phase == IRC_POINT) {
    const double e = E[b];
    if (!(e < y.E_n)) {
      for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
        r[i] = rn[i];
        f[i] = fn[i];
      }
      z.fmax2 = atom_max2(fn, dimi, red);  // (its barriers: every thread has read E[b])
      if (threadIdx.x == 0) E[b] = y.E_n;
      y.end = 2;
    } else {
      const int64_t n = y.n_points;
      for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
        const double ri = r[i];
        rn[i] = ri;
        fn[i] = f[i];
        if (p.R_path) p.R_path[(b * p.max_points + n) * dimi + i] = ri;
      }
      if (p.E_path && threadIdx.x == 0) p.E_path[b * p.max_points + n] = e;
      y.n_points = n + 1;
      y.E_n = e;
      z.fmax2 = atom_max2(f, dimi, red);
      y.end = z.fmax2 < p.fmax2 ? 1 : (y.n_points == p.max_points ? 3 : 0);
    }
    y.phase = IRC_K1;
    z.n_steps = y.n_points;
    z.conv = y.end;
  }
  if (y.end || !advance) {
    __syncthreads();  // every thread has read the state
    if (threadIdx.x == 0) {
      st[b] = z;
      is[b] = y;
    }
    return;
  }
  double q = 0.0;
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    const double g = __dmul_rn(sqrt(s[i]), f[i]);
    q = __dadd_rn(q, __dmul_rn(g, g));
  }
  q = block_sum(q, red);
  const double nrm = sqrt(q);
  const int ph = y.phase;
  const double c = ph == IRC_K3 ? p.h : (ph == IRC_K4 ? p.h6 : p.hh);
  for (int i = threadIdx.x; i < dimi; i += MD_THREADS) {
    const double ri = sqrt(s[i]);
    const double d = q == 0.0 ? 0.0 : __ddiv_rn(__dmul_rn(ri, f[i]), nrm);
    double x = d;  // what the stage moves along: d, or K after k4
    if (ph == IRC_K1) {
      k[i] = d;
    } else if (ph == IRC_K4) {
      x = __dadd_rn(k[i], d);
    } else {
      k[i] = __dadd_rn(k[i], __dmul_rn(2.0, d));
    }
    r[i] = __dadd_rn(rn[i], __dmul_rn(ri, __dmul_rn(c, x)));
  }
  y.phase = ph == IRC_K4 ? IRC_POINT : ph + 1;
  __syncthreads();  // every thread has read the state
  if (threadIdx.x == 0) {
    st[b] = z;
    is[b] = y;
  }
}

}  // namespace

}  // namespace sgdml

// md.cuh: the checks of a window table, shared with mbar.cu
int sgdml::umbrella_windows_check(int64_t n_windows, int n_cv, const int* type, const double* centers,
                                  const double* kappas) {
  SG_ARG(centers != nullptr && kappas != nullptr);
  SG_ARG(!is_device_ptr(centers) && !is_device_ptr(kappas));
  for (int64_t i = 0; i < n_windows * n_cv; ++i) {
    const double c = centers[i], k = kappas[i];
    if (!std::isfinite(c)) return fail_arg("every window centre must be finite");
    if (!(std::isfinite(k) && k >= 0.0)) return fail_arg("every force constant must be finite and >= 0");
    if (type[i % n_cv] == CV_DIHEDRAL && !(c > -M_PI && c <= M_PI))
      return fail_arg("a dihedral's window centre must lie in (-pi, pi]");
  }
  return 0;
}

// ============================================================== driver (sgdml_b200_md_*, _remd_run, _pimd_*, _relax_*)
// The state of n_rep replicas stays in device memory between steps and between runs.  One step is the integrator
// kernel, then the forces and energies of the new positions (force_eval_run, predict.cuh) written back into the
// state.  That sequence is captured once into a CUDA graph and replayed n_steps times on the caller's stream;
// everything a run changes (dt, gamma, kT, seed, frame buffers) lives in device memory, and the step counter is
// advanced by the integrator, so the graph bakes in no run.
using namespace sgdml;

namespace {

// The parameters of every integrator, at the head of the handle's upload block.  A call fills only its own.
struct StepParams {
  MdParams md;
  PimdParams pimd;
  RelaxParams relax;
  NebParams neb;
  RemdParams remd;
  NptParams npt;
  MetadParams metad;
  DimerParams dimer;
  UmbrellaParams umbrella;
  IrcParams irc;
};
constexpr size_t STEP_PARAMS_BYTES = (sizeof(StepParams) + 255) & ~(size_t)255;  // where the tables start
// The umbrella parameters took the block past 768 bytes, so the tables start at 1024.  Every kernel that reads a table
// gets its address as an argument, and a captured graph is keyed on the block, so the move changes no step.
static_assert(STEP_PARAMS_BYTES == 1024, "the tables start at 1024 bytes");

// What a captured step bakes in besides the force evaluation: the integrator (MdKind), the replicas per group (the
// grids of the NEB and exchange kernels) and the upload block (the tab and sigma kernel arguments point into it).
struct StepKey {
  int kind, group;
  const char* blk;
  bool operator==(const StepKey& o) const { return kind == o.kind && group == o.group && blk == o.blk; }
};

// What a handle is, fixed at creation (sgdml_b200_pimd_create makes PLAIN handles with one bead, RING with more): it
// decides which entry points take the handle (check_kind) and how its state's forces are evaluated.
enum HandleKind { PLAIN, RING, NPT, METAD, UMBRELLA };

}  // namespace

struct sgdml_b200_md {
  HandleKind kind = PLAIN;
  int64_t n_rep = 0;
  int dimi = 0;
  int nb = 1;  // beads per ring polymer: replica p nb + j is bead j of polymer p (1 for sgdml_b200_md_create)
  ForceEval* fe = nullptr;  // the handle's own predictor workspace: predict calls never touch it, MD never theirs
  double *R = nullptr, *V = nullptr, *F = nullptr, *E = nullptr;  // state: (n_rep, 3N) x 3, (n_rep)
  double *Fs = nullptr, *Es = nullptr;  // outputs of the force evaluation that precedes a capture
  uint64_t* step = nullptr;             // (n_rep) step counters, all equal
  uint64_t step_host = 0;               // their value once the queued runs have finished
  bool has_state = false;
  double* s = nullptr;                  // (3N) inverse mass
  std::vector<double> s_host;           // s on the host
  // The upload block on the device (blk) and its pinned mirror (hblk): StepParams, then the tables -- the PIMD table
  // C (nb x nb) and the four mode tables (nb each), sigma (rows, 3N), the noise scale per mode or temperature, and the
  // ladder beta, lam_up, lam_dn (rows each).  A call fills its part of the mirror once the previous call's upload has
  // read it (uploaded), then uploads the prefix it uses in one copy.
  char *blk = nullptr, *hblk = nullptr;
  int rows = 0;  // max(nb, the largest n_temps so far)
  cudaEvent_t uploaded = nullptr;
  cudaStream_t gs = nullptr;  // capture stream
  cudaEvent_t ge = nullptr;
  cudaGraphExec_t exec = nullptr;
  StepKey graph_key = {};     // the key of the captured step
  int n_kernels = 0;
  // replicas per group of the current call: images per band (NEB), temperatures per ladder (replica exchange), else 1
  int group = 1;
  // geometry optimisation (sgdml_b200_relax_*), allocated by the first relaxation
  RelaxState* rst = nullptr;  // (n_rep) per-replica optimiser state
  int* hActive = nullptr;     // mapped pinned: unconverged replicas, written by k_relax_count
  int* dActive = nullptr;     // its device address
  cudaEvent_t counted = nullptr;
  double *S = nullptr, *Y = nullptr, *rho = nullptr;        // L-BFGS ring, m_cap pairs per replica
  double *r_prev = nullptr, *g_prev = nullptr;              // (n_rep, 3N)
  int m_cap = 0;
  // nudged elastic band (sgdml_b200_neb_fire), allocated by the first NEB call
  double* Fn = nullptr;       // (n_rep, 3N) NEB forces of the interior images
  int* climb_idx = nullptr;   // (n_rep) the highest interior image of each band (the first n_rep / P entries)
  // dimer search (sgdml_b200_dimer_fire), allocated by the first dimer call; F-dagger goes to Fn
  double *dmode = nullptr, *dtheta = nullptr;  // (n_rep / 2, 3N) unit modes, and T (or a caller's modes in transit)
  DimerState* dstate = nullptr;               // (n_rep / 2)
  int* dbad = nullptr;                        // (n_rep / 2) k_dimer_init's verdict per mode
  bool has_modes = false;                     // dmode holds the modes of an earlier call
  // reaction path (sgdml_b200_irc_rk4), allocated by the first IRC call
  double *irc_rn = nullptr, *irc_fn = nullptr, *irc_k = nullptr;  // (n_rep, 3N) the newest point's R and F, RK4 sum
  double* irc_v = nullptr;                    // (n_rep / 2, 3N) the caller's modes in transit, normalised in place
  IrcState* istate = nullptr;                 // (n_rep)
  int* ibad = nullptr;                        // (n_rep / 2) k_irc_init's verdict per mode
  // replica exchange (sgdml_b200_remd_run), allocated by the first replica-exchange call
  int* walker = nullptr;      // (n_rep) walker label per slot
  int64_t* xcount = nullptr;  // (2, n_rep) accepted and attempted swaps of the current run
  // NPT (sgdml_b200_npt_create): one cell per replica, made with the handle; null on every other handle
  NptCell* cell = nullptr;    // (n_rep) barostat state
  Lattice* lat = nullptr;     // (n_rep) the cells the descriptor kernel reads: a L0 and L0^-1 / a, a = exp(eps / 3)
  double *W = nullptr, *Ws = nullptr;  // (n_rep, 9) virial of the state, and of the evaluation that precedes a capture
  // metadynamics (sgdml_b200_metad_create): null on every other handle.  The model's forces go to Fm, and k_metad_bias
  // completes F; the hill store's pointers, its capacity and the CVs live in the mirror's MetadParams.
  double* Fm = nullptr;        // (n_rep, 3N) the model's forces of the state
  double *cv = nullptr, *Vb = nullptr, *Fb = nullptr;  // the state's CVs, bias energy and bias force
  double *hc = nullptr, *hw = nullptr, *hh = nullptr;  // the hill store: centres, widths, heights
  int64_t* hcount = nullptr;   // (n_groups) committed hills per group
  std::vector<int64_t> hcount_host;  // the same, once the queued runs have finished
  int64_t n_groups = 0;
  // umbrella sampling (sgdml_b200_umbrella_create): Fm, cv, Vb and Fb as on a metadynamics handle, the walker labels
  // and swap counts as on a replica exchange, and the window table, whose address is in the mirror's UmbrellaParams
  double* win = nullptr;       // (2, n_windows, n_cv) centres, then force constants

  // the block's parts in blk or hblk
  StepParams* params(char* b) const { return reinterpret_cast<StepParams*>(b); }
  double* tab(char* b) const { return reinterpret_cast<double*>(b + STEP_PARAMS_BYTES); }
  double* sigma(char* b) const { return tab(b) + nb * nb + 4 * nb; }
  double* ladder(char* b) const { return sigma(b) + (size_t)rows * dimi; }
};

namespace {

void md_free(sgdml_b200_md* md) {
  cudaDeviceSynchronize();  // blocks go back to the cache: nothing may still use them
  if (md->exec) cudaGraphExecDestroy(md->exec);
  if (md->gs) cudaStreamDestroy(md->gs);
  if (md->ge) cudaEventDestroy(md->ge);
  if (md->uploaded) cudaEventDestroy(md->uploaded);
  if (md->counted) cudaEventDestroy(md->counted);
  force_eval_destroy(md->fe);
  for (double* p : {md->R, md->V, md->F, md->E, md->Fs, md->Es, md->s}) cached_free(p);
  for (double* p : {md->S, md->Y, md->rho, md->r_prev, md->g_prev, md->Fn, md->W, md->Ws}) cached_free(p);
  for (double* p : {md->Fm, md->cv, md->Vb, md->Fb, md->hc, md->hw, md->hh, md->dmode, md->dtheta}) cached_free(p);
  for (double* p : {md->irc_rn, md->irc_fn, md->irc_k, md->irc_v}) cached_free(p);
  cached_free(md->istate);
  cached_free(md->ibad);
  cached_free(md->dstate);
  cached_free(md->dbad);
  cached_free(md->hcount);
  cached_free(md->win);
  cached_free(md->step);
  cached_free(md->blk);
  cached_free(md->rst);
  cached_free(md->climb_idx);
  cached_free(md->walker);
  cached_free(md->xcount);
  cached_free(md->cell);
  cached_free(md->lat);
  cudaFreeHost(md->hblk);
  cudaFreeHost(md->hActive);
  delete md;
}

// The block holds `rows` sigma and ladder rows: nb at creation, more when a replica exchange needs them.  A grown
// block moves, which changes the step key.  The mirror starts as zeros.
int reserve(sgdml_b200_md* md, int rows) {
  if (rows <= md->rows) return 0;
  if (md->blk != nullptr) SG_CUDA(cudaDeviceSynchronize());  // the old block goes back: nothing may still use it
  cached_free(md->blk);
  cudaFreeHost(md->hblk);
  md->blk = md->hblk = nullptr;
  md->rows = 0;
  const size_t bytes =
      STEP_PARAMS_BYTES + sizeof(double) * ((size_t)md->nb * md->nb + 4 * md->nb + (size_t)rows * (md->dimi + 3));
  SG_CUDA(cached_malloc(&md->blk, bytes));
  SG_CUDA(cudaMallocHost(&md->hblk, bytes));
  std::memset(md->hblk, 0, bytes);
  md->rows = rows;
  return 0;
}

// uploads the block's first bytes up to `end` (in hblk) on s, and marks when the mirror is free again
int upload(sgdml_b200_md* md, const void* end, cudaStream_t s) {
  const size_t bytes = (size_t)(static_cast<const char*>(end) - md->hblk);
  SG_CUDA(cudaMemcpyAsync(md->blk, md->hblk, bytes, cudaMemcpyHostToDevice, s));
  SG_CUDA(cudaEventRecord(md->uploaded, s));
  return 0;
}

// The outputs of one call, each a (caller's pointer, bytes) pair; a null pointer or 0 bytes is no output.  The kernels
// write a caller's device array in place and a host array into one device staging block, which finish() copies back.
// The stream is synchronised before that block goes back to the cache on every path: after an error return, launches
// already queued may still write into it.
class Outputs {
 public:
  struct Out {
    void* user;
    size_t bytes;
  };
  explicit Outputs(cudaStream_t s) : s_(s) {}
  Outputs(const Outputs&) = delete;
  Outputs& operator=(const Outputs&) = delete;
  ~Outputs() {
    if (block_ == nullptr) return;
    if (!synced_) cudaStreamSynchronize(s_);
    cached_free(block_);
  }
  int init(std::initializer_list<Out> outs) {  // at most MAX_OUTS
    size_t off[MAX_OUTS], total = 0;
    for (const Out& o : outs) {
      const int i = n_++;
      out_[i] = o;
      dev_[i] = o.bytes > 0 ? o.user : nullptr;
      staged_[i] = dev_[i] != nullptr && !is_device_ptr(o.user);
      off[i] = total;
      if (staged_[i]) total += (o.bytes + 255) & ~(size_t)255;
    }
    if (total == 0) return 0;
    SG_CUDA(cached_malloc(&block_, total));
    for (int i = 0; i < n_; ++i)
      if (staged_[i]) dev_[i] = block_ + off[i];
    return 0;
  }
  // where the kernels write output i (null: none)
  template <class T = double>
  T* dev(int i) const {
    return static_cast<T*>(dev_[i]);
  }
  // queues the copies of device arrays src[0], src[1], ... into outputs first, first + 1, ... (those that are outputs)
  int copy_from(int first, std::initializer_list<const void*> src) {
    int i = first;
    for (const void* p : src) {
      if (dev_[i] != nullptr) SG_CUDA(cudaMemcpyAsync(dev_[i], p, out_[i].bytes, cudaMemcpyDeviceToDevice, s_));
      ++i;
    }
    return 0;
  }
  // queues the copies to the host arrays and, if there are any, waits for them
  int finish() {
    for (int i = 0; i < n_; ++i)
      if (staged_[i]) SG_CUDA(cudaMemcpyAsync(out_[i].user, dev_[i], out_[i].bytes, cudaMemcpyDeviceToHost, s_));
    if (block_ != nullptr) {
      SG_CUDA(cudaStreamSynchronize(s_));
      synced_ = true;
    }
    return 0;
  }

 private:
  static constexpr int MAX_OUTS = 14;
  cudaStream_t s_;
  int n_ = 0;
  Out out_[MAX_OUTS];
  void* dev_[MAX_OUTS];
  bool staged_[MAX_OUTS];
  char* block_ = nullptr;
  bool synced_ = false;
};

// what one step of the handle's graph integrates
enum MdKind {
  MD_CLASSICAL = 0, MD_RING_POLYMER = 1, MD_FIRE = 2, MD_LBFGS = 3, MD_NEB_FIRE = 4, MD_REMD = 5, MD_NPT = 6,
  MD_METAD = 7, MD_DIMER = 8, MD_UMBRELLA = 9, MD_IRC = 10
};

// the integrator of sgdml_b200_md_run, sgdml_b200_remd_run, sgdml_b200_npt_run, sgdml_b200_umbrella_run,
// sgdml_b200_pimd_run, sgdml_b200_relax_*, sgdml_b200_neb_fire, sgdml_b200_dimer_fire or sgdml_b200_irc_rk4;
// advance == 0 completes a run's last step (MD; a replica exchange or umbrella run first exchanges that last state) or
// only tests convergence (relaxation, NEB: after the force projection, dimer: with the curvature, IRC: a new point).
// L-BFGS keeps its direction in V, which relax_impl zeroes after.
int md_integrate(sgdml_b200_md* md, int kind, int advance, cudaStream_t s) {
  StepParams* p = md->params(md->blk);
  switch (kind) {
    case MD_RING_POLYMER:
      k_pimd_step<<<(unsigned)(md->n_rep / md->nb), MD_THREADS, 0, s>>>(&p->pimd, md->tab(md->blk), md->s,
                                                                      md->sigma(md->blk), md->R, md->V, md->F, md->E,
                                                                      md->step, md->dimi, md->nb, advance);
      break;
    case MD_FIRE:
      k_fire_step<<<(unsigned)md->n_rep, MD_THREADS, 0, s>>>(&p->relax, md->rst, md->R, md->V, md->F, md->dimi,
                                                             advance);
      break;
    case MD_LBFGS:
      k_lbfgs_step<<<(unsigned)md->n_rep, MD_THREADS, 0, s>>>(&p->relax, md->rst, md->R, md->V, md->F, md->E,
                                                              md->dimi, advance);
      break;
    case MD_NEB_FIRE: {
      const int64_t n_bands = md->n_rep / md->group;
      k_neb_force<<<(unsigned)(n_bands * (md->group - 2)), MD_THREADS, 0, s>>>(&p->neb, md->R, md->F, md->E, md->Fn,
                                                                              md->climb_idx, md->dimi);
      SG_CUDA(cudaGetLastError());
      count_launch(KID_MISC);
      k_neb_fire_step<<<(unsigned)n_bands, MD_THREADS, 0, s>>>(&p->neb, md->rst, md->R, md->V, md->Fn, md->dimi,
                                                               advance);
      break;
    }
    case MD_DIMER:
      k_dimer_step<<<(unsigned)(md->n_rep / 2), MD_THREADS, 0, s>>>(&p->dimer, md->rst, md->dstate, md->R, md->V, md->F,
                                                                   md->Fn, md->dmode, md->dtheta, md->dimi, advance);
      break;
    case MD_IRC:
      k_irc_step<<<(unsigned)md->n_rep, MD_THREADS, 0, s>>>(&p->irc, md->rst, md->istate, md->s, md->R, md->F, md->E,
                                                            md->irc_rn, md->irc_fn, md->irc_k, md->dimi, advance);
      break;
    case MD_NPT:
      k_npt_step<<<(unsigned)md->n_rep, MD_THREADS, 0, s>>>(&p->md, &p->npt, md->s, md->sigma(md->blk), md->R, md->V,
                                                            md->F, md->E, md->W, md->cell, md->lat, md->step, md->dimi,
                                                            advance);
      break;
    case MD_REMD:
    case MD_UMBRELLA:
      if (kind == MD_REMD)
        k_remd_exchange<<<(unsigned)(md->n_rep / md->group), MD_THREADS, 0, s>>>(&p->remd, &p->md, md->s, md->R, md->V,
                                                                                md->F, md->E, md->walker, md->step,
                                                                                md->dimi);
      else
        k_umbrella_exchange<<<(unsigned)(md->n_rep / md->group), MD_THREADS, 0, s>>>(
            &p->remd, &p->umbrella, &p->md, md->s, md->R, md->V, md->F, md->Fm, md->E, md->walker, md->step, md->dimi);
      SG_CUDA(cudaGetLastError());
      count_launch(KID_MISC);
      [[fallthrough]];
    default:
      k_md_step<<<(unsigned)md->n_rep, MD_THREADS, 0, s>>>(&p->md, md->s, md->sigma(md->blk), md->R, md->V, md->F,
                                                           md->E, md->step, md->dimi, advance);
  }
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

// F and E (and on an NPT handle W, each replica in its own cell) of the positions in R
int md_forces(sgdml_b200_md* md, double* F, double* E, double* W, cudaStream_t s) {
  if (md->kind != NPT) return force_eval_run(md->fe, md->R, F, E, s);
  return force_eval_run_cells(md->fe, md->R, md->lat, F, E, W, s);
}

// The umbrella restraints of the state in R on top of the model's forces in Fm
int umbrella_bias(sgdml_b200_md* md, cudaStream_t s) {
  k_umbrella_bias<<<(unsigned)md->n_rep, MD_THREADS, 0, s>>>(&md->params(md->blk)->umbrella, md->R, md->Fm, md->F,
                                                             md->dimi);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

// The state's forces and energies: on a metadynamics or umbrella handle the model's F into Fm, then k_metad_bias
// (deposit: inside a run) or k_umbrella_bias completes F; on every other handle md_forces
int md_state_forces(sgdml_b200_md* md, int deposit, cudaStream_t s) {
  if (md->kind != METAD && md->kind != UMBRELLA) return md_forces(md, md->F, md->E, md->W, s);
  SG_TRY(md_forces(md, md->Fm, md->E, nullptr, s));
  if (md->kind == UMBRELLA) return umbrella_bias(md, s);
  StepParams* p = md->params(md->blk);
  k_metad_bias<<<(unsigned)md->n_rep, MD_THREADS, 0, s>>>(&p->metad, &p->md, md->R, md->Fm, md->F, md->step, md->dimi,
                                                          deposit);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

int md_step(sgdml_b200_md* md, int kind, cudaStream_t s) {
  SG_TRY(md_integrate(md, kind, 1, s));
  return md_state_forces(md, 1, s);
}

// the step graph, captured again whenever the force evaluation it bakes in is stale or its key changes
int md_graph(sgdml_b200_md* md, int kind, cudaStream_t s) {
  const StepKey key = {kind, md->group, md->blk};
  if (md->exec != nullptr && md->graph_key == key && !force_eval_stale(md->fe)) return 0;
  if (md->exec != nullptr) {
    cudaGraphExecDestroy(md->exec);
    md->exec = nullptr;
  }
  if (md->gs == nullptr) {
    SG_CUDA(cudaStreamCreateWithFlags(&md->gs, cudaStreamNonBlocking));
    SG_CUDA(cudaEventCreateWithFlags(&md->ge, cudaEventDisableTiming));
  }
  // captured on a private stream (the caller's may be the legacy stream); after the caller's queued work
  SG_CUDA(cudaEventRecord(md->ge, s));
  SG_CUDA(cudaStreamWaitEvent(md->gs, md->ge, 0));
  // the force evaluation once un-captured, into scratch outputs: sets the kernels' shared-memory attributes
  SG_TRY(md_forces(md, md->Fs, md->Es, md->Ws, md->gs));
  SG_CUDA(cudaStreamSynchronize(md->gs));
  SG_TRY(capture_graph(md->gs, [&] { return md_step(md, kind, md->gs); }, &md->exec, &md->n_kernels));
  force_eval_mark(md->fe);
  md->graph_key = key;
  return 0;
}

// n_steps steps of the handle's integrator: graph replays, or plain launches with SGDML_B200_GRAPH=0 or profiling
int md_replay(sgdml_b200_md* md, int kind, int64_t n_steps, cudaStream_t s) {
  if (g_graph_enabled() && !profiling_enabled()) {
    SG_TRY(md_graph(md, kind, s));
    for (int64_t k = 0; k < n_steps; ++k) {
      SG_CUDA(cudaGraphLaunch(md->exec, s));
      count_launch(KID_PREDICT_AUX, md->n_kernels);  // the kernels of a replay are launches too
    }
  } else {
    for (int64_t k = 0; k < n_steps; ++k) SG_TRY(md_step(md, kind, s));
  }
  return 0;
}

// ------------------------------------------------------------------ MD, replica-exchange and PIMD runs
// What a run writes, by Outputs slot: the frames, a ring polymer's estimator frames, a replica exchange's walker
// frames, final walker labels and counts, an NPT run's cell and pressure frames, then a metadynamics run's CV and
// bias-energy frames.
enum RunOut {
  OUT_R, OUT_V, OUT_EPOT, OUT_EKIN, OUT_KPRIM, OUT_KCV, OUT_WALKER_F, OUT_WALKERS, OUT_NACC, OUT_NATT, OUT_CELL,
  OUT_PRESS, OUT_CV, OUT_BIAS, N_RUN_OUTS
};

// The run's constants, once on the host in double precision.  First the fields MdParams and PimdParams share.
template <class P>
void run_params(P& p, const sgdml_b200_md* md, double dt, uint64_t seed, int64_t n_frames, int64_t stride,
                const Outputs& out) {
  p.h = 0.5 * dt;
  p.key[0] = (uint32_t)seed;
  p.key[1] = (uint32_t)(seed >> 32);
  p.stride = n_frames > 0 ? (int)stride : 0;
  p.run_start = md->step_host;
  p.R_f = out.dev(OUT_R);
  p.V_f = out.dev(OUT_V);
  p.Ep_f = out.dev(OUT_EPOT);
  p.Ek_f = out.dev(OUT_EKIN);
}

// MD: c1 and the (n_temps, 3N) sigma table, one row per temperature kT[k] (n_temps = 1 for sgdml_b200_md_run); returns
// the end of what it filled
const double* md_params(sgdml_b200_md* md, double dt, double gamma, const double* kT, int n_temps) {
  MdParams& p = md->params(md->hblk)->md;
  double* sigma = md->sigma(md->hblk);
  const int dimi = md->dimi;
  p.c1 = std::exp(-gamma * dt);
  p.use_O = gamma > 0.0 ? 1 : 0;
  p.n_temps = n_temps;
  for (int k = 0; k < n_temps; ++k)
    for (int i = 0; i < dimi; ++i)
      sigma[(size_t)k * dimi + i] = std::sqrt((1.0 - p.c1 * p.c1) * kT[k] * md->s_host[(size_t)i]);
  return sigma + (size_t)n_temps * dimi;
}

// What a replica-exchange run (sgdml_b200_remd_run) adds to an MD run: its ladder (kT on the host, checked) and its
// schedule.
struct RemdRun {
  int n_temps;
  const double* kT;
  int64_t every;
};

// the replica-exchange state, made at the first replica-exchange call, which sets the walker labels to the identity
int remd_alloc(sgdml_b200_md* md, cudaStream_t s) {
  const size_t n = (size_t)md->n_rep;
  if (md->xcount == nullptr) SG_CUDA(cached_malloc(&md->xcount, 2 * sizeof(int64_t) * n));
  if (md->walker == nullptr) {
    SG_CUDA(cached_malloc(&md->walker, sizeof(int) * n));
    k_remd_identity<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(md->walker, md->n_rep);
    SG_CUDA(cudaGetLastError());
    count_launch(KID_MISC);
  }
  return 0;
}

// the exchange's parameters and ladder (after run_params and md_params); beta and lam are computed here, on the host
// in double precision.  Returns the end of what it filled.
const double* remd_params(sgdml_b200_md* md, const RemdRun& x, const Outputs& out) {
  const int nt = x.n_temps;
  StepParams& hp = *md->params(md->hblk);
  const MdParams& p = hp.md;
  RemdParams& q = hp.remd;
  q.key[0] = p.key[0];
  q.key[1] = p.key[1];
  q.run_start = p.run_start;
  q.stride = p.stride;
  q.every = x.every;
  q.n_temps = nt;
  double *beta = md->ladder(md->hblk), *up = beta + md->rows, *dn = up + md->rows;
  for (int k = 0; k < nt; ++k) beta[k] = 1.0 / x.kT[k];
  for (int k = 0; k + 1 < nt; ++k) {
    up[k] = std::sqrt(x.kT[k + 1] / x.kT[k]);
    dn[k] = std::sqrt(x.kT[k] / x.kT[k + 1]);
  }
  q.beta = md->ladder(md->blk);
  q.lam_up = q.beta + md->rows;
  q.lam_dn = q.lam_up + md->rows;
  q.n_acc = md->xcount;
  q.n_att = md->xcount + md->n_rep;
  q.W_f = out.dev<int>(OUT_WALKER_F);
  return dn + (nt - 1);
}

// What an NPT run (sgdml_b200_npt_run) adds to an MD run: the barostat's target pressure, compressibility and time
// constant, checked.
struct NptRun {
  double P0, beta_T, tau_p;
};

// the barostat's constants, on the host in double precision (after run_params)
void npt_params(sgdml_b200_md* md, const NptRun& b, double dt, double kT, const Outputs& out) {
  NptParams& q = md->params(md->hblk)->npt;
  const double rate = b.beta_T / b.tau_p;
  q.P0 = b.P0;
  q.c_a = rate * dt;
  q.c_b = 2.0 * kT * rate * dt;
  q.cell_f = out.dev(OUT_CELL);
  q.P_f = out.dev(OUT_PRESS);
}

// What a metadynamics run (sgdml_b200_metad_run) adds to an MD run: the deposition, checked, and the hills it deposits
// per walker.
struct MetadRun {
  double w0, dkT;
  const double* widths;
  int64_t pace, n_dep;
};

// the deposit's constants and the frame outputs (the CVs and the store's pointers are the handle's, already there)
void metad_params(sgdml_b200_md* md, const MetadRun& m, const Outputs& out) {
  MetadParams& q = md->params(md->hblk)->metad;
  q.w0 = m.w0;
  q.dkT = m.dkT;
  q.pace = m.pace;
  for (int j = 0; j < q.n_cv; ++j) q.width[j] = m.widths[j];
  q.cv_f = out.dev(OUT_CV);
  q.bias_f = out.dev(OUT_BIAS);
}

// An umbrella run (sgdml_b200_umbrella_run): RemdParams' schedule, counters and walker frames, one temperature's beta,
// and the CV and restraint frames (after run_params; the CVs and the window table are the handle's, already there)
void umbrella_params(sgdml_b200_md* md, int64_t every, double kT, const Outputs& out) {
  StepParams& hp = *md->params(md->hblk);
  const MdParams& p = hp.md;
  RemdParams& x = hp.remd;
  UmbrellaParams& q = hp.umbrella;
  x.key[0] = p.key[0];
  x.key[1] = p.key[1];
  x.run_start = p.run_start;
  x.stride = p.stride;
  x.every = every;
  x.n_temps = q.n_windows;
  x.beta = x.lam_up = x.lam_dn = nullptr;
  x.n_acc = md->xcount;
  x.n_att = md->xcount + md->n_rep;
  x.W_f = out.dev<int>(OUT_WALKER_F);
  q.beta = kT > 0.0 ? 1.0 / kT : 0.0;
  q.cv_f = out.dev(OUT_CV);
  q.bias_f = out.dev(OUT_BIAS);
}

// Grows every group's hill store to at least `need` slots, keeping its hills, before anything of the call is queued.
// The store's pointers and capacity are in the mirror's MetadParams, which the caller uploads.
int metad_reserve(sgdml_b200_md* md, int64_t need) {
  MetadParams& q = md->params(md->hblk)->metad;
  if (need <= q.cap) return 0;
  const int64_t cap = std::max(need, 2 * q.cap);
  const size_t nc = (size_t)q.n_cv, G = (size_t)md->n_groups;
  double *c = nullptr, *w = nullptr, *h = nullptr;
  SG_CUDA(cudaDeviceSynchronize());  // queued work may still use the old store
  SG_CUDA(cached_malloc(&c, sizeof(double) * G * cap * nc));
  SG_CUDA(cached_malloc(&w, sizeof(double) * G * cap * nc));
  SG_CUDA(cached_malloc(&h, sizeof(double) * G * cap));
  if (q.cap > 0) {
    const size_t rc = sizeof(double) * q.cap * nc, rh = sizeof(double) * q.cap;
    SG_CUDA(cudaMemcpy2D(c, sizeof(double) * cap * nc, md->hc, rc, rc, G, cudaMemcpyDeviceToDevice));
    SG_CUDA(cudaMemcpy2D(w, sizeof(double) * cap * nc, md->hw, rc, rc, G, cudaMemcpyDeviceToDevice));
    SG_CUDA(cudaMemcpy2D(h, sizeof(double) * cap, md->hh, rh, rh, G, cudaMemcpyDeviceToDevice));
  }
  cached_free(md->hc);
  cached_free(md->hw);
  cached_free(md->hh);
  md->hc = q.centers = c;
  md->hw = q.widths = w;
  md->hh = q.heights = h;
  q.cap = cap;
  return 0;
}

// PIMD: the estimator constants, C, the mode tables and the (P, 3N) sigma table (tests/pimd_oracle.py restates them);
// returns the end of what it filled
const double* pimd_params(sgdml_b200_md* md, const Outputs& out, double dt, double kT, double hbar, double gamma,
                          double lambda) {
  const int nb = md->nb, dimi = md->dimi;
  PimdParams& p = md->params(md->hblk)->pimd;
  double* sigma = md->sigma(md->hblk);
  const double h = 0.5 * dt;
  const double kTP = nb * kT;
  const double wP = kTP / hbar;
  p.use_O = gamma > 0.0 || (lambda > 0.0 && nb > 1) ? 1 : 0;
  p.kprim0 = 0.5 * (double)(dimi * nb) * kT;
  p.kspring = 0.5 * wP * wP / nb;
  p.kcv0 = 0.5 * dimi * kT;
  p.kvir = 0.5 / nb;
  p.Kp_f = out.dev(OUT_KPRIM);
  p.Kcv_f = out.dev(OUT_KCV);
  double* C = md->tab(md->hblk);
  double *m_cos = C + nb * nb, *m_sow = m_cos + nb, *m_msin = m_sow + nb, *m_c1 = m_msin + nb;
  for (int j = 0; j < nb; ++j)
    for (int k = 0; k < nb; ++k) {
      double c;
      if (k == 0)
        c = std::sqrt(1.0 / nb);
      else if (2 * k < nb)
        c = std::sqrt(2.0 / nb) * std::cos(2.0 * M_PI * j * k / nb);
      else if (2 * k == nb)
        c = std::sqrt(1.0 / nb) * (j % 2 ? -1.0 : 1.0);
      else
        c = std::sqrt(2.0 / nb) * std::sin(2.0 * M_PI * j * k / nb);
      C[j * nb + k] = c;
    }
  for (int k = 0; k < nb; ++k) {
    double g = gamma;
    m_cos[k] = 1.0;
    m_sow[k] = h;
    m_msin[k] = 0.0;
    if (k > 0) {
      const double wk = 2.0 * wP * std::sin(M_PI * k / nb);
      m_cos[k] = std::cos(wk * h);
      m_sow[k] = std::sin(wk * h) / wk;
      m_msin[k] = -wk * std::sin(wk * h);
      g = 2.0 * lambda * wk;
    }
    m_c1[k] = std::exp(-g * dt);
    for (int i = 0; i < dimi; ++i)
      sigma[(size_t)k * dimi + i] = std::sqrt((1.0 - m_c1[k] * m_c1[k]) * kTP * md->s_host[(size_t)i]);
  }
  return sigma + (size_t)nb * dimi;
}

// Which kinds of handle an entry point accepts: the rows of the table next to sgdml_b200_md_create in
// include/sgdml_b200.h, each with the creators of its kinds for the refusal.
struct Accepts {
  unsigned kinds;  // bit k: HandleKind k
  const char* needs;
};
constexpr Accepts ANY_KIND = {1u << PLAIN | 1u << RING | 1u << NPT | 1u << METAD | 1u << UMBRELLA, "a handle"};
constexpr Accepts PLAIN_KIND = {1u << PLAIN, "a handle of sgdml_b200_md_create (or sgdml_b200_pimd_create, one bead)"};
constexpr Accepts PLAIN_OR_RING = {1u << PLAIN | 1u << RING, "a handle of sgdml_b200_md_create or _pimd_create"};
constexpr Accepts NPT_KIND = {1u << NPT, "an NPT handle (sgdml_b200_npt_create)"};
constexpr Accepts METAD_KIND = {1u << METAD, "a metadynamics handle (sgdml_b200_metad_create)"};
constexpr Accepts UMBRELLA_KIND = {1u << UMBRELLA, "an umbrella handle (sgdml_b200_umbrella_create)"};

// the first check of every entry point that takes a handle
int check_kind(const sgdml_b200_md* md, const char* entry, const Accepts& a) {
  SG_ARG(md != nullptr);
  if ((a.kinds >> md->kind & 1u) == 0) return fail_arg((std::string(entry) + " needs " + a.needs).c_str());
  return 0;
}

// One call of md_run: the arguments every run shares, then those only one integrator reads
struct Run {
  int64_t n_steps, stride;
  double dt, kT, gamma;  // kT: a replica exchange's first temperature
  uint64_t seed;
  void* outs[N_RUN_OUTS];
  double hbar, lambda;  // MD_RING_POLYMER
  RemdRun remd;         // MD_REMD; MD_UMBRELLA: n_temps = n_windows and every (kT unused)
  NptRun npt;           // MD_NPT
  MetadRun metad;       // MD_METAD
};

// the checks every run shares; a rejected call queues nothing
int run_check(const sgdml_b200_md* md, const Run& r, const char* entry) {
  SG_ARG(r.n_steps >= 0 && r.stride >= 0 && r.stride <= INT32_MAX);
  SG_ARG(std::isfinite(r.dt) && r.dt > 0.0);
  SG_ARG(std::isfinite(r.kT) && r.kT >= 0.0);
  if (md->nb == 1 && r.kT > 0.0 && r.gamma == 0.0)
    return fail_arg("kT > 0 needs a friction gamma > 0 (a thermostat without coupling)");
  if (r.stride > 0 && r.n_steps % r.stride != 0) return fail_arg("n_steps must be a multiple of stride");
  if (!md->has_state) return fail_arg((std::string(entry) + ": no state yet (call sgdml_b200_md_set_state)").c_str());
  return 0;
}

// sgdml_b200_md_run (MD_CLASSICAL), _pimd_run (MD_RING_POLYMER), _remd_run (MD_REMD), _npt_run (MD_NPT),
// _metad_run (MD_METAD) and _umbrella_run (MD_UMBRELLA), after their checks: n_steps steps, then the completing launch.
int md_run(sgdml_b200_md* md, int kind, const Run& r, cudaStream_t s) {
  const bool exch = kind == MD_REMD || kind == MD_UMBRELLA;
  if (r.n_steps == 0 && !exch) return 0;  // (an exchange run still reports its labels and zero counts)
  md->group = exch ? r.remd.n_temps : 1;
  const int64_t n_rep = md->n_rep, n_frames = r.stride > 0 ? r.n_steps / r.stride : 0;
  const size_t fr = sizeof(double) * (size_t)(n_frames * n_rep);
  const size_t fp = sizeof(double) * (size_t)(n_frames * (n_rep / md->nb));
  const size_t nc = sizeof(int64_t) * (size_t)(n_rep / md->group * (md->group - 1));  // (n_ladders, n_temps - 1)
  const int n_cv = kind == MD_METAD     ? md->params(md->hblk)->metad.n_cv
                   : kind == MD_UMBRELLA ? md->params(md->hblk)->umbrella.n_cv
                                         : 0;
  void* const* outs = r.outs;
  Outputs out(s);
  SG_TRY(out.init({{outs[OUT_R], fr * md->dimi}, {outs[OUT_V], fr * md->dimi}, {outs[OUT_EPOT], fr},
                   {outs[OUT_EKIN], fr}, {outs[OUT_KPRIM], fp}, {outs[OUT_KCV], fp},
                   {outs[OUT_WALKER_F], sizeof(int) * (size_t)(n_frames * n_rep)},
                   {outs[OUT_WALKERS], sizeof(int) * (size_t)n_rep}, {outs[OUT_NACC], nc}, {outs[OUT_NATT], nc},
                   {outs[OUT_CELL], 9 * fr}, {outs[OUT_PRESS], fr}, {outs[OUT_CV], fr * n_cv}, {outs[OUT_BIAS], fr}}));
  SG_TRY(force_eval_prepare(md->fe));
  if (kind == MD_REMD) {
    SG_TRY(reserve(md, r.remd.n_temps));
    SG_TRY(remd_alloc(md, s));
  }
  if (exch) SG_CUDA(cudaMemsetAsync(md->xcount, 0, 2 * sizeof(int64_t) * (size_t)n_rep, s));  // the run's counts
  SG_CUDA(cudaEventSynchronize(md->uploaded));  // the previous call has read the mirror
  if (kind == MD_METAD) {
    int64_t need = 0;
    for (int64_t c : md->hcount_host) need = std::max(need, c);
    SG_TRY(metad_reserve(md, need + (int64_t)md->params(md->hblk)->metad.n_walkers * r.metad.n_dep));
  }
  StepParams& p = *md->params(md->hblk);
  const double* end;
  if (kind == MD_RING_POLYMER) {
    run_params(p.pimd, md, r.dt, r.seed, n_frames, r.stride, out);
    end = pimd_params(md, out, r.dt, r.kT, r.hbar, r.gamma, r.lambda);
  } else {
    run_params(p.md, md, r.dt, r.seed, n_frames, r.stride, out);
    end = kind == MD_REMD ? md_params(md, r.dt, r.gamma, r.remd.kT, r.remd.n_temps)
                          : md_params(md, r.dt, r.gamma, &r.kT, 1);
    switch (kind) {
      case MD_REMD: end = remd_params(md, r.remd, out); break;
      case MD_NPT: npt_params(md, r.npt, r.dt, r.kT, out); break;
      case MD_METAD: metad_params(md, r.metad, out); break;
      case MD_UMBRELLA: umbrella_params(md, r.remd.every, r.kT, out); break;
    }
  }
  SG_TRY(upload(md, end, s));
  if (r.n_steps > 0) {
    SG_TRY(md_replay(md, kind, r.n_steps, s));
    md->step_host += (uint64_t)r.n_steps;
    SG_TRY(md_integrate(md, kind, 0, s));  // the second half-kick of the last step (and its frame)
    if (kind == MD_METAD && r.metad.n_dep > 0) {  // the run's hills become committed
      const int64_t add = (int64_t)md->params(md->hblk)->metad.n_walkers * r.metad.n_dep;
      k_metad_commit<<<(unsigned)((md->n_groups + 255) / 256), 256, 0, s>>>(md->hcount, md->n_groups, add);
      SG_CUDA(cudaGetLastError());
      count_launch(KID_MISC);
      for (int64_t& c : md->hcount_host) c += add;
    }
  }
  if (exch) SG_TRY(out.copy_from(OUT_WALKERS, {md->walker, md->xcount, md->xcount + n_rep}));
  return out.finish();
}

// ------------------------------------------------------------------ geometry optimisation (sgdml_b200_relax_*)
constexpr int64_t RELAX_BLOCK = 16;  // replays between convergence read-backs
int64_t g_relax_block = 0;           // sgdml_b200_set_relax_block (test hook): 0 = RELAX_BLOCK

// the optimiser state, made at the first relaxation; the L-BFGS ring grows to `memory` pairs per replica, and the NEB,
// dimer and IRC buffers are made at the first call of that kind
int relax_alloc(sgdml_b200_md* md, int memory, int kind) {
  const bool neb = kind == MD_NEB_FIRE, dimer = kind == MD_DIMER;
  if (kind == MD_IRC && md->istate == nullptr) {
    const size_t st = sizeof(double) * (size_t)(md->n_rep * md->dimi);
    for (double** p : {&md->irc_rn, &md->irc_fn, &md->irc_k}) SG_CUDA(cached_malloc(p, st));
    SG_CUDA(cached_malloc(&md->irc_v, st / 2));
    SG_CUDA(cached_malloc(&md->ibad, sizeof(int) * (size_t)(md->n_rep / 2)));
    SG_CUDA(cached_malloc(&md->istate, sizeof(IrcState) * (size_t)md->n_rep));
  }
  if (md->rst == nullptr) SG_CUDA(cached_malloc(&md->rst, sizeof(RelaxState) * (size_t)md->n_rep));
  if (md->hActive == nullptr) {
    SG_CUDA(cudaHostAlloc(&md->hActive, sizeof(int), cudaHostAllocMapped));
    SG_CUDA(cudaHostGetDevicePointer((void**)&md->dActive, md->hActive, 0));
  }
  if (md->counted == nullptr) SG_CUDA(cudaEventCreateWithFlags(&md->counted, cudaEventDisableTiming));
  if (neb) {
    if (md->climb_idx == nullptr) SG_CUDA(cached_malloc(&md->climb_idx, sizeof(int) * (size_t)md->n_rep));
  }
  if ((neb || dimer) && md->Fn == nullptr)
    SG_CUDA(cached_malloc(&md->Fn, sizeof(double) * (size_t)(md->n_rep * md->dimi)));
  if (dimer && md->dstate == nullptr) {
    const size_t nd = (size_t)(md->n_rep / 2);
    SG_CUDA(cached_malloc(&md->dmode, sizeof(double) * nd * md->dimi));
    SG_CUDA(cached_malloc(&md->dtheta, sizeof(double) * nd * md->dimi));
    SG_CUDA(cached_malloc(&md->dbad, sizeof(int) * nd));
    SG_CUDA(cached_malloc(&md->dstate, sizeof(DimerState) * nd));
  }
  if (memory > md->m_cap) {
    const size_t vec = sizeof(double) * (size_t)(md->n_rep * md->dimi);
    SG_CUDA(cudaDeviceSynchronize());  // the old ring goes back to the cache: nothing may still use it
    for (double** p : {&md->S, &md->Y, &md->rho}) {
      cached_free(*p);
      *p = nullptr;
    }
    md->m_cap = 0;
    SG_CUDA(cached_malloc(&md->S, vec * memory));
    SG_CUDA(cached_malloc(&md->Y, vec * memory));
    SG_CUDA(cached_malloc(&md->rho, sizeof(double) * (size_t)md->n_rep * memory));
    if (md->r_prev == nullptr) {
      SG_CUDA(cached_malloc(&md->r_prev, vec));
      SG_CUDA(cached_malloc(&md->g_prev, vec));
    }
    md->m_cap = memory;
  }
  return 0;
}

// What a dimer search (sgdml_b200_dimer_fire) adds to relax_impl: the caller's modes (null: the handle's) and its
// outputs per dimer.
struct DimerRun {
  const double* modes;
  double* curvature_out;
  int64_t* n_rot_out;
  double* modes_out;
};

// The start of a dimer search, after the upload: k_dimer_init on scratch (the modes into Fn's first n_dimers rows,
// the images into the next), the verdict read back, and only then the commit -- modes, images, a zero DimerState --
// and one un-captured force evaluation of every replica.  A bad mode is an argument error with the handle unchanged.
// A rejected call has still overwritten dtheta (the caller's modes in transit), Fn (the scratch rows) and the dimer
// part of the upload block: none of them carries anything from one call to the next -- every dimer call rewrites all
// three before it reads them, and Fn's rows are rewritten by every NEB force evaluation -- so keep it that way when
// using them across calls.
int dimer_start(sgdml_b200_md* md, const double* modes, cudaStream_t s) {
  const int64_t nd = md->n_rep / 2;
  const size_t row = sizeof(double) * (size_t)md->dimi, rows = row * (size_t)nd;
  const double* src = md->dmode;
  if (modes != nullptr) {
    SG_CUDA(cudaMemcpyAsync(md->dtheta, modes, rows, cudaMemcpyDefault, s));
    src = md->dtheta;
  }
  double* nd_s = md->Fn;
  double* img_s = md->Fn + nd * md->dimi;
  k_dimer_init<<<(unsigned)nd, MD_THREADS, 0, s>>>(&md->params(md->blk)->dimer, md->R, src, nd_s, img_s, md->dbad,
                                                    md->dimi);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  std::vector<int> bad((size_t)nd);
  SG_CUDA(cudaMemcpyAsync(bad.data(), md->dbad, sizeof(int) * (size_t)nd, cudaMemcpyDeviceToHost, s));
  SG_CUDA(cudaStreamSynchronize(s));
  for (int b : bad)
    if (b) return fail_arg("sgdml_b200_dimer_fire: every mode must be finite and not (almost) a rigid motion");
  SG_CUDA(cudaMemcpyAsync(md->dmode, nd_s, rows, cudaMemcpyDeviceToDevice, s));
  SG_CUDA(cudaMemcpy2DAsync(md->R + md->dimi, 2 * row, img_s, row, row, (size_t)nd, cudaMemcpyDeviceToDevice, s));
  SG_CUDA(cudaMemsetAsync(md->dstate, 0, sizeof(DimerState) * (size_t)nd, s));
  md->has_modes = true;
  return md_state_forces(md, 0, s);
}

// What an IRC call (sgdml_b200_irc_rk4) adds to relax_impl: the caller's modes and its outputs per branch.
struct IrcRun {
  const double* modes;
  double *R_path, *E_path;
};

// The start of an IRC call, after the upload: the modes into irc_v, k_irc_init's check on them, the verdict read back,
// and only then its commit and one un-captured force evaluation of every replica (point 1).  A bad mode is an argument
// error with the handle unchanged; a rejected call has overwritten only irc_v, ibad and the IRC part of the upload
// block, which every IRC call rewrites before reading them.
int irc_start(sgdml_b200_md* md, const double* modes, cudaStream_t s) {
  const int64_t np = md->n_rep / 2;
  SG_CUDA(cudaMemcpyAsync(md->irc_v, modes, sizeof(double) * (size_t)(np * md->dimi), cudaMemcpyDefault, s));
  const IrcParams* q = &md->params(md->blk)->irc;
  for (int commit = 0; commit < 2; ++commit) {
    k_irc_init<<<(unsigned)np, MD_THREADS, 0, s>>>(q, md->s, md->R, md->F, md->E, md->irc_v, md->ibad, md->irc_rn,
                                                   md->irc_fn, md->istate, md->dimi, commit);
    SG_CUDA(cudaGetLastError());
    count_launch(KID_MISC);
    if (commit) break;
    std::vector<int> bad((size_t)np);
    SG_CUDA(cudaMemcpyAsync(bad.data(), md->ibad, sizeof(int) * (size_t)np, cudaMemcpyDeviceToHost, s));
    SG_CUDA(cudaStreamSynchronize(s));
    for (int b : bad)
      if (b) return fail_arg("sgdml_b200_irc_rk4: every mode must be finite with a nonzero mass-weighted norm");
  }
  return md_state_forces(md, 0, s);
}

// Relaxes every replica (or NEB band, or dimer) from the handle's state: blocks of step-graph replays, each followed
// by the convergence test and a count of unconverged units read back through mapped pinned memory; stops when none is
// left or after max_steps.  The unit of convergence is a group of g consecutive replicas: g = 1 for relaxation, g = P
// for NEB (whose climbing_out gets each band's highest interior image), g = 2 for the dimer (dm: its modes and
// outputs), g = 1 for the IRC (ir: its modes and outputs; n_steps_out and conv_out get n_points and end).  call: the
// entry point's RelaxParams (FIRE, L-BFGS; the handle's L-BFGS ring is added here), NebParams (NEB), DimerParams
// (dimer) or IrcParams (IRC; the path outputs are added here).  memory: L-BFGS pairs per replica to allocate (0: none).
// Frozen units make the block length a matter of cost only.  V is zero before and after.
int relax_impl(sgdml_b200_md* md, int kind, int g, int memory, const StepParams& call, int64_t max_steps,
               int64_t* n_steps_out, int* conv_out, double* fmax_out, int* climbing_out, cudaStream_t s,
               const DimerRun* dm = nullptr, const IrcRun* ir = nullptr) {
  md->group = g;
  const int64_t n_rep = md->n_rep;
  const int64_t n_units = n_rep / g;
  SG_TRY(force_eval_prepare(md->fe));
  SG_TRY(relax_alloc(md, memory, kind));
  Outputs out(s);
  const size_t un = (size_t)n_units;
  SG_TRY(out.init({{n_steps_out, sizeof(int64_t) * un}, {conv_out, sizeof(int) * un},
                   {fmax_out, sizeof(double) * un}, {climbing_out, sizeof(int) * un},
                   {dm ? dm->curvature_out : nullptr, sizeof(double) * un},
                   {dm ? dm->n_rot_out : nullptr, sizeof(int64_t) * un},
                   {dm ? dm->modes_out : nullptr, sizeof(double) * un * md->dimi},
                   {ir ? ir->R_path : nullptr, sizeof(double) * un * (size_t)(call.irc.max_points * md->dimi)},
                   {ir ? ir->E_path : nullptr, sizeof(double) * un * (size_t)call.irc.max_points}}));
  SG_CUDA(cudaEventSynchronize(md->uploaded));  // the previous call has read the mirror
  StepParams& p = *md->params(md->hblk);
  if (kind == MD_NEB_FIRE) {
    p.neb = call.neb;
  } else if (kind == MD_DIMER) {
    p.dimer = call.dimer;
  } else if (kind == MD_IRC) {
    p.irc = call.irc;
    p.irc.R_path = out.dev(7);
    p.irc.E_path = out.dev(8);
  } else {
    p.relax = call.relax;
    p.relax.m_cap = md->m_cap;
    p.relax.S = md->S;
    p.relax.Y = md->Y;
    p.relax.rho = md->rho;
    p.relax.r_prev = md->r_prev;
    p.relax.g_prev = md->g_prev;
  }
  SG_TRY(upload(md, &p + 1, s));
  if (kind == MD_DIMER) SG_TRY(dimer_start(md, dm->modes, s));
  if (kind == MD_IRC) SG_TRY(irc_start(md, ir->modes, s));
  const size_t st = sizeof(double) * (size_t)(n_rep * md->dimi);
  SG_CUDA(cudaMemsetAsync(md->rst, 0, sizeof(RelaxState) * (size_t)n_units, s));
  SG_CUDA(cudaMemsetAsync(md->V, 0, st, s));
  const int64_t block = g_relax_block > 0 ? g_relax_block : RELAX_BLOCK;
  for (int64_t done = 0;;) {
    SG_TRY(md_integrate(md, kind, 0, s));  // the test on the current forces
    k_relax_count<<<1, MD_THREADS, 0, s>>>(md->rst, n_units, md->dActive);
    SG_CUDA(cudaGetLastError());
    count_launch(KID_MISC);
    SG_CUDA(cudaEventRecord(md->counted, s));
    SG_CUDA(cudaEventSynchronize(md->counted));
    if (*(volatile int*)md->hActive == 0 || done >= max_steps) break;
    const int64_t n = std::min(block, max_steps - done);
    SG_TRY(md_replay(md, kind, n, s));
    done += n;
  }
  SG_CUDA(cudaMemsetAsync(md->V, 0, st, s));  // a following MD run starts at rest
  k_relax_report<<<(unsigned)((n_units + 255) / 256), 256, 0, s>>>(md->rst, n_units, out.dev<int64_t>(0),
                                                                  out.dev<int>(1), out.dev<double>(2));
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  SG_TRY(out.copy_from(3, {md->climb_idx}));  // the last test ran k_neb_force at the final positions
  if (kind == MD_DIMER) {
    k_dimer_report<<<(unsigned)((n_units + 255) / 256), 256, 0, s>>>(md->dstate, n_units, out.dev<double>(4),
                                                                    out.dev<int64_t>(5));
    SG_CUDA(cudaGetLastError());
    count_launch(KID_MISC);
    SG_TRY(out.copy_from(6, {md->dmode}));
  }
  return out.finish();
}

// the checks both optimisers share; a rejected call queues nothing
int relax_check(const sgdml_b200_md* md, int64_t max_steps, double fmax, double maxstep, const char* entry) {
  SG_ARG(max_steps >= 0);
  SG_ARG(std::isfinite(fmax) && fmax >= 0.0);
  SG_ARG(std::isfinite(maxstep) && maxstep > 0.0);
  if (!md->has_state) return fail_arg((std::string(entry) + ": no state yet (call sgdml_b200_md_set_state)").c_str());
  return 0;
}

// A handle of the given kind, n_rep = n_poly nb replicas; the caller has checked the counts and parsed the arguments of
// its kind.  init, if given, makes the kind's own part; a failure anywhere frees the whole handle.
int md_create(sgdml_b200_md** out, sgdml_b200_model* m, HandleKind kind, int64_t n_rep, int nb, const double* inv_mass,
              const std::function<int(sgdml_b200_md*)>& init = nullptr) {
  SG_ARG(!is_device_ptr(inv_mass));
  int64_t n_atoms = 0;
  SG_TRY(sgdml_b200_model_dims(m, &n_atoms, nullptr, nullptr));
  for (int i = 0; i < n_atoms; ++i)
    if (!(std::isfinite(inv_mass[i]) && inv_mass[i] > 0.0)) return fail_arg("inv_mass must be finite and > 0");
  sgdml_b200_md* md = new sgdml_b200_md();
  md->kind = kind;
  md->n_rep = n_rep;
  md->nb = nb;
  md->dimi = 3 * (int)n_atoms;
  auto body = [&]() -> int {
    SG_TRY(force_eval_create(m, n_rep, &md->fe));
    const size_t st = sizeof(double) * (size_t)(n_rep * md->dimi);
    for (double** p : {&md->R, &md->V, &md->F, &md->Fs}) SG_CUDA(cached_malloc(p, st));
    SG_CUDA(cached_malloc(&md->E, sizeof(double) * n_rep));
    SG_CUDA(cached_malloc(&md->Es, sizeof(double) * n_rep));
    SG_CUDA(cached_malloc(&md->step, sizeof(uint64_t) * n_rep));
    SG_CUDA(cached_malloc(&md->s, sizeof(double) * md->dimi));
    SG_TRY(reserve(md, nb));
    SG_CUDA(cudaEventCreateWithFlags(&md->uploaded, cudaEventDisableTiming));
    md->s_host.resize((size_t)md->dimi);
    for (int i = 0; i < md->dimi; ++i) md->s_host[(size_t)i] = inv_mass[i / 3];
    SG_CUDA(cudaMemcpy(md->s, md->s_host.data(), sizeof(double) * md->dimi, cudaMemcpyHostToDevice));
    SG_TRY(force_eval_prepare(md->fe));
    return init ? init(md) : 0;
  };
  if (const int rc = body()) {
    md_free(md);
    return rc;
  }
  *out = md;
  return 0;
}

// The cells of an NPT handle from (n_rep, 9) HOST lattices and inverses, each checked as sgdml_b200_predict_virial_cells
// checks them: the barostat state (eps = 0, V0 = |det L0|) and the cells the descriptor kernel reads.  Nothing is queued.
int npt_parse(const double* lattices, const double* lattice_invs, int64_t n_rep, std::vector<NptCell>* cells,
              std::vector<Lattice>* lats) {
  SG_ARG(lattices != nullptr && lattice_invs != nullptr);
  SG_ARG(!is_device_ptr(lattices) && !is_device_ptr(lattice_invs));
  cells->assign((size_t)n_rep, NptCell());
  lats->assign((size_t)n_rep, Lattice());
  for (int64_t g = 0; g < n_rep; ++g) {
    Lattice& l = (*lats)[(size_t)g];
    NptCell& c = (*cells)[(size_t)g];
    l.on = 1;
    std::copy(lattices + 9 * g, lattices + 9 * g + 9, l.vec);
    std::copy(lattice_invs + 9 * g, lattice_invs + 9 * g + 9, l.inv);
    SG_TRY(check_cell(l));
    const double* a = l.vec;
    c.eps = 0.0;
    c.V0 = std::fabs(a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6]) +
                     a[2] * (a[3] * a[7] - a[4] * a[6]));
    std::copy(l.vec, l.vec + 9, c.L0);
    std::copy(l.inv, l.inv + 9, c.L0inv);
  }
  return 0;
}

// installs parsed cells on an NPT handle, and with a state evaluates F, E and W in them
int npt_install(sgdml_b200_md* md, const std::vector<NptCell>& cells, const std::vector<Lattice>& lats,
                cudaStream_t s) {
  SG_CUDA(cudaMemcpyAsync(md->cell, cells.data(), sizeof(NptCell) * cells.size(), cudaMemcpyHostToDevice, s));
  SG_CUDA(cudaMemcpyAsync(md->lat, lats.data(), sizeof(Lattice) * lats.size(), cudaMemcpyHostToDevice, s));
  if (md->has_state) {
    SG_TRY(force_eval_prepare(md->fe));
    SG_TRY(md_forces(md, md->F, md->E, md->W, s));
  }
  SG_CUDA(cudaStreamSynchronize(s));  // (the host vectors go out of scope)
  return 0;
}

// The CVs of sgdml_b200_metad_create and _umbrella_create from HOST arrays, checked: the types, and the atoms of
// each CV distinct and in [0, n_atoms).  Nothing is queued.
int cv_parse(int64_t n_cv, const int* cv_type, const int64_t* cv_atoms, int64_t n_atoms, int* type, int (*atoms)[4]) {
  SG_ARG(n_cv >= 1 && n_cv <= MD_MAX_CV);
  SG_ARG(!is_device_ptr(cv_type) && !is_device_ptr(cv_atoms));
  for (int j = 0; j < n_cv; ++j) {
    if (cv_type[j] != CV_DISTANCE && cv_type[j] != CV_ANGLE && cv_type[j] != CV_DIHEDRAL)
      return fail_arg("cv_type must be 0 (distance), 1 (angle) or 2 (dihedral)");
    type[j] = cv_type[j];
    const int na = cv_type[j] + 2;
    for (int p = 0; p < na; ++p) {
      const int64_t a = cv_atoms[4 * j + p];
      if (a < 0 || a >= n_atoms) return fail_arg("cv_atoms must lie in [0, N)");
      for (int o = 0; o < p; ++o)
        if (cv_atoms[4 * j + o] == a) return fail_arg("the atoms of a CV must be distinct");
      atoms[j][p] = (int)a;
    }
  }
  return 0;
}

// The buffers of a biased handle (metadynamics, umbrella): the model's forces Fm, the state's CVs, bias energy and
// bias force, the last zero where no CV reaches
int bias_alloc(sgdml_b200_md* md, int n_cv) {
  const size_t st = sizeof(double) * (size_t)(md->n_rep * md->dimi);
  SG_CUDA(cached_malloc(&md->Fm, st));
  SG_CUDA(cached_malloc(&md->Fb, st));
  SG_CUDA(cached_malloc(&md->cv, sizeof(double) * (size_t)(md->n_rep * n_cv)));
  SG_CUDA(cached_malloc(&md->Vb, sizeof(double) * (size_t)md->n_rep));
  SG_CUDA(cudaMemset(md->Fb, 0, st));  // the coordinates no CV touches keep a zero bias force
  return 0;
}

// The window table (centres, then force constants) of an umbrella handle from (n_windows, n_cv) HOST arrays, checked.
// Nothing is queued.
int windows_parse(int64_t n_windows, int n_cv, const int* type, const double* centers, const double* kappas,
                  std::vector<double>* win) {
  SG_TRY(umbrella_windows_check(n_windows, n_cv, type, centers, kappas));
  const size_t n = (size_t)(n_windows * n_cv);
  win->assign(centers, centers + n);
  win->insert(win->end(), kappas, kappas + n);
  return 0;
}

// The CV, bias-energy and bias-force rows of a biased handle's state
int bias_get(sgdml_b200_md* md, int n_cv, double* cv, double* V_bias, double* F_bias, const char* entry,
             cudaStream_t s) {
  if (!md->has_state) return fail_arg((std::string(entry) + ": no state yet (call sgdml_b200_md_set_state)").c_str());
  const size_t n = (size_t)md->n_rep;
  Outputs out(s);
  SG_TRY(out.init({{cv, sizeof(double) * n * n_cv}, {V_bias, sizeof(double) * n}, {F_bias, sizeof(double) * n * md->dimi}}));
  SG_TRY(out.copy_from(0, {md->cv, md->Vb, md->Fb}));
  return out.finish();
}

}  // namespace

extern "C" {

int sgdml_b200_md_create(sgdml_b200_md** out, sgdml_b200_model* m, int64_t n_rep, const double* inv_mass) {
  SG_TRY(require_device());
  SG_ARG(out != nullptr && m != nullptr && inv_mass != nullptr);
  SG_ARG(n_rep >= 1 && n_rep <= INT32_MAX);
  return md_create(out, m, PLAIN, n_rep, 1, inv_mass);
}

int sgdml_b200_pimd_create(sgdml_b200_md** out, sgdml_b200_model* m, int64_t n_poly, int64_t n_beads,
                           const double* inv_mass) {
  SG_TRY(require_device());
  SG_ARG(out != nullptr && m != nullptr && inv_mass != nullptr);
  SG_ARG(n_beads >= 1 && n_beads <= PIMD_MAX_BEADS);
  SG_ARG(n_poly >= 1 && n_poly <= INT32_MAX / n_beads);
  return md_create(out, m, n_beads > 1 ? RING : PLAIN, n_poly * n_beads, (int)n_beads, inv_mass);
}

int sgdml_b200_npt_create(sgdml_b200_md** out, sgdml_b200_model* m, int64_t n_rep, const double* inv_mass,
                          const double* lattices, const double* lattice_invs) {
  SG_TRY(require_device());
  SG_ARG(out != nullptr && m != nullptr && inv_mass != nullptr);
  SG_ARG(n_rep >= 1 && n_rep <= INT32_MAX);
  std::vector<NptCell> cells;
  std::vector<Lattice> lats;
  SG_TRY(npt_parse(lattices, lattice_invs, n_rep, &cells, &lats));
  return md_create(out, m, NPT, n_rep, 1, inv_mass, [&](sgdml_b200_md* md) -> int {
    SG_CUDA(cached_malloc(&md->cell, sizeof(NptCell) * (size_t)n_rep));
    SG_CUDA(cached_malloc(&md->lat, sizeof(Lattice) * (size_t)n_rep));
    SG_CUDA(cached_malloc(&md->W, sizeof(double) * 9 * (size_t)n_rep));
    SG_CUDA(cached_malloc(&md->Ws, sizeof(double) * 9 * (size_t)n_rep));
    SG_CUDA(cudaMemset(md->W, 0, sizeof(double) * 9 * (size_t)n_rep));
    return npt_install(md, cells, lats, 0);
  });
}

int sgdml_b200_npt_set_cells(sgdml_b200_md* md, const double* lattices, const double* lattice_invs, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_npt_set_cells", NPT_KIND));
  std::vector<NptCell> cells;
  std::vector<Lattice> lats;
  SG_TRY(npt_parse(lattices, lattice_invs, md->n_rep, &cells, &lats));
  return npt_install(md, cells, lats, (cudaStream_t)stream);
}

int sgdml_b200_npt_get_cells(sgdml_b200_md* md, double* lattices, double* lattice_invs, double* W, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_npt_get_cells", NPT_KIND));
  cudaStream_t s = (cudaStream_t)stream;
  const size_t row = 9 * sizeof(double), n = (size_t)md->n_rep;
  Outputs out(s);
  SG_TRY(out.init({{lattices, row * n}, {lattice_invs, row * n}, {W, row * n}}));
  const char* base = reinterpret_cast<const char*>(md->lat);
  const size_t off[2] = {offsetof(Lattice, vec), offsetof(Lattice, inv)};
  for (int k = 0; k < 2; ++k)
    if (out.dev(k) != nullptr)
      SG_CUDA(cudaMemcpy2DAsync(out.dev(k), row, base + off[k], sizeof(Lattice), row, n, cudaMemcpyDeviceToDevice, s));
  SG_TRY(out.copy_from(2, {md->W}));
  return out.finish();
}

int sgdml_b200_metad_create(sgdml_b200_md** out, sgdml_b200_model* m, int64_t n_groups, int64_t n_walkers,
                            const double* inv_mass, int64_t n_cv, const int* cv_type, const int64_t* cv_atoms) {
  SG_TRY(require_device());
  SG_ARG(out != nullptr && m != nullptr && inv_mass != nullptr && cv_type != nullptr && cv_atoms != nullptr);
  SG_ARG(n_groups >= 1 && n_walkers >= 1 && n_groups <= INT32_MAX / n_walkers);
  int64_t n_atoms = 0;
  SG_TRY(sgdml_b200_model_dims(m, &n_atoms, nullptr, nullptr));
  MetadParams q = {};
  SG_TRY(cv_parse(n_cv, cv_type, cv_atoms, n_atoms, q.type, q.atoms));
  q.n_cv = (int)n_cv;
  q.n_walkers = (int)n_walkers;
  const int64_t n_rep = n_groups * n_walkers;
  return md_create(out, m, METAD, n_rep, 1, inv_mass, [&](sgdml_b200_md* md) -> int {
    SG_TRY(bias_alloc(md, (int)n_cv));
    SG_CUDA(cached_malloc(&md->hcount, sizeof(int64_t) * (size_t)n_groups));
    SG_CUDA(cudaMemset(md->hcount, 0, sizeof(int64_t) * (size_t)n_groups));
    md->n_groups = n_groups;
    md->hcount_host.assign((size_t)n_groups, 0);
    q.count = md->hcount;
    q.cv = md->cv;
    q.Vb = md->Vb;
    q.Fb = md->Fb;
    StepParams* p = md->params(md->hblk);
    p->metad = q;
    SG_TRY(upload(md, p + 1, 0));
    SG_CUDA(cudaStreamSynchronize(0));
    return 0;
  });
}

int sgdml_b200_metad_run(sgdml_b200_md* md, int64_t n_steps, double dt, double gamma, double kT, double w0,
                         const double* widths, int64_t pace, double dkT, uint64_t seed, int64_t stride,
                         double* R_frames, double* V_frames, double* E_pot_frames, double* E_kin_frames,
                         double* cv_frames, double* bias_frames, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_metad_run", METAD_KIND));
  Run r = {n_steps, stride, dt, kT, gamma, seed, {R_frames, V_frames, E_pot_frames, E_kin_frames}};
  r.outs[OUT_CV] = cv_frames;
  r.outs[OUT_BIAS] = bias_frames;
  SG_TRY(run_check(md, r, "sgdml_b200_metad_run"));
  SG_ARG(std::isfinite(gamma) && gamma >= 0.0);
  SG_ARG(std::isfinite(w0) && w0 >= 0.0);
  SG_ARG(pace >= 1);
  SG_ARG(dkT > 0.0);  // finite or +inf (NaN fails)
  SG_ARG(widths != nullptr && !is_device_ptr(widths));
  const MetadParams& q = md->params(md->hblk)->metad;
  for (int j = 0; j < q.n_cv; ++j)
    if (!(std::isfinite(widths[j]) && widths[j] > 0.0)) return fail_arg("every width must be finite and > 0");
  const uint64_t a = md->step_host, e = md->step_host + (uint64_t)n_steps, pc = (uint64_t)pace;
  r.metad = {w0, dkT, widths, pace, (int64_t)(e / pc - a / pc)};
  return md_run(md, MD_METAD, r, (cudaStream_t)stream);
}

int sgdml_b200_metad_get_hills(sgdml_b200_md* md, int64_t* n_hills, double* centers, double* widths,
                               double* heights, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_metad_get_hills", METAD_KIND));
  SG_ARG(n_hills != nullptr && !is_device_ptr(n_hills));
  cudaStream_t s = (cudaStream_t)stream;
  const MetadParams& q = md->params(md->hblk)->metad;
  const size_t nc = (size_t)q.n_cv;
  int64_t total = 0;
  for (int64_t c : md->hcount_host) total += c;
  Outputs out(s);
  SG_TRY(out.init({{centers, sizeof(double) * total * nc}, {widths, sizeof(double) * total * nc},
                   {heights, sizeof(double) * total}}));
  int64_t off = 0;
  for (int64_t g = 0; g < md->n_groups; ++g) {
    const int64_t c = md->hcount_host[(size_t)g];
    n_hills[g] = c;
    if (c == 0) continue;
    const size_t row = sizeof(double) * c * nc, src = (size_t)(g * q.cap) * nc;
    if (out.dev(0)) SG_CUDA(cudaMemcpyAsync(out.dev(0) + off * nc, md->hc + src, row, cudaMemcpyDeviceToDevice, s));
    if (out.dev(1)) SG_CUDA(cudaMemcpyAsync(out.dev(1) + off * nc, md->hw + src, row, cudaMemcpyDeviceToDevice, s));
    if (out.dev(2))
      SG_CUDA(cudaMemcpyAsync(out.dev(2) + off, md->hh + g * q.cap, sizeof(double) * c, cudaMemcpyDeviceToDevice, s));
    off += c;
  }
  return out.finish();
}

int sgdml_b200_metad_set_hills(sgdml_b200_md* md, const int64_t* n_hills, const double* centers,
                               const double* widths, const double* heights, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_metad_set_hills", METAD_KIND));
  SG_ARG(n_hills != nullptr && !is_device_ptr(n_hills));
  int64_t total = 0, need = 0;
  for (int64_t g = 0; g < md->n_groups; ++g) {
    SG_ARG(n_hills[g] >= 0);
    total += n_hills[g];
    need = std::max(need, n_hills[g]);
  }
  const int nc = md->params(md->hblk)->metad.n_cv;
  if (total > 0) {
    SG_ARG(centers != nullptr && widths != nullptr && heights != nullptr);
    SG_ARG(!is_device_ptr(centers) && !is_device_ptr(widths) && !is_device_ptr(heights));
    for (int64_t k = 0; k < total; ++k) {
      if (!std::isfinite(heights[k])) return fail_arg("every height must be finite");
      for (int j = 0; j < nc; ++j) {
        if (!std::isfinite(centers[k * nc + j])) return fail_arg("every centre must be finite");
        if (!(std::isfinite(widths[k * nc + j]) && widths[k * nc + j] > 0.0))
          return fail_arg("every width must be finite and > 0");
      }
    }
  }
  cudaStream_t s = (cudaStream_t)stream;
  SG_CUDA(cudaEventSynchronize(md->uploaded));  // the previous call has read the mirror
  SG_TRY(metad_reserve(md, need));
  StepParams* p = md->params(md->hblk);
  const MetadParams& q = p->metad;
  int64_t off = 0;
  for (int64_t g = 0; g < md->n_groups; ++g) {
    const int64_t c = n_hills[g];
    if (c == 0) continue;
    const size_t row = sizeof(double) * c * nc, dst = (size_t)(g * q.cap) * nc;
    SG_CUDA(cudaMemcpyAsync(md->hc + dst, centers + off * nc, row, cudaMemcpyHostToDevice, s));
    SG_CUDA(cudaMemcpyAsync(md->hw + dst, widths + off * nc, row, cudaMemcpyHostToDevice, s));
    SG_CUDA(cudaMemcpyAsync(md->hh + g * q.cap, heights + off, sizeof(double) * c, cudaMemcpyHostToDevice, s));
    off += c;
  }
  md->hcount_host.assign(n_hills, n_hills + md->n_groups);
  SG_CUDA(cudaMemcpyAsync(md->hcount, md->hcount_host.data(), sizeof(int64_t) * md->n_groups, cudaMemcpyHostToDevice,
                          s));
  SG_TRY(upload(md, p + 1, s));
  if (md->has_state) {
    SG_TRY(force_eval_prepare(md->fe));
    SG_TRY(md_state_forces(md, 0, s));
  }
  SG_CUDA(cudaStreamSynchronize(s));  // (the caller's arrays and the counts' host vector)
  return 0;
}

int sgdml_b200_metad_get_bias(sgdml_b200_md* md, double* cv, double* V_bias, double* F_bias, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_metad_get_bias", METAD_KIND));
  return bias_get(md, md->params(md->hblk)->metad.n_cv, cv, V_bias, F_bias, "sgdml_b200_metad_get_bias",
                  (cudaStream_t)stream);
}

int sgdml_b200_umbrella_create(sgdml_b200_md** out, sgdml_b200_model* m, int64_t n_ladders, int64_t n_windows,
                               const double* inv_mass, int64_t n_cv, const int* cv_type, const int64_t* cv_atoms,
                               const double* centers, const double* kappas) {
  SG_TRY(require_device());
  SG_ARG(out != nullptr && m != nullptr && inv_mass != nullptr && cv_type != nullptr && cv_atoms != nullptr);
  SG_ARG(n_ladders >= 1 && n_windows >= 1 && n_ladders <= INT32_MAX / n_windows);
  int64_t n_atoms = 0;
  SG_TRY(sgdml_b200_model_dims(m, &n_atoms, nullptr, nullptr));
  UmbrellaParams q = {};
  SG_TRY(cv_parse(n_cv, cv_type, cv_atoms, n_atoms, q.type, q.atoms));
  q.n_cv = (int)n_cv;
  q.n_windows = (int)n_windows;
  std::vector<double> win;
  SG_TRY(windows_parse(n_windows, q.n_cv, q.type, centers, kappas, &win));
  return md_create(out, m, UMBRELLA, n_ladders * n_windows, 1, inv_mass, [&](sgdml_b200_md* md) -> int {
    SG_TRY(bias_alloc(md, q.n_cv));
    SG_CUDA(cached_malloc(&md->win, sizeof(double) * win.size()));
    SG_CUDA(cudaMemcpy(md->win, win.data(), sizeof(double) * win.size(), cudaMemcpyHostToDevice));
    SG_TRY(remd_alloc(md, 0));
    q.win = md->win;
    q.cv = md->cv;
    q.Vb = md->Vb;
    q.Fb = md->Fb;
    StepParams* p = md->params(md->hblk);
    p->umbrella = q;
    SG_TRY(upload(md, p + 1, 0));
    SG_CUDA(cudaStreamSynchronize(0));
    return 0;
  });
}

int sgdml_b200_umbrella_set_windows(sgdml_b200_md* md, const double* centers, const double* kappas, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_umbrella_set_windows", UMBRELLA_KIND));
  const UmbrellaParams& q = md->params(md->hblk)->umbrella;
  std::vector<double> win;
  SG_TRY(windows_parse(q.n_windows, q.n_cv, q.type, centers, kappas, &win));
  cudaStream_t s = (cudaStream_t)stream;
  SG_CUDA(cudaMemcpyAsync(md->win, win.data(), sizeof(double) * win.size(), cudaMemcpyHostToDevice, s));
  if (md->has_state) SG_TRY(umbrella_bias(md, s));  // Fm is the state's: only the restraints change
  SG_CUDA(cudaStreamSynchronize(s));  // (the table's host vector goes out of scope)
  return 0;
}

int sgdml_b200_umbrella_run(sgdml_b200_md* md, int64_t n_steps, double dt, double gamma, double kT, uint64_t seed,
                            int64_t exchange_every, int64_t stride, double* R_frames, double* V_frames,
                            double* E_pot_frames, double* E_kin_frames, double* cv_frames, double* bias_frames,
                            int* walker_frames, int* walkers_out, int64_t* n_accepted, int64_t* n_attempted,
                            void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_umbrella_run", UMBRELLA_KIND));
  Run r = {n_steps, stride, dt, kT, gamma, seed,
           {R_frames, V_frames, E_pot_frames, E_kin_frames, nullptr, nullptr, walker_frames, walkers_out, n_accepted,
            n_attempted}};
  r.outs[OUT_CV] = cv_frames;
  r.outs[OUT_BIAS] = bias_frames;
  SG_TRY(run_check(md, r, "sgdml_b200_umbrella_run"));
  SG_ARG(std::isfinite(gamma) && gamma >= 0.0);
  SG_ARG(exchange_every >= 0);
  const int nw = md->params(md->hblk)->umbrella.n_windows;
  if (exchange_every > 0 && !(kT > 0.0 && nw >= 2))
    return fail_arg("sgdml_b200_umbrella_run: exchanges need kT > 0 and n_windows >= 2");
  r.remd = {nw, nullptr, exchange_every};
  return md_run(md, MD_UMBRELLA, r, (cudaStream_t)stream);
}

int sgdml_b200_umbrella_get_bias(sgdml_b200_md* md, double* cv, double* V_bias, double* F_bias, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_umbrella_get_bias", UMBRELLA_KIND));
  return bias_get(md, md->params(md->hblk)->umbrella.n_cv, cv, V_bias, F_bias, "sgdml_b200_umbrella_get_bias",
                  (cudaStream_t)stream);
}

int sgdml_b200_md_destroy(sgdml_b200_md* md) {
  if (md != nullptr) md_free(md);
  return 0;
}

int sgdml_b200_md_set_state(sgdml_b200_md* md, const double* R, const double* V, uint64_t step, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_md_set_state", ANY_KIND));
  SG_ARG(R != nullptr);
  cudaStream_t s = (cudaStream_t)stream;
  const size_t st = sizeof(double) * (size_t)(md->n_rep * md->dimi);
  SG_TRY(force_eval_prepare(md->fe));
  SG_CUDA(cudaMemcpyAsync(md->R, R, st, cudaMemcpyDefault, s));
  if (V != nullptr)
    SG_CUDA(cudaMemcpyAsync(md->V, V, st, cudaMemcpyDefault, s));
  else
    SG_CUDA(cudaMemsetAsync(md->V, 0, st, s));
  const std::vector<uint64_t> steps((size_t)md->n_rep, step);
  SG_CUDA(cudaMemcpyAsync(md->step, steps.data(), sizeof(uint64_t) * md->n_rep, cudaMemcpyHostToDevice, s));
  SG_TRY(md_state_forces(md, 0, s));
  if (md->walker != nullptr) {  // a replica exchange's walkers start again from their slots
    k_remd_identity<<<(unsigned)((md->n_rep + 255) / 256), 256, 0, s>>>(md->walker, md->n_rep);
    SG_CUDA(cudaGetLastError());
    count_launch(KID_MISC);
  }
  SG_CUDA(cudaStreamSynchronize(s));  // (the counters' host vector goes out of scope)
  md->step_host = step;
  md->has_state = true;
  return 0;
}

int sgdml_b200_md_get_state(sgdml_b200_md* md, double* R, double* V, double* F, double* E_pot, uint64_t* step,
                            void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_md_get_state", ANY_KIND));
  if (!md->has_state) return fail_arg("sgdml_b200_md_get_state: no state yet (call sgdml_b200_md_set_state)");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t st = sizeof(double) * (size_t)(md->n_rep * md->dimi);
  Outputs out(s);
  SG_TRY(out.init({{R, st}, {V, st}, {F, st}, {E_pot, sizeof(double) * md->n_rep}, {step, sizeof(uint64_t)}}));
  SG_TRY(out.copy_from(0, {md->R, md->V, md->kind == METAD || md->kind == UMBRELLA ? md->Fm : md->F, md->E, md->step}));
  return out.finish();
}

int sgdml_b200_md_run(sgdml_b200_md* md, int64_t n_steps, double dt, double gamma, double kT, uint64_t seed,
                      int64_t stride, double* R_frames, double* V_frames, double* E_pot_frames, double* E_kin_frames,
                      void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_md_run", PLAIN_KIND));
  const Run r = {n_steps, stride, dt, kT, gamma, seed, {R_frames, V_frames, E_pot_frames, E_kin_frames}};
  SG_TRY(run_check(md, r, "sgdml_b200_md_run"));
  SG_ARG(std::isfinite(gamma) && gamma >= 0.0);
  return md_run(md, MD_CLASSICAL, r, (cudaStream_t)stream);
}

int sgdml_b200_npt_run(sgdml_b200_md* md, int64_t n_steps, double dt, double gamma, double kT, double P0,
                       double beta_T, double tau_p, uint64_t seed, int64_t stride, double* R_frames,
                       double* V_frames, double* E_pot_frames, double* E_kin_frames, double* cell_frames,
                       double* P_frames, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_npt_run", NPT_KIND));
  Run r = {n_steps, stride, dt, kT, gamma, seed, {R_frames, V_frames, E_pot_frames, E_kin_frames}};
  r.outs[OUT_CELL] = cell_frames;
  r.outs[OUT_PRESS] = P_frames;
  SG_TRY(run_check(md, r, "sgdml_b200_npt_run"));
  SG_ARG(std::isfinite(gamma) && gamma >= 0.0);
  SG_ARG(std::isfinite(P0));
  SG_ARG(std::isfinite(beta_T) && beta_T >= 0.0);
  SG_ARG(std::isfinite(tau_p) && tau_p > 0.0);
  r.npt = {P0, beta_T, tau_p};
  return md_run(md, MD_NPT, r, (cudaStream_t)stream);
}

int sgdml_b200_remd_run(sgdml_b200_md* md, int64_t n_temps, const double* kT, int64_t n_steps, double dt, double gamma,
                        uint64_t seed, int64_t exchange_every, int64_t stride, double* R_frames, double* V_frames,
                        double* E_pot_frames, double* E_kin_frames, int* walker_frames, int* walkers_out,
                        int64_t* n_accepted, int64_t* n_attempted, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_remd_run", PLAIN_KIND));
  SG_ARG(kT != nullptr);
  SG_ARG(n_temps >= 2 && md->n_rep % n_temps == 0);
  SG_ARG(!is_device_ptr(kT));
  for (int64_t k = 0; k < n_temps; ++k)
    if (!(std::isfinite(kT[k]) && kT[k] > 0.0)) return fail_arg("sgdml_b200_remd_run: every kT must be finite and > 0");
  SG_ARG(std::isfinite(gamma) && gamma > 0.0);
  SG_ARG(exchange_every >= 0);
  Run r = {n_steps, stride, dt, kT[0], gamma, seed,
           {R_frames, V_frames, E_pot_frames, E_kin_frames, nullptr, nullptr, walker_frames, walkers_out, n_accepted,
            n_attempted}};
  SG_TRY(run_check(md, r, "sgdml_b200_remd_run"));
  r.remd = {(int)n_temps, kT, exchange_every};
  return md_run(md, MD_REMD, r, (cudaStream_t)stream);
}

int sgdml_b200_pimd_run(sgdml_b200_md* md, int64_t n_steps, double dt, double kT, double hbar, double gamma,
                        double lambda, uint64_t seed, int64_t stride, double* R_frames, double* V_frames,
                        double* E_pot_frames, double* E_kin_frames, double* K_prim_frames, double* K_cv_frames,
                        void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_pimd_run", PLAIN_OR_RING));
  const Run r = {n_steps, stride, dt, kT, gamma, seed,
                 {R_frames, V_frames, E_pot_frames, E_kin_frames, K_prim_frames, K_cv_frames}, hbar, lambda};
  SG_TRY(run_check(md, r, "sgdml_b200_pimd_run"));
  SG_ARG(std::isfinite(hbar) && hbar > 0.0);
  SG_ARG(std::isfinite(gamma) && gamma >= 0.0);
  SG_ARG(std::isfinite(lambda) && lambda >= 0.0);
  if (md->nb > 1 && kT == 0.0) return fail_arg("a ring polymer (n_beads > 1) needs kT > 0");
  return md_run(md, MD_RING_POLYMER, r, (cudaStream_t)stream);
}

int sgdml_b200_relax_fire(sgdml_b200_md* md, int64_t max_steps, double fmax, double maxstep, double dt, double dtmax,
                          int64_t* n_steps_out, int* converged_out, double* fmax_out, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_relax_fire", PLAIN_OR_RING));
  SG_TRY(relax_check(md, max_steps, fmax, maxstep, "sgdml_b200_relax_fire"));
  SG_ARG(std::isfinite(dt) && dt > 0.0);
  SG_ARG(std::isfinite(dtmax) && dtmax > 0.0);
  StepParams c = {};
  c.relax.fmax2 = fmax * fmax;
  c.relax.maxstep = maxstep;
  c.relax.dt0 = dt;
  c.relax.dtmax = dtmax;
  return relax_impl(md, MD_FIRE, 1, 0, c, max_steps, n_steps_out, converged_out, fmax_out, nullptr,
                    (cudaStream_t)stream);
}

int sgdml_b200_relax_lbfgs(sgdml_b200_md* md, int64_t max_steps, double fmax, double maxstep, int memory, double h0,
                           int64_t* n_steps_out, int* converged_out, double* fmax_out, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_relax_lbfgs", PLAIN_OR_RING));
  SG_TRY(relax_check(md, max_steps, fmax, maxstep, "sgdml_b200_relax_lbfgs"));
  SG_ARG(memory >= 1 && memory <= LBFGS_MAX_MEMORY);
  SG_ARG(std::isfinite(h0) && h0 > 0.0);
  StepParams c = {};
  c.relax.fmax2 = fmax * fmax;
  c.relax.maxstep = maxstep;
  c.relax.h0 = h0;
  c.relax.memory = memory;
  return relax_impl(md, MD_LBFGS, 1, memory, c, max_steps, n_steps_out, converged_out, fmax_out, nullptr,
                    (cudaStream_t)stream);
}

int sgdml_b200_neb_fire(sgdml_b200_md* md, int64_t n_images, int64_t max_steps, double fmax, double k, int climb,
                        double maxstep, double dt, double dtmax, int64_t* n_steps_out, int* converged_out,
                        double* fmax_out, int* climbing_out, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_neb_fire", PLAIN_KIND));
  SG_TRY(relax_check(md, max_steps, fmax, maxstep, "sgdml_b200_neb_fire"));
  SG_ARG(n_images >= 3 && md->n_rep % n_images == 0);
  SG_ARG((n_images - 2) * md->dimi <= INT32_MAX);
  SG_ARG(std::isfinite(k) && k >= 0.0);
  SG_ARG(std::isfinite(dt) && dt > 0.0);
  SG_ARG(std::isfinite(dtmax) && dtmax > 0.0);
  StepParams c = {};
  c.neb.fmax2 = fmax * fmax;
  c.neb.maxstep = maxstep;
  c.neb.dt0 = dt;
  c.neb.dtmax = dtmax;
  c.neb.k = k;
  c.neb.climb = climb != 0 ? 1 : 0;
  c.neb.P = (int)n_images;
  return relax_impl(md, MD_NEB_FIRE, (int)n_images, 0, c, max_steps, n_steps_out, converged_out, fmax_out,
                    climbing_out, (cudaStream_t)stream);
}

int sgdml_b200_dimer_fire(sgdml_b200_md* md, const double* modes, int64_t max_steps, double fmax, double separation,
                          double cos_trial, double sin_trial, double rot_min, double maxstep, double dt, double dtmax,
                          int64_t* n_steps_out, int* converged_out, double* fmax_out, double* curvature_out,
                          int64_t* n_rot_out, double* modes_out, void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_dimer_fire", PLAIN_KIND));
  SG_TRY(relax_check(md, max_steps, fmax, maxstep, "sgdml_b200_dimer_fire"));
  if (md->n_rep % 2 != 0) return fail_arg("sgdml_b200_dimer_fire: n_rep must be even (a centre and an image per dimer)");
  if (modes == nullptr && !md->has_modes)
    return fail_arg("sgdml_b200_dimer_fire: no modes yet (pass modes on the handle's first dimer call)");
  SG_ARG(std::isfinite(separation) && separation > 0.0);
  SG_ARG(std::isfinite(cos_trial) && cos_trial > 0.0 && std::isfinite(sin_trial) && sin_trial > 0.0);
  SG_ARG(std::fabs(cos_trial * cos_trial + sin_trial * sin_trial - 1.0) < 1e-12);
  SG_ARG(std::isfinite(rot_min) && rot_min >= 0.0);
  SG_ARG(std::isfinite(dt) && dt > 0.0);
  SG_ARG(std::isfinite(dtmax) && dtmax > 0.0);
  StepParams c = {};
  DimerParams& q = c.dimer;
  q.D = separation;
  q.c_t = cos_trial;
  q.s_t = sin_trial;
  q.s2_t = 2.0 * sin_trial * cos_trial;
  q.omc2_t = 2.0 * sin_trial * sin_trial;
  q.rot_min = rot_min;
  q.fmax2 = fmax * fmax;
  q.maxstep = maxstep;
  q.dt0 = dt;
  q.dtmax = dtmax;
  q.periodic = force_eval_periodic(md->fe) ? 1 : 0;
  const DimerRun dm = {modes, curvature_out, n_rot_out, modes_out};
  return relax_impl(md, MD_DIMER, 2, 0, c, max_steps, n_steps_out, converged_out, fmax_out, nullptr,
                    (cudaStream_t)stream, &dm);
}

int sgdml_b200_irc_rk4(sgdml_b200_md* md, const double* modes, int64_t max_points, double step, double fmax,
                       double* R_path, double* E_path, int64_t* n_points_out, int* end_out, double* fmax_out,
                       void* stream) {
  SG_TRY(require_device());
  SG_TRY(check_kind(md, "sgdml_b200_irc_rk4", PLAIN_KIND));
  if (md->n_rep % 2 != 0) return fail_arg("sgdml_b200_irc_rk4: n_rep must be even (two branches per saddle)");
  if (!md->has_state) return fail_arg("sgdml_b200_irc_rk4: no state yet (call sgdml_b200_md_set_state)");
  SG_ARG(modes != nullptr);
  SG_ARG(max_points >= 2 && max_points <= INT64_MAX / 4 / md->n_rep / md->dimi);
  SG_ARG(std::isfinite(step) && step > 0.0);
  SG_ARG(std::isfinite(fmax) && fmax >= 0.0);
  StepParams c = {};
  IrcParams& q = c.irc;
  q.h = step;
  q.hh = step / 2.0;
  q.h6 = step / 6.0;
  q.fmax2 = fmax * fmax;
  q.max_points = max_points;
  const IrcRun ir = {modes, R_path, E_path};
  return relax_impl(md, MD_IRC, 1, 0, c, 4 * (max_points - 1), n_points_out, end_out, fmax_out, nullptr,
                    (cudaStream_t)stream, nullptr, &ir);
}

int sgdml_b200_set_relax_block(int64_t n_steps) {
  SG_ARG(n_steps >= 0);
  g_relax_block = n_steps;
  return 0;
}

}  // extern "C"
