// Path (a), assembly: the symmetric Matern-5/2 Hessian-kernel matrix K (SURVEY.md section 8
// rows a-K / a-KT) -- reference sgdml/train.py:97-232 (_assemble_kernel_mat_wkr),
// train.py:1260-1535 (_assemble_kernel_mat), torchtools.py:110-392 (GDMLTorchAssemble).
//
// Design.  The reference materialises the dense Jacobians (D x 3N, six non-zeros per
// row) and runs three S-fold einsums plus a 3N x D x 3N product per block
// (train.py:209-226).  Here the Jacobian never exists.  With the antisymmetric pair vectors
//   G_m[a][g] = (r_a - r_g)/|r_a - r_g|^3      (J_m[d(a,g), atom a] = -G_m[a][g])
// and P the atom permutation that induces the descriptor permutation perm_p, block (i,j) is
//   K_ij[a][b] = sum_p  c1_p u_p[a] (x) v_p[b]  -  c2_p T_p[a][b]          (3x3 per atom pair)
//   delta_p[d] = x_i[d] - x_j[perm_p[d]],  n_p = sqrt5 |delta_p|,  e_p = exp(-n_p/sig)
//   c1_p = 25 e_p/(3 sig^4),   c2_p = 5 (sig^2 + sig n_p) e_p/(3 sig^4)       (train.py:179-220)
//   u_p[a] = -sum_g G_i[a][g] delta_p[d(a,g)]                                  (= J_i^T delta_p)
//   v_p[b] = -sum_g G_j[b][g] delta_p[d(P^-1 b, P^-1 g)]                        (= J_j^(p)T delta_p)
//   T_p[a][b] = sum_g G_i[a][g] (x) G_j[Pa][Pg]   if b == P a,
//             = -G_i[a][P^-1 b] (x) G_j[Pa][b]    otherwise                     (= J_i^T J_j^(p))
// i.e. ~33 N^2 FMAs per permutation instead of the reference's ~2 D 3N (3S + 3N) per block.
// One CTA owns row point i and a tile of TJ column points; the per-(j,p) vectors are staged in
// shared memory; each thread then owns 3x3 atom-pair sub-blocks and writes them once.
#include <algorithm>

#include "common.cuh"
#include "desc.cuh"

namespace sgdml {

struct AsmArgs {
  const double* R_desc;    // (M, D)
  const double* R_d_desc;  // (M, D, 3)
  const int* dperm;        // (S, D) descriptor perms
  const int* aperm;        // (S, N) atom perms P
  const int* apinv;        // (S, N) inverse atom perms
  const int* jpts;         // (nJ) training point of each block-column
  const int64_t* dest;     // (nJ, 3N) destination column in K or -1
  int N, D, M, S, nJ, TJ;
  int i0;                  // first row point of this call (row-sharded assembly): K row block = i - i0
  unsigned mN, mNN, mPer;  // ceil(2^32 / d) for d = N, N*N, 5N
  int NK;                  // kept column atoms per column point, at most (N unless a column subset is assembled)
  unsigned mNK, mNNK;      // ceil(2^32 / d) for d = NK, N*NK
  int sym;                 // full square matrix: compute blocks j >= i only and mirror them (K_ji = K_ij^T)
  double sig, scale;
  double* K;
  int64_t ldk;
};

// expands compressed g (D,3) into the antisymmetric table G (N,N,3), zero diagonal, and the
// descriptor x (D) into the symmetric table X (N,N)
__device__ void load_pair_tables(const double* __restrict__ g, const double* __restrict__ x, int N,
                                 double* __restrict__ G, double* __restrict__ X, int warp, int lane, int nw) {
  for (int a = warp; a < N; a += nw)
    for (int b = lane; b < N; b += 32) {
      double v0 = 0.0, v1 = 0.0, v2 = 0.0, xv = 0.0;
      if (a != b) {
        const int hi = a > b ? a : b, lo = a > b ? b : a;
        const int d = pair_index(hi, lo);
        const double sgn = a > b ? 1.0 : -1.0;
        v0 = sgn * g[d * 3 + 0];
        v1 = sgn * g[d * 3 + 1];
        v2 = sgn * g[d * 3 + 2];
        xv = x[d];
      }
      const int idx = a * N + b;
      G[idx * 3 + 0] = v0;
      G[idx * 3 + 1] = v1;
      G[idx * 3 + 2] = v2;
      X[idx] = xv;
    }
}

// exact x / d for 0 <= x < 2^20, 1 <= d < 2^12 with m = ceil(2^32 / d): runtime integer division
// compiles to an XU-pipe sequence that throttled the first version of this kernel
__device__ __forceinline__ int fastdiv(int x, unsigned m) { return (int)__umulhi((unsigned)x, m); }

__device__ __forceinline__ int ceil_div_dev(int a, int b) { return (a + b - 1) / b; }

constexpr int ASM_NI = 4;  // 3x3 atom-pair sub-blocks per thread (accumulators live in registers)

// One CTA: row point i, a tile of TJ column points.  Permutations are the OUTER loop; for each
// permutation the per-point vectors (delta table, u, v, diagonal sums) are rebuilt in shared
// memory with unit-stride loops over atom tables, then every thread adds the permutation's
// contribution to its 3x3 sub-blocks, which stay in registers until the single final store.
__global__ void __launch_bounds__(256, 2) k_assemble(const AsmArgs p) {
  extern __shared__ __align__(16) double sm[];
  const int N = p.N, S = p.S, TJ = p.TJ;
  const int N3 = 3 * N, NN = N * N, NN3 = NN * 3;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;

  const int i = p.i0 + blockIdx.y;
  const int jt0 = blockIdx.x * TJ;
  const int tj = min(TJ, p.nJ - jt0);
  if (p.sym && jt0 + tj - 1 < i) return;  // (sym: jpts is the identity) every column point of the tile is < i

  double* Gi = sm;                 // NN3
  double* Xi = Gi + NN3;           // NN
  double* Gj = Xi + NN;            // TJ*NN3
  double* Xj = Gj + TJ * NN3;      // TJ*NN
  double* Dl = Xj + TJ * NN;       // TJ*NN   delta table in the j frame (current permutation)
  double* u = Dl + TJ * NN;        // TJ*N3
  double* v = u + TJ * N3;         // TJ*N3
  double* Dg = v + TJ * N3;        // TJ*3*N3
  double* cc = Dg + TJ * 3 * N3;   // S*TJ*2
  double* n2p = cc + S * TJ * 2;   // TJ*8  per-warp partial sums of squared deltas (each pair twice)
  int* sP = reinterpret_cast<int*>(n2p + TJ * 8);  // S*N
  int* sPi = sP + S * N;                                // S*N
  int* need = sPi + S * N;                              // TJ*N: column atom b of point t has at least one kept column
  int* klist = need + TJ * N;                           // TJ*N: the kept column atoms of point t, compact
  int* nk = klist + TJ * N;                             // TJ: how many

  load_pair_tables(p.R_d_desc + (int64_t)i * p.D * 3, p.R_desc + (int64_t)i * p.D, N, Gi, Xi, warp, lane, nw);
  for (int t = 0; t < tj; ++t) {
    const int j = p.jpts[jt0 + t];
    load_pair_tables(p.R_d_desc + (int64_t)j * p.D * 3, p.R_desc + (int64_t)j * p.D, N, Gj + t * NN3, Xj + t * NN, warp,
                     lane, nw);
  }
  for (int idx = tid; idx < S * N; idx += nt) {
    sP[idx] = p.aperm[idx];
    sPi[idx] = p.apinv[idx];
  }
  // column subsets (the Nystroem set-up keeps ~10 of a point's 3N columns): the per-permutation vectors v[b] and the
  // diagonal sums Dg[P^-1 b] are only needed for column atoms b with a kept column
  for (int idx = tid; idx < tj * N; idx += nt) {
    const int64_t* dst = p.dest + (int64_t)(jt0 + idx / N) * N3 + 3 * (idx % N);
    need[idx] = (dst[0] >= 0 || dst[1] >= 0 || dst[2] >= 0) ? 1 : 0;
  }
  // compact list of the kept column atoms of every column point: the sub-blocks are dealt out over (row atom, kept
  // column atom) pairs, so a column subset with few kept atoms per point needs no grid.z split
  if (tid < tj) {
    int c = 0;
    for (int b = 0; b < N; ++b) {
      const int64_t* dst = p.dest + (int64_t)(jt0 + tid) * N3 + 3 * b;
      if (dst[0] >= 0 || dst[1] >= 0 || dst[2] >= 0) klist[tid * N + c++] = b;
    }
    nk[tid] = c;
  }
  __syncthreads();

  // this thread's output items: (t, a, b) = column point, row atom, kept column atom
  int it_t[ASM_NI], it_a[ASM_NI], it_b[ASM_NI];
  double acc[ASM_NI][9];
#pragma unroll
  for (int q = 0; q < ASM_NI; ++q) {
    const int it = (int)blockIdx.z * ASM_NI * nt + tid + q * nt;  // grid.z splits the sub-blocks of large molecules
    bool ok = it < tj * N * p.NK;
    const int t = ok ? fastdiv(it, p.mNNK) : 0;
    if (p.sym && jt0 + t < i) ok = false;  // mirrored from block (j, i) instead
    const int ak = ok ? it - t * N * p.NK : 0;
    it_a[q] = fastdiv(ak, p.mNK);
    const int k = ak - it_a[q] * p.NK;
    if (k >= nk[t]) ok = false;
    it_b[q] = ok ? klist[t * N + k] : 0;
    it_t[q] = ok ? t : -1;
#pragma unroll
    for (int e = 0; e < 9; ++e) acc[q][e] = 0.0;
  }

  const double sig = p.sig;
  const double sig2 = sig * sig;
  const double inv_div = 1.0 / (3.0 * sig2 * sig2);  // 1/mat52_base_div (train.py:179)

  for (int pp = 0; pp < S; ++pp) {
    const int* P = sP + pp * N;
    const int* Pi = sPi + pp * N;
    // ---- S1: delta table in the j frame, Dl[b][g] = x_i[d(P^-1 b, P^-1 g)] - x_j[d(b, g)]
    //          (= delta_p[d(P^-1 b, P^-1 g)], train.py:199) and sum of squares; all warps, rows of
    //          the (t, b) plane round-robin over warps, g over lanes
    for (int t = 0; t < tj; ++t) {
      double s2 = 0.0;
      for (int e = tid; e < NN; e += nt) {
        const int b = fastdiv(e, p.mN);
        const int g = e - b * N;
        const double dl = Xi[Pi[b] * N + Pi[g]] - Xj[t * NN + e];
        Dl[t * NN + e] = dl;
        s2 = fma(dl, dl, s2);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      if (lane == 0) n2p[t * 8 + warp] = s2;  // fixed-order reduction below: bit-reproducible K
    }
    __syncthreads();

    // ---- S2: u[a] = -sum_g G_i[a][g] Dl[Pa][Pg],  v[b] = -sum_g G_j[b][g] Dl[b][g],
    //          Dg[a][c][c'] = sum_g G_i[a][g][c] G_j[Pa][Pg][c']      (units of 3 outputs each)
    {
      // Matern factors of this permutation (one thread per column point, from the tail of the CTA)
      if (tid >= nt - tj) {
        const int t = nt - 1 - tid;
        double n2 = 0.0;
        for (int w = 0; w < nw; ++w) n2 += n2p[t * 8 + w];
        const double nrm = sqrt(5.0) * sqrt(0.5 * n2);  // every pair twice; train.py:201
        const double base = exp(-nrm / sig) * inv_div * 5.0;          // train.py:202
        cc[(pp * TJ + t) * 2 + 0] = base * 5.0;                       // c1 (train.py:211)
        cc[(pp * TJ + t) * 2 + 1] = (sig2 + sig * nrm) * base;        // c2 (train.py:219)
      }
      const int per = 5 * N;  // N (u) + N (v) + 3N (Dg rows a,c)
      for (int idx = tid; idx < tj * per; idx += nt) {
        const int t = fastdiv(idx, p.mPer);
        const int r = idx - t * per;
        const double* Gjt = Gj + t * NN3;
        const double* Dlt = Dl + t * NN;
        if (r < N) {  // u[a][0..2]
          const int a = r, pa = P[a];
          const double* gi = Gi + a * N3;
          const double* dl = Dlt + pa * N;
          double s0 = 0.0, s1 = 0.0, s2 = 0.0;
          for (int g = 0; g < N; ++g) {
            const double d = dl[P[g]];
            s0 = fma(gi[g * 3 + 0], d, s0);
            s1 = fma(gi[g * 3 + 1], d, s1);
            s2 = fma(gi[g * 3 + 2], d, s2);
          }
          u[t * N3 + 3 * a + 0] = -s0;
          u[t * N3 + 3 * a + 1] = -s1;
          u[t * N3 + 3 * a + 2] = -s2;
        } else if (r < 2 * N) {  // v[b][0..2]
          const int b = r - N;
          if (!need[t * N + b]) continue;
          const double* gj = Gjt + b * N3;
          const double* dl = Dlt + b * N;
          double s0 = 0.0, s1 = 0.0, s2 = 0.0;
          for (int g = 0; g < N; ++g) {
            const double d = dl[g];
            s0 = fma(gj[g * 3 + 0], d, s0);
            s1 = fma(gj[g * 3 + 1], d, s1);
            s2 = fma(gj[g * 3 + 2], d, s2);
          }
          v[t * N3 + 3 * b + 0] = -s0;
          v[t * N3 + 3 * b + 1] = -s1;
          v[t * N3 + 3 * b + 2] = -s2;
        } else {  // Dg[a][c][0..2]
          const int ac = r - 2 * N;
          const int a = (int)__umulhi((unsigned)ac, 0x55555556u), c = ac - 3 * a;
          if (!need[t * N + P[a]]) continue;  // only read for the sub-block (a, b = P a)
          const double* gi = Gi + a * N3 + c;
          const double* gj = Gjt + P[a] * N3;
          double s0 = 0.0, s1 = 0.0, s2 = 0.0;
          for (int g = 0; g < N; ++g) {
            const double x = gi[g * 3];
            const double* y = gj + P[g] * 3;
            s0 = fma(x, y[0], s0);
            s1 = fma(x, y[1], s1);
            s2 = fma(x, y[2], s2);
          }
          Dg[t * 3 * N3 + ac * 3 + 0] = s0;
          Dg[t * 3 * N3 + ac * 3 + 1] = s1;
          Dg[t * 3 * N3 + ac * 3 + 2] = s2;
        }
      }
    }
    __syncthreads();

    // ---- S3: acc[a][b] += c1 u[a] (x) v[b] - c2 T[a][b]
#pragma unroll
    for (int q = 0; q < ASM_NI; ++q) {
      const int t = it_t[q];
      if (t < 0) continue;
      const int a = it_a[q], b = it_b[q];
      const double c1 = cc[(pp * TJ + t) * 2 + 0], c2 = cc[(pp * TJ + t) * 2 + 1];
      const double* ua = u + t * N3 + 3 * a;
      const double* vb = v + t * N3 + 3 * b;
      const int pa = P[a];
      double t0[3], t1[3];  // T[a][b] = t0[c] * t1[c'] (outer product) unless b == P a
      if (b != pa) {
        const double* gi = Gi + (a * N + Pi[b]) * 3;
        const double* gj = Gj + t * NN3 + (pa * N + b) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          t0[c] = c2 * gi[c];   // -c2 * (-gi (x) gj) = +c2 gi (x) gj
          t1[c] = gj[c];
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const double cu = c1 * ua[c];
#pragma unroll
          for (int c2i = 0; c2i < 3; ++c2i)
            acc[q][c * 3 + c2i] = fma(t0[c], t1[c2i], fma(cu, vb[c2i], acc[q][c * 3 + c2i]));
        }
      } else {
        const double* dg = Dg + t * 3 * N3 + 9 * a;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const double cu = c1 * ua[c];
#pragma unroll
          for (int c2i = 0; c2i < 3; ++c2i)
            acc[q][c * 3 + c2i] = fma(-c2, dg[c * 3 + c2i], fma(cu, vb[c2i], acc[q][c * 3 + c2i]));
        }
      }
    }
    // (no barrier here: the next S1 only writes Dl / cc[pp+1]; u, v, Dg are rewritten after it)
  }

  // ---- single store of the finished 3x3 sub-blocks (+ the mirrored block in symmetric mode)
#pragma unroll
  for (int q = 0; q < ASM_NI; ++q) {
    const int t = it_t[q];
    if (t < 0) continue;
    const int a = it_a[q], b = it_b[q];
    const int64_t* dst = p.dest + (int64_t)(jt0 + t) * N3 + 3 * b;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double* Krow = p.K + ((int64_t)(i - p.i0) * N3 + 3 * a + c) * p.ldk;
#pragma unroll
      for (int c2i = 0; c2i < 3; ++c2i) {
        const int64_t col = dst[c2i];
        if (col >= 0) Krow[col] = p.scale * acc[q][c * 3 + c2i];
      }
    }
    if (p.sym && jt0 + t > i) {  // (sym implies i0 == 0)
      const int j = jt0 + t;
#pragma unroll
      for (int c2i = 0; c2i < 3; ++c2i) {
        double* Krow = p.K + ((int64_t)j * N3 + 3 * b + c2i) * p.ldk + (int64_t)i * N3 + 3 * a;
#pragma unroll
        for (int c = 0; c < 3; ++c) Krow[c] = p.scale * acc[q][c * 3 + c2i];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// k_assemble_v4: the default small-molecule kernel, built for many permutations and column subsets as well (BASELINE
// config 3: N = 42, S = 243, the Nystroem set-up keeps ~9 of a point's 126 columns).  Against k_assemble, what the
// first kernel's profile showed (few warps active, a mostly idle FP64 pipe, barrier / short-scoreboard / wait stalls):
//  * permutations are processed in CHUNKS of PG: phase A computes the per-(point, permutation) vectors u, v, Dg of the
//    whole chunk in one go, with the delta table evaluated on the fly (delta_p[Pa][Pg] = x_i[a][g] - x_j[Pa][Pg]; no
//    staged table); three CTA barriers per chunk instead of two per permutation;
//  * phase A is enumerated TYPE-major over the chunk -- all u rows, then the v rows, then the Dg rows -- so a warp runs
//    one kind of row task, and v / Dg rows exist only for column atoms with a kept column (compact list); |delta|^2
//    comes out of the u rows, which are always needed;
//  * the atom-permutation tables are bytes (20 KB instead of 82 KB at S = 243, N = 42), which leaves room for chunks of
//    up to 16 permutations next to the four pair tables of a 42-atom block;
//  * the pair tables have ODD row strides (3N | 1, N | 1 doubles): threads of a warp work on different table rows, and
//    with N = 42 even strides put every fourth row on the same banks;
//  * a CTA walks over `tiles_per_cta` column tiles with the row point's tables resident.
// Phase B (the 3x3 sub-block accumulation in registers) is that of k_assemble.
__device__ void load_pair_tables_strided(const double* __restrict__ g, const double* __restrict__ x, int N, int gs, int xs,
                                         double* __restrict__ G, double* __restrict__ X, int warp, int lane, int nw) {
  for (int a = warp; a < N; a += nw)
    for (int b = lane; b < N; b += 32) {
      double v0 = 0.0, v1 = 0.0, v2 = 0.0, xv = 0.0;
      if (a != b) {
        const int hi = a > b ? a : b, lo = a > b ? b : a;
        const int d = pair_index(hi, lo);
        const double sgn = a > b ? 1.0 : -1.0;
        v0 = sgn * g[d * 3 + 0];
        v1 = sgn * g[d * 3 + 1];
        v2 = sgn * g[d * 3 + 2];
        xv = x[d];
      }
      G[a * gs + b * 3 + 0] = v0;
      G[a * gs + b * 3 + 1] = v1;
      G[a * gs + b * 3 + 2] = v2;
      X[a * xs + b] = xv;
    }
}

__global__ void __launch_bounds__(256, 2) k_assemble_v4(const AsmArgs p, int PG, int tiles_per_cta) {
  extern __shared__ __align__(16) double sm[];
  const int N = p.N, S = p.S, TJ = p.TJ, NK = p.NK;
  const int N3 = 3 * N;
  const int GS = N3 | 1, XS = N | 1;  // odd row strides of the pair tables
  const int tid = threadIdx.x, nt = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;
  const int i = p.i0 + blockIdx.y;

  double* Gi = sm;                        // N*GS
  double* Xi = Gi + N * GS;               // N*XS
  double* Gj = Xi + N * XS;               // TJ*N*GS
  double* Xj = Gj + TJ * N * GS;          // TJ*N*XS
  double* uS = Xj + TJ * N * XS;          // TJ*PG*N3
  double* vS = uS + TJ * PG * N3;         // TJ*PG*N3   (rows of kept column atoms only)
  double* DgS = vS + TJ * PG * N3;        // TJ*PG*3*N3 (rows a = P^-1 b of kept column atoms b only)
  double* n2p = DgS + TJ * PG * 3 * N3;   // TJ*PG*N    per-u-row sums of squared deltas (each pair twice)
  double* cc = n2p + TJ * PG * N;         // TJ*PG*2
  int* klist = reinterpret_cast<int*>(cc + TJ * PG * 2);  // TJ*N: the kept column atoms of point t, compact
  int* nk = klist + TJ * N;                                    // TJ: how many
  unsigned char* sP = reinterpret_cast<unsigned char*>(nk + TJ);  // S*N
  unsigned char* sPi = sP + S * N;                                     // S*N

  load_pair_tables_strided(p.R_d_desc + (int64_t)i * p.D * 3, p.R_desc + (int64_t)i * p.D, N, GS, XS, Gi, Xi, warp, lane,
                           nw);
  for (int idx = tid; idx < S * N; idx += nt) {
    sP[idx] = (unsigned char)p.aperm[idx];
    sPi[idx] = (unsigned char)p.apinv[idx];
  }
  const double sig = p.sig;
  const double sig2 = sig * sig;
  const double inv_div = 1.0 / (3.0 * sig2 * sig2);  // 1/mat52_base_div (train.py:179)

  const int tile_begin = blockIdx.x * tiles_per_cta;
  const int tile_end = min(tile_begin + tiles_per_cta, ceil_div_dev(p.nJ, TJ));
  for (int tile = tile_begin; tile < tile_end; ++tile) {
    const int jt0 = tile * TJ;
    const int tj = min(TJ, p.nJ - jt0);
    if (p.sym && jt0 + tj - 1 < i) continue;  // (sym: jpts is the identity) every column point of the tile is < i
    __syncthreads();  // the previous tile's phase B has finished with Gj / the vectors
    for (int t = 0; t < tj; ++t) {
      const int j = p.jpts[jt0 + t];
      load_pair_tables_strided(p.R_d_desc + (int64_t)j * p.D * 3, p.R_desc + (int64_t)j * p.D, N, GS, XS, Gj + t * N * GS,
                               Xj + t * N * XS, warp, lane, nw);
    }
    for (int tw = warp; tw < tj; tw += nw) {  // compact list of the kept column atoms of point tw (ballot over atoms)
      int c = 0;
      for (int b0 = 0; b0 < N; b0 += 32) {
        const int b = b0 + lane;
        bool kept = false;
        if (b < N) {
          const int64_t* dst = p.dest + (int64_t)(jt0 + tw) * N3 + 3 * b;
          kept = dst[0] >= 0 || dst[1] >= 0 || dst[2] >= 0;
        }
        const unsigned m = __ballot_sync(0xffffffffu, kept);
        if (kept) klist[tw * N + c + __popc(m & ((1u << lane) - 1u))] = b;
        c += __popc(m);
      }
      if (lane == 0) nk[tw] = c;
    }
    __syncthreads();
    // this thread's output items: (t, a, b) = column point, row atom, kept column atom
    int it_t[ASM_NI], it_a[ASM_NI], it_b[ASM_NI];
    double acc[ASM_NI][9];
#pragma unroll
    for (int q = 0; q < ASM_NI; ++q) {
      const int it = (int)blockIdx.z * ASM_NI * nt + tid + q * nt;  // grid.z splits the sub-blocks of large molecules
      bool ok = it < tj * N * NK;
      const int t = ok ? fastdiv(it, p.mNNK) : 0;
      if (p.sym && jt0 + t < i) ok = false;  // mirrored from block (j, i) instead
      const int ak = ok ? it - t * N * NK : 0;
      it_a[q] = fastdiv(ak, p.mNK);
      const int k = ak - it_a[q] * NK;
      if (k >= nk[t]) ok = false;
      it_b[q] = ok ? klist[t * N + k] : 0;
      it_t[q] = ok ? t : -1;
#pragma unroll
      for (int e = 0; e < 9; ++e) acc[q][e] = 0.0;
    }

    for (int p0 = 0; p0 < S; p0 += PG) {
      const int pg = min(PG, S - p0);
      // ---- phase A, type-major over the chunk's (column point, permutation) slots
      const int n_slots = tj * pg;
      const int nU = n_slots * N, nV = n_slots * NK, nD = 3 * nV;
      for (int idx = tid; idx < nU + nV + nD; idx += nt) {
        if (idx < nU) {
          // u[a] = -sum_g G_i[a][g] delta[a][g],  delta[a][g] = x_i[a][g] - x_j[Pa][Pg]  (i frame)
          const int sl = fastdiv(idx, p.mN);
          const int a = idx - sl * N;
          const int t = sl / pg, pl = sl - t * pg;
          const unsigned char* P = sP + (p0 + pl) * N;
          const double* gi = Gi + a * GS;
          const double* xi = Xi + a * XS;
          const double* xj = Xj + t * N * XS + P[a] * XS;
          double s0 = 0.0, s1 = 0.0, s2 = 0.0, q2 = 0.0;
          for (int g = 0; g < N; ++g) {
            const double d = xi[g] - xj[P[g]];
            q2 = fma(d, d, q2);
            s0 = fma(gi[g * 3 + 0], d, s0);
            s1 = fma(gi[g * 3 + 1], d, s1);
            s2 = fma(gi[g * 3 + 2], d, s2);
          }
          const int slot = t * PG + pl;
          double* u = uS + slot * N3 + 3 * a;
          u[0] = -s0;
          u[1] = -s1;
          u[2] = -s2;
          n2p[slot * N + a] = q2;
        } else if (idx < nU + nV) {
          // v[b] = -sum_g G_j[b][g] delta[P^-1 b][P^-1 g]  for the kept column atoms b
          const int e = idx - nU;
          const int sl = fastdiv(e, p.mNK);
          const int k = e - sl * NK;
          const int t = sl / pg, pl = sl - t * pg;
          if (k >= nk[t]) continue;
          const int b = klist[t * N + k];
          const unsigned char* Pi = sPi + (p0 + pl) * N;
          const double* gj = Gj + t * N * GS + b * GS;
          const double* xj = Xj + t * N * XS + b * XS;
          const double* xi = Xi + Pi[b] * XS;
          double s0 = 0.0, s1 = 0.0, s2 = 0.0;
          for (int g = 0; g < N; ++g) {
            const double d = xi[Pi[g]] - xj[g];
            s0 = fma(gj[g * 3 + 0], d, s0);
            s1 = fma(gj[g * 3 + 1], d, s1);
            s2 = fma(gj[g * 3 + 2], d, s2);
          }
          double* v = vS + (t * PG + pl) * N3 + 3 * b;
          v[0] = -s0;
          v[1] = -s1;
          v[2] = -s2;
        } else {
          // Dg[a][c][0..2] = sum_g G_i[a][g][c] G_j[Pa][Pg][0..2]  for a = P^-1 b, b a kept column atom
          const int e = idx - nU - nV;
          const int e3 = (int)__umulhi((unsigned)e, 0x55555556u), c = e - 3 * e3;
          const int sl = fastdiv(e3, p.mNK);
          const int k = e3 - sl * NK;
          const int t = sl / pg, pl = sl - t * pg;
          if (k >= nk[t]) continue;
          const int b = klist[t * N + k];
          const unsigned char* P = sP + (p0 + pl) * N;
          const int a = sPi[(p0 + pl) * N + b];
          const double* gi = Gi + a * GS + c;
          const double* gj = Gj + t * N * GS + b * GS;  // b = P a
          double s0 = 0.0, s1 = 0.0, s2 = 0.0;
          for (int g = 0; g < N; ++g) {
            const double x = gi[g * 3];
            const double* y = gj + P[g] * 3;
            s0 = fma(x, y[0], s0);
            s1 = fma(x, y[1], s1);
            s2 = fma(x, y[2], s2);
          }
          double* dg = DgS + (t * PG + pl) * 3 * N3 + (a * 3 + c) * 3;
          dg[0] = s0;
          dg[1] = s1;
          dg[2] = s2;
        }
      }
      __syncthreads();
      // ---- Matern factors of the chunk (fixed-order sum of the row partials: bit-reproducible K)
      if (tid < n_slots) {
        const int t = tid / pg, pl = tid - t * pg;
        const int slot = t * PG + pl;
        double n2 = 0.0;
        for (int a = 0; a < N; ++a) n2 += n2p[slot * N + a];
        const double nrm = sqrt(5.0) * sqrt(0.5 * n2);  // every pair twice; train.py:201
        const double base = exp(-nrm / sig) * inv_div * 5.0;          // train.py:202
        cc[slot * 2 + 0] = base * 5.0;                                 // c1 (train.py:211)
        cc[slot * 2 + 1] = (sig2 + sig * nrm) * base;                  // c2 (train.py:219)
      }
      __syncthreads();
      // ---- phase B: acc[a][b] += c1 u[a] (x) v[b] - c2 T[a][b] for the permutations of the chunk
      for (int pl = 0; pl < pg; ++pl) {
        const unsigned char* P = sP + (p0 + pl) * N;
        const unsigned char* Pi = sPi + (p0 + pl) * N;
#pragma unroll
        for (int q = 0; q < ASM_NI; ++q) {
          const int t = it_t[q];
          if (t < 0) continue;
          const int slot = t * PG + pl;
          const int a = it_a[q], b = it_b[q];
          const double c1 = cc[slot * 2 + 0], c2 = cc[slot * 2 + 1];
          const double* ua = uS + slot * N3 + 3 * a;
          const double* vb = vS + slot * N3 + 3 * b;
          const int pa = P[a];
          if (b != pa) {
            const double* gi = Gi + a * GS + Pi[b] * 3;
            const double* gj = Gj + t * N * GS + pa * GS + b * 3;
            double t0[3], t1[3];  // T[a][b] = -gi (x) gj  ->  -c2 T = +c2 gi (x) gj
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              t0[c] = c2 * gi[c];
              t1[c] = gj[c];
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const double cu = c1 * ua[c];
#pragma unroll
              for (int c2i = 0; c2i < 3; ++c2i)
                acc[q][c * 3 + c2i] = fma(t0[c], t1[c2i], fma(cu, vb[c2i], acc[q][c * 3 + c2i]));
            }
          } else {
            const double* dg = DgS + slot * 3 * N3 + 9 * a;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const double cu = c1 * ua[c];
#pragma unroll
              for (int c2i = 0; c2i < 3; ++c2i)
                acc[q][c * 3 + c2i] = fma(-c2, dg[c * 3 + c2i], fma(cu, vb[c2i], acc[q][c * 3 + c2i]));
            }
          }
        }
      }
      if (p0 + PG < S) __syncthreads();  // the next chunk overwrites the vectors
    }

    // ---- single store of the finished 3x3 sub-blocks (+ the mirrored block in symmetric mode)
#pragma unroll
    for (int q = 0; q < ASM_NI; ++q) {
      const int t = it_t[q];
      if (t < 0) continue;
      const int a = it_a[q], b = it_b[q];
      const int64_t* dst = p.dest + (int64_t)(jt0 + t) * N3 + 3 * b;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        double* Krow = p.K + ((int64_t)(i - p.i0) * N3 + 3 * a + c) * p.ldk;
#pragma unroll
        for (int c2i = 0; c2i < 3; ++c2i) {
          const int64_t col = dst[c2i];
          if (col >= 0) Krow[col] = p.scale * acc[q][c * 3 + c2i];
        }
      }
      if (p.sym && jt0 + t > i) {  // (sym implies i0 == 0)
        const int j = jt0 + t;
#pragma unroll
        for (int c2i = 0; c2i < 3; ++c2i) {
          double* Krow = p.K + ((int64_t)j * N3 + 3 * b + c2i) * p.ldk + (int64_t)i * N3 + 3 * a;
#pragma unroll
          for (int c = 0; c < 3; ++c) Krow[c] = p.scale * acc[q][c * 3 + c2i];
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// k_assemble_v5: k_assemble_v4 on the COMPRESSED pair arrays -- x (D) and g (D x 3) of the row point and of the column
// point(s) sit in shared memory exactly as stored (4 D doubles per point instead of the 4 N^2 of the expanded
// antisymmetric tables), looked up through the pair index d(a, g) = max(max - 1)/2 + min with the sign of a - g.  That
// halves the table footprint: molecules up to ~64 atoms (BASELINE config 5: C60, N = 60, S = 120) keep everything on chip
// with chunks of 11 permutations, where k_assemble_large walks per-CTA slabs in global memory one permutation at a time.
__device__ __forceinline__ int pidx(int a, int g) { return a > g ? a * (a - 1) / 2 + g : g * (g - 1) / 2 + a; }

__global__ void __launch_bounds__(256, 2) k_assemble_v5(const AsmArgs p, int PG, int tiles_per_cta) {
  extern __shared__ __align__(16) double sm[];
  const int N = p.N, S = p.S, TJ = p.TJ, NK = p.NK;
  const int N3 = 3 * N, D = p.D, D3 = 3 * p.D;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;
  const int i = p.i0 + blockIdx.y;

  double* gI = sm;                        // 3D   compressed pair vectors of the row point, as stored: g[d][0..2]
  double* xI = gI + D3;                   // D    descriptor of the row point
  double* gJ = xI + D;                    // TJ*3D
  double* xJ = gJ + TJ * D3;              // TJ*D
  double* uS = xJ + TJ * D;               // TJ*PG*N3
  double* vS = uS + TJ * PG * N3;         // TJ*PG*N3   (rows of kept column atoms only)
  double* DgS = vS + TJ * PG * N3;        // TJ*PG*3*N3 (rows a = P^-1 b of kept column atoms b only)
  double* n2p = DgS + TJ * PG * 3 * N3;   // TJ*PG*N    per-u-row sums of squared deltas (each pair twice)
  double* cc = n2p + TJ * PG * N;         // TJ*PG*2
  int* klist = reinterpret_cast<int*>(cc + TJ * PG * 2);  // TJ*N: the kept column atoms of point t, compact
  int* nk = klist + TJ * N;                                    // TJ: how many
  unsigned char* sP = reinterpret_cast<unsigned char*>(nk + TJ);  // S*N
  unsigned char* sPi = sP + S * N;                                     // S*N

  for (int e = tid; e < D3; e += nt) gI[e] = p.R_d_desc[(int64_t)i * D3 + e];
  for (int e = tid; e < D; e += nt) xI[e] = p.R_desc[(int64_t)i * D + e];
  for (int idx = tid; idx < S * N; idx += nt) {
    sP[idx] = (unsigned char)p.aperm[idx];
    sPi[idx] = (unsigned char)p.apinv[idx];
  }
  const double sig = p.sig;
  const double sig2 = sig * sig;
  const double inv_div = 1.0 / (3.0 * sig2 * sig2);  // 1/mat52_base_div (train.py:179)

  const int tile_begin = blockIdx.x * tiles_per_cta;
  const int tile_end = min(tile_begin + tiles_per_cta, ceil_div_dev(p.nJ, TJ));
  for (int tile = tile_begin; tile < tile_end; ++tile) {
    const int jt0 = tile * TJ;
    const int tj = min(TJ, p.nJ - jt0);
    if (p.sym && jt0 + tj - 1 < i) continue;  // (sym: jpts is the identity) every column point of the tile is < i
    __syncthreads();  // the previous tile's phase B has finished with Gj / the vectors
    for (int t = 0; t < tj; ++t) {
      const int j = p.jpts[jt0 + t];
      for (int e = tid; e < D3; e += nt) gJ[t * D3 + e] = p.R_d_desc[(int64_t)j * D3 + e];
      for (int e = tid; e < D; e += nt) xJ[t * D + e] = p.R_desc[(int64_t)j * D + e];
    }
    for (int tw = warp; tw < tj; tw += nw) {  // compact list of the kept column atoms of point tw (ballot over atoms)
      int c = 0;
      for (int b0 = 0; b0 < N; b0 += 32) {
        const int b = b0 + lane;
        bool kept = false;
        if (b < N) {
          const int64_t* dst = p.dest + (int64_t)(jt0 + tw) * N3 + 3 * b;
          kept = dst[0] >= 0 || dst[1] >= 0 || dst[2] >= 0;
        }
        const unsigned m = __ballot_sync(0xffffffffu, kept);
        if (kept) klist[tw * N + c + __popc(m & ((1u << lane) - 1u))] = b;
        c += __popc(m);
      }
      if (lane == 0) nk[tw] = c;
    }
    __syncthreads();
    // this thread's output items: (t, a, b) = column point, row atom, kept column atom
    int it_t[ASM_NI], it_a[ASM_NI], it_b[ASM_NI];
    double acc[ASM_NI][9];
#pragma unroll
    for (int q = 0; q < ASM_NI; ++q) {
      const int it = (int)blockIdx.z * ASM_NI * nt + tid + q * nt;  // grid.z splits the sub-blocks of large molecules
      bool ok = it < tj * N * NK;
      const int t = ok ? fastdiv(it, p.mNNK) : 0;
      if (p.sym && jt0 + t < i) ok = false;  // mirrored from block (j, i) instead
      const int ak = ok ? it - t * N * NK : 0;
      it_a[q] = fastdiv(ak, p.mNK);
      const int k = ak - it_a[q] * NK;
      if (k >= nk[t]) ok = false;
      it_b[q] = ok ? klist[t * N + k] : 0;
      it_t[q] = ok ? t : -1;
#pragma unroll
      for (int e = 0; e < 9; ++e) acc[q][e] = 0.0;
    }

    for (int p0 = 0; p0 < S; p0 += PG) {
      const int pg = min(PG, S - p0);
      // ---- phase A, type-major over the chunk's (column point, permutation) slots
      const int n_slots = tj * pg;
      const int nU = n_slots * N, nV = n_slots * NK, nD = 3 * nV;
      for (int idx = tid; idx < nU + nV + nD; idx += nt) {
        if (idx < nU) {
          // u[a] = -sum_g G_i[a][g] delta[a][g],  delta[a][g] = x_i[a][g] - x_j[Pa][Pg]  (i frame)
          const int sl = fastdiv(idx, p.mN);
          const int a = idx - sl * N;
          const int t = sl / pg, pl = sl - t * pg;
          const unsigned char* P = sP + (p0 + pl) * N;
          const double* xj = xJ + t * D;
          const int pa = P[a];
          double s0 = 0.0, s1 = 0.0, s2 = 0.0, q2 = 0.0;
          for (int g = 0; g < N; ++g) {
            if (g == a) continue;
            const int di = pidx(a, g), dj = pidx(pa, P[g]);
            const double d = xI[di] - xj[dj];
            q2 = fma(d, d, q2);
            const double w = a > g ? d : -d;  // G_i[a][g] = sgn(a - g) g_i[d(a,g)]
            const double* gi = gI + 3 * di;
            s0 = fma(gi[0], w, s0);
            s1 = fma(gi[1], w, s1);
            s2 = fma(gi[2], w, s2);
          }
          const int slot = t * PG + pl;
          double* u = uS + slot * N3 + 3 * a;
          u[0] = -s0;
          u[1] = -s1;
          u[2] = -s2;
          n2p[slot * N + a] = q2;
        } else if (idx < nU + nV) {
          // v[b] = -sum_g G_j[b][g] delta[P^-1 b][P^-1 g]  for the kept column atoms b
          const int e = idx - nU;
          const int sl = fastdiv(e, p.mNK);
          const int k = e - sl * NK;
          const int t = sl / pg, pl = sl - t * pg;
          if (k >= nk[t]) continue;
          const int b = klist[t * N + k];
          const unsigned char* Pi = sPi + (p0 + pl) * N;
          const double* xj = xJ + t * D;
          const int pib = Pi[b];
          double s0 = 0.0, s1 = 0.0, s2 = 0.0;
          for (int g = 0; g < N; ++g) {
            if (g == b) continue;
            const int dj = pidx(b, g), di = pidx(pib, Pi[g]);
            const double d = xI[di] - xj[dj];
            const double w = b > g ? d : -d;
            const double* gj = gJ + t * D3 + 3 * dj;
            s0 = fma(gj[0], w, s0);
            s1 = fma(gj[1], w, s1);
            s2 = fma(gj[2], w, s2);
          }
          double* v = vS + (t * PG + pl) * N3 + 3 * b;
          v[0] = -s0;
          v[1] = -s1;
          v[2] = -s2;
        } else {
          // Dg[a][c][0..2] = sum_g G_i[a][g][c] G_j[Pa][Pg][0..2]  for a = P^-1 b, b a kept column atom
          const int e = idx - nU - nV;
          const int e3 = (int)__umulhi((unsigned)e, 0x55555556u), c = e - 3 * e3;
          const int sl = fastdiv(e3, p.mNK);
          const int k = e3 - sl * NK;
          const int t = sl / pg, pl = sl - t * pg;
          if (k >= nk[t]) continue;
          const int b = klist[t * N + k];
          const unsigned char* P = sP + (p0 + pl) * N;
          const int a = sPi[(p0 + pl) * N + b];
          double s0 = 0.0, s1 = 0.0, s2 = 0.0;
          for (int g = 0; g < N; ++g) {
            if (g == a) continue;
            const int pg = P[g];
            const int di = pidx(a, g), dj = pidx(b, pg);  // b = P a
            const double gic = gI[3 * di + c];
            const double x = ((a > g) == (b > pg)) ? gic : -gic;  // sgn(a - g) sgn(Pa - Pg)
            const double* y = gJ + t * D3 + 3 * dj;
            s0 = fma(x, y[0], s0);
            s1 = fma(x, y[1], s1);
            s2 = fma(x, y[2], s2);
          }
          double* dg = DgS + (t * PG + pl) * 3 * N3 + (a * 3 + c) * 3;
          dg[0] = s0;
          dg[1] = s1;
          dg[2] = s2;
        }
      }
      __syncthreads();
      // ---- Matern factors of the chunk (fixed-order sum of the row partials: bit-reproducible K)
      if (tid < n_slots) {
        const int t = tid / pg, pl = tid - t * pg;
        const int slot = t * PG + pl;
        double n2 = 0.0;
        for (int a = 0; a < N; ++a) n2 += n2p[slot * N + a];
        const double nrm = sqrt(5.0) * sqrt(0.5 * n2);  // every pair twice; train.py:201
        const double base = exp(-nrm / sig) * inv_div * 5.0;          // train.py:202
        cc[slot * 2 + 0] = base * 5.0;                                 // c1 (train.py:211)
        cc[slot * 2 + 1] = (sig2 + sig * nrm) * base;                  // c2 (train.py:219)
      }
      __syncthreads();
      // ---- phase B: acc[a][b] += c1 u[a] (x) v[b] - c2 T[a][b] for the permutations of the chunk
      for (int pl = 0; pl < pg; ++pl) {
        const unsigned char* P = sP + (p0 + pl) * N;
        const unsigned char* Pi = sPi + (p0 + pl) * N;
#pragma unroll
        for (int q = 0; q < ASM_NI; ++q) {
          const int t = it_t[q];
          if (t < 0) continue;
          const int slot = t * PG + pl;
          const int a = it_a[q], b = it_b[q];
          const double c1 = cc[slot * 2 + 0], c2 = cc[slot * 2 + 1];
          const double* ua = uS + slot * N3 + 3 * a;
          const double* vb = vS + slot * N3 + 3 * b;
          const int pa = P[a];
          if (b != pa) {
            const int pib = Pi[b];
            const double* gi = gI + 3 * pidx(a, pib);
            const double* gj = gJ + t * D3 + 3 * pidx(pa, b);
            const double sg = ((a > pib) == (pa > b)) ? c2 : -c2;  // sgn(a - P^-1 b) sgn(Pa - b) c2
            double t0[3], t1[3];  // T[a][b] = -G_i[a][P^-1 b] (x) G_j[Pa][b]  ->  -c2 T = +c2 G_i (x) G_j
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              t0[c] = sg * gi[c];
              t1[c] = gj[c];
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const double cu = c1 * ua[c];
#pragma unroll
              for (int c2i = 0; c2i < 3; ++c2i)
                acc[q][c * 3 + c2i] = fma(t0[c], t1[c2i], fma(cu, vb[c2i], acc[q][c * 3 + c2i]));
            }
          } else {
            const double* dg = DgS + slot * 3 * N3 + 9 * a;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const double cu = c1 * ua[c];
#pragma unroll
              for (int c2i = 0; c2i < 3; ++c2i)
                acc[q][c * 3 + c2i] = fma(-c2, dg[c * 3 + c2i], fma(cu, vb[c2i], acc[q][c * 3 + c2i]));
            }
          }
        }
      }
      if (p0 + PG < S) __syncthreads();  // the next chunk overwrites the vectors
    }

    // ---- single store of the finished 3x3 sub-blocks (+ the mirrored block in symmetric mode)
#pragma unroll
    for (int q = 0; q < ASM_NI; ++q) {
      const int t = it_t[q];
      if (t < 0) continue;
      const int a = it_a[q], b = it_b[q];
      const int64_t* dst = p.dest + (int64_t)(jt0 + t) * N3 + 3 * b;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        double* Krow = p.K + ((int64_t)(i - p.i0) * N3 + 3 * a + c) * p.ldk;
#pragma unroll
        for (int c2i = 0; c2i < 3; ++c2i) {
          const int64_t col = dst[c2i];
          if (col >= 0) Krow[col] = p.scale * acc[q][c * 3 + c2i];
        }
      }
      if (p.sym && jt0 + t > i) {  // (sym implies i0 == 0)
        const int j = jt0 + t;
#pragma unroll
        for (int c2i = 0; c2i < 3; ++c2i) {
          double* Krow = p.K + ((int64_t)j * N3 + 3 * b + c2i) * p.ldk + (int64_t)i * N3 + 3 * a;
#pragma unroll
          for (int c = 0; c < 3; ++c) Krow[c] = p.scale * acc[q][c * 3 + c2i];
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Large molecules (N > ~50: the atom tables of one block no longer fit in shared memory; BASELINE
// configs 4 and 5).  Same mathematics and the same summation order as k_assemble, but the tables
// live in a private slab of global memory per CTA (L1/L2 resident), the CTAs are persistent
// (2 per SM, each walking a contiguous range of (row point, column point) blocks so the row tables
// are rebuilt only when i changes), and the per-permutation vectors u, v, Dg of ALL permutations
// are kept so that the 3x3 sub-blocks can be accumulated in register-sized passes without
// recomputing them.  Only the delta table (N*N doubles) stays in shared memory when it fits.
__global__ void __launch_bounds__(256, 2)
    k_assemble_large(const AsmArgs p, double* slabs, int64_t slab_stride, int64_t n_work, int dl_in_smem) {
  extern __shared__ __align__(16) double sm[];
  __shared__ double n2p[8];
  const int N = p.N, S = p.S;
  const int N3 = 3 * N, NN = N * N, NN3 = NN * 3;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;

  double* sl = slabs + (int64_t)blockIdx.x * slab_stride;
  double* Gi = sl;                    // NN3
  double* Xi = Gi + NN3;              // NN
  double* Gj = Xi + NN;               // NN3
  double* Xj = Gj + NN3;              // NN
  double* uS = Xj + NN;               // S*N3
  double* vS = uS + (int64_t)S * N3;  // S*N3
  double* DgS = vS + (int64_t)S * N3;        // S*3*N3
  double* cc = DgS + (int64_t)S * 3 * N3;    // S*2
  double* Dl = dl_in_smem ? sm : cc + 2 * S;  // NN

  const double sig = p.sig;
  const double sig2 = sig * sig;
  const double inv_div = 1.0 / (3.0 * sig2 * sig2);

  const int64_t w0 = n_work * (int64_t)blockIdx.x / gridDim.x;
  const int64_t w1 = n_work * ((int64_t)blockIdx.x + 1) / gridDim.x;
  int cur_i = -1;
  for (int64_t w = w0; w < w1; ++w) {
    const int i = p.i0 + (int)(w / p.nJ);
    const int jt = (int)(w % p.nJ);
    const int j = p.jpts[jt];
    __syncthreads();  // the previous block's accumulation passes have finished reading the slab
    if (i != cur_i) {
      load_pair_tables(p.R_d_desc + (int64_t)i * p.D * 3, p.R_desc + (int64_t)i * p.D, N, Gi, Xi, warp, lane, nw);
      cur_i = i;
    }
    load_pair_tables(p.R_d_desc + (int64_t)j * p.D * 3, p.R_desc + (int64_t)j * p.D, N, Gj, Xj, warp, lane, nw);
    __syncthreads();

    // ---- phase A: per-permutation vectors (S1 + S2 of k_assemble), kept for all permutations
    for (int pp = 0; pp < S; ++pp) {
      const int* P = p.aperm + pp * N;
      const int* Pi = p.apinv + pp * N;
      double s2 = 0.0;
      for (int e = tid; e < NN; e += nt) {
        const int b = fastdiv(e, p.mN);
        const int g = e - b * N;
        const double dl = Xi[Pi[b] * N + Pi[g]] - Xj[e];
        Dl[e] = dl;
        s2 = fma(dl, dl, s2);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      if (lane == 0) n2p[warp] = s2;
      __syncthreads();
      if (tid == nt - 1) {
        double n2 = 0.0;
        for (int w8 = 0; w8 < nw; ++w8) n2 += n2p[w8];
        const double nrm = sqrt(5.0) * sqrt(0.5 * n2);
        const double base = exp(-nrm / sig) * inv_div * 5.0;
        cc[pp * 2 + 0] = base * 5.0;
        cc[pp * 2 + 1] = (sig2 + sig * nrm) * base;
      }
      double* u = uS + (int64_t)pp * N3;
      double* v = vS + (int64_t)pp * N3;
      double* Dg = DgS + (int64_t)pp * 3 * N3;
      for (int r = tid; r < 5 * N; r += nt) {
        if (r < N) {
          const int a = r, pa = P[a];
          const double* gi = Gi + a * N3;
          const double* dl = Dl + pa * N;
          double s0 = 0.0, s1 = 0.0, s2b = 0.0;
          for (int g = 0; g < N; ++g) {
            const double d = dl[P[g]];
            s0 = fma(gi[g * 3 + 0], d, s0);
            s1 = fma(gi[g * 3 + 1], d, s1);
            s2b = fma(gi[g * 3 + 2], d, s2b);
          }
          u[3 * a + 0] = -s0;
          u[3 * a + 1] = -s1;
          u[3 * a + 2] = -s2b;
        } else if (r < 2 * N) {
          const int b = r - N;
          const double* gj = Gj + b * N3;
          const double* dl = Dl + b * N;
          double s0 = 0.0, s1 = 0.0, s2b = 0.0;
          for (int g = 0; g < N; ++g) {
            const double d = dl[g];
            s0 = fma(gj[g * 3 + 0], d, s0);
            s1 = fma(gj[g * 3 + 1], d, s1);
            s2b = fma(gj[g * 3 + 2], d, s2b);
          }
          v[3 * b + 0] = -s0;
          v[3 * b + 1] = -s1;
          v[3 * b + 2] = -s2b;
        } else {
          const int ac = r - 2 * N;
          const int a = (int)__umulhi((unsigned)ac, 0x55555556u), c = ac - 3 * a;
          const double* gi = Gi + a * N3 + c;
          const double* gj = Gj + P[a] * N3;
          double s0 = 0.0, s1 = 0.0, s2b = 0.0;
          for (int g = 0; g < N; ++g) {
            const double x = gi[g * 3];
            const double* y = gj + P[g] * 3;
            s0 = fma(x, y[0], s0);
            s1 = fma(x, y[1], s1);
            s2b = fma(x, y[2], s2b);
          }
          Dg[ac * 3 + 0] = s0;
          Dg[ac * 3 + 1] = s1;
          Dg[ac * 3 + 2] = s2b;
        }
      }
      __syncthreads();  // Dl and n2p are rewritten by the next permutation
    }

    // ---- phase B: passes of ASM_NI sub-blocks per thread over the N*N atom pairs (S3 of k_assemble)
    for (int base0 = 0; base0 < NN; base0 += ASM_NI * nt) {
      int it_a[ASM_NI], it_b[ASM_NI];
      double acc[ASM_NI][9];
#pragma unroll
      for (int q = 0; q < ASM_NI; ++q) {
        const int it = base0 + tid + q * nt;
        bool ok = it < NN;
        int a_ = ok ? fastdiv(it, p.mN) : -1;
        const int b_ = ok ? it - a_ * N : 0;
        if (ok) {  // sub-blocks whose three columns are all dropped are never stored: skip them
          const int64_t* dst = p.dest + (int64_t)jt * N3 + 3 * b_;
          if (dst[0] < 0 && dst[1] < 0 && dst[2] < 0) a_ = -1;
        }
        it_a[q] = a_;
        it_b[q] = b_;
#pragma unroll
        for (int e = 0; e < 9; ++e) acc[q][e] = 0.0;
      }
      for (int pp = 0; pp < S; ++pp) {
        const int* P = p.aperm + pp * N;
        const int* Pi = p.apinv + pp * N;
        const double c1 = cc[pp * 2 + 0], c2 = cc[pp * 2 + 1];
        const double* u = uS + (int64_t)pp * N3;
        const double* v = vS + (int64_t)pp * N3;
        const double* Dg = DgS + (int64_t)pp * 3 * N3;
#pragma unroll
        for (int q = 0; q < ASM_NI; ++q) {
          const int a = it_a[q], b = it_b[q];
          if (a < 0) continue;
          const double* ua = u + 3 * a;
          const double* vb = v + 3 * b;
          const int pa = P[a];
          if (b != pa) {
            const double* gi = Gi + (a * N + Pi[b]) * 3;
            const double* gj = Gj + (pa * N + b) * 3;
            double t0[3], t1[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              t0[c] = c2 * gi[c];
              t1[c] = gj[c];
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const double cu = c1 * ua[c];
#pragma unroll
              for (int c2i = 0; c2i < 3; ++c2i)
                acc[q][c * 3 + c2i] = fma(t0[c], t1[c2i], fma(cu, vb[c2i], acc[q][c * 3 + c2i]));
            }
          } else {
            const double* dg = Dg + 9 * a;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const double cu = c1 * ua[c];
#pragma unroll
              for (int c2i = 0; c2i < 3; ++c2i)
                acc[q][c * 3 + c2i] = fma(-c2, dg[c * 3 + c2i], fma(cu, vb[c2i], acc[q][c * 3 + c2i]));
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < ASM_NI; ++q) {
        const int a = it_a[q], b = it_b[q];
        if (a < 0) continue;
        const int64_t* dst = p.dest + (int64_t)jt * N3 + 3 * b;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          double* Krow = p.K + ((int64_t)(i - p.i0) * N3 + 3 * a + c) * p.ldk;
#pragma unroll
          for (int c2i = 0; c2i < 3; ++c2i) {
            const int64_t col = dst[c2i];
            if (col >= 0) Krow[col] = p.scale * acc[q][c * 3 + c2i];
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Energy constraints in the kernel (use_E_cstr; reference train.py:234-300): the M extra rows and columns of
// the (3NM + M) x (3NM + M) matrix.  One CTA per pair (i, j), one thread per atom b of point j:
//   delta_p[d(P^-1 b, P^-1 g)] = x_i[d(P^-1 b, P^-1 g)] - x_j[d(b, g)],   n_p = sqrt5 |delta_p|,
//   v_p[b] = -sum_g G_j[b][g] delta_p[...]                                  (= J_j^(p)T delta_p, as in k_assemble)
//   r[b]   = -sum_p c_p v_p[b],  c_p = 5 (n_p + sig) exp(-n_p/sig) / (3 sig^3)        (train.py:237-248)
//   K[n + i, blk_j] = r  and, by the same formula with the roles exchanged (train.py:266-294), K[blk_j, n + i] = r;
//   K[n + j, n + i] = -sum_p (1 + (n_p/sig)(1 + n_p/(3 sig))) exp(-n_p/sig)           (train.py:296-300)
// No tables: the pair quantities are read straight from the compressed arrays (L1/L2 resident); the work is
// O(S N^2) per pair against O(S N^2 * 33) for the force-force block.
// The per-pair part, shared by k_assemble_ecstr and k_assemble_ecstr_rows: for the pair (i, j) returns r[b] of
// atom b = threadIdx.x of point j in (r0, r1, r2) and, in thread 0, the sum over permutations of the K_ee terms in
// kee (the matrix entry is -scale * kee).  Block-wide:
// every thread of the CTA calls it; red holds one double per warp (blockDim.x = N rounded up to a warp multiple, so
// up to 32 warps at the assembly's bound of N <= 1023; the order of every sum depends only on N).
__device__ __forceinline__ void ecstr_pair(const double* __restrict__ xi, const double* __restrict__ xj,
                                           const double* __restrict__ gj, const int* __restrict__ aperm_inv, int N,
                                           int S, double sig, double* red, double& s_cp, double& s_kee, double& r0,
                                           double& r1, double& r2, double& kee) {
  const int b = threadIdx.x;
  r0 = 0.0, r1 = 0.0, r2 = 0.0, kee = 0.0;
  for (int pp = 0; pp < S; ++pp) {
    const int* Pi = aperm_inv + pp * N;
    double v0 = 0.0, v1 = 0.0, v2 = 0.0, s2 = 0.0;
    if (b < N) {
      const int pb = Pi[b];
      for (int g = 0; g < N; ++g) {
        if (g == b) continue;
        const int pg = Pi[g];
        const int d1 = pb > pg ? pair_index(pb, pg) : pair_index(pg, pb);
        const int d2 = b > g ? pair_index(b, g) : pair_index(g, b);
        const double sgn = b > g ? 1.0 : -1.0;  // G_j[b][g] = +g_d for b > g, -g_d otherwise
        const double dl = xi[d1] - xj[d2];
        s2 = fma(dl, dl, s2);
        v0 = fma(sgn * gj[d2 * 3 + 0], dl, v0);
        v1 = fma(sgn * gj[d2 * 3 + 1], dl, v1);
        v2 = fma(sgn * gj[d2 * 3 + 2], dl, v2);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s2;
    __syncthreads();
    if (threadIdx.x == 0) {
      double n2 = 0.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) n2 += red[w];
      const double nrm = sqrt(5.0) * sqrt(0.5 * n2);  // every pair was visited twice
      const double e = exp(-nrm / sig);
      s_cp = 5.0 * (nrm + sig) * e / (3.0 * sig * sig * sig);
      const double t = nrm / sig;
      s_kee = (1.0 + t * (1.0 + nrm / (3.0 * sig))) * e;
    }
    __syncthreads();
    const double cp = s_cp;
    // v_p = -(sum): r -= c_p v_p  ->  r += c_p (sum)
    r0 = fma(cp, v0, r0);
    r1 = fma(cp, v1, r1);
    r2 = fma(cp, v2, r2);
    if (threadIdx.x == 0) kee += s_kee;
    __syncthreads();  // red / s_cp are rewritten by the next permutation
  }
}

__global__ void __launch_bounds__(1024) k_assemble_ecstr(const double* __restrict__ R_desc, const double* __restrict__ R_d_desc,
                                                        const int* __restrict__ aperm_inv, int N, int D, int M, int S,
                                                        double sig, double scale, double* __restrict__ K, int64_t ldk) {
  __shared__ double red[32];
  __shared__ double s_cp, s_kee;
  const int i = blockIdx.y, j = blockIdx.x;
  const int b = threadIdx.x;  // atom of point j (blockDim.x = N rounded up to a warp multiple)
  const double* xi = R_desc + (int64_t)i * D;
  const double* xj = R_desc + (int64_t)j * D;
  const double* gj = R_d_desc + (int64_t)j * D * 3;
  const int64_t n = (int64_t)M * 3 * N;
  double r0, r1, r2, kee;
  ecstr_pair(xi, xj, gj, aperm_inv, N, S, sig, red, s_cp, s_kee, r0, r1, r2, kee);
  if (b < N) {
    const int64_t col = (int64_t)j * 3 * N + 3 * b;
    double* rowE = K + (n + i) * ldk + col;
    rowE[0] = scale * r0;
    rowE[1] = scale * r1;
    rowE[2] = scale * r2;
    K[(col + 0) * ldk + n + i] = scale * r0;
    K[(col + 1) * ldk + n + i] = scale * r1;
    K[(col + 2) * ldk + n + i] = scale * r2;
  }
  if (threadIdx.x == 0) K[(n + j) * ldk + n + i] = -scale * kee;
}

// Energy parts of a row block of K_nm (sgdml_b200_assemble_ecstr_rows): row point a = m_begin + blockIdx.y, column
// item blockIdx.x.  An item is either one energy column 3NM + q at output column dst >= 0 -- the pair (q, a) gives
// the force rows of a (r) and the energy row of a (K_ee) in that column -- or the selected force columns of point q
// (dst = -1 - t, fdest[t*3N + k] = output column of component k or -1) -- the pair (a, q) gives the energy row of a
// in them.  Force rows come first in K (n_rowpts * 3N of them), then one energy row per row point.
__global__ void __launch_bounds__(1024) k_assemble_ecstr_rows(const double* __restrict__ R_desc,
                                                             const double* __restrict__ R_d_desc,
                                                             const int* __restrict__ aperm_inv, int N, int D, int S,
                                                             double sig, double scale, const int* __restrict__ item_pt,
                                                             const int64_t* __restrict__ item_dst,
                                                             const int64_t* __restrict__ fdest, int m_begin,
                                                             int64_t n_frows, double* __restrict__ K, int64_t ldk) {
  __shared__ double red[32];
  __shared__ double s_cp, s_kee;
  const int a = m_begin + (int)blockIdx.y, q = item_pt[blockIdx.x];
  const int64_t dst = item_dst[blockIdx.x];
  const bool ecol = dst >= 0;
  const int i = ecol ? q : a, j = ecol ? a : q;
  const int b = threadIdx.x;
  double r0, r1, r2, kee;
  ecstr_pair(R_desc + (int64_t)i * D, R_desc + (int64_t)j * D, R_d_desc + (int64_t)j * D * 3, aperm_inv, N, S, sig, red,
             s_cp, s_kee, r0, r1, r2, kee);
  const int N3 = 3 * N;
  double* rowE = K + (n_frows + blockIdx.y) * ldk;
  if (ecol) {
    if (b < N) {
      double* Kf = K + ((int64_t)blockIdx.y * N3 + 3 * b) * ldk + dst;
      Kf[0] = scale * r0;
      Kf[ldk] = scale * r1;
      Kf[2 * ldk] = scale * r2;
    }
    if (threadIdx.x == 0) rowE[dst] = -scale * kee;
  } else if (b < N) {
    const int64_t* d3 = fdest + (-1 - dst) * N3 + 3 * b;
    if (d3[0] >= 0) rowE[d3[0]] = scale * r0;
    if (d3[1] >= 0) rowE[d3[1]] = scale * r1;
    if (d3[2] >= 0) rowE[d3[2]] = scale * r2;
  }
}

// bound on the slabs of k_assemble_large, one per persistent CTA (sgdml_b200_assemble_rows)
constexpr size_t ASM_SLAB_BYTES_MAX = (size_t)2 << 30;

static size_t asm_large_slab_doubles(int N, int S) {
  const size_t N3 = 3 * (size_t)N, NN = (size_t)N * N;
  return 2 * (NN * 3 + NN) + (size_t)S * (2 * N3 + 3 * N3 + 2) + NN;
}

static size_t asm_v4_smem_bytes(int N, int S, int TJ, int PG) {
  const size_t N3 = 3 * (size_t)N, GS = N3 | 1, XS = (size_t)N | 1;
  const size_t dbl = (size_t)N * (GS + XS) * (1 + TJ) + (size_t)TJ * PG * (2 * N3 + 3 * N3 + N + 2);
  return dbl * 8 + ((size_t)TJ * N + TJ) * 4 + 2 * (size_t)S * N + 16;
}

static size_t asm_v5_smem_bytes(int N, int S, int TJ, int PG) {
  const size_t N3 = 3 * (size_t)N, D = (size_t)N * (N - 1) / 2;
  const size_t dbl = 4 * D * (1 + TJ) + (size_t)TJ * PG * (2 * N3 + 3 * N3 + N + 2);
  return dbl * 8 + ((size_t)TJ * N + TJ) * 4 + 2 * (size_t)S * N + 16;
}

static size_t asm_smem_bytes(int N, int D, int S, int TJ) {
  (void)D;
  const size_t N3 = 3 * (size_t)N, NN = (size_t)N * N;
  size_t dbl = NN * 3 + NN + (size_t)TJ * (NN * 3 + NN + NN + 2 * N3 + 3 * N3) + (size_t)S * TJ * 2 + (size_t)TJ * 8;
  return dbl * 8 + 2 * (size_t)S * N * 4 + 2 * (size_t)TJ * N * 4 + (size_t)TJ * 4 + 16;
}

}  // namespace sgdml

using namespace sgdml;

// Recovers the atom permutation P that induces a descriptor permutation (dperm[d(a,b)] =
// d(P a, P b)); returns false if dperm is not induced by any atom permutation.
static bool atom_perm_from_desc_perm(const int* dperm, int N, int* P) {
  const int D = N * (N - 1) / 2;
  if (N == 2) {
    P[0] = 0;
    P[1] = 1;
    return dperm[0] == 0;
  }
  for (int a = 0; a < N; ++a) {
    // two pairs containing a
    int o1 = (a == 0) ? 1 : 0, o2 = -1;
    for (int o = 0; o < N; ++o)
      if (o != a && o != o1) {
        o2 = o;
        break;
      }
    auto d_of = [](int x, int y) { return x > y ? x * (x - 1) / 2 + y : y * (y - 1) / 2 + x; };
    int e1 = dperm[d_of(a, o1)], e2 = dperm[d_of(a, o2)];
    int a1, b1, a2, b2;
    pair_from_d(e1, a1, b1);
    pair_from_d(e2, a2, b2);
    int common = -1;
    if (a1 == a2 || a1 == b2) common = a1;
    if (b1 == a2 || b1 == b2) common = (common == -1) ? b1 : -2;
    if (common < 0) return false;
    P[a] = common;
  }
  // verify
  std::vector<char> seen((size_t)N, 0);
  for (int a = 0; a < N; ++a) {
    if (P[a] < 0 || P[a] >= N || seen[(size_t)P[a]]) return false;
    seen[(size_t)P[a]] = 1;
  }
  for (int a = 1; a < N; ++a)
    for (int b = 0; b < a; ++b) {
      int pa = P[a], pb = P[b];
      int e = pa > pb ? pa * (pa - 1) / 2 + pb : pb * (pb - 1) / 2 + pa;
      if (dperm[a * (a - 1) / 2 + b] != e) return false;
    }
  (void)D;
  return true;
}

static int g_asm_variant = 0;  // 0: by size; 1: always the large-molecule kernel (tests)
static int g_asm_kernel = 0;  // small-molecule kernel: 0 = by size (default), 2 = k_assemble (per-permutation phases), 4 = k_assemble_v4 (chunked), 5 = k_assemble_v5 (chunked, compressed pair arrays)
static int g_asm_max_rowpts = 65535;  // row points per launch of k_assemble (grid.y limit; lowered by tests)

extern "C" int sgdml_b200_set_assemble_variant(int variant) {
  // 0 / 1: kernel choice; 1000 + r (test hook): at most r row points per launch of the small-molecule kernel
  if (variant >= 1000) {
    SG_ARG(variant - 1000 >= 1 && variant - 1000 <= 65535);
    g_asm_max_rowpts = variant - 1000;
    return 0;
  }
  if (variant == 2 || variant == 4 || variant == 5) {  // which small-molecule kernel
    g_asm_kernel = variant;
    return 0;
  }
  SG_ARG(variant == 0 || variant == 1);
  g_asm_variant = variant;
  if (variant == 0) g_asm_kernel = 0;  // back to the defaults
  return 0;
}

extern "C" int sgdml_b200_assemble_rows(const double* R_desc, const double* R_d_desc, const int64_t* tril_perms_lin,
                                        int64_t n_atoms, int64_t n_train, int64_t n_perms, double sig,
                                        const int64_t* col_idxs, int64_t n_cols, double scale, int64_t m_begin,
                                        int64_t m_end, double* K, int64_t ldk, void* stream) {
  SG_TRY(require_device());
  SG_ARG(R_desc != nullptr && R_d_desc != nullptr && tril_perms_lin != nullptr && K != nullptr);
  SG_ARG(n_atoms >= 2 && n_train >= 1 && n_perms >= 1 && sig > 0);
  SG_ARG(m_begin >= 0 && m_begin < m_end && m_end <= n_train);
  const int N = (int)n_atoms, M = (int)n_train, S = (int)n_perms;
  const int D = N * (N - 1) / 2, N3 = 3 * N;
  const int64_t n = (int64_t)M * N3;
  const int n_rowpts = (int)(m_end - m_begin);
  const int64_t n_rows = (int64_t)n_rowpts * N3;
  if (col_idxs == nullptr) SG_ARG(n_cols == n);
  SG_ARG(n_cols >= 1 && n_cols <= n && ldk >= n_cols);
  cudaStream_t s = (cudaStream_t)stream;

  // ---- integer tables (host)
  std::vector<int64_t> lin((size_t)S * D);
  if (is_device_ptr(tril_perms_lin))
    SG_CUDA(cudaMemcpy(lin.data(), tril_perms_lin, sizeof(int64_t) * lin.size(), cudaMemcpyDeviceToHost));
  else
    std::copy(tril_perms_lin, tril_perms_lin + lin.size(), lin.begin());
  std::vector<int> dperm((size_t)S * D), aperm((size_t)S * N), apinv((size_t)S * N);
  for (int pp = 0; pp < S; ++pp) {
    for (int d = 0; d < D; ++d) {
      const int64_t e = lin[(size_t)d * S + pp] - (int64_t)pp * D;
      SG_ARG(e >= 0 && e < D);
      dperm[(size_t)pp * D + d] = (int)e;
    }
    if (!atom_perm_from_desc_perm(&dperm[(size_t)pp * D], N, &aperm[(size_t)pp * N]))
      return fail_arg("tril_perms_lin is not induced by atom permutations (utils/desc.py:509-539)");
    for (int a = 0; a < N; ++a) apinv[(size_t)pp * N + aperm[(size_t)pp * N + a]] = a;
  }
  // block-columns and destination map (train.py:1357-1407)
  std::vector<int> jpts;
  std::vector<int64_t> dest;
  if (col_idxs == nullptr) {
    jpts.resize((size_t)M);
    dest.resize((size_t)M * N3);
    for (int j = 0; j < M; ++j) {
      jpts[(size_t)j] = j;
      for (int k = 0; k < N3; ++k) dest[(size_t)j * N3 + k] = (int64_t)j * N3 + k;
    }
  } else {
    std::vector<int64_t> cols((size_t)n_cols);
    if (is_device_ptr(col_idxs))
      SG_CUDA(cudaMemcpy(cols.data(), col_idxs, sizeof(int64_t) * cols.size(), cudaMemcpyDeviceToHost));
    else
      std::copy(col_idxs, col_idxs + n_cols, cols.begin());
    for (int64_t c = 0; c < n_cols; ++c) {
      SG_ARG(cols[(size_t)c] >= 0 && cols[(size_t)c] < n);
      if (c > 0 && cols[(size_t)c] <= cols[(size_t)c - 1])
        return fail_arg("col_idxs must be sorted ascending without duplicates (train.py:1341-1345)");
      const int j = (int)(cols[(size_t)c] / N3), k = (int)(cols[(size_t)c] % N3);
      if (jpts.empty() || jpts.back() != j) {
        jpts.push_back(j);
        dest.insert(dest.end(), (size_t)N3, (int64_t)-1);
      }
      dest[(jpts.size() - 1) * N3 + k] = c;
    }
  }
  const int nJ = (int)jpts.size();
  // kept column atoms per column point, at most: the sub-blocks of a block are dealt out over N * NK (row atom, kept
  // column atom) pairs -- N * N for the full matrix, far fewer for the column subsets of the Nystroem set-up
  int NK = 1;
  for (int jt = 0; jt < nJ; ++jt) {
    int c = 0;
    for (int b = 0; b < N; ++b) {
      const int64_t* d3 = &dest[(size_t)jt * N3 + 3 * b];
      if (d3[0] >= 0 || d3[1] >= 0 || d3[2] >= 0) ++c;
    }
    NK = std::max(NK, c);
  }

  // ---- tile size: at most ASM_NI 3x3 sub-blocks per thread, and shared memory small enough for
  //      two co-resident CTAs per SM
  int TJ = 0, n_chunks = 1;
  bool large = g_asm_variant == 1;
  for (int t = 8; t >= 1 && !large; --t)
    if ((int64_t)t * N * N <= (int64_t)ASM_NI * 256 && asm_smem_bytes(N, D, S, t) <= 110 * 1024) {
      TJ = t;
      break;
    }
  if (TJ == 0 && !large) {
    // mid-sized molecule: one column point per CTA, its N*N sub-blocks split over grid.z (the
    // per-permutation vectors are then recomputed by every chunk)
    TJ = 1;
    n_chunks = (int)(((int64_t)N * NK + ASM_NI * 256 - 1) / (ASM_NI * 256));
    if (asm_smem_bytes(N, D, S, 1) > 220 * 1024) large = true;  // tables beyond shared memory: k_assemble_large
  }
  // v5 kernel (compressed pair arrays on chip): for molecules whose expanded tables do not fit shared memory, up to
  // ~64 atoms; one column point per CTA, chunks of up to 16 permutations
  int PG5 = std::min(S, 16);
  while (PG5 > 1 && asm_v5_smem_bytes(N, S, 1, PG5) > 220 * 1024) --PG5;
  const size_t smem5 = asm_v5_smem_bytes(N, S, 1, PG5);
  const bool fits5 = N <= 255 && smem5 <= 220 * 1024 && (PG5 >= 4 || PG5 == S);
  const bool use_v5 = g_asm_variant != 1 && fits5 && (g_asm_kernel == 5 || (g_asm_kernel == 0 && large));
  if (use_v5) {
    large = false;
    TJ = 1;
    n_chunks = (int)(((int64_t)N * NK + ASM_NI * 256 - 1) / (ASM_NI * 256));
  }
  if (large) TJ = 1;
  TJ = std::min(TJ, nJ);
  const size_t smem = asm_smem_bytes(N, D, S, TJ);
  SG_ARG((int64_t)N * N < (1 << 20) && N < 4096);  // fastdiv range

  Staged sX, sG, sK;
  SG_TRY(sX.init(R_desc, sizeof(double) * (size_t)M * D, true, s));
  SG_TRY(sG.init(R_d_desc, sizeof(double) * (size_t)M * D * 3, true, s));
  const bool K_host = !is_device_ptr(K);
  SG_TRY(sK.init(K, sizeof(double) * (size_t)n_rows * ldk, false, s));
  if (K_host && ldk != n_cols) SG_CUDA(cudaMemsetAsync(sK.dev(), 0, sizeof(double) * (size_t)n_rows * ldk, s));

  int *d_dperm = nullptr, *d_aperm = nullptr, *d_apinv = nullptr, *d_jpts = nullptr;
  int64_t* d_dest = nullptr;
  double* d_slabs = nullptr;
  // the integer tables (and the large-molecule kernel's slabs) live in persistent workspaces: a cudaMalloc / cudaFree
  // pair per table costs milliseconds once the K buffer and the factorisation workspaces exist
  auto cleanup = [&]() {};
  auto body = [&]() -> int {
    SG_TRY(ws_get(WS_ASM_DPERM, sizeof(int) * dperm.size(), (void**)&d_dperm));
    SG_TRY(ws_get(WS_ASM_APERM, sizeof(int) * aperm.size(), (void**)&d_aperm));
    SG_TRY(ws_get(WS_ASM_APINV, sizeof(int) * apinv.size(), (void**)&d_apinv));
    SG_TRY(ws_get(WS_ASM_JPTS, sizeof(int) * jpts.size(), (void**)&d_jpts));
    SG_TRY(ws_get(WS_ASM_DEST, sizeof(int64_t) * dest.size(), (void**)&d_dest));
    SG_CUDA(cudaMemcpyAsync(d_dperm, dperm.data(), sizeof(int) * dperm.size(), cudaMemcpyHostToDevice, s));
    SG_CUDA(cudaMemcpyAsync(d_aperm, aperm.data(), sizeof(int) * aperm.size(), cudaMemcpyHostToDevice, s));
    SG_CUDA(cudaMemcpyAsync(d_apinv, apinv.data(), sizeof(int) * apinv.size(), cudaMemcpyHostToDevice, s));
    SG_CUDA(cudaMemcpyAsync(d_jpts, jpts.data(), sizeof(int) * jpts.size(), cudaMemcpyHostToDevice, s));
    SG_CUDA(cudaMemcpyAsync(d_dest, dest.data(), sizeof(int64_t) * dest.size(), cudaMemcpyHostToDevice, s));
    AsmArgs a;
    a.R_desc = (const double*)sX.dev();
    a.R_d_desc = (const double*)sG.dev();
    a.dperm = d_dperm;
    a.aperm = d_aperm;
    a.apinv = d_apinv;
    a.jpts = d_jpts;
    a.dest = d_dest;
    a.N = N;
    a.D = D;
    a.M = M;
    a.S = S;
    a.nJ = nJ;
    a.TJ = TJ;
    a.i0 = (int)m_begin;
    // symmetric mode (upper block triangle computed, lower mirrored) needs every row point in this call
    a.sym = (col_idxs == nullptr && n_rowpts == M && !large) ? 1 : 0;
    a.mN = (unsigned)((0x100000000ull + N - 1) / N);
    a.mNN = (unsigned)((0x100000000ull + (uint64_t)N * N - 1) / ((uint64_t)N * N));
    a.mPer = (unsigned)((0x100000000ull + 5 * N - 1) / (5 * N));
    a.NK = NK;
    a.mNK = (unsigned)((0x100000000ull + NK - 1) / NK);
    a.mNNK = (unsigned)((0x100000000ull + (uint64_t)N * NK - 1) / ((uint64_t)N * NK));
    a.sig = sig;
    a.scale = scale;
    a.K = (double*)sK.dev();
    a.ldk = ldk;
    if (!large) {
      // rows on grid.y, column tiles on grid.x; grid.y is limited to 65535, so longer row ranges (the
      // iterative solver assembles K_nm over ALL training points of a rank) run as several launches,
      // each with its own first row point and K row offset
      const int max_rows_per_launch = g_asm_max_rowpts;
      if (n_rowpts > max_rows_per_launch) a.sym = 0;  // the mirrored store addresses absolute row points
      // v4 kernel: chunks of up to 16 permutations; two CTAs per SM when everything fits in ~110 KB, else one
      int PG4 = std::min(S, 16);
      while (PG4 > 1 && (asm_v4_smem_bytes(N, S, TJ, PG4) > 220 * 1024 || TJ * PG4 > 256)) --PG4;
      if (PG4 == S && asm_v4_smem_bytes(N, S, TJ, PG4) > 110 * 1024) {
        int q = PG4;
        while (q > 8 && asm_v4_smem_bytes(N, S, TJ, q) > 110 * 1024) --q;
        if (asm_v4_smem_bytes(N, S, TJ, q) <= 110 * 1024) PG4 = q;
      }
      const size_t smem4 = asm_v4_smem_bytes(N, S, TJ, PG4);
      // chosen by timing the variants (tools/asm_variants.py) at BASELINE config 2 (full matrix) and on the Ac-Ala3 shape
      // (S = 243, random column subsets): v4 was the fastest on both -- v4 is the default
      const bool use_v4 = N <= 255 && smem4 <= 220 * 1024 && TJ * PG4 <= 256 && (g_asm_kernel == 4 || g_asm_kernel == 0);
      const int tiles_per_cta = 4;
      if (use_v5) {
        SG_CUDA(cudaFuncSetAttribute(k_assemble_v5, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem5));
      } else if (use_v4) {
        SG_CUDA(cudaFuncSetAttribute(k_assemble_v4, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem4));
      } else
        SG_CUDA(cudaFuncSetAttribute(k_assemble, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      ProfScope ps(KID_ASSEMBLE, s);
      for (int r0 = 0; r0 < n_rowpts; r0 += max_rows_per_launch) {
        const int nr = std::min(max_rows_per_launch, n_rowpts - r0);
        AsmArgs ac = a;
        ac.i0 = (int)m_begin + r0;
        ac.K = a.K + (int64_t)r0 * N3 * ldk;
        if (use_v5) {
          dim3 grid((unsigned)ceil_div(nJ, tiles_per_cta), (unsigned)nr, (unsigned)n_chunks);
          k_assemble_v5<<<grid, 256, smem5, s>>>(ac, PG5, tiles_per_cta);
        } else if (use_v4) {
          dim3 grid((unsigned)ceil_div(ceil_div(nJ, TJ), tiles_per_cta), (unsigned)nr, (unsigned)n_chunks);
          k_assemble_v4<<<grid, 256, smem4, s>>>(ac, PG4, tiles_per_cta);
        } else {
          dim3 grid((unsigned)ceil_div(nJ, TJ), (unsigned)nr, (unsigned)n_chunks);
          k_assemble<<<grid, 256, smem, s>>>(ac);
        }
        SG_CUDA(cudaGetLastError());
        count_launch(KID_ASSEMBLE);
      }
    } else {
      int dev = 0, n_sm = 0;
      SG_CUDA(cudaGetDevice(&dev));
      SG_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
      const int64_t n_work = (int64_t)n_rowpts * nJ;
      const size_t dl_bytes = sizeof(double) * (size_t)N * N;
      const int dl_in_smem = dl_bytes <= 100 * 1024 ? 1 : 0;  // two CTAs per SM keep their delta tables on chip
      const size_t slab = (asm_large_slab_doubles(N, S) + 1) / 2 * 2;
      // persistent, 2 per SM; fewer once the slabs (kept in a workspace until sgdml_b200_release_workspaces) would pass
      // ASM_SLAB_BYTES_MAX: on 132 SMs from N ~ 335 at S = 3 (214 CTAs of 10 MB at N = 370); C60 takes 0.3 GB
      const int64_t slab_ctas = std::max<int64_t>(1, (int64_t)(ASM_SLAB_BYTES_MAX / (sizeof(double) * slab)));
      const int n_cta = (int)std::min<int64_t>(std::min<int64_t>(n_work, 2 * (int64_t)n_sm), slab_ctas);
      SG_TRY(ws_get(WS_ASM_SLABS, sizeof(double) * slab * (size_t)n_cta, (void**)&d_slabs));
      if (dl_in_smem)
        SG_CUDA(cudaFuncSetAttribute(k_assemble_large, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dl_bytes));
      ProfScope ps(KID_ASSEMBLE, s);
      k_assemble_large<<<n_cta, 256, dl_in_smem ? dl_bytes : 0, s>>>(a, d_slabs, (int64_t)slab, n_work, dl_in_smem);
      SG_CUDA(cudaGetLastError());
      count_launch(KID_ASSEMBLE);
    }
    SG_TRY(sK.finish(s));
    // the integer tables are read by the kernel: wait before freeing them
    SG_CUDA(cudaStreamSynchronize(s));
    return 0;
  };
  int rc = body();
  cleanup();
  return rc;
}

extern "C" int sgdml_b200_assemble(const double* R_desc, const double* R_d_desc, const int64_t* tril_perms_lin,
                                   int64_t n_atoms, int64_t n_train, int64_t n_perms, double sig,
                                   const int64_t* col_idxs, int64_t n_cols, double scale, double* K, int64_t ldk,
                                   void* stream) {
  return sgdml_b200_assemble_rows(R_desc, R_d_desc, tril_perms_lin, n_atoms, n_train, n_perms, sig, col_idxs, n_cols,
                                  scale, 0, n_train, K, ldk, stream);
}

// Inverse atom permutations (S x N) of tril_perms_lin, the tables of the energy-constraint kernels.
static int ecstr_apinv(const int64_t* tril_perms_lin, int N, int S, std::vector<int>& apinv) {
  const int D = N * (N - 1) / 2;
  std::vector<int64_t> lin((size_t)S * D);
  if (is_device_ptr(tril_perms_lin))
    SG_CUDA(cudaMemcpy(lin.data(), tril_perms_lin, sizeof(int64_t) * lin.size(), cudaMemcpyDeviceToHost));
  else
    std::copy(tril_perms_lin, tril_perms_lin + lin.size(), lin.begin());
  std::vector<int> dperm((size_t)D), aperm((size_t)N);
  apinv.assign((size_t)S * N, 0);
  for (int pp = 0; pp < S; ++pp) {
    for (int d = 0; d < D; ++d) {
      const int64_t e = lin[(size_t)d * S + pp] - (int64_t)pp * D;
      SG_ARG(e >= 0 && e < D);
      dperm[(size_t)d] = (int)e;
    }
    if (!atom_perm_from_desc_perm(dperm.data(), N, aperm.data()))
      return fail_arg("tril_perms_lin is not induced by atom permutations (utils/desc.py:509-539)");
    for (int a = 0; a < N; ++a) apinv[(size_t)pp * N + aperm[(size_t)a]] = a;
  }
  return 0;
}

// GDMLTrain._assemble_kernel_mat(use_E_cstr=True), train.py:234-300: fills the M energy rows and columns (and the
// M x M energy-energy block) of the (3NM + M)-square matrix whose force-force part sgdml_b200_assemble writes.
extern "C" int sgdml_b200_assemble_ecstr(const double* R_desc, const double* R_d_desc, const int64_t* tril_perms_lin,
                                         int64_t n_atoms, int64_t n_train, int64_t n_perms, double sig, double scale,
                                         double* K, int64_t ldk, void* stream) {
  SG_TRY(require_device());
  SG_ARG(R_desc != nullptr && R_d_desc != nullptr && tril_perms_lin != nullptr && K != nullptr);
  SG_ARG(n_atoms >= 2 && n_atoms <= 1023 && n_train >= 1 && n_train <= 65535 && n_perms >= 1 && sig > 0);
  const int N = (int)n_atoms, M = (int)n_train, S = (int)n_perms;
  const int D = N * (N - 1) / 2;
  const int64_t nt = (int64_t)M * 3 * N + M;
  SG_ARG(ldk >= nt && is_device_ptr(K));
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<int> apinv;
  SG_TRY(ecstr_apinv(tril_perms_lin, N, S, apinv));
  Staged sX, sG;
  SG_TRY(sX.init(R_desc, sizeof(double) * (size_t)M * D, true, s));
  SG_TRY(sG.init(R_d_desc, sizeof(double) * (size_t)M * D * 3, true, s));
  int* d_apinv = nullptr;
  SG_CUDA(cudaMalloc(&d_apinv, sizeof(int) * apinv.size()));
  auto body = [&]() -> int {
    SG_CUDA(cudaMemcpyAsync(d_apinv, apinv.data(), sizeof(int) * apinv.size(), cudaMemcpyHostToDevice, s));
    ProfScope ps(KID_ASSEMBLE, s);
    k_assemble_ecstr<<<dim3((unsigned)M, (unsigned)M), (N + 31) / 32 * 32, 0, s>>>(
        (const double*)sX.dev(), (const double*)sG.dev(), d_apinv, N, D, M, S, sig, scale, K, ldk);
    SG_CUDA(cudaGetLastError());
    count_launch(KID_ASSEMBLE);
    SG_CUDA(cudaStreamSynchronize(s));
    return 0;
  };
  int rc = body();
  cudaFree(d_apinv);
  return rc;
}

// Row block of the energy-constrained K_nm (the Nystroem set-up of iterative.py:232-247 with use_E_cstr): the force
// prefix of the column list goes through sgdml_b200_assemble_rows, every other entry through k_assemble_ecstr_rows,
// which computes each (row point, column point) pair the list touches once.
extern "C" int sgdml_b200_assemble_ecstr_rows(const double* R_desc, const double* R_d_desc,
                                              const int64_t* tril_perms_lin, int64_t n_atoms, int64_t n_train,
                                              int64_t n_perms, double sig, const int64_t* col_idxs, int64_t n_cols,
                                              double scale, int64_t m_begin, int64_t m_end, double* K, int64_t ldk,
                                              void* stream) {
  SG_TRY(require_device());
  SG_ARG(R_desc != nullptr && R_d_desc != nullptr && tril_perms_lin != nullptr && col_idxs != nullptr && K != nullptr);
  SG_ARG(n_atoms >= 2 && n_atoms <= 1023 && n_train >= 1 && n_train <= 65535 && n_perms >= 1 && sig > 0);
  SG_ARG(m_begin >= 0 && m_begin < m_end && m_end <= n_train);
  const int N = (int)n_atoms, M = (int)n_train, S = (int)n_perms;
  const int D = N * (N - 1) / 2, N3 = 3 * N;
  const int64_t n = (int64_t)M * N3, nt = n + M;
  SG_ARG(n_cols >= 1 && n_cols <= nt && ldk >= n_cols && is_device_ptr(K));
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<int64_t> cols((size_t)n_cols);
  if (is_device_ptr(col_idxs))
    SG_CUDA(cudaMemcpy(cols.data(), col_idxs, sizeof(int64_t) * cols.size(), cudaMemcpyDeviceToHost));
  else
    std::copy(col_idxs, col_idxs + n_cols, cols.begin());
  int64_t n_fcols = 0;
  for (int64_t c = 0; c < n_cols; ++c) {
    SG_ARG(cols[(size_t)c] >= 0 && cols[(size_t)c] < nt);
    if (c > 0 && cols[(size_t)c] <= cols[(size_t)c - 1])
      return fail_arg("col_idxs must be sorted ascending without duplicates (train.py:1341-1345)");
    if (cols[(size_t)c] < n) ++n_fcols;
  }
  std::vector<int> apinv;
  SG_TRY(ecstr_apinv(tril_perms_lin, N, S, apinv));
  // force rows x force columns: exactly the row block sgdml_b200_assemble_rows writes
  if (n_fcols > 0)
    SG_TRY(sgdml_b200_assemble_rows(R_desc, R_d_desc, tril_perms_lin, n_atoms, n_train, n_perms, sig, col_idxs,
                                    n_fcols, scale, m_begin, m_end, K, ldk, stream));
  // column items: one per force-column point (with its destination map), one per energy column
  std::vector<int> item_pt;
  std::vector<int64_t> item_dst, fdest;
  for (int64_t c = 0; c < n_fcols; ++c) {
    const int q = (int)(cols[(size_t)c] / N3), k = (int)(cols[(size_t)c] % N3);
    if (item_pt.empty() || item_pt.back() != q) {
      item_dst.push_back(-1 - (int64_t)item_pt.size());
      item_pt.push_back(q);
      fdest.insert(fdest.end(), (size_t)N3, (int64_t)-1);
    }
    fdest[(item_pt.size() - 1) * N3 + k] = c;
  }
  for (int64_t c = n_fcols; c < n_cols; ++c) {
    item_pt.push_back((int)(cols[(size_t)c] - n));
    item_dst.push_back(c);
  }
  const int64_t n_items = (int64_t)item_pt.size();
  const int n_rowpts = (int)(m_end - m_begin);
  Staged sX, sG;
  SG_TRY(sX.init(R_desc, sizeof(double) * (size_t)M * D, true, s));
  SG_TRY(sG.init(R_d_desc, sizeof(double) * (size_t)M * D * 3, true, s));
  int *d_apinv = nullptr, *d_pt = nullptr;
  int64_t *d_dst = nullptr, *d_fdest = nullptr;
  auto body = [&]() -> int {
    SG_CUDA(cudaMalloc(&d_apinv, sizeof(int) * apinv.size()));
    SG_CUDA(cudaMalloc(&d_pt, sizeof(int) * (size_t)n_items));
    SG_CUDA(cudaMalloc(&d_dst, sizeof(int64_t) * (size_t)n_items));
    SG_CUDA(cudaMalloc(&d_fdest, sizeof(int64_t) * std::max<size_t>(fdest.size(), 1)));
    SG_CUDA(cudaMemcpyAsync(d_apinv, apinv.data(), sizeof(int) * apinv.size(), cudaMemcpyHostToDevice, s));
    SG_CUDA(cudaMemcpyAsync(d_pt, item_pt.data(), sizeof(int) * (size_t)n_items, cudaMemcpyHostToDevice, s));
    SG_CUDA(cudaMemcpyAsync(d_dst, item_dst.data(), sizeof(int64_t) * (size_t)n_items, cudaMemcpyHostToDevice, s));
    if (!fdest.empty())
      SG_CUDA(cudaMemcpyAsync(d_fdest, fdest.data(), sizeof(int64_t) * fdest.size(), cudaMemcpyHostToDevice, s));
    ProfScope ps(KID_ASSEMBLE, s);
    k_assemble_ecstr_rows<<<dim3((unsigned)n_items, (unsigned)n_rowpts), (N + 31) / 32 * 32, 0, s>>>(
        (const double*)sX.dev(), (const double*)sG.dev(), d_apinv, N, D, S, sig, scale, d_pt, d_dst, d_fdest,
        (int)m_begin, (int64_t)n_rowpts * N3, K, ldk);
    SG_CUDA(cudaGetLastError());
    count_launch(KID_ASSEMBLE);
    SG_CUDA(cudaStreamSynchronize(s));  // the tables are freed below
    return 0;
  };
  int rc = body();
  cudaFree(d_apinv);
  cudaFree(d_pt);
  cudaFree(d_dst);
  cudaFree(d_fdest);
  return rc;
}
