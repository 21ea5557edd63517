// Permutation discovery, stage one (utils/perm.py:53-235, bipartite_match): for every pair of training geometries the
// assignment of the atoms of one to the atoms of the other that best aligns the eigenvectors of their distance
// matrices, and the distance-matrix mismatch before and after it.  One CTA per (geometry i, range of 16 geometries j):
//   cost = -|V_i| |V_j|^T                  tiled FP64 FMA product through shared memory   (perm.py:70)
//   penalty = max|cost| between species    folded into the solver's cost lookup            (perm.py:71, 97-98)
//   assignment                             shortest augmenting paths, perm_solve.cuh       (perm.py:73)
//   |adj_i - adj_j|_F, |adj_i[perm][:, perm] - adj_j|_F, and what perm.py:78-85 keeps of them.
// Up to 112 atoms the cost matrix and |V_i| stay in shared memory while the CTA walks its j; beyond that the cost matrix
// lives in a slab of global memory per (persistent) CTA and |V_i| is read through L2.  The code is the same: only the
// pointers differ.  Every reduction has a fixed order, so results are bit-identical between runs and between the
// all-pairs and the pair-list form.
#include <algorithm>

#include "common.cuh"
#include "perm_solve.cuh"

namespace sgdml {
namespace {

constexpr int PM_JC = 16;          // geometries j per work item
constexpr int PM_SMEM_ATOMS = 112; // largest N with the cost matrix and |V_i| in shared memory
constexpr int PM_TILE = 32;        // the product is computed in 32 x 32 tiles

struct PermPlan {
  int in_smem;       // 1: cost matrix and |V_i| in shared memory, 0: cost matrix in a global slab
  int threads;       // 32 / 64 / 128 / 256
  int ld;            // row stride of the cost matrix (odd: conflict-free column walks)
  size_t smem;       // dynamic shared memory bytes
  int64_t slab;      // doubles per CTA in the global slab (0 when in_smem)
  int ctas_per_sm;   // persistent CTAs per SM
};

int perm_kc(int threads) { return threads == 32 ? 8 : 16; }

PermPlan make_plan(int n) {
  PermPlan p;
  p.in_smem = n <= PM_SMEM_ATOMS;
  p.threads = n <= 32 ? 32 : n <= 64 ? 64 : n <= 128 ? 128 : 256;
  p.ld = n | 1;
  const size_t mat = (size_t)n * p.ld;
  size_t doubles = (p.in_smem ? 2 * mat : 0) + 2 * (size_t)perm_kc(p.threads) * (PM_TILE + 1) + 3 * (size_t)n + 16 + 2 * 8;
  size_t bytes = doubles * 8 + (2 * 8 + 4 * (size_t)n) * 4 + (size_t)n;
  p.smem = (bytes + 15) / 16 * 16;
  p.slab = p.in_smem ? 0 : (int64_t)mat;
  p.ctas_per_sm = p.in_smem ? 32 : 2;
  return p;
}

struct PermArgs {
  const double* adj;
  const double* absv;
  const int* z;
  int n_geo, n;
  const int64_t* pairs;  // device, or NULL for all pairs
  int64_t n_pairs;
  double* match_cost;
  int32_t* perms;
  uint8_t* has_perm;
  double* slab;
  int64_t slab_stride;
  int64_t n_items;
  int chunks_per_row;
  int in_smem, ld;
};

template <int T>
struct BlockTeam {
  int tid;
  static constexpr int size = T;
  double* red_val;  // [2][8]
  int* red_idx;     // [2][8]
  mutable int parity;
  __device__ __forceinline__ void sync() const {
    if (T == 32)
      __syncwarp();
    else
      __syncthreads();
  }
  __device__ __forceinline__ perm::ArgMin argmin(perm::ArgMin a) const {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      perm::ArgMin b;
      b.val = __shfl_xor_sync(0xffffffffu, a.val, o);
      b.idx = __shfl_xor_sync(0xffffffffu, a.idx, o);
      a = perm::argmin2(a, b);
    }
    // with NaN among the values the butterfly's lanes may disagree: lane 0 decides
    a.val = __shfl_sync(0xffffffffu, a.val, 0);
    a.idx = __shfl_sync(0xffffffffu, a.idx, 0);
    if (T == 32) return a;
    // one barrier per call: the scratch alternates, and a thread can only be two calls ahead of another after that one
    // has passed the barrier in between
    double* rv = red_val + 8 * parity;
    int* ri = red_idx + 8 * parity;
    parity ^= 1;
    if ((tid & 31) == 0) {
      rv[tid >> 5] = a.val;
      ri[tid >> 5] = a.idx;
    }
    __syncthreads();
    perm::ArgMin r;
    r.val = rv[0];
    r.idx = ri[0];
#pragma unroll
    for (int w = 1; w < T / 32; ++w) {
      perm::ArgMin b;
      b.val = rv[w];
      b.idx = ri[w];
      r = perm::argmin2(r, b);
    }
    return r;
  }
};

// Fixed-order block reductions (lane tree, then the warps in order); red: 8 doubles of shared memory.
template <int T, bool MAX>
__device__ __forceinline__ double block_reduce(double x, double* red, int tid) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double y = __shfl_xor_sync(0xffffffffu, x, o);
    x = MAX ? fmax(x, y) : x + y;
  }
  if (T == 32) return x;
  __syncthreads();  // earlier readers of red are done
  if ((tid & 31) == 0) red[tid >> 5] = x;
  __syncthreads();
  double r = red[0];
#pragma unroll
  for (int w = 1; w < T / 32; ++w) r = MAX ? fmax(r, red[w]) : r + red[w];
  return r;
}

// C[a][b] = -sum_k A[a][k] B[b][k] for a, b < n (A, B, C in shared or global memory); returns this thread's max |C|.
// TA x 32 tiles (TA = 16 for a single warp, which keeps its accumulators in registers at 16 CTAs per SM, else 32), k in
// slices of KC staged transposed in shared memory; thread t owns column t % 32 of the tile and the rows
// t / 32 + (T / 32) r.
template <int T, int KC>
__device__ __forceinline__ double neg_product_nt(const double* A, int lda, const double* __restrict__ B, int ldb,
                                                 double* C, int ldc, int n, double* As, double* Bs, int tid) {
  constexpr int TA = T == 32 ? 16 : PM_TILE;
  constexpr int R = TA * PM_TILE / T;
  constexpr int LDS = PM_TILE + 1;
  const int tb = tid & 31, ta = tid >> 5;
  double mx = 0.0;
  for (int a0 = 0; a0 < n; a0 += TA) {
    for (int b0 = 0; b0 < n; b0 += PM_TILE) {
      double acc[R];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = 0.0;
      for (int k0 = 0; k0 < n; k0 += KC) {
        for (int e = tid; e < PM_TILE * KC; e += T) {
          const int row = e / KC, kk = e % KC;
          const bool kin = k0 + kk < n;
          if (row < TA) As[kk * LDS + row] = (kin && a0 + row < n) ? A[(int64_t)(a0 + row) * lda + k0 + kk] : 0.0;
          Bs[kk * LDS + row] = (kin && b0 + row < n) ? B[(int64_t)(b0 + row) * ldb + k0 + kk] : 0.0;
        }
        if (T == 32) __syncwarp(); else __syncthreads();
#pragma unroll
        for (int kk = 0; kk < KC; ++kk) {
          const double bv = Bs[kk * LDS + tb];
#pragma unroll
          for (int r = 0; r < R; ++r) acc[r] = fma(As[kk * LDS + ta + (T / 32) * r], bv, acc[r]);
        }
        if (T == 32) __syncwarp(); else __syncthreads();
      }
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int a = a0 + ta + (T / 32) * r, b = b0 + tb;
        if (a < n && b < n) {
          C[(int64_t)a * ldc + b] = -acc[r];
          mx = fmax(mx, fabs(acc[r]));
        }
      }
    }
  }
  return mx;
}

// Register budget: 128 per thread (4 / 2 CTAs of 128 / 256 threads per SM); the single-warp variant gets 168 (12 CTAs per
// SM), below which its 16 x 32 product tile spills.
template <int T>
__global__ void __launch_bounds__(T, T == 32 ? 12 : 512 / T) k_bipartite_match(const PermArgs p) {
  constexpr int KC = T == 32 ? 8 : 16;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x, n = p.n, ld = p.ld;
  const size_t mat = (size_t)n * ld;
  double* sd = reinterpret_cast<double*>(smem_raw);
  double* cost = p.in_smem ? sd : p.slab + (int64_t)blockIdx.x * p.slab_stride;
  double* vi_s = sd + (p.in_smem ? mat : 0);
  double* As = sd + (p.in_smem ? 2 * mat : 0);
  double* Bs = As + KC * (PM_TILE + 1);
  double* u = Bs + KC * (PM_TILE + 1);
  double* v = u + n;
  double* spc = v + n;
  double* red = spc + n;        // 8 (+ 8 spare)
  double* red_val = red + 16;   // 2 x 8
  int* red_idx = reinterpret_cast<int*>(red_val + 16);  // 2 x 8
  int* path = red_idx + 16;
  int* row4col = path + n;
  int* col4row = row4col + n;
  int* zs = col4row + n;
  unsigned char* sc = reinterpret_cast<unsigned char*>(zs + n);

  BlockTeam<T> tm;
  tm.tid = tid;
  tm.red_val = red_val;
  tm.red_idx = red_idx;
  tm.parity = 0;

  for (int a = tid; a < n; a += T) zs[a] = p.z[a];
  int resident = -1;  // geometry whose |V| is in vi_s
  const int64_t nn = (int64_t)n * n;

  for (int64_t w = blockIdx.x; w < p.n_items; w += gridDim.x) {
    int64_t e0, e1;  // list entries, or j range of row gi
    int gi = 0;
    if (p.pairs != nullptr) {
      e0 = w * PM_JC;
      e1 = min(e0 + (int64_t)PM_JC, p.n_pairs);
    } else {
      gi = (int)(w / p.chunks_per_row);
      e0 = gi + 1 + (w % p.chunks_per_row) * (int64_t)PM_JC;
      e1 = min(e0 + (int64_t)PM_JC, (int64_t)p.n_geo);
    }
    for (int64_t e = e0; e < e1; ++e) {
      int gj;
      int64_t out;
      if (p.pairs != nullptr) {
        gi = (int)p.pairs[2 * e];
        gj = (int)p.pairs[2 * e + 1];
        out = e;
      } else {
        gj = (int)e;
        out = (int64_t)gi * p.n_geo - (int64_t)gi * (gi + 1) / 2 + (gj - gi - 1);
      }
      const double* Vi = p.absv + gi * nn;
      int ldvi = n;
      tm.sync();  // the previous pair's readers of cost, col4row and vi_s are done
      if (p.in_smem) {
        if (resident != gi) {
          for (int64_t q = tid; q < nn; q += T) vi_s[(q / n) * ld + q % n] = Vi[q];
          resident = gi;
          tm.sync();
        }
        Vi = vi_s;
        ldvi = ld;
      }
      double mx = neg_product_nt<T, KC>(Vi, ldvi, p.absv + gj * nn, n, cost, ld, n, As, Bs, tid);
      mx = block_reduce<T, true>(mx, red, tid);
      tm.sync();
      perm::lap_solve(tm, n, cost, ld, mx, zs, u, v, spc, path, row4col, col4row, sc);

      const double* adj_i = p.adj + gi * nn;
      const double* adj_j = p.adj + gj * nn;
      double s_before = 0.0, s_after = 0.0;
      for (int64_t q = tid; q < nn; q += T) {
        const int a = (int)(q / n), b = (int)(q % n);
        const double aj = adj_j[q];
        const double d0 = adj_i[q] - aj;
        const double d1 = adj_i[(int64_t)col4row[a] * n + col4row[b]] - aj;
        s_before = fma(d0, d0, s_before);
        s_after = fma(d1, d1, s_after);
      }
      s_before = sqrt(block_reduce<T, false>(s_before, red, tid));
      s_after = sqrt(block_reduce<T, false>(s_after, red, tid));
      if (tid == 0) {
        // perm.py:81-85; np.isclose(score_before, score) with its default tolerances
        const bool worse = s_after >= s_before;
        const bool close = fabs(s_before - s_after) <= 1e-8 + 1e-5 * fabs(s_after);
        const int64_t mc = p.pairs != nullptr ? out : (int64_t)gi * p.n_geo + gj;
        p.match_cost[mc] = worse ? s_before : s_after;
        if (p.has_perm != nullptr) p.has_perm[out] = (!worse && !close) ? 1 : 0;
      }
      if (p.perms != nullptr)
        for (int a = tid; a < n; a += T) p.perms[out * n + a] = col4row[a];
    }
  }
}

template <int T>
int launch_match(const PermArgs& a, const PermPlan& plan, int grid, cudaStream_t s) {
  SG_CUDA(cudaFuncSetAttribute(k_bipartite_match<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem));
  k_bipartite_match<T><<<grid, T, plan.smem, s>>>(a);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

}  // namespace
}  // namespace sgdml

using namespace sgdml;

extern "C" {

int sgdml_b200_bipartite_match_plan(int64_t n_atoms, int64_t* out) {
  SG_ARG(out != nullptr && n_atoms >= 2 && n_atoms <= 1023);
  const PermPlan p = make_plan((int)n_atoms);
  out[0] = p.in_smem ? 0 : 1;
  out[1] = p.threads;
  out[2] = (int64_t)p.smem;
  out[3] = p.slab;
  out[4] = p.ctas_per_sm;
  return 0;
}

int sgdml_b200_bipartite_match(const double* adj, const double* absv, const int64_t* z, int64_t n_geo, int64_t n_atoms,
                               const int64_t* pairs, int64_t n_pairs, double* match_cost, int32_t* perms,
                               uint8_t* has_perm, void* stream) {
  // argument checks first: none of them needs a device
  SG_ARG(adj != nullptr && absv != nullptr && z != nullptr && match_cost != nullptr);
  SG_ARG(n_atoms >= 2 && n_atoms <= 1023);
  SG_ARG(n_geo >= 1 && n_geo <= 65535);
  std::vector<int64_t> hp;
  if (pairs != nullptr) {
    SG_ARG(n_pairs >= 0);
    SG_TRY(read_int64s(pairs, (size_t)(2 * n_pairs), hp));
    for (int64_t e = 0; e < n_pairs; ++e)
      if (hp[2 * e] < 0 || hp[2 * e] >= hp[2 * e + 1] || hp[2 * e + 1] >= n_geo)
        return fail_arg("pairs must be (i, j) with 0 <= i < j < n_geo");
  }
  SG_TRY(require_device());
  const int64_t n_out = pairs != nullptr ? n_pairs : n_geo * (n_geo - 1) / 2;
  if (n_out == 0) return 0;
  std::vector<int64_t> hz64;
  SG_TRY(read_int64s(z, (size_t)n_atoms, hz64));
  std::vector<int> hz(hz64.begin(), hz64.end());

  cudaStream_t s = (cudaStream_t)stream;
  const int n = (int)n_atoms;
  const PermPlan plan = make_plan(n);
  const size_t geo_bytes = sizeof(double) * (size_t)n_geo * n * n;
  Staged sAdj, sV, sZ, sP, sCost, sPerm, sHas;
  SG_TRY(sAdj.init(adj, geo_bytes, true, s));
  SG_TRY(sV.init(absv, geo_bytes, true, s));
  SG_TRY(sZ.init(hz.data(), sizeof(int) * (size_t)n, true, s));
  if (pairs != nullptr) SG_TRY(sP.init(hp.data(), sizeof(int64_t) * (size_t)(2 * n_pairs), true, s));
  // all pairs: only the upper triangle of the (M, M) output is written, so a host buffer's other entries travel along
  SG_TRY(sCost.init(match_cost, sizeof(double) * (size_t)(pairs != nullptr ? n_pairs : n_geo * n_geo), pairs == nullptr, s));
  SG_TRY(sPerm.init(perms, sizeof(int32_t) * (size_t)n_out * n, false, s));
  SG_TRY(sHas.init(has_perm, (size_t)n_out, false, s));

  PermArgs a;
  a.adj = (const double*)sAdj.dev();
  a.absv = (const double*)sV.dev();
  a.z = (const int*)sZ.dev();
  a.n_geo = (int)n_geo;
  a.n = n;
  a.pairs = (const int64_t*)sP.dev();
  a.n_pairs = n_pairs;
  a.match_cost = (double*)sCost.dev();
  a.perms = (int32_t*)sPerm.dev();
  a.has_perm = (uint8_t*)sHas.dev();
  a.in_smem = plan.in_smem;
  a.ld = plan.ld;
  a.chunks_per_row = (int)((n_geo - 1 + PM_JC - 1) / PM_JC);
  a.n_items = pairs != nullptr ? (n_pairs + PM_JC - 1) / PM_JC : (n_geo - 1) * (int64_t)a.chunks_per_row;
  const int grid = (int)std::min<int64_t>(a.n_items, (int64_t)num_sms() * plan.ctas_per_sm);
  a.slab = nullptr;
  a.slab_stride = plan.slab;
  if (!plan.in_smem) {
    void* slab = nullptr;
    SG_TRY(ws_get(WS_PERM_SLAB, sizeof(double) * (size_t)plan.slab * grid, &slab));
    a.slab = (double*)slab;
  }
  {
    ProfScope ps(KID_MISC, s);
    switch (plan.threads) {
      case 32: SG_TRY(launch_match<32>(a, plan, grid, s)); break;
      case 64: SG_TRY(launch_match<64>(a, plan, grid, s)); break;
      case 128: SG_TRY(launch_match<128>(a, plan, grid, s)); break;
      default: SG_TRY(launch_match<256>(a, plan, grid, s)); break;
    }
  }
  SG_TRY(sCost.finish(s));
  SG_TRY(sPerm.finish(s));
  SG_TRY(sHas.finish(s));
  // the slab and the staged index arrays are reused by the next call: wait for the kernel
  SG_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
