// Normal-mode analysis on the device (include/sgdml_b200.h: sgdml_b200_vib_project, sgdml_b200_symeig_batched):
// the mass-weighted Hessian with its rigid modes moved to the top of the spectrum, and a batched symmetric eigensolver
// (parallel cyclic Jacobi, one CTA per matrix).  Every reduction runs in a fixed order and nothing uses atomics, so
// both calls return the same bits on every call.
#include <cfloat>

#include "common.cuh"

namespace sgdml {

namespace {

// A rotation is dropped from the rigid basis when Gram-Schmidt leaves less than this fraction of its norm: a linear
// geometry (bent by less than ~1e-6 rad) keeps 2 rotations.
constexpr double RIGID_TOL = 1e-6;
constexpr int VIB_THREADS = 256;
constexpr int SYMEIG_THREADS = 512;
constexpr int SYMEIG_MAX_SWEEPS = 60;

// Sum over the CTA in a fixed order: lanes by a shuffle tree, then the warps' partials in warp order.  Every thread gets
// the result.
template <int NT>
__device__ double block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();  // red may still be read from the previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < NT / 32; ++w) s += red[w];
  return s;
}

// One CTA per geometry: the rigid basis B (6 x n, rows a = tx, ty, tz, rx, ry, rz, n = 3N) in mass-weighted coordinates,
// orthonormalised by two Gram-Schmidt passes in that order; kept vectors are compacted to the first rows, the others are
// zero.  Translations: sqrt(m_i) e_c; rotations about the centre of mass: sqrt(m_i) (e_a x (r_i - r_com)).  Periodic
// models keep the translations only.
__global__ void __launch_bounds__(VIB_THREADS) k_vib_basis(const double* __restrict__ R,
                                                           const double* __restrict__ ism, int n_atoms, int periodic,
                                                           double* __restrict__ B, int64_t* __restrict__ n_rigid) {
  __shared__ double red[VIB_THREADS / 32];
  const int64_t g = blockIdx.x;
  const int n = 3 * n_atoms;
  const double* r = R + g * n;
  double* b = B + g * 6 * n;
  double mt = 0.0, mx = 0.0, my = 0.0, mz = 0.0;
  for (int i = threadIdx.x; i < n_atoms; i += blockDim.x) {
    const double mi = 1.0 / (ism[i] * ism[i]);
    mt += mi;
    mx += mi * r[3 * i + 0];
    my += mi * r[3 * i + 1];
    mz += mi * r[3 * i + 2];
  }
  mt = block_sum<VIB_THREADS>(mt, red);
  const double cx = block_sum<VIB_THREADS>(mx, red) / mt;
  const double cy = block_sum<VIB_THREADS>(my, red) / mt;
  const double cz = block_sum<VIB_THREADS>(mz, red) / mt;
  int kept = 0;
  const int n_raw = periodic ? 3 : 6;
  for (int a = 0; a < 6; ++a) {
    double* v = b + kept * n;  // candidate goes to the first free row
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
      const int i = j / 3, c = j - 3 * i;
      const double sm = 1.0 / ism[i];
      double x = 0.0;
      if (a < 3) {
        x = c == a ? sm : 0.0;
      } else if (a < n_raw) {
        const double dx = r[3 * i + 0] - cx, dy = r[3 * i + 1] - cy, dz = r[3 * i + 2] - cz;
        const auto d = [dx, dy, dz](int k) { return k == 0 ? dx : k == 1 ? dy : dz; };
        const int ax = a - 3;  // (e_ax x d)_c = eps_{c ax k} d_k
        const int c1 = (c + 1) % 3, c2 = (c + 2) % 3;
        x = (ax == c1 ? d(c2) : 0.0) - (ax == c2 ? d(c1) : 0.0);
        x *= sm;
      }
      v[j] = x;
    }
    __syncthreads();
    double nn = 0.0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) nn += v[j] * v[j];
    const double norm0 = sqrt(block_sum<VIB_THREADS>(nn, red));
    for (int pass = 0; pass < 2; ++pass) {
      for (int k = 0; k < kept; ++k) {
        const double* u = b + k * n;
        double dp = 0.0;
        for (int j = threadIdx.x; j < n; j += blockDim.x) dp += u[j] * v[j];
        dp = block_sum<VIB_THREADS>(dp, red);
        for (int j = threadIdx.x; j < n; j += blockDim.x) v[j] -= dp * u[j];
        __syncthreads();
      }
    }
    nn = 0.0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) nn += v[j] * v[j];
    const double norm = sqrt(block_sum<VIB_THREADS>(nn, red));
    const bool keep = norm0 > 0.0 && norm > RIGID_TOL * norm0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) v[j] = keep ? v[j] / norm : 0.0;
    __syncthreads();
    kept += keep ? 1 : 0;
  }
  for (int k = kept; k < 6; ++k)
    for (int j = threadIdx.x; j < n; j += blockDim.x) b[k * n + j] = 0.0;
  if (threadIdx.x == 0) n_rigid[g] = kept;
}

// Hm_ij = 1/2 (H_ij + H_ji) (s_i s_j) with s the inverse square roots of the masses: exactly symmetric
__device__ __forceinline__ double hm_entry(const double* __restrict__ h, const double* __restrict__ ism, int n, int i,
                                           int j) {
  return (0.5 * (h[(int64_t)i * n + j] + h[(int64_t)j * n + i])) * (ism[i / 3] * ism[j / 3]);
}

// One warp per row i of one geometry's Hm: Y[a][i] = (Hm B^T)_ia for the 6 basis rows, rowabs[i] = sum_j |Hm_ij|
__global__ void __launch_bounds__(256) k_vib_rows(const double* __restrict__ H, const double* __restrict__ ism,
                                                  const double* __restrict__ B, int n, double* __restrict__ Y,
                                                  double* __restrict__ rowabs) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= n) return;
  const int64_t g = blockIdx.y;
  const double* h = H + g * n * n;
  const double* b = B + g * 6 * n;
  double y[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  double ra = 0.0;
  for (int j = lane; j < n; j += 32) {
    const double x = hm_entry(h, ism, n, i, j);
    ra += fabs(x);
#pragma unroll
    for (int a = 0; a < 6; ++a) y[a] = fma(x, b[a * n + j], y[a]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ra += __shfl_xor_sync(0xffffffffu, ra, o);
#pragma unroll
    for (int a = 0; a < 6; ++a) y[a] += __shfl_xor_sync(0xffffffffu, y[a], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int a = 0; a < 6; ++a) Y[(g * 6 + a) * n + i] = y[a];
    rowabs[g * n + i] = ra;
  }
}

// One CTA per geometry: Z = B Hm B^T (6 x 6, symmetrised) and the shift c = 2 |Hm|_inf + 1 -> Z[g][0..35], Z[g][36]
__global__ void __launch_bounds__(VIB_THREADS) k_vib_small(const double* __restrict__ B, const double* __restrict__ Y,
                                                           const double* __restrict__ rowabs, int n,
                                                           double* __restrict__ Z) {
  __shared__ double red[VIB_THREADS / 32];
  __shared__ double z[36];
  const int64_t g = blockIdx.x;
  const double* b = B + g * 6 * n;
  const double* y = Y + g * 6 * n;
  for (int ab = 0; ab < 36; ++ab) {
    const int a = ab / 6, c = ab - 6 * a;
    double s = 0.0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s = fma(b[a * n + j], y[c * n + j], s);
    s = block_sum<VIB_THREADS>(s, red);
    if (threadIdx.x == 0) z[ab] = s;
  }
  double mx = 0.0;
  for (int j = threadIdx.x; j < n; j += blockDim.x) mx = fmax(mx, rowabs[g * n + j]);
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 36) {
    const int a = threadIdx.x / 6, c = threadIdx.x - 6 * a;
    Z[g * 40 + threadIdx.x] = 0.5 * (z[a * 6 + c] + z[c * 6 + a]);
  }
  if (threadIdx.x == 0) {
    double m = 0.0;
    for (int w = 0; w < VIB_THREADS / 32; ++w) m = fmax(m, red[w]);
    Z[g * 40 + 36] = 2.0 * m + 1.0;
  }
}

// One thread per entry:  Hp = P Hm P + c B^T B,  P = I - B^T B, expanded as
//   Hp_ij = Hm_ij - (B^T Y)_ij - (B^T Y)_ji + (B^T Z B)_ij + c (B^T B)_ij,
// every entry evaluated at (min(i, j), max(i, j)) so that Hp is exactly symmetric.
__global__ void __launch_bounds__(256) k_vib_assemble(const double* __restrict__ H, const double* __restrict__ ism,
                                                      const double* __restrict__ B, const double* __restrict__ Y,
                                                      const double* __restrict__ Z, int n, int64_t n_geo,
                                                      double* __restrict__ Hp) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nn = (int64_t)n * n;
  if (idx >= n_geo * nn) return;
  const int64_t g = idx / nn;
  const int64_t ij = idx - g * nn;
  const int i0 = (int)(ij / n), j0 = (int)(ij - (int64_t)i0 * n);
  const int i = min(i0, j0), j = max(i0, j0);
  const double* b = B + g * 6 * n;
  const double* y = Y + g * 6 * n;
  const double* z = Z + g * 40;
  double bi[6], bj[6];
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    bi[a] = b[a * n + i];
    bj[a] = b[a * n + j];
  }
  double pij = 0.0, pji = 0.0, quad = 0.0, rig = 0.0;
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    pij = fma(bi[a], y[a * n + j], pij);
    pji = fma(bj[a], y[a * n + i], pji);
    rig = fma(bi[a], bj[a], rig);
    double zb = 0.0;
#pragma unroll
    for (int c = 0; c < 6; ++c) zb = fma(z[a * 6 + c], bj[c], zb);
    quad = fma(bi[a], zb, quad);
  }
  Hp[idx] = hm_entry(H + g * nn, ism, n, i, j) - pij - pji + quad + z[36] * rig;
}

// ---------------------------------------------------------------- batched symmetric eigensolver
// Parallel cyclic Jacobi, one CTA per matrix, A in shared memory (row stride ld, odd), V in the output (global, row
// major, columns the eigenvectors).  A sweep is m - 1 rounds of the round-robin ordering of m = n + (n odd) indices; a
// round rotates m / 2 disjoint pairs: rotation angles first, then all row updates, all column updates (of A and V), then
// the 2 x 2 blocks set to their exact rotated values.  A pair is rotated when |a_pq| > eps |A|_F / n, so the entries
// left off the diagonal total at most eps |A|_F in Frobenius norm; sweeps stop after one without a rotation.
__device__ __forceinline__ void rr_pair(int r, int k, int m, int& p, int& q) {
  // circle method: index m - 1 stays, the others turn; round r pairs (r, m - 1) and ((r + k), (r - k)) mod (m - 1)
  int x, y;
  if (k == 0) {
    x = r;
    y = m - 1;
  } else {
    x = (r + k) % (m - 1);
    y = (r - k + (m - 1)) % (m - 1);
  }
  p = min(x, y);
  q = max(x, y);
}

__global__ void __launch_bounds__(SYMEIG_THREADS) k_symeig_jacobi(const double* __restrict__ Ain, int n,
                                                                  double* __restrict__ w, double* __restrict__ Vout) {
  extern __shared__ double sj_sm[];
  const int ld = n | 1;
  const int m = n + (n & 1);
  const int h = m / 2;
  double* A = sj_sm;                              // n x ld
  double* rc = A + (size_t)n * ld;                // h: cos
  double* rs = rc + h;                            // h: sin
  double* ra = rs + h;                            // h: new a_pp
  double* rb = ra + h;                            // h: new a_qq
  double* red = rb + h;                           // SYMEIG_THREADS / 32
  int* rp = reinterpret_cast<int*>(red + SYMEIG_THREADS / 32);  // h
  int* rq = rp + h;                                             // h
  int* rank = rq + h;                                           // n
  __shared__ int rotated;
  const int64_t g = blockIdx.x;
  const double* a_in = Ain + g * n * n;
  double* V = Vout + g * n * n;
  double fro = 0.0;
  for (int idx = threadIdx.x; idx < n * n; idx += blockDim.x) {
    const int i = idx / n, j = idx - i * n;
    const double x = a_in[idx];
    A[i * ld + j] = x;
    V[idx] = i == j ? 1.0 : 0.0;
    fro = fma(x, x, fro);
  }
  fro = sqrt(block_sum<SYMEIG_THREADS>(fro, red));
  const double thr = DBL_EPSILON * fro / n;
  for (int sweep = 0; sweep < SYMEIG_MAX_SWEEPS; ++sweep) {
    if (threadIdx.x == 0) rotated = 0;
    __syncthreads();
    for (int r = 0; r < m - 1; ++r) {
      for (int k = threadIdx.x; k < h; k += blockDim.x) {
        int p, q;
        rr_pair(r, k, m, p, q);
        double c = 1.0, s = 0.0;
        if (q < n) {
          const double apq = A[p * ld + q], app = A[p * ld + p], aqq = A[q * ld + q];
          if (fabs(apq) > thr) {
            const double theta = (aqq - app) / (2.0 * apq);
            const double t =
                fabs(theta) > 1e150 ? 0.5 / theta : copysign(1.0, theta) / (fabs(theta) + sqrt(fma(theta, theta, 1.0)));
            c = 1.0 / sqrt(fma(t, t, 1.0));
            s = t * c;
            // rows and columns p, q turn with this pair's rotation only, so its 2 x 2 block ends exactly diagonal
            ra[k] = app - t * apq;
            rb[k] = aqq + t * apq;
            rotated = 1;
          } else {
            q = n;  // no rotation
          }
        }
        rp[k] = p;
        rq[k] = q;
        rc[k] = c;
        rs[k] = s;
      }
      __syncthreads();
      for (int idx = threadIdx.x; idx < h * n; idx += blockDim.x) {  // rows p, q
        const int j = idx / h, k = idx - j * h;
        const int q = rq[k];
        if (q >= n) continue;
        const int p = rp[k];
        const double c = rc[k], s = rs[k];
        const double ap = A[p * ld + j], aq = A[q * ld + j];
        A[p * ld + j] = c * ap - s * aq;
        A[q * ld + j] = s * ap + c * aq;
      }
      __syncthreads();
      for (int idx = threadIdx.x; idx < h * n; idx += blockDim.x) {  // columns p, q of A and V
        const int i = idx / h, k = idx - i * h;
        const int q = rq[k];
        if (q >= n) continue;
        const int p = rp[k];
        const double c = rc[k], s = rs[k];
        const double ap = A[i * ld + p], aq = A[i * ld + q];
        A[i * ld + p] = c * ap - s * aq;
        A[i * ld + q] = s * ap + c * aq;
        const double vp = V[(int64_t)i * n + p], vq = V[(int64_t)i * n + q];
        V[(int64_t)i * n + p] = c * vp - s * vq;
        V[(int64_t)i * n + q] = s * vp + c * vq;
      }
      __syncthreads();
      for (int k = threadIdx.x; k < h; k += blockDim.x) {  // the rotated 2 x 2 blocks, exactly
        const int q = rq[k];
        if (q >= n) continue;
        const int p = rp[k];
        A[p * ld + p] = ra[k];
        A[q * ld + q] = rb[k];
        A[p * ld + q] = 0.0;
        A[q * ld + p] = 0.0;
      }
      __syncthreads();
    }
    if (rotated == 0) break;
    __syncthreads();  // rotated is reset at the next sweep's start
  }
  // ascending order, ties by index: rank_i = #{j : d_j < d_i or (d_j == d_i and j < i)}
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double di = A[i * ld + i];
    int rk = 0;
    for (int j = 0; j < n; ++j) {
      const double dj = A[j * ld + j];
      rk += (dj < di || (dj == di && j < i)) ? 1 : 0;
    }
    rank[i] = rk;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) w[g * n + rank[i]] = A[i * ld + i];
  __syncthreads();
  for (int idx = threadIdx.x; idx < n * n; idx += blockDim.x) {
    const int i = idx / n, j = idx - i * n;
    A[i * ld + j] = V[idx];
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < n * n; idx += blockDim.x) {
    const int i = idx / n, j = idx - i * n;
    V[(int64_t)i * n + rank[j]] = A[i * ld + j];
  }
}

size_t symeig_smem(int n) {
  const int ld = n | 1, h = (n + (n & 1)) / 2;
  return sizeof(double) * ((size_t)n * ld + 4 * h + SYMEIG_THREADS / 32) + sizeof(int) * (2 * h + n);
}

}  // namespace

}  // namespace sgdml

using namespace sgdml;

int sgdml_b200_symeig_max_n(void) { return SGDML_B200_SYMEIG_MAX_N; }

int sgdml_b200_vib_project(const double* H, const double* R, const double* inv_sqrt_mass, int64_t n_geo,
                           int64_t n_atoms, int periodic, double* Hp, int64_t* n_rigid, void* stream) {
  SG_TRY(require_device());
  SG_ARG(H != nullptr && R != nullptr && inv_sqrt_mass != nullptr && Hp != nullptr && n_rigid != nullptr);
  SG_ARG(n_geo >= 0 && n_atoms >= 1 && n_atoms <= 1023 && (periodic == 0 || periodic == 1));
  SG_ARG(is_device_ptr(H) && is_device_ptr(R) && is_device_ptr(inv_sqrt_mass) && is_device_ptr(Hp) &&
         is_device_ptr(n_rigid));
  SG_ARG(H != Hp);
  if (n_geo == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int n = 3 * (int)n_atoms;
  double *B = nullptr, *Y = nullptr, *rowabs = nullptr, *Z = nullptr;
  SG_CUDA(cached_malloc(&B, sizeof(double) * n_geo * 6 * n));
  SG_CUDA(cached_malloc(&Y, sizeof(double) * n_geo * 6 * n));
  SG_CUDA(cached_malloc(&rowabs, sizeof(double) * n_geo * n));
  SG_CUDA(cached_malloc(&Z, sizeof(double) * n_geo * 40));
  int rc = 0;
  {
    ProfScope ps(KID_MISC, s);
    k_vib_basis<<<(unsigned)n_geo, VIB_THREADS, 0, s>>>(R, inv_sqrt_mass, (int)n_atoms, periodic, B, n_rigid);
    k_vib_rows<<<dim3((unsigned)ceil_div(n, 8), (unsigned)n_geo), 256, 0, s>>>(H, inv_sqrt_mass, B, n, Y, rowabs);
    k_vib_small<<<(unsigned)n_geo, VIB_THREADS, 0, s>>>(B, Y, rowabs, n, Z);
    k_vib_assemble<<<(unsigned)ceil_div(n_geo * n * n, 256), 256, 0, s>>>(H, inv_sqrt_mass, B, Y, Z, n, n_geo, Hp);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) rc = fail_cuda(e, "vib_project launch", __FILE__, __LINE__);
    count_launch(KID_MISC, 4);
  }
  const cudaError_t e = cudaStreamSynchronize(s);  // the scratch goes back to the cache
  for (double* p : {B, Y, rowabs, Z}) cached_free(p);
  if (rc != 0) return rc;
  SG_CUDA(e);
  return 0;
}

int sgdml_b200_symeig_batched(const double* A, int64_t n, int64_t n_geo, double* w, double* V, void* stream) {
  SG_TRY(require_device());
  SG_ARG(A != nullptr && w != nullptr && V != nullptr);
  SG_ARG(n >= 1 && n <= SGDML_B200_SYMEIG_MAX_N && n_geo >= 0 && n_geo <= 2147483647);
  SG_ARG(is_device_ptr(A) && is_device_ptr(w) && is_device_ptr(V));
  SG_ARG(A != V);
  if (n_geo == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem = symeig_smem((int)n);
  if (smem > 48 * 1024)
    SG_CUDA(cudaFuncSetAttribute(k_symeig_jacobi, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ProfScope ps(KID_MISC, s);
  k_symeig_jacobi<<<(unsigned)n_geo, SYMEIG_THREADS, smem, s>>>(A, (int)n, w, V);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}
