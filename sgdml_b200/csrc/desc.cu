// Representation layer (SURVEY.md section 8, rows a-D1..a-D4, a-P0): inverse-distance
// descriptor, compressed Jacobian, Jacobian-vector products and the integer
// atom-perm -> descriptor-perm map.
#include "common.cuh"
#include "desc.cuh"

namespace sgdml {

// ---------------------------------------------------------------- a-D1: from_R
// reference: utils/desc.py:80-110 (_pdist), 139-163, 166-205, 288-365
// lat.on != 0: minimum-image convention (minimum_image, desc.cuh).  Thread idx = g * dim_d + d.
__device__ __forceinline__ void desc_from_R_body(int64_t idx, int64_t g, const double* __restrict__ R, int n_atoms,
                                                 int dim_d, double* __restrict__ R_desc,
                                                 double* __restrict__ R_d_desc, const Lattice& lat) {
  int d = (int)(idx - g * dim_d);
  int a, b;
  pair_from_d(d, a, b);
  const double* r = R + g * 3 * n_atoms;
  double dx = r[3 * a + 0] - r[3 * b + 0];
  double dy = r[3 * a + 1] - r[3 * b + 1];
  double dz = r[3 * a + 2] - r[3 * b + 2];
  minimum_image(lat, dx, dy, dz);
  double dist = sqrt(dot3(dx, dy, dz, dx, dy, dz));
  double inv = 1.0 / dist;
  double inv3 = 1.0 / (dist * dist * dist);
  if (R_desc) R_desc[idx] = inv;
  if (R_d_desc) {
    R_d_desc[idx * 3 + 0] = dx * inv3;
    R_d_desc[idx * 3 + 1] = dy * inv3;
    R_d_desc[idx * 3 + 2] = dz * inv3;
  }
}
// lats == nullptr: every geometry in the cell `lat`, a kernel argument, so the bulk path reads no cell from memory.
// Otherwise geometry g takes lats[g]; with small D one block spans several geometries, so every thread reads its own
// geometry's cell (152 B, shared through L1 by the D threads of that geometry).
__global__ void k_desc_from_R(const double* __restrict__ R, int64_t n_geo, int n_atoms, int dim_d,
                              double* __restrict__ R_desc, double* __restrict__ R_d_desc, const Lattice lat,
                              const Lattice* __restrict__ lats) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_geo * dim_d) return;
  const int64_t g = idx / dim_d;
  if (lats != nullptr)
    desc_from_R_body(idx, g, R, n_atoms, dim_d, R_desc, R_d_desc, lats[g]);
  else
    desc_from_R_body(idx, g, R, n_atoms, dim_d, R_desc, R_d_desc, lat);
}

// ---------------------------------------------------------------- a-D3: (J v)_d = g_d . (v_b - v_a)
// reference: utils/desc.py:368-385
__global__ void k_d_desc_dot_vec(const double* __restrict__ R_d_desc, const double* __restrict__ vecs,
                                 int64_t n_geo, int n_atoms, int dim_d, double* __restrict__ out,
                                 int64_t out_stride) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = n_geo * dim_d;
  if (idx >= total) return;
  int64_t g = idx / dim_d;
  int d = (int)(idx - g * dim_d);
  int a, b;
  pair_from_d(d, a, b);
  const double* v = vecs + g * 3 * n_atoms;
  out[g * out_stride + d] = d_desc_dot(R_d_desc + idx * 3, a, b, [v](int i) { return v[i]; });
}

// ---------------------------------------------------------------- a-D4: J^T w
// reference: utils/desc.py:388-408.  One thread per (geometry, atom, component).
__global__ void k_vec_dot_d_desc(const double* __restrict__ R_d_desc, const double* __restrict__ vecs,
                                 int64_t n_geo, int n_atoms, int dim_d, int64_t vec_stride,
                                 double* __restrict__ out) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = n_geo * 3 * n_atoms;
  if (idx >= total) return;
  int64_t g = idx / (3 * n_atoms);
  int rem = (int)(idx - g * 3 * n_atoms);
  int k = rem / 3, c = rem - 3 * k;
  const double* gd = R_d_desc + g * dim_d * 3;
  const double* w = vecs + g * vec_stride;
  double s = 0.0;
  for (int o = 0; o < n_atoms; ++o) {
    if (o == k) continue;
    if (o > k) {  // pair (a=o, b=k): atom b gets +g w
      int d = pair_index(o, k);
      s += gd[d * 3 + c] * w[d];
    } else {  // pair (a=k, b=o): atom a gets -g w
      int d = pair_index(k, o);
      s -= gd[d * 3 + c] * w[d];
    }
  }
  out[idx] = s;
}

int launch_desc_from_R(const double* R, int64_t n_geo, int n_atoms, double* R_desc, double* R_d_desc,
                       cudaStream_t s, const Lattice& lat, const Lattice* lats_dev) {
  if (n_geo == 0) return 0;
  const int D = n_atoms * (n_atoms - 1) / 2;
  int64_t total = n_geo * D;
  ProfScope ps(KID_DESC, s);
  k_desc_from_R<<<ceil_div(total, 256), 256, 0, s>>>(R, n_geo, n_atoms, D, R_desc, R_d_desc, lat, lats_dev);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_DESC);
  return 0;
}

int launch_d_desc_dot_vec(const double* R_d_desc, const double* vecs, int64_t n_geo, int n_atoms, double* out,
                          int64_t out_stride, cudaStream_t s) {
  if (n_geo == 0) return 0;
  const int D = n_atoms * (n_atoms - 1) / 2;
  int64_t total = n_geo * D;
  k_d_desc_dot_vec<<<ceil_div(total, 256), 256, 0, s>>>(R_d_desc, vecs, n_geo, n_atoms, D, out, out_stride);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_DESC);
  return 0;
}

int launch_vec_dot_d_desc(const double* R_d_desc, const double* vecs, int64_t n_geo, int n_atoms,
                          int64_t vec_stride, double* out, cudaStream_t s) {
  if (n_geo == 0) return 0;
  const int D = n_atoms * (n_atoms - 1) / 2;
  int64_t total = n_geo * 3 * n_atoms;
  k_vec_dot_d_desc<<<ceil_div(total, 256), 256, 0, s>>>(R_d_desc, vecs, n_geo, n_atoms, D, vec_stride, out);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_DESC);
  return 0;
}

// lattice / lattice_inv: 9 HOST doubles each (3 x 3 row-major, lattice vectors as columns), or both NULL
int lattice_from_host(const double* lattice, const double* lattice_inv, Lattice* l) {
  l->on = 0;
  if (lattice == nullptr && lattice_inv == nullptr) return 0;
  SG_ARG(lattice != nullptr && lattice_inv != nullptr);
  SG_ARG(!is_device_ptr(lattice) && !is_device_ptr(lattice_inv));
  for (int i = 0; i < 9; ++i) {
    l->vec[i] = lattice[i];
    l->inv[i] = lattice_inv[i];
  }
  l->on = 1;
  return 0;
}
}  // namespace sgdml

using namespace sgdml;

extern "C" {

// a-P0: utils/desc.py:509-539 + train.py:897-904.  Host integer code, bit-exact.
int sgdml_b200_tril_perms_lin(const int64_t* perms, int64_t n_perms, int64_t n_atoms, int64_t* out) {
  SG_ARG(perms != nullptr && out != nullptr);
  SG_ARG(n_perms >= 1 && n_atoms >= 2);
  const int64_t D = n_atoms * (n_atoms - 1) / 2;
  for (int64_t p = 0; p < n_perms; ++p) {
    const int64_t* pm = perms + p * n_atoms;
    // validate: must be a permutation of 0..N-1
    std::vector<char> seen((size_t)n_atoms, 0);
    for (int64_t a = 0; a < n_atoms; ++a) {
      if (pm[a] < 0 || pm[a] >= n_atoms || seen[(size_t)pm[a]]) return fail_arg("perms rows must be permutations of 0..N-1");
      seen[(size_t)pm[a]] = 1;
    }
    int64_t d = 0;
    for (int64_t a = 1; a < n_atoms; ++a) {
      for (int64_t b = 0; b < a; ++b, ++d) {
        int64_t pa = pm[a], pb = pm[b];
        int64_t hi = pa > pb ? pa : pb, lo = pa > pb ? pb : pa;
        int64_t e = hi * (hi - 1) / 2 + lo;
        out[d * n_perms + p] = e + p * D;
      }
    }
  }
  return 0;
}

int sgdml_b200_desc_from_R_pbc(const double* R, int64_t n_geo, int64_t n_atoms, const double* lattice,
                               const double* lattice_inv, double* R_desc, double* R_d_desc, void* stream) {
  SG_TRY(require_device());
  SG_ARG(R != nullptr && n_geo >= 0 && n_atoms >= 2);
  if (n_geo == 0) return 0;
  Lattice l;
  SG_TRY(lattice_from_host(lattice, lattice_inv, &l));
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t D = n_atoms * (n_atoms - 1) / 2;
  Staged sR, sX, sG;
  SG_TRY(sR.init(R, sizeof(double) * n_geo * 3 * n_atoms, true, s));
  SG_TRY(sX.init(R_desc, sizeof(double) * n_geo * D, false, s));
  SG_TRY(sG.init(R_d_desc, sizeof(double) * n_geo * D * 3, false, s));
  SG_TRY(launch_desc_from_R((const double*)sR.dev(), n_geo, (int)n_atoms, (double*)sX.dev(), (double*)sG.dev(), s, l,
                            nullptr));
  SG_TRY(sX.finish(s));
  SG_TRY(sG.finish(s));
  if (sR.staged() || sX.staged() || sG.staged()) SG_CUDA(cudaStreamSynchronize(s));
  return 0;
}

int sgdml_b200_desc_from_R(const double* R, int64_t n_geo, int64_t n_atoms, double* R_desc, double* R_d_desc,
                           void* stream) {
  SG_TRY(require_device());
  SG_ARG(R != nullptr && n_geo >= 0 && n_atoms >= 2);
  if (n_geo == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t D = n_atoms * (n_atoms - 1) / 2;
  Staged sR, sX, sG;
  SG_TRY(sR.init(R, sizeof(double) * n_geo * 3 * n_atoms, true, s));
  SG_TRY(sX.init(R_desc, sizeof(double) * n_geo * D, false, s));
  SG_TRY(sG.init(R_d_desc, sizeof(double) * n_geo * D * 3, false, s));
  SG_TRY(launch_desc_from_R((const double*)sR.dev(), n_geo, (int)n_atoms, (double*)sX.dev(), (double*)sG.dev(), s,
                            Lattice{}, nullptr));
  SG_TRY(sX.finish(s));
  SG_TRY(sG.finish(s));
  if (sR.staged() || sX.staged() || sG.staged()) SG_CUDA(cudaStreamSynchronize(s));
  return 0;
}

int sgdml_b200_d_desc_dot_vec(const double* R_d_desc, const double* vecs, int64_t n_geo, int64_t n_atoms,
                              double* out, void* stream) {
  SG_TRY(require_device());
  SG_ARG(R_d_desc != nullptr && vecs != nullptr && out != nullptr && n_geo >= 0 && n_atoms >= 2);
  if (n_geo == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t D = n_atoms * (n_atoms - 1) / 2;
  Staged sG, sV, sO;
  SG_TRY(sG.init(R_d_desc, sizeof(double) * n_geo * D * 3, true, s));
  SG_TRY(sV.init(vecs, sizeof(double) * n_geo * 3 * n_atoms, true, s));
  SG_TRY(sO.init(out, sizeof(double) * n_geo * D, false, s));
  SG_TRY(launch_d_desc_dot_vec((const double*)sG.dev(), (const double*)sV.dev(), n_geo, (int)n_atoms,
                               (double*)sO.dev(), D, s));
  SG_TRY(sO.finish(s));
  if (sG.staged() || sV.staged() || sO.staged()) SG_CUDA(cudaStreamSynchronize(s));
  return 0;
}

int sgdml_b200_vec_dot_d_desc(const double* R_d_desc, const double* vecs, int64_t n_geo, int64_t n_atoms,
                              double* out, void* stream) {
  SG_TRY(require_device());
  SG_ARG(R_d_desc != nullptr && vecs != nullptr && out != nullptr && n_geo >= 0 && n_atoms >= 2);
  if (n_geo == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t D = n_atoms * (n_atoms - 1) / 2;
  Staged sG, sV, sO;
  SG_TRY(sG.init(R_d_desc, sizeof(double) * n_geo * D * 3, true, s));
  SG_TRY(sV.init(vecs, sizeof(double) * n_geo * D, true, s));
  SG_TRY(sO.init(out, sizeof(double) * n_geo * 3 * n_atoms, false, s));
  SG_TRY(launch_vec_dot_d_desc((const double*)sG.dev(), (const double*)sV.dev(), n_geo, (int)n_atoms, D,
                               (double*)sO.dev(), s));
  SG_TRY(sO.finish(s));
  if (sG.staged() || sV.staged() || sO.staged()) SG_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
