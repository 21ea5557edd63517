// Pair indexing shared by the kernels: d <-> (a, b), a > b, in np.tril_indices(N,-1)
// order, i.e. d = a(a-1)/2 + b  (reference utils/desc.py:109-110).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sgdml {

__host__ __device__ __forceinline__ int pair_index(int a, int b) {  // requires a > b
  return a * (a - 1) / 2 + b;
}

__host__ __device__ __forceinline__ void pair_from_d(int d, int& a, int& b) {
  // a = largest integer with a(a-1)/2 <= d
  int t = (int)((1.0 + sqrt(8.0 * (double)d + 1.0)) * 0.5);
  while (t * (t - 1) / 2 > d) --t;
  while ((t + 1) * t / 2 <= d) ++t;
  a = t;
  b = d - t * (t - 1) / 2;
}

// periodic cell for the minimum-image convention (utils/desc.py:44-77): 3 x 3 row-major, lattice vectors as columns
struct Lattice {
  int on;
  double vec[9];
  double inv[9];
};
int lattice_from_host(const double* lattice, const double* lattice_inv, Lattice* l);

// a x + b y + c z as fma(c, z, fma(a, x, b y)), with the roundings spelled out: which product the compiler fuses
// otherwise depends on the code around the expression, and the descriptor kernels must round alike
__device__ __forceinline__ double dot3(double a, double b, double c, double x, double y, double z) {
  return __fma_rn(c, z, __fma_rn(a, x, __dmul_rn(b, y)));
}

// minimum-image convention (utils/desc.py:44-77): d -= lat @ rint(lat_inv @ d), lattice vectors as the COLUMNS of
// lat; np.around and rint both round half to even.  Every descriptor kernel wraps through here, so all of them pick
// the same images, also at exact rounding ties.
__device__ __forceinline__ void minimum_image(const Lattice& lat, double& dx, double& dy, double& dz) {
  if (!lat.on) return;
  const double c0 = rint(dot3(lat.inv[0], lat.inv[1], lat.inv[2], dx, dy, dz));
  const double c1 = rint(dot3(lat.inv[3], lat.inv[4], lat.inv[5], dx, dy, dz));
  const double c2 = rint(dot3(lat.inv[6], lat.inv[7], lat.inv[8], dx, dy, dz));
  dx -= dot3(lat.vec[0], lat.vec[1], lat.vec[2], c0, c1, c2);
  dy -= dot3(lat.vec[3], lat.vec[4], lat.vec[5], c0, c1, c2);
  dz -= dot3(lat.vec[6], lat.vec[7], lat.vec[8], c0, c1, c2);
}

// (J v)_d = g_d . (v_b - v_a) for pair d = (a, b), v read through v(i): k_d_desc_dot_vec's arithmetic, also the tangent
// rows of sgdml_b200_predict_hvp (v a row of V) and sgdml_b200_predict_hessian (v = e_i, where every product is exact)
template <class VecAt>
__device__ __forceinline__ double d_desc_dot(const double* gd, int a, int b, VecAt v) {
  double s = gd[0] * (v(3 * b + 0) - v(3 * a + 0));
  s += gd[1] * (v(3 * b + 1) - v(3 * a + 1));
  s += gd[2] * (v(3 * b + 2) - v(3 * a + 2));
  return s;
}

// host-side launchers defined in desc.cu (device pointers only), reused by predict.cu
// lats_dev == nullptr: every geometry in the cell `lat` (passed by value); otherwise geometry g in lats_dev[g], n_geo
// cells in DEVICE memory
int launch_desc_from_R(const double* R, int64_t n_geo, int n_atoms, double* R_desc, double* R_d_desc,
                       cudaStream_t s, const Lattice& lat, const Lattice* lats_dev);
int launch_d_desc_dot_vec(const double* R_d_desc, const double* vecs, int64_t n_geo, int n_atoms, double* out,
                          int64_t out_stride, cudaStream_t s);
int launch_vec_dot_d_desc(const double* R_d_desc, const double* vecs, int64_t n_geo, int n_atoms,
                          int64_t vec_stride, double* out, cudaStream_t s);

}  // namespace sgdml
