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

// host-side launchers defined in desc.cu (device pointers only), reused by predict.cu
int launch_desc_from_R(const double* R, int64_t n_geo, int n_atoms, double* R_desc, double* R_d_desc,
                       cudaStream_t s, const Lattice* lat = nullptr);
// the same with the cell read by the kernel from DEVICE memory at lat_dev (a captured graph's per-call cell)
int launch_desc_from_R_lp(const double* R, int64_t n_geo, int n_atoms, double* R_desc, double* R_d_desc,
                          cudaStream_t s, const Lattice* lat_dev);
// one cell per geometry: lats_dev (n_geo) in DEVICE memory, cell g for geometry g
int launch_desc_from_R_cells(const double* R, int64_t n_geo, int n_atoms, double* R_desc, double* R_d_desc,
                             cudaStream_t s, const Lattice* lats_dev);
int launch_d_desc_dot_vec(const double* R_d_desc, const double* vecs, int64_t n_geo, int n_atoms, double* out,
                          int64_t out_stride, cudaStream_t s);
int launch_vec_dot_d_desc(const double* R_d_desc, const double* vecs, int64_t n_geo, int n_atoms,
                          int64_t vec_stride, double* out, cudaStream_t s);

}  // namespace sgdml
