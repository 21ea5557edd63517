// Internal interface of the dense-solve kernels (solve.cu), shared with nystroem.cu.
#pragma once
#include "common.cuh"

namespace sgdml {

constexpr int NB = 128;  // Cholesky panel width / TRSM block

struct GemmArgs {
  int64_t m, n, k;
  const double* A;
  int64_t lda;
  const double* B;
  int64_t ldb;
  double* C;
  int64_t ldc;
  double alpha, beta;
  int mode;  // 0: C = alpha A B^T + beta C ; 1: C += A B^T (accumulators start from C)
  int tri;   // 1: C square, only tiles touching the lower triangle are computed
  const int* abort_flag;  // optional: skip all work when *abort_flag != 0
};

// device pointers only
int launch_gemm(const GemmArgs& a, cudaStream_t s);
int potrf_device(double* A, int64_t n, int64_t lda, int* info_host, cudaStream_t s, bool analytic_solver = false);
int potrs_device(const double* L, int64_t n, int64_t lda, double* B, int64_t nrhs, int64_t ldb, cudaStream_t s);
int trsm_right_lt_device(const double* L, int64_t m, int64_t ldl, double* X, int64_t n_rows, int64_t ldx,
                         cudaStream_t s);

// csrc/nystroem.cu: the two halves of the preconditioner application on device vectors (stream-ordered, no
// synchronisation); part must hold m * xtv_chunks(n_rows) doubles
int64_t xtv_chunks(int64_t n_rows);
int xt_v_device(const double* X, int64_t n_rows, int64_t m, int64_t ldx, const double* v_dev, double* t_dev,
                double* part, cudaStream_t s);
int x_t_minus_v_device(const double* X, int64_t n_rows, int64_t m, int64_t ldx, double lam, const double* t_dev,
                       const double* v_dev, double* out_dev, cudaStream_t s);

// csrc/ozaki.cu: an operand cut into int8 slices (unit-major pre-swizzled layout) and the GEMM on such operands
struct OzOperand {
  int8_t* units = nullptr;   // [k-block][slice][row tile][8192]
  int* exps = nullptr;       // row exponents
  int64_t rows_pad = 0, kp = 0;
};
size_t ozaki_units_bytes(int64_t rows, int64_t k, int n_slices);
size_t ozaki_exps_bytes(int64_t rows);
int ozaki_split(const double* X, int64_t rows, int64_t k, int64_t ldx, int n_slices, int8_t* units, int* exps,
                OzOperand* out, cudaStream_t s);
// C (m x n, ldc) = (overwrite ? 0 : C) + alpha * A B^T for pre-split operands; stream-ordered, no allocation
int ozaki_gemm(const OzOperand& a, const OzOperand& b, int64_t m, int64_t n, double alpha, int overwrite, double* C,
               int64_t ldc, int n_slices, cudaStream_t s);

// csrc/ozaki.cu: C += alpha A B^T (overwrite: C = alpha A B^T) through n_slices int8 slices per operand on the int8
// tensor cores (wgmma)
int ozaki_gemm_nt_device(int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda, const double* B,
                         int64_t ldb, double* C, int64_t ldc, int n_slices, int tri, int overwrite, cudaStream_t s);
int ozaki_syrk_workspace_bytes(int64_t max_rows, int64_t max_k, int n_slices, size_t* plane_bytes, size_t* exp_bytes);
int ozaki_syrk_device(int64_t n, int64_t k, double alpha, const double* X, int64_t ldx, double* C, int64_t ldc,
                      int n_slices, int8_t* planes, int* exps, cudaStream_t s);

}  // namespace sgdml
