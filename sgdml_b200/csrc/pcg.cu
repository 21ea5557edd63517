// Device-resident preconditioned conjugate gradient (SURVEY.md section 8 rows a-S2 / 8b `sgdml_b200_pcg`) --
// reference sgdml/solvers/iterative.py:740-752 (scipy.sparse.linalg.cg on the operators of
// iterative.py:120-142 and 183-206).
//
//   solve (-K + lam I) x = y,   A v = lam v - K v,   K v = predict_train(alphas = v) (raw sums),
//   P v = (X (X^T v) - v) / lam  with X = B^T the Nystroem factor (iterative.py:136-138)
//
// Every vector (x, r, p, z, A p) lives in HBM for the whole solve; the CG scalars are produced by
// two-stage deterministic reductions on the device and consumed from device memory by the next kernel, so an
// iteration is a pure launch sequence: set_alphas -> fused predictor on the training points -> 2 vector
// kernels -> 2 GEMV kernels of the preconditioner -> 2 vector kernels.  The host reads back a residual
// history every `check_every` iterations (that is where the reference's callbacks, checkpoints and restart
// logic hook in, iterative.py:640-735) and nothing else.
//
// Several GPUs (SURVEY 8e): every rank keeps the full replicated vectors and computes the scalars
// redundantly (bit-identical: fixed reduction order); the K.v rows and the rows of the Nystroem factor are
// sharded by training point, and the two exchanges per iteration -- one all-gather of n doubles after K.v, one
// all-reduce of m doubles plus one all-gather of n doubles in P.v -- go through a caller-supplied exchange
// function on DEVICE buffers in stream order (the Python host plugs torch.distributed / NCCL in there; the
// library itself links no communication library).
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "solve.cuh"

namespace sgdml {

constexpr int PCG_NT = 256;
constexpr int PCG_ELEMS_PER_CTA = 2048;
constexpr int PCG_MAX_CTAS = 1024;

// scalar slots (device)
enum { SC_RZ = 0, SC_PAP = 1, SC_ALPHA = 2, SC_BETA = 3, SC_RESID = 4, SC_DONE = 5, SC_ITERS = 6, SC_TOL = 7, SC_COUNT = 8 };

// block-wide sum in a fixed order (warp shuffles, then warp 0 over the 8 warp sums)
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (warp == 0) {
    s = (lane < PCG_NT / 32) ? red[lane] : 0.0;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  return s;  // valid in thread 0
}

// every CTA owns a fixed contiguous range: the partial sums, and hence the scalars, are bit-reproducible
__device__ __forceinline__ void cta_range(int64_t n, int64_t& i0, int64_t& i1) {
  const int64_t per = (n + gridDim.x - 1) / gridDim.x;
  i0 = (int64_t)blockIdx.x * per;
  i1 = min(n, i0 + per);
}

// r = y - lam x + kv  (= y - A x);  partial[b] = sum r^2
__global__ void __launch_bounds__(PCG_NT) k_pcg_init_r(int64_t n, double lam, const double* __restrict__ y,
                                                      const double* __restrict__ x, const double* __restrict__ kv,
                                                      double* __restrict__ r, double* __restrict__ partial) {
  __shared__ double red[PCG_NT / 32];
  int64_t i0, i1;
  cta_range(n, i0, i1);
  double s = 0.0;
  for (int64_t i = i0 + threadIdx.x; i < i1; i += PCG_NT) {
    const double v = (kv != nullptr) ? (y[i] - lam * x[i]) + kv[i] : y[i];
    r[i] = v;
    s = fma(v, v, s);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// ap = lam p - kv (in place over kv);  partial[b] = sum p . ap
__global__ void __launch_bounds__(PCG_NT) k_pcg_ap(int64_t n, double lam, const double* __restrict__ p,
                                                  double* __restrict__ kv_ap, double* __restrict__ partial) {
  __shared__ double red[PCG_NT / 32];
  int64_t i0, i1;
  cta_range(n, i0, i1);
  double s = 0.0;
  for (int64_t i = i0 + threadIdx.x; i < i1; i += PCG_NT) {
    const double pv = p[i];
    const double a = lam * pv - kv_ap[i];
    kv_ap[i] = a;
    s = fma(pv, a, s);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// partial[b] = sum a . b
__global__ void __launch_bounds__(PCG_NT) k_pcg_dot(int64_t n, const double* __restrict__ a, const double* __restrict__ b,
                                                   double* __restrict__ partial) {
  __shared__ double red[PCG_NT / 32];
  int64_t i0, i1;
  cta_range(n, i0, i1);
  double s = 0.0;
  for (int64_t i = i0 + threadIdx.x; i < i1; i += PCG_NT) s = fma(a[i], b[i], s);
  s = block_sum(s, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// x += alpha p; r -= alpha ap; partial[b] = sum r^2   (alpha from device memory; 0 once converged)
__global__ void __launch_bounds__(PCG_NT) k_pcg_update(int64_t n, const double* __restrict__ sc,
                                                      const double* __restrict__ p, const double* __restrict__ ap,
                                                      double* __restrict__ x, double* __restrict__ r,
                                                      double* __restrict__ partial) {
  __shared__ double red[PCG_NT / 32];
  int64_t i0, i1;
  cta_range(n, i0, i1);
  const double alpha = sc[SC_ALPHA];
  double s = 0.0;
  for (int64_t i = i0 + threadIdx.x; i < i1; i += PCG_NT) {
    x[i] = fma(alpha, p[i], x[i]);
    const double v = fma(-alpha, ap[i], r[i]);
    r[i] = v;
    s = fma(v, v, s);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// v = -v  (the energy rows of K.v with energy constraints: the operator returns [F; -E], iterative.py:196-198)
__global__ void __launch_bounds__(PCG_NT) k_pcg_neg(int64_t n, double* __restrict__ v) {
  const int64_t i = (int64_t)blockIdx.x * PCG_NT + threadIdx.x;
  if (i < n) v[i] = -v[i];
}

// p = z + beta p
__global__ void __launch_bounds__(PCG_NT) k_pcg_p(int64_t n, const double* __restrict__ sc, const double* __restrict__ z,
                                                 double* __restrict__ p) {
  const double beta = sc[SC_BETA];
  const int64_t i = (int64_t)blockIdx.x * PCG_NT + threadIdx.x;
  if (i < n) p[i] = fma(beta, p[i], z[i]);
}

// one CTA: sums the per-CTA partials in a fixed order and updates the scalar block.
//   mode 0: resid = sqrt(sum), rz untouched                 (initial residual)
//   mode 1: pAp = sum; alpha = done ? 0 : rz / pAp
//   mode 2: resid = sqrt(sum); hist[slot] = resid; if not done: ++iters, done = resid <= tol
//   mode 3: rz_new = sum; beta = first ? 0 : rz_new / rz; rz = rz_new
__global__ void __launch_bounds__(PCG_NT) k_pcg_scalar(const double* __restrict__ partial, int n_part, int mode,
                                                      int slot_or_first, double* __restrict__ sc,
                                                      double* __restrict__ hist) {
  __shared__ double red[PCG_NT / 32];
  double s = 0.0;
  for (int i = threadIdx.x; i < n_part; i += PCG_NT) s += partial[i];
  s = block_sum(s, red);
  if (threadIdx.x != 0) return;
  if (mode == 0) {
    sc[SC_RESID] = sqrt(s);
  } else if (mode == 1) {
    sc[SC_PAP] = s;
    sc[SC_ALPHA] = (sc[SC_DONE] != 0.0) ? 0.0 : sc[SC_RZ] / s;
  } else if (mode == 2) {
    const double resid = sqrt(s);
    sc[SC_RESID] = resid;
    hist[slot_or_first] = resid;
    if (sc[SC_DONE] == 0.0) {
      sc[SC_ITERS] += 1.0;
      // NaN (breakdown) also stops the iteration: the host sees it in the history
      if (!(resid > sc[SC_TOL])) sc[SC_DONE] = 1.0;
    }
  } else {
    const double rz_old = sc[SC_RZ];
    sc[SC_BETA] = slot_or_first ? 0.0 : s / rz_old;
    sc[SC_RZ] = s;
  }
}

}  // namespace sgdml

using namespace sgdml;

namespace {

struct PcgWs {
  double *x, *r, *p, *z, *kv, *t, *part_xt, *partial, *sc, *hist, *vloc, *zloc;
};

int pcg_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(PCG_MAX_CTAS, (n + PCG_ELEMS_PER_CTA - 1) / PCG_ELEMS_PER_CTA)); }

int64_t pcg_ws_doubles(int64_t n, int64_t n_rows_loc, int64_t m_ind, int64_t check_every) {
  if (n < 1 || n_rows_loc < 0 || m_ind < 0 || check_every < 1) return -1;
  return 5 * n + m_ind + m_ind * xtv_chunks(std::max<int64_t>(n_rows_loc, 1)) + PCG_MAX_CTAS + SC_COUNT + check_every + 8;
}

// The energy-constrained solve stages this rank's two segments of a vector (force rows, energy rows) contiguously,
// in the row order of X_loc: two more n_rows_loc-vectors after the common layout.
int64_t pcg_ecstr_ws_doubles(int64_t n, int64_t n_rows_loc, int64_t m_ind, int64_t check_every) {
  const int64_t base = pcg_ws_doubles(n, n_rows_loc, m_ind, check_every);
  return base < 0 ? -1 : base + 2 * n_rows_loc;
}

// sgdml_b200_pcg (ecstr = false) and sgdml_b200_pcg_ecstr (ecstr = true): one implementation; with ecstr = false
// every launch and every exchange is the force-only solve's.
int pcg_impl(bool ecstr, sgdml_b200_model* model, int64_t m_begin, int64_t m_end, const double* X_loc, int64_t m_ind,
             int64_t ldx, double lam, const double* y, double* x, int x_is_zero, double tol_abs, int64_t max_iters,
             int64_t check_every, double* workspace, int64_t workspace_doubles, sgdml_b200_exchange_fn exchange,
             void* exchange_ctx, sgdml_b200_pcg_progress_fn progress, void* progress_ctx, int64_t* iters_out,
             double* resid_out, void* stream) {
  SG_TRY(require_device());
  SG_ARG(model != nullptr && y != nullptr && x != nullptr && workspace != nullptr && iters_out != nullptr &&
         resid_out != nullptr);
  SG_ARG(lam > 0.0 && tol_abs >= 0.0 && max_iters >= 0 && check_every >= 1);
  int64_t n_atoms = 0, n_train = 0;
  SG_TRY(sgdml_b200_model_dims(model, &n_atoms, &n_train, nullptr));
  const int64_t dimi = 3 * n_atoms, n_f = dimi * n_train, n = n_f + (ecstr ? n_train : 0);
  SG_ARG(m_begin >= 0 && m_begin <= m_end && m_end <= n_train);
  SG_ARG(exchange != nullptr || (m_begin == 0 && m_end == n_train));  // one rank evaluates everything
  const int64_t n_pts_loc = m_end - m_begin, n_frows_loc = n_pts_loc * dimi;
  const int64_t n_rows_loc = n_frows_loc + (ecstr ? n_pts_loc : 0);
  SG_ARG(m_ind >= 0 && (m_ind == 0 || (X_loc != nullptr && ldx >= m_ind && is_device_ptr(X_loc))));
  SG_ARG(is_device_ptr(workspace) &&
         workspace_doubles >= (ecstr ? pcg_ecstr_ws_doubles : pcg_ws_doubles)(n, n_rows_loc, m_ind, check_every));
  cudaStream_t s = (cudaStream_t)stream;

  PcgWs w;
  {
    double* q = workspace;
    w.x = q, q += n;
    w.r = q, q += n;
    w.p = q, q += n;
    w.z = q, q += n;
    w.kv = q, q += n;
    w.t = q, q += m_ind;
    w.part_xt = q, q += m_ind * xtv_chunks(std::max<int64_t>(n_rows_loc, 1));
    w.partial = q, q += PCG_MAX_CTAS;
    w.sc = q, q += SC_COUNT;
    w.hist = q, q += check_every;
    w.vloc = ecstr ? q : nullptr, q += ecstr ? n_rows_loc : 0;
    w.zloc = ecstr ? q : nullptr;
  }
  const int G = pcg_grid(n);
  const int64_t off_loc = m_begin * dimi;

  // K v for the replicated vector v (device) into w.kv: rows of this rank, then the all-gather.  With energy
  // constraints v = [v_F; v_E] and K v = [F; -E] of the predictor with alphas_F = v_F, alphas_E = v_E.
  auto k_vec = [&](const double* v) -> int {
    SG_TRY(sgdml_b200_model_set_alphas(model, v, stream));
    if (ecstr) SG_TRY(sgdml_b200_model_set_alphas_E(model, v + n_f, stream));
    if (m_end > m_begin) {
      double* e_loc = ecstr ? w.kv + n_f + m_begin : nullptr;
      SG_TRY(sgdml_b200_predict_train(model, m_begin, m_end, 0, e_loc, w.kv + off_loc, stream));
      if (ecstr) {
        k_pcg_neg<<<ceil_div(n_pts_loc, PCG_NT), PCG_NT, 0, s>>>(n_pts_loc, e_loc);
        SG_CUDA(cudaGetLastError());
        count_launch(KID_MISC);
      }
    }
    if (exchange != nullptr && exchange(exchange_ctx, 1, w.kv, n_f) != 0) return fail_arg("exchange (all-gather of K.v) failed");
    if (ecstr && exchange != nullptr && exchange(exchange_ctx, 2, w.kv + n_f, n_train) != 0)
      return fail_arg("exchange (all-gather of the energy rows of K.v) failed");
    return 0;
  };
  // this rank's rows of a replicated vector in the row order of X_loc (force rows, then energy rows) and back
  auto gather_loc = [&](const double* v, double* loc) -> int {
    SG_CUDA(cudaMemcpyAsync(loc, v + off_loc, sizeof(double) * n_frows_loc, cudaMemcpyDeviceToDevice, s));
    SG_CUDA(cudaMemcpyAsync(loc + n_frows_loc, v + n_f + m_begin, sizeof(double) * n_pts_loc, cudaMemcpyDeviceToDevice, s));
    return 0;
  };
  auto scatter_loc = [&](const double* loc, double* v) -> int {
    SG_CUDA(cudaMemcpyAsync(v + off_loc, loc, sizeof(double) * n_frows_loc, cudaMemcpyDeviceToDevice, s));
    SG_CUDA(cudaMemcpyAsync(v + n_f + m_begin, loc + n_frows_loc, sizeof(double) * n_pts_loc, cudaMemcpyDeviceToDevice, s));
    return 0;
  };
  // z = P r
  auto p_vec = [&]() -> int {
    if (m_ind == 0) {  // no preconditioner: z = r
      SG_CUDA(cudaMemcpyAsync(w.z, w.r, sizeof(double) * n, cudaMemcpyDeviceToDevice, s));
      return 0;
    }
    const double* r_loc = ecstr ? w.vloc : w.r + off_loc;
    double* z_loc = ecstr ? w.zloc : w.z + off_loc;
    if (ecstr && n_rows_loc > 0) SG_TRY(gather_loc(w.r, w.vloc));
    if (n_rows_loc > 0) {
      SG_TRY(xt_v_device(X_loc, n_rows_loc, m_ind, ldx, r_loc, w.t, w.part_xt, s));
    } else {
      SG_CUDA(cudaMemsetAsync(w.t, 0, sizeof(double) * m_ind, s));
    }
    if (exchange != nullptr && exchange(exchange_ctx, 0, w.t, m_ind) != 0) return fail_arg("exchange (all-reduce of X^T v) failed");
    if (n_rows_loc > 0) SG_TRY(x_t_minus_v_device(X_loc, n_rows_loc, m_ind, ldx, lam, w.t, r_loc, z_loc, s));
    if (ecstr && n_rows_loc > 0) SG_TRY(scatter_loc(w.zloc, w.z));
    if (exchange != nullptr && exchange(exchange_ctx, 1, w.z, n_f) != 0) return fail_arg("exchange (all-gather of P.v) failed");
    if (ecstr && exchange != nullptr && exchange(exchange_ctx, 2, w.z + n_f, n_train) != 0)
      return fail_arg("exchange (all-gather of the energy rows of P.v) failed");
    return 0;
  };
  auto scalar = [&](int mode, int arg) -> int {
    k_pcg_scalar<<<1, PCG_NT, 0, s>>>(w.partial, G, mode, arg, w.sc, w.hist);
    SG_CUDA(cudaGetLastError());
    return 0;
  };

  // ---- set-up: x0, r0 = y - A x0, z0 = P r0, p0 = z0, rz
  Staged sY;
  SG_TRY(sY.init(y, sizeof(double) * n, true, s));
  const double* yd = (const double*)sY.dev();
  if (x_is_zero) {
    SG_CUDA(cudaMemsetAsync(w.x, 0, sizeof(double) * n, s));
  } else {
    SG_CUDA(cudaMemcpyAsync(w.x, x, sizeof(double) * n, cudaMemcpyDefault, s));
    SG_TRY(k_vec(w.x));
  }
  {
    double h_sc[SC_COUNT] = {0};
    h_sc[SC_TOL] = tol_abs;
    SG_CUDA(cudaMemcpyAsync(w.sc, h_sc, sizeof(h_sc), cudaMemcpyHostToDevice, s));
    SG_CUDA(cudaStreamSynchronize(s));  // h_sc is a stack buffer
  }
  k_pcg_init_r<<<G, PCG_NT, 0, s>>>(n, lam, yd, w.x, x_is_zero ? nullptr : w.kv, w.r, w.partial);
  SG_CUDA(cudaGetLastError());
  SG_TRY(scalar(0, 0));
  SG_TRY(p_vec());
  k_pcg_dot<<<G, PCG_NT, 0, s>>>(n, w.r, w.z, w.partial);
  SG_CUDA(cudaGetLastError());
  SG_TRY(scalar(3, 1));
  k_pcg_p<<<ceil_div(n, PCG_NT), PCG_NT, 0, s>>>(n, w.sc, w.z, w.p);  // beta = 0: p = z
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC, 5);

  double h_sc[SC_COUNT];
  std::vector<double> h_hist((size_t)check_every);
  SG_CUDA(cudaMemcpyAsync(h_sc, w.sc, sizeof(h_sc), cudaMemcpyDeviceToHost, s));
  SG_CUDA(cudaStreamSynchronize(s));
  int64_t iters = 0;
  double resid = h_sc[SC_RESID];
  bool stop = !(resid > tol_abs);

  // ---- iterations, in chunks of at most check_every between two looks at the residual
  int64_t chunk = std::min<int64_t>(check_every, 4);  // short first chunks: a good preconditioner converges in a handful
  while (!stop && iters < max_iters) {
    const int64_t todo = std::min<int64_t>(chunk, max_iters - iters);
    for (int64_t j = 0; j < todo; ++j) {
      SG_TRY(k_vec(w.p));
      k_pcg_ap<<<G, PCG_NT, 0, s>>>(n, lam, w.p, w.kv, w.partial);
      SG_CUDA(cudaGetLastError());
      SG_TRY(scalar(1, 0));
      k_pcg_update<<<G, PCG_NT, 0, s>>>(n, w.sc, w.p, w.kv, w.x, w.r, w.partial);
      SG_CUDA(cudaGetLastError());
      SG_TRY(scalar(2, (int)j));
      SG_TRY(p_vec());
      k_pcg_dot<<<G, PCG_NT, 0, s>>>(n, w.r, w.z, w.partial);
      SG_CUDA(cudaGetLastError());
      SG_TRY(scalar(3, 0));
      k_pcg_p<<<ceil_div(n, PCG_NT), PCG_NT, 0, s>>>(n, w.sc, w.z, w.p);
      SG_CUDA(cudaGetLastError());
      count_launch(KID_MISC, 7);
    }
    SG_CUDA(cudaMemcpyAsync(h_sc, w.sc, sizeof(h_sc), cudaMemcpyDeviceToHost, s));
    SG_CUDA(cudaMemcpyAsync(h_hist.data(), w.hist, sizeof(double) * (size_t)todo, cudaMemcpyDeviceToHost, s));
    SG_CUDA(cudaStreamSynchronize(s));
    const int64_t iters_new = (int64_t)h_sc[SC_ITERS] - iters;  // < todo if the tolerance was reached inside the chunk
    const double prev = resid;
    iters += iters_new;
    resid = h_sc[SC_RESID];
    if (h_sc[SC_DONE] != 0.0 || !(resid == resid)) stop = true;
    if (progress != nullptr && iters_new > 0 && progress(progress_ctx, iters, h_hist.data(), iters_new) != 0) stop = true;
    // next chunk: as many iterations as the current convergence rate says are still needed (so that the
    // solve stops close to the first iteration below the tolerance, like the reference's loop), capped
    if (!stop) {
      int64_t next = check_every;
      if (resid < prev && resid > tol_abs && iters_new > 0) {
        const double rate = std::log(prev / resid) / (double)iters_new;  // > 0
        const double need = std::log(resid / std::max(tol_abs, 1e-300)) / rate;
        next = (int64_t)std::max(1.0, std::min((double)check_every, std::ceil(need)));
      }
      chunk = next;
    }
  }
  SG_CUDA(cudaMemcpyAsync(x, w.x, sizeof(double) * n, cudaMemcpyDefault, s));
  SG_CUDA(cudaStreamSynchronize(s));
  *iters_out = iters;
  *resid_out = resid;
  return 0;
}

}  // namespace

extern "C" {

int64_t sgdml_b200_pcg_workspace_doubles(int64_t n, int64_t n_rows_loc, int64_t m_ind, int64_t check_every) {
  return pcg_ws_doubles(n, n_rows_loc, m_ind, check_every);
}

int64_t sgdml_b200_pcg_ecstr_workspace_doubles(int64_t n, int64_t n_rows_loc, int64_t m_ind, int64_t check_every) {
  return pcg_ecstr_ws_doubles(n, n_rows_loc, m_ind, check_every);
}

int sgdml_b200_pcg(sgdml_b200_model* model, int64_t m_begin, int64_t m_end, const double* X_loc, int64_t m_ind,
                   int64_t ldx, double lam, const double* y, double* x, int x_is_zero, double tol_abs,
                   int64_t max_iters, int64_t check_every, double* workspace, int64_t workspace_doubles,
                   sgdml_b200_exchange_fn exchange, void* exchange_ctx, sgdml_b200_pcg_progress_fn progress,
                   void* progress_ctx, int64_t* iters_out, double* resid_out, void* stream) {
  return pcg_impl(false, model, m_begin, m_end, X_loc, m_ind, ldx, lam, y, x, x_is_zero, tol_abs, max_iters,
                  check_every, workspace, workspace_doubles, exchange, exchange_ctx, progress, progress_ctx, iters_out,
                  resid_out, stream);
}

int sgdml_b200_pcg_ecstr(sgdml_b200_model* model, int64_t m_begin, int64_t m_end, const double* X_loc, int64_t m_ind,
                         int64_t ldx, double lam, const double* y, double* x, int x_is_zero, double tol_abs,
                         int64_t max_iters, int64_t check_every, double* workspace, int64_t workspace_doubles,
                         sgdml_b200_exchange_fn exchange, void* exchange_ctx, sgdml_b200_pcg_progress_fn progress,
                         void* progress_ctx, int64_t* iters_out, double* resid_out, void* stream) {
  return pcg_impl(true, model, m_begin, m_end, X_loc, m_ind, ldx, lam, y, x, x_is_zero, tol_abs, max_iters,
                  check_every, workspace, workspace_doubles, exchange, exchange_ctx, progress, progress_ctx, iters_out,
                  resid_out, stream);
}

}  // extern "C"
