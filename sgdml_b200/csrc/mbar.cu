// MBAR on the device (sgdml_b200_umbrella_mbar; Shirts & Chodera, J. Chem. Phys. 129, 124105 (2008), eq. 11): the
// self-consistent reduced free energies of umbrella windows from pooled CV samples, and the unbiased weight of every
// sample.  The contract, with its reduction order, is in md.cuh; the restraint is md.cuh's umbrella_restraint, the
// function the step graph evaluates, so u_kn here has the bits of beta times the bias energy the run wrote.
//
// One iteration is four launches: k_mbar_logsum (L_n, one thread per sample), k_mbar_partial (per-CTA (max, sum) pairs
// of -u_kn - L_n, grid (CTAs, windows)), k_mbar_combine (one CTA per window: f_k') and k_mbar_update (shift, residual,
// stop).  Iterations are queued in blocks of MBAR_BLOCK between host read-backs of the stop flag; once set, every
// kernel of the rest of the block returns at once, so the iteration count is exact.  u_kn is recomputed where it is
// needed, never stored: the K x n matrix of a large pool does not fit, and recomputing it costs a few FP64 operations.
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "md.cuh"

namespace sgdml {
namespace {

constexpr int64_t MBAR_BLOCK = 16;  // iterations between read-backs of the stop flag

struct MbarParams {
  int n_cv, K;
  int type[MD_MAX_CV];
  double beta;
  int64_t n;
  const double* S;    // (n, n_cv) samples
  const double* win;  // (K, n_cv) centres, then (K, n_cv) force constants
  const double* lnN;  // (K) ln N_k (-inf for an empty window)
};

struct MbarState {
  int64_t n_iter;
  double resid;
  int done;
};

// u_kn = beta b_k(s_n); k == K is the unbiased state, u = 0
__device__ __forceinline__ double mbar_u(const MbarParams& p, int k, int64_t n) {
  if (k == p.K) return 0.0;
  const double b =
      umbrella_restraint(p.n_cv, p.type, p.S + n * p.n_cv, p.win + k * p.n_cv, p.win + (p.K + k) * p.n_cv, nullptr);
  return __dmul_rn(p.beta, b);
}

__device__ __forceinline__ void lse_fold(double& m, double& S, double x) {
  if (x > m) {
    S = __dadd_rn(__dmul_rn(S, exp(__dsub_rn(m, x))), 1.0);
    m = x;
  } else {
    S = __dadd_rn(S, exp(__dsub_rn(x, m)));
  }
}

__device__ __forceinline__ void lse_merge(double& m, double& S, double m2, double S2) {
  if (S2 == 0.0) return;
  if (S == 0.0) {
    m = m2;
    S = S2;
  } else if (m2 > m) {
    S = __dadd_rn(__dmul_rn(S, exp(__dsub_rn(m, m2))), S2);
    m = m2;
  } else {
    S = __dadd_rn(S, __dmul_rn(S2, exp(__dsub_rn(m2, m))));
  }
}

// the fixed tree over the CTA's pairs: red[t] += red[t + w] for w = MBAR_THREADS / 2, ..., 1; thread 0 gets the result
__device__ __forceinline__ void lse_tree(double& m, double& S, double* rm, double* rs) {
  const int t = threadIdx.x;
  rm[t] = m;
  rs[t] = S;
  __syncthreads();
  for (int w = MBAR_THREADS / 2; w > 0; w >>= 1) {
    if (t < w) {
      double a = rm[t], b = rs[t];
      lse_merge(a, b, rm[t + w], rs[t + w]);
      rm[t] = a;
      rs[t] = b;
    }
    __syncthreads();
  }
  m = rm[0];
  S = rs[0];
}

// L_n = m_n + log(sum_k exp(a_kn - m_n)), a_kn = (ln N_k + f_k) - u_kn, m_n = max_k a_kn
__global__ void __launch_bounds__(MBAR_THREADS) k_mbar_logsum(const MbarParams* __restrict__ P,
                                                             const double* __restrict__ f, double* __restrict__ L,
                                                             const MbarState* gate) {
  const MbarParams& p = *P;
  if (gate != nullptr && gate->done) return;
  const int64_t n = (int64_t)blockIdx.x * MBAR_THREADS + threadIdx.x;
  if (n >= p.n) return;
  double m = -INFINITY;
  for (int k = 0; k < p.K; ++k) m = fmax(m, __dsub_rn(__dadd_rn(p.lnN[k], f[k]), mbar_u(p, k, n)));
  double S = 0.0;
  for (int k = 0; k < p.K; ++k) S = __dadd_rn(S, exp(__dsub_rn(__dsub_rn(__dadd_rn(p.lnN[k], f[k]), mbar_u(p, k, n)), m)));
  L[n] = __dadd_rn(m, log(S));
}

// the (max, sum) pair of -u_kn - L_n over the samples of CTA blockIdx.x, window k = k0 + blockIdx.y
__global__ void __launch_bounds__(MBAR_THREADS) k_mbar_partial(const MbarParams* __restrict__ P,
                                                              const double* __restrict__ L, int k0,
                                                              double2* __restrict__ part, const MbarState* gate) {
  __shared__ double rm[MBAR_THREADS], rs[MBAR_THREADS];
  const MbarParams& p = *P;
  if (gate != nullptr && gate->done) return;
  const int k = k0 + (int)blockIdx.y;
  const int64_t first = (int64_t)blockIdx.x * MBAR_CHUNK;
  const int64_t last = min(first + (int64_t)MBAR_CHUNK, p.n);
  double m = -INFINITY, S = 0.0;
  for (int64_t n = first + threadIdx.x; n < last; n += MBAR_THREADS) lse_fold(m, S, __dsub_rn(-mbar_u(p, k, n), L[n]));
  lse_tree(m, S, rm, rs);
  if (threadIdx.x == 0) part[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = make_double2(m, S);
}

// f_out[k0 + blockIdx.x] = -logsumexp over the n_part pairs of that window
__global__ void __launch_bounds__(MBAR_THREADS) k_mbar_combine(const double2* __restrict__ part, int n_part, int k0,
                                                              double* __restrict__ f_out, const MbarState* gate) {
  __shared__ double rm[MBAR_THREADS], rs[MBAR_THREADS];
  if (gate != nullptr && gate->done) return;
  const double2* q = part + (int64_t)blockIdx.x * n_part;
  double m = -INFINITY, S = 0.0;
  for (int c = threadIdx.x; c < n_part; c += MBAR_THREADS) lse_merge(m, S, q[c].x, q[c].y);
  lse_tree(m, S, rm, rs);
  if (threadIdx.x == 0) f_out[k0 + blockIdx.x] = -__dadd_rn(m, log(S));
}

// f' = f' - f'_0, resid = max_k |f'_k - f_k|, f = f', and the stop test (one thread)
__global__ void k_mbar_update(double* __restrict__ f, const double* __restrict__ fn, int K, double tol,
                              int64_t max_iter, MbarState* st) {
  if (st->done) return;
  double r = 0.0;
  const double f0 = fn[0];
  for (int k = 0; k < K; ++k) {
    const double v = __dsub_rn(fn[k], f0);
    const double d = fabs(__dsub_rn(v, f[k]));
    r = (d > r || d != d) ? d : r;
    f[k] = v;
  }
  st->resid = r;
  st->n_iter += 1;
  if (!(r >= tol) || st->n_iter >= max_iter) st->done = 1;
}

// log w_n = f_u - L_n
__global__ void k_mbar_logw(const double* __restrict__ L, const double* __restrict__ fu, int64_t n,
                            double* __restrict__ log_w) {
  const int64_t i = (int64_t)blockIdx.x * MBAR_THREADS + threadIdx.x;
  if (i < n) log_w[i] = __dsub_rn(*fu, L[i]);
}

// bad[0] = 1 when a sample is not finite
__global__ void k_mbar_check(const double* __restrict__ S, int64_t count, int* bad) {
  const int64_t i = (int64_t)blockIdx.x * MBAR_THREADS + threadIdx.x;
  if (i < count && !isfinite(S[i])) *bad = 1;
}

template <class T>
struct DevBuf {  // a cached device block, freed after the stream has finished with it
  T* p = nullptr;
  cudaStream_t s;
  explicit DevBuf(cudaStream_t st) : s(st) {}
  ~DevBuf() {
    if (p == nullptr) return;
    cudaStreamSynchronize(s);
    cached_free(p);
  }
  int alloc(size_t count) {
    SG_CUDA(cached_malloc(&p, sizeof(T) * count));
    return 0;
  }
};

int launched() {
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC);
  return 0;
}

}  // namespace
}  // namespace sgdml

using namespace sgdml;

extern "C" int sgdml_b200_umbrella_mbar(int64_t n_windows, int64_t n_cv, const int* cv_type, const double* centers,
                                        const double* kappas, double beta, int64_t n_samples, const double* samples,
                                        const int64_t* n_per_window, double tol, int64_t max_iter, double* f,
                                        double* log_w, int64_t* n_iter, double* resid, void* stream) {
  SG_TRY(require_device());
  SG_ARG(cv_type != nullptr && samples != nullptr && n_per_window != nullptr);
  SG_ARG(n_windows >= 1 && n_windows <= 65535);
  SG_ARG(n_cv >= 1 && n_cv <= MD_MAX_CV);
  SG_ARG(!is_device_ptr(cv_type) && !is_device_ptr(n_per_window));
  SG_ARG(n_iter == nullptr || !is_device_ptr(n_iter));
  SG_ARG(resid == nullptr || !is_device_ptr(resid));
  SG_ARG(std::isfinite(beta) && beta > 0.0);
  SG_ARG(std::isfinite(tol) && tol >= 0.0);
  SG_ARG(max_iter >= 1);
  SG_ARG(n_samples >= 1 && n_samples <= ((int64_t)1 << 40));
  MbarParams p = {};
  p.n_cv = (int)n_cv;
  p.K = (int)n_windows;
  p.beta = beta;
  p.n = n_samples;
  for (int j = 0; j < n_cv; ++j) {
    if (cv_type[j] != CV_DISTANCE && cv_type[j] != CV_ANGLE && cv_type[j] != CV_DIHEDRAL)
      return fail_arg("cv_type must be 0 (distance), 1 (angle) or 2 (dihedral)");
    p.type[j] = cv_type[j];
  }
  SG_TRY(umbrella_windows_check(n_windows, p.n_cv, p.type, centers, kappas));
  const int K = p.K;
  std::vector<double> tab((size_t)(3 * K * n_cv + K));  // centres, force constants, ln N
  std::memcpy(tab.data(), centers, sizeof(double) * K * n_cv);
  std::memcpy(tab.data() + K * n_cv, kappas, sizeof(double) * K * n_cv);
  double* lnN = tab.data() + 2 * K * n_cv;
  int64_t total = 0;
  for (int k = 0; k < K; ++k) {
    if (n_per_window[k] < 0) return fail_arg("every n_per_window must be >= 0");
    total += n_per_window[k];
    lnN[k] = n_per_window[k] > 0 ? std::log((double)n_per_window[k]) : -INFINITY;
  }
  if (total != n_samples) return fail_arg("n_per_window must sum to n_samples");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t count = n_samples * n_cv;
  Staged S_in;
  SG_TRY(S_in.init(samples, sizeof(double) * count, true, s));
  p.S = static_cast<const double*>(S_in.dev());
  const int C = ceil_div(n_samples, MBAR_CHUNK);
  const unsigned gn = (unsigned)ceil_div(n_samples, MBAR_THREADS);
  DevBuf<double> dtab(s), fbuf(s), L(s);
  DevBuf<double2> part(s);
  DevBuf<MbarState> st(s);
  DevBuf<MbarParams> dp(s);
  DevBuf<int> bad(s);
  SG_TRY(bad.alloc(1));
  SG_CUDA(cudaMemsetAsync(bad.p, 0, sizeof(int), s));
  k_mbar_check<<<(unsigned)ceil_div(count, MBAR_THREADS), MBAR_THREADS, 0, s>>>(p.S, count, bad.p);
  SG_TRY(launched());
  int bad_h = 0;
  SG_CUDA(cudaMemcpyAsync(&bad_h, bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  SG_CUDA(cudaStreamSynchronize(s));
  if (bad_h) return fail_arg("sgdml_b200_umbrella_mbar: every sample must be finite");
  SG_TRY(dtab.alloc(tab.size()));
  SG_TRY(fbuf.alloc(2 * (size_t)K + 1));  // f, then f' (K + 1 entries: the last is the unbiased state's)
  SG_TRY(L.alloc((size_t)n_samples));
  SG_TRY(part.alloc((size_t)C * K));
  SG_TRY(st.alloc(1));
  SG_TRY(dp.alloc(1));
  SG_CUDA(cudaMemcpyAsync(dtab.p, tab.data(), sizeof(double) * tab.size(), cudaMemcpyHostToDevice, s));
  SG_CUDA(cudaMemsetAsync(fbuf.p, 0, sizeof(double) * (2 * (size_t)K + 1), s));
  SG_CUDA(cudaMemsetAsync(st.p, 0, sizeof(MbarState), s));
  p.win = dtab.p;
  p.lnN = dtab.p + 2 * K * n_cv;
  SG_CUDA(cudaMemcpyAsync(dp.p, &p, sizeof(MbarParams), cudaMemcpyHostToDevice, s));
  double *fk = fbuf.p, *fn = fbuf.p + K;
  MbarState hst = {};
  for (int64_t queued = 0; queued < max_iter;) {
    const int64_t nb = std::min(MBAR_BLOCK, max_iter - queued);
    for (int64_t i = 0; i < nb; ++i) {
      k_mbar_logsum<<<gn, MBAR_THREADS, 0, s>>>(dp.p, fk, L.p, st.p);
      SG_TRY(launched());
      k_mbar_partial<<<dim3((unsigned)C, (unsigned)K), MBAR_THREADS, 0, s>>>(dp.p, L.p, 0, part.p, st.p);
      SG_TRY(launched());
      k_mbar_combine<<<(unsigned)K, MBAR_THREADS, 0, s>>>(part.p, C, 0, fn, st.p);
      SG_TRY(launched());
      k_mbar_update<<<1, 1, 0, s>>>(fk, fn, K, tol, max_iter, st.p);
      SG_TRY(launched());
    }
    queued += nb;
    SG_CUDA(cudaMemcpyAsync(&hst, st.p, sizeof(MbarState), cudaMemcpyDeviceToHost, s));
    SG_CUDA(cudaStreamSynchronize(s));
    if (hst.done) break;
  }
  // the weights of the final f: L once more, then the unbiased state's f_u (row K of the reduction)
  k_mbar_logsum<<<gn, MBAR_THREADS, 0, s>>>(dp.p, fk, L.p, nullptr);
  SG_TRY(launched());
  k_mbar_partial<<<dim3((unsigned)C, 1), MBAR_THREADS, 0, s>>>(dp.p, L.p, K, part.p, nullptr);
  SG_TRY(launched());
  k_mbar_combine<<<1, MBAR_THREADS, 0, s>>>(part.p, C, K, fn, nullptr);
  SG_TRY(launched());
  Staged f_out, w_out;
  SG_TRY(f_out.init(f, f ? sizeof(double) * K : 0, false, s));
  SG_TRY(w_out.init(log_w, log_w ? sizeof(double) * n_samples : 0, false, s));
  if (log_w != nullptr) {
    k_mbar_logw<<<gn, MBAR_THREADS, 0, s>>>(L.p, fn + K, n_samples, static_cast<double*>(w_out.dev()));
    SG_TRY(launched());
    SG_TRY(w_out.finish(s));
  }
  if (f != nullptr) {
    SG_CUDA(cudaMemcpyAsync(f_out.dev(), fk, sizeof(double) * K, cudaMemcpyDeviceToDevice, s));
    SG_TRY(f_out.finish(s));
  }
  SG_CUDA(cudaStreamSynchronize(s));
  if (n_iter != nullptr) *n_iter = hst.n_iter;
  if (resid != nullptr) *resid = hst.resid;
  return 0;
}
