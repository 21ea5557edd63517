// Path (a), dense solve (SURVEY.md section 8 row a-S1): FP64 Cholesky factorisation and
// triangular solves replacing scipy.linalg.cho_factor / cho_solve (LAPACK dpotrf/dpotrs) in
// sgdml/solvers/analytic.py:94-99 and iterative.py:447-449.
//
// Design.  K stays in HBM from assembly to the solve (the reference round-trips every
// block-column through the host, torchtools.py:233).  Blocked right-looking Cholesky on the
// lower triangle of the row-major matrix, panel width NB = 128:
//   1. k_potf2_tile   one CTA factorises the 128 x 128 diagonal block in shared memory;
//   2. k_trsm_strip   64-row strips of the panel solve X L11^T = P by true substitution
//                     (no explicit inverse: diagonal blocks of sGDML kernels have condition
//                     numbers ~1e11, lam = 1e-10) and also emit -X into a workspace;
//   3. k_gemm_nt      trailing update C += (-X) X^T on the FP64 tensor pipe (mma.sync
//                     m8n8k4.f64 -> SASS DMMA; wgmma has no f64 type), lower tiles only,
//                     4-stage cp.async pipeline, fragment-major shared-memory tiles.
// FP64 throughout: TF32/BF16 factorisations cannot deliver 1e-6 forces at cond ~4e11.
#include <cuda.h>  // CUtensorMap types only: cuTensorMapEncodeTiled is resolved at run time (no libcuda link)

#include <algorithm>
#include <cmath>
#include <cstdlib>

#include "common.cuh"
#include "solve.cuh"

namespace sgdml {


// ====================================================================== GEMM  C (+)= A B^T
template <int BM_, int BN_, int WM_, int WN_, int BK_, int STAGES_>
struct GCfg {
  static constexpr int BM = BM_, BN = BN_, WM = WM_, WN = WN_;
  static constexpr int BK = BK_, STAGES = STAGES_, NT = 256;
  static constexpr int KP = BK / 2;                 // 16-byte pairs per tile row
  static constexpr int QA = BM * KP / NT, QB = BN * KP / NT;  // cp.async ops per thread per stage
  static constexpr int KSTEPS = BK / 4;
  static constexpr int TR = BM / (8 * WM), TC = BN / (8 * WN);
  static constexpr int A_DBL = BM * BK, B_DBL = BN * BK;
  static constexpr size_t SMEM_BYTES = (size_t)STAGES * (A_DBL + B_DBL) * 8;
  static_assert(WM * WN == 8, "8 warps");
  static_assert(BM % (8 * WM) == 0 && BN % (8 * WN) == 0, "warp tiling");
  static_assert((BM * KP) % NT == 0 && (BN * KP) % NT == 0, "loader mapping");
  static_assert(QA <= KSTEPS && QB <= KSTEPS, "one A and one B op per k-step at most");
  static_assert(BM % BN == 0, "triangular enumeration assumes BM = r BN");
};

// shared-memory tile layout: [k/4][row][4] so that one DMMA fragment (8 rows x 4 k) is 256
// contiguous bytes -> conflict-free LDS.64
template <class G>
__global__ void __launch_bounds__(256) k_gemm_nt(const GemmArgs p) {
  extern __shared__ __align__(128) double gsm[];
  if (p.abort_flag != nullptr && *p.abort_flag != 0) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int lr = lane >> 2, lc = lane & 3;

  // ---- tile coordinates
  int64_t ti, tj;
  if (p.tri) {
    // L2-friendly rasterisation of the lower triangle: super-tiles of GS x GS row tiles are
    // enumerated in triangular order, tiles inside a super-tile row-major, so that the ~132
    // co-resident CTAs share a small set of A and B operand panels.
    constexpr int r = G::BM / G::BN;
    constexpr int GS = 8;
    constexpr int PER = GS * GS * r;
    const int64_t sb = blockIdx.x / PER;
    const int local = (int)(blockIdx.x - sb * PER);
    int64_t t = (int64_t)((sqrt(8.0 * (double)sb + 1.0) - 1.0) * 0.5);
    while ((t + 1) * (t + 2) / 2 <= sb) ++t;
    while (t * (t + 1) / 2 > sb) --t;
    const int64_t sj = sb - t * (t + 1) / 2;
    ti = t * GS + local / (GS * r);
    tj = sj * GS * r + local % (GS * r);
    if (tj * G::BN >= (ti + 1) * G::BM) return;  // strictly above the diagonal
  } else {
    const int64_t ntn = (p.n + G::BN - 1) / G::BN;
    ti = blockIdx.x / ntn;
    tj = blockIdx.x - ti * ntn;
  }
  const int64_t m0 = ti * G::BM, n0 = tj * G::BN;
  if (m0 >= p.m || n0 >= p.n) return;

  const int wm = warp / G::WN, wn = warp % G::WN;
  const int row0 = wm * G::TR * 8, col0 = wn * G::TC * 8;

  const int KT = (int)((p.k + G::BK - 1) / G::BK);
  // one 16-byte cp.async of the A (or B) tile of k-tile `kt`: op index q of this thread
  auto load_a = [&](int kt, int q) {
    double* As = gsm + (size_t)(kt % G::STAGES) * (G::A_DBL + G::B_DBL);
    const int64_t k0 = (int64_t)kt * G::BK;
    const int op = tid + q * G::NT;
    const int row = op / G::KP, kp = op % G::KP;
    const bool ok = (m0 + row < p.m) && (k0 + 2 * kp < p.k);
    const double* src = ok ? p.A + (m0 + row) * p.lda + k0 + 2 * kp : p.A;
    cp_async16_pred(As + ((kp >> 1) * G::BM + row) * 4 + (kp & 1) * 2, src, ok);
  };
  auto load_b = [&](int kt, int q) {
    double* Bs = gsm + (size_t)(kt % G::STAGES) * (G::A_DBL + G::B_DBL) + G::A_DBL;
    const int64_t k0 = (int64_t)kt * G::BK;
    const int op = tid + q * G::NT;
    const int row = op / G::KP, kp = op % G::KP;
    const bool ok = (n0 + row < p.n) && (k0 + 2 * kp < p.k);
    const double* src = ok ? p.B + (n0 + row) * p.ldb + k0 + 2 * kp : p.B;
    cp_async16_pred(Bs + ((kp >> 1) * G::BN + row) * 4 + (kp & 1) * 2, src, ok);
  };

  // pipeline prologue first, so that the C-tile loads below overlap with it
#pragma unroll
  for (int st = 0; st < G::STAGES - 1; ++st) {
    if (st < KT) {
#pragma unroll
      for (int q = 0; q < G::QA; ++q) load_a(st, q);
#pragma unroll
      for (int q = 0; q < G::QB; ++q) load_b(st, q);
    }
    cp_async_commit();
  }

  double acc[G::TR][G::TC][2];
  if (p.mode == 1) {
#pragma unroll
    for (int i = 0; i < G::TR; ++i) {
      const int64_t r = m0 + row0 + i * 8 + lr;
#pragma unroll
      for (int j = 0; j < G::TC; ++j) {
        const int64_t c = n0 + col0 + j * 8 + 2 * lc;
        double2 v = make_double2(0.0, 0.0);
        if (r < p.m && c + 1 < p.n)
          v = *reinterpret_cast<const double2*>(p.C + r * p.ldc + c);
        else if (r < p.m && c < p.n)
          v.x = p.C[r * p.ldc + c];
        acc[i][j][0] = v.x;
        acc[i][j][1] = v.y;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < G::TR; ++i)
#pragma unroll
      for (int j = 0; j < G::TC; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  }

  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<G::STAGES - 2>();
    __syncthreads();
    const bool more = (kt + G::STAGES - 1 < KT);
    const double* As = gsm + (size_t)(kt % G::STAGES) * (G::A_DBL + G::B_DBL);
    const double* Bs = As + G::A_DBL;
#pragma unroll
    for (int ks = 0; ks < G::KSTEPS; ++ks) {
      // the next stage's loads are spread over the k-steps: a burst of LDGSTS right after the
      // barrier blocks the fragment LDS behind it in the LSU queue and starves the DMMA pipe
      if (more) {
        if (ks < G::QA) load_a(kt + G::STAGES - 1, ks);
        if (ks < G::QB) load_b(kt + G::STAGES - 1, ks);
      }
      double fa[G::TR], fb[G::TC];
#pragma unroll
      for (int i = 0; i < G::TR; ++i) fa[i] = As[(ks * G::BM + row0 + i * 8 + lr) * 4 + lc];
#pragma unroll
      for (int j = 0; j < G::TC; ++j) fb[j] = Bs[(ks * G::BN + col0 + j * 8 + lr) * 4 + lc];
#pragma unroll
      for (int i = 0; i < G::TR; ++i)
#pragma unroll
        for (int j = 0; j < G::TC; ++j) dmma884(acc[i][j][0], acc[i][j][1], fa[i], fb[j]);
    }
    cp_async_commit();
  }
  cp_async_wait<0>();

  // ---- epilogue (mode 0 reads the old C values of a whole fragment row first, so that the
  //      loads are independent instead of one exposed round trip per element)
#pragma unroll
  for (int i = 0; i < G::TR; ++i) {
    const int64_t r = m0 + row0 + i * 8 + lr;
    if (r >= p.m) continue;
    double old0[G::TC], old1[G::TC];
    if (p.mode == 0 && p.beta != 0.0) {
#pragma unroll
      for (int j = 0; j < G::TC; ++j) {
        const int64_t c = n0 + col0 + j * 8 + 2 * lc;
        const double* src = p.C + r * p.ldc + c;
        old0[j] = (c < p.n) ? src[0] : 0.0;
        old1[j] = (c + 1 < p.n) ? src[1] : 0.0;
      }
    }
#pragma unroll
    for (int j = 0; j < G::TC; ++j) {
      const int64_t c = n0 + col0 + j * 8 + 2 * lc;
      if (c >= p.n) continue;
      double* dst = p.C + r * p.ldc + c;
      double v0 = acc[i][j][0], v1 = acc[i][j][1];
      if (p.mode == 0) {
        v0 *= p.alpha;
        v1 *= p.alpha;
        if (p.beta != 0.0) {
          v0 += p.beta * old0[j];
          v1 += p.beta * old1[j];
        }
      }
      if (c + 1 < p.n)
        *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
      else
        dst[0] = v0;
    }
  }
}

// slow reference path for unaligned / odd shapes (also the on-GPU cross-check in tests)
__global__ void k_gemm_nt_naive(const GemmArgs p) {
  if (p.abort_flag != nullptr && *p.abort_flag != 0) return;
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= p.n) return;
  for (int64_t r = blockIdx.y; r < p.m; r += gridDim.y) {
    if (p.tri && c > r) continue;
    double s = 0.0;
    for (int64_t kk = 0; kk < p.k; ++kk) s = fma(p.A[r * p.lda + kk], p.B[c * p.ldb + kk], s);
    double* dst = p.C + r * p.ldc + c;
    if (p.mode == 1)
      *dst += s;
    else
      *dst = p.alpha * s + (p.beta != 0.0 ? p.beta * *dst : 0.0);
  }
}


// ====================================================================== TMA variant of the GEMM
// Same tiles and DMMA inner loop as k_gemm_nt, but the operand pipeline is Blackwell/Hopper style:
// one elected thread issues cp.async.bulk.tensor (2-D tensor maps, 128-byte swizzle, SASS UTMALDG)
// into a 3-stage ring, completion is signalled on mbarriers (full: transaction bytes; empty: one
// arrival per consumer warp) -- no per-thread address arithmetic, no LDGSTS, and no CTA-wide barrier
// in the main loop.  Each stage holds two 128-row x 16-double boxes per operand (a box row is exactly
// the 128-byte swizzle span); a fragment element (row, k) lives at
//   box + row*128 + ((chunk ^ (row & 7)) << 4) + (k & 1)*8,   chunk = (k & 15) >> 1.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

constexpr int TG_BM = 128, TG_BN = 128, TG_BK = 32, TG_STAGES = 3;
constexpr int TG_BOX_BYTES = 128 * 128;                     // 128 rows x 16 doubles
constexpr int TG_STAGE_BYTES = 4 * TG_BOX_BYTES;            // A: 2 boxes, B: 2 boxes
constexpr size_t TG_SMEM_BYTES = (size_t)TG_STAGES * TG_STAGE_BYTES + 64;

__global__ void __launch_bounds__(256) k_gemm_nt_tma(const __grid_constant__ CUtensorMap tmA,
                                                     const __grid_constant__ CUtensorMap tmB, const GemmArgs p) {
  extern __shared__ __align__(1024) unsigned char tsm2[];
  if (p.abort_flag != nullptr && *p.abort_flag != 0) return;
  uint64_t* full = reinterpret_cast<uint64_t*>(tsm2 + (size_t)TG_STAGES * TG_STAGE_BYTES);
  uint64_t* empty = full + TG_STAGES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int lr = lane >> 2, lc = lane & 3;
  constexpr int WM = 2, WN = 4, TR = TG_BM / (8 * WM), TC = TG_BN / (8 * WN);

  int64_t ti, tj;
  if (p.tri) {
    constexpr int GS = 8;
    constexpr int PER = GS * GS;
    const int64_t sb = blockIdx.x / PER;
    const int local = (int)(blockIdx.x - sb * PER);
    int64_t t = (int64_t)((sqrt(8.0 * (double)sb + 1.0) - 1.0) * 0.5);
    while ((t + 1) * (t + 2) / 2 <= sb) ++t;
    while (t * (t + 1) / 2 > sb) --t;
    const int64_t sj = sb - t * (t + 1) / 2;
    ti = t * GS + local / GS;
    tj = sj * GS + local % GS;
    if (tj * TG_BN >= (ti + 1) * TG_BM) return;
  } else {
    const int64_t ntn = (p.n + TG_BN - 1) / TG_BN;
    ti = blockIdx.x / ntn;
    tj = blockIdx.x - ti * ntn;
  }
  const int64_t m0 = ti * TG_BM, n0 = tj * TG_BN;
  if (m0 >= p.m || n0 >= p.n) return;

  if (tid == 0) {
#pragma unroll
    for (int st = 0; st < TG_STAGES; ++st) {
      mbar_init(&full[st], 1);
      mbar_init(&empty[st], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int KT = (int)((p.k + TG_BK - 1) / TG_BK);
  auto issue = [&](int kt) {
    const int st = kt % TG_STAGES;
    unsigned char* base = tsm2 + (size_t)st * TG_STAGE_BYTES;
    const int k0 = kt * TG_BK;
    mbar_arrive_expect_tx(&full[st], (uint32_t)TG_STAGE_BYTES);
    tma_load_2d(base, &tmA, k0, (int)m0, &full[st]);
    tma_load_2d(base + TG_BOX_BYTES, &tmA, k0 + 16, (int)m0, &full[st]);
    tma_load_2d(base + 2 * TG_BOX_BYTES, &tmB, k0, (int)n0, &full[st]);
    tma_load_2d(base + 3 * TG_BOX_BYTES, &tmB, k0 + 16, (int)n0, &full[st]);
  };
  if (tid == 0) {
    issue(0);
    if (KT > 1) issue(1);
  }

  const int wm = warp / WN, wn = warp % WN;
  const int row0 = wm * TR * 8, col0 = wn * TC * 8;
  double acc[TR][TC][2];
  if (p.mode == 1) {
#pragma unroll
    for (int i = 0; i < TR; ++i) {
      const int64_t r = m0 + row0 + i * 8 + lr;
#pragma unroll
      for (int j = 0; j < TC; ++j) {
        const int64_t c = n0 + col0 + j * 8 + 2 * lc;
        double2 v = make_double2(0.0, 0.0);
        if (r < p.m && c + 1 < p.n)
          v = *reinterpret_cast<const double2*>(p.C + r * p.ldc + c);
        else if (r < p.m && c < p.n)
          v.x = p.C[r * p.ldc + c];
        acc[i][j][0] = v.x;
        acc[i][j][1] = v.y;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < TR; ++i)
#pragma unroll
      for (int j = 0; j < TC; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  }

  // per-lane constants of the swizzled fragment addresses
  const int a_row_off = (row0 + lr) * 128 + ((lc & 1) << 3);
  const int b_row_off = (col0 + lr) * 128 + ((lc & 1) << 3);
  const int half = lc >> 1;

  for (int kt = 0; kt < KT; ++kt) {
    if (tid == 0 && kt + 2 < KT) {
      // stage (kt+2)%3 was last read for tile kt-1: wait until all 8 consumer warps released it
      if (kt >= 1) mbar_wait(&empty[(kt + 2) % TG_STAGES], (uint32_t)(((kt - 1) / TG_STAGES) & 1));
      issue(kt + 2);
    }
    const int st = kt % TG_STAGES;
    mbar_wait(&full[st], (uint32_t)((kt / TG_STAGES) & 1));
    const unsigned char* As = tsm2 + (size_t)st * TG_STAGE_BYTES;
    const unsigned char* Bs = As + 2 * TG_BOX_BYTES;
#pragma unroll
    for (int ks = 0; ks < TG_BK / 4; ++ks) {
      const int box = ks >> 2;
      const int sw = (((2 * (ks & 3) + half) ^ lr) << 4);
      double fa[TR], fb[TC];
#pragma unroll
      for (int i = 0; i < TR; ++i)
        fa[i] = *reinterpret_cast<const double*>(As + box * TG_BOX_BYTES + a_row_off + i * 8 * 128 + sw);
#pragma unroll
      for (int j = 0; j < TC; ++j)
        fb[j] = *reinterpret_cast<const double*>(Bs + box * TG_BOX_BYTES + b_row_off + j * 8 * 128 + sw);
#pragma unroll
      for (int i = 0; i < TR; ++i)
#pragma unroll
        for (int j = 0; j < TC; ++j) dmma884(acc[i][j][0], acc[i][j][1], fa[i], fb[j]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
  }

#pragma unroll
  for (int i = 0; i < TR; ++i) {
    const int64_t r = m0 + row0 + i * 8 + lr;
    if (r >= p.m) continue;
    double old0[TC], old1[TC];
    if (p.mode == 0 && p.beta != 0.0) {
#pragma unroll
      for (int j = 0; j < TC; ++j) {
        const int64_t c = n0 + col0 + j * 8 + 2 * lc;
        const double* src = p.C + r * p.ldc + c;
        old0[j] = (c < p.n) ? src[0] : 0.0;
        old1[j] = (c + 1 < p.n) ? src[1] : 0.0;
      }
    }
#pragma unroll
    for (int j = 0; j < TC; ++j) {
      const int64_t c = n0 + col0 + j * 8 + 2 * lc;
      if (c >= p.n) continue;
      double* dst = p.C + r * p.ldc + c;
      double v0 = acc[i][j][0], v1 = acc[i][j][1];
      if (p.mode == 0) {
        v0 *= p.alpha;
        v1 *= p.alpha;
        if (p.beta != 0.0) {
          v0 += p.beta * old0[j];
          v1 += p.beta * old1[j];
        }
      }
      if (c + 1 < p.n)
        *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
      else
        dst[0] = v0;
    }
  }
}

typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled tmap_encoder() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiled>(ptr);
  }
  return fn;
}

// row-major (rows x cols) FP64 matrix with row stride ld -> 2-D map with 16 x 128 boxes, 128 B swizzle
static int make_operand_map(CUtensorMap* tm, const double* base, int64_t rows, int64_t cols, int64_t ld) {
  PFN_tmapEncodeTiled enc = tmap_encoder();
  if (enc == nullptr) {
    set_last_error("cuTensorMapEncodeTiled is not available from this driver");
    return SGDML_B200_ERR_UNSUPPORTED;
  }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 8};
  cuuint32_t box[2] = {16, 128};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<double*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[128];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    set_last_error(buf);
    return SGDML_B200_ERR_ARG;
  }
  return 0;
}

static int launch_gemm_tma(const GemmArgs& a, cudaStream_t s) {
  static bool configured[64] = {false};
  int dev = 0;
  SG_CUDA(cudaGetDevice(&dev));
  if (dev >= 0 && dev < 64 && !configured[dev]) {
    SG_CUDA(cudaFuncSetAttribute(k_gemm_nt_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TG_SMEM_BYTES));
    configured[dev] = true;
  }
  CUtensorMap tmA, tmB;
  SG_TRY(make_operand_map(&tmA, a.A, a.m, a.k, a.lda));
  SG_TRY(make_operand_map(&tmB, a.B, a.n, a.k, a.ldb));
  const int64_t ntm = (a.m + TG_BM - 1) / TG_BM, ntn = (a.n + TG_BN - 1) / TG_BN;
  int64_t blocks;
  if (a.tri) {
    const int64_t sr = (ntm + 7) / 8;
    blocks = sr * (sr + 1) / 2 * 64;
  } else {
    blocks = ntm * ntn;
  }
  if (blocks == 0) return 0;
  ProfScope ps(KID_GEMM, s);
  k_gemm_nt_tma<<<(unsigned)blocks, 256, TG_SMEM_BYTES, s>>>(tmA, tmB, a);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_GEMM);
  return 0;
}

using GBig = GCfg<128, 128, 2, 4, 32, 3>;   // 196 KB smem, 1 CTA/SM

static int g_gemm_variant = 3;  // 0: 128x128 cp.async, 2: scalar, 3: 128x128 TMA (default)

template <class G>
static int launch_gemm_t(const GemmArgs& a, cudaStream_t s) {
  static bool configured[64] = {false};
  int dev = 0;
  SG_CUDA(cudaGetDevice(&dev));
  if (dev >= 0 && dev < 64 && !configured[dev]) {
    SG_CUDA(cudaFuncSetAttribute(k_gemm_nt<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G::SMEM_BYTES));
    configured[dev] = true;
  }
  int64_t blocks;
  const int64_t ntm = (a.m + G::BM - 1) / G::BM, ntn = (a.n + G::BN - 1) / G::BN;
  if (a.tri) {
    const int64_t sr = (ntm + 7) / 8;
    blocks = sr * (sr + 1) / 2 * 64 * (G::BM / G::BN);
  } else
    blocks = ntm * ntn;
  if (blocks == 0) return 0;
  ProfScope ps(KID_GEMM, s);
  k_gemm_nt<G><<<(unsigned)blocks, G::NT, G::SMEM_BYTES, s>>>(a);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_GEMM);
  return 0;
}

static bool gemm_fast_ok(const GemmArgs& a) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return (a.lda % 2 == 0) && (a.ldb % 2 == 0) && (a.ldc % 2 == 0) && (a.k % 2 == 0) && al16(a.A) && al16(a.B) &&
         al16(a.C);
}

int launch_gemm(const GemmArgs& a, cudaStream_t s) {
  if (a.m <= 0 || a.n <= 0) return 0;
  if (g_gemm_variant == 2 || !gemm_fast_ok(a)) {
    dim3 grid((unsigned)((a.n + 127) / 128), (unsigned)std::min<int64_t>(a.m, 65535));
    ProfScope ps(KID_GEMM, s);
    k_gemm_nt_naive<<<grid, 128, 0, s>>>(a);
    SG_CUDA(cudaGetLastError());
    count_launch(KID_GEMM);
    return 0;
  }
  if (g_gemm_variant == 3 && tmap_encoder() != nullptr) return launch_gemm_tma(a, s);  // else: cp.async tiles
  return launch_gemm_t<GBig>(a, s);
}

// ====================================================================== potf2 on one tile
// Factorises the nb x nb (nb <= 128) diagonal block at A (row stride lda) in shared memory.
// info: set to (k0 + j + 1) if the pivot j is not positive (LAPACK dpotrf convention).
// Register-resident right-looking factorisation: thread (ty, tx) of a 32 x 32 grid owns the
// 4 x 4 elements (ty + 32a, tx + 32b); per column only the pivot column travels through shared
// memory (double buffered -> one barrier per column).
__global__ void __launch_bounds__(1024) k_potf2_tile(double* __restrict__ A, int64_t lda, int nb, int64_t k0,
                                                     int* __restrict__ info) {
  __shared__ double colbuf[2][NB];
  __shared__ int bad;
  if (*info != 0) return;
  const int tid = threadIdx.x;
  const int tx = tid & 31, ty = tid >> 5;
  double a[4][4];
#pragma unroll
  for (int ai = 0; ai < 4; ++ai)
#pragma unroll
    for (int bi = 0; bi < 4; ++bi) {
      const int i = ty + 32 * ai, l = tx + 32 * bi;
      a[ai][bi] = (i < nb && l <= i) ? A[(int64_t)i * lda + l] : 0.0;
    }
  if (tid == 0) bad = 0;
  __syncthreads();
  bool failed = false;
#pragma unroll
  for (int bj = 0; bj < 4; ++bj) {
    if (failed) break;
    for (int jj = 0; jj < 32; ++jj) {
      const int j = bj * 32 + jj;
      if (j >= nb) break;
      double* cb = colbuf[j & 1];
      if (tx == jj) {  // owners of column j publish it (raw values)
#pragma unroll
        for (int ai = 0; ai < 4; ++ai) {
          const int i = ty + 32 * ai;
          if (i >= j && i < nb) cb[i] = a[ai][bj];
        }
      }
      __syncthreads();
      const double ajj = cb[j];
      if (!(ajj > 0.0)) {  // not positive definite (also catches NaN); uniform across the CTA
        if (tid == 0) bad = j + 1;
        failed = true;
        break;
      }
      // one rsqrt instead of sqrt + division (two ~400-cycle dependent sequences per column)
      const double dinv = rsqrt(ajj);
      const double d = ajj * dinv;
      double ci[4], cl[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = ty + 32 * q, l = tx + 32 * q;
        ci[q] = (i > j && i < nb) ? cb[i] * dinv : 0.0;
        cl[q] = (l > j && l < nb) ? cb[l] * dinv : 0.0;
      }
#pragma unroll
      for (int ai = 0; ai < 4; ++ai)
#pragma unroll
        for (int bi = 0; bi < 4; ++bi) {
          const int i = ty + 32 * ai, l = tx + 32 * bi;
          if (l > j && l <= i) a[ai][bi] = fma(-ci[ai], cl[bi], a[ai][bi]);
        }
      if (tx == jj) {  // finalise column j in the owners' registers
#pragma unroll
        for (int ai = 0; ai < 4; ++ai) {
          const int i = ty + 32 * ai;
          if (i == j)
            a[ai][bj] = d;
          else if (i > j)
            a[ai][bj] *= dinv;
        }
      }
    }
  }
  __syncthreads();
  if (bad != 0) {
    if (tid == 0) *info = (int)(k0 + bad);
    return;
  }
#pragma unroll
  for (int ai = 0; ai < 4; ++ai)
#pragma unroll
    for (int bi = 0; bi < 4; ++bi) {
      const int i = ty + 32 * ai, l = tx + 32 * bi;
      if (i < nb && l <= i) A[(int64_t)i * lda + l] = a[ai][bi];
    }
}

// ====================================================================== panel TRSM strips
// Solves X L11^T = P for a strip of RS rows of the panel P (rows x kb, kb <= NB) below the
// diagonal block L11 (kb x kb, lower), by blocked forward substitution in shared memory.
// Writes X over P and -X into W (row stride NB) for the trailing update.
constexpr int RS = 64;   // rows per strip
constexpr int SB = 32;   // substitution block
__global__ void __launch_bounds__(256) k_trsm_strip(const double* __restrict__ L11, int64_t lda, int kb,
                                                    double* __restrict__ Pbase, int64_t ldp, int64_t n_rows,
                                                    double* __restrict__ W, int64_t ldw,
                                                    const int* __restrict__ info) {
  extern __shared__ __align__(16) double tsm[];
  constexpr int LD = NB + 4;  // == 4 mod 16: conflict-free DMMA fragment loads
  double* L = tsm;            // NB x LD
  double* X = L + NB * LD;    // RS x LD
  __shared__ double rdiag[NB];  // 1 / L[c][c]: the substitution multiplies instead of dividing
  if (info != nullptr && *info != 0) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int lr = lane >> 2, lc = lane & 3;
  const int64_t r0 = (int64_t)blockIdx.x * RS;
  const int rows = (int)min((int64_t)RS, n_rows - r0);
  double* P = Pbase + r0 * ldp;

  for (int idx = tid; idx < NB * NB; idx += 256) {
    const int i = idx / NB, j = idx - i * NB;
    L[i * LD + j] = (i < kb && j <= i) ? L11[(int64_t)i * lda + j] : ((i == j) ? 1.0 : 0.0);
  }
  for (int idx = tid; idx < RS * NB; idx += 256) {
    const int i = idx / NB, j = idx - i * NB;
    X[i * LD + j] = (i < rows && j < kb) ? P[(int64_t)i * ldp + j] : 0.0;
  }
  if (tid < NB) rdiag[tid] = (tid < kb) ? 1.0 / L11[(int64_t)tid * lda + tid] : 1.0;
  __syncthreads();

  for (int jb = 0; jb < NB / SB; ++jb) {
    const int c0 = jb * SB;
    if (c0 >= kb) break;
    if (jb > 0) {
      // X[:, c0:c0+SB] -= X[:, 0:c0] * L[c0:c0+SB, 0:c0]^T ; warp w owns rows 8w..8w+7
      double acc[SB / 8][2];
#pragma unroll
      for (int j = 0; j < SB / 8; ++j) acc[j][0] = acc[j][1] = 0.0;
      const double* xa = X + (warp * 8 + lr) * LD + lc;
      const double* lb = L + (c0 + lr) * LD + lc;
      for (int ks = 0; ks < c0 / 4; ++ks) {
        const double fa = xa[ks * 4];
#pragma unroll
        for (int j = 0; j < SB / 8; ++j) dmma884(acc[j][0], acc[j][1], fa, lb[j * 8 * LD + ks * 4]);
      }
#pragma unroll
      for (int j = 0; j < SB / 8; ++j) {
        double* dst = X + (warp * 8 + lr) * LD + c0 + j * 8 + 2 * lc;
        dst[0] -= acc[j][0];
        dst[1] -= acc[j][1];
      }
    }
    __syncthreads();
    // substitution inside the SB x SB diagonal block: thread r < RS owns row r
    if (tid < RS) {
      double x[SB];
#pragma unroll
      for (int c = 0; c < SB; ++c) x[c] = X[tid * LD + c0 + c];
#pragma unroll
      for (int c = 0; c < SB; ++c) {
        const double xc = x[c] * rdiag[c0 + c];
        x[c] = xc;
#pragma unroll
        for (int l = c + 1; l < SB; ++l) x[l] = fma(-xc, L[(c0 + l) * LD + c0 + c], x[l]);
      }
#pragma unroll
      for (int c = 0; c < SB; ++c) X[tid * LD + c0 + c] = x[c];
    }
    __syncthreads();
  }

  for (int idx = tid; idx < RS * NB; idx += 256) {
    const int i = idx / NB, j = idx - i * NB;
    if (i < rows && j < kb) {
      const double v = X[i * LD + j];
      P[(int64_t)i * ldp + j] = v;
      W[(r0 + i) * ldw + j] = -v;
    }
  }
}

// ====================================================================== triangular solves
// forward:  z_blk = L_kk^-1 r_blk ; backward: x_blk = L_kk^-T r_blk ; one CTA, nb <= 128.
// B is (n, nrhs) row-major with row stride ldb; each thread owns one right-hand side.
__global__ void __launch_bounds__(128) k_trsv_diag(const double* __restrict__ A, int64_t lda, int64_t k0, int nb,
                                                   double* __restrict__ B, int64_t nrhs, int64_t ldb, int backward) {
  extern __shared__ double Ls[];  // nb x (NB+1)
  constexpr int LD = NB + 1;
  const double* Lkk = A + k0 * lda + k0;
  for (int idx = threadIdx.x; idx < nb * nb; idx += blockDim.x) {
    const int i = idx / nb, j = idx - i * nb;
    Ls[i * LD + j] = (j <= i) ? Lkk[(int64_t)i * lda + j] : 0.0;
  }
  __syncthreads();
  for (int64_t rhs = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; rhs < nrhs;
       rhs += (int64_t)gridDim.x * blockDim.x) {
    double* b = B + k0 * ldb + rhs;
    if (!backward) {
      for (int i = 0; i < nb; ++i) {
        double s = b[(int64_t)i * ldb];
        for (int j = 0; j < i; ++j) s = fma(-Ls[i * LD + j], b[(int64_t)j * ldb], s);
        b[(int64_t)i * ldb] = s / Ls[i * LD + i];
      }
    } else {
      for (int i = nb - 1; i >= 0; --i) {
        double s = b[(int64_t)i * ldb];
        for (int j = i + 1; j < nb; ++j) s = fma(-Ls[j * LD + i], b[(int64_t)j * ldb], s);
        b[(int64_t)i * ldb] = s / Ls[i * LD + i];
      }
    }
  }
}

// single right-hand side (the common case): the CTA stages the diagonal block in shared memory,
// then ONE warp runs the substitution with the solution in registers (4 entries per lane) and
// warp shuffles for the pivot broadcast -- no block-wide barrier per column.
__global__ void __launch_bounds__(256) k_trsv_diag1(const double* __restrict__ A, int64_t lda, int64_t k0, int nb,
                                                    double* __restrict__ b, int64_t ldb, int backward) {
  extern __shared__ double Ls[];  // NB x (NB+1)
  constexpr int LD = NB + 1;
  const double* Lkk = A + k0 * lda + k0;
  const int tid = threadIdx.x;
  for (int idx = tid; idx < NB * NB; idx += blockDim.x) {
    const int i = idx / NB, j = idx - i * NB;
    Ls[i * LD + j] = (i < nb && j <= i) ? Lkk[(int64_t)i * lda + j] : ((i == j) ? 1.0 : 0.0);
  }
  double* rd = Ls + NB * LD;  // NB reciprocals of the diagonal
  if (tid < NB) rd[tid] = (tid < nb) ? 1.0 / Lkk[(int64_t)tid * lda + tid] : 1.0;
  __syncthreads();
  if (tid >= 32) return;
  const int lane = tid;
  double x[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = lane + 32 * q;
    x[q] = (i < nb) ? b[(k0 + i) * ldb] : 0.0;
  }
  if (!backward) {
#pragma unroll
    for (int qj = 0; qj < 4; ++qj) {
      for (int jj = 0; jj < 32; ++jj) {
        const int j = qj * 32 + jj;
        const double xj = __shfl_sync(0xffffffffu, x[qj], jj) * rd[j];
        if (lane == jj) x[qj] = xj;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int i = lane + 32 * q;
          if (i > j) x[q] = fma(-Ls[i * LD + j], xj, x[q]);
        }
      }
    }
  } else {
#pragma unroll
    for (int qj = 3; qj >= 0; --qj) {
      for (int jj = 31; jj >= 0; --jj) {
        const int j = qj * 32 + jj;
        const double xj = __shfl_sync(0xffffffffu, x[qj], jj) * rd[j];
        if (lane == jj) x[qj] = xj;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int i = lane + 32 * q;
          if (i < j) x[q] = fma(-Ls[j * LD + i], xj, x[q]);
        }
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = lane + 32 * q;
    if (i < nb) b[(k0 + i) * ldb] = x[q];
  }
}

// forward update: B[k0+nb:, :] -= L[k0+nb:, k0:k0+nb] * B[k0:k0+nb, :]   (one warp per row)
__global__ void __launch_bounds__(256) k_trsv_update_fwd(const double* __restrict__ A, int64_t lda, int64_t k0,
                                                         int nb, int64_t n, double* __restrict__ B, int64_t nrhs,
                                                         int64_t ldb) {
  const int lane = threadIdx.x & 31;
  const int64_t row = k0 + nb + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const double* Lr = A + row * lda + k0;
  for (int64_t rhs = 0; rhs < nrhs; ++rhs) {
    double s = 0.0;
    for (int j = lane; j < nb; j += 32) s = fma(Lr[j], B[(k0 + j) * ldb + rhs], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) B[row * ldb + rhs] -= s;
  }
}

// backward update: B[0:k0, :] -= L[k0:k0+nb, 0:k0]^T * B[k0:k0+nb, :]   (one thread per column j)
__global__ void __launch_bounds__(256) k_trsv_update_bwd(const double* __restrict__ A, int64_t lda, int64_t k0,
                                                         int nb, double* __restrict__ B, int64_t nrhs, int64_t ldb) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= k0) return;
  for (int64_t rhs = 0; rhs < nrhs; ++rhs) {
    double s = 0.0;
    for (int r = 0; r < nb; ++r) s = fma(A[(k0 + r) * lda + j], B[(k0 + r) * ldb + rhs], s);
    B[j * ldb + rhs] -= s;
  }
}

__global__ void k_add_diag(double* __restrict__ A, int64_t n, int64_t lda, double lam) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) A[i * lda + i] += lam;
}

__global__ void k_negate_copy(const double* __restrict__ src, double* __restrict__ dst, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = -src[i];
}

// FP64 tensor-pipe peak probe: 8 independent accumulator pairs per warp, register operands only
__global__ void __launch_bounds__(256) k_dmma_peak(double* out, int iters, double a, double b) {
  double c0[8], c1[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    c0[i] = i;
    c1[i] = -i;
  }
  const double ra = a + threadIdx.x * 1e-12, rb = b;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) dmma884(c0[i], c1[i], ra, rb);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += c0[i] + c1[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// ---------------------------------------------------------------------- host drivers (device pointers)
// Two-level blocking: inner panels of NB = 128 columns (potf2 tile + substitution strips), whose
// trailing update is applied eagerly only inside the current outer block of NBO columns; the rest
// of the matrix receives ONE lazy update per outer block with k = NBO, so every C tile is read and
// written n/NBO times instead of n/NB times and the GEMM prologue/epilogue is amortised over 4x
// more math.
constexpr int NBO_MAX = 1024;

// Slice count of the lazy trailing updates (csrc/ozaki.cu): -1 = automatic, 0 = FP64 DMMA, 2..7 = int8 slices on the
// wgmma tensor cores.  Automatic: SGDML_B200_OZAKI_SLICES if set (values below 2 mean FP64, as for
// SGDML_B200_OZAKI_PREDICT_SLICES), otherwise FP64.  Measured on an H100 SXM at a 400 W
// power limit (BASELINE config 2, n = 63 000): solve 3.46 s with FP64 DMMA trailing updates, 3.65 s with 7 int8 slices
// (at a 700 W limit: 2.84 s against 2.88 s) -- the FP64 path is both faster and exact there.
static int g_solve_slices = -1;
static int resolve_slices() {
  if (g_solve_slices >= 0) return g_solve_slices;
  const char* oz = getenv("SGDML_B200_OZAKI_SLICES");
  if (oz != nullptr) {
    const int v = atoi(oz);
    return v >= 2 ? std::min(7, v) : 0;
  }
  return 0;
}

int potrf_device(double* A, int64_t n, int64_t lda, int* info_host, cudaStream_t s, bool analytic_solver) {
  int* d_info = nullptr;
  double* W = nullptr;  // -X of the current outer block (the device buffers are persistent workspaces: csrc/core.cu ws_get)
  // outer block: wide for large matrices (fewer passes over C), narrower when n is small
  const int NBO = (n >= 16384) ? NBO_MAX : ((n >= 4096) ? 512 : 256);
  const int oz_slices = resolve_slices();
  int8_t* oz_planes = nullptr;  // slice planes of the current outer panel (int8 path)
  int* oz_exps = nullptr;
  SG_TRY(ws_get(WS_POTRF_INFO, sizeof(int), (void**)&d_info));
  SG_TRY(ws_get(WS_POTRF_W, sizeof(double) * (size_t)n * NBO, (void**)&W));
  if (oz_slices > 0) {
    size_t pb = 0, eb = 0;
    SG_TRY(ozaki_syrk_workspace_bytes(n, NBO, oz_slices, &pb, &eb));
    SG_TRY(ws_get(WS_OZ_PLANES, pb, (void**)&oz_planes));
    SG_TRY(ws_get(WS_OZ_EXPS, eb, (void**)&oz_exps));
  }
  SG_CUDA(cudaMemsetAsync(d_info, 0, sizeof(int), s));
  const size_t trsm_smem = sizeof(double) * (NB + RS) * (NB + 4);
  SG_CUDA(cudaFuncSetAttribute(k_trsm_strip, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)trsm_smem));
  for (int64_t K0 = 0; K0 < n; K0 += NBO) {
    const int64_t K1 = std::min<int64_t>(K0 + NBO, n);  // end of the outer block
    for (int64_t k0 = K0; k0 < K1; k0 += NB) {
      const int kb = (int)std::min<int64_t>(NB, n - k0);
      {
        ProfScope ps(KID_POTF2, s);
        k_potf2_tile<<<1, 1024, 0, s>>>(A + k0 * lda + k0, lda, kb, k0, d_info);
        SG_CUDA(cudaGetLastError());
        count_launch(KID_POTF2);
      }
      const int64_t rem = n - k0 - kb;
      if (rem <= 0) break;
      {
        ProfScope ps(KID_TRSM, s);
        k_trsm_strip<<<(unsigned)((rem + RS - 1) / RS), 256, trsm_smem, s>>>(
            A + k0 * lda + k0, lda, kb, A + (k0 + kb) * lda + k0, lda, rem, W + (k0 + kb) * NBO + (k0 - K0), NBO, d_info);
        SG_CUDA(cudaGetLastError());
        count_launch(KID_TRSM);
      }
      const int64_t cols_in = K1 - (k0 + kb);  // columns of the outer block still to be factorised
      if (cols_in > 0) {
        GemmArgs g;
        g.m = rem;
        g.n = cols_in;
        g.k = kb;
        g.A = W + (k0 + kb) * NBO + (k0 - K0);  // -X
        g.lda = NBO;
        g.B = A + (k0 + kb) * lda + k0;  // X rows of the outer block
        g.ldb = lda;
        g.C = A + (k0 + kb) * lda + (k0 + kb);
        g.ldc = lda;
        g.alpha = 1.0;
        g.beta = 1.0;
        g.mode = 1;
        g.tri = 0;
        g.abort_flag = d_info;
        SG_TRY(launch_gemm(g, s));
      }
    }
    const int64_t rem = n - K1;
    if (rem <= 0) break;
    if (oz_slices > 0) {
      // the trailing update on the int8 tensor cores (csrc/ozaki.cu), C -= X X^T through exact int8 slice products
      const double* X = A + K1 * lda + K0;
      SG_TRY(ozaki_syrk_device(rem, K1 - K0, -1.0, X, lda, A + K1 * lda + K1, lda, oz_slices, oz_planes, oz_exps, s));
      continue;
    }
    GemmArgs g;
    g.m = rem;
    g.n = rem;
    g.k = K1 - K0;
    g.A = W + K1 * NBO;  // -X, all panels of the outer block
    g.lda = NBO;
    g.B = A + K1 * lda + K0;
    g.ldb = lda;
    g.C = A + K1 * lda + K1;
    g.ldc = lda;
    g.alpha = 1.0;
    g.beta = 1.0;
    g.mode = 1;
    g.tri = 1;
    g.abort_flag = d_info;
    SG_TRY(launch_gemm(g, s));
  }
  SG_CUDA(cudaMemcpyAsync(info_host, d_info, sizeof(int), cudaMemcpyDeviceToHost, s));
  SG_CUDA(cudaStreamSynchronize(s));
  return 0;
}

int potrs_device(const double* L, int64_t n, int64_t lda, double* B, int64_t nrhs, int64_t ldb, cudaStream_t s) {
  ProfScope ps(KID_TRSV, s);
  count_launch(KID_TRSV, (int)(4 * ((n + NB - 1) / NB) - 2));
  const size_t smem = sizeof(double) * (NB * (NB + 1) + NB);
  SG_CUDA(cudaFuncSetAttribute(k_trsv_diag, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  SG_CUDA(cudaFuncSetAttribute(k_trsv_diag1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // forward: L z = b
  for (int64_t k0 = 0; k0 < n; k0 += NB) {
    const int nb = (int)std::min<int64_t>(NB, n - k0);
    if (nrhs == 1)
      k_trsv_diag1<<<1, 256, smem, s>>>(L, lda, k0, nb, B, ldb, 0);
    else
      k_trsv_diag<<<(unsigned)std::min<int64_t>((nrhs + 127) / 128, 1024), 128, smem, s>>>(L, lda, k0, nb, B, nrhs, ldb,
                                                                                          0);
    SG_CUDA(cudaGetLastError());
    const int64_t rem = n - k0 - nb;
    if (rem > 0) {
      k_trsv_update_fwd<<<(unsigned)((rem + 7) / 8), 256, 0, s>>>(L, lda, k0, nb, n, B, nrhs, ldb);
      SG_CUDA(cudaGetLastError());
    }
  }
  // backward: L^T x = z
  const int64_t last = ((n - 1) / NB) * NB;
  for (int64_t k0 = last; k0 >= 0; k0 -= NB) {
    const int nb = (int)std::min<int64_t>(NB, n - k0);
    if (nrhs == 1)
      k_trsv_diag1<<<1, 256, smem, s>>>(L, lda, k0, nb, B, ldb, 1);
    else
      k_trsv_diag<<<(unsigned)std::min<int64_t>((nrhs + 127) / 128, 1024), 128, smem, s>>>(L, lda, k0, nb, B, nrhs, ldb,
                                                                                          1);
    SG_CUDA(cudaGetLastError());
    if (k0 > 0) {
      k_trsv_update_bwd<<<(unsigned)((k0 + 255) / 256), 256, 0, s>>>(L, lda, k0, nb, B, nrhs, ldb);
      SG_CUDA(cudaGetLastError());
    }
  }
  return 0;
}

// X <- X L^-T for a lower-triangular L (m x m) and X (n_rows x m), right-looking over 128-column
// blocks: substitution strips for the diagonal block, DMMA GEMM for the remaining columns.
int trsm_right_lt_device(const double* L, int64_t m, int64_t ldl, double* X, int64_t n_rows, int64_t ldx,
                         cudaStream_t s) {
  double* Wn = nullptr;
  SG_CUDA(cudaMalloc(&Wn, sizeof(double) * (size_t)n_rows * NB));
  auto body = [&]() -> int {
    const size_t trsm_smem = sizeof(double) * (NB + RS) * (NB + 4);
    SG_CUDA(cudaFuncSetAttribute(k_trsm_strip, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)trsm_smem));
    for (int64_t k0 = 0; k0 < m; k0 += NB) {
      const int kb = (int)std::min<int64_t>(NB, m - k0);
      {
        ProfScope ps(KID_TRSM, s);
        k_trsm_strip<<<(unsigned)((n_rows + RS - 1) / RS), 256, trsm_smem, s>>>(L + k0 * ldl + k0, ldl, kb, X + k0, ldx,
                                                                               n_rows, Wn, NB, nullptr);
        SG_CUDA(cudaGetLastError());
        count_launch(KID_TRSM);
      }
      const int64_t rest = m - k0 - kb;
      if (rest > 0) {
        GemmArgs g;
        g.m = n_rows;
        g.n = rest;
        g.k = kb;
        g.A = Wn;  // -X_blk
        g.lda = NB;
        g.B = L + (k0 + kb) * ldl + k0;
        g.ldb = ldl;
        g.C = X + (k0 + kb);
        g.ldc = ldx;
        g.alpha = 1.0;
        g.beta = 1.0;
        g.mode = 1;
        g.tri = 0;
        g.abort_flag = nullptr;
        SG_TRY(launch_gemm(g, s));
      }
    }
    SG_CUDA(cudaStreamSynchronize(s));
    return 0;
  };
  int rc = body();
  cudaFree(Wn);
  return rc;
}

}  // namespace sgdml

using namespace sgdml;

extern "C" {

int sgdml_b200_potrf(double* A, int64_t n, int64_t lda, void* stream) {
  SG_TRY(require_device());
  SG_ARG(A != nullptr && n >= 1 && lda >= n);
  cudaStream_t s = (cudaStream_t)stream;
  Staged sA;
  SG_TRY(sA.init(A, sizeof(double) * (size_t)n * lda, true, s));
  int info = 0;
  SG_TRY(potrf_device((double*)sA.dev(), n, lda, &info, s));
  SG_TRY(sA.finish(s));
  if (sA.staged()) SG_CUDA(cudaStreamSynchronize(s));
  if (info > 0) {
    char buf[160];
    snprintf(buf, sizeof(buf), "%d-th leading minor of the array is not positive definite", info);
    set_last_error(buf);
  }
  return info;
}

int sgdml_b200_potrs(const double* L, int64_t n, int64_t lda, double* B, int64_t nrhs, int64_t ldb, void* stream) {
  SG_TRY(require_device());
  SG_ARG(L != nullptr && B != nullptr && n >= 1 && lda >= n && nrhs >= 1 && ldb >= nrhs);
  cudaStream_t s = (cudaStream_t)stream;
  Staged sL, sB;
  SG_TRY(sL.init(L, sizeof(double) * (size_t)n * lda, true, s));
  SG_TRY(sB.init(B, sizeof(double) * (size_t)n * ldb, true, s));
  SG_TRY(potrs_device((const double*)sL.dev(), n, lda, (double*)sB.dev(), nrhs, ldb, s));
  SG_TRY(sB.finish(s));
  if (sL.staged() || sB.staged()) SG_CUDA(cudaStreamSynchronize(s));
  return 0;
}

int sgdml_b200_solve_analytic(double* Kneg, int64_t n, int64_t lda, double lam, const double* y, double* alphas,
                              void* stream) {
  SG_TRY(require_device());
  SG_ARG(Kneg != nullptr && y != nullptr && alphas != nullptr && n >= 1 && lda >= n);
  cudaStream_t s = (cudaStream_t)stream;
  Staged sK, sY, sX;
  SG_TRY(sK.init(Kneg, sizeof(double) * (size_t)n * lda, true, s));
  SG_TRY(sY.init(y, sizeof(double) * (size_t)n, true, s));
  SG_TRY(sX.init(alphas, sizeof(double) * (size_t)n, false, s));
  double* K = (double*)sK.dev();
  k_add_diag<<<ceil_div(n, 256), 256, 0, s>>>(K, n, lda, lam);  // analytic.py:82
  SG_CUDA(cudaGetLastError());
  count_launch(KID_MISC, 2);
  int info = 0;
  SG_TRY(potrf_device(K, n, lda, &info, s, true));  // analytic.py:94-96
  if (info > 0) {
    char buf[160];
    snprintf(buf, sizeof(buf), "%d-th leading minor of the array is not positive definite", info);
    set_last_error(buf);
    return info;
  }
  double* tmp = nullptr;
  SG_TRY(ws_get(WS_SOLVE_TMP, sizeof(double) * (size_t)n, (void**)&tmp));
  auto body = [&]() -> int {
    SG_CUDA(cudaMemcpyAsync(tmp, sY.dev(), sizeof(double) * (size_t)n, cudaMemcpyDeviceToDevice, s));
    SG_TRY(potrs_device(K, n, lda, tmp, 1, 1, s));  // analytic.py:97-99
    k_negate_copy<<<ceil_div(n, 256), 256, 0, s>>>(tmp, (double*)sX.dev(), n);
    SG_CUDA(cudaGetLastError());
    SG_TRY(sX.finish(s));
    SG_CUDA(cudaStreamSynchronize(s));
    return 0;
  };
  return body();
}

int sgdml_b200_dgemm_nt(int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda, const double* B,
                        int64_t ldb, double beta, double* C, int64_t ldc, void* stream) {
  SG_TRY(require_device());
  SG_ARG(A != nullptr && B != nullptr && C != nullptr && m >= 1 && n >= 1 && k >= 1);
  SG_ARG(lda >= k && ldb >= k && ldc >= n);
  cudaStream_t s = (cudaStream_t)stream;
  Staged sA, sB, sC;
  SG_TRY(sA.init(A, sizeof(double) * (size_t)m * lda, true, s));
  SG_TRY(sB.init(B, sizeof(double) * (size_t)n * ldb, true, s));
  SG_TRY(sC.init(C, sizeof(double) * (size_t)m * ldc, true, s));
  GemmArgs g;
  g.m = m;
  g.n = n;
  g.k = k;
  g.A = (const double*)sA.dev();
  g.lda = lda;
  g.B = (const double*)sB.dev();
  g.ldb = ldb;
  g.C = (double*)sC.dev();
  g.ldc = ldc;
  g.alpha = alpha;
  g.beta = beta;
  g.mode = 0;
  g.tri = 0;
  g.abort_flag = nullptr;
  SG_TRY(launch_gemm(g, s));
  SG_TRY(sC.finish(s));
  if (sA.staged() || sB.staged() || sC.staged()) SG_CUDA(cudaStreamSynchronize(s));
  return 0;
}

int sgdml_b200_gemm_nt_args(int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                            const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int mode, int tri,
                            const int* abort_flag, void* stream) {
  SG_TRY(require_device());
  SG_ARG(A != nullptr && B != nullptr && C != nullptr && m >= 1 && n >= 1 && k >= 1);
  SG_ARG(lda >= k && ldb >= k && ldc >= n);
  SG_ARG((mode == 0 || mode == 1) && (tri == 0 || tri == 1) && (tri == 0 || m == n));
  SG_ARG(is_device_ptr(A) && is_device_ptr(B) && is_device_ptr(C) && (abort_flag == nullptr || is_device_ptr(abort_flag)));
  GemmArgs g;
  g.m = m;
  g.n = n;
  g.k = k;
  g.A = A;
  g.lda = lda;
  g.B = B;
  g.ldb = ldb;
  g.C = C;
  g.ldc = ldc;
  g.alpha = alpha;
  g.beta = beta;
  g.mode = mode;
  g.tri = tri;
  g.abort_flag = abort_flag;
  return launch_gemm(g, (cudaStream_t)stream);
}

int sgdml_b200_fp64_peak_tflops(double* tflops) {
  SG_TRY(require_device());
  SG_ARG(tflops != nullptr);
  double* out = nullptr;
  const int grid = num_sms() * 4, iters = 1 << 14;
  SG_CUDA(cudaMalloc(&out, sizeof(double) * (size_t)grid * 256));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  double best = 0.0;
  for (int rep = 0; rep < 5; ++rep) {
    cudaEventRecord(e0, 0);
    k_dmma_peak<<<grid, 256>>>(out, iters, 1.0000001, 1e-9);
    cudaEventRecord(e1, 0);
    cudaEventSynchronize(e1);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    const double tf = 2.0 * 256.0 * 8.0 * iters * 8.0 * grid / (ms * 1e-3) * 1e-12;
    if (rep > 0 && tf > best) best = tf;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(out);
  SG_CUDA(cudaGetLastError());
  *tflops = best;
  return 0;
}

// Sustained variant: keeps the DMMA pipe saturated for `seconds` (power-capped clocks settle
// well below the burst clock on a 1 kW part) and reports the throughput of the second half.
int sgdml_b200_fp64_peak_tflops_sustained(double seconds, double* tflops) {
  SG_TRY(require_device());
  SG_ARG(tflops != nullptr && seconds > 0.0 && seconds <= 30.0);
  double* out = nullptr;
  const int grid = num_sms() * 4, iters = 1 << 14;
  SG_CUDA(cudaMalloc(&out, sizeof(double) * (size_t)grid * 256));
  cudaEvent_t e0, e1, e2;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventCreate(&e2);
  // calibrate one launch
  cudaEventRecord(e0, 0);
  k_dmma_peak<<<grid, 256>>>(out, iters, 1.0000001, 1e-9);
  cudaEventRecord(e1, 0);
  cudaEventSynchronize(e1);
  float ms1 = 1.f;
  cudaEventElapsedTime(&ms1, e0, e1);
  const int n_launch = (int)(seconds * 1e3 / ms1) + 2;
  const int half = n_launch / 2;
  for (int i = 0; i < half; ++i) k_dmma_peak<<<grid, 256>>>(out, iters, 1.0000001, 1e-9);
  cudaEventRecord(e1, 0);
  for (int i = half; i < n_launch; ++i) k_dmma_peak<<<grid, 256>>>(out, iters, 1.0000001, 1e-9);
  cudaEventRecord(e2, 0);
  cudaEventSynchronize(e2);
  float ms = 1.f;
  cudaEventElapsedTime(&ms, e1, e2);
  *tflops = 2.0 * 256.0 * 8.0 * iters * 8.0 * grid * (double)(n_launch - half) / (ms * 1e-3) * 1e-12;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaEventDestroy(e2);
  cudaFree(out);
  SG_CUDA(cudaGetLastError());
  return 0;
}

int sgdml_b200_set_solve_slices(int n_slices) {
  SG_ARG(n_slices == -1 || n_slices == 0 || (n_slices >= 2 && n_slices <= 7));
  g_solve_slices = n_slices;
  return 0;
}

int sgdml_b200_get_solve_slices(void) { return resolve_slices(); }

int sgdml_b200_set_gemm_variant(int v) {
  SG_ARG(v == 0 || v == 2 || v == 3);
  g_gemm_variant = v;
  return 0;
}

}  // extern "C"
