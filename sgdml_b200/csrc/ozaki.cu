// FP64 GEMM on the Hopper tensor cores: C += alpha * A * B^T with A and B cut into signed 7-bit slices (int8)
// and every slice-pair product computed EXACTLY by wgmma (s8 x s8 -> s32, accumulators in registers):
// Ozaki-style error-free splitting.  This is the int8 form of the Cholesky trailing update of path (a)
// (reference: scipy cho_factor = LAPACK dpotrf, sgdml/solvers/analytic.py:94-96).  The H100 data sheet gives
// 67 TFLOP/s of FP64 tensor-core throughput and 1979 TOP/s of dense int8; 28 exact int8 GEMMs (7 slices)
// bring the latter to ~70 TFLOP/s-equivalent at best, so which path is faster is a measured choice
// (csrc/solve.cu resolve_slices).
//
//   x_ij = 2^(e_i) * sum_{p=1..S} q_ij^(p) 2^(-7p),   |q^(p)| <= 64,   e_i per ROW
//   (A B^T)_ij = 2^(ea_i + eb_j) * sum_{L=2..S+1} 2^(-7L) * sum_{p+q=L} (A^(p) B^(q)T)_ij
// The inner sums are integers below 2^31 (64^2 * k * S with k <= 2^14), so the int32 tensor-core
// accumulation is exact; pairs with p + q > S + 1 are dropped (below the last kept bit).
// tools/ozaki_study.py (CPU, exact) shows what that buys on the sGDML system: with S = 7 the trained
// forces agree with the FP64 factorisation to 2e-11 at cond(K) = 2e10; S = 8 is FP64-equivalent.
//
// Kernel structure (persistent, one CTA per SM, 128 x 32 tiles of C, 288 threads, warp-specialised):
//   layout   the split kernel writes the slices UNIT-MAJOR and PRE-SWIZZLED: a pipeline unit -- slice p of one
//            64-wide k-block for a tile of 128 rows -- is one contiguous 8 KB block of global memory holding
//            exactly the bytes of the canonical K-major 64-byte-swizzle shared-memory tile, so a unit is fetched
//            with one 1-D bulk copy (cp.async.bulk, TMA engine) that streams whole DRAM pages; a 32-row B tile is
//            a contiguous quarter of a unit.
//   warps 8-11 producer (one thread): a pipeline stage holds one k-block -- the S slices of A (8 KB each), then the S slices of B
//            (2 KB each) in slice order -- filled by 2 S bulk copies; 3 stages at S = 7 (210 KB)
//   warps 0-7  two consumer warpgroups, 64 rows of the tile each: one m64 n32 k32 wgmma per slice pair into the
//            register accumulator of its level (16 registers each, 16 S in all).  The level accumulators are summed
//            smallest level first in FP64, scaled by 2^(ea_i + eb_j) and added to C straight from registers.
//   raster   CTAs walk the tiles super-tile by super-tile (8 x 32 tiles = 1024 x 1024 of C), so the slices
//            the concurrently running CTAs read (2 x 1024 rows) stay L2-resident while they are reused
#include <cuda.h>

#include <cfloat>

#include "common.cuh"
#include "solve.cuh"

namespace sgdml {

constexpr int OZ_BITS = 7;
constexpr int OZ_MAX_S = 7;
constexpr int OZ_BM = 128, OZ_BN = 32;
constexpr int OZ_KPAD = 128;                               // the contraction length is padded to a multiple of this
// BK = bytes (= int8 elements) of k per pipeline unit = width of one swizzle row (64-byte swizzle)
constexpr int OZ_BK = 64;
constexpr int OZ_RING_BYTES = 210 * 1024;
constexpr int OZ_MAX_RING = 8;
constexpr int OZ_MMA_K = 32;                               // k per wgmma for 8-bit operands
constexpr int OZ_A_BYTES = OZ_BM * OZ_BK;                  // 8 KB: one unit of a 128-row tile (global and shared)
constexpr int OZ_B_BYTES = OZ_BN * OZ_BK;                  // 2 KB
constexpr int OZ_UNIT_BYTES = OZ_A_BYTES + OZ_B_BYTES;     // 10 KB; both parts 1024-byte aligned
constexpr int OZ_GSM = 8, OZ_GSN = 32;                     // super-tile: 8 x 32 tiles = 1024 x 1024 elements of C

// ---------------------------------------------------------------- splitting kernels
// Row exponent + S rounds of (scale by 2^7, round to nearest, subtract): x = 2^e sum_p q_p 2^(-7p), |q_p| <= 64.
// A row that holds a NaN or an infinity gets the exponent OZ_EXP_NONFINITE and all-zero slices; the epilogue writes NaN
// to every entry of C in its row (A) or column (B).  fmax skips NaN, so without the mark such a row would be sliced as if
// the entry were zero (and an infinity would leave the row's other slices out of int8 range).
constexpr int OZ_EXP_NONFINITE = 1 << 20;
__device__ __forceinline__ int oz_row_exponent(const double* __restrict__ x, int64_t k, int lane) {
  double amax = 0.0;
  bool finite = true;
  for (int64_t j = lane; j < k; j += 32) {
    const double a = fabs(x[j]);
    amax = fmax(amax, a);
    finite = finite && a <= DBL_MAX;  // false for NaN and infinities
  }
  if (!__all_sync(0xffffffffu, finite)) return OZ_EXP_NONFINITE;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  int e = 0;
  if (amax > 0.0) {
    frexp(amax, &e);  // amax = f 2^e, f in [0.5, 1)
    e += 1;           // |x| 2^-e < 1/2
  }
  return e;
}

// Plain layout (bring-up aid only): planes [S][rows_pad][kp] int8, zero padded; exps [rows_pad].
__global__ void __launch_bounds__(256) k_ozaki_split(const double* __restrict__ X, int64_t rows, int64_t k, int64_t ldx,
                                                    int S, int64_t rows_pad, int64_t kp, int8_t* __restrict__ planes,
                                                    int* __restrict__ exps) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows_pad) return;
  if (r >= rows) {  // padding rows: zeros
    for (int p = 0; p < S; ++p)
      for (int64_t j = lane; j < kp; j += 32) planes[((int64_t)p * rows_pad + r) * kp + j] = 0;
    if (lane == 0) exps[r] = 0;
    return;
  }
  const double* x = X + r * ldx;
  const int e = oz_row_exponent(x, k, lane);
  if (lane == 0) exps[r] = e;
  for (int64_t j = lane; j < kp; j += 32) {
    double v = (j < k && e != OZ_EXP_NONFINITE) ? ldexp(x[j], -e) : 0.0;
    for (int p = 0; p < S; ++p) {
      v *= (double)(1 << OZ_BITS);
      const double q = rint(v);  // |q| <= 64, remainder in [-1/2, 1/2]
      planes[((int64_t)p * rows_pad + r) * kp + j] = (int8_t)(int)q;
      v -= q;
    }
  }
}

// Unit-major pre-swizzled layout (what the GEMM reads): units [kb][p][row tile of 128] of 8192 bytes each; inside a
// unit, row r (0..127) is 64 bytes at r*64 and its 16-byte chunk c is stored at chunk c ^ ((r >> 1) & 3) -- the
// byte image of the canonical K-major SWIZZLE_64B shared-memory tile, so that a unit is fetched by ONE contiguous
// bulk copy (a 32-row B tile is a contiguous quarter of a unit: the swizzle only involves row bits 1-2).
// One warp per row; every lane converts 4 consecutive k (one 32-bit store per slice).
__global__ void __launch_bounds__(256) k_ozaki_split_sw(const double* __restrict__ X, int64_t rows, int64_t k,
                                                       int64_t ldx, int S, int64_t rows_pad, int64_t kp,
                                                       int8_t* __restrict__ units, int* __restrict__ exps) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows_pad) return;
  const int64_t RT = rows_pad / OZ_BM, rt = r / OZ_BM;
  const int rin = (int)(r - rt * OZ_BM);
  const int sw = (rin >> 1) & 3;
  int e = 0;
  const double* x = X + r * ldx;
  if (r < rows) e = oz_row_exponent(x, k, lane);
  if (lane == 0) exps[r] = e;
  const bool live = r < rows && e != OZ_EXP_NONFINITE;
  // x 2^-e, rounded once (= ldexp(x, -e)): 2^-e is a double for e >= -1023 (2^-1025 is subnormal but exact); below that,
  // for rows whose largest entry is under 2^-1025, scale in two exact steps through 2^512
  const bool tiny = e < -1021;
  const double pre = tiny ? 0x1p512 : 1.0;
  const double sc = ldexp(1.0, tiny ? -e - 512 : -e);  // exact power of two
  for (int64_t j0 = (int64_t)lane * 4; j0 < kp; j0 += 128) {
    double v[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) v[t] = (live && j0 + t < k) ? x[j0 + t] * pre * sc : 0.0;
    const int64_t kb = j0 / OZ_BK;
    const int jj = (int)(j0 - kb * OZ_BK);  // byte within the 64-byte row: chunk jj/16, offset jj%16 (multiple of 4)
    const int off = rin * OZ_BK + (((jj >> 4) ^ sw) << 4) + (jj & 15);
    for (int p = 0; p < S; ++p) {
      uint32_t word = 0;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        v[t] *= (double)(1 << OZ_BITS);
        const double q = rint(v[t]);
        v[t] -= q;
        word |= ((uint32_t)(int)q & 0xffu) << (8 * t);
      }
      *reinterpret_cast<uint32_t*>(units + (((kb * S + p) * RT + rt) * (int64_t)OZ_A_BYTES + off)) = word;
    }
  }
}

// ---------------------------------------------------------------- wgmma helpers
// Shared-memory matrix descriptor (sm_90 wgmma), K-major operand in the canonical 64-byte-swizzle layout: rows are
// 64 bytes apart, an 8-row swizzle atom is 512 bytes, the 16-byte chunk index of a row is XORed with bits [1,3) of
// the row number.
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1) |
//   [32,46) stride byte offset >> 4 (512 B between 8-row groups) | [49,52) base offset = 0 (atoms 512-byte aligned) |
//   [62,64) layout type = 2 (SWIZZLE_64B)
__device__ __forceinline__ uint64_t gmma_desc_kmajor_sw64(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((8 * OZ_BK) >> 4) << 32;
  d |= (uint64_t)2 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// D (64 x 32, int32, registers) += A (64 x 32) * B (32 x 32)^T, signed 8-bit, both K-major in shared memory
__device__ __forceinline__ void wgmma_s8_n32(int* d, uint64_t da, uint64_t db) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n"
      "}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "l"(da), "l"(db), "n"(1));
}

struct OzArgs {
  int64_t m, n;      // C is m x n (rows of A, rows of B)
  int64_t kp;        // padded contraction length (multiple of OZ_KPAD)
  int64_t rt_a, rt_b;  // 128-row tiles per slice of A / B (the unit strides)
  int S;             // slices per operand
  int tri;           // 1: only tiles that touch the lower triangle (m == n, A and B the same row set)
  double alpha;      // +1 or -1 (any finite value works)
  const int8_t* ua;  // units of A: [kb][p][rt_a][8192]
  const int8_t* ub;  // units of B
  const int* ea;     // row exponents of A (m_pad)
  const int* eb;     // row exponents of B (n_pad)
  double* C;
  int64_t ldc;
  int* dbg_levels;   // bring-up: raw int32 level sums, [S][m][n] (NULL in production)
  int overwrite;     // 1: C = alpha A B^T (the old contents of C are not read)
  int dbg_flags;     // timing experiments (SGDML_B200_OZAKI_DBG): 1 = no global read-modify-write in the epilogue,
                     // 2 = no wgmma issued, 4 = epilogue reads only one level
};

struct OzSmemTail {
  uint64_t full[OZ_MAX_RING];
  uint64_t empty[OZ_MAX_RING];
};

constexpr size_t OZ_SMEM_BYTES = (size_t)OZ_RING_BYTES + sizeof(OzSmemTail) + 1024;
static_assert(OZ_SMEM_BYTES <= 232448, "exceeds 227 KB of shared memory");

// CTA number -> tile (tm, tn), super-tile by super-tile; false if the CTA has no tile
__device__ __forceinline__ bool oz_tile_of_cta(const OzArgs& p, int64_t cta, int64_t& tm, int64_t& tn) {
  constexpr int PER = OZ_GSM * OZ_GSN;
  const int64_t ntm = (p.m + OZ_BM - 1) / OZ_BM, ntn = (p.n + OZ_BN - 1) / OZ_BN;
  const int64_t sb = cta / PER;
  const int local = (int)(cta - sb * PER);
  int64_t si, sj;
  if (p.tri) {  // super-tiles of the lower triangle (1024 x 1024 each): row t holds t + 1 of them
    int64_t t = (int64_t)((sqrt(8.0 * (double)sb + 1.0) - 1.0) * 0.5);
    while ((t + 1) * (t + 2) / 2 <= sb) ++t;
    while (t * (t + 1) / 2 > sb) --t;
    si = t;
    sj = sb - t * (t + 1) / 2;
  } else {
    const int64_t nsn = (ntn + OZ_GSN - 1) / OZ_GSN;
    si = sb / nsn;
    sj = sb - si * nsn;
  }
  // inside a super-tile the n tiles of one m tile are adjacent: concurrently resident CTAs share the A tile
  tm = si * OZ_GSM + local / OZ_GSN;
  tn = sj * OZ_GSN + local % OZ_GSN;
  if (tm >= ntm || tn >= ntn) return false;
  if (p.tri && tn * OZ_BN > tm * OZ_BM + OZ_BM - 1) return false;  // entirely above the diagonal
  return true;
}

// The wgmma sequence of one k32 step for one consumer warpgroup: one m64 n32 k32 product per slice pair (pa, q),
// pa + q <= S + 1, into the accumulator of level pa + q.  S is a template parameter, so the pair schedule (28 pairs
// for S = 7) is a compile-time list and the accumulator indices are constants: the level accumulators stay in
// registers.  Every product has the same shape on its own 16 registers; wider products over several consecutive
// levels (N = 64, 128) would overlap the windows of other slices' products at other alignments, and ptxas then
// serialises the whole wgmma pipeline (C7511).
template <int S, int PA, int Q>
__device__ __forceinline__ void oz_issue_slice(int* acc, uint64_t desc_hi, uint32_t a_lo, uint32_t b_lo) {
  if constexpr (PA + Q <= S + 1) {
    // A tiles are 8192 B apart (+512 in the >> 4 address field), B tiles 2048 B (+128)
    const uint64_t da = desc_hi | (uint64_t)((a_lo + (uint32_t)(PA - 1) * (OZ_A_BYTES >> 4)) & 0x3FFF);
    const uint64_t db = desc_hi | (uint64_t)((b_lo + (uint32_t)(Q - 1) * (OZ_B_BYTES >> 4)) & 0x3FFF);
    wgmma_s8_n32(acc + 16 * (PA + Q - 2), da, db);
    oz_issue_slice<S, PA, Q + 1>(acc, desc_hi, a_lo, b_lo);
  }
}
template <int S, int PA>
__device__ __forceinline__ void oz_issue_kstep(int* acc, uint64_t desc_hi, uint32_t a_lo, uint32_t b_lo) {
  if constexpr (PA <= S) {
    oz_issue_slice<S, PA, 1>(acc, desc_hi, a_lo, b_lo);
    oz_issue_kstep<S, PA + 1>(acc, desc_hi, a_lo, b_lo);
  }
}

constexpr int OZ_CONSUMERS = 256;               // warps 0-7: two consumer warpgroups
constexpr int OZ_THREADS = OZ_CONSUMERS + 128;  // warps 8-11: producer warpgroup (one thread issues the copies)

// PERSISTENT: a CTA walks over the tiles  blockIdx.x, blockIdx.x + gridDim.x, ...  of the super-tile raster (so the
// CTAs that run at the same time still work on neighbouring tiles).  The producer streams the k-block stages of one
// tile after the other without a bubble; the read-modify-write of C at the end of a tile overlaps the loads of the
// next tile's first stages.
template <int S>
__global__ void __launch_bounds__(OZ_THREADS, 1) k_ozaki_gemm(const OzArgs p, int64_t n_ids) {
  extern __shared__ unsigned char oz_raw[];
  // 1024-byte alignment for the swizzled tiles
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(oz_raw) + 1023) & ~(uintptr_t)1023);
  // a pipeline stage holds one k-block: the S slices of A (8 KB each), then the S slices of B (2 KB each) in slice order
  constexpr int STAGE_BYTES = S * OZ_UNIT_BYTES;
  constexpr int NST_FIT = OZ_RING_BYTES / STAGE_BYTES;
  constexpr int NST = NST_FIT < OZ_MAX_RING ? NST_FIT : OZ_MAX_RING;
  static_assert(NST >= 2, "at least two k-blocks in flight");
  OzSmemTail* tail = reinterpret_cast<OzSmemTail*>(smem + (size_t)OZ_RING_BYTES);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int i = 0; i < NST; ++i) {
      mbar_init(&tail->full[i], 1);
      mbar_init(&tail->empty[i], OZ_CONSUMERS / 32);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int KB = (int)(p.kp / OZ_BK);

  if (warp >= OZ_CONSUMERS / 32) {
    // ===================================================== producer: 2 S contiguous bulk copies per k-block
    // the register file goes to the consumers' level accumulators (128 x 40 + 256 x 232 <= 64 K registers)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (tid == OZ_CONSUMERS) {
      const int64_t a_stride = p.rt_a * (int64_t)OZ_A_BYTES, b_stride = p.rt_b * (int64_t)OZ_A_BYTES;  // per (kb, slice)
      int st = 0;
      uint32_t round = 0;
      for (int64_t id = blockIdx.x; id < n_ids; id += gridDim.x) {
        int64_t tm, tn;
        if (!oz_tile_of_cta(p, id, tm, tn)) continue;
        const int64_t n0 = tn * OZ_BN;
        const int8_t* a_src = p.ua + tm * (int64_t)OZ_A_BYTES;
        const int8_t* b_src = p.ub + (n0 / OZ_BM) * (int64_t)OZ_A_BYTES + (n0 % OZ_BM) * OZ_BK;
        for (int kb = 0; kb < KB; ++kb) {
          if (round > 0) mbar_wait(&tail->empty[st], (round - 1) & 1);  // the stage's previous k-block is consumed
          unsigned char* base = smem + (size_t)st * STAGE_BYTES;
          mbar_arrive_expect_tx(&tail->full[st], (uint32_t)STAGE_BYTES);
#pragma unroll
          for (int sl = 0; sl < S; ++sl) {
            bulk_g2s(base + sl * OZ_A_BYTES, a_src + sl * a_stride, OZ_A_BYTES, &tail->full[st]);
            bulk_g2s(base + S * OZ_A_BYTES + sl * OZ_B_BYTES, b_src + sl * b_stride, OZ_B_BYTES, &tail->full[st]);
          }
          a_src += (int64_t)S * a_stride;
          b_src += (int64_t)S * b_stride;
          if (++st == NST) {
            st = 0;
            ++round;
          }
        }
      }
    }
    return;
  }

  // ===================================================== consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63 of a tile
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = warp >> 2;
  const uint64_t desc_hi = gmma_desc_kmajor_sw64(0);  // everything but the 14-bit start-address field
  const uint32_t smem_base = smem_u32(smem);
  const bool no_mma = (p.dbg_flags & 2) != 0;
  int st = 0;
  uint32_t round = 0;
  for (int64_t id = blockIdx.x; id < n_ids; id += gridDim.x) {
    int64_t tm, tn;
    if (!oz_tile_of_cta(p, id, tm, tn)) continue;
    int acc[16 * S];  // level L = 2 .. S + 1 in acc[16 (L - 2) .. 16 (L - 2) + 15]
#pragma unroll
    for (int i = 0; i < 16 * S; ++i) acc[i] = 0;
    int prev = -1;  // stage of the previous k-block, released once its products have completed
    for (int kb = 0; kb < KB; ++kb) {
      mbar_wait(&tail->full[st], round & 1);
      if (!no_mma) {
        const uint32_t a0 = smem_base + (uint32_t)st * STAGE_BYTES + (uint32_t)wg * (64 * OZ_BK);
        const uint32_t b0 = smem_base + (uint32_t)st * STAGE_BYTES + (uint32_t)(S * OZ_A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < OZ_BK / OZ_MMA_K; ++ks)  // K advance inside the 64-byte swizzle row: +32 B = +2
          oz_issue_kstep<S, 1>(acc, desc_hi, ((a0 >> 4) + 2 * ks) & 0x3FFF, ((b0 >> 4) + 2 * ks) & 0x3FFF);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's products have completed: its stage may be refilled
      }
      if (prev >= 0 && lane == 0) mbar_arrive(&tail->empty[prev]);
      prev = st;
      if (++st == NST) {
        st = 0;
        ++round;
      }
    }
    wgmma_wait<0>();
    if (prev >= 0 && lane == 0) mbar_arrive(&tail->empty[prev]);

    // ---- epilogue: thread holds rows r0, r0 + 8 and columns n0 + 8 j + 2 (lane % 4) + {0, 1}, j = 0..3
    //      (acc[16 l + 4 j + {0, 1}] on row r0, acc[16 l + 4 j + {2, 3}] on row r0 + 8)
    const int64_t m0 = tm * OZ_BM, n0 = tn * OZ_BN;
    const int64_t r0 = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
    double v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = 0.0;
#pragma unroll
    for (int level = S + 1; level >= 2; --level) {  // smallest contributions first
      if ((p.dbg_flags & 4) && level > 2) continue;
      const double w = __longlong_as_double((long long)(1023 - OZ_BITS * level) << 52);  // 2^(-7 level), exact
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = fma((double)acc[16 * (level - 2) + i], w, v[i]);
      if (p.dbg_levels != nullptr) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int64_t r = r0 + 8 * ((i >> 1) & 1), c = n0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
          if (r < p.m && c < p.n) p.dbg_levels[((int64_t)(level - 2) * p.m + r) * p.n + c] = acc[16 * (level - 2) + i];
        }
      }
    }
    if (p.dbg_flags & 1) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t r = r0 + 8 * h;
      if (r >= p.m) continue;
      const int ea = p.ea[r];
      double* crow = p.C + r * p.ldc;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (((i >> 1) & 1) != h) continue;
        const int64_t c = n0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        if (c >= p.n) continue;
        const int eb = p.eb[c];
        // one scaling by 2^(ea + eb), = ldexp(alpha v, ea + eb): 2^ea alone is infinite for a row whose largest entry
        // is >= 2^1023 (ea = 1025).  In the normal range the power of two is built from its bits (one rounding either way).
        const int es = ea + eb;
        const double av = p.alpha * v[i];
        double upd;
        if (ea == OZ_EXP_NONFINITE || eb == OZ_EXP_NONFINITE)
          upd = __longlong_as_double(0x7ff8000000000000ll);
        else if (es >= -1022 && es <= 1023)
          upd = av * __longlong_as_double((long long)(es + 1023) << 52);
        else
          upd = ldexp(av, es);
        crow[c] = p.overwrite ? upd : crow[c] + upd;
      }
    }
  }
}

// ---------------------------------------------------------------- host side
static size_t oz_plane_bytes(int64_t rows, int64_t k, int S) {
  const int64_t rows_pad = (rows + OZ_BM - 1) / OZ_BM * OZ_BM, kp = (k + OZ_KPAD - 1) / OZ_KPAD * OZ_KPAD;
  return (size_t)S * rows_pad * kp;
}

// slices X (rows x k) into caller-provided device memory (unit-major pre-swizzled layout)
static int oz_split_into(const double* X, int64_t rows, int64_t k, int64_t ldx, int S, int8_t* units, int* exps,
                         OzOperand* o, cudaStream_t s) {
  o->rows_pad = (rows + OZ_BM - 1) / OZ_BM * OZ_BM;
  o->kp = (k + OZ_KPAD - 1) / OZ_KPAD * OZ_KPAD;
  o->units = units;
  o->exps = exps;
  k_ozaki_split_sw<<<ceil_div(o->rows_pad, 8), 256, 0, s>>>(X, rows, k, ldx, S, o->rows_pad, o->kp, o->units, o->exps);
  SG_CUDA(cudaGetLastError());
  count_launch(KID_GEMM);
  return 0;
}

static int oz_launch(const OzOperand& oa, const OzOperand& ob, int64_t m, int64_t n, double alpha, double* C,
                     int64_t ldc, int S, int tri, cudaStream_t s, int* dbg_levels = nullptr, int overwrite = 0) {
  static bool configured[64] = {false};
  int dev = 0;
  SG_CUDA(cudaGetDevice(&dev));
  if (dev >= 0 && dev < 64 && !configured[dev]) {
    SG_CUDA(cudaFuncSetAttribute(k_ozaki_gemm<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM_BYTES));
    SG_CUDA(cudaFuncSetAttribute(k_ozaki_gemm<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM_BYTES));
    SG_CUDA(cudaFuncSetAttribute(k_ozaki_gemm<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM_BYTES));
    SG_CUDA(cudaFuncSetAttribute(k_ozaki_gemm<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM_BYTES));
    SG_CUDA(cudaFuncSetAttribute(k_ozaki_gemm<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM_BYTES));
    SG_CUDA(cudaFuncSetAttribute(k_ozaki_gemm<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM_BYTES));
    configured[dev] = true;
  }
  SG_ARG(oa.kp == ob.kp);
  OzArgs a;
  a.m = m;
  a.n = n;
  a.kp = oa.kp;
  a.rt_a = oa.rows_pad / OZ_BM;
  a.rt_b = ob.rows_pad / OZ_BM;
  a.S = S;
  a.tri = tri;
  a.alpha = alpha;
  a.ua = oa.units;
  a.ub = ob.units;
  a.ea = oa.exps;
  a.eb = ob.exps;
  a.C = C;
  a.ldc = ldc;
  a.dbg_levels = dbg_levels;
  a.overwrite = overwrite;
  {
    const char* df = getenv("SGDML_B200_OZAKI_DBG");
    a.dbg_flags = df ? atoi(df) : 0;
  }
  const int64_t ntm = ceil_div(m, OZ_BM), ntn = ceil_div(n, OZ_BN);
  int64_t n_super;
  if (tri) {
    const int64_t sr = (ntm + OZ_GSM - 1) / OZ_GSM;  // 1024-row super-tile rows; (GSM * BM == GSN * BN)
    n_super = sr * (sr + 1) / 2;
  } else {
    n_super = ((ntm + OZ_GSM - 1) / OZ_GSM) * ((ntn + OZ_GSN - 1) / OZ_GSN);
  }
  const int64_t blocks = n_super * OZ_GSM * OZ_GSN;
  SG_ARG(blocks < ((int64_t)1 << 31));
  const unsigned grid = (unsigned)std::min<int64_t>(blocks, (int64_t)num_sms());
  ProfScope ps(KID_GEMM, s);
  switch (S) {
    case 2: k_ozaki_gemm<2><<<grid, OZ_THREADS, OZ_SMEM_BYTES, s>>>(a, blocks); break;
    case 3: k_ozaki_gemm<3><<<grid, OZ_THREADS, OZ_SMEM_BYTES, s>>>(a, blocks); break;
    case 4: k_ozaki_gemm<4><<<grid, OZ_THREADS, OZ_SMEM_BYTES, s>>>(a, blocks); break;
    case 5: k_ozaki_gemm<5><<<grid, OZ_THREADS, OZ_SMEM_BYTES, s>>>(a, blocks); break;
    case 6: k_ozaki_gemm<6><<<grid, OZ_THREADS, OZ_SMEM_BYTES, s>>>(a, blocks); break;
    case 7: k_ozaki_gemm<7><<<grid, OZ_THREADS, OZ_SMEM_BYTES, s>>>(a, blocks); break;
    default: return fail_arg("2 <= n_slices <= 7");
  }
  SG_CUDA(cudaGetLastError());
  count_launch(KID_GEMM);
  return 0;
}
static_assert(OZ_GSM * OZ_BM == OZ_GSN * OZ_BN, "square super-tiles (the triangular raster relies on it)");

// ---- operand-level interface (csrc/predict.cu keeps the slices of the model matrices between calls)
size_t ozaki_units_bytes(int64_t rows, int64_t k, int S) { return oz_plane_bytes(rows, k, S); }
size_t ozaki_exps_bytes(int64_t rows) { return sizeof(int) * (size_t)((rows + OZ_BM - 1) / OZ_BM * OZ_BM); }
int ozaki_split(const double* X, int64_t rows, int64_t k, int64_t ldx, int S, int8_t* units, int* exps, OzOperand* o,
                cudaStream_t s) {
  SG_ARG(S >= 2 && S <= OZ_MAX_S && rows >= 1 && k >= 1 && k <= (1 << 14));
  return oz_split_into(X, rows, k, ldx, S, units, exps, o, s);
}
int ozaki_gemm(const OzOperand& a, const OzOperand& b, int64_t m, int64_t n, double alpha, int overwrite, double* C,
               int64_t ldc, int S, cudaStream_t s) {
  SG_ARG(a.kp == b.kp && m <= a.rows_pad && n <= b.rows_pad);
  return oz_launch(a, b, m, n, alpha, C, ldc, S, 0, s, nullptr, overwrite);
}

// Workspace of the symmetric update used by potrf: allocated once per factorisation (a cudaMalloc /
// cudaFree pair costs milliseconds in a process that holds tens of GB -- see csrc/core.cu), reused by every
// outer step, no host synchronisation in between.
int ozaki_syrk_workspace_bytes(int64_t max_rows, int64_t max_k, int S, size_t* plane_bytes, size_t* exp_bytes) {
  *plane_bytes = oz_plane_bytes(max_rows, max_k, S);
  *exp_bytes = sizeof(int) * (size_t)((max_rows + OZ_BM - 1) / OZ_BM * OZ_BM);
  return 0;
}

// C (n x n, lower-triangle tiles) += alpha X X^T with X (n x k): stream-ordered, no allocation
int ozaki_syrk_device(int64_t n, int64_t k, double alpha, const double* X, int64_t ldx, double* C, int64_t ldc, int S,
                      int8_t* planes, int* exps, cudaStream_t s) {
  SG_ARG(S >= 2 && S <= OZ_MAX_S && n >= 1 && k >= 1 && k <= (1 << 14));
  OzOperand o;
  SG_TRY(oz_split_into(X, n, k, ldx, S, planes, exps, &o, s));
  return oz_launch(o, o, n, n, alpha, C, ldc, S, 1, s);
}

// C (m x n, ldc) += alpha * A (m x k, lda) * B (n x k, ldb)^T through S int8 slices per operand.
// tri != 0: m == n and only tiles touching the lower triangle are updated.  All pointers on the device.
// Self-contained form (allocates and frees its slice planes, synchronises the stream): tests and the
// predictor experiment; the Cholesky uses ozaki_syrk_device.
int ozaki_gemm_nt_device(int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda, const double* B,
                         int64_t ldb, double* C, int64_t ldc, int S, int tri, int overwrite, cudaStream_t s) {
  SG_ARG(S >= 2 && S <= OZ_MAX_S && m >= 1 && n >= 1 && k >= 1);
  SG_ARG(k <= (1 << 14));  // int32 accumulation stays exact: 64^2 * k * S < 2^31
  const bool same = (A == B && m == n && lda == ldb);
  int8_t *pa = nullptr, *pb = nullptr;
  int *xa = nullptr, *xb = nullptr;
  auto cleanup = [&]() {
    cudaFree(pa);
    cudaFree(xa);
    cudaFree(pb);
    cudaFree(xb);
  };
  auto body = [&]() -> int {
    OzOperand oa, ob;
    SG_CUDA(cudaMalloc(&pa, oz_plane_bytes(m, k, S)));
    SG_CUDA(cudaMalloc(&xa, sizeof(int) * (size_t)((m + OZ_BM - 1) / OZ_BM * OZ_BM)));
    SG_TRY(oz_split_into(A, m, k, lda, S, pa, xa, &oa, s));
    if (same) {
      ob = oa;
    } else {
      SG_CUDA(cudaMalloc(&pb, oz_plane_bytes(n, k, S)));
      SG_CUDA(cudaMalloc(&xb, sizeof(int) * (size_t)((n + OZ_BM - 1) / OZ_BM * OZ_BM)));
      SG_TRY(oz_split_into(B, n, k, ldb, S, pb, xb, &ob, s));
    }
    SG_TRY(oz_launch(oa, ob, m, n, alpha, C, ldc, S, tri, s, nullptr, overwrite));
    SG_CUDA(cudaStreamSynchronize(s));  // the planes are freed below
    return 0;
  };
  int rc = body();
  cleanup();
  return rc;
}

// Bring-up aid: runs the split and the int8 products and hands back every intermediate.
//   planes_a [S][m_pad][kp] int8 (plain row-major layout), exps_a [m_pad], planes_b / exps_b likewise,
//   levels [S][m][n] int32 (all device pointers; any of them may be NULL).  C receives C + A B^T as usual.
int ozaki_debug_device(int64_t m, int64_t n, int64_t k, const double* A, int64_t lda, const double* B, int64_t ldb,
                       double* C, int64_t ldc, int S, int8_t* planes_a, int* exps_a, int8_t* planes_b, int* exps_b,
                       int* levels, cudaStream_t s) {
  SG_ARG(S >= 2 && S <= OZ_MAX_S && m >= 1 && n >= 1 && k >= 1 && k <= (1 << 14));
  int8_t *pa = nullptr, *pb = nullptr;
  int *xa = nullptr, *xb = nullptr;
  auto cleanup = [&]() {
    cudaFree(pa);
    cudaFree(xa);
    cudaFree(pb);
    cudaFree(xb);
  };
  auto body = [&]() -> int {
    OzOperand oa, ob;
    const size_t ba = oz_plane_bytes(m, k, S), bb = oz_plane_bytes(n, k, S);
    const int64_t mp = (m + OZ_BM - 1) / OZ_BM * OZ_BM, np = (n + OZ_BM - 1) / OZ_BM * OZ_BM, kp = (k + OZ_KPAD - 1) / OZ_KPAD * OZ_KPAD;
    const size_t ea = sizeof(int) * (size_t)mp, eb = sizeof(int) * (size_t)np;
    SG_CUDA(cudaMalloc(&pa, ba));
    SG_CUDA(cudaMalloc(&xa, ea));
    SG_CUDA(cudaMalloc(&pb, bb));
    SG_CUDA(cudaMalloc(&xb, eb));
    // the plain-layout planes for the caller (their exponents are the ones the GEMM uses too)
    if (planes_a) {
      k_ozaki_split<<<ceil_div(mp, 8), 256, 0, s>>>(A, m, k, lda, S, mp, kp, planes_a, xa);
      SG_CUDA(cudaGetLastError());
    }
    if (planes_b) {
      k_ozaki_split<<<ceil_div(np, 8), 256, 0, s>>>(B, n, k, ldb, S, np, kp, planes_b, xb);
      SG_CUDA(cudaGetLastError());
    }
    SG_TRY(oz_split_into(A, m, k, lda, S, pa, xa, &oa, s));
    SG_TRY(oz_split_into(B, n, k, ldb, S, pb, xb, &ob, s));
    if (exps_a) SG_CUDA(cudaMemcpyAsync(exps_a, xa, ea, cudaMemcpyDeviceToDevice, s));
    if (exps_b) SG_CUDA(cudaMemcpyAsync(exps_b, xb, eb, cudaMemcpyDeviceToDevice, s));
    if (C != nullptr) SG_TRY(oz_launch(oa, ob, m, n, 1.0, C, ldc, S, 0, s, levels));
    SG_CUDA(cudaStreamSynchronize(s));
    return 0;
  };
  int rc = body();
  cleanup();
  return rc;
}

}  // namespace sgdml

using namespace sgdml;

extern "C" int sgdml_b200_ozaki_debug(int64_t m, int64_t n, int64_t k, const double* A, int64_t lda, const double* B,
                                      int64_t ldb, double* C, int64_t ldc, int n_slices, int8_t* planes_a, int* exps_a,
                                      int8_t* planes_b, int* exps_b, int* levels, void* stream) {
  SG_TRY(require_device());
  SG_ARG(A != nullptr && B != nullptr && lda >= k && ldb >= k);
  return ozaki_debug_device(m, n, k, A, lda, B, ldb, C, ldc, n_slices, planes_a, exps_a, planes_b, exps_b, levels,
                            (cudaStream_t)stream);
}

extern "C" int sgdml_b200_ozaki_gemm_nt(int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                                        const double* B, int64_t ldb, double* C, int64_t ldc, int n_slices, int tri,
                                        void* stream) {
  SG_TRY(require_device());
  SG_ARG(A != nullptr && B != nullptr && C != nullptr && lda >= k && ldb >= k && ldc >= n);
  SG_ARG(is_device_ptr(A) && is_device_ptr(B) && is_device_ptr(C));
  if (tri) SG_ARG(m == n);
  return ozaki_gemm_nt_device(m, n, k, alpha, A, lda, B, ldb, C, ldc, n_slices, tri, 0, (cudaStream_t)stream);
}

extern "C" int sgdml_b200_ozaki_gemm_args(int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                                          const double* B, int64_t ldb, double* C, int64_t ldc, int n_slices, int tri,
                                          int overwrite, void* stream) {
  SG_TRY(require_device());
  SG_ARG(A != nullptr && B != nullptr && C != nullptr && lda >= k && ldb >= k && ldc >= n);
  SG_ARG((tri == 0 || tri == 1) && (tri == 0 || m == n) && (overwrite == 0 || overwrite == 1));
  SG_ARG(is_device_ptr(A) && is_device_ptr(B) && is_device_ptr(C));
  return ozaki_gemm_nt_device(m, n, k, alpha, A, lda, B, ldb, C, ldc, n_slices, tri, overwrite, (cudaStream_t)stream);
}
