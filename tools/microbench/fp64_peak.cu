// FP64 pipe microbenchmarks for H100 (sm_90a). Decides DFMA-vs-DMMA for the
// sgdml_b200 kernels and provides the FP64 roofline denominator.
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o fp64_peak fp64_peak.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { \
  printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1);} } while (0)

template <int CHAINS>
__global__ void __launch_bounds__(256) k_dfma(double* out, int iters, double a, double b) {
  double acc[CHAINS];
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) acc[i] = threadIdx.x * 1e-9 + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < CHAINS; ++i) acc[i] = fma(acc[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// mma.sync m8n8k4 f64: 256 FMA per warp instruction
template <int CHAINS>
__global__ void __launch_bounds__(256) k_dmma884(double* out, int iters, double a, double b) {
  double c0[CHAINS], c1[CHAINS];
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) { c0[i] = i; c1[i] = -i; }
  double ra = a + threadIdx.x * 1e-12, rb = b;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < CHAINS; ++i) {
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                   : "+d"(c0[i]), "+d"(c1[i]) : "d"(ra), "d"(rb));
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) s += c0[i] + c1[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// m16n8k4 f64: A 2 regs, B 1 reg, C 4 regs: 512 FMA / warp instr
template <int CHAINS>
__global__ void __launch_bounds__(256) k_dmma1684(double* out, int iters, double a, double b) {
  double c[CHAINS][4];
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) { c[i][0] = i; c[i][1] = -i; c[i][2] = 1; c[i][3] = 2; }
  double ra0 = a + threadIdx.x * 1e-12, ra1 = a * 0.5, rb = b;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < CHAINS; ++i) {
      asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                   : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3]) : "d"(ra0), "d"(ra1), "d"(rb));
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// m16n8k8 f64: A 4 regs, B 2 regs, C 4 regs: 1024 FMA / warp instr
template <int CHAINS>
__global__ void __launch_bounds__(256) k_dmma1688(double* out, int iters, double a, double b) {
  double c[CHAINS][4];
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) { c[i][0] = i; c[i][1] = -i; c[i][2] = 1; c[i][3] = 2; }
  double ra0 = a + threadIdx.x * 1e-12, ra1 = a * 0.5, ra2 = a * 0.25, ra3 = a * 0.125, rb0 = b, rb1 = b * 0.5;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < CHAINS; ++i) {
      asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                   : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3])
                   : "d"(ra0), "d"(ra1), "d"(ra2), "d"(ra3), "d"(rb0), "d"(rb1));
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// m16n8k16 f64: A 8 regs, B 4 regs, C 4 regs: 2048 FMA / warp instr
template <int CHAINS>
__global__ void __launch_bounds__(256) k_dmma16816(double* out, int iters, double a, double b) {
  double c[CHAINS][4];
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) { c[i][0] = i; c[i][1] = -i; c[i][2] = 1; c[i][3] = 2; }
  double ra[8], rb[4];
#pragma unroll
  for (int i = 0; i < 8; ++i) ra[i] = a / (i + 1) + threadIdx.x * 1e-12;
#pragma unroll
  for (int i = 0; i < 4; ++i) rb[i] = b / (i + 1);
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < CHAINS; ++i) {
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                   : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3])
                   : "d"(ra[0]), "d"(ra[1]), "d"(ra[2]), "d"(ra[3]), "d"(ra[4]), "d"(ra[5]), "d"(ra[6]), "d"(ra[7]),
                     "d"(rb[0]), "d"(rb[1]), "d"(rb[2]), "d"(rb[3]));
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// mixed: half the warps DFMA, half DMMA m8n8k4 -> do the pipes overlap?
__global__ void __launch_bounds__(256) k_mixed(double* out, int iters, double a, double b) {
  int warp = threadIdx.x >> 5;
  double s = 0;
  if (warp & 1) {
    double acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = threadIdx.x * 1e-9 + i;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fma(acc[i], a, b);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) s += acc[i];
  } else {
    double c0[8], c1[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { c0[i] = i; c1[i] = -i; }
    double ra = a + threadIdx.x * 1e-12, rb = b;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                     : "+d"(c0[i]), "+d"(c1[i]) : "d"(ra), "d"(rb));
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) s += c0[i] + c1[i];
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// exp / sqrt throughput in double
__global__ void __launch_bounds__(256) k_exp(double* out, int iters, double a) {
  double x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = -(threadIdx.x * 1e-3 + i) * a;
  double s = 0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 4; ++i) { s += exp(x[i]); x[i] -= 1e-7; }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void __launch_bounds__(256) k_sqrt(double* out, int iters, double a) {
  double x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = (threadIdx.x * 1e-3 + i + 1) * a;
  double s = 0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 4; ++i) { s += sqrt(x[i]); x[i] += 1e-7; }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// fp32 FFMA peak for reference (and for possible double-single tricks)
__global__ void __launch_bounds__(256) k_ffma(float* out, int iters, float a, float b) {
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = threadIdx.x * 1e-6f + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = fmaf(acc[i], a, b);
  }
  float s = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <typename F>
double time_ms(F launch, int reps = 5) {
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  launch(); launch();
  CK(cudaDeviceSynchronize());
  double best = 1e30;
  for (int r = 0; r < reps; ++r) {
    CK(cudaEventRecord(e0));
    launch();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    if (ms < best) best = ms;
  }
  return best;
}

int main() {
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  int sms = p.multiProcessorCount;
  printf("device %s sms %d clock %d kHz\n", p.name, sms, p.clockRate);
  double* out; CK(cudaMalloc(&out, sizeof(double) * sms * 8 * 256));
  const int iters = 1 << 15;
  for (int bps = 1; bps <= 8; bps *= 2) {
    int grid = sms * bps;
    double ms, tf;
    ms = time_ms([&] { k_dfma<8><<<grid, 256>>>(out, iters, 1.0000001, 1e-9); });
    tf = 2.0 * 8 * iters * 256.0 * grid / ms * 1e-9;
    printf("dfma<8>      blocks/SM %d  %.3f ms  %.2f TFLOP/s\n", bps, ms, tf);
    ms = time_ms([&] { k_dfma<16><<<grid, 256>>>(out, iters, 1.0000001, 1e-9); });
    tf = 2.0 * 16 * iters * 256.0 * grid / ms * 1e-9;
    printf("dfma<16>     blocks/SM %d  %.3f ms  %.2f TFLOP/s\n", bps, ms, tf);
    ms = time_ms([&] { k_dmma884<8><<<grid, 256>>>(out, iters, 1.0000001, 1e-9); });
    tf = 2.0 * 256 * 8 * iters * 8.0 * grid / ms * 1e-9;
    printf("dmma m8n8k4   blocks/SM %d  %.3f ms  %.2f TFLOP/s\n", bps, ms, tf);
    ms = time_ms([&] { k_dmma1684<8><<<grid, 256>>>(out, iters, 1.0000001, 1e-9); });
    tf = 2.0 * 512 * 8 * iters * 8.0 * grid / ms * 1e-9;
    printf("dmma m16n8k4  blocks/SM %d  %.3f ms  %.2f TFLOP/s\n", bps, ms, tf);
    ms = time_ms([&] { k_dmma1688<8><<<grid, 256>>>(out, iters, 1.0000001, 1e-9); });
    tf = 2.0 * 1024 * 8 * iters * 8.0 * grid / ms * 1e-9;
    printf("dmma m16n8k8  blocks/SM %d  %.3f ms  %.2f TFLOP/s\n", bps, ms, tf);
    ms = time_ms([&] { k_dmma16816<8><<<grid, 256>>>(out, iters, 1.0000001, 1e-9); });
    tf = 2.0 * 2048 * 8 * iters * 8.0 * grid / ms * 1e-9;
    printf("dmma m16n8k16 blocks/SM %d  %.3f ms  %.2f TFLOP/s\n", bps, ms, tf);
    ms = time_ms([&] { k_mixed<<<grid, 256>>>(out, iters, 1.0000001, 1e-9); });
    tf = (2.0 * 8 * iters * 128.0 + 2.0 * 256 * 8 * iters * 4.0) * grid / ms * 1e-9;
    printf("mixed dfma+dmma blocks/SM %d  %.3f ms  %.2f TFLOP/s (sum)\n", bps, ms, tf);
  }
  {
    int grid = sms * 8;
    double ms = time_ms([&] { k_exp<<<grid, 256>>>(out, 4096, 1.0); });
    printf("exp(double): %.3f ms  %.1f Gexp/s\n", ms, 4.0 * 4096 * 256.0 * grid / ms * 1e-6);
    ms = time_ms([&] { k_sqrt<<<grid, 256>>>(out, 4096, 1.0); });
    printf("sqrt(double): %.3f ms  %.1f Gsqrt/s\n", ms, 4.0 * 4096 * 256.0 * grid / ms * 1e-6);
    ms = time_ms([&] { k_ffma<<<grid, 256>>>((float*)out, iters, 1.0000001f, 1e-9f); });
    printf("ffma: %.3f ms  %.2f TFLOP/s\n", ms, 2.0 * 16 * iters * 256.0 * grid / ms * 1e-9);
  }
  return 0;
}
