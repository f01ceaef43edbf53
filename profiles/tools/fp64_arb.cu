// Microbenchmark: arbitration of the FP64 pipe between a warp issuing scalar FP64 instructions and
// 0..3 other warps of the same SM sub-partition streaming DMMA.8x8x4 (or, with BIG, DMMA.16x8x16:
// the same flop in 8x fewer, longer instructions).  One CTA per SM, 16 warps; warps 0-3 (one per
// sub-partition) run the scalar stream and time it with clock64; warps of groups 1..NDW run DMMA
// streams for longer than that; the remaining warps exit.
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

__device__ __forceinline__ void dmma16816(double& c0, double& c1, double& c2, double& c3, double a,
                                          double b) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, "
      "{%4,%4,%4,%4,%4,%4,%4,%4}, {%5,%5,%5,%5}, {%0,%1,%2,%3};\n"
      : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
      : "d"(a), "d"(b));
}

// MODE 0: independent DFMA x8; 1: dependent DFMA chain; 2: the scalar warp interleaves
// 1 DMMA.8x8x4 per KI scalar instructions (mixed stream)
template <int MODE, int KI, bool BIG>
__global__ void __launch_bounds__(512, 1) k_arb(double* out, int ndw, int n_scalar, long long* cyc) {
  const int grp = threadIdx.x >> 7;
  double c0[8], c1[8], s[8];
  for (int i = 0; i < 8; i++) c0[i] = threadIdx.x * 1e-3 + i, c1[i] = i * 0.5, s[i] = 1.0 + i;
  double a = threadIdx.x * 1e-6, b = 1.0 + threadIdx.x * 1e-7;
  const double m = 1.0 + 1e-9, d = 1e-7;
  if (grp == 0) {
    // let the DMMA warps get going first
    for (int i = 0; i < 64; i++) dmma884(c0[i & 7], c1[i & 7], a, b);
    const long long t0 = clock64();
    for (int it = 0; it < n_scalar / 8; ++it) {
      if (MODE == 0) {
#pragma unroll
        for (int i = 0; i < 8; i++) s[i] = fma(s[i], m, d);
      } else if (MODE == 1) {
#pragma unroll
        for (int i = 0; i < 8; i++) s[0] = fma(s[0], m, d);
      } else {
#pragma unroll
        for (int i = 0; i < 8; i++) {
          s[i] = fma(s[i], m, d);
          if ((i % KI) == KI - 1) dmma884(c0[i & 7], c1[i & 7], a, b);
        }
      }
    }
    const long long t1 = clock64();
    if ((threadIdx.x & 31) == 0 && blockIdx.x == 0) cyc[threadIdx.x >> 5] = t1 - t0;
  } else if (grp <= ndw) {
    if (BIG) {
      for (int it = 0; it < n_scalar * 6 / 4; ++it) {  // the flop of the DMMA.8x8x4 stream
#pragma unroll
        for (int i = 0; i < 4; i++) dmma16816(c0[2 * i], c1[2 * i], c0[2 * i + 1], c1[2 * i + 1], a, b);
      }
    } else {
      for (int it = 0; it < n_scalar * 6; ++it) {
#pragma unroll
        for (int i = 0; i < 8; i++) dmma884(c0[i], c1[i], a, b);
      }
    }
  }
  double r = 0;
  for (int i = 0; i < 8; i++) r += c0[i] + c1[i] + s[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = r;
}

template <int MODE, int KI, bool BIG>
static void run(const char* name, double* out, long long* cyc) {
  const int n_scalar = 4096;
  printf("%-44s", name);
  for (int ndw = 0; ndw <= 3; ++ndw) {
    k_arb<MODE, KI, BIG><<<132, 512>>>(out, ndw, n_scalar, cyc);
    cudaDeviceSynchronize();
    long long h[4];
    cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    printf("  %d DMMA warps: %7.2f", ndw, (double)h[0] / n_scalar);
  }
  printf("   cycles per scalar instr\n");
}

int main() {
  double* out;
  long long* cyc;
  cudaMalloc(&out, 132 * 512 * sizeof(double));
  cudaMalloc(&cyc, 16 * sizeof(long long));
  printf("DMMA warps stream DMMA.8x8x4:\n");
  run<0, 1, false>("independent DFMA stream", out, cyc);
  run<1, 1, false>("dependent DFMA chain", out, cyc);
  run<2, 1, false>("1 DMMA per 1 DFMA (mixed stream)", out, cyc);
  run<2, 2, false>("1 DMMA per 2 DFMA", out, cyc);
  run<2, 4, false>("1 DMMA per 4 DFMA", out, cyc);
  run<2, 8, false>("1 DMMA per 8 DFMA", out, cyc);
  printf("DMMA warps stream DMMA.16x8x16:\n");
  run<0, 1, true>("independent DFMA stream", out, cyc);
  run<1, 1, true>("dependent DFMA chain", out, cyc);
  printf("status %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
