// FP64 rates of the device: DMMA throughput for every f64 mma.sync shape (m8n8k4, and the
// m16n8k4 / m16n8k8 / m16n8k16 shapes added by sm_90), the latency of each shape (one warp, one
// dependent accumulator chain), and scalar DFMA throughput.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_peak fp64_peak.cu
#include <cstdio>
#include <cuda_runtime.h>

// one f64 MMA of shape M x N x K: A fragment NA doubles, B NB, C/D NC (per lane)
template <int M, int K> struct Dmma;
template <> struct Dmma<8, 4> {
  static constexpr int NA = 1, NB = 1, NC = 2;
  static __device__ __forceinline__ void mma(double (&c)[NC], const double (&a)[NA], const double (&b)[NB]) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
  }
};
template <> struct Dmma<16, 4> {
  static constexpr int NA = 2, NB = 1, NC = 4;
  static __device__ __forceinline__ void mma(double (&c)[NC], const double (&a)[NA], const double (&b)[NB]) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
  }
};
template <> struct Dmma<16, 8> {
  static constexpr int NA = 4, NB = 2, NC = 4;
  static __device__ __forceinline__ void mma(double (&c)[NC], const double (&a)[NA], const double (&b)[NB]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
  }
};
template <> struct Dmma<16, 16> {
  static constexpr int NA = 8, NB = 4, NC = 4;
  static __device__ __forceinline__ void mma(double (&c)[NC], const double (&a)[NA], const double (&b)[NB]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                   "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
  }
};

// ILP independent accumulator chains per warp; with ILP = 1 and one warp, `cyc` receives the
// cycles per instruction of the dependent chain (latency)
template <int M, int K, int ILP>
__global__ void k_dmma(double* out, int iters, long long* cyc) {
  using D = Dmma<M, K>;
  double c[ILP][D::NC], a[D::NA], b[D::NB];
  for (int i = 0; i < ILP; i++) for (int j = 0; j < D::NC; j++) c[i][j] = threadIdx.x * 1e-3 + i + j;
  for (int j = 0; j < D::NA; j++) a[j] = threadIdx.x * 1e-6 + j;
  for (int j = 0; j < D::NB; j++) b[j] = 1.0 + threadIdx.x * 1e-7 * j;
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < ILP; i++) D::mma(c[i], a, b);
  }
  double s = 0;
  for (int i = 0; i < ILP; i++) for (int j = 0; j < D::NC; j++) s += c[i][j];
  const long long t1 = clock64();
  if (cyc != nullptr && threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int ILP>
__global__ void k_dfma(double* out, int iters) {
  double c[ILP];
  for (int i = 0; i < ILP; i++) c[i] = threadIdx.x * 1e-3 + i;
  double a = 1.0 + threadIdx.x * 1e-9, b = threadIdx.x * 1e-7;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < ILP; i++) c[i] = fma(c[i], a, b);
  }
  double s = 0;
  for (int i = 0; i < ILP; i++) s += c[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <typename F> float timeit(F f) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0), cudaEventCreate(&e1);
  f();
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  f();
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms;
  cudaEventElapsedTime(&ms, e0, e1);
  return ms;
}

template <int M, int K>
static void shape(double* out, long long* cyc, int sms, double clk_hz, int iters) {
  // throughput: 8 independent chains per warp, two blocks of 4..32 warps per SM
  const double flop = 2.0 * M * 8 * K;
  for (int warps : {4, 8, 16, 32}) {
    const int thr = warps * 32, blocks = sms * (2048 / thr > 2 ? 2 : 2048 / thr);
    const int it = iters * 32 / (M * K);  // the same flop for every shape
    const float ms = timeit([&] { k_dmma<M, K, 8><<<blocks, thr>>>(out, it, nullptr); });
    if (cudaGetLastError() != cudaSuccess) {  // e.g. too many registers for the block size
      printf("dmma m%dn8k%-2d warps/blk=%2d: launch failed\n", M, K, warps);
      continue;
    }
    const double tf = (double)blocks * warps * it * 8 * flop / ms * 1e-9;
    printf("dmma m%dn8k%-2d warps/blk=%2d blocks=%d: %6.2f TF  %6.1f flop/clk/SM at %.0f MHz\n",
           M, K, warps, blocks, tf, tf * 1e12 / (sms * clk_hz), clk_hz * 1e-6);
  }
  // latency: one warp, one dependent chain
  const int it = 4096;
  k_dmma<M, K, 1><<<1, 32>>>(out, it, cyc);
  cudaDeviceSynchronize();
  long long h;
  cudaMemcpy(&h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
  printf("dmma m%dn8k%-2d dependent chain: %.1f cycles per instruction\n", M, K, (double)h / it);
}

int main() {
  int dev = 0, sms = 132, clk_khz = 1980000;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, dev);
  double* out;
  long long* cyc;
  cudaMalloc(&out, (size_t)sms * 8 * 1024 * sizeof(double));
  cudaMalloc(&cyc, sizeof(long long));
  const int iters = 20000;  // m8n8k4 instructions per chain; fewer for the larger shapes
  shape<8, 4>(out, cyc, sms, clk_khz * 1e3, iters);
  shape<16, 4>(out, cyc, sms, clk_khz * 1e3, iters);
  shape<16, 8>(out, cyc, sms, clk_khz * 1e3, iters);
  shape<16, 16>(out, cyc, sms, clk_khz * 1e3, iters);
  for (int warps : {4, 8, 16, 32}) {
    const int thr = warps * 32, blocks = sms * (2048 / thr > 2 ? 2 : 2048 / thr);
    const float ms = timeit([&] { k_dfma<8><<<blocks, thr>>>(out, iters); });
    printf("dfma      warps/blk=%2d blocks=%d: %6.2f TF\n", warps, blocks,
           (double)blocks * thr * iters * 8 * 2.0 / ms * 1e-9);
  }
  printf("status %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
