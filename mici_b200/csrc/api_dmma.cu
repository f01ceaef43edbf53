// libmici_b200.so -- C-ABI entry points (include/mici_b200.h): dispatch of the FP64 tensor-core leapfrog kernel K1.
// Host-side argument checking and kernel dispatch only; all arithmetic is in the .cuh kernels.
#include "api_common.cuh"
#include "leapfrog_dmma.cuh"

// leapfrog_dmma.cuh defines mb200::leapfrog_dmma_dispatch (declared in api_common.cuh)

namespace mb200 {

// One element per thread in whole warps: exp_short_chain votes over all 32 lanes, so lanes past
// n evaluate exp(0) and do not store.
__global__ void exp_short_chain_selftest_kernel(const double* __restrict__ x, double* __restrict__ y,
                                                int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const double v = exp_short_chain(i < n ? x[i] : 0.0);
  if (i < n) y[i] = v;
}

}  // namespace mb200

using namespace mb200;

extern "C" {

int mb200_selftest_exp_short_chain(const double* x, double* y, int64_t n, void* stream) {
  if (n < 0) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (n == 0) return 0;
  if (!x || !y) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  const DeviceScope device_scope(x);
  constexpr int threads = 256;
  const int64_t blocks = (n + threads - 1) / threads;
  if (blocks > 0x7fffffff) return fail(MB200_ERR_INVALID_ARG, "n too large");
  exp_short_chain_selftest_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(x, y, n);
  return check_launch("exp_short_chain_selftest_kernel");
}

}  // extern "C"
