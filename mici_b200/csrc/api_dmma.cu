// libmici_b200.so -- C-ABI entry points (include/mici_b200.h): launch of the FP64 tensor-core leapfrog kernel K1.
// Host-side argument checking and kernel dispatch only; all arithmetic is in the .cuh kernels.
#include "api_common.cuh"
#include "leapfrog_dmma.cuh"

namespace mb200 {

// One launch of K1 with DP padded columns, PC: per-chain step sizes.  One CTA per SM; a CTA takes
// up to 8 row tiles of 8 chains per pass, fewer for small batches so that the tiles spread over
// all SMs.
template <class Target, int DP, bool PC>
static int k1_run(const EuclidArgs& a) {
  const int sms = num_sms();
  const int64_t total_tiles = (a.n + 7) / 8;
  int64_t tpc = (total_tiles + sms - 1) / sms;  // tiles per CTA and pass
  if (tpc > DMMA_TILES_PER_CTA) tpc = DMMA_TILES_PER_CTA;
  auto al16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  const int even = (a.dim & 1) == 0;
  const int vec2 = even && al16(a.q_in) && al16(a.p_in) && al16(a.q_out) && al16(a.p_out);
  const int tma_rows = even && al16(a.minv);  // persistent: CTAs loop over passes of tpc tiles
  return eu_launch(leapfrog_dmma_kernel<Target, DP, PC>, "leapfrog_dmma_kernel",
                   (total_tiles + tpc - 1) / tpc, 1, DMMA_THREADS, sizeof(DmmaSmem<DP>), a.st,
                   a.q_in, a.p_in, a.q_out, a.p_out, a.dir, a.sched.step_sizes, a.n, a.dim,
                   PC ? 1.0 : a.eps, a.n_steps, a.minv, a.m, a.h_out, a.status, a.n_done, (int)tpc,
                   vec2, tma_rows);
}

// Called where k1_serves(): the tile width DP is the dimension rounded up to a multiple of 32
template <class Target>
int k1_launch(const EuclidArgs& a) {
  auto run = [&](auto pc) {
    constexpr bool PC = decltype(pc)::value;
    if (a.dim <= 32) return k1_run<Target, 32, PC>(a);
    if (a.dim <= 64) return k1_run<Target, 64, PC>(a);
    if (a.dim <= 96) return k1_run<Target, 96, PC>(a);
    return k1_run<Target, 128, PC>(a);
  };
  return a.sched.step_sizes != nullptr ? run(std::true_type()) : run(std::false_type());
}
template int k1_launch<StdGaussianTarget>(const EuclidArgs&);
template int k1_launch<NealFunnelTarget>(const EuclidArgs&);
template int k1_launch<BananaTarget>(const EuclidArgs&);

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
