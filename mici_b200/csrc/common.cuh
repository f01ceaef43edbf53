// Shared device helpers for libmici_b200 (sm_90a).  Also compiled by NVRTC for user-written
// targets (csrc/user_target.cuh): NVRTC has no system headers, but declares the vector types
// and device math functions itself.
#pragma once
#ifndef __CUDACC_RTC__
#include <cuda_runtime.h>
#include <stdint.h>
#endif

#include "../../include/mici_b200.h"

namespace mb200 {

constexpr unsigned FULL_MASK = 0xffffffffu;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}

__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(FULL_MASK, v, o));
  return v;
}

// max that propagates NaN (numpy's abs(x).max() returns NaN if any entry is NaN;
// solvers.py:25-27 + the `np.isnan(error)` checks at :80, :449)
__device__ __forceinline__ double nanmax(double a, double b) {
  return (a != a) ? a : ((b != b) ? b : fmax(a, b));
}

__device__ __forceinline__ double warp_nanmax(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = nanmax(v, __shfl_xor_sync(FULL_MASK, v, o));
  return v;
}

// Model parameters passed by value in the kernel argument buffer.
struct ModelArgs {
  int target_id;
  double tp[MB200_MAX_PARAMS];
  const double* taux;
  int rmetric_id;
  double mp[MB200_MAX_PARAMS];
  const double* maux;
  // optional per-chain overrides of the scalar step_size / n_steps arguments of the implicit and
  // constrained kernels (device arrays [n_chains] or NULL), passed in by their entry points
  const double* step_sizes;
  const int32_t* n_steps_pc;
  // per-CTA global scratch of the global-workspace dense metric policy (dense_global.cuh):
  // CTA b owns [workspace + b * ws_stride, + ws_stride) doubles
  double* workspace;
  size_t ws_stride;
  // optional call counters [n_chains][MB200_N_COUNTERS] (mb200_set_call_counters) or NULL
  int32_t* counters;
};

// Splitting schedule of a symmetric composition integrator (integrators.py:176-378): flow i is
// h1_flow (momentum kick) or h2_flow (position drift) over coef[i] * dt.  Leapfrog is
// {0.5 kick, 1 drift, 0.5 kick}.
constexpr int MB200_MAX_FLOWS = 16;
struct FlowSchedule {
  int n;
  unsigned drift_mask;  // bit i set: flow i is an h2_flow (drift), else an h1_flow (kick)
  double coef[MB200_MAX_FLOWS];
  // optional per-chain overrides (device arrays [n_chains]; NULL = the scalar arguments):
  // step sizes (one adapter state per chain during warm-up, adapters.py:262-283, 373) and
  // trajectory lengths (MetropolisRandomIntegrationTransition, transitions.py:355-412)
  const double* step_sizes;
  const int32_t* n_steps;
  // GaussianEuclideanMetricSystem (systems.py:369-474): h2 = q.q/2 + p.M^-1 p/2 and the drift is
  // the exact rotation of (q, p).  rot: metric diagonal [dim] (diagonal metric) or, for a dense
  // metric, per drift flow the three symmetric matrices [U cos U^T | U (sin w) U^T |
  // -U (sin / w) U^T] built on the host from eigh(M) for |dt| = coef * step_size.
  int gaussian;
  const double* rot;
};

}  // namespace mb200
