// User-written target models, compiled at run time by NVRTC (mici_b200/jit.py) together with the
// general-dimension Euclidean kernels of leapfrog_generic.cuh.
//
// The user writes two device functions:
//
//   __device__ double neg_log_dens(const mb200::Chain& c);               // returns l(q)
//   __device__ void grad_neg_log_dens(const mb200::Chain& c, double* g);  // writes dl/dq to g[0, dim)
//
// Rules:
//  - All 32 lanes of the chain's warp call each function together, and must reach every c.sum()
//    together.
//  - Every g[i], i < dim, is written by at least one lane; lanes that write the same entry write
//    the same value.
//  - neg_log_dens returns the same value on every lane.
//  - The kernel synchronises the warp before and after each call: never synchronise beyond the
//    warp (no __syncthreads()).
// A serial loop run redundantly on every lane is legal, just slow; the intended style is
// `for (int i = c.lane; i < c.dim; i += 32)` with c.sum() for reductions.  The code is compiled
// with -fmad=false, as the library is, so products and sums round as they do in NumPy; write
// fma() where a fused multiply-add is wanted.
#pragma once
#include "leapfrog_generic.cuh"

namespace mb200 {

// What a user function sees of one chain.
struct Chain {
  int dim;
  int lane;                           // 0 .. 31
  const double* q;                    // the whole position vector [dim], shared memory
  double params[MB200_MAX_PARAMS];    // mb200_model.target_params
  const double* aux;                  // mb200_model.target_aux (device array) or NULL
  // warp all-reduce in a fixed butterfly order: every lane gets the same value
  __device__ __forceinline__ double sum(double x) const { return warp_sum(x); }
};

}  // namespace mb200

__device__ double neg_log_dens(const mb200::Chain& c);
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g);

namespace mb200 {

struct UserTarget {
  static constexpr bool WHOLE_VECTOR = true;
  static constexpr int NRED = 0;
  double tp[MB200_MAX_PARAMS];
  const double* taux;
  __device__ UserTarget(const ModelArgs& m, int) : taux(m.taux) {
#pragma unroll
    for (int i = 0; i < MB200_MAX_PARAMS; ++i) tp[i] = m.tp[i];
  }
  __device__ __forceinline__ Chain chain(const double* q, int dim, int lane) const {
    Chain c;
    c.dim = dim;
    c.lane = lane;
    c.q = q;
#pragma unroll
    for (int i = 0; i < MB200_MAX_PARAMS; ++i) c.params[i] = tp[i];
    c.aux = taux;
    return c;
  }
  __device__ __forceinline__ void grad(const double* q, int dim, int lane, double* g) const {
    grad_neg_log_dens(chain(q, dim, lane), g);
  }
  __device__ __forceinline__ double nld(const double* q, int dim, int lane) const {
    return neg_log_dens(chain(q, dim, lane));
  }
};

}  // namespace mb200
