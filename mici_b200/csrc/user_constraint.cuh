// User-written constraint functions, compiled at run time by NVRTC (mici_b200/jit.py) together
// with the constrained leapfrog and projection kernels of constrained.cuh (K6).
//
// Besides neg_log_dens and grad_neg_log_dens (user_target.cuh), the user writes
//
//   __device__ void constr(const mb200::Chain& c, double* out);          // out[k] = c_k(q), k < N_CONSTR
//   __device__ void jacob_constr(const mb200::Chain& c, double* J);      // J[k * dim + i] = dc_k / dq_i
//
// and, for a density with respect to the Lebesgue measure (dens_wrt_hausdorff=False) or a
// GaussianDenseConstrainedEuclideanMetricSystem, the constraint's matrix-Hessian product
//
//   __device__ void mhp_constr(const mb200::Chain& c, const double* m, double* out);
//                                          // out[j] = sum_{k,i} m[k * dim + i] d2c_k / dq_i dq_j
//
// mb200::N_CONSTR (1 .. 8) is the number of constraints; the host defines it when it compiles
// (MB200_USER_N_CONSTR), and MB200_USER_MHP_CONSTR when the source defines mhp_constr, so a model
// used only with the Hausdorff density need not write it.
//
// The rules of user_target.cuh apply to every function: all 32 lanes call it together and reach
// every c.sum() together; every output entry is written by at least one lane, and lanes that write
// the same entry write the same value; no __syncthreads(); compiled with -fmad=false.  The
// constraint Jacobian is whole rows of dim entries: entries beyond a constraint's support must be
// written too (as 0).
#pragma once
#include "user_target.cuh"
#include "constrained.cuh"

#ifndef MB200_USER_N_CONSTR
#error "MB200_USER_N_CONSTR (the number of constraints) must be defined"
#endif

namespace mb200 {
constexpr int N_CONSTR = MB200_USER_N_CONSTR;
static_assert(N_CONSTR >= 1 && N_CONSTR <= 8, "N_CONSTR must be in [1, 8]");
}  // namespace mb200

__device__ void constr(const mb200::Chain& c, double* out);
__device__ void jacob_constr(const mb200::Chain& c, double* J);
#ifdef MB200_USER_MHP_CONSTR
__device__ void mhp_constr(const mb200::Chain& c, const double* m, double* out);
#endif

namespace mb200 {

// K6's target interface (constrained.cuh) over the user functions.  Each call writes the chain's
// pair-layout registers (i = 2 lane + 64 (e >> 1) + (e & 1)) to the warp's staging area, calls the
// user function between two __syncwarp()s and reads the results back into registers.  Staging
// area of a warp with NV = 2 KP values per lane: q [64 KP], NC rows of dim entries (J, or the
// operand m of mhp) [NC * 64 KP], one output vector [64 KP].
struct UserConstrainedTarget {
  static constexpr int NC = N_CONSTR;
  static constexpr bool STAGED = true;
  UserTarget base;  // params and aux
  double* stage;

  __device__ UserConstrainedTarget(const ModelArgs& m, int dim, double* stage_area)
      : base(m, dim), stage(stage_area) {}

  template <int NV>
  __device__ __forceinline__ double* rows() const {
    return stage + 32 * NV;
  }
  template <int NV>
  __device__ __forceinline__ double* out() const {
    return stage + 32 * NV * (NC + 1);
  }
  // writes q (the area is read only inside user calls, which end at a __syncwarp())
  template <int NV>
  __device__ __forceinline__ Chain stage_q(int lane, int dim, const double (&q)[NV]) const {
#pragma unroll
    for (int e = 0; e < NV; ++e) stage[2 * lane + 64 * (e >> 1) + (e & 1)] = q[e];
    __syncwarp();
    return base.chain(stage, dim, lane);
  }
  template <int NV>
  __device__ __forceinline__ void read(int lane, int dim, const double* src,
                                       double (&v)[NV]) const {
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
      v[e] = (i < dim) ? src[i] : 0.0;
    }
  }

  template <int NV>
  __device__ __forceinline__ void grad(int lane, int dim, const double (&q)[NV],
                                       double (&g)[NV]) const {
    const Chain c = stage_q(lane, dim, q);
    grad_neg_log_dens(c, out<NV>());
    __syncwarp();
    read(lane, dim, out<NV>(), g);
  }

  template <int NV>
  __device__ __forceinline__ double nld(int lane, int dim, const double (&q)[NV]) const {
    const Chain c = stage_q(lane, dim, q);
    const double v = neg_log_dens(c);
    __syncwarp();
    return v;
  }

  template <int NV>
  __device__ __forceinline__ void constr_jacob(int lane, int dim, const double (&q)[NV],
                                               double (&c)[NC], double (&J)[NC][NV]) const {
    const Chain ch = stage_q(lane, dim, q);
    constr(ch, out<NV>());
    jacob_constr(ch, rows<NV>());
    __syncwarp();
#pragma unroll
    for (int a = 0; a < NC; ++a) {
      c[a] = out<NV>()[a];
      read(lane, dim, rows<NV>() + a * dim, J[a]);
    }
  }

  template <int NV>
  __device__ __forceinline__ void mhp(int lane, int dim, const double (&q)[NV],
                                      const double (&m)[NC][NV], double (&o)[NV]) const {
#ifdef MB200_USER_MHP_CONSTR
    __syncwarp();  // the rows area may still be read from the previous call
#pragma unroll
    for (int a = 0; a < NC; ++a)
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
        if (i < dim) rows<NV>()[a * dim + i] = m[a][e];
      }
    const Chain c = stage_q(lane, dim, q);
    mhp_constr(c, rows<NV>(), out<NV>());
    __syncwarp();
    read(lane, dim, out<NV>(), o);
#else
    // never reached: the host refuses the Lebesgue density and the Gaussian system for an image
    // built without mhp_constr
#pragma unroll
    for (int e = 0; e < NV; ++e) o[e] = 0.0;
#endif
  }
};

}  // namespace mb200
