// Device-side target models (closed registry; SURVEY.md section 7 "hard part 6").
//
// The reference takes arbitrary Python callables `neg_log_dens` / `grad_neg_log_dens`
// (systems.py:88-95); a fused GPU gradient cannot, so the benchmark targets are compiled in.
// The NumPy statements of the same models used by the oracle are in oracle/targets.py.
//
// "Pair" interface used by the Euclidean leapfrog kernels: a chain's position vector is owned
// in aligned pairs of consecutive coordinates (i, i+1), i even, by whatever threads the kernel
// layout chooses.  A gradient evaluation is
//   1. red[r] = sum over pairs of accumulate(...)         (per-chain sum reductions, NRED of them)
//   2. grad_pair(...) using the reduced values.
// Coordinates with index >= dim are phantom (value 0) and must not contribute.
#pragma once
#include "common.cuh"

namespace mb200 {

// exp(x) with a short dependent chain for the tensor-core kernel, where the exp(-v) of a group's
// chains sits on the critical path of the group's update phase: x = k ln2 + r, |r| <= ln2/2, e^r
// by its degree-13 Taylor polynomial in Estrin form (truncation 4e-18 relative; depth 4 after r
// instead of libm's 11-deep Horner chain), scaled by 2^k through the exponent bits.  Agrees with libm's exp to ~2 ulp for
// |x| < 700; exp_short_chain sends the other arguments to libm.
__device__ __forceinline__ double exp_short_chain_poly(double x) {
  const double t = fma(x, 1.4426950408889634, 6755399441055744.0);  // 2^52 + 2^51: rint in low bits
  const double k = t - 6755399441055744.0;
  double r = fma(k, -6.93147180369123816490e-01, x);   // ln2 high part
  r = fma(k, -1.90821492927058770002e-10, r);          // ln2 low part
  const double r2 = r * r, r4 = r2 * r2, r8 = r4 * r4;
  const double p0 = fma(r, 1.0, 1.0);
  const double p1 = fma(r, 1.0 / 6.0, 0.5);
  const double p2 = fma(r, 1.0 / 120.0, 1.0 / 24.0);
  const double p3 = fma(r, 1.0 / 5040.0, 1.0 / 720.0);
  const double p4 = fma(r, 1.0 / 362880.0, 1.0 / 40320.0);
  const double p5 = fma(r, 1.0 / 39916800.0, 1.0 / 3628800.0);
  const double p6 = fma(r, 1.0 / 6227020800.0, 1.0 / 479001600.0);
  const double q0 = fma(p1, r2, p0), q1 = fma(p3, r2, p2), q2 = fma(p5, r2, p4);
  const double s0 = fma(q1, r4, q0), s1 = fma(p6, r4, q2);
  const double e = fma(s1, r8, s0);
  const long long bits = __double_as_longlong(e) + ((long long)k << 52);
  return __longlong_as_double(bits);
}

// Arguments outside [-700, 700] (or non-finite) take libm's exp.  Called by all 32 lanes of a warp
// at once: the polynomial runs branch-free on every lane, and libm's exp only in a warp-uniform
// branch, taken when some lane's argument is out of range.
__device__ __forceinline__ double exp_short_chain(double x) {
  const bool in_range = fabs(x) < 700.0;
  const double e = exp_short_chain_poly(in_range ? x : 0.0);
  if (__any_sync(FULL_MASK, !in_range)) return in_range ? e : exp(x);
  return e;
}

struct StdGaussianTarget {
  static constexpr int NRED = 0;
  __device__ StdGaussianTarget(const ModelArgs&, int) {}
  __device__ __forceinline__ void accumulate(int, double, double, double*) const {}
  __device__ __forceinline__ void grad_pair(int, double q0, double q1, const double*, double& g0,
                                            double& g1) const {
    g0 = q0;
    g1 = q1;
  }
  // contribution of the pair to l(q) (summed over pairs by the caller)
  __device__ __forceinline__ double nld_pair(int, double q0, double q1, const double*) const {
    return 0.5 * (q0 * q0 + q1 * q1);
  }
  // ---- tile interface of the tensor-core kernel (leapfrog_dmma.cuh), see the note below
  static constexpr bool TILE_SUM = false, ROW_SCALAR = false, LINEAR = true, COORD0 = false;
  __device__ __forceinline__ double row_scalar(double) const { return 1.0; }
  __device__ __forceinline__ double kick_coef(double mh, double) const { return mh; }
  __device__ __forceinline__ double grad0(double q0, double, double) const { return q0; }
  __device__ __forceinline__ void kick_pair_nl(double, double, double, double&, double&) const {}
};

// Tile interface (tensor-core kernel).  The kernel owns coordinates in aligned pairs and applies
// the momentum kick p += mh * grad l(q) (mh = -step/2) with as few fp64 instructions as possible:
//   LINEAR      grad_i = rs * q_i for every coordinate (but possibly coordinate 0): the kick is
//               one FMA per coordinate with the per-chain coefficient kick_coef(mh, rs);
//               otherwise kick_pair_nl(mh, x, y, p0, p1) applies the pair's kick itself
//   ROW_SCALAR  rs = row_scalar(q[0]) is evaluated once per chain by the warp that holds
//               coordinate 0, all 32 lanes at once (one chain per lane)
//   TILE_SUM    S = sum over coordinates of q_i^2 (coordinate 0 excluded when COORD0) is
//               reduced per chain
//   COORD0      coordinate 0's gradient is grad0(q[0], S, rs) instead of the generic form

// v = q[0], x = q[1:]:  l = v^2/18 + (D-1) v/2 + exp(-v) |x|^2 / 2
struct NealFunnelTarget {
  // red[0] = |x|^2, red[1] = exp(-v).  exp(-v) is "reduced" with a single contributor (the
  // owner of coordinate 0), so it is evaluated once per chain instead of once per thread.
  static constexpr int NRED = 2;
  int dim;
  __device__ NealFunnelTarget(const ModelArgs&, int d) : dim(d) {}
  __device__ __forceinline__ void accumulate(int i, double q0, double q1, double* red) const {
    if (i == 0) {
      red[0] += q1 * q1;
      red[1] += exp(-q0);
    } else {
      red[0] += q0 * q0 + q1 * q1;
    }
  }
  __device__ __forceinline__ void grad_pair(int i, double q0, double q1, const double* red,
                                            double& g0, double& g1) const {
    const double e = red[1];
    g0 = (i == 0) ? (q0 / 9.0 + 0.5 * (dim - 1) - 0.5 * e * red[0]) : e * q0;
    g1 = e * q1;
  }
  __device__ __forceinline__ double nld_pair(int i, double q0, double, const double* red) const {
    if (i != 0) return 0.0;
    return q0 * q0 / 18.0 + 0.5 * (dim - 1) * q0 + 0.5 * red[1] * red[0];
  }
  // ---- tile interface of the tensor-core kernel: grad_i = exp(-v) x_i for i >= 1;
  // grad_0 = v/9 + (D-1)/2 - exp(-v) |x|^2 / 2, with v/9 as a multiplication by the rounded
  // reciprocal and the sum as two FMAs (the fp64 division is a ~15-deep dependent chain on the
  // critical path of a 4-warp group; differs from grad_pair's `q0 / 9.0` by at most 1 ulp)
  static constexpr bool TILE_SUM = true, ROW_SCALAR = true, LINEAR = true, COORD0 = true;
  __device__ __forceinline__ double row_scalar(double v) const { return exp_short_chain(-v); }
  __device__ __forceinline__ double kick_coef(double mh, double rs) const { return mh * rs; }
  __device__ __forceinline__ double grad0(double v, double xx, double rs) const {
    return fma(-0.5 * rs, xx, fma(v, 1.0 / 9.0, 0.5 * (dim - 1)));
  }
  __device__ __forceinline__ void kick_pair_nl(double, double, double, double&, double&) const {}
};

// pairs (x, y) = (q[2k], q[2k+1]):  l = sum x^2/8 + (y - b x^2)^2 / 2
struct BananaTarget {
  static constexpr int NRED = 0;
  double b;
  __device__ BananaTarget(const ModelArgs& m, int) : b(m.tp[0]) {}
  __device__ __forceinline__ void accumulate(int, double, double, double*) const {}
  __device__ __forceinline__ void grad_pair(int, double x, double y, const double*, double& g0,
                                            double& g1) const {
    const double r = y - b * x * x;
    g0 = x / 4.0 - 2.0 * b * x * r;
    g1 = r;
  }
  __device__ __forceinline__ double nld_pair(int, double x, double y, const double*) const {
    const double r = y - b * x * x;
    return x * x / 8.0 + 0.5 * r * r;
  }
  // ---- tile interface of the tensor-core kernel: the gradient is not linear in q
  static constexpr bool TILE_SUM = false, ROW_SCALAR = false, LINEAR = false, COORD0 = false;
  __device__ __forceinline__ double row_scalar(double) const { return 1.0; }
  __device__ __forceinline__ double kick_coef(double mh, double) const { return mh; }
  __device__ __forceinline__ double grad0(double q0, double, double) const { return q0; }
  __device__ __forceinline__ void kick_pair_nl(double mh, double x, double y, double& p0,
                                               double& p1) const {
    double g0, g1;
    grad_pair(0, x, y, nullptr, g0, g1);
    p0 = fma(mh, g0, p0);
    p1 = fma(mh, g1, p1);
  }
};

}  // namespace mb200
