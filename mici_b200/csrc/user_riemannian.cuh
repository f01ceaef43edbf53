// User-written targets and metrics on the diagonal and scalar Riemannian systems, compiled at run
// time by NVRTC (mici_b200/jit.py) together with the implicit-integrator, velocity and
// momentum-refresh kernels of riemannian.cuh (K9).
//
// Besides neg_log_dens and grad_neg_log_dens (user_target.cuh), the user writes one pair:
//
//   // DiagonalRiemannianMetricSystem: M(q) = diag(d(q))
//   __device__ void metric_diagonal(const mb200::Chain& c, double* d);           // d[i] = d_i(q)
//   __device__ void vjp_metric_diagonal(const mb200::Chain& c, const double* w, double* out);
//                                                          // out[j] = sum_i w[i] dd_i / dq_j
//   // ScalarRiemannianMetricSystem: M(q) = s(q) I
//   __device__ double metric_scalar(const mb200::Chain& c);        // s(q), the same on every lane
//   __device__ void vjp_metric_scalar(const mb200::Chain& c, double w, double* out);
//                                                          // out[j] = w ds / dq_j
//
// The rules of user_target.cuh apply to every function.  Inside the metric functions c.params
// and c.aux are the metric's own (mb200_model.rmetric_params / rmetric_aux); c.q is the position.
// Each chain runs on one 32-thread CTA, a single warp, with its vectors in shared memory; every
// call sits between two __syncwarp()s, so lanes may read entries other lanes wrote in an earlier
// call or in the same call before a c.sum().  A d_i or s that is not positive (or NaN) fails as
// with the registry metrics: LinAlgError outside a fixed-point solve, ConvergenceError inside one.
//
// The host defines MB200_USER_DIAGONAL_METRIC or MB200_USER_SCALAR_METRIC and puts
// MB200_USER_METRIC_FUNCTIONS after the user sources: that binds the pair to the policies, so a
// missing function is reported at the end of the user's own source.
#pragma once
#include "user_target.cuh"
#include "riemannian.cuh"

#if defined(MB200_USER_DIAGONAL_METRIC) == defined(MB200_USER_SCALAR_METRIC)
#error "define exactly one of MB200_USER_DIAGONAL_METRIC and MB200_USER_SCALAR_METRIC"
#endif

namespace mb200 {

static_assert(RM_COMPACT_THREADS == 32, "the user contract is per warp: one chain per 32-thread CTA");

// Riemannian block interface (riemannian.cuh) over the user's target functions: l and grad l
// only, no Hessian
struct UserRTarget {
  static constexpr bool DENSE_MTP = false;
  static constexpr bool HAS_HESSIAN = false;
  static constexpr int NEED = 1;
  UserTarget u;  // target_params and target_aux
  int dim;
  __device__ UserRTarget(const ModelArgs& m, int d) : u(m, d), dim(d) {}
  __device__ void attach(double*) const {}
  __device__ double nld(const Blk& k, const double* q) const {
    __syncwarp();
    const double v = u.nld(q, dim, k.lane);
    __syncwarp();
    return v;
  }
  __device__ void grad(const Blk& k, const double* q, double* g) const {
    __syncwarp();
    u.grad(q, dim, k.lane, g);
    __syncwarp();
  }
  __device__ void hess(const Blk&, const double*, double*, int) const {}
  __device__ __forceinline__ int need_col(int, int) const { return -1; }
  __device__ void mtp_entries(const Blk&, const double*, const double*, double*) const {}
};
static_assert(UserRTarget::DENSE_MTP == UserRTargetTraits::DENSE_MTP, "host launch traits");

// The metric's view of a chain: rmetric_params and rmetric_aux
struct UserMetricArgs {
  double mp[MB200_MAX_PARAMS];
  const double* maux;
  int dim;
  __device__ UserMetricArgs(const ModelArgs& m, int d) : maux(m.maux), dim(d) {
#pragma unroll
    for (int i = 0; i < MB200_MAX_PARAMS; ++i) mp[i] = m.mp[i];
  }
  __device__ __forceinline__ Chain chain(const Blk& k, const double* q) const {
    Chain c;
    c.dim = dim;
    c.lane = k.lane;
    c.q = q;
#pragma unroll
    for (int i = 0; i < MB200_MAX_PARAMS; ++i) c.params[i] = mp[i];
    c.aux = maux;
    return c;
  }
};

// Bound by MB200_USER_METRIC_FUNCTIONS after the user sources: static diag / vjp (diagonal) or
// scalar / vjp (scalar) calling the user's pair
struct UserMetricFunctions;

// DiagonalMetric's model interface over metric_diagonal / vjp_metric_diagonal
template <class F = UserMetricFunctions>
struct UserDiagModel {
  UserMetricArgs a;
  __device__ UserDiagModel(const ModelArgs& m, int d) : a(m, d) {}
  __device__ void diag(const Blk& k, const double* q, double* d) const {
    __syncwarp();
    F::diag(a.chain(k, q), d);
    __syncwarp();
  }
  __device__ void vjp(const Blk& k, const double* q, const double* wv, double* out) const {
    __syncwarp();
    F::vjp(a.chain(k, q), wv, out);
    __syncwarp();
  }
};

// ScalarMetric's model interface over metric_scalar / vjp_metric_scalar
template <class F = UserMetricFunctions>
struct UserScalarModel {
  UserMetricArgs a;
  __device__ UserScalarModel(const ModelArgs& m, int d) : a(m, d) {}
  __device__ double scalar(const Blk& k, int, const double* q) const {
    __syncwarp();
    const double s = F::scalar(a.chain(k, q));
    __syncwarp();
    return s;
  }
  __device__ void vjp(const Blk& k, int, const double* q, double g, double* out) const {
    __syncwarp();
    F::vjp(a.chain(k, q), g, out);
    __syncwarp();
  }
};

template <class Target>
using UserDiagonalMetric = DiagonalMetric<Target, UserDiagModel<>>;
template <class Target>
using UserScalarMetric = ScalarMetric<Target, UserScalarModel<>>;

template <class P>
constexpr bool user_policy_traits_match() {
  using H = UserRPolicyTraits<UserRTarget>;
  return P::SOFTABS == H::SOFTABS && P::COMPACT == H::COMPACT && P::N_MATS == H::N_MATS &&
         P::MIN_BLOCKS == H::MIN_BLOCKS && P::THREADS == H::THREADS;
}
static_assert(user_policy_traits_match<DiagonalMetric<UserRTarget, QuadraticDiagModel>>() &&
                  user_policy_traits_match<ScalarMetric<UserRTarget, QuadraticScalarModel>>(),
              "host launch traits");

}  // namespace mb200

#ifdef MB200_USER_DIAGONAL_METRIC
#define MB200_USER_METRIC_FUNCTIONS                                                             \
  struct mb200::UserMetricFunctions {                                                           \
    static __device__ __forceinline__ void diag(const mb200::Chain& c, double* d) {             \
      metric_diagonal(c, d);                                                                    \
    }                                                                                           \
    static __device__ __forceinline__ void vjp(const mb200::Chain& c, const double* w,          \
                                               double* out) {                                   \
      vjp_metric_diagonal(c, w, out);                                                           \
    }                                                                                           \
  };
#else
#define MB200_USER_METRIC_FUNCTIONS                                                             \
  struct mb200::UserMetricFunctions {                                                           \
    static __device__ __forceinline__ double scalar(const mb200::Chain& c) {                    \
      return metric_scalar(c);                                                                  \
    }                                                                                           \
    static __device__ __forceinline__ void vjp(const mb200::Chain& c, double w, double* out) {  \
      vjp_metric_scalar(c, w, out);                                                             \
    }                                                                                           \
  };
#endif
