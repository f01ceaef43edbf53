// User-written targets and metrics on the diagonal, scalar, dense and Cholesky-factored Riemannian
// systems, compiled at run time by NVRTC (mici_b200/jit.py) together with the implicit-integrator,
// velocity and momentum-refresh kernels of riemannian.cuh (K9, K10, K14) or, for a dense metric, of
// the global-workspace dense policy of dense_global.cuh (K2g, K13).
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
//   // DenseRiemannianMetricSystem: M(q) dense, positive definite
//   __device__ void metric_dense(const mb200::CtaChain& c, double* M, int ld);
//                                          // M[i * ld + j] = M_ij(q) for all 0 <= i, j < dim
//   __device__ void vjp_metric_dense(const mb200::CtaChain& c, const double* V, int ld,
//                                    double* out);
//           // out[k] = sum_ij V[i * ld + j] dM_ij / dq_k, V symmetric, every out[k], k < dim
//   // CholeskyFactoredRiemannianMetricSystem: M(q) = L(q) L(q)^T, L lower triangular
//   __device__ void metric_chol(const mb200::CtaChain& c, double* L, int ld);
//                  // L[i * ld + j] = L_ij(q) for 0 <= j <= i < dim; the upper triangle is never read
//   __device__ void vjp_metric_chol(const mb200::CtaChain& c, const double* V, int ld,
//                                   double* out);
//           // out[k] = sum_{j <= i} V[i * ld + j] dL_ij / dq_k, every out[k], k < dim; V is lower
//           // triangular and its entries above the diagonal must not be read
//
// The rules of user_target.cuh apply to every function.  Inside the metric functions c.params
// and c.aux are the metric's own (mb200_model.rmetric_params / rmetric_aux); c.q is the position.
// Each chain runs on one 32-thread CTA, a single warp, with its vectors in shared memory; every
// call sits between two __syncwarp()s, so lanes may read entries other lanes wrote in an earlier
// call or in the same call before a c.sum().  A d_i or s that is not positive (or NaN) fails as
// with the registry metrics: LinAlgError outside a fixed-point solve, ConvergenceError inside one.
//
// The dense metric runs on the global-workspace dense policy: one 256-thread CTA per chain, the
// D x D matrices in a per-CTA global workspace.  Its two functions are called by the WHOLE CTA
// and see the chain through mb200::CtaChain: c.lane in [0, c.n_lanes), c.n_lanes == 256, and
// c.sum(), a CTA all-reduce in a fixed order that every thread must reach.  Each call sits
// between two __syncthreads(); M and V are in global memory (L2), q and out in shared memory.
// The intended style is `for (int i = c.lane; i < c.dim; i += c.n_lanes)` over rows, or over the
// D^2 entries.  The target keeps its warp contract: warp 0 alone calls neg_log_dens /
// grad_neg_log_dens while the other warps wait, so one CudaTarget source runs on every system.
// As in the reference (DenseRiemannianMetricSystem, numpy.linalg.cholesky):
//  - every entry of the dim x dim matrix, both triangles, must be finite; one that is not is a
//    LinAlgError;
//  - only the lower triangle is factored (the upper one is never read);
//  - a pivot that is not positive is a LinAlgError;
//  - inside a fixed-point solve both failures are a ConvergenceError.
// The policy, not the user, writes the identity padding of the rows and columns from dim to the
// padded dimension (a multiple of 32) after every fill.  dim <= 576.
//
// The Cholesky-factored metric runs on the triangular-factored policy CholeskyFactoredMetric (K10):
// one 256-thread CTA (MB200_RM_CHOL_THREADS) per chain, with the same CtaChain view and the same
// rules as the dense metric: both functions are called by the whole CTA, each call between two
// __syncthreads(), and the target keeps its warp contract through warp 0.  L and V are [dim x
// (dim + 1)] matrices in shared memory up to D = 112 and in a per-CTA global workspace beyond;
// q and out are in shared memory.  The policy forms V itself, lower triangle only: diag(2 / L_ii)
// for the gradient of log|M| and tril(-2 (M^-1 p)(L^-1 p)^T) for that of the quadratic form, and
// calls vjp_metric_chol once for each.  As in the reference (TriangularFactoredPositiveDefinite-
// Matrix): a non-finite entry of the lower triangle is a LinAlgError (the policy checks the
// lower triangle after every fill), a ConvergenceError inside a fixed-point solve; a negative
// diagonal entry is legal; a zero one fails only where L is solved with.  dim <= 1016, where the
// per-chain vectors alone fill the shared memory.
//
// The host defines exactly one of MB200_USER_DIAGONAL_METRIC, MB200_USER_SCALAR_METRIC,
// MB200_USER_DENSE_METRIC and MB200_USER_CHOLESKY_METRIC and puts MB200_USER_METRIC_FUNCTIONS
// after the user sources: that binds the pair to the policies, so a missing function is reported
// at the end of the user's own source.
#pragma once
#include "user_target.cuh"
#include "riemannian.cuh"

#if defined(MB200_USER_DIAGONAL_METRIC) + defined(MB200_USER_SCALAR_METRIC) + \
        defined(MB200_USER_DENSE_METRIC) + defined(MB200_USER_CHOLESKY_METRIC) != 1
#error "define exactly one of MB200_USER_DIAGONAL_METRIC, MB200_USER_SCALAR_METRIC, MB200_USER_DENSE_METRIC and MB200_USER_CHOLESKY_METRIC"
#endif

#ifdef MB200_USER_DENSE_METRIC
#include "dense_global.cuh"
#endif

namespace mb200 {

static_assert(RM_COMPACT_THREADS == 32, "the user contract is per warp: one chain per 32-thread CTA");

// Riemannian block interface (riemannian.cuh) over the user's target functions: l and grad l
// only, no Hessian
struct UserRTarget : UserRTargetTraits {
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

// What a dense or Cholesky-factored metric function sees of one chain: the whole CTA
struct CtaChain {
  int dim;
  int lane;                         // 0 .. n_lanes - 1: the thread of the CTA
  int n_lanes;                      // 256
  const double* q;                  // the whole position vector [dim], shared memory
  double params[MB200_MAX_PARAMS];  // mb200_model.rmetric_params
  const double* aux;                // mb200_model.rmetric_aux (device array) or NULL
  Blk blk;
  // CTA all-reduce in a fixed order (warp butterflies, then the warp totals in order): every
  // thread gets the same value
  __device__ __forceinline__ double sum(double x) const { return block_sum(blk, x); }
};

// The target's warp contract on a 256-thread CTA (the dense and Cholesky-factored policies):
// warp 0 calls the user functions, the other warps wait at the barrier; the value of l reaches
// every thread through shared memory (the reduction scratch's slot 32, which block_sum /
// block_nanmax / block_prefix_suffix never use)
struct UserRTargetCta : UserRTarget {
  __device__ UserRTargetCta(const ModelArgs& m, int d) : UserRTarget(m, d) {}
  __device__ double nld(const Blk& k, const double* q) const {
    __syncthreads();
    if (k.warp == 0) {
      const double v = u.nld(q, dim, k.lane);
      if (k.lane == 0) k.red[32] = v;
    }
    __syncthreads();
    return k.red[32];
  }
  __device__ void grad(const Blk& k, const double* q, double* g) const {
    __syncthreads();
    if (k.warp == 0) u.grad(q, dim, k.lane, g);
    __syncthreads();
  }
};

// The CTA-wide metric's view of a chain: rmetric_params and rmetric_aux, read from the kernel's
// ModelArgs parameter at each call rather than held in registers across the integrator
struct UserCtaMetricArgs {
  const ModelArgs& m;
  int dim;
  __device__ UserCtaMetricArgs(const ModelArgs& mm, int d) : m(mm), dim(d) {}
  __device__ __forceinline__ CtaChain chain(const Blk& k, const double* q) const {
    CtaChain c;
    c.dim = dim;
    c.lane = k.tid;
    c.n_lanes = k.nthr;
    c.q = q;
#pragma unroll
    for (int i = 0; i < MB200_MAX_PARAMS; ++i) c.params[i] = m.mp[i];
    c.aux = m.maux;
    c.blk = k;
    return c;
  }
};

// CholeskyFactoredMetric's model interface over metric_chol / vjp_metric_chol: fill, then the
// policy's own finiteness check of the lower triangle (the user function returns nothing), and
// the VJP of a lower-triangular V (DENSE_VJP: the policy forms V in w.M2)
template <class F = UserMetricFunctions>
struct UserCholModel : UserCtaMetricArgs, UserCholModelTraits {
  __device__ UserCholModel(const ModelArgs& m, int d) : UserCtaMetricArgs(m, d) {}
  // true iff every entry of the lower triangle is finite
  __device__ bool fill(const Blk& k, const double* q, double* L, int ld) const {
    __syncthreads();
    F::chol(chain(k, q), L, ld);
    __syncthreads();
    bool bad = false;
    for (int i = k.warp; i < dim; i += k.nwarp)
      for (int j = k.lane; j <= i; j += 32)
        if (!isfinite(L[i * ld + j])) bad = true;
    return !bad;
  }
  __device__ void vjp_tril(const Blk& k, const double* q, const double* V, int ld,
                           double* out) const {
    __syncthreads();
    F::vjp(chain(k, q), V, ld, out);
    __syncthreads();
  }
};

template <class Target>
using UserCholeskyMetric = CholeskyFactoredMetric<Target, UserCholModel<>>;
static_assert(MB200_RM_CHOL_THREADS == 256, "the Cholesky user contract is per 256-thread CTA");

#ifdef MB200_USER_DENSE_METRIC
// GlobalDenseMetricT's model interface over metric_dense / vjp_metric_dense: fill and the dense
// VJP, no entry and no rank-one VJP (the policy forms V = -w w^T for the generic route)
template <class F = UserMetricFunctions>
struct UserDenseModel {
  double mp[MB200_MAX_PARAMS];
  const double* maux;
  int dim;
  __device__ UserDenseModel(const ModelArgs& m, int d) : maux(m.maux), dim(d) {
#pragma unroll
    for (int i = 0; i < MB200_MAX_PARAMS; ++i) mp[i] = m.mp[i];
  }
  __device__ __forceinline__ CtaChain chain(const Blk& k, const double* q) const {
    CtaChain c;
    c.dim = dim;
    c.lane = k.tid;
    c.n_lanes = k.nthr;
    c.q = q;
#pragma unroll
    for (int i = 0; i < MB200_MAX_PARAMS; ++i) c.params[i] = mp[i];
    c.aux = maux;
    c.blk = k;
    return c;
  }
  __device__ void fill(const Blk& k, const double* q, double* M, int ld) const {
    __syncthreads();
    F::dense(chain(k, q), M, ld);
    __syncthreads();
  }
  __device__ void vjp_dense(const Blk& k, const double* q, const double* V, int ld,
                            double* out) const {
    __syncthreads();
    F::vjp(chain(k, q), V, ld, out);
    __syncthreads();
  }
};

template <class Target>
using UserDenseMetric = GlobalDenseMetricT<Target, UserDenseModel<>>;
static_assert(DG_THREADS == 256, "the dense user contract is per 256-thread CTA");
#endif

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
#elif defined(MB200_USER_DENSE_METRIC)
#define MB200_USER_METRIC_FUNCTIONS                                                             \
  struct mb200::UserMetricFunctions {                                                           \
    static __device__ __forceinline__ void dense(const mb200::CtaChain& c, double* M, int ld) { \
      metric_dense(c, M, ld);                                                                   \
    }                                                                                           \
    static __device__ __forceinline__ void vjp(const mb200::CtaChain& c, const double* V,       \
                                               int ld, double* out) {                           \
      vjp_metric_dense(c, V, ld, out);                                                          \
    }                                                                                           \
  };
#elif defined(MB200_USER_CHOLESKY_METRIC)
#define MB200_USER_METRIC_FUNCTIONS                                                             \
  struct mb200::UserMetricFunctions {                                                           \
    static __device__ __forceinline__ void chol(const mb200::CtaChain& c, double* L, int ld) {  \
      metric_chol(c, L, ld);                                                                    \
    }                                                                                           \
    static __device__ __forceinline__ void vjp(const mb200::CtaChain& c, const double* V,       \
                                               int ld, double* out) {                           \
      vjp_metric_chol(c, V, ld, out);                                                           \
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
