// libmici_b200.so -- C-ABI entry points (include/mici_b200.h): implicit integrators on Riemannian-metric systems.
// Host-side argument checking and kernel dispatch only; all arithmetic is in the .cuh kernels.
#include "api_common.cuh"
#include "riemannian.cuh"

namespace mb200 {

template <class Target, template <class> class MetricT>
static int launch_implicit(const double* q_in, const double* p_in, double* q_out, double* p_out,
                           const int32_t* dir, int64_t n, int dim, double eps, int n_steps,
                           const ModelArgs& m, double fp_tol, double fp_div, int fp_max,
                           double rev_tol, double* h_out, int32_t* status, int32_t* n_done,
                           int32_t* fp_iters, cudaStream_t st, int midpoint, int fp_solver) {
  auto kern = implicit_leapfrog_kernel<Target, MetricT>;
  int n_mats = MetricT<Target>::N_MATS;
  // SoftAbs: a third matrix enables warm-started eigensolves; use it when two CTAs still fit
  if (MetricT<Target>::SOFTABS && rm_smem_doubles(dim, 3) * sizeof(double) <= 113 * 1024) n_mats = 3;
  if (MetricT<Target>::SOFTABS && Target::DENSE_MTP) n_mats = 3;  // the third holds Z = A U
  constexpr bool compact = rm_compact_policy<MetricT<Target>>::value;
  size_t smem = (compact ? rm_compact_doubles(dim, midpoint) : rm_smem_doubles(dim, n_mats)) *
                sizeof(double);
  bool in_ws = false;
  if (compact && smem > 227 * 1024)
    return fail(MB200_ERR_UNSUPPORTED, "dim %d: per-chain vectors (%zu bytes) exceed shared memory",
                dim, smem);
  constexpr int ws_mats = rm_workspace_mats<MetricT<Target>>::value;
  if (smem > 227 * 1024) {
    // SoftAbs and Cholesky-factored metrics beyond shared memory: the same kernels with the
    // matrices in a per-CTA global workspace (L2-resident operands: slower, but the reference
    // has no dimension limit)
    if (ws_mats == 0)
      return fail(MB200_ERR_UNSUPPORTED,
                  "dim %d: per-chain metric (%zu bytes) exceeds shared memory", dim, smem);
    n_mats = RM_NMATS_IN_WORKSPACE + ws_mats;
    smem = rm_smem_doubles(dim, n_mats) * sizeof(double);
    in_ws = true;
    if (smem > 227 * 1024) return fail(MB200_ERR_UNSUPPORTED, "dim %d too large", dim);
  }
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "smem attr: %s", cudaGetErrorString(e));
  int per_sm = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, MetricT<Target>::THREADS, smem);
  if (per_sm < 1) per_sm = 1;
  if (in_ws && per_sm > 2) per_sm = 2;
  int64_t blocks = (int64_t)num_sms() * per_sm;
  if (blocks > n) blocks = n;
  ModelArgs margs = m;
  const size_t per_cta = ws_mats * ((((size_t)dim * (dim + 1)) + 1) & ~(size_t)1);
  DgScratch scratch(nullptr, 0, in_ws ? per_cta * blocks * sizeof(double) : 0, st);
  if (in_ws) {
    if (scratch.ptr == nullptr) return fail(MB200_ERR_CUDA, "metric workspace allocation failed");
    margs.workspace = scratch.ptr;
    margs.ws_stride = per_cta;
  }
  kern<<<(unsigned)blocks, MetricT<Target>::THREADS, smem, st>>>(
      q_in, p_in, q_out, p_out, dir, n, dim, eps, n_steps, margs, fp_tol, fp_div, fp_max, rev_tol,
      h_out, status, n_done, fp_iters, n_mats, midpoint, fp_solver);
  return check_launch("implicit_leapfrog_kernel");
}

// Dense metrics whose factor does not fit in shared memory (and every Hadamard metric) run through
// the global-workspace policy (api_dense.cu); the rank-1 metric keeps its Sherman-Morrison form
// as an OPTIONAL policy (rmetric_params[2] != 0) and for targets the dense policy is not
// compiled for.
static bool wants_global_dense(const ModelArgs& m, int dim) {
  if (m.rmetric_id == MB200_RMETRIC_HADAMARD) return true;
  if (m.rmetric_id != MB200_RMETRIC_RANK1) return false;
  const bool fits = rm_smem_doubles(dim, 1) * sizeof(double) <= 227 * 1024;
  return !fits && m.mp[2] == 0.0 && m.target_id == MB200_TARGET_QUADRATIC &&
         dense_global_supported(dim);
}

static bool is_compact_rmetric(int id) {
  return id == MB200_RMETRIC_DIAG_QUADRATIC || id == MB200_RMETRIC_DIAG_FUNNEL_FISHER ||
         id == MB200_RMETRIC_SCALAR_QUADRATIC;
}

// Target / metric pairs of the O(D) metrics.  `L` is one of the launch functors below: its
// `run<Target, MetricT>()` launches the entry point's kernel for that pair.
template <class L>
static int compact_dispatch(const ModelArgs& m, int dim, const L& l) {
  if (m.rmetric_id != MB200_RMETRIC_DIAG_FUNNEL_FISHER && !(m.mp[0] > 0.0 && m.mp[1] >= 0.0))
    return fail(MB200_ERR_INVALID_ARG, "metric parameters need a > 0 and b >= 0");
  if (m.target_id == MB200_TARGET_BANANA && (dim & 1))
    return fail(MB200_ERR_INVALID_ARG, "banana target needs even dim");
  if (m.target_id == MB200_TARGET_QUADRATIC && !m.taux)
    return fail(MB200_ERR_INVALID_ARG, "quadratic target needs its precision matrix");
  if (m.rmetric_id == MB200_RMETRIC_DIAG_FUNNEL_FISHER) {
    if (m.target_id != MB200_TARGET_NEAL_FUNNEL)
      return fail(MB200_ERR_UNSUPPORTED, "the funnel Fisher metric needs the funnel target (got %d)",
                  m.target_id);
    return l.template run<FunnelRTarget, FunnelFisherMetric>();
  }
  const bool diag = m.rmetric_id == MB200_RMETRIC_DIAG_QUADRATIC;
  switch (m.target_id) {
    case MB200_TARGET_STD_GAUSSIAN:
      return diag ? l.template run<StdGaussianRTarget, QuadraticDiagonalMetric>()
                  : l.template run<StdGaussianRTarget, ScalarMetric>();
    case MB200_TARGET_BANANA:
      return diag ? l.template run<BananaRTarget, QuadraticDiagonalMetric>()
                  : l.template run<BananaRTarget, ScalarMetric>();
    case MB200_TARGET_NEAL_FUNNEL:
      return diag ? l.template run<FunnelRTarget, QuadraticDiagonalMetric>()
                  : l.template run<FunnelRTarget, ScalarMetric>();
    case MB200_TARGET_QUADRATIC:
      return diag ? l.template run<QuadraticRTarget, QuadraticDiagonalMetric>()
                  : l.template run<QuadraticRTarget, ScalarMetric>();
    default:
      return fail(MB200_ERR_UNSUPPORTED, "target %d not available with diagonal / scalar metrics",
                  m.target_id);
  }
}

// Target / metric pairs of the Cholesky-factored metric (same targets and argument checks as
// compact_dispatch); `L` as there
template <class L>
static int chol_dispatch(const ModelArgs& m, int dim, const L& l) {
  if (!m.maux)
    return fail(MB200_ERR_INVALID_ARG, "Cholesky-factored metric needs its base factor (rmetric_aux)");
  if (m.target_id == MB200_TARGET_BANANA && (dim & 1))
    return fail(MB200_ERR_INVALID_ARG, "banana target needs even dim");
  if (m.target_id == MB200_TARGET_QUADRATIC && !m.taux)
    return fail(MB200_ERR_INVALID_ARG, "quadratic target needs its precision matrix");
  switch (m.target_id) {
    case MB200_TARGET_STD_GAUSSIAN: return l.template run<StdGaussianRTarget, QuadraticCholeskyMetric>();
    case MB200_TARGET_BANANA: return l.template run<BananaRTarget, QuadraticCholeskyMetric>();
    case MB200_TARGET_NEAL_FUNNEL: return l.template run<FunnelRTarget, QuadraticCholeskyMetric>();
    case MB200_TARGET_QUADRATIC: return l.template run<QuadraticRTarget, QuadraticCholeskyMetric>();
    default:
      return fail(MB200_ERR_UNSUPPORTED, "target %d not available with a Cholesky-factored metric",
                  m.target_id);
  }
}

struct ImplicitLaunch {
  const double *q_in, *p_in;
  double *q_out, *p_out;
  const int32_t* dir;
  int64_t n;
  int dim;
  double eps;
  int n_steps;
  const ModelArgs& m;
  double fp_tol, fp_div;
  int fp_max;
  double rev_tol;
  double* h_out;
  int32_t *status, *n_done, *fp_iters;
  cudaStream_t st;
  int midpoint, fp_solver;
  template <class Target, template <class> class MetricT>
  int run() const {
    return launch_implicit<Target, MetricT>(q_in, p_in, q_out, p_out, dir, n, dim, eps, n_steps, m,
                                            fp_tol, fp_div, fp_max, rev_tol, h_out, status, n_done,
                                            fp_iters, st, midpoint, fp_solver);
  }
};

static int implicit_dispatch(const double* q_in, const double* p_in, double* q_out, double* p_out,
                             const int32_t* dir, int64_t n, int dim, double eps, int n_steps,
                             const ModelArgs& m, double fp_tol, double fp_div, int fp_max,
                             double rev_tol, double* h_out, int32_t* status, int32_t* n_done,
                             int32_t* fp_iters, cudaStream_t st, int midpoint = 0,
                             int fp_solver = 0, void* ws = nullptr, int64_t ws_bytes = 0) {
  if (fp_solver != MB200_FP_SOLVER_DIRECT && fp_solver != MB200_FP_SOLVER_STEFFENSEN)
    return fail(MB200_ERR_INVALID_ARG, "unknown fixed-point solver %d", fp_solver);
  const DeviceScope device_scope(q_in);
  if (wants_global_dense(m, dim))
    return dense_global_implicit(q_in, p_in, q_out, p_out, dir, n, dim, eps, n_steps, m, fp_tol,
                                 fp_div, fp_max, rev_tol, h_out, status, n_done, fp_iters, st,
                                 midpoint, fp_solver, ws, ws_bytes);
#define MB200_ARGS                                                                           \
  q_in, p_in, q_out, p_out, dir, n, dim, eps, n_steps, m, fp_tol, fp_div, fp_max, rev_tol,   \
      h_out, status, n_done, fp_iters, st, midpoint, fp_solver
  if (m.rmetric_id == MB200_RMETRIC_SOFTABS) {
    if (!(m.mp[0] > 0.0)) return fail(MB200_ERR_INVALID_ARG, "softabs_coeff must be positive");
    switch (m.target_id) {
      case MB200_TARGET_BANANA:
        if (dim & 1) return fail(MB200_ERR_INVALID_ARG, "banana target needs even dim");
        return launch_implicit<BananaRTarget, SoftAbsMetric>(MB200_ARGS);
      case MB200_TARGET_QUARTIC:
        if (!m.taux) return fail(MB200_ERR_INVALID_ARG, "quartic target needs its directions");
        if (midpoint)
          return fail(MB200_ERR_UNSUPPORTED, "implicit midpoint: quartic target not available");
        return launch_implicit<QuarticRTarget, SoftAbsMetric>(MB200_ARGS);
      default:
        return fail(MB200_ERR_UNSUPPORTED, "target %d has no device Hessian / MTP (SoftAbs metric)",
                    m.target_id);
    }
  }
  if (m.rmetric_id == MB200_RMETRIC_RANK1) {
    if (!m.maux) return fail(MB200_ERR_INVALID_ARG, "rank-1 metric needs its base matrix (rmetric_aux)");
    if (m.target_id == MB200_TARGET_QUADRATIC && !m.taux)
      return fail(MB200_ERR_INVALID_ARG, "quadratic target needs its precision matrix");
    if (m.target_id == MB200_TARGET_BANANA && (dim & 1))
      return fail(MB200_ERR_INVALID_ARG, "banana target needs even dim");
    // per-chain Cholesky factor in shared memory when it fits (or when forced), else the
    // Sherman-Morrison form that never materialises M(q); mp[2] != 0 forces the latter
    // (dimensions beyond shared memory reach this point only with the Sherman-Morrison policy
    // forced or for targets the global-workspace dense policy is not compiled for)
    const bool fits = rm_smem_doubles(dim, 1) * sizeof(double) <= 227 * 1024;
    const bool woodbury = !fits || m.mp[2] != 0.0;
    switch (m.target_id) {
      case MB200_TARGET_QUADRATIC:
        return woodbury ? launch_implicit<QuadraticRTarget, Rank1WoodburyMetric>(MB200_ARGS)
                        : launch_implicit<QuadraticRTarget, Rank1DenseMetric>(MB200_ARGS);
      case MB200_TARGET_STD_GAUSSIAN:
        return woodbury ? launch_implicit<StdGaussianRTarget, Rank1WoodburyMetric>(MB200_ARGS)
                        : launch_implicit<StdGaussianRTarget, Rank1DenseMetric>(MB200_ARGS);
      case MB200_TARGET_BANANA:
        return woodbury ? launch_implicit<BananaRTarget, Rank1WoodburyMetric>(MB200_ARGS)
                        : launch_implicit<BananaRTarget, Rank1DenseMetric>(MB200_ARGS);
      default:
        return fail(MB200_ERR_UNSUPPORTED, "target %d not available for Riemannian systems", m.target_id);
    }
  }
#undef MB200_ARGS
  if (is_compact_rmetric(m.rmetric_id))
    return compact_dispatch(m, dim, ImplicitLaunch{q_in, p_in, q_out, p_out, dir, n, dim, eps,
                                                   n_steps, m, fp_tol, fp_div, fp_max, rev_tol,
                                                   h_out, status, n_done, fp_iters, st, midpoint,
                                                   fp_solver});
  if (m.rmetric_id == MB200_RMETRIC_CHOL_QUADRATIC)
    return chol_dispatch(m, dim, ImplicitLaunch{q_in, p_in, q_out, p_out, dir, n, dim, eps, n_steps,
                                                m, fp_tol, fp_div, fp_max, rev_tol, h_out, status,
                                                n_done, fp_iters, st, midpoint, fp_solver});
  return fail(MB200_ERR_INVALID_ARG, "unknown rmetric_id %d", m.rmetric_id);
}

template <class Target, template <class> class MetricT>
static int launch_sample_momentum(const double* q, const double* z, double* p_out, int64_t n,
                                  int dim, const ModelArgs& m, int32_t* status, cudaStream_t st) {
  auto kern = riemannian_sample_momentum_kernel<Target, MetricT>;
  int n_mats = MetricT<Target>::N_MATS;
  constexpr bool compact = rm_compact_policy<MetricT<Target>>::value;
  size_t smem = (compact ? rm_compact_doubles(dim, 0) : rm_smem_doubles(dim, n_mats)) * sizeof(double);
  bool in_ws = false;
  constexpr int ws_mats = rm_workspace_mats<MetricT<Target>>::value;
  if (smem > 227 * 1024) {
    if (ws_mats == 0) return fail(MB200_ERR_UNSUPPORTED, "dim %d too large", dim);
    n_mats = RM_NMATS_IN_WORKSPACE + ws_mats;
    smem = rm_smem_doubles(dim, n_mats) * sizeof(double);
    in_ws = true;
    if (smem > 227 * 1024) return fail(MB200_ERR_UNSUPPORTED, "dim %d too large", dim);
  }
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "smem attr: %s", cudaGetErrorString(e));
  int64_t blocks = (int64_t)num_sms() * 2;
  if (compact) {  // small CTAs: as many as fit
    int per_sm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, MetricT<Target>::THREADS, smem);
    blocks = (int64_t)num_sms() * (per_sm > 1 ? per_sm : 1);
  }
  if (blocks > n) blocks = n;
  ModelArgs margs = m;
  const size_t per_cta = ws_mats * ((((size_t)dim * (dim + 1)) + 1) & ~(size_t)1);
  DgScratch scratch(nullptr, 0, in_ws ? per_cta * blocks * sizeof(double) : 0, st);
  if (in_ws) {
    if (scratch.ptr == nullptr) return fail(MB200_ERR_CUDA, "metric workspace allocation failed");
    margs.workspace = scratch.ptr;
    margs.ws_stride = per_cta;
  }
  kern<<<(unsigned)blocks, MetricT<Target>::THREADS, smem, st>>>(q, z, p_out, n, dim, margs, status,
                                                                  n_mats);
  return check_launch("riemannian_sample_momentum_kernel");
}

template <class Target, template <class> class MetricT>
static int launch_velocity(const double* q, const double* p, double* vel, int64_t n, int dim,
                           const ModelArgs& m, int32_t* status, cudaStream_t st) {
  auto kern = riemannian_velocity_kernel<Target, MetricT>;
  int n_mats = MetricT<Target>::N_MATS;
  constexpr bool compact = rm_compact_policy<MetricT<Target>>::value;
  size_t smem = (compact ? rm_compact_doubles(dim, 0) : rm_smem_doubles(dim, n_mats)) * sizeof(double);
  bool in_ws = false;
  constexpr int ws_mats = rm_workspace_mats<MetricT<Target>>::value;
  if (smem > 227 * 1024) {
    if (ws_mats == 0) return fail(MB200_ERR_UNSUPPORTED, "dim %d too large", dim);
    n_mats = RM_NMATS_IN_WORKSPACE + ws_mats;
    smem = rm_smem_doubles(dim, n_mats) * sizeof(double);
    in_ws = true;
    if (smem > 227 * 1024) return fail(MB200_ERR_UNSUPPORTED, "dim %d too large", dim);
  }
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "smem attr: %s", cudaGetErrorString(e));
  int64_t blocks = (int64_t)num_sms() * 2;
  if (compact) {  // small CTAs: as many as fit
    int per_sm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, MetricT<Target>::THREADS, smem);
    blocks = (int64_t)num_sms() * (per_sm > 1 ? per_sm : 1);
  }
  if (blocks > n) blocks = n;
  ModelArgs margs = m;
  const size_t per_cta = ws_mats * ((((size_t)dim * (dim + 1)) + 1) & ~(size_t)1);
  DgScratch scratch(nullptr, 0, in_ws ? per_cta * blocks * sizeof(double) : 0, st);
  if (in_ws) {
    if (scratch.ptr == nullptr) return fail(MB200_ERR_CUDA, "metric workspace allocation failed");
    margs.workspace = scratch.ptr;
    margs.ws_stride = per_cta;
  }
  kern<<<(unsigned)blocks, MetricT<Target>::THREADS, smem, st>>>(q, p, vel, n, dim, margs, status,
                                                                  n_mats);
  return check_launch("riemannian_velocity_kernel");
}

// sqrt(M(q)) v (velocity = false) or M(q)^-1 v (velocity = true) for the compact metrics
struct VectorLaunch {
  const double *q, *v;
  double* out;
  int64_t n;
  int dim;
  const ModelArgs& m;
  int32_t* status;
  cudaStream_t st;
  bool velocity;
  template <class Target, template <class> class MetricT>
  int run() const {
    return velocity ? launch_velocity<Target, MetricT>(q, v, out, n, dim, m, status, st)
                    : launch_sample_momentum<Target, MetricT>(q, v, out, n, dim, m, status, st);
  }
};

}  // namespace mb200

using namespace mb200;

extern "C" {

int mb200_implicit_leapfrog_riemannian(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, const mb200_model* model, int32_t fp_solver,
    double fp_convergence_tol, double fp_divergence_tol, int32_t fp_max_iters,
    double reverse_check_tol, double* h_out, int32_t* status, int32_t* n_done, int32_t* fp_iters,
    void* workspace, int64_t workspace_bytes, void* stream) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos_in || !mom_in || !pos_out || !mom_out || !model)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1 || n_steps < 0 || fp_max_iters < 0)
    return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (n_chains == 0) return 0;
  return implicit_dispatch(pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size,
                           n_steps, to_args(model, step_sizes, n_steps_per_chain),
                           fp_convergence_tol, fp_divergence_tol, fp_max_iters, reverse_check_tol,
                           h_out, status, n_done, fp_iters, (cudaStream_t)stream, 0, fp_solver,
                           workspace, workspace_bytes);
}

// Per-chain buffers live in shared memory except for the global-workspace dense metric policy
// (D x D matrices per resident CTA).  A caller that passes less (or NULL) still works: the
// library then takes the scratch from the stream-ordered allocator for the duration of the call.
int64_t mb200_implicit_workspace_bytes(int64_t n_chains, int32_t dim, const mb200_model* model) {
  if (!model || n_chains <= 0 || dim < 1) return 0;
  const ModelArgs m = to_args(model);
  return wants_global_dense(m, dim) ? dense_global_workspace_bytes(n_chains, dim) : 0;
}

int mb200_hamiltonian_riemannian(const double* pos, const double* mom, int64_t n_chains,
                                 int32_t dim, const mb200_model* model, double* h_out,
                                 int32_t* status, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos || !mom || !model || !h_out) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (n_chains == 0) return 0;
  // zero steps: state written back unchanged in place, h evaluated
  return implicit_dispatch(pos, mom, const_cast<double*>(pos), const_cast<double*>(mom), nullptr,
                           n_chains, dim, 0.0, 0, to_args(model), 1e-9, 1e10, 100, 2e-8, h_out,
                           status, nullptr, nullptr, (cudaStream_t)stream, 0, 0, workspace,
                           workspace_bytes);
}

int mb200_selftest_fixed_point(int32_t func_id, int32_t fp_solver, const double* x0,
                               const double* y, int64_t n, int32_t dim, double convergence_tol,
                                      double divergence_tol, int32_t max_iters, double* x_out,
                                      int32_t* iters_out, int32_t* status, void* stream) {
  if (!x0 || !y || !x_out || !iters_out || !status)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n < 0 || dim < 1 || func_id < 0 || func_id > 4) return fail(MB200_ERR_INVALID_ARG, "bad arguments");
  if (n == 0) return 0;
  const DeviceScope device_scope(x0);
  const size_t smem = (size_t)(3 * dim + 40) * sizeof(double);
  int64_t blocks = n < 4096 ? n : 4096;
  fixed_point_selftest_kernel<<<(unsigned)blocks, 64, smem, (cudaStream_t)stream>>>(
      func_id, fp_solver, x0, y, n, dim, convergence_tol, divergence_tol, max_iters, x_out, iters_out,
      status);
  return check_launch("fixed_point_selftest_kernel");
}

int mb200_selftest_eigh(const double* matrices, int64_t n_matrices, int32_t dim, int32_t warm_from,
                        double* eigval, double* eigvec, int32_t* status, void* stream) {
  if (!matrices || !eigval || !eigvec || !status)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_matrices < 0 || dim < 1 || warm_from >= n_matrices)
    return fail(MB200_ERR_INVALID_ARG, "bad arguments");
  if (n_matrices == 0) return 0;
  const DeviceScope device_scope(matrices);
  const size_t smem = rm_smem_doubles(dim, 3) * sizeof(double);
  if (smem > 227 * 1024) return fail(MB200_ERR_UNSUPPORTED, "dim %d too large for the self-test", dim);
  cudaError_t e = cudaFuncSetAttribute(eigh_selftest_kernel,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "smem attr: %s", cudaGetErrorString(e));
  int64_t blocks = n_matrices < 1024 ? n_matrices : 1024;
  eigh_selftest_kernel<<<(unsigned)blocks, RM_THREADS, smem, (cudaStream_t)stream>>>(
      matrices, n_matrices, dim, warm_from, eigval, eigvec, status);
  return check_launch("eigh_selftest_kernel");
}

int mb200_implicit_midpoint_riemannian(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, const mb200_model* model, int32_t fp_solver,
    double fp_convergence_tol, double fp_divergence_tol, int32_t fp_max_iters,
    double reverse_check_tol, double* h_out, int32_t* status, int32_t* n_done, int32_t* fp_iters,
    void* stream) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos_in || !mom_in || !pos_out || !mom_out || !model)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1 || n_steps < 0 || fp_max_iters < 0)
    return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  return implicit_dispatch(pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size,
                           n_steps, to_args(model, step_sizes, n_steps_per_chain),
                           fp_convergence_tol, fp_divergence_tol,
                           fp_max_iters, reverse_check_tol, h_out, status, n_done, fp_iters,
                           (cudaStream_t)stream, 1, fp_solver);
}

int mb200_sample_momentum_riemannian(const double* pos, const double* normals, double* mom_out,
                                     int64_t n_chains, int32_t dim, const mb200_model* model,
                                     int32_t* status, void* stream) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos || !normals || !mom_out || !model) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  const DeviceScope device_scope(pos);
  const ModelArgs m = to_args(model);
  cudaStream_t st = (cudaStream_t)stream;
#define MB200_ARGS pos, normals, mom_out, n_chains, dim, m, status, st
  if (wants_global_dense(m, dim))
    return dense_global_vector(pos, normals, mom_out, n_chains, dim, m, status, st, 0);
  if (m.rmetric_id == MB200_RMETRIC_SOFTABS) {
    if (m.target_id == MB200_TARGET_BANANA) return launch_sample_momentum<BananaRTarget, SoftAbsMetric>(MB200_ARGS);
    if (m.target_id == MB200_TARGET_QUARTIC) return launch_sample_momentum<QuarticRTarget, SoftAbsMetric>(MB200_ARGS);
    return fail(MB200_ERR_UNSUPPORTED, "target %d has no device Hessian", m.target_id);
  }
  if (m.rmetric_id == MB200_RMETRIC_RANK1) {
    if (!m.maux) return fail(MB200_ERR_INVALID_ARG, "rank-1 metric needs its base matrix");
    if (rm_smem_doubles(dim, 1) * sizeof(double) > 227 * 1024)
      return fail(MB200_ERR_UNSUPPORTED,
                  "dim %d: the Cholesky factor of M(q) does not fit in shared memory", dim);
    switch (m.target_id) {
      case MB200_TARGET_QUADRATIC: return launch_sample_momentum<QuadraticRTarget, Rank1DenseMetric>(MB200_ARGS);
      case MB200_TARGET_STD_GAUSSIAN: return launch_sample_momentum<StdGaussianRTarget, Rank1DenseMetric>(MB200_ARGS);
      case MB200_TARGET_BANANA: return launch_sample_momentum<BananaRTarget, Rank1DenseMetric>(MB200_ARGS);
      default: return fail(MB200_ERR_UNSUPPORTED, "target %d not available", m.target_id);
    }
  }
#undef MB200_ARGS
  if (is_compact_rmetric(m.rmetric_id))
    return compact_dispatch(m, dim, VectorLaunch{pos, normals, mom_out, n_chains, dim, m, status,
                                                 st, false});
  if (m.rmetric_id == MB200_RMETRIC_CHOL_QUADRATIC)
    return chol_dispatch(m, dim, VectorLaunch{pos, normals, mom_out, n_chains, dim, m, status, st,
                                              false});
  return fail(MB200_ERR_INVALID_ARG, "unknown rmetric_id %d", m.rmetric_id);
}

int mb200_dh_dmom_riemannian(const double* pos, const double* mom, double* vel_out,
                             int64_t n_chains, int32_t dim, const mb200_model* model,
                             int32_t* status, void* stream) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos || !mom || !vel_out || !model) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  const DeviceScope device_scope(pos);
  const ModelArgs m = to_args(model);
  cudaStream_t st = (cudaStream_t)stream;
#define MB200_ARGS pos, mom, vel_out, n_chains, dim, m, status, st
  if (wants_global_dense(m, dim))
    return dense_global_vector(pos, mom, vel_out, n_chains, dim, m, status, st, 1);
  if (m.rmetric_id == MB200_RMETRIC_SOFTABS) {
    if (m.target_id == MB200_TARGET_BANANA) return launch_velocity<BananaRTarget, SoftAbsMetric>(MB200_ARGS);
    if (m.target_id == MB200_TARGET_QUARTIC) return launch_velocity<QuarticRTarget, SoftAbsMetric>(MB200_ARGS);
    return fail(MB200_ERR_UNSUPPORTED, "target %d has no device Hessian", m.target_id);
  }
  if (m.rmetric_id == MB200_RMETRIC_RANK1) {
    if (!m.maux) return fail(MB200_ERR_INVALID_ARG, "rank-1 metric needs its base matrix");
    const bool fits = rm_smem_doubles(dim, 1) * sizeof(double) <= 227 * 1024;
    const bool woodbury = !fits || m.mp[2] != 0.0;
    switch (m.target_id) {
      case MB200_TARGET_QUADRATIC:
        return woodbury ? launch_velocity<QuadraticRTarget, Rank1WoodburyMetric>(MB200_ARGS)
                        : launch_velocity<QuadraticRTarget, Rank1DenseMetric>(MB200_ARGS);
      case MB200_TARGET_STD_GAUSSIAN:
        return woodbury ? launch_velocity<StdGaussianRTarget, Rank1WoodburyMetric>(MB200_ARGS)
                        : launch_velocity<StdGaussianRTarget, Rank1DenseMetric>(MB200_ARGS);
      case MB200_TARGET_BANANA:
        return woodbury ? launch_velocity<BananaRTarget, Rank1WoodburyMetric>(MB200_ARGS)
                        : launch_velocity<BananaRTarget, Rank1DenseMetric>(MB200_ARGS);
      default: return fail(MB200_ERR_UNSUPPORTED, "target %d not available", m.target_id);
    }
  }
#undef MB200_ARGS
  if (is_compact_rmetric(m.rmetric_id))
    return compact_dispatch(m, dim, VectorLaunch{pos, mom, vel_out, n_chains, dim, m, status, st,
                                                 true});
  if (m.rmetric_id == MB200_RMETRIC_CHOL_QUADRATIC)
    return chol_dispatch(m, dim, VectorLaunch{pos, mom, vel_out, n_chains, dim, m, status, st, true});
  return fail(MB200_ERR_INVALID_ARG, "unknown rmetric_id %d", m.rmetric_id);
}

}  // extern "C"
