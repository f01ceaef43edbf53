// libmici_b200.so -- C-ABI entry points (include/mici_b200.h): implicit integrators on Riemannian-metric systems.
// Host-side argument checking and kernel dispatch only; all arithmetic is in the .cuh kernels.
#include "api_common.cuh"
#include "riemannian.cuh"

namespace mb200 {

// What a Riemannian entry point computes (the Hamiltonian alone is a leapfrog of zero steps)
enum class RmOp { Leapfrog, Midpoint, SampleMomentum, Velocity };

// Launch plan of the three Riemannian kernels outside the global-workspace dense policy: the
// chain's layout, the per-CTA global workspace of the policies whose matrices do not fit in
// shared memory, and the grid.  `launch(blocks, smem, margs, layout)` starts `kern`.
template <class Target, template <class> class MetricT, class Kernel, class Launch>
static int rm_launch(Kernel kern, const char* name, RmOp op, int64_t n, int dim,
                     const ModelArgs& m, cudaStream_t st, const Launch& launch) {
  using Metric = MetricT<Target>;
  constexpr bool compact = Metric::PLACE == RM_COMPACT;
  const bool implicit = op == RmOp::Leapfrog || op == RmOp::Midpoint;
  RmLayout layout{dim, Metric::PLACE, Metric::N_MATS, 0, op == RmOp::Midpoint};
  // SoftAbs integrators: a third matrix enables warm-started eigensolves; use it when two CTAs
  // still fit (DENSE_MTP targets always: the third holds Z = A U)
  if (Metric::SOFTABS && implicit) {
    RmLayout three = layout;
    three.smem_mats = 3;
    if (rm_smem_bytes(three) <= 113 * 1024 || Target::DENSE_MTP) layout = three;
  }
  size_t smem = rm_smem_bytes(layout);
  if (smem > RM_SMEM_BYTES) {
    if (compact && implicit)
      return fail(MB200_ERR_UNSUPPORTED,
                  "dim %d: per-chain vectors (%zu bytes) exceed shared memory", dim, smem);
    // SoftAbs and Cholesky-factored metrics beyond shared memory: the same kernels with the
    // matrices in a per-CTA global workspace (L2-resident operands: slower, but the reference
    // has no dimension limit)
    if (Metric::WORKSPACE_MATS == 0)
      return implicit ? fail(MB200_ERR_UNSUPPORTED,
                             "dim %d: per-chain metric (%zu bytes) exceeds shared memory", dim, smem)
                      : fail(MB200_ERR_UNSUPPORTED, "dim %d too large", dim);
    layout.smem_mats = 0;
    layout.ws_mats = Metric::WORKSPACE_MATS;
    smem = rm_smem_bytes(layout);
    if (smem > RM_SMEM_BYTES) return fail(MB200_ERR_UNSUPPORTED, "dim %d too large", dim);
  }
  const bool in_ws = layout.ws_mats > 0;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "smem attr: %s", cudaGetErrorString(e));
  // the integrators and the small CTAs of the compact policies: as many CTAs as fit (at most two
  // per SM with the workspace); the vector kernels of the matrix policies: two per SM
  int per_sm = 2;
  if (implicit || compact) {
    per_sm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, Metric::THREADS, smem);
    if (per_sm < 1) per_sm = 1;
    if (in_ws && per_sm > 2) per_sm = 2;
  }
  int64_t blocks = (int64_t)num_sms() * per_sm;
  if (blocks > n) blocks = n;
  ModelArgs margs = m;
  const size_t per_cta = layout.ws_mats * layout.ws_mat_doubles();
  DgScratch scratch(nullptr, 0, in_ws ? per_cta * blocks * sizeof(double) : 0, st);
  if (in_ws) {
    if (scratch.ptr == nullptr) return fail(MB200_ERR_CUDA, "metric workspace allocation failed");
    margs.workspace = scratch.ptr;
    margs.ws_stride = per_cta;
  }
  launch((unsigned)blocks, smem, margs, layout);
  return check_launch(name);
}

// a user image's Cholesky-factored policy as the host plans it
template <class Target>
using UserCholeskyPlan = CholeskyFactoredMetric<Target, UserCholModelTraits>;

// Launch functors of the operations: `run<Target, MetricT>()` starts the operation's kernel for
// that pair, `global(hadamard)` its global-workspace dense form (api_dense.cu), `image<Traits>()`
// the kernel of the loaded user image `user` (user_riemannian.cuh), planned as the registry
// policy `Traits` over UserRTargetTraits, whose launch constants the image's policy shares
using ImplicitKernel = decltype(&implicit_leapfrog_kernel<StdGaussianRTarget, QuadraticDiagonalMetric>);
using VectorKernel = decltype(&riemannian_velocity_kernel<StdGaussianRTarget, QuadraticDiagonalMetric>);

template <RmOp OP>
struct ImplicitLaunch {
  static constexpr RmOp op = OP;
  const ImplicitArgs& a;
  const UserRiemannianKernels* user;
  template <class Target, template <class> class MetricT>
  int run() const {
    return launch<Target, MetricT>(implicit_leapfrog_kernel<Target, MetricT>);
  }
  template <template <class> class Traits>
  int image() const {
    return launch<UserRTargetTraits, Traits>(reinterpret_cast<ImplicitKernel>(user->implicit));
  }
  template <class Target, template <class> class MetricT>
  int launch(ImplicitKernel kern) const {
    return rm_launch<Target, MetricT>(
        kern, "implicit_leapfrog_kernel", OP, a.n, a.dim, a.m, a.st,
        [&](unsigned blocks, size_t smem, const ModelArgs& margs, const RmLayout& layout) {
          rm_start(kern, blocks, MetricT<Target>::THREADS, smem, a.st, a.q_in, a.p_in, a.q_out,
                   a.p_out, a.dir, a.n, a.dim, a.eps, a.n_steps, margs, a.fp_tol, a.fp_div,
                   a.fp_max, a.rev_tol, a.h_out, a.status, a.n_done, a.fp_iters, layout,
                   (int)(OP == RmOp::Midpoint), a.fp_solver);
        });
  }
  int global(bool hadamard) const { return dense_global_implicit(a, hadamard); }
  int image_global() const { return dense_global_implicit_image(a, user->implicit); }
};

template <RmOp OP>
struct VectorLaunch {
  static constexpr RmOp op = OP;
  static constexpr bool velocity = OP == RmOp::Velocity;
  const VectorArgs& a;
  const UserRiemannianKernels* user;
  template <class Target, template <class> class MetricT>
  int run() const {
    return launch<Target, MetricT>(riemannian_vector_kernel<Target, MetricT, velocity>());
  }
  template <template <class> class Traits>
  int image() const {
    return launch<UserRTargetTraits, Traits>(
        reinterpret_cast<VectorKernel>(velocity ? user->velocity : user->momentum));
  }
  template <class Target, template <class> class MetricT>
  int launch(VectorKernel kern) const {
    return rm_launch<Target, MetricT>(
        kern, velocity ? "riemannian_velocity_kernel" : "riemannian_sample_momentum_kernel", OP,
        a.n, a.dim, a.m, a.st,
        [&](unsigned blocks, size_t smem, const ModelArgs& margs, const RmLayout& layout) {
          rm_start(kern, blocks, MetricT<Target>::THREADS, smem, a.st, a.q, a.v, a.out, a.n, a.dim,
                   margs, a.status, layout);
        });
  }
  int global(bool hadamard) const { return dense_global_vector(a, velocity, hadamard); }
  int image_global() const {
    return dense_global_vector_image(a, velocity ? user->velocity : user->momentum);
  }
};

// The caller-provided workspace an implicit leapfrog of this model takes (the global-workspace
// dense policy only); launches nothing
struct WorkspaceQuery {
  static constexpr RmOp op = RmOp::Leapfrog;
  int64_t n;
  int dim;
  int64_t* bytes;
  const UserRiemannianKernels* user = nullptr;
  template <class Target, template <class> class MetricT>
  int run() const { return 0; }
  template <template <class> class>
  int image() const { return 0; }
  int image_global() const { return 0; }
  int global(bool) const {
    *bytes = dense_global_workspace_bytes(n, dim);
    return 0;
  }
};

// `l` on the targets a metric policy is compiled for: std-Gaussian, banana, quadratic and (FUNNEL)
// Neal's funnel; `metric` completes the error of any other target
template <template <class> class MetricT, bool FUNNEL, class L>
static int run_on_target(int target_id, const L& l, const char* metric) {
  switch (target_id) {
    case MB200_TARGET_STD_GAUSSIAN: return l.template run<StdGaussianRTarget, MetricT>();
    case MB200_TARGET_BANANA: return l.template run<BananaRTarget, MetricT>();
    case MB200_TARGET_QUADRATIC: return l.template run<QuadraticRTarget, MetricT>();
    case MB200_TARGET_NEAL_FUNNEL:
      if constexpr (FUNNEL) return l.template run<FunnelRTarget, MetricT>();
  }
  return fail(MB200_ERR_UNSUPPORTED, "target %d not available %s", target_id, metric);
}

// Which kernel serves a Riemannian model, for every operation L::op: checks the model (the same
// checks whatever the operation), picks the metric policy and the target, and hands them to `l`.
// An operation's exclusions sit next to the route they restrict.  A loaded user image (l.user,
// the *_user entry points) serves a user target with the image's own user metric, planned from
// the registry policy it runs over user models: the compact ones (diagonal, scalar), the
// triangular-factored one (MB200_RMETRIC_USER_CHOLESKY: 256-thread CTAs, the factor and V per
// chain), or, for a dense one (MB200_RMETRIC_USER_DENSE), the global-workspace launch plan with its
// limits.
template <class L>
static int rm_dispatch(const ModelArgs& m, int dim, const L& l) {
  constexpr RmOp op = L::op;
  const int t = m.target_id;
  if (l.user != nullptr) {
    if (t != MB200_TARGET_USER)
      return fail(MB200_ERR_INVALID_ARG, "user-image entry point needs target_id MB200_TARGET_USER");
    if (m.rmetric_id != l.user->rmetric_id)
      return fail(MB200_ERR_INVALID_ARG, "rmetric_id %d does not match the user image's (%d)",
                  m.rmetric_id, l.user->rmetric_id);
    if (l.user->rmetric_id == MB200_RMETRIC_USER_CHOLESKY)
      return l.template image<UserCholeskyPlan>();
    if (l.user->rmetric_id == MB200_RMETRIC_USER_SCALAR)
      return l.template image<QuadraticScalarMetric>();
    if (l.user->rmetric_id != MB200_RMETRIC_USER_DENSE)
      return l.template image<QuadraticDiagonalMetric>();
    if (op == RmOp::Midpoint)
      return fail(MB200_ERR_UNSUPPORTED,
                  "implicit midpoint is not available for the global-workspace dense metric");
    if (!dense_global_supported(dim))
      return fail(MB200_ERR_UNSUPPORTED, "dim %d: panel buffers exceed shared memory", dim);
    return l.image_global();
  }
  // one per-chain D x D matrix (the rank-1 metric's Cholesky factor) fits in shared memory
  const bool fits = rm_smem_bytes(RmLayout{dim, RM_MATRICES, 1, 0, true}) <= RM_SMEM_BYTES;

  // Global-workspace dense policy: every Hadamard metric, and the rank-1 metric whose factor does
  // not fit in shared memory on the quadratic target, unless the Sherman-Morrison form is forced
  // (rmetric_params[2] != 0)
  if (m.rmetric_id == MB200_RMETRIC_HADAMARD ||
      (m.rmetric_id == MB200_RMETRIC_RANK1 && !fits && m.mp[2] == 0.0 &&
       t == MB200_TARGET_QUADRATIC && dense_global_supported(dim))) {
    if (op == RmOp::Midpoint)
      return fail(MB200_ERR_UNSUPPORTED,
                  "implicit midpoint is not available for the global-workspace dense metric");
    if (!dense_global_supported(dim))
      return fail(MB200_ERR_UNSUPPORTED, "dim %d: panel buffers exceed shared memory", dim);
    if (!m.maux) return fail(MB200_ERR_INVALID_ARG, "dense metric needs its matrices (rmetric_aux)");
    if (t != MB200_TARGET_QUADRATIC)
      return fail(MB200_ERR_UNSUPPORTED,
                  "target %d not compiled for the global-workspace dense metric", t);
    if (!m.taux) return fail(MB200_ERR_INVALID_ARG, "quadratic target needs its precision matrix");
    return l.global(m.rmetric_id == MB200_RMETRIC_HADAMARD);
  }

  if (m.rmetric_id == MB200_RMETRIC_SOFTABS) {
    if (!(m.mp[0] > 0.0)) return fail(MB200_ERR_INVALID_ARG, "softabs_coeff must be positive");
    if (t == MB200_TARGET_BANANA) {
      if (dim & 1) return fail(MB200_ERR_INVALID_ARG, "banana target needs even dim");
      return l.template run<BananaRTarget, SoftAbsMetric>();
    }
    if (t == MB200_TARGET_QUARTIC) {
      if (!m.taux) return fail(MB200_ERR_INVALID_ARG, "quartic target needs its directions");
      if (op == RmOp::Midpoint)
        return fail(MB200_ERR_UNSUPPORTED, "implicit midpoint: quartic target not available");
      return l.template run<QuarticRTarget, SoftAbsMetric>();
    }
    return fail(MB200_ERR_UNSUPPORTED, "target %d has no device Hessian / MTP (SoftAbs metric)", t);
  }

  // the other metrics' own arguments, then their targets'
  switch (m.rmetric_id) {
    case MB200_RMETRIC_RANK1:
      if (!m.maux)
        return fail(MB200_ERR_INVALID_ARG, "rank-1 metric needs its base matrix (rmetric_aux)");
      break;
    case MB200_RMETRIC_DIAG_QUADRATIC:
    case MB200_RMETRIC_SCALAR_QUADRATIC:
      if (!(m.mp[0] > 0.0 && m.mp[1] >= 0.0))
        return fail(MB200_ERR_INVALID_ARG, "metric parameters need a > 0 and b >= 0");
      break;
    case MB200_RMETRIC_DIAG_FUNNEL_FISHER: break;
    case MB200_RMETRIC_CHOL_QUADRATIC:
      if (!m.maux)
        return fail(MB200_ERR_INVALID_ARG,
                    "Cholesky-factored metric needs its base factor (rmetric_aux)");
      break;
    default: return fail(MB200_ERR_INVALID_ARG, "unknown rmetric_id %d", m.rmetric_id);
  }
  if (t == MB200_TARGET_BANANA && (dim & 1))
    return fail(MB200_ERR_INVALID_ARG, "banana target needs even dim");
  if (t == MB200_TARGET_QUADRATIC && !m.taux)
    return fail(MB200_ERR_INVALID_ARG, "quadratic target needs its precision matrix");

  switch (m.rmetric_id) {
    case MB200_RMETRIC_RANK1:
      // per-chain Cholesky factor in shared memory when it fits, else the Sherman-Morrison form
      // that never materialises M(q); rmetric_params[2] != 0 forces the latter for the integrators
      // and the velocity (the momentum refresh needs the factor)
      if (!fits || (m.mp[2] != 0.0 && op != RmOp::SampleMomentum)) {
        if constexpr (op == RmOp::SampleMomentum)
          return fail(MB200_ERR_UNSUPPORTED,
                      "dim %d: the Cholesky factor of M(q) does not fit in shared memory", dim);
        else
          return run_on_target<Rank1WoodburyMetric, false>(t, l, "for Riemannian systems");
      }
      return run_on_target<Rank1DenseMetric, false>(t, l, "for Riemannian systems");
    case MB200_RMETRIC_DIAG_FUNNEL_FISHER:
      if (t != MB200_TARGET_NEAL_FUNNEL)
        return fail(MB200_ERR_UNSUPPORTED,
                    "the funnel Fisher metric needs the funnel target (got %d)", t);
      return l.template run<FunnelRTarget, FunnelFisherMetric>();
    case MB200_RMETRIC_DIAG_QUADRATIC:
      return run_on_target<QuadraticDiagonalMetric, true>(t, l, "with diagonal / scalar metrics");
    case MB200_RMETRIC_SCALAR_QUADRATIC:
      return run_on_target<QuadraticScalarMetric, true>(t, l, "with diagonal / scalar metrics");
    default:
      return run_on_target<QuadraticCholeskyMetric, true>(t, l, "with a Cholesky-factored metric");
  }
}

// The handle of a Riemannian *_user entry point: an image of mb200_user_riemannian_load
static int riemannian_image(const void* handle, const UserRiemannianKernels** u) {
  if (!handle) return fail(MB200_ERR_INVALID_ARG, "user_image is NULL");
  *u = &user_riemannian_kernels(handle);
  if ((*u)->rmetric_id == 0)
    return fail(MB200_ERR_INVALID_ARG,
                "user image has no Riemannian kernels (mb200_user_riemannian_load)");
  return 0;
}

template <RmOp OP>
static int implicit_dispatch(const ImplicitArgs& a, const UserRiemannianKernels* user = nullptr) {
  if (a.fp_solver != MB200_FP_SOLVER_DIRECT && a.fp_solver != MB200_FP_SOLVER_STEFFENSEN)
    return fail(MB200_ERR_INVALID_ARG, "unknown fixed-point solver %d", a.fp_solver);
  const DeviceScope device_scope(a.q_in);
  return rm_dispatch(a.m, a.dim, ImplicitLaunch<OP>{a, user});
}

template <RmOp OP>
static int vector_dispatch(const VectorArgs& a, const UserRiemannianKernels* user = nullptr) {
  const DeviceScope device_scope(a.q);
  return rm_dispatch(a.m, a.dim, VectorLaunch<OP>{a, user});
}

// The bodies of the entry points: the registry ones (user == NULL) and their _user twins, whose
// image serves a user target with its user metric

// implicit leapfrog / midpoint steps (zero steps: the Hamiltonian of the state)
template <RmOp OP>
static int implicit_entry(const double* pos_in, const double* mom_in, double* pos_out,
                          double* mom_out, const int32_t* dir, int64_t n_chains, int dim,
                          double step_size, const double* step_sizes, int n_steps,
                          const int32_t* n_steps_per_chain, const mb200_model* model,
                          int fp_solver, double fp_convergence_tol, double fp_divergence_tol,
                          int fp_max_iters, double reverse_check_tol, double* h_out,
                          int32_t* status, int32_t* n_done, int32_t* fp_iters, void* workspace,
                          int64_t workspace_bytes, void* stream,
                          const UserRiemannianKernels* user) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos_in || !mom_in || !pos_out || !mom_out || !model)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1 || n_steps < 0 || fp_max_iters < 0)
    return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  return implicit_dispatch<OP>(
      ImplicitArgs{pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, n_steps,
                   to_args(model, step_sizes, n_steps_per_chain), fp_convergence_tol,
                   fp_divergence_tol, fp_max_iters, reverse_check_tol, h_out, status, n_done,
                   fp_iters, fp_solver, workspace, workspace_bytes, (cudaStream_t)stream},
      user);
}

static int hamiltonian_entry(const double* pos, const double* mom, int64_t n_chains, int dim,
                             const mb200_model* model, double* h_out, int32_t* status,
                             void* workspace, int64_t workspace_bytes, void* stream,
                             const UserRiemannianKernels* user) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos || !mom || !model || !h_out) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  // zero steps: state written back unchanged in place, h evaluated
  return implicit_dispatch<RmOp::Leapfrog>(
      ImplicitArgs{pos, mom, const_cast<double*>(pos), const_cast<double*>(mom), nullptr, n_chains,
                   dim, 0.0, 0, to_args(model), 1e-9, 1e10, 100, 2e-8, h_out, status, nullptr,
                   nullptr, MB200_FP_SOLVER_DIRECT, workspace, workspace_bytes,
                   (cudaStream_t)stream},
      user);
}

// momentum refresh (SampleMomentum: v = normals) or velocity (Velocity: v = mom)
template <RmOp OP>
static int vector_entry(const double* pos, const double* v, double* out, int64_t n_chains,
                        int dim, const mb200_model* model, int32_t* status, void* stream,
                        const UserRiemannianKernels* user) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos || !v || !out || !model) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  return vector_dispatch<OP>(
      VectorArgs{pos, v, out, n_chains, dim, to_args(model), status, (cudaStream_t)stream}, user);
}

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
  return implicit_entry<RmOp::Leapfrog>(
      pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, step_sizes, n_steps,
      n_steps_per_chain, model, fp_solver, fp_convergence_tol, fp_divergence_tol, fp_max_iters,
      reverse_check_tol, h_out, status, n_done, fp_iters, workspace, workspace_bytes, stream,
      nullptr);
}

// Per-chain buffers live in shared memory except for the global-workspace dense metric policy
// (D x D matrices per resident CTA).  A caller that passes less (or NULL) still works: the
// library then takes the scratch from the stream-ordered allocator for the duration of the call.
int64_t mb200_implicit_workspace_bytes(int64_t n_chains, int32_t dim, const mb200_model* model) {
  if (!model || n_chains <= 0 || dim < 1) return 0;
  // a user image's diagonal / scalar policies keep every per-chain vector in shared memory, its
  // Cholesky-factored policy allocates its per-CTA workspace itself (as the registry one does);
  // its dense policy is the global-workspace one
  if (model->rmetric_id == MB200_RMETRIC_USER_DIAGONAL ||
      model->rmetric_id == MB200_RMETRIC_USER_SCALAR ||
      model->rmetric_id == MB200_RMETRIC_USER_CHOLESKY)
    return 0;
  if (model->rmetric_id == MB200_RMETRIC_USER_DENSE)
    return dense_global_supported(dim) ? dense_global_workspace_bytes(n_chains, dim) : 0;
  int64_t bytes = 0;
  rm_dispatch(to_args(model), dim, WorkspaceQuery{n_chains, dim, &bytes});
  return bytes;
}

int mb200_hamiltonian_riemannian(const double* pos, const double* mom, int64_t n_chains,
                                 int32_t dim, const mb200_model* model, double* h_out,
                                 int32_t* status, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  return hamiltonian_entry(pos, mom, n_chains, dim, model, h_out, status, workspace,
                           workspace_bytes, stream, nullptr);
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
  const size_t smem = rm_smem_bytes(eigh_selftest_layout(dim));
  if (smem > RM_SMEM_BYTES)
    return fail(MB200_ERR_UNSUPPORTED, "dim %d too large for the self-test", dim);
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
  return implicit_entry<RmOp::Midpoint>(
      pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, step_sizes, n_steps,
      n_steps_per_chain, model, fp_solver, fp_convergence_tol, fp_divergence_tol, fp_max_iters,
      reverse_check_tol, h_out, status, n_done, fp_iters, nullptr, 0, stream, nullptr);
}

int mb200_sample_momentum_riemannian(const double* pos, const double* normals, double* mom_out,
                                     int64_t n_chains, int32_t dim, const mb200_model* model,
                                     int32_t* status, void* stream) {
  return vector_entry<RmOp::SampleMomentum>(pos, normals, mom_out, n_chains, dim, model, status,
                                            stream, nullptr);
}

int mb200_dh_dmom_riemannian(const double* pos, const double* mom, double* vel_out,
                             int64_t n_chains, int32_t dim, const mb200_model* model,
                             int32_t* status, void* stream) {
  return vector_entry<RmOp::Velocity>(pos, mom, vel_out, n_chains, dim, model, status, stream,
                                      nullptr);
}

// The _user twins: a user target with the user metric of the loaded image `user_image`
// (mb200_user_riemannian_load), checked first; the registry entry points' bodies otherwise

int mb200_implicit_leapfrog_riemannian_user(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, const mb200_model* model, int32_t fp_solver,
    double fp_convergence_tol, double fp_divergence_tol, int32_t fp_max_iters,
    double reverse_check_tol, double* h_out, int32_t* status, int32_t* n_done, int32_t* fp_iters,
    void* workspace, int64_t workspace_bytes, void* stream, const void* user_image) {
  const UserRiemannianKernels* u;
  if (const int rc = riemannian_image(user_image, &u)) return rc;
  return implicit_entry<RmOp::Leapfrog>(
      pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, step_sizes, n_steps,
      n_steps_per_chain, model, fp_solver, fp_convergence_tol, fp_divergence_tol, fp_max_iters,
      reverse_check_tol, h_out, status, n_done, fp_iters, workspace, workspace_bytes, stream, u);
}

int mb200_implicit_midpoint_riemannian_user(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, const mb200_model* model, int32_t fp_solver,
    double fp_convergence_tol, double fp_divergence_tol, int32_t fp_max_iters,
    double reverse_check_tol, double* h_out, int32_t* status, int32_t* n_done, int32_t* fp_iters,
    void* stream, const void* user_image) {
  const UserRiemannianKernels* u;
  if (const int rc = riemannian_image(user_image, &u)) return rc;
  return implicit_entry<RmOp::Midpoint>(
      pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, step_sizes, n_steps,
      n_steps_per_chain, model, fp_solver, fp_convergence_tol, fp_divergence_tol, fp_max_iters,
      reverse_check_tol, h_out, status, n_done, fp_iters, nullptr, 0, stream, u);
}

int mb200_hamiltonian_riemannian_user(const double* pos, const double* mom, int64_t n_chains,
                                      int32_t dim, const mb200_model* model, double* h_out,
                                      int32_t* status, void* workspace, int64_t workspace_bytes,
                                      void* stream, const void* user_image) {
  const UserRiemannianKernels* u;
  if (const int rc = riemannian_image(user_image, &u)) return rc;
  return hamiltonian_entry(pos, mom, n_chains, dim, model, h_out, status, workspace,
                           workspace_bytes, stream, u);
}

int mb200_sample_momentum_riemannian_user(const double* pos, const double* normals,
                                          double* mom_out, int64_t n_chains, int32_t dim,
                                          const mb200_model* model, int32_t* status, void* stream,
                                          const void* user_image) {
  const UserRiemannianKernels* u;
  if (const int rc = riemannian_image(user_image, &u)) return rc;
  return vector_entry<RmOp::SampleMomentum>(pos, normals, mom_out, n_chains, dim, model, status,
                                            stream, u);
}

int mb200_dh_dmom_riemannian_user(const double* pos, const double* mom, double* vel_out,
                                  int64_t n_chains, int32_t dim, const mb200_model* model,
                                  int32_t* status, void* stream, const void* user_image) {
  const UserRiemannianKernels* u;
  if (const int rc = riemannian_image(user_image, &u)) return rc;
  return vector_entry<RmOp::Velocity>(pos, mom, vel_out, n_chains, dim, model, status, stream, u);
}

}  // extern "C"
