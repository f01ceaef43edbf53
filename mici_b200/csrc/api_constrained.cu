// libmici_b200.so -- C-ABI entry points (include/mici_b200.h): constrained (RATTLE / geodesic) leapfrog family.
// Host-side argument checking and kernel dispatch only; all arithmetic is in the .cuh kernels.
#include "api_common.cuh"
#include "constrained.cuh"

namespace mb200 {

// The Gaussian split's w vector and eigenvector matrices (all NULL for the plain system)
struct GaussianArgs {
  const double* omega;
  const double* eigvec;
  const double* eigvec_t;
};

constexpr int CS_WARPS = 4;  // chains (one warp each) per CTA of the warp-per-chain kernels

// CTAs for n chains at `per_cta` chains per CTA, at most 16 per SM (grid-stride loop beyond)
static unsigned cs_blocks(int64_t n, int per_cta) {
  int64_t blocks = (n + per_cta - 1) / per_cta;
  const int64_t cap = (int64_t)num_sms() * 16;
  return (unsigned)(blocks > cap ? cap : blocks);
}

// A constrained target and its per-lane element count KP, as the dispatch below hands them over
template <class T, int KP_>
struct CsShape {
  using Target = T;
  static constexpr int KP = KP_;
  template <bool GAUSS>
  static size_t smem() {
    return (size_t)CS_WARPS * cs_smem_per_warp<T, KP, GAUSS>() * sizeof(double);
  }
};

// The same for the kernels of a user image (UserConstrainedTarget): the metric product's rows and
// the user constraint's staging area
template <bool GAUSS>
static size_t cs_user_smem(const UserConstraintKernels& u) {
  return (size_t)CS_WARPS *
         (constrained_smem_doubles(u.n_constr, u.kp, GAUSS) +
          user_constraint_stage_per_warp(u.n_constr, u.kp)) *
         sizeof(double);
}

// A constrained operation for constrained_target_dispatch: `registry(CsShape<Target, KP>{})`
// starts its library kernel, `image(u)` the same kernel from the loaded user image `user` (NULL
// for a registry target)
template <class Registry, class Image>
struct CsLaunch {
  const UserConstraintKernels* user;
  Registry registry;
  Image image;
};
template <class Registry, class Image>
static CsLaunch<Registry, Image> cs_launch(const void* user_target, Registry registry,
                                           Image image) {
  return {user_target ? &user_constraint_kernels(user_target) : nullptr, registry, image};
}

// Target / size dispatch shared by the constrained entry points.  A user image serves
// dim <= 256 with one constraint and dim <= 128 with several, at the KP the sphere and
// multi-sphere targets use for that dim, which must be the KP it was compiled for.
template <class Launch>
static int constrained_target_dispatch(const ModelArgs& m, int dim, const Launch& launch) {
  if (launch.user != nullptr) {
    const UserConstraintKernels& u = *launch.user;
    if (m.target_id != MB200_TARGET_USER)
      return fail(MB200_ERR_INVALID_ARG,
                  "user-target entry point needs target_id MB200_TARGET_USER");
    if (u.n_constr < 1)
      return fail(MB200_ERR_INVALID_ARG,
                  "user target has no constraint kernels (mb200_user_constraint_load)");
    const int max_dim = u.n_constr == 1 ? 256 : 128;
    if (dim > max_dim)
      return fail(MB200_ERR_UNSUPPORTED, "user constraint: dim %d > %d not supported", dim,
                  max_dim);
    const int kp = dim <= 64 ? 1 : (dim <= 128 ? 2 : 4);
    if (kp != u.kp)
      return fail(MB200_ERR_INVALID_ARG, "user constraint image has kp %d; dim %d needs kp %d",
                  u.kp, dim, kp);
    return launch.image(u);
  }
  const auto& launch_registry = launch.registry;
  switch (m.target_id) {
    case MB200_TARGET_TORUS:
      if (dim != 3) return fail(MB200_ERR_INVALID_ARG, "torus target needs dim == 3");
      return launch_registry(CsShape<TorusTarget, 1>{});
    case MB200_TARGET_SPHERE:
      if (dim <= 64) return launch_registry(CsShape<SphereTarget, 1>{});
      if (dim <= 128) return launch_registry(CsShape<SphereTarget, 2>{});
      if (dim <= 256) return launch_registry(CsShape<SphereTarget, 4>{});
      return fail(MB200_ERR_UNSUPPORTED, "sphere target: dim %d > 256 not supported", dim);
    case MB200_TARGET_MULTI_SPHERE: {
      const int nc = (int)m.tp[0];
      if ((nc != 2 && nc != 4 && nc != 8) || dim % nc != 0 || dim > 128)
        return fail(MB200_ERR_UNSUPPORTED,
                    "multi-sphere target: n_constr must be 2, 4 or 8, dim a multiple <= 128");
      if (dim <= 64) {
        if (nc == 2) return launch_registry(CsShape<MultiSphereTarget<2>, 1>{});
        if (nc == 4) return launch_registry(CsShape<MultiSphereTarget<4>, 1>{});
        return launch_registry(CsShape<MultiSphereTarget<8>, 1>{});
      }
      if (nc == 2) return launch_registry(CsShape<MultiSphereTarget<2>, 2>{});
      if (nc == 4) return launch_registry(CsShape<MultiSphereTarget<4>, 2>{});
      return launch_registry(CsShape<MultiSphereTarget<8>, 2>{});
    }
    default:
      return fail(MB200_ERR_UNSUPPORTED, "target %d defines no constraint", m.target_id);
  }
}

// Argument checks shared by the plain and the Gaussian-split entry points (the torus one-thread
// kernel serves the plain system's Hausdorff density only).
template <bool GAUSS>
static int constrained_leapfrog_dispatch(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, int32_t n_inner_step, int32_t metric_kind,
    const double* metric_inv, const GaussianArgs& ga, const mb200_model* model,
    int32_t projection_solver, double constraint_tol, double position_tol, double divergence_tol,
    int32_t max_iters, int32_t max_line_search_iters, double reverse_check_tol, double* h_out,
    int32_t* status, int32_t* n_done, int32_t* newton_iters, void* stream,
    const void* user_target = nullptr) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos_in || !mom_in || !pos_out || !mom_out || !model)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1 || n_steps < 0 || n_inner_step < 1 || max_iters < 0 ||
      max_line_search_iters < 0)
    return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (projection_solver < 0 || projection_solver > 2)
    return fail(MB200_ERR_INVALID_ARG, "unknown projection solver %d", projection_solver);
  if (metric_kind < 0 || metric_kind > 2) return fail(MB200_ERR_INVALID_ARG, "bad metric_kind");
  if (metric_kind != MB200_METRIC_IDENTITY && !metric_inv)
    return fail(MB200_ERR_INVALID_ARG, "metric_inv is NULL");
  if (GAUSS && !ga.omega) return fail(MB200_ERR_INVALID_ARG, "metric_omega is NULL");
  if (GAUSS && metric_kind == MB200_METRIC_DENSE && (!ga.eigvec || !ga.eigvec_t))
    return fail(MB200_ERR_INVALID_ARG, "metric_eigvec / metric_eigvec_t is NULL");
  if (n_chains == 0) return 0;
  const DeviceScope device_scope(pos_in);
  const ModelArgs m = to_args(model, step_sizes, n_steps_per_chain);
  cudaStream_t st = (cudaStream_t)stream;
  // config C3: torus, identity metric, Newton projection, Hausdorff density -> one THREAD per chain
  if (!GAUSS && m.target_id == MB200_TARGET_TORUS && dim == 3 &&
      metric_kind == MB200_METRIC_IDENTITY && projection_solver == MB200_PROJ_SOLVER_NEWTON &&
      m.tp[MB200_MAX_PARAMS - 1] == 0.0) {
    // latency bound per chain: spread small batches over as many warps as there are
    // sub-partitions (measured: 8 lanes per warp 0.287 ms, 32 lanes 0.300 ms at 4096 chains)
    const int lanes = n_chains >= (int64_t)num_sms() * 4 * 32 ? 32 : 8;
    constrained_torus_thread_kernel<<<cs_blocks(n_chains, lanes), 32, 0, st>>>(
        pos_in, mom_in, pos_out, mom_out, dir, n_chains, step_size, n_steps, n_inner_step, m,
        constraint_tol, position_tol, divergence_tol, max_iters, reverse_check_tol, h_out, status,
        n_done, newton_iters, lanes);
    return check_launch("constrained_torus_thread_kernel");
  }
  auto registry = [&](auto shape) {
    using S = decltype(shape);
    constrained_leapfrog_kernel<typename S::Target, S::KP, GAUSS>
        <<<cs_blocks(n_chains, CS_WARPS), CS_WARPS * 32, S::template smem<GAUSS>(), st>>>(
            pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, n_steps,
            n_inner_step, metric_kind, metric_inv, m, constraint_tol, position_tol,
            divergence_tol, max_iters, reverse_check_tol, h_out, status, n_done, newton_iters,
            projection_solver, max_line_search_iters, ga.omega, ga.eigvec, ga.eigvec_t);
    return check_launch("constrained_leapfrog_kernel");
  };
  auto image = [&](const UserConstraintKernels& u) {
    // the Lebesgue density's gradient and the Gaussian system run the matrix-Hessian product
    if (!u.mhp_constr && (GAUSS || m.tp[MB200_MAX_PARAMS - 1] != 0.0))
      return fail(MB200_ERR_INVALID_ARG,
                  "user constraint defines no mhp_constr, which the %s needs",
                  GAUSS ? "Gaussian system" : "Lebesgue density");
    using Kernel = decltype(&constrained_leapfrog_kernel<SphereTarget, 1, GAUSS>);
    return eu_launch(reinterpret_cast<Kernel>(u.leapfrog[GAUSS]), "constrained_leapfrog_kernel",
                     (n_chains + CS_WARPS - 1) / CS_WARPS, 16, CS_WARPS * 32,
                     cs_user_smem<GAUSS>(u), st, pos_in, mom_in, pos_out, mom_out, dir, n_chains,
                     dim, step_size, n_steps, n_inner_step, metric_kind, metric_inv, m,
                     constraint_tol, position_tol, divergence_tol, max_iters, reverse_check_tol,
                     h_out, status, n_done, newton_iters, projection_solver,
                     max_line_search_iters, ga.omega, ga.eigvec, ga.eigvec_t);
  };
  return constrained_target_dispatch(m, dim, cs_launch(user_target, registry, image));
}

template <bool GAUSS>
static int project_dispatch(const double* pos, const double* mom_in, double* mom_out,
                            int64_t n_chains, int32_t dim, int32_t metric_kind,
                            const double* metric_inv, const mb200_model* model, void* stream,
                            const void* user_target = nullptr) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos || !mom_in || !mom_out || !model) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (metric_kind < 0 || metric_kind > 2) return fail(MB200_ERR_INVALID_ARG, "bad metric_kind");
  if (metric_kind != MB200_METRIC_IDENTITY && !metric_inv)
    return fail(MB200_ERR_INVALID_ARG, "metric_inv is NULL");
  const DeviceScope device_scope(pos);
  const ModelArgs m = to_args(model);
  auto registry = [&](auto shape) {
    using S = decltype(shape);
    constrained_project_kernel<typename S::Target, S::KP, GAUSS>
        <<<cs_blocks(n_chains, CS_WARPS), CS_WARPS * 32, S::template smem<GAUSS>(),
           (cudaStream_t)stream>>>(pos, mom_in, mom_out, n_chains, dim, metric_kind, metric_inv, m);
    return check_launch("constrained_project_kernel");
  };
  auto image = [&](const UserConstraintKernels& u) {
    using Kernel = decltype(&constrained_project_kernel<SphereTarget, 1, GAUSS>);
    return eu_launch(reinterpret_cast<Kernel>(u.project[GAUSS]), "constrained_project_kernel",
                     (n_chains + CS_WARPS - 1) / CS_WARPS, 16, CS_WARPS * 32,
                     cs_user_smem<GAUSS>(u), (cudaStream_t)stream, pos, mom_in, mom_out, n_chains,
                     dim, metric_kind, metric_inv, m);
  };
  return constrained_target_dispatch(m, dim, cs_launch(user_target, registry, image));
}

}  // namespace mb200

using namespace mb200;

extern "C" {

int mb200_constrained_leapfrog_euclidean(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, int32_t n_inner_step, int32_t metric_kind,
    const double* metric_inv, const mb200_model* model, int32_t projection_solver,
    double constraint_tol, double position_tol, double divergence_tol, int32_t max_iters,
    int32_t max_line_search_iters, double reverse_check_tol, double* h_out, int32_t* status,
    int32_t* n_done, int32_t* newton_iters, void* stream) {
  return constrained_leapfrog_dispatch<false>(
      pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, step_sizes, n_steps,
      n_steps_per_chain, n_inner_step, metric_kind, metric_inv, GaussianArgs{nullptr, nullptr, nullptr},
      model, projection_solver, constraint_tol, position_tol, divergence_tol, max_iters,
      max_line_search_iters, reverse_check_tol, h_out, status, n_done, newton_iters, stream);
}

int mb200_constrained_leapfrog_gaussian_euclidean(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, int32_t n_inner_step, int32_t metric_kind,
    const double* metric_inv, const double* metric_omega, const double* metric_eigvec,
    const double* metric_eigvec_t, const mb200_model* model, int32_t projection_solver,
    double constraint_tol, double position_tol, double divergence_tol, int32_t max_iters,
    int32_t max_line_search_iters, double reverse_check_tol, double* h_out, int32_t* status,
    int32_t* n_done, int32_t* newton_iters, void* stream) {
  return constrained_leapfrog_dispatch<true>(
      pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, step_sizes, n_steps,
      n_steps_per_chain, n_inner_step, metric_kind, metric_inv,
      GaussianArgs{metric_omega, metric_eigvec, metric_eigvec_t}, model, projection_solver,
      constraint_tol, position_tol, divergence_tol, max_iters, max_line_search_iters,
      reverse_check_tol, h_out, status, n_done, newton_iters, stream);
}

int mb200_project_onto_cotangent_space(const double* pos, const double* mom_in, double* mom_out,
                                       int64_t n_chains, int32_t dim, int32_t metric_kind,
                                       const double* metric_inv, const mb200_model* model,
                                       void* stream) {
  return project_dispatch<false>(pos, mom_in, mom_out, n_chains, dim, metric_kind, metric_inv,
                                 model, stream);
}

int mb200_project_onto_cotangent_space_gaussian(const double* pos, const double* mom_in,
                                                double* mom_out, int64_t n_chains, int32_t dim,
                                                int32_t metric_kind, const double* metric_inv,
                                                const mb200_model* model, void* stream) {
  return project_dispatch<true>(pos, mom_in, mom_out, n_chains, dim, metric_kind, metric_inv,
                                model, stream);
}

int mb200_constrained_leapfrog_euclidean_user(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, int32_t n_inner_step, int32_t metric_kind,
    const double* metric_inv, const mb200_model* model, int32_t projection_solver,
    double constraint_tol, double position_tol, double divergence_tol, int32_t max_iters,
    int32_t max_line_search_iters, double reverse_check_tol, double* h_out, int32_t* status,
    int32_t* n_done, int32_t* newton_iters, void* stream, const void* user_target) {
  if (!user_target) return fail(MB200_ERR_INVALID_ARG, "user_target is NULL");
  return constrained_leapfrog_dispatch<false>(
      pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, step_sizes, n_steps,
      n_steps_per_chain, n_inner_step, metric_kind, metric_inv, GaussianArgs{nullptr, nullptr, nullptr},
      model, projection_solver, constraint_tol, position_tol, divergence_tol, max_iters,
      max_line_search_iters, reverse_check_tol, h_out, status, n_done, newton_iters, stream,
      user_target);
}

int mb200_constrained_leapfrog_gaussian_euclidean_user(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, int32_t n_inner_step, int32_t metric_kind,
    const double* metric_inv, const double* metric_omega, const double* metric_eigvec,
    const double* metric_eigvec_t, const mb200_model* model, int32_t projection_solver,
    double constraint_tol, double position_tol, double divergence_tol, int32_t max_iters,
    int32_t max_line_search_iters, double reverse_check_tol, double* h_out, int32_t* status,
    int32_t* n_done, int32_t* newton_iters, void* stream, const void* user_target) {
  if (!user_target) return fail(MB200_ERR_INVALID_ARG, "user_target is NULL");
  return constrained_leapfrog_dispatch<true>(
      pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size, step_sizes, n_steps,
      n_steps_per_chain, n_inner_step, metric_kind, metric_inv,
      GaussianArgs{metric_omega, metric_eigvec, metric_eigvec_t}, model, projection_solver,
      constraint_tol, position_tol, divergence_tol, max_iters, max_line_search_iters,
      reverse_check_tol, h_out, status, n_done, newton_iters, stream, user_target);
}

int mb200_project_onto_cotangent_space_user(const double* pos, const double* mom_in,
                                            double* mom_out, int64_t n_chains, int32_t dim,
                                            int32_t metric_kind, const double* metric_inv,
                                            const mb200_model* model, void* stream,
                                            const void* user_target) {
  if (!user_target) return fail(MB200_ERR_INVALID_ARG, "user_target is NULL");
  return project_dispatch<false>(pos, mom_in, mom_out, n_chains, dim, metric_kind, metric_inv,
                                 model, stream, user_target);
}

int mb200_project_onto_cotangent_space_gaussian_user(const double* pos, const double* mom_in,
                                                     double* mom_out, int64_t n_chains,
                                                     int32_t dim, int32_t metric_kind,
                                                     const double* metric_inv,
                                                     const mb200_model* model, void* stream,
                                                     const void* user_target) {
  if (!user_target) return fail(MB200_ERR_INVALID_ARG, "user_target is NULL");
  return project_dispatch<true>(pos, mom_in, mom_out, n_chains, dim, metric_kind, metric_inv,
                                model, stream, user_target);
}

}  // extern "C"
