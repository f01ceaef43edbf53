/*
 * mici_b200.h -- C ABI of libmici_b200.so: batched-chain Hamiltonian integrator steps on
 * NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary for ONE hot path of matt-graham/mici: `Integrator.step`
 * evaluated over many independent chains.  Each entry point replaces the per-chain Python
 * call chain named in its comment (paths relative to the reference tree).  The reference is
 * pure Python with no FFI; a maintainer binds these with `ctypes` (see INTEGRATION.md).
 *
 * Conventions
 *  - All array pointers are DEVICE pointers (e.g. torch.Tensor.data_ptr()), fp64, row-major
 *    `[n_chains x dim]`, 16-byte aligned.  `target_params` is a HOST pointer (<= 8 doubles,
 *    copied by value into the launch).
 *  - `dir` may be NULL (all chains +1) or int32[n_chains] with entries +-1; the signed time
 *    step of a chain is `dir * step_size` (integrators.py:79).
 *  - Integrator entry points take `double step_size, const double* step_sizes, int32_t n_steps,
 *    const int32_t* n_steps_per_chain`.  `step_sizes` is NULL or a device array [n_chains]: when
 *    given, chain c uses step_sizes[c] instead of step_size (during warm-up every chain carries
 *    its own dual-averaging step size: adapters.py:262-283, 373; the initial coarse search halves
 *    / doubles it chain by chain: adapters.py:285-343).  `n_steps_per_chain` is NULL or a device
 *    array [n_chains]: when given, chain c takes min(n_steps_per_chain[c], n_steps) steps
 *    (MetropolisRandomIntegrationTransition, transitions.py:355-412).
 *  - Out-of-place: `*_out` may alias `*_in` (in-place) or be distinct buffers, so that
 *    `Integrator.step` keeps its "returns a new state, argument untouched" contract
 *    (integrators.py:78-80, tests/test_integrators.py:110-124) without an extra copy.
 *  - Return value: 0 = launched, <0 = argument / launch error (message via
 *    mb200_last_error()).  Never throws.  Launches are asynchronous on `stream`
 *    (a cudaStream_t passed as void*; NULL = legacy default stream).
 *  - Per-chain outcome replaces the reference's exceptions (errors.py:10-27):
 *    `status[i]` is one of MB200_STATUS_*; a chain whose step fails keeps the state it had
 *    BEFORE the failing step and takes no further steps in that launch (the reference's
 *    transitions abort the trajectory on IntegratorError: transitions.py:292-295).
 *    `n_done[i]` (optional) counts completed steps.
 *  - Re-entrant: no global mutable state apart from a thread-local error string.
 */
#ifndef MICI_B200_H
#define MICI_B200_H

#ifndef __CUDACC_RTC__
#include <stdint.h>
#else /* NVRTC (user targets, mici_b200/jit.py): no system headers; LP64 integer types */
typedef int int32_t;
typedef unsigned int uint32_t;
typedef long int64_t;
typedef unsigned long uint64_t;
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define MB200_VERSION 101

/* per-chain status codes */
#define MB200_STATUS_OK 0
#define MB200_STATUS_CONVERGENCE 1    /* mici.errors.ConvergenceError      */
#define MB200_STATUS_NON_REVERSIBLE 2 /* mici.errors.NonReversibleStepError */
#define MB200_STATUS_LINALG 3         /* mici.errors.LinAlgError            */

/* error returns */
#define MB200_ERR_INVALID_ARG (-1)
#define MB200_ERR_UNSUPPORTED (-2)
#define MB200_ERR_CUDA (-3)

/* fixed metric of a Euclidean system (systems.py:332-346 coercion) */
#define MB200_METRIC_IDENTITY 0 /* metric_inv ignored                         */
#define MB200_METRIC_DIAGONAL 1 /* metric_inv = 1/diag, [dim]                 */
#define MB200_METRIC_DENSE 2    /* metric_inv = explicit dense M^-1, [dim*dim] */

/* closed registry of target models compiled into the library (SURVEY.md 7.6) */
#define MB200_TARGET_STD_GAUSSIAN 0 /* l = |q|^2/2                      params: -            */
#define MB200_TARGET_NEAL_FUNNEL 1  /* Neal's funnel                    params: -            */
#define MB200_TARGET_BANANA 2       /* paired banana                    params: b            */
#define MB200_TARGET_QUADRATIC 3    /* l = q^T P q / 2                  aux: P [dim*dim]     */
#define MB200_TARGET_TORUS 4        /* density on torus (README:315-337) params: R, r, alpha */
#define MB200_TARGET_SPHERE 5       /* tilted density on unit sphere    params: -            */
#define MB200_TARGET_MULTI_SPHERE 6 /* n_constr unit spheres on consecutive blocks  params: n_constr (2, 4 or 8) */
#define MB200_TARGET_QUARTIC 7      /* l = |q|^2/2 + gamma/4 sum_m (a_m.q)^4   params: gamma; aux: A [dim*dim] (dense Hessian; SoftAbs systems) */
/* a user-written target compiled at run time (mb200_user_target_load); only the *_user entry
 * points accept it, every registry entry point rejects it as an unknown target */
#define MB200_TARGET_USER 64
/* constrained targets: target_params[MB200_MAX_PARAMS - 1] != 0 means the density is given with
 * respect to the Lebesgue measure (dens_wrt_hausdorff=False, systems.py:853-861): h1 and dh1_dpos
 * carry log det gram / 2 and its gradient (systems.py:1024-1031) */

/* position-dependent metrics of Riemannian systems */
#define MB200_RMETRIC_SOFTABS 0 /* SoftAbs of target Hessian (matrices.py:1631-1685); params: softabs_coeff */
#define MB200_RMETRIC_RANK1 1   /* dense M(q) = B + c q q^T;  aux: [B | B^-1] (2*dim*dim), params: c, log|B|, force_woodbury, generic_rank1_vjp */
#define MB200_RMETRIC_HADAMARD 2 /* dense M(q) = B + c (q q^T) o S (full rank); aux: [B | S] (2*dim*dim), params: c, -, -, generic_rank1_vjp */
/* O(D) metrics (DiagonalRiemannianMetricSystem / ScalarRiemannianMetricSystem, systems.py:1405-1571);
 * targets: std-Gaussian, banana, funnel, quadratic (the funnel Fisher metric: funnel only) */
#define MB200_RMETRIC_DIAG_QUADRATIC 3     /* diagonal d_i = a + b q_i^2;  params: a > 0, b >= 0 */
#define MB200_RMETRIC_DIAG_FUNNEL_FISHER 4 /* diagonal d = [1/9 + (D-1)/2, e^-v, ..., e^-v], v = q[0]: the funnel's expected Fisher information */
#define MB200_RMETRIC_SCALAR_QUADRATIC 5   /* scaled identity s I, s = a + b |q|^2;  params: a > 0, b >= 0 */
/* Cholesky-factored metric M = L L^T given by its lower factor (CholeskyFactoredRiemannianMetricSystem,
 * systems.py:1574-1653); targets: std-Gaussian, banana, funnel, quadratic */
#define MB200_RMETRIC_CHOL_QUADRATIC 6 /* L(q) = L0 + c tril(q q^T);  aux: L0 [dim*dim] row-major, upper triangle zero (never read), params: c */
/* user-written diagonal / scalar / dense / Cholesky-factored metrics compiled at run time with a user target
 * (mb200_user_riemannian_load); only the Riemannian *_user entry points accept them, every registry
 * entry point rejects them as an unknown rmetric_id.  params / aux: the metric's own */
#define MB200_RMETRIC_USER_DIAGONAL 32
#define MB200_RMETRIC_USER_SCALAR 33
#define MB200_RMETRIC_USER_DENSE 34 /* global-workspace dense policy: dim <= 576, no implicit midpoint */
#define MB200_RMETRIC_USER_CHOLESKY 35 /* triangular-factored policy: dim <= 1016 */

/* fixed-point solvers fused into the implicit integrators (solvers.py:47-94, 97-154) */
#define MB200_FP_SOLVER_DIRECT 0
#define MB200_FP_SOLVER_STEFFENSEN 1

/* projection solvers fused into the constrained integrator (solvers.py:346-469, 195-343, 472-614) */
#define MB200_PROJ_SOLVER_NEWTON 0
#define MB200_PROJ_SOLVER_QUASI_NEWTON 1
#define MB200_PROJ_SOLVER_NEWTON_LINE_SEARCH 2

#define MB200_MAX_PARAMS 8

typedef struct mb200_model {
  int32_t target_id;                       /* MB200_TARGET_*                              */
  int32_t n_target_params;
  double target_params[MB200_MAX_PARAMS];
  const double* target_aux;                /* device pointer or NULL                      */
  int32_t rmetric_id;                      /* MB200_RMETRIC_* (Riemannian entry points)   */
  int32_t n_rmetric_params;
  double rmetric_params[MB200_MAX_PARAMS];
  const double* rmetric_aux;               /* device pointer or NULL                      */
} mb200_model;

int mb200_version(void);
const char* mb200_last_error(void);

/*
 * Call counters -- the device-side counterpart of ChainState._call_counts (states.py:44-72,
 * 160-300: every memoised system method bumps a counter that the samplers report).
 * `counters` is a device array [n_chains][MB200_N_COUNTERS] of int32 (or NULL to switch the
 * counting off).  Every later integrator launch issued FROM THE CALLING THREAD adds, per chain,
 * what that chain evaluated during the launch (rejected step attempts included, the optional
 * h_out energy evaluation excluded):
 *   MB200_COUNT_GRAD          grad_neg_log_dens evaluations
 *   MB200_COUNT_METRIC        Riemannian systems: metric builds (Cholesky factorisations /
 *                             eigendecompositions); constrained systems: constraint-Jacobian
 *                             evaluations; 0 otherwise
 *   MB200_COUNT_QUAD_VJP      VJPs of the quadratic form p.M(q)^-1 p (Riemannian systems)
 *   MB200_COUNT_SOLVER_ITERS  fixed-point / Newton iterations, summed over all steps
 * The counts are accumulated (+=): zero the array to start a new tally.
 */
#define MB200_N_COUNTERS 4
#define MB200_COUNT_GRAD 0
#define MB200_COUNT_METRIC 1
#define MB200_COUNT_QUAD_VJP 2
#define MB200_COUNT_SOLVER_ITERS 3
int mb200_set_call_counters(int32_t* counters);

/*
 * n_steps explicit leapfrog steps on a Euclidean-metric system, fused gradient.
 * Replaces: LeapfrogIntegrator.step/_step (integrators.py:63-80, 170-173) +
 *           System.h1_flow/dh1_dpos/grad_neg_log_dens (systems.py:109-152) +
 *           EuclideanMetricSystem.h2_flow/dh2_dmom (systems.py:352-363) +
 *           explicit-inverse matvec (matrices.py:222-226, 1183-1188).
 * "Next" row N4: symmetric composition (splitting) integrators --
 * SymmetricCompositionIntegrator and the BCSS 2/3/4-stage schemes (integrators.py:176-378):
 *   coefficients  NULL: the leapfrog schedule {0.5, 1, 0.5} (n_flows / initial_h1_flow_step are
 *                 ignored).  Else a HOST array of the full symmetric sequence of n_flows (odd)
 *                 coefficients (integrators.py:268-277): each step applies the alternating flows
 *                 a, b, a, ..., a over coefficients[i] * dt, a = h1_flow (kick) if
 *                 initial_h1_flow_step else h2_flow (drift).
 * h_out (optional, [n_chains]): Hamiltonian of the returned state (systems.py:187-196,348-350).
 * n_done[c] receives the number of steps chain c took.  With a dense metric, the leapfrog
 * schedule, n_steps_per_chain == NULL and n_steps > 0 it runs on the tensor-core kernel (which
 * applies per-chain step sizes on the momentum side: tile s = eps_c * dir * p against the
 * unscaled metric); otherwise on the general-dimension kernel.
 */
int mb200_leapfrog_euclidean(const double* pos_in, const double* mom_in, double* pos_out,
                             double* mom_out, const int32_t* dir, int64_t n_chains, int32_t dim,
                             double step_size, const double* step_sizes, int32_t n_steps,
                             const int32_t* n_steps_per_chain, int32_t n_flows,
                             const double* coefficients, int32_t initial_h1_flow_step,
                             int32_t metric_kind, const double* metric_inv,
                             const mb200_model* model, double* h_out, int32_t* status,
                             int32_t* n_done, void* stream);

/* Diagnostic: identical contract, but always through the general-dimension kernel (never the
 * tensor-core kernel); used by the tests to cross-check the two implementations. */
int mb200_leapfrog_euclidean_generic(const double* pos_in, const double* mom_in, double* pos_out,
                                     double* mom_out, const int32_t* dir, int64_t n_chains,
                                     int32_t dim, double step_size, const double* step_sizes,
                                     int32_t n_steps, const int32_t* n_steps_per_chain,
                                     int32_t n_flows, const double* coefficients,
                                     int32_t initial_h1_flow_step, int32_t metric_kind,
                                     const double* metric_inv, const mb200_model* model,
                                     double* h_out, int32_t* status, int32_t* n_done,
                                     void* stream);

/* Hamiltonian h = l(q) + p.M^-1 p / 2 of a Euclidean-metric system (systems.py:187-196, 348-350). */
int mb200_hamiltonian_euclidean(const double* pos, const double* mom, int64_t n_chains,
                                int32_t dim, int32_t metric_kind, const double* metric_inv,
                                const mb200_model* model, double* h_out, void* stream);

/*
 * Individual Euclidean-system quantities for callers outside `Integrator.step`
 * (System.neg_log_dens / grad_neg_log_dens: systems.py:97-119; dh2_dmom / h2: systems.py:348-354).
 * Any of nld_out [n], grad_out [n*dim], vel_out [n*dim] (= M^-1 p), kin_out [n] (= p.M^-1 p/2)
 * may be NULL.
 */
int mb200_euclidean_eval(const double* pos, const double* mom, int64_t n_chains, int32_t dim,
                         int32_t metric_kind, const double* metric_inv, const mb200_model* model,
                         double* nld_out, double* grad_out, double* vel_out, double* kin_out,
                         void* stream);

/*
 * User-written targets (mici_b200/csrc/user_target.cuh): a model's two device functions compiled
 * at run time, by NVRTC, together with the general-dimension Euclidean kernels.
 *  - mb200_user_target_load: loads a CUBIN `image` of `image_bytes` (cudaLibraryLoadData; the
 *    kernels are device-independent) and looks up its `n_names` = 10 kernels by their lowered
 *    names, in this order: leapfrog_generic_kernel<UserTarget, KP, CPW, false> for (KP, CPW) =
 *    (1, 4), (2, 4), (4, 2), (8, 1), (16, 1), then euclidean_eval_kernel<UserTarget, KP> for
 *    KP = 1, 2, 4, 8, 16.  *handle receives the loaded target.
 *  - mb200_user_target_unload: releases a handle.
 *  - mb200_leapfrog_euclidean_user, mb200_hamiltonian_euclidean_user, mb200_euclidean_eval_user:
 *    the same contracts as mb200_leapfrog_euclidean (always on the general-dimension kernel),
 *    mb200_hamiltonian_euclidean and mb200_euclidean_eval, for model->target_id ==
 *    MB200_TARGET_USER and the loaded `user_target`; dim <= 1024.
 * The library does not link NVRTC: compiling is the caller's job (mici_b200/jit.py).
 */
int mb200_user_target_load(const void* image, int64_t image_bytes, const char* const* names,
                           int32_t n_names, void** handle);
int mb200_user_target_unload(void* handle);
int mb200_leapfrog_euclidean_user(const double* pos_in, const double* mom_in, double* pos_out,
                                  double* mom_out, const int32_t* dir, int64_t n_chains,
                                  int32_t dim, double step_size, const double* step_sizes,
                                  int32_t n_steps, const int32_t* n_steps_per_chain,
                                  int32_t n_flows, const double* coefficients,
                                  int32_t initial_h1_flow_step, int32_t metric_kind,
                                  const double* metric_inv, const mb200_model* model,
                                  double* h_out, int32_t* status, int32_t* n_done, void* stream,
                                  const void* user_target);
int mb200_hamiltonian_euclidean_user(const double* pos, const double* mom, int64_t n_chains,
                                     int32_t dim, int32_t metric_kind, const double* metric_inv,
                                     const mb200_model* model, double* h_out, void* stream,
                                     const void* user_target);
int mb200_euclidean_eval_user(const double* pos, const double* mom, int64_t n_chains, int32_t dim,
                              int32_t metric_kind, const double* metric_inv,
                              const mb200_model* model, double* nld_out, double* grad_out,
                              double* vel_out, double* kin_out, void* stream,
                              const void* user_target);

/*
 * n_steps constrained (RATTLE / geodesic) leapfrog steps with Newton projection.
 * Replaces: ConstrainedLeapfrogIntegrator.step (integrators.py:929-984) +
 *           solve_projection_onto_manifold_{newton, quasi_newton, newton_with_line_search}
 *           (solvers.py:346-469, 195-343, 472-614; projection_solver = MB200_PROJ_SOLVER_*) +
 *           DenseConstrainedEuclideanMetricSystem methods (systems.py:786-873, 1006-1022),
 *           dens_wrt_hausdorff=True.
 * newton_iters (optional, [n_chains]): total Newton iterations used by the chain.
 */
int mb200_constrained_leapfrog_euclidean(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, int32_t n_inner_step, int32_t metric_kind,
    const double* metric_inv, const mb200_model* model, int32_t projection_solver,
    double constraint_tol, double position_tol, double divergence_tol, int32_t max_iters,
    int32_t max_line_search_iters, double reverse_check_tol, double* h_out, int32_t* status,
    int32_t* n_done, int32_t* newton_iters, void* stream);

/*
 * The same for GaussianDenseConstrainedEuclideanMetricSystem (systems.py:1034-1184): h2 =
 * q.q/2 + p.M^-1 p/2, whose flow is the exact rotation of (q, p) in the eigenbasis of M; the
 * projection solvers use dh2_flow_dmom(|dt|) = (U diag(sin(w|dt|) w) U^T, U diag(cos(w|dt|)) U^T);
 * the Gram matrices are inverted through their eigendecomposition (DenseSymmetricMatrix); the
 * density is always with respect to the Lebesgue measure.  With (eigval, U) the metric's
 * eigendecomposition:
 *   metric_omega    [dim] w = 1 / eigval^(1/2) (device; ones for the identity metric)
 *   metric_eigvec   [dim*dim] U, row-major (device; dense metric only, else NULL)
 *   metric_eigvec_t [dim*dim] U^T, row-major (device; dense metric only, else NULL)
 * sin(w |dt|) and cos(w |dt|) are evaluated per chain, so step_sizes may vary per chain with
 * every metric kind.  Other arguments, targets and sizes as for
 * mb200_constrained_leapfrog_euclidean.
 */
int mb200_constrained_leapfrog_gaussian_euclidean(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, int32_t n_inner_step, int32_t metric_kind,
    const double* metric_inv, const double* metric_omega, const double* metric_eigvec,
    const double* metric_eigvec_t, const mb200_model* model, int32_t projection_solver,
    double constraint_tol, double position_tol, double divergence_tol, int32_t max_iters,
    int32_t max_line_search_iters, double reverse_check_tol, double* h_out, int32_t* status,
    int32_t* n_done, int32_t* newton_iters, void* stream);

/*
 * n_steps implicit generalised-leapfrog steps on a Riemannian-metric system, fixed-point
 * solves by direct iteration.
 * Replaces: ImplicitLeapfrogIntegrator.step (integrators.py:482-544; NB every sub-map gets the
 *           full dir*step_size, SURVEY.md H3) + solve_fixed_point_direct / _steffensen
 *           (solvers.py:47-154, selected by fp_solver) +
 *           RiemannianMetricSystem derivatives (systems.py:1360-1402) +
 *           DensePositiveDefiniteMatrix / SoftAbsRegularizedPositiveDefiniteMatrix arithmetic
 *           (matrices.py:1161-1188, 1631-1685).
 * fp_iters (optional, [n_chains*4]): iterations of the four fixed-point solves of the LAST
 *           completed step.  workspace: device scratch of mb200_implicit_workspace_bytes().
 */
int mb200_implicit_leapfrog_riemannian(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, const mb200_model* model, int32_t fp_solver,
    double fp_convergence_tol, double fp_divergence_tol, int32_t fp_max_iters,
    double reverse_check_tol, double* h_out, int32_t* status, int32_t* n_done, int32_t* fp_iters,
    void* workspace, int64_t workspace_bytes, void* stream);

int64_t mb200_implicit_workspace_bytes(int64_t n_chains, int32_t dim, const mb200_model* model);

/* Hamiltonian of a Riemannian system: l(q) + log|M(q)|/2 + p.M(q)^-1 p / 2 (systems.py:1375-1390). */
int mb200_hamiltonian_riemannian(const double* pos, const double* mom, int64_t n_chains,
                                 int32_t dim, const mb200_model* model, double* h_out,
                                 int32_t* status, void* workspace, int64_t workspace_bytes,
                                 void* stream);

/*
 * "Next" row N1: Metropolis accept / reject of a static-HMC transition for all chains.
 * Replaces: MetropolisIntegrationTransition._sample_n_step, transitions.py:275-315 (the part
 * after the trajectory): accept_prob = exp(min(0, h_init - h_prop)) (0 if NaN, 0 if the
 * trajectory failed at its first step), accepted iff status == 0 and uniforms < accept_prob;
 * pos/mom are overwritten with the proposal where accepted; dir is negated where rejected
 * (:299, :314).  accept_prob / accept_stat / accepted may be NULL.
 */
int mb200_metropolis_select(double* pos, double* mom, const double* pos_prop,
                            const double* mom_prop, const double* h_init, const double* h_prop,
                            const int32_t* status, const int32_t* n_done, int32_t* dir,
                            const double* uniforms, int64_t n_chains, int32_t dim,
                            double* accept_prob, double* accept_stat, int32_t* accepted,
                            void* stream);

/*
 * Diagnostic: the fused fixed-point solvers (K4; fp_solver = MB200_FP_SOLVER_*:
 * solve_fixed_point_direct solvers.py:47-94, solve_fixed_point_steffensen :97-154) on the
 * reference's own known-answer problems
 * (reference tests/test_solvers.py:25-47): func_id 0 babylonian (y/x + x)/2, 1 ratio
 * (x+y)/(x+1), 2 cosine, 3 doubling 2x, 4 quadratic 1 + x^2; x0, y, x_out are [n*dim].
 */
int mb200_selftest_fixed_point(int32_t func_id, int32_t fp_solver, const double* x0,
                               const double* y, int64_t n, int32_t dim, double convergence_tol,
                               double divergence_tol, int32_t max_iters, double* x_out,
                               int32_t* iters_out, int32_t* status, void* stream);

/*
 * Diagnostic: the per-chain symmetric eigensolver (K3, parallel cyclic Jacobi; replaces
 * numpy.linalg.eigh at matrices.py:437, 1658) on arbitrary dense symmetric matrices
 * [n_matrices x dim x dim].  eigvec holds the eigenvectors as columns (row-major), eigval is
 * unsorted.  warm_from >= 0: each solve is warm-started from the eigenvectors of matrix
 * `warm_from` (the V^T H V path used between successive fixed-point iterates); -1: cold.
 */
int mb200_selftest_eigh(const double* matrices, int64_t n_matrices, int32_t dim, int32_t warm_from,
                        double* eigval, double* eigvec, int32_t* status, void* stream);

/*
 * Diagnostic: the blocked DMMA factorisation of the global-workspace dense metric policy
 * (csrc/dense_global.cuh) on arbitrary SPD matrices [n_matrices*dim*dim], one CTA per matrix:
 * lower Cholesky factor, explicit inverse, solution of M x = rhs and log|M| -- the operations of
 * DensePositiveDefiniteMatrix (matrices.py:1161-1188, 982-984) that tests compare with
 * numpy.linalg.  status 3 where the factorisation fails.
 */
int mb200_selftest_dense_factor(const double* matrices, const double* rhs, int64_t n_matrices,
                                int32_t dim, double* chol_out, double* inv_out, double* sol_out,
                                double* logdet_out, int32_t* status, void* stream);

/*
 * Diagnostic: y[i] = exp(x[i]) as the tensor-core leapfrog evaluates it (the funnel's exp(-v) in
 * K1: a short-chain polynomial for |x| < 700, libm's exp otherwise), one element per thread in
 * warps of 32 consecutive elements; x and y are device arrays [n].
 */
int mb200_selftest_exp_short_chain(const double* x, double* y, int64_t n, void* stream);

/*
 * "Next" row N4: n_steps implicit-midpoint steps on a Riemannian-metric system.
 * Replaces: ImplicitMidpointIntegrator.step (integrators.py:547-681): a direct fixed-point solve
 * in z = (q, p) for the forward half-step, an explicit Euler half-step, and a reversibility
 * check by a second fixed-point solve.  fp_iters (optional, [n_chains*4]): iterations of the two
 * solves of the last completed step in slots 0 and 1.  Other arguments as for
 * mb200_implicit_leapfrog_riemannian.
 */
int mb200_implicit_midpoint_riemannian(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, const mb200_model* model, int32_t fp_solver,
    double fp_convergence_tol, double fp_divergence_tol, int32_t fp_max_iters,
    double reverse_check_tol, double* h_out, int32_t* status, int32_t* n_done, int32_t* fp_iters,
    void* stream);

/*
 * Momentum refresh for the non-Euclidean systems (row N1).
 *  - mb200_project_onto_cotangent_space: p -= J^T (J M^-1 J^T)^-1 J M^-1 p for every chain
 *    (ConstrainedEuclideanMetricSystem.project_onto_cotangent_space, systems.py:863-873; the
 *    second half of ConstrainedTractableFlowSystem.sample_momentum, systems.py:613-616).
 *  - mb200_sample_momentum_riemannian: mom = sqrt(M(q)) z (RiemannianMetricSystem.sample_momentum,
 *    systems.py:1401-1402; sqrt = U sqrt(softabs) U^T for SoftAbs, the Cholesky factor for dense
 *    metrics); `normals` are standard-normal variates [n*dim]; status 3 where M(q) cannot be built.
 */
int mb200_project_onto_cotangent_space(const double* pos, const double* mom_in, double* mom_out,
                                       int64_t n_chains, int32_t dim, int32_t metric_kind,
                                       const double* metric_inv, const mb200_model* model,
                                       void* stream);
/* The same projection with the Gram matrix inverted through its eigendecomposition, as
 * GaussianDenseConstrainedEuclideanMetricSystem does (systems.py:1157-1169). */
int mb200_project_onto_cotangent_space_gaussian(const double* pos, const double* mom_in,
                                                double* mom_out, int64_t n_chains, int32_t dim,
                                                int32_t metric_kind, const double* metric_inv,
                                                const mb200_model* model, void* stream);

/*
 * User-written constraints (mici_b200/csrc/user_constraint.cuh): a model's target and constraint
 * device functions compiled at run time, by NVRTC, together with the Euclidean kernels of
 * mb200_user_target_load and the constrained leapfrog and projection kernels.
 *  - mb200_user_constraint_load: as mb200_user_target_load, for an image of `n_names` = 14
 *    kernels: the 10 of mb200_user_target_load, then, with T = UserConstrainedTarget,
 *    constrained_leapfrog_kernel<T, kp, false>, constrained_leapfrog_kernel<T, kp, true>,
 *    constrained_project_kernel<T, kp, false>, constrained_project_kernel<T, kp, true>.
 *    n_constr (1 .. 8) and kp (1, 2 or 4) are those the image was compiled for; mhp_constr != 0
 *    when it defines mhp_constr.  The handle also serves the Euclidean *_user entry points and is
 *    released by mb200_user_target_unload.
 *  - mb200_constrained_leapfrog_euclidean_user, mb200_constrained_leapfrog_gaussian_euclidean_user,
 *    mb200_project_onto_cotangent_space_user, mb200_project_onto_cotangent_space_gaussian_user:
 *    the contracts of the entry points without `_user`, for model->target_id ==
 *    MB200_TARGET_USER and a `user_target` from mb200_user_constraint_load.  dim <= 256 with one
 *    constraint, dim <= 128 with several, and dim must select the image's kp (1: dim <= 64,
 *    2: dim <= 128, 4: dim <= 256).  The Lebesgue density and the Gaussian system need an image
 *    with mhp_constr.
 */
int mb200_user_constraint_load(const void* image, int64_t image_bytes, const char* const* names,
                               int32_t n_names, int32_t n_constr, int32_t kp, int32_t mhp_constr,
                               void** handle);
int mb200_constrained_leapfrog_euclidean_user(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, int32_t n_inner_step, int32_t metric_kind,
    const double* metric_inv, const mb200_model* model, int32_t projection_solver,
    double constraint_tol, double position_tol, double divergence_tol, int32_t max_iters,
    int32_t max_line_search_iters, double reverse_check_tol, double* h_out, int32_t* status,
    int32_t* n_done, int32_t* newton_iters, void* stream, const void* user_target);
int mb200_constrained_leapfrog_gaussian_euclidean_user(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, int32_t n_inner_step, int32_t metric_kind,
    const double* metric_inv, const double* metric_omega, const double* metric_eigvec,
    const double* metric_eigvec_t, const mb200_model* model, int32_t projection_solver,
    double constraint_tol, double position_tol, double divergence_tol, int32_t max_iters,
    int32_t max_line_search_iters, double reverse_check_tol, double* h_out, int32_t* status,
    int32_t* n_done, int32_t* newton_iters, void* stream, const void* user_target);
int mb200_project_onto_cotangent_space_user(const double* pos, const double* mom_in,
                                            double* mom_out, int64_t n_chains, int32_t dim,
                                            int32_t metric_kind, const double* metric_inv,
                                            const mb200_model* model, void* stream,
                                            const void* user_target);
int mb200_project_onto_cotangent_space_gaussian_user(const double* pos, const double* mom_in,
                                                     double* mom_out, int64_t n_chains,
                                                     int32_t dim, int32_t metric_kind,
                                                     const double* metric_inv,
                                                     const mb200_model* model, void* stream,
                                                     const void* user_target);

int mb200_sample_momentum_riemannian(const double* pos, const double* normals, double* mom_out,
                                     int64_t n_chains, int32_t dim, const mb200_model* model,
                                     int32_t* status, void* stream);

/*
 * RiemannianMetricSystem.dh2_dmom / System.dh_dmom (systems.py:1398-1399, 202-207): the velocity
 * M(q)^-1 p of every chain, read by the no-U-turn criteria (transitions.py:434-435, 472-473).
 * status 3 (and NaN velocities) where M(q) cannot be built.
 */
int mb200_dh_dmom_riemannian(const double* pos, const double* mom, double* vel_out,
                             int64_t n_chains, int32_t dim, const mb200_model* model,
                             int32_t* status, void* stream);

/*
 * User-written targets and metrics on the diagonal, scalar, dense and Cholesky-factored Riemannian
 * systems (mici_b200/csrc/user_riemannian.cuh): a user target and a user diagonal, scalar, dense
 * or Cholesky-factored metric compiled at run time, by NVRTC, together with the Riemannian kernels
 * of the compact policies, of the triangular-factored policy or of the global-workspace dense
 * policy (mici_b200/csrc/dense_global.cuh).
 *  - mb200_user_riemannian_load: loads a CUBIN `image` of `n_names` = 3 kernels, with
 *    T = UserRTarget and M = UserDiagonalMetric (rmetric_id MB200_RMETRIC_USER_DIAGONAL) or
 *    UserScalarMetric (MB200_RMETRIC_USER_SCALAR), or T = UserRTargetCta and M = UserDenseMetric
 *    (MB200_RMETRIC_USER_DENSE) or UserCholeskyMetric (MB200_RMETRIC_USER_CHOLESKY):
 *    implicit_leapfrog_kernel<T, M>,
 *    riemannian_velocity_kernel<T, M>, riemannian_sample_momentum_kernel<T, M>.  The handle is
 *    released by mb200_user_target_unload.  It serves only the Riemannian *_user entry points;
 *    the Euclidean and constrained ones refuse it, and these refuse every other handle.
 *  - mb200_implicit_leapfrog_riemannian_user, mb200_implicit_midpoint_riemannian_user,
 *    mb200_hamiltonian_riemannian_user, mb200_sample_momentum_riemannian_user,
 *    mb200_dh_dmom_riemannian_user: the contracts of the entry points without `_user`, for
 *    model->target_id == MB200_TARGET_USER, model->rmetric_id == the handle's rmetric_id and a
 *    `user_image` from mb200_user_riemannian_load; anything else is MB200_ERR_INVALID_ARG and
 *    launches nothing.  No workspace is needed for the diagonal and scalar metrics
 *    (mb200_implicit_workspace_bytes returns 0).
 *  - A dense image runs on the launch plan of the global-workspace dense policy: one CTA of 256
 *    threads per SM, the per-CTA D x D matrices in `workspace` (mb200_implicit_workspace_bytes
 *    bytes; less or NULL: a stream-ordered allocation for the call).  Refused before any launch:
 *    the implicit midpoint (MB200_ERR_UNSUPPORTED, as for the registry Hadamard metric) and
 *    dim > 576 (MB200_ERR_UNSUPPORTED).
 *  - A Cholesky-factored image runs on the launch plan of the registry's Cholesky-factored metric
 *    with two per-chain matrices (the factor L and the matrix V the policy differentiates): one
 *    256-thread CTA per chain, both matrices in shared memory up to dim 112 and in a per-CTA
 *    global workspace that the library allocates itself (stream-ordered) beyond;
 *    mb200_implicit_workspace_bytes returns 0.  Both integrators are supported.  dim > 1016, where
 *    the per-chain vectors exceed shared memory, is MB200_ERR_UNSUPPORTED before any launch.
 */
int mb200_user_riemannian_load(const void* image, int64_t image_bytes, const char* const* names,
                               int32_t n_names, int32_t rmetric_id, void** handle);
int mb200_implicit_leapfrog_riemannian_user(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, const mb200_model* model, int32_t fp_solver,
    double fp_convergence_tol, double fp_divergence_tol, int32_t fp_max_iters,
    double reverse_check_tol, double* h_out, int32_t* status, int32_t* n_done, int32_t* fp_iters,
    void* workspace, int64_t workspace_bytes, void* stream, const void* user_image);
int mb200_implicit_midpoint_riemannian_user(
    const double* pos_in, const double* mom_in, double* pos_out, double* mom_out,
    const int32_t* dir, int64_t n_chains, int32_t dim, double step_size, const double* step_sizes,
    int32_t n_steps, const int32_t* n_steps_per_chain, const mb200_model* model, int32_t fp_solver,
    double fp_convergence_tol, double fp_divergence_tol, int32_t fp_max_iters,
    double reverse_check_tol, double* h_out, int32_t* status, int32_t* n_done, int32_t* fp_iters,
    void* stream, const void* user_image);
int mb200_hamiltonian_riemannian_user(const double* pos, const double* mom, int64_t n_chains,
                                      int32_t dim, const mb200_model* model, double* h_out,
                                      int32_t* status, void* workspace, int64_t workspace_bytes,
                                      void* stream, const void* user_image);
int mb200_sample_momentum_riemannian_user(const double* pos, const double* normals,
                                          double* mom_out, int64_t n_chains, int32_t dim,
                                          const mb200_model* model, int32_t* status, void* stream,
                                          const void* user_image);
int mb200_dh_dmom_riemannian_user(const double* pos, const double* mom, double* vel_out,
                                  int64_t n_chains, int32_t dim, const mb200_model* model,
                                  int32_t* status, void* stream, const void* user_image);

/*
 * "Next" row N4: GaussianEuclideanMetricSystem (systems.py:369-474) -- the target density is
 * given relative to the standard Gaussian measure, h1 = l(q), h2 = q.q/2 + p.M^-1 p/2 and
 * h2_flow is the exact rotation of (q, p) in the eigenbasis of M (systems.py:464-474).  Leapfrog
 * (coefficients NULL) or a symmetric composition over these flows; h_out includes q.q/2.
 *   rotation  identity metric: NULL.  diagonal metric: the metric diagonal [dim] (device).
 *             dense metric: for every drift flow of the schedule, in order, three symmetric
 *             [dim x dim] device matrices  U cos(w t) U^T | U (sin(w t) w) U^T |
 *             -U (sin(w t) / w) U^T  with (eigval, U) = eigh(M), w = eigval^-1/2,
 *             t = coefficient * step_size (the sign of dir is applied by the kernel).
 *   step_sizes  optional per-chain step sizes (identity / diagonal metric only), else NULL.
 * n_steps = 0 with h_out evaluates the Hamiltonian only.
 */
int mb200_leapfrog_gaussian_euclidean(const double* pos_in, const double* mom_in, double* pos_out,
                                      double* mom_out, const int32_t* dir, int64_t n_chains,
                                      int32_t dim, double step_size, const double* step_sizes,
                                      int32_t n_steps, int32_t n_flows, const double* coefficients,
                                      int32_t initial_h1_flow_step, int32_t metric_kind,
                                      const double* metric_inv, const double* rotation,
                                      const mb200_model* model, double* h_out, int32_t* status,
                                      int32_t* n_done, void* stream);

/*
 * "Next" row N4: dynamic-length HMC transitions (NUTS) on a Euclidean-metric system with the
 * explicit leapfrog integrator, one whole transition per chain per call --
 * DynamicIntegrationTransition.sample / _build_tree (transitions.py:610-770) with
 * MultinomialDynamicIntegrationTransition (:773-809; slice_variant = 0) or
 * SliceDynamicIntegrationTransition (:812-858; slice_variant = 1) weights and the
 * riemannian_ (euclidean_criterion = 0, the reference's default) or euclidean_no_u_turn_criterion
 * (:405-470).  Every chain builds its own tree (one warp per chain); with a shared dense metric
 * and dim <= 128 the chains of a group of 8 advance leaf by leaf in lock-step and the product
 * M^-1 grad l(q) of the group is one tensor-pipe (DMMA) tile product per leaf (nuts_dmma.cuh).
 *   uniforms   [n_chains x n_uniforms] device array of U[0,1) variates; chain c consumes
 *              uniforms[c][0 .. n_uniforms_used[c]) in the order the reference calls
 *              rng.uniform().  2 max_tree_depth + 2^max_tree_depth variates always suffice;
 *              a chain that runs out reports status 1.
 *   workspace  >= mb200_nuts_workspace_bytes(n_chains, dim, max_tree_depth) bytes (device)
 *   outputs    pos_out / mom_out the returned state; h_out its Hamiltonian; n_step,
 *              av_metrop_accept_prob, reject_prob, tree_depth, diverging as the reference's
 *              transition statistics (transitions.py:713-769); dir_out the `dir` attribute of
 *              the returned state object (the direction its leaf was integrated in; for the
 *              initial state the direction of the last doubling started from it,
 *              transitions.py:731) -- the next stage's step-size search reads it
 *              (adapters.py:321).  Any of these may be NULL.
 * step_sizes: optional per-chain step sizes (device, [n_chains]) replacing step_size.
 */
int64_t mb200_nuts_workspace_bytes(int64_t n_chains, int32_t dim, int32_t max_tree_depth);
int mb200_nuts_euclidean(const double* pos_in, const double* mom_in, double* pos_out,
                         double* mom_out, int64_t n_chains, int32_t dim, double step_size,
                         const double* step_sizes, int32_t metric_kind, const double* metric_inv,
                         const mb200_model* model, int32_t slice_variant,
                         int32_t euclidean_criterion, int32_t extra_subtree_checks,
                         int32_t max_tree_depth, double max_delta_h, const double* uniforms,
                         int32_t n_uniforms, void* workspace, int64_t workspace_bytes,
                         double* h_out, int32_t* n_step, double* av_metrop_accept_prob,
                         double* reject_prob, int32_t* tree_depth, int32_t* diverging,
                         int32_t* n_uniforms_used, int32_t* dir_out, int32_t* status,
                         void* stream);

/*
 * Host-buffer form of mb200_leapfrog_euclidean -- the call a NumPy-state caller makes
 * (the reference's ChainState arrays live in host memory: states.py:160-305).  pos / mom / dir /
 * status are HOST pointers (page-locked memory makes the copies asynchronous); metric_inv stays a
 * device pointer.  The batch is cut into n_chunks row blocks aligned to the CTA granularity of
 * the kernel; block k is copied in, stepped and copied out on streams[k % n_streams], so that the
 * host->device copy of later blocks and the device->host copy of earlier blocks overlap the
 * kernels (chains are independent: chunking changes results at most in the last bits -- the
 * tensor-core kernel picks its accumulation split by launch size).  `scratch` is a device buffer
 * of at least mb200_host_scratch_bytes(n_chains, dim) bytes owned by the caller and must not be
 * shared by concurrent calls.  synchronize != 0: wait for all streams before returning.
 * PAGEABLE host buffers (plain NumPy arrays) are detected and staged by the library itself: a
 * small pool of worker threads copies each row block through a pinned bounce buffer (grow-only,
 * owned by the library), so that the host copies of one block overlap the DMA and the kernel of
 * the others; such a call is always synchronous.
 */
/*
 * Dynamic transitions for ANY integrator / system pair (constrained, implicit, compositions):
 * the tree bookkeeping of DynamicIntegrationTransition (transitions.py:528-581, 610-770) as
 * device kernels around batched integrator steps.  The caller advances all chains in lock-step:
 *   begin(initial pos, mom, dh_dmom, h)
 *   for depth in 0 .. max_tree_depth-1:
 *     start(depth) -> per-chain direction, edge state, active mask      [stop if none active]
 *     for k in 1 .. 2^depth:  one batched Integrator.step of the edge state with those
 *       directions, system.h and system.dh_dmom of the result, then leaf(k, 2^depth, ...)
 *     finish(depth)
 *   end() -> returned state and statistics
 * `status` of a leaf is the integrator's per-chain status: != 0 terminates that chain's tree and
 * sets convergence_error / non_reversible_step (transitions.py:670-676).  Uniform variates are
 * consumed per chain in the reference's order, as in mb200_nuts_euclidean.  workspace:
 * mb200_nuts_workspace_bytes(); chain_state: mb200_nuts_generic_state_bytes().  flags_out bits:
 * 0 diverging, 1 convergence_error, 2 non_reversible_step, 3 ran out of uniform variates.
 */
typedef struct mb200_nuts_options {
  int32_t max_tree_depth;
  int32_t slice_variant;
  int32_t euclidean_criterion;
  int32_t extra_subtree_checks;
  double max_delta_h;
  const double* uniforms;   /* [n_chains * n_uniforms] */
  int32_t n_uniforms;
} mb200_nuts_options;

int64_t mb200_nuts_generic_state_bytes(int64_t n_chains);
int mb200_nuts_generic_begin(const double* pos, const double* mom, const double* vel,
                             const double* h, int64_t n_chains, int32_t dim,
                             const mb200_nuts_options* options, void* workspace,
                             int64_t workspace_bytes, void* chain_state, int64_t chain_state_bytes,
                             void* stream);
int mb200_nuts_generic_start(int64_t n_chains, int32_t dim, int32_t depth,
                             const mb200_nuts_options* options, void* workspace, void* chain_state,
                             double* pos_edge, double* mom_edge, int32_t* dir_out, int32_t* active,
                             void* stream);
int mb200_nuts_generic_leaf(const double* pos, const double* mom, const double* vel,
                            const double* h, const int32_t* status, int64_t n_chains, int32_t dim,
                            int32_t k, int32_t n_leaves, const mb200_nuts_options* options,
                            void* workspace, void* chain_state, int32_t* active, void* stream);
int mb200_nuts_generic_finish(int64_t n_chains, int32_t dim, int32_t depth,
                              const mb200_nuts_options* options, void* workspace, void* chain_state,
                              void* stream);
int mb200_nuts_generic_end(int64_t n_chains, int32_t dim, const mb200_nuts_options* options,
                           void* workspace, void* chain_state, double* pos_out, double* mom_out,
                           double* h_out, int32_t* n_step, double* av_metrop_accept_prob,
                           double* reject_prob, int32_t* tree_depth, int32_t* flags_out,
                           int32_t* n_uniforms_used, int32_t* dir_out, void* stream);

int64_t mb200_host_scratch_bytes(int64_t n_chains, int32_t dim);
int mb200_leapfrog_euclidean_host(const double* pos_in, const double* mom_in, double* pos_out,
                                  double* mom_out, const int32_t* dir, int64_t n_chains,
                                  int32_t dim, double step_size, int32_t n_steps,
                                  int32_t metric_kind, const double* metric_inv,
                                  const mb200_model* model, int32_t* status, int32_t n_chunks,
                                  void* const* streams, int32_t n_streams, void* scratch,
                                  int64_t scratch_bytes, int32_t synchronize);

#ifdef __cplusplus
}
#endif
#endif /* MICI_B200_H */
