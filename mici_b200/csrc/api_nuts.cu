// libmici_b200.so -- C-ABI entry points (include/mici_b200.h): dynamic (NUTS) transitions, Metropolis selection, version / error text.
// Host-side argument checking and kernel dispatch only; all arithmetic is in the .cuh kernels.
#include "api_common.cuh"
#include "nuts.cuh"
#include "nuts_dmma.cuh"
#include "nuts_generic.cuh"
#include "transitions.cuh"

namespace mb200 {

// Arguments and launches of fused Euclidean NUTS (eu_dispatch)
struct NutsLaunch {
  static constexpr EuOp op = EuOp::Nuts;
  const double *q_in, *p_in;
  double *q_out, *p_out;
  int64_t n;
  int dim;
  double eps;
  int metric_kind;
  const double* minv;
  ModelArgs m;
  NutsArgs a;
  double* ws;
  double* h_out;
  int32_t* n_step;
  double *av_accept, *reject_prob;
  int32_t *depth, *diverging, *n_used, *dir_out, *status;
  cudaStream_t st;

  // Shared dense metric, dim <= 128: groups of 8 chains in lock-step, mat-vecs on the tensor pipe.
  // Measured on C1 (depth 6; free-running nuts_euclidean_kernel: 95 M leapfrog steps/s): one
  // group per CTA 205 M, two groups 172 M (register spills at the 128-register budget and a
  // workspace working set beyond L2), 16 chains in one lock-step 168 M; at dim = 64 (depth 8) two
  // groups 377 M, one group 300 M, free-running 215 M.
  template <class Target, int L>
  int dmma() const {
    constexpr int KP = EU_LAYOUTS[L].kp, GROUPS = KP == 1 ? 2 : 1, WARPS = 8 * GROUPS;
    return eu_launch(nuts_dmma_kernel<Target, KP, GROUPS>, "nuts_dmma_kernel",
                     (n + WARPS - 1) / WARPS, 0, WARPS * 32, NutsDmmaLayout<KP, GROUPS>::smem_bytes(),
                     st, q_in, p_in, q_out, p_out, n, dim, eps, minv, m, a, ws, h_out, n_step,
                     av_accept, reject_prob, depth, diverging, n_used, dir_out, status);
  }

  // Free-running: one warp per chain
  template <class Target, int L>
  int warp() const {
    constexpr int KP = EU_LAYOUTS[L].kp;
    NutsArgs args = a;
    // dense metric that fits in shared memory next to the staging rows: the warps of a CTA share
    // it (12 warps for 64 < dim <= 128, where one CTA per SM fits; 8 otherwise -- measured)
    const size_t metric_bytes = (size_t)dim * dim * sizeof(double);
    const int staged_warps = KP == 2 ? 12 : 8;
    args.stage_metric = metric_kind == MB200_METRIC_DENSE &&
                        metric_bytes + staged_warps * 64 * KP * sizeof(double) <= 200 * 1024;
    const int warps = args.stage_metric ? staged_warps : 4;
    const size_t smem =
        (size_t)warps * 64 * KP * sizeof(double) + (args.stage_metric ? metric_bytes : 0);
    return eu_launch(nuts_euclidean_kernel<Target, KP>, "nuts_euclidean_kernel",
                     (n + warps - 1) / warps, 0, warps * 32, smem, st, q_in, p_in, q_out, p_out, n,
                     dim, eps, metric_kind, minv, m, args, ws, h_out, n_step, av_accept,
                     reject_prob, depth, diverging, n_used, dir_out, status);
  }
};

}  // namespace mb200

using namespace mb200;

extern "C" {

int mb200_version(void) { return MB200_VERSION; }

const char* mb200_last_error(void) { return g_err; }

int mb200_set_call_counters(int32_t* counters) {
  tl_counters = counters;
  return 0;
}


int mb200_metropolis_select(double* pos, double* mom, const double* pos_prop,
                            const double* mom_prop, const double* h_init, const double* h_prop,
                            const int32_t* status, const int32_t* n_done, int32_t* dir,
                            const double* uniforms, int64_t n_chains, int32_t dim,
                            double* accept_prob, double* accept_stat, int32_t* accepted,
                            void* stream) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos || !mom || !pos_prop || !mom_prop || !h_init || !h_prop || !uniforms)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (n_chains == 0) return 0;
  const DeviceScope device_scope(pos);
  int64_t blocks = (n_chains * dim + 255) / 256;
  const int64_t cap = (int64_t)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  metropolis_select_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      pos, mom, pos_prop, mom_prop, h_init, h_prop, status, n_done, dir, uniforms, n_chains, dim,
      accept_prob, accept_stat, accepted);
  return check_launch("metropolis_select_kernel");
}

int64_t mb200_nuts_workspace_bytes(int64_t n_chains, int32_t dim, int32_t max_tree_depth) {
  if (n_chains < 0 || dim < 1 || dim > 1024 || max_tree_depth < 1 ||
      max_tree_depth > NUTS_MAX_DEPTH)
    return -1;
  return (int64_t)(nuts_workspace_doubles_per_chain(dim, max_tree_depth) * sizeof(double)) *
         n_chains;
}

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
                         void* stream) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos_in || !mom_in || !pos_out || !mom_out || !model || !uniforms || !workspace)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1 || n_uniforms < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (max_tree_depth < 1 || max_tree_depth > NUTS_MAX_DEPTH)
    return fail(MB200_ERR_INVALID_ARG, "max_tree_depth must be in [1, %d]", NUTS_MAX_DEPTH);
  if (const int rc = eu_check_metric(metric_kind, metric_inv)) return rc;
  // need < 0: dim > 1024, which the dispatch reports
  const int64_t need = mb200_nuts_workspace_bytes(n_chains, dim, max_tree_depth);
  if (need >= 0 && workspace_bytes < need)
    return fail(MB200_ERR_INVALID_ARG, "workspace too small: %lld < %lld bytes",
                (long long)workspace_bytes, (long long)need);
  const DeviceScope device_scope(pos_in);
  NutsArgs a;
  a.max_depth = max_tree_depth;
  a.max_delta_h = max_delta_h;
  a.euclidean_criterion = euclidean_criterion;
  a.extra_checks = extra_subtree_checks;
  a.slice = slice_variant;
  a.uniforms = uniforms;
  a.n_uniforms = n_uniforms;
  a.step_sizes = step_sizes;
  a.stage_metric = 0;
  const ModelArgs m = to_args(model);
  return eu_dispatch(m, dim, metric_kind,
                     NutsLaunch{pos_in, mom_in, pos_out, mom_out, n_chains, dim, step_size,
                                metric_kind, metric_inv, m, a, (double*)workspace, h_out, n_step,
                                av_metrop_accept_prob, reject_prob, tree_depth, diverging,
                                n_uniforms_used, dir_out, status, (cudaStream_t)stream});
}

// ---------------------------------------------------------------- generic dynamic transitions
namespace {

mb200::NutsGenArgs gen_args(const mb200_nuts_options* o) {
  mb200::NutsGenArgs a;
  a.max_depth = o->max_tree_depth;
  a.slice = o->slice_variant;
  a.euclid = o->euclidean_criterion;
  a.extra = o->extra_subtree_checks;
  a.max_delta_h = o->max_delta_h;
  a.uniforms = o->uniforms;
  a.n_uniforms = o->n_uniforms;
  return a;
}

int gen_check(int64_t n, int32_t dim, const mb200_nuts_options* o, const void* ws, const void* cs) {
  if (!o || !ws || !cs || !o->uniforms) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n < 0 || dim < 1 || dim > 1024) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (o->max_tree_depth < 1 || o->max_tree_depth > NUTS_MAX_DEPTH || o->n_uniforms < 1)
    return fail(MB200_ERR_INVALID_ARG, "max_tree_depth must be in [1, %d]", NUTS_MAX_DEPTH);
  return 0;
}

unsigned gen_blocks(int64_t n) {
  const int64_t cap = (int64_t)num_sms() * 8;
  int64_t b = (n + 3) / 4;
  return (unsigned)(b < cap ? (b < 1 ? 1 : b) : cap);
}

}  // namespace

int64_t mb200_nuts_generic_state_bytes(int64_t n_chains) {
  return n_chains < 0 ? -1 : n_chains * (int64_t)sizeof(NutsGenState);
}

int mb200_nuts_generic_begin(const double* pos, const double* mom, const double* vel,
                             const double* h, int64_t n_chains, int32_t dim,
                             const mb200_nuts_options* options, void* workspace,
                             int64_t workspace_bytes, void* chain_state, int64_t chain_state_bytes,
                             void* stream) {
  if (n_chains == 0) return 0;
  if (!pos || !mom || !vel || !h) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (int rc = gen_check(n_chains, dim, options, workspace, chain_state)) return rc;
  if (workspace_bytes < mb200_nuts_workspace_bytes(n_chains, dim, options->max_tree_depth) ||
      chain_state_bytes < mb200_nuts_generic_state_bytes(n_chains))
    return fail(MB200_ERR_INVALID_ARG, "workspace / chain state too small");
  const DeviceScope device_scope(pos);
  const NutsGenArgs a = gen_args(options);
  cudaStream_t st = (cudaStream_t)stream;
  with_layout(dim, [&](auto lay) {
    constexpr int KP = EU_LAYOUTS[decltype(lay)::value].kp;
    nuts_generic_begin_kernel<KP><<<gen_blocks(n_chains), 128, 0, st>>>(
        pos, mom, vel, h, n_chains, dim, a, (double*)workspace, (NutsGenState*)chain_state);
    return 0;
  });
  return check_launch("nuts_generic_begin_kernel");
}

int mb200_nuts_generic_start(int64_t n_chains, int32_t dim, int32_t depth,
                             const mb200_nuts_options* options, void* workspace, void* chain_state,
                             double* pos_edge, double* mom_edge, int32_t* dir_out, int32_t* active,
                             void* stream) {
  if (n_chains == 0) return 0;
  if (!pos_edge || !mom_edge || !dir_out || !active)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (int rc = gen_check(n_chains, dim, options, workspace, chain_state)) return rc;
  const DeviceScope device_scope(pos_edge);
  const NutsGenArgs a = gen_args(options);
  cudaStream_t st = (cudaStream_t)stream;
  with_layout(dim, [&](auto lay) {
    constexpr int KP = EU_LAYOUTS[decltype(lay)::value].kp;
    nuts_generic_start_kernel<KP><<<gen_blocks(n_chains), 128, 0, st>>>(
        n_chains, dim, depth, a, (double*)workspace, (NutsGenState*)chain_state, pos_edge,
        mom_edge, dir_out, active);
    return 0;
  });
  return check_launch("nuts_generic_start_kernel");
}

int mb200_nuts_generic_leaf(const double* pos, const double* mom, const double* vel,
                            const double* h, const int32_t* status, int64_t n_chains, int32_t dim,
                            int32_t k, int32_t n_leaves, const mb200_nuts_options* options,
                            void* workspace, void* chain_state, int32_t* active, void* stream) {
  if (n_chains == 0) return 0;
  if (!pos || !mom || !vel || !h || !status || !active)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (int rc = gen_check(n_chains, dim, options, workspace, chain_state)) return rc;
  const DeviceScope device_scope(pos);
  const NutsGenArgs a = gen_args(options);
  cudaStream_t st = (cudaStream_t)stream;
  with_layout(dim, [&](auto lay) {
    constexpr int KP = EU_LAYOUTS[decltype(lay)::value].kp;
    nuts_generic_leaf_kernel<KP><<<gen_blocks(n_chains), 128, 0, st>>>(
        pos, mom, vel, h, status, n_chains, dim, k, n_leaves, a, (double*)workspace,
        (NutsGenState*)chain_state, active);
    return 0;
  });
  return check_launch("nuts_generic_leaf_kernel");
}

int mb200_nuts_generic_finish(int64_t n_chains, int32_t dim, int32_t depth,
                              const mb200_nuts_options* options, void* workspace, void* chain_state,
                              void* stream) {
  if (n_chains == 0) return 0;
  if (int rc = gen_check(n_chains, dim, options, workspace, chain_state)) return rc;
  const DeviceScope device_scope(workspace);
  const NutsGenArgs a = gen_args(options);
  cudaStream_t st = (cudaStream_t)stream;
  with_layout(dim, [&](auto lay) {
    constexpr int KP = EU_LAYOUTS[decltype(lay)::value].kp;
    nuts_generic_finish_kernel<KP><<<gen_blocks(n_chains), 128, 0, st>>>(
        n_chains, dim, depth, a, (double*)workspace, (NutsGenState*)chain_state);
    return 0;
  });
  return check_launch("nuts_generic_finish_kernel");
}

int mb200_nuts_generic_end(int64_t n_chains, int32_t dim, const mb200_nuts_options* options,
                           void* workspace, void* chain_state, double* pos_out, double* mom_out,
                           double* h_out, int32_t* n_step, double* av_metrop_accept_prob,
                           double* reject_prob, int32_t* tree_depth, int32_t* flags_out,
                           int32_t* n_uniforms_used, int32_t* dir_out, void* stream) {
  if (n_chains == 0) return 0;
  if (!pos_out || !mom_out || !h_out || !n_step || !av_metrop_accept_prob || !reject_prob ||
      !tree_depth || !flags_out || !n_uniforms_used || !dir_out)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (int rc = gen_check(n_chains, dim, options, workspace, chain_state)) return rc;
  const DeviceScope device_scope(pos_out);
  const NutsGenArgs a = gen_args(options);
  cudaStream_t st = (cudaStream_t)stream;
  with_layout(dim, [&](auto lay) {
    constexpr int KP = EU_LAYOUTS[decltype(lay)::value].kp;
    nuts_generic_end_kernel<KP><<<gen_blocks(n_chains), 128, 0, st>>>(
        n_chains, dim, a, (const double*)workspace, (const NutsGenState*)chain_state, pos_out,
        mom_out, h_out, n_step, av_metrop_accept_prob, reject_prob, tree_depth, flags_out,
        n_uniforms_used, dir_out);
    return 0;
  });
  return check_launch("nuts_generic_end_kernel");
}

}  // extern "C"
