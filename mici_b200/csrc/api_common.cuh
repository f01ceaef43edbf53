// Host-side helpers shared by the translation units of libmici_b200.so (argument checking, error
// text, model-argument packing).  The library is split into one .cu per kernel family so that the
// families compile in parallel (`make -j`); the C ABI (include/mici_b200.h) is unchanged.
#pragma once
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <type_traits>

#include "common.cuh"
#include "targets.cuh"

namespace mb200 {

inline thread_local char g_err[512] = "";

inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

// a type as a value (also keeps a parameter out of template argument deduction)
template <class T>
struct TypeTag {
  using type = T;
};

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return 0;
}

inline thread_local int32_t* tl_counters = nullptr;  // mb200_set_call_counters

// Kernel arguments of a model.  step_sizes / n_steps_pc: the optional per-chain device arrays of
// the implicit and constrained entry points (NULL: every chain uses the scalar argument).
inline ModelArgs to_args(const mb200_model* m, const double* step_sizes = nullptr,
                         const int32_t* n_steps_pc = nullptr) {
  ModelArgs a;
  memset(&a, 0, sizeof(a));
  a.step_sizes = step_sizes;
  a.n_steps_pc = n_steps_pc;
  a.counters = tl_counters;
  a.target_id = m->target_id;
  for (int i = 0; i < MB200_MAX_PARAMS; ++i) a.tp[i] = m->target_params[i];
  a.taux = m->target_aux;
  a.rmetric_id = m->rmetric_id;
  for (int i = 0; i < MB200_MAX_PARAMS; ++i) a.mp[i] = m->rmetric_params[i];
  a.maux = m->rmetric_aux;
  return a;
}

// SM count of the CURRENT device (queried per call: a process may drive several devices).
inline int num_sms() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 132;
}

// Makes the device that owns `ptr` current for the lifetime of the object (the caller may have a
// different current device: ADVICE r1) and restores the previous one afterwards.
struct DeviceScope {
  int prev = -1;
  explicit DeviceScope(const void* ptr) {
    cudaPointerAttributes at;
    if (ptr != nullptr && cudaPointerGetAttributes(&at, ptr) == cudaSuccess &&
        at.type == cudaMemoryTypeDevice) {
      int cur = 0;
      cudaGetDevice(&cur);
      if (cur != at.device) {
        prev = cur;
        cudaSetDevice(at.device);
      }
    } else {
      cudaGetLastError();  // clear a possible "invalid value" from a host pointer
    }
  }
  ~DeviceScope() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// Workspace: caller-provided when large enough, else a stream-ordered allocation that is freed
// (stream-ordered) right after the launch -- entry points without a workspace parameter
// (momentum refresh, velocity, implicit midpoint) use the latter.
struct DgScratch {
  double* ptr = nullptr;
  bool owned = false;
  cudaStream_t st;
  DgScratch(void* user, int64_t user_bytes, size_t need, cudaStream_t s) : st(s) {
    if (need == 0) return;
    if (user != nullptr && user_bytes >= (int64_t)need &&
        (reinterpret_cast<uintptr_t>(user) & 15) == 0) {
      ptr = static_cast<double*>(user);
    } else if (cudaMallocAsync(reinterpret_cast<void**>(&ptr), need, s) == cudaSuccess) {
      owned = true;
    } else {
      ptr = nullptr;
    }
  }
  ~DgScratch() {
    if (owned && ptr != nullptr) cudaFreeAsync(ptr, st);
  }
};

// ---- Euclidean family: which kernel serves a model (api_euclid.cu, api_nuts.cu, api_dmma.cu) ----

// Arguments of one Euclidean leapfrog launch (zero steps evaluate the Hamiltonian only).
// allow_k1: the caller lets the tensor-core kernel K1 serve the call (mb200_leapfrog_euclidean
// with the default leapfrog schedule); k1_serves() decides whether it does.
struct EuclidArgs {
  const double *q_in, *p_in;
  double *q_out, *p_out;
  const int32_t* dir;
  int64_t n;
  int dim;
  double eps;
  int n_steps;
  FlowSchedule sched;
  int metric_kind;
  const double* minv;
  ModelArgs m;
  double* h_out;
  int32_t *status, *n_done;
  cudaStream_t st;
  bool allow_k1;
};

// K1's domain: one trajectory length for every chain, n_steps > 0, a dense metric,
// 8 <= dim <= 128, a registry target, and per-chain step sizes or a finite non-zero eps (K1 stages
// eps * M^-1 in shared memory)
inline bool k1_serves(int metric_kind, int dim, double eps, const double* step_sizes, int n_steps,
                      const int32_t* n_steps_pc, int target_id) {
  return n_steps_pc == nullptr && n_steps > 0 && metric_kind == MB200_METRIC_DENSE && dim >= 8 &&
         dim <= 128 && (step_sizes != nullptr || (eps != 0.0 && isfinite(eps))) &&
         (target_id == MB200_TARGET_STD_GAUSSIAN || target_id == MB200_TARGET_NEAL_FUNNEL ||
          target_id == MB200_TARGET_BANANA);
}

// K1 for one registry target (api_dmma.cu)
template <class Target>
int k1_launch(const EuclidArgs& a);

// (KP, CPW) of the warp-per-chain Euclidean kernels -- K1g, evaluation, fused NUTS and the generic
// NUTS steps -- by dimension: layout l serves dim <= max_dim.  A user target's kernel table
// (mb200_user_target_load) is in this order, and mici_b200/jit.py LAYOUTS lists it: keep the two
// in step.
struct EuLayout {
  int max_dim, kp, cpw;
};
constexpr EuLayout EU_LAYOUTS[] = {{64, 1, 4}, {128, 2, 4}, {256, 4, 2}, {512, 8, 1}, {1024, 16, 1}};
constexpr int N_EU_LAYOUTS = sizeof(EU_LAYOUTS) / sizeof(EU_LAYOUTS[0]);

// f(std::integral_constant<int, l>()) for the layout l of `dim`
template <int L = 0, class F>
int with_layout(int dim, const F& f) {
  if constexpr (L == N_EU_LAYOUTS)
    return fail(MB200_ERR_UNSUPPORTED, "dim %d > 1024 not supported", dim);
  else
    return dim <= EU_LAYOUTS[L].max_dim ? f(std::integral_constant<int, L>())
                                        : with_layout<L + 1>(dim, f);
}

// Starts `kern` on min(blocks, cap) CTAs of `threads` threads with `smem` bytes of dynamic shared
// memory (opted in above the default 48 KB); cap is `per_sm` CTAs per SM, or as many as fit when
// per_sm == 0.  A failure reads "<name>: <CUDA error>".
template <class... P>
int eu_launch(void (*kern)(P...), const char* name, int64_t blocks, int per_sm, int threads,
              size_t smem, cudaStream_t st, typename TypeTag<P>::type... args) {
  const void* k = (const void*)kern;
  cudaError_t e = cudaSuccess;
  if (smem > 48 * 1024)
    e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess && per_sm == 0) {
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, threads, smem);
    if (per_sm < 1) per_sm = 1;
  }
  if (e == cudaSuccess) {
    const int64_t cap = (int64_t)num_sms() * per_sm;
    void* argv[] = {&args...};
    e = cudaLaunchKernel(k, dim3((unsigned)(blocks < cap ? blocks : cap)), dim3(threads), argv,
                         smem, st);
  }
  if (e != cudaSuccess) {
    cudaGetLastError();  // reported here: clear it from the runtime's error state
    return fail(MB200_ERR_CUDA, "%s: %s", name, cudaGetErrorString(e));
  }
  return check_launch(name);
}

// the metric arguments every Euclidean entry point takes
inline int eu_check_metric(int metric_kind, const double* minv) {
  if (metric_kind < 0 || metric_kind > 2) return fail(MB200_ERR_INVALID_ARG, "bad metric_kind");
  if (metric_kind != MB200_METRIC_IDENTITY && !minv)
    return fail(MB200_ERR_INVALID_ARG, "metric_inv is NULL");
  return 0;
}

enum class EuOp { Leapfrog, Eval, Nuts };

// Which kernel serves a Euclidean model, for every operation L::op.  Checks the model the same way
// whatever the operation, picks the route, and hands the target type and the layout to `l`:
//   l.k1<Target>()        K1, the tensor-core leapfrog (l.k1_ok: k1_serves)
//   l.dmma<Target, L>()   fused NUTS in lock-step on the tensor pipe (dense metric, 8 <= dim <= 128)
//   l.warp<Target, L>()   the library's warp-per-chain kernel of the operation
//   l.image(L)            the same kernel from the loaded user-target image l.user
template <class L>
int eu_dispatch(const ModelArgs& m, int dim, int metric_kind, const L& l) {
  if (m.target_id == MB200_TARGET_BANANA && (dim & 1))
    return fail(MB200_ERR_INVALID_ARG, "banana target needs even dim");
  if constexpr (L::op != EuOp::Nuts) {
    if (l.user != nullptr) {
      if (m.target_id != MB200_TARGET_USER)
        return fail(MB200_ERR_INVALID_ARG,
                    "user-target entry point needs target_id MB200_TARGET_USER");
      return with_layout(dim, [&](auto lay) { return l.image(lay.value); });
    }
  }
  auto route = [&](auto target) {
    using Target = typename decltype(target)::type;
    if constexpr (L::op == EuOp::Leapfrog)
      if (l.k1_ok()) return l.template k1<Target>();
    return with_layout(dim, [&](auto lay) {
      constexpr int LAY = decltype(lay)::value;
      if constexpr (L::op == EuOp::Nuts && EU_LAYOUTS[LAY].kp <= 2)
        if (metric_kind == MB200_METRIC_DENSE && dim >= 8) return l.template dmma<Target, LAY>();
      return l.template warp<Target, LAY>();
    });
  };
  switch (m.target_id) {
    case MB200_TARGET_STD_GAUSSIAN: return route(TypeTag<StdGaussianTarget>());
    case MB200_TARGET_NEAL_FUNNEL: return route(TypeTag<NealFunnelTarget>());
    case MB200_TARGET_BANANA: return route(TypeTag<BananaTarget>());
  }
  return fail(MB200_ERR_UNSUPPORTED, "target %d not available for Euclidean systems", m.target_id);
}

// The constrained kernels of a user image loaded by mb200_user_constraint_load, compiled for
// n_constr constraints at kp, indexed by GAUSS.  n_constr == 0: an image of
// mb200_user_target_load, which carries none.
struct UserConstraintKernels {
  int n_constr, kp;
  bool mhp_constr;
  const void* leapfrog[2];
  const void* project[2];
};
// the constrained part of a loaded user image (api_euclid.cu)
const UserConstraintKernels& user_constraint_kernels(const void* handle);

// The Riemannian kernels of a user image loaded by mb200_user_riemannian_load, for one (user
// target, user metric) pair: the implicit leapfrog / midpoint, velocity and momentum-refresh
// kernels of the metric kind rmetric_id.  rmetric_id == 0: an image of mb200_user_target_load or
// mb200_user_constraint_load, which carries none (and whose Euclidean kernels this one lacks).
struct UserRiemannianKernels {
  int rmetric_id;
  const void* implicit;
  const void* velocity;
  const void* momentum;
};
// the Riemannian part of a loaded user image (api_euclid.cu)
const UserRiemannianKernels& user_riemannian_kernels(const void* handle);

// Starts `kern` -- a library kernel, or a kernel of a loaded user image (a cudaKernel_t, which
// only cudaLaunchKernel can start: a <<<>>> launch would call it as the kernel's host stub) --
// with the argument types of the library's own instantiations
template <class... P>
inline void rm_start(void (*kern)(P...), unsigned blocks, int threads, size_t smem,
                     cudaStream_t st, typename TypeTag<P>::type... args) {
  void* argv[] = {&args...};
  cudaLaunchKernel((const void*)kern, dim3(blocks), dim3(threads), argv, smem, st);
}

// Arguments of one implicit-integrator launch on a Riemannian system (leapfrog or midpoint steps;
// zero steps evaluate the Hamiltonian only).  ws / ws_bytes: the caller's workspace, or NULL.
struct ImplicitArgs {
  const double *q_in, *p_in;
  double *q_out, *p_out;
  const int32_t* dir;
  int64_t n;
  int dim;
  double eps;
  int n_steps;
  ModelArgs m;
  double fp_tol, fp_div;
  int fp_max;
  double rev_tol;
  double* h_out;
  int32_t *status, *n_done, *fp_iters;
  int fp_solver;
  void* ws;
  int64_t ws_bytes;
  cudaStream_t st;
};

// Arguments of one per-chain metric-vector product on a Riemannian system: sqrt(M(q)) v
// (momentum refresh) or M(q)^-1 v (velocity)
struct VectorArgs {
  const double *q, *v;
  double* out;
  int64_t n;
  int dim;
  ModelArgs m;
  int32_t* status;
  cudaStream_t st;
};

// implemented in api_dense.cu (global-workspace dense metric policy, dense_global.cuh); the
// route to it is decided, and its arguments checked, in api_riemannian.cu
int64_t dense_global_workspace_bytes(int64_t n_chains, int dim);
bool dense_global_supported(int dim);
int dense_global_implicit(const ImplicitArgs& a, bool hadamard);
int dense_global_vector(const VectorArgs& a, bool velocity, bool hadamard);
// the same launch plan for the kernel `kern` of a loaded user image (MB200_RMETRIC_USER_DENSE)
int dense_global_implicit_image(const ImplicitArgs& a, const void* kern);
int dense_global_vector_image(const VectorArgs& a, const void* kern);

}  // namespace mb200
