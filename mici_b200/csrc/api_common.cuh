// Host-side helpers shared by the translation units of libmici_b200.so (argument checking, error
// text, model-argument packing).  The library is split into one .cu per kernel family so that the
// families compile in parallel (`make -j`); the C ABI (include/mici_b200.h) is unchanged.
#pragma once
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "common.cuh"

namespace mb200 {

inline thread_local char g_err[512] = "";

inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

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

// implemented in api_dmma.cu (tensor-core leapfrog); MB200_ERR_UNSUPPORTED = outside its domain
int leapfrog_dmma_dispatch(const double* q_in, const double* p_in, double* q_out, double* p_out,
                           const int32_t* dir, const double* step_sizes, int64_t n, int dim,
                           double eps, int n_steps, const double* minv, const ModelArgs& m,
                           double* h_out, int32_t* status, int32_t* n_done, cudaStream_t st);

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

}  // namespace mb200
