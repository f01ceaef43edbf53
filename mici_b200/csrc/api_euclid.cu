// libmici_b200.so -- C-ABI entry points (include/mici_b200.h): Euclidean-metric leapfrog family (general-dimension kernel, evaluation pieces, host-buffer path).
// Host-side argument checking and kernel dispatch only; all arithmetic is in the .cuh kernels.
#include "api_common.cuh"
#include "leapfrog_generic.cuh"

#include <condition_variable>
#include <cstring>
#include <functional>
#include <mutex>
#include <queue>
#include <string>
#include <thread>
#include <vector>

namespace mb200 {

// ---- host-buffer path for PAGEABLE memory ----------------------------------------------------
// cudaMemcpyAsync on pageable memory is staged by the driver through one internal buffer and
// serialises with the caller (measured: 9.7 ms per 8192 x 128 launch against 0.9 ms from pinned
// memory).  The library stages such buffers itself: a few worker threads each take one row
// block end to end -- memcpy into a pinned bounce buffer, H2D + kernel + D2H on the block's
// stream, wait for its event, memcpy out of the bounce buffer -- so the host copies of one block
// overlap the DMA and the kernel of the others.
class HostStager {
 public:
  static HostStager& get() {
    static HostStager* s = new HostStager;  // never destroyed: its detached workers outlive main
    return *s;
  }
  // grow-only pinned bounce buffer of at least `bytes`
  void* bounce(size_t bytes) {
    if (bytes > cap_) {
      if (buf_) cudaFreeHost(buf_);
      buf_ = nullptr, cap_ = 0;
      if (cudaHostAlloc(&buf_, bytes, cudaHostAllocPortable) != cudaSuccess) return nullptr;
      cap_ = bytes;
    }
    return buf_;
  }
  // runs the tasks on the pool (the caller's thread takes part), returns when all are done
  void run(std::vector<std::function<void()>>& tasks) {
    const int want = (int)tasks.size() - 1 < MAX_WORKERS ? (int)tasks.size() - 1 : MAX_WORKERS;
    {
      std::lock_guard<std::mutex> lk(mu_);
      while (n_workers_ < want) {
        std::thread([this] { loop(); }).detach();
        ++n_workers_;
      }
      pending_ = (int)tasks.size();
      for (auto& t : tasks) queue_.push(&t);
    }
    cv_.notify_all();
    for (;;) {  // help out
      std::function<void()>* t = nullptr;
      {
        std::lock_guard<std::mutex> lk(mu_);
        if (!queue_.empty()) t = queue_.front(), queue_.pop();
      }
      if (!t) break;
      (*t)();
      finish_one();
    }
    std::unique_lock<std::mutex> lk(mu_);
    done_cv_.wait(lk, [this] { return pending_ == 0; });
  }
  std::mutex call_mu;  // one host-path call at a time owns the bounce buffer

 private:
  static constexpr int MAX_WORKERS = 7;
  void finish_one() {
    std::lock_guard<std::mutex> lk(mu_);
    if (--pending_ == 0) done_cv_.notify_all();
  }
  void loop() {
    for (;;) {
      std::function<void()>* t;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [this] { return !queue_.empty(); });
        t = queue_.front(), queue_.pop();
      }
      (*t)();
      finish_one();
    }
  }
  std::mutex mu_;
  std::condition_variable cv_, done_cv_;
  std::queue<std::function<void()>*> queue_;
  int n_workers_ = 0;
  int pending_ = 0;
  void* buf_ = nullptr;
  size_t cap_ = 0;
};

static bool is_pageable(const void* ptr) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
    cudaGetLastError();
    return true;
  }
  return a.type == cudaMemoryTypeUnregistered;
}

// A loaded user-target image (mb200_user_target_load): its general-dimension leapfrog kernels
// leapfrog_generic_kernel<UserTarget, KP, CPW, false> and evaluation kernels
// euclidean_eval_kernel<UserTarget, KP>, one per layout of EU_LAYOUTS.  Their parameters are those
// of the library's own instantiations.
using LeapfrogKernel = decltype(&leapfrog_generic_kernel<StdGaussianTarget, 1, 4, false>);
using EvalKernel = decltype(&euclidean_eval_kernel<StdGaussianTarget, 1>);
struct UserKernels {
  cudaLibrary_t lib;
  UserRiemannianKernels rm;  // mb200_user_riemannian_load only, which has no other kernels
  LeapfrogKernel leapfrog[N_EU_LAYOUTS];
  EvalKernel eval[N_EU_LAYOUTS];
  UserConstraintKernels constr;  // mb200_user_constraint_load only
};

const UserConstraintKernels& user_constraint_kernels(const void* handle) {
  return static_cast<const UserKernels*>(handle)->constr;
}

const UserRiemannianKernels& user_riemannian_kernels(const void* handle) {
  return static_cast<const UserKernels*>(handle)->rm;
}

// The handle of a Euclidean *_user entry point: an image with the Euclidean kernels
static int euclidean_image(const void* handle, const UserKernels** u) {
  if (!handle) return fail(MB200_ERR_INVALID_ARG, "user_target is NULL");
  *u = static_cast<const UserKernels*>(handle);
  if ((*u)->rm.rmetric_id != 0)
    return fail(MB200_ERR_INVALID_ARG,
                "a Riemannian user image (mb200_user_riemannian_load) has no Euclidean kernels");
  return 0;
}

// Loads `image` and looks up its kernels: the Euclidean table, then (n_names > 2 N_EU_LAYOUTS)
// the constrained one, in the order of include/mici_b200.h; or, for an image of
// mb200_user_riemannian_load (rm.rmetric_id != 0), its three Riemannian kernels only
static int user_image_load(const void* image, const char* const* names, int n_names,
                           const UserConstraintKernels& constr, const UserRiemannianKernels& rm,
                           void** handle) {
  UserKernels* u = new UserKernels();
  u->constr = constr;
  u->rm = rm;
  cudaError_t e = cudaLibraryLoadData(&u->lib, image, nullptr, nullptr, 0, nullptr, nullptr, 0);
  if (e != cudaSuccess) {
    delete u;
    return fail(MB200_ERR_CUDA, "cudaLibraryLoadData: %s", cudaGetErrorString(e));
  }
  for (int i = 0; i < n_names; ++i) {
    cudaKernel_t k;
    e = cudaLibraryGetKernel(&k, u->lib, names[i]);
    if (e != cudaSuccess) {
      cudaLibraryUnload(u->lib);
      delete u;
      return fail(MB200_ERR_CUDA, "cudaLibraryGetKernel(%s): %s", names[i], cudaGetErrorString(e));
    }
    const int c = i - 2 * N_EU_LAYOUTS;
    if (rm.rmetric_id != 0)
      (i == 0 ? u->rm.implicit : i == 1 ? u->rm.velocity : u->rm.momentum) =
          reinterpret_cast<const void*>(k);
    else if (i < N_EU_LAYOUTS)
      u->leapfrog[i] = reinterpret_cast<LeapfrogKernel>(k);
    else if (c < 0)
      u->eval[i - N_EU_LAYOUTS] = reinterpret_cast<EvalKernel>(k);
    else if (c < 2)
      u->constr.leapfrog[c] = reinterpret_cast<const void*>(k);
    else
      u->constr.project[c - 2] = reinterpret_cast<const void*>(k);
  }
  *handle = u;
  return 0;
}

// Splitting schedule of the C-ABI arguments: n_flows (odd) coefficients alternating a, b, ..., a
// with a = h1_flow (kick) if initial_h1_flow_step else h2_flow (drift) (integrators.py:268-281);
// coefficients == NULL is the leapfrog schedule {0.5 kick, 1 drift, 0.5 kick}.
static int make_schedule(FlowSchedule& s, int n_flows, const double* coefficients,
                         int initial_h1_flow_step) {
  memset(&s, 0, sizeof(s));
  if (coefficients == nullptr) {
    s.n = 3;
    s.drift_mask = 0x2u;
    s.coef[0] = 0.5, s.coef[1] = 1.0, s.coef[2] = 0.5;
    return 0;
  }
  if (n_flows < 1 || n_flows > MB200_MAX_FLOWS || (n_flows & 1) == 0)
    return fail(MB200_ERR_INVALID_ARG, "n_flows must be odd and in [1, %d]", MB200_MAX_FLOWS);
  s.n = n_flows;
  for (int i = 0; i < n_flows; ++i) {
    s.coef[i] = coefficients[i];
    const bool is_a = (i & 1) == 0;
    if (initial_h1_flow_step ? !is_a : is_a) s.drift_mask |= 1u << i;
  }
  return 0;
}

// Launch functors of the leapfrog and the evaluation (eu_dispatch).  whole_vector: a user target
// stages each chain's position and gradient in shared memory (user_target.cuh), 2 * 64 KP doubles
// per warp more.
struct LeapfrogLaunch {
  static constexpr EuOp op = EuOp::Leapfrog;
  const EuclidArgs& a;
  const UserKernels* user;
  bool k1_ok() const {
    return a.allow_k1 && k1_serves(a.metric_kind, a.dim, a.eps, a.sched.step_sizes, a.n_steps,
                                   a.sched.n_steps, a.m.target_id);
  }
  template <class Target>
  int k1() const {
    return k1_launch<Target>(a);
  }
  template <class Target, int L>
  int warp() const {
    constexpr int KP = EU_LAYOUTS[L].kp, CPW = EU_LAYOUTS[L].cpw;
    return run(a.sched.gaussian ? leapfrog_generic_kernel<Target, KP, CPW, true>
                                : leapfrog_generic_kernel<Target, KP, CPW, false>,
               L, false);
  }
  int image(int l) const { return run(user->leapfrog[l], l, true); }
  int run(LeapfrogKernel kern, int l, bool whole_vector) const {
    constexpr int WARPS = 4;
    const int kp = EU_LAYOUTS[l].kp, cpw = EU_LAYOUTS[l].cpw;
    const size_t smem = (size_t)WARPS * (cpw + (whole_vector ? 2 : 0)) * 64 * kp * sizeof(double);
    const int64_t groups = (a.n + cpw - 1) / cpw;
    return eu_launch(kern, "leapfrog_generic_kernel", (groups + WARPS - 1) / WARPS, 16, WARPS * 32,
                     smem, a.st, a.q_in, a.p_in, a.q_out, a.p_out, a.dir, a.n, a.dim, a.eps,
                     a.n_steps, a.sched, a.metric_kind, a.minv, a.m, a.h_out, a.status, a.n_done);
  }
};

struct EvalLaunch {
  static constexpr EuOp op = EuOp::Eval;
  const double *q, *p;
  int64_t n;
  int dim;
  int metric_kind;
  const double* minv;
  ModelArgs m;
  double *nld, *grad, *vel, *kin;
  cudaStream_t st;
  const UserKernels* user;
  template <class Target, int L>
  int warp() const {
    return run(euclidean_eval_kernel<Target, EU_LAYOUTS[L].kp>, L, false);
  }
  int image(int l) const { return run(user->eval[l], l, true); }
  int run(EvalKernel kern, int l, bool whole_vector) const {
    constexpr int WARPS = 4;
    const size_t smem = (size_t)WARPS * (whole_vector ? 3 : 1) * 64 * EU_LAYOUTS[l].kp * sizeof(double);
    return eu_launch(kern, "euclidean_eval_kernel", (n + WARPS - 1) / WARPS, 16, WARPS * 32, smem,
                     st, q, p, n, dim, metric_kind, minv, m, nld, grad, vel, kin);
  }
};

// mb200_leapfrog_euclidean (allow_k1), _generic, _user (user != NULL) and
// mb200_leapfrog_gaussian_euclidean (a.sched.gaussian)
static int leapfrog_euclidean_impl(EuclidArgs a, const mb200_model* model,
                                   const UserKernels* user = nullptr) {
  if (a.n == 0 && a.dim >= 1 && a.n_steps >= 0) return 0;  // empty batch: nothing to do
  if (!a.q_in || !a.p_in || !a.q_out || !a.p_out || !model)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (a.n < 0 || a.dim < 1 || a.n_steps < 0) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (const int rc = eu_check_metric(a.metric_kind, a.minv)) return rc;
  const DeviceScope device_scope(a.q_in);
  a.m = to_args(model);
  return eu_dispatch(a.m, a.dim, a.metric_kind, LeapfrogLaunch{a, user});
}

static int leapfrog_euclidean_entry(const double* q_in, const double* p_in, double* q_out,
                                    double* p_out, const int32_t* dir, int64_t n, int dim,
                                    double eps, const double* step_sizes, int n_steps,
                                    const int32_t* n_steps_pc, int n_flows,
                                    const double* coefficients, int initial_h1_flow_step,
                                    int metric_kind, const double* minv, const mb200_model* model,
                                    double* h_out, int32_t* status, int32_t* n_done,
                                    cudaStream_t st, bool allow_k1,
                                    const UserKernels* user = nullptr) {
  FlowSchedule s;
  if (const int rc = make_schedule(s, n_flows, coefficients, initial_h1_flow_step)) return rc;
  s.step_sizes = step_sizes;
  s.n_steps = n_steps_pc;
  // K1 runs the leapfrog schedule only
  return leapfrog_euclidean_impl({q_in, p_in, q_out, p_out, dir, n, dim, eps, n_steps, s,
                                  metric_kind, minv, ModelArgs(), h_out, status, n_done, st,
                                  allow_k1 && coefficients == nullptr},
                                 model, user);
}

// mb200_euclidean_eval and mb200_euclidean_eval_user (user != NULL)
static int euclidean_eval_impl(const double* pos, const double* mom, int64_t n_chains, int dim,
                               int metric_kind, const double* metric_inv,
                               const mb200_model* model, double* nld_out, double* grad_out,
                               double* vel_out, double* kin_out, cudaStream_t st,
                               const UserKernels* user) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos || !mom || !model) return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (const int rc = eu_check_metric(metric_kind, metric_inv)) return rc;
  const DeviceScope device_scope(pos);
  const ModelArgs m = to_args(model);
  return eu_dispatch(m, dim, metric_kind,
                     EvalLaunch{pos, mom, n_chains, dim, metric_kind, metric_inv, m, nld_out,
                                grad_out, vel_out, kin_out, st, user});
}

}  // namespace mb200

using namespace mb200;

extern "C" {

int mb200_leapfrog_euclidean(const double* pos_in, const double* mom_in, double* pos_out,
                             double* mom_out, const int32_t* dir, int64_t n_chains, int32_t dim,
                             double step_size, const double* step_sizes, int32_t n_steps,
                             const int32_t* n_steps_per_chain, int32_t n_flows,
                             const double* coefficients, int32_t initial_h1_flow_step,
                             int32_t metric_kind, const double* metric_inv,
                             const mb200_model* model, double* h_out, int32_t* status,
                             int32_t* n_done, void* stream) {
  return leapfrog_euclidean_entry(pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size,
                                  step_sizes, n_steps, n_steps_per_chain, n_flows, coefficients,
                                  initial_h1_flow_step, metric_kind, metric_inv, model, h_out,
                                  status, n_done, (cudaStream_t)stream, true);
}

// Same arithmetic through the general-dimension kernel only (used by tests to cross-check the
// tensor-core kernel; not part of the reference-facing surface).
int mb200_leapfrog_euclidean_generic(const double* pos_in, const double* mom_in, double* pos_out,
                                     double* mom_out, const int32_t* dir, int64_t n_chains,
                                     int32_t dim, double step_size, const double* step_sizes,
                                     int32_t n_steps, const int32_t* n_steps_per_chain,
                                     int32_t n_flows, const double* coefficients,
                                     int32_t initial_h1_flow_step, int32_t metric_kind,
                                     const double* metric_inv, const mb200_model* model,
                                     double* h_out, int32_t* status, int32_t* n_done,
                                     void* stream) {
  return leapfrog_euclidean_entry(pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size,
                                  step_sizes, n_steps, n_steps_per_chain, n_flows, coefficients,
                                  initial_h1_flow_step, metric_kind, metric_inv, model, h_out,
                                  status, n_done, (cudaStream_t)stream, false);
}

int mb200_hamiltonian_euclidean(const double* pos, const double* mom, int64_t n_chains,
                                int32_t dim, int32_t metric_kind, const double* metric_inv,
                                const mb200_model* model, double* h_out, void* stream) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!h_out) return fail(MB200_ERR_INVALID_ARG, "h_out is NULL");
  // zero leapfrog steps: loads the state, evaluates h, writes the (unchanged) state back in place
  return mb200_leapfrog_euclidean_generic(pos, mom, const_cast<double*>(pos),
                                          const_cast<double*>(mom), nullptr, n_chains, dim, 0.0,
                                          nullptr, 0, nullptr, 0, nullptr, 0, metric_kind,
                                          metric_inv, model, h_out, nullptr, nullptr, stream);
}

int mb200_euclidean_eval(const double* pos, const double* mom, int64_t n_chains, int32_t dim,
                         int32_t metric_kind, const double* metric_inv, const mb200_model* model,
                         double* nld_out, double* grad_out, double* vel_out, double* kin_out,
                         void* stream) {
  return euclidean_eval_impl(pos, mom, n_chains, dim, metric_kind, metric_inv, model, nld_out,
                             grad_out, vel_out, kin_out, (cudaStream_t)stream, nullptr);
}

int mb200_leapfrog_gaussian_euclidean(const double* pos_in, const double* mom_in, double* pos_out,
                                      double* mom_out, const int32_t* dir, int64_t n_chains,
                                      int32_t dim, double step_size, const double* step_sizes,
                                      int32_t n_steps, int32_t n_flows, const double* coefficients,
                                      int32_t initial_h1_flow_step, int32_t metric_kind,
                                      const double* metric_inv, const double* rotation,
                                      const mb200_model* model, double* h_out, int32_t* status,
                                      int32_t* n_done, void* stream) {
  FlowSchedule s;
  if (const int rc = make_schedule(s, n_flows, coefficients, initial_h1_flow_step)) return rc;
  if (metric_kind != MB200_METRIC_IDENTITY && !rotation && n_chains > 0)
    return fail(MB200_ERR_INVALID_ARG, "rotation is NULL");
  if (metric_kind == MB200_METRIC_DENSE && step_sizes)
    return fail(MB200_ERR_UNSUPPORTED,
                "per-chain step sizes need per-chain rotation matrices for a dense metric");
  s.gaussian = 1;
  s.rot = rotation;
  s.step_sizes = step_sizes;
  return leapfrog_euclidean_impl({pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size,
                                  n_steps, s, metric_kind, metric_inv, ModelArgs(), h_out, status,
                                  n_done, (cudaStream_t)stream, false},
                                 model);
}

int mb200_user_target_load(const void* image, int64_t image_bytes, const char* const* names,
                           int32_t n_names, void** handle) {
  if (!image || image_bytes <= 0 || !names || !handle)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_names != 2 * N_EU_LAYOUTS)
    return fail(MB200_ERR_INVALID_ARG, "expected %d kernel names, got %d", 2 * N_EU_LAYOUTS,
                n_names);
  return user_image_load(image, names, n_names, UserConstraintKernels{}, UserRiemannianKernels{},
                         handle);
}

int mb200_user_constraint_load(const void* image, int64_t image_bytes, const char* const* names,
                               int32_t n_names, int32_t n_constr, int32_t kp, int32_t mhp_constr,
                               void** handle) {
  if (!image || image_bytes <= 0 || !names || !handle)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_names != 2 * N_EU_LAYOUTS + 4)
    return fail(MB200_ERR_INVALID_ARG, "expected %d kernel names, got %d", 2 * N_EU_LAYOUTS + 4,
                n_names);
  if (n_constr < 1 || n_constr > 8 || (kp != 1 && kp != 2 && kp != 4))
    return fail(MB200_ERR_INVALID_ARG, "n_constr must be in [1, 8] and kp 1, 2 or 4");
  return user_image_load(image, names, n_names,
                         UserConstraintKernels{n_constr, kp, mhp_constr != 0, {}, {}},
                         UserRiemannianKernels{}, handle);
}

int mb200_user_riemannian_load(const void* image, int64_t image_bytes, const char* const* names,
                               int32_t n_names, int32_t rmetric_id, void** handle) {
  if (!image || image_bytes <= 0 || !names || !handle)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_names != 3) return fail(MB200_ERR_INVALID_ARG, "expected 3 kernel names, got %d", n_names);
  if (rmetric_id != MB200_RMETRIC_USER_DIAGONAL && rmetric_id != MB200_RMETRIC_USER_SCALAR &&
      rmetric_id != MB200_RMETRIC_USER_DENSE && rmetric_id != MB200_RMETRIC_USER_CHOLESKY)
    return fail(MB200_ERR_INVALID_ARG,
                "rmetric_id must be MB200_RMETRIC_USER_DIAGONAL, MB200_RMETRIC_USER_SCALAR, "
                "MB200_RMETRIC_USER_DENSE or MB200_RMETRIC_USER_CHOLESKY");
  return user_image_load(image, names, n_names, UserConstraintKernels{},
                         UserRiemannianKernels{rmetric_id, nullptr, nullptr, nullptr}, handle);
}

int mb200_user_target_unload(void* handle) {
  if (!handle) return fail(MB200_ERR_INVALID_ARG, "null handle");
  UserKernels* u = static_cast<UserKernels*>(handle);
  const cudaError_t e = cudaLibraryUnload(u->lib);
  delete u;
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "cudaLibraryUnload: %s", cudaGetErrorString(e));
  return 0;
}

int mb200_leapfrog_euclidean_user(const double* pos_in, const double* mom_in, double* pos_out,
                                  double* mom_out, const int32_t* dir, int64_t n_chains,
                                  int32_t dim, double step_size, const double* step_sizes,
                                  int32_t n_steps, const int32_t* n_steps_per_chain,
                                  int32_t n_flows, const double* coefficients,
                                  int32_t initial_h1_flow_step, int32_t metric_kind,
                                  const double* metric_inv, const mb200_model* model,
                                  double* h_out, int32_t* status, int32_t* n_done, void* stream,
                                  const void* user_target) {
  const UserKernels* u;
  if (const int rc = euclidean_image(user_target, &u)) return rc;
  return leapfrog_euclidean_entry(pos_in, mom_in, pos_out, mom_out, dir, n_chains, dim, step_size,
                                  step_sizes, n_steps, n_steps_per_chain, n_flows, coefficients,
                                  initial_h1_flow_step, metric_kind, metric_inv, model, h_out,
                                  status, n_done, (cudaStream_t)stream, false, u);
}

int mb200_hamiltonian_euclidean_user(const double* pos, const double* mom, int64_t n_chains,
                                     int32_t dim, int32_t metric_kind, const double* metric_inv,
                                     const mb200_model* model, double* h_out, void* stream,
                                     const void* user_target) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!h_out) return fail(MB200_ERR_INVALID_ARG, "h_out is NULL");
  // zero leapfrog steps, as mb200_hamiltonian_euclidean
  return mb200_leapfrog_euclidean_user(pos, mom, const_cast<double*>(pos),
                                       const_cast<double*>(mom), nullptr, n_chains, dim, 0.0,
                                       nullptr, 0, nullptr, 0, nullptr, 0, metric_kind,
                                       metric_inv, model, h_out, nullptr, nullptr, stream,
                                       user_target);
}

int mb200_euclidean_eval_user(const double* pos, const double* mom, int64_t n_chains, int32_t dim,
                              int32_t metric_kind, const double* metric_inv,
                              const mb200_model* model, double* nld_out, double* grad_out,
                              double* vel_out, double* kin_out, void* stream,
                              const void* user_target) {
  const UserKernels* u;
  if (const int rc = euclidean_image(user_target, &u)) return rc;
  return euclidean_eval_impl(pos, mom, n_chains, dim, metric_kind, metric_inv, model, nld_out,
                             grad_out, vel_out, kin_out, (cudaStream_t)stream, u);
}

int64_t mb200_host_scratch_bytes(int64_t n_chains, int32_t dim) {
  if (n_chains < 0 || dim < 1) return -1;
  return n_chains * ((int64_t)4 * dim * (int64_t)sizeof(double) + 2 * (int64_t)sizeof(int32_t));
}

int mb200_leapfrog_euclidean_host(const double* pos_in, const double* mom_in, double* pos_out,
                                  double* mom_out, const int32_t* dir, int64_t n_chains,
                                  int32_t dim, double step_size, int32_t n_steps,
                                  int32_t metric_kind, const double* metric_inv,
                                  const mb200_model* model, int32_t* status, int32_t n_chunks,
                                  void* const* streams, int32_t n_streams, void* scratch,
                                  int64_t scratch_bytes, int32_t synchronize) {
  if (n_chains == 0 && dim >= 1) return 0;
  if (!pos_in || !mom_in || !pos_out || !mom_out || !model || !streams || !scratch)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_chains < 0 || dim < 1 || n_steps < 0 || n_chunks < 1 || n_streams < 1)
    return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (scratch_bytes < mb200_host_scratch_bytes(n_chains, dim))
    return fail(MB200_ERR_INVALID_ARG, "scratch too small");
  const DeviceScope device_scope(scratch);
  const size_t nd = (size_t)n_chains * dim;
  double* d_qi = (double*)scratch;
  double* d_pi = d_qi + nd;
  double* d_qo = d_pi + nd;
  double* d_po = d_qo + nd;
  int32_t* d_status = (int32_t*)(d_po + nd);
  int32_t* d_dir = d_status + n_chains;
  // chunk boundaries on the granularity of a CTA of the kernel that will run (64 chains for K1, 16
  // for K1g), so that the chunks together launch no more CTAs than one launch over all chains would
  const int64_t align =
      k1_serves(metric_kind, dim, step_size, nullptr, n_steps, nullptr, model->target_id) ? 64 : 16;
  int64_t per = (n_chains + n_chunks - 1) / n_chunks;
  per = (per + align - 1) / align * align;
  if (is_pageable(pos_in) || is_pageable(mom_in) || is_pageable(pos_out) || is_pageable(mom_out)) {
    // pageable buffers: staged through pinned bounce buffers by the worker pool; the call is
    // synchronous (as CUDA's own pageable copies are)
    HostStager& hs = HostStager::get();
    std::lock_guard<std::mutex> call_lock(hs.call_mu);
    const size_t vec_bytes = nd * sizeof(double);
    char* pin = (char*)hs.bounce(4 * vec_bytes + 2 * (size_t)n_chains * sizeof(int32_t));
    if (!pin) return fail(MB200_ERR_CUDA, "host path: cannot allocate the pinned bounce buffer");
    double* b_qi = (double*)pin;
    double* b_pi = b_qi + nd;
    double* b_qo = b_pi + nd;
    double* b_po = b_qo + nd;
    int32_t* b_status = (int32_t*)(b_po + nd);
    int32_t* b_dir = b_status + n_chains;
    int dev = 0;
    cudaGetDevice(&dev);
    std::vector<std::function<void()>> tasks;
    std::vector<int> rcs;
    std::vector<std::string> msgs;
    int n_tasks = 0;
    for (int64_t lo = 0; lo < n_chains; lo += per) ++n_tasks;
    rcs.assign(n_tasks, 0), msgs.resize(n_tasks);
    int c = 0;
    for (int64_t lo = 0; lo < n_chains; lo += per, ++c) {
      const int64_t len = (lo + per <= n_chains) ? per : n_chains - lo;
      cudaStream_t st = (cudaStream_t)streams[c % n_streams];
      const size_t off = (size_t)lo * dim, bytes = (size_t)len * dim * sizeof(double);
      tasks.emplace_back([=, &rcs, &msgs] {
        cudaSetDevice(dev);
        memcpy(b_qi + off, pos_in + off, bytes);
        memcpy(b_pi + off, mom_in + off, bytes);
        if (dir) memcpy(b_dir + lo, dir + lo, len * sizeof(int32_t));
        cudaMemcpyAsync(d_qi + off, b_qi + off, bytes, cudaMemcpyHostToDevice, st);
        cudaMemcpyAsync(d_pi + off, b_pi + off, bytes, cudaMemcpyHostToDevice, st);
        if (dir)
          cudaMemcpyAsync(d_dir + lo, b_dir + lo, len * sizeof(int32_t), cudaMemcpyHostToDevice, st);
        int rc = mb200_leapfrog_euclidean(d_qi + off, d_pi + off, d_qo + off, d_po + off,
                                          dir ? d_dir + lo : nullptr, len, dim, step_size, nullptr,
                                          n_steps, nullptr, 0, nullptr, 0, metric_kind, metric_inv,
                                          model, nullptr, d_status + lo, nullptr, st);
        if (rc != 0) {
          rcs[c] = rc, msgs[c] = g_err;
          return;
        }
        cudaMemcpyAsync(b_qo + off, d_qo + off, bytes, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(b_po + off, d_po + off, bytes, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(b_status + lo, d_status + lo, len * sizeof(int32_t),
                        cudaMemcpyDeviceToHost, st);
        // NB several blocks may share a stream: wait for THIS block's work only
        cudaEvent_t ev;
        cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        cudaEventRecord(ev, st);
        const cudaError_t e = cudaEventSynchronize(ev);
        cudaEventDestroy(ev);
        if (e != cudaSuccess) {
          rcs[c] = MB200_ERR_CUDA, msgs[c] = cudaGetErrorString(e);
          return;
        }
        memcpy(pos_out + off, b_qo + off, bytes);
        memcpy(mom_out + off, b_po + off, bytes);
        if (status) memcpy(status + lo, b_status + lo, len * sizeof(int32_t));
      });
    }
    hs.run(tasks);
    for (int i = 0; i < n_tasks; ++i)
      if (rcs[i] != 0) return fail(rcs[i], "host path (block %d): %s", i, msgs[i].c_str());
    return 0;
  }
  int c = 0;
  for (int64_t lo = 0; lo < n_chains; lo += per, ++c) {
    const int64_t len = (lo + per <= n_chains) ? per : n_chains - lo;
    cudaStream_t st = (cudaStream_t)streams[c % n_streams];
    const size_t off = (size_t)lo * dim, bytes = (size_t)len * dim * sizeof(double);
    cudaMemcpyAsync(d_qi + off, pos_in + off, bytes, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(d_pi + off, mom_in + off, bytes, cudaMemcpyHostToDevice, st);
    if (dir) cudaMemcpyAsync(d_dir + lo, dir + lo, len * sizeof(int32_t), cudaMemcpyHostToDevice, st);
    const int rc = mb200_leapfrog_euclidean(d_qi + off, d_pi + off, d_qo + off, d_po + off,
                                            dir ? d_dir + lo : nullptr, len, dim, step_size,
                                            nullptr, n_steps, nullptr, 0, nullptr, 0, metric_kind,
                                            metric_inv, model, nullptr, d_status + lo, nullptr, st);
    if (rc != 0) return rc;
    cudaMemcpyAsync(pos_out + off, d_qo + off, bytes, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(mom_out + off, d_po + off, bytes, cudaMemcpyDeviceToHost, st);
    if (status)
      cudaMemcpyAsync(status + lo, d_status + lo, len * sizeof(int32_t), cudaMemcpyDeviceToHost, st);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "host path: %s", cudaGetErrorString(e));
  if (synchronize) {
    const int used = c < n_streams ? c : n_streams;
    for (int i = 0; i < used; ++i) {
      e = cudaStreamSynchronize((cudaStream_t)streams[i]);
      if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "host path: %s", cudaGetErrorString(e));
    }
  }
  return 0;
}

}  // extern "C"
