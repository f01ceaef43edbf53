// libmici_b200.so -- C-ABI glue of the global-workspace dense metric policy (dense_global.cuh):
// implicit leapfrog / Hamiltonian / momentum refresh / velocity on Riemannian systems whose
// per-chain D x D metric does not fit in shared memory (config C4: D = 512), and the diagnostic
// entry point of the blocked factorisation.
#include "api_common.cuh"
#include "dense_global.cuh"

namespace mb200 {

static int dg_blocks(int64_t n) {
  const int64_t cap = (int64_t)num_sms();  // one CTA per SM (its shared memory is ~200 KB)
  return (int)(n < cap ? n : cap);
}

int64_t dense_global_workspace_bytes(int64_t n_chains, int dim) {
  return (int64_t)dg_blocks(n_chains) * (int64_t)dg_workspace_doubles(dim) * (int64_t)sizeof(double);
}

bool dense_global_supported(int dim) {
  return rm_smem_bytes(dg_layout(dim)) <= RM_SMEM_BYTES;
}

// The kernels this plan starts: a registry instantiation, or a kernel of a loaded user image (a
// cudaKernel_t) with the same parameters
using DgImplicitKernel = decltype(&implicit_leapfrog_kernel<QuadraticRTarget, GlobalDenseRank1>);
using DgVectorKernel = decltype(&riemannian_velocity_kernel<QuadraticRTarget, GlobalDenseRank1>);

static int dg_launch_implicit(DgImplicitKernel kern, const ImplicitArgs& a) {
  const RmLayout layout = dg_layout(a.dim);
  const size_t smem = rm_smem_bytes(layout);
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "smem attr: %s", cudaGetErrorString(e));
  const int blocks = dg_blocks(a.n);
  DgScratch scratch(a.ws, a.ws_bytes, (size_t)dense_global_workspace_bytes(a.n, a.dim), a.st);
  if (scratch.ptr == nullptr) return fail(MB200_ERR_CUDA, "dense metric workspace allocation failed");
  ModelArgs m = a.m;
  m.workspace = scratch.ptr;
  m.ws_stride = dg_workspace_doubles(a.dim);
  rm_start(kern, (unsigned)blocks, DG_THREADS, smem, a.st, a.q_in, a.p_in, a.q_out, a.p_out, a.dir,
           a.n, a.dim, a.eps, a.n_steps, m, a.fp_tol, a.fp_div, a.fp_max, a.rev_tol, a.h_out,
           a.status, a.n_done, a.fp_iters, layout, 0, a.fp_solver);
  return check_launch("implicit_leapfrog_kernel (global dense metric)");
}

int dense_global_implicit(const ImplicitArgs& a, bool hadamard) {
  return dg_launch_implicit(hadamard ? implicit_leapfrog_kernel<QuadraticRTarget, GlobalDenseHadamard>
                                     : implicit_leapfrog_kernel<QuadraticRTarget, GlobalDenseRank1>,
                            a);
}

int dense_global_implicit_image(const ImplicitArgs& a, const void* kern) {
  return dg_launch_implicit(reinterpret_cast<DgImplicitKernel>(kern), a);
}

static int dg_launch_vec(DgVectorKernel kern, const VectorArgs& a) {
  const RmLayout layout = dg_layout(a.dim);
  const size_t smem = rm_smem_bytes(layout);
  const int blocks = dg_blocks(a.n);
  DgScratch scratch(nullptr, 0, (size_t)dense_global_workspace_bytes(a.n, a.dim), a.st);
  if (scratch.ptr == nullptr) return fail(MB200_ERR_CUDA, "dense metric workspace allocation failed");
  ModelArgs m = a.m;
  m.workspace = scratch.ptr;
  m.ws_stride = dg_workspace_doubles(a.dim);
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "smem attr: %s", cudaGetErrorString(e));
  rm_start(kern, (unsigned)blocks, DG_THREADS, smem, a.st, a.q, a.v, a.out, a.n, a.dim, m,
           a.status, layout);
  return check_launch("riemannian vector kernel (global dense metric)");
}

// velocity: out = M(q)^-1 v ; else out = chol(M(q)) v
int dense_global_vector(const VectorArgs& a, bool velocity, bool hadamard) {
  if (velocity)
    return dg_launch_vec(hadamard ? riemannian_velocity_kernel<QuadraticRTarget, GlobalDenseHadamard>
                                  : riemannian_velocity_kernel<QuadraticRTarget, GlobalDenseRank1>,
                         a);
  return dg_launch_vec(
      hadamard ? riemannian_sample_momentum_kernel<QuadraticRTarget, GlobalDenseHadamard>
               : riemannian_sample_momentum_kernel<QuadraticRTarget, GlobalDenseRank1>,
      a);
}

int dense_global_vector_image(const VectorArgs& a, const void* kern) {
  return dg_launch_vec(reinterpret_cast<DgVectorKernel>(kern), a);
}

}  // namespace mb200

using namespace mb200;

extern "C" {

int mb200_selftest_dense_factor(const double* matrices, const double* rhs, int64_t n_matrices,
                                int32_t dim, double* chol_out, double* inv_out, double* sol_out,
                                double* logdet_out, int32_t* status, void* stream) {
  if (!matrices || !rhs || !chol_out || !inv_out || !sol_out || !logdet_out || !status)
    return fail(MB200_ERR_INVALID_ARG, "null pointer argument");
  if (n_matrices < 0 || dim < 1) return fail(MB200_ERR_INVALID_ARG, "bad sizes");
  if (n_matrices == 0) return 0;
  if (!dense_global_supported(dim))
    return fail(MB200_ERR_UNSUPPORTED, "dim %d: panel buffers exceed shared memory", dim);
  const DeviceScope device_scope(matrices);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = rm_smem_bytes(dg_layout(dim));
  cudaError_t e = cudaFuncSetAttribute(dense_global_selftest_kernel,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail(MB200_ERR_CUDA, "smem attr: %s", cudaGetErrorString(e));
  const int blocks = dg_blocks(n_matrices);
  DgScratch scratch(nullptr, 0, (size_t)dense_global_workspace_bytes(n_matrices, dim), st);
  if (scratch.ptr == nullptr) return fail(MB200_ERR_CUDA, "workspace allocation failed");
  ModelArgs m;
  memset(&m, 0, sizeof(m));
  m.workspace = scratch.ptr;
  m.ws_stride = dg_workspace_doubles(dim);
  dense_global_selftest_kernel<<<(unsigned)blocks, DG_THREADS, smem, st>>>(
      matrices, rhs, n_matrices, dim, m, chol_out, inv_out, sol_out, logdet_out, status);
  return check_launch("dense_global_selftest_kernel");
}

}  // extern "C"
