// K2 / K3 / K4 / K5: implicit generalised leapfrog on a Riemannian-metric system --
// one CTA per chain, everything for the chain resident in shared memory.
//
// Replaces, per chain (reference paths):
//   ImplicitLeapfrogIntegrator._step and sub-steps          integrators.py:482-544
//   solve_fixed_point_direct                                solvers.py:47-94
//   RiemannianMetricSystem.{metric,h1,dh1_dpos,h2,dh2_dpos,dh2_dmom}   systems.py:1360-1402
//   DensePositiveDefiniteMatrix (Cholesky, solves, logdet, gradients)  matrices.py:1161-1188
//   SoftAbsRegularizedPositiveDefiniteMatrix (eigh, softabs, gradients) matrices.py:1631-1685
//
// Per-chain control flow (fixed-point convergence / divergence, reversibility failure) is the
// CTA's own uniform control flow: chains that converge early simply retire their CTA and the
// next chain is scheduled, so divergent iteration counts cost no idle lanes.
//
// K3 (symmetric eigensolver) is a parallel cyclic two-sided Jacobi iteration: D/2 disjoint
// rotations per round (round-robin ordering), each round applied as R^T A R on 2x2 blocks, the
// eigenvectors accumulated as U R.  Jacobi is used because it is the most accurate dense
// symmetric eigensolver (relative accuracy of eigenvectors), which the divided differences in
// grad_quadratic_form_inv (matrices.py:1679-1685) need, and because it parallelises over a CTA
// without any serial tridiagonal phase.
#pragma once
#ifndef __CUDACC_RTC__
#include <cfloat>
#elif !defined(DBL_EPSILON)
#define DBL_EPSILON 2.2204460492503131e-16  // NVRTC (user_riemannian.cuh) has no <cfloat>
#endif

#include "common.cuh"

namespace mb200 {

constexpr int RM_THREADS = 256;
constexpr int RM_MAX_SWEEPS = 40;

// Address-space statements for pointer VALUES whose origin the compiler cannot see (pointers that
// reach a non-inlined function through a struct in memory would otherwise be dereferenced with
// generic LD / ST instead of LDS / STS or LDG / STG).
#define RM_SHARED(p) __builtin_assume(__isShared(p))
#define RM_GLOBAL(p) __builtin_assume(__isGlobal(p))

struct Blk {
  int tid, nthr, lane, warp, nwarp;
  double* red;  // [34] reduction scratch
};

__device__ __forceinline__ double block_sum(const Blk& b, double v) {
  v = warp_sum(v);
  __syncthreads();
  if (b.lane == 0) b.red[b.warp] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < b.nwarp; ++w) t += b.red[w];
  return t;
}

__device__ __forceinline__ double block_nanmax(const Blk& b, double v) {
  v = warp_nanmax(v);
  __syncthreads();
  if (b.lane == 0) b.red[b.warp] = v;
  __syncthreads();
  double t = b.red[0];
  for (int w = 1; w < b.nwarp; ++w) t = nanmax(t, b.red[w]);
  return t;
}

// true on all threads iff `flag` is true on any thread
__device__ __forceinline__ bool block_any(const Blk&, bool flag) {
  return __syncthreads_or(flag ? 1 : 0) != 0;
}

// ---------------------------------------------------------------------------------------------
// Targets (block-cooperative interface; vectors in shared memory)
// ---------------------------------------------------------------------------------------------

struct BananaRTarget {
  static constexpr bool DENSE_MTP = false;
  __device__ void attach(double*) const {}
  static constexpr bool HAS_HESSIAN = true;
  static constexpr int NEED = 2;  // entries of a D x D gradient matrix needed per row by mtp
  double b;
  int dim;
  __device__ BananaRTarget(const ModelArgs& m, int d) : b(m.tp[0]), dim(d) {}

  __device__ double nld(const Blk& k, const double* q) const {
    double s = 0.0;
    for (int i = 2 * k.tid; i < dim; i += 2 * k.nthr) {
      const double x = q[i], y = q[i + 1], r = y - b * x * x;
      s += x * x / 8.0 + 0.5 * r * r;
    }
    return block_sum(k, s);
  }
  __device__ void grad(const Blk& k, const double* q, double* g) const {
    for (int i = 2 * k.tid; i < dim; i += 2 * k.nthr) {
      const double x = q[i], y = q[i + 1], r = y - b * x * x;
      g[i] = x / 4.0 - 2.0 * b * x * r;
      g[i + 1] = r;
    }
  }
  // dense Hessian (block diagonal for this model, but produced and consumed as a dense matrix)
  __device__ void hess(const Blk& k, const double* q, double* A, int ld) const {
    for (int idx = k.tid; idx < dim * dim; idx += k.nthr) {
      const int i = idx / dim, j = idx - i * dim;
      const int pi = i & ~1;
      double v = 0.0;
      if ((j & ~1) == pi) {
        const double x = q[pi], y = q[pi + 1];
        if (i == pi && j == pi) v = 0.25 - 2.0 * b * y + 6.0 * b * b * x * x;
        else if (i == pi + 1 && j == pi + 1) v = 1.0;
        else v = -2.0 * b * x;
      }
      A[i * ld + j] = v;
    }
  }
  // columns of row `a` of the matrix argument that the matrix-Tressian product reads
  __device__ __forceinline__ int need_col(int a, int j) const {
    if ((a & 1) == 0) return a + j;  // (x,x), (x,y)
    return j == 0 ? a - 1 : -1;      // (y,x)
  }
  // mtp(V)_k = sum_ij V_ij d^3 l / dq_i dq_j dq_k  from the needed entries Vn[a][j]
  __device__ void mtp_entries(const Blk& k, const double* q, const double* Vn, double* out) const {
    for (int i = 2 * k.tid; i < dim; i += 2 * k.nthr) {
      const double x = q[i];
      const double vxx = Vn[i * NEED + 0], vxy = Vn[i * NEED + 1], vyx = Vn[(i + 1) * NEED + 0];
      out[i] = vxx * (12.0 * b * b * x) - 2.0 * b * (vxy + vyx);
      out[i + 1] = -2.0 * b * vxx;
    }
  }
};

struct QuadraticRTarget {
  static constexpr bool DENSE_MTP = false;
  __device__ void attach(double*) const {}
  static constexpr bool HAS_HESSIAN = false;
  static constexpr int NEED = 1;
  const double* P;
  int dim;
  __device__ QuadraticRTarget(const ModelArgs& m, int d) : P(m.taux), dim(d) {}
  __device__ void grad(const Blk& k, const double* q, double* g) const {
    for (int i = k.tid; i < dim; i += k.nthr) {
      const double* row = P + (size_t)i * dim;
      double s = 0.0;
      for (int j = 0; j < dim; ++j) s = fma(row[j], q[j], s);
      g[i] = s;
    }
  }
  __device__ double nld(const Blk& k, const double* q) const {
    double s = 0.0;
    for (int i = k.tid; i < dim; i += k.nthr) {
      const double* row = P + (size_t)i * dim;
      double t = 0.0;
      for (int j = 0; j < dim; ++j) t = fma(row[j], q[j], t);
      s = fma(q[i], t, s);
    }
    return 0.5 * block_sum(k, s);
  }
  __device__ void hess(const Blk&, const double*, double*, int) const {}
  __device__ __forceinline__ int need_col(int, int) const { return -1; }
  __device__ void mtp_entries(const Blk&, const double*, const double*, double*) const {}
};

struct StdGaussianRTarget {
  static constexpr bool DENSE_MTP = false;
  __device__ void attach(double*) const {}
  static constexpr bool HAS_HESSIAN = false;
  static constexpr int NEED = 1;
  int dim;
  __device__ StdGaussianRTarget(const ModelArgs&, int d) : dim(d) {}
  __device__ void grad(const Blk& k, const double* q, double* g) const {
    for (int i = k.tid; i < dim; i += k.nthr) g[i] = q[i];
  }
  __device__ double nld(const Blk& k, const double* q) const {
    double s = 0.0;
    for (int i = k.tid; i < dim; i += k.nthr) s = fma(q[i], q[i], s);
    return 0.5 * block_sum(k, s);
  }
  __device__ void hess(const Blk&, const double*, double*, int) const {}
  __device__ __forceinline__ int need_col(int, int) const { return -1; }
  __device__ void mtp_entries(const Blk&, const double*, const double*, double*) const {}
};

// Neal's funnel, v = q[0], x = q[1:]: l = v^2/18 + (D-1) v/2 + exp(-v) |x|^2/2 (the expressions
// of the NumPy model, oracle/targets.py NealFunnel).  No Hessian: diagonal / scalar metrics only.
struct FunnelRTarget {
  static constexpr bool DENSE_MTP = false;
  __device__ void attach(double*) const {}
  static constexpr bool HAS_HESSIAN = false;
  static constexpr int NEED = 1;
  int dim;
  __device__ FunnelRTarget(const ModelArgs&, int d) : dim(d) {}
  __device__ double xsq(const Blk& k, const double* q) const {
    double s = 0.0;
    for (int i = 1 + k.tid; i < dim; i += k.nthr) s = fma(q[i], q[i], s);
    return block_sum(k, s);
  }
  __device__ double nld(const Blk& k, const double* q) const {
    const double s = xsq(k, q), v = q[0];
    return (v * v / 18.0 + 0.5 * (dim - 1) * v) + 0.5 * exp(-v) * s;
  }
  __device__ void grad(const Blk& k, const double* q, double* g) const {
    const double s = xsq(k, q), v = q[0], e = exp(-v);
    for (int i = k.tid; i < dim; i += k.nthr)
      g[i] = (i == 0) ? (v / 9.0 + 0.5 * (dim - 1)) - 0.5 * e * s : e * q[i];
  }
  __device__ void hess(const Blk&, const double*, double*, int) const {}
  __device__ __forceinline__ int need_col(int, int) const { return -1; }
  __device__ void mtp_entries(const Blk&, const double*, const double*, double*) const {}
};

// l(q) = |q|^2/2 + (gamma/4) sum_m (a_m . q)^4, A = directions [D x D] in global memory (shared
// by all chains, L2-resident).  Dense Hessian I + 3 gamma A^T diag(s^2) A, s = A q; the
// matrix-Tressian product mtp(V)_k = 6 gamma sum_m s_m (a_m^T V a_m) a_mk needs the whole of V:
// the SoftAbs policy hands this target the factors of V instead of entries (DENSE_MTP):
//   V = U diag(d) U^T           ->  a_m^T V a_m = sum_i d_i Z_mi^2,          Z = A U
//   V = -U ((e e^T) o J) U^T    ->  a_m^T V a_m = -(z_m o e)^T J (z_m o e)
struct QuarticRTarget {
  static constexpr bool DENSE_MTP = true;
  static constexpr bool HAS_HESSIAN = true;
  static constexpr int NEED = 1;
  const double* A;
  double gamma;
  int dim;
  mutable double* sbuf;  // [dim] shared scratch for s = A q (attached after the carve)
  __device__ QuarticRTarget(const ModelArgs& m, int d)
      : A(m.taux), gamma(m.tp[0]), dim(d), sbuf(nullptr) {}
  __device__ void attach(double* scratch) const { sbuf = scratch; }

  // s = A q into sbuf (one warp per direction)
  __device__ void project(const Blk& k, const double* q) const {
    for (int m = k.warp; m < dim; m += k.nwarp) {
      double t = 0.0;
      for (int j = k.lane; j < dim; j += 32) t = fma(A[(size_t)m * dim + j], q[j], t);
      t = warp_sum(t);
      if (k.lane == 0) sbuf[m] = t;
    }
    __syncthreads();
  }
  // out_k = base_k + coef * sum_m A_mk w_m  (coalesced over k)
  __device__ void back_project(const Blk& k, const double* wv, double coef, const double* base,
                               double* out) const {
    for (int i = k.tid; i < dim; i += k.nthr) {
      double t = 0.0;
      for (int m = 0; m < dim; ++m) t = fma(A[(size_t)m * dim + i], wv[m], t);
      out[i] = (base != nullptr ? base[i] : 0.0) + coef * t;
    }
    __syncthreads();
  }
  __device__ double nld(const Blk& k, const double* q) const {
    project(k, q);
    double t = 0.0;
    for (int i = k.tid; i < dim; i += k.nthr) {
      const double s2 = sbuf[i] * sbuf[i];
      t += 0.5 * (q[i] * q[i]) + 0.25 * gamma * (s2 * s2);
    }
    return block_sum(k, t);
  }
  __device__ void grad(const Blk& k, const double* q, double* g) const {
    project(k, q);
    for (int i = k.tid; i < dim; i += k.nthr) sbuf[i] = sbuf[i] * sbuf[i] * sbuf[i];
    __syncthreads();
    back_project(k, sbuf, gamma, q, g);
  }
  // H = I + 3 gamma A^T diag(s^2) A, 4x4 register tiles
  __device__ void hess(const Blk& k, const double* q, double* H, int ld) const {
    project(k, q);
    for (int i = k.tid; i < dim; i += k.nthr) sbuf[i] = 3.0 * gamma * (sbuf[i] * sbuf[i]);
    __syncthreads();
    const int tn = (dim + 3) / 4;
    for (int t = k.tid; t < tn * tn; t += k.nthr) {
      const int i0 = 4 * (t / tn), j0 = 4 * (t % tn);
      double acc[4][4];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
      for (int m = 0; m < dim; ++m) {
        const double* row = A + (size_t)m * dim;
        const double wm = sbuf[m];
        double x[4], y[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          x[a] = (i0 + a < dim) ? wm * row[i0 + a] : 0.0;
          y[a] = (j0 + a < dim) ? row[j0 + a] : 0.0;
        }
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) acc[a][b] = fma(x[a], y[b], acc[a][b]);
      }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b)
          if (i0 + a < dim && j0 + b < dim)
            H[(i0 + a) * ld + j0 + b] = acc[a][b] + ((i0 + a == j0 + b) ? 1.0 : 0.0);
    }
    __syncthreads();
  }
  __device__ __forceinline__ int need_col(int, int) const { return -1; }
  __device__ void mtp_entries(const Blk&, const double*, const double*, double*) const {}

  // Z = A U (directions in the eigenbasis), Z [dim x dim] stride ld in shared memory
  __device__ void eigen_directions(const Blk& k, const double* U, int ld, double* Z) const {
    const int tn = (dim + 3) / 4;
    for (int t = k.tid; t < tn * tn; t += k.nthr) {
      const int m0 = 4 * (t / tn), j0 = 4 * (t % tn);
      double acc[4][4];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
      for (int i = 0; i < dim; ++i) {
        double x[4], y[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          x[a] = (m0 + a < dim) ? A[(size_t)(m0 + a) * dim + i] : 0.0;
          y[a] = (j0 + a < dim) ? U[i * ld + j0 + a] : 0.0;
        }
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) acc[a][b] = fma(x[a], y[b], acc[a][b]);
      }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b)
          if (m0 + a < dim && j0 + b < dim) Z[(m0 + a) * ld + j0 + b] = acc[a][b];
    }
    __syncthreads();
  }
  // out = mtp(U diag(d) U^T): t_m = sum_i d_i Z_mi^2
  __device__ void mtp_diag(const Blk& k, const double* q, const double* Z, int ld, const double* d,
                           double* tm, double* out) const {
    project(k, q);
    for (int m = k.warp; m < dim; m += k.nwarp) {
      double t = 0.0;
      for (int i = k.lane; i < dim; i += 32) t = fma(d[i] * Z[m * ld + i], Z[m * ld + i], t);
      t = warp_sum(t);
      if (k.lane == 0) tm[m] = sbuf[m] * t;
    }
    __syncthreads();
    back_project(k, tm, 6.0 * gamma, nullptr, out);
  }
  // out = mtp(-U ((e e^T) o J) U^T): t_m = -(z_m o e)^T J (z_m o e); one warp per direction,
  // y = z_m o e staged per warp in `ybuf` [nwarp * dim]
  __device__ void mtp_quad(const Blk& k, const double* q, const double* Z, int ld, const double* e,
                           const double* J, int ldj, double* ybuf, double* tm, double* out) const {
    project(k, q);
    double* y = ybuf + (size_t)k.warp * dim;
    for (int m = k.warp; m < dim; m += k.nwarp) {
      for (int i = k.lane; i < dim; i += 32) y[i] = Z[m * ld + i] * e[i];
      __syncwarp();
      double t = 0.0;
      for (int j = k.lane; j < dim; j += 32) {
        double u = 0.0;
        for (int i = 0; i < dim; ++i) u = fma(y[i], J[i * ldj + j], u);
        t = fma(u, y[j], t);
      }
      t = warp_sum(t);
      if (k.lane == 0) tm[m] = -(sbuf[m] * t);
      __syncwarp();
    }
    __syncthreads();
    back_project(k, tm, 6.0 * gamma, nullptr, out);
  }
};

// ---------------------------------------------------------------------------------------------
// shared-memory workspace of one chain
// ---------------------------------------------------------------------------------------------
struct RmWork {
  int dim, ld;
  double *M1, *M2, *M3;  // [dim*ld] each (M2: SoftAbs; M3: SoftAbs warm start, when it fits)
  double *q, *p, *qs, *ps, *x0, *x1, *x2, *base, *v1, *v2, *v3, *lam, *sa, *gsa, *ev, *Vn;
  double *z0, *z1, *z2, *zb, *zp;  // [2*dim] implicit midpoint: iterates, base, previous (q, p)
  double *rc, *rs;  // rotation cos / sin [dim/2 + 1]
  int *top, *bot;   // round-robin index arrays [dim/2 + 1]
  double* extra;    // shared memory beyond the carved vectors (global-dense policy: panel buffers)
};

// shared-memory doubles the global-workspace dense policy (dense_global.cuh) needs beyond the
// vectors: the panel [(np - 32) x 36], the diagonal block and its inverse [32 x 36] each
__host__ __device__ inline int dg_padded_dim(int dim) { return (dim + 31) & ~31; }
__host__ __device__ inline size_t dg_smem_doubles(int dim) {
  const int np = dg_padded_dim(dim);
  return (size_t)(np > 32 ? np - 32 : 32) * 36 + 2 * 32 * 36;
}
// opt-in dynamic shared memory of one CTA on sm_90 (228 KB per SM, 1 KB of it reserved per CTA)
constexpr size_t RM_SMEM_BYTES = 227 * 1024;

// Where a chain's buffers live.  Every metric policy declares its PLACE; those that rm_launch
// plans also declare the per-chain D x D matrices they keep in shared memory (N_MATS) and how many
// of them move to the per-CTA global workspace when those do not fit (WORKSPACE_MATS, 0: no such
// route).
enum RmPlace : int {
  // the O(D) policies (diagonal and scalar metrics): the integrator's vectors plus ev (policy
  // scratch), lam (d(q)) and sa (1 / d(q)), and the implicit-midpoint vectors only for implicit
  // midpoint; no matrices, no eigensolver or Cholesky buffers: at D = 128 a chain needs 14.6 KB
  // (leapfrog), so that many chains share an SM
  RM_COMPACT,
  // the matrix policies: every vector, and the matrices in shared memory or, beyond it (SoftAbs
  // at D > ~100, the Cholesky-factored metric's factor at D > ~150), in the per-CTA global
  // workspace: the algorithms are unchanged, the operands are simply L2-resident
  RM_MATRICES,
  // the global-workspace dense policy (dense_global.cuh): the integrator's vectors and ev, then
  // its panel buffers (dg_smem_doubles) from `extra`
  RM_DENSE_GLOBAL,
};

// The layout of one chain's buffers: planned on the host (rm_launch, the dense-global launchers)
// and passed to the kernels
struct RmLayout {
  int dim;
  RmPlace place;
  int smem_mats;  // RM_MATRICES: per-chain D x (D + 1) matrices in shared memory
  int ws_mats;    // ... or in the per-CTA global workspace (then smem_mats == 0)
  bool zvecs;     // RM_COMPACT: the implicit-midpoint vectors too (RM_MATRICES: always)
  // doubles from one workspace matrix to the next (each starts 16-byte aligned); a CTA's
  // workspace is ws_mats of them
  __host__ __device__ size_t ws_mat_doubles() const {
    return ((size_t)dim * (dim + 1) + 1) & ~(size_t)1;
  }
};

// Carves the buffers of layout `l` from shared memory `s` and this CTA's workspace `gmats`: every
// pointer of `w` (those the layout lacks are NULL), the reduction scratch blk.red [40 doubles],
// `extra` (what follows it) and *tscratch, the [dim] scratch of DENSE_MTP targets.  Returns the
// doubles of shared memory the layout takes; the host sizes a launch by running it from a null
// base (rm_smem_bytes), so the size and the pointers cannot disagree.  Vectors are dpad apart:
//   RM_COMPACT       q p qs ps x0 x1 x2 base v1 v2 v3 ev lam sa [z0 z1 z2 zb zp] red
//   RM_DENSE_GLOBAL  q p qs ps x0 x1 x2 base v1 v2 v3 ev red, panel buffers
//   RM_MATRICES      [M1 M2 M3] q p qs ps x0 x1 x2 base v1 v2 v3 lam sa gsa ev Vn z0 z1 z2 zb zp
//                    rc rs top bot red
// where Vn and z0 .. zp take 2 dpad each, rc, rs and top / bot (ints) dpad / 2 + 2 each.
__host__ __device__ __forceinline__ size_t rm_carve(const RmLayout& l, double* s, double* gmats,
                                                    Blk& blk, RmWork& w, double** tscratch) {
  double* const s0 = s;
  const int dim = l.dim;
  const int ld = dim + 1;
  const int dpad = (dim + 1) & ~1;
  w.dim = dim;
  w.ld = ld;
  size_t beyond = 0;  // doubles the policy carves from `extra` itself
  if (l.place == RM_COMPACT) {
    w.M1 = w.M2 = w.M3 = nullptr;
    double** cv[] = {&w.q,  &w.p,  &w.qs, &w.ps, &w.x0, &w.x1, &w.x2,
                     &w.base, &w.v1, &w.v2, &w.v3, &w.ev, &w.lam, &w.sa};
    for (auto v : cv) {
      *v = s;
      s += dpad;
    }
    w.gsa = w.Vn = nullptr;
    w.rc = w.rs = nullptr;
    w.top = w.bot = nullptr;
    if (l.zvecs) {
      double** zv[] = {&w.z0, &w.z1, &w.z2, &w.zb, &w.zp};
      for (auto v : zv) {
        *v = s;
        s += 2 * dpad;
      }
    } else {
      w.z0 = w.z1 = w.z2 = w.zb = w.zp = nullptr;
    }
  } else if (l.place == RM_DENSE_GLOBAL) {
    w.M1 = w.M2 = w.M3 = nullptr;
    double** cv[] = {&w.q, &w.p, &w.qs, &w.ps, &w.x0, &w.x1, &w.x2, &w.base, &w.v1, &w.v2, &w.v3,
                     &w.ev};
    for (auto v : cv) {
      *v = s;
      s += dpad;
    }
    w.lam = w.sa = w.gsa = w.Vn = nullptr;
    w.z0 = w.z1 = w.z2 = w.zb = w.zp = nullptr;
    w.rc = w.rs = nullptr;
    w.top = w.bot = nullptr;
    beyond = dg_smem_doubles(dim);
  } else {
    if (l.ws_mats > 0) {
      const int km = l.ws_mats;
      const size_t sq = l.ws_mat_doubles();
      w.M1 = km >= 1 ? gmats : nullptr;
      w.M2 = km >= 2 ? gmats + sq : nullptr;
      w.M3 = km >= 3 ? gmats + 2 * sq : nullptr;
    } else {
      const int nm = l.smem_mats;
      w.M1 = nm >= 1 ? s : nullptr;
      if (nm >= 1) s += (size_t)dim * ld;
      w.M2 = nm >= 2 ? s : nullptr;
      if (nm >= 2) s += (size_t)dim * ld;
      w.M3 = nm >= 3 ? s : nullptr;
      if (nm >= 3) s += (size_t)dim * ld;
    }
    double** vecs[] = {&w.q, &w.p, &w.qs, &w.ps, &w.x0, &w.x1, &w.x2, &w.base, &w.v1,
                       &w.v2, &w.v3, &w.lam, &w.sa, &w.gsa, &w.ev};
    for (auto v : vecs) {
      *v = s;
      s += dpad;
    }
    w.Vn = s;  // NEED <= 2 entries per coordinate
    s += 2 * dpad;
    w.z0 = s;
    s += 2 * dpad;
    w.z1 = s;
    s += 2 * dpad;
    w.z2 = s;
    s += 2 * dpad;
    w.zb = s;
    s += 2 * dpad;
    w.zp = s;
    s += 2 * dpad;
    w.rc = s;
    s += dpad / 2 + 2;
    w.rs = s;
    s += dpad / 2 + 2;
    w.top = reinterpret_cast<int*>(s);
    w.bot = w.top + (dpad / 2 + 2);
    s += dpad / 2 + 2;
  }
  blk.red = s;
  s += 40;
  w.extra = s;
  // DENSE_MTP targets (SoftAbs, RM_THREADS): the per-warp staging rows and the per-direction
  // results take (nwarp + 1) x dim doubles of the Vn / z0 .. zp region, which is contiguous, and
  // this scratch the next dim: the region's 12 dpad hold (nwarp + 2) x dim
  static_assert(RM_THREADS / 32 + 2 <= 12, "DENSE_MTP scratch beyond the Vn / z region");
  *tscratch = w.Vn != nullptr ? w.Vn + (size_t)(blk.nwarp + 1) * dim : nullptr;
  return (size_t)(s - s0) + beyond;
}

__host__ __device__ inline size_t rm_smem_bytes(const RmLayout& l) {
  Blk blk{};
  RmWork w;
  double* tscratch;
  return rm_carve(l, nullptr, nullptr, blk, w, &tscratch) * sizeof(double);
}

// The start of every Riemannian kernel: the CTA's Blk, and the chain's buffers carved by layout
// `l` from dynamic shared memory and this CTA's share of m.workspace.  Returns the scratch of
// DENSE_MTP targets (Target::attach).  COMPACT: the kernel's policy is an RM_COMPACT one, so
// every layout it is launched with is; a matrix policy's kernel is never launched with one.
// STEPS: the kernel integrates (the velocity and momentum kernels take no step, so a compact
// layout carves no midpoint vectors for them).  Stating both at compile time leaves only the
// carves that can run in the kernel.
template <bool COMPACT, bool STEPS = true>
__device__ __forceinline__ double* rm_begin(RmLayout l, const ModelArgs& m, Blk& blk,
                                            RmWork& w) {
  extern __shared__ double smem[];
  blk.tid = threadIdx.x, blk.nthr = blockDim.x, blk.lane = threadIdx.x & 31;
  blk.warp = threadIdx.x >> 5, blk.nwarp = blockDim.x >> 5;
  l.place = COMPACT ? RM_COMPACT : l.place == RM_DENSE_GLOBAL ? RM_DENSE_GLOBAL : RM_MATRICES;
  if (!STEPS) l.zvecs = false;
  double* tscratch;
  rm_carve(l, smem,
           m.workspace != nullptr ? m.workspace + (size_t)blockIdx.x * m.ws_stride : nullptr, blk,
           w, &tscratch);
  return tscratch;
}

// true for policies whose build() accepts a metric that cannot be solved with (a zero pivot of
// a triangular factor: `static constexpr bool CAN_BE_SINGULAR = true` and a `singular()`
// member); the velocity kernel and the energy then report it
template <class M, class = void>
struct rm_singular_policy {
  static constexpr bool value = false;
};
template <class M>
struct rm_singular_policy<M, decltype(void(M::CAN_BE_SINGULAR))> {
  static constexpr bool value = M::CAN_BE_SINGULAR;
};

// ---------------------------------------------------------------------------------------------
// K3: symmetric eigendecomposition A = U diag(lam) U^T by parallel cyclic Jacobi.
// A [dim x dim, stride ld] is destroyed (its diagonal becomes lam); U receives the eigenvectors
// as columns.  Returns false if not converged / non-finite (-> LinAlgError, matrices.py:437).
// ---------------------------------------------------------------------------------------------
// Round-robin (circle method) schedule over np "seats": in round r of np-1, pair t couples seats
//   t == 0 : (np-1, r)          t > 0 : ((r+t) mod (np-1), (r-t) mod (np-1))
// so every unordered pair meets exactly once per sweep; no schedule arrays.  Matrix indices are
// dealt to the seats such that round 0 couples the adjacent indices (0,1), (2,3), ...: models
// whose Hessian couples coordinates in consecutive pairs then finish all their rotations in the
// first round and every other round is skipped by the look-ahead.
__device__ __forceinline__ int rr_seat_index(int np, int seat) {
  if (seat == np - 1) return 1;
  if (seat == 0) return 0;
  const int m = np >> 1;
  return seat < m ? 2 * seat : 2 * (np - 1 - seat) + 1;
}
__device__ __forceinline__ void rr_pair(int np, int r, int t, int& p, int& q) {
  const int m1 = np - 1;
  int a, b;
  if (t == 0) {
    a = m1;
    b = r;
  } else {
    a = r + t;
    if (a >= m1) a -= m1;
    b = r - t;
    if (b < 0) b += m1;
  }
  a = rr_seat_index(np, a);
  b = rr_seat_index(np, b);
  p = a < b ? a : b;
  q = a < b ? b : a;
}

// `warm`: U already holds an orthogonal basis V and A holds V^T H V (nearly diagonal); the
// rotations are accumulated onto V, so that on return U holds the eigenvectors of H.
// SH: A and U are known to live in shared memory.  RmWork's pointers reach this (non-inlined)
// function through memory, so the compiler cannot see their address space and would emit generic
// LD / ST for every access; the assumptions below turn them back into LDS / STS (measured: C2
// 137 k -> 194 k steps/s, dense-Hessian C2 13.5 k -> 17.5 k).
template <bool SH>
__device__ inline bool jacobi_eigh_impl(const Blk& k, RmWork& w, double* A, double* U, bool warm) {
  const int n = w.dim, ld = w.ld;
  double* const rc = w.rc;
  double* const rs = w.rs;
  int* const top = w.top;
  int* const bot = w.bot;
  __builtin_assume(__isShared(rc));
  __builtin_assume(__isShared(rs));
  __builtin_assume(__isShared(top));
  __builtin_assume(__isShared(bot));
  if (SH) {
    __builtin_assume(__isShared(A));
    __builtin_assume(__isShared(U));
  }
  const int m = (n + 1) / 2;  // pairs per round (odd n: one index idles each round)
  const int np = 2 * m;       // padded player count; index n (if odd) is a bye
  if (!warm)
    for (int idx = k.tid; idx < n * n; idx += k.nthr) {
      const int i = idx / n, j = idx - i * n;
      U[i * ld + j] = (i == j) ? 1.0 : 0.0;
    }
  // scale for the convergence test
  double dmax = 0.0;
  for (int idx = k.tid; idx < n * n; idx += k.nthr) {
    const int i = idx / n, j = idx - i * n;
    dmax = nanmax(dmax, fabs(A[i * ld + j]));
  }
  const double scale = block_nanmax(k, dmax);
  if (!(scale == scale) || isinf(scale)) return false;
  if (scale == 0.0) return true;
  const double tol = 1e-15 * scale;

  // thread grid for the update phases: tx indexes column pairs, ty strides over row pairs / rows
  // (no integer divisions in the inner loops; the round's pair table is written once to w.top /
  // w.bot by the parameter phase)
  const int tx = k.tid & 31, ty = k.tid >> 5, ny = k.nthr >> 5;
  // look-ahead votes: two banks of [nwarp] ints in the reduction scratch (k.red[16..32) is unused
  // by block_sum / block_nanmax), alternated per pass so that no extra barrier protects them
  int* flag_banks = reinterpret_cast<int*>(k.red + 16);
  __builtin_assume(__isShared(flag_banks));
  int pass = 0;
  for (int sweep = 0; sweep < RM_MAX_SWEEPS; ++sweep) {
    double off = 0.0;
    for (int round = 0; round < np - 1;) {
      // --- look-ahead: warp v examines round `round + v`.  Warp 0 also produces the rotation
      // parameters of the current round.  Rounds in which no pair needs a rotation (every pair
      // already decoupled: block-structured matrices, late sweeps) are skipped up to nwarp at a
      // time with a single barrier; a matrix that needs every rotation pays the same two
      // barriers per round as without the look-ahead.
      const int rr = round + k.warp;
      bool need = false;
      double off_w = 0.0;
      if (rr < np - 1) {
        for (int t = k.lane; t < m; t += 32) {
          int p, q;
          rr_pair(np, rr, t, p, q);
          double c = 1.0, s = 0.0;
          if (q < n) {
            const double apq = A[p * ld + q];
            off_w = fmax(off_w, fabs(apq));
            if (fabs(apq) > 1e-300 && fabs(apq) > 1e-18 * scale) {
              need = true;
              if (k.warp == 0) {
                // t = sign(tau) / (|tau| + sqrt(1 + tau^2)), tau = (aqq - app) / (2 apq), written
                // as t = sign * |b| / (|d| + sqrt(d^2 + b^2)) with d = aqq - app, b = 2 apq, and
                // c = 1 / sqrt(1 + t^2) through rsqrt + one Newton step: ONE division and two
                // rsqrt in the dependent chain instead of three divisions and two sqrt -- this
                // chain is the serial part of every round (all other warps wait for it).  How
                // well t annihilates a_pq only affects convergence; orthogonality needs
                // c^2 + s^2 = 1, which the Newton step restores to rounding.
                const double app = A[p * ld + p], aqq = A[q * ld + q];
                const double d = aqq - app, b2 = 2.0 * apq;
                const double w2 = fma(d, d, b2 * b2);
                double tt;
                if (w2 < 1e300 && w2 > 1e-300) {
                  const double h = w2 * rsqrt(w2);
                  tt = fabs(b2) / (fabs(d) + h);
                } else {  // out of range for the squared form: the textbook expression
                  const double tau = d / b2;
                  tt = 1.0 / (fabs(tau) + sqrt(1.0 + tau * tau));
                }
                if (d != 0.0 && (d < 0.0) != (b2 < 0.0)) tt = -tt;  // sign(tau); tau = 0 -> +1
                const double x = fma(tt, tt, 1.0);
                double r = rsqrt(x);
                r = r * fma(-0.5 * x, r * r, 1.5);
                c = r;
                s = tt * c;
              }
            }
          }
          if (k.warp == 0) {
            rc[t] = c;
            rs[t] = s;
            top[t] = p;
            bot[t] = q;
          }
        }
      }
      int* flags = flag_banks + (pass & 1) * 16;
      ++pass;
      const bool warp_need = __any_sync(FULL_MASK, need);
      if (k.lane == 0) flags[k.warp] = warp_need ? 1 : 0;
      __syncthreads();
      // first round of the batch that needs a rotation: one load per lane and a ballot (a
      // sequential scan of the flags was a chain of up to nwarp dependent shared-memory loads
      // per pass -- 15 % of the samples of the block-diagonal C2 case)
      const unsigned vote =
          __ballot_sync(FULL_MASK, k.lane < k.nwarp && flags[k.lane < k.nwarp ? k.lane : 0] != 0);
      const int first = vote != 0u ? __ffs(vote) - 1 : k.nwarp;
      if (k.warp <= first) off = fmax(off, off_w);  // rounds consumed now (skipped or rotated)
      if (first > 0) {  // rounds round .. round+first-1 need no rotation
        round += first;
        continue;
      }
      // --- A <- R^T A R on 2x2 blocks (pair a rows, pair b cols), U <- U R
      for (int b = tx; b < m; b += 32) {
        const int pb = top[b], qb = bot[b];
        const double cb = rc[b], sb = rs[b];
        const bool vb = qb < n;
        for (int a = ty; a < m; a += ny) {
          const double sa = rs[a];
          if (sa == 0.0 && sb == 0.0) continue;  // both rotations are the identity
          const int pa = top[a], qa = bot[a];
          const double ca = rc[a];
          const bool va = qa < n;
          if (va && vb) {
            const double a00 = A[pa * ld + pb], a01 = A[pa * ld + qb];
            const double a10 = A[qa * ld + pb], a11 = A[qa * ld + qb];
            // rows: (r0, r1) = (ca*x0 - sa*x1, sa*x0 + ca*x1)
            const double r00 = fma(ca, a00, -(sa * a10)), r01 = fma(ca, a01, -(sa * a11));
            const double r10 = fma(sa, a00, ca * a10), r11 = fma(sa, a01, ca * a11);
            // cols
            A[pa * ld + pb] = fma(cb, r00, -(sb * r01));
            A[pa * ld + qb] = fma(sb, r00, cb * r01);
            A[qa * ld + pb] = fma(cb, r10, -(sb * r11));
            A[qa * ld + qb] = fma(sb, r10, cb * r11);
          } else if (va && !vb) {  // single column pb (< n), rotated rows only
            const double a0 = A[pa * ld + pb], a1 = A[qa * ld + pb];
            A[pa * ld + pb] = fma(ca, a0, -(sa * a1));
            A[qa * ld + pb] = fma(sa, a0, ca * a1);
          } else if (!va && vb) {  // single row pa (< n), rotated cols only
            const double a0 = A[pa * ld + pb], a1 = A[pa * ld + qb];
            A[pa * ld + pb] = fma(cb, a0, -(sb * a1));
            A[pa * ld + qb] = fma(sb, a0, cb * a1);
          }
        }
        if (vb && sb != 0.0) {
          // four rows per pass: all loads before the stores (independent round trips)
          int i = ty;
          for (; i + 3 * ny < n; i += 4 * ny) {
            double u0[4], u1[4];
#pragma unroll
            for (int e = 0; e < 4; ++e)
              u0[e] = U[(i + e * ny) * ld + pb], u1[e] = U[(i + e * ny) * ld + qb];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              U[(i + e * ny) * ld + pb] = fma(cb, u0[e], -(sb * u1[e]));
              U[(i + e * ny) * ld + qb] = fma(sb, u0[e], cb * u1[e]);
            }
          }
          for (; i < n; i += ny) {
            const double u0 = U[i * ld + pb], u1 = U[i * ld + qb];
            U[i * ld + pb] = fma(cb, u0, -(sb * u1));
            U[i * ld + qb] = fma(sb, u0, cb * u1);
          }
        }
      }
      __syncthreads();
      ++round;
    }
    const double offmax = block_nanmax(k, off);
    if (!(offmax == offmax)) return false;
    if (offmax <= tol) return true;  // the sweep just done squares this again
  }
  return false;
}

__device__ inline bool jacobi_eigh(const Blk& k, RmWork& w, double* A, double* U, bool warm = false) {
  return __isShared(A) ? jacobi_eigh_impl<true>(k, w, A, U, warm)
                       : jacobi_eigh_impl<false>(k, w, A, U, warm);
}

// C = op(X) * Y for n x n shared-memory matrices (stride ld), op = transpose if XT.  4x4 register
// tiles, one per thread.  C must not alias X or Y.
__device__ __forceinline__ void rm_dmma(double& c0, double& c1, double a, double b) {
  asm volatile(
      "mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
      : "+d"(c0), "+d"(c1)
      : "d"(a), "d"(b));
}

// The same product on the FP64 tensor pipe (DMMA m8n8k4) for n a multiple of 32: one 16 x 32
// output tile per warp and pass, operands read from shared memory as fragments (A by rows, or by
// columns for X^T; B by rows).
template <bool XT>
__device__ inline void smem_matmul_dmma(const Blk& k, int n, int ld, const double* X,
                                        const double* Y, double* C) {
  const int r = k.lane >> 2, c = k.lane & 3;
  const int tr = n / 16, tc = n / 32;
  for (int t = k.warp; t < tr * tc; t += k.nwarp) {
    const int i0 = 16 * (t / tc), j0 = 32 * (t % tc);
    double acc[2][4][2];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) acc[mt][nt][0] = 0.0, acc[mt][nt][1] = 0.0;
#pragma unroll 4
    for (int ks = 0; ks < n / 4; ++ks) {
      double a[2], b[4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
        a[mt] = XT ? X[(4 * ks + c) * ld + i0 + 8 * mt + r] : X[(i0 + 8 * mt + r) * ld + 4 * ks + c];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) b[nt] = Y[(4 * ks + c) * ld + j0 + 8 * nt + r];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) rm_dmma(acc[mt][nt][0], acc[mt][nt][1], a[mt], b[nt]);
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        C[(i0 + 8 * mt + r) * ld + j0 + 8 * nt + 2 * c] = acc[mt][nt][0];
        C[(i0 + 8 * mt + r) * ld + j0 + 8 * nt + 2 * c + 1] = acc[mt][nt][1];
      }
  }
  __syncthreads();
}

template <bool XT>
__device__ inline void smem_matmul(const Blk& k, int n, int ld, const double* X, const double* Y,
                                   double* C) {
  if ((n & 31) == 0) {
    smem_matmul_dmma<XT>(k, n, ld, X, Y, C);
    return;
  }
  const int tn = (n + 3) / 4;
  for (int t = k.tid; t < tn * tn; t += k.nthr) {
    const int i0 = 4 * (t / tn), j0 = 4 * (t % tn);
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
    for (int kk = 0; kk < n; ++kk) {
      double x[4], y[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int i = i0 + a;
        x[a] = (i < n) ? (XT ? X[kk * ld + i] : X[i * ld + kk]) : 0.0;
        const int j = j0 + a;
        y[a] = (j < n) ? Y[kk * ld + j] : 0.0;
      }
      // exact: skipping a product with an all-zero operand adds nothing (operands are finite)
      if ((x[0] == 0.0 && x[1] == 0.0 && x[2] == 0.0 && x[3] == 0.0) ||
          (y[0] == 0.0 && y[1] == 0.0 && y[2] == 0.0 && y[3] == 0.0))
        continue;
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fma(x[a], y[b], acc[a][b]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b)
        if (i0 + a < n && j0 + b < n) C[(i0 + a) * ld + j0 + b] = acc[a][b];
  }
  __syncthreads();
}

#ifndef __CUDACC_RTC__  // library self-tests: kept out of the run-time compiled user images
// three matrices in shared memory: the eigenvectors, the matrix, and the warm start's product
__host__ __device__ inline RmLayout eigh_selftest_layout(int dim) {
  return RmLayout{dim, RM_MATRICES, 3, 0, true};
}

// Diagnostic kernel: K3 on arbitrary dense symmetric matrices (one CTA per matrix).  With
// `warm_from` >= 0 the solve of matrix i is warm-started from the eigenvectors of matrix
// `warm_from` (exercising the V^T H V path used between fixed-point iterates).
static __global__ void __launch_bounds__(RM_THREADS)
    eigh_selftest_kernel(const double* __restrict__ mats, int64_t n_mats, int dim, int warm_from,
                         double* __restrict__ eigval, double* __restrict__ eigvec,
                         int32_t* __restrict__ status) {
  extern __shared__ double smem[];
  Blk blk;
  blk.tid = threadIdx.x, blk.nthr = blockDim.x, blk.lane = threadIdx.x & 31;
  blk.warp = threadIdx.x >> 5, blk.nwarp = blockDim.x >> 5;
  RmWork w;
  double* tscratch;
  rm_carve(eigh_selftest_layout(dim), smem, nullptr, blk, w, &tscratch);
  const int ld = w.ld;
  for (int64_t mi = blockIdx.x; mi < n_mats; mi += gridDim.x) {
    __syncthreads();
    bool ok = true;
    bool warm = false;
    if (warm_from >= 0) {
      const double* src = mats + (size_t)warm_from * dim * dim;
      for (int idx = blk.tid; idx < dim * dim; idx += blk.nthr)
        w.M2[(idx / dim) * ld + idx % dim] = src[idx];
      __syncthreads();
      ok = jacobi_eigh(blk, w, w.M2, w.M1);
      warm = ok;
    }
    const double* src = mats + (size_t)mi * dim * dim;
    for (int idx = blk.tid; idx < dim * dim; idx += blk.nthr)
      w.M2[(idx / dim) * ld + idx % dim] = src[idx];
    __syncthreads();
    if (warm) {
      smem_matmul<false>(blk, dim, ld, w.M2, w.M1, w.M3);
      smem_matmul<true>(blk, dim, ld, w.M1, w.M3, w.M2);
      for (int idx = blk.tid; idx < dim * dim; idx += blk.nthr) {
        const int i = idx / dim, j = idx - i * dim;
        if (i < j) {
          const double v = 0.5 * (w.M2[i * ld + j] + w.M2[j * ld + i]);
          w.M2[i * ld + j] = v;
          w.M2[j * ld + i] = v;
        }
      }
      __syncthreads();
    }
    ok = jacobi_eigh(blk, w, w.M2, w.M1, warm);
    for (int idx = blk.tid; idx < dim * dim; idx += blk.nthr)
      eigvec[(size_t)mi * dim * dim + idx] = w.M1[(idx / dim) * ld + idx % dim];
    for (int i = blk.tid; i < dim; i += blk.nthr) eigval[mi * dim + i] = w.M2[i * ld + i];
    if (blk.tid == 0) status[mi] = ok ? 0 : MB200_STATUS_LINALG;
  }
}
#endif

// ---------------------------------------------------------------------------------------------
// K2: in-place lower Cholesky factor of the SPD matrix M [dim x dim, stride ld]
// (numpy.linalg.cholesky, matrices.py:1165-1169).  Returns false on a non-positive / non-finite
// pivot (-> LinAlgError "Cholesky factorisation failed", matrices.py:1170-1172).
// ---------------------------------------------------------------------------------------------
__device__ inline bool cholesky_inplace(const Blk& k, double* M, int n, int ld) {
  for (int j = 0; j < n; ++j) {
    __syncthreads();
    const double d = M[j * ld + j];
    const bool bad = !(d > 0.0) || isinf(d);
    if (bad) return false;  // uniform: every thread reads the same value
    const double l = sqrt(d);
    __syncthreads();
    for (int i = j + k.tid; i < n; i += k.nthr) M[i * ld + j] = (i == j) ? l : M[i * ld + j] / l;
    __syncthreads();
    // trailing update of the lower triangle: M[i][c] -= L[i][j] * L[c][j], j < c <= i
    const int rem = n - j - 1;
    for (int idx = k.tid; idx < rem * rem; idx += k.nthr) {
      const int i = j + 1 + idx / rem, c = j + 1 + idx % rem;
      if (c <= i) M[i * ld + c] -= M[i * ld + j] * M[c * ld + j];
    }
  }
  __syncthreads();
  return true;
}

// Forward / back substitution with a lower factor L (scipy solve_triangular, matrices.py:897-912).
// Column-oriented so that each elimination step is parallel over rows.  The two halves are also
// used on their own (the Cholesky-factored metric needs L^-1 b).
// x = L^-1 b (forward substitution); x may alias b
__device__ __forceinline__ void cholesky_forward(const Blk& k, const double* L, int n, int ld,
                                                 const double* b, double* x) {
  for (int i = k.tid; i < n; i += k.nthr) x[i] = b[i];
  __syncthreads();
  for (int j = 0; j < n; ++j) {  // L y = b
    if (k.tid == 0) x[j] /= L[j * ld + j];
    __syncthreads();
    const double xj = x[j];
    for (int i = j + 1 + k.tid; i < n; i += k.nthr) x[i] -= L[i * ld + j] * xj;
    __syncthreads();
  }
}
// x <- L^-T x in place (back substitution)
__device__ __forceinline__ void cholesky_back(const Blk& k, const double* L, int n, int ld,
                                              double* x) {
  for (int j = n - 1; j >= 0; --j) {  // L^T x = y
    if (k.tid == 0) x[j] /= L[j * ld + j];
    __syncthreads();
    const double xj = x[j];
    for (int i = k.tid; i < j; i += k.nthr) x[i] -= L[j * ld + i] * xj;
    __syncthreads();
  }
}
// x = (L L^T)^-1 b; x may alias b
__device__ inline void cholesky_solve(const Blk& k, const double* L, int n, int ld,
                                      const double* b, double* x) {
  cholesky_forward(k, L, n, ld, b, x);
  cholesky_back(k, L, n, ld, x);
}

// ---------------------------------------------------------------------------------------------
// Metric policies.  build(q) -> 0 ok, else status of the failure kind; methods mirror
// RiemannianMetricSystem's use of the matrix object (systems.py:1375-1402).
// ---------------------------------------------------------------------------------------------

// SoftAbs of the target Hessian (matrices.py:1631-1685)
template <class Target>
struct SoftAbsMetric {
  static constexpr bool SOFTABS = true;
  static constexpr RmPlace PLACE = RM_MATRICES;
  static constexpr int N_MATS = 2;
  // beyond shared memory: eigenvectors, work / divided-difference and warm-start matrices
  static constexpr int WORKSPACE_MATS = 3;
  // register budget: two CTAs per SM (<= 128 registers); stated explicitly because ptxas's own
  // choice flips with unrelated code changes (48 vs 80 registers measured 3.4x apart on C4)
  static constexpr int MIN_BLOCKS = 2;
  static constexpr int THREADS = RM_THREADS;
  const Target& t;
  double alpha;
  bool have_j;     // divided-difference matrix J built in w.M2 for the current metric?
  bool j_finite;   // ... and all of its entries are finite
  bool have_prev;  // w.M1 holds the eigenvectors of the previous build (warm start available)
  bool have_z;     // DENSE_MTP targets: Z = A U of the current metric is in w.M3

  __device__ SoftAbsMetric(const Target& tt, const ModelArgs& m)
      : t(tt), alpha(m.mp[0]), have_j(false), j_finite(false), have_prev(false), have_z(false) {}
  // forget the previous eigenvectors (start of every integrator step: bounds the loss of
  // orthogonality from accumulating rotations over many warm-started solves)
  __device__ void reset() { have_prev = false; }

  // returns 0, or MB200_STATUS_LINALG (eigh failure) / -1 (ValueError: non-positive eigenvalues)
  __device__ int build(const Blk& k, RmWork& w, const double* q) {
    have_j = false;
    have_z = false;  // w.M3 is the warm start's scratch during the build
    t.hess(k, q, w.M2, w.ld);
    __syncthreads();
    // Warm start: successive fixed-point iterates move q only slightly, so the previous
    // eigenvectors V almost diagonalise the new Hessian: iterate on V^T H V (2 products of
    // D^3 flop) and accumulate the rotations onto V -- 3-4 sweeps instead of 8-9.
    const bool warm = have_prev && w.M3 != nullptr;
    if (warm) {
      smem_matmul<false>(k, w.dim, w.ld, w.M2, w.M1, w.M3);  // T = H V
      smem_matmul<true>(k, w.dim, w.ld, w.M1, w.M3, w.M2);   // A = V^T T
      // symmetrise (the two products round differently above and below the diagonal)
      for (int idx = k.tid; idx < w.dim * w.dim; idx += k.nthr) {
        const int i = idx / w.dim, j = idx - i * w.dim;
        if (i < j) {
          const double v = 0.5 * (w.M2[i * w.ld + j] + w.M2[j * w.ld + i]);
          w.M2[i * w.ld + j] = v;
          w.M2[j * w.ld + i] = v;
        }
      }
      __syncthreads();
    }
    have_prev = false;
    if (!jacobi_eigh(k, w, w.M2, w.M1, warm)) return MB200_STATUS_LINALG;
    have_prev = true;
    bool bad = false;
    for (int i = k.tid; i < w.dim; i += k.nthr) {
      const double x = w.M2[i * w.ld + i];
      const double ax = alpha * x;
      const double s = x / tanh(x * alpha);                            // :1662-1664
      const double sh = sinh(ax);
      w.lam[i] = x;
      w.sa[i] = s;
      w.gsa[i] = 1.0 / tanh(ax) - ax / (sh * sh);                      // :1666-1671
      if (!(s > 0.0)) bad = true;  // EigendecomposedPositiveDefiniteMatrix: ValueError (:1606-1609)
    }
    if (block_any(k, bad)) return -1;
    return 0;
  }
  __device__ double log_abs_det(const Blk& k, RmWork& w) const {
    double s = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) s += log(fabs(w.sa[i]));
    return block_sum(k, s);
  }
  // out = M^-1 v = U ((U^T v) / s)   (matrices.py:1555-1556 with 1/eigval); out must not alias v
  __device__ void inv_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    const int n = w.dim, ld = w.ld;
    for (int j = k.tid; j < n; j += k.nthr) {
      double s = 0.0;
      for (int i = 0; i < n; ++i) s = fma(w.M1[i * ld + j], v[i], s);
      w.ev[j] = s / w.sa[j];
    }
    __syncthreads();
    for (int i = k.tid; i < n; i += k.nthr) {
      double s = 0.0;
      for (int j = 0; j < n; ++j) s = fma(w.M1[i * ld + j], w.ev[j], s);
      out[i] = s;
    }
    __syncthreads();
  }
  // out = sqrt(M) v = U (sqrt(s) o (U^T v))   (EigendecomposedPositiveDefiniteMatrix.sqrt,
  // matrices.py:1618-1628); out must not alias v
  __device__ bool sqrt_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    const int n = w.dim, ld = w.ld;
    for (int j = k.tid; j < n; j += k.nthr) {
      double s = 0.0;
      for (int i = 0; i < n; ++i) s = fma(w.M1[i * ld + j], v[i], s);
      w.ev[j] = sqrt(w.sa[j]) * s;
    }
    __syncthreads();
    for (int i = k.tid; i < n; i += k.nthr) {
      double s = 0.0;
      for (int j = 0; j < n; ++j) s = fma(w.M1[i * ld + j], w.ev[j], s);
      out[i] = s;
    }
    __syncthreads();
    return true;
  }
  // out = vjp(grad_log_abs_det), grad_log_abs_det = U diag(gs/s) U^T   (:1673-1676)
  __device__ void vjp_grad_log_abs_det(const Blk& k, RmWork& w, const double* q, double* out) {
    const int n = w.dim, ld = w.ld;
    if constexpr (Target::DENSE_MTP) {
      if (!have_z) {
        t.eigen_directions(k, w.M1, ld, w.M3);
        have_z = true;
      }
      for (int i = k.tid; i < n; i += k.nthr) w.ev[i] = w.gsa[i] / w.sa[i];
      __syncthreads();
      t.mtp_diag(k, q, w.M3, ld, w.ev, w.Vn + (size_t)k.nwarp * n, out);
      return;
    }
    for (int idx = k.tid; idx < n * Target::NEED; idx += k.nthr) {
      const int a = idx / Target::NEED, j = idx - a * Target::NEED;
      const int b = t.need_col(a, j);
      double s = 0.0;
      if (b >= 0)
        for (int i = 0; i < n; ++i)
          s = fma(w.M1[a * ld + i] * (w.gsa[i] / w.sa[i]), w.M1[b * ld + i], s);
      w.Vn[idx] = s;
    }
    __syncthreads();
    t.mtp_entries(k, q, w.Vn, out);
    __syncthreads();
  }
  // out = vjp(grad_quadratic_form_inv(p)) = vjp(-U ((e e^T) o J) U^T), e = U^T p / s  (:1678-1685)
  __device__ void vjp_grad_quad_inv(const Blk& k, RmWork& w, const double* q, const double* p,
                                    double* out) {
    const int n = w.dim, ld = w.ld;
    if (!have_j) {  // J depends on the metric only: build once per metric, reuse per iteration
      bool bad = false;
      for (int idx = k.tid; idx < n * n; idx += k.nthr) {
        const int i = idx / n, j = idx - i * n;
        const double v = (i == j) ? w.gsa[i] : (w.sa[i] - w.sa[j]) / (w.lam[i] - w.lam[j]);
        if (!isfinite(v)) bad = true;
        w.M2[i * ld + j] = v;
      }
      j_finite = !block_any(k, bad);  // (0 * inf must stay NaN: only skip zeros if J is finite)
      have_j = true;
    }
    for (int j = k.tid; j < n; j += k.nthr) {
      double s = 0.0;
      for (int i = 0; i < n; ++i) s = fma(w.M1[i * ld + j], p[i], s);
      w.ev[j] = s / w.sa[j];
    }
    __syncthreads();
    if constexpr (Target::DENSE_MTP) {
      if (!have_z) {
        t.eigen_directions(k, w.M1, ld, w.M3);
        have_z = true;
      }
      // per-warp staging rows and the per-direction results live in Vn (2 dpad doubles) and the
      // z buffers that follow it (unused by the leapfrog integrator): (nwarp + 1) dim <= 12 dpad
      t.mtp_quad(k, q, w.M3, ld, w.ev, w.M2, ld, w.Vn, w.Vn + (size_t)k.nwarp * n, out);
      return;
    }
    // V = -U G U^T with G = diag(e) J diag(e).  When a third matrix is available and one pass of
    // 16 x 32 DMMA tiles covers the product (D = 32, 64 with 8 warps), P = U G runs on the tensor
    // pipe (this contraction was 30 % of the C2 step as scalar code) and only the NEED entries
    // per row of V = -P U^T are formed.
    if (w.M3 != nullptr && (n & 31) == 0 && (n / 16) * (n / 32) <= k.nwarp) {
      for (int idx = k.tid; idx < n * n; idx += k.nthr) {
        const int i = idx / n, j = idx - i * n;
        w.M3[i * ld + j] = (w.ev[i] * w.M2[i * ld + j]) * w.ev[j];
      }
      __syncthreads();
      {
        const int r = k.lane >> 2, c = k.lane & 3;
        const int tc = n / 32, tile = k.warp;
        const bool active = tile < (n / 16) * tc;
        const int i0 = 16 * (tile / tc), j0 = 32 * (tile % tc);
        double acc[2][4][2];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) acc[mt][nt][0] = 0.0, acc[mt][nt][1] = 0.0;
        if (active) {
#pragma unroll 4
          for (int ks = 0; ks < n / 4; ++ks) {
            double a[2], b[4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) a[mt] = w.M1[(i0 + 8 * mt + r) * ld + 4 * ks + c];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) b[nt] = w.M3[(4 * ks + c) * ld + j0 + 8 * nt + r];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int nt = 0; nt < 4; ++nt) rm_dmma(acc[mt][nt][0], acc[mt][nt][1], a[mt], b[nt]);
          }
        }
        __syncthreads();  // every warp has read G: P may overwrite it
        if (active) {
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
              w.M3[(i0 + 8 * mt + r) * ld + j0 + 8 * nt + 2 * c] = acc[mt][nt][0];
              w.M3[(i0 + 8 * mt + r) * ld + j0 + 8 * nt + 2 * c + 1] = acc[mt][nt][1];
            }
        }
        __syncthreads();
      }
      for (int idx = k.warp; idx < n * Target::NEED; idx += k.nwarp) {
        const int a = idx / Target::NEED, jn = idx - a * Target::NEED;
        const int b = t.need_col(a, jn);
        double sacc = 0.0;
        if (b >= 0)
          for (int j = k.lane; j < n; j += 32) sacc = fma(w.M3[a * ld + j], w.M1[b * ld + j], sacc);
        sacc = warp_sum(sacc);
        if (k.lane == 0) w.Vn[idx] = -sacc;
      }
      __syncthreads();
      t.mtp_entries(k, q, w.Vn, out);
      __syncthreads();
      return;
    }
    // one warp per row a: t_j = sum_i (U_ai e_i) J_ij, then V(a,b) = -sum_j t_j e_j U_bj
    double* trow = w.v3;  // reused per warp below via registers; v3 holds (U_a o e) of the row
    (void)trow;
    for (int a = k.warp; a < n; a += k.nwarp) {
      double acc[Target::NEED];
#pragma unroll
      for (int jn = 0; jn < Target::NEED; ++jn) acc[jn] = 0.0;
      for (int j = k.lane; j < n; j += 32) {
        double tj = 0.0;
        for (int i = 0; i < n; ++i) {
          const double ue = w.M1[a * ld + i] * w.ev[i];  // warp-uniform
          if (ue == 0.0 && j_finite) continue;            // exact zero term (sparse eigenvectors)
          tj = fma(ue, w.M2[i * ld + j], tj);
        }
        tj *= w.ev[j];
#pragma unroll
        for (int jn = 0; jn < Target::NEED; ++jn) {
          const int b = t.need_col(a, jn);
          if (b >= 0) acc[jn] = fma(tj, w.M1[b * ld + j], acc[jn]);
        }
      }
#pragma unroll
      for (int jn = 0; jn < Target::NEED; ++jn) {
        const double s = warp_sum(acc[jn]);
        if (k.lane == 0) w.Vn[a * Target::NEED + jn] = -s;
      }
    }
    __syncthreads();
    t.mtp_entries(k, q, w.Vn, out);
    __syncthreads();
  }
};

// Dense metric M(q) = B + c q q^T (DenseRiemannianMetricSystem, systems.py:1710-1760) with
// DensePositiveDefiniteMatrix arithmetic (matrices.py:1161-1188).  The two gradient matrices are
// never formed: vjp(V) = c (V + V^T) q needs only V q, i.e. M^-1 q for grad_log_abs_det = M^-1
// (:1175-1177) and -w (w.q) for grad_quadratic_form_inv = -w w^T, w = M^-1 p (:1179-1181).
template <class Target>
struct Rank1DenseMetric {
  static constexpr bool SOFTABS = false;
  static constexpr RmPlace PLACE = RM_MATRICES;
  static constexpr int N_MATS = 1;
  static constexpr int WORKSPACE_MATS = 0;
  static constexpr int MIN_BLOCKS = 2;
  static constexpr int THREADS = RM_THREADS;
  const Target& t;
  const double* B;
  double c;
  __device__ Rank1DenseMetric(const Target& tt, const ModelArgs& m) : t(tt), B(m.maux), c(m.mp[0]) {}
  __device__ void reset() {}

  __device__ int build(const Blk& k, RmWork& w, const double* q) {
    const int n = w.dim, ld = w.ld;
    bool bad = false;
    for (int idx = k.tid; idx < n * n; idx += k.nthr) {
      const int i = idx / n, j = idx - i * n;
      const double v = B[idx] + c * (q[i] * q[j]);
      if (!isfinite(v)) bad = true;
      w.M1[i * ld + j] = v;
    }
    if (block_any(k, bad)) return MB200_STATUS_LINALG;  // "Array is not finite" (:211-215)
    if (!cholesky_inplace(k, w.M1, n, ld)) return MB200_STATUS_LINALG;
    return 0;
  }
  __device__ double log_abs_det(const Blk& k, RmWork& w) const {
    double s = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) s += log(fabs(w.M1[i * w.ld + i]));
    return 2.0 * block_sum(k, s);  // matrices.py:982-984
  }
  __device__ void inv_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    cholesky_solve(k, w.M1, w.dim, w.ld, v, out);
  }
  // out = L v (sqrt of a DensePositiveDefiniteMatrix is its Cholesky factor, matrices.py:1212-1216)
  __device__ bool sqrt_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    for (int i = k.tid; i < w.dim; i += k.nthr) {
      double s = 0.0;
      for (int j = 0; j <= i; ++j) s = fma(w.M1[i * w.ld + j], v[j], s);
      out[i] = s;
    }
    __syncthreads();
    return true;
  }
  __device__ void vjp_grad_log_abs_det(const Blk& k, RmWork& w, const double* q, double* out) const {
    cholesky_solve(k, w.M1, w.dim, w.ld, q, w.ev);  // M^-1 q
    for (int i = k.tid; i < w.dim; i += k.nthr) out[i] = c * (w.ev[i] + w.ev[i]);
    __syncthreads();
  }
  __device__ void vjp_grad_quad_inv(const Blk& k, RmWork& w, const double* q, const double* p,
                                    double* out) {
    cholesky_solve(k, w.M1, w.dim, w.ld, p, w.ev);  // w = M^-1 p
    double s = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) s = fma(w.ev[i], q[i], s);
    const double wq = block_sum(k, s);
    // V q = -(w w^T) q = -w (w.q);  c (V + V^T) q = 2 c V q
    for (int i = k.tid; i < w.dim; i += k.nthr) {
      const double vq = -(w.ev[i] * wq);
      out[i] = c * (vq + vq);
    }
    __syncthreads();
  }
};

// The same metric M(q) = B + c q q^T for dimensions whose D x D factor does not fit in shared
// memory (config C4, D = 512): the matrix is never formed.  With the shared explicit inverse
// B^-1 (built on the host exactly like a fixed dense metric, matrices.py:1183-1188) and
// u = B^-1 q, the matrix-determinant and Sherman-Morrison identities give
//   log|M|  = log|B| + log(1 + c q.u)
//   M^-1 v  = B^-1 v - u (c (u.v) / (1 + c q.u))
//   M^-1 q  = u / (1 + c q.u)
// -- O(D^2) per metric instead of the reference's O(D^3) Cholesky (matrices.py:1161-1173);
// equal to it up to rounding (checked against the D = 512 reference fixture).
template <class Target>
struct Rank1WoodburyMetric {
  static constexpr bool SOFTABS = false;
  static constexpr RmPlace PLACE = RM_MATRICES;
  static constexpr int N_MATS = 0;
  static constexpr int WORKSPACE_MATS = 0;
  static constexpr int MIN_BLOCKS = 2;
  static constexpr int THREADS = RM_THREADS;
  const Target& t;
  const double* Binv;
  double c, logdet_b, denom;
  __device__ Rank1WoodburyMetric(const Target& tt, const ModelArgs& m)
      : t(tt), Binv(m.maux + (size_t)tt.dim * tt.dim), c(m.mp[0]), logdet_b(m.mp[1]), denom(1.0) {}
  __device__ void reset() {}

  // out = B^-1 v (B^-1 symmetric: column-wise reads are coalesced across threads)
  __device__ void binv_matvec(const Blk& k, int n, const double* v, double* out) const {
    for (int i = k.tid; i < n; i += k.nthr) {
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      int j = 0;
      for (; j + 3 < n; j += 4) {
        s0 = fma(Binv[(size_t)j * n + i], v[j], s0);
        s1 = fma(Binv[(size_t)(j + 1) * n + i], v[j + 1], s1);
        s2 = fma(Binv[(size_t)(j + 2) * n + i], v[j + 2], s2);
        s3 = fma(Binv[(size_t)(j + 3) * n + i], v[j + 3], s3);
      }
      for (; j < n; ++j) s0 = fma(Binv[(size_t)j * n + i], v[j], s0);
      out[i] = (s0 + s1) + (s2 + s3);
    }
    __syncthreads();
  }
  // u = B^-1 q kept in w.lam (unused by dense metrics)
  __device__ int build(const Blk& k, RmWork& w, const double* q) {
    binv_matvec(k, w.dim, q, w.lam);
    double s = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) s = fma(q[i], w.lam[i], s);
    denom = 1.0 + c * block_sum(k, s);
    if (!(denom > 0.0) || isinf(denom)) return MB200_STATUS_LINALG;  // M not SPD / not finite
    return 0;
  }
  __device__ double log_abs_det(const Blk&, RmWork&) const { return logdet_b + log(denom); }
  // the Cholesky factor of M(q) is not available in this form
  __device__ bool sqrt_matvec(const Blk&, RmWork&, const double*, double*) const { return false; }
  __device__ void inv_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    binv_matvec(k, w.dim, v, out);
    double s = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) s = fma(w.lam[i], v[i], s);
    const double f = c * block_sum(k, s) / denom;
    for (int i = k.tid; i < w.dim; i += k.nthr) out[i] -= w.lam[i] * f;
    __syncthreads();
  }
  __device__ void vjp_grad_log_abs_det(const Blk& k, RmWork& w, const double*, double* out) const {
    for (int i = k.tid; i < w.dim; i += k.nthr) {
      const double mq = w.lam[i] / denom;  // (M^-1 q)_i
      out[i] = c * (mq + mq);
    }
    __syncthreads();
  }
  __device__ void vjp_grad_quad_inv(const Blk& k, RmWork& w, const double* q, const double* p,
                                    double* out) {
    inv_matvec(k, w, p, w.ev);  // w = M^-1 p
    double s = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) s = fma(w.ev[i], q[i], s);
    const double wq = block_sum(k, s);
    for (int i = k.tid; i < w.dim; i += k.nthr) {
      const double vq = -(w.ev[i] * wq);
      out[i] = c * (vq + vq);
    }
    __syncthreads();
  }
};

// ---------------------------------------------------------------------------------------------
// O(D) metrics: DiagonalRiemannianMetricSystem (PositiveDiagonalMatrix, matrices.py:709-792) and
// ScalarRiemannianMetricSystem (PositiveScaledIdentityMatrix, matrices.py:595-706).  Every
// expression below is the NumPy expression of the reference matrix class, in its order of
// operations (1 / d is formed first and then multiplied, never p / d).  These policies use the
// compact vector set and a small CTA: the per-chain work per metric is a few passes over D
// elements, so a 256-thread CTA would leave most lanes idle at the D of the hierarchical models.
// ---------------------------------------------------------------------------------------------
#ifndef MB200_RM_COMPACT_THREADS
#define MB200_RM_COMPACT_THREADS 32  // measured against 64 and 128 on C7 (DESIGN.md, K9)
#endif
constexpr int RM_COMPACT_THREADS = MB200_RM_COMPACT_THREADS;
constexpr int RM_COMPACT_MIN_BLOCKS = 65536 / 128 / RM_COMPACT_THREADS;  // <= 128 registers

// diagonal models d(q) and their VJPs w -> sum_i w_i dd_i/dq
// MB200_RMETRIC_DIAG_QUADRATIC: d_i = a + b q_i^2, vjp(w)_i = 2 b w_i q_i
struct QuadraticDiagModel {
  double a, b;
  int dim;
  __device__ QuadraticDiagModel(const ModelArgs& m, int d) : a(m.mp[0]), b(m.mp[1]), dim(d) {}
  __device__ void diag(const Blk& k, const double* q, double* d) const {
    for (int i = k.tid; i < dim; i += k.nthr) d[i] = a + b * (q[i] * q[i]);
  }
  __device__ void vjp(const Blk& k, const double* q, const double* wv, double* out) const {
    for (int i = k.tid; i < dim; i += k.nthr) out[i] = 2.0 * b * wv[i] * q[i];
  }
};

// MB200_RMETRIC_DIAG_FUNNEL_FISHER: expected Fisher information of the funnel,
// d = [1/9 + (D-1)/2, e^-v, ..., e^-v];  vjp(w) = [-e^-v sum_{i>=1} w_i, 0, ..., 0]
struct FunnelFisherDiagModel {
  int dim;
  __device__ FunnelFisherDiagModel(const ModelArgs&, int d) : dim(d) {}
  __device__ void diag(const Blk& k, const double* q, double* d) const {
    const double e = exp(-q[0]);
    const double d0 = 1.0 / 9.0 + 0.5 * (dim - 1);
    for (int i = k.tid; i < dim; i += k.nthr) d[i] = (i == 0) ? d0 : e;
  }
  __device__ void vjp(const Blk& k, const double* q, const double* wv, double* out) const {
    double s = 0.0;
    for (int i = 1 + k.tid; i < dim; i += k.nthr) s += wv[i];
    s = block_sum(k, s);
    const double e = exp(-q[0]);
    for (int i = k.tid; i < dim; i += k.nthr) out[i] = (i == 0) ? -e * s : 0.0;
  }
};

template <class Target, class Model>
struct DiagonalMetric {
  static constexpr bool SOFTABS = false;
  static constexpr RmPlace PLACE = RM_COMPACT;
  static constexpr int N_MATS = 0;
  static constexpr int WORKSPACE_MATS = 0;
  static constexpr int MIN_BLOCKS = RM_COMPACT_MIN_BLOCKS;
  static constexpr int THREADS = RM_COMPACT_THREADS;
  const Target& t;
  Model model;
  __device__ DiagonalMetric(const Target& tt, const ModelArgs& m) : t(tt), model(m, tt.dim) {}
  __device__ void reset() {}

  // d in w.lam, 1 / d in w.sa; LinAlgError status unless every d_i > 0 (NaN fails), the check
  // of PositiveDiagonalMatrix (matrices.py:778-780)
  __device__ int build(const Blk& k, RmWork& w, const double* q) {
    model.diag(k, q, w.lam);
    bool bad = false;
    for (int i = k.tid; i < w.dim; i += k.nthr) {
      const double d = w.lam[i];
      w.sa[i] = 1.0 / d;
      if (!(d > 0.0)) bad = true;
    }
    return block_any(k, bad) ? MB200_STATUS_LINALG : 0;
  }
  // sum(log |d|)  (SymmetricMatrix.log_abs_det, matrices.py:458-459)
  __device__ double log_abs_det(const Blk& k, RmWork& w) const {
    double s = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) s += log(fabs(w.lam[i]));
    return block_sum(k, s);
  }
  // (1 / d) * v
  __device__ void inv_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    for (int i = k.tid; i < w.dim; i += k.nthr) out[i] = w.sa[i] * v[i];
    __syncthreads();
  }
  // d ** 0.5 * v
  __device__ bool sqrt_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    for (int i = k.tid; i < w.dim; i += k.nthr) out[i] = sqrt(w.lam[i]) * v[i];
    __syncthreads();
    return true;
  }
  // vjp(grad_log_abs_det) with grad_log_abs_det = 1.0 / d  (matrices.py:758-759)
  __device__ void vjp_grad_log_abs_det(const Blk& k, RmWork& w, const double* q, double* out) {
    model.vjp(k, q, w.sa, out);
    __syncthreads();
  }
  // vjp(grad_quadratic_form_inv(p)) with grad_quadratic_form_inv(p) = -((1 / d) * p) ** 2
  // (matrices.py:761-762)
  __device__ void vjp_grad_quad_inv(const Blk& k, RmWork& w, const double* q, const double* p,
                                    double* out) {
    for (int i = k.tid; i < w.dim; i += k.nthr) {
      const double x = w.sa[i] * p[i];
      w.ev[i] = -(x * x);
    }
    __syncthreads();  // a model VJP may read entries other threads wrote (funnel: sum over i >= 1)
    model.vjp(k, q, w.ev, out);
    __syncthreads();
  }
};

template <class Target>
using QuadraticDiagonalMetric = DiagonalMetric<Target, QuadraticDiagModel>;
template <class Target>
using FunnelFisherMetric = DiagonalMetric<Target, FunnelFisherDiagModel>;

// scalar models s(q) and their VJPs w -> w ds/dq (w a block-uniform scalar), over dim entries
// MB200_RMETRIC_SCALAR_QUADRATIC: s = a + b |q|^2, vjp(w)_i = 2 b w q_i
struct QuadraticScalarModel {
  double a, b;
  __device__ QuadraticScalarModel(const ModelArgs& m, int) : a(m.mp[0]), b(m.mp[1]) {}
  __device__ double scalar(const Blk& k, int dim, const double* q) const {
    double acc = 0.0;
    for (int i = k.tid; i < dim; i += k.nthr) acc = fma(q[i], q[i], acc);
    return a + b * block_sum(k, acc);
  }
  __device__ void vjp(const Blk& k, int dim, const double* q, double g, double* out) const {
    for (int i = k.tid; i < dim; i += k.nthr) out[i] = 2.0 * b * g * q[i];
  }
};

// M(q) = s(q) I.  The scalar and its reciprocal are block-uniform registers.
template <class Target, class Model>
struct ScalarMetric {
  static constexpr bool SOFTABS = false;
  static constexpr RmPlace PLACE = RM_COMPACT;
  static constexpr int N_MATS = 0;
  static constexpr int WORKSPACE_MATS = 0;
  static constexpr int MIN_BLOCKS = RM_COMPACT_MIN_BLOCKS;
  static constexpr int THREADS = RM_COMPACT_THREADS;
  const Target& t;
  Model model;
  double s, inv_s;
  __device__ ScalarMetric(const Target& tt, const ModelArgs& m)
      : t(tt), model(m, tt.dim), s(1.0), inv_s(1.0) {}
  __device__ void reset() {}

  // LinAlgError status unless s > 0 (NaN fails): PositiveScaledIdentityMatrix (matrices.py:692-694)
  __device__ int build(const Blk& k, RmWork& w, const double* q) {
    s = model.scalar(k, w.dim, q);
    inv_s = 1.0 / s;
    return (s > 0.0) ? 0 : MB200_STATUS_LINALG;
  }
  // D * log(|s|)  (matrices.py:659-667)
  __device__ double log_abs_det(const Blk&, RmWork& w) const { return w.dim * log(fabs(s)); }
  // (1 / s) * v
  __device__ void inv_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    for (int i = k.tid; i < w.dim; i += k.nthr) out[i] = inv_s * v[i];
    __syncthreads();
  }
  // s ** 0.5 * v
  __device__ bool sqrt_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    const double r = sqrt(s);
    for (int i = k.tid; i < w.dim; i += k.nthr) out[i] = r * v[i];
    __syncthreads();
    return true;
  }
  // vjp(D / s)  (grad_log_abs_det, matrices.py:669-670)
  __device__ void vjp_grad_log_abs_det(const Blk& k, RmWork& w, const double* q, double* out) {
    const double g = w.dim / s;
    model.vjp(k, w.dim, q, g, out);
    __syncthreads();
  }
  // vjp(-sum(p ** 2) / s ** 2)  (grad_quadratic_form_inv, matrices.py:672-673)
  __device__ void vjp_grad_quad_inv(const Blk& k, RmWork& w, const double* q, const double* p,
                                    double* out) {
    double acc = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) acc = fma(p[i], p[i], acc);
    const double g = -block_sum(k, acc) / (s * s);
    model.vjp(k, w.dim, q, g, out);
    __syncthreads();
  }
};

template <class Target>
using QuadraticScalarMetric = ScalarMetric<Target, QuadraticScalarModel>;

// What the host's launch plan (rm_launch) reads of a user image's target (UserRTarget of
// user_riemannian.cuh derives from it); the image's policies are the registry's, over user models
struct UserRTargetTraits {
  static constexpr bool DENSE_MTP = false;
};

// ---------------------------------------------------------------------------------------------
// K10: CholeskyFactoredRiemannianMetricSystem (systems.py:1574-1653): the metric is given by its
// lower-triangular factor L(q), M = L L^T, with TriangularFactoredPositiveDefiniteMatrix
// arithmetic (matrices.py:795-1114): no factorisation, O(D^2) per metric.
// ---------------------------------------------------------------------------------------------
#ifndef MB200_RM_CHOL_THREADS
#define MB200_RM_CHOL_THREADS 256  // measured against 64 and 128 on C8 (DESIGN.md, K10)
#endif

// Inclusive prefix sums P_k = sum_{j<=k} b_j q_j and inclusive suffix sums S_k = sum_{i>=k} a_i q_i
// over the CTA, a tile of nthr elements at a time (warp shuffles, warp totals in k.red[0..8) and
// k.red[16..24): at most 256 threads).  P and S must not alias a, b or q.
__device__ inline void block_prefix_suffix(const Blk& k, int n, const double* a, const double* b,
                                           const double* q, double* P, double* S) {
  double carry_p = 0.0, carry_s = 0.0;
  for (int base = 0; base < n; base += k.nthr) {
    const int i = base + k.tid;  // prefix element of this thread
    const int r = n - 1 - i;     // suffix element of this thread (descending)
    double x = i < n ? b[i] * q[i] : 0.0;
    double y = i < n ? a[r] * q[r] : 0.0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double xo = __shfl_up_sync(FULL_MASK, x, o), yo = __shfl_up_sync(FULL_MASK, y, o);
      if (k.lane >= o) x += xo, y += yo;
    }
    __syncthreads();  // the previous tile's (or a block reduction's) readers of k.red are done
    if (k.lane == 31) k.red[k.warp] = x, k.red[16 + k.warp] = y;
    __syncthreads();
    double px = carry_p, py = carry_s;
    for (int v = 0; v < k.warp; ++v) px += k.red[v], py += k.red[16 + v];
    if (i < n) P[i] = px + x, S[r] = py + y;
    for (int v = 0; v < k.nwarp; ++v) carry_p += k.red[v], carry_s += k.red[16 + v];
  }
  __syncthreads();
}

// MB200_RMETRIC_CHOL_QUADRATIC: L(q) = L0 + c tril(q q^T), L0 = aux [D x D] row-major lower
// triangular (the host zeroes its upper triangle; it is never read here).  VJPs of the two
// structured lower-triangular arguments the policy produces, sum_ij V_ij dL_ij/dq_k with
// dL_ij/dq_k = c (delta_ik q_j + q_i delta_jk), j <= i -- V is never formed:
//   V = diag(d)          ->  c (d_k q_k + d_k q_k)
//   V = tril(s a b^T)    ->  c s (a_k sum_{j<=k} b_j q_j + b_k sum_{i>=k} a_i q_i)
struct QuadraticCholModel {
  const double* L0;
  double c;
  int dim;
  __device__ QuadraticCholModel(const ModelArgs& m, int d) : L0(m.maux), c(m.mp[0]), dim(d) {}
  // lower triangle of L(q) into L (stride ld); true iff every entry written is finite
  __device__ bool fill(const Blk& k, const double* q, double* L, int ld) const {
    bool bad = false;
    for (int idx = k.tid; idx < dim * dim; idx += k.nthr) {
      const int i = idx / dim, j = idx - i * dim;
      if (j > i) continue;
      const double v = L0[idx] + c * (q[i] * q[j]);
      if (!isfinite(v)) bad = true;
      L[i * ld + j] = v;
    }
    return !bad;
  }
  __device__ void vjp_diag(const Blk& k, const double* q, const double* d, double* out) const {
    for (int i = k.tid; i < dim; i += k.nthr) {
      const double x = d[i] * q[i];
      out[i] = c * (x + x);
    }
  }
  // P, S: [dim] shared scratch for the scans
  __device__ void vjp_outer(const Blk& k, const double* q, double s, const double* a,
                            const double* b, double* P, double* S, double* out) const {
    block_prefix_suffix(k, dim, a, b, q, P, S);
    for (int i = k.tid; i < dim; i += k.nthr)
      out[i] = c * (s * (a[i] * P[i] + b[i] * S[i]));
  }
};

// true for Cholesky models that differentiate a lower-triangular V itself (`static constexpr bool
// DENSE_VJP = true` and vjp_tril(k, q, V, ld, out): out[k] = sum_{j<=i} V_ij dL_ij/dq_k, the
// user models of user_riemannian.cuh); the policy then forms V in a second per-chain matrix, w.M2.
// The registry model declares nothing and takes the structured VJPs vjp_diag / vjp_outer.
template <class M, class = void>
struct chol_dense_vjp {
  static constexpr bool value = false;
};
template <class M>
struct chol_dense_vjp<M, decltype(void(M::DENSE_VJP))> {
  static constexpr bool value = M::DENSE_VJP;
};

// TriangularFactoredPositiveDefiniteMatrix(L, factor_is_lower=True):
//   log|M| = 2 sum log|L_ii|                          (matrices.py:982-984, 850-852)
//   M^-1 v = L^-T (L^-1 v), no inverse formed          (:1110-1111, 897-912)
//   sqrt(M) z = L z                                     (:1113-1114)
//   grad_log_abs_det = diag(2 / diag L)                 (:1048-1050)
//   grad_quadratic_form_inv(p) = tril(-2 (M^-1 p)(L^-1 p)^T)   (:1052-1058)
// build() fails (LinAlgError status) only for a non-finite entry of the lower triangle
// (ExplicitArrayMatrix, :207-215); a zero or negative diagonal entry is accepted, as by the
// reference: a zero pivot surfaces through IEEE arithmetic in the solves (-> ConvergenceError
// inside a fixed-point solve) and through singular() in the velocity and energy evaluations.
// A DENSE_VJP model (chol_dense_vjp) gets the two gradients as lower-triangular matrices V in w.M2
// (its strict upper triangle is never written), one vjp_tril call each, as the reference's
// vjp_metric_chol_func(q)(V) does.
template <class Target, class Model>
struct CholeskyFactoredMetric {
  static constexpr bool SOFTABS = false;
  static constexpr bool CAN_BE_SINGULAR = true;
  static constexpr RmPlace PLACE = RM_MATRICES;
  // the factor [dim x (dim + 1)], and V for a DENSE_VJP model; in the per-CTA global workspace
  // beyond D ~ 150 (one matrix) or D ~ 113 (two)
  static constexpr int N_MATS = chol_dense_vjp<Model>::value ? 2 : 1;
  static constexpr int WORKSPACE_MATS = N_MATS;
  static constexpr int THREADS = MB200_RM_CHOL_THREADS;
  // <= 128 registers; a DENSE_VJP model: up to 255, since the user functions and the target's
  // parameters would not fit beside the policy's state without spilling
  static constexpr int MIN_BLOCKS = chol_dense_vjp<Model>::value ? 1 : 65536 / 128 / THREADS;
  const Target& t;
  Model model;
  __device__ CholeskyFactoredMetric(const Target& tt, const ModelArgs& m) : t(tt), model(m, tt.dim) {}
  __device__ void reset() {}

  __device__ int build(const Blk& k, RmWork& w, const double* q) {
    const bool ok = model.fill(k, q, w.M1, w.ld);
    return block_any(k, !ok) ? MB200_STATUS_LINALG : 0;  // "Array is not finite" (:207-215)
  }
  // a zero diagonal entry: scipy's solve_triangular raises LinAlgError ("singular matrix")
  __device__ bool singular(const Blk& k, RmWork& w) const {
    bool z = false;
    for (int i = k.tid; i < w.dim; i += k.nthr)
      if (w.M1[i * w.ld + i] == 0.0) z = true;
    return block_any(k, z);
  }
  __device__ double log_abs_det(const Blk& k, RmWork& w) const {
    double s = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) s += log(fabs(w.M1[i * w.ld + i]));
    return 2.0 * block_sum(k, s);
  }
  __device__ void inv_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    cholesky_solve(k, w.M1, w.dim, w.ld, v, out);
  }
  __device__ bool sqrt_matvec(const Blk& k, RmWork& w, const double* v, double* out) const {
    for (int i = k.tid; i < w.dim; i += k.nthr) {
      double s = 0.0;
      for (int j = 0; j <= i; ++j) s = fma(w.M1[i * w.ld + j], v[j], s);
      out[i] = s;
    }
    __syncthreads();
    return true;
  }
  // d = 2 / diag L in w.ev; a DENSE_VJP model: V = diag(d) in w.M2, strict lower triangle zero
  __device__ void vjp_grad_log_abs_det(const Blk& k, RmWork& w, const double* q, double* out) {
    if constexpr (chol_dense_vjp<Model>::value) {
      const int ld = w.ld;
      for (int i = k.warp; i < w.dim; i += k.nwarp)  // one row per warp: coalesced
        for (int j = k.lane; j <= i; j += 32)
          w.M2[i * ld + j] = j == i ? 2.0 / w.M1[i * ld + i] : 0.0;
      __syncthreads();
      model.vjp_tril(k, q, w.M2, ld, out);
    } else {
      for (int i = k.tid; i < w.dim; i += k.nthr) w.ev[i] = 2.0 / w.M1[i * w.ld + i];
      __syncthreads();
      model.vjp_diag(k, q, w.ev, out);
    }
    __syncthreads();
  }
  // b = L^-1 p in w.lam (computed once: M^-1 p = L^-T b continues from it), a = M^-1 p in w.ev;
  // scan scratch w.sa, w.gsa.  A DENSE_VJP model: V = tril(-2 a b^T) in w.M2
  __device__ void vjp_grad_quad_inv(const Blk& k, RmWork& w, const double* q, const double* p,
                                    double* out) {
    cholesky_forward(k, w.M1, w.dim, w.ld, p, w.lam);
    for (int i = k.tid; i < w.dim; i += k.nthr) w.ev[i] = w.lam[i];
    __syncthreads();
    cholesky_back(k, w.M1, w.dim, w.ld, w.ev);
    if constexpr (chol_dense_vjp<Model>::value) {
      const int ld = w.ld;
      for (int i = k.warp; i < w.dim; i += k.nwarp) {
        const double a = w.ev[i];
        for (int j = k.lane; j <= i; j += 32) w.M2[i * ld + j] = -2.0 * (a * w.lam[j]);
      }
      __syncthreads();
      model.vjp_tril(k, q, w.M2, ld, out);
    } else {
      model.vjp_outer(k, q, -2.0, w.ev, w.lam, w.sa, w.gsa, out);
    }
    __syncthreads();
  }
};

template <class Target>
using QuadraticCholeskyMetric = CholeskyFactoredMetric<Target, QuadraticCholModel>;

// What rm_launch reads of the model of a user image's Cholesky-factored policy (UserCholModel of
// user_riemannian.cuh derives from it): CholeskyFactoredMetric<UserRTargetTraits,
// UserCholModelTraits> carries the image policy's launch constants
struct UserCholModelTraits {
  static constexpr bool DENSE_VJP = true;
};

// ---------------------------------------------------------------------------------------------
// K4: solve_fixed_point_direct (solvers.py:47-94) for one chain, block-cooperative.
// `func(x_in, x_out)` returns 0 or a failure code (any failure inside the solver is a
// ConvergenceError, :89-92).  The same iterate sequence and the same stopping rule as the
// reference: x = func(x0); error = max|x - x0| (NaN-propagating); diverged if error > div_tol or
// NaN; converged -- returning the NEW iterate -- if error < tol; else x0 = x.  Iterates alternate
// between the buffers xa (holding x0 on entry) and xb; on success *result points at the solution.
// ---------------------------------------------------------------------------------------------
template <class F>
__device__ inline int fixed_point_direct(const Blk& k, int dim, double* xa, double* xb, F func,
                                         double tol, double div_tol, int max_iters,
                                         double** result, int& iters) {
  double* xin = xa;
  double* xout = xb;
  for (int i = 0; i < max_iters; ++i) {
    if (func(xin, xout) != 0) return MB200_STATUS_CONVERGENCE;
    double e = 0.0;
    for (int j = k.tid; j < dim; j += k.nthr) e = nanmax(e, fabs(xout[j] - xin[j]));
    const double err = block_nanmax(k, e);
    ++iters;
    if (err > div_tol || err != err) return MB200_STATUS_CONVERGENCE;
    if (err < tol) {
      *result = xout;
      return 0;
    }
    double* tmp = xin;
    xin = xout;
    xout = tmp;
  }
  return MB200_STATUS_CONVERGENCE;
}

// solve_fixed_point_steffensen (solvers.py:97-154): Aitken-extrapolated iteration, two function
// evaluations per iteration: x1 = f(x0), x2 = f(x1), x = x0 - (x1 - x0)^2 / (x2 - 2 x1 + x0) with
// exact-zero denominators replaced by machine epsilon (:130-133); same divergence / convergence
// tests on |x - x0| as the direct solver.  Iterates live in xa (x0 on entry), xb, xc.
template <class F>
__device__ inline int fixed_point_steffensen(const Blk& k, int dim, double* xa, double* xb,
                                             double* xc, F func, double tol, double div_tol,
                                             int max_iters, double** result, int& iters) {
  double* x0 = xa;
  double* x1 = xb;
  double* x2 = xc;
  for (int i = 0; i < max_iters; ++i) {
    if (func(x0, x1) != 0) return MB200_STATUS_CONVERGENCE;
    if (func(x1, x2) != 0) return MB200_STATUS_CONVERGENCE;
    double e = 0.0;
    for (int j = k.tid; j < dim; j += k.nthr) {
      double denom = __dadd_rn(__dsub_rn(x2[j], __dmul_rn(2.0, x1[j])), x0[j]);
      if (fabs(denom) == 0.0) denom = DBL_EPSILON;
      const double d1 = __dsub_rn(x1[j], x0[j]);
      const double x = __dsub_rn(x0[j], __dmul_rn(d1, d1) / denom);
      e = nanmax(e, fabs(x - x0[j]));
      x2[j] = x;
    }
    const double err = block_nanmax(k, e);
    ++iters;
    if (err > div_tol || err != err) return MB200_STATUS_CONVERGENCE;
    if (err < tol) {
      *result = x2;
      return 0;
    }
    double* tmp = x0;
    x0 = x2;
    x2 = tmp;
  }
  return MB200_STATUS_CONVERGENCE;
}

#ifndef __CUDACC_RTC__  // library self-tests: kept out of the run-time compiled user images
// Diagnostic kernel: K4 on the reference's own known-answer problems
// (reference tests/test_solvers.py:25-47): 0 babylonian (y/x + x)/2, 1 ratio (x+y)/(x+1),
// 2 cosine, 3 doubling 2x, 4 quadratic 1 + x^2.  One CTA per problem instance.
static __global__ void __launch_bounds__(64)
    fixed_point_selftest_kernel(int func_id, int solver, const double* __restrict__ x0,
                                const double* __restrict__ y, int64_t n, int dim, double tol,
                                double div_tol, int max_iters, double* __restrict__ x_out,
                                int32_t* __restrict__ iters_out, int32_t* __restrict__ status) {
  extern __shared__ double smem[];
  Blk k;
  k.tid = threadIdx.x, k.nthr = blockDim.x, k.lane = threadIdx.x & 31;
  k.warp = threadIdx.x >> 5, k.nwarp = blockDim.x >> 5;
  double* xa = smem;
  double* xb = smem + dim;
  double* xc = smem + 2 * dim;
  k.red = smem + 3 * dim;
  for (int64_t ch = blockIdx.x; ch < n; ch += gridDim.x) {
    __syncthreads();
    for (int j = k.tid; j < dim; j += k.nthr) xa[j] = x0[ch * dim + j];
    __syncthreads();
    auto func = [&](const double* xin, double* xout) {
      for (int j = k.tid; j < dim; j += k.nthr) {
        const double x = xin[j], yy = y[ch * dim + j];
        double r;
        if (func_id == 0) r = (yy / x + x) / 2.0;
        else if (func_id == 1) r = (x + yy) / (x + 1.0);
        else if (func_id == 2) r = cos(x);
        else if (func_id == 3) r = 2.0 * x;
        else r = 1.0 + x * x;
        xout[j] = r;
      }
      __syncthreads();
      return 0;
    };
    double* sol = xa;
    int iters = 0;
    const int st = solver == 1 ? fixed_point_steffensen(k, dim, xa, xb, xc, func, tol, div_tol,
                                                        max_iters, &sol, iters)
                               : fixed_point_direct(k, dim, xa, xb, func, tol, div_tol, max_iters,
                                                    &sol, iters);
    for (int j = k.tid; j < dim; j += k.nthr) x_out[ch * dim + j] = sol[j];
    if (k.tid == 0) {
      iters_out[ch] = iters;
      status[ch] = st;
    }
  }
}
#endif

// ---------------------------------------------------------------------------------------------
// K4 + K5: the integrator
// ---------------------------------------------------------------------------------------------
template <class Target, class Metric>
struct ImplicitLeapfrog {
  const Blk& k;
  RmWork& w;
  const Target& t;
  Metric& m;
  double fp_tol, fp_div, rev_tol;
  int fp_max;
  int fp_solver;  // MB200_FP_SOLVER_DIRECT / MB200_FP_SOLVER_STEFFENSEN
  // call counters of the chain in flight (block-uniform; mb200_set_call_counters):
  // gradients of l, metric builds (factorisations / eigendecompositions), VJPs of the
  // quadratic form p.M^-1 p, fixed-point iterations
  int n_grad = 0, n_build = 0, n_quad = 0, n_fp = 0;
  __device__ __forceinline__ int build_(const double* q) {
    ++n_build;
    return m.build(k, w, q);
  }
  __device__ __forceinline__ void grad_(const double* q, double* g) {
    ++n_grad;
    t.grad(k, q, g);
  }
  __device__ __forceinline__ void quad_(const double* q, const double* p, double* out) {
    ++n_quad;
    m.vjp_grad_quad_inv(k, w, q, p, out);
  }

  // K4 on this chain's buffers (see fixed_point_direct below)
  template <class F>
  __device__ int fixed_point(F func, double** result, int& iters) {
    if (fp_solver == MB200_FP_SOLVER_STEFFENSEN)
      return fixed_point_steffensen(k, w.dim, w.x0, w.x1, w.x2, func, fp_tol, fp_div, fp_max,
                                    result, iters);
    return fixed_point_direct(k, w.dim, w.x0, w.x1, func, fp_tol, fp_div, fp_max, result, iters);
  }

  // dh1_dpos = grad l + vjp(grad_log_abs_det) / 2   (systems.py:1381-1385); metric of q current
  __device__ void kick_h1(double dt) {
    grad_(w.q, w.v1);
    m.vjp_grad_log_abs_det(k, w, w.q, w.v2);
    for (int i = k.tid; i < w.dim; i += k.nthr)
      w.p[i] = __dsub_rn(w.p[i], __dmul_rn(dt, __dadd_rn(w.v1[i], __dmul_rn(0.5, w.v2[i]))));
    __syncthreads();
  }

  // one step; q, p in w.q / w.p updated in place; returns status
  __device__ int step(double dt, int* iters4) {
    const int n = w.dim;
    int st;
    int it_b = 0, it_crev = 0, it_c = 0, it_brev = 0;
    // ---- _step_a (:493-494)
    m.reset();
    st = build_(w.q);
    if (st != 0) return MB200_STATUS_LINALG;
    kick_h1(dt);
    // ---- _step_b_fwd (:496-502): p = p0 - dt * dh2_dpos(q, p), metric fixed
    for (int i = k.tid; i < n; i += k.nthr) w.base[i] = w.p[i], w.x0[i] = w.p[i];
    __syncthreads();
    double* sol;
    auto fb = [&](double sdt) {
      return [&, sdt](const double* xin, double* xout) {
        quad_(w.q, xin, w.v1);
        for (int i = k.tid; i < n; i += k.nthr)
          xout[i] = __dsub_rn(w.base[i], __dmul_rn(sdt, __dmul_rn(0.5, w.v1[i])));
        __syncthreads();
        return 0;
      };
    };
    st = fixed_point(fb(dt), &sol, it_b);
    iters4[0] = it_b;
    if (st != 0) return st;
    for (int i = k.tid; i < n; i += k.nthr) w.p[i] = sol[i];
    __syncthreads();
    // ---- _step_c_fwd (:517-528): q += dt * M(q)^-1 p, then reverse check with _step_c_adj(-dt)
    for (int i = k.tid; i < n; i += k.nthr) w.v3[i] = w.q[i];  // pos_init
    __syncthreads();
    m.inv_matvec(k, w, w.p, w.v1);
    for (int i = k.tid; i < n; i += k.nthr) w.q[i] = __dadd_rn(w.q[i], __dmul_rn(dt, w.v1[i]));
    __syncthreads();
    // fixed point in q: x = base + sdt * M(x)^-1 p, new metric every iteration (:530-536)
    auto fc = [&](double sdt) {
      return [&, sdt](const double* xin, double* xout) {
        const int bs = build_(xin);
        if (bs != 0) return 1;
        m.inv_matvec(k, w, w.p, w.v1);
        for (int i = k.tid; i < n; i += k.nthr)
          xout[i] = __dadd_rn(w.base[i], __dmul_rn(sdt, w.v1[i]));
        __syncthreads();
        return 0;
      };
    };
    for (int i = k.tid; i < n; i += k.nthr) w.base[i] = w.q[i], w.x0[i] = w.q[i];
    __syncthreads();
    st = fixed_point(fc(-dt), &sol, it_crev);
    iters4[1] = it_crev;
    if (st != 0) return st;
    {
      double e = 0.0;
      for (int i = k.tid; i < n; i += k.nthr) e = nanmax(e, fabs(sol[i] - w.v3[i]));
      const double rev = block_nanmax(k, e);
      if (rev > rev_tol) return MB200_STATUS_NON_REVERSIBLE;
    }
    // ---- _step_c_adj (:530-536)
    for (int i = k.tid; i < n; i += k.nthr) w.base[i] = w.q[i], w.x0[i] = w.q[i];
    __syncthreads();
    st = fixed_point(fc(dt), &sol, it_c);
    iters4[2] = it_c;
    if (st != 0) return st;
    for (int i = k.tid; i < n; i += k.nthr) w.q[i] = sol[i];
    __syncthreads();
    // ---- _step_b_adj (:504-515): p -= dt * dh2_dpos(q, p) at the new metric, then reverse check
    st = build_(w.q);
    if (st != 0) return MB200_STATUS_LINALG;
    for (int i = k.tid; i < n; i += k.nthr) w.v3[i] = w.p[i];  // mom_init
    __syncthreads();
    quad_(w.q, w.p, w.v1);
    for (int i = k.tid; i < n; i += k.nthr)
      w.p[i] = __dsub_rn(w.p[i], __dmul_rn(dt, __dmul_rn(0.5, w.v1[i])));
    __syncthreads();
    for (int i = k.tid; i < n; i += k.nthr) w.base[i] = w.p[i], w.x0[i] = w.p[i];
    __syncthreads();
    st = fixed_point(fb(-dt), &sol, it_brev);
    iters4[3] = it_brev;
    if (st != 0) return st;
    {
      double e = 0.0;
      for (int i = k.tid; i < n; i += k.nthr) e = nanmax(e, fabs(sol[i] - w.v3[i]));
      const double rev = block_nanmax(k, e);
      if (rev > rev_tol) return MB200_STATUS_NON_REVERSIBLE;
    }
    // ---- _step_a
    kick_h1(dt);
    return MB200_STATUS_OK;
  }

  // ---- ImplicitMidpointIntegrator (integrators.py:547-681), "next" row N4 ----------------
  // dh/dz at (q, p): vel = dh_dmom = M(q)^-1 p; force = dh_dpos = dh1_dpos + dh2_dpos
  // (systems.py:198-207, 1381-1399).  Returns 0 or the metric-build failure.
  __device__ int hamiltonian_gradient(const double* q, const double* p, double* vel,
                                      double* force) {
    if (build_(q) != 0) return 1;
    m.inv_matvec(k, w, p, vel);
    grad_(q, w.v1);
    m.vjp_grad_log_abs_det(k, w, q, w.v2);
    quad_(q, p, w.v3);
    for (int i = k.tid; i < w.dim; i += k.nthr)
      force[i] = __dadd_rn(__dadd_rn(w.v1[i], __dmul_rn(0.5, w.v2[i])), __dmul_rn(0.5, w.v3[i]));
    __syncthreads();
    return 0;
  }

  // _step_a_fwd (:609-626): fixed point z = z0 + [dt dh_dmom(z); -dt dh_dpos(z)] in z = (q, p),
  // starting from (and based at) the (q, p) held in w.zb.  Solution pointer in *sol.
  __device__ int midpoint_fwd(double dt, double** sol, int& iters) {
    const int n = w.dim;
    for (int i = k.tid; i < 2 * n; i += k.nthr) w.z0[i] = w.zb[i];
    __syncthreads();
    auto func = [&](const double* zin, double* zout) {
      if (hamiltonian_gradient(zin, zin + n, w.x0, w.x1) != 0) return 1;
      for (int i = k.tid; i < n; i += k.nthr) {
        zout[i] = __dadd_rn(w.zb[i], __dmul_rn(dt, w.x0[i]));
        zout[n + i] = __dadd_rn(w.zb[n + i], __dmul_rn(-dt, w.x1[i]));
      }
      __syncthreads();
      return 0;
    };
    if (fp_solver == MB200_FP_SOLVER_STEFFENSEN)
      return fixed_point_steffensen(k, 2 * n, w.z0, w.z1, w.z2, func, fp_tol, fp_div, fp_max, sol,
                                    iters);
    return fixed_point_direct(k, 2 * n, w.z0, w.z1, func, fp_tol, fp_div, fp_max, sol, iters);
  }

  // one implicit-midpoint step (:679-681): _step_a_fwd(dt/2) then _step_a_adj(dt/2)
  __device__ int midpoint_step(double dt_full, int* iters4) {
    const int n = w.dim;
    const double dt = dt_full / 2;
    m.reset();
    int it_fwd = 0, it_rev = 0;
    double* sol;
    for (int i = k.tid; i < n; i += k.nthr) w.zb[i] = w.q[i], w.zb[n + i] = w.p[i];
    __syncthreads();
    int st = midpoint_fwd(dt, &sol, it_fwd);
    iters4[0] = it_fwd;
    if (st != 0) return st;
    for (int i = k.tid; i < n; i += k.nthr) w.q[i] = sol[i], w.p[i] = sol[n + i];
    __syncthreads();
    // _step_a_adj (:628-647): explicit Euler half-step from state_prev ...
    if (hamiltonian_gradient(w.q, w.p, w.x0, w.x1) != 0) return MB200_STATUS_LINALG;
    for (int i = k.tid; i < n; i += k.nthr) {
      w.zp[i] = w.q[i], w.zp[n + i] = w.p[i];  // state_prev
      w.q[i] = __dadd_rn(w.q[i], __dmul_rn(dt, w.x0[i]));
      w.p[i] = __dsub_rn(w.p[i], __dmul_rn(dt, w.x1[i]));
    }
    __syncthreads();
    // ... then the reversibility check: _step_a_fwd(state_back, -dt) must return to state_prev
    for (int i = k.tid; i < n; i += k.nthr) w.zb[i] = w.q[i], w.zb[n + i] = w.p[i];
    __syncthreads();
    st = midpoint_fwd(-dt, &sol, it_rev);
    iters4[1] = it_rev;
    if (st != 0) return st;
    double e = 0.0;
    for (int i = k.tid; i < 2 * n; i += k.nthr) e = nanmax(e, fabs(sol[i] - w.zp[i]));
    const double rev = block_nanmax(k, e);
    if (rev > rev_tol) return MB200_STATUS_NON_REVERSIBLE;
    return MB200_STATUS_OK;
  }

  // h = l(q) + log|M|/2 + p.M^-1 p/2   (systems.py:1375-1390); NaN if the metric cannot be built
  __device__ double hamiltonian() {
    m.reset();
    if (m.build(k, w, w.q) != 0) return nan("");  // diagnostics: not counted
    if constexpr (rm_singular_policy<Metric>::value)
      if (m.singular(k, w)) return nan("");
    m.inv_matvec(k, w, w.p, w.v1);
    double s = 0.0;
    for (int i = k.tid; i < w.dim; i += k.nthr) s = fma(w.p[i], w.v1[i], s);
    const double kin = block_sum(k, s);
    const double lad = m.log_abs_det(k, w);
    const double l = t.nld(k, w.q);
    return (l + 0.5 * lad) + 0.5 * kin;
  }
};

template <class Target, template <class> class MetricT>
__global__ void __launch_bounds__(MetricT<Target>::THREADS, MetricT<Target>::MIN_BLOCKS)
    implicit_leapfrog_kernel(const double* q_in, const double* p_in, double* q_out, double* p_out,
                             const int32_t* __restrict__ dir, int64_t n_chains, int dim,
                             double step_size, int n_steps, ModelArgs model, double fp_tol,
                             double fp_div, int fp_max, double rev_tol,
                             double* __restrict__ h_out, int32_t* __restrict__ status,
                             int32_t* __restrict__ n_done, int32_t* __restrict__ fp_iters,
                             RmLayout layout, int midpoint, int fp_solver) {
  Blk blk;
  RmWork w;
  double* const tscratch = rm_begin<MetricT<Target>::PLACE == RM_COMPACT>(layout, model, blk, w);
  const Target target(model, dim);
  target.attach(tscratch);
  MetricT<Target> metric(target, model);
  ImplicitLeapfrog<Target, MetricT<Target>> integ{blk,    w,      target,  metric,
                                                  fp_tol, fp_div, rev_tol, fp_max, fp_solver};

  for (int64_t ch = blockIdx.x; ch < n_chains; ch += gridDim.x) {
    __syncthreads();
    for (int i = blk.tid; i < dim; i += blk.nthr) {
      w.q[i] = q_in[(size_t)ch * dim + i];
      w.p[i] = p_in[(size_t)ch * dim + i];
    }
    __syncthreads();
    const double eps = model.step_sizes != nullptr ? model.step_sizes[ch] : step_size;
    const double dt = (dir != nullptr) ? (double)dir[ch] * eps : eps;
    const int ns = model.n_steps_pc != nullptr ? min(model.n_steps_pc[ch], n_steps) : n_steps;
    int st = MB200_STATUS_OK, done = 0;
    int it4[4] = {0, 0, 0, 0};
    integ.n_grad = integ.n_build = integ.n_quad = integ.n_fp = 0;
    for (int s = 0; s < ns && st == MB200_STATUS_OK; ++s) {
      for (int i = blk.tid; i < dim; i += blk.nthr) w.qs[i] = w.q[i], w.ps[i] = w.p[i];
      __syncthreads();
      int it_step[4] = {0, 0, 0, 0};
      st = midpoint ? integ.midpoint_step(dt, it_step) : integ.step(dt, it_step);
      integ.n_fp += it_step[0] + it_step[1] + it_step[2] + it_step[3];
      if (st == MB200_STATUS_OK) {
        ++done;
#pragma unroll
        for (int j = 0; j < 4; ++j) it4[j] = it_step[j];
      } else {
        __syncthreads();
        for (int i = blk.tid; i < dim; i += blk.nthr) w.q[i] = w.qs[i], w.p[i] = w.ps[i];
        __syncthreads();
      }
    }
    for (int i = blk.tid; i < dim; i += blk.nthr) {
      q_out[(size_t)ch * dim + i] = w.q[i];
      p_out[(size_t)ch * dim + i] = w.p[i];
    }
    if (h_out != nullptr) {
      const double h = integ.hamiltonian();
      if (blk.tid == 0) h_out[ch] = h;
    }
    if (blk.tid == 0) {
      if (status != nullptr) status[ch] = st;
      if (n_done != nullptr) n_done[ch] = done;
      if (fp_iters != nullptr)
        for (int j = 0; j < 4; ++j) fp_iters[ch * 4 + j] = it4[j];
      if (model.counters != nullptr) {  // the energy evaluation above is not counted
        int32_t* c = model.counters + ch * MB200_N_COUNTERS;
        c[MB200_COUNT_GRAD] += integ.n_grad, c[MB200_COUNT_METRIC] += integ.n_build;
        c[MB200_COUNT_QUAD_VJP] += integ.n_quad, c[MB200_COUNT_SOLVER_ITERS] += integ.n_fp;
      }
    }
  }
}

// mom = sqrt(M(q)) z for every chain: RiemannianMetricSystem.sample_momentum (systems.py:1401-1402).
template <class Target, template <class> class MetricT>
__global__ void __launch_bounds__(MetricT<Target>::THREADS, MetricT<Target>::MIN_BLOCKS)
    riemannian_sample_momentum_kernel(const double* __restrict__ q_in, const double* __restrict__ z,
                                      double* __restrict__ p_out, int64_t n_chains, int dim,
                                      ModelArgs model, int32_t* __restrict__ status,
                                      RmLayout layout) {
  Blk blk;
  RmWork w;
  double* const tscratch =
      rm_begin<MetricT<Target>::PLACE == RM_COMPACT, false>(layout, model, blk, w);
  const Target target(model, dim);
  target.attach(tscratch);
  MetricT<Target> metric(target, model);
  for (int64_t ch = blockIdx.x; ch < n_chains; ch += gridDim.x) {
    __syncthreads();
    for (int i = blk.tid; i < dim; i += blk.nthr) {
      w.q[i] = q_in[(size_t)ch * dim + i];
      w.v1[i] = z[(size_t)ch * dim + i];
    }
    __syncthreads();
    metric.reset();
    int st = metric.build(blk, w, w.q) != 0 ? MB200_STATUS_LINALG : MB200_STATUS_OK;
    if (st == MB200_STATUS_OK && !metric.sqrt_matvec(blk, w, w.v1, w.v2)) st = MB200_STATUS_LINALG;
    for (int i = blk.tid; i < dim; i += blk.nthr)
      p_out[(size_t)ch * dim + i] = (st == MB200_STATUS_OK) ? w.v2[i] : nan("");
    if (blk.tid == 0 && status != nullptr) status[ch] = st;
  }
}

// vel = M(q)^-1 p for every chain: RiemannianMetricSystem.dh2_dmom / dh_dmom (systems.py:1398-1399,
// 202-207), read by the no-U-turn criteria (transitions.py:434-435, 472-473).
template <class Target, template <class> class MetricT>
__global__ void __launch_bounds__(MetricT<Target>::THREADS, MetricT<Target>::MIN_BLOCKS)
    riemannian_velocity_kernel(const double* __restrict__ q_in, const double* __restrict__ p_in,
                               double* __restrict__ vel_out, int64_t n_chains, int dim,
                               ModelArgs model, int32_t* __restrict__ status,
                                      RmLayout layout) {
  Blk blk;
  RmWork w;
  double* const tscratch =
      rm_begin<MetricT<Target>::PLACE == RM_COMPACT, false>(layout, model, blk, w);
  const Target target(model, dim);
  target.attach(tscratch);
  MetricT<Target> metric(target, model);
  for (int64_t ch = blockIdx.x; ch < n_chains; ch += gridDim.x) {
    __syncthreads();
    for (int i = blk.tid; i < dim; i += blk.nthr) {
      w.q[i] = q_in[(size_t)ch * dim + i];
      w.p[i] = p_in[(size_t)ch * dim + i];
    }
    __syncthreads();
    metric.reset();
    int st = metric.build(blk, w, w.q) != 0 ? MB200_STATUS_LINALG : MB200_STATUS_OK;
    if constexpr (rm_singular_policy<MetricT<Target>>::value)
      if (st == MB200_STATUS_OK && metric.singular(blk, w)) st = MB200_STATUS_LINALG;
    if (st == MB200_STATUS_OK) metric.inv_matvec(blk, w, w.p, w.v1);
    for (int i = blk.tid; i < dim; i += blk.nthr)
      vel_out[(size_t)ch * dim + i] = (st == MB200_STATUS_OK) ? w.v1[i] : nan("");
    if (blk.tid == 0 && status != nullptr) status[ch] = st;
  }
}

// The velocity kernel (VELOCITY) or the momentum-refresh kernel of a target / metric pair; only
// the one asked for is instantiated
template <class Target, template <class> class MetricT, bool VELOCITY>
inline auto riemannian_vector_kernel() {
  if constexpr (VELOCITY)
    return riemannian_velocity_kernel<Target, MetricT>;
  else
    return riemannian_sample_momentum_kernel<Target, MetricT>;
}

}  // namespace mb200
