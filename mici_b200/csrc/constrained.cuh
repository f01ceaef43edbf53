// K6: constrained (RATTLE / geodesic) leapfrog with Newton projection -- one warp per chain.
//
// Replaces, per chain (reference paths):
//   ConstrainedLeapfrogIntegrator._step/_step_a/_step_b            integrators.py:929-984
//   solve_projection_onto_manifold_newton                          solvers.py:346-469
//   ConstrainedEuclideanMetricSystem.project_onto_cotangent_space  systems.py:863-873
//   DenseConstrainedEuclideanMetricSystem.jacob_constr_inner_product systems.py:1006-1022
//   dh2_flow_dmom = (|dt| M^-1, I)                                 systems.py:794-799
//
// One warp owns one chain for the whole launch; vectors are in registers in the pair layout of
// metric_ops.cuh.  Every branch (Newton convergence, divergence, reversibility failure) is
// uniform across the warp, so chains in other warps proceed independently: the per-chain
// convergence mask of the reference's Python loop is the warp's own control flow.  The C x C
// systems (C = Target::NC <= 8) are solved redundantly in registers by every lane.  The same
// kernels with GAUSS = true run GaussianDenseConstrainedEuclideanMetricSystem (systems.py:1034-1184).
#pragma once
#include "metric_ops.cuh"
#include "targets.cuh"

namespace mb200 {

// ---------------------------------------------------------------------------------------------
// Constrained targets (warp-cooperative interface, pair layout)
//   grad(lane, dim, q, g)               gradient of l
//   nld(lane, dim, q)                   l(q), same value on all lanes
//   constr_jacob(lane, dim, q, c, J)    c(q) [NC] on all lanes; J[NC][NV] columns owned by lane
//   mhp(lane, dim, q, m, out)           out_j = sum_{k,i} m[k][i] d^2 c_k / dq_i dq_j
// User-written constraints implement the same interface (UserConstrainedTarget,
// user_constraint.cuh).
// ---------------------------------------------------------------------------------------------

// Torus in R^3 (reference README.md:315-337): rho = sqrt(x^2+y^2), theta = atan2(y, x),
// phi = atan2(z, rho - R);  l = log1p(r cos(phi)/R) - log1p(alpha sin(4 theta) cos(phi));
// c = (rho - R)^2 + z^2 - r^2.
struct TorusTarget {
  static constexpr int NC = 1;
  double R, r, alpha;
  __device__ TorusTarget(const ModelArgs& m, int) : R(m.tp[0]), r(m.tp[1]), alpha(m.tp[2]) {}

  template <int NV>
  __device__ __forceinline__ void gather(const double (&q)[NV], double& x, double& y,
                                         double& z) const {
    x = __shfl_sync(FULL_MASK, q[0], 0);
    y = __shfl_sync(FULL_MASK, q[1], 0);
    z = __shfl_sync(FULL_MASK, q[0], 1);
  }

  template <int NV>
  __device__ __forceinline__ void grad(int lane, int, const double (&q)[NV],
                                       double (&g)[NV]) const {
    double x, y, z;
    gather(q, x, y, z);
    const double a = r / R;
    const double rho2 = x * x + y * y;
    const double rho = sqrt(rho2);
    const double u = rho - R;
    const double theta = atan2(y, x);
    const double phi = atan2(z, u);
    double s4, c4, sp, cp;
    sincos(4.0 * theta, &s4, &c4);
    sincos(phi, &sp, &cp);
    const double d1 = 1.0 + a * cp;
    const double d2 = 1.0 + alpha * s4 * cp;
    const double dl_dphi = -a * sp / d1 + alpha * s4 * sp / d2;
    const double dl_dth = -4.0 * alpha * c4 * cp / d2;
    const double w = u * u + z * z;
    const double dphi_du = -z / w;
    const double dphi_dz = u / w;
    const double gx = dl_dth * (-y / rho2) + dl_dphi * dphi_du * (x / rho);
    const double gy = dl_dth * (x / rho2) + dl_dphi * dphi_du * (y / rho);
    const double gz = dl_dphi * dphi_dz;
#pragma unroll
    for (int e = 0; e < NV; ++e) g[e] = 0.0;
    if (lane == 0) g[0] = gx, g[1] = gy;
    if (lane == 1) g[0] = gz;
  }

  template <int NV>
  __device__ __forceinline__ double nld(int, int, const double (&q)[NV]) const {
    double x, y, z;
    gather(q, x, y, z);
    const double rho = sqrt(x * x + y * y);
    const double theta = atan2(y, x);
    const double phi = atan2(z, rho - R);
    return log1p(r * cos(phi) / R) - log1p(sin(4.0 * theta) * cos(phi) * alpha);
  }

  template <int NV>
  __device__ __forceinline__ void constr_jacob(int lane, int, const double (&q)[NV],
                                               double (&c)[NC], double (&J)[NC][NV]) const {
    double x, y, z;
    gather(q, x, y, z);
    const double rho = sqrt(x * x + y * y);
    const double d = rho - R;
    c[0] = d * d + z * z - r * r;
    const double f = 2.0 * d / rho;
#pragma unroll
    for (int e = 0; e < NV; ++e) J[0][e] = 0.0;
    if (lane == 0) J[0][0] = f * x, J[0][1] = f * y;
    if (lane == 1) J[0][0] = 2.0 * z;
  }

  // out_j = sum_{k,i} m[k][i] d^2 c_k / dq_i dq_j (matrix-Hessian product, systems.py:964-975):
  // with f = 2 (rho - R) / rho and g = 2 R / rho^3 the Hessian of c is
  // [[f + g x^2, g x y, 0], [g x y, f + g y^2, 0], [0, 0, 2]]
  template <int NV>
  __device__ __forceinline__ void mhp(int lane, int, const double (&q)[NV],
                                      const double (&m)[NC][NV], double (&out)[NV]) const {
    double x, y, z;
    gather(q, x, y, z);
    const double mx = __shfl_sync(FULL_MASK, m[0][0], 0);
    const double my = __shfl_sync(FULL_MASK, m[0][1], 0);
    const double mz = __shfl_sync(FULL_MASK, m[0][0], 1);
    const double rho = sqrt(x * x + y * y);
    const double f = 2.0 * (rho - R) / rho;
    const double g = 2.0 * R / (rho * rho * rho);
#pragma unroll
    for (int e = 0; e < NV; ++e) out[e] = 0.0;
    if (lane == 0) {
      out[0] = mx * (f + g * x * x) + my * (g * x * y);
      out[1] = mx * (g * x * y) + my * (f + g * y * y);
    }
    if (lane == 1) out[0] = 2.0 * mz;
  }
};

// Unit sphere in R^D: l = |q|^2/2 + q[0];  c = |q|^2 - 1.
struct SphereTarget {
  static constexpr int NC = 1;
  __device__ SphereTarget(const ModelArgs&, int) {}

  template <int NV>
  __device__ __forceinline__ void grad(int lane, int dim, const double (&q)[NV],
                                       double (&g)[NV]) const {
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
      g[e] = (i < dim) ? q[e] : 0.0;
      if (i == 0) g[e] += 1.0;
    }
  }

  template <int NV>
  __device__ __forceinline__ double nld(int, int, const double (&q)[NV]) const {
    double s = 0.0;
#pragma unroll
    for (int e = 0; e < NV; ++e) s = fma(q[e], q[e], s);
    s = warp_sum(s);
    return 0.5 * s + __shfl_sync(FULL_MASK, q[0], 0);
  }

  template <int NV>
  __device__ __forceinline__ void constr_jacob(int, int, const double (&q)[NV], double (&c)[NC],
                                               double (&J)[NC][NV]) const {
    double s = 0.0;
#pragma unroll
    for (int e = 0; e < NV; ++e) s = fma(q[e], q[e], s);
    c[0] = warp_sum(s) - 1.0;
#pragma unroll
    for (int e = 0; e < NV; ++e) J[0][e] = 2.0 * q[e];
  }

  template <int NV>
  __device__ __forceinline__ void mhp(int, int, const double (&)[NV], const double (&m)[NC][NV],
                                      double (&out)[NV]) const {
#pragma unroll
    for (int e = 0; e < NV; ++e) out[e] = 2.0 * m[0][e];  // Hessian of c is 2 I
  }
};

// NCON unit spheres: consecutive blocks of dim / NCON coordinates, c_k = |q_block_k|^2 - 1;
// l = |q|^2/2 + q[0].  With a dense metric the Gram matrix is a full NCON x NCON matrix.
template <int NCON>
struct MultiSphereTarget {
  static constexpr int NC = NCON;
  int block;
  __device__ MultiSphereTarget(const ModelArgs&, int dim) : block(dim / NCON) {}

  template <int NV>
  __device__ __forceinline__ void grad(int lane, int dim, const double (&q)[NV],
                                       double (&g)[NV]) const {
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
      g[e] = (i < dim) ? q[e] : 0.0;
      if (i == 0) g[e] += 1.0;
    }
  }

  template <int NV>
  __device__ __forceinline__ double nld(int, int, const double (&q)[NV]) const {
    double s = 0.0;
#pragma unroll
    for (int e = 0; e < NV; ++e) s = fma(q[e], q[e], s);
    s = warp_sum(s);
    return 0.5 * s + __shfl_sync(FULL_MASK, q[0], 0);
  }

  template <int NV>
  __device__ __forceinline__ void constr_jacob(int lane, int dim, const double (&q)[NV],
                                               double (&c)[NC], double (&J)[NC][NV]) const {
#pragma unroll
    for (int a = 0; a < NC; ++a) {
      double s = 0.0;
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
        const bool mine = i < dim && i / block == a;
        J[a][e] = mine ? 2.0 * q[e] : 0.0;
        if (mine) s = fma(q[e], q[e], s);
      }
      c[a] = warp_sum(s) - 1.0;
    }
  }

  template <int NV>
  __device__ __forceinline__ void mhp(int lane, int dim, const double (&)[NV],
                                      const double (&m)[NC][NV], double (&out)[NV]) const {
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
      double v = 0.0;
#pragma unroll
      for (int a = 0; a < NC; ++a)
        if (i < dim && i / block == a) v = 2.0 * m[a][e];
      out[e] = v;
    }
  }
};

// ---------------------------------------------------------------------------------------------
// small dense C x C algebra in registers (every lane holds the full matrix)
// ---------------------------------------------------------------------------------------------

// x = G^-1 u via the explicit inverse of the SPD Gram matrix built from its Cholesky factor,
// as DensePositiveDefiniteMatrix.inv does (matrices.py:1161-1188): inv = L^-T (L^-1).
template <int C>
__device__ __forceinline__ void spd_inverse_apply(const double (&G)[C][C], const double (&u)[C],
                                                  double (&x)[C]) {
  double L[C][C];
#pragma unroll
  for (int i = 0; i < C; ++i)
#pragma unroll
    for (int j = 0; j < C; ++j) L[i][j] = 0.0;
#pragma unroll
  for (int j = 0; j < C; ++j) {
    double d = G[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
    d = sqrt(d);
    L[j][j] = d;
#pragma unroll
    for (int i = j + 1; i < C; ++i) {
      double s = G[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k];
      L[i][j] = s / d;
    }
  }
  // Linv = L^-1 (lower), then inv = Linv^T Linv
  double Li[C][C];
#pragma unroll
  for (int j = 0; j < C; ++j) {
#pragma unroll
    for (int i = 0; i < C; ++i) {
      if (i < j) {
        Li[i][j] = 0.0;
      } else {
        double s = (i == j) ? 1.0 : 0.0;
#pragma unroll
        for (int k = 0; k < C; ++k)
          if (k >= j && k < i) s -= L[i][k] * Li[k][j];
        Li[i][j] = s / L[i][i];
      }
    }
  }
#pragma unroll
  for (int i = 0; i < C; ++i) {
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < C; ++j) {
      double a = 0.0;
#pragma unroll
      for (int k = 0; k < C; ++k) a = fma(Li[k][i], Li[k][j], a);
      s = fma(a, u[j], s);
    }
    x[i] = s;
  }
}

// Ginv = explicit inverse of the SPD matrix G (as spd_inverse_apply builds it) and
// half_logdet = sum log L_ii = log det G / 2 (DensePositiveDefiniteMatrix.log_abs_det / 2,
// matrices.py:982-984, systems.py:836-838)
template <int C>
__device__ __forceinline__ void spd_inverse_logdet(const double (&G)[C][C], double (&Ginv)[C][C],
                                                   double& half_logdet) {
  half_logdet = 0.0;
#pragma unroll
  for (int b = 0; b < C; ++b) {
    double u[C], x[C];
#pragma unroll
    for (int a = 0; a < C; ++a) u[a] = (a == b) ? 1.0 : 0.0;
    spd_inverse_apply<C>(G, u, x);
#pragma unroll
    for (int a = 0; a < C; ++a) Ginv[a][b] = x[a];
  }
  // Cholesky diagonal again (cheap for C <= 8)
  double L[C][C];
#pragma unroll
  for (int j = 0; j < C; ++j) {
    double d = G[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
    d = sqrt(d);
    L[j][j] = d;
    half_logdet += log(fabs(d));
#pragma unroll
    for (int i = j + 1; i < C; ++i) {
      double t = G[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) t -= L[i][k] * L[j][k];
      L[i][j] = t / d;
    }
  }
}

// x = R^-1 c by LU with partial pivoting (scipy.linalg.lu_factor / lu_solve:
// matrices.py:1311, 1371-1384)
template <int C>
__device__ __forceinline__ void lu_solve(double (&R)[C][C], const double (&c)[C],
                                         double (&x)[C]) {
  double b[C];
#pragma unroll
  for (int i = 0; i < C; ++i) b[i] = c[i];
#pragma unroll
  for (int k = 0; k < C; ++k) {
    int piv = k;
    double best = fabs(R[k][k]);
#pragma unroll
    for (int i = k + 1; i < C; ++i) {
      const double a = fabs(R[i][k]);
      if (a > best) best = a, piv = i;
    }
#pragma unroll
    for (int i = k + 1; i < C; ++i) {
      if (i == piv) {
#pragma unroll
        for (int j = 0; j < C; ++j) {
          const double t = R[k][j];
          R[k][j] = R[i][j];
          R[i][j] = t;
        }
        const double t = b[k];
        b[k] = b[i];
        b[i] = t;
      }
    }
#pragma unroll
    for (int i = k + 1; i < C; ++i) {
      const double f = R[i][k] / R[k][k];
#pragma unroll
      for (int j = k + 1; j < C; ++j) R[i][j] -= f * R[k][j];
      b[i] -= f * b[k];
    }
  }
#pragma unroll
  for (int i = C - 1; i >= 0; --i) {
    double s = b[i];
#pragma unroll
    for (int j = i + 1; j < C; ++j) s -= R[i][j] * x[j];
    x[i] = s / R[i][i];
  }
}

// Eigendecomposition G = V diag(lam) V^T of a symmetric C x C matrix by cyclic Jacobi rotations
// (every lane redundantly, only the upper triangle of A is read and written).  Stands in for
// numpy.linalg.eigh of DenseSymmetricMatrix (matrices.py:436-438); at C = 1 it returns lam = G,
// V = 1 exactly as LAPACK does.  The eigenvalues come out unsorted; a non-finite entry makes
// every output NaN-contaminated, which the callers' NaN tests turn into a ConvergenceError.
template <int C>
__device__ __forceinline__ void jacobi_eigh(const double (&G)[C][C], double (&lam)[C],
                                            double (&V)[C][C]) {
  double A[C][C];
#pragma unroll
  for (int i = 0; i < C; ++i)
#pragma unroll
    for (int j = 0; j < C; ++j) A[i][j] = G[i][j], V[i][j] = (i == j) ? 1.0 : 0.0;
#pragma unroll 1
  for (int sweep = 0; sweep < 16; ++sweep) {
    double off = 0.0;
#pragma unroll
    for (int i = 0; i < C; ++i)
#pragma unroll
      for (int j = i + 1; j < C; ++j) off = fma(A[i][j], A[i][j], off);
    if (!(off > 0.0)) break;  // diagonal, or NaN
#pragma unroll
    for (int p = 0; p < C; ++p)
#pragma unroll
      for (int q = p + 1; q < C; ++q) {
        const double apq = A[p][q];
        const double g = 100.0 * fabs(apq);
        if (sweep > 3 && fabs(A[p][p]) + g == fabs(A[p][p]) && fabs(A[q][q]) + g == fabs(A[q][q])) {
          A[p][q] = 0.0;  // below the diagonal's resolution (Numerical Recipes' jacobi)
        } else if (apq != 0.0) {
          const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
          const double tn = copysign(1.0, theta) / (fabs(theta) + sqrt(fma(theta, theta, 1.0)));
          const double c = 1.0 / sqrt(fma(tn, tn, 1.0)), s = tn * c;
          A[p][p] -= tn * apq;
          A[q][q] += tn * apq;
          A[p][q] = 0.0;
#pragma unroll
          for (int r = 0; r < C; ++r) {
            if (r == p || r == q) continue;
            double& arp = r < p ? A[r][p] : A[p][r];
            double& arq = r < q ? A[r][q] : A[q][r];
            const double x = arp, y = arq;
            arp = c * x - s * y;
            arq = s * x + c * y;
          }
#pragma unroll
          for (int r = 0; r < C; ++r) {
            const double x = V[r][p], y = V[r][q];
            V[r][p] = c * x - s * y;
            V[r][q] = s * x + c * y;
          }
        }
      }
  }
#pragma unroll
  for (int i = 0; i < C; ++i) lam[i] = A[i][i];
}

// x = G^-1 u with G^-1 = EigendecomposedSymmetricMatrix(V, 1 / lam), the inverse of a
// DenseSymmetricMatrix (matrices.py:1446-1447, 1568-1569): V (diag(1/lam) (V^T u)).
template <int C>
__device__ __forceinline__ void eig_inverse_apply(const double (&lam)[C], const double (&V)[C][C],
                                                  const double (&u)[C], double (&x)[C]) {
  double y[C];
#pragma unroll
  for (int i = 0; i < C; ++i) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < C; ++k) s = fma(V[k][i], u[k], s);
    y[i] = (1.0 / lam[i]) * s;
  }
#pragma unroll
  for (int i = 0; i < C; ++i) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < C; ++k) s = fma(V[i][k], y[k], s);
    x[i] = s;
  }
}

// Per-chain data of the Gaussian split (GaussianEuclideanMetricSystem, systems.py:464-474, and
// dh2_flow_dmom, systems.py:1171-1184): w = 1 / eigval^(1/2) of the metric and sin(w |dt|),
// cos(w |dt|) for the chain's inner step, in the pair layout of the eigen-coordinates.
template <int NV>
struct GaussianRotation {
  double om[NV], sw[NV], cw[NV];
};

template <class Target, int KP, bool GAUSS = false>
struct ConstrainedOps {
  static constexpr int NV = 2 * KP;
  static constexpr int C = Target::NC;

  const Target& t;
  int metric_kind;
  const double* minv;
  int dim, lane;
  double* psm;
  int solver, max_ls;
  // GAUSS only: w and the metric's eigenvectors U (row-major) and U^T (NULL unless dense)
  const double* omega = nullptr;
  const double* eigvec = nullptr;
  const double* eigvec_t = nullptr;
  GaussianRotation<NV> rot = {};

  // sin / cos of w |dt| for this chain (CUDA's sincos; NumPy's sin / cos may differ in the last
  // bit).  Padding coordinates get w = 1 and hold zeros.
  __device__ __forceinline__ void set_rotation(double adt) {
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
      const double om = (i < dim) ? omega[i] : 1.0;
      rot.om[e] = om;
      sincos(om * adt, &rot.sw[e], &rot.cw[e]);
    }
  }
  // R vectors to eigen-coordinates, U^T x (inv_metric_apply forms A^T x, A = U), and back, U y
  // (A = U^T).  Identity and diagonal metrics have U = I and skip the products.
  template <int R>
  __device__ __forceinline__ void to_eig(const double (&a)[R][NV], double (&out)[R][NV]) const {
    inv_metric_apply<KP, R>(metric_kind == MB200_METRIC_DENSE ? MB200_METRIC_DENSE
                                                              : MB200_METRIC_IDENTITY,
                            eigvec, dim, lane, psm, a, out);
  }
  template <int R>
  __device__ __forceinline__ void from_eig(const double (&a)[R][NV], double (&out)[R][NV]) const {
    inv_metric_apply<KP, R>(metric_kind == MB200_METRIC_DENSE ? MB200_METRIC_DENSE
                                                              : MB200_METRIC_IDENTITY,
                            eigvec_t, dim, lane, psm, a, out);
  }

  // h2_flow(dt): q += dt M^-1 p (systems.py:362-363), or for the Gaussian split the exact
  // rotation (systems.py:464-474), rotated in the eigenbasis, then multiplied and added:
  //   q' = U (cos(w dt) U^T q + (sin(w dt) w) U^T p),  p' = U (cos(w dt) U^T p - (sin(w dt)/w) U^T q)
  __device__ __forceinline__ void drift(double (&q)[NV], double (&p)[NV], double dt) const {
    if constexpr (GAUSS) {
      double x[2][NV], y[2][NV];
#pragma unroll
      for (int e = 0; e < NV; ++e) x[0][e] = q[e], x[1][e] = p[e];
      to_eig<2>(x, y);
      const double sgn = dt < 0.0 ? -1.0 : 1.0;  // sin is odd: sin(w dt) = sgn sin(w |dt|)
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        const double sn = sgn * rot.sw[e], cs = rot.cw[e], om = rot.om[e];
        x[0][e] = __dadd_rn(__dmul_rn(cs, y[0][e]), __dmul_rn(__dmul_rn(sn, om), y[1][e]));
        x[1][e] = __dsub_rn(__dmul_rn(cs, y[1][e]), __dmul_rn(__ddiv_rn(sn, om), y[0][e]));
      }
      from_eig<2>(x, y);
#pragma unroll
      for (int e = 0; e < NV; ++e) q[e] = y[0][e], p[e] = y[1][e];
    } else {
      double v[NV];
      inv_metric_vec(p, v);
#pragma unroll
      for (int e = 0; e < NV; ++e) q[e] = __dadd_rn(q[e], __dmul_rn(dt, v[e]));
    }
  }

  // S_a = dh2_flow_pos_dmom(|dt|) Jp_a^T: |dt| M^-1 Jp_a^T (systems.py:794-799), or
  // U (sin(w |dt|) w  .*  U^T Jp_a^T) for the Gaussian split (systems.py:1171-1184)
  __device__ __forceinline__ void flow_rows(const double (&Jp)[C][NV], double adt,
                                            double (&S)[C][NV]) const {
    if constexpr (GAUSS) {
      double y[C][NV];
      to_eig<C>(Jp, y);
#pragma unroll
      for (int a = 0; a < C; ++a)
#pragma unroll
        for (int e = 0; e < NV; ++e) y[a][e] = __dmul_rn(__dmul_rn(rot.sw[e], rot.om[e]), y[a][e]);
      from_eig<C>(y, S);
    } else {
      inv_metric_rows(Jp, S);
#pragma unroll
      for (int a = 0; a < C; ++a)
#pragma unroll
        for (int e = 0; e < NV; ++e) S[a][e] = adt * S[a][e];
    }
  }

  // on convergence: p -= sign(dt) dh2_flow_mom_dmom mu (solvers.py:331, 457, 586), with
  // dh2_flow_mom_dmom = I, or U diag(cos(w |dt|)) U^T for the Gaussian split
  __device__ __forceinline__ void finish(double (&p)[NV], const double (&mu)[NV], double dt) const {
    const double sgn = (dt > 0.0) ? 1.0 : ((dt < 0.0) ? -1.0 : 0.0);
    if constexpr (GAUSS) {
      double x[1][NV], y[1][NV];
#pragma unroll
      for (int e = 0; e < NV; ++e) x[0][e] = mu[e];
      to_eig<1>(x, y);
#pragma unroll
      for (int e = 0; e < NV; ++e) y[0][e] = __dmul_rn(sgn * rot.cw[e], y[0][e]);
      from_eig<1>(y, x);
#pragma unroll
      for (int e = 0; e < NV; ++e) p[e] = __dsub_rn(p[e], x[0][e]);
    } else {
#pragma unroll
      for (int e = 0; e < NV; ++e) p[e] = __dsub_rn(p[e], sgn * mu[e]);
    }
  }

  // Gram-matrix inverse: DensePositiveDefiniteMatrix (Cholesky) for DenseConstrained...System
  // (systems.py:1006-1022), DenseSymmetricMatrix (eigh) for the Gaussian one (:1157-1169)
  __device__ __forceinline__ void gram_solve(const double (&G)[C][C], const double (&u)[C],
                                             double (&x)[C]) const {
    if constexpr (GAUSS) {
      double lam[C], V[C][C];
      jacobi_eigh<C>(G, lam, V);
      eig_inverse_apply<C>(lam, V, u, x);
    } else {
      spd_inverse_apply<C>(G, u, x);
    }
  }
  __device__ __forceinline__ void gram_inverse_logdet(const double (&G)[C][C],
                                                      double (&Ginv)[C][C],
                                                      double& half_logdet) const {
    if constexpr (GAUSS) {
      double lam[C], V[C][C];
      jacobi_eigh<C>(G, lam, V);
      double s = 0.0;  // SymmetricMatrix.log_abs_det (matrices.py:457-459)
#pragma unroll
      for (int i = 0; i < C; ++i) s += log(fabs(lam[i]));
      half_logdet = 0.5 * s;
#pragma unroll
      for (int a = 0; a < C; ++a)
#pragma unroll
        for (int b = 0; b < C; ++b) {
          double v = 0.0;
#pragma unroll
          for (int k = 0; k < C; ++k) v = fma(V[a][k] * (1.0 / lam[k]), V[b][k], v);
          Ginv[a][b] = v;
        }
    } else {
      spd_inverse_logdet<C>(G, Ginv, half_logdet);
    }
  }

  __device__ __forceinline__ void inv_metric_rows(const double (&a)[C][NV],
                                                  double (&out)[C][NV]) const {
    inv_metric_apply<KP, C>(metric_kind, minv, dim, lane, psm, a, out);
  }
  __device__ __forceinline__ void inv_metric_vec(const double (&a)[NV], double (&out)[NV]) const {
    double ai[1][NV], oi[1][NV];
#pragma unroll
    for (int e = 0; e < NV; ++e) ai[0][e] = a[e];
    inv_metric_apply<KP, 1>(metric_kind, minv, dim, lane, psm, ai, oi);
#pragma unroll
    for (int e = 0; e < NV; ++e) out[e] = oi[0][e];
  }
  static __device__ __forceinline__ double dot(const double (&a)[NV], const double (&b)[NV]) {
    double s = 0.0;
#pragma unroll
    for (int e = 0; e < NV; ++e) s = fma(a[e], b[e], s);
    return warp_sum(s);
  }
  static __device__ __forceinline__ double maxabs(const double (&a)[NV]) {
    double m = 0.0;
#pragma unroll
    for (int e = 0; e < NV; ++e) m = nanmax(m, fabs(a[e]));
    return warp_nanmax(m);
  }

  // dh1_dpos (systems.py:858-861): grad l, plus -- for a density given with respect to the
  // Lebesgue measure (dens_wrt_hausdorff=False) -- grad_log_det_sqrt_gram =
  // mhp_constr(inv_gram @ J @ M^-1) (systems.py:1024-1031).  Returns log det gram / 2 in *ldsg.
  __device__ __forceinline__ void dh1(const double (&q)[NV], double (&g)[NV], bool lebesgue,
                                      double* ldsg = nullptr) const {
    t.grad(lane, dim, q, g);
    if (!lebesgue) return;
    double c[C], J[C][NV], W[C][NV], G[C][C], Ginv[C][C], m[C][NV], extra[NV], hl;
    t.constr_jacob(lane, dim, q, c, J);
    inv_metric_rows(J, W);  // rows of J M^-1 (M symmetric)
#pragma unroll
    for (int a = 0; a < C; ++a)
#pragma unroll
      for (int b = 0; b < C; ++b) G[a][b] = dot(J[a], W[b]);
    gram_inverse_logdet(G, Ginv, hl);
#pragma unroll
    for (int a = 0; a < C; ++a)
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        double v = 0.0;
#pragma unroll
        for (int b = 0; b < C; ++b) v = fma(Ginv[a][b], W[b][e], v);
        m[a][e] = v;
      }
    t.mhp(lane, dim, q, m, extra);
#pragma unroll
    for (int e = 0; e < NV; ++e) g[e] = __dadd_rn(g[e], extra[e]);
    if (ldsg != nullptr) *ldsg = hl;
  }

  // p <- p - J^T (J M^-1 J^T)^-1 J M^-1 p     (systems.py:863-873)
  __device__ __forceinline__ void project(double (&p)[NV], const double (&q)[NV]) const {
    double c[C], J[C][NV], W[C][NV], G[C][C], u[C], w[C], v[NV];
    t.constr_jacob(lane, dim, q, c, J);
    inv_metric_rows(J, W);  // W_d = M^-1 J_d^T
#pragma unroll
    for (int a = 0; a < C; ++a)
#pragma unroll
      for (int b = 0; b < C; ++b) G[a][b] = dot(J[a], W[b]);
    inv_metric_vec(p, v);
#pragma unroll
    for (int a = 0; a < C; ++a) u[a] = dot(J[a], v);
    gram_solve(G, u, w);
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      double s = 0.0;
#pragma unroll
      for (int a = 0; a < C; ++a) s = fma(J[a][e], w[a], s);
      p[e] = __dsub_rn(p[e], s);
    }
  }

  // h2_flow then Newton retraction onto the manifold (integrators.py:929-942,
  // solvers.py:346-469).  Returns false on ConvergenceError.
  __device__ __forceinline__ bool retract_newton(double (&q)[NV], double (&p)[NV],
                                          const double (&q_prev)[NV], double dt,
                                          double constraint_tol, double position_tol,
                                          double divergence_tol, int max_iters,
                                          int& iters) const {
    drift(q, p, dt);
    double mu[NV];
#pragma unroll
    for (int e = 0; e < NV; ++e) mu[e] = 0.0;
    double cp[C], Jp[C][NV], S[C][NV];
    t.constr_jacob(lane, dim, q_prev, cp, Jp);
    const double adt = fabs(dt);
    flow_rows(Jp, adt, S);  // S_a = |dt| M^-1 Jp_a^T
    for (int i = 0; i < max_iters; ++i) {
      double c[C], J[C][NV], R[C][C], x[C];
      t.constr_jacob(lane, dim, q, c, J);
      double err = 0.0;
#pragma unroll
      for (int a = 0; a < C; ++a) err = nanmax(err, fabs(c[a]));
#pragma unroll
      for (int a = 0; a < C; ++a)
#pragma unroll
        for (int b = 0; b < C; ++b) R[a][b] = dot(J[a], S[b]);
      lu_solve<C>(R, c, x);
      double dmu[NV], dpos[NV];
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        double s = 0.0, d = 0.0;
#pragma unroll
        for (int a = 0; a < C; ++a) s = fma(Jp[a][e], x[a], s), d = fma(S[a][e], x[a], d);
        dmu[e] = s;
        dpos[e] = d;
      }
      ++iters;
      if (err > divergence_tol || err != err) return false;
      if (err < constraint_tol && maxabs(dpos) < position_tol) {
        finish(p, mu, dt);
        return true;
      }
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        mu[e] = __dadd_rn(mu[e], dmu[e]);
        q[e] = __dsub_rn(q[e], dpos[e]);
      }
    }
    return false;
  }

  // solve_projection_onto_manifold_quasi_newton (solvers.py:195-343): the residual Jacobian is
  // frozen at the previous state, J_prev (|dt| M^-1) J_prev^T (an SPD Gram matrix whose explicit
  // inverse is built once from its Cholesky factor, systems.py:1013-1016, matrices.py:1161-1188).
  __device__ __forceinline__ bool retract_quasi_newton(double (&q)[NV], double (&p)[NV],
                                                       const double (&q_prev)[NV], double dt,
                                                       double constraint_tol, double position_tol,
                                                       double divergence_tol, int max_iters,
                                                       int& iters) const {
    drift(q, p, dt);
    double mu[NV];
#pragma unroll
    for (int e = 0; e < NV; ++e) mu[e] = 0.0;
    double cp[C], Jp[C][NV], S[C][NV], G[C][C];
    t.constr_jacob(lane, dim, q_prev, cp, Jp);
    const double adt = fabs(dt);
    flow_rows(Jp, adt, S);
#pragma unroll
    for (int a = 0; a < C; ++a)
#pragma unroll
      for (int b = 0; b < C; ++b) G[a][b] = dot(Jp[a], S[b]);
    // the Gaussian split's eigendecomposition of G, once per solve like the reference's `.inv`
    double lam[C], V[C][C];
    if constexpr (GAUSS) jacobi_eigh<C>(G, lam, V);
    for (int i = 0; i < max_iters; ++i) {
      double c[C], J[C][NV], x[C];
      t.constr_jacob(lane, dim, q, c, J);  // (only c is used: the Jacobian stays frozen)
      double err = 0.0;
#pragma unroll
      for (int a = 0; a < C; ++a) err = nanmax(err, fabs(c[a]));
      if constexpr (GAUSS)
        eig_inverse_apply<C>(lam, V, c, x);
      else
        spd_inverse_apply<C>(G, c, x);
      double dmu[NV], dpos[NV];
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        double s = 0.0, d = 0.0;
#pragma unroll
        for (int a = 0; a < C; ++a) s = fma(Jp[a][e], x[a], s), d = fma(S[a][e], x[a], d);
        dmu[e] = s;
        dpos[e] = d;
      }
      ++iters;
      if (err > divergence_tol || err != err) return false;
      if (err < constraint_tol && maxabs(dpos) < position_tol) {
        finish(p, mu, dt);
        return true;
      }
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        mu[e] = __dadd_rn(mu[e], dmu[e]);
        q[e] = __dsub_rn(q[e], dpos[e]);
      }
    }
    return false;
  }

  // solve_projection_onto_manifold_newton_with_line_search (solvers.py:472-614): full Newton
  // direction, step halved (at most max_ls times) until |c| decreases.  The reference's order of
  // tests is kept: divergence only from the second iteration (:574), convergence tested before
  // the update with the previous iteration's step (:580-584), and after an unsuccessful line
  // search the position stays at the last trial step while mu advances by the halved one
  // (:597-604).
  __device__ __forceinline__ bool retract_newton_line_search(
      double (&q)[NV], double (&p)[NV], const double (&q_prev)[NV], double dt,
      double constraint_tol, double position_tol, double divergence_tol, int max_iters,
      int max_ls, int& iters) const {
    drift(q, p, dt);
    double mu[NV], dpos[NV];
#pragma unroll
    for (int e = 0; e < NV; ++e) mu[e] = 0.0, dpos[e] = 0.0;
    double cp[C], Jp[C][NV], S[C][NV];
    t.constr_jacob(lane, dim, q_prev, cp, Jp);
    const double adt = fabs(dt);
    flow_rows(Jp, adt, S);
    double step = 1.0;
    for (int i = 0; i < max_iters; ++i) {
      double c[C], J[C][NV], R[C][C], x[C];
      t.constr_jacob(lane, dim, q, c, J);
      double err = 0.0;
#pragma unroll
      for (int a = 0; a < C; ++a) err = nanmax(err, fabs(c[a]));
      ++iters;
      if (i > 0 && (err > divergence_tol || err != err)) return false;
      double sd[NV];
#pragma unroll
      for (int e = 0; e < NV; ++e) sd[e] = step * dpos[e];
      if (err < constraint_tol && (i == 0 || maxabs(sd) < position_tol)) {
        finish(p, mu, dt);
        return true;
      }
#pragma unroll
      for (int a = 0; a < C; ++a)
#pragma unroll
        for (int b = 0; b < C; ++b) R[a][b] = dot(J[a], S[b]);
      lu_solve<C>(R, c, x);
      double dmu[NV], qc[NV];
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        double s = 0.0, d = 0.0;
#pragma unroll
        for (int a = 0; a < C; ++a) s = fma(Jp[a][e], x[a], s), d = fma(S[a][e], x[a], d);
        dmu[e] = s;
        dpos[e] = -d;
        qc[e] = q[e];
      }
      step = 1.0;
      for (int l = 0; l < max_ls; ++l) {
#pragma unroll
        for (int e = 0; e < NV; ++e) q[e] = __dadd_rn(qc[e], __dmul_rn(step, dpos[e]));
        double c2[C], J2[C][NV];
        t.constr_jacob(lane, dim, q, c2, J2);
        double e2 = 0.0;
#pragma unroll
        for (int a = 0; a < C; ++a) e2 = nanmax(e2, fabs(c2[a]));
        if (e2 < err) break;
        step *= 0.5;
      }
#pragma unroll
      for (int e = 0; e < NV; ++e) mu[e] = __dadd_rn(mu[e], __dmul_rn(step, dmu[e]));
    }
    return false;
  }

  // projection solver selected by the integrator (integrators.py:862; MB200_PROJ_SOLVER_*)
  __device__ __forceinline__ bool retract(double (&q)[NV], double (&p)[NV],
                                          const double (&q_prev)[NV], double dt,
                                          double constraint_tol, double position_tol,
                                          double divergence_tol, int max_iters,
                                          int& iters) const {
    if (solver == MB200_PROJ_SOLVER_QUASI_NEWTON)
      return retract_quasi_newton(q, p, q_prev, dt, constraint_tol, position_tol, divergence_tol,
                                  max_iters, iters);
    if (solver == MB200_PROJ_SOLVER_NEWTON_LINE_SEARCH)
      return retract_newton_line_search(q, p, q_prev, dt, constraint_tol, position_tol,
                                        divergence_tol, max_iters, max_ls, iters);
    return retract_newton(q, p, q_prev, dt, constraint_tol, position_tol, divergence_tol,
                          max_iters, iters);
  }
};

// Shared-memory doubles per warp: the rows staged by the dense metric product (C of them; the
// Gaussian split also rotates q and p together)
__host__ __device__ constexpr int constrained_smem_doubles(int c, int kp, bool gauss) {
  return (c > 1 ? c : (gauss ? 2 : 1)) * 64 * kp;
}
template <int C, int KP, bool GAUSS>
__host__ __device__ constexpr int constrained_smem_per_warp() {
  return constrained_smem_doubles(C, KP, GAUSS);
}

// A user-written constraint (user_constraint.cuh) declares STAGED = true: it sees whole vectors
// and stages each chain's q, NC rows of J (or of the matrix-Hessian product's operand) and one
// output vector through per-warp shared memory of its own, after the metric product's.  Registry
// targets declare nothing and get nothing.
template <class T>
__host__ __device__ constexpr auto cs_staged(int) -> decltype(T::STAGED) {
  return T::STAGED;
}
template <class T>
__host__ __device__ constexpr bool cs_staged(long) {
  return false;
}
__host__ __device__ constexpr int user_constraint_stage_per_warp(int nc, int kp) {
  return (nc + 2) * 64 * kp;
}
template <class Target, int KP, bool GAUSS>
__host__ __device__ constexpr int cs_smem_per_warp() {
  return constrained_smem_per_warp<Target::NC, KP, GAUSS>() +
         (cs_staged<Target>(0) ? user_constraint_stage_per_warp(Target::NC, KP) : 0);
}
// The kernel's target; a staged one gets its area, behind the metric product's in `warp_smem`
template <class Target, int KP, bool GAUSS>
__device__ __forceinline__ Target cs_target(const ModelArgs& m, int dim, double* warp_smem) {
  if constexpr (cs_staged<Target>(0))
    return Target(m, dim, warp_smem + constrained_smem_per_warp<Target::NC, KP, GAUSS>());
  else
    return Target(m, dim);
}

// GAUSS selects the flow policy of GaussianDenseConstrainedEuclideanMetricSystem
// (systems.py:1034-1184): the h2 drift is the exact rotation, the solvers use
// dh2_flow_dmom = (U diag(sin(w|dt|) w) U^T, U diag(cos(w|dt|)) U^T), the Gram matrices are
// inverted through their eigendecomposition, h2 carries q.q/2 and the density is always with
// respect to the Lebesgue measure.  omega / eigvec / eigvec_t are read only when GAUSS.
template <class Target, int KP, bool GAUSS = false>
__global__ void __launch_bounds__(128)
    constrained_leapfrog_kernel(const double* q_in, const double* p_in, double* q_out,
                                double* p_out, const int32_t* __restrict__ dir, int64_t n_chains,
                                int dim, double step_size, int n_steps, int n_inner,
                                int metric_kind, const double* __restrict__ minv, ModelArgs model,
                                double constraint_tol, double position_tol, double divergence_tol,
                                int max_iters, double rev_tol, double* __restrict__ h_out,
                                int32_t* __restrict__ status, int32_t* __restrict__ n_done,
                                int32_t* __restrict__ newton_iters, int proj_solver,
                                int max_line_search_iters, const double* __restrict__ omega,
                                const double* __restrict__ eigvec,
                                const double* __restrict__ eigvec_t) {
  constexpr int NV = 2 * KP;
  constexpr int SM_PER_WARP = cs_smem_per_warp<Target, KP, GAUSS>();
  extern __shared__ double smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const Target target =
      cs_target<Target, KP, GAUSS>(model, dim, smem + (size_t)warp * SM_PER_WARP);
  ConstrainedOps<Target, KP, GAUSS> ops{target,      metric_kind,
                                        minv,        dim,
                                        lane,        smem + (size_t)warp * SM_PER_WARP,
                                        proj_solver, max_line_search_iters,
                                        omega,       eigvec,
                                        eigvec_t};
  const bool even = (dim & 1) == 0;

  for (int64_t ch = (int64_t)blockIdx.x * wpb + warp; ch < n_chains;
       ch += (int64_t)gridDim.x * wpb) {
    double q[NV], p[NV], g[NV];
    const double eps = model.step_sizes != nullptr ? model.step_sizes[ch] : step_size;
    const double dt = (dir != nullptr) ? (double)dir[ch] * eps : eps;
    const int ns = model.n_steps_pc != nullptr ? min(model.n_steps_pc[ch], n_steps) : n_steps;
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int i = 2 * lane + 64 * k;
      double q0 = 0, q1 = 0, p0 = 0, p1 = 0;
      if (i < dim) {
        const size_t o = (size_t)ch * dim + i;
        if (even) {
          const double2 a = *reinterpret_cast<const double2*>(q_in + o);
          const double2 b = *reinterpret_cast<const double2*>(p_in + o);
          q0 = a.x, q1 = a.y, p0 = b.x, p1 = b.y;
        } else {
          q0 = q_in[o], p0 = p_in[o];
          if (i + 1 < dim) q1 = q_in[o + 1], p1 = p_in[o + 1];
        }
      }
      q[2 * k] = q0, q[2 * k + 1] = q1, p[2 * k] = p0, p[2 * k + 1] = p1;
    }
    // dens_wrt_hausdorff=False
    const bool lebesgue = GAUSS || model.tp[MB200_MAX_PARAMS - 1] != 0.0;
    ops.dh1(q, g, lebesgue);
    int st = MB200_STATUS_OK, done = 0, iters = 0;
    // constraint-Jacobian evaluations: one per projection, one per retraction (at the previous
    // position) plus one per Newton iteration, one per Lebesgue-density gradient
    int n_proj = 0, n_retr = 0;
    const double dt_inner = dt / n_inner;
    if constexpr (GAUSS) ops.set_rotation(fabs(dt_inner));
    for (int s = 0; s < ns && st == MB200_STATUS_OK; ++s) {
      double qs[NV], ps[NV];
#pragma unroll
      for (int e = 0; e < NV; ++e) qs[e] = q[e], ps[e] = p[e];
      // _step_a(dt/2)
#pragma unroll
      for (int e = 0; e < NV; ++e) p[e] = __dsub_rn(p[e], __dmul_rn(0.5 * dt, g[e]));
      ops.project(p, q);
      ++n_proj;
      // _step_b(dt)
      for (int i = 0; i < n_inner && st == MB200_STATUS_OK; ++i) {
        double qprev[NV];
#pragma unroll
        for (int e = 0; e < NV; ++e) qprev[e] = q[e];
        ++n_retr;
        if (!ops.retract(q, p, qprev, dt_inner, constraint_tol, position_tol, divergence_tol,
                         max_iters, iters)) {
          st = MB200_STATUS_CONVERGENCE;
          break;
        }
        ops.project(p, q);
        ++n_proj, ++n_retr;
        double qb[NV], pb[NV];
#pragma unroll
        for (int e = 0; e < NV; ++e) qb[e] = q[e], pb[e] = p[e];
        if (!ops.retract(qb, pb, q, -dt_inner, constraint_tol, position_tol, divergence_tol,
                         max_iters, iters)) {
          st = MB200_STATUS_CONVERGENCE;
          break;
        }
        double diff[NV];
#pragma unroll
        for (int e = 0; e < NV; ++e) diff[e] = qb[e] - qprev[e];
        const double rev = ConstrainedOps<Target, KP>::maxabs(diff);
        if (rev > rev_tol) st = MB200_STATUS_NON_REVERSIBLE;
      }
      if (st == MB200_STATUS_OK) {
        // _step_a(dt/2)
        ops.dh1(q, g, lebesgue);
#pragma unroll
        for (int e = 0; e < NV; ++e) p[e] = __dsub_rn(p[e], __dmul_rn(0.5 * dt, g[e]));
        ops.project(p, q);
        ++n_proj;
        ++done;
      } else {
#pragma unroll
        for (int e = 0; e < NV; ++e) q[e] = qs[e], p[e] = ps[e];
      }
    }
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int i = 2 * lane + 64 * k;
      if (i < dim) {
        const size_t o = (size_t)ch * dim + i;
        if (even) {
          *reinterpret_cast<double2*>(q_out + o) = make_double2(q[2 * k], q[2 * k + 1]);
          *reinterpret_cast<double2*>(p_out + o) = make_double2(p[2 * k], p[2 * k + 1]);
        } else {
          q_out[o] = q[2 * k], p_out[o] = p[2 * k];
          if (i + 1 < dim) q_out[o + 1] = q[2 * k + 1], p_out[o + 1] = p[2 * k + 1];
        }
      }
    }
    if (h_out != nullptr) {
      double v[NV];
      ops.inv_metric_vec(p, v);
      const double kin = ConstrainedOps<Target, KP>::dot(p, v);
      double l = target.nld(lane, dim, q);
      if (lebesgue) {  // h1 = l + log det gram / 2 (systems.py:853-856)
        double gtmp[NV], ldsg = 0.0;
        ops.dh1(q, gtmp, true, &ldsg);
        l += ldsg;
      }
      if constexpr (GAUSS) {  // h1 + (q.q/2 + p.M^-1 p/2) (systems.py:451-454)
        const double qq = ConstrainedOps<Target, KP>::dot(q, q);
        if (lane == 0) h_out[ch] = l + (0.5 * qq + 0.5 * kin);
      } else {
        if (lane == 0) h_out[ch] = l + 0.5 * kin;
      }
    }
    if (lane == 0) {
      if (status != nullptr) status[ch] = st;
      if (n_done != nullptr) n_done[ch] = done;
      if (newton_iters != nullptr) newton_iters[ch] = iters;
      if (model.counters != nullptr) {
        int32_t* cnt = model.counters + ch * MB200_N_COUNTERS;
        cnt[MB200_COUNT_GRAD] += 1 + done;
        cnt[MB200_COUNT_METRIC] += n_proj + n_retr + iters + (lebesgue ? 1 + done : 0);
        cnt[MB200_COUNT_SOLVER_ITERS] += iters;
      }
    }
  }
}

// Projection of momenta onto the cotangent space of the constraint manifold for all chains:
// ConstrainedTractableFlowSystem.sample_momentum (systems.py:613-616) draws from N(0, M) and
// then applies project_onto_cotangent_space (systems.py:863-873); this is that second half.
// GAUSS: the Gram matrix is inverted through its eigendecomposition (systems.py:1157-1169).
template <class Target, int KP, bool GAUSS = false>
__global__ void __launch_bounds__(128)
    constrained_project_kernel(const double* __restrict__ q_in, const double* p_in, double* p_out,
                               int64_t n_chains, int dim, int metric_kind,
                               const double* __restrict__ minv, ModelArgs model) {
  constexpr int NV = 2 * KP;
  constexpr int SM_PER_WARP = cs_smem_per_warp<Target, KP, GAUSS>();
  extern __shared__ double smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const Target target =
      cs_target<Target, KP, GAUSS>(model, dim, smem + (size_t)warp * SM_PER_WARP);
  const ConstrainedOps<Target, KP, GAUSS> ops{target, metric_kind, minv, dim, lane,
                                              smem + (size_t)warp * SM_PER_WARP, 0, 0};
  for (int64_t ch = (int64_t)blockIdx.x * wpb + warp; ch < n_chains;
       ch += (int64_t)gridDim.x * wpb) {
    double q[NV], p[NV];
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
      q[e] = (i < dim) ? q_in[(size_t)ch * dim + i] : 0.0;
      p[e] = (i < dim) ? p_in[(size_t)ch * dim + i] : 0.0;
    }
    ops.project(p, q);
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
      if (i < dim) p_out[(size_t)ch * dim + i] = p[e];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// K6t: the torus configuration (C3: D = 3, one constraint, identity metric, Newton projection,
// density with respect to the Hausdorff measure) with ONE THREAD per chain.
//
// The warp-per-chain kernel above keeps 3 coordinates in 2 of a warp's 32 lanes and spends most of
// its instructions on warp reductions of two values; with D = 3 the whole chain state fits in a
// thread's registers and every reduction is a handful of scalar operations.  The arithmetic below
// follows the warp kernel operation for operation (same fma / add association as its lane
// layout produces: lane 0 holds x, y, lane 1 holds z), so both kernels agree bit for bit.
// ---------------------------------------------------------------------------------------------
struct Vec3 {
  double x, y, z;
};

struct TorusThread {
  double R, r, alpha;
  __device__ __forceinline__ static double dot(const Vec3& a, const Vec3& b) {
    const double s0 = fma(a.y, b.y, fma(a.x, b.x, 0.0));
    const double s1 = fma(a.z, b.z, 0.0);
    return s0 + s1;
  }
  __device__ __forceinline__ static double maxabs(const Vec3& a) {
    const double m0 = nanmax(nanmax(0.0, fabs(a.x)), fabs(a.y));
    const double m1 = nanmax(nanmax(0.0, fabs(a.z)), 0.0);
    return nanmax(m0, m1);
  }
  __device__ __forceinline__ Vec3 grad(const Vec3& q) const {
    const double x = q.x, y = q.y, z = q.z;
    const double a = r / R;
    const double rho2 = x * x + y * y;
    const double rho = sqrt(rho2);
    const double u = rho - R;
    const double theta = atan2(y, x);
    const double phi = atan2(z, u);
    double s4, c4, sp, cp;
    sincos(4.0 * theta, &s4, &c4);
    sincos(phi, &sp, &cp);
    const double d1 = 1.0 + a * cp;
    const double d2 = 1.0 + alpha * s4 * cp;
    const double dl_dphi = -a * sp / d1 + alpha * s4 * sp / d2;
    const double dl_dth = -4.0 * alpha * c4 * cp / d2;
    const double w = u * u + z * z;
    const double dphi_du = -z / w;
    const double dphi_dz = u / w;
    Vec3 g;
    g.x = dl_dth * (-y / rho2) + dl_dphi * dphi_du * (x / rho);
    g.y = dl_dth * (x / rho2) + dl_dphi * dphi_du * (y / rho);
    g.z = dl_dphi * dphi_dz;
    return g;
  }
  __device__ __forceinline__ double nld(const Vec3& q) const {
    const double rho = sqrt(q.x * q.x + q.y * q.y);
    const double theta = atan2(q.y, q.x);
    const double phi = atan2(q.z, rho - R);
    return log1p(r * cos(phi) / R) - log1p(sin(4.0 * theta) * cos(phi) * alpha);
  }
  __device__ __forceinline__ void constr_jacob(const Vec3& q, double& c, Vec3& J) const {
    const double rho = sqrt(q.x * q.x + q.y * q.y);
    const double d = rho - R;
    c = d * d + q.z * q.z - r * r;
    const double f = 2.0 * d / rho;
    J.x = f * q.x, J.y = f * q.y, J.z = 2.0 * q.z;
  }
  // p <- p - J^T (J J^T)^-1 J p  (identity metric; spd_inverse_apply<1> spelled out)
  __device__ __forceinline__ void project(Vec3& p, const Vec3& q) const {
    double c;
    Vec3 J;
    constr_jacob(q, c, J);
    const double G = dot(J, J);
    const double u = dot(J, p);
    const double L = sqrt(G);
    const double Li = 1.0 / L;
    const double a = fma(Li, Li, 0.0);
    const double w = fma(a, u, 0.0);
    p.x = __dsub_rn(p.x, fma(J.x, w, 0.0));
    p.y = __dsub_rn(p.y, fma(J.y, w, 0.0));
    p.z = __dsub_rn(p.z, fma(J.z, w, 0.0));
  }
  // h2_flow then Newton retraction (solvers.py:346-469), as ConstrainedOps::retract_newton
  __device__ __forceinline__ bool retract(Vec3& q, Vec3& p, const Vec3& q_prev, double dt,
                                          double ctol, double ptol, double dtol, int max_iters,
                                          int& iters) const {
    q.x = __dadd_rn(q.x, __dmul_rn(dt, p.x));
    q.y = __dadd_rn(q.y, __dmul_rn(dt, p.y));
    q.z = __dadd_rn(q.z, __dmul_rn(dt, p.z));
    Vec3 mu = {0.0, 0.0, 0.0}, Jp, S;
    double cp;
    constr_jacob(q_prev, cp, Jp);
    const double adt = fabs(dt);
    S.x = adt * Jp.x, S.y = adt * Jp.y, S.z = adt * Jp.z;
    for (int i = 0; i < max_iters; ++i) {
      double c;
      Vec3 J;
      constr_jacob(q, c, J);
      const double err = nanmax(0.0, fabs(c));
      const double Rm = dot(J, S);
      const double xs = c / Rm;  // lu_solve<1>
      Vec3 dmu, dpos;
      dmu.x = fma(Jp.x, xs, 0.0), dmu.y = fma(Jp.y, xs, 0.0), dmu.z = fma(Jp.z, xs, 0.0);
      dpos.x = fma(S.x, xs, 0.0), dpos.y = fma(S.y, xs, 0.0), dpos.z = fma(S.z, xs, 0.0);
      ++iters;
      if (err > dtol || err != err) return false;
      if (err < ctol && maxabs(dpos) < ptol) {
        const double sgn = (dt > 0.0) ? 1.0 : ((dt < 0.0) ? -1.0 : 0.0);
        p.x = __dsub_rn(p.x, sgn * mu.x);
        p.y = __dsub_rn(p.y, sgn * mu.y);
        p.z = __dsub_rn(p.z, sgn * mu.z);
        return true;
      }
      mu.x = __dadd_rn(mu.x, dmu.x), mu.y = __dadd_rn(mu.y, dmu.y), mu.z = __dadd_rn(mu.z, dmu.z);
      q.x = __dsub_rn(q.x, dpos.x), q.y = __dsub_rn(q.y, dpos.y), q.z = __dsub_rn(q.z, dpos.z);
    }
    return false;
  }
};

__global__ void __launch_bounds__(32)
    constrained_torus_thread_kernel(const double* q_in, const double* p_in, double* q_out,
                                    double* p_out, const int32_t* __restrict__ dir,
                                    int64_t n_chains, double step_size, int n_steps, int n_inner,
                                    ModelArgs model, double constraint_tol, double position_tol,
                                    double divergence_tol, int max_iters, double rev_tol,
                                    double* __restrict__ h_out, int32_t* __restrict__ status,
                                    int32_t* __restrict__ n_done,
                                    int32_t* __restrict__ newton_iters, int lanes) {
  const TorusThread t{model.tp[0], model.tp[1], model.tp[2]};
  if ((int)threadIdx.x >= lanes) return;
  for (int64_t ch = (int64_t)blockIdx.x * lanes + threadIdx.x; ch < n_chains;
       ch += (int64_t)gridDim.x * lanes) {
    Vec3 q = {q_in[ch * 3], q_in[ch * 3 + 1], q_in[ch * 3 + 2]};
    Vec3 p = {p_in[ch * 3], p_in[ch * 3 + 1], p_in[ch * 3 + 2]};
    const double eps = model.step_sizes != nullptr ? model.step_sizes[ch] : step_size;
    const double dt = (dir != nullptr) ? (double)dir[ch] * eps : eps;
    const int ns = model.n_steps_pc != nullptr ? min(model.n_steps_pc[ch], n_steps) : n_steps;
    Vec3 g = t.grad(q);
    int st = MB200_STATUS_OK, done = 0, iters = 0, n_proj = 0, n_retr = 0;
    const double dt_inner = dt / n_inner;
    for (int s = 0; s < ns && st == MB200_STATUS_OK; ++s) {
      const Vec3 qs = q, ps = p;
      p.x = __dsub_rn(p.x, __dmul_rn(0.5 * dt, g.x));
      p.y = __dsub_rn(p.y, __dmul_rn(0.5 * dt, g.y));
      p.z = __dsub_rn(p.z, __dmul_rn(0.5 * dt, g.z));
      t.project(p, q);
      ++n_proj;
      for (int i = 0; i < n_inner && st == MB200_STATUS_OK; ++i) {
        const Vec3 qprev = q;
        ++n_retr;
        if (!t.retract(q, p, qprev, dt_inner, constraint_tol, position_tol, divergence_tol,
                       max_iters, iters)) {
          st = MB200_STATUS_CONVERGENCE;
          break;
        }
        t.project(p, q);
        ++n_proj, ++n_retr;
        Vec3 qb = q, pb = p;
        if (!t.retract(qb, pb, q, -dt_inner, constraint_tol, position_tol, divergence_tol,
                       max_iters, iters)) {
          st = MB200_STATUS_CONVERGENCE;
          break;
        }
        const Vec3 diff = {qb.x - qprev.x, qb.y - qprev.y, qb.z - qprev.z};
        if (TorusThread::maxabs(diff) > rev_tol) st = MB200_STATUS_NON_REVERSIBLE;
      }
      if (st == MB200_STATUS_OK) {
        g = t.grad(q);
        p.x = __dsub_rn(p.x, __dmul_rn(0.5 * dt, g.x));
        p.y = __dsub_rn(p.y, __dmul_rn(0.5 * dt, g.y));
        p.z = __dsub_rn(p.z, __dmul_rn(0.5 * dt, g.z));
        t.project(p, q);
        ++n_proj;
        ++done;
      } else {
        q = qs, p = ps;
      }
    }
    q_out[ch * 3] = q.x, q_out[ch * 3 + 1] = q.y, q_out[ch * 3 + 2] = q.z;
    p_out[ch * 3] = p.x, p_out[ch * 3 + 1] = p.y, p_out[ch * 3 + 2] = p.z;
    if (h_out != nullptr) h_out[ch] = t.nld(q) + 0.5 * TorusThread::dot(p, p);
    if (status != nullptr) status[ch] = st;
    if (n_done != nullptr) n_done[ch] = done;
    if (newton_iters != nullptr) newton_iters[ch] = iters;
    if (model.counters != nullptr) {
      int32_t* cnt = model.counters + ch * MB200_N_COUNTERS;
      cnt[MB200_COUNT_GRAD] += 1 + done;
      cnt[MB200_COUNT_METRIC] += n_proj + n_retr + iters;
      cnt[MB200_COUNT_SOLVER_ITERS] += iters;
    }
  }
}

}  // namespace mb200
