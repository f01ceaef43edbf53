"""User-written constraints of the user-constraint tests (``CudaTarget(..., n_constr=...)``): the
registry's constrained targets rewritten as user sources (``csrc/user_constraint.cuh``), and
models the registry cannot express, with the NumPy statements of the same models that the
reference is run with to make the ``uc_*`` fixtures (tests/make_user_constraint_golden.py)."""

import numpy as np


def CudaTarget(*args, **kwargs):  # noqa: N802
    from mici_b200.targets import CudaTarget as cls  # noqa: PLC0415

    return cls(*args, **kwargs)


# l = |q|^2/2 + q[0] (the sphere and multi-sphere targets share it)
_NLD_SQUARE_PLUS_FIRST = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) s += c.q[i] * c.q[i];
  return 0.5 * c.sum(s) + c.q[0];
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  for (int i = c.lane; i < c.dim; i += 32) g[i] = c.q[i] + (i == 0 ? 1.0 : 0.0);
}
"""

# unit sphere c = |q|^2 - 1, Hessian 2 I
SPHERE = _NLD_SQUARE_PLUS_FIRST + r"""
__device__ void constr(const mb200::Chain& c, double* out) {
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) s += c.q[i] * c.q[i];
  s = c.sum(s);
  if (c.lane == 0) out[0] = s - 1.0;
}
__device__ void jacob_constr(const mb200::Chain& c, double* J) {
  for (int i = c.lane; i < c.dim; i += 32) J[i] = 2.0 * c.q[i];
}
__device__ void mhp_constr(const mb200::Chain& c, const double* m, double* out) {
  for (int i = c.lane; i < c.dim; i += 32) out[i] = 2.0 * m[i];
}
"""

# N_CONSTR unit spheres on consecutive blocks of dim / N_CONSTR coordinates
MULTI_SPHERE = _NLD_SQUARE_PLUS_FIRST + r"""
__device__ void constr(const mb200::Chain& c, double* out) {
  const int block = c.dim / mb200::N_CONSTR;
  for (int k = 0; k < mb200::N_CONSTR; ++k) {
    double s = 0.0;
    for (int i = k * block + c.lane; i < (k + 1) * block; i += 32) s += c.q[i] * c.q[i];
    s = c.sum(s);
    if (c.lane == 0) out[k] = s - 1.0;
  }
}
__device__ void jacob_constr(const mb200::Chain& c, double* J) {
  const int block = c.dim / mb200::N_CONSTR;
  for (int k = 0; k < mb200::N_CONSTR; ++k)
    for (int i = c.lane; i < c.dim; i += 32) J[k * c.dim + i] = i / block == k ? 2.0 * c.q[i] : 0.0;
}
__device__ void mhp_constr(const mb200::Chain& c, const double* m, double* out) {
  const int block = c.dim / mb200::N_CONSTR;
  for (int i = c.lane; i < c.dim; i += 32) out[i] = 2.0 * m[(i / block) * c.dim + i];
}
"""

# torus in R^3, params (R, r, alpha):  rho = sqrt(x^2 + y^2), theta = atan2(y, x),
# phi = atan2(z, rho - R);  l = log1p(r cos(phi) / R) - log1p(alpha sin(4 theta) cos(phi));
# c = (rho - R)^2 + z^2 - r^2.  Every lane computes the three coordinates.
TORUS = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const double R = c.params[0], r = c.params[1], alpha = c.params[2];
  const double x = c.q[0], y = c.q[1], z = c.q[2];
  const double rho = sqrt(x * x + y * y);
  const double theta = atan2(y, x), phi = atan2(z, rho - R);
  return log1p(r * cos(phi) / R) - log1p(sin(4.0 * theta) * cos(phi) * alpha);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const double R = c.params[0], r = c.params[1], alpha = c.params[2];
  const double x = c.q[0], y = c.q[1], z = c.q[2];
  const double a = r / R, rho2 = x * x + y * y, rho = sqrt(rho2), u = rho - R;
  const double theta = atan2(y, x), phi = atan2(z, u);
  double s4, c4, sp, cp;
  sincos(4.0 * theta, &s4, &c4);
  sincos(phi, &sp, &cp);
  const double d1 = 1.0 + a * cp, d2 = 1.0 + alpha * s4 * cp;
  const double dl_dphi = -a * sp / d1 + alpha * s4 * sp / d2;
  const double dl_dth = -4.0 * alpha * c4 * cp / d2;
  const double w = u * u + z * z, dphi_du = -z / w, dphi_dz = u / w;
  if (c.lane == 0) {
    g[0] = dl_dth * (-y / rho2) + dl_dphi * dphi_du * (x / rho);
    g[1] = dl_dth * (x / rho2) + dl_dphi * dphi_du * (y / rho);
    g[2] = dl_dphi * dphi_dz;
  }
}
__device__ void constr(const mb200::Chain& c, double* out) {
  const double R = c.params[0], r = c.params[1];
  const double x = c.q[0], y = c.q[1], z = c.q[2];
  const double d = sqrt(x * x + y * y) - R;
  if (c.lane == 0) out[0] = d * d + z * z - r * r;
}
__device__ void jacob_constr(const mb200::Chain& c, double* J) {
  const double R = c.params[0];
  const double x = c.q[0], y = c.q[1], z = c.q[2];
  const double rho = sqrt(x * x + y * y), f = 2.0 * (rho - R) / rho;
  if (c.lane == 0) J[0] = f * x, J[1] = f * y, J[2] = 2.0 * z;
}
// Hessian [[f + g x^2, g x y, 0], [g x y, f + g y^2, 0], [0, 0, 2]], f = 2 (rho - R) / rho,
// g = 2 R / rho^3
__device__ void mhp_constr(const mb200::Chain& c, const double* m, double* out) {
  const double R = c.params[0];
  const double x = c.q[0], y = c.q[1];
  const double rho = sqrt(x * x + y * y);
  const double f = 2.0 * (rho - R) / rho, g = 2.0 * R / (rho * rho * rho);
  if (c.lane == 0) {
    out[0] = m[0] * (f + g * x * x) + m[1] * (g * x * y);
    out[1] = m[0] * (g * x * y) + m[1] * (f + g * y * y);
    out[2] = 2.0 * m[2];
  }
}
"""

SOURCES = {"sphere": SPHERE, "multi_sphere": MULTI_SPHERE, "torus": TORUS}


def registry_as_user(target):
    """The constrained ``CudaTarget`` computing the same model as a registry constrained target
    (the multi-sphere's n_constr parameter becomes N_CONSTR)."""
    params = () if target.name == "multi_sphere" else target.params
    return CudaTarget(target.dim, SOURCES[target.name], params=params, name=target.name,
                      n_constr=target.n_constr, mhp_constr=True)


# ---------------------------------------------------------------- models the registry lacks
# Each: CUDA source and NumPy callables of the same model (the NumPy side drives the unmodified
# reference in tests/make_user_constraint_golden.py and imports nothing of mici_b200).

# SO(3): q = Q row-major (Q[r][c] = q[3 r + c]), c_p = (Q^T Q - I)[a, b] for the upper-triangle
# pairs p = (a, b) in np.triu_indices(3) order (N_CONSTR = 6, overlapping Jacobian rows); matrix
# von Mises-Fisher density exp(tr(F^T Q)), F row-major in aux: l = -sum F * Q.
SO3 = r"""
__device__ __forceinline__ void so3_pair(int p, int& a, int& b) {
  const int A[6] = {0, 0, 0, 1, 1, 2}, B[6] = {0, 1, 2, 1, 2, 2};
  a = A[p], b = B[p];
}
__device__ double neg_log_dens(const mb200::Chain& c) {
  double s = 0.0;
  for (int i = 0; i < 9; ++i) s += c.aux[i] * c.q[i];
  return -s;
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  for (int i = c.lane; i < 9; i += 32) g[i] = -c.aux[i];
}
__device__ void constr(const mb200::Chain& c, double* out) {
  for (int p = c.lane; p < 6; p += 32) {
    int a, b;
    so3_pair(p, a, b);
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += c.q[3 * k + a] * c.q[3 * k + b];
    out[p] = s - (a == b ? 1.0 : 0.0);
  }
}
__device__ void jacob_constr(const mb200::Chain& c, double* J) {
  for (int idx = c.lane; idx < 6 * 9; idx += 32) {
    const int p = idx / 9, i = idx % 9, r = i / 3, col = i % 3;
    int a, b;
    so3_pair(p, a, b);
    double v = 0.0;
    if (col == a) v += c.q[3 * r + b];
    if (col == b) v += c.q[3 * r + a];
    J[idx] = v;
  }
}
"""
SO3_PAIRS = tuple(zip(*np.triu_indices(3)))


def _so3_f():
    rng = np.random.default_rng(3303)
    return rng.normal(size=(3, 3)) * 2.0


def so3():
    return CudaTarget(9, SO3, aux=_so3_f().ravel(), name="so3", n_constr=6)


def so3_numpy():
    f = _so3_f().ravel()

    def nld(q):
        return -np.sum(f * q)

    def grad(q):
        return -f.copy()

    def constr(q):
        m = q.reshape(3, 3)
        return (m.T @ m - np.identity(3))[np.triu_indices(3)]

    def jacob(q):
        m = q.reshape(3, 3)
        j = np.zeros((6, 9))
        for p, (a, b) in enumerate(SO3_PAIRS):
            for r in range(3):
                j[p, 3 * r + a] += m[r, b]
                j[p, 3 * r + b] += m[r, a]
        return j

    return {"neg_log_dens": nld, "grad_neg_log_dens": grad, "constr": constr,
            "jacob_constr": jacob}


def so3_start(rng, n):
    q = np.empty((n, 9))
    for i in range(n):
        m, r = np.linalg.qr(rng.normal(size=(3, 3)))
        q[i] = (m * np.sign(np.diag(r))).ravel()
    return q


# A generator constraint on the Gaussian system: q = (theta0, theta1, u[5]), observations
# y_k = theta0 + theta1 u_k + u_k^3 / 3 (y in aux, N_CONSTR = 5); c_k = that - y_k, whose Hessian
# depends on q.  Prior beyond the Gaussian reference measure: l = |theta|^2 / (2 s^2), s = params[0].
GENERATOR = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const double s = c.params[0];
  return (c.q[0] * c.q[0] + c.q[1] * c.q[1]) / (2.0 * s * s);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const double s2 = c.params[0] * c.params[0];
  for (int i = c.lane; i < c.dim; i += 32) g[i] = i < 2 ? c.q[i] / s2 : 0.0;
}
__device__ void constr(const mb200::Chain& c, double* out) {
  for (int k = c.lane; k < mb200::N_CONSTR; k += 32) {
    const double u = c.q[2 + k];
    out[k] = c.q[0] + c.q[1] * u + u * u * u / 3.0 - c.aux[k];
  }
}
__device__ void jacob_constr(const mb200::Chain& c, double* J) {
  for (int idx = c.lane; idx < mb200::N_CONSTR * c.dim; idx += 32) {
    const int k = idx / c.dim, i = idx % c.dim;
    const double u = c.q[2 + k];
    J[idx] = i == 0 ? 1.0 : (i == 1 ? u : (i == 2 + k ? c.q[1] + u * u : 0.0));
  }
}
// Hessian of c_k: d2/dtheta1 du_k = 1, d2/du_k^2 = 2 u_k
__device__ void mhp_constr(const mb200::Chain& c, const double* m, double* out) {
  for (int j = c.lane; j < c.dim; j += 32) {
    double v = 0.0;
    if (j == 1) {
      for (int k = 0; k < mb200::N_CONSTR; ++k) v += m[k * c.dim + 2 + k];
    } else if (j >= 2) {
      const int k = j - 2;
      v = m[k * c.dim + 1] + 2.0 * c.q[j] * m[k * c.dim + j];
    }
    out[j] = v;
  }
}
"""
GENERATOR_N = 5
GENERATOR_DIM = 2 + GENERATOR_N
GENERATOR_PARAMS = (2.0,)


def _generator_truth():
    rng = np.random.default_rng(5505)
    theta = np.array([0.3, 0.8])
    u = rng.normal(size=GENERATOR_N)
    return theta, u, theta[0] + theta[1] * u + u**3 / 3.0


def generator():
    return CudaTarget(GENERATOR_DIM, GENERATOR, params=GENERATOR_PARAMS, aux=_generator_truth()[2],
                      name="generator", n_constr=GENERATOR_N, mhp_constr=True)


def generator_numpy():
    (s,) = GENERATOR_PARAMS
    y = _generator_truth()[2]
    n = GENERATOR_N

    def nld(q):
        return (q[0] * q[0] + q[1] * q[1]) / (2.0 * s * s)

    def grad(q):
        g = np.zeros_like(q)
        g[:2] = q[:2] / (s * s)
        return g

    def constr(q):
        u = q[2:]
        return q[0] + q[1] * u + u * u * u / 3.0 - y

    def jacob(q):
        u = q[2:]
        j = np.zeros((n, q.shape[0]))
        j[:, 0] = 1.0
        j[:, 1] = u
        j[np.arange(n), 2 + np.arange(n)] = q[1] + u * u
        return j

    def mhp(q):
        def prod(m):
            out = np.zeros(q.shape[0])
            out[1] = sum(m[k, 2 + k] for k in range(n))
            out[2:] = m[np.arange(n), 1] + 2.0 * q[2:] * m[np.arange(n), 2 + np.arange(n)]
            return out
        return prod

    return {"neg_log_dens": nld, "grad_neg_log_dens": grad, "constr": constr,
            "jacob_constr": jacob, "mhp_constr": mhp}


def generator_start(rng, n):
    """Points on the manifold: theta near the truth, u solving the cubic for each y_k."""
    y = _generator_truth()[2]
    q = np.empty((n, GENERATOR_DIM))
    for i in range(n):
        theta = _generator_truth()[0] + 0.2 * rng.normal(size=2)
        theta[1] = abs(theta[1])  # u^3/3 + theta1 u monotone: one real root per y_k
        u = np.empty(GENERATOR_N)
        for k in range(GENERATOR_N):
            roots = np.roots([1.0 / 3.0, 0.0, theta[1], theta[0] - y[k]])
            u[k] = roots[np.argmin(abs(roots.imag))].real
            for _ in range(3):  # polish to rounding
                u[k] -= (theta[0] + theta[1] * u[k] + u[k] ** 3 / 3.0 - y[k]) / (theta[1] + u[k] ** 2)
        q[i] = np.concatenate([theta, u])
    return q


# The l4 sphere sum q_i^4 = 1 (N_CONSTR = 1, Hessian diag(12 q^2)); l = |q|^2 / 2 + q[0]
L4_SPHERE = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) s += c.q[i] * c.q[i];
  return 0.5 * c.sum(s) + c.q[0];
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  for (int i = c.lane; i < c.dim; i += 32) g[i] = c.q[i] + (i == 0 ? 1.0 : 0.0);
}
__device__ void constr(const mb200::Chain& c, double* out) {
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) {
    const double q2 = c.q[i] * c.q[i];
    s += q2 * q2;
  }
  s = c.sum(s);
  if (c.lane == 0) out[0] = s - 1.0;
}
__device__ void jacob_constr(const mb200::Chain& c, double* J) {
  for (int i = c.lane; i < c.dim; i += 32) J[i] = 4.0 * c.q[i] * c.q[i] * c.q[i];
}
__device__ void mhp_constr(const mb200::Chain& c, const double* m, double* out) {
  for (int i = c.lane; i < c.dim; i += 32) out[i] = 12.0 * c.q[i] * c.q[i] * m[i];
}
"""
L4_DIM = 200


def l4_sphere():
    return CudaTarget(L4_DIM, L4_SPHERE, name="l4_sphere", n_constr=1, mhp_constr=True)


def l4_sphere_numpy():
    def nld(q):
        return 0.5 * (q @ q) + q[0]

    def grad(q):
        g = q.copy()
        g[0] += 1.0
        return g

    return {"neg_log_dens": nld, "grad_neg_log_dens": grad,
            "constr": lambda q: np.array([np.sum(q**4) - 1.0]),
            "jacob_constr": lambda q: (4.0 * q**3)[None, :],
            "mhp_constr": lambda q: (lambda m: 12.0 * q * q * m[0])}


def l4_start(rng, n):
    x = rng.normal(size=(n, L4_DIM))
    return x / np.sum(x**4, axis=1, keepdims=True) ** 0.25


# name -> (CudaTarget factory, NumPy callables, start-state sampler)
UC_MODELS = {
    "so3": (so3, so3_numpy, so3_start),
    "generator": (generator, generator_numpy, generator_start),
    "l4_sphere": (l4_sphere, l4_sphere_numpy, l4_start),
}
