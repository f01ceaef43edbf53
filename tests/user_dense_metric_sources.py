"""User-written CUDA targets and dense metrics of the user-dense-metric tests
(``csrc/user_riemannian.cuh``, ``DenseRiemannianMetricSystem``): the registry's quadratic target
and its rank-1 and Hadamard metrics rewritten as user sources, each written with the registry
kernel's expressions in the registry kernel's order, so that both compute the same values; and
models the registry cannot express, with the NumPy twins that the reference runs to make their
fixtures.

The targets keep the warp contract (``mb200::Chain``); the dense metric functions are called by
the chain's whole 256-thread CTA (``mb200::CtaChain``)."""

import numpy as np

from user_riemannian_sources import LOGISTIC, Logistic, _logistic_data

# l = q.P q / 2 with P in aux (riemannian.cuh QuadraticRTarget: the same per-row dot products)
QUADRATIC = r"""
__device__ void prec_row(const mb200::Chain& c, int i, double& s) {
  const double* row = c.aux + (size_t)i * c.dim;
  s = 0.0;
  for (int j = 0; j < c.dim; ++j) s = fma(row[j], c.q[j], s);
}
__device__ double neg_log_dens(const mb200::Chain& c) {
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) {
    double t;
    prec_row(c, i, t);
    s = fma(c.q[i], t, s);
  }
  return 0.5 * c.sum(s);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  for (int i = c.lane; i < c.dim; i += 32) prec_row(c, i, g[i]);
}
"""

# M = B + c q q^T, aux = B, params (c): dense_global.cuh Rank1Model.  One row per warp, lanes
# along the row, for the fill and the VJP.
RANK1_DENSE = r"""
__device__ void metric_dense(const mb200::CtaChain& c, double* M, int ld) {
  const int n = c.dim, w = c.lane >> 5, l = c.lane & 31, nw = c.n_lanes >> 5;
  const double k = c.params[0];
  for (int i = w; i < n; i += nw)
    for (int j = l; j < n; j += 32) M[(size_t)i * ld + j] = c.aux[(size_t)i * n + j] + k * (c.q[i] * c.q[j]);
}
__device__ void vjp_metric_dense(const mb200::CtaChain& c, const double* V, int ld, double* out) {
  const int n = c.dim, w = c.lane >> 5, l = c.lane & 31, nw = c.n_lanes >> 5;
  for (int i = w; i < n; i += nw) {
    double s = 0.0;
    for (int j = l; j < n; j += 32) s = fma(V[(size_t)i * ld + j], c.q[j], s);
    s = mb200::warp_sum(s);
    if (l == 0) out[i] = c.params[0] * (s + s);
  }
}
"""

# M = B + c (q q^T) o S, aux = [B | S], params (c): dense_global.cuh HadamardModel
HADAMARD_DENSE = r"""
__device__ void metric_dense(const mb200::CtaChain& c, double* M, int ld) {
  const int n = c.dim, w = c.lane >> 5, l = c.lane & 31, nw = c.n_lanes >> 5;
  const double* B = c.aux;
  const double* S = c.aux + (size_t)n * n;
  const double k = c.params[0];
  for (int i = w; i < n; i += nw)
    for (int j = l; j < n; j += 32)
      M[(size_t)i * ld + j] = B[(size_t)i * n + j] + k * ((c.q[i] * c.q[j]) * S[(size_t)i * n + j]);
}
__device__ void vjp_metric_dense(const mb200::CtaChain& c, const double* V, int ld, double* out) {
  const int n = c.dim, w = c.lane >> 5, l = c.lane & 31, nw = c.n_lanes >> 5;
  const double* S = c.aux + (size_t)n * n;
  for (int i = w; i < n; i += nw) {
    double s = 0.0;
    for (int j = l; j < n; j += 32) s = fma(V[(size_t)i * ld + j] * S[(size_t)i * n + j], c.q[j], s);
    s = mb200::warp_sum(s);
    if (l == 0) out[i] = c.params[0] * (s + s);
  }
}
"""

# Bayesian logistic regression's Fisher metric G(q) = X^T diag(s (1 - s)) X + I / v0, s = sigma(X q)
# with X [N x D] in aux and params (v0, N), N <= 64: the per-row weights go through a static
# shared-memory array, written by one warp per data row, then every thread fills entries.
# vjp: out_k = sum_n s_n (1 - s_n) (1 - 2 s_n) (x_n . V x_n) x_nk
LOGISTIC_DENSE_FISHER = r"""
#define LR_MAX_ROWS 64
__device__ void metric_dense(const mb200::CtaChain& c, double* M, int ld) {
  __shared__ double lam[LR_MAX_ROWS];
  const int N = (int)c.params[1], D = c.dim, w = c.lane >> 5, l = c.lane & 31, nw = c.n_lanes >> 5;
  const double* X = c.aux;
  for (int n = w; n < N; n += nw) {
    double z = 0.0;
    for (int k = l; k < D; k += 32) z += X[n * D + k] * c.q[k];
    z = mb200::warp_sum(z);
    const double s = 1.0 / (1.0 + exp(-z));
    if (l == 0) lam[n] = s * (1.0 - s);
  }
  __syncthreads();
  for (int idx = c.lane; idx < D * D; idx += c.n_lanes) {
    const int i = idx / D, j = idx - i * D;
    double g = 0.0;
    for (int n = 0; n < N; ++n) g += (X[n * D + i] * X[n * D + j]) * lam[n];
    M[(size_t)i * ld + j] = (i == j) ? g + 1.0 / c.params[0] : g;
  }
}
__device__ void vjp_metric_dense(const mb200::CtaChain& c, const double* V, int ld, double* out) {
  __shared__ double coef[LR_MAX_ROWS];
  const int N = (int)c.params[1], D = c.dim, w = c.lane >> 5, l = c.lane & 31, nw = c.n_lanes >> 5;
  const double* X = c.aux;
  for (int n = w; n < N; n += nw) {
    double z = 0.0, a = 0.0;
    for (int i = l; i < D; i += 32) {
      const double xi = X[n * D + i];
      double t = 0.0;
      for (int j = 0; j < D; ++j) t += V[(size_t)i * ld + j] * X[n * D + j];
      z += xi * c.q[i];
      a += xi * t;
    }
    z = mb200::warp_sum(z);
    a = mb200::warp_sum(a);
    const double s = 1.0 / (1.0 + exp(-z));
    if (l == 0) coef[n] = s * (1.0 - s) * (1.0 - 2.0 * s) * a;
  }
  __syncthreads();
  for (int k = c.lane; k < D; k += c.n_lanes) {
    double o = 0.0;
    for (int n = 0; n < N; ++n) o += coef[n] * X[n * D + k];
    out[k] = o;
  }
}
"""

# Log-Gaussian Cox process on a square grid of D cells: counts y, cell area m, prior mean mu and
# prior precision C^-1:  l(x) = sum_i (m e^x_i - y_i x_i) + (x - mu).C^-1 (x - mu) / 2,
# target aux = [C^-1 | y], params (m, mu)
LGCP = r"""
__device__ double prior_row(const mb200::Chain& c, int i) {
  const double* row = c.aux + (size_t)i * c.dim;
  double t = 0.0;
  for (int j = 0; j < c.dim; ++j) t = fma(row[j], c.q[j] - c.params[1], t);
  return t;
}
__device__ double neg_log_dens(const mb200::Chain& c) {
  const double* y = c.aux + (size_t)c.dim * c.dim;
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) {
    const double x = c.q[i];
    s += (c.params[0] * exp(x) - y[i] * x) + 0.5 * (x - c.params[1]) * prior_row(c, i);
  }
  return c.sum(s);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const double* y = c.aux + (size_t)c.dim * c.dim;
  for (int i = c.lane; i < c.dim; i += 32)
    g[i] = (c.params[0] * exp(c.q[i]) - y[i]) + prior_row(c, i);
}
"""

# its Riemannian-manifold metric G(x) = C^-1 + diag(m e^x), aux = C^-1, params (m);
# vjp: out_k = V_kk m e^x_k
LGCP_METRIC = r"""
__device__ void metric_dense(const mb200::CtaChain& c, double* M, int ld) {
  const int n = c.dim, w = c.lane >> 5, l = c.lane & 31, nw = c.n_lanes >> 5;
  for (int i = w; i < n; i += nw) {
    const double d = c.params[0] * exp(c.q[i]);
    for (int j = l; j < n; j += 32) {
      const double v = c.aux[(size_t)i * n + j];
      M[(size_t)i * ld + j] = (i == j) ? v + d : v;
    }
  }
}
__device__ void vjp_metric_dense(const mb200::CtaChain& c, const double* V, int ld, double* out) {
  for (int k = c.lane; k < c.dim; k += c.n_lanes)
    out[k] = V[(size_t)k * ld + k] * (c.params[0] * exp(c.q[k]));
}
"""


class LogisticDenseFisher:
    """NumPy twin of LOGISTIC_DENSE_FISHER."""

    def __init__(self, X, v0):
        self.X, self.v0 = np.asarray(X, float), float(v0)

    def metric_func(self, q):
        s = 1.0 / (1.0 + np.exp(-(self.X @ q)))
        return (self.X.T * (s * (1.0 - s))) @ self.X + np.identity(self.X.shape[1]) / self.v0

    def vjp_metric_func(self, q):
        s = 1.0 / (1.0 + np.exp(-(self.X @ q)))

        def vjp(V):
            a = np.einsum("ni,ij,nj->n", self.X, V, self.X)
            return self.X.T @ (s * (1.0 - s) * (1.0 - 2.0 * s) * a)

        return vjp


class Lgcp:
    """NumPy twin of LGCP."""

    def __init__(self, prec, y, m, mu):
        self.prec, self.y, self.m, self.mu = np.asarray(prec), np.asarray(y), float(m), float(mu)
        self.dim = self.y.shape[0]

    def neg_log_dens(self, x):
        r = x - self.mu
        return np.sum(self.m * np.exp(x) - self.y * x) + 0.5 * r @ self.prec @ r

    def grad_neg_log_dens(self, x):
        return self.m * np.exp(x) - self.y + self.prec @ (x - self.mu)


class LgcpMetric:
    """NumPy twin of LGCP_METRIC."""

    def __init__(self, prec, m):
        self.prec, self.m = np.asarray(prec), float(m)

    def metric_func(self, x):
        return self.prec + np.diag(self.m * np.exp(x))

    def vjp_metric_func(self, x):
        d = self.m * np.exp(x)
        return lambda V: np.diagonal(V) * d


def _lgcp_data(side, seed=20261018):
    """A ``side x side`` grid on the unit square: exponential covariance C_ij = s2 exp(-|u_i - u_j|
    / beta), one latent field drawn from N(mu, C), Poisson counts of rate m e^x."""
    rng = np.random.default_rng([seed, side])
    g = (np.arange(side) + 0.5) / side
    u = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
    dist = np.linalg.norm(u[:, None, :] - u[None, :, :], axis=-1)
    s2, beta, mu, m = 1.0, 0.3, 0.5, 1.0
    cov = s2 * np.exp(-dist / beta)
    x = mu + np.linalg.cholesky(cov) @ rng.standard_normal(side * side)
    y = rng.poisson(m * np.exp(x)).astype(float)
    return np.linalg.inv(cov), y, m, mu


def ud_model(name):
    """``(NumPy target, NumPy metric, (target source, params, aux), (metric source, params,
    aux))`` of a dense model the registry cannot express: ``logistic`` (D = 25, 40 rows),
    ``lgcp64`` and ``lgcp144``."""
    if name == "logistic":
        X, y = _logistic_data()
        v0 = 4.0
        return (Logistic(X, y, v0), LogisticDenseFisher(X, v0),
                (LOGISTIC, (v0, X.shape[0]), np.concatenate([X.ravel(), y])),
                (LOGISTIC_DENSE_FISHER, (v0, X.shape[0]), X.ravel().copy()))
    if name in ("lgcp64", "lgcp144"):
        prec, y, m, mu = _lgcp_data(8 if name == "lgcp64" else 12)
        prec = 0.5 * (prec + prec.T)
        return (Lgcp(prec, y, m, mu), LgcpMetric(prec, m),
                (LGCP, (m, mu), np.concatenate([prec.ravel(), y])),
                (LGCP_METRIC, (m,), prec.ravel().copy()))
    raise KeyError(name)


UD_MODELS = ("logistic", "lgcp64", "lgcp144")

# (target source, metric source) of every test model, for the compile tests
COMPILE_PAIRS = {
    "rank1": (QUADRATIC, RANK1_DENSE),
    "hadamard": (QUADRATIC, HADAMARD_DENSE),
    "logistic": (LOGISTIC, LOGISTIC_DENSE_FISHER),
    "lgcp": (LGCP, LGCP_METRIC),
}
