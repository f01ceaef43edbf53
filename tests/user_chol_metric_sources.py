"""User-written CUDA targets and Cholesky-factor metrics of the user-Cholesky-metric tests
(``csrc/user_riemannian.cuh``, ``CholeskyFactoredRiemannianMetricSystem``): the registry's
quadratic Cholesky-factor model rewritten as user sources, and a hierarchical AR(1) model the
registry cannot express, with the NumPy twins that the reference runs to make its fixtures.

The targets keep the warp contract (``mb200::Chain``); the metric functions are called by the
chain's whole 256-thread CTA (``mb200::CtaChain``)."""

import numpy as np

from user_dense_metric_sources import QUADRATIC  # noqa: F401  (l = q.P q / 2, P in aux)
from user_riemannian_sources import BANANA, FUNNEL, STD_GAUSSIAN  # noqa: F401

# (a) L(q) = L0 + c tril(q q^T), L0 = aux [D x D] row-major, params (c): riemannian.cuh
# QuadraticCholModel.  The fill has the registry's expression; the VJP forms
# out_k = c (sum_{j <= k} V_kj q_j + sum_{i >= k} V_ik q_i) from V itself, so its sums run in
# another order than the registry's prefix / suffix scans.
QUADRATIC_CHOL = r"""
__device__ void metric_chol(const mb200::CtaChain& c, double* L, int ld) {
  const int n = c.dim;
  const double k = c.params[0];
  for (int idx = c.lane; idx < n * n; idx += c.n_lanes) {
    const int i = idx / n, j = idx - i * n;
    if (j > i) continue;
    L[i * ld + j] = c.aux[idx] + k * (c.q[i] * c.q[j]);
  }
}
__device__ void vjp_metric_chol(const mb200::CtaChain& c, const double* V, int ld, double* out) {
  const int n = c.dim;
  for (int k = c.lane; k < n; k += c.n_lanes) {
    double r = 0.0, t = 0.0;
    for (int j = 0; j <= k; ++j) r = fma(V[k * ld + j], c.q[j], r);
    for (int i = k; i < n; ++i) t = fma(V[i * ld + k], c.q[i], t);
    out[k] = c.params[0] * (r + t);
  }
}
"""

# (b) Hierarchical AR(1): q = (a, b, x_0 .. x_{T-1}), phi = tanh a, sigma = e^b, the latent series
# x a stationary AR(1) of coefficient phi and innovation scale sigma, observed as y = aux[T] with
# noise scale s = params[0]; a, b ~ N(0, 1).  With S = (1 - phi^2) x_0^2 + sum_{t>=1} (x_t -
# phi x_{t-1})^2 and 1/sigma^2 = e^{-2b}:
#   l = a^2/2 + b^2/2 + T b - log(1 - phi^2)/2 + S / (2 sigma^2) + sum_t (x_t - y_t)^2 / (2 s^2)
#   dl/da = a + phi - (1 - phi^2) / sigma^2 (phi x_0^2 + sum_{t>=1} x_{t-1} (x_t - phi x_{t-1}))
#   dl/db = b + T - S / sigma^2
AR1_HIER = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const int T = c.dim - 2;
  const double a = c.q[0], b = c.q[1], phi = tanh(a), is2 = exp(-2.0 * b);
  const double s2 = c.params[0] * c.params[0];
  const double* x = c.q + 2;
  double e = 0.0, o = 0.0;
  for (int t = c.lane; t < T; t += 32) {
    const double d = t == 0 ? 0.0 : x[t] - phi * x[t - 1];
    e += t == 0 ? (1.0 - phi * phi) * (x[0] * x[0]) : d * d;
    const double r = x[t] - c.aux[t];
    o += r * r;
  }
  e = c.sum(e);
  o = c.sum(o);
  return 0.5 * (a * a) + 0.5 * (b * b) + T * b - 0.5 * log(1.0 - phi * phi) + 0.5 * (e * is2) +
         o / (2.0 * s2);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const int T = c.dim - 2;
  const double a = c.q[0], b = c.q[1], phi = tanh(a), is2 = exp(-2.0 * b);
  const double s2 = c.params[0] * c.params[0];
  const double* x = c.q + 2;
  double e = 0.0, h = 0.0;
  for (int t = c.lane; t < T; t += 32) {
    const double d = t == 0 ? 0.0 : x[t] - phi * x[t - 1];
    e += t == 0 ? (1.0 - phi * phi) * (x[0] * x[0]) : d * d;
    h += t == 0 ? phi * (x[0] * x[0]) : x[t - 1] * d;
    double gt = t == 0 ? (1.0 - phi * phi) * x[0] : d;
    if (t + 1 < T) gt -= phi * (x[t + 1] - phi * x[t]);
    g[2 + t] = gt * is2 + (x[t] - c.aux[t]) / s2;
  }
  e = c.sum(e);
  h = c.sum(h);
  if (c.lane == 0) {
    g[0] = a + phi - (1.0 - phi * phi) * is2 * h;
    g[1] = b + T - e * is2;
  }
}
"""

# Its metric, M = L L^T with L = blockdiag(diag(alpha, beta), L_x), params (alpha, beta): L_x the
# lower-bidiagonal Cholesky factor of the AR(1) prior precision Q_x = L_x L_x^T,
#   (L_x)_tt = 1/sigma (t < T-1),  (L_x)_{T-1,T-1} = sqrt(1 - phi^2)/sigma,  (L_x)_{t+1,t} = -phi/sigma.
# Every entry of L_x is proportional to 1/sigma, so dL/db = -L on the x block; dL/da:
# -phi sqrt(1 - phi^2)/sigma at (T-1, T-1), -(1 - phi^2)/sigma below the diagonal.  The VJP
# reduces over the whole factor into out[0] and out[1] (c.sum); out[k] = 0 for k >= 2.
AR1_HIER_CHOL = r"""
__device__ double ar1_factor(int i, int j, int T, double alpha, double beta, double phi,
                             double isig) {
  if (i < 2 || j < 2) return i != j ? 0.0 : (i == 0 ? alpha : beta);
  const int t = i - 2, u = j - 2;
  if (t == u) return t == T - 1 ? sqrt(1.0 - phi * phi) * isig : isig;
  return t == u + 1 ? -phi * isig : 0.0;
}
__device__ void metric_chol(const mb200::CtaChain& c, double* L, int ld) {
  const int n = c.dim, T = n - 2;
  const double phi = tanh(c.q[0]), isig = exp(-c.q[1]);
  for (int i = c.lane >> 5; i < n; i += c.n_lanes >> 5)
    for (int j = c.lane & 31; j <= i; j += 32)
      L[i * ld + j] = ar1_factor(i, j, T, c.params[0], c.params[1], phi, isig);
}
__device__ void vjp_metric_chol(const mb200::CtaChain& c, const double* V, int ld, double* out) {
  const int n = c.dim, T = n - 2;
  const double phi = tanh(c.q[0]), isig = exp(-c.q[1]), w = 1.0 - phi * phi;
  double da = 0.0, db = 0.0;
  for (int t = c.lane; t < T; t += c.n_lanes) {
    const int i = 2 + t;
    const double vd = V[i * ld + i];
    db -= vd * (t == T - 1 ? sqrt(w) * isig : isig);
    if (t == T - 1) da -= vd * (phi * sqrt(w) * isig);
    if (t > 0) {
      const double vo = V[i * ld + i - 1];
      db -= vo * (-phi * isig);
      da -= vo * (w * isig);
    }
  }
  da = c.sum(da);
  db = c.sum(db);
  for (int k = c.lane; k < n; k += c.n_lanes) out[k] = k == 0 ? da : (k == 1 ? db : 0.0);
}
"""


class Ar1Hier:
    """NumPy twin of AR1_HIER."""

    def __init__(self, y, obs_sd):
        self.y, self.s = np.asarray(y, dtype=np.float64), float(obs_sd)
        self.dim = self.y.shape[0] + 2

    def _parts(self, q):
        a, b, x = q[0], q[1], q[2:]
        phi = np.tanh(a)
        d = x[1:] - phi * x[:-1]
        return a, b, x, phi, np.exp(-2.0 * b), d

    def neg_log_dens(self, q):
        a, b, x, phi, is2, d = self._parts(q)
        T = x.shape[0]
        e = (1.0 - phi * phi) * (x[0] * x[0]) + np.sum(d * d)
        o = np.sum((x - self.y) ** 2)
        return (0.5 * (a * a) + 0.5 * (b * b) + T * b - 0.5 * np.log(1.0 - phi * phi)
                + 0.5 * (e * is2) + o / (2.0 * self.s**2))

    def grad_neg_log_dens(self, q):
        a, b, x, phi, is2, d = self._parts(q)
        T = x.shape[0]
        e = (1.0 - phi * phi) * (x[0] * x[0]) + np.sum(d * d)
        h = phi * (x[0] * x[0]) + np.sum(x[:-1] * d)
        gx = np.concatenate([[(1.0 - phi * phi) * x[0]], d])
        gx[:-1] -= phi * d
        g = np.empty_like(q)
        g[0] = a + phi - (1.0 - phi * phi) * is2 * h
        g[1] = b + T - e * is2
        g[2:] = gx * is2 + (x - self.y) / self.s**2
        return g


class Ar1HierChol:
    """NumPy twin of AR1_HIER_CHOL: the factor and the VJP the reference takes."""

    def __init__(self, alpha, beta):
        self.alpha, self.beta = float(alpha), float(beta)

    def metric_func(self, q):
        n = q.shape[0]
        T = n - 2
        phi, isig = np.tanh(q[0]), np.exp(-q[1])
        L = np.zeros((n, n))
        L[0, 0], L[1, 1] = self.alpha, self.beta
        t = np.arange(2, n)
        L[t, t] = isig
        L[n - 1, n - 1] = np.sqrt(1.0 - phi * phi) * isig
        L[t[1:], t[:-1]] = -phi * isig
        Lx, Q = L[2:, 2:], ar1_precision(q)
        if np.isfinite(Q).all() and np.isfinite(L).all():  # L_x is the factor of Q_x
            assert T >= 2 and np.allclose(Lx @ Lx.T, Q, rtol=0, atol=1e-12 * np.abs(Q).max())
        return L

    def vjp_metric_func(self, q):
        n = q.shape[0]
        phi, isig = np.tanh(q[0]), np.exp(-q[1])
        w = 1.0 - phi * phi
        t = np.arange(2, n)

        def vjp(V):
            V = np.tril(V)
            diag = np.full(n - 2, isig)
            diag[-1] = np.sqrt(w) * isig
            out = np.zeros(n)
            out[1] = -(np.sum(V[t, t] * diag) + np.sum(V[t[1:], t[:-1]] * (-phi * isig)))
            out[0] = -(V[n - 1, n - 1] * (phi * np.sqrt(w) * isig)
                       + np.sum(V[t[1:], t[:-1]] * (w * isig)))
            return out

        return vjp


def ar1_precision(q):
    """The AR(1) prior precision Q_x of the position ``q`` (the x block of M(q))."""
    T = q.shape[0] - 2
    phi, is2 = np.tanh(q[0]), np.exp(-2.0 * q[1])
    Q = np.diag(np.r_[1.0, np.full(T - 2, 1.0 + phi * phi), 1.0]) * is2
    i = np.arange(T - 1)
    Q[i + 1, i] = Q[i, i + 1] = -phi * is2
    return Q


AR1_TRUTH = (1.0, -0.5)  # (a, b): phi = tanh 1 = 0.76, sigma = e^-0.5 = 0.61
AR1_OBS_SD = 0.5


def _ar1_data(T, seed=20261018):
    rng = np.random.default_rng([seed, T])
    phi, sig = np.tanh(AR1_TRUTH[0]), np.exp(AR1_TRUTH[1])
    x = np.empty(T)
    x[0] = sig / np.sqrt(1.0 - phi * phi) * rng.standard_normal()
    for t in range(1, T):
        x[t] = phi * x[t - 1] + sig * rng.standard_normal()
    return x, x + AR1_OBS_SD * rng.standard_normal(T)


def ul_model(name):
    """``(NumPy target, NumPy metric, (target source, params, aux), (metric source, params,
    aux))`` of the hierarchical AR(1) model ``ar1_64`` (T = 64, D = 66: the factor and V in
    shared memory) or ``ar1_254`` (T = 254, D = 256: in the per-CTA workspace)."""
    T = {"ar1_64": 64, "ar1_254": 254}[name]
    _, y = _ar1_data(T)
    alpha, beta = np.sqrt(T), np.sqrt(2.0 * T)
    return (Ar1Hier(y, AR1_OBS_SD), Ar1HierChol(alpha, beta),
            (AR1_HIER, (AR1_OBS_SD,), y.copy()), (AR1_HIER_CHOL, (alpha, beta), None))


def ul_start(name, n_chains, rng):
    """Positions near the model's truth: (a, b) + 0.1 N(0, 1) and the latent series + 0.2 N(0, 1)."""
    T = {"ar1_64": 64, "ar1_254": 254}[name]
    x, _ = _ar1_data(T)
    pos = np.empty((n_chains, T + 2))
    pos[:, :2] = np.asarray(AR1_TRUTH) + 0.1 * rng.standard_normal((n_chains, 2))
    pos[:, 2:] = x + 0.2 * rng.standard_normal((n_chains, T))
    return pos


UL_MODELS = ("ar1_64", "ar1_254")

# (target source, metric source) of every test model, for the compile tests
COMPILE_PAIRS = {
    "quadratic_chol": (QUADRATIC, QUADRATIC_CHOL),
    "std_gaussian_chol": (STD_GAUSSIAN, QUADRATIC_CHOL),
    "banana_chol": (BANANA, QUADRATIC_CHOL),
    "funnel_chol": (FUNNEL, QUADRATIC_CHOL),
    "ar1_hier": (AR1_HIER, AR1_HIER_CHOL),
}
