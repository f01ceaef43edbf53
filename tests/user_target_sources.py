"""User-written CUDA targets of the user-target tests (``mici_b200.targets.CudaTarget``), with the
NumPy statements of the same models that the reference is run with to make the ``ut_*``
fixtures (tests/make_user_target_golden.py).  The NumPy side imports nothing of mici_b200:
``CudaTarget`` is imported only where a CUDA target is built."""

import numpy as np


def CudaTarget(*args, **kwargs):  # noqa: N802
    from mici_b200.targets import CudaTarget as cls  # noqa: PLC0415

    return cls(*args, **kwargs)

# ---------------------------------------------------------------- registry models, rewritten

STD_GAUSSIAN = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) s += c.q[i] * c.q[i];
  return 0.5 * c.sum(s);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  for (int i = c.lane; i < c.dim; i += 32) g[i] = c.q[i];
}
"""

# v = q[0], x = q[1:]:  l = v^2/18 + (D-1) v/2 + exp(-v) |x|^2 / 2
FUNNEL = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  double xx = 0.0;
  for (int i = 1 + c.lane; i < c.dim; i += 32) xx += c.q[i] * c.q[i];
  xx = c.sum(xx);
  const double v = c.q[0];
  return v * v / 18.0 + 0.5 * (c.dim - 1) * v + 0.5 * exp(-v) * xx;
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  double xx = 0.0;
  for (int i = 1 + c.lane; i < c.dim; i += 32) xx += c.q[i] * c.q[i];
  xx = c.sum(xx);
  const double v = c.q[0], e = exp(-v);
  for (int i = 1 + c.lane; i < c.dim; i += 32) g[i] = e * c.q[i];
  if (c.lane == 0) g[0] = v / 9.0 + 0.5 * (c.dim - 1) - 0.5 * e * xx;
}
"""

# pairs (x, y) = (q[2k], q[2k+1]):  l = sum x^2/8 + (y - b x^2)^2 / 2, b = params[0]
BANANA = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const double b = c.params[0];
  double s = 0.0;
  for (int i = 2 * c.lane; i < c.dim; i += 64) {
    const double x = c.q[i], r = c.q[i + 1] - b * x * x;
    s += x * x / 8.0 + 0.5 * r * r;
  }
  return c.sum(s);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const double b = c.params[0];
  for (int i = 2 * c.lane; i < c.dim; i += 64) {
    const double x = c.q[i], r = c.q[i + 1] - b * x * x;
    g[i] = x / 4.0 - 2.0 * b * x * r;
    g[i + 1] = r;
  }
}
"""


def registry_as_user(target):
    """The ``CudaTarget`` computing the same model as a registry target."""
    src = {"std_gaussian": STD_GAUSSIAN, "neal_funnel": FUNNEL, "banana": BANANA}[target.name]
    return CudaTarget(target.dim, src, params=target.params, name=target.name)


# ---------------------------------------------------------------- models the registry lacks

# Non-centred eight schools, q = (mu, log tau, theta~[8]); theta = mu + tau theta~.
# params: prior scales (s_mu, s_tau); aux: y[8] then sigma[8].
#   l = mu^2/(2 s_mu^2) + log_tau^2/(2 s_tau^2) + |theta~|^2/2 + sum (theta_j - y_j)^2 / (2 sigma_j^2)
EIGHT_SCHOOLS = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const double mu = c.q[0], lt = c.q[1], tau = exp(lt);
  double s = 0.0;
  if (c.lane < 8) {
    const double tt = c.q[2 + c.lane], y = c.aux[c.lane], sg = c.aux[8 + c.lane];
    const double r = mu + tau * tt - y;
    s = 0.5 * tt * tt + r * r / (2.0 * sg * sg);
  }
  s = c.sum(s);
  const double sm = c.params[0], st = c.params[1];
  return mu * mu / (2.0 * sm * sm) + lt * lt / (2.0 * st * st) + s;
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const double mu = c.q[0], lt = c.q[1], tau = exp(lt);
  double rm = 0.0, rt = 0.0;
  if (c.lane < 8) {
    const double tt = c.q[2 + c.lane], y = c.aux[c.lane], sg = c.aux[8 + c.lane];
    const double r = (mu + tau * tt - y) / (sg * sg);
    g[2 + c.lane] = tt + r * tau;
    rm = r;
    rt = r * tau * tt;
  }
  rm = c.sum(rm);
  rt = c.sum(rt);
  const double sm = c.params[0], st = c.params[1];
  if (c.lane == 0) {
    g[0] = mu / (sm * sm) + rm;
    g[1] = lt / (st * st) + rt;
  }
}
"""
EIGHT_SCHOOLS_Y = np.array([28.0, 8.0, -3.0, 7.0, -1.0, 1.0, 18.0, 12.0])
EIGHT_SCHOOLS_SIGMA = np.array([15.0, 10.0, 16.0, 11.0, 9.0, 11.0, 10.0, 18.0])
EIGHT_SCHOOLS_PARAMS = (5.0, 5.0)


def eight_schools():
    aux = np.concatenate([EIGHT_SCHOOLS_Y, EIGHT_SCHOOLS_SIGMA])
    return CudaTarget(10, EIGHT_SCHOOLS, params=EIGHT_SCHOOLS_PARAMS, aux=aux, name="eight_schools")


def eight_schools_numpy():
    y, sg = EIGHT_SCHOOLS_Y, EIGHT_SCHOOLS_SIGMA
    sm, st = EIGHT_SCHOOLS_PARAMS

    def nld(q):
        mu, lt, tt = q[0], q[1], q[2:]
        r = mu + np.exp(lt) * tt - y
        return mu**2 / (2 * sm**2) + lt**2 / (2 * st**2) + np.sum(0.5 * tt**2 + r**2 / (2 * sg**2))

    def grad(q):
        mu, lt, tt = q[0], q[1], q[2:]
        tau = np.exp(lt)
        r = (mu + tau * tt - y) / sg**2
        return np.concatenate([[mu / sm**2 + r.sum(), lt / st**2 + (r * tau * tt).sum()],
                               tt + r * tau])

    return nld, grad


# Latent AR(1) series x[D] observed with unit noise, y = aux[D]; params: (phi, sigma).
#   l = x0^2 (1 - phi^2) / (2 s^2) + sum_{t>=1} (x_t - phi x_{t-1})^2 / (2 s^2) + sum (x_t - y_t)^2 / 2
# Each coordinate's gradient reads its neighbours x_{t-1}, x_{t+1}, held by other lanes.
AR1 = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const double phi = c.params[0], s2 = c.params[1] * c.params[1];
  double s = 0.0;
  for (int t = c.lane; t < c.dim; t += 32) {
    const double x = c.q[t], o = x - c.aux[t];
    const double e = (t == 0) ? x * x * (1.0 - phi * phi) : (x - phi * c.q[t - 1]) * (x - phi * c.q[t - 1]);
    s += e / (2.0 * s2) + 0.5 * o * o;
  }
  return c.sum(s);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const double phi = c.params[0], s2 = c.params[1] * c.params[1];
  for (int t = c.lane; t < c.dim; t += 32) {
    const double x = c.q[t];
    double d = (t == 0) ? x * (1.0 - phi * phi) / s2 : (x - phi * c.q[t - 1]) / s2;
    if (t + 1 < c.dim) d -= phi * (c.q[t + 1] - phi * x) / s2;
    g[t] = d + (x - c.aux[t]);
  }
}
"""
AR1_DIM = 100
AR1_PARAMS = (0.9, 0.5)


def _ar1_data():
    return np.random.default_rng(20261017).normal(size=AR1_DIM).cumsum() * 0.3


def ar1():
    return CudaTarget(AR1_DIM, AR1, params=AR1_PARAMS, aux=_ar1_data(), name="ar1")


def ar1_numpy():
    phi, sig = AR1_PARAMS
    s2 = sig * sig
    y = _ar1_data()

    def nld(q):
        e = np.concatenate([[q[0] * q[0] * (1 - phi * phi)], (q[1:] - phi * q[:-1]) ** 2])
        o = q - y
        return np.sum(e / (2 * s2) + 0.5 * o * o)

    def grad(q):
        d = np.empty_like(q)
        d[0] = q[0] * (1 - phi * phi) / s2
        d[1:] = (q[1:] - phi * q[:-1]) / s2
        d[:-1] -= phi * (q[1:] - phi * q[:-1]) / s2
        return d + (q - y)

    return nld, grad


# Bayesian logistic regression, beta[D]: design X [N x D] (row-major) then labels y[N] in aux;
# params: (N, prior scale s).  eta = X beta;
#   l = sum_i log1p(exp(eta_i)) - y_i eta_i + |beta|^2 / (2 s^2),  grad = X^T (sigmoid(eta) - y) + beta / s^2
LOGISTIC = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const int n = (int)c.params[0];
  const double s = c.params[1];
  const double* x = c.aux;
  const double* y = c.aux + (size_t)n * c.dim;
  double acc = 0.0;
  for (int i = c.lane; i < n; i += 32) {
    double eta = 0.0;
    for (int j = 0; j < c.dim; ++j) eta += x[(size_t)i * c.dim + j] * c.q[j];
    acc += log1p(exp(eta)) - y[i] * eta;
  }
  double bb = 0.0;
  for (int j = c.lane; j < c.dim; j += 32) bb += c.q[j] * c.q[j];
  return c.sum(acc) + c.sum(bb) / (2.0 * s * s);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const int n = (int)c.params[0];
  const double s = c.params[1];
  const double* x = c.aux;
  const double* y = c.aux + (size_t)n * c.dim;
  // each lane takes its own rows; column sums of X^T r reduced over the warp one coordinate at a time
  double r[8];
  int m = 0;
  for (int i = c.lane; i < n; i += 32, ++m) {
    double eta = 0.0;
    for (int j = 0; j < c.dim; ++j) eta += x[(size_t)i * c.dim + j] * c.q[j];
    r[m] = 1.0 / (1.0 + exp(-eta)) - y[i];
  }
  for (int j = 0; j < c.dim; ++j) {
    double p = 0.0;
    int k = 0;
    for (int i = c.lane; i < n; i += 32, ++k) p += x[(size_t)i * c.dim + j] * r[k];
    p = c.sum(p);
    if (c.lane == 0) g[j] = p + c.q[j] / (s * s);
  }
}
"""
LOGISTIC_N, LOGISTIC_DIM, LOGISTIC_SCALE = 200, 25, 2.0  # LOGISTIC keeps <= 8 rows per lane


def _logistic_data():
    rng = np.random.default_rng(4242)
    x = rng.normal(size=(LOGISTIC_N, LOGISTIC_DIM)) / np.sqrt(LOGISTIC_DIM)
    beta = rng.normal(size=LOGISTIC_DIM)
    y = (rng.uniform(size=LOGISTIC_N) < 1 / (1 + np.exp(-x @ beta))).astype(np.float64)
    return x, y


def logistic():
    x, y = _logistic_data()
    return CudaTarget(LOGISTIC_DIM, LOGISTIC, params=(LOGISTIC_N, LOGISTIC_SCALE),
                      aux=np.concatenate([x.ravel(), y]), name="logistic")


def logistic_numpy():
    x, y = _logistic_data()
    s2 = LOGISTIC_SCALE**2

    def nld(q):
        eta = x @ q
        return np.sum(np.log1p(np.exp(eta)) - y * eta) + q @ q / (2 * s2)

    def grad(q):
        eta = x @ q
        return x.T @ (1 / (1 + np.exp(-eta)) - y) + q / s2

    return nld, grad


# dimension of each model (the fixture generator needs it without building a CudaTarget)
DIMS = {"eight_schools": 10, "ar1": AR1_DIM, "logistic": LOGISTIC_DIM}
USER_MODELS = {"eight_schools": (eight_schools, eight_schools_numpy),
               "ar1": (ar1, ar1_numpy),
               "logistic": (logistic, logistic_numpy)}
ALL_SOURCES = {"std_gaussian": STD_GAUSSIAN, "funnel": FUNNEL, "banana": BANANA,
               "eight_schools": EIGHT_SCHOOLS, "ar1": AR1, "logistic": LOGISTIC}
