"""User-written CUDA targets and metrics of the user-Riemannian tests: the registry's diagonal and
scalar Riemannian models rewritten as user sources (``csrc/user_riemannian.cuh``), each written
with the registry kernel's expressions in the registry kernel's order, so that both compute the
same values; and models the registry cannot express, with the NumPy twins that the reference
runs to make their fixtures."""

import numpy as np

# v = q[0], x = q[1:]:  l = v^2/18 + (D-1) v/2 + exp(-v) |x|^2 / 2 (riemannian.cuh FunnelRTarget)
FUNNEL = r"""
__device__ double xsq(const mb200::Chain& c) {
  double s = 0.0;
  for (int i = 1 + c.lane; i < c.dim; i += 32) s = fma(c.q[i], c.q[i], s);
  return c.sum(s);
}
__device__ double neg_log_dens(const mb200::Chain& c) {
  const double s = xsq(c), v = c.q[0];
  return (v * v / 18.0 + 0.5 * (c.dim - 1) * v) + 0.5 * exp(-v) * s;
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const double s = xsq(c), v = c.q[0], e = exp(-v);
  for (int i = c.lane; i < c.dim; i += 32)
    g[i] = (i == 0) ? (v / 9.0 + 0.5 * (c.dim - 1)) - 0.5 * e * s : e * c.q[i];
}
"""

# the funnel's expected Fisher information d = [1/9 + (D-1)/2, e^-v, ..., e^-v]
FUNNEL_FISHER = r"""
__device__ void metric_diagonal(const mb200::Chain& c, double* d) {
  const double e = exp(-c.q[0]);
  const double d0 = 1.0 / 9.0 + 0.5 * (c.dim - 1);
  for (int i = c.lane; i < c.dim; i += 32) d[i] = (i == 0) ? d0 : e;
}
__device__ void vjp_metric_diagonal(const mb200::Chain& c, const double* w, double* out) {
  double s = 0.0;
  for (int i = 1 + c.lane; i < c.dim; i += 32) s += w[i];
  s = c.sum(s);
  const double e = exp(-c.q[0]);
  for (int i = c.lane; i < c.dim; i += 32) out[i] = (i == 0) ? -e * s : 0.0;
}
"""

# l = |q|^2 / 2
STD_GAUSSIAN = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) s = fma(c.q[i], c.q[i], s);
  return 0.5 * c.sum(s);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  for (int i = c.lane; i < c.dim; i += 32) g[i] = c.q[i];
}
"""

# pairs (x, y) = (q[2k], q[2k+1]):  l = sum x^2/8 + (y - b x^2)^2 / 2, b = params[0]
BANANA = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const double b = c.params[0];
  double s = 0.0;
  for (int i = 2 * c.lane; i < c.dim; i += 64) {
    const double x = c.q[i], y = c.q[i + 1], r = y - b * x * x;
    s += x * x / 8.0 + 0.5 * r * r;
  }
  return c.sum(s);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const double b = c.params[0];
  for (int i = 2 * c.lane; i < c.dim; i += 64) {
    const double x = c.q[i], y = c.q[i + 1], r = y - b * x * x;
    g[i] = x / 4.0 - 2.0 * b * x * r;
    g[i + 1] = r;
  }
}
"""

# d_i = a + b q_i^2, (a, b) = params[0:2]
QUADRATIC_DIAGONAL = r"""
__device__ void metric_diagonal(const mb200::Chain& c, double* d) {
  const double a = c.params[0], b = c.params[1];
  for (int i = c.lane; i < c.dim; i += 32) d[i] = a + b * (c.q[i] * c.q[i]);
}
__device__ void vjp_metric_diagonal(const mb200::Chain& c, const double* w, double* out) {
  const double b = c.params[1];
  for (int i = c.lane; i < c.dim; i += 32) out[i] = 2.0 * b * w[i] * c.q[i];
}
"""

# s = a + b |q|^2, (a, b) = params[0:2]
QUADRATIC_SCALAR = r"""
__device__ double metric_scalar(const mb200::Chain& c) {
  double acc = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) acc = fma(c.q[i], c.q[i], acc);
  return c.params[0] + c.params[1] * c.sum(acc);
}
__device__ void vjp_metric_scalar(const mb200::Chain& c, double w, double* out) {
  const double b = c.params[1];
  for (int i = c.lane; i < c.dim; i += 32) out[i] = 2.0 * b * w * c.q[i];
}
"""

# (name, target source, metric kind, metric source): every pair the CPU tests compile
PAIRS = {
    "funnel_fisher": (FUNNEL, "diagonal", FUNNEL_FISHER),
    "std_gaussian_diag": (STD_GAUSSIAN, "diagonal", QUADRATIC_DIAGONAL),
    "banana_diag": (BANANA, "diagonal", QUADRATIC_DIAGONAL),
    "std_gaussian_scalar": (STD_GAUSSIAN, "scalar", QUADRATIC_SCALAR),
    "banana_scalar": (BANANA, "scalar", QUADRATIC_SCALAR),
    "funnel_scalar": (FUNNEL, "scalar", QUADRATIC_SCALAR),
}

# ------------------------------------------------------------ models the registry cannot express
#
# Each model: CUDA target and metric sources, and their NumPy twins, which the unmodified
# reference takes as its callables to make the ur_* fixtures (tests/make_user_riemannian_golden.py)
# and the oracle runs with (tests/riemannian_diag_cases.py's OracleSystem).  Every expression is
# the same in both, in the same order, except that the CUDA sums run in the warp's order.

# Centred eight schools, q = [mu, log tau, theta_1..J] (D = J + 2):
#   mu ~ N(0, v0), log tau ~ N(0, 1), theta_j ~ N(mu, tau^2), y_j ~ N(theta_j, sigma_j^2)
# target params: (v0,), target aux: [y (J) | sigma (J)]; the metric is the expected Fisher
# information, d = [1/v0 + J e^{-2 lt}, 1 + 2 J, e^{-2 lt} + 1/sigma_j^2], depending on log tau;
# metric params: (v0,), metric aux: sigma (J).
EIGHT_SCHOOLS = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const int J = c.dim - 2;
  const double mu = c.q[0], lt = c.q[1], e = exp(-2.0 * lt);
  double s = 0.0;
  for (int j = c.lane; j < J; j += 32) {
    const double th = c.q[2 + j], sg = c.aux[J + j];
    const double r = th - mu, u = c.aux[j] - th;
    s += 0.5 * (r * r) * e + u * u / (2.0 * (sg * sg));
  }
  s = c.sum(s);
  return mu * mu / (2.0 * c.params[0]) + 0.5 * (lt * lt) + J * lt + s;
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const int J = c.dim - 2;
  const double mu = c.q[0], lt = c.q[1], e = exp(-2.0 * lt);
  double sr = 0.0, srr = 0.0;
  for (int j = c.lane; j < J; j += 32) {
    const double th = c.q[2 + j], sg = c.aux[J + j], r = th - mu;
    sr += r;
    srr += r * r;
    g[2 + j] = r * e + (th - c.aux[j]) / (sg * sg);
  }
  sr = c.sum(sr);
  srr = c.sum(srr);
  if (c.lane == 0) {
    g[0] = mu / c.params[0] - sr * e;
    g[1] = lt - srr * e + J;
  }
}
"""
EIGHT_SCHOOLS_FISHER = r"""
__device__ void metric_diagonal(const mb200::Chain& c, double* d) {
  const int J = c.dim - 2;
  const double e = exp(-2.0 * c.q[1]);
  for (int j = c.lane; j < J; j += 32) d[2 + j] = e + 1.0 / (c.aux[j] * c.aux[j]);
  if (c.lane == 0) {
    d[0] = 1.0 / c.params[0] + J * e;
    d[1] = 1.0 + 2.0 * J;
  }
}
__device__ void vjp_metric_diagonal(const mb200::Chain& c, const double* w, double* out) {
  const int J = c.dim - 2;
  double s = 0.0;
  for (int j = c.lane; j < J; j += 32) s += w[2 + j];
  s = c.sum(s);
  const double e = exp(-2.0 * c.q[1]);
  for (int i = c.lane; i < c.dim; i += 32) out[i] = (i == 1) ? -2.0 * e * (J * w[0] + s) : 0.0;
}
"""


class EightSchools:
    """NumPy twin of EIGHT_SCHOOLS."""

    def __init__(self, y, sigma, v0):
        self.y, self.sigma, self.v0 = np.asarray(y, float), np.asarray(sigma, float), float(v0)
        self.dim = len(self.y) + 2

    def neg_log_dens(self, q):
        J = len(self.y)
        mu, lt, th = q[0], q[1], q[2:]
        e = np.exp(-2.0 * lt)
        r, u = th - mu, self.y - th
        s = np.sum(0.5 * (r * r) * e + u * u / (2.0 * (self.sigma * self.sigma)))
        return mu * mu / (2.0 * self.v0) + 0.5 * (lt * lt) + J * lt + s

    def grad_neg_log_dens(self, q):
        J = len(self.y)
        mu, lt, th = q[0], q[1], q[2:]
        e = np.exp(-2.0 * lt)
        r = th - mu
        g = np.empty_like(q)
        g[2:] = r * e + (th - self.y) / (self.sigma * self.sigma)
        g[0] = mu / self.v0 - np.sum(r) * e
        g[1] = lt - np.sum(r * r) * e + J
        return g


class EightSchoolsFisher:
    """NumPy twin of EIGHT_SCHOOLS_FISHER."""

    kind = "diagonal"

    def __init__(self, sigma, v0):
        self.sigma, self.v0 = np.asarray(sigma, float), float(v0)

    def metric_func(self, q):
        J = len(self.sigma)
        e = np.exp(-2.0 * q[1])
        d = np.empty_like(q)
        d[2:] = e + 1.0 / (self.sigma * self.sigma)
        d[0] = 1.0 / self.v0 + J * e
        d[1] = 1.0 + 2.0 * J
        return d

    def vjp_metric_func(self, q):
        J = len(self.sigma)

        def vjp(w):
            out = np.zeros_like(q)
            out[1] = -2.0 * np.exp(-2.0 * q[1]) * (J * w[0] + np.sum(w[2:]))
            return out

        return vjp


# Bayesian logistic regression, N data rows x_n in R^D, labels y_n in {0, 1}, prior N(0, v0 I):
#   l = sum_n [log1p(exp(z_n)) - y_n z_n] + |q|^2 / (2 v0),  z = X q
# params (both): (v0, N); target aux: [X (N x D, row-major) | y (N)]; metric aux: X.
# Fisher diagonal d_k = sum_n x_nk^2 s_n (1 - s_n) + 1/v0, s = sigmoid(z); its VJP
#   out_j = sum_n s_n (1 - s_n) (1 - 2 s_n) (sum_k w_k x_nk^2) x_nj
# needs two warp reductions per data row.
LOGISTIC = r"""
__device__ double neg_log_dens(const mb200::Chain& c) {
  const int N = (int)c.params[1];
  const double* X = c.aux;
  double qq = 0.0;
  for (int k = c.lane; k < c.dim; k += 32) qq += c.q[k] * c.q[k];
  double l = c.sum(qq) / (2.0 * c.params[0]);
  for (int n = 0; n < N; ++n) {
    double z = 0.0;
    for (int k = c.lane; k < c.dim; k += 32) z += X[n * c.dim + k] * c.q[k];
    z = c.sum(z);
    l += log1p(exp(z)) - c.aux[N * c.dim + n] * z;
  }
  return l;
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const int N = (int)c.params[1];
  const double* X = c.aux;
  for (int k = c.lane; k < c.dim; k += 32) g[k] = c.q[k] / c.params[0];
  for (int n = 0; n < N; ++n) {
    double z = 0.0;
    for (int k = c.lane; k < c.dim; k += 32) z += X[n * c.dim + k] * c.q[k];
    z = c.sum(z);
    const double r = 1.0 / (1.0 + exp(-z)) - c.aux[N * c.dim + n];
    for (int k = c.lane; k < c.dim; k += 32) g[k] += r * X[n * c.dim + k];
  }
}
"""
LOGISTIC_FISHER = r"""
__device__ void metric_diagonal(const mb200::Chain& c, double* d) {
  const int N = (int)c.params[1];
  const double* X = c.aux;
  for (int k = c.lane; k < c.dim; k += 32) d[k] = 0.0;
  for (int n = 0; n < N; ++n) {
    double z = 0.0;
    for (int k = c.lane; k < c.dim; k += 32) z += X[n * c.dim + k] * c.q[k];
    z = c.sum(z);
    const double s = 1.0 / (1.0 + exp(-z)), v = s * (1.0 - s);
    for (int k = c.lane; k < c.dim; k += 32) d[k] += X[n * c.dim + k] * X[n * c.dim + k] * v;
  }
  for (int k = c.lane; k < c.dim; k += 32) d[k] += 1.0 / c.params[0];
}
__device__ void vjp_metric_diagonal(const mb200::Chain& c, const double* w, double* out) {
  const int N = (int)c.params[1];
  const double* X = c.aux;
  for (int j = c.lane; j < c.dim; j += 32) out[j] = 0.0;
  for (int n = 0; n < N; ++n) {
    double z = 0.0, a = 0.0;
    for (int k = c.lane; k < c.dim; k += 32) {
      const double x = X[n * c.dim + k];
      z += x * c.q[k];
      a += w[k] * (x * x);
    }
    z = c.sum(z);
    a = c.sum(a);
    const double s = 1.0 / (1.0 + exp(-z)), coef = s * (1.0 - s) * (1.0 - 2.0 * s) * a;
    for (int j = c.lane; j < c.dim; j += 32) out[j] += coef * X[n * c.dim + j];
  }
}
"""


class Logistic:
    """NumPy twin of LOGISTIC."""

    def __init__(self, X, y, v0):
        self.X, self.y, self.v0 = np.asarray(X, float), np.asarray(y, float), float(v0)
        self.dim = self.X.shape[1]

    def neg_log_dens(self, q):
        z = self.X @ q
        return (q @ q) / (2.0 * self.v0) + np.sum(np.log1p(np.exp(z)) - self.y * z)

    def grad_neg_log_dens(self, q):
        z = self.X @ q
        return q / self.v0 + self.X.T @ (1.0 / (1.0 + np.exp(-z)) - self.y)


class LogisticFisher:
    """NumPy twin of LOGISTIC_FISHER."""

    kind = "diagonal"

    def __init__(self, X, v0):
        self.X, self.v0 = np.asarray(X, float), float(v0)

    def metric_func(self, q):
        s = 1.0 / (1.0 + np.exp(-(self.X @ q)))
        return (self.X * self.X).T @ (s * (1.0 - s)) + 1.0 / self.v0

    def vjp_metric_func(self, q):
        s = 1.0 / (1.0 + np.exp(-(self.X @ q)))

        def vjp(w):
            a = (self.X * self.X) @ w
            return self.X.T @ (s * (1.0 - s) * (1.0 - 2.0 * s) * a)

        return vjp


# Multivariate Student-t with nu degrees of freedom (params (nu,) in both):
#   l = (nu + D)/2 log(1 + |q|^2/nu),  s(q) = (nu + D) / (nu + |q|^2)
STUDENT_T = r"""
__device__ double qq(const mb200::Chain& c) {
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) s += c.q[i] * c.q[i];
  return c.sum(s);
}
__device__ double neg_log_dens(const mb200::Chain& c) {
  const double nu = c.params[0];
  return 0.5 * (nu + c.dim) * log1p(qq(c) / nu);
}
__device__ void grad_neg_log_dens(const mb200::Chain& c, double* g) {
  const double nu = c.params[0], f = (nu + c.dim) / (nu + qq(c));
  for (int i = c.lane; i < c.dim; i += 32) g[i] = f * c.q[i];
}
"""
STUDENT_T_SCALAR = r"""
__device__ double sq(const mb200::Chain& c) {
  double s = 0.0;
  for (int i = c.lane; i < c.dim; i += 32) s += c.q[i] * c.q[i];
  return c.sum(s);
}
__device__ double metric_scalar(const mb200::Chain& c) {
  return (c.params[0] + c.dim) / (c.params[0] + sq(c));
}
__device__ void vjp_metric_scalar(const mb200::Chain& c, double w, double* out) {
  const double r = c.params[0] + sq(c), f = -2.0 * (c.params[0] + c.dim) / (r * r) * w;
  for (int i = c.lane; i < c.dim; i += 32) out[i] = f * c.q[i];
}
"""


class StudentT:
    """NumPy twin of STUDENT_T."""

    def __init__(self, dim, nu):
        self.dim, self.nu = int(dim), float(nu)

    def neg_log_dens(self, q):
        return 0.5 * (self.nu + self.dim) * np.log1p((q @ q) / self.nu)

    def grad_neg_log_dens(self, q):
        return (self.nu + self.dim) / (self.nu + q @ q) * q


class StudentTScalar:
    """NumPy twin of STUDENT_T_SCALAR."""

    kind = "scalar"

    def __init__(self, dim, nu):
        self.dim, self.nu = int(dim), float(nu)

    def metric_func(self, q):
        return (self.nu + self.dim) / (self.nu + q @ q)

    def vjp_metric_func(self, q):
        r = self.nu + q @ q
        return lambda w: -2.0 * (self.nu + self.dim) / (r * r) * w * q


def _eight_schools_data():
    y = np.array([28.0, 8.0, -3.0, 7.0, -1.0, 1.0, 18.0, 12.0])
    sigma = np.array([15.0, 10.0, 16.0, 11.0, 9.0, 11.0, 10.0, 18.0])
    return y, sigma


def _logistic_data(n=40, dim=25, seed=20261017):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, dim)) / np.sqrt(dim)
    beta = rng.standard_normal(dim)
    y = (rng.uniform(size=n) < 1.0 / (1.0 + np.exp(-(X @ beta)))).astype(float)
    return X, y


def ur_model(name):
    """``(NumPy target, NumPy metric, (target source, params, aux), (metric kind, source, params,
    aux))`` of a model the registry cannot express."""
    if name == "eight_schools":
        y, sigma = _eight_schools_data()
        v0 = 25.0
        return (EightSchools(y, sigma, v0), EightSchoolsFisher(sigma, v0),
                (EIGHT_SCHOOLS, (v0,), np.concatenate([y, sigma])),
                ("diagonal", EIGHT_SCHOOLS_FISHER, (v0,), sigma))
    if name == "logistic":
        X, y = _logistic_data()
        v0 = 4.0
        return (Logistic(X, y, v0), LogisticFisher(X, v0),
                (LOGISTIC, (v0, X.shape[0]), np.concatenate([X.ravel(), y])),
                ("diagonal", LOGISTIC_FISHER, (v0, X.shape[0]), X.ravel().copy()))
    if name == "student_t":
        dim, nu = 6, 5.0
        return (StudentT(dim, nu), StudentTScalar(dim, nu), (STUDENT_T, (nu,), None),
                ("scalar", STUDENT_T_SCALAR, (nu,), None))
    raise KeyError(name)


UR_MODELS = ("eight_schools", "logistic", "student_t")
