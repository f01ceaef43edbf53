"""Synthetic benchmark / parity problems (SURVEY.md section 8(d), BASELINE.json configs).

Host-side *input generation* only: shapes, seeds, shared metrics and initial states for the
five configurations C0..C4.  Everything is fp64 and generated with
``numpy.random.default_rng(BASE_SEED + k)`` so that the CUDA path, the oracle and the
reference all see identical inputs.  No integrator arithmetic lives here.
"""

from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

BASE_SEED = 20260924


@dataclass
class Problem:
    """A fully specified integrator workload.

    Attributes:
        name: config label (``"C0"`` .. ``"C4"``).
        integrator: ``"leapfrog"`` | ``"implicit_leapfrog"`` | ``"constrained_leapfrog"``.
        system: ``"euclidean"`` | ``"softabs_riemannian"`` | ``"dense_riemannian"`` |
            ``"diagonal_riemannian"`` | ``"scalar_riemannian"`` | ``"cholesky_riemannian"`` |
            ``"constrained_euclidean"`` | ``"gaussian_constrained_euclidean"``.
        target: target-model name (``mici_b200.targets`` registry key).
        target_params: constructor kwargs of the target model.
        metric: ``None`` (identity), 1-D (diagonal) or 2-D (dense SPD) array -- the fixed
            metric of Euclidean systems.
        metric_model / metric_params: position-dependent metric (dense, diagonal, scalar and
            Cholesky-factored Riemannian systems).
        step_size: integrator ``step_size``.
        pos, mom: ``[n_chains, dim]`` initial states.
    """

    name: str
    integrator: str
    system: str
    target: str
    target_params: dict
    step_size: float
    pos: np.ndarray
    mom: np.ndarray
    metric: np.ndarray | None = None
    metric_model: str | None = None
    metric_params: dict = field(default_factory=dict)
    system_kwargs: dict = field(default_factory=dict)
    integrator_kwargs: dict = field(default_factory=dict)

    @property
    def n_chains(self):
        return self.pos.shape[0]

    @property
    def dim(self):
        return self.pos.shape[1]

    @property
    def algorithmic_bytes_per_chain_step(self):
        """B_alg = 4 * D * 8: read q, p and write q, p in fp64 (SURVEY.md 8(d))."""
        return 32 * self.dim


def dense_spd_metric(rng, dim):
    """M = A A^T / D + I with A_ij ~ N(0, 1): condition number ~5."""
    a = rng.standard_normal((dim, dim))
    return a @ a.T / dim + np.identity(dim)


def c0_std_gaussian(n_chains=4, dim=10, seed=BASE_SEED + 0):
    rng = np.random.default_rng(seed)
    return Problem(
        name="C0",
        integrator="leapfrog",
        system="euclidean",
        target="std_gaussian",
        target_params={"dim": dim},
        step_size=0.1,
        pos=rng.standard_normal((n_chains, dim)),
        mom=rng.standard_normal((n_chains, dim)),
    )


def c1_funnel(n_chains=8192, dim=128, seed=BASE_SEED + 1, metric_kind="dense",
              integrator="leapfrog"):
    rng = np.random.default_rng(seed)
    metric = dense_spd_metric(rng, dim)
    pos = 0.1 * rng.standard_normal((n_chains, dim))
    z = rng.standard_normal((n_chains, dim))
    if metric_kind == "dense":
        mom = z @ np.linalg.cholesky(metric).T  # p0 = L z per chain
    elif metric_kind == "diagonal":
        metric = np.ascontiguousarray(metric.diagonal())
        mom = z * np.sqrt(metric)
    else:
        metric = None
        mom = z
    return Problem(
        name="C1",
        integrator=integrator,
        system="euclidean",
        target="neal_funnel",
        target_params={"dim": dim},
        step_size=0.01,
        pos=pos,
        mom=mom,
        metric=metric,
    )


def g1_gaussian_split(n_chains=256, dim=32, seed=BASE_SEED + 6, metric_kind="dense",
                      integrator="leapfrog", target="banana"):
    """Extra parity case for row N4: ``GaussianEuclideanMetricSystem`` (systems.py:369-474) --
    the registered target is the density relative to the standard Gaussian measure, the
    drift is the exact rotation in the eigenbasis of the metric."""
    rng = np.random.default_rng(seed)
    metric = dense_spd_metric(rng, dim)
    pos = 0.7 * rng.standard_normal((n_chains, dim))
    z = rng.standard_normal((n_chains, dim))
    if metric_kind == "dense":
        mom = z @ np.linalg.cholesky(metric).T
    elif metric_kind == "diagonal":
        metric = np.ascontiguousarray(metric.diagonal())
        mom = z * np.sqrt(metric)
    else:
        metric = None
        mom = z
    params = {"dim": dim, "b": 0.5} if target == "banana" else {"dim": dim}
    return Problem(
        name="G1",
        integrator=integrator,
        system="gaussian_euclidean",
        target=target,
        target_params=params,
        step_size=0.15,
        pos=pos,
        mom=mom,
        metric=metric,
    )


def c2_softabs_banana(n_chains=2048, dim=64, seed=BASE_SEED + 2, integrator="implicit_leapfrog"):
    rng = np.random.default_rng(seed)
    return Problem(
        name="C2",
        integrator=integrator,
        system="softabs_riemannian",
        target="banana",
        target_params={"dim": dim, "b": 0.5},
        step_size=0.1,
        pos=0.5 * rng.standard_normal((n_chains, dim)),
        mom=rng.standard_normal((n_chains, dim)),
        system_kwargs={"softabs_coeff": 1.0},
    )


def c6_softabs_quartic(n_chains=2048, dim=64, seed=BASE_SEED + 9, gamma=1.0,
                       integrator="implicit_leapfrog"):
    """C2's system (SoftAbs metric, implicit leapfrog) on a target with a DENSE Hessian:
    l = |q|^2/2 + (gamma/4) sum_m (a_m . q)^4 with D random directions.  The banana of C2 has a
    2 x 2 block-diagonal Hessian that a Jacobi eigensolver diagonalises in one round; this target
    needs every rotation of every sweep."""
    rng = np.random.default_rng(seed)
    directions = rng.standard_normal((dim, dim)) / np.sqrt(dim)
    return Problem(
        name="C6",
        integrator=integrator,
        system="softabs_riemannian",
        target="quartic",
        target_params={"directions": directions, "gamma": gamma},
        step_size=0.1,
        pos=0.5 * rng.standard_normal((n_chains, dim)),
        mom=rng.standard_normal((n_chains, dim)),
        system_kwargs={"softabs_coeff": 1.0},
    )


def c3_torus(n_chains=4096, seed=BASE_SEED + 3, R=1.0, r=0.5, alpha=0.9,
             dens_wrt_hausdorff=True):
    rng = np.random.default_rng(seed)
    theta, phi = rng.uniform(0, 2 * np.pi, size=(2, n_chains))
    pos = np.stack(
        [
            (R + r * np.cos(phi)) * np.cos(theta),
            (R + r * np.cos(phi)) * np.sin(theta),
            r * np.sin(phi),
        ],
        -1,
    )
    mom = rng.standard_normal((n_chains, 3))
    # project the initial momentum onto the cotangent space (identity metric):
    # p -= J^T (J J^T)^-1 J p with J = [2(rho-R)x/rho, 2(rho-R)y/rho, 2z]
    rho = np.sqrt(pos[:, 0] ** 2 + pos[:, 1] ** 2)
    f = 2.0 * (rho - R) / rho
    jac = np.stack([f * pos[:, 0], f * pos[:, 1], 2.0 * pos[:, 2]], -1)
    mom = mom - jac * ((jac * mom).sum(-1) / (jac * jac).sum(-1))[:, None]
    return Problem(
        name="C3",
        integrator="constrained_leapfrog",
        system="constrained_euclidean",
        target="torus",
        target_params={"R": R, "r": r, "alpha": alpha},
        step_size=0.1,
        pos=pos,
        mom=mom,
        integrator_kwargs={"n_inner_step": 1},
        system_kwargs={"dens_wrt_hausdorff": dens_wrt_hausdorff},
    )


def c4_dense_riemannian(n_chains=8192, dim=512, seed=BASE_SEED + 4, coeff=0.1,
                        integrator="implicit_leapfrog"):
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((dim, dim))
    prec = np.identity(dim) + 0.1 * (g @ g.T) / dim
    base = dense_spd_metric(rng, dim)
    pos = 0.5 * rng.standard_normal((n_chains, dim))
    mom = rng.standard_normal((n_chains, dim)) @ np.linalg.cholesky(base).T
    return Problem(
        name="C4",
        integrator=integrator,
        system="dense_riemannian",
        target="quadratic",
        target_params={"prec": prec},
        step_size=0.05,
        pos=pos,
        mom=mom,
        metric_model="rank1",
        metric_params={"base": base, "coeff": coeff},
    )


def c5_dense_hadamard(n_chains=8192, dim=512, seed=BASE_SEED + 7, coeff=0.1,
                      integrator="implicit_leapfrog"):
    """C4's system with a metric that has NO low-rank structure: M(q) = B + c (q q^T) o S.  The
    quadratic target and the SPD matrices are generated like C4's; the metric can only be handled
    by the generic dense path (per-chain Cholesky + explicit inverse + dense VJP)."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((dim, dim))
    prec = np.identity(dim) + 0.1 * (g @ g.T) / dim
    base = dense_spd_metric(rng, dim)
    scale = dense_spd_metric(rng, dim)
    pos = 0.5 * rng.standard_normal((n_chains, dim))
    mom = rng.standard_normal((n_chains, dim)) @ np.linalg.cholesky(base).T
    return Problem(
        name="C5",
        integrator=integrator,
        system="dense_riemannian",
        target="quadratic",
        target_params={"prec": prec},
        step_size=0.05,
        pos=pos,
        mom=mom,
        metric_model="hadamard",
        metric_params={"base": base, "scale": scale, "coeff": coeff},
    )


def funnel_fisher_diagonal(q):
    """The funnel's expected Fisher information d(q) = [1/9 + (D-1)/2, e^-v, ..., e^-v] for a
    batch ``q`` [n, D] (the metric of ``mici_b200.targets.FunnelFisherMetric``)."""
    d = np.empty_like(q)
    d[:, 0] = 1.0 / 9.0 + 0.5 * (q.shape[1] - 1)
    d[:, 1:] = np.exp(-q[:, :1])
    return d


def c7_funnel_riemannian(n_chains=8192, dim=128, seed=BASE_SEED + 10, metric_kind="fisher",
                         integrator="implicit_leapfrog"):
    """The funnel of C1 on a Riemannian system with an O(D) position-dependent metric:
    ``metric_kind="fisher"`` -- ``DiagonalRiemannianMetricSystem`` with the funnel's expected
    Fisher information; ``"scalar"`` -- ``ScalarRiemannianMetricSystem`` with s = 1 + |q|^2 / D.
    Momenta are drawn from N(0, M(q)) at the initial positions.  Step sizes chosen on the CPU
    oracle (10 steps): Fisher 0.2 -- all of the first 256 chains complete, median |h error| 1.9;
    scalar 0.05 -- all of the first 64 complete, median |h error| 0.8 (at 0.1 the median error is
    250 and at 0.2 only 84 % complete: one scale for all coordinates cannot follow the funnel's
    neck)."""
    rng = np.random.default_rng(seed)
    pos = 0.5 * rng.standard_normal((n_chains, dim))
    z = rng.standard_normal((n_chains, dim))
    if metric_kind == "fisher":
        system, model, params = "diagonal_riemannian", "funnel_fisher", {}
        mom = z * np.sqrt(funnel_fisher_diagonal(pos))
    elif metric_kind == "scalar":
        system, model, params = "scalar_riemannian", "scalar_quadratic", {"a": 1.0, "b": 1.0 / dim}
        mom = z * np.sqrt(1.0 + (pos * pos).sum(1) / dim)[:, None]
    else:
        raise ValueError(metric_kind)
    return Problem(
        name="C7",
        integrator=integrator,
        system=system,
        target="neal_funnel",
        target_params={"dim": dim},
        step_size=0.2 if metric_kind == "fisher" else 0.05,
        pos=pos,
        mom=mom,
        metric_model=model,
        metric_params=params,
    )


def chol_quadratic_factor(pos, base_factor, coeff):
    """L(q) = L0 + c tril(q q^T) for a batch ``pos`` [n, D] (the factor of
    ``mici_b200.targets.QuadraticCholeskyMetric``), [n, D, D]."""
    return base_factor + coeff * np.tril(pos[:, :, None] * pos[:, None, :])


def c8_cholesky_riemannian(n_chains=8192, dim=128, seed=BASE_SEED + 11, coeff=None,
                           integrator="implicit_leapfrog", step_size=0.1):
    """``CholeskyFactoredRiemannianMetricSystem`` on the quadratic target of C4 (precision
    P = I + 0.1 G G^T / D, generated the same way): L(q) = chol(P) + c tril(q q^T) with
    c = 1/D, so M(0) = P, the target's Fisher information.  Momenta are drawn from N(0, M(q))
    at the initial positions (p = L(q) z).  Step size chosen on the CPU oracle (10 steps, first
    64 chains, every chain completing at each size): 0.1 -- median |h error| 0.037, 6.8
    fixed-point iterations per solve; 0.2 -- 0.023, 8.3; 0.4 -- 0.18, 11.0.  0.1 is the
    largest size at which the solves stay below 7 iterations."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((dim, dim))
    prec = np.identity(dim) + 0.1 * (g @ g.T) / dim
    base = np.linalg.cholesky(prec)
    coeff = 1.0 / dim if coeff is None else float(coeff)
    pos = 0.5 * rng.standard_normal((n_chains, dim))
    z = rng.standard_normal((n_chains, dim))
    # L(q) z = L0 z + c q o cumsum(q o z): the rows of tril(q q^T) z
    mom = z @ base.T + coeff * pos * np.cumsum(pos * z, axis=1)
    return Problem(
        name="C8",
        integrator=integrator,
        system="cholesky_riemannian",
        target="quadratic",
        target_params={"prec": prec},
        step_size=step_size,
        pos=pos,
        mom=mom,
        metric_model="chol_quadratic",
        metric_params={"base_factor": base, "coeff": coeff},
    )


def sphere_constrained(n_chains=64, dim=10, seed=BASE_SEED + 5, metric_kind="dense",
                       dens_wrt_hausdorff=True):
    """Extra parity case for K6 beyond C3: unit sphere in R^dim, tilted Gaussian density,
    optional diagonal / dense metric (exercises the general-dimension constrained path)."""
    rng = np.random.default_rng(seed)
    pos = rng.standard_normal((n_chains, dim))
    pos /= np.linalg.norm(pos, axis=1, keepdims=True)
    mom = rng.standard_normal((n_chains, dim))
    if metric_kind == "dense":
        metric = dense_spd_metric(rng, dim)
    elif metric_kind == "diagonal":
        metric = rng.uniform(0.5, 2.0, dim)
    else:
        metric = None
    # project the momentum onto the cotangent space: p -= J^T (J M^-1 J^T)^-1 J M^-1 p, J = 2 q^T
    if metric is None:
        minv_j = pos
        minv_p = mom
    elif metric.ndim == 1:
        minv_j = pos / metric
        minv_p = mom / metric
    else:
        minv = np.linalg.inv(metric)
        minv_j = pos @ minv
        minv_p = mom @ minv
    lam = (pos * minv_p).sum(-1) / (pos * minv_j).sum(-1)
    mom = mom - lam[:, None] * pos
    return Problem(
        name="S1",
        integrator="constrained_leapfrog",
        system="constrained_euclidean",
        target="sphere",
        target_params={"dim": dim},
        step_size=0.2,
        pos=pos,
        mom=mom,
        metric=metric,
        integrator_kwargs={"n_inner_step": 1},
        system_kwargs={"dens_wrt_hausdorff": dens_wrt_hausdorff},
    )


def multi_sphere_constrained(n_chains=32, dim=16, n_constr=4, seed=BASE_SEED + 8,
                             metric_kind="dense", dens_wrt_hausdorff=True):
    """Extra parity case for K6 with SEVERAL constraints (C = n_constr <= 8): consecutive blocks
    of dim / n_constr coordinates each on their unit sphere; with a dense metric the Gram matrix
    and the Newton residual Jacobian are full C x C matrices."""
    rng = np.random.default_rng(seed)
    block = dim // n_constr
    pos = rng.standard_normal((n_chains, n_constr, block))
    pos /= np.linalg.norm(pos, axis=2, keepdims=True)
    pos = pos.reshape(n_chains, dim)
    mom = rng.standard_normal((n_chains, dim))
    if metric_kind == "dense":
        metric = dense_spd_metric(rng, dim)
        minv = np.linalg.inv(metric)
    elif metric_kind == "diagonal":
        metric = rng.uniform(0.5, 2.0, dim)
        minv = np.diag(1.0 / metric)
    else:
        metric = None
        minv = np.identity(dim)
    for i in range(n_chains):  # p -= J^T (J M^-1 J^T)^-1 J M^-1 p
        jac = np.zeros((n_constr, dim))
        for k in range(n_constr):
            jac[k, k * block:(k + 1) * block] = 2.0 * pos[i, k * block:(k + 1) * block]
        gram = jac @ minv @ jac.T
        mom[i] -= jac.T @ np.linalg.solve(gram, jac @ (minv @ mom[i]))
    return Problem(
        name="S2",
        integrator="constrained_leapfrog",
        system="constrained_euclidean",
        target="multi_sphere",
        target_params={"dim": dim, "n_constr": n_constr},
        step_size=0.15,
        pos=pos,
        mom=mom,
        metric=metric,
        integrator_kwargs={"n_inner_step": 1},
        system_kwargs={"dens_wrt_hausdorff": dens_wrt_hausdorff},
    )


def c9_gaussian_constrained(n_chains=8192, dim=128, n_constr=8, seed=BASE_SEED + 12,
                            step_size=0.1):
    """C9: GaussianDenseConstrainedEuclideanMetricSystem on the multi-sphere target, C = 8,
    D = 128, dense metric, Newton projection; start states on the manifold with projected momenta
    as in ``multi_sphere_constrained``.  Step size 0.1, chosen on the CPU oracle: every step of the
    reference fixture at this shape (gc_multi_sphere_c8_dense_d128, 3 chains, 5 steps) and of the
    C = 8, D = 32 fixture (8 chains, 20 steps) converges."""
    base = multi_sphere_constrained(n_chains=n_chains, dim=dim, n_constr=n_constr, seed=seed,
                                    metric_kind="dense")
    base.name = "C9"
    base.system = "gaussian_constrained_euclidean"
    base.system_kwargs = {}
    base.step_size = step_size
    return base


CONFIGS = {
    "C0": c0_std_gaussian,
    "C1": c1_funnel,
    "C2": c2_softabs_banana,
    "C3": c3_torus,
    "C4": c4_dense_riemannian,
    "C5": c5_dense_hadamard,
    "C6": c6_softabs_quartic,
    "C7": c7_funnel_riemannian,
    "C8": c8_cholesky_riemannian,
    "C9": c9_gaussian_constrained,
    "S1": sphere_constrained,
    "S2": multi_sphere_constrained,
    "G1": g1_gaussian_split,
}


def make_problem(name, **kwargs):
    """Build config ``name`` (``"C0"``..``"C4"``), optionally overriding sizes/seed."""
    return CONFIGS[name](**kwargs)
