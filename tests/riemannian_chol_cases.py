"""TEST INFRASTRUCTURE ONLY -- the NumPy oracle and the reference fixtures of the
Cholesky-factored Riemannian-metric system (``CholeskyFactoredRiemannianMetricSystem``,
reference systems.py:1574-1653).

* ``CholeskyFactoredMetricValue``: ``TriangularFactoredPositiveDefiniteMatrix(L,
  factor_is_lower=True)`` arithmetic (reference matrices.py:795-1114), expression for expression.
* ``QuadraticChol``: the NumPy model L(q) = L0 + c tril(q q^T) with the explicit VJP callable
  the reference takes.
* ``patched_drivers()``: makes ``oracle.drivers`` (oracle and reference runners, HMC / NUTS /
  staged sampling) handle the system ``"cholesky_riemannian"``; the oracle's implicit
  integrators, solvers and transitions are used unchanged.
* Case tables kept apart from the other fixtures'; ``OPENBLAS_NUM_THREADS=1 python
  tests/riemannian_chol_cases.py`` regenerates the ``rc_*.npz`` fixtures from the unmodified
  reference.
"""

from __future__ import annotations

import contextlib
import os
import sys

import numpy as np
import scipy.linalg as sla

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mici_b200 import problems as pb  # noqa: E402
from oracle import drivers as dr  # noqa: E402
from oracle import mici_oracle as mo  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
SYSTEM = "cholesky_riemannian"


# -------------------------------------------------------------------------- metric value


class CholeskyFactoredMetricValue:
    """``TriangularFactoredPositiveDefiniteMatrix(L, factor_is_lower=True)``."""

    def __init__(self, factor):
        # TriangularMatrix: _make_array_triangular (:795-797, :821), then
        # ExplicitArrayMatrix.__init__'s asarray_chkfinite -> LinAlgError (:207-215)
        self.factor = mo._chkfinite(np.tril(factor))

    @property
    def log_abs_det(self):  # 2 * factor.log_abs_det (:982-984, :850-852)
        return 2 * np.log(np.abs(self.factor.diagonal())).sum()

    def _inv_factor_matvec(self, v):  # L.inv @ v (InverseTriangularMatrix, :897-903)
        return sla.solve_triangular(self.factor, v, lower=True, check_finite=False)

    def inv_matvec(self, v):
        # inv = TriangularFactoredPositiveDefiniteMatrix(factor=L.inv.T) (:1110-1111);
        # inv @ v = inv.factor @ (inv.factor.T @ v) (:1042-1043)
        return sla.solve_triangular(self.factor.T, self._inv_factor_matvec(v), lower=False,
                                    check_finite=False)

    def sqrt_matvec(self, v):  # sqrt is the factor itself (:1113-1114)
        return self.factor @ v

    @property
    def grad_log_abs_det(self):  # :1048-1050
        return np.diag(2 / self.factor.diagonal())

    def grad_quadratic_form_inv(self, v):  # :1052-1058
        inv_factor_vector = self._inv_factor_matvec(v)
        inv_vector = self.inv_matvec(v)
        return np.tril(-2 * np.outer(inv_vector, inv_factor_vector))  # sign = 1


# -------------------------------------------------------------------------- metric model


class QuadraticChol:
    """L(q) = L0 + c tril(q q^T), VJP V -> c (V q + V^T q)."""

    def __init__(self, base_factor, coeff):
        self.base_factor = np.asarray(base_factor, dtype=np.float64)
        self.coeff = float(coeff)

    def metric_func(self, q):
        return self.base_factor + self.coeff * np.tril(np.outer(q, q))

    def vjp_metric_func(self, q):
        c = self.coeff
        return lambda V: c * (V @ q + V.T @ q)


def metric_model(problem):
    return QuadraticChol(**problem.metric_params)


class OracleSystem(mo.RiemannianSystem):
    """``mo.RiemannianSystem`` with a Cholesky-factored metric value."""

    def __init__(self, target, model):
        super().__init__(target, "cholesky", metric_model=model)

    def metric(self, q):
        self.n_metric_evals += 1
        return CholeskyFactoredMetricValue(self.metric_model.metric_func(q))

    def vjp(self, q):
        return self.metric_model.vjp_metric_func(q)


# ------------------------------------------------------------------ drivers extension

_ORIG_STEP_FN = dr.oracle_step_fn
_ORIG_BUILD_REFERENCE = dr.build_reference


def oracle_step_fn(problem, counts=None, **overrides):
    if problem.system != SYSTEM:
        return _ORIG_STEP_FN(problem, counts=counts, **overrides)
    system = OracleSystem(dr.build_target(problem), metric_model(problem))
    ikw = dict(problem.integrator_kwargs)
    ikw.update(overrides)
    eps = problem.step_size
    fn = (mo.implicit_midpoint_step if problem.integrator == "implicit_midpoint"
          else mo.implicit_leapfrog_step)

    def step(q, p, d):
        c = {} if counts is None else counts
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            out = fn(q, p, d * eps, system, counts=c, **ikw)
        if counts is not None:
            counts.setdefault("all_fp_iters", []).append(list(c.get("fp_iters", [])))
        return out

    return step, system.h, system


def build_reference(problem, **overrides):
    if problem.system != SYSTEM:
        return _ORIG_BUILD_REFERENCE(problem, **overrides)
    mici = dr.import_reference()
    target = dr.build_target(problem)
    model = metric_model(problem)
    system = mici.systems.CholeskyFactoredRiemannianMetricSystem(
        neg_log_dens=target.neg_log_dens, metric_chol_func=model.metric_func,
        vjp_metric_chol_func=model.vjp_metric_func, grad_neg_log_dens=target.grad_neg_log_dens)
    ikw = dict(problem.integrator_kwargs)
    ikw.update(overrides)
    if isinstance(ikw.get("fixed_point_solver"), str):
        ikw["fixed_point_solver"] = getattr(mici.solvers,
                                            "solve_fixed_point_" + ikw["fixed_point_solver"])
    cls = {"implicit_leapfrog": mici.integrators.ImplicitLeapfrogIntegrator,
           "implicit_midpoint": mici.integrators.ImplicitMidpointIntegrator}[problem.integrator]
    return system, cls(system, problem.step_size, **ikw)


@contextlib.contextmanager
def patched_drivers():
    """``oracle.drivers`` runners that also build the Cholesky-factored system."""
    prev = dr.oracle_step_fn, dr.build_reference
    dr.oracle_step_fn, dr.build_reference = oracle_step_fn, build_reference
    try:
        yield dr
    finally:
        dr.oracle_step_fn, dr.build_reference = prev


# -------------------------------------------------------------------------- problems


def make_problem(target, dim, n_chains, step_size, seed, coeff=None, integrator="implicit_leapfrog",
                 pos_scale=0.5, integrator_kwargs=None, base_factor=None, pos=None):
    """A small Cholesky-factored problem: L0 the Cholesky factor of a random SPD matrix (unless
    given), c = 1/D (unless given), positions ``pos_scale * N(0, I)`` (unless given), momenta
    p = L(q) z.  The quadratic target's precision is generated like C4's."""
    rng = np.random.default_rng(seed)
    tparams = {"dim": dim}
    if target == "banana":
        tparams["b"] = 0.5
    elif target == "quadratic":
        g = rng.standard_normal((dim, dim))
        tparams = {"prec": np.identity(dim) + 0.1 * (g @ g.T) / dim}
    if base_factor is None:
        base_factor = np.linalg.cholesky(pb.dense_spd_metric(rng, dim))
    coeff = 1.0 / dim if coeff is None else float(coeff)
    q = pos_scale * rng.standard_normal((n_chains, dim))
    if pos is not None:
        q = np.array(pos, dtype=np.float64)
    z = rng.standard_normal((n_chains, dim))
    model = QuadraticChol(base_factor, coeff)
    mom = np.stack([np.tril(model.metric_func(q[c])) @ z[c] for c in range(n_chains)])
    return pb.Problem(
        name="RC", integrator=integrator, system=SYSTEM, target=target, target_params=tparams,
        step_size=step_size, pos=q, mom=mom, metric_model="chol_quadratic",
        metric_params={"base_factor": np.asarray(base_factor, dtype=np.float64), "coeff": coeff},
        integrator_kwargs=dict(integrator_kwargs or {}),
    )


def singular_start_positions(n_chains=8, dim=3, seed=pb.BASE_SEED + 70):
    """q0 = +-1 (L00 = -1 + q0^2 = 0 exactly: singular), q0 = +-0.5 (L00 < 0) and |q0| = 2
    (L00 > 0), the other coordinates 0.5 N(0, 1)."""
    q = 0.5 * np.random.default_rng(seed).standard_normal((n_chains, dim))
    q[:, 0] = [1.0, -1.0, 0.5, -0.5, 2.0, -2.0, 1.0, 0.5][:n_chains]
    return q


S = pb.BASE_SEED + 100
# (a step size of 0.02: near L00 = 0 the metric is nearly singular and the dynamics are stiff;
# at 0.1 every negative-diagonal chain fails its first step)
STD3 = dict(target="std_gaussian", dim=3, n_chains=8, step_size=0.02, seed=S + 30,
            base_factor=np.diag([-1.0, 1.0, 1.0]), coeff=1.0, pos=singular_start_positions())
# name: (make_problem kwargs, step counts).  Mixed directions: chain i runs with dir (-1)^i.
CASES = {
    "rc_std_d1": (dict(target="std_gaussian", dim=1, n_chains=8, step_size=0.1, seed=S + 1,
                       coeff=0.5), (1, 5, 20)),
    "rc_banana_d2": (dict(target="banana", dim=2, n_chains=8, step_size=0.1, seed=S + 2,
                          coeff=0.5), (1, 5, 20)),
    "rc_std_d5": (dict(target="std_gaussian", dim=5, n_chains=8, step_size=0.1, seed=S + 3),
                  (1, 5, 20)),
    "rc_banana_d8": (dict(target="banana", dim=8, n_chains=8, step_size=0.1, seed=S + 4),
                     (1, 5, 20)),
    "rc_funnel_d10": (dict(target="neal_funnel", dim=10, n_chains=8, step_size=0.05, seed=S + 5),
                      (1, 5, 20)),
    "rc_std_d33": (dict(target="std_gaussian", dim=33, n_chains=6, step_size=0.1, seed=S + 6),
                   (1, 5, 20)),
    "rc_quadratic_d64": (dict(target="quadratic", dim=64, n_chains=6, step_size=0.1, seed=S + 7),
                         (1, 5, 20)),
    "rc_quadratic_d128": (dict(target="quadratic", dim=128, n_chains=4, step_size=0.1,
                               seed=S + 8), (1, 5, 20)),
    # beyond shared memory: the factor lives in the per-CTA global workspace
    "rc_quadratic_d200": (dict(target="quadratic", dim=200, n_chains=3, step_size=0.1,
                               seed=S + 9), (1, 5)),
    # negative-diagonal, exactly singular and regular starts (L0 = diag(-1, 1, 1), c = 1)
    "rc_std_d3_singular": (STD3, (1, 5, 20)),
    # implicit midpoint and the Steffensen solver
    "rc_banana_d8_midpoint": (dict(target="banana", dim=8, n_chains=8, step_size=0.1, seed=S + 10,
                                   integrator="implicit_midpoint"), (1, 5, 20)),
    "rc_std_d5_steffensen": (dict(target="std_gaussian", dim=5, n_chains=8, step_size=0.1,
                                  seed=S + 11,
                                  integrator_kwargs={"fixed_point_solver": "steffensen"}),
                             (1, 5, 20)),
    "rc_funnel_d10_midpoint_steffensen": (
        dict(target="neal_funnel", dim=10, n_chains=8, step_size=0.05, seed=S + 12,
             integrator="implicit_midpoint",
             integrator_kwargs={"fixed_point_solver": "steffensen"}), (1, 5, 20)),
}
# big steps: chains fail with ConvergenceError and with NonReversibleStepError
FAILURE_CASES = {
    "rc_banana_d8_bigstep": (dict(target="banana", dim=8, n_chains=24, step_size=0.5, seed=S + 13,
                                  pos_scale=1.0, coeff=0.5), (1, 5)),
    "rc_std_d5_bigstep": (dict(target="std_gaussian", dim=5, n_chains=24, step_size=0.9,
                               seed=S + 14, pos_scale=1.0, coeff=0.5), (1, 5)),
}
# static HMC: (problem kwargs, n_iter, n_step, seed)
HMC_CASES = {
    "rc_hmc_banana_d4": (dict(target="banana", dim=4, n_chains=4, step_size=0.15, seed=S + 15),
                         4, 5, 717),
}
# NUTS (DynamicMultinomialHMC's transition): (problem kwargs, n_iter, seed, max_tree_depth)
NUTS_CASES = {
    "rc_nuts_std_d5": (dict(target="std_gaussian", dim=5, n_chains=3, step_size=0.2, seed=S + 16),
                       3, 718, 4),
}
# dual-averaging warm-up + main stage through StaticMetropolisHMC.sample_chains:
# (problem kwargs, n_warm_up_iter, n_main_iter, n_step, seed)
ADAPT_CASES = {
    "rc_adapt_std_d5_dualavg": (dict(target="std_gaussian", dim=5, n_chains=4, step_size=0.15,
                                     seed=S + 17), 10, 3, 3, 719),
}
ADAPT_SPECS = [("dual_averaging", {})]
ALL_INTEGRATOR_CASES = {**CASES, **FAILURE_CASES}


# D x D BLAS mat-vecs (the quadratic target's gradient, the VJP callable) large enough for
# OpenBLAS to split over threads, whose rounding then depends on the thread count BLAS was
# started with: the fixtures are generated with OPENBLAS_NUM_THREADS=1
BLAS_THREADED_CASES = ("rc_quadratic_d128", "rc_quadratic_d200")


def case_problem(name):
    kw = {**ALL_INTEGRATOR_CASES, **{k: (v[0],) for k, v in HMC_CASES.items()},
          **{k: (v[0],) for k, v in NUTS_CASES.items()},
          **{k: (v[0],) for k, v in ADAPT_CASES.items()}}[name][0]
    return make_problem(**kw)


def case_dirs(problem):
    return np.where(np.arange(problem.n_chains) % 2 == 0, 1, -1).astype(np.int32)


def oracle_integrator_run(problem, n_steps, dirs):
    """Oracle run plus the fixed-point iterations of every chain's last completed step."""
    its = np.zeros((problem.n_chains, 4), dtype=np.int32)
    with patched_drivers(), np.errstate(divide="ignore", invalid="ignore"):
        out = dr.oracle_run(problem, n_steps, dirs=dirs)
        for c in range(problem.n_chains):
            if out["n_done"][c] == 0:
                continue
            counts = {}
            step, _, _ = dr.oracle_step_fn(problem, counts=counts)
            q, p = problem.pos[c].copy(), problem.mom[c].copy()
            for _ in range(int(out["n_done"][c])):
                q, p = step(q, p, int(dirs[c]))
            last = counts["all_fp_iters"][-1]
            its[c, :len(last)] = last
    out["fp_iters"] = its
    return out


def load_fixture(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))


def oracle_adapt_run(name):
    """The oracle's staged run of an ``ADAPT_CASES`` entry, through the stages the reference's
    sampler chose (stored with the fixture)."""
    from oracle.make_golden import STAGE_CODES

    names = {code: which for which, code in STAGE_CODES.items()}
    g = load_fixture(name)
    stages = [(int(n), names[int(c)]) for n, c in zip(g["stage_n_iter"], g["stage_which"])]
    _, _, _, n_step, seed = ADAPT_CASES[name]
    with patched_drivers():
        return dr.oracle_sample_chains(case_problem(name), stages, n_step, seed, ADAPT_SPECS)


def generate(names=None):  # pragma: no cover - run by hand against the unmodified reference
    if names:
        from oracle.make_golden import STAGE_CODES, reference_stage_list

        with patched_drivers():
            for name in names:
                _, n_warm, n_main, n_step, seed = ADAPT_CASES[name]
                ref = dr.reference_sample_chains(case_problem(name), n_warm, n_main, n_step, seed,
                                                 ADAPT_SPECS)
                stages = reference_stage_list(ADAPT_SPECS, None, n_warm, n_main)
                np.savez(os.path.join(GOLDEN_DIR, name + ".npz"),
                         stage_n_iter=np.array([n for n, _ in stages]),
                         stage_which=np.array([STAGE_CODES[w] for _, w in stages]), **ref)
                print(name, "step size", float(ref["step_size"]), "n_step", ref["n_step"].tolist())
        return
    generate(list(ADAPT_CASES))
    with patched_drivers(), np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for name, (_, step_counts) in ALL_INTEGRATOR_CASES.items():
            problem = case_problem(name)
            dirs = case_dirs(problem)
            rec = {"step_counts": np.array(step_counts), "dirs": dirs,
                   "step_size": problem.step_size}
            for n in step_counts:
                ref = dr.reference_run(problem, n, dirs=dirs)
                orc = oracle_integrator_run(problem, n, dirs)
                for k in ("pos", "mom", "status", "n_done", "h"):
                    rec[f"{k}_{n}"] = ref[k]
                rec[f"fp_iters_{n}"] = orc["fp_iters"]
                print(name, n, "status", ref["status"].tolist())
            np.savez(os.path.join(GOLDEN_DIR, name + ".npz"), **rec)
        for name, (_, n_iter, n_step, seed) in HMC_CASES.items():
            ref = dr.reference_hmc(case_problem(name), n_iter, n_step, seed)
            np.savez(os.path.join(GOLDEN_DIR, name + ".npz"), **ref)
            print(name, "accept", ref["accept_stat"].round(3).tolist())
        for name, (_, n_iter, seed, depth) in NUTS_CASES.items():
            ref = dr.reference_nuts(case_problem(name), n_iter, seed, max_tree_depth=depth)
            np.savez(os.path.join(GOLDEN_DIR, name + ".npz"), **ref)
            print(name, "n_step", ref["n_step"].tolist())


if __name__ == "__main__":
    generate(sys.argv[1:])
