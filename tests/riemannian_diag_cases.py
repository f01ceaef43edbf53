"""TEST INFRASTRUCTURE ONLY -- the NumPy oracle and the reference fixtures of the diagonal and
scalar Riemannian-metric systems (``DiagonalRiemannianMetricSystem`` /
``ScalarRiemannianMetricSystem``, reference systems.py:1405-1571).

* ``DiagonalMetricValue`` / ``ScalarMetricValue``: ``PositiveDiagonalMatrix`` /
  ``PositiveScaledIdentityMatrix`` arithmetic (reference matrices.py:595-792), expression for
  expression -- the kernels follow their order of operations.
* NumPy metric models (``QuadraticDiag``, ``FunnelFisher``, ``QuadraticScalar``) with the
  explicit VJP callables the reference takes.
* ``patched_drivers()``: makes ``oracle.drivers`` (oracle and reference runners, HMC / NUTS /
  staged sampling) handle the systems ``"diagonal_riemannian"`` and ``"scalar_riemannian"``;
  the oracle's implicit integrators, solvers and transitions are used unchanged.
* Case tables kept apart from ``oracle/make_golden.py``'s (the existing fixtures stay as they
  are); ``python tests/riemannian_diag_cases.py`` regenerates the ``rd_*.npz`` fixtures from the
  unmodified reference.
"""

from __future__ import annotations

import contextlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mici_b200 import problems as pb  # noqa: E402
from oracle import drivers as dr  # noqa: E402
from oracle import mici_oracle as mo  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
NEW_SYSTEMS = ("diagonal_riemannian", "scalar_riemannian")


# ------------------------------------------------------------------------- metric values


class DiagonalMetricValue:
    """``PositiveDiagonalMatrix(d)`` (matrices.py:709-792)."""

    def __init__(self, diagonal):
        if not np.all(diagonal > 0):  # :778-780
            raise ValueError("Diagonal values must all be positive.")
        self.diagonal = diagonal
        self.inv = 1.0 / diagonal  # _construct_inv (:783-784)

    @property
    def log_abs_det(self):  # SymmetricMatrix.log_abs_det (:458-459)
        return np.log(np.abs(self.diagonal)).sum()

    def inv_matvec(self, v):
        return self.inv * v

    def sqrt_matvec(self, v):  # _construct_sqrt (:786-787)
        return self.diagonal**0.5 * v

    @property
    def grad_log_abs_det(self):  # :758-759
        return 1.0 / self.diagonal

    def grad_quadratic_form_inv(self, v):  # :761-762
        return -((self.inv * v) ** 2)


class ScalarMetricValue:
    """``PositiveScaledIdentityMatrix(s, size=D)`` (matrices.py:595-706)."""

    def __init__(self, scalar, size):
        if scalar <= 0:  # :692-694
            raise ValueError("Scalar multiplier must be positive.")
        self.scalar = scalar
        self.size = size

    @property
    def log_abs_det(self):  # :659-667
        return self.size * np.log(abs(self.scalar))

    def inv_matvec(self, v):  # _construct_inv (:703-704), _left_matrix_multiply (:626-627)
        return (1 / self.scalar) * v

    def sqrt_matvec(self, v):  # :706
        return self.scalar**0.5 * v

    @property
    def grad_log_abs_det(self):  # :669-670
        return self.size / self.scalar

    def grad_quadratic_form_inv(self, v):  # :672-673
        return -np.sum(v**2) / self.scalar**2


# --------------------------------------------------------------------- metric models


class QuadraticDiag:
    """d_i = a + b q_i^2; at a = b = 1 the reference test's ``1 + q**2`` with VJP ``2 * m * q``."""

    kind = "diagonal"

    def __init__(self, a=1.0, b=1.0):
        self.a, self.b = float(a), float(b)

    def metric_func(self, q):
        return self.a + self.b * (q * q)

    def vjp_metric_func(self, q):
        return lambda w: 2 * self.b * w * q


class FunnelFisher:
    """The funnel's expected Fisher information, d = [1/9 + (D-1)/2, e^-v, ..., e^-v]."""

    kind = "diagonal"

    def metric_func(self, q):
        d = np.empty_like(q)
        d[0] = 1.0 / 9.0 + 0.5 * (q.shape[0] - 1)
        d[1:] = np.exp(-q[0])
        return d

    def vjp_metric_func(self, q):
        def vjp(w):
            out = np.zeros_like(q)
            out[0] = -np.exp(-q[0]) * np.sum(w[1:])
            return out

        return vjp


class QuadraticScalar:
    """s = a + b |q|^2, VJP w -> 2 b w q."""

    kind = "scalar"

    def __init__(self, a=1.0, b=1.0):
        self.a, self.b = float(a), float(b)

    def metric_func(self, q):
        return self.a + self.b * (q @ q)

    def vjp_metric_func(self, q):
        return lambda w: 2 * self.b * w * q


MODELS = {"diag_quadratic": QuadraticDiag, "funnel_fisher": FunnelFisher,
          "scalar_quadratic": QuadraticScalar}


def metric_model(problem):
    return MODELS[problem.metric_model](**problem.metric_params)


class OracleSystem(mo.RiemannianSystem):
    """``mo.RiemannianSystem`` with a diagonal / scalar metric value: the oracle's implicit
    integrators call ``metric``, ``vjp``, ``h``, ``dh1_dpos``, ``dh2_dpos`` and ``dh2_dmom``."""

    def __init__(self, target, model):
        super().__init__(target, model.kind, metric_model=model)

    def metric(self, q):
        self.n_metric_evals += 1
        if self.kind == "diagonal":
            return DiagonalMetricValue(self.metric_model.metric_func(q))
        return ScalarMetricValue(self.metric_model.metric_func(q), q.shape[0])

    def vjp(self, q):
        return self.metric_model.vjp_metric_func(q)


# ------------------------------------------------------------------ drivers extension

_ORIG_STEP_FN = dr.oracle_step_fn
_ORIG_BUILD_REFERENCE = dr.build_reference


def oracle_step_fn(problem, counts=None, **overrides):
    if problem.system not in NEW_SYSTEMS:
        return _ORIG_STEP_FN(problem, counts=counts, **overrides)
    system = OracleSystem(dr.build_target(problem), metric_model(problem))
    ikw = dict(problem.integrator_kwargs)
    ikw.update(overrides)
    eps = problem.step_size
    fn = (mo.implicit_midpoint_step if problem.integrator == "implicit_midpoint"
          else mo.implicit_leapfrog_step)

    def step(q, p, d):
        c = {} if counts is None else counts
        out = fn(q, p, d * eps, system, counts=c, **ikw)
        if counts is not None:
            counts.setdefault("all_fp_iters", []).append(list(c.get("fp_iters", [])))
        return out

    return step, system.h, system


def build_reference(problem, **overrides):
    if problem.system not in NEW_SYSTEMS:
        return _ORIG_BUILD_REFERENCE(problem, **overrides)
    mici = dr.import_reference()
    target = dr.build_target(problem)
    model = metric_model(problem)
    if problem.system == "diagonal_riemannian":
        system = mici.systems.DiagonalRiemannianMetricSystem(
            neg_log_dens=target.neg_log_dens, metric_diagonal_func=model.metric_func,
            vjp_metric_diagonal_func=model.vjp_metric_func,
            grad_neg_log_dens=target.grad_neg_log_dens)
    else:
        system = mici.systems.ScalarRiemannianMetricSystem(
            neg_log_dens=target.neg_log_dens, metric_scalar_func=model.metric_func,
            vjp_metric_scalar_func=model.vjp_metric_func,
            grad_neg_log_dens=target.grad_neg_log_dens)
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
    """``oracle.drivers`` runners that also build the diagonal / scalar systems."""
    prev = dr.oracle_step_fn, dr.build_reference
    dr.oracle_step_fn, dr.build_reference = oracle_step_fn, build_reference
    try:
        yield dr
    finally:
        dr.oracle_step_fn, dr.build_reference = prev


# -------------------------------------------------------------------------- problems


def make_problem(target, dim, metric, n_chains, step_size, seed, integrator="implicit_leapfrog",
                 metric_params=None, pos_scale=0.5, integrator_kwargs=None):
    """A small Riemannian problem: positions ``pos_scale * N(0, I)``, momenta from N(0, M(q))."""
    rng = np.random.default_rng(seed)
    pos = pos_scale * rng.standard_normal((n_chains, dim))
    z = rng.standard_normal((n_chains, dim))
    params = {"a": 1.0, "b": 1.0} if metric_params is None else dict(metric_params)
    model = MODELS[metric](**params) if metric != "funnel_fisher" else FunnelFisher()
    if model.kind == "diagonal":
        mom = z * np.sqrt(np.stack([model.metric_func(q) for q in pos]))
        system = "diagonal_riemannian"
    else:
        mom = z * np.sqrt(np.array([model.metric_func(q) for q in pos]))[:, None]
        system = "scalar_riemannian"
    tparams = {"dim": dim, "b": 0.5} if target == "banana" else {"dim": dim}
    return pb.Problem(
        name="RD", integrator=integrator, system=system, target=target, target_params=tparams,
        step_size=step_size, pos=pos, mom=mom, metric_model=metric,
        metric_params={} if metric == "funnel_fisher" else params,
        integrator_kwargs=dict(integrator_kwargs or {}),
    )


S = pb.BASE_SEED
# name: (make_problem kwargs, step counts).  Mixed directions: chain i runs with dir (-1)^i.
CASES = {
    "rd_dq_std_d1": (dict(target="std_gaussian", dim=1, metric="diag_quadratic", n_chains=8,
                          step_size=0.1, seed=S + 11), (1, 5, 20)),
    "rd_dq_std_d2": (dict(target="std_gaussian", dim=2, metric="diag_quadratic", n_chains=8,
                          step_size=0.1, seed=S + 12), (1, 5, 20)),
    "rd_dq_banana_d2": (dict(target="banana", dim=2, metric="diag_quadratic", n_chains=8,
                             step_size=0.1, seed=S + 13), (1, 5, 20)),
    "rd_dq_std_d5": (dict(target="std_gaussian", dim=5, metric="diag_quadratic", n_chains=8,
                          step_size=0.1, seed=S + 14), (1, 5, 20)),
    "rd_dq_std_d33": (dict(target="std_gaussian", dim=33, metric="diag_quadratic", n_chains=8,
                           step_size=0.05, seed=S + 15), (1, 5, 20)),
    "rd_dq_banana_d32": (dict(target="banana", dim=32, metric="diag_quadratic", n_chains=8,
                              step_size=0.05, seed=S + 16), (1, 5, 20)),
    "rd_ff_funnel_d10": (dict(target="neal_funnel", dim=10, metric="funnel_fisher", n_chains=8,
                              step_size=0.2, seed=S + 17), (1, 5, 20)),
    "rd_ff_funnel_d128": (dict(target="neal_funnel", dim=128, metric="funnel_fisher", n_chains=6,
                               step_size=0.2, seed=S + 18), (1, 5, 20)),
    "rd_sc_std_d5": (dict(target="std_gaussian", dim=5, metric="scalar_quadratic", n_chains=8,
                          step_size=0.1, seed=S + 19), (1, 5, 20)),
    "rd_sc_banana_d64": (dict(target="banana", dim=64, metric="scalar_quadratic", n_chains=6,
                              step_size=0.05, seed=S + 20, metric_params={"a": 1.0, "b": 1 / 64}),
                         (1, 5, 20)),
    # implicit midpoint and the Steffensen solver
    "rd_dq_banana_d8_midpoint": (dict(target="banana", dim=8, metric="diag_quadratic", n_chains=8,
                                      step_size=0.1, seed=S + 21, integrator="implicit_midpoint"),
                                 (1, 5, 20)),
    "rd_ff_funnel_d10_midpoint": (dict(target="neal_funnel", dim=10, metric="funnel_fisher",
                                       n_chains=8, step_size=0.2, seed=S + 22,
                                       integrator="implicit_midpoint"), (1, 5, 20)),
    "rd_sc_std_d5_midpoint": (dict(target="std_gaussian", dim=5, metric="scalar_quadratic",
                                   n_chains=8, step_size=0.1, seed=S + 23,
                                   integrator="implicit_midpoint"), (1, 5, 20)),
    "rd_dq_std_d5_steffensen": (dict(target="std_gaussian", dim=5, metric="diag_quadratic",
                                     n_chains=8, step_size=0.1, seed=S + 24,
                                     integrator_kwargs={"fixed_point_solver": "steffensen"}),
                                (1, 5, 20)),
    "rd_ff_funnel_d10_midpoint_steffensen": (
        dict(target="neal_funnel", dim=10, metric="funnel_fisher", n_chains=8, step_size=0.2,
             seed=S + 25, integrator="implicit_midpoint",
             integrator_kwargs={"fixed_point_solver": "steffensen"}), (1, 5, 20)),
}
# big steps: chains fail with ConvergenceError and with NonReversibleStepError
FAILURE_CASES = {
    "rd_dq_banana_d8_bigstep": (dict(target="banana", dim=8, metric="diag_quadratic",
                                     n_chains=24, step_size=0.4, seed=S + 26, pos_scale=1.0),
                                (1, 5)),
    "rd_ff_funnel_d10_bigstep": (dict(target="neal_funnel", dim=10, metric="funnel_fisher",
                                      n_chains=24, step_size=0.6, seed=S + 27, pos_scale=1.0),
                                 (1, 5)),
    "rd_sc_std_d5_bigstep": (dict(target="std_gaussian", dim=5, metric="scalar_quadratic",
                                  n_chains=24, step_size=0.8, seed=S + 28, pos_scale=0.5),
                             (1, 5)),
}
# static HMC: (problem kwargs, n_iter, n_step, seed)
HMC_CASES = {
    "rd_hmc_ff_funnel_d10": (dict(target="neal_funnel", dim=10, metric="funnel_fisher",
                                  n_chains=4, step_size=0.2, seed=S + 29), 4, 5, 707),
    "rd_hmc_sc_std_d5": (dict(target="std_gaussian", dim=5, metric="scalar_quadratic",
                              n_chains=4, step_size=0.15, seed=S + 30), 4, 5, 708),
}
# NUTS (DynamicMultinomialHMC's transition): (problem kwargs, n_iter, seed, max_tree_depth)
NUTS_CASES = {
    "rd_nuts_dq_banana_d4": (dict(target="banana", dim=4, metric="diag_quadratic", n_chains=3,
                                  step_size=0.2, seed=S + 31), 3, 709, 4),
    "rd_nuts_sc_std_d5": (dict(target="std_gaussian", dim=5, metric="scalar_quadratic",
                               n_chains=3, step_size=0.2, seed=S + 32), 3, 710, 4),
}
# dual-averaging warm-up + main stage through StaticMetropolisHMC.sample_chains:
# (problem kwargs, n_warm_up_iter, n_main_iter, n_step, seed)
ADAPT_CASES = {
    "rd_adapt_ff_funnel_d10_dualavg": (dict(target="neal_funnel", dim=10, metric="funnel_fisher",
                                            n_chains=4, step_size=0.2, seed=S + 33), 10, 3, 3, 711),
    "rd_adapt_sc_std_d5_dualavg": (dict(target="std_gaussian", dim=5, metric="scalar_quadratic",
                                        n_chains=4, step_size=0.15, seed=S + 34), 10, 3, 3, 712),
}
ADAPT_SPECS = [("dual_averaging", {})]
ALL_INTEGRATOR_CASES = {**CASES, **FAILURE_CASES}


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
    with patched_drivers():
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
    with patched_drivers():
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
