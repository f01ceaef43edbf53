"""TEST INFRASTRUCTURE ONLY -- the NumPy oracle and the reference fixtures of the Gaussian
constrained system (``GaussianDenseConstrainedEuclideanMetricSystem``, reference
systems.py:1034-1184).

* ``GaussianConstrainedSystem``: ``mo.ConstrainedSystem`` with the Gaussian split -- h2 =
  q.q/2 + p.M^-1 p/2, Gram matrices as ``DenseSymmetricMatrix`` inverted through
  ``numpy.linalg.eigh`` (matrices.py:436-459, 1414-1447), ``dh2_flow_dmom`` as two
  ``EigendecomposedSymmetricMatrix`` (:1529-1575) -- expression for expression.
* ``constrained_leapfrog_step`` and the three projection solvers with those operators
  (solvers.py:195-614, integrators.py:929-984).
* ``patched_drivers()``: makes ``oracle.drivers`` handle the system
  ``"gaussian_constrained_euclidean"``; the oracle's transitions are used unchanged.
* Case tables kept apart from the other fixtures'; ``OPENBLAS_NUM_THREADS=1 python
  tests/gaussian_constrained_cases.py`` regenerates the ``gc_*.npz`` fixtures from the unmodified
  reference.
"""

from __future__ import annotations

import contextlib
import copy
import os
import sys

import numpy as np
import numpy.linalg as nla
import scipy.linalg as sla

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mici_b200 import problems as pb  # noqa: E402
from oracle import drivers as dr  # noqa: E402
from oracle import mici_oracle as mo  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
SYSTEM = "gaussian_constrained_euclidean"


# ------------------------------------------------------------------------ matrix operators


class EigOperator:
    """``EigendecomposedSymmetricMatrix(eigvec, eigval)`` (matrices.py:1529-1575); ``u`` None for
    the identity eigenvectors of identity / diagonal metrics (matrices.py:519-528, 743-749)."""

    def __init__(self, u, eigval):
        self.u = u
        self.eigval = eigval

    def __matmul__(self, x):
        # eigvec @ (diag_eigval @ (eigvec.T @ x)); DiagonalMatrix @ 2-D is diagonal[:, None] * x
        y = x if self.u is None else self.u.T @ x
        e = self.eigval
        y = (e[:, None] * y if y.ndim == 2 else e * y) if np.ndim(e) and np.size(e) > 1 else e * y
        return y if self.u is None else self.u @ y


def eigh_inverse(array):
    """``DenseSymmetricMatrix(array).inv`` (matrices.py:1446-1447): eigh, then 1 / eigval."""
    eigval, v = nla.eigh(array)
    return EigOperator(v, 1 / eigval), eigval


class GaussianConstrainedSystem(mo.ConstrainedSystem):
    def __init__(self, target, metric=None):
        super().__init__(target, metric, dens_wrt_hausdorff=False)
        eigval, u = mo.metric_eig(self.metric)
        if self.metric.kind == "identity":
            eigval = np.ones(target.dim)  # IdentityMatrix.eigval is its diagonal (:519-521)
        self.eigval, self.u = eigval, u
        self.omega = 1.0 / eigval**0.5

    def inv_metric_right(self, a):
        """``a @ metric.inv`` (``metric._right_matrix_multiply``)."""
        m = self.metric
        if m.kind == "identity":
            return a
        if m.kind == "diagonal":
            return m.inv_diagonal * a
        return a @ m.inv_array

    def gram(self, q):
        jac = self.jacob_constr(q)
        return jac @ self.inv_metric_mat(jac.T)  # systems.py:1163-1166

    def h1(self, q):
        eigval = nla.eigh(self.gram(q))[0]
        return self.target.neg_log_dens(q) + 0.5 * np.log(np.abs(eigval)).sum()

    def h2(self, q, p):
        return 0.5 * q @ q + 0.5 * (self.inv_metric_right(p) @ p)  # systems.py:451-454

    def h(self, q, p):
        return self.h1(q) + self.h2(q, p)

    def dh1_dpos(self, q):
        jac = self.jacob_constr(q)
        inv_gram, _ = eigh_inverse(jac @ self.inv_metric_mat(jac.T))
        m = self.inv_metric_right(inv_gram @ jac)
        return self.target.grad_neg_log_dens(q) + self.target.mhp_constr(q)(m)

    def project_onto_cotangent_space(self, mom, q):
        jac = self.jacob_constr(q)
        inv_gram, _ = eigh_inverse(jac @ self.inv_metric_mat(jac.T))
        return mom - jac.T @ (inv_gram @ (jac @ self.inv_metric_mat(mom)))

    def h2_flow(self, q, p, dt):
        return mo.gaussian_h2_flow(q, p, dt, self.metric)

    def dh2_flow_dmom(self, dt):
        sin_omega_dt, cos_omega_dt = np.sin(self.omega * dt), np.cos(self.omega * dt)
        return EigOperator(self.u, sin_omega_dt * self.omega), EigOperator(self.u, cos_omega_dt)


# ------------------------------------------------------------------------------- solvers


def _finish(p, mu, time_step, dmom):
    # state.mom -= np.sign(time_step) * dh2_flow_mom_dmom @ mu: (sign * matrix) @ mu
    return p - EigOperator(dmom.u, np.sign(time_step) * dmom.eigval) @ mu


def solve_newton(q, p, q_prev, time_step, system, constraint_tol=1e-9, position_tol=1e-8,
                 divergence_tol=1e10, max_iters=50, counts=None):
    """solvers.py:346-469 with the Gaussian split's dh2_flow_dmom."""
    q, p, mu = q.copy(), p.copy(), np.zeros_like(q)
    jac_prev = system.jacob_constr(q_prev)
    dpos_op, dmom = system.dh2_flow_dmom(abs(time_step))
    error = np.nan
    try:
        for i in range(max_iters):
            jac = system.jacob_constr(q)
            c = system.constr(q)
            error = mo.maximum_norm(c)
            res_jac = mo._chkfinite(jac @ (dpos_op @ jac_prev.T))
            lu_piv = sla.lu_factor(res_jac, check_finite=False)
            delta_mu = jac_prev.T @ sla.lu_solve(lu_piv, c, 0, check_finite=False)
            delta_pos = dpos_op @ delta_mu
            if error > divergence_tol or np.isnan(error):
                raise mo.OracleIntegratorError(mo.STATUS_CONVERGENCE, f"Newton diverged at {i}")
            if error < constraint_tol and mo.maximum_norm(delta_pos) < position_tol:
                if counts is not None:
                    counts.setdefault("newton_iters", []).append(i + 1)
                return q, _finish(p, mu, time_step, dmom)
            mu += delta_mu
            q -= delta_pos
    except (ValueError, mo._LinAlgError, nla.LinAlgError) as e:
        raise mo.OracleIntegratorError(mo.STATUS_CONVERGENCE, f"{type(e)} in Newton") from e
    raise mo.OracleIntegratorError(mo.STATUS_CONVERGENCE, f"Newton did not converge, |c|={error}")


def solve_quasi_newton(q, p, q_prev, time_step, system, constraint_tol=1e-9, position_tol=1e-8,
                       divergence_tol=1e10, max_iters=50, counts=None):
    """solvers.py:195-343: the frozen Gram matrix J_prev S J_prev^T is a DenseSymmetricMatrix."""
    q, p, mu = q.copy(), p.copy(), np.zeros_like(q)
    jac_prev = system.jacob_constr(q_prev)
    dpos_op, dmom = system.dh2_flow_dmom(abs(time_step))
    error = np.nan
    try:
        inv_g, _ = eigh_inverse(jac_prev @ (dpos_op @ jac_prev.T))
        for i in range(max_iters):
            c = system.constr(q)
            error = mo.maximum_norm(c)
            delta_mu = jac_prev.T @ (inv_g @ c)
            delta_pos = dpos_op @ delta_mu
            if error > divergence_tol or np.isnan(error):
                raise mo.OracleIntegratorError(mo.STATUS_CONVERGENCE, f"quasi-Newton diverged {i}")
            if error < constraint_tol and mo.maximum_norm(delta_pos) < position_tol:
                if counts is not None:
                    counts.setdefault("newton_iters", []).append(i + 1)
                return q, _finish(p, mu, time_step, dmom)
            mu += delta_mu
            q -= delta_pos
    except (ValueError, mo._LinAlgError, nla.LinAlgError) as e:
        raise mo.OracleIntegratorError(mo.STATUS_CONVERGENCE, f"{type(e)} in quasi-Newton") from e
    raise mo.OracleIntegratorError(mo.STATUS_CONVERGENCE, f"quasi-Newton: |c|={error}")


def solve_newton_line_search(q, p, q_prev, time_step, system, constraint_tol=1e-9,
                             position_tol=1e-8, divergence_tol=1e10, max_iters=50,
                             max_line_search_iters=10, counts=None):
    """solvers.py:472-614 with the Gaussian split's dh2_flow_dmom."""
    q, p, mu = q.copy(), p.copy(), np.zeros_like(q)
    jac_prev = system.jacob_constr(q_prev)
    dpos_op, dmom = system.dh2_flow_dmom(abs(time_step))
    delta_pos, step_size = None, None
    error = np.nan
    for i in range(max_iters):
        try:
            jac = system.jacob_constr(q)
            c = system.constr(q)
            error = mo.maximum_norm(c)
            if i > 0 and (error > divergence_tol or np.isnan(error)):
                raise mo.OracleIntegratorError(mo.STATUS_CONVERGENCE, f"Newton diverged at {i}")
            if error < constraint_tol and (
                    i == 0 or mo.maximum_norm(step_size * delta_pos) < position_tol):
                if counts is not None:
                    counts.setdefault("newton_iters", []).append(i + 1)
                return q, _finish(p, mu, time_step, dmom)
            res_jac = mo._chkfinite(jac @ (dpos_op @ jac_prev.T))
            lu_piv = sla.lu_factor(res_jac, check_finite=False)
            delta_mu = jac_prev.T @ sla.lu_solve(lu_piv, c, 0, check_finite=False)
            delta_pos = -(dpos_op @ delta_mu)
            pos_curr = q.copy()
            step_size = 1.0
            for _ in range(max_line_search_iters):
                q = pos_curr + step_size * delta_pos
                if mo.maximum_norm(system.constr(q)) < error:
                    break
                step_size *= 0.5
            mu += step_size * delta_mu
        except (ValueError, mo._LinAlgError, nla.LinAlgError) as e:
            raise mo.OracleIntegratorError(mo.STATUS_CONVERGENCE, f"{type(e)} in Newton") from e
    raise mo.OracleIntegratorError(mo.STATUS_CONVERGENCE, f"Newton did not converge, |c|={error}")


SOLVERS = {"newton": solve_newton, "quasi_newton": solve_quasi_newton,
           "newton_with_line_search": solve_newton_line_search}


def constrained_leapfrog_step(q, p, time_step, system, n_inner_step=1, reverse_check_tol=2e-8,
                              projection_solver_kwargs=None, counts=None,
                              projection_solver="newton"):
    """One ``ConstrainedLeapfrogIntegrator.step`` (integrators.py:929-984) on the Gaussian system."""
    kw = {} if projection_solver_kwargs is None else projection_solver_kwargs
    solve = SOLVERS[projection_solver]
    q = np.array(q, dtype=np.float64)
    p = np.array(p, dtype=np.float64)

    def retract(q, p, q_prev, dt):
        q, p = system.h2_flow(q, p, dt)
        return solve(q, p, q_prev, dt, system, counts=counts, **kw)

    try:
        p = p - (0.5 * time_step) * system.dh1_dpos(q)
        p = system.project_onto_cotangent_space(p, q)
        dt_inner = time_step / n_inner_step
        for _ in range(n_inner_step):
            q_prev = q.copy()
            q, p = retract(q, p, q_prev, dt_inner)
            p = system.project_onto_cotangent_space(p, q)
            q_back, _ = retract(q.copy(), p.copy(), q, -dt_inner)
            rev_diff = mo.maximum_norm(q_back - q_prev)
            if rev_diff > reverse_check_tol:
                raise mo.OracleIntegratorError(mo.STATUS_NON_REVERSIBLE, f"rev diff {rev_diff}")
        p = p - (0.5 * time_step) * system.dh1_dpos(q)
        p = system.project_onto_cotangent_space(p, q)
    except (ValueError, mo._LinAlgError) as e:
        raise mo.OracleIntegratorError(mo.STATUS_LINALG, str(e)) from e
    return q, p


# ------------------------------------------------------------------ drivers extension

_ORIG = {}


def oracle_step_fn(problem, counts=None, **overrides):
    if problem.system != SYSTEM:
        return _ORIG["oracle_step_fn"](problem, counts=counts, **overrides)
    system = GaussianConstrainedSystem(dr.build_target(problem), problem.metric)
    ikw = dict(problem.integrator_kwargs)
    ikw.update(overrides)
    eps = problem.step_size

    def step(q, p, d):
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            return constrained_leapfrog_step(q, p, d * eps, system, counts=counts, **ikw)

    def h(q, p):
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            return system.h(q, p)

    return step, h, system


def build_reference(problem, **overrides):
    if problem.system != SYSTEM:
        return _ORIG["build_reference"](problem, **overrides)
    mici = dr.import_reference()
    target = dr.build_target(problem)
    system = mici.systems.GaussianDenseConstrainedEuclideanMetricSystem(
        neg_log_dens=target.neg_log_dens, constr=target.constr, metric=problem.metric,
        grad_neg_log_dens=target.grad_neg_log_dens, jacob_constr=target.jacob_constr,
        mhp_constr=target.mhp_constr)
    ikw = dict(problem.integrator_kwargs)
    ikw.update(overrides)
    if isinstance(ikw.get("projection_solver"), str):
        ikw["projection_solver"] = getattr(
            mici.solvers, "solve_projection_onto_manifold_" + ikw["projection_solver"])
    return system, mici.integrators.ConstrainedLeapfrogIntegrator(system, problem.step_size, **ikw)


def _sample_momentum(problem, system):
    if problem.system != SYSTEM:
        return _ORIG["_sample_momentum"](problem, system)
    return mo.constrained_sample_momentum(system)


def _velocity_fn(problem, system):
    if problem.system != SYSTEM:
        return _ORIG["_velocity_fn"](problem, system)
    return lambda q, p: system.inv_metric_mat(p)


@contextlib.contextmanager
def patched_drivers():
    """``oracle.drivers`` runners that also build the Gaussian constrained system."""
    names = ("oracle_step_fn", "build_reference", "_sample_momentum", "_velocity_fn")
    prev = {n: getattr(dr, n) for n in names}
    _ORIG.update(prev)
    for n in names:
        setattr(dr, n, globals()[n])
    try:
        yield dr
    finally:
        for n, f in prev.items():
            setattr(dr, n, f)


# -------------------------------------------------------------------------- problems


def make_problem(kind, metric_kind, dim=None, n_chains=8, step_size=0.2, seed=0, n_constr=None,
                 integrator_kwargs=None, zero_block=False):
    """Sphere, multi-sphere or torus start states of the existing constrained problems, with the
    Gaussian system and the given metric."""
    s = pb.BASE_SEED + 200 + seed
    if kind == "sphere":
        base = pb.sphere_constrained(n_chains=n_chains, dim=dim, seed=s, metric_kind=metric_kind)
    elif kind == "multi_sphere":
        base = pb.multi_sphere_constrained(n_chains=n_chains, dim=dim, n_constr=n_constr, seed=s,
                                           metric_kind=metric_kind)
    else:
        base = pb.c3_torus(n_chains=n_chains, seed=s)
    prob = copy.copy(base)
    prob.system = SYSTEM
    prob.name = "GC"
    prob.step_size = step_size
    prob.pos = base.pos.copy()
    prob.mom = base.mom.copy()
    if zero_block:  # q = 0 on the first sphere block of chain 0: the Gram matrix is singular
        prob.pos[0, : dim // n_constr] = 0.0
    prob.system_kwargs = {}
    prob.integrator_kwargs = {"n_inner_step": 1, **(integrator_kwargs or {})}
    return prob


QN = {"projection_solver": "quasi_newton"}
LS = {"projection_solver": "newton_with_line_search"}
# name: (make_problem kwargs, step counts).  Mixed directions: chain i runs with dir (-1)^i.
CASES = {
    "gc_sphere_identity_d5": (dict(kind="sphere", metric_kind="identity", dim=5, seed=1), (1, 5, 20)),
    "gc_sphere_dense_d10": (dict(kind="sphere", metric_kind="dense", dim=10, seed=2), (1, 5, 20)),
    "gc_sphere_diag_d70_inner2": (dict(kind="sphere", metric_kind="diagonal", dim=70, seed=3,
                                       integrator_kwargs={"n_inner_step": 2}), (1, 5)),
    "gc_sphere_dense_d200": (dict(kind="sphere", metric_kind="dense", dim=200, n_chains=3, seed=4,
                                  step_size=0.05),
                             (1, 5)),
    "gc_multi_sphere_c2_identity_d12": (dict(kind="multi_sphere", metric_kind="identity", dim=12,
                                             n_constr=2, seed=5, step_size=0.15), (1, 5, 20)),
    "gc_multi_sphere_c4_dense_d16": (dict(kind="multi_sphere", metric_kind="dense", dim=16,
                                          n_constr=4, seed=6, step_size=0.15), (1, 5, 20)),
    "gc_multi_sphere_c4_diag_d72_inner2": (dict(kind="multi_sphere", metric_kind="diagonal",
                                                dim=72, n_constr=4, seed=7, step_size=0.15,
                                                integrator_kwargs={"n_inner_step": 2}), (1, 5)),
    "gc_multi_sphere_c8_dense_d32": (dict(kind="multi_sphere", metric_kind="dense", dim=32,
                                          n_constr=8, seed=8, step_size=0.1), (1, 5, 20)),
    "gc_multi_sphere_c8_dense_d128": (dict(kind="multi_sphere", metric_kind="dense", dim=128,
                                           n_constr=8, n_chains=3, seed=9, step_size=0.1), (1, 5)),
    "gc_torus": (dict(kind="torus", metric_kind="identity", n_chains=8, seed=10, step_size=0.2),
                 (1, 5, 20)),
    "gc_multi_sphere_c4_dense_d16_quasi_newton": (
        dict(kind="multi_sphere", metric_kind="dense", dim=16, n_constr=4, seed=11,
             step_size=0.15, integrator_kwargs=QN), (1, 5, 20)),
    "gc_sphere_dense_d10_quasi_newton": (dict(kind="sphere", metric_kind="dense", dim=10, seed=12,
                                              integrator_kwargs=QN), (1, 5)),
    "gc_multi_sphere_c2_dense_d12_line_search": (
        dict(kind="multi_sphere", metric_kind="dense", dim=12, n_constr=2, seed=13,
             step_size=0.15, integrator_kwargs=LS), (1, 5, 20)),
    "gc_multi_sphere_c2_identity_d12_singular": (
        dict(kind="multi_sphere", metric_kind="identity", dim=12, n_constr=2, seed=14,
             step_size=0.15, zero_block=True), (1, 5)),
}
# big steps: chains fail with ConvergenceError and with NonReversibleStepError
FAILURE_CASES = {
    "gc_sphere_dense_d10_bigstep": (dict(kind="sphere", metric_kind="dense", dim=10, n_chains=24,
                                         seed=15, step_size=0.7), (1, 5)),
    "gc_multi_sphere_c4_identity_d16_bigstep": (
        dict(kind="multi_sphere", metric_kind="identity", dim=16, n_constr=4, n_chains=24,
             seed=16, step_size=0.6), (1, 5)),
}
HMC_CASES = {
    "gc_hmc_sphere_dense_d10": (dict(kind="sphere", metric_kind="dense", dim=10, n_chains=4,
                                     seed=17), 4, 5, 817),
}
NUTS_CASES = {
    "gc_nuts_multi_sphere_c2_d12": (dict(kind="multi_sphere", metric_kind="identity", dim=12,
                                         n_constr=2, n_chains=3, seed=18, step_size=0.15),
                                    3, 818, 4),
}
ADAPT_CASES = {
    "gc_adapt_sphere_diag_d10_dualavg": (dict(kind="sphere", metric_kind="diagonal", dim=10,
                                              n_chains=4, seed=19), 10, 3, 3, 819),
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
    """Oracle run plus the total Newton iterations of every chain."""
    its = np.zeros(problem.n_chains, dtype=np.int32)
    with patched_drivers():
        out = dr.oracle_run(problem, n_steps, dirs=dirs)
        for c in range(problem.n_chains):
            counts = {}
            step, _, _ = dr.oracle_step_fn(problem, counts=counts)
            q, p = problem.pos[c].copy(), problem.mom[c].copy()
            for _ in range(n_steps):
                try:
                    q, p = step(q, p, int(dirs[c]))
                except mo.OracleIntegratorError:
                    break
            its[c] = sum(counts.get("newton_iters", []))
    out["newton_iters"] = its
    return out


def load_fixture(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))


def oracle_adapt_run(name):
    from oracle.make_golden import STAGE_CODES

    names = {code: which for which, code in STAGE_CODES.items()}
    g = load_fixture(name)
    stages = [(int(n), names[int(c)]) for n, c in zip(g["stage_n_iter"], g["stage_which"])]
    _, _, _, n_step, seed = ADAPT_CASES[name]
    with patched_drivers():
        return dr.oracle_sample_chains(case_problem(name), stages, n_step, seed, ADAPT_SPECS)


def generate(names=None):  # pragma: no cover - run by hand against the unmodified reference
    from oracle.make_golden import STAGE_CODES, reference_stage_list

    with patched_drivers(), np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for name, (_, n_warm, n_main, n_step, seed) in ADAPT_CASES.items():
            ref = dr.reference_sample_chains(case_problem(name), n_warm, n_main, n_step, seed,
                                             ADAPT_SPECS)
            stages = reference_stage_list(ADAPT_SPECS, None, n_warm, n_main)
            np.savez(os.path.join(GOLDEN_DIR, name + ".npz"),
                     stage_n_iter=np.array([n for n, _ in stages]),
                     stage_which=np.array([STAGE_CODES[w] for _, w in stages]), **ref)
            print(name, "step size", float(ref["step_size"]))
        for name, (_, step_counts) in ALL_INTEGRATOR_CASES.items():
            if names and name not in names:
                continue
            problem = case_problem(name)
            dirs = case_dirs(problem)
            rec = {"step_counts": np.array(step_counts), "dirs": dirs,
                   "step_size": problem.step_size}
            for n in step_counts:
                ref = dr.reference_run(problem, n, dirs=dirs)
                orc = oracle_integrator_run(problem, n, dirs)
                for k in ("pos", "mom", "status", "n_done", "h"):
                    rec[f"{k}_{n}"] = ref[k]
                rec[f"newton_iters_{n}"] = orc["newton_iters"]
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
