"""Make the ``tests/golden/uc_*.npz`` fixtures of tests/test_user_constraint_gpu.py: constrained
models that the registry cannot express, run through the unmodified reference, which takes their
NumPy callables (tests/user_constraint_sources.py) natively.  Start states lie on the manifold to
rounding; momenta are projected onto its cotangent space by the reference system.  Needs the
reference (``oracle/_ref``, placed by ``build()``):

    python tests/make_user_constraint_golden.py [case ...]
"""

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

from oracle import drivers as dr  # noqa: E402
from oracle import mici_oracle as mo  # noqa: E402
from user_constraint_sources import UC_MODELS  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")

# name -> (model, system, dens_wrt_hausdorff, n_chains, metric kind, projection solver,
#          step size, kind, kind arguments, seed)
#   system "dense": DenseConstrainedEuclideanMetricSystem; "gaussian":
#   GaussianDenseConstrainedEuclideanMetricSystem (always the Lebesgue density)
#   kind "steps": n_steps constrained leapfrog steps per count, mixed directions;
#   kind "hmc": static HMC, (n_iter, n_step)
CASES = {
    "uc_so3_dense_newton": ("so3", "dense", True, 6, "dense", "newton", 0.1, "steps", (1, 5, 20), 1),
    "uc_hmc_so3_dense": ("so3", "dense", True, 4, "dense", "newton", 0.2, "hmc", (4, 5), 2),
    "uc_generator_gaussian_dense": ("generator", "gaussian", False, 6, "dense", "newton", 0.1,
                                    "steps", (1, 5, 20), 3),
    "uc_l4_sphere_diag_quasi_newton": ("l4_sphere", "dense", False, 4, "diagonal", "quasi_newton",
                                       0.02, "steps", (1, 5), 4),
    # a step at which the frozen-Jacobian iteration fails for 1 of 16 chains in the first step
    # and 5 of 16 within three (ConvergenceError)
    "uc_l4_sphere_diag_quasi_newton_bigstep": ("l4_sphere", "dense", False, 16, "diagonal",
                                               "quasi_newton", 0.1, "steps", (1, 3), 5),
}


def mixed_dirs(n):
    d = np.ones(n, dtype=np.int32)
    d[1::3] = -1
    return d


def reference_system(name, metric):
    mici = dr.import_reference()
    model, system_kind, hausdorff = CASES[name][:3]
    fns = UC_MODELS[model][1]()
    if system_kind == "gaussian":
        return mici.systems.GaussianDenseConstrainedEuclideanMetricSystem(metric=metric, **fns)
    return mici.systems.DenseConstrainedEuclideanMetricSystem(
        metric=metric, dens_wrt_hausdorff=hausdorff, **fns)


def inputs(name):
    """Seeded start positions on the manifold, cotangent momenta and the metric of a case."""
    mici = dr.import_reference()
    model, _, _, n, kind, _, _, _, _, seed = CASES[name]
    rng = np.random.default_rng(seed)
    pos = UC_MODELS[model][2](rng, n)
    dim = pos.shape[1]
    if kind == "identity":
        metric = None
    elif kind == "diagonal":
        metric = rng.uniform(0.5, 2.0, size=dim)
    else:
        a = rng.normal(size=(dim, dim)) / np.sqrt(dim)
        metric = a @ a.T + np.identity(dim)
    system = reference_system(name, metric)
    mom = np.empty_like(pos)
    for i in range(n):
        state = mici.states.ChainState(pos=pos[i].copy(), mom=np.zeros(dim), dir=1)
        mom[i] = system.project_onto_cotangent_space(rng.normal(size=dim), state)
    return pos, mom, metric, system


def make(name):
    mici = dr.import_reference()
    _, _, _, n, _, solver, eps, kind, arg, seed = CASES[name]
    pos, mom, metric, system = inputs(name)
    integ = mici.integrators.ConstrainedLeapfrogIntegrator(
        system, eps,
        projection_solver=getattr(mici.solvers, "solve_projection_onto_manifold_" + solver))
    out = {"pos0": pos, "mom0": mom, "step_size": np.array(eps)}
    if metric is not None:
        out["metric"] = metric
    if kind == "steps":
        dirs = mixed_dirs(n)
        out["dirs"] = dirs
        for n_steps in arg:
            q, p, h = pos.copy(), mom.copy(), np.full(n, np.nan)
            status, n_done = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
            for i in range(n):
                state = mici.states.ChainState(pos=pos[i].copy(), mom=mom[i].copy(),
                                               dir=int(dirs[i]))
                for _ in range(n_steps):
                    try:
                        state = integ.step(state)
                    except mici.errors.ConvergenceError:
                        status[i] = mo.STATUS_CONVERGENCE
                        break
                    except mici.errors.NonReversibleStepError:
                        status[i] = mo.STATUS_NON_REVERSIBLE
                        break
                    n_done[i] += 1
                q[i], p[i] = state.pos, state.mom
                if status[i] == 0:
                    h[i] = system.h(state)
            out.update({f"pos_{n_steps}": q, f"mom_{n_steps}": p, f"h_{n_steps}": h,
                        f"status_{n_steps}": status, f"n_done_{n_steps}": n_done})
        out["step_counts"] = np.array(arg)
    else:
        n_iter, n_step = arg
        int_tr = mici.transitions.MetropolisStaticIntegrationTransition(system, integ, n_step)
        mom_tr = mici.transitions.IndependentMomentumTransition(system)
        keys = ("n_step", "metrop_accept_prob", "accept_stat")
        trace = np.empty((n_iter, n, pos.shape[1]))
        stats = {k: np.empty((n_iter, n)) for k in keys}
        dirs = np.ones(n, dtype=np.int32)
        for i in range(n):
            rng = np.random.default_rng([seed, i])
            state = mici.states.ChainState(pos=pos[i].copy(), mom=mom[i].copy(), dir=1)
            for it in range(n_iter):
                state, _ = mom_tr.sample(state, rng)
                state, st = int_tr.sample(state, rng)
                trace[it, i] = state.pos
                for k in keys:
                    stats[k][it, i] = st[k]
            dirs[i] = state.dir
        out.update(trace=trace, dir=dirs, seed=np.array(seed), n_iter=np.array(n_iter),
                   n_step_arg=np.array(n_step), **stats)
    np.savez(os.path.join(GOLDEN_DIR, name + ".npz"), **out)
    summary = {k: v for k, v in out.items() if k.startswith("status_")}
    print(f"{name}: written", {k: np.bincount(v, minlength=3).tolist() for k, v in summary.items()})


if __name__ == "__main__":
    for case in sys.argv[1:] or CASES:
        make(case)
