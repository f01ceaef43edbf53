"""Make the ``tests/golden/ut_*.npz`` fixtures of tests/test_user_target_gpu.py: models that the
target registry cannot express, run through the unmodified reference, which takes their NumPy
callables (tests/user_target_sources.py) natively.  Needs the reference (``oracle/_ref``, placed
by ``build()``):

    python tests/make_user_target_golden.py
"""

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

from oracle import drivers as dr  # noqa: E402
from user_target_sources import DIMS, USER_MODELS  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")

# name -> (model, n_chains, metric kind, integrator, step size, kind, kind arguments, seed)
#   kind "steps": n_steps leapfrog steps per count, mixed directions
#   kind "hmc":   static HMC, (n_iter, n_step);  "nuts": DynamicMultinomialHMC, n_iter
CASES = {
    "ut_eight_schools_identity": ("eight_schools", 8, "identity", "leapfrog", 0.1, "steps", (1, 5, 20), 1),
    "ut_ar1_diag": ("ar1", 6, "diagonal", "leapfrog", 0.05, "steps", (1, 20), 2),
    "ut_ar1_diag_bcss3": ("ar1", 6, "diagonal", "bcss3", 0.08, "steps", (1, 20), 3),
    "ut_logistic_dense": ("logistic", 8, "dense", "leapfrog", 0.2, "steps", (1, 5, 20), 4),
    "ut_hmc_logistic_dense": ("logistic", 6, "dense", "leapfrog", 0.3, "hmc", (5, 6), 5),
    "ut_nuts_logistic_dense": ("logistic", 4, "dense", "leapfrog", 0.25, "nuts", 4, 6),
}
INTEGRATORS = {"leapfrog": "LeapfrogIntegrator", "bcss3": "BCSSThreeStageIntegrator"}


def mixed_dirs(n):
    d = np.ones(n, dtype=np.int32)
    d[1::3] = -1
    return d


def inputs(name):
    """Seeded initial positions, momenta and metric of a case."""
    model, n, kind, _, _, _, _, seed = CASES[name]
    dim = DIMS[model]
    rng = np.random.default_rng([seed, dim])
    pos = 0.5 * rng.normal(size=(n, dim))
    mom = rng.normal(size=(n, dim))
    if kind == "identity":
        metric = None
    elif kind == "diagonal":
        metric = rng.uniform(0.5, 2.0, size=dim)
    else:
        a = rng.normal(size=(dim, dim)) / np.sqrt(dim)
        metric = a @ a.T + np.identity(dim)
    return pos, mom, metric


def make(name):
    mici = dr.import_reference()
    model, n, _, integ_name, eps, kind, arg, seed = CASES[name]
    nld, grad = USER_MODELS[model][1]()
    pos, mom, metric = inputs(name)
    system = mici.systems.EuclideanMetricSystem(neg_log_dens=nld, metric=metric,
                                                grad_neg_log_dens=grad)
    integ = getattr(mici.integrators, INTEGRATORS[integ_name])(system, eps)
    out = {"pos0": pos, "mom0": mom, "step_size": np.array(eps)}
    if metric is not None:
        out["metric"] = metric
    if kind == "steps":
        dirs = mixed_dirs(n)
        out["dirs"] = dirs
        for n_steps in arg:
            q, p, h = np.empty_like(pos), np.empty_like(mom), np.empty(n)
            for i in range(n):
                state = mici.states.ChainState(pos=pos[i].copy(), mom=mom[i].copy(), dir=int(dirs[i]))
                for _ in range(n_steps):
                    state = integ.step(state)
                q[i], p[i], h[i] = state.pos, state.mom, system.h(state)
            out.update({f"pos_{n_steps}": q, f"mom_{n_steps}": p, f"h_{n_steps}": h})
        out["step_counts"] = np.array(arg)
    else:
        if kind == "hmc":
            n_iter, n_step = arg
            int_tr = mici.transitions.MetropolisStaticIntegrationTransition(system, integ, n_step)
            keys = ("n_step", "metrop_accept_prob", "accept_stat")
        else:
            n_iter = arg
            int_tr = mici.transitions.MultinomialDynamicIntegrationTransition(system, integ)
            keys = ("n_step", "tree_depth", "diverging", "av_metrop_accept_prob", "accept_stat")
        mom_tr = mici.transitions.IndependentMomentumTransition(system)
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
        out.update(trace=trace, dir=dirs, seed=np.array(seed), n_iter=np.array(n_iter), **stats)
        if kind == "hmc":
            out["n_step_arg"] = np.array(n_step)
    np.savez(os.path.join(GOLDEN_DIR, name + ".npz"), **out)
    print(f"{name}: written")


if __name__ == "__main__":
    for case in sys.argv[1:] or CASES:
        make(case)
