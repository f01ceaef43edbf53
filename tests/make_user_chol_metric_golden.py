"""Make the ``tests/golden/ul_*.npz`` fixtures of tests/test_user_chol_metric_gpu.py: the
hierarchical AR(1) model with its closed-form Cholesky factor (tests/user_chol_metric_sources.py),
which the registry cannot express, run through the unmodified reference's
``CholeskyFactoredRiemannianMetricSystem``, which takes its NumPy ``metric_chol_func`` /
``vjp_metric_chol_func`` natively.  The case tables, the problems and the oracle hook live here
too, so the tests build the same inputs.  Needs the reference (``oracle/_ref``, placed by
``build()``):

    OPENBLAS_NUM_THREADS=1 python tests/make_user_chol_metric_golden.py [case ...]
"""

import contextlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

import riemannian_chol_cases as rc  # noqa: E402
from mici_b200 import problems as pb  # noqa: E402
from oracle import drivers as dr  # noqa: E402
from user_chol_metric_sources import ul_model, ul_start  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")

# integrator cases: (model, n_chains, step size, seed, step counts, integrator, integrator kwargs)
CASES = {
    "ul_ar1_64_leapfrog": ("ar1_64", 6, 0.1, 1, (1, 5, 20), "implicit_leapfrog", {}),
    "ul_ar1_64_midpoint": ("ar1_64", 6, 0.1, 2, (1, 5, 20), "implicit_midpoint", {}),
    "ul_ar1_64_steffensen": ("ar1_64", 6, 0.1, 3, (1, 5, 20), "implicit_leapfrog",
                             {"fixed_point_solver": "steffensen"}),
    "ul_ar1_254_leapfrog": ("ar1_254", 3, 0.1, 4, (1, 5), "implicit_leapfrog", {}),
}
# a big step: some chains end in ConvergenceError within 5 steps
FAILURE_CASES = {
    "ul_ar1_64_bigstep": ("ar1_64", 12, 0.25, 5, (1, 5), "implicit_leapfrog", {}),
}
# static HMC: (model, n_chains, step size, seed, n_iter, n_step, rng seed)
HMC_CASES = {"ul_hmc_ar1_64": ("ar1_64", 4, 0.1, 6, 4, 5, 911)}
# NUTS: (model, n_chains, step size, seed, n_iter, rng seed, max tree depth)
NUTS_CASES = {"ul_nuts_ar1_64": ("ar1_64", 3, 0.1, 7, 3, 912, 4)}
# dual-averaging warm-up + main stage: (model, n_chains, step size, seed, n_warm, n_main, n_step,
# rng seed)
ADAPT_CASES = {"ul_adapt_ar1_64_dualavg": ("ar1_64", 4, 0.1, 8, 10, 3, 3, 913)}


def problem(model, n_chains, step_size, seed, integrator="implicit_leapfrog",
            integrator_kwargs=None):
    """Seeded positions near the model's truth and momenta from N(0, M(q)): ``mom = L(q) z``."""
    _, metric, _, _ = ul_model(model)
    rng = np.random.default_rng([20261019, seed])
    pos = ul_start(model, n_chains, rng)
    z = rng.standard_normal(pos.shape)
    mom = np.stack([metric.metric_func(q) @ zi for q, zi in zip(pos, z)])
    return pb.Problem(
        name="UL", integrator=integrator, system=rc.SYSTEM, target="ul_" + model,
        target_params={}, step_size=step_size, pos=pos, mom=mom, metric_model="ul_" + model,
        metric_params={}, integrator_kwargs=dict(integrator_kwargs or {}))


def case_problem(name):
    if name in CASES or name in FAILURE_CASES:
        model, n, eps, seed, _, integ, ikw = {**CASES, **FAILURE_CASES}[name]
        return problem(model, n, eps, seed, integ, ikw)
    model, n, eps, seed = {**HMC_CASES, **NUTS_CASES, **ADAPT_CASES}[name][:4]
    return problem(model, n, eps, seed)


@contextlib.contextmanager
def patched():
    """``oracle.drivers`` extended to the Cholesky-factored system (riemannian_chol_cases) and to
    the ``ul_*`` models: the oracle and the reference build their NumPy twins."""
    build_target, metric_model = dr.build_target, rc.metric_model

    def target(p):
        return ul_model(p.target[3:])[0] if p.target.startswith("ul_") else build_target(p)

    def metric(p):
        if p.metric_model and p.metric_model.startswith("ul_"):
            return ul_model(p.metric_model[3:])[1]
        return metric_model(p)

    dr.build_target, rc.metric_model = target, metric
    try:
        with rc.patched_drivers():
            yield dr
    finally:
        dr.build_target, rc.metric_model = build_target, metric_model


def make(name):
    p = case_problem(name)
    with patched():
        if name in CASES or name in FAILURE_CASES:
            steps = {**CASES, **FAILURE_CASES}[name][4]
            dirs = rc.case_dirs(p)
            rec = {"step_counts": np.array(steps), "dirs": dirs, "step_size": p.step_size}
            for n in steps:
                ref = dr.reference_run(p, n, dirs=dirs)
                orc = rc.oracle_integrator_run(p, n, dirs)
                for k in ("pos", "mom", "status", "n_done", "h"):
                    rec[f"{k}_{n}"] = ref[k]
                rec[f"fp_iters_{n}"] = orc["fp_iters"]
                print(name, n, "status", ref["status"].tolist())
        elif name in HMC_CASES:
            _, _, _, _, n_iter, n_step, seed = HMC_CASES[name]
            rec = dr.reference_hmc(p, n_iter, n_step, seed)
            print(name, "accept", rec["accept_stat"].round(3).tolist())
        elif name in NUTS_CASES:
            _, _, _, _, n_iter, seed, depth = NUTS_CASES[name]
            rec = dr.reference_nuts(p, n_iter, seed, max_tree_depth=depth)
            print(name, "n_step", rec["n_step"].tolist())
        else:
            from oracle.make_golden import STAGE_CODES, reference_stage_list

            _, _, _, _, n_warm, n_main, n_step, seed = ADAPT_CASES[name]
            ref = dr.reference_sample_chains(p, n_warm, n_main, n_step, seed, rc.ADAPT_SPECS)
            stages = reference_stage_list(rc.ADAPT_SPECS, None, n_warm, n_main)
            rec = dict(stage_n_iter=np.array([n for n, _ in stages]),
                       stage_which=np.array([STAGE_CODES[w] for _, w in stages]), **ref)
            print(name, "step size", float(ref["step_size"]), "n_step", ref["n_step"].tolist())
    np.savez(os.path.join(GOLDEN_DIR, name + ".npz"), **rec)


ALL = (*CASES, *FAILURE_CASES, *HMC_CASES, *NUTS_CASES, *ADAPT_CASES)

if __name__ == "__main__":
    for case in sys.argv[1:] or ALL:
        make(case)
