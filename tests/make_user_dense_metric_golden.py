"""Make the ``tests/golden/ud_*.npz`` fixtures of tests/test_user_dense_metric_gpu.py: dense
Riemannian models that the registry cannot express (tests/user_dense_metric_sources.py), run
through the unmodified reference's ``DenseRiemannianMetricSystem``, which takes their NumPy
``metric_func`` / ``vjp_metric_func`` natively.  The case tables, the problems and the oracle
hook live here too, so the tests build the same inputs.  Needs the reference (``oracle/_ref``,
placed by ``build()``):

    python tests/make_user_dense_metric_golden.py [case ...]
"""

import contextlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

import riemannian_diag_cases as rc  # noqa: E402
from mici_b200 import problems as pb  # noqa: E402
from oracle import drivers as dr  # noqa: E402
from user_dense_metric_sources import ud_model  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")

_POS_SCALE = {"logistic": 0.5, "lgcp64": 0.3, "lgcp144": 0.3}
_POS_MEAN = {"logistic": 0.0, "lgcp64": 0.5, "lgcp144": 0.5}

# integrator cases: (model, n_chains, step size, seed, step counts, integrator kwargs)
CASES = {
    "ud_lr_leapfrog": ("logistic", 6, 0.2, 1, (1, 5, 20), {}),
    "ud_lr_steffensen": ("logistic", 6, 0.2, 2, (1, 5, 20),
                         {"fixed_point_solver": "steffensen"}),
    "ud_lgcp64_leapfrog": ("lgcp64", 6, 0.1, 3, (1, 5, 20), {}),
    "ud_lgcp64_steffensen": ("lgcp64", 6, 0.1, 4, (1, 5, 20),
                             {"fixed_point_solver": "steffensen"}),
    "ud_lgcp144_leapfrog": ("lgcp144", 4, 0.1, 5, (1, 5, 20), {}),
}
# a big step: some chains end in ConvergenceError within 5 steps
FAILURE_CASES = {
    "ud_lgcp64_bigstep": ("lgcp64", 12, 0.35, 6, (1, 5), {}),
}
# static HMC: (model, n_chains, step size, seed, n_iter, n_step, rng seed)
HMC_CASES = {"ud_hmc_lr": ("logistic", 4, 0.2, 7, 4, 5, 811)}
# NUTS: (model, n_chains, step size, seed, n_iter, rng seed, max tree depth)
NUTS_CASES = {"ud_nuts_lgcp64": ("lgcp64", 3, 0.1, 8, 3, 812, 4)}
# dual-averaging warm-up + main stage: (model, n_chains, step size, seed, n_warm, n_main, n_step,
# rng seed)
ADAPT_CASES = {"ud_adapt_lr_dualavg": ("logistic", 4, 0.2, 9, 10, 3, 3, 813)}


def problem(model, n_chains, step_size, seed, integrator_kwargs=None):
    """Seeded positions and momenta from N(0, M(q)): ``mom = chol(M(q)) z``."""
    target, metric, _, _ = ud_model(model)
    rng = np.random.default_rng([20261018, seed])
    pos = _POS_MEAN[model] + _POS_SCALE[model] * rng.standard_normal((n_chains, target.dim))
    z = rng.standard_normal((n_chains, target.dim))
    mom = np.stack([np.linalg.cholesky(metric.metric_func(q)) @ zi for q, zi in zip(pos, z)])
    return pb.Problem(
        name="UD", integrator="implicit_leapfrog", system="dense_riemannian",
        target="ud_" + model, target_params={}, step_size=step_size, pos=pos, mom=mom,
        metric_model="ud_" + model, metric_params={},
        integrator_kwargs=dict(integrator_kwargs or {}))


def case_problem(name):
    if name in CASES or name in FAILURE_CASES:
        model, n, eps, seed, _, ikw = {**CASES, **FAILURE_CASES}[name]
        return problem(model, n, eps, seed, ikw)
    model, n, eps, seed = {**HMC_CASES, **NUTS_CASES, **ADAPT_CASES}[name][:4]
    return problem(model, n, eps, seed)


@contextlib.contextmanager
def patched():
    """``oracle.drivers`` extended to the ``ud_*`` models: the oracle and the reference build
    their NumPy twins."""
    build_target, build_metric = dr.build_target, dr.build_metric_model

    def target(p):
        return ud_model(p.target[3:])[0] if p.target.startswith("ud_") else build_target(p)

    def metric(p):
        if p.metric_model and p.metric_model.startswith("ud_"):
            return ud_model(p.metric_model[3:])[1]
        return build_metric(p)

    dr.build_target, dr.build_metric_model = target, metric
    try:
        yield dr
    finally:
        dr.build_target, dr.build_metric_model = build_target, build_metric


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
