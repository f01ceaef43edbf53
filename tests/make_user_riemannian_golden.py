"""Make the ``tests/golden/ur_*.npz`` fixtures of tests/test_user_riemannian_gpu.py: diagonal and
scalar Riemannian models that the registry cannot express (tests/user_riemannian_sources.py),
run through the unmodified reference, which takes their NumPy callables natively.  The case
tables, the problems and the oracle hook live here too, so the tests build the same inputs.
Needs the reference (``oracle/_ref``, placed by ``build()``):

    python tests/make_user_riemannian_golden.py [case ...]
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
from user_riemannian_sources import ur_model  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")

# model -> (start position scale per coordinate, or a scalar)
_POS_SCALE = {"eight_schools": 0.5, "logistic": 0.5, "student_t": 1.0}

# integrator cases: (model, integrator, n_chains, step size, seed, step counts)
CASES = {
    "ur_es_leapfrog": ("eight_schools", "implicit_leapfrog", 8, 0.1, 1, (1, 5, 20)),
    "ur_es_midpoint": ("eight_schools", "implicit_midpoint", 8, 0.1, 2, (1, 5, 20)),
    "ur_lr_leapfrog": ("logistic", "implicit_leapfrog", 6, 0.2, 3, (1, 5, 20)),
    "ur_lr_midpoint": ("logistic", "implicit_midpoint", 6, 0.2, 4, (1, 5, 20)),
    "ur_st_leapfrog": ("student_t", "implicit_leapfrog", 8, 0.3, 5, (1, 5, 20)),
    "ur_st_midpoint": ("student_t", "implicit_midpoint", 8, 0.3, 6, (1, 5, 20)),
}
# a big step: within 5 steps 6 of 24 chains fail with ConvergenceError (at larger steps the
# iterates overflow exp(-2 log tau), where whether a chain fails by divergence or by
# irreversibility turns on rounding)
FAILURE_CASES = {
    "ur_es_leapfrog_bigstep": ("eight_schools", "implicit_leapfrog", 24, 0.7, 7, (1, 5)),
}
# static HMC: (model, n_chains, step size, seed, n_iter, n_step, rng seed)
HMC_CASES = {"ur_hmc_st": ("student_t", 4, 0.3, 8, 4, 5, 801)}
# NUTS: (model, n_chains, step size, seed, n_iter, rng seed, max tree depth)
NUTS_CASES = {"ur_nuts_es": ("eight_schools", 3, 0.15, 9, 3, 802, 4)}
# dual-averaging warm-up + main stage: (model, n_chains, step size, seed, n_warm, n_main, n_step,
# rng seed)
ADAPT_CASES = {"ur_adapt_lr_dualavg": ("logistic", 4, 0.2, 10, 10, 3, 3, 803)}


def problem(model, integrator, n_chains, step_size, seed):
    """Seeded positions and momenta from N(0, M(q)), as riemannian_diag_cases.make_problem."""
    target, metric, _, (kind, _, _, _) = ur_model(model)
    rng = np.random.default_rng([20261017, seed])
    pos = _POS_SCALE[model] * rng.standard_normal((n_chains, target.dim))
    z = rng.standard_normal((n_chains, target.dim))
    if kind == "diagonal":
        mom = z * np.sqrt(np.stack([metric.metric_func(q) for q in pos]))
    else:
        mom = z * np.sqrt(np.array([metric.metric_func(q) for q in pos]))[:, None]
    return pb.Problem(
        name="UR", integrator=integrator, system=kind + "_riemannian", target="ur_" + model,
        target_params={}, step_size=step_size, pos=pos, mom=mom, metric_model="ur_" + model,
        metric_params={})


def case_problem(name):
    if name in CASES or name in FAILURE_CASES:
        model, integrator, n, eps, seed, _ = {**CASES, **FAILURE_CASES}[name]
        return problem(model, integrator, n, eps, seed)
    model, n, eps, seed = {**HMC_CASES, **NUTS_CASES, **ADAPT_CASES}[name][:4]
    return problem(model, "implicit_leapfrog", n, eps, seed)


@contextlib.contextmanager
def patched():
    """``oracle.drivers`` and the diagonal / scalar oracle of riemannian_diag_cases, extended to
    the ``ur_*`` models: the oracle and the reference build their NumPy twins."""
    build_target = dr.build_target

    def build(p):
        if p.target.startswith("ur_"):
            return ur_model(p.target[3:])[0]
        return build_target(p)

    models = {"ur_" + m: (lambda m=m: ur_model(m)[1])
              for m in ("eight_schools", "logistic", "student_t")}
    dr.build_target = build
    rc.MODELS.update(models)
    try:
        with rc.patched_drivers() as d:
            yield d
    finally:
        dr.build_target = build_target
        for k in models:
            rc.MODELS.pop(k, None)


def make(name):
    p = case_problem(name)
    with patched():
        if name in CASES or name in FAILURE_CASES:
            steps = {**CASES, **FAILURE_CASES}[name][5]
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
