"""User-written Cholesky-factor metrics on CholeskyFactoredRiemannianMetricSystem, on the device:
the registry's quadratic factor model rewritten as user sources (tests/user_chol_metric_sources.py)
against the reference fixtures of the registry model (tests/golden/rc_*.npz) and against the
registry kernels on identical inputs; the hierarchical AR(1) model, which the registry cannot
express, against fixtures of the unmodified reference (tests/golden/ul_*.npz,
tests/make_user_chol_metric_golden.py) and against the NumPy oracle; and chains whose factor is
not finite or is singular, which must leave every other chain unchanged."""

import numpy as np
import pytest
import torch

from mici_b200 import engine, jit, problems, targets, transitions
from mici_b200.errors import LinAlgError
from mici_b200.integrators import ImplicitLeapfrogIntegrator
from mici_b200.states import ChainState
from mici_b200.systems import CholeskyFactoredRiemannianMetricSystem
from mici_b200.targets import CudaCholeskyMetric, CudaTarget

import make_user_chol_metric_golden as ul
import riemannian_chol_cases as rc
import user_chol_metric_sources as ucs
from golden_util import ATOL, RTOL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

TARGETS = {"std_gaussian": ucs.STD_GAUSSIAN, "banana": ucs.BANANA, "neal_funnel": ucs.FUNNEL,
           "quadratic": ucs.QUADRATIC}


@pytest.fixture(scope="module", autouse=True)
def _compiled_images():
    """Compile the module's five images at once (NVRTC runs outside the GIL)."""
    from concurrent.futures import ThreadPoolExecutor  # noqa: PLC0415

    pairs = [(src, name, ucs.QUADRATIC_CHOL, "quadratic_chol") for name, src in TARGETS.items()]
    pairs.append((ucs.AR1_HIER, "ar1_hier", ucs.AR1_HIER_CHOL, "metric"))
    with ThreadPoolExecutor(len(pairs)) as pool:
        list(pool.map(lambda a: jit.compile_target(a[0], a[1], metric=("cholesky", a[2], a[3])),
                      pairs))


def user_system(problem):
    """The problem's registry target and quadratic factor model rewritten as user sources, or the
    user sources of a ``ul_*`` model."""
    if problem.target.startswith("ul_"):
        _, _, (tsrc, tparams, taux), (msrc, mparams, maux) = ucs.ul_model(problem.target[3:])
        target = CudaTarget(problem.pos.shape[1], tsrc, params=tparams, aux=taux, name="ar1_hier")
        return CholeskyFactoredRiemannianMetricSystem(
            target, CudaCholeskyMetric(msrc, params=mparams, aux=maux, name="metric"))
    t = targets.make_target(problem.target, **problem.target_params)
    mm = targets.make_metric_model(problem.metric_model, **problem.metric_params)
    target = CudaTarget(t.dim, TARGETS[problem.target], params=t.params, aux=t.aux,
                        name=problem.target)
    metric = CudaCholeskyMetric(ucs.QUADRATIC_CHOL, params=mm.params, aux=mm.aux,
                                name="quadratic_chol")
    return CholeskyFactoredRiemannianMetricSystem(target, metric)


def run(problem, n_steps, system=None, dirs=None):
    integ = engine.build_integrator(problem, system=system)
    state = engine.build_state(problem, DEV, dirs=dirs)
    new = integ.step_n(state, n_steps, return_h=True)
    torch.cuda.synchronize()
    return {k: getattr(new, a).cpu().numpy()
            for k, a in (("pos", "pos"), ("mom", "mom"), ("status", "status"),
                         ("n_done", "n_done"), ("h", "h"), ("iters", "solver_iters"))}


def _check_integrator_fixture(name, problem, g, system):
    """pos / mom at rtol 1e-10 (1e-9 after 20 Steffensen steps, as for the registry), h at rtol
    1e-10; status and completed steps exactly; the fixed-point iterations of the last completed
    step exactly with the direct solver and in all but one solve in a hundred with Steffensen's,
    whose extrapolation can move an iterate across the tolerance on last-bit differences."""
    for n in g["step_counts"]:
        out = run(problem, int(n), system=system, dirs=g["dirs"])
        lbl = f"{name}[{n}]"
        rtol = 1e-9 if "steffensen" in name and n == 20 else RTOL
        np.testing.assert_array_equal(out["status"], g[f"status_{n}"], err_msg=lbl)
        np.testing.assert_array_equal(out["n_done"], g[f"n_done_{n}"], err_msg=lbl)
        np.testing.assert_allclose(out["pos"], g[f"pos_{n}"], rtol=rtol, atol=ATOL, err_msg=lbl)
        np.testing.assert_allclose(out["mom"], g[f"mom_{n}"], rtol=rtol, atol=ATOL, err_msg=lbl)
        np.testing.assert_array_equal(np.isnan(out["h"]), np.isnan(g[f"h_{n}"]), err_msg=lbl)
        ok = np.isfinite(g[f"h_{n}"])
        np.testing.assert_allclose(out["h"][ok], g[f"h_{n}"][ok], rtol=RTOL, atol=1e-9,
                                   err_msg=lbl)
        done = out["n_done"] > 0
        if "steffensen" in name:
            differ = out["iters"][done] != g[f"fp_iters_{n}"][done]
            assert differ.sum() <= max(1, differ.size // 100), (lbl, out["iters"])
        else:
            np.testing.assert_array_equal(out["iters"][done], g[f"fp_iters_{n}"][done],
                                          err_msg=lbl)


@pytest.mark.parametrize("name", sorted(rc.ALL_INTEGRATOR_CASES))
def test_registry_model_as_user_sources_matches_reference_fixture(name):
    """Every rc_* integrator case: D = 1 .. 200 (both layouts), both integrators, both solvers,
    big steps, and the negative-diagonal / exactly singular starts."""
    problem = rc.case_problem(name)
    _check_integrator_fixture(name, problem, rc.load_fixture(name), user_system(problem))


@pytest.mark.parametrize("name", sorted({**ul.CASES, **ul.FAILURE_CASES}))
def test_ar1_model_matches_reference_fixture(name):
    """The hierarchical AR(1) model at T = 64 (D = 66, shared memory) and T = 254 (D = 256, the
    per-CTA workspace): leapfrog, midpoint, Steffensen, and a big step at which some chains end
    in ConvergenceError or NonReversibleStepError."""
    problem = ul.case_problem(name)
    g = rc.load_fixture(name)
    _check_integrator_fixture(name, problem, g, user_system(problem))
    if name in ul.FAILURE_CASES:
        assert (g[f"status_{g['step_counts'][-1]}"] != 0).any()


def _case(name):
    if name.startswith("ul_"):
        return ul.case_problem(name), rc.load_fixture(name)
    return rc.case_problem(name), rc.load_fixture(name)


@pytest.mark.parametrize("name", sorted(rc.HMC_CASES) + sorted(ul.HMC_CASES))
def test_batched_hmc_matches_reference_fixture(name):
    """Static HMC, momentum refresh through the user image included."""
    problem, g = _case(name)
    n_iter, n_step, seed = (ul.HMC_CASES[name][4:] if name in ul.HMC_CASES
                            else rc.HMC_CASES[name][1:])
    integ = engine.build_integrator(problem, system=user_system(problem))
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    final, stats, trace = transitions.sample_hmc(integ.system, integ, state, rngs, n_iter, n_step,
                                                 trace_pos=True)
    torch.cuda.synchronize()
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-9, atol=1e-11)
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"])
    np.testing.assert_array_equal(stats["n_step"].cpu().numpy(), g["n_step"])
    np.testing.assert_allclose(stats["metrop_accept_prob"].cpu().numpy(), g["metrop_accept_prob"],
                               rtol=1e-8, atol=1e-12)


@pytest.mark.parametrize("name", sorted(rc.NUTS_CASES) + sorted(ul.NUTS_CASES))
def test_nuts_matches_reference_fixture(name):
    """MultinomialDynamicIntegrationTransition through the lock-step generic NUTS path."""
    problem, g = _case(name)
    n_iter, seed, depth = (ul.NUTS_CASES[name][4:] if name in ul.NUTS_CASES
                           else rc.NUTS_CASES[name][1:])
    integ = engine.build_integrator(problem, system=user_system(problem))
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    final, stats, trace = transitions.sample_chains(
        integ.system, integ, state, rngs, 0, n_iter,
        integration_transition=transitions.MultinomialDynamicIntegrationTransition(
            integ.system, integ, max_tree_depth=depth))
    torch.cuda.synchronize()
    for k in ("n_step", "tree_depth", "diverging"):
        np.testing.assert_array_equal(stats[k].cpu().numpy().astype(np.float64), g[k], err_msg=k)
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"][-1])
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-8, atol=1e-10)
    for k in ("av_metrop_accept_prob", "accept_stat"):
        np.testing.assert_allclose(stats[k].cpu().numpy(), g[k], rtol=1e-7, atol=1e-10, err_msg=k)


@pytest.mark.parametrize("name", sorted(rc.ADAPT_CASES) + sorted(ul.ADAPT_CASES))
def test_dual_averaging_warm_up_matches_reference_fixture(name):
    """Dual-averaging warm-up plus a main stage through ``StaticMetropolisHMC.sample_chains``."""
    from mici_b200 import adapters, samplers  # noqa: PLC0415

    problem, g = _case(name)
    n_warm, n_main, n_step, seed = (ul.ADAPT_CASES[name][4:] if name in ul.ADAPT_CASES
                                    else rc.ADAPT_CASES[name][1:])
    integ = engine.build_integrator(problem, system=user_system(problem))
    state = engine.build_state(problem, DEV)
    sampler = samplers.StaticMetropolisHMC(integ.system, integ, np.random.default_rng(seed),
                                           n_step)
    out = sampler.sample_chains(n_warm, n_main, state,
                                adapters=[adapters.DualAveragingStepSizeAdapter()],
                                trace_warm_up=True, n_worker=1, display_progress=False)
    torch.cuda.synchronize()
    stats = {k: v.transpose(0, 1).cpu().numpy() for k, v in out.statistics.items()}
    pos = out.traces["pos"].transpose(0, 1).cpu().numpy()
    np.testing.assert_array_equal(stats["n_step"], g["n_step"])
    np.testing.assert_array_equal(out.final_states.dir.cpu().numpy(), g["final_dir"])
    k = 4
    np.testing.assert_allclose(stats["accept_stat"][:k], g["accept_stat"][:k], rtol=1e-7,
                               atol=1e-10)
    np.testing.assert_allclose(pos[:k], g["pos"][:k], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(stats["accept_stat"], g["accept_stat"], rtol=1e-2, atol=1e-3)
    np.testing.assert_allclose(pos, g["pos"], rtol=1e-3, atol=1e-4)
    assert integ.step_size == pytest.approx(float(g["step_size"]), rel=1e-4)


def _compare(reg, usr, label):
    for k in ("status", "n_done", "iters"):
        np.testing.assert_array_equal(usr[k], reg[k], err_msg=f"{label} {k}")
    for k in ("pos", "mom", "h"):
        np.testing.assert_allclose(usr[k], reg[k], rtol=RTOL, atol=ATOL, err_msg=f"{label} {k}")


@pytest.mark.parametrize("integrator", ["implicit_leapfrog", "implicit_midpoint"])
@pytest.mark.parametrize("dim,n_chains", [(5, 1024), (64, 1024), (128, 512), (200, 264),
                                          (1016, 132)])
def test_user_quadratic_factor_against_registry_on_identical_inputs(dim, n_chains, integrator):
    """C8 in mixed directions, 3 steps: the registry's quadratic factor model against the same
    model written as user sources.  Status, completed steps and fixed-point iterations identical;
    pos, mom and h within rtol 1e-10.  Both fill L with the same expression; the user VJP sums
    V q and V^T q in another order than the registry's scans, so the results are not expected to
    agree bit for bit.  D = 5 and 64 run both sides in shared memory; at D = 128 the user image
    (two matrices per chain) runs on the workspace route while the registry stays in shared
    memory; at 200 and 1016 (the user bound) both use the workspace."""
    problem = problems.make_problem("C8", n_chains=n_chains, dim=dim, integrator=integrator)
    dirs = np.where(np.arange(n_chains) % 2 == 0, 1, -1).astype(np.int32)
    reg = run(problem, 3, system=engine.build_system(problem), dirs=dirs)
    usr = run(problem, 3, system=user_system(problem), dirs=dirs)
    assert (reg["status"] == 0).mean() > 0.9
    _compare(reg, usr, f"C8 D={dim} {integrator}")


@pytest.mark.parametrize("name", ["ul_ar1_64_leapfrog", "ul_ar1_254_leapfrog",
                                  "ul_ar1_64_midpoint"])
def test_h_dh_dmom_and_sample_momentum_match_oracle(name):
    """h at rtol 1e-12, the velocity at rtol 1e-12 and the momentum refresh L(q) z at rtol 1e-13,
    against the NumPy oracle of the same model."""
    problem = ul.case_problem(name)
    system = user_system(problem)
    state = engine.build_state(problem, DEV)
    h = system.h(state).cpu().numpy()
    vel = system.dh_dmom(state).cpu().numpy()
    rngs = [np.random.default_rng([5, c]) for c in range(problem.n_chains)]
    mom = system.sample_momentum(state, rngs).cpu().numpy()
    with ul.patched() as dr:
        _, h_fn, osys = dr.oracle_step_fn(problem)
        for c in range(problem.n_chains):
            q, p = problem.pos[c], problem.mom[c]
            assert h[c] == pytest.approx(h_fn(q, p), rel=1e-12)
            np.testing.assert_allclose(vel[c], osys.dh2_dmom(q, p), rtol=1e-12, atol=1e-14)
            z = np.random.default_rng([5, c]).normal(size=problem.pos.shape[1])
            np.testing.assert_allclose(mom[c], osys.metric(q).sqrt_matvec(z), rtol=1e-13,
                                       atol=1e-14)


def test_failing_factors_are_errors_and_leave_the_other_chains_bit_identical():
    """L(q) = diag(-1, 1, ..., 1) + tril(q q^T) (the user quadratic factor, c = 1): chain 1
    starts where L is not finite (LinAlgError in dh_dmom, sample_momentum and a step), chain 2
    with q0 = 1, L00 = 0 exactly (dh_dmom raises, h is NaN, a step ends in ConvergenceError,
    sample_momentum succeeds), chain 4 with q0 = 0.5, L00 < 0 (legal).  The other chains'
    outputs are bit-identical to a run without chains 1 and 2."""
    dim, n = 24, 8
    base = np.identity(dim)
    base[0, 0] = -1.0
    target = CudaTarget(dim, ucs.STD_GAUSSIAN, name="std_gaussian")
    metric = CudaCholeskyMetric(ucs.QUADRATIC_CHOL, params=(1.0,), aux=base,
                                name="quadratic_chol")
    system = CholeskyFactoredRiemannianMetricSystem(target, metric)
    rng = np.random.default_rng(9)
    pos, mom = 0.1 * rng.standard_normal((n, dim)), 0.1 * rng.standard_normal((n, dim))
    pos[:, 0] = 2.0
    pos[1, 3] = 1e200
    pos[2, 0] = 1.0
    pos[4, 0] = 0.5
    bad = [1, 2]
    good = [c for c in range(n) if c not in bad]

    def state(rows):
        return ChainState(pos=torch.as_tensor(pos[rows], device=DEV),
                          mom=torch.as_tensor(mom[rows], device=DEV), dir=1)

    for rows in ([0, 1], [0, 2]):
        with pytest.raises(LinAlgError):
            system.dh_dmom(state(rows))
    with pytest.raises(LinAlgError):
        system.sample_momentum(state([0, 1]), [np.random.default_rng(c) for c in range(2)])
    system.sample_momentum(state([0, 2, 4]), [np.random.default_rng(c) for c in range(3)])
    h = system.h(state(list(range(n)))).cpu().numpy()
    assert np.isnan(h[[1, 2]]).all() and np.isfinite(h[good]).all()
    integ = ImplicitLeapfrogIntegrator(system, 0.02)
    outs = []
    for rows in (list(range(n)), good):
        new = integ.step_n(state(rows), 2, return_h=True)
        outs.append({k: getattr(new, k).cpu().numpy()
                     for k in ("pos", "mom", "h", "status", "n_done", "solver_iters")})
    full, sub = outs
    assert full["status"][1] == 3 and full["status"][2] == 1, full["status"]
    assert (full["status"][good] == 0).all(), full["status"]
    for k in sub:
        np.testing.assert_array_equal(full[k][good], sub[k], err_msg=k)
