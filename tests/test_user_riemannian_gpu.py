"""User-written targets and metrics on the diagonal and scalar Riemannian systems, on the device:
the registry's models rewritten as user sources (tests/user_riemannian_sources.py) against the
reference fixtures of the registry models (tests/golden/rd_*.npz) and against the registry
kernels on identical inputs; models the registry cannot express (eight schools, logistic
regression, Student-t) against fixtures of the unmodified reference (tests/golden/ur_*.npz,
tests/make_user_riemannian_golden.py) and against the NumPy oracle; and the failure of a metric
that is not positive."""

import numpy as np
import pytest
import torch

from mici_b200 import engine, problems, targets, transitions
from mici_b200.errors import LinAlgError
from mici_b200.systems import DiagonalRiemannianMetricSystem, ScalarRiemannianMetricSystem
from mici_b200.targets import CudaDiagonalMetric, CudaScalarMetric, CudaTarget

import make_user_riemannian_golden as ur
import riemannian_diag_cases as rc
import user_riemannian_sources as us
from golden_util import ATOL, RTOL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

TARGETS = {"std_gaussian": us.STD_GAUSSIAN, "banana": us.BANANA, "neal_funnel": us.FUNNEL}
METRICS = {"diag_quadratic": (CudaDiagonalMetric, us.QUADRATIC_DIAGONAL),
           "funnel_fisher": (CudaDiagonalMetric, us.FUNNEL_FISHER),
           "scalar_quadratic": (CudaScalarMetric, us.QUADRATIC_SCALAR)}


def user_system(problem):
    """The problem's registry target and metric rewritten as user sources, or the user sources of
    a ``ur_*`` model."""
    if problem.target.startswith("ur_"):
        _, _, (tsrc, tparams, taux), (kind, msrc, mparams, maux) = us.ur_model(problem.target[3:])
        target = CudaTarget(problem.pos.shape[1], tsrc, params=tparams, aux=taux,
                            name=problem.target)
        if kind == "diagonal":
            return DiagonalRiemannianMetricSystem(
                target, CudaDiagonalMetric(msrc, params=mparams, aux=maux, name="metric"))
        return ScalarRiemannianMetricSystem(
            target, CudaScalarMetric(msrc, params=mparams, aux=maux, name="metric"))
    t = targets.make_target(problem.target, **problem.target_params)
    mm = targets.make_metric_model(problem.metric_model, **problem.metric_params)
    cls, msrc = METRICS[problem.metric_model]
    target = CudaTarget(t.dim, TARGETS[problem.target], params=t.params, name=problem.target)
    metric = cls(msrc, params=mm.params, name=problem.metric_model)
    system_cls = (DiagonalRiemannianMetricSystem if cls is CudaDiagonalMetric
                  else ScalarRiemannianMetricSystem)
    return system_cls(target, metric)


def run(problem, n_steps, system=None, dirs=None, chains=None):
    integ = engine.build_integrator(problem, system=system)
    state = engine.build_state(problem, DEV, dirs=dirs, chains=chains)
    new = integ.step_n(state, n_steps, return_h=True)
    torch.cuda.synchronize()
    return {k: getattr(new, a).cpu().numpy()
            for k, a in (("pos", "pos"), ("mom", "mom"), ("status", "status"),
                         ("n_done", "n_done"), ("h", "h"), ("iters", "solver_iters"))}


def _case(name):
    """(problem, fixture) of an rd_* case (registry model as user sources) or a ur_* case."""
    if name.startswith("ur_"):
        return ur.case_problem(name), rc.load_fixture(name)
    return rc.case_problem(name), rc.load_fixture(name)


def _registry_expressible(names):
    return sorted(n for n in names if rc.case_problem(n).target in TARGETS)


INTEGRATOR_CASES = (_registry_expressible(rc.ALL_INTEGRATOR_CASES)
                    + sorted({**ur.CASES, **ur.FAILURE_CASES}))


@pytest.mark.parametrize("name", INTEGRATOR_CASES)
def test_user_sources_match_reference_fixture(name):
    """The tolerances of test_diagonal_riemannian_gpu.py: pos / mom at rtol 1e-10, atol 1e-12 (1e-9
    for 20 Steffensen steps), h at rtol 1e-10; status, completed steps and fixed-point iterations
    exactly.  Implicit leapfrog and midpoint over 1 / 5 / 20 steps in mixed directions, and the
    big-step failures."""
    problem, g = _case(name)
    system = user_system(problem)
    for n in g["step_counts"]:
        out = run(problem, int(n), system=system, dirs=g["dirs"])
        lbl = f"{name}[{n}]"
        rtol = 1e-9 if "steffensen" in name and n == 20 else RTOL
        np.testing.assert_array_equal(out["status"], g[f"status_{n}"], err_msg=lbl)
        np.testing.assert_array_equal(out["n_done"], g[f"n_done_{n}"], err_msg=lbl)
        np.testing.assert_allclose(out["pos"], g[f"pos_{n}"], rtol=rtol, atol=ATOL, err_msg=lbl)
        np.testing.assert_allclose(out["mom"], g[f"mom_{n}"], rtol=rtol, atol=ATOL, err_msg=lbl)
        ok = np.isfinite(g[f"h_{n}"])
        np.testing.assert_allclose(out["h"][ok], g[f"h_{n}"][ok], rtol=RTOL, atol=1e-9,
                                   err_msg=lbl)
        done = out["n_done"] > 0
        np.testing.assert_array_equal(out["iters"][done], g[f"fp_iters_{n}"][done], err_msg=lbl)


def _compare(reg, usr, label):
    for k in ("status", "n_done", "iters"):
        np.testing.assert_array_equal(usr[k], reg[k], err_msg=f"{label} {k}")
    for k in ("pos", "mom", "h"):
        np.testing.assert_allclose(usr[k], reg[k], rtol=1e-9, atol=0, err_msg=f"{label} {k}")
    return all(np.array_equal(usr[k], reg[k], equal_nan=True) for k in ("pos", "mom", "h"))


@pytest.mark.parametrize("metric_kind,dim,midpoint", [
    ("fisher", 128, False), ("scalar", 128, False), ("fisher", 128, True), ("scalar", 1024, False),
    ("fisher", 1024, False)])
def test_user_against_registry_on_identical_inputs(metric_kind, dim, midpoint):
    """C7 (funnel, 8192 chains, 10 implicit steps) and D = 1024: status, completed steps,
    fixed-point iterations and call counters identical; pos, mom and h to 1e-9 relative."""
    n_chains = 8192 if dim == 128 else 1024
    problem = problems.make_problem(
        "C7", n_chains=n_chains, dim=dim, metric_kind=metric_kind,
        integrator="implicit_midpoint" if midpoint else "implicit_leapfrog")
    reg_sys, usr_sys = engine.build_system(problem), user_system(problem)
    counts = []
    outs = []
    for system in (reg_sys, usr_sys):
        from mici_b200 import _lib  # noqa: PLC0415

        c = torch.zeros((n_chains, 4), dtype=torch.int32, device=DEV)
        _lib.check(_lib.load().mb200_set_call_counters(_lib.ptr(c)), "counters")
        try:
            outs.append(run(problem, 10, system=system))
        finally:
            _lib.load().mb200_set_call_counters(None)
        counts.append(c.cpu().numpy())
    bitwise = _compare(outs[0], outs[1], f"C7 {metric_kind} D={dim}")
    np.testing.assert_array_equal(counts[1], counts[0])
    print(f"user vs registry, {metric_kind} D={dim} midpoint={midpoint}: bitwise equal: {bitwise}")


@pytest.mark.parametrize("name", sorted(rc.HMC_CASES) + sorted(ur.HMC_CASES))
def test_batched_hmc_matches_reference_fixture(name):
    """Static HMC, momentum refresh through the user image included, as the registry test."""
    problem, g = _case(name)
    _, n_iter, n_step, seed = (rc.HMC_CASES[name] if name in rc.HMC_CASES
                               else ur.HMC_CASES[name][3:])
    integ = engine.build_integrator(problem, system=user_system(problem))
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    final, stats, trace = transitions.sample_hmc(integ.system, integ, state, rngs, n_iter, n_step,
                                                 trace_pos=True)
    torch.cuda.synchronize()
    np.testing.assert_allclose(trace.cpu().numpy()[0], g["pos"][0], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-9, atol=1e-11)
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"])
    np.testing.assert_array_equal(stats["n_step"].cpu().numpy(), g["n_step"])
    np.testing.assert_allclose(stats["metrop_accept_prob"].cpu().numpy(), g["metrop_accept_prob"],
                               rtol=1e-8, atol=1e-12)


@pytest.mark.parametrize("name", sorted(rc.NUTS_CASES) + sorted(ur.NUTS_CASES))
def test_nuts_matches_reference_fixture(name):
    """MultinomialDynamicIntegrationTransition through the lock-step generic NUTS path."""
    problem, g = _case(name)
    if name in rc.NUTS_CASES:
        _, n_iter, seed, depth = rc.NUTS_CASES[name]
    else:
        _, _, _, _, n_iter, seed, depth = ur.NUTS_CASES[name]
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


@pytest.mark.parametrize("name", sorted(rc.ADAPT_CASES) + sorted(ur.ADAPT_CASES))
def test_dual_averaging_warm_up_matches_reference_fixture(name):
    """Dual-averaging warm-up plus a main stage through ``StaticMetropolisHMC.sample_chains``,
    at the tolerances of the registry test."""
    from mici_b200 import adapters, samplers  # noqa: PLC0415

    problem, g = _case(name)
    n_warm, n_main, n_step, seed = (rc.ADAPT_CASES[name][1:] if name in rc.ADAPT_CASES
                                    else ur.ADAPT_CASES[name][4:])
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


@pytest.mark.parametrize("name", ["rd_dq_banana_d8_midpoint", "rd_ff_funnel_d10",
                                  "rd_sc_banana_d64", "rd_dq_std_d33", "ur_es_leapfrog",
                                  "ur_lr_leapfrog", "ur_st_leapfrog"])
def test_h_dh_dmom_and_sample_momentum_match_oracle(name):
    """h at rtol 1e-12, the velocity and the momentum refresh at rtol 1e-15, against the NumPy
    oracle of the same model, as the registry test."""
    problem, _ = _case(name)
    system = user_system(problem)
    state = engine.build_state(problem, DEV)
    h = system.h(state).cpu().numpy()
    vel = system.dh_dmom(state).cpu().numpy()
    rngs = [np.random.default_rng([5, c]) for c in range(problem.n_chains)]
    mom = system.sample_momentum(state, rngs).cpu().numpy()
    with ur.patched() as dr:
        _, h_fn, osys = dr.oracle_step_fn(problem)
        for c in range(problem.n_chains):
            q = problem.pos[c]
            assert h[c] == pytest.approx(h_fn(q, problem.mom[c]), rel=1e-12)
            np.testing.assert_allclose(vel[c], osys.dh2_dmom(q, problem.mom[c]), rtol=1e-15,
                                       atol=0)
            z = np.random.default_rng([5, c]).normal(size=problem.pos.shape[1])
            np.testing.assert_allclose(mom[c], osys.metric(q).sqrt_matvec(z), rtol=1e-15, atol=0)


def test_non_positive_user_metric_is_a_linalg_error_and_ends_a_step_in_convergence_error():
    """d_i = a + b q_i^2 with a < 0: dh_dmom raises LinAlgError; an integrator step whose
    fixed-point iterates leave the positive region ends with ConvergenceError (status 1)."""
    from mici_b200.integrators import ImplicitLeapfrogIntegrator  # noqa: PLC0415
    from mici_b200.states import ChainState  # noqa: PLC0415

    target = CudaTarget(4, us.STD_GAUSSIAN)
    bad = DiagonalRiemannianMetricSystem(target, CudaDiagonalMetric(us.QUADRATIC_DIAGONAL,
                                                                    params=(-1.0, 1.0)))
    g = torch.Generator().manual_seed(3)
    state = ChainState(pos=(0.1 * torch.randn((4, 4), generator=g, dtype=torch.float64)).to(DEV),
                       mom=torch.randn((4, 4), generator=g, dtype=torch.float64).to(DEV), dir=1)
    with pytest.raises(LinAlgError):
        bad.dh_dmom(state)
    # s = a + b |q|^2 is positive at q = 0 and crosses zero inside the position fixed point
    scalar = ScalarRiemannianMetricSystem(target, CudaScalarMetric(us.QUADRATIC_SCALAR,
                                                                  params=(1e-3, -1.0)))
    state = ChainState(pos=torch.zeros((4, 4), dtype=torch.float64, device=DEV),
                       mom=torch.full((4, 4), 0.5, dtype=torch.float64, device=DEV), dir=1)
    new = ImplicitLeapfrogIntegrator(scalar, 0.5).step_n(state, 1, return_h=True)
    assert set(new.status.cpu().tolist()) == {1}, new.status
