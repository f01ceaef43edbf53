"""User-written dense metrics on DenseRiemannianMetricSystem, on the device: the registry's rank-1
and Hadamard metrics rewritten as user sources (tests/user_dense_metric_sources.py) against the
reference fixtures of the registry models (c4_dense_riemannian_*, c5_hadamard_*) and against the
registry kernels on identical inputs; models the registry cannot express (logistic regression with
its dense Fisher metric, the log-Gaussian Cox process) against fixtures of the unmodified reference
(tests/golden/ud_*.npz, tests/make_user_dense_metric_golden.py) and against the NumPy oracle; and
chains whose metric is not finite or not positive definite, which must leave every other chain
unchanged."""

import numpy as np
import pytest
import torch

from mici_b200 import engine, jit, problems, targets, transitions
from mici_b200.errors import LinAlgError
from mici_b200.integrators import ImplicitLeapfrogIntegrator
from mici_b200.states import ChainState
from mici_b200.systems import DenseRiemannianMetricSystem
from mici_b200.targets import CudaDenseMetric, CudaTarget

import make_user_dense_metric_golden as ud
import riemannian_diag_cases as rc
import user_dense_metric_sources as uds
from golden_util import ATOL, RTOL, assert_matches_golden, load_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

REGISTRY_METRICS = {"rank1": uds.RANK1_DENSE, "hadamard": uds.HADAMARD_DENSE}


@pytest.fixture(scope="module", autouse=True)
def _compiled_images():
    """Compile the module's four images at once (NVRTC runs outside the GIL): each takes about a
    minute of one CPU core."""
    from concurrent.futures import ThreadPoolExecutor  # noqa: PLC0415

    pairs = [(uds.QUADRATIC, "quadratic", m, name) for name, m in REGISTRY_METRICS.items()]
    pairs += [(tsrc, "ud_" + model.rstrip("0123456789"), msrc, "metric")
              for model, ((tsrc, _, _), (msrc, _, _)) in
              ((m, uds.ud_model(m)[2:]) for m in ("logistic", "lgcp64"))]
    with ThreadPoolExecutor(len(pairs)) as pool:
        list(pool.map(lambda a: jit.compile_target(a[0], a[1], metric=("dense", a[2], a[3])),
                      pairs))


def user_system(problem):
    """The problem's registry quadratic target and rank-1 / Hadamard metric rewritten as user
    sources, or the user sources of a ``ud_*`` model."""
    if problem.target.startswith("ud_"):
        _, _, (tsrc, tparams, taux), (msrc, mparams, maux) = uds.ud_model(problem.target[3:])
        # one image for the LGCP at every size
        target = CudaTarget(problem.pos.shape[1], tsrc, params=tparams, aux=taux,
                            name=problem.target.rstrip("0123456789"))
        return DenseRiemannianMetricSystem(
            target, CudaDenseMetric(msrc, params=mparams, aux=maux, name="metric"))
    t = targets.make_target(problem.target, **problem.target_params)
    mm = targets.make_metric_model(problem.metric_model, **problem.metric_params)
    target = CudaTarget(t.dim, uds.QUADRATIC, aux=t.aux, name="quadratic")
    metric = CudaDenseMetric(REGISTRY_METRICS[problem.metric_model], params=mm.params[:1],
                             aux=mm.base if problem.metric_model == "rank1" else mm.aux,
                             name=problem.metric_model)
    return DenseRiemannianMetricSystem(target, metric)


def run(problem, n_steps, system=None, dirs=None, chains=None):
    integ = engine.build_integrator(problem, system=system)
    state = engine.build_state(problem, DEV, dirs=dirs, chains=chains)
    new = integ.step_n(state, n_steps, return_h=True)
    torch.cuda.synchronize()
    return {k: getattr(new, a).cpu().numpy()
            for k, a in (("pos", "pos"), ("mom", "mom"), ("status", "status"),
                         ("n_done", "n_done"), ("h", "h"), ("iters", "solver_iters"))}


REGISTRY_CASES = ["c4_dense_riemannian_d64", "c4_dense_riemannian_d512", "c5_hadamard_d24",
                  "c5_hadamard_d100", "c5_hadamard_d512"]


@pytest.mark.parametrize("name", REGISTRY_CASES)
def test_registry_models_as_user_sources_match_reference_fixture(name):
    """At the tolerances of the registry test (test_parity_gpu.py)."""
    problem, dirs, overrides, g = load_case(name)
    system = user_system(problem)
    for n_steps in g["step_counts"]:
        integ = engine.build_integrator(problem, system=system, **overrides)
        state = engine.build_state(problem, DEV, dirs=dirs)
        new = integ.step_n(state, int(n_steps), return_h=True)
        out = {k: getattr(new, k).cpu().numpy() for k in ("pos", "mom", "status", "n_done", "h")}
        ok = out["status"] == 0
        out["h"] = np.where(ok, out["h"], np.nan)
        gg = dict(g)
        gg[f"h_{n_steps}"] = np.where(ok, g[f"h_{n_steps}"], np.nan)
        assert_matches_golden(out, gg, int(n_steps), label=f"{name}[{n_steps}]")


def _compare(reg, usr, label):
    for k in ("status", "n_done", "iters"):
        np.testing.assert_array_equal(usr[k], reg[k], err_msg=f"{label} {k}")
    for k in ("pos", "mom", "h"):
        np.testing.assert_allclose(usr[k], reg[k], rtol=1e-9, atol=0, err_msg=f"{label} {k}")
    return all(np.array_equal(usr[k], reg[k], equal_nan=True) for k in ("pos", "mom"))


@pytest.mark.parametrize("dim,n_chains", [(5, 1024), (33, 1024), (100, 1024), (512, 264)])
def test_user_hadamard_against_registry_generic_route_on_identical_inputs(dim, n_chains):
    """C5 in mixed directions, 3 implicit leapfrog steps: the registry's Hadamard metric on its
    generic rank-one route (V = -w w^T formed, then the dense VJP) against the same metric
    written as user sources.  Status, completed steps and fixed-point iterations identical; pos,
    mom and h to 1e-9 relative.  Both fill and differentiate M(q) with the same expressions, so
    pos and mom agree bit for bit; h differs only in the order of the target's sum."""
    problem = problems.make_problem("C5", n_chains=n_chains, dim=dim)
    problem.metric_params = dict(problem.metric_params, generic_rank1_vjp=True)
    dirs = np.where(np.arange(n_chains) % 2 == 0, 1, -1).astype(np.int32)
    reg = run(problem, 3, system=engine.build_system(problem), dirs=dirs)
    usr = run(problem, 3, system=user_system(problem), dirs=dirs)
    assert (reg["status"] == 0).mean() > 0.5
    assert _compare(reg, usr, f"C5 D={dim}")


INTEGRATOR_CASES = sorted({**ud.CASES, **ud.FAILURE_CASES})


@pytest.mark.parametrize("name", INTEGRATOR_CASES)
def test_user_dense_models_match_reference_fixture(name):
    """Logistic regression with its dense Fisher metric (D = 25) and the LGCP (D = 64, 144):
    implicit leapfrog over 1 / 5 / 20 steps in mixed directions, both fixed-point solvers, and a
    big step at which some chains end in ConvergenceError.  pos / mom at rtol 1e-10 (1e-8 with
    the Steffensen solver, whose extrapolation divides by differences of iterates near the
    convergence tolerance and so amplifies the rounding difference between the blocked DMMA
    Cholesky and LAPACK's: up to 3.8e-9 measured after 20 steps), h at rtol 1e-10; status and
    completed steps exactly; fixed-point iterations exactly with the direct solver.  With
    Steffensen's solver the count is itself sensitive to that rounding: once in the LGCP case
    (one solve of one chain after 5 steps) an extrapolated iterate landed on the other side of
    the tolerance and the solve ran 18 more iterations to the same solution, so there at most one
    solve in a hundred may differ."""
    problem = ud.case_problem(name)
    g = rc.load_fixture(name)
    system = user_system(problem)
    for n in g["step_counts"]:
        out = run(problem, int(n), system=system, dirs=g["dirs"])
        lbl = f"{name}[{n}]"
        rtol = 1e-8 if "steffensen" in name else RTOL
        np.testing.assert_array_equal(out["status"], g[f"status_{n}"], err_msg=lbl)
        np.testing.assert_array_equal(out["n_done"], g[f"n_done_{n}"], err_msg=lbl)
        np.testing.assert_allclose(out["pos"], g[f"pos_{n}"], rtol=rtol, atol=ATOL, err_msg=lbl)
        np.testing.assert_allclose(out["mom"], g[f"mom_{n}"], rtol=rtol, atol=ATOL, err_msg=lbl)
        ok = np.isfinite(g[f"h_{n}"])
        np.testing.assert_allclose(out["h"][ok], g[f"h_{n}"][ok], rtol=RTOL, atol=1e-9,
                                   err_msg=lbl)
        done = out["n_done"] > 0
        if "steffensen" in name:
            differ = out["iters"][done] != g[f"fp_iters_{n}"][done]
            assert differ.sum() <= max(1, differ.size // 100), (lbl, out["iters"], g[f"fp_iters_{n}"])
        else:
            np.testing.assert_array_equal(out["iters"][done], g[f"fp_iters_{n}"][done],
                                          err_msg=lbl)
    if name in ud.FAILURE_CASES:
        assert (g[f"status_{g['step_counts'][-1]}"] == 1).any()


@pytest.mark.parametrize("name", sorted(ud.HMC_CASES))
def test_batched_hmc_matches_reference_fixture(name):
    """Static HMC, momentum refresh through the user image included."""
    problem, g = ud.case_problem(name), rc.load_fixture(name)
    n_iter, n_step, seed = ud.HMC_CASES[name][4:]
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


@pytest.mark.parametrize("name", sorted(ud.NUTS_CASES))
def test_nuts_matches_reference_fixture(name):
    """MultinomialDynamicIntegrationTransition through the lock-step generic NUTS path."""
    problem, g = ud.case_problem(name), rc.load_fixture(name)
    n_iter, seed, depth = ud.NUTS_CASES[name][4:]
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


@pytest.mark.parametrize("name", sorted(ud.ADAPT_CASES))
def test_dual_averaging_warm_up_matches_reference_fixture(name):
    """Dual-averaging warm-up plus a main stage through ``StaticMetropolisHMC.sample_chains``."""
    from mici_b200 import adapters, samplers  # noqa: PLC0415

    problem, g = ud.case_problem(name), rc.load_fixture(name)
    n_warm, n_main, n_step, seed = ud.ADAPT_CASES[name][4:]
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


@pytest.mark.parametrize("name", ["ud_lr_leapfrog", "ud_lgcp64_leapfrog", "ud_lgcp144_leapfrog"])
def test_h_dh_dmom_and_sample_momentum_match_oracle(name):
    """h at rtol 1e-12, the velocity and the momentum refresh at rtol 1e-11 (a blocked Cholesky
    against LAPACK's), against the NumPy oracle of the same model."""
    problem = ud.case_problem(name)
    system = user_system(problem)
    state = engine.build_state(problem, DEV)
    h = system.h(state).cpu().numpy()
    vel = system.dh_dmom(state).cpu().numpy()
    rngs = [np.random.default_rng([5, c]) for c in range(problem.n_chains)]
    mom = system.sample_momentum(state, rngs).cpu().numpy()
    with ud.patched() as dr:
        _, h_fn, osys = dr.oracle_step_fn(problem)
        for c in range(problem.n_chains):
            q, p = problem.pos[c], problem.mom[c]
            assert h[c] == pytest.approx(h_fn(q, p), rel=1e-12)
            np.testing.assert_allclose(vel[c], osys.dh2_dmom(q, p), rtol=1e-11, atol=1e-13)
            z = np.random.default_rng([5, c]).normal(size=problem.pos.shape[1])
            np.testing.assert_allclose(mom[c], osys.metric(q).sqrt_matvec(z), rtol=1e-11,
                                       atol=1e-13)


def test_failing_metrics_are_errors_and_leave_the_other_chains_bit_identical():
    """M = I + c (q q^T) o 1 with c = -1 (the Hadamard sources, B = I, S = all ones): positive
    definite only for |q| < 1.  Chain 1 starts where M is not finite, chain 2 where it is
    indefinite, chain 5 where it is positive definite but its position iterate leaves that region
    (ConvergenceError).  dh_dmom and sample_momentum raise LinAlgError; inside an integrator step
    the three chains fail; the other chains' outputs are bit-identical to a run without them."""
    dim, n = 40, 8
    target = CudaTarget(dim, uds.QUADRATIC, aux=np.identity(dim), name="quadratic")
    metric = CudaDenseMetric(uds.HADAMARD_DENSE, params=(-1.0,),
                             aux=np.concatenate([np.identity(dim).ravel(), np.ones(dim * dim)]),
                             name="hadamard")
    system = DenseRiemannianMetricSystem(target, metric)
    rng = np.random.default_rng(7)
    pos, mom = 0.01 * rng.standard_normal((n, dim)), 0.01 * rng.standard_normal((n, dim))
    pos[1, 0] = 1e200
    pos[2] = 0.5
    pos[5], mom[5] = 0.0, 2.0
    bad = [1, 2, 5]
    good = [c for c in range(n) if c not in bad]

    def state(rows):
        return ChainState(pos=torch.as_tensor(pos[rows], device=DEV),
                          mom=torch.as_tensor(mom[rows], device=DEV), dir=1)

    with pytest.raises(LinAlgError):
        system.dh_dmom(state(list(range(n))))
    with pytest.raises(LinAlgError):
        system.sample_momentum(state(list(range(n))),
                               [np.random.default_rng(c) for c in range(n)])
    integ = ImplicitLeapfrogIntegrator(system, 0.1)
    outs = []
    for rows in (list(range(n)), good):
        new = integ.step_n(state(rows), 2, return_h=True)
        outs.append({k: getattr(new, k).cpu().numpy()
                     for k in ("pos", "mom", "h", "status", "n_done", "solver_iters")})
    full, sub = outs
    assert (full["status"][[1, 2]] != 0).all(), full["status"]
    assert full["status"][5] == 1, full["status"]
    assert (full["status"][good] == 0).all()
    for k in sub:
        np.testing.assert_array_equal(full[k][good], sub[k], err_msg=k)
    vel = system.dh_dmom(state(good)).cpu().numpy()
    assert np.isfinite(vel).all()
