"""GaussianDenseConstrainedEuclideanMetricSystem on the device: the constrained leapfrog kernel
with the Gaussian-split flow policy (csrc/constrained.cuh, GAUSS = true) against the reference
fixtures (tests/golden/gc_*.npz, tests/gaussian_constrained_cases.py) and the NumPy oracle."""

import numpy as np
import pytest
import torch

from mici_b200 import engine, problems, transitions

import gaussian_constrained_cases as gc
from golden_util import ATOL, RTOL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def run_cuda(problem, n_steps, dirs=None):
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV, dirs=dirs)
    new = integ.step_n(state, n_steps, return_h=True)
    torch.cuda.synchronize()
    return {k: getattr(new, a).cpu().numpy()
            for k, a in (("pos", "pos"), ("mom", "mom"), ("status", "status"),
                         ("n_done", "n_done"), ("h", "h"), ("iters", "solver_iters"))}


@pytest.mark.parametrize("name", sorted(gc.ALL_INTEGRATOR_CASES))
def test_cuda_matches_reference_fixture(name):
    """pos / mom at rtol 1e-10, atol 1e-12; h at rtol 1e-10, atol 1e-9; status, completed steps
    and the total Newton iterations of chains that complete every step exactly (a failing solve's
    iterations are counted by the kernel and not by the oracle)."""
    problem, g = gc.case_problem(name), gc.load_fixture(name)
    for n in g["step_counts"]:
        out = run_cuda(problem, int(n), dirs=g["dirs"])
        lbl = f"{name}[{n}]"
        np.testing.assert_array_equal(out["status"], g[f"status_{n}"], err_msg=lbl)
        np.testing.assert_array_equal(out["n_done"], g[f"n_done_{n}"], err_msg=lbl)
        np.testing.assert_allclose(out["pos"], g[f"pos_{n}"], rtol=RTOL, atol=ATOL, err_msg=lbl)
        np.testing.assert_allclose(out["mom"], g[f"mom_{n}"], rtol=RTOL, atol=ATOL, err_msg=lbl)
        np.testing.assert_allclose(out["h"], g[f"h_{n}"], rtol=RTOL, atol=1e-9, err_msg=lbl)
        ok = g[f"status_{n}"] == 0
        np.testing.assert_array_equal(out["iters"][ok], g[f"newton_iters_{n}"][ok], err_msg=lbl)


@pytest.mark.parametrize("name", ["gc_sphere_dense_d10", "gc_multi_sphere_c4_diag_d72_inner2",
                                  "gc_multi_sphere_c8_dense_d32", "gc_torus",
                                  "gc_sphere_dense_d200"])
def test_h_dh_dmom_projection_and_sample_momentum_match_oracle(name):
    problem = gc.case_problem(name)
    system = engine.build_integrator(problem).system
    state = engine.build_state(problem, DEV)
    h = system.h(state).cpu().numpy()
    vel = system.dh_dmom(state).cpu().numpy()
    rng = np.random.default_rng(3)
    raw = rng.standard_normal(problem.pos.shape)
    proj = system.project_onto_cotangent_space(torch.as_tensor(raw, device=DEV), state)
    proj = proj.cpu().numpy()
    rngs = [np.random.default_rng([5, c]) for c in range(problem.n_chains)]
    mom = system.sample_momentum(state, rngs).cpu().numpy()
    with gc.patched_drivers() as dr:
        _, h_fn, osys = dr.oracle_step_fn(problem)
        sample = dr._sample_momentum(problem, osys)
        for c in range(problem.n_chains):
            q, p = problem.pos[c], problem.mom[c]
            assert h[c] == pytest.approx(h_fn(q, p), rel=1e-12, abs=1e-12)
            np.testing.assert_allclose(vel[c], osys.inv_metric_mat(p), rtol=1e-12, atol=1e-14)
            want = osys.project_onto_cotangent_space(raw[c], q)
            np.testing.assert_allclose(proj[c], want, rtol=1e-11, atol=1e-13)
            jac = osys.jacob_constr(q)
            assert np.abs(jac @ osys.inv_metric_mat(proj[c])).max() < 1e-12 * max(
                1.0, np.abs(raw[c]).max())
            np.testing.assert_allclose(mom[c], sample(q, np.random.default_rng([5, c])),
                                       rtol=1e-11, atol=1e-13)


@pytest.mark.parametrize("name", ["gc_sphere_identity_d5", "gc_sphere_diag_d70_inner2",
                                  "gc_multi_sphere_c4_dense_d16", "gc_sphere_dense_d10_bigstep",
                                  "gc_multi_sphere_c2_dense_d12_line_search"])
def test_per_chain_step_sizes_and_lengths_match_individual_launches(name):
    problem = gc.case_problem(name)
    integ = engine.build_integrator(problem)
    n = problem.n_chains
    rng = np.random.default_rng(12)
    eps = problem.step_size * rng.choice([0.5, 1.0, 2.0], n)
    ns = rng.integers(0, 5, n).astype(np.int32)
    dirs = torch.as_tensor(rng.choice([-1, 1], n).astype(np.int32), device=DEV)
    state = engine.build_state(problem, DEV)
    state.dir = dirs
    integ.step_size = torch.as_tensor(eps, device=DEV)
    got = integ.step_n(state, torch.as_tensor(ns, device=DEV), return_h=True)
    torch.cuda.synchronize()
    for c in range(n):
        integ.step_size = float(eps[c])
        one = engine.build_state(problem, DEV, chains=slice(c, c + 1))
        one.dir = dirs[c:c + 1]
        ref = integ.step_n(one, int(ns[c]), return_h=True)
        assert int(got.status[c]) == int(ref.status[0]) and int(got.n_done[c]) == int(ref.n_done[0])
        assert torch.equal(got.pos[c], ref.pos[0]) and torch.equal(got.mom[c], ref.mom[0])
        assert torch.equal(got.h[c], ref.h[0])
        assert torch.equal(got.solver_iters[c], ref.solver_iters[0])


@pytest.mark.parametrize("name", ["gc_sphere_dense_d10", "gc_multi_sphere_c4_dense_d16_quasi_newton"])
def test_call_counters_match_oracle(name):
    """Per chain over 5 steps: 1 + 5 gradients; constraint-Jacobian evaluations: 3 projections,
    2 retractions plus the Newton iterations, and 1 + 5 Lebesgue-density gradients."""
    problem = gc.case_problem(name)
    integ = engine.build_integrator(problem)
    integ.count_calls()
    out = integ.step_n(engine.build_state(problem, DEV), 5)
    torch.cuda.synchronize()
    got = integ.call_counts.cpu().numpy()
    orc = gc.oracle_integrator_run(problem, 5, np.ones(problem.n_chains, dtype=np.int32))
    assert (out.n_done.cpu().numpy() == 5).all()
    for c in range(problem.n_chains):
        it = int(orc["newton_iters"][c])
        want = [6, 5 * 3 + 5 * 2 + it + 6, 0, it]
        np.testing.assert_array_equal(got[c], want, err_msg=f"chain {c}")


@pytest.mark.parametrize("name", sorted(gc.HMC_CASES))
def test_batched_hmc_matches_reference_fixture(name):
    problem = gc.case_problem(name)
    _, n_iter, n_step, seed = gc.HMC_CASES[name]
    g = gc.load_fixture(name)
    integ = engine.build_integrator(problem)
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


@pytest.mark.parametrize("name", sorted(gc.NUTS_CASES))
def test_nuts_matches_reference_fixture(name):
    problem = gc.case_problem(name)
    _, n_iter, seed, depth = gc.NUTS_CASES[name]
    g = gc.load_fixture(name)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    final, stats, trace = transitions.sample_chains(
        integ.system, integ, state, rngs, 0, n_iter,
        integration_transition=transitions.MultinomialDynamicIntegrationTransition(
            integ.system, integ, max_tree_depth=depth))
    torch.cuda.synchronize()
    for k in ("n_step", "tree_depth", "diverging"):
        np.testing.assert_array_equal(stats[k].cpu().numpy().astype(np.float64), g[k], err_msg=k)
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(stats["accept_stat"].cpu().numpy(), g["accept_stat"], rtol=1e-7,
                               atol=1e-10)


@pytest.mark.parametrize("name", sorted(gc.ADAPT_CASES))
def test_dual_averaging_warm_up_matches_reference_fixture(name):
    from mici_b200 import adapters, samplers

    problem, g = gc.case_problem(name), gc.load_fixture(name)
    _, n_warm, n_main, n_step, seed = gc.ADAPT_CASES[name]
    integ = engine.build_integrator(problem)
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
    np.testing.assert_allclose(pos[:4], g["pos"][:4], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(pos, g["pos"], rtol=1e-3, atol=1e-4)
    assert integ.step_size == pytest.approx(float(g["step_size"]), rel=1e-4)


DROPIN_CASES = {
    "gauss_constr_static": ("gc_hmc_sphere_dense_d10", "StaticMetropolisHMC", 3, {"n_step": 5}),
    "gauss_constr_dynamic": ("gc_nuts_multi_sphere_c2_d12", "DynamicMultinomialHMC", 2,
                             {"max_tree_depth": 4}),
}


@pytest.mark.skipif(not gc.dr.reference_available(),
                    reason="reference package not available (oracle/_ref missing)")
@pytest.mark.parametrize("name", sorted(DROPIN_CASES))
def test_stock_mici_sampler_over_new_system(name):
    from test_dropin_gpu import _run_stock_sampler

    case, sampler_name, n_iter, skw = DROPIN_CASES[name]
    mici = gc.dr.import_reference()
    problem = gc.case_problem(case)
    sampler_cls = getattr(mici.samplers, sampler_name)
    with gc.patched_drivers() as dr:
        ref_system, ref_integrator = dr.build_reference(problem)
    ref = _run_stock_sampler(mici, sampler_cls, ref_system, ref_integrator, problem, n_iter, 4242,
                             **skw)
    integ = engine.build_integrator(problem)
    new = _run_stock_sampler(mici, sampler_cls, integ.system, integ, problem, n_iter, 4242, **skw)
    for k in ("n_step", "convergence_error", "non_reversible_step"):
        np.testing.assert_array_equal(new[2][k], ref[2][k], err_msg=k)
    np.testing.assert_allclose(new[2]["accept_stat"], ref[2]["accept_stat"], rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(new[0], ref[0], rtol=1e-8, atol=1e-10)


def test_c9_full_size_constraints_reversibility_and_energy():
    problem = problems.make_problem("C9")
    integ = engine.build_integrator(problem)
    system = integ.system
    state = engine.build_state(problem, DEV)
    h0 = system.h(state)
    fwd = integ.step_n(state, 10, return_h=True)
    torch.cuda.synchronize()
    ok = fwd.status == 0
    assert ok.float().mean() > 0.9
    q = fwd.pos[ok].view(-1, 8, 16)
    assert ((q * q).sum(-1) - 1.0).abs().max().item() < 1e-8
    fwd.dir = torch.full((problem.n_chains,), -1, dtype=torch.int32, device=DEV)
    back = integ.step_n(fwd, 10)
    torch.cuda.synchronize()
    both = ok & (back.status == 0)
    assert both.float().mean() > 0.9
    assert (back.pos[both] - state.pos[both]).abs().max().item() < 1e-7
    long = integ.step_n(state, 50, return_h=True)
    torch.cuda.synchronize()
    done = long.status == 0
    assert done.float().mean() > 0.8
    dh = (long.h[done] - h0[done]).abs()
    assert torch.isfinite(dh).all() and dh.median().item() < 1.0
