"""The Cholesky-factored Riemannian-metric system on the device: implicit leapfrog / midpoint
kernels with the triangular-factored metric policy (csrc/riemannian.cuh CholeskyFactoredMetric)
against the reference fixtures (tests/golden/rc_*.npz, tests/riemannian_chol_cases.py) and
against the NumPy oracle on the same seeded inputs."""

import numpy as np
import pytest
import torch

from mici_b200 import engine, problems, transitions
from mici_b200.errors import LinAlgError

import riemannian_chol_cases as rc
from golden_util import ATOL, RTOL
from test_cholesky_riemannian_oracle import failure_table_problem

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def run_cuda(problem, n_steps, dirs=None, return_h=True):
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV, dirs=dirs)
    pos0, mom0 = state.pos.clone(), state.mom.clone()
    new = integ.step_n(state, n_steps, return_h=return_h)
    torch.cuda.synchronize()
    # Integrator.step must not mutate its argument (reference tests/test_integrators.py:110-124)
    torch.testing.assert_close(state.pos, pos0, rtol=0, atol=0, equal_nan=True)
    torch.testing.assert_close(state.mom, mom0, rtol=0, atol=0, equal_nan=True)
    return {k: (None if getattr(new, a) is None else getattr(new, a).cpu().numpy())
            for k, a in (("pos", "pos"), ("mom", "mom"), ("status", "status"),
                         ("n_done", "n_done"), ("h", "h"), ("iters", "solver_iters"))}


@pytest.mark.parametrize("name", sorted(rc.ALL_INTEGRATOR_CASES))
def test_cuda_matches_reference_fixture(name):
    """pos / mom at rtol 1e-10, atol 1e-12; h at rtol 1e-10, atol 1e-9; status, completed steps
    and the fixed-point iterations of the last completed step exactly."""
    problem, g = rc.case_problem(name), rc.load_fixture(name)
    dirs = g["dirs"]
    for n in g["step_counts"]:
        out = run_cuda(problem, int(n), dirs=dirs)
        lbl = f"{name}[{n}]"
        # Aitken extrapolation divides by second differences of the iterates, which amplifies the
        # last-bit differences of exp(-v) (libm vs CUDA) over 20 funnel steps: measured 3.2e-10
        # relative on one of 80 coordinates (as for the diagonal metrics' Steffensen fixtures)
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
        np.testing.assert_array_equal(out["iters"][done], g[f"fp_iters_{n}"][done], err_msg=lbl)


@pytest.mark.parametrize("name", ["rc_banana_d8_midpoint", "rc_funnel_d10", "rc_quadratic_d64",
                                  "rc_std_d33", "rc_quadratic_d200"])
def test_h_dh_dmom_and_sample_momentum_match_oracle(name):
    problem = rc.case_problem(name)
    system = engine.build_integrator(problem).system
    state = engine.build_state(problem, DEV)
    h = system.h(state).cpu().numpy()
    vel = system.dh_dmom(state).cpu().numpy()
    with rc.patched_drivers() as dr:
        _, h_fn, osys = dr.oracle_step_fn(problem)
        for c in range(problem.n_chains):
            q, p = problem.pos[c], problem.mom[c]
            assert h[c] == pytest.approx(h_fn(q, p), rel=1e-12)
            np.testing.assert_allclose(vel[c], osys.dh2_dmom(q, p), rtol=1e-12, atol=1e-14)
    rngs = [np.random.default_rng([5, c]) for c in range(problem.n_chains)]
    mom = system.sample_momentum(state, rngs).cpu().numpy()
    for c in range(problem.n_chains):
        z = np.random.default_rng([5, c]).normal(size=problem.dim)
        np.testing.assert_allclose(mom[c], osys.metric(problem.pos[c]).sqrt_matvec(z),
                                   rtol=1e-13, atol=1e-14)


def test_failure_semantics_match_the_reference_class():
    """L(q) = diag(-1, 1, 1) + tril(q q^T): q0 = 1 (L00 = 0), q0 = inf, q0 = 0.5 (L00 < 0).
    h: NaN, NaN, the oracle's value; dh_dmom: LinAlgError, LinAlgError, the oracle's value;
    sample_momentum: L z, LinAlgError, L z; one step: ConvergenceError, LinAlgError, completes
    (as the oracle and the reference, tests/test_cholesky_riemannian_oracle.py)."""
    problem = failure_table_problem()
    integ = engine.build_integrator(problem)
    system = integ.system
    state = engine.build_state(problem, DEV)
    h = system.h(state).cpu().numpy()
    assert np.isnan(h[0]) and np.isnan(h[1])
    with rc.patched_drivers() as dr:
        _, h_fn, osys = dr.oracle_step_fn(problem)
        ref = dr.oracle_run(problem, 1)
    q_neg, p = problem.pos[2], problem.mom[2]
    assert h[2] == pytest.approx(h_fn(q_neg, p), rel=1e-12)
    for c, ok in enumerate((False, False, True)):
        one = engine.build_state(problem, DEV, chains=slice(c, c + 1))
        if ok:
            np.testing.assert_allclose(system.dh_dmom(one).cpu().numpy()[0],
                                       osys.dh2_dmom(q_neg, p), rtol=1e-12, atol=1e-14)
        else:
            with pytest.raises(LinAlgError):
                system.dh_dmom(one)
    for c, ok in enumerate((True, False, True)):
        one = engine.build_state(problem, DEV, chains=slice(c, c + 1))
        rngs = [np.random.default_rng([6, c])]
        if ok:
            z = np.random.default_rng([6, c]).normal(size=3)
            fac = np.diag([-1.0, 1.0, 1.0]) + np.tril(np.outer(problem.pos[c], problem.pos[c]))
            np.testing.assert_allclose(system.sample_momentum(one, rngs).cpu().numpy()[0],
                                       fac @ z, rtol=1e-15, atol=1e-15)
        else:
            with pytest.raises(LinAlgError):
                system.sample_momentum(one, rngs)
    out = run_cuda(problem, 1)
    np.testing.assert_array_equal(out["status"], [1, 3, 0])
    np.testing.assert_array_equal(out["status"], ref["status"])
    np.testing.assert_allclose(out["pos"][2], ref["pos"][2], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(out["mom"][2], ref["mom"][2], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("name", ["rc_funnel_d10", "rc_std_d5_bigstep", "rc_banana_d8_midpoint",
                                  "rc_std_d3_singular"])
def test_per_chain_step_sizes_and_lengths_match_individual_launches(name):
    problem = rc.case_problem(name)
    integ = engine.build_integrator(problem)
    n = problem.n_chains
    rng = np.random.default_rng(12)
    eps = problem.step_size * rng.choice([0.5, 1.0, 2.0, 4.0], n)
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
        assert torch.equal(got.h[c], ref.h[0]) or (torch.isnan(got.h[c]) and torch.isnan(ref.h[0]))
        assert torch.equal(got.solver_iters[c], ref.solver_iters[0])


@pytest.mark.parametrize("name", ["rc_funnel_d10", "rc_quadratic_d64", "rc_banana_d8_midpoint",
                                  "rc_std_d5_steffensen", "rc_funnel_d10_midpoint_steffensen"])
def test_call_counters_match_oracle(name):
    """Per chain over 5 steps, from the oracle's fixed-point iteration counts of every step:
    leapfrog -- 2 gradients, it1 + it2 + 2 metric builds, it0 + it3 + 1 quadratic-form VJPs;
    midpoint -- one gradient, build and VJP per evaluation of dh/dz (every fixed-point function
    call plus the explicit half-step).  Steffensen calls the function twice per iteration.
    Chains with a solve of more than 20 iterations on the oracle are left out: such a solve
    hovers at the convergence tolerance and its count follows last-bit rounding (one funnel
    chain's Steffensen midpoint solve takes 67 iterations on the oracle; that chain's five-step
    total was 100 iterations on the device against the oracle's 134)."""
    problem = rc.case_problem(name)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    integ.count_calls()
    out = integ.step_n(state, 5)
    torch.cuda.synchronize()
    got = integ.call_counts.cpu().numpy()
    done = out.n_done.cpu().numpy()
    calls = 2 if "steffensen" in name else 1
    midpoint = problem.integrator == "implicit_midpoint"
    full = np.flatnonzero(done == 5)
    compared = 0
    with rc.patched_drivers() as dr:
        for c in full:
            counts = {}
            step, _, _ = dr.oracle_step_fn(problem, counts=counts)
            q, p = problem.pos[c], problem.mom[c]
            for _ in range(5):
                q, p = step(q, p, 1)
            it = np.array(counts["all_fp_iters"], dtype=np.int64)
            if it.max() > 20:
                continue
            compared += 1
            want = np.zeros(4, dtype=np.int64)
            want[3] = it.sum()
            if midpoint:
                want[:3] = calls * it.sum() + len(it)
            else:
                want[0] = 2 * len(it)
                want[1] = calls * (it[:, 1] + it[:, 2]).sum() + 2 * len(it)
                want[2] = calls * (it[:, 0] + it[:, 3]).sum() + len(it)
            np.testing.assert_array_equal(got[c], want, err_msg=f"chain {c}")
    assert compared >= problem.n_chains // 2


@pytest.mark.parametrize("name", sorted(rc.HMC_CASES))
def test_batched_hmc_matches_reference_fixture(name):
    problem = rc.case_problem(name)
    _, n_iter, n_step, seed = rc.HMC_CASES[name]
    g = rc.load_fixture(name)
    integ = engine.build_integrator(problem)
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


@pytest.mark.parametrize("name", sorted(rc.NUTS_CASES))
def test_nuts_matches_reference_fixture(name):
    problem = rc.case_problem(name)
    _, n_iter, seed, depth = rc.NUTS_CASES[name]
    g = rc.load_fixture(name)
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
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"][-1])
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-8, atol=1e-10)
    for k in ("av_metrop_accept_prob", "accept_stat"):
        np.testing.assert_allclose(stats[k].cpu().numpy(), g[k], rtol=1e-7, atol=1e-10, err_msg=k)


@pytest.mark.parametrize("name", sorted(rc.ADAPT_CASES))
def test_dual_averaging_warm_up_matches_reference_fixture(name):
    from mici_b200 import adapters, samplers

    problem, g = rc.case_problem(name), rc.load_fixture(name)
    _, n_warm, n_main, n_step, seed = rc.ADAPT_CASES[name]
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
    np.testing.assert_array_equal(out.final_states.dir.cpu().numpy(), g["final_dir"])
    k = 4
    np.testing.assert_allclose(stats["accept_stat"][:k], g["accept_stat"][:k], rtol=1e-7,
                               atol=1e-10)
    np.testing.assert_allclose(pos[:k], g["pos"][:k], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(stats["accept_stat"], g["accept_stat"], rtol=1e-2, atol=1e-3)
    np.testing.assert_allclose(pos, g["pos"], rtol=1e-3, atol=1e-4)
    assert integ.step_size == pytest.approx(float(g["step_size"]), rel=1e-4)


DROPIN_CASES = {
    # name: (fixture case of the problem, stock sampler, n_iter, sampler kwargs)
    "chol_banana_static": ("rc_hmc_banana_d4", "StaticMetropolisHMC", 4, {"n_step": 5}),
    "chol_std_dynamic": ("rc_nuts_std_d5", "DynamicMultinomialHMC", 3, {"max_tree_depth": 4}),
}


@pytest.mark.skipif(not rc.dr.reference_available(),
                    reason="reference package not available (oracle/_ref missing)")
@pytest.mark.parametrize("name", sorted(DROPIN_CASES))
def test_stock_mici_sampler_over_new_system(name):
    """The unmodified reference samplers drive the new system and the CUDA implicit leapfrog with
    one NumPy-held ``mici.states.ChainState`` per chain and reproduce the all-reference chains."""
    from test_dropin_gpu import _run_stock_sampler

    case, sampler_name, n_iter, skw = DROPIN_CASES[name]
    mici = rc.dr.import_reference()
    problem = rc.case_problem(case)
    sampler_cls = getattr(mici.samplers, sampler_name)
    with rc.patched_drivers() as dr:
        ref_system, ref_integrator = dr.build_reference(problem)
    ref = _run_stock_sampler(mici, sampler_cls, ref_system, ref_integrator, problem, n_iter, 4242,
                             **skw)
    integ = engine.build_integrator(problem)
    new = _run_stock_sampler(mici, sampler_cls, integ.system, integ, problem, n_iter, 4242, **skw)
    for k in ("n_step", "convergence_error", "non_reversible_step"):
        np.testing.assert_array_equal(new[2][k], ref[2][k], err_msg=k)
    np.testing.assert_allclose(new[2]["accept_stat"], ref[2]["accept_stat"], rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(new[1], ref[1], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(new[0], ref[0], rtol=1e-8, atol=1e-10)


REF_TEST_SEED = 3046987125  # reference tests/test_integrators.py:8


@pytest.mark.parametrize("dim", [1, 2, 5])
@pytest.mark.parametrize("integrator", ["implicit_leapfrog", "implicit_midpoint"])
def test_reference_property_checks(dim, integrator):
    """The reference's own integrator checks (tests/test_integrators.py:8-110) with its protocol:
    five states with pos, mom ~ N(0, I) from its seed, step size 0.1; reversibility after
    n_step 1 / 5 / 20 steps and back; approximate energy conservation over 200 steps (mean of h
    over the first 100 values minus the mean over the rest); no input mutation.  Std-Gaussian
    target, L(q) = chol(A A^T / D + I) + tril(q q^T) / (2 D).  The reference tests no
    Cholesky-factored system; the bound is its implicit-leapfrog tolerance for Riemannian
    systems, 1e-3, for both integrators (the oracle's largest statistic: 3.1e-4 leapfrog,
    2.7e-4 midpoint, above the 2e-4 the reference sets for the midpoint on its diagonal
    system)."""
    h_diff_tol = 1e-3
    problem = rc.make_problem("std_gaussian", dim, n_chains=5, step_size=0.1,
                              seed=problems.BASE_SEED + 80 + dim, integrator=integrator,
                              coeff=0.5 / dim)
    qp = np.random.default_rng(REF_TEST_SEED).standard_normal((5, 2, dim))
    problem.pos, problem.mom = qp[:, 0].copy(), qp[:, 1].copy()
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    pos0, mom0 = state.pos.clone(), state.mom.clone()
    for n_step in (1, 5, 20):
        fwd = integ.step_n(state, n_step)
        assert torch.equal(state.pos, pos0) and torch.equal(state.mom, mom0)
        assert int((fwd.status != 0).sum()) == 0
        fwd.dir = -1
        back = integ.step_n(fwd, n_step)
        torch.testing.assert_close(back.pos, pos0, rtol=0, atol=1e-8)
        torch.testing.assert_close(back.mom, mom0, rtol=0, atol=1e-8)
    hs, s = [integ.system.h(state)], state
    for _ in range(200):
        s = integ.step_n(s, 1, return_h=True)
        assert int((s.status != 0).sum()) == 0
        hs.append(s.h)
    hs = torch.stack(hs)
    diff = hs[:100].mean(0) - hs[100:].mean(0)
    assert float(diff.abs().max()) < h_diff_tol


@pytest.mark.parametrize("integrator", ["implicit_leapfrog", "implicit_midpoint"])
def test_d512_matches_oracle(integrator):
    """D = 512: the factor (2 MB) lives in the per-CTA global workspace.  4 chains, 3 steps,
    oracle parity and a round trip."""
    problem = rc.make_problem("quadratic", 512, n_chains=4, step_size=0.05,
                              seed=problems.BASE_SEED + 90, integrator=integrator)
    dirs = np.array([1, -1, 1, -1], dtype=np.int32)
    out = run_cuda(problem, 3, dirs=dirs)
    with rc.patched_drivers() as dr:
        ref = dr.oracle_run(problem, 3, dirs=dirs)
    np.testing.assert_array_equal(out["status"], ref["status"])
    np.testing.assert_array_equal(out["status"], 0)
    np.testing.assert_allclose(out["pos"], ref["pos"], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(out["mom"], ref["mom"], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(out["h"], ref["h"], rtol=RTOL)
    integ = engine.build_integrator(problem)
    fwd = integ.step_n(engine.build_state(problem, DEV), 3)
    fwd.dir = -1
    back = integ.step_n(fwd, 3)
    torch.testing.assert_close(back.pos.cpu(), torch.as_tensor(problem.pos), rtol=0, atol=1e-8)
    torch.testing.assert_close(back.mom.cpu(), torch.as_tensor(problem.mom), rtol=0, atol=1e-8)


def test_full_size_c8_reversibility_and_energy():
    """All 8192 chains x D = 128: 10 steps forward, flip dir, 10 back; chains that completed both
    return to their start within 1e-8.  Energy: the median |h(10 steps) - h(0)| over completed
    chains is 0.04 on the CPU oracle's first 64 chains; the bound leaves a 2.5x margin."""
    problem = problems.make_problem("C8")
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    h0 = integ.system.h(state)
    fwd = integ.step_n(state, 10, return_h=True)
    ok = fwd.status == 0
    assert float(ok.double().mean()) > 0.99
    dh = (fwd.h - h0)[ok].abs()
    assert float(dh.median()) < 0.1
    fwd.dir = -1
    back = integ.step_n(fwd, 10)
    both = ok & (back.status == 0)
    assert float(both.double().mean()) > 0.99
    torch.testing.assert_close(back.pos[both], state.pos[both], rtol=0, atol=1e-8)
    torch.testing.assert_close(back.mom[both], state.mom[both], rtol=0, atol=1e-8)
