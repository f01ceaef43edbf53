"""CPU checks of the diagonal / scalar Riemannian-metric systems: the NumPy oracle
(tests/riemannian_diag_cases.py) reproduces every reference fixture bit for bit, a live check
against the importable reference, and the host classes' argument validation."""

import numpy as np
import pytest

from mici_b200 import engine, problems, systems, targets

import riemannian_diag_cases as rc


@pytest.mark.parametrize("name", sorted(rc.ALL_INTEGRATOR_CASES))
def test_oracle_reproduces_fixture_bit_for_bit(name):
    problem, g = rc.case_problem(name), rc.load_fixture(name)
    for n in g["step_counts"]:
        out = rc.oracle_integrator_run(problem, int(n), g["dirs"])
        for k in ("pos", "mom", "status", "n_done", "h"):
            np.testing.assert_array_equal(out[k], g[f"{k}_{n}"], err_msg=f"{name}[{n}] {k}")
        np.testing.assert_array_equal(out["fp_iters"], g[f"fp_iters_{n}"])


def test_failure_fixtures_hold_both_failure_kinds():
    kinds = set()
    for name in rc.FAILURE_CASES:
        kinds |= set(rc.load_fixture(name)["status_5"].tolist())
    assert {1, 2} <= kinds


@pytest.mark.parametrize("name", sorted(rc.HMC_CASES))
def test_oracle_hmc_reproduces_fixture(name):
    _, n_iter, n_step, seed = rc.HMC_CASES[name]
    g = rc.load_fixture(name)
    with rc.patched_drivers() as dr:
        out = dr.oracle_hmc(rc.case_problem(name), n_iter, n_step, seed)
    for k in ("pos", "dir", "n_step", "metrop_accept_prob", "accept_stat"):
        np.testing.assert_array_equal(out[k], g[k], err_msg=k)


@pytest.mark.parametrize("name", sorted(rc.NUTS_CASES))
def test_oracle_nuts_reproduces_fixture(name):
    _, n_iter, seed, depth = rc.NUTS_CASES[name]
    g = rc.load_fixture(name)
    with rc.patched_drivers() as dr:
        out = dr.oracle_nuts(rc.case_problem(name), n_iter, seed, max_tree_depth=depth)
    for k in ("pos", "dir", "n_step", "tree_depth", "accept_stat"):
        np.testing.assert_array_equal(out[k], g[k], err_msg=k)


@pytest.mark.skipif(not rc.dr.reference_available(), reason="reference package not available")
@pytest.mark.parametrize("name", ["rd_ff_funnel_d10", "rd_sc_std_d5_bigstep",
                                  "rd_dq_banana_d8_midpoint"])
def test_oracle_matches_live_reference(name):
    problem = rc.case_problem(name)
    dirs = rc.case_dirs(problem)
    with rc.patched_drivers() as dr:
        ref = dr.reference_run(problem, 5, dirs=dirs)
        out = dr.oracle_run(problem, 5, dirs=dirs)
    for k in ("pos", "mom", "status", "n_done", "h"):
        np.testing.assert_array_equal(out[k], ref[k], err_msg=k)


def test_constructors_and_parameter_validation():
    funnel, gauss = targets.NealFunnel(4), targets.StdGaussian(4)
    s = systems.DiagonalRiemannianMetricSystem(funnel, targets.FunnelFisherMetric())
    assert s._rmetric_id == targets.RMETRIC_DIAG_FUNNEL_FISHER
    s = systems.DiagonalRiemannianMetricSystem(gauss, targets.QuadraticDiagonalMetric(2.0, 0.5))
    assert s._rmetric_params == (2.0, 0.5)
    s = systems.ScalarRiemannianMetricSystem(gauss, targets.QuadraticScalarMetric(b=0.0))
    assert s._rmetric_id == targets.RMETRIC_SCALAR_QUADRATIC and s._rmetric_params == (1.0, 0.0)
    with pytest.raises(TypeError):
        systems.DiagonalRiemannianMetricSystem(gauss, lambda q: 1 + q**2)
    with pytest.raises(TypeError):
        systems.DiagonalRiemannianMetricSystem(gauss, targets.QuadraticScalarMetric())
    with pytest.raises(TypeError):
        systems.DiagonalRiemannianMetricSystem(gauss, targets.FunnelFisherMetric())
    with pytest.raises(TypeError):
        systems.ScalarRiemannianMetricSystem(gauss, targets.QuadraticDiagonalMetric())
    with pytest.raises(ValueError, match="fused into the kernels"):
        systems.DiagonalRiemannianMetricSystem(
            gauss, targets.QuadraticDiagonalMetric(), vjp_metric_diagonal_func=lambda q: q)
    with pytest.raises(ValueError, match="fused into the kernels"):
        systems.ScalarRiemannianMetricSystem(
            gauss, targets.QuadraticScalarMetric(), vjp_metric_scalar_func=lambda q: q)
    for bad in ({"a": 0.0}, {"a": -1.0}, {"b": -0.1}, {"a": float("nan")}):
        with pytest.raises(ValueError):
            targets.QuadraticDiagonalMetric(**bad)
        with pytest.raises(ValueError):
            targets.QuadraticScalarMetric(**bad)


@pytest.mark.parametrize("kind", ["fisher", "scalar"])
def test_c7_builds_its_system(kind):
    problem = problems.make_problem("C7", n_chains=4, dim=16, metric_kind=kind)
    system = engine.build_system(problem)
    cls = (systems.DiagonalRiemannianMetricSystem if kind == "fisher"
           else systems.ScalarRiemannianMetricSystem)
    assert isinstance(system, cls)
    # momenta drawn from N(0, M(q)): p / sqrt(d(q)) is the seeded standard-normal draw
    z = np.random.default_rng(problems.BASE_SEED + 10)
    z.standard_normal((4, 16))
    z = z.standard_normal((4, 16))
    d = (problems.funnel_fisher_diagonal(problem.pos) if kind == "fisher"
         else (1.0 + (problem.pos**2).sum(1) / 16)[:, None])
    np.testing.assert_allclose(problem.mom / np.sqrt(d), z, rtol=1e-14)


@pytest.mark.parametrize("name", sorted(rc.ADAPT_CASES))
def test_oracle_warm_up_reproduces_fixture(name):
    """Dual-averaging warm-up + main stage: the oracle's adapters and transitions reproduce the
    reference's ``StaticMetropolisHMC.sample_chains`` bit for bit."""
    out, g = rc.oracle_adapt_run(name), rc.load_fixture(name)
    for k in ("pos", "accept_stat", "n_step", "final_pos", "final_mom", "final_dir",
              "step_size"):
        np.testing.assert_array_equal(out[k], g[k], err_msg=k)
