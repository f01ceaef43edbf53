"""CPU checks of the Cholesky-factored Riemannian-metric system: the NumPy oracle
(tests/riemannian_chol_cases.py) reproduces every reference fixture bit for bit, the failure
semantics of the reference's triangular-factored matrix class, a live check against the
importable reference, and the host class's argument validation."""

import os

import numpy as np
import pytest

from mici_b200 import engine, problems, systems, targets

import riemannian_chol_cases as rc
from oracle import mici_oracle as mo


@pytest.mark.parametrize("name", sorted(rc.ALL_INTEGRATOR_CASES))
def test_oracle_reproduces_fixture_bit_for_bit(name):
    """Bit for bit, except in the cases whose D x D mat-vecs BLAS may split over threads
    (``rc.BLAS_THREADED_CASES``, D = 128 and 200): there pos / mom / h to rtol 1e-13 unless BLAS
    was started with one thread (measured: 1.3e-15 absolute between 8 threads and 1)."""
    problem, g = rc.case_problem(name), rc.load_fixture(name)
    exact = name not in rc.BLAS_THREADED_CASES or os.environ.get("OPENBLAS_NUM_THREADS") == "1"
    for n in g["step_counts"]:
        out = rc.oracle_integrator_run(problem, int(n), g["dirs"])
        for k in ("status", "n_done"):
            np.testing.assert_array_equal(out[k], g[f"{k}_{n}"], err_msg=f"{name}[{n}] {k}")
        for k in ("pos", "mom", "h"):
            if exact:
                np.testing.assert_array_equal(out[k], g[f"{k}_{n}"], err_msg=f"{name}[{n}] {k}")
            else:
                np.testing.assert_allclose(out[k], g[f"{k}_{n}"], rtol=1e-13, atol=1e-14,
                                           err_msg=f"{name}[{n}] {k}")
        np.testing.assert_array_equal(out["fp_iters"], g[f"fp_iters_{n}"])


def test_failure_fixtures_hold_both_failure_kinds():
    kinds = set()
    for name in rc.FAILURE_CASES:
        kinds |= set(rc.load_fixture(name)["status_5"].tolist())
    assert {1, 2} <= kinds


def test_singular_fixture_covers_every_start_kind():
    """The chains of ``rc_std_d3_singular`` start singular (L00 = 0), with L00 < 0 and with
    L00 > 0; the singular ones fail their first step with ConvergenceError, the others
    complete it."""
    problem, g = rc.case_problem("rc_std_d3_singular"), rc.load_fixture("rc_std_d3_singular")
    l00 = -1.0 + problem.pos[:, 0] ** 2
    assert (l00 == 0).sum() >= 2 and (l00 < 0).sum() >= 2 and (l00 > 0).sum() >= 2
    np.testing.assert_array_equal(g["status_1"][l00 == 0], mo.STATUS_CONVERGENCE)
    np.testing.assert_array_equal(g["n_done_1"][l00 == 0], 0)
    np.testing.assert_array_equal(g["status_1"][l00 != 0], 0)
    assert np.isnan(g["h_1"][l00 == 0]).all() and np.isfinite(g["h_1"][l00 != 0]).all()


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
    """Trajectory, directions and tree sizes bit for bit; the acceptance statistic of the
    existing oracle NUTS transition (oracle/mici_oracle.py) sums its terms in another order
    than the reference and differs from it by 1 ulp in one of nine values here."""
    _, n_iter, seed, depth = rc.NUTS_CASES[name]
    g = rc.load_fixture(name)
    with rc.patched_drivers() as dr:
        out = dr.oracle_nuts(rc.case_problem(name), n_iter, seed, max_tree_depth=depth)
    for k in ("pos", "dir", "n_step", "tree_depth"):
        np.testing.assert_array_equal(out[k], g[k], err_msg=k)
    np.testing.assert_allclose(out["accept_stat"], g["accept_stat"], rtol=2.3e-16, atol=0)


@pytest.mark.parametrize("name", sorted(rc.ADAPT_CASES))
def test_oracle_warm_up_reproduces_fixture(name):
    out, g = rc.oracle_adapt_run(name), rc.load_fixture(name)
    for k in ("pos", "accept_stat", "n_step", "final_pos", "final_mom", "final_dir",
              "step_size"):
        np.testing.assert_array_equal(out[k], g[k], err_msg=k)


def failure_table_problem():
    """L(q) = diag(-1, 1, 1) + tril(q q^T), D = 3: q0 = 1 (L00 = 0), q0 = inf (non-finite L),
    q0 = 0.5 (L00 < 0); step size 0.05 (at 0.1 the negative-diagonal chain's first step does
    not converge)."""
    pos = np.array([[1.0, 0.3, -0.2], [np.inf, 0.3, -0.2], [0.5, 0.3, -0.2]])
    problem = rc.make_problem("std_gaussian", 3, 3, 0.05, problems.BASE_SEED + 71,
                              base_factor=np.diag([-1.0, 1.0, 1.0]), coeff=1.0, pos=pos[[2, 2, 2]])
    problem.pos = pos
    problem.mom = np.array([[0.4, -0.1, 0.7]] * 3)
    return problem


def test_oracle_failure_semantics():
    """h, dh_dmom and sample_momentum of the oracle at the three failure rows: singular --
    LinAlgError, LinAlgError, L z; non-finite -- LinAlgError everywhere; negative diagonal --
    finite.  An integrator step: ConvergenceError, LinAlgError, completes."""
    problem = failure_table_problem()
    with rc.patched_drivers() as dr, np.errstate(divide="ignore", invalid="ignore"):
        step, h_fn, osys = dr.oracle_step_fn(problem)
        q_sing, q_inf, q_neg = problem.pos
        p = problem.mom[0]
        z = np.array([0.3, -1.2, 0.5])
        with pytest.raises(np.linalg.LinAlgError):
            h_fn(q_sing, p)
        with pytest.raises(np.linalg.LinAlgError):
            osys.dh2_dmom(q_sing, p)
        l_sing = np.diag([-1.0, 1.0, 1.0]) + np.tril(np.outer(q_sing, q_sing))
        np.testing.assert_array_equal(osys.metric(q_sing).sqrt_matvec(z), l_sing @ z)
        for fn in (lambda: h_fn(q_inf, p), lambda: osys.dh2_dmom(q_inf, p),
                   lambda: osys.metric(q_inf)):
            with pytest.raises(mo._LinAlgError):
                fn()
        assert np.isfinite(h_fn(q_neg, p)) and np.isfinite(osys.dh2_dmom(q_neg, p)).all()
        out = dr.oracle_run(problem, 1)
    np.testing.assert_array_equal(out["status"], [mo.STATUS_CONVERGENCE, mo.STATUS_LINALG, 0])


@pytest.mark.skipif(not rc.dr.reference_available(), reason="reference package not available")
def test_reference_failure_semantics():
    """The same rows through the unmodified reference."""
    mici = rc.dr.import_reference()
    problem = failure_table_problem()
    with rc.patched_drivers() as dr, np.errstate(divide="ignore", invalid="ignore"):
        system, _ = dr.build_reference(problem)
        out = dr.reference_run(problem, 1)
        for i, (h_ok, v_ok, s_ok) in enumerate([(False, False, True), (False, False, False),
                                                (True, True, True)]):
            state = mici.states.ChainState(pos=problem.pos[i].copy(), mom=problem.mom[i].copy(),
                                           dir=1)
            for ok, fn in ((h_ok, system.h), (v_ok, system.dh_dmom),
                           (s_ok, lambda s: system.sample_momentum(s, np.random.default_rng(1)))):
                if ok:
                    assert np.isfinite(fn(state)).all()
                else:
                    # mici's LinAlgError from the finiteness check, scipy's (numpy's) from a
                    # triangular solve with a zero pivot
                    with pytest.raises((mici.errors.LinAlgError, np.linalg.LinAlgError)):
                        fn(state)
    np.testing.assert_array_equal(out["status"], [mo.STATUS_CONVERGENCE, mo.STATUS_LINALG, 0])


@pytest.mark.skipif(not rc.dr.reference_available(), reason="reference package not available")
@pytest.mark.parametrize("name", ["rc_std_d5", "rc_banana_d8_midpoint", "rc_std_d3_singular"])
def test_oracle_matches_live_reference(name):
    problem = rc.case_problem(name)
    dirs = rc.case_dirs(problem)
    with rc.patched_drivers() as dr, np.errstate(divide="ignore", invalid="ignore"):
        ref = dr.reference_run(problem, 5, dirs=dirs)
        out = dr.oracle_run(problem, 5, dirs=dirs)
    for k in ("pos", "mom", "status", "n_done", "h"):
        np.testing.assert_array_equal(out[k], ref[k], err_msg=k)


def test_constructor_and_argument_validation():
    gauss = targets.StdGaussian(4)
    base = np.tril(np.arange(16.0).reshape(4, 4)) + np.identity(4)
    full = base + np.triu(np.ones((4, 4)), 1)
    m = targets.QuadraticCholeskyMetric(full, 0.25)
    np.testing.assert_array_equal(m.aux, base)  # upper triangle zeroed on the host
    assert m.aux.flags.c_contiguous and m.params == (0.25,)
    s = systems.CholeskyFactoredRiemannianMetricSystem(gauss, m)
    assert s._rmetric_id == targets.RMETRIC_CHOL_QUADRATIC == 6
    assert s._rmetric_params == (0.25,) and s._rmetric_aux is m.aux
    assert targets.METRIC_REGISTRY["chol_quadratic"] is targets.QuadraticCholeskyMetric
    # negative and zero diagonal entries and a negative coefficient are legal
    targets.QuadraticCholeskyMetric(np.diag([-1.0, 0.0, 1.0]), -2.0)
    with pytest.raises(ValueError, match="dimension 4"):
        systems.CholeskyFactoredRiemannianMetricSystem(
            gauss, targets.QuadraticCholeskyMetric(np.identity(5), 0.1))
    with pytest.raises(TypeError):
        systems.CholeskyFactoredRiemannianMetricSystem(gauss, lambda q: np.identity(4))
    with pytest.raises(TypeError):
        systems.CholeskyFactoredRiemannianMetricSystem(gauss, targets.QuadraticScalarMetric())
    with pytest.raises(ValueError, match="fused into the kernels"):
        systems.CholeskyFactoredRiemannianMetricSystem(gauss, m, vjp_metric_chol_func=lambda q: q)
    with pytest.raises(ValueError):
        systems.CholeskyFactoredRiemannianMetricSystem(gauss, m, grad_neg_log_dens=lambda q: q)
    with pytest.raises(TypeError):
        systems.CholeskyFactoredRiemannianMetricSystem(lambda q: q @ q / 2, m)
    for bad in (np.ones((3, 4)), np.ones(4), [[np.nan, 0.0], [0.0, 1.0]]):
        with pytest.raises(ValueError):
            targets.QuadraticCholeskyMetric(bad, 0.1)
    for c in (np.inf, np.nan):
        with pytest.raises(ValueError):
            targets.QuadraticCholeskyMetric(np.identity(3), c)


def test_c8_builds_its_system():
    problem = problems.make_problem("C8", n_chains=4, dim=16)
    system = engine.build_system(problem)
    assert isinstance(system, systems.CholeskyFactoredRiemannianMetricSystem)
    base, c = problem.metric_params["base_factor"], problem.metric_params["coeff"]
    prec = problem.target_params["prec"]
    np.testing.assert_allclose(base @ base.T, prec, rtol=1e-13, atol=1e-13)
    assert c == 1 / 16
    # momenta drawn from N(0, M(q)): L(q)^-1 p is the seeded standard-normal draw
    rng = np.random.default_rng(problems.BASE_SEED + 11)
    rng.standard_normal((16, 16))
    rng.standard_normal((4, 16))
    z = rng.standard_normal((4, 16))
    fac = problems.chol_quadratic_factor(problem.pos, base, c)
    got = np.stack([np.linalg.solve(fac[i], problem.mom[i]) for i in range(4)])
    np.testing.assert_allclose(got, z, rtol=1e-12, atol=1e-12)
