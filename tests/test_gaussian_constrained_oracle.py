"""CPU tests of GaussianDenseConstrainedEuclideanMetricSystem: the host class's argument checks,
the NumPy oracle (tests/gaussian_constrained_cases.py) against the reference fixtures
(tests/golden/gc_*.npz), and against the live reference where a copy is present."""

import os

import numpy as np
import pytest

from mici_b200 import systems, targets

import gaussian_constrained_cases as gc


def test_host_class_signature_and_checks():
    t = targets.make_target("sphere", dim=5)
    s = systems.GaussianDenseConstrainedEuclideanMetricSystem(t, t)
    assert not s.dens_wrt_hausdorff
    assert isinstance(s, systems.GaussianEuclideanMetricSystem)
    assert isinstance(s, systems.DenseConstrainedEuclideanMetricSystem)
    mro = type(s).__mro__
    assert mro.index(systems.GaussianEuclideanMetricSystem) < mro.index(
        systems.DenseConstrainedEuclideanMetricSystem)
    with pytest.raises(TypeError):
        systems.GaussianDenseConstrainedEuclideanMetricSystem(t, t, dens_wrt_hausdorff=False)
    with pytest.raises(TypeError):
        systems.GaussianDenseConstrainedEuclideanMetricSystem(lambda q: q @ q, t)
    with pytest.raises(ValueError):
        systems.GaussianDenseConstrainedEuclideanMetricSystem(t, t, mhp_constr=lambda q: q)
    with pytest.raises(ValueError):
        systems.GaussianDenseConstrainedEuclideanMetricSystem(t, t, jacob_constr=lambda q: q)
    with pytest.raises(ValueError):
        systems.GaussianDenseConstrainedEuclideanMetricSystem(t, targets.make_target("sphere", dim=5))


# D x D BLAS products large enough for OpenBLAS to split over threads, whose rounding then
# depends on the thread count: the fixtures are generated with OPENBLAS_NUM_THREADS=1 (measured
# otherwise: 1.9e-15 absolute on one momentum coordinate of 384 at D = 128)
BLAS_THREADED_CASES = ("gc_multi_sphere_c8_dense_d128", "gc_sphere_dense_d200")


@pytest.mark.parametrize("name", sorted(gc.ALL_INTEGRATOR_CASES))
def test_oracle_reproduces_reference_fixture(name):
    """Bit for bit: pos, mom, status, completed steps and h (rtol 1e-13 for the two large dense
    cases unless OpenBLAS runs one thread)."""
    problem, g = gc.case_problem(name), gc.load_fixture(name)
    exact = name not in BLAS_THREADED_CASES or os.environ.get("OPENBLAS_NUM_THREADS") == "1"
    for n in g["step_counts"]:
        with gc.patched_drivers() as dr, np.errstate(divide="ignore", invalid="ignore"):
            out = dr.oracle_run(problem, int(n), dirs=g["dirs"])
        for k in ("status", "n_done", "pos", "mom", "h"):
            lbl = f"{name}[{n}] {k}"
            if exact or k in ("status", "n_done"):
                np.testing.assert_array_equal(out[k], g[f"{k}_{n}"], err_msg=lbl)
            else:
                np.testing.assert_allclose(out[k], g[f"{k}_{n}"], rtol=1e-13, atol=1e-14,
                                           err_msg=lbl)


@pytest.mark.parametrize("name", sorted(gc.HMC_CASES))
def test_oracle_hmc_reproduces_reference_fixture(name):
    _, n_iter, n_step, seed = gc.HMC_CASES[name]
    g = gc.load_fixture(name)
    with gc.patched_drivers() as dr:
        out = dr.oracle_hmc(gc.case_problem(name), n_iter, n_step, seed)
    for k in ("pos", "dir", "n_step", "accept_stat"):
        np.testing.assert_array_equal(out[k], g[k], err_msg=k)


@pytest.mark.parametrize("name", sorted(gc.NUTS_CASES))
def test_oracle_nuts_reproduces_reference_fixture(name):
    _, n_iter, seed, depth = gc.NUTS_CASES[name]
    g = gc.load_fixture(name)
    with gc.patched_drivers() as dr:
        out = dr.oracle_nuts(gc.case_problem(name), n_iter, seed, max_tree_depth=depth)
    for k in ("pos", "dir", "n_step", "tree_depth"):
        np.testing.assert_array_equal(out[k], g[k], err_msg=k)
    np.testing.assert_allclose(out["accept_stat"], g["accept_stat"], rtol=1e-14, atol=1e-15)


@pytest.mark.parametrize("name", sorted(gc.ADAPT_CASES))
def test_oracle_warm_up_reproduces_reference_fixture(name):
    g = gc.load_fixture(name)
    out = gc.oracle_adapt_run(name)
    for k in ("pos", "final_pos", "final_mom", "step_size"):
        np.testing.assert_array_equal(out[k], g[k], err_msg=k)


@pytest.mark.skipif(not gc.dr.reference_available(), reason="reference copy not present")
@pytest.mark.parametrize("name", ["gc_multi_sphere_c4_dense_d16", "gc_torus",
                                  "gc_multi_sphere_c2_identity_d12_singular"])
def test_oracle_matches_live_reference(name):
    problem, g = gc.case_problem(name), gc.load_fixture(name)
    with gc.patched_drivers() as dr, np.errstate(divide="ignore", invalid="ignore"):
        ref = dr.reference_run(problem, 5, dirs=g["dirs"])
        out = dr.oracle_run(problem, 5, dirs=g["dirs"])
    for k in ("status", "n_done", "pos", "mom", "h"):
        np.testing.assert_array_equal(out[k], ref[k], err_msg=k)
