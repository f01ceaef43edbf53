"""User-written targets (``CudaTarget``) on the GPU: registry models rewritten as user sources
against the reference fixtures, the user funnel against the registry's general kernel, and models
the registry cannot express against fixtures of the unmodified reference (ut_*)."""

import ctypes
import os

import numpy as np
import pytest
import torch

from mici_b200 import _lib, engine, integrators, systems, transitions
from mici_b200.states import ChainState

from golden_util import ATOL, RTOL, assert_matches_golden, load_case, load_hmc_case, load_nuts_case
from user_target_sources import FUNNEL, USER_MODELS, registry_as_user

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _user_integrator(problem):
    """The problem's integrator, on an EuclideanMetricSystem holding the user rewrite of its
    registry target."""
    ref = engine.build_system(problem)
    system = systems.EuclideanMetricSystem(registry_as_user(ref.target), metric=ref.metric)
    return engine.build_integrator(problem, system=system)


@pytest.mark.parametrize("name", [
    "c0_std_gaussian", "c1_funnel_identity", "c1_funnel_diag", "c1_funnel_dense",
    "c1_funnel_dense_d24", "n4_bcss2_funnel_d24", "n4_bcss3_funnel_d40_diag",
    "n4_bcss4_funnel_d130"])
def test_registry_models_as_user_sources_match_reference_fixtures(name):
    problem, dirs, overrides, g = load_case(name)
    integ = _user_integrator(problem)
    for n_steps in g["step_counts"]:
        state = engine.build_state(problem, DEV, dirs=dirs)
        new = integ.step_n(state, int(n_steps), return_h=True)
        out = {k: getattr(new, k).cpu().numpy() for k in ("pos", "mom", "status", "n_done", "h")}
        assert_matches_golden(out, g, int(n_steps), label=f"{name}[{n_steps}]")
        # the system's own pieces on the user image
        h = integ.system.h(new)
        np.testing.assert_allclose(h.cpu().numpy(), out["h"], rtol=1e-12, atol=1e-12)


def test_user_funnel_static_hmc_matches_reference_fixture():
    problem, n_iter, n_step, seed, g = load_hmc_case("hmc_c1_funnel_d16")
    integ = _user_integrator(problem)
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    final, stats, trace = transitions.sample_hmc(integ.system, integ, state, rngs, n_iter, n_step,
                                                 trace_pos=True)
    np.testing.assert_array_equal(stats["accepted"].cpu().numpy(), g["accepted"].astype(bool))
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-9, atol=1e-11)
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"])


def test_user_funnel_nuts_runs_lock_step_and_matches_reference_fixture():
    problem, n_iter, seed, opts, g = load_nuts_case("nuts_c1_multinomial_d10")
    assert not opts
    integ = _user_integrator(problem)
    tr = transitions.MultinomialDynamicIntegrationTransition(integ.system, integ)
    assert not tr._fused
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    final, stats, trace = transitions.sample_chains(integ.system, integ, state, rngs, 0, n_iter,
                                                    integration_transition=tr)
    for k in ("n_step", "tree_depth", "diverging"):
        np.testing.assert_array_equal(stats[k].cpu().numpy().astype(np.float64), g[k], err_msg=k)
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(stats["accept_stat"].cpu().numpy(), g["accept_stat"], rtol=1e-7,
                               atol=1e-10)


def _generic_launch(fn, args, user=None):
    lib = _lib.load()
    rc = getattr(lib, fn)(*args, *(() if user is None else (user,)))
    _lib.check(rc, fn)


def _user_vs_registry(n, dim, n_steps, seed):
    """The user funnel and the registry funnel through the general-dimension kernel on identical
    inputs: mixed directions, per-chain step sizes and lengths, dense metric, call counters."""
    rng = np.random.default_rng(seed)
    q = torch.as_tensor(rng.normal(size=(n, dim)) * 0.5, device=DEV)
    p = torch.as_tensor(rng.normal(size=(n, dim)), device=DEV)
    a = rng.normal(size=(dim, dim)) / np.sqrt(dim)
    metric = a @ a.T + np.identity(dim)
    dirs = torch.as_tensor(np.where(np.arange(n) % 3 == 1, -1, 1).astype(np.int32), device=DEV)
    eps = torch.as_tensor(rng.uniform(0.02, 0.08, size=n), device=DEV)
    lengths = torch.as_tensor(rng.integers(0, n_steps + 1, size=n).astype(np.int32), device=DEV)
    from mici_b200.targets import CudaTarget, NealFunnel

    outs = []
    for target in (NealFunnel(dim), CudaTarget(dim, FUNNEL)):
        system = systems.EuclideanMetricSystem(target, metric=metric)
        model = system._model(q.device)
        minv = system.metric.inv_device(q.device)
        counts = torch.zeros(n, 4, dtype=torch.int32, device=DEV)
        o = {k: torch.empty_like(q) for k in ("pos", "mom")}
        o["h"] = torch.empty(n, dtype=torch.float64, device=DEV)
        o["status"] = torch.empty(n, dtype=torch.int32, device=DEV)
        o["n_done"] = torch.empty(n, dtype=torch.int32, device=DEV)
        args = (_lib.ptr(q), _lib.ptr(p), _lib.ptr(o["pos"]), _lib.ptr(o["mom"]), _lib.ptr(dirs),
                n, dim, 0.0, _lib.ptr(eps), n_steps, _lib.ptr(lengths), 0, None, 1, 2,
                _lib.ptr(minv), ctypes.byref(model), _lib.ptr(o["h"]), _lib.ptr(o["status"]),
                _lib.ptr(o["n_done"]), _lib.current_stream_ptr(q.device))
        _lib.load().mb200_set_call_counters(_lib.ptr(counts))
        try:
            if isinstance(target, CudaTarget):
                _generic_launch("mb200_leapfrog_euclidean_user", args, target.handle())
            else:
                _generic_launch("mb200_leapfrog_euclidean_generic", args)
        finally:
            _lib.load().mb200_set_call_counters(None)
        o["counts"] = counts
        outs.append({k: v.cpu().numpy() for k, v in o.items()})
    reg, usr = outs
    for k in ("pos", "mom", "h"):
        np.testing.assert_allclose(usr[k], reg[k], rtol=1e-10, atol=1e-12, err_msg=k)
    for k in ("status", "n_done", "counts"):
        np.testing.assert_array_equal(usr[k], reg[k], err_msg=k)


@pytest.mark.parametrize("n_steps", [1, 5, 20])
def test_user_funnel_equals_registry_general_kernel_at_c1_size(n_steps):
    _user_vs_registry(8192, 128, n_steps, n_steps)


@pytest.mark.parametrize("dim", [300, 1024])
def test_user_funnel_equals_registry_general_kernel_one_chain_per_warp(dim):
    """D > 256: the CPW = 1 layouts (KP = 8, 16), whose shared memory exceeds 48 KB."""
    _user_vs_registry(257, dim, 5, dim)


def test_repeat_handle_lookup_is_a_dictionary_access(monkeypatch):
    """After the first launch, a user target's launches find its loaded image without compiling,
    hashing or loading again."""
    from mici_b200 import jit
    from mici_b200.targets import CudaTarget

    target = CudaTarget(16, FUNNEL + "\n// handle probe\n")
    system = systems.EuclideanMetricSystem(target)
    integ = integrators.LeapfrogIntegrator(system, 0.05)
    state = ChainState(pos=torch.zeros(5, 16, dtype=torch.float64, device=DEV),
                       mom=torch.ones(5, 16, dtype=torch.float64, device=DEV), dir=1)
    first = integ.step_n(state, 2, return_h=True)

    def fail(*a, **k):
        raise AssertionError("looked up the slow way")

    for name in ("compile_target", "cache_key", "_headers_digest", "version"):
        monkeypatch.setattr(jit, name, fail)
    again = integ.step_n(state, 2, return_h=True)
    torch.testing.assert_close(again.pos, first.pos, rtol=0, atol=0)
    torch.testing.assert_close(system.h(again), first.h, rtol=0, atol=0)


def test_user_funnel_eval_pieces_equal_registry():
    from mici_b200.targets import CudaTarget, NealFunnel

    for dim in (7, 64, 200, 1024):
        rng = np.random.default_rng(dim)
        state = ChainState(pos=torch.as_tensor(rng.normal(size=(37, dim)) * 0.5, device=DEV),
                           mom=torch.as_tensor(rng.normal(size=(37, dim)), device=DEV), dir=1)
        reg = systems.EuclideanMetricSystem(NealFunnel(dim), metric=np.linspace(1, 2, dim))
        usr = systems.EuclideanMetricSystem(CudaTarget(dim, FUNNEL), metric=np.linspace(1, 2, dim))
        for fn in ("neg_log_dens", "grad_neg_log_dens", "h"):
            torch.testing.assert_close(getattr(usr, fn)(state), getattr(reg, fn)(state),
                                       rtol=1e-12, atol=1e-12, msg=f"{fn} dim {dim}")


# ---------------------------------------------------------------- ut_* fixtures


def _ut(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    from make_user_target_golden import CASES, INTEGRATORS

    model, n, _, integ_name, eps, kind, arg, seed = CASES[name]
    target = USER_MODELS[model][0]()
    system = systems.EuclideanMetricSystem(target, metric=g.get("metric"))
    integ = getattr(integrators, INTEGRATORS[integ_name])(system, float(g["step_size"]))
    state = ChainState(pos=torch.as_tensor(g["pos0"], device=DEV),
                       mom=torch.as_tensor(g["mom0"], device=DEV), dir=1)
    return g, integ, state, kind, arg, seed


@pytest.mark.parametrize("name", ["ut_eight_schools_identity", "ut_ar1_diag", "ut_ar1_diag_bcss3",
                                  "ut_logistic_dense"])
def test_user_models_steps_match_reference(name):
    g, integ, state, _, counts, _ = _ut(name)
    state.dir = torch.as_tensor(g["dirs"], device=DEV)
    for n_steps in counts:
        new = integ.step_n(state, n_steps, return_h=True)
        assert not new.status.any()
        np.testing.assert_allclose(new.pos.cpu().numpy(), g[f"pos_{n_steps}"], rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(new.mom.cpu().numpy(), g[f"mom_{n_steps}"], rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(new.h.cpu().numpy(), g[f"h_{n_steps}"], rtol=RTOL, atol=1e-9)


def test_user_logistic_static_hmc_matches_reference():
    g, integ, state, _, (n_iter, n_step), seed = _ut("ut_hmc_logistic_dense")
    rngs = [np.random.default_rng([seed, i]) for i in range(state.pos.shape[0])]
    final, stats, trace = transitions.sample_hmc(integ.system, integ, state, rngs, n_iter, n_step,
                                                 trace_pos=True)
    np.testing.assert_allclose(trace.cpu().numpy(), g["trace"], rtol=1e-9, atol=1e-11)
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"])
    np.testing.assert_allclose(stats["metrop_accept_prob"].cpu().numpy(), g["metrop_accept_prob"],
                               rtol=1e-8, atol=1e-12)


def test_user_logistic_dynamic_multinomial_hmc_matches_reference():
    g, integ, state, _, n_iter, seed = _ut("ut_nuts_logistic_dense")
    rngs = [np.random.default_rng([seed, i]) for i in range(state.pos.shape[0])]
    tr = transitions.MultinomialDynamicIntegrationTransition(integ.system, integ)
    final, stats, trace = transitions.sample_chains(integ.system, integ, state, rngs, 0, n_iter,
                                                    integration_transition=tr)
    for k in ("n_step", "tree_depth", "diverging"):
        np.testing.assert_array_equal(stats[k].cpu().numpy().astype(np.float64), g[k], err_msg=k)
    np.testing.assert_allclose(trace.cpu().numpy(), g["trace"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(stats["av_metrop_accept_prob"].cpu().numpy(),
                               g["av_metrop_accept_prob"], rtol=1e-7, atol=1e-10)
