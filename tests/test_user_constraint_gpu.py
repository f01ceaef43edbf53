"""User-written constraints (``CudaTarget(..., n_constr=...)``) on the GPU: the registry's
constrained targets rewritten as user sources against the reference fixtures, the user
constraint against the registry one on the same warp kernel with identical inputs, and models the
registry cannot express against fixtures of the unmodified reference (uc_*)."""
import os

import ctypes
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from mici_b200 import _lib, engine, integrators, samplers, solvers, systems, transitions
from mici_b200.adapters import DualAveragingStepSizeAdapter
from mici_b200.states import ChainState
from mici_b200.targets import CudaTarget, MultiSphere, Sphere

import gaussian_constrained_cases as gc
from golden_util import ATOL, RTOL, assert_matches_golden, load_case, load_hmc_case, load_nuts_case
from make_user_constraint_golden import CASES as UC_CASES
from user_constraint_sources import MULTI_SPHERE, SPHERE, UC_MODELS, registry_as_user

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

CASES = ["s1_sphere_identity_d5", "s1_sphere_dense_d10", "s1_sphere_dense_d10_lebesgue",
         "s1_sphere_diag_d70_inner2", "s2_multi_sphere_c4_dense_d16",
         "s2_multi_sphere_c8_dense_d32_lebesgue", "s2_multi_sphere_c8_quasi_newton_d16",
         "c3_torus", "c3_torus_lebesgue", "c3_torus_bigstep", "n4_line_search_torus"]
GC_CASES = ["gc_sphere_dense_d10", "gc_sphere_dense_d200", "gc_multi_sphere_c8_dense_d128"]


def _user_system(ref):
    """A constrained system like the registry system `ref`, holding the user rewrite of its
    target."""
    target = registry_as_user(ref.target)
    if isinstance(ref, systems.GaussianDenseConstrainedEuclideanMetricSystem):
        return systems.GaussianDenseConstrainedEuclideanMetricSystem(target, metric=ref.metric)
    return systems.DenseConstrainedEuclideanMetricSystem(
        target, metric=ref.metric, dens_wrt_hausdorff=ref.dens_wrt_hausdorff)


def _user_integrator(problem, **overrides):
    return engine.build_integrator(problem, system=_user_system(engine.build_system(problem)),
                                   **overrides)


@pytest.fixture(scope="module", autouse=True)
def _compiled_images():
    """Compile every image this module uses up front, in parallel (one NVRTC compile of the
    constrained kernels takes about a minute of one CPU core)."""
    problems = [load_case(n)[0] for n in CASES] + [gc.case_problem(n) for n in GC_CASES]
    problems += [load_hmc_case("hmc_s1_sphere_d20_dense")[0],
                 load_nuts_case("nuts_c3_torus_constrained")[0],
                 gc.case_problem("gc_nuts_multi_sphere_c2_d12")]
    targets = [registry_as_user(engine.build_system(p).target) for p in problems]
    targets += [CudaTarget(200, SPHERE, n_constr=1, mhp_constr=True, name="sphere"),
                CudaTarget(128, MULTI_SPHERE, n_constr=8, mhp_constr=True, name="multi_sphere")]
    targets += [make() for make, _, _ in UC_MODELS.values()]
    with ThreadPoolExecutor(8) as pool:
        list(pool.map(lambda t: t.compile(), targets))


def _run(integ, problem, n_steps, dirs):
    state = engine.build_state(problem, DEV, dirs=dirs)
    new = integ.step_n(state, n_steps, return_h=True)
    torch.cuda.synchronize()
    return {k: getattr(new, a).cpu().numpy()
            for k, a in (("pos", "pos"), ("mom", "mom"), ("status", "status"),
                         ("n_done", "n_done"), ("h", "h"), ("iters", "solver_iters"))}


@pytest.mark.parametrize("name", CASES)
def test_registry_constraints_as_user_sources_match_reference_fixtures(name):
    problem, dirs, overrides, g = load_case(name)
    integ = _user_integrator(problem, **(overrides or {}))
    for n_steps in g["step_counts"]:
        out = _run(integ, problem, int(n_steps), dirs)
        ok = out["status"] == 0
        out["h"] = np.where(ok, out["h"], np.nan)
        gg = dict(g)
        gg[f"h_{n_steps}"] = np.where(ok, g[f"h_{n_steps}"], np.nan)
        assert_matches_golden(out, gg, int(n_steps), label=f"{name}[{n_steps}]",
                              kind_flip_frac=0.05 if name.endswith("bigstep") else 0.0)


@pytest.mark.parametrize("name", GC_CASES)
def test_gaussian_system_with_user_constraint_matches_reference_fixtures(name):
    problem, g = gc.case_problem(name), gc.load_fixture(name)
    integ = _user_integrator(problem)
    for n in g["step_counts"]:
        out = _run(integ, problem, int(n), g["dirs"])
        lbl = f"{name}[{n}]"
        np.testing.assert_array_equal(out["status"], g[f"status_{n}"], err_msg=lbl)
        np.testing.assert_array_equal(out["n_done"], g[f"n_done_{n}"], err_msg=lbl)
        np.testing.assert_allclose(out["pos"], g[f"pos_{n}"], rtol=RTOL, atol=ATOL, err_msg=lbl)
        np.testing.assert_allclose(out["mom"], g[f"mom_{n}"], rtol=RTOL, atol=ATOL, err_msg=lbl)
        np.testing.assert_allclose(out["h"], g[f"h_{n}"], rtol=RTOL, atol=1e-9, err_msg=lbl)
        ok = g[f"status_{n}"] == 0
        np.testing.assert_array_equal(out["iters"][ok], g[f"newton_iters_{n}"][ok], err_msg=lbl)


def test_user_sphere_static_hmc_matches_reference_fixture():
    problem, n_iter, n_step, seed, g = load_hmc_case("hmc_s1_sphere_d20_dense")
    integ = _user_integrator(problem)
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    final, stats, trace = transitions.sample_hmc(integ.system, integ, state, rngs, n_iter, n_step,
                                                 trace_pos=True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(stats["accepted"].cpu().numpy(), g["accepted"].astype(bool))
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-9, atol=1e-11)
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"])
    np.testing.assert_array_equal(stats["n_step"].cpu().numpy(), g["n_step"])


def _nuts_matches(problem, n_iter, seed, g, depth=None, keys=("n_step", "tree_depth", "diverging")):
    integ = _user_integrator(problem)
    kw = {} if depth is None else {"max_tree_depth": depth}
    tr = transitions.MultinomialDynamicIntegrationTransition(integ.system, integ, **kw)
    assert not tr._fused
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    final, stats, trace = transitions.sample_chains(integ.system, integ, state, rngs, 0, n_iter,
                                                    integration_transition=tr)
    torch.cuda.synchronize()
    for k in keys:
        if k in g:
            np.testing.assert_array_equal(stats[k].cpu().numpy().astype(np.float64), g[k],
                                          err_msg=k)
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(stats["accept_stat"].cpu().numpy(), g["accept_stat"], rtol=1e-7,
                               atol=1e-10)


def test_user_torus_nuts_runs_lock_step_and_matches_reference_fixture():
    problem, n_iter, seed, opts, g = load_nuts_case("nuts_c3_torus_constrained")
    assert set(opts) <= {"max_tree_depth"}
    _nuts_matches(problem, n_iter, seed, g, depth=opts.get("max_tree_depth"),
                  keys=("n_step", "tree_depth", "diverging", "convergence_error",
                        "non_reversible_step"))


def test_gaussian_user_multi_sphere_nuts_matches_reference_fixture():
    name = "gc_nuts_multi_sphere_c2_d12"
    _, n_iter, seed, depth = gc.NUTS_CASES[name]
    _nuts_matches(gc.case_problem(name), n_iter, seed, gc.load_fixture(name), depth=depth)


def _sample_with_adapter(target, metric, pos, seed, random_n_step):
    system = systems.DenseConstrainedEuclideanMetricSystem(target, metric=metric)
    integ = integrators.ConstrainedLeapfrogIntegrator(system, 0.2)
    rng = np.random.default_rng(seed)
    sampler = (samplers.RandomMetropolisHMC(system, integ, rng, (2, 6)) if random_n_step
               else samplers.StaticMetropolisHMC(system, integ, rng, 4))
    pos = torch.as_tensor(pos, device=DEV)
    state = ChainState(pos=pos, mom=torch.zeros_like(pos), dir=1)
    out = sampler.sample_chains(6, 4, state, adapters=[DualAveragingStepSizeAdapter()],
                                n_worker=1, display_progress=False)
    return out, integ


@pytest.mark.parametrize("random_n_step", (False, True))
def test_sample_chains_with_adapter_user_equals_registry(random_n_step):
    """Static and random HMC through sample_chains with dual-averaging step-size adaptation: the
    user sphere follows the registry sphere on the same seeds."""
    dim, n = 12, 8
    rng = np.random.default_rng(5)
    pos = rng.normal(size=(n, dim))
    pos /= np.linalg.norm(pos, axis=1, keepdims=True)
    a = rng.normal(size=(dim, dim)) / np.sqrt(dim)
    metric = a @ a.T + np.identity(dim)
    reg, ireg = _sample_with_adapter(Sphere(dim), metric, pos, 11, random_n_step)
    usr, iusr = _sample_with_adapter(CudaTarget(dim, SPHERE, n_constr=1, mhp_constr=True,
                                                name="sphere"), metric, pos, 11, random_n_step)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(usr.statistics["n_step"].cpu().numpy(),
                                  reg.statistics["n_step"].cpu().numpy())
    np.testing.assert_allclose(usr.traces["pos"].cpu().numpy(), reg.traces["pos"].cpu().numpy(),
                               rtol=1e-8, atol=1e-10)
    assert iusr.step_size == pytest.approx(ireg.step_size, rel=1e-8)


def _launch(target, q, p, dirs, eps, lengths, n_steps, metric, solver, counts, gaussian=False):
    """One launch of the warp kernel on `target` (registry or user) with per-chain step sizes and
    lengths, mixed directions, a dense metric and call counters."""
    n, dim = q.shape
    cls = (systems.GaussianDenseConstrainedEuclideanMetricSystem if gaussian
           else systems.DenseConstrainedEuclideanMetricSystem)
    system = cls(target, metric=metric)
    model = system._model(q.device)
    o = {k: torch.empty_like(q) for k in ("pos", "mom")}
    o["h"] = torch.empty(n, dtype=torch.float64, device=DEV)
    for k in ("status", "n_done", "iters"):
        o[k] = torch.empty(n, dtype=torch.int32, device=DEV)
    extra = tuple(_lib.ptr(x) for x in system.rotation_args(q.device)) if gaussian else ()
    entry = ("mb200_constrained_leapfrog_gaussian_euclidean" if gaussian
             else "mb200_constrained_leapfrog_euclidean")
    user = ()
    if isinstance(target, CudaTarget):
        entry += "_user"
        user = (target.handle(),)
    counts.zero_()
    _lib.load().mb200_set_call_counters(_lib.ptr(counts))
    try:
        rc = getattr(_lib.load(), entry)(
            _lib.ptr(q), _lib.ptr(p), _lib.ptr(o["pos"]), _lib.ptr(o["mom"]), _lib.ptr(dirs), n,
            dim, 0.0, _lib.ptr(eps), n_steps, _lib.ptr(lengths), 1, 2,
            _lib.ptr(system.metric.inv_device(q.device)), *extra, ctypes.byref(model), solver,
            1e-9, 1e-8, 1e10, 50, 10, 2e-8, _lib.ptr(o["h"]), _lib.ptr(o["status"]),
            _lib.ptr(o["n_done"]), _lib.ptr(o["iters"]), _lib.current_stream_ptr(q.device), *user)
        _lib.check(rc, entry)
    finally:
        _lib.load().mb200_set_call_counters(None)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in o.items()}
    out["counts"] = counts.cpu().numpy()
    return out


@pytest.mark.parametrize("kind,n,dim,gaussian", [("multi_sphere", 8192, 128, False),
                                                 ("multi_sphere", 8192, 128, True),
                                                 ("sphere", 2048, 200, False)])
def test_user_constraint_equals_registry_on_the_warp_kernel(kind, n, dim, gaussian):
    rng = np.random.default_rng(dim + n)
    n_constr = 8 if kind == "multi_sphere" else 1
    block = dim // n_constr
    q = rng.normal(size=(n, dim))
    for k in range(n_constr):  # on the manifold to rounding
        q[:, k * block:(k + 1) * block] /= np.linalg.norm(q[:, k * block:(k + 1) * block], axis=1,
                                                          keepdims=True)
    a = rng.normal(size=(dim, dim)) / np.sqrt(dim)
    metric = a @ a.T + np.identity(dim)
    p = rng.normal(size=(n, dim)) @ np.linalg.cholesky(metric).T
    q, p = (torch.as_tensor(x, device=DEV) for x in (q, p))
    dirs = torch.as_tensor(np.where(np.arange(n) % 3 == 1, -1, 1).astype(np.int32), device=DEV)
    hi = 0.3 if kind == "multi_sphere" else 0.03  # most chains complete their steps
    eps = torch.as_tensor(rng.uniform(hi / 6, hi, size=n), device=DEV)
    lengths = torch.as_tensor(rng.integers(0, 6, size=n).astype(np.int32), device=DEV)
    counts = torch.zeros(n, 4, dtype=torch.int32, device=DEV)
    if kind == "multi_sphere":
        reg_t = MultiSphere(dim, 8)
        usr_t = CudaTarget(dim, MULTI_SPHERE, n_constr=8, mhp_constr=True, name="multi_sphere")
    else:
        reg_t = Sphere(dim)
        usr_t = CudaTarget(dim, SPHERE, n_constr=1, mhp_constr=True, name="sphere")
    p = systems.DenseConstrainedEuclideanMetricSystem(reg_t, metric=metric) \
        .project_onto_cotangent_space(p, ChainState(pos=q, mom=p, dir=1))
    for solver in (0, 1, 2):
        reg = _launch(reg_t, q, p, dirs, eps, lengths, 5, metric, solver, counts, gaussian)
        usr = _launch(usr_t, q, p, dirs, eps, lengths, 5, metric, solver, counts, gaussian)
        lbl = f"{kind} solver {solver}"
        assert (reg["n_done"] > 0).mean() > 0.5, lbl
        for k in ("status", "n_done", "iters", "counts"):
            np.testing.assert_array_equal(usr[k], reg[k], err_msg=f"{lbl} {k}")
        for k in ("pos", "mom", "h"):
            np.testing.assert_allclose(usr[k], reg[k], rtol=1e-9, atol=1e-12, err_msg=f"{lbl} {k}")


def test_user_projection_equals_registry():
    dim, n = 40, 64
    rng = np.random.default_rng(3)
    q = rng.normal(size=(n, dim))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q, p = (torch.as_tensor(x, device=DEV) for x in (q, rng.normal(size=(n, dim))))
    state = ChainState(pos=q, mom=p, dir=1)
    for cls in (systems.DenseConstrainedEuclideanMetricSystem,
                systems.GaussianDenseConstrainedEuclideanMetricSystem):
        reg = cls(Sphere(dim), metric=np.linspace(1, 2, dim))
        usr = cls(CudaTarget(dim, SPHERE, n_constr=1, mhp_constr=True, name="sphere"),
                  metric=np.linspace(1, 2, dim))
        np.testing.assert_allclose(usr.project_onto_cotangent_space(p, state).cpu().numpy(),
                                   reg.project_onto_cotangent_space(p, state).cpu().numpy(),
                                   rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(usr.h(state).cpu().numpy(), reg.h(state).cpu().numpy(),
                                   rtol=1e-12)


# ---------------------------------------------------------------- models the registry lacks


def _uc_case(name):
    """The fixture of a uc_* case and the integrator that reproduces it: the model's CudaTarget
    on the case's system, metric, projection solver and step size."""
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    model, system_kind, hausdorff, _, _, solver, eps = UC_CASES[name][:7]
    target = UC_MODELS[model][0]()
    metric = g.get("metric")
    if system_kind == "gaussian":
        system = systems.GaussianDenseConstrainedEuclideanMetricSystem(target, metric=metric)
    else:
        system = systems.DenseConstrainedEuclideanMetricSystem(target, metric=metric,
                                                               dens_wrt_hausdorff=hausdorff)
    integ = integrators.ConstrainedLeapfrogIntegrator(
        system, eps,
        projection_solver=getattr(solvers, "solve_projection_onto_manifold_" + solver))
    return g, integ


@pytest.mark.parametrize("name", [n for n, c in UC_CASES.items() if c[7] == "steps"])
def test_models_the_registry_cannot_express_match_reference_fixtures(name):
    """SO(3) (six overlapping constraints, F in aux), a generator constraint on the Gaussian
    system (five constraints sharing theta, non-constant Hessian) and the l4 sphere at D = 200
    (KP 4, Lebesgue density, quasi-Newton), the last also at a step where chains fail."""
    g, integ = _uc_case(name)
    for n in g["step_counts"]:
        state = ChainState(pos=torch.as_tensor(g["pos0"], device=DEV),
                           mom=torch.as_tensor(g["mom0"], device=DEV),
                           dir=torch.as_tensor(g["dirs"], device=DEV))
        new = integ.step_n(state, int(n), return_h=True)
        torch.cuda.synchronize()
        out = {k: getattr(new, k).cpu().numpy() for k in ("pos", "mom", "status", "n_done", "h")}
        assert_matches_golden(out, g, int(n), label=f"{name}[{n}]")
    if name.endswith("bigstep"):
        assert (g[f"status_{n}"] == 1).any() and (g[f"status_{n}"] == 0).any()


def test_so3_static_hmc_matches_reference_fixture():
    g, integ = _uc_case("uc_hmc_so3_dense")
    n_iter, n_step, seed = int(g["n_iter"]), int(g["n_step_arg"]), int(g["seed"])
    state = ChainState(pos=torch.as_tensor(g["pos0"], device=DEV),
                       mom=torch.as_tensor(g["mom0"], device=DEV), dir=1)
    rngs = [np.random.default_rng([seed, i]) for i in range(g["pos0"].shape[0])]
    final, stats, trace = transitions.sample_hmc(integ.system, integ, state, rngs, n_iter, n_step,
                                                 trace_pos=True)
    torch.cuda.synchronize()
    np.testing.assert_allclose(trace.cpu().numpy(), g["trace"], rtol=1e-9, atol=1e-11)
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"])
    np.testing.assert_array_equal(stats["n_step"].cpu().numpy(), g["n_step"])
    np.testing.assert_allclose(stats["metrop_accept_prob"].cpu().numpy(), g["metrop_accept_prob"],
                               rtol=1e-8, atol=1e-12)
