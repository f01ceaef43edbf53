"""GPU parity tests: the CUDA path (through the C ABI) against the reference fixtures
(tests/golden, generated from the unmodified reference) and against the oracle port on the
same seeded inputs.  Tolerance: rtol 1e-10 (north_star), atol 1e-12 (SURVEY.md 8(d))."""

import numpy as np
import pytest
import torch

from mici_b200 import engine, problems
from oracle import drivers as dr

from golden_util import ATOL, RTOL, assert_matches_golden, case_names, load_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

HMC_NAMES = ["hmc_c1_funnel_d16", "hmc_c0_std_gaussian", "hmc_c2_softabs_d8", "hmc_c4_dense_d12",
             "hmc_c3_torus", "hmc_s1_sphere_d20_dense", "hmc_c1_random_n_step",
             "hmc_g1_gaussian_split_d16"]


def run_cuda(problem, n_steps, dirs=None, overrides=None, chains=None, return_h=True):
    integ = engine.build_integrator(problem, **(overrides or {}))
    state = engine.build_state(problem, DEV, dirs=dirs, chains=chains)
    pos0, mom0 = state.pos.clone(), state.mom.clone()
    new = integ.step_n(state, n_steps, return_h=return_h)
    torch.cuda.synchronize()
    # Integrator.step must not mutate its argument (reference tests/test_integrators.py:110-124)
    assert torch.equal(state.pos, pos0) and torch.equal(state.mom, mom0)
    assert new.pos.data_ptr() != state.pos.data_ptr()
    return {
        "pos": new.pos.cpu().numpy(),
        "mom": new.mom.cpu().numpy(),
        "status": new.status.cpu().numpy(),
        "n_done": new.n_done.cpu().numpy(),
        "h": new.h.cpu().numpy() if return_h else None,
        "iters": None if new.solver_iters is None else new.solver_iters.cpu().numpy(),
    }


@pytest.mark.parametrize("name", case_names() + case_names(failures=True))
def test_cuda_matches_reference_fixture(name):
    problem, dirs, overrides, g = load_case(name)
    for n_steps in g["step_counts"]:
        out = run_cuda(problem, int(n_steps), dirs=dirs, overrides=overrides)
        ok = out["status"] == 0
        out["h"] = np.where(ok, out["h"], np.nan)
        gg = dict(g)
        gg[f"h_{n_steps}"] = np.where(ok, g[f"h_{n_steps}"], np.nan)
        assert_matches_golden(out, gg, int(n_steps), label=f"{name}[{n_steps}]",
                              kind_flip_frac=0.05 if name.endswith("bigstep") else 0.0)


@pytest.mark.parametrize("cfg,kwargs", [
    ("C0", {"n_chains": 37, "dim": 10}),
    ("C1", {"n_chains": 64}),
    ("C1", {"n_chains": 33, "dim": 9}),
    ("C1", {"n_chains": 19, "dim": 130}),
    ("C1", {"n_chains": 5, "dim": 300}),
    ("C1", {"n_chains": 40, "dim": 96, "metric_kind": "diagonal"}),
    ("C3", {"n_chains": 64}),
])
def test_cuda_matches_oracle_port(cfg, kwargs):
    problem = problems.make_problem(cfg, **kwargs)
    dirs = np.where(np.arange(problem.n_chains) % 2 == 0, 1, -1).astype(np.int32)
    for n_steps in (1, 5, 20):
        ref = dr.oracle_run(problem, n_steps, dirs=dirs)
        out = run_cuda(problem, n_steps, dirs=dirs)
        np.testing.assert_array_equal(out["status"], ref["status"])
        np.testing.assert_allclose(out["pos"], ref["pos"], rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(out["mom"], ref["mom"], rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(out["h"], ref["h"], rtol=RTOL, atol=1e-9)


@pytest.mark.parametrize("cfg,kwargs", [("C1", {"n_chains": 48}), ("C3", {"n_chains": 48})])
def test_step_n_equals_repeated_step(cfg, kwargs):
    problem = problems.make_problem(cfg, **kwargs)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    fused = integ.step_n(state, 7)
    s = state
    for _ in range(7):
        s = integ.step(s)
    torch.cuda.synchronize()
    assert torch.equal(fused.pos, s.pos) and torch.equal(fused.mom, s.mom)


def test_dmma_and_generic_leapfrog_kernels_agree():
    """The tensor-core leapfrog kernel against the general-dimension kernel (same C ABI)."""
    import ctypes

    from mici_b200 import _lib

    problem = problems.make_problem("C1", n_chains=500)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    fast = integ.step_n(state, 10, return_h=True)
    sysm = integ.system
    n, dim = state.pos.shape
    model = sysm._model(state.pos.device)
    q, p = torch.empty_like(state.pos), torch.empty_like(state.mom)
    h = torch.empty(n, dtype=torch.float64, device=DEV)
    rc = _lib.load().mb200_leapfrog_euclidean_generic(
        _lib.ptr(state.pos), _lib.ptr(state.mom), _lib.ptr(q), _lib.ptr(p), None, n, dim,
        problem.step_size, None, 10, None, 0, None, 0, sysm.metric.kind,
        _lib.ptr(sysm.metric.inv_device(state.pos.device)),
        ctypes.byref(model), _lib.ptr(h), None, None, _lib.current_stream_ptr(state.pos.device))
    assert rc == 0
    torch.cuda.synchronize()
    torch.testing.assert_close(fast.pos, q, rtol=1e-11, atol=1e-13)
    torch.testing.assert_close(fast.mom, p, rtol=1e-11, atol=1e-13)
    torch.testing.assert_close(fast.h, h, rtol=1e-11, atol=1e-10)


def test_reversibility_full_size_c1():
    """Size-independent property at BASELINE's full C1 size (reference
    tests/test_integrators.py:75-91): n steps forward, flip dir, n steps back."""
    problem = problems.make_problem("C1")
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    fwd = integ.step_n(state, 20)
    fwd.dir = -1
    back = integ.step_n(fwd, 20)
    torch.cuda.synchronize()
    torch.testing.assert_close(back.pos, state.pos, rtol=0, atol=1e-9)
    torch.testing.assert_close(back.mom, state.mom, rtol=0, atol=1e-8)


def test_energy_conservation_full_size_c1():
    """tests/test_integrators.py:93-108 style check on all 8192 chains."""
    problem = problems.make_problem("C1")
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    h0 = integ.system.h(state)
    new = integ.step_n(state, 200, return_h=True)
    torch.cuda.synchronize()
    assert torch.isfinite(new.h).all()
    assert (new.h - h0).abs().max().item() < 5e-2


def test_constraint_satisfaction_full_size_c3():
    """tests/test_integrators.py:159-197: |c(q)| < 1e-8 and J M^-1 p = 0 after steps."""
    problem = problems.make_problem("C3")
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    new = integ.step_n(state, 10)
    torch.cuda.synchronize()
    ok = new.status == 0
    assert ok.float().mean().item() > 0.9
    q, p = new.pos[ok], new.mom[ok]
    rho = torch.sqrt(q[:, 0] ** 2 + q[:, 1] ** 2)
    c = (rho - 1.0) ** 2 + q[:, 2] ** 2 - 0.25
    assert c.abs().max().item() < 1e-8
    f = 2.0 * (rho - 1.0) / rho
    jac = torch.stack([f * q[:, 0], f * q[:, 1], 2.0 * q[:, 2]], -1)
    assert (jac * p).sum(-1).abs().max().item() < 1e-8


def test_single_chain_state_raises_like_reference():
    from mici_b200 import ChainState
    from mici_b200.errors import IntegratorError

    problem = problems.make_problem("C3", n_chains=64)
    problem.step_size = 0.4
    ref = dr.oracle_run(problem, 1)
    bad = int(np.nonzero(ref["status"])[0][0])
    good = int(np.nonzero(ref["status"] == 0)[0][0])
    integ = engine.build_integrator(problem)
    for idx, should_raise in ((bad, True), (good, False)):
        st = ChainState(
            pos=torch.as_tensor(problem.pos[idx], device=DEV),
            mom=torch.as_tensor(problem.mom[idx], device=DEV),
            dir=1,
        )
        if should_raise:
            with pytest.raises(IntegratorError):
                integ.step(st)
        else:
            new = integ.step(st)
            np.testing.assert_allclose(new.pos.cpu().numpy(), ref["pos"][idx], rtol=RTOL, atol=ATOL)


def test_rank1_low_rank_form_matches_cholesky_form_and_fixture():
    """The Sherman-Morrison metric policy (used when the per-chain factor does not fit in shared
    memory) against the per-chain Cholesky policy and the reference fixture at D = 64."""
    problem, dirs, overrides, g = load_case("c4_dense_riemannian_d64")
    chol = run_cuda(problem, 5, dirs=dirs, overrides=overrides)
    problem.metric_params = dict(problem.metric_params, force_low_rank_form=True)
    low = run_cuda(problem, 5, dirs=dirs, overrides=overrides)
    assert_matches_golden(low, g, 5, label="low-rank form")
    np.testing.assert_array_equal(low["status"], chol["status"])
    np.testing.assert_allclose(low["pos"], chol["pos"], rtol=1e-11, atol=1e-13)
    np.testing.assert_allclose(low["mom"], chol["mom"], rtol=1e-11, atol=1e-13)
    np.testing.assert_array_equal(low["iters"], chol["iters"])


def test_implicit_solver_iteration_counts_match_oracle():
    """H2 (SURVEY.md 7.2): the fused fixed-point solves stop on the same iterate as
    solve_fixed_point_direct (solvers.py:77-88) -- compare per-chain iteration counts."""
    for cfg, kwargs in (("C2", {"n_chains": 24, "dim": 8}), ("C4", {"n_chains": 6, "dim": 16})):
        problem = problems.make_problem(cfg, **kwargs)
        counts = {}
        ref = dr.oracle_run(problem, 1, counts=counts)
        out = run_cuda(problem, 1)
        np.testing.assert_array_equal(out["status"], ref["status"])
        ok = ref["status"] == 0
        ref_iters = np.array([c for c in counts["all_fp_iters"]])
        np.testing.assert_array_equal(out["iters"][ok], ref_iters[ok])


def test_riemannian_hamiltonian_matches_oracle():
    for cfg, kwargs in (("C2", {"n_chains": 16, "dim": 8}), ("C4", {"n_chains": 4, "dim": 32})):
        problem = problems.make_problem(cfg, **kwargs)
        integ = engine.build_integrator(problem)
        state = engine.build_state(problem, DEV)
        h = integ.system.h(state).cpu().numpy()
        ref = dr.oracle_run(problem, 0)
        np.testing.assert_allclose(h, ref["h_init"], rtol=RTOL, atol=1e-10)


def test_softabs_full_size_c2_reversibility_and_energy():
    """Full BASELINE size C2 (2048 chains, D = 64): size-independent properties
    (tests/test_integrators.py:75-108)."""
    problem = problems.make_problem("C2")
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    h0 = integ.system.h(state)
    fwd = integ.step_n(state, 3, return_h=True)
    ok = fwd.status == 0
    assert ok.float().mean().item() > 0.95
    dh = (fwd.h - h0)[ok].abs()
    assert dh.median().item() < 0.1 and dh.max().item() < 2.0  # step 2*eps = 0.2 (H3), D = 64
    fwd.dir = -1
    back = integ.step_n(fwd, 3)
    torch.cuda.synchronize()
    both = ok & (back.status == 0)
    torch.testing.assert_close(back.pos[both], state.pos[both], rtol=0, atol=1e-6)


def test_host_buffer_path_equals_device_path():
    """`step_n_host` (pinned host buffers, chunked over streams) returns exactly what the
    device-resident `step_n` returns: chunking the independent chains changes no result."""
    problem = problems.make_problem("C1", n_chains=777)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    ref = integ.step_n(state, 6)
    pos_h = torch.as_tensor(problem.pos).pin_memory()
    mom_h = torch.as_tensor(problem.mom).pin_memory()
    pos, mom, status = integ.step_n_host(pos_h, mom_h, 6, device=DEV, n_chunks=4)
    torch.cuda.synchronize()
    assert torch.equal(pos, ref.pos.cpu()) and torch.equal(mom, ref.mom.cpu())
    assert torch.equal(status, ref.status.cpu())
    # pageable (NumPy-backed) buffers -- what the reference's ChainState holds -- take the
    # library's own staging pipeline (worker threads + pinned bounce buffers); mixed directions
    pos_n, mom_n = np.array(problem.pos), np.array(problem.mom)
    dirs = torch.as_tensor(np.where(np.arange(777) % 3 == 0, -1, 1).astype(np.int32))
    state.dir = dirs.to(DEV)
    ref = integ.step_n(state, 6)
    for _ in range(2):  # the second call reuses the bounce buffer and the workers
        pos, mom, status = integ.step_n_host(torch.from_numpy(pos_n), torch.from_numpy(mom_n), 6,
                                             dir=dirs, device=DEV, n_chunks=5)
        assert not pos.is_pinned()
        assert torch.equal(pos, ref.pos.cpu()) and torch.equal(mom, ref.mom.cpu())
        assert torch.equal(status, ref.status.cpu())


@pytest.mark.parametrize("name", HMC_NAMES)
def test_batched_hmc_transition_matches_reference_fixture(name):
    """Row N1 on the device: whole static-HMC iterations (momentum refresh, fused trajectory,
    energy, Metropolis select, direction flips) against the reference's own transition classes,
    every chain consuming the variates of its own seeded NumPy stream."""
    from golden_util import load_hmc_case
    from mici_b200 import transitions

    problem, n_iter, n_step, seed, g = load_hmc_case(name)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    if isinstance(n_step, tuple):
        final, stats, trace = transitions.sample_chains(integ.system, integ, state, rngs, 0, n_iter,
                                                        n_step_range=n_step)
    else:
        final, stats, trace = transitions.sample_hmc(integ.system, integ, state, rngs, n_iter,
                                                     n_step, trace_pos=True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(stats["accepted"].cpu().numpy(), g["accepted"].astype(bool))
    # first transition (one trajectory from the shared initial state): north_star's tolerance;
    # later iterations compound through accept / reject decisions and fixed-point solves
    np.testing.assert_allclose(trace.cpu().numpy()[0], g["pos"][0], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-9, atol=1e-11)
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"])
    np.testing.assert_array_equal(stats["n_step"].cpu().numpy(), g["n_step"])
    np.testing.assert_allclose(stats["metrop_accept_prob"].cpu().numpy(), g["metrop_accept_prob"],
                               rtol=1e-8, atol=1e-12)


def test_batched_hmc_full_size_c1_device_rng():
    """8192 chains x D=128, variates generated on the device: acceptance statistics are sane
    and every state stays finite."""
    from mici_b200 import transitions

    problem = problems.make_problem("C1")
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1234)
    final, stats, _ = transitions.sample_hmc(integ.system, integ, state, gen, 4, 20)
    torch.cuda.synchronize()
    assert torch.isfinite(final.pos).all() and torch.isfinite(final.mom).all()
    acc = stats["accept_stat"].mean().item()
    assert 0.5 < acc <= 1.0
    assert (stats["n_step"] == 20).all()


# ---- K4 on the reference's own solver known answers (reference tests/test_solvers.py:25-80)
def _fixed_point_gpu(func_id, x0, y, tol, max_iters=100, div_tol=1e10, solver=0):
    from mici_b200 import _lib

    x0 = torch.as_tensor(np.atleast_2d(x0), device=DEV).contiguous()
    y = torch.as_tensor(np.atleast_2d(y), device=DEV).contiguous()
    n, dim = x0.shape
    out = torch.empty_like(x0)
    iters = torch.empty(n, dtype=torch.int32, device=DEV)
    status = torch.empty(n, dtype=torch.int32, device=DEV)
    rc = _lib.load().mb200_selftest_fixed_point(
        func_id, solver, _lib.ptr(x0), _lib.ptr(y), n, dim, tol, div_tol, max_iters, _lib.ptr(out),
        _lib.ptr(iters), _lib.ptr(status), _lib.current_stream_ptr(x0.device))
    assert rc == 0
    torch.cuda.synchronize()
    return out.cpu().numpy(), iters.cpu().numpy(), status.cpu().numpy()


@pytest.mark.parametrize("solver", [0, 1])
@pytest.mark.parametrize("prob,func_id", [("babylonian", 0), ("ratio", 1), ("cosine", 2)])
@pytest.mark.parametrize("tol", [1e-6, 1e-8, 1e-10])
def test_fused_fixed_point_solver_known_answers(prob, func_id, tol, solver):
    import os

    from oracle import mici_oracle as mo
    from oracle.make_golden import GOLDEN_DIR

    y = np.array([3.0, 5.0, 7.0]) if func_id < 2 else np.array([0.0])
    x0 = np.ones_like(y)
    fixed_point = y**0.5 if func_id < 2 else np.array([0.7390851332151607])
    x, iters, status = _fixed_point_gpu(func_id, x0, y, tol, solver=solver)
    assert status[0] == 0
    assert np.abs(x[0] - fixed_point).max() < tol  # reference test_solvers.py:65-80
    g = np.load(os.path.join(GOLDEN_DIR, "solver_known_answers.npz"))
    key = ("steffensen_" if solver else "") + f"{prob}_{tol:g}"
    np.testing.assert_allclose(x[0], g[key], rtol=1e-13)  # same iterate returned
    funcs = {0: lambda v: (y / v + v) / 2, 1: lambda v: (v + y) / (v + 1), 2: np.cos}
    ref_solver = mo.solve_fixed_point_steffensen if solver else mo.solve_fixed_point_direct
    _, n_ref = ref_solver(funcs[func_id], x0, convergence_tol=tol)
    assert iters[0] == n_ref  # same stopping iteration (H2)


@pytest.mark.parametrize("func_id", [3, 4])
def test_fused_fixed_point_solver_divergence_and_max_iters(func_id):
    _, _, status = _fixed_point_gpu(func_id, np.arange(3.0), np.zeros(3), 1e-9, max_iters=10000)
    assert status[0] == 1  # ConvergenceError (reference test_solvers.py:83-93)
    _, _, status = _fixed_point_gpu(2, np.array([1.0]), np.array([0.0]), 1e-10, max_iters=1)
    assert status[0] == 1  # max_iters exceeded (reference test_solvers.py:96-107)


# ---- K3 (Jacobi eigensolver) on dense symmetric matrices against numpy.linalg.eigh
@pytest.mark.parametrize("dim", [1, 2, 3, 7, 16, 33, 64, 77])
@pytest.mark.parametrize("warm", [False, True])
def test_jacobi_eigensolver_dense_matrices(dim, warm):
    from mici_b200 import _lib

    rng = np.random.default_rng(100 + dim)
    n = 6
    base = rng.standard_normal((dim, dim))
    mats = np.empty((n, dim, dim))
    for i in range(n):
        a = base + (0.05 if warm else 1.0) * rng.standard_normal((dim, dim))
        mats[i] = 0.5 * (a + a.T)
    if dim >= 7:
        mats[1][np.abs(mats[1]) < 0.8] = 0.0  # sparse symmetric matrix (identity-rotation skips)
        mats[1] = 0.5 * (mats[1] + mats[1].T)
        mats[2] = np.diag(rng.standard_normal(dim))  # already diagonal
    m = torch.as_tensor(mats, device=DEV).contiguous()
    val = torch.empty((n, dim), dtype=torch.float64, device=DEV)
    vec = torch.empty((n, dim, dim), dtype=torch.float64, device=DEV)
    st = torch.empty(n, dtype=torch.int32, device=DEV)
    rc = _lib.load().mb200_selftest_eigh(_lib.ptr(m), n, dim, 0 if warm else -1, _lib.ptr(val),
                                         _lib.ptr(vec), _lib.ptr(st), _lib.current_stream_ptr(m.device))
    assert rc == 0
    torch.cuda.synchronize()
    assert (st == 0).all()
    val, vec = val.cpu().numpy(), vec.cpu().numpy()
    for i in range(n):
        ref = np.linalg.eigvalsh(mats[i])
        scale = max(1.0, np.abs(ref).max())
        np.testing.assert_allclose(np.sort(val[i]), ref, rtol=0, atol=5e-14 * scale)
        u = vec[i]
        np.testing.assert_allclose(u.T @ u, np.identity(dim), atol=1e-13)
        np.testing.assert_allclose(u @ np.diag(val[i]) @ u.T, mats[i], atol=1e-13 * scale)


@pytest.mark.parametrize("cfg,kwargs", [
    ("C3", {"n_chains": 64}),
    ("S1", {"n_chains": 48, "dim": 40, "metric_kind": "dense"}),
    ("S1", {"n_chains": 48, "dim": 150, "metric_kind": "diagonal"}),
])
def test_project_onto_cotangent_space_matches_oracle(cfg, kwargs):
    """systems.py:863-873 for all chains in one launch."""
    from oracle import mici_oracle as mo

    problem = problems.make_problem(cfg, **kwargs)
    system = engine.build_system(problem)
    rng = np.random.default_rng(3)
    mom = rng.standard_normal(problem.pos.shape)
    state = engine.build_state(problem, DEV)
    got = system.project_onto_cotangent_space(torch.as_tensor(mom, device=DEV), state).cpu().numpy()
    osys = mo.ConstrainedSystem(dr.build_target(problem), problem.metric)
    want = np.stack([osys.project_onto_cotangent_space(mom[i], problem.pos[i])
                     for i in range(problem.n_chains)])
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=ATOL)
    # the projected momentum is in the cotangent space: J M^-1 p = 0
    for i in range(0, problem.n_chains, 7):
        jac = osys.jacob_constr(problem.pos[i])
        resid = jac @ osys.inv_metric_mat(got[i][:, None])
        assert np.abs(resid).max() < 1e-12 * max(1.0, np.abs(mom[i]).max() * np.abs(jac).max())


@pytest.mark.parametrize("cfg,kwargs", [
    ("C2", {"n_chains": 40, "dim": 16}),
    ("C2", {"n_chains": 10, "dim": 64}),
    ("C4", {"n_chains": 40, "dim": 24}),
    ("C4", {"n_chains": 6, "dim": 128}),
])
def test_riemannian_sample_momentum_matches_oracle(cfg, kwargs):
    """sqrt(M(q)) z (systems.py:1401-1402): U sqrt(softabs) U^T z for SoftAbs, L z for dense."""
    problem = problems.make_problem(cfg, **kwargs)
    system = engine.build_system(problem)
    state = engine.build_state(problem, DEV)
    _, _, osys = dr.oracle_step_fn(problem)
    rngs = [np.random.default_rng([5, i]) for i in range(problem.n_chains)]
    got = system.sample_momentum(state, rngs).cpu().numpy()
    want = np.stack([osys.metric(problem.pos[i]).sqrt_matvec(
        np.random.default_rng([5, i]).normal(size=problem.dim)) for i in range(problem.n_chains)])
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-11)


def test_riemannian_sample_momentum_unavailable_in_low_rank_form():
    """The OPTIONAL Sherman-Morrison policy has no Cholesky factor of M(q); the default dense
    policy at D = 512 (global-workspace blocked Cholesky) samples like the oracle."""
    problem = problems.make_problem("C4", n_chains=4, dim=512)
    problem.metric_params = dict(problem.metric_params, force_low_rank_form=True)
    system = engine.build_system(problem)
    state = engine.build_state(problem, DEV)
    with pytest.raises(RuntimeError, match="does not fit"):
        system.sample_momentum(state, np.random.default_rng(0))


@pytest.mark.parametrize("cfg,kwargs", [
    ("C4", {"n_chains": 4, "dim": 512}),
    ("C5", {"n_chains": 5, "dim": 200}),
])
def test_global_dense_metric_momentum_velocity_and_energy_match_oracle(cfg, kwargs):
    """sqrt(M) z, M^-1 p and h through the global-workspace dense policy (D > 160)."""
    problem = problems.make_problem(cfg, **kwargs)
    system = engine.build_system(problem)
    state = engine.build_state(problem, DEV)
    _, h_fn, osys = dr.oracle_step_fn(problem)
    rngs = [np.random.default_rng([7, i]) for i in range(problem.n_chains)]
    got = system.sample_momentum(state, rngs).cpu().numpy()
    want = np.stack([osys.metric(problem.pos[i]).sqrt_matvec(
        np.random.default_rng([7, i]).normal(size=problem.dim)) for i in range(problem.n_chains)])
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-11)
    vel = system.dh_dmom(state).cpu().numpy()
    want_v = np.stack([osys.metric(problem.pos[i]).inv_matvec(problem.mom[i])
                       for i in range(problem.n_chains)])
    np.testing.assert_allclose(vel, want_v, rtol=1e-9, atol=1e-11)
    h = system.h(state).cpu().numpy()
    want_h = np.array([h_fn(problem.pos[i], problem.mom[i]) for i in range(problem.n_chains)])
    np.testing.assert_allclose(h, want_h, rtol=1e-10)


@pytest.mark.parametrize("dim", [5, 32, 33, 64, 100, 200, 512])
def test_blocked_dmma_cholesky_inverse_and_solve_match_numpy(dim):
    """csrc/dense_global.cuh on random SPD matrices: L, M^-1, M^-1 b and log|M| vs numpy.linalg
    (the arithmetic of DensePositiveDefiniteMatrix, matrices.py:1161-1188, 982-984)."""
    import ctypes

    from mici_b200 import _lib

    rng = np.random.default_rng(dim)
    n_mats = 6
    a = rng.standard_normal((n_mats, dim, dim))
    mats = a @ a.transpose(0, 2, 1) / dim + np.identity(dim)
    mats[-1] = mats[-1] - 3.0 * np.identity(dim)  # not positive definite: status 3
    rhs = rng.standard_normal((n_mats, dim))
    d_m = torch.as_tensor(mats, device=DEV).contiguous()
    d_b = torch.as_tensor(rhs, device=DEV).contiguous()
    chol = torch.zeros_like(d_m)
    inv = torch.zeros_like(d_m)
    sol = torch.zeros_like(d_b)
    logdet = torch.zeros(n_mats, dtype=torch.float64, device=DEV)
    status = torch.full((n_mats,), -1, dtype=torch.int32, device=DEV)
    rc = _lib.load().mb200_selftest_dense_factor(
        _lib.ptr(d_m), _lib.ptr(d_b), n_mats, dim, _lib.ptr(chol), _lib.ptr(inv), _lib.ptr(sol),
        _lib.ptr(logdet), _lib.ptr(status), _lib.current_stream_ptr(torch.device(DEV)))
    _lib.check(rc, "mb200_selftest_dense_factor")
    torch.cuda.synchronize()
    st = status.cpu().numpy()
    assert list(st[:-1]) == [0] * (n_mats - 1) and st[-1] == 3
    for i in range(n_mats - 1):
        want_l = np.linalg.cholesky(mats[i])
        np.testing.assert_allclose(chol[i].cpu().numpy(), want_l, rtol=1e-11, atol=1e-13)
        np.testing.assert_allclose(inv[i].cpu().numpy(), np.linalg.inv(mats[i]), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(sol[i].cpu().numpy(), np.linalg.solve(mats[i], rhs[i]),
                                   rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(float(logdet[i]), np.linalg.slogdet(mats[i])[1], rtol=1e-12)


ADAPT_NAMES = ["adapt_c1_dualavg_variance", "adapt_c1_dualavg_covariance", "adapt_c0_dualavg_min",
               "adapt_c0_variance_first", "adapt_c3_torus_dualavg", "adapt_c2_softabs_d6_dualavg",
               "adapt_nuts_c0_dualavg", "adapt_nuts_c1_dualavg_variance"]
NUTS_NAMES = ["nuts_c1_multinomial_d10", "nuts_c1_slice_euclidean_d16",
              "nuts_c0_depth4_no_extra_checks", "nuts_c1_diag_divergent", "nuts_c1_identity_d70",
              # constrained / implicit integrators: lock-step leaves + mb200_nuts_generic_* kernels
              "nuts_c3_torus_constrained", "nuts_c2_softabs_d4_implicit"]


def _dynamic_transition(integ, opts):
    from mici_b200 import transitions

    opts = dict(opts)
    cls = (transitions.SliceDynamicIntegrationTransition if opts.pop("variant", "multinomial") == "slice"
           else transitions.MultinomialDynamicIntegrationTransition)
    crit = getattr(transitions, opts.pop("criterion", "riemannian") + "_no_u_turn_criterion")
    return cls(integ.system, integ, termination_criterion=crit,
               do_extra_subtree_checks=opts.pop("extra_checks", True), **opts)


def _build_adapters(specs):
    from mici_b200 import adapters

    cls = {"dual_averaging": adapters.DualAveragingStepSizeAdapter,
           "online_variance": adapters.OnlineVarianceMetricAdapter,
           "online_covariance": adapters.OnlineCovarianceMetricAdapter}
    out = []
    for name, kw in specs:
        kw = dict(kw)
        if "log_step_size_reducer" in kw:
            kw["log_step_size_reducer"] = getattr(adapters, kw["log_step_size_reducer"])
        out.append(cls[name](**kw))
    return out


@pytest.mark.parametrize("name", ADAPT_NAMES)
def test_batched_adaptive_sampling_matches_reference_fixture(name):
    """Row N3 on the device: staged warm-up (windowed stager, per-chain dual-averaging step sizes
    through ``mb200_leapfrog_euclidean``'s ``step_sizes``, online variance / covariance metric
    adaptation, momentum resampling) + main stage, against the reference's own
    ``StaticMetropolisHMC.sample_chains`` -- every chain consuming its own NumPy stream.
    Discrete outcomes (trajectory lengths, accept / reject, directions) must agree exactly."""
    from golden_util import load_adapt_case
    from mici_b200 import stagers, transitions

    problem, specs, sk, n_warm, n_main, n_step, seed, _, g = load_adapt_case(name)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    base = np.random.default_rng(seed)
    stager = None if sk is None else stagers.WindowedWarmUpStager(**sk)
    # through the sampler front ends (reference call signature); the per-chain generators are
    # derived from the sampler's generator exactly as the reference derives them
    from mici_b200 import samplers

    if isinstance(n_step, dict):
        opts = dict(n_step)
        cls = (samplers.DynamicSliceHMC if opts.pop("variant", "multinomial") == "slice"
               else samplers.DynamicMultinomialHMC)
        crit = getattr(transitions, opts.pop("criterion", "riemannian") + "_no_u_turn_criterion")
        sampler = cls(integ.system, integ, base, termination_criterion=crit,
                      do_extra_subtree_checks=opts.pop("extra_checks", True), **opts)
    else:
        sampler = samplers.StaticMetropolisHMC(integ.system, integ, base, n_step)
    out = sampler.sample_chains(n_warm, n_main, state, adapters=_build_adapters(specs),
                                stager=stager, trace_warm_up=True, n_worker=1,
                                display_progress=False)
    final = out.final_states
    trace = out.traces["pos"].transpose(0, 1)
    stats = {k: v.transpose(0, 1) for k, v in out.statistics.items()}
    h_last = out.traces["hamiltonian"][:, -1]
    np.testing.assert_allclose(h_last.cpu().numpy(), integ.system.h(final).cpu().numpy(),
                               rtol=1e-12)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(stats["n_step"].cpu().numpy(), g["n_step"])
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["final_dir"])
    eps_trace, acc = stats["step_size"].cpu().numpy(), stats["accept_stat"].cpu().numpy()
    pos = trace.cpu().numpy()
    # the first transitions: plain parity
    k = 4
    np.testing.assert_allclose(eps_trace[:k], g["step_size_trace"][:k], rtol=1e-9)
    np.testing.assert_allclose(acc[:k], g["accept_stat"][:k], rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(pos[:k], g["pos"][:k], rtol=1e-8, atol=1e-10)
    # whole run: dual averaging deliberately probes step sizes far beyond the stability limit
    # early on (log step size regularised towards log(10 eps0)), where the leapfrog map
    # amplifies rounding differences by orders of magnitude per transition; measured deviation
    # over the 25-46 transitions is <= 1e-5 in positions / step sizes, 4e-5 absolute in accept_stat
    np.testing.assert_allclose(eps_trace, g["step_size_trace"], rtol=1e-3)
    np.testing.assert_allclose(acc, g["accept_stat"], rtol=1e-2, atol=1e-3)
    np.testing.assert_allclose(pos, g["pos"], rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(final.mom.cpu().numpy(), g["final_mom"], rtol=1e-3, atol=1e-4)
    assert isinstance(integ.step_size, float)
    assert integ.step_size == pytest.approx(float(g["step_size"]), rel=1e-4)
    if g["metric"].size:
        np.testing.assert_allclose(integ.system.metric.array, g["metric"], rtol=1e-4, atol=1e-8)


def test_per_chain_step_sizes_and_lengths_match_individual_launches():
    """``mb200_leapfrog_euclidean`` with per-chain step sizes and lengths: chain c with step size
    eps_c and n_c steps equals chain c of a plain launch with the scalar (eps_c, n_c) -- bit for
    bit on the same kernel."""
    problem = problems.make_problem("C1", n_chains=37, dim=48)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    rng = np.random.default_rng(9)
    eps = rng.uniform(0.005, 0.05, problem.n_chains)
    ns = rng.integers(0, 7, problem.n_chains).astype(np.int32)
    dirs = torch.as_tensor(rng.choice([-1, 1], problem.n_chains).astype(np.int32), device=DEV)
    state.dir = dirs
    integ.step_size = torch.as_tensor(eps, device=DEV)
    got = integ.step_n(state, torch.as_tensor(ns, device=DEV), return_h=True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.n_done.cpu().numpy(), ns)
    from oracle import mici_oracle as mo

    target, metric = dr.build_target(problem), mo.coerce_metric(problem.metric)
    for c in range(problem.n_chains):
        q, p = mo.leapfrog_steps(problem.pos[c], problem.mom[c], float(dirs[c]) * eps[c],
                                 int(ns[c]), target, metric)
        np.testing.assert_allclose(got.pos[c].cpu().numpy(), q, rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(got.mom[c].cpu().numpy(), p, rtol=RTOL, atol=ATOL)
        assert float(got.h[c]) == pytest.approx(mo.euclidean_h(q, p, target, metric), rel=1e-10)
    # composition integrators take the same per-chain arguments
    problem2 = problems.make_problem("C1", n_chains=9, dim=20, integrator="bcss3")
    integ2 = engine.build_integrator(problem2)
    st2 = engine.build_state(problem2, DEV)
    eps2 = np.linspace(0.01, 0.05, 9)
    integ2.step_size = torch.as_tensor(eps2, device=DEV)
    got2 = integ2.step_n(st2, 3)
    for c in (0, 4, 8):
        integ2.step_size = float(eps2[c])
        ref = integ2.step_n(engine.build_state(problem2, DEV, chains=slice(c, c + 1)), 3)
        assert torch.equal(got2.pos[c], ref.pos[0]) and torch.equal(got2.mom[c], ref.mom[0])
    # one scalar step size with per-chain lengths (no step-size array); a diagonal metric keeps
    # the single-chain launches on the same general-dimension kernel
    problem3 = problems.make_problem("C1", n_chains=11, dim=24, metric_kind="diagonal")
    integ3 = engine.build_integrator(problem3)
    st3 = engine.build_state(problem3, DEV)
    ns3 = rng.integers(0, 7, problem3.n_chains).astype(np.int32)
    dirs3 = torch.as_tensor(rng.choice([-1, 1], problem3.n_chains).astype(np.int32), device=DEV)
    st3.dir = dirs3
    got3 = integ3.step_n(st3, torch.as_tensor(ns3, device=DEV), return_h=True)
    np.testing.assert_array_equal(got3.n_done.cpu().numpy(), ns3)
    for c in range(problem3.n_chains):
        one = engine.build_state(problem3, DEV, chains=slice(c, c + 1))
        one.dir = dirs3[c:c + 1]
        ref = integ3.step_n(one, int(ns3[c]), return_h=True)
        assert torch.equal(got3.pos[c], ref.pos[0]) and torch.equal(got3.mom[c], ref.mom[0])
        assert torch.equal(got3.h[c], ref.h[0])


@pytest.mark.parametrize("dim, n_chains", [(48, 37), (128, 70)])
def test_per_chain_step_sizes_on_the_dmma_kernel(dim, n_chains):
    """Per-chain step sizes with ONE trajectory length stay on the DMMA kernel (K1, momentum
    tile scaled by eps_c): every chain equals the oracle's leapfrog with its own step size; a
    chain with eps_c = 0 does not move and gets the energy of its unmoved state."""
    problem = problems.make_problem("C1", n_chains=n_chains, dim=dim)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    rng = np.random.default_rng(11)
    eps = rng.uniform(0.005, 0.04, n_chains)
    eps[3] = 0.0
    dirs = torch.as_tensor(rng.choice([-1, 1], n_chains).astype(np.int32), device=DEV)
    state.dir = dirs
    integ.step_size = torch.as_tensor(eps, device=DEV)
    got = integ.step_n(state, 6, return_h=True)
    torch.cuda.synchronize()
    assert int((got.status != 0).sum()) == 0
    assert torch.equal(got.pos[3], state.pos[3]) and torch.equal(got.mom[3], state.mom[3])
    from oracle import mici_oracle as mo

    target, metric = dr.build_target(problem), mo.coerce_metric(problem.metric)
    for c in range(n_chains):
        q, p = mo.leapfrog_steps(problem.pos[c], problem.mom[c], float(dirs[c]) * eps[c], 6,
                                 target, metric)
        np.testing.assert_allclose(got.pos[c].cpu().numpy(), q, rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(got.mom[c].cpu().numpy(), p, rtol=RTOL, atol=ATOL)
        assert float(got.h[c]) == pytest.approx(mo.euclidean_h(q, p, target, metric), rel=1e-10)


@pytest.mark.parametrize("dim, offset", [(47, 0), (48, 1), (127, 1)])
def test_dmma_kernel_odd_dim_and_unaligned_state(dim, offset):
    """K1 with an odd dimension (phantom last coordinate, plain staging of the metric) and with
    state arrays that are only 8-byte aligned (scalar loads / stores): equals the oracle."""
    n_chains = 45
    problem = problems.make_problem("C1", n_chains=n_chains, dim=dim)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    if offset:
        for name in ("pos", "mom"):
            buf = torch.empty(n_chains * dim + offset, dtype=torch.float64, device=DEV)
            view = buf[offset:].view(n_chains, dim)
            view.copy_(getattr(state, name))
            setattr(state, name, view)
        assert state.pos.data_ptr() % 16 == 8
    got = integ.step_n(state, 5, return_h=True)
    torch.cuda.synchronize()
    from oracle import mici_oracle as mo

    target, metric = dr.build_target(problem), mo.coerce_metric(problem.metric)
    for c in range(0, n_chains, 4):
        q, p = mo.leapfrog_steps(problem.pos[c], problem.mom[c], float(integ.step_size), 5,
                                 target, metric)
        np.testing.assert_allclose(got.pos[c].cpu().numpy(), q, rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(got.mom[c].cpu().numpy(), p, rtol=RTOL, atol=ATOL)
        assert float(got.h[c]) == pytest.approx(mo.euclidean_h(q, p, target, metric), rel=1e-10)


def test_initial_step_size_search_matches_oracle():
    """DualAveragingStepSizeAdapter._find_and_set_init_step_size (adapters.py:285-352), all
    chains at once with per-chain halving / doubling."""
    import warnings

    from mici_b200 import adapters, transitions
    from oracle import mici_oracle as mo

    problem = problems.make_problem("C1", n_chains=64, dim=24)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    tr = transitions.MetropolisStaticIntegrationTransition(integ.system, integ, 1)
    got = adapters.DualAveragingStepSizeAdapter()._find_and_set_init_step_size(
        state, integ.system, integ).cpu().numpy()
    target, metric = dr.build_target(problem), mo.coerce_metric(problem.metric)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = np.array([
            mo.find_init_step_size(
                problem.pos[c], problem.mom[c], 1,
                lambda q, p, d, e: mo.leapfrog_steps(q, p, d * e, 1, target, metric),
                lambda q, p: mo.euclidean_h(q, p, target, metric))
            for c in range(problem.n_chains)])
    np.testing.assert_array_equal(got, want)
    assert tr.integrator.step_size is integ.step_size and len(set(got.tolist())) > 1


@pytest.mark.parametrize("metric_kind,dim", [("identity", 9), ("diagonal", 40), ("dense", 33)])
def test_gaussian_split_h2_flow_and_energy_match_oracle(metric_kind, dim):
    """GaussianEuclideanMetricSystem.h2_flow / h2 / h (systems.py:450-474) on their own."""
    from oracle import mici_oracle as mo

    problem = problems.make_problem("G1", n_chains=24, dim=dim if dim % 2 == 0 else dim + 1,
                                    metric_kind=metric_kind)
    system = engine.build_system(problem)
    metric = mo.coerce_metric(problem.metric)
    target = dr.build_target(problem)
    for dt in (0.3, -0.7):
        state = engine.build_state(problem, DEV)
        system.h2_flow(state, dt)
        for c in range(0, problem.n_chains, 5):
            q, p = mo.gaussian_h2_flow(problem.pos[c], problem.mom[c], dt, metric)
            np.testing.assert_allclose(state.pos[c].cpu().numpy(), q, rtol=RTOL, atol=ATOL)
            np.testing.assert_allclose(state.mom[c].cpu().numpy(), p, rtol=RTOL, atol=ATOL)
    state = engine.build_state(problem, DEV)
    h = system.h(state).cpu().numpy()
    h2 = system.h2(state).cpu().numpy()
    for c in range(0, problem.n_chains, 5):
        want = mo.gaussian_euclidean_h(problem.pos[c], problem.mom[c], target, metric)
        assert h[c] == pytest.approx(want, rel=1e-11)
        assert h2[c] == pytest.approx(want - target.neg_log_dens(problem.pos[c]), rel=1e-10)


@pytest.mark.parametrize("cfg,kwargs", [
    ("C3", {"n_chains": 40}),
    ("S1", {"n_chains": 12, "dim": 20, "metric_kind": "dense"}),
    ("C2", {"n_chains": 10, "dim": 8}),
    ("C4", {"n_chains": 8, "dim": 16}),
    ("C2", {"n_chains": 6, "dim": 8, "integrator": "implicit_midpoint"}),
])
def test_per_chain_launch_of_implicit_and_constrained_integrators(cfg, kwargs):
    """Per-chain step sizes and lengths: chain c with (eps_c, n_c) equals chain c of a scalar
    launch with that step size and length -- bit for bit, status and iteration counts included
    (large step sizes make some chains fail)."""
    problem = problems.make_problem(cfg, **kwargs)
    integ = engine.build_integrator(problem)
    n = problem.n_chains
    rng = np.random.default_rng(12)
    eps = problem.step_size * rng.choice([0.5, 1.0, 2.0, 6.0], n)
    ns = rng.integers(0, 4, n).astype(np.int32)
    dirs = torch.as_tensor(rng.choice([-1, 1], n).astype(np.int32), device=DEV)
    state = engine.build_state(problem, DEV)
    state.dir = dirs
    integ.step_size = torch.as_tensor(eps, device=DEV)
    got = integ.step_n(state, torch.as_tensor(ns, device=DEV), return_h=True)
    torch.cuda.synchronize()
    n_failed = 0
    for c in range(n):
        integ.step_size = float(eps[c])
        one = engine.build_state(problem, DEV, chains=slice(c, c + 1))
        one.dir = dirs[c:c + 1]
        ref = integ.step_n(one, int(ns[c]), return_h=True)
        assert int(got.status[c]) == int(ref.status[0]) and int(got.n_done[c]) == int(ref.n_done[0])
        assert torch.equal(got.pos[c], ref.pos[0]) and torch.equal(got.mom[c], ref.mom[0])
        assert torch.equal(got.h[c], ref.h[0]) or (torch.isnan(got.h[c]) and torch.isnan(ref.h[0]))
        assert torch.equal(got.solver_iters[c], ref.solver_iters[0])
        n_failed += int(ref.status[0] != 0)
    assert n_failed < n


@pytest.mark.parametrize("cfg,kwargs", [("C3", {"n_chains": 48}), ("C2", {"n_chains": 12, "dim": 6})])
def test_initial_step_size_search_with_failing_steps_matches_oracle(cfg, kwargs):
    """adapters.py:285-352 including the ``except IntegratorError`` branch (:338-340): at step
    size 1 most constrained / implicit steps fail, each chain halves on its own."""
    import warnings

    from mici_b200 import adapters
    from oracle import mici_oracle as mo

    problem = problems.make_problem(cfg, **kwargs)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    got = adapters.DualAveragingStepSizeAdapter()._find_and_set_init_step_size(
        state, integ.system, integ).cpu().numpy()
    ctx = dr._AdaptiveContext(problem)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = np.array([mo.find_init_step_size(problem.pos[c], problem.mom[c], 1, ctx.step_eps,
                                                ctx.h) for c in range(problem.n_chains)])
    # a failure / success decision right at a solver threshold may differ for isolated chains
    # (ill-conditioned: see the *bigstep fixtures); the search then ends one halving apart
    differs = got != want
    assert differs.mean() <= 0.05, (got, want)
    assert np.all((got[differs] == want[differs] / 2) | (got[differs] == want[differs] * 2))
    assert (got < 1).any()


@pytest.mark.parametrize("name", NUTS_NAMES)
def test_dynamic_transition_matches_reference_fixture(name):
    """Row N4 on the device: whole NUTS transitions (tree doubling, multinomial / slice
    progressive sampling, no-U-turn checks, divergence test) in one launch, one warp per chain,
    against the reference's own transition classes; every chain consumes exactly the uniforms
    its NumPy generator would have produced for it."""
    from golden_util import load_nuts_case
    from mici_b200 import transitions

    problem, n_iter, seed, opts, g = load_nuts_case(name)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([seed, i]) for i in range(problem.n_chains)]
    final, stats, trace = transitions.sample_chains(
        integ.system, integ, state, rngs, 0, n_iter,
        integration_transition=_dynamic_transition(integ, opts))
    torch.cuda.synchronize()
    for k in ("n_step", "tree_depth", "diverging", "convergence_error", "non_reversible_step"):
        if k in g:
            np.testing.assert_array_equal(stats[k].cpu().numpy().astype(np.float64), g[k],
                                          err_msg=k)
    np.testing.assert_array_equal(final.dir.cpu().numpy(), g["dir"][-1])
    np.testing.assert_allclose(trace.cpu().numpy(), g["pos"], rtol=1e-8, atol=1e-10)
    for k in ("av_metrop_accept_prob", "accept_stat", "reject_prob"):
        np.testing.assert_allclose(stats[k].cpu().numpy(), g[k], rtol=1e-7, atol=1e-10, err_msg=k)
    # the generators were advanced by exactly what the reference consumes: replay the chains
    # through the oracle on fresh generators and compare the next draw of every stream
    import warnings

    from oracle import mici_oracle as mo

    step, h_fn, system = dr.oracle_step_fn(problem)
    sample_mom, vel = dr._sample_momentum(problem, system), dr._velocity_fn(problem, system)
    for i in range(problem.n_chains):
        g_ref = np.random.default_rng([seed, i])
        q = problem.pos[i].copy()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for _ in range(n_iter):
                q, _, _ = mo.nuts_transition(q, sample_mom(q, g_ref), g_ref.uniform, step, h_fn,
                                             vel, **opts)
        assert rngs[i].uniform() == g_ref.uniform()


@pytest.mark.parametrize("cfg,kwargs,eps,opts", [
    ("C1", {"n_chains": 24, "dim": 16}, 0.15, {}),
    ("C1", {"n_chains": 16, "dim": 70, "metric_kind": "diagonal"}, 0.2,
     {"variant": "slice", "criterion": "euclidean", "max_tree_depth": 6}),
])
def test_generic_dynamic_transition_equals_fused_kernel(cfg, kwargs, eps, opts):
    """The lock-step generic path (batched steps + bookkeeping kernels) and the fused one-launch
    kernel are two implementations of the same transition: identical discrete outcomes and
    uniform consumption, states equal to rounding, on a Euclidean system where both apply."""
    problem = problems.make_problem(cfg, **kwargs)
    problem.step_size = eps
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    out = []
    for fused in (True, False):
        tr = _dynamic_transition(integ, opts)
        tr._fused = fused
        rngs = [np.random.default_rng([91, i]) for i in range(problem.n_chains)]
        st = state
        for _ in range(3):
            st, stats = tr.sample(st, rngs)
        out.append((st, stats, [r.uniform() for r in rngs]))
    (a, sa, ua), (b, sb, ub) = out
    for k in ("n_step", "tree_depth", "diverging"):
        assert torch.equal(sa[k], sb[k]), k
    assert ua == ub
    assert torch.equal(a.dir, b.dir)
    np.testing.assert_allclose(b.pos.cpu().numpy(), a.pos.cpu().numpy(), rtol=1e-9, atol=1e-11)


def test_dynamic_transition_full_size_device_rng():
    """8192 chains x D=128 with device-generated uniforms: finite states, sane statistics."""
    from mici_b200 import transitions

    problem = problems.make_problem("C1")
    problem.step_size = 0.05
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    tr = transitions.MultinomialDynamicIntegrationTransition(integ.system, integ, max_tree_depth=6)
    final, stats, _ = transitions.sample_chains(integ.system, integ, state, gen, 0, 3,
                                                integration_transition=tr, trace_pos=False)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(final.pos).all()) and bool(torch.isfinite(final.mom).all())
    assert int(stats["n_step"].min()) >= 1 and int(stats["tree_depth"].max()) <= 5
    assert 0.3 < float(stats["accept_stat"].mean()) <= 1.0
    assert not bool(stats["diverging"].any())


def _nuts_setup(cfg, kwargs, seed=3046987125):
    from mici_b200 import transitions

    problem = problems.make_problem(cfg, **kwargs)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(seed % (2**31))
    tr = transitions.MultinomialDynamicIntegrationTransition(integ.system, integ)
    return problem, integ, state, gen, tr, transitions.IndependentMomentumTransition(integ.system)


def test_dual_averaging_controls_accept_statistic():
    """Mirror of the reference's ``DualAveragingStepSizeAdapterTests.test_adaptation``
    (reference tests/test_adapters.py:102-128): 500 adaptive dynamic transitions on a standard
    Gaussian, then 500 with the finalised step size -- here for 32 chains at once, each with its
    own step size while adapting."""
    from mici_b200 import adapters

    problem, integ, state, gen, tr, mom_tr = _nuts_setup("C0", {"n_chains": 32, "dim": 10})
    integ.step_size = None
    adapter = adapters.DualAveragingStepSizeAdapter()
    a_state = adapter.initialize(state, tr)
    assert integ.step_size.shape == (32,)
    for _ in range(500):
        state, _ = mom_tr.sample(state, gen)
        state, stats = tr.sample(state, gen)
        adapter.update(a_state, state, stats, tr)
    adapter.finalize(a_state, state, tr, gen)
    err = a_state["adapt_stat_error"].abs().cpu().numpy()
    assert err.mean() < 0.02 and err.max() < 0.1
    assert isinstance(integ.step_size, float) and 0.1 < integ.step_size < 3.0
    total = 0.0
    for _ in range(500):
        state, _ = mom_tr.sample(state, gen)
        state, stats = tr.sample(state, gen)
        total += float(stats["accept_stat"].mean())
    assert abs(adapter.adapt_stat_target - total / 500) < 0.05


@pytest.mark.parametrize("kind", ["variance", "covariance"])
def test_metric_adapters_match_direct_estimates(kind):
    """Mirror of the reference's ``TestOnlineVarianceMetricAdapter`` /
    ``TestOnlineCovarianceMetricAdapter`` (reference tests/test_adapters.py:212-300): Welford
    states after 10 dynamic transitions and the finalised metric against NumPy estimates from
    the recorded samples -- pooled over all chains, which is what the chain-by-chain merge of the
    reference (adapters.py:487-505, 615-634) computes."""
    from mici_b200 import adapters

    problem, integ, state, gen, tr, mom_tr = _nuts_setup(
        "C1", {"n_chains": 24, "dim": 10, "metric_kind": "identity"})
    integ.step_size = 0.2
    adapter = (adapters.OnlineVarianceMetricAdapter() if kind == "variance"
               else adapters.OnlineCovarianceMetricAdapter())
    a_state = adapter.initialize(state, tr)
    samples = []
    for _ in range(10):
        state, _ = mom_tr.sample(state, gen)
        state, stats = tr.sample(state, gen)
        samples.append(state.pos.cpu().numpy().copy())
        adapter.update(a_state, state, stats, tr)
    samples = np.stack(samples)  # [10, n_chains, dim]
    assert a_state["iter"] == 10
    np.testing.assert_allclose(a_state["mean"].cpu().numpy(), samples.mean(0), rtol=1e-10, atol=1e-13)
    centred = samples - samples.mean(0)
    if kind == "variance":
        np.testing.assert_allclose(a_state["sum_diff_sq"].cpu().numpy(), (centred**2).sum(0),
                                   rtol=1e-9, atol=1e-12)
    else:
        np.testing.assert_allclose(a_state["sum_diff_outer"].cpu().numpy(),
                                   np.einsum("tcj,tck->jk", centred, centred), rtol=1e-9, atol=1e-11)
    adapter.finalize(a_state, state, tr, gen)
    flat = samples.reshape(-1, problem.dim)
    n = flat.shape[0]
    weight = n / (adapter.reg_iter_offset + n)
    metric = integ.system.metric
    if kind == "variance":
        reg = weight * flat.var(axis=0, ddof=1) + (1 - weight) * adapter.reg_scale
        assert metric.kind == 1
        np.testing.assert_allclose(metric.array, 1 / reg, rtol=1e-9)
    else:
        reg = weight * np.cov(flat, rowvar=False, ddof=1) + (
            1 - weight) * adapter.reg_scale * np.identity(problem.dim)
        assert metric.kind == 2
        np.testing.assert_allclose(metric.inv, reg, rtol=1e-8, atol=1e-12)
    assert bool(torch.isfinite(state.mom).all())  # momenta resampled under the new metric


def test_correlated_momentum_transition():
    """transitions.py:145-198: partial refresh with the variates of each chain's own stream."""
    from mici_b200 import transitions
    from oracle import mici_oracle as mo

    problem = problems.make_problem("C1", n_chains=6, dim=8)
    system = engine.build_system(problem)
    state = engine.build_state(problem, DEV)
    rngs = [np.random.default_rng([3, i]) for i in range(problem.n_chains)]
    coeff = 0.4
    new, stats = transitions.CorrelatedMomentumTransition(system, coeff).sample(state, rngs)
    assert stats is None
    metric = mo.coerce_metric(problem.metric)
    for i in range(problem.n_chains):
        ind = metric.sqrt_matvec(np.random.default_rng([3, i]).standard_normal(problem.dim))
        want = problem.mom[i] * (1.0 - coeff**2) ** 0.5 + coeff * ind
        np.testing.assert_allclose(new.mom[i].cpu().numpy(), want, rtol=1e-12, atol=1e-14)
    with pytest.raises(ValueError):
        transitions.CorrelatedMomentumTransition(system, 1.5)
