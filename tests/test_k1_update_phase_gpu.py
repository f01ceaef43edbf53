"""The tensor-core leapfrog kernel (K1) on batches whose last CTA mixes groups of one and two row
tiles and ends in a partially live tile, at every dimension class of the kernel, with one shared
step size and with per-chain step sizes.  These shapes exercise the update phase's per-chain
scalar (the funnel's exp(-v), evaluated for all of a group's chains in one pass of the warp that
holds coordinate 0) and its reductions for every tile count."""

import ctypes

import numpy as np
import pytest
import torch

from mici_b200 import _lib, engine, integrators, problems

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# K1 gives a CTA up to 8 row tiles of 8 chains and spreads them over the SMs (132 on an H100 SXM):
#   8236 chains = 1030 tiles: 128 CTAs of 8 tiles, the last CTA 6 tiles (groups of 2, 2, 1 and 1
#                 tiles), the last tile holds 4 live chains;
#   1100 chains = 138 tiles: 69 CTAs of 2 tiles (groups of one tile), the last tile 4 live chains.
BATCHES = [8236, 1100]
DIMS = [32, 64, 96, 128]


def _setup(n_chains, dim, per_chain):
    problem = problems.make_problem("C1", n_chains=n_chains, dim=dim)
    system = engine.build_system(problem)
    if per_chain:
        rng = np.random.default_rng(20261015 + dim)
        step = torch.as_tensor(problem.step_size * rng.uniform(0.5, 1.5, n_chains),
                               dtype=torch.float64, device=DEV)
    else:
        step = problem.step_size
    integ = integrators.LeapfrogIntegrator(system, step)
    dirs = np.where(np.arange(n_chains) % 3 == 0, -1, 1).astype(np.int32)
    state = engine.build_state(problem, DEV, dirs=dirs)
    return problem, integ, state, step


@pytest.mark.parametrize("per_chain", [False, True], ids=["shared_eps", "per_chain_eps"])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("n_chains", BATCHES)
def test_k1_agrees_with_generic_kernel(n_chains, dim, per_chain):
    """K1 against the general-dimension kernel K1g (same C ABI, tolerances of
    test_dmma_and_generic_leapfrog_kernels_agree)."""
    problem, integ, state, step = _setup(n_chains, dim, per_chain)
    n_steps = 10
    fast = integ.step_n(state, n_steps, return_h=True)
    sysm = integ.system
    n = state.pos.shape[0]
    model = sysm._model(state.pos.device)
    q, p = torch.empty_like(state.pos), torch.empty_like(state.mom)
    h = torch.empty(n, dtype=torch.float64, device=DEV)
    eps, eps_t = (0.0, step) if per_chain else (step, None)
    rc = _lib.load().mb200_leapfrog_euclidean_generic(
        _lib.ptr(state.pos), _lib.ptr(state.mom), _lib.ptr(q), _lib.ptr(p), _lib.ptr(state.dir),
        n, dim, eps, _lib.ptr(eps_t), n_steps, None, 0, None, 0, sysm.metric.kind,
        _lib.ptr(sysm.metric.inv_device(state.pos.device)),
        ctypes.byref(model), _lib.ptr(h), None, None, _lib.current_stream_ptr(state.pos.device))
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.isfinite(fast.pos).all() and torch.isfinite(fast.mom).all()
    torch.testing.assert_close(fast.pos, q, rtol=1e-11, atol=1e-13)
    torch.testing.assert_close(fast.mom, p, rtol=1e-11, atol=1e-13)
    torch.testing.assert_close(fast.h, h, rtol=1e-11, atol=1e-10)


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("n_chains", BATCHES)
def test_k1_step_n_equals_repeated_step(n_chains, dim):
    """One fused launch of k steps equals k launches of one step, bit for bit: the two half-kicks
    at a step boundary stay two separately rounded updates.  (With per-chain step sizes the kernel
    carries eps_c * p and divides by eps_c on the way out, so launch boundaries round there.)"""
    _, integ, state, _ = _setup(n_chains, dim, False)
    k = 5
    fused = integ.step_n(state, k)
    s = state
    for _ in range(k):
        s = integ.step(s)
    torch.cuda.synchronize()
    assert torch.equal(fused.pos, s.pos) and torch.equal(fused.mom, s.mom)
