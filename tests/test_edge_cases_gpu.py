"""GPU edge cases of the boundary: empty / ragged batches, minimum and maximum dimensions,
batches larger than one wave of CTAs, aliasing outputs, scalar directions -- all against the
oracle port on the same inputs."""

import ctypes

import numpy as np
import pytest
import torch

from mici_b200 import ChainState, _lib, engine, problems
from mici_b200.errors import Error
from oracle import drivers as dr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RTOL, ATOL = 1e-10, 1e-12


def _check(problem, n_steps, dirs=None, chains=None):
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV, dirs=dirs)
    out = integ.step_n(state, n_steps, return_h=True)
    torch.cuda.synchronize()
    sl = slice(None) if chains is None else chains
    ref = dr.oracle_run(problem, n_steps, dirs=None if dirs is None else np.asarray(dirs)[sl], chains=sl)
    np.testing.assert_array_equal(out.status.cpu().numpy()[sl], ref["status"])
    np.testing.assert_allclose(out.pos.cpu().numpy()[sl], ref["pos"], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(out.mom.cpu().numpy()[sl], ref["mom"], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(out.h.cpu().numpy()[sl], ref["h"], rtol=RTOL, atol=1e-9)
    return out


@pytest.mark.parametrize("cfg", ["C1", "C2", "C3", "C4"])
def test_empty_batch(cfg):
    kw = {"C1": {"dim": 16}, "C2": {"dim": 8}, "C3": {}, "C4": {"dim": 16}}[cfg]
    problem = problems.make_problem(cfg, n_chains=4, **kw)
    integ = engine.build_integrator(problem)
    dim = problem.dim
    state = ChainState(pos=torch.empty((0, dim), dtype=torch.float64, device=DEV),
                       mom=torch.empty((0, dim), dtype=torch.float64, device=DEV), dir=1)
    out = integ.step_n(state, 3, return_h=True)
    assert out.pos.shape == (0, dim) and out.status.shape == (0,)


@pytest.mark.parametrize("n_chains", [1, 7, 8, 9, 55, 56, 57, 63, 64, 65, 113, 129])
def test_ragged_batches_dense_leapfrog(n_chains):
    """Row tiles of 8 chains and CTAs of 64: every partial-tile / partial-CTA shape."""
    problem = problems.make_problem("C1", n_chains=n_chains, dim=32)
    dirs = np.where(np.arange(n_chains) % 3 == 0, -1, 1).astype(np.int32)
    _check(problem, 4, dirs=dirs)


def test_more_chains_than_one_wave_of_ctas():
    """n > 132 * 64 chains (H100 SXM: 132 SMs): the persistent CTAs loop over a second block."""
    n = 132 * 64 + 61
    problem = problems.make_problem("C1", n_chains=n, dim=16)
    chains = np.r_[0:8, 64 * 131 : 64 * 131 + 8, 132 * 64 - 3 : n]  # first, last-of-wave, second pass
    out = _check(problem, 3, chains=chains)
    assert bool(torch.isfinite(out.pos).all()) and int(out.n_done.min()) == 3


@pytest.mark.parametrize("dim,metric_kind", [
    (1, "dense"), (2, "dense"), (3, "diagonal"), (8, "dense"), (126, "dense"), (128, "dense"),
    (129, "dense"), (127, "identity"), (512, "diagonal"), (1024, "identity"),
])
def test_dimension_range_euclidean(dim, metric_kind):
    problem = problems.make_problem("C1", n_chains=5, dim=dim, metric_kind=metric_kind)
    _check(problem, 2)


def test_dimension_above_maximum_is_rejected():
    problem = problems.make_problem("C1", n_chains=2, dim=1025, metric_kind="identity")
    integ = engine.build_integrator(problem)
    with pytest.raises(Error, match="1024"):
        integ.step(engine.build_state(problem, DEV))


def test_scalar_negative_direction_and_single_chain_state():
    problem = problems.make_problem("C1", n_chains=6, dim=24)
    integ = engine.build_integrator(problem)
    st = ChainState(pos=torch.as_tensor(problem.pos, device=DEV),
                    mom=torch.as_tensor(problem.mom, device=DEV), dir=-1)
    out = integ.step_n(st, 5)
    ref = dr.oracle_run(problem, 5, dirs=-np.ones(6, dtype=np.int32))
    np.testing.assert_allclose(out.pos.cpu().numpy(), ref["pos"], rtol=RTOL, atol=ATOL)
    one = ChainState(pos=torch.as_tensor(problem.pos[2], device=DEV),
                     mom=torch.as_tensor(problem.mom[2], device=DEV), dir=-1)
    new = integ.step_n(one, 5)
    assert new.pos.shape == (24,)
    np.testing.assert_allclose(new.pos.cpu().numpy(), ref["pos"][2], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("cfg,kw,entry", [
    ("C1", {"n_chains": 70, "dim": 64}, "leapfrog"),
    ("C1", {"n_chains": 9, "dim": 11}, "leapfrog"),
])
def test_leapfrog_outputs_may_alias_inputs(cfg, kw, entry):
    """include/mici_b200.h: `*_out` may alias `*_in` (in-place update)."""
    problem = problems.make_problem(cfg, **kw)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    ref = integ.step_n(state, 3)
    pos, mom = state.pos.clone(), state.mom.clone()
    sysm = integ.system
    model = sysm._model(pos.device)
    rc = _lib.load().mb200_leapfrog_euclidean(
        _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(pos), _lib.ptr(mom), None, pos.shape[0],
        pos.shape[1], problem.step_size, None, 3, None, 0, None, 0, sysm.metric.kind,
        _lib.ptr(sysm.metric.inv_device(pos.device)), ctypes.byref(model), None, None, None,
        _lib.current_stream_ptr(pos.device))
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(pos, ref.pos) and torch.equal(mom, ref.mom)


def test_invalid_leapfrog_arguments_return_errors_not_crashes():
    lib = _lib.load()
    problem = problems.make_problem("C1", n_chains=4, dim=8)
    integ = engine.build_integrator(problem)
    state = engine.build_state(problem, DEV)
    model = integ.system._model(state.pos.device)
    args = lambda **o: [  # noqa: E731
        _lib.ptr(state.pos), _lib.ptr(state.mom), _lib.ptr(state.pos), _lib.ptr(state.mom), None,
        o.get("n", 4), o.get("dim", 8), 0.1, None, o.get("n_steps", 1), None, 0, None, 0,
        o.get("kind", 2),
        o.get("minv", _lib.ptr(integ.system.metric.inv_device(state.pos.device))),
        ctypes.byref(model), None, None, None, _lib.current_stream_ptr(state.pos.device)]
    assert lib.mb200_leapfrog_euclidean(*args(n=-1)) == -1
    assert lib.mb200_leapfrog_euclidean(*args(dim=0)) == -1
    assert lib.mb200_leapfrog_euclidean(*args(n_steps=-2)) == -1
    assert lib.mb200_leapfrog_euclidean(*args(kind=7)) == -1
    assert lib.mb200_leapfrog_euclidean(*args(minv=None)) == -1
    assert b"metric_inv" in lib.mb200_last_error()
    model.target_id = 99
    assert lib.mb200_leapfrog_euclidean(*args()) == -2


def test_non_finite_inputs_propagate_like_numpy():
    """The explicit leapfrog never raises in the reference: NaN / inf simply propagate."""
    problem = problems.make_problem("C1", n_chains=16, dim=32)
    problem.pos[3, 5] = np.nan
    problem.mom[9, 0] = np.inf
    integ = engine.build_integrator(problem)
    out = integ.step_n(engine.build_state(problem, DEV), 2)
    ref = dr.oracle_run(problem, 2)
    got = out.pos.cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(ref["pos"]))
    ok = np.isfinite(ref["pos"]).all(1)
    np.testing.assert_allclose(got[ok], ref["pos"][ok], rtol=RTOL, atol=ATOL)
    assert (out.status == 0).all()


def test_numpy_chain_state_in_numpy_out():
    """A state holding NumPy arrays (the reference's own ChainState storage) steps through the
    same kernels and comes back as NumPy; a 1-D state raises the reference exceptions."""
    problem = problems.make_problem("C1", n_chains=5, dim=24)
    integ = engine.build_integrator(problem)
    st = ChainState(pos=problem.pos[1].copy(), mom=problem.mom[1].copy(), dir=1)
    new = integ.step(st)
    assert isinstance(new.pos, np.ndarray) and new.pos.shape == (24,)
    ref = dr.oracle_run(problem, 1)
    np.testing.assert_allclose(new.pos, ref["pos"][1], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(new.mom, ref["mom"][1], rtol=RTOL, atol=ATOL)
    np.testing.assert_array_equal(st.pos, problem.pos[1])  # argument untouched
    h = integ.system.h(new)
    np.testing.assert_allclose(h, ref["h"][1], rtol=RTOL)

    class ForeignState:  # duck-typed stand-in for mici.states.ChainState
        def __init__(self, pos, mom, dir):  # noqa: A002
            self.pos, self.mom, self.dir = pos, mom, dir

        def copy(self):
            return ForeignState(self.pos.copy(), self.mom.copy(), self.dir)

        def __contains__(self, name):
            return name in ("pos", "mom", "dir")

    fs = ForeignState(problem.pos[2].copy(), problem.mom[2].copy(), -1)
    out = integ.step(fs)
    assert isinstance(out, ForeignState) and out.dir == -1
    ref2 = dr.oracle_run(problem, 1, dirs=-np.ones(5, dtype=np.int32))
    np.testing.assert_allclose(out.pos, ref2["pos"][2], rtol=RTOL, atol=ATOL)


def test_trace_write_out_from_device_buffers_reference_file_layout(tmp_path):
    """Row N2 on the GPU: per-iteration traces of a batched HMC run live in device buffers
    ``[n_iter, n_chains, ...]`` and are written as the reference's per-chain memory-mappable
    ``{prefix}_{index}_{key}.npy`` files (samplers.py:104-138); reading them back the way
    ``interop.convert_to_inference_data`` does (interop.py:54-96: ``np.load(..., mmap_mode)``)
    returns the traced positions."""
    from mici_b200 import traces, transitions

    prob = problems.make_problem("C1", n_chains=24, dim=16)
    integ = engine.build_integrator(prob)
    state = engine.build_state(prob, "cuda:0")
    n_iter = 5
    buf = traces.TraceBuffer(n_iter, prob.n_chains, (prob.dim,), device="cuda:0")
    hbuf = traces.TraceBuffer(n_iter, prob.n_chains, (), device="cuda:0")
    gen = torch.Generator(device="cuda:0")
    gen.manual_seed(3)
    mom_tr = transitions.IndependentMomentumTransition(integ.system)
    int_tr = transitions.MetropolisStaticIntegrationTransition(integ.system, integ, n_step=4)
    for _ in range(n_iter):
        state, _ = mom_tr.sample(state, gen)
        state, stats = int_tr.sample(state, gen)
        buf.append(state.pos)
        hbuf.append(integ.system.h(state))
    gathered = traces.gather_traces({"pos": buf.data, "hamiltonian": hbuf.data}, prob.n_chains)
    paths = traces.write_chain_traces(tmp_path, "trace", gathered)
    assert len(paths["pos"]) == prob.n_chains
    assert paths["pos"][3].name == "trace_3_pos.npy"
    for i in (0, 7, 23):
        mm = np.load(paths["pos"][i], mmap_mode="r")
        assert mm.shape == (n_iter, prob.dim)
        np.testing.assert_array_equal(np.asarray(mm), buf.data[:, i].cpu().numpy())
        hm = np.load(paths["hamiltonian"][i], mmap_mode="r")
        np.testing.assert_array_equal(np.asarray(hm), hbuf.data[:, i].cpu().numpy())


def test_kernel_side_call_counters():
    """``mb200_set_call_counters``: per-chain tallies written by the kernels themselves."""
    # K1 (tensor-core leapfrog): one gradient per step plus the initial one
    prob = problems.make_problem("C1", n_chains=19, dim=32)
    integ = engine.build_integrator(prob).count_calls()
    state = engine.build_state(prob, DEV)
    integ.step_n(state, 5)
    integ.step_n(state, 2)
    c = integ.call_counts.cpu().numpy()
    assert (c[:, 0] == 6 + 3).all() and (c[:, 1:] == 0).all()
    assert integ.call_count_totals()["grad_neg_log_dens"] == 19 * 9
    # three-stage composition on the general kernel: one gradient per drift
    prob = problems.make_problem("C1", n_chains=5, dim=20, integrator="bcss3")
    integ = engine.build_integrator(prob).count_calls()
    integ.step_n(engine.build_state(prob, DEV), 4)
    got = integ.call_counts.cpu().numpy()[:, 0]
    assert (got == 1 + 4 * 3).all()  # flows a b a b a b a: three drifts per step
    # implicit leapfrog (SoftAbs): builds / VJPs follow the fixed-point iteration counts
    prob = problems.make_problem("C2", n_chains=6, dim=8)
    integ = engine.build_integrator(prob).count_calls()
    out = integ.step_n(engine.build_state(prob, DEV), 1)
    it = out.solver_iters.cpu().numpy()
    c = integ.call_counts.cpu().numpy()
    ok = out.status.cpu().numpy() == 0
    assert ok.all()
    np.testing.assert_array_equal(c[:, 3], it.sum(1))
    np.testing.assert_array_equal(c[:, 1], it[:, 1] + it[:, 2] + 2)  # metric builds
    np.testing.assert_array_equal(c[:, 2], it[:, 0] + it[:, 3] + 1)  # quadratic-form VJPs
    np.testing.assert_array_equal(c[:, 0], 2)
    # constrained leapfrog: 3 projections + 2 retractions per step, one Jacobian per Newton
    # iteration; the thread-per-chain torus kernel and the warp kernel (sphere) count alike
    for cfg, kw in (("C3", dict(n_chains=40)), ("S1", dict(n_chains=9, dim=10))):
        prob = problems.make_problem(cfg, **kw)
        integ = engine.build_integrator(prob).count_calls()
        out = integ.step_n(engine.build_state(prob, DEV), 3)
        assert int((out.status != 0).sum()) == 0
        c = integ.call_counts.cpu().numpy()
        it = out.solver_iters.cpu().numpy().reshape(-1)
        np.testing.assert_array_equal(c[:, 3], it)
        np.testing.assert_array_equal(c[:, 1], 5 * 3 + it)
        np.testing.assert_array_equal(c[:, 0], 4)
    # switched off again: later launches leave the tally alone
    integ.count_calls(False)
    integ.step_n(engine.build_state(prob, DEV), 1)
    assert integ.call_counts is None
