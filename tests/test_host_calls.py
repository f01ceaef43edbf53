"""Every host-side library call of the systems, integrators and transitions, pinned.

``_lib.load`` is replaced by a recording fake that never launches anything, the stream by a
constant, and ``CudaTarget.handle`` by a sentinel pointer, so no kernel runs and nothing is
compiled.  Each case records, per C call: the symbol, every scalar, the ``mb200_model`` and
``mb200_nuts_options`` fields, and for every pointer whether it is NULL, which named tensor it
points to, or a buffer the host path allocated itself (``new``).  Where the host reads an output
back (status, active, flags, uniforms used) the fake writes fixed values through the pointer:
every chain succeeds, every lock-step tree stays active, and every chain uses 3 uniforms.

Without a GPU the cases run on CPU tensors.  The cases that need a CUDA device (NumPy states,
cotangent projections, Riemannian momentum draws, host-buffer stepping) run where one exists;
they launch nothing either.
"""

from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from mici_b200 import _lib, integrators, systems, targets, transitions
from mici_b200.solvers import (
    solve_fixed_point_steffensen,
    solve_projection_onto_manifold_newton_with_line_search,
    solve_projection_onto_manifold_quasi_newton,
)
from mici_b200.states import ChainState

STREAM = 0x5EA
USER = 0xC0DE
N, DIM = 3, 4
WS_BYTES = 4096

# symbol -> (index of n_chains, {index of an int32 [n] output the host reads: value})
_OUTPUTS = {
    "mb200_leapfrog_euclidean": (5, {18: 0}),
    "mb200_leapfrog_euclidean_user": (5, {18: 0}),
    "mb200_leapfrog_gaussian_euclidean": (5, {18: 0}),
    "mb200_constrained_leapfrog_euclidean": (5, {23: 0}),
    "mb200_constrained_leapfrog_euclidean_user": (5, {23: 0}),
    "mb200_constrained_leapfrog_gaussian_euclidean": (5, {26: 0}),
    "mb200_constrained_leapfrog_gaussian_euclidean_user": (5, {26: 0}),
    "mb200_implicit_leapfrog_riemannian": (5, {18: 0}),
    "mb200_implicit_midpoint_riemannian": (5, {18: 0}),
    "mb200_hamiltonian_riemannian": (2, {6: 0}),
    "mb200_dh_dmom_riemannian": (3, {6: 0}),
    "mb200_sample_momentum_riemannian": (3, {6: 0}),
    "mb200_nuts_euclidean": (4, {25: 0, 26: 3, 28: 0}),
    "mb200_nuts_generic_start": (0, {9: 1}),
    "mb200_nuts_generic_end": (0, {12: 0, 13: 3}),
}
# symbol -> (index of the host coefficient array, index of its length)
_COEFFICIENTS = {
    "mb200_leapfrog_euclidean": (12, 11),
    "mb200_leapfrog_euclidean_user": (12, 11),
    "mb200_leapfrog_gaussian_euclidean": (11, 10),
}


class _CudaArray:
    def __init__(self, address, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4",
                                         "data": (address, False), "version": 2}


class Recorder:
    """Stand-in for the loaded library: records each call as one line of text."""

    def __init__(self, device):
        self.device = device
        self.calls = []
        self.named = {}
        self.owners = []

    def name(self, label, value):
        if isinstance(value, torch.Tensor):
            # holding the tensor keeps its address from being reused by a later buffer
            self.named[value.data_ptr()] = (label, value)
        return value

    def _labels(self):
        labels = {p: label for p, (label, _) in self.named.items()}
        for prefix, owner in self.owners:
            for k, v in list(getattr(owner, "_dev", {}).items()):
                key = k[0] if isinstance(k, tuple) else k
                for i, t in enumerate(v if isinstance(v, tuple) else (v,)):
                    if isinstance(t, torch.Tensor):
                        sub = f"[{i}]" if isinstance(v, tuple) else ""
                        labels.setdefault(t.data_ptr(), f"{prefix}.{key}{sub}")
            counts = getattr(owner, "call_counts", None)
            if isinstance(counts, torch.Tensor):
                labels[counts.data_ptr()] = f"{prefix}.call_counts"
        labels[STREAM] = "stream"
        labels[USER] = "user"
        return labels

    def _ptr(self, value, labels):
        if value is None or value == 0:
            return "NULL"
        return "@" + labels.get(value, "new")

    def _arg(self, a, labels):
        if a is None:
            return "NULL"
        if isinstance(a, ctypes.c_void_p):
            return self._ptr(a.value, labels)
        if type(a).__name__ == "CArgObject":
            obj = a._obj
            if isinstance(obj, _lib.Model):
                tp = {i: v for i, v in enumerate(obj.target_params) if v}
                rp = {i: v for i, v in enumerate(obj.rmetric_params) if v}
                return (f"Model(target={obj.target_id}/{obj.n_target_params} {tp} "
                        f"aux={self._ptr(obj.target_aux, labels)} rmetric={obj.rmetric_id}/"
                        f"{obj.n_rmetric_params} {rp} raux={self._ptr(obj.rmetric_aux, labels)})")
            if isinstance(obj, _lib.NutsOptions):
                return (f"Nuts(depth={obj.max_tree_depth} slice={obj.slice_variant} "
                        f"euclid={obj.euclidean_criterion} extra={obj.extra_subtree_checks} "
                        f"max_dh={obj.max_delta_h!r} uni={self._ptr(obj.uniforms, labels)} "
                        f"n_uni={obj.n_uniforms})")
            raise AssertionError(f"unexpected by-reference argument {obj!r}")
        if isinstance(a, (bool, int, float)):
            return f"{type(a).__name__}:{a!r}"
        raise AssertionError(f"unexpected argument {a!r}")

    def _write(self, address, n, value):
        if address is None:
            return
        if self.device.type == "cuda":
            torch.as_tensor(_CudaArray(address, n), device=self.device).fill_(value)
        else:
            (ctypes.c_int32 * n).from_address(address)[:] = [value] * n

    def __getattr__(self, symbol):
        if not symbol.startswith("mb200_"):
            raise AttributeError(symbol)

        def call(*args):
            labels = self._labels()
            text = [self._arg(a, labels) for a in args]
            if symbol in _COEFFICIENTS:
                i, k = _COEFFICIENTS[symbol]
                if args[i] is not None:
                    text[i] = "host" + repr(list((ctypes.c_double * args[k]).from_address(
                        args[i].value)))
            self.calls.append(f"{symbol}({', '.join(text)})")
            if symbol in _OUTPUTS:
                n_index, outs = _OUTPUTS[symbol]
                for i, v in outs.items():
                    a = args[i]
                    self._write(None if a is None else a.value, args[n_index], v)
            if symbol.endswith("_bytes"):
                return WS_BYTES
            return 0

        return call


@pytest.fixture
def rec(monkeypatch):
    def make(device):
        r = Recorder(torch.device(device))
        monkeypatch.setattr(_lib, "load", lambda: r)
        return r

    monkeypatch.setattr(_lib, "current_stream_ptr", lambda device: ctypes.c_void_p(STREAM))
    monkeypatch.setattr(targets.CudaTarget, "handle", lambda self: ctypes.c_void_p(USER))
    return make


# ----------------------------------------------------------------------------------------------
# models

def _spd(dim, seed):
    a = np.random.default_rng(seed).standard_normal((dim, dim))
    return a @ a.T + dim * np.eye(dim)


def _metric(kind):
    return {"identity": None, "diag": np.arange(1.0, DIM + 1), "dense": _spd(DIM, 1)}[kind]


USER_SRC = "/* recorded, never compiled */"


def _user(**kw):
    return targets.CudaTarget(DIM, USER_SRC, params=(0.5,), aux=np.ones(3), **kw)


def _system(name):
    m, t = name.split(":")[0], name.split(":")[1] if ":" in name else "registry"
    user = t == "user"
    if m.startswith("eu_"):
        target = _user() if user else targets.NealFunnel(DIM)
        return systems.EuclideanMetricSystem(target, metric=_metric(m[3:]))
    if m.startswith("gauss_eu_"):
        return systems.GaussianEuclideanMetricSystem(targets.Quadratic(_spd(DIM, 2)),
                                                     metric=_metric(m[9:]))
    if m == "constr_hausdorff":
        target = _user(n_constr=1) if user else targets.Sphere(DIM)
        return systems.ConstrainedEuclideanMetricSystem(target, metric=_metric("diag"))
    if m == "constr_lebesgue":
        target = _user(n_constr=1, mhp_constr=True) if user else targets.MultiSphere(DIM, 2)
        return systems.DenseConstrainedEuclideanMetricSystem(target, metric=_metric("dense"),
                                                             dens_wrt_hausdorff=False)
    if m.startswith("gauss_constr_"):
        target = _user(n_constr=1, mhp_constr=True) if user else targets.Sphere(DIM)
        return systems.GaussianDenseConstrainedEuclideanMetricSystem(target,
                                                                     metric=_metric(m[13:]))
    if m == "rm_dense":
        return systems.DenseRiemannianMetricSystem(targets.NealFunnel(DIM),
                                                   targets.Rank1Metric(_spd(DIM, 3), 0.5))
    if m == "rm_softabs":
        return systems.SoftAbsRiemannianMetricSystem(targets.Quartic(_spd(DIM, 4)),
                                                     softabs_coeff=2.0)
    if m == "rm_scalar":
        return systems.ScalarRiemannianMetricSystem(targets.NealFunnel(DIM),
                                                    targets.QuadraticScalarMetric(1.0, 0.5))
    if m == "rm_diag":
        return systems.DiagonalRiemannianMetricSystem(targets.NealFunnel(DIM),
                                                      targets.FunnelFisherMetric())
    if m == "rm_chol":
        return systems.CholeskyFactoredRiemannianMetricSystem(
            targets.StdGaussian(DIM), targets.QuadraticCholeskyMetric(np.tril(_spd(DIM, 5)), 0.1))
    raise KeyError(name)


def _watch(r, system, integrator=None):
    r.owners.append(("sys", system))
    if getattr(system, "metric", None) is not None and hasattr(system, "_metric"):
        r.owners.append(("metric", system._metric))
    if integrator is not None:
        r.owners.append(("integ", integrator))


def _state(r, device, n=N, dir=1, numpy=False):  # noqa: A002
    g = np.random.default_rng(7)
    pos, mom = g.standard_normal((n, DIM)), g.standard_normal((n, DIM))
    if numpy:
        return ChainState(pos=pos, mom=mom, dir=dir)
    pos = r.name("pos", torch.as_tensor(pos, device=device))
    mom = r.name("mom", torch.as_tensor(mom, device=device))
    if isinstance(dir, torch.Tensor):
        dir = r.name("dir", dir.to(device))  # noqa: A001
    return ChainState(pos=pos, mom=mom, dir=dir)


def _run(r, ops):
    for op in ops:
        try:
            op()
        except Exception as e:  # noqa: BLE001
            r.calls.append(f"raises {type(e).__name__}: {e}")
    return r.calls


# ----------------------------------------------------------------------------------------------
# cases: name -> function(recorder, device) running the operations

SYSTEM_METHODS = ("h", "neg_log_dens", "grad_neg_log_dens", "h2", "dh2_dmom", "dh_dmom")


def _system_case(name, methods=SYSTEM_METHODS, momentum=True):
    def case(r, device):
        s = _system(name)
        _watch(r, s)
        st = _state(r, device)
        ops = [lambda m=m: getattr(s, m)(st) for m in methods]
        if momentum:
            ops += [lambda: s.sample_momentum(st, np.random.default_rng(1)),
                    lambda: s.sample_momentum(st, [np.random.default_rng(i) for i in range(N)])]
        return _run(r, ops)
    return case


def _integrator(name, system):
    if name == "leapfrog":
        return integrators.LeapfrogIntegrator(system, step_size=0.25)
    if name == "bcss2":
        return integrators.BCSSTwoStageIntegrator(system, step_size=0.25)
    if name == "bcss3":
        return integrators.BCSSThreeStageIntegrator(system, step_size=0.25)
    if name == "implicit_leapfrog":
        return integrators.ImplicitLeapfrogIntegrator(system, step_size=0.25)
    if name == "implicit_leapfrog_steffensen":
        return integrators.ImplicitLeapfrogIntegrator(
            system, step_size=0.25, reverse_check_tol=1e-7,
            fixed_point_solver=solve_fixed_point_steffensen,
            fixed_point_solver_kwargs={"max_iters": 33, "convergence_tol": 1e-11})
    if name == "implicit_midpoint":
        return integrators.ImplicitMidpointIntegrator(system, step_size=0.25)
    if name == "constrained":
        return integrators.ConstrainedLeapfrogIntegrator(system, step_size=0.25)
    if name == "constrained_line_search":
        return integrators.ConstrainedLeapfrogIntegrator(
            system, step_size=0.25, n_inner_step=2, reverse_check_tol=1e-6,
            projection_solver=solve_projection_onto_manifold_newton_with_line_search,
            projection_solver_kwargs={"max_iters": 20, "max_line_search_iters": 4})
    if name == "constrained_quasi_newton":
        return integrators.ConstrainedLeapfrogIntegrator(
            system, step_size=0.25, projection_solver=solve_projection_onto_manifold_quasi_newton,
            projection_solver_kwargs={"constraint_tol": 1e-10})
    raise KeyError(name)


def _step_case(integ_name, sys_name):
    def case(r, device):
        s = _system(sys_name)
        it = _integrator(integ_name, s)
        _watch(r, s, it)
        st = _state(r, device)
        st_rev = _state(r, device, dir=torch.tensor([1, -1, 1], dtype=torch.int32))
        eps_t = r.name("eps_t", torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64, device=device))
        len_t = r.name("len_t", torch.tensor([1, 4, 2], dtype=torch.int32, device=device))
        single = ChainState(pos=st.pos[1], mom=st.mom[1], dir=-1)

        def per_chain_eps():
            it.step_size = eps_t
            try:
                it.step_n(st, 2, return_h=True)
            finally:
                it.step_size = 0.25

        def counted():
            it.count_calls()
            try:
                it.step_n(st_rev, 2)
                it.step_n(st_rev, 1, return_h=True)
            finally:
                it.count_calls(False)

        return _run(r, [
            lambda: it.step_n(st, 3),
            lambda: it.step_n(st, 3, return_h=True),
            per_chain_eps,
            lambda: it.step_n(st, len_t),
            lambda: it.step_n(st_rev, len_t, return_h=True),
            counted,
            lambda: it.step(single),
        ])
    return case


def _gaussian_flow_case(sys_name):
    def case(r, device):
        s = _system(sys_name)
        _watch(r, s)
        dt_t = r.name("dt", torch.tensor([0.1, -0.2, 0.3], dtype=torch.float64, device=device))
        return _run(r, [lambda: s.h2_flow(_state(r, device), 0.3),
                        lambda: s.h2_flow(_state(r, device), -0.3),
                        lambda: s.h2_flow(_state(r, device), dt_t)])
    return case


def _metropolis_case(sys_name, integ_name):
    def case(r, device):
        s = _system(sys_name)
        it = _integrator(integ_name, s)
        _watch(r, s, it)
        tr = transitions.MetropolisStaticIntegrationTransition(s, it, 3)
        tr_rand = transitions.MetropolisRandomIntegrationTransition(s, it, (1, 5))
        gens = [np.random.default_rng(i) for i in range(N)]
        return _run(r, [lambda: tr.sample(_state(r, device, dir=-1), gens),
                        lambda: tr.sample(_state(r, device), np.random.default_rng(3)),
                        lambda: tr_rand.sample(_state(r, device), np.random.default_rng(4))])
    return case


def _replayed(seeds, used):
    """The generator states after each chain consumed exactly `used` uniforms."""
    out = []
    for s in seeds:
        g = np.random.default_rng(s)
        g.uniform(size=used)
        out.append(g.bit_generator.state)
    return out


def _nuts_case(sys_name, integ_name, fused, depth):
    def case(r, device):
        s = _system(sys_name)
        it = _integrator(integ_name, s)
        _watch(r, s, it)
        multi = transitions.MultinomialDynamicIntegrationTransition(s, it, max_tree_depth=depth)
        sl = transitions.SliceDynamicIntegrationTransition(
            s, it, max_tree_depth=depth, max_delta_h=50.0, do_extra_subtree_checks=False,
            termination_criterion=transitions.euclidean_no_u_turn_criterion)
        assert multi._fused == fused and sl._fused == fused
        gens = [np.random.default_rng(10 + i) for i in range(N)]
        eps_t = r.name("eps_t", torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64, device=device))

        def per_chain():
            it.step_size = eps_t
            try:
                sl.sample(_state(r, device), np.random.default_rng(5))
            finally:
                it.step_size = 0.25

        def replay():
            multi.sample(_state(r, device), gens)
            assert [g.bit_generator.state for g in gens] == _replayed(range(10, 10 + N), 3)

        return _run(r, [replay, per_chain])
    return case


def _momentum_case(sys_name, **state_kw):
    def case(r, device):
        s = _system(sys_name)
        _watch(r, s)
        st = _state(r, device, **state_kw)
        return _run(r, [lambda: s.sample_momentum(st, np.random.default_rng(1)),
                        lambda: s.sample_momentum(st, torch.Generator(device=device))])
    return case


def _project_case(sys_name):
    def case(r, device):
        s = _system(sys_name)
        _watch(r, s)
        st = _state(r, device)
        mom = r.name("mom2", torch.ones(N, DIM, dtype=torch.float64, device=device))
        return _run(r, [lambda: s.project_onto_cotangent_space(mom, st),
                        lambda: s.project_onto_cotangent_space(mom[0], ChainState(pos=st.pos[0])),
                        lambda: s.sample_momentum(st, np.random.default_rng(1))])
    return case


def _numpy_case(sys_name, integ_name):
    def case(r, device):
        s = _system(sys_name)
        it = _integrator(integ_name, s)
        _watch(r, s, it)
        st = _state(r, device, numpy=True)
        single = ChainState(pos=st.pos[0], mom=st.mom[0], dir=1)
        ops = [lambda m=m: getattr(s, m)(st) for m in ("h", "dh2_dmom")]
        if hasattr(s, "neg_log_dens"):
            ops += [lambda: s.neg_log_dens(single), lambda: s.grad_neg_log_dens(st)]
        return _run(r, ops + [lambda: it.step_n(st, 2), lambda: it.step(single),
                              lambda: s.sample_momentum(st, np.random.default_rng(1))])
    return case


def _host_case(sys_name, integ_name):
    def case(r, device):
        s = _system(sys_name)
        it = _integrator(integ_name, s)
        _watch(r, s, it)
        g = np.random.default_rng(7)
        pos = r.name("host_pos", torch.as_tensor(g.standard_normal((8, DIM))))
        mom = r.name("host_mom", torch.as_tensor(g.standard_normal((8, DIM))))
        return _run(r, [lambda: it.step_n_host(pos, mom, 3, n_chunks=3),
                        lambda: it.step_n_host(pos, mom, 2, dir=-1, n_chunks=2)])
    return case


CPU_CASES = {}
for _m in ("eu_identity", "eu_diag", "eu_dense", "eu_dense:user", "gauss_eu_identity",
           "gauss_eu_dense", "constr_hausdorff", "constr_hausdorff:user", "constr_lebesgue",
           "constr_lebesgue:user", "gauss_constr_dense", "gauss_constr_diag:user"):
    CPU_CASES[f"system/{_m}"] = _system_case(_m, momentum=not _m.startswith(("constr",
                                                                              "gauss_constr")))
for _m in ("rm_dense", "rm_softabs", "rm_scalar", "rm_diag", "rm_chol"):
    CPU_CASES[f"system/{_m}"] = _system_case(_m, methods=("h", "dh2_dmom", "dh_dmom"),
                                             momentum=False)
for _m in ("gauss_eu_identity", "gauss_eu_diag", "gauss_eu_dense"):
    CPU_CASES[f"h2_flow/{_m}"] = _gaussian_flow_case(_m)
for _i, _m in (("leapfrog", "eu_identity"), ("leapfrog", "eu_dense"), ("leapfrog", "eu_diag:user"),
               ("bcss2", "eu_diag"), ("bcss3", "eu_dense:user"), ("leapfrog", "gauss_eu_diag"),
               ("bcss2", "gauss_eu_dense"), ("implicit_leapfrog", "rm_dense"),
               ("implicit_leapfrog_steffensen", "rm_softabs"), ("implicit_midpoint", "rm_scalar"),
               ("implicit_leapfrog", "rm_diag"), ("implicit_midpoint", "rm_chol"),
               ("constrained", "constr_hausdorff"), ("constrained", "constr_hausdorff:user"),
               ("constrained_line_search", "constr_lebesgue"),
               ("constrained_quasi_newton", "constr_lebesgue:user"),
               ("constrained", "gauss_constr_dense"),
               ("constrained_line_search", "gauss_constr_identity:user")):
    CPU_CASES[f"step_n/{_i}/{_m}"] = _step_case(_i, _m)
for _i, _m in (("leapfrog", "eu_dense"), ("implicit_leapfrog", "rm_diag"),
               ("constrained", "constr_hausdorff:user")):
    CPU_CASES[f"metropolis/{_i}/{_m}"] = _metropolis_case(_m, _i)
for _i, _m, _f in (("leapfrog", "eu_diag", True), ("leapfrog", "eu_dense:user", False),
                   ("bcss2", "eu_identity", False), ("implicit_leapfrog", "rm_dense", False),
                   ("constrained", "gauss_constr_dense", False)):
    CPU_CASES[f"nuts/{_i}/{_m}"] = _nuts_case(_m, _i, _f, 2)

CUDA_CASES = {}
for _m in ("eu_dense", "gauss_eu_diag", "rm_dense", "rm_softabs", "rm_scalar", "rm_diag",
           "rm_chol"):
    CUDA_CASES[f"sample_momentum/{_m}"] = _momentum_case(_m)
CUDA_CASES["sample_momentum/rm_chol/numpy"] = _momentum_case("rm_chol", numpy=True)
for _m in ("constr_hausdorff", "constr_lebesgue:user", "gauss_constr_dense",
           "gauss_constr_diag:user"):
    CUDA_CASES[f"project/{_m}"] = _project_case(_m)
for _i, _m in (("leapfrog", "eu_dense"), ("leapfrog", "eu_identity:user"),
               ("leapfrog", "gauss_eu_dense"), ("implicit_leapfrog", "rm_dense"),
               ("constrained", "constr_hausdorff"), ("constrained", "gauss_constr_dense:user")):
    CUDA_CASES[f"numpy/{_i}/{_m}"] = _numpy_case(_m, _i)
for _i, _m in (("leapfrog", "eu_dense"), ("leapfrog", "eu_identity"), ("leapfrog", "eu_diag:user"),
               ("leapfrog", "gauss_eu_diag"), ("bcss2", "eu_diag")):
    CUDA_CASES[f"step_n_host/{_i}/{_m}"] = _host_case(_m, _i)


@pytest.mark.parametrize("case", sorted(CPU_CASES))
def test_host_calls(rec, case):
    r = rec("cpu")
    assert CPU_CASES[case](r, torch.device("cpu")) == EXPECTED[case]


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CUDA_CASES))
def test_host_calls_cuda(rec, case):
    r = rec("cuda")
    calls = CUDA_CASES[case](r, torch.device("cuda"))
    torch.cuda.synchronize()
    assert calls == EXPECTED[case]


EXPECTED = {}
EXPECTED['h2_flow/gauss_eu_dense'] = [
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.3, NULL, int:1, int:1, host[1.0], int:0, int:2, @metric.inv, @metric.rot, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @new, int:3, int:4, float:0.3, NULL, int:1, int:1, host[1.0], int:0, int:2, @metric.inv, @metric.rot, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @stream)',
    'raises NotImplementedError: per-chain step sizes with a dense Gaussian-split metric',
]
EXPECTED['h2_flow/gauss_eu_diag'] = [
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.3, NULL, int:1, int:1, host[1.0], int:0, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @new, int:3, int:4, float:0.3, NULL, int:1, int:1, host[1.0], int:0, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @new, int:3, int:4, float:0.0, @new, int:1, int:1, host[1.0], int:0, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @stream)',
]
EXPECTED['h2_flow/gauss_eu_identity'] = [
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.3, NULL, int:1, int:1, host[1.0], int:0, int:0, NULL, NULL, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @new, int:3, int:4, float:0.3, NULL, int:1, int:1, host[1.0], int:0, int:0, NULL, NULL, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @new, int:3, int:4, float:0.0, @new, int:1, int:1, host[1.0], int:0, int:0, NULL, NULL, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @stream)',
]
EXPECTED['metropolis/constrained/constr_hausdorff:user'] = [
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_metropolis_select(@new, @new, @new, @new, @new, @new, @new, @new, @new, @new, int:3, int:4, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_metropolis_select(@new, @new, @new, @new, @new, @new, @new, @new, @new, @new, int:3, int:4, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @new, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_metropolis_select(@new, @new, @new, @new, @new, @new, @new, @new, @new, @new, int:3, int:4, @new, @new, @new, @stream)',
]
EXPECTED['metropolis/implicit_leapfrog/rm_diag'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_metropolis_select(@new, @new, @new, @new, @new, @new, @new, @new, @new, @new, int:3, int:4, @new, @new, @new, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_metropolis_select(@new, @new, @new, @new, @new, @new, @new, @new, @new, @new, int:3, int:4, @new, @new, @new, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @new, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_metropolis_select(@new, @new, @new, @new, @new, @new, @new, @new, @new, @new, int:3, int:4, @new, @new, @new, @stream)',
]
EXPECTED['metropolis/leapfrog/eu_dense'] = [
    'mb200_hamiltonian_euclidean(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_metropolis_select(@new, @new, @new, @new, @new, @new, @new, @new, @new, @new, int:3, int:4, @new, @new, @new, @stream)',
    'mb200_hamiltonian_euclidean(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_metropolis_select(@new, @new, @new, @new, @new, @new, @new, @new, @new, @new, int:3, int:4, @new, @new, @new, @stream)',
    'mb200_hamiltonian_euclidean(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @new, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_metropolis_select(@new, @new, @new, @new, @new, @new, @new, @new, @new, @new, int:3, int:4, @new, @new, @new, @stream)',
]
EXPECTED['nuts/bcss2/eu_identity'] = [
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_generic_state_bytes(int:3)',
    'mb200_hamiltonian_euclidean(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_begin(@pos, @mom, @new, @new, int:3, int:4, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, int:4096, @new, int:4096, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:0, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:0, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:2, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:2, int:2, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_end(int:3, int:4, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_generic_state_bytes(int:3)',
    'mb200_hamiltonian_euclidean(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_begin(@pos, @mom, @new, @new, int:3, int:4, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, int:4096, @new, int:4096, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:0, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:0, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:2, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:2, int:2, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_end(int:3, int:4, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
]
EXPECTED['nuts/constrained/gauss_constr_dense'] = [
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_generic_state_bytes(int:3)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_begin(@pos, @mom, @new, @new, int:3, int:4, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, int:4096, @new, int:4096, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:0, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:0, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:2, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:2, int:2, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_end(int:3, int:4, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_generic_state_bytes(int:3)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_begin(@pos, @mom, @new, @new, int:3, int:4, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, int:4096, @new, int:4096, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:0, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:0, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:2, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:2, int:2, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_end(int:3, int:4, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
]
EXPECTED['nuts/implicit_leapfrog/rm_dense'] = [
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_generic_state_bytes(int:3)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_nuts_generic_begin(@pos, @mom, @new, @new, int:3, int:4, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, int:4096, @new, int:4096, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:0, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@new, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:0, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@new, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:2, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@new, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:2, int:2, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_end(int:3, int:4, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_generic_state_bytes(int:3)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_nuts_generic_begin(@pos, @mom, @new, @new, int:3, int:4, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, int:4096, @new, int:4096, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:0, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@new, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:0, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@new, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:2, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@new, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:2, int:2, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_end(int:3, int:4, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
]
EXPECTED['nuts/leapfrog/eu_dense:user'] = [
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_generic_state_bytes(int:3)',
    'mb200_hamiltonian_euclidean_user(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @stream, @user)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_begin(@pos, @mom, @new, @new, int:3, int:4, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, int:4096, @new, int:4096, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:0, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:0, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:2, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:3, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:2, int:2, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:1, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_end(int:3, int:4, Nuts(depth=2 slice=0 euclid=0 extra=1 max_dh=1000.0 uni=@new n_uni=8), @sys.nuts_ws, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_generic_state_bytes(int:3)',
    'mb200_hamiltonian_euclidean_user(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @stream, @user)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_begin(@pos, @mom, @new, @new, int:3, int:4, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, int:4096, @new, int:4096, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:0, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:0, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_start(int:3, int:4, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:1, int:2, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_nuts_generic_leaf(@new, @new, @new, @new, @new, int:3, int:4, int:2, int:2, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @stream)',
    'mb200_nuts_generic_finish(int:3, int:4, int:1, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @stream)',
    'mb200_nuts_generic_end(int:3, int:4, Nuts(depth=2 slice=1 euclid=1 extra=0 max_dh=50.0 uni=@new n_uni=9), @sys.nuts_ws, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
]
EXPECTED['nuts/leapfrog/eu_diag'] = [
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_euclidean(@pos, @mom, @new, @new, int:3, int:4, float:0.25, NULL, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, int:0, int:1, int:2, float:1000.0, @new, int:8, @sys.nuts_ws, int:4096, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
    'mb200_nuts_workspace_bytes(int:3, int:4, int:2)',
    'mb200_nuts_euclidean(@pos, @mom, @new, @new, int:3, int:4, float:0.0, @eps_t, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:1, int:1, int:0, int:2, float:50.0, @new, int:9, @sys.nuts_ws, int:4096, @new, @new, @new, @new, @new, @new, @new, @new, @new, @stream)',
]
EXPECTED['step_n/bcss2/eu_diag'] = [
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
]
EXPECTED['step_n/bcss2/gauss_eu_dense'] = [
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:2, @metric.inv, @metric.rot, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:2, @metric.inv, @metric.rot, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'raises NotImplementedError: per-chain step sizes with a dense Gaussian-split metric',
    'raises NotImplementedError: per-chain trajectory lengths: plain Euclidean systems only',
    'raises NotImplementedError: per-chain trajectory lengths: plain Euclidean systems only',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:2, @metric.inv, @metric.rot, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:2, @metric.inv, @metric.rot, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:2, @metric.inv, @metric.rot, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
]
EXPECTED['step_n/bcss3/eu_dense:user'] = [
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:7, host[0.11888010966548, 0.29619504261126, 0.38111989033452, 0.40760991477748, 0.38111989033452, 0.29619504261126, 0.11888010966548], int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:7, host[0.11888010966548, 0.29619504261126, 0.38111989033452, 0.40760991477748, 0.38111989033452, 0.29619504261126, 0.11888010966548], int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:7, host[0.11888010966548, 0.29619504261126, 0.38111989033452, 0.40760991477748, 0.38111989033452, 0.29619504261126, 0.11888010966548], int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:7, host[0.11888010966548, 0.29619504261126, 0.38111989033452, 0.40760991477748, 0.38111989033452, 0.29619504261126, 0.11888010966548], int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:7, host[0.11888010966548, 0.29619504261126, 0.38111989033452, 0.40760991477748, 0.38111989033452, 0.29619504261126, 0.11888010966548], int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:7, host[0.11888010966548, 0.29619504261126, 0.38111989033452, 0.40760991477748, 0.38111989033452, 0.29619504261126, 0.11888010966548], int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:7, host[0.11888010966548, 0.29619504261126, 0.38111989033452, 0.40760991477748, 0.38111989033452, 0.29619504261126, 0.11888010966548], int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:7, host[0.11888010966548, 0.29619504261126, 0.38111989033452, 0.40760991477748, 0.38111989033452, 0.29619504261126, 0.11888010966548], int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
]
EXPECTED['step_n/constrained/constr_hausdorff'] = [
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_constrained_leapfrog_euclidean(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
]
EXPECTED['step_n/constrained/constr_hausdorff:user'] = [
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_constrained_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
]
EXPECTED['step_n/constrained/gauss_constr_dense'] = [
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_constrained_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
]
EXPECTED['step_n/constrained_line_search/constr_lebesgue'] = [
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:2, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, NULL, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:2, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:2, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, @new, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:2, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, NULL, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:2, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:2, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, NULL, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:2, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_constrained_leapfrog_euclidean(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:2, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, NULL, @new, @new, @new, @stream)',
]
EXPECTED['step_n/constrained_line_search/gauss_constr_identity:user'] = [
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:2, int:0, NULL, @metric.gauss_constr[0], NULL, NULL, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, NULL, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:2, int:0, NULL, @metric.gauss_constr[0], NULL, NULL, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, @new, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:2, int:0, NULL, @metric.gauss_constr[0], NULL, NULL, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, @new, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:2, int:0, NULL, @metric.gauss_constr[0], NULL, NULL, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, NULL, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:2, int:0, NULL, @metric.gauss_constr[0], NULL, NULL, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, @new, @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:2, int:0, NULL, @metric.gauss_constr[0], NULL, NULL, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, NULL, @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:2, int:0, NULL, @metric.gauss_constr[0], NULL, NULL, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, @new, @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:2, int:0, NULL, @metric.gauss_constr[0], NULL, NULL, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:2, float:1e-09, float:1e-08, float:10000000000.0, int:20, int:4, float:1e-06, NULL, @new, @new, @new, @stream, @user)',
]
EXPECTED['step_n/constrained_quasi_newton/constr_lebesgue:user'] = [
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:1, float:1e-10, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:1, float:1e-10, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:1, float:1e-10, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:1, float:1e-10, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:1, float:1e-10, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:1, float:1e-10, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:1, float:1e-10, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_constrained_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:1, float:1e-10, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
]
EXPECTED['step_n/implicit_leapfrog/rm_dense'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_implicit_workspace_bytes(int:1, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
]
EXPECTED['step_n/implicit_leapfrog/rm_diag'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_implicit_workspace_bytes(int:1, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
]
EXPECTED['step_n/implicit_leapfrog_steffensen/rm_softabs'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), int:1, float:1e-11, float:10000000000.0, int:33, float:1e-07, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), int:1, float:1e-11, float:10000000000.0, int:33, float:1e-07, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), int:1, float:1e-11, float:10000000000.0, int:33, float:1e-07, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), int:1, float:1e-11, float:10000000000.0, int:33, float:1e-07, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), int:1, float:1e-11, float:10000000000.0, int:33, float:1e-07, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), int:1, float:1e-11, float:10000000000.0, int:33, float:1e-07, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), int:1, float:1e-11, float:10000000000.0, int:33, float:1e-07, @new, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_implicit_workspace_bytes(int:1, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), int:1, float:1e-11, float:10000000000.0, int:33, float:1e-07, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
]
EXPECTED['step_n/implicit_midpoint/rm_chol'] = [
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_implicit_midpoint_riemannian(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @stream)',
]
EXPECTED['step_n/implicit_midpoint/rm_scalar'] = [
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_implicit_midpoint_riemannian(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, @new, @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_implicit_midpoint_riemannian(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @stream)',
]
EXPECTED['step_n/leapfrog/eu_dense'] = [
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
]
EXPECTED['step_n/leapfrog/eu_diag:user'] = [
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean_user(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream, @user)',
    'mb200_set_call_counters(NULL)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
]
EXPECTED['step_n/leapfrog/eu_identity'] = [
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, NULL, int:0, NULL, int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:0, NULL, int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:4, @len_t, int:0, NULL, int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, NULL, int:0, NULL, int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
]
EXPECTED['step_n/leapfrog/gauss_eu_diag'] = [
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, @eps_t, int:2, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'raises NotImplementedError: per-chain trajectory lengths: plain Euclidean systems only',
    'raises NotImplementedError: per-chain trajectory lengths: plain Euclidean systems only',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:2, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_set_call_counters(@integ.call_counts)',
    'mb200_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, @dir, int:3, int:4, float:0.25, NULL, int:1, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @new, @new, @stream)',
    'mb200_set_call_counters(NULL)',
    'mb200_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:1, int:4, float:0.25, NULL, int:1, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
]
EXPECTED['system/constr_hausdorff'] = [
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/constr_hausdorff:user'] = [
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval_user(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval_user(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/constr_lebesgue'] = [
    'mb200_constrained_leapfrog_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=6/1 {0: 2.0, 7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/constr_lebesgue:user'] = [
    'mb200_constrained_leapfrog_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval_user(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval_user(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/eu_dense'] = [
    'mb200_hamiltonian_euclidean(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/eu_dense:user'] = [
    'mb200_hamiltonian_euclidean_user(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @stream, @user)',
    'mb200_euclidean_eval_user(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval_user(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/eu_diag'] = [
    'mb200_hamiltonian_euclidean(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:1, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:1, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/eu_identity'] = [
    'mb200_hamiltonian_euclidean(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/gauss_constr_dense'] = [
    'mb200_constrained_leapfrog_gaussian_euclidean(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/gauss_constr_diag:user'] = [
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@pos, @mom, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:1, @metric.inv, @metric.gauss_constr[0], NULL, NULL, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval_user(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval_user(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/gauss_eu_dense'] = [
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/gauss_eu_identity'] = [
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@pos, @mom, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['system/rm_chol'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), @new, @stream)',
]
EXPECTED['system/rm_dense'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
]
EXPECTED['system/rm_diag'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), @new, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), @new, @stream)',
]
EXPECTED['system/rm_scalar'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), @new, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), @new, @stream)',
]
EXPECTED['system/rm_softabs'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL))',
    'mb200_hamiltonian_riemannian(@pos, @mom, int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), @new, @stream)',
    'mb200_dh_dmom_riemannian(@pos, @mom, @new, int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), @new, @stream)',
]
EXPECTED['numpy/constrained/constr_hausdorff'] = [
    'mb200_constrained_leapfrog_euclidean(@new, @new, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:1, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:1, int:4, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_constrained_leapfrog_euclidean(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:2, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_constrained_leapfrog_euclidean(@new, @new, @new, @new, NULL, int:1, int:4, float:0.25, NULL, int:1, NULL, int:1, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:1, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_project_onto_cotangent_space(@new, @new, @new, int:3, int:4, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @stream)',
]
EXPECTED['numpy/constrained/gauss_constr_dense:user'] = [
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@new, @new, @new, @new, NULL, int:3, int:4, float:0.0, NULL, int:0, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval_user(@new, @new, int:1, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval_user(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream, @user)',
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:2, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
    'mb200_constrained_leapfrog_gaussian_euclidean_user(@new, @new, @new, @new, NULL, int:1, int:4, float:0.25, NULL, int:1, NULL, int:1, int:2, @metric.inv, @metric.gauss_constr[0], @metric.gauss_constr[1], @metric.gauss_constr[2], Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), int:0, float:1e-09, float:1e-08, float:10000000000.0, int:50, int:10, float:2e-08, NULL, @new, @new, @new, @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_project_onto_cotangent_space_gaussian_user(@new, @new, @new, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @stream, @user)',
]
EXPECTED['numpy/implicit_leapfrog/rm_dense'] = [
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_hamiltonian_riemannian(@new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_dh_dmom_riemannian(@new, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_implicit_workspace_bytes(int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:2, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_implicit_workspace_bytes(int:1, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux))',
    'mb200_implicit_leapfrog_riemannian(@new, @new, @new, @new, NULL, int:1, int:4, float:0.25, NULL, int:1, NULL, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), int:0, float:1e-09, float:10000000000.0, int:100, float:2e-08, NULL, @new, @new, @new, @sys.ws, int:4096, @stream)',
    'mb200_sample_momentum_riemannian(@new, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
]
EXPECTED['numpy/leapfrog/eu_dense'] = [
    'mb200_hamiltonian_euclidean(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:1, int:4, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:2, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, NULL, int:1, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['numpy/leapfrog/eu_identity:user'] = [
    'mb200_hamiltonian_euclidean_user(@new, @new, int:3, int:4, int:0, NULL, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:0, NULL, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval_user(@new, @new, int:1, int:4, int:0, NULL, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream, @user)',
    'mb200_euclidean_eval_user(@new, @new, int:3, int:4, int:0, NULL, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:2, NULL, int:0, NULL, int:1, int:0, NULL, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, NULL, int:1, int:4, float:0.25, NULL, int:1, NULL, int:0, NULL, int:1, int:0, NULL, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
]
EXPECTED['numpy/leapfrog/gauss_eu_dense'] = [
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, NULL, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:1, int:4, int:2, @metric.inv, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @new, NULL, NULL, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.inv, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, NULL, NULL, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:2, int:0, NULL, int:1, int:2, @metric.inv, @metric.rot, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@new, @new, @new, @new, NULL, int:1, int:4, float:0.25, NULL, int:1, int:0, NULL, int:1, int:2, @metric.inv, @metric.rot, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['project/constr_hausdorff'] = [
    'mb200_project_onto_cotangent_space(@pos, @mom2, @new, int:3, int:4, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @stream)',
    'mb200_project_onto_cotangent_space(@pos, @mom2, @new, int:1, int:4, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:1, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_project_onto_cotangent_space(@pos, @new, @new, int:3, int:4, int:1, @metric.inv, Model(target=5/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @stream)',
]
EXPECTED['project/constr_lebesgue:user'] = [
    'mb200_project_onto_cotangent_space_user(@pos, @mom2, @new, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @stream, @user)',
    'mb200_project_onto_cotangent_space_user(@pos, @mom2, @new, int:1, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_project_onto_cotangent_space_user(@pos, @new, @new, int:3, int:4, int:2, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @stream, @user)',
]
EXPECTED['project/gauss_constr_dense'] = [
    'mb200_project_onto_cotangent_space_gaussian(@pos, @mom2, @new, int:3, int:4, int:2, @metric.inv, Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), @stream)',
    'mb200_project_onto_cotangent_space_gaussian(@pos, @mom2, @new, int:1, int:4, int:2, @metric.inv, Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_project_onto_cotangent_space_gaussian(@pos, @new, @new, int:3, int:4, int:2, @metric.inv, Model(target=5/0 {7: 1.0} aux=NULL rmetric=0/0 {} raux=NULL), @stream)',
]
EXPECTED['project/gauss_constr_diag:user'] = [
    'mb200_project_onto_cotangent_space_gaussian_user(@pos, @mom2, @new, int:3, int:4, int:1, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @stream, @user)',
    'mb200_project_onto_cotangent_space_gaussian_user(@pos, @mom2, @new, int:1, int:4, int:1, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @stream, @user)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:1, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_project_onto_cotangent_space_gaussian_user(@pos, @new, @new, int:3, int:4, int:1, @metric.inv, Model(target=64/1 {0: 0.5, 7: 1.0} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), @stream, @user)',
]
EXPECTED['sample_momentum/eu_dense'] = [
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:2, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['sample_momentum/gauss_eu_diag'] = [
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:1, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
    'mb200_euclidean_eval(@new, @new, int:3, int:4, int:1, @metric.sqrt_t, Model(target=0/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, NULL, @new, NULL, @stream)',
]
EXPECTED['sample_momentum/rm_chol'] = [
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), @new, @stream)',
]
EXPECTED['sample_momentum/rm_chol/numpy'] = [
    'mb200_sample_momentum_riemannian(@new, @new, @new, int:3, int:4, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_sample_momentum_riemannian(@new, @new, @new, int:3, int:4, Model(target=0/0 {} aux=NULL rmetric=6/1 {0: 0.1} raux=@sys.rmetric_aux), @new, @stream)',
]
EXPECTED['sample_momentum/rm_dense'] = [
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=1/4 {0: 0.5, 1: 8.631391553616007} raux=@sys.rmetric_aux), @new, @stream)',
]
EXPECTED['sample_momentum/rm_diag'] = [
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), @new, @stream)',
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=4/0 {} raux=NULL), @new, @stream)',
]
EXPECTED['sample_momentum/rm_scalar'] = [
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), @new, @stream)',
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=1/0 {} aux=NULL rmetric=5/2 {0: 1.0, 1: 0.5} raux=NULL), @new, @stream)',
]
EXPECTED['sample_momentum/rm_softabs'] = [
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), @new, @stream)',
    'mb200_sample_momentum_riemannian(@pos, @new, @new, int:3, int:4, Model(target=7/1 {0: 1.0} aux=@sys.target_aux rmetric=0/1 {0: 2.0} raux=NULL), @new, @stream)',
]
EXPECTED['step_n_host/bcss2/eu_diag'] = [
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, NULL, int:2, int:4, float:0.25, NULL, int:3, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:4, int:4, float:0.25, NULL, int:2, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_euclidean(@new, @new, @new, @new, @new, int:4, int:4, float:0.25, NULL, int:2, NULL, int:5, host[0.21132486540518713, 0.5, 0.5773502691896257, 0.5, 0.21132486540518713], int:1, int:1, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
]
EXPECTED['step_n_host/leapfrog/eu_dense'] = [
    'mb200_host_scratch_bytes(int:8, int:4)',
    'mb200_leapfrog_euclidean_host(@host_pos, @host_mom, @new, @new, NULL, int:8, int:4, float:0.25, int:3, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, int:3, @new, int:3, @sys.host_scratch, int:4096, int:1)',
    'mb200_host_scratch_bytes(int:8, int:4)',
    'mb200_leapfrog_euclidean_host(@host_pos, @host_mom, @new, @new, @new, int:8, int:4, float:0.25, int:2, int:2, @metric.inv, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, int:2, @new, int:2, @sys.host_scratch, int:4096, int:1)',
]
EXPECTED['step_n_host/leapfrog/eu_diag:user'] = [
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, NULL, int:2, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:4, int:4, float:0.25, NULL, int:2, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
    'mb200_leapfrog_euclidean_user(@new, @new, @new, @new, @new, int:4, int:4, float:0.25, NULL, int:2, NULL, int:0, NULL, int:1, int:1, @metric.inv, Model(target=64/1 {0: 0.5} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream, @user)',
]
EXPECTED['step_n_host/leapfrog/eu_identity'] = [
    'mb200_host_scratch_bytes(int:8, int:4)',
    'mb200_leapfrog_euclidean_host(@host_pos, @host_mom, @new, @new, NULL, int:8, int:4, float:0.25, int:3, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, int:3, @new, int:3, @sys.host_scratch, int:4096, int:1)',
    'mb200_host_scratch_bytes(int:8, int:4)',
    'mb200_leapfrog_euclidean_host(@host_pos, @host_mom, @new, @new, @new, int:8, int:4, float:0.25, int:2, int:0, NULL, Model(target=1/0 {} aux=NULL rmetric=0/0 {} raux=NULL), @new, int:2, @new, int:2, @sys.host_scratch, int:4096, int:1)',
]
EXPECTED['step_n_host/leapfrog/gauss_eu_diag'] = [
    'mb200_leapfrog_gaussian_euclidean(@new, @new, @new, @new, NULL, int:2, int:4, float:0.25, NULL, int:3, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@new, @new, @new, @new, NULL, int:3, int:4, float:0.25, NULL, int:3, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:4, int:4, float:0.25, NULL, int:2, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
    'mb200_leapfrog_gaussian_euclidean(@new, @new, @new, @new, @new, int:4, int:4, float:0.25, NULL, int:2, int:0, NULL, int:1, int:1, @metric.inv, @metric.diag, Model(target=3/0 {} aux=@sys.target_aux rmetric=0/0 {} raux=NULL), NULL, @new, @new, @stream)',
]
