"""User-written targets and metrics on the diagonal and scalar Riemannian systems, without a GPU:
NVRTC compilation of the Riemannian image, compile errors, the systems' constructor rules, the
image cache, copies, the library calls the systems and integrators make, and the C entry points'
routing."""

import copy
import ctypes
import pickle
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import test_host_calls as hc
from mici_b200 import _lib, integrators, jit, systems, targets, transitions
from mici_b200.errors import TargetCompileError
from mici_b200.targets import (
    CudaDiagonalMetric,
    CudaRiemannianPair,
    CudaScalarMetric,
    CudaTarget,
    FunnelFisherMetric,
    NealFunnel,
    QuadraticDiagonalMetric,
    QuadraticScalarMetric,
)

from test_user_target import _elf_symbols
from user_riemannian_sources import (
    FUNNEL,
    FUNNEL_FISHER,
    PAIRS,
    QUADRATIC_DIAGONAL,
    QUADRATIC_SCALAR,
    STD_GAUSSIAN,
    UR_MODELS,
    ur_model,
)

USER_DIAG, USER_SCALAR = 32, 33


# ---------------------------------------------------------------------------------- compilation

def test_example_pairs_compile_to_sm90a_images_with_the_three_kernels():
    def build(item):
        name, (tsrc, kind, msrc) = item
        return name, jit.compile_target(tsrc, name, metric=(kind, msrc, name + "_metric"))

    with ThreadPoolExecutor(len(PAIRS)) as pool:
        images = dict(pool.map(build, PAIRS.items()))
    for name, (_, cubin, names) in images.items():
        kind = PAIRS[name][1]
        assert cubin[:4] == b"\x7fELF"
        assert int.from_bytes(cubin[0x30:0x34], "little") & 0xFF == 90  # sm_90(a)
        assert len(names) == 3 and _elf_symbols(cubin) >= set(names)
        assert ["implicit_leapfrog" in names[0], "velocity" in names[1],
                "sample_momentum" in names[2]] == [True] * 3
        want = "UserDiagonalMetric" if kind == "diagonal" else "UserScalarMetric"
        assert all("UserRTarget" in n and want in n for n in names)


@pytest.mark.parametrize("model", UR_MODELS)
def test_models_beyond_the_registry_compile(model):
    _, _, (tsrc, _, _), (kind, msrc, _, _) = ur_model(model)
    _, cubin, names = jit.compile_target(tsrc, model, metric=(kind, msrc, model + "_metric"))
    assert len(names) == 3 and _elf_symbols(cubin) >= set(names)


def test_missing_metric_vjp_is_a_compile_error_at_the_end_of_the_metric_source():
    src = FUNNEL_FISHER.replace("vjp_metric_diagonal(", "other_vjp(")
    with pytest.raises(TargetCompileError) as e:
        jit.compile_target(FUNNEL, "funnel", metric=("diagonal", src, "fisher_no_vjp"))
    line = len(src.splitlines()) + 1
    assert "vjp_metric_diagonal" in e.value.log
    assert f"fisher_no_vjp.cu({line})" in e.value.log


def test_metric_syntax_error_reports_the_metric_line():
    src = QUADRATIC_SCALAR + "__device__ double broken() { return q1; }\n"
    with pytest.raises(TargetCompileError) as e:
        jit.compile_target(STD_GAUSSIAN, "gauss", metric=("scalar", src, "broken_scalar"))
    assert f"broken_scalar.cu({len(src.splitlines())})" in e.value.log


# ---------------------------------------------------------------------------- constructor rules

def _target(dim=6, **kw):
    return CudaTarget(dim, FUNNEL, **kw)


def test_user_metrics_are_accepted_with_an_unconstrained_cuda_target():
    s = systems.DiagonalRiemannianMetricSystem(_target(), CudaDiagonalMetric(FUNNEL_FISHER))
    assert s._rmetric_id == USER_DIAG and isinstance(s._user_pair, CudaRiemannianPair)
    s = systems.ScalarRiemannianMetricSystem(
        _target(), CudaScalarMetric(QUADRATIC_SCALAR, params=(1.0, 0.5), aux=[1.0, 2.0]))
    assert s._rmetric_id == USER_SCALAR and s._rmetric_params == (1.0, 0.5)
    assert np.array_equal(s._rmetric_aux, [1.0, 2.0])
    # registry models are unchanged
    s = systems.DiagonalRiemannianMetricSystem(NealFunnel(6), FunnelFisherMetric())
    assert s._user_pair is None and not s._user_targets


@pytest.mark.parametrize("make", [
    # a user metric with a registry target
    lambda: systems.DiagonalRiemannianMetricSystem(NealFunnel(6), CudaDiagonalMetric(FUNNEL_FISHER)),
    lambda: systems.ScalarRiemannianMetricSystem(NealFunnel(6), CudaScalarMetric(QUADRATIC_SCALAR)),
    # a metric of the other kind
    lambda: systems.DiagonalRiemannianMetricSystem(_target(), CudaScalarMetric(QUADRATIC_SCALAR)),
    lambda: systems.ScalarRiemannianMetricSystem(_target(), CudaDiagonalMetric(FUNNEL_FISHER)),
    lambda: systems.DiagonalRiemannianMetricSystem(NealFunnel(6), CudaScalarMetric(QUADRATIC_SCALAR)),
    # a constrained CudaTarget
    lambda: systems.DiagonalRiemannianMetricSystem(_target(n_constr=1),
                                                   CudaDiagonalMetric(FUNNEL_FISHER)),
    lambda: systems.ScalarRiemannianMetricSystem(_target(n_constr=1),
                                                 CudaScalarMetric(QUADRATIC_SCALAR)),
    # a CudaTarget with a registry metric
    lambda: systems.ScalarRiemannianMetricSystem(_target(), QuadraticScalarMetric()),
    lambda: systems.DiagonalRiemannianMetricSystem(_target(), QuadraticDiagonalMetric()),
    # the other Riemannian systems take no user metric
    lambda: systems.CholeskyFactoredRiemannianMetricSystem(_target(), CudaDiagonalMetric("")),
    lambda: systems.DenseRiemannianMetricSystem(_target(), CudaDiagonalMetric("")),
])
def test_refused_pairs_raise_type_error(make):
    with pytest.raises(TypeError):
        make()


def test_cuda_target_with_registry_metric_keeps_its_error_text():
    with pytest.raises(TypeError, match="does not take a CudaTarget: user targets run on "
                                        "EuclideanMetricSystem"):
        systems.DiagonalRiemannianMetricSystem(_target(), QuadraticDiagonalMetric())


def test_metric_constructor_validation():
    for cls in (CudaDiagonalMetric, CudaScalarMetric):
        with pytest.raises(ValueError):
            cls(42)
        with pytest.raises(ValueError):
            cls(FUNNEL_FISHER, params=range(9))
        with pytest.raises(ValueError):
            cls(FUNNEL_FISHER, aux=["a"])
        with pytest.raises(ValueError):
            cls(FUNNEL_FISHER, name="not an identifier")
        m = cls(FUNNEL_FISHER, params=range(8), aux=[[1, 2]])
        assert m.params == tuple(float(i) for i in range(8)) and m.aux.dtype == np.float64


# ----------------------------------------------------------------------------------- cache keys

def test_cache_keys_cover_the_image_kind_and_both_sources(monkeypatch):
    compiled = []

    def fake(source, name, constraint=(), metric=()):
        compiled.append((name, constraint, metric))
        return b"\x7fELF-stub", tuple(f"k{i}" for i in range(3 if metric else 10))

    monkeypatch.setattr(jit, "_compile", fake)
    src = FUNNEL + "\n// riemannian cache probe\n"
    diag = ("diagonal", FUNNEL_FISHER, "m")
    other = ("diagonal", QUADRATIC_DIAGONAL, "m")
    scalar = ("scalar", FUNNEL_FISHER, "m")
    for metric in (None, diag, other, scalar):
        jit.compile_target(src, "t", metric=metric)
    before = dict(jit.stats)
    jit.compile_target(src, "t", metric=diag)  # repeat: a hit
    assert jit.stats["hits"] == before["hits"] + 1 and len(compiled) == 4
    keys = {jit.cache_key(src, "t", (), jit._metric(m)) for m in (None, diag, other, scalar)}
    assert len(keys) == 4 and jit.cache_key(src, "t") in keys


def test_pair_handle_is_the_riemannian_image(monkeypatch):
    loaded = []
    monkeypatch.setattr(jit, "load_target", lambda *a, **k: loaded.append((a, k)) or "h")
    t, m = _target(), CudaScalarMetric(QUADRATIC_SCALAR, name="sm")
    system = systems.ScalarRiemannianMetricSystem(t, m)
    assert targets.user_handle(system._user_pair) == "h"
    assert loaded == [((t.source, t.name), {"metric": ("scalar", m.source, "sm")})]


# --------------------------------------------------------------------------------------- copies

def test_system_and_integrator_survive_deepcopy_and_pickle():
    t = _target(params=(1.5,), aux=np.arange(3.0), name="funnel")
    m = CudaDiagonalMetric(FUNNEL_FISHER, params=(0.5,), aux=np.ones(2), name="fisher")
    integ = integrators.ImplicitLeapfrogIntegrator(systems.DiagonalRiemannianMetricSystem(t, m), 0.1)
    for clone in (copy.deepcopy(integ), pickle.loads(pickle.dumps(integ))):
        s = clone.system
        assert isinstance(s, systems.DiagonalRiemannianMetricSystem)
        assert s.target.source == t.source and s.metric_model.source == m.source
        assert s.metric_model.name == "fisher" and np.array_equal(s.metric_model.aux, m.aux)
        assert s._user_pair.target.source == t.source and s._user_pair.metric.kind == "diagonal"
        assert s._rmetric_id == USER_DIAG and s._rmetric_params == (0.5,)


# ------------------------------------------------------------------------------- recorded calls

PAIR = 0xBEEF  # the fake handle of every (target, metric) image


@pytest.fixture
def rec(monkeypatch):
    for name in ("mb200_implicit_leapfrog_riemannian", "mb200_implicit_midpoint_riemannian",
                 "mb200_hamiltonian_riemannian", "mb200_dh_dmom_riemannian",
                 "mb200_sample_momentum_riemannian"):
        monkeypatch.setitem(hc._OUTPUTS, name + "_user", hc._OUTPUTS[name])
    monkeypatch.setattr(_lib, "current_stream_ptr", lambda device: ctypes.c_void_p(hc.STREAM))
    monkeypatch.setattr(CudaRiemannianPair, "handle", lambda self: ctypes.c_void_p(PAIR))
    monkeypatch.setattr(CudaTarget, "handle", lambda self: ctypes.c_void_p(hc.USER))

    class PairRecorder(hc.Recorder):
        def _labels(self):
            return {**super()._labels(), PAIR: "pair"}

    def make(device):
        r = PairRecorder(torch.device(device))
        monkeypatch.setattr(_lib, "load", lambda: r)
        return r

    return make


def _user_system(kind):
    t = CudaTarget(hc.DIM, FUNNEL, params=(0.5,), aux=np.ones(3))
    if kind == "diagonal":
        return systems.DiagonalRiemannianMetricSystem(
            t, CudaDiagonalMetric(FUNNEL_FISHER, params=(2.0, 3.0), aux=np.ones(2)))
    return systems.ScalarRiemannianMetricSystem(t, CudaScalarMetric(QUADRATIC_SCALAR,
                                                                    params=(1.0, 0.25)))


def _ops(system, state, device):
    integ = integrators.ImplicitLeapfrogIntegrator(system, 0.1)
    mid = integrators.ImplicitMidpointIntegrator(system, 0.1)
    ops = [lambda: system.h(state), lambda: system.dh_dmom(state),
           lambda: integ.step_n(state, 2), lambda: mid.step_n(state, 2),
           lambda: transitions.MetropolisRandomIntegrationTransition(
               system, integ, (1, 3)).sample(state, np.random.default_rng(0)),
           lambda: transitions.MultinomialDynamicIntegrationTransition(
               system, integ, max_tree_depth=2).sample(state, np.random.default_rng(0))]
    if device == "cuda":
        ops.append(lambda: system.sample_momentum(state, np.random.default_rng(0)))
    return ops


@pytest.mark.parametrize("kind", ("diagonal", "scalar"))
def test_every_riemannian_call_goes_to_the_user_twin_with_the_pair_image(rec, kind):
    device = "cuda" if torch.cuda.is_available() else "cpu"
    r = rec(device)
    system = _user_system(kind)
    hc._watch(r, system)
    state = hc._state(r, device)
    calls = hc._run(r, _ops(system, state, device))
    assert not [c for c in calls if c.startswith("raises")], calls
    rm_calls = [c for c in calls if "riemannian" in c and "workspace" not in c]
    symbols = {c.split("(")[0] for c in rm_calls}
    want = {"mb200_hamiltonian_riemannian_user", "mb200_dh_dmom_riemannian_user",
            "mb200_implicit_leapfrog_riemannian_user", "mb200_implicit_midpoint_riemannian_user"}
    if device == "cuda":
        want.add("mb200_sample_momentum_riemannian_user")
    assert symbols == want, symbols
    rmetric = (f"rmetric={USER_DIAG}/2 {{0: 2.0, 1: 3.0}} raux=@sys.rmetric_aux" if kind == "diagonal"
               else f"rmetric={USER_SCALAR}/2 {{0: 1.0, 1: 0.25}} raux=NULL")
    for c in rm_calls:
        assert f"Model(target=64/1 {{0: 0.5}} aux=@sys.target_aux {rmetric})" in c, c
        # the handle appended is the pair's image, never the target's own
        assert c.endswith(", @stream, @pair)"), c


# -------------------------------------------------------------------------------------- routing

INVALID, CUDA = -1, -3


@pytest.fixture(scope="module")
def lib():
    import os

    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge

        ge.build()
    return _lib.load()


BUF = np.zeros(64)
PTR = BUF.ctypes.data


def _handle(rmetric_id):
    """A stand-in for a loaded image: the library's handle layout (api_euclid.cu UserKernels)
    starts with the library handle, then the Riemannian kernel table, whose first field is the
    rmetric id the image serves; every kernel pointer is NULL, so a routed call fails at launch."""
    h = np.zeros(32, dtype=np.uint64)
    h.view(np.int32)[2] = rmetric_id
    return h


def _model(target, rmetric):
    m = _lib.Model()
    m.target_id, m.rmetric_id = target, rmetric
    m.rmetric_params[0], m.rmetric_params[1] = 1.0, 0.5
    return m


def _call(lib, op, m, handle, dim=8):
    n = 4
    h = None if handle is None else handle.ctypes.data
    if op in ("leapfrog", "midpoint"):
        args = [PTR, PTR, PTR, PTR, None, n, dim, 0.1, None, 1, None, ctypes.byref(m), 0, 1e-9,
                1e10, 100, 2e-8, PTR, PTR, PTR, PTR]
        if op == "leapfrog":
            rc = lib.mb200_implicit_leapfrog_riemannian_user(*args, None, 0, None, h)
        else:
            rc = lib.mb200_implicit_midpoint_riemannian_user(*args, None, h)
    elif op == "hamiltonian":
        rc = lib.mb200_hamiltonian_riemannian_user(PTR, PTR, n, dim, ctypes.byref(m), PTR, PTR,
                                                   None, 0, None, h)
    else:
        rc = getattr(lib, f"mb200_{op}_riemannian_user")(PTR, PTR, PTR, n, dim, ctypes.byref(m),
                                                        PTR, None, h)
    return rc, lib.mb200_last_error().decode()


OPS = ("leapfrog", "midpoint", "hamiltonian", "sample_momentum", "dh_dmom")
needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(),
                                  reason="routed calls would launch kernels on host pointers")


@needs_no_gpu
@pytest.mark.parametrize("op", OPS)
def test_user_twins_refuse_wrong_models_and_handles(lib, op):
    cases = [
        (_model(1, USER_DIAG), _handle(USER_DIAG), "user-image entry point needs target_id"),
        (_model(64, USER_SCALAR), _handle(USER_DIAG), "rmetric_id 33 does not match"),
        (_model(64, 4), _handle(USER_DIAG), "rmetric_id 4 does not match"),
        (_model(64, USER_DIAG), _handle(0), "user image has no Riemannian kernels"),
        (_model(64, USER_DIAG), None, "user_image is NULL"),
    ]
    for m, h, msg in cases:
        rc, err = _call(lib, op, m, h)
        assert rc == INVALID and err.startswith(msg), (op, rc, err)


@needs_no_gpu
@pytest.mark.parametrize("op", OPS)
def test_routed_user_calls_fail_only_at_their_first_cuda_call(lib, op):
    kernel = {"sample_momentum": "riemannian_sample_momentum_kernel",
              "dh_dmom": "riemannian_velocity_kernel"}.get(op, "implicit_leapfrog_kernel")
    for rmetric in (USER_DIAG, USER_SCALAR):
        rc, err = _call(lib, op, _model(64, rmetric), _handle(rmetric))
        assert rc == CUDA, (op, rc, err)
        assert err.startswith("smem attr") or err.startswith(kernel), err


@needs_no_gpu
@pytest.mark.parametrize("op", OPS)
def test_user_metric_ids_stay_unknown_on_the_registry_entry_points(lib, op):
    from test_dispatch_routing import riemannian_call

    for target in (0, 1, 64):
        for rmetric in (USER_DIAG, USER_SCALAR):
            rc, err = riemannian_call(lib, op, _model(target, rmetric), 8)
            assert rc == INVALID and err == f"unknown rmetric_id {rmetric}", (rc, err)


@needs_no_gpu
def test_euclidean_and_constrained_entry_points_refuse_a_riemannian_handle(lib):
    m = _model(64, 0)
    h = _handle(USER_DIAG).ctypes.data
    rc = lib.mb200_hamiltonian_euclidean_user(PTR, PTR, 4, 8, 0, None, ctypes.byref(m), PTR, None, h)
    assert rc == INVALID and lib.mb200_last_error().decode().startswith("a Riemannian user image")
    rc = lib.mb200_euclidean_eval_user(PTR, PTR, 4, 8, 0, None, ctypes.byref(m), PTR, PTR, PTR, PTR,
                                       None, h)
    assert rc == INVALID and lib.mb200_last_error().decode().startswith("a Riemannian user image")
    rc = lib.mb200_project_onto_cotangent_space_user(PTR, PTR, PTR, 4, 8, 0, None, ctypes.byref(m),
                                                     None, h)
    assert rc == INVALID and "no constraint kernels" in lib.mb200_last_error().decode()


def test_workspace_query_is_zero_for_user_metrics(lib):
    for rmetric in (USER_DIAG, USER_SCALAR):
        assert lib.mb200_implicit_workspace_bytes(4, 8, ctypes.byref(_model(64, rmetric))) == 0


def test_loader_checks_its_arguments(lib):
    h = ctypes.c_void_p()
    names = (ctypes.c_char_p * 3)(b"a", b"b", b"c")
    assert lib.mb200_user_riemannian_load(b"x", 1, names, 2, USER_DIAG, ctypes.byref(h)) == INVALID
    assert lib.mb200_user_riemannian_load(b"x", 1, names, 3, 4, ctypes.byref(h)) == INVALID
    assert "rmetric_id must be" in lib.mb200_last_error().decode()
