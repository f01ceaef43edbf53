"""User-written Cholesky-factor metrics on CholeskyFactoredRiemannianMetricSystem, without a GPU:
NVRTC compilation of the Cholesky image, compile errors, the system's constructor rules, the image
cache, copies, the library calls the system, both implicit integrators, HMC and lock-step NUTS
make, and the C entry points' refusals and workspace query."""

import copy
import ctypes
import pickle
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import test_host_calls as hc
from mici_b200 import integrators, jit, systems, transitions
from mici_b200.errors import TargetCompileError
from mici_b200.targets import (
    CudaCholeskyMetric,
    CudaDenseMetric,
    CudaDiagonalMetric,
    CudaRiemannianPair,
    CudaScalarMetric,
    CudaTarget,
    QuadraticCholeskyMetric,
    StdGaussian,
)

from test_user_riemannian import (  # noqa: F401  (rec: the recording-library fixture)
    CUDA,
    INVALID,
    PTR,
    _call,
    _handle,
    _model,
    lib,
    needs_no_gpu,
    rec,
)
from test_user_target import _elf_symbols
from user_chol_metric_sources import AR1_HIER, AR1_HIER_CHOL, COMPILE_PAIRS, QUADRATIC, QUADRATIC_CHOL
from user_dense_metric_sources import HADAMARD_DENSE
from user_riemannian_sources import FUNNEL_FISHER, QUADRATIC_SCALAR

USER_CHOL, USER_DENSE, USER_DIAG = 35, 34, 32
UNSUPPORTED = -2


# ---------------------------------------------------------------------------------- compilation

def test_test_models_compile_to_sm90a_images_with_the_three_cholesky_kernels():
    def build(item):
        name, (tsrc, msrc) = item
        return name, jit.compile_target(tsrc, "t_" + name, metric=("cholesky", msrc, "m_" + name))

    with ThreadPoolExecutor(len(COMPILE_PAIRS)) as pool:
        images = dict(pool.map(build, COMPILE_PAIRS.items()))
    for _, cubin, names in images.values():
        assert cubin[:4] == b"\x7fELF"
        assert int.from_bytes(cubin[0x30:0x34], "little") & 0xFF == 90  # sm_90(a)
        assert len(names) == 3 and _elf_symbols(cubin) >= set(names)
        assert ["implicit_leapfrog" in names[0], "velocity" in names[1],
                "sample_momentum" in names[2]] == [True] * 3
        assert all("UserRTargetCta" in n and "UserCholeskyMetric" in n for n in names)
        assert not any("selftest" in s for s in _elf_symbols(cubin))


def test_missing_vjp_metric_chol_is_a_compile_error_at_the_end_of_the_metric_source():
    src = AR1_HIER_CHOL.replace("vjp_metric_chol(", "other_vjp(")
    with pytest.raises(TargetCompileError) as e:
        jit.compile_target(AR1_HIER, "ar1", metric=("cholesky", src, "ar1_no_vjp"))
    assert "vjp_metric_chol" in e.value.log
    assert f"ar1_no_vjp.cu({len(src.splitlines()) + 1})" in e.value.log


def test_a_warp_contract_metric_function_does_not_compile_as_a_cholesky_metric():
    src = (
        "__device__ void metric_chol(const mb200::Chain& c, double* L, int ld) {\n"
        "  for (int i = c.lane; i < c.dim; i += 32) L[i * ld + i] = 1.0;\n"
        "}\n"
        "__device__ void vjp_metric_chol(const mb200::CtaChain& c, const double* V, int ld,\n"
        "                                double* out) {\n"
        "  for (int k = c.lane; k < c.dim; k += c.n_lanes) out[k] = 0.0;\n"
        "}\n")
    with pytest.raises(TargetCompileError) as e:
        jit.compile_target(QUADRATIC, "quad", metric=("cholesky", src, "chol_warp_fill"))
    assert '"const mb200::CtaChain" to "const mb200::Chain"' in e.value.log
    assert f"chol_warp_fill.cu({len(src.splitlines()) + 1})" in e.value.log


# ---------------------------------------------------------------------------- constructor rules

def _target(dim=6, **kw):
    return CudaTarget(dim, QUADRATIC, aux=np.identity(dim), **kw)


def _chol(**kw):
    return CudaCholeskyMetric(QUADRATIC_CHOL, **kw)


def test_cholesky_user_metric_is_accepted_with_an_unconstrained_cuda_target():
    s = systems.CholeskyFactoredRiemannianMetricSystem(_target(),
                                                       _chol(params=(0.5,), aux=np.ones(36)))
    assert s._rmetric_id == USER_CHOL and isinstance(s._user_pair, CudaRiemannianPair)
    assert s._user_pair.metric.kind == "cholesky" and s._rmetric_params == (0.5,)
    assert np.array_equal(s._rmetric_aux, np.ones(36))
    # the user metric has no base factor to check against the target's dimension
    systems.CholeskyFactoredRiemannianMetricSystem(_target(9), _chol(aux=np.ones(4)))
    # registry models are unchanged, the base-factor size check included
    s = systems.CholeskyFactoredRiemannianMetricSystem(StdGaussian(3),
                                                       QuadraticCholeskyMetric(np.identity(3), 0.1))
    assert s._user_pair is None and not s._user_targets
    with pytest.raises(ValueError, match="The base factor is 2 x 2"):
        systems.CholeskyFactoredRiemannianMetricSystem(StdGaussian(3),
                                                       QuadraticCholeskyMetric(np.identity(2), 0.1))


def test_dimension_limit_is_1016():
    systems.CholeskyFactoredRiemannianMetricSystem(CudaTarget(1016, QUADRATIC), _chol())
    with pytest.raises(ValueError, match="dim <= 1016, got 1017"):
        systems.CholeskyFactoredRiemannianMetricSystem(CudaTarget(1017, QUADRATIC), _chol())


@pytest.mark.parametrize("make", [
    # a user Cholesky metric with a registry target
    lambda: systems.CholeskyFactoredRiemannianMetricSystem(StdGaussian(3), _chol()),
    # the other user metrics on the Cholesky system
    lambda: systems.CholeskyFactoredRiemannianMetricSystem(_target(), CudaDiagonalMetric(FUNNEL_FISHER)),
    lambda: systems.CholeskyFactoredRiemannianMetricSystem(_target(), CudaScalarMetric(QUADRATIC_SCALAR)),
    lambda: systems.CholeskyFactoredRiemannianMetricSystem(_target(), CudaDenseMetric(HADAMARD_DENSE)),
    # a Cholesky user metric on the other systems
    lambda: systems.DenseRiemannianMetricSystem(_target(), _chol()),
    lambda: systems.DiagonalRiemannianMetricSystem(_target(), _chol()),
    lambda: systems.ScalarRiemannianMetricSystem(_target(), _chol()),
    # a constrained CudaTarget
    lambda: systems.CholeskyFactoredRiemannianMetricSystem(_target(n_constr=1), _chol()),
])
def test_refused_pairs_raise_type_error(make):
    with pytest.raises(TypeError):
        make()


def test_unchanged_messages():
    with pytest.raises(TypeError, match="does not take a CudaTarget: user targets run on "
                                        "EuclideanMetricSystem"):
        systems.CholeskyFactoredRiemannianMetricSystem(
            _target(3), QuadraticCholeskyMetric(np.identity(3), 0.1))
    with pytest.raises(ValueError, match="The metric VJP is fused into the kernels."):
        systems.CholeskyFactoredRiemannianMetricSystem(_target(), _chol(),
                                                       vjp_metric_chol_func=lambda q: q)


def test_metric_constructor_validation():
    with pytest.raises(ValueError):
        CudaCholeskyMetric(42)
    with pytest.raises(ValueError):
        CudaCholeskyMetric(QUADRATIC_CHOL, params=range(9))
    with pytest.raises(ValueError):
        CudaCholeskyMetric(QUADRATIC_CHOL, name="not an identifier")
    m = CudaCholeskyMetric(QUADRATIC_CHOL, params=range(8), aux=[[1, 2]])
    assert m.params == tuple(float(i) for i in range(8)) and m.aux.dtype == np.float64
    assert m.kind == "cholesky" and m.rmetric_id == USER_CHOL


# ----------------------------------------------------------------------------------- cache keys

def test_cache_keys_keep_the_metric_kind(monkeypatch):
    compiled = []

    def fake(source, name, constraint=(), metric=()):
        compiled.append((name, metric))
        return b"\x7fELF-stub", ("k0", "k1", "k2")

    monkeypatch.setattr(jit, "_compile", fake)
    src = QUADRATIC + "\n// cholesky cache probe\n"
    dense = ("dense", QUADRATIC_CHOL, "m")
    chol = ("cholesky", QUADRATIC_CHOL, "m")
    other = ("cholesky", AR1_HIER_CHOL, "m")
    for metric in (dense, chol, other):
        jit.compile_target(src, "t", metric=metric)
    before = dict(jit.stats)
    jit.compile_target(src, "t", metric=chol)  # repeat: a hit
    assert jit.stats["hits"] == before["hits"] + 1 and len(compiled) == 3
    keys = {jit.cache_key(src, "t", (), jit._metric(m)) for m in (dense, chol, other)}
    assert len(keys) == 3


def test_cholesky_translation_unit_and_kernel_names():
    tu = jit.translation_unit(QUADRATIC, "t", metric=("cholesky", AR1_HIER_CHOL, "m"))
    assert tu.endswith(f'#line {len(AR1_HIER_CHOL.splitlines()) + 1} "m.cu"\n'
                       "MB200_USER_METRIC_FUNCTIONS\n")
    assert jit._defines((), ("cholesky", AR1_HIER_CHOL, "m")) == ("-DMB200_USER_CHOLESKY_METRIC",)
    t, m = "mb200::UserRTargetCta", "mb200::UserCholeskyMetric"
    assert jit.riemannian_name_expressions("cholesky") == (
        f"&mb200::implicit_leapfrog_kernel<{t}, {m}>",
        f"&mb200::riemannian_velocity_kernel<{t}, {m}>",
        f"&mb200::riemannian_sample_momentum_kernel<{t}, {m}>")
    assert jit.RIEMANNIAN_RMETRIC_IDS["cholesky"] == USER_CHOL


# --------------------------------------------------------------------------------------- copies

def test_system_and_integrator_survive_deepcopy_and_pickle():
    t = _target(name="quad")
    m = _chol(params=(0.5,), aux=np.ones(36), name="qchol")
    for cls in (integrators.ImplicitLeapfrogIntegrator, integrators.ImplicitMidpointIntegrator):
        integ = cls(systems.CholeskyFactoredRiemannianMetricSystem(t, m), 0.1)
        for clone in (copy.deepcopy(integ), pickle.loads(pickle.dumps(integ))):
            s = clone.system
            assert isinstance(s, systems.CholeskyFactoredRiemannianMetricSystem)
            assert s.target.source == t.source and s.metric_model.source == m.source
            assert s.metric_model.name == "qchol" and np.array_equal(s.metric_model.aux, m.aux)
            assert s._user_pair.metric.kind == "cholesky"
            assert s._rmetric_id == USER_CHOL and s._rmetric_params == (0.5,)


# ------------------------------------------------------------------------------- recorded calls

def test_every_cholesky_call_goes_to_the_user_twin_with_the_pair_image(rec):  # noqa: F811
    device = "cuda" if torch.cuda.is_available() else "cpu"
    r = rec(device)
    t = CudaTarget(hc.DIM, QUADRATIC, aux=np.identity(hc.DIM))
    system = systems.CholeskyFactoredRiemannianMetricSystem(
        t, _chol(params=(0.25,), aux=np.identity(hc.DIM)))
    hc._watch(r, system)
    state = hc._state(r, device)
    leapfrog = integrators.ImplicitLeapfrogIntegrator(system, 0.1)
    midpoint = integrators.ImplicitMidpointIntegrator(system, 0.1)
    ops = [lambda: system.h(state), lambda: system.dh_dmom(state),
           lambda: leapfrog.step_n(state, 2), lambda: midpoint.step_n(state, 2),
           lambda: transitions.MetropolisRandomIntegrationTransition(
               system, leapfrog, (1, 3)).sample(state, np.random.default_rng(0)),
           lambda: transitions.MultinomialDynamicIntegrationTransition(
               system, leapfrog, max_tree_depth=2).sample(state, np.random.default_rng(0))]
    if device == "cuda":
        ops.append(lambda: system.sample_momentum(state, np.random.default_rng(0)))
    calls = hc._run(r, ops)
    assert not [c for c in calls if c.startswith("raises")], calls
    rm_calls = [c for c in calls if "riemannian" in c and "workspace" not in c]
    symbols = {c.split("(")[0] for c in rm_calls}
    want = {"mb200_hamiltonian_riemannian_user", "mb200_dh_dmom_riemannian_user",
            "mb200_implicit_leapfrog_riemannian_user", "mb200_implicit_midpoint_riemannian_user"}
    if device == "cuda":
        want.add("mb200_sample_momentum_riemannian_user")
    assert symbols == want, symbols
    for c in rm_calls:
        assert (f"Model(target=64/0 {{}} aux=@sys.target_aux "
                f"rmetric={USER_CHOL}/1 {{0: 0.25}} raux=@sys.rmetric_aux)") in c, c
        assert c.endswith(", @stream, @pair)"), c


# ------------------------------------------------------------------------------------ C entry

OPS = ("leapfrog", "midpoint", "hamiltonian", "sample_momentum", "dh_dmom")


@needs_no_gpu
@pytest.mark.parametrize("op", OPS)
def test_cholesky_image_refusals_launch_nothing(lib, op):  # noqa: F811
    cases = [
        # a registry target
        (_model(1, USER_CHOL), _handle(USER_CHOL), "user-image entry point needs target_id"),
        # mismatched rmetric ids, both ways
        (_model(64, USER_DENSE), _handle(USER_CHOL), "rmetric_id 34 does not match"),
        (_model(64, USER_CHOL), _handle(USER_DIAG), "rmetric_id 35 does not match"),
        # a Euclidean or constrained image (no Riemannian kernels)
        (_model(64, USER_CHOL), _handle(0), "user image has no Riemannian kernels"),
    ]
    for m, h, msg in cases:
        rc, err = _call(lib, op, m, h)
        assert rc == INVALID and err.startswith(msg), (op, rc, err)
    rc, err = _call(lib, op, _model(64, USER_CHOL), _handle(USER_CHOL), dim=1017)
    assert rc == UNSUPPORTED and err == "dim 1017 too large", (op, rc, err)


@needs_no_gpu
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("dim", [8, 113, 1016])
def test_routed_cholesky_calls_fail_only_at_their_first_cuda_call(lib, op, dim):  # noqa: F811
    """Both integrators are routed; the first CUDA call of the launch plan is the kernel's
    shared-memory attribute, on both sides of the shared-memory / workspace crossover."""
    rc, err = _call(lib, op, _model(64, USER_CHOL), _handle(USER_CHOL), dim=dim)
    assert rc == CUDA and err.startswith("smem attr"), (op, rc, err)


@needs_no_gpu
@pytest.mark.parametrize("op", OPS)
def test_cholesky_id_stays_unknown_on_the_registry_entry_points(lib, op):  # noqa: F811
    from test_dispatch_routing import riemannian_call

    for target in (0, 1, 64):
        rc, err = riemannian_call(lib, op, _model(target, USER_CHOL), 8)
        assert rc == INVALID and err == f"unknown rmetric_id {USER_CHOL}", (rc, err)


@needs_no_gpu
def test_euclidean_entry_points_refuse_a_cholesky_handle(lib):  # noqa: F811
    m = _model(64, 0)
    h = _handle(USER_CHOL).ctypes.data
    rc = lib.mb200_hamiltonian_euclidean_user(PTR, PTR, 4, 8, 0, None, ctypes.byref(m), PTR, None, h)
    assert rc == INVALID and lib.mb200_last_error().decode().startswith("a Riemannian user image")


def test_workspace_query_for_the_cholesky_id_is_zero(lib):  # noqa: F811
    """The library allocates the per-CTA workspace of the Cholesky-factored policy itself."""
    ws = lib.mb200_implicit_workspace_bytes
    for dim in (8, 112, 113, 1016, 1017):
        assert ws(4, dim, ctypes.byref(_model(64, USER_CHOL))) == 0


@needs_no_gpu
def test_loader_accepts_the_cholesky_id(lib):  # noqa: F811
    h = ctypes.c_void_p()
    names = (ctypes.c_char_p * 3)(b"a", b"b", b"c")
    # the arguments pass; loading the (not loadable) image is the first CUDA call
    assert lib.mb200_user_riemannian_load(b"x", 1, names, 3, USER_CHOL, ctypes.byref(h)) == CUDA
    assert lib.mb200_last_error().decode().startswith("cudaLibraryLoadData")
    for bad in (31, 36, 6):
        assert lib.mb200_user_riemannian_load(b"x", 1, names, 3, bad, ctypes.byref(h)) == INVALID
