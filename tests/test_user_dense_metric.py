"""User-written dense metrics on DenseRiemannianMetricSystem, without a GPU: NVRTC compilation of
the dense image, compile errors, the system's constructor rules, the image cache, copies, the
library calls the system, the implicit leapfrog, HMC and lock-step NUTS make, and the C entry
points' refusals and workspace query."""

import copy
import ctypes
import pickle
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import test_host_calls as hc
from mici_b200 import _lib, integrators, jit, systems, transitions
from mici_b200.errors import TargetCompileError
from mici_b200.targets import (
    CudaDenseMetric,
    CudaDiagonalMetric,
    CudaRiemannianPair,
    CudaScalarMetric,
    CudaTarget,
    HadamardMetric,
    Quadratic,
    Rank1Metric,
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
from user_dense_metric_sources import (
    COMPILE_PAIRS,
    HADAMARD_DENSE,
    LGCP,
    LGCP_METRIC,
    QUADRATIC,
    RANK1_DENSE,
)
from user_riemannian_sources import FUNNEL_FISHER, QUADRATIC_SCALAR

USER_DENSE, USER_DIAG = 34, 32


# ---------------------------------------------------------------------------------- compilation

def test_test_models_compile_to_sm90a_images_with_the_three_dense_kernels():
    def build(item):
        name, (tsrc, msrc) = item
        return name, jit.compile_target(tsrc, "t_" + name, metric=("dense", msrc, "m_" + name))

    with ThreadPoolExecutor(len(COMPILE_PAIRS)) as pool:
        images = dict(pool.map(build, COMPILE_PAIRS.items()))
    for _, cubin, names in images.values():
        assert cubin[:4] == b"\x7fELF"
        assert int.from_bytes(cubin[0x30:0x34], "little") & 0xFF == 90  # sm_90(a)
        assert len(names) == 3 and _elf_symbols(cubin) >= set(names)
        assert ["implicit_leapfrog" in names[0], "velocity" in names[1],
                "sample_momentum" in names[2]] == [True] * 3
        assert all("UserRTargetCta" in n and "UserDenseMetric" in n for n in names)
        # the library's self-test kernel stays out of the user image
        assert not any("selftest" in s for s in _elf_symbols(cubin))


def test_missing_vjp_metric_dense_is_a_compile_error_at_the_end_of_the_metric_source():
    src = LGCP_METRIC.replace("vjp_metric_dense(", "other_vjp(")
    with pytest.raises(TargetCompileError) as e:
        jit.compile_target(LGCP, "lgcp", metric=("dense", src, "lgcp_no_vjp"))
    assert "vjp_metric_dense" in e.value.log
    assert f"lgcp_no_vjp.cu({len(src.splitlines()) + 1})" in e.value.log


def test_a_warp_contract_metric_function_does_not_compile_as_a_dense_metric():
    src = (
        "__device__ void metric_dense(const mb200::Chain& c, double* M, int ld) {\n"
        "  for (int i = c.lane; i < c.dim; i += 32) M[i * ld + i] = 1.0;\n"
        "}\n"
        "__device__ void vjp_metric_dense(const mb200::CtaChain& c, const double* V, int ld,\n"
        "                                 double* out) {\n"
        "  for (int k = c.lane; k < c.dim; k += c.n_lanes) out[k] = 0.0;\n"
        "}\n")
    with pytest.raises(TargetCompileError) as e:
        jit.compile_target(LGCP, "lgcp", metric=("dense", src, "lgcp_warp_fill"))
    assert '"const mb200::CtaChain" to "const mb200::Chain"' in e.value.log
    assert f"lgcp_warp_fill.cu({len(src.splitlines()) + 1})" in e.value.log


# ---------------------------------------------------------------------------- constructor rules

def _target(dim=6, **kw):
    return CudaTarget(dim, QUADRATIC, aux=np.identity(dim), **kw)


def _dense(**kw):
    return CudaDenseMetric(HADAMARD_DENSE, **kw)


def test_dense_user_metric_is_accepted_with_an_unconstrained_cuda_target():
    s = systems.DenseRiemannianMetricSystem(_target(), _dense(params=(0.5,), aux=np.ones(72)))
    assert s._rmetric_id == USER_DENSE and isinstance(s._user_pair, CudaRiemannianPair)
    assert s._user_pair.metric.kind == "dense" and s._rmetric_params == (0.5,)
    assert np.array_equal(s._rmetric_aux, np.ones(72))
    # registry models are unchanged
    s = systems.DenseRiemannianMetricSystem(Quadratic(np.identity(3)),
                                            HadamardMetric(np.identity(3), np.ones((3, 3)), 0.1))
    assert s._user_pair is None and not s._user_targets


def test_dimension_limit_is_576():
    systems.DenseRiemannianMetricSystem(CudaTarget(576, QUADRATIC), _dense())
    with pytest.raises(ValueError, match="576"):
        systems.DenseRiemannianMetricSystem(CudaTarget(577, QUADRATIC), _dense())


@pytest.mark.parametrize("make", [
    # a user dense metric with a registry target
    lambda: systems.DenseRiemannianMetricSystem(Quadratic(np.identity(3)), _dense()),
    # a diagonal or scalar user metric on the dense system
    lambda: systems.DenseRiemannianMetricSystem(_target(), CudaDiagonalMetric(FUNNEL_FISHER)),
    lambda: systems.DenseRiemannianMetricSystem(_target(), CudaScalarMetric(QUADRATIC_SCALAR)),
    # a dense user metric on the other systems
    lambda: systems.DiagonalRiemannianMetricSystem(_target(), _dense()),
    lambda: systems.ScalarRiemannianMetricSystem(_target(), _dense()),
    # a constrained CudaTarget
    lambda: systems.DenseRiemannianMetricSystem(_target(n_constr=1), _dense()),
])
def test_refused_pairs_raise_type_error(make):
    with pytest.raises(TypeError):
        make()


def test_unchanged_messages():
    with pytest.raises(TypeError, match="does not take a CudaTarget: user targets run on "
                                        "EuclideanMetricSystem"):
        systems.DenseRiemannianMetricSystem(_target(3), Rank1Metric(np.identity(3), 0.1))
    with pytest.raises(ValueError, match="The metric VJP is fused into the kernels."):
        systems.DenseRiemannianMetricSystem(_target(), _dense(), vjp_metric_func=lambda q: q)


def test_metric_constructor_validation():
    with pytest.raises(ValueError):
        CudaDenseMetric(42)
    with pytest.raises(ValueError):
        CudaDenseMetric(HADAMARD_DENSE, params=range(9))
    with pytest.raises(ValueError):
        CudaDenseMetric(HADAMARD_DENSE, name="not an identifier")
    m = CudaDenseMetric(HADAMARD_DENSE, params=range(8), aux=[[1, 2]])
    assert m.params == tuple(float(i) for i in range(8)) and m.aux.dtype == np.float64
    assert m.kind == "dense" and m.rmetric_id == USER_DENSE


# ----------------------------------------------------------------------------------- cache keys

def test_cache_keys_keep_the_metric_kind(monkeypatch):
    compiled = []

    def fake(source, name, constraint=(), metric=()):
        compiled.append((name, metric))
        return b"\x7fELF-stub", ("k0", "k1", "k2")

    monkeypatch.setattr(jit, "_compile", fake)
    src = QUADRATIC + "\n// dense cache probe\n"
    diag = ("diagonal", RANK1_DENSE, "m")
    dense = ("dense", RANK1_DENSE, "m")
    other = ("dense", HADAMARD_DENSE, "m")
    for metric in (diag, dense, other):
        jit.compile_target(src, "t", metric=metric)
    before = dict(jit.stats)
    jit.compile_target(src, "t", metric=dense)  # repeat: a hit
    assert jit.stats["hits"] == before["hits"] + 1 and len(compiled) == 3
    keys = {jit.cache_key(src, "t", (), jit._metric(m)) for m in (diag, dense, other)}
    assert len(keys) == 3


def test_dense_translation_unit_and_kernel_names():
    tu = jit.translation_unit(QUADRATIC, "t", metric=("dense", LGCP_METRIC, "m"))
    assert tu.endswith(f'#line {len(LGCP_METRIC.splitlines()) + 1} "m.cu"\n'
                       "MB200_USER_METRIC_FUNCTIONS\n")
    assert jit._defines((), ("dense", LGCP_METRIC, "m")) == ("-DMB200_USER_DENSE_METRIC",)
    assert jit.riemannian_name_expressions("dense") == (
        "&mb200::implicit_leapfrog_kernel<mb200::UserRTargetCta, mb200::UserDenseMetric>",
        "&mb200::riemannian_velocity_kernel<mb200::UserRTargetCta, mb200::UserDenseMetric>",
        "&mb200::riemannian_sample_momentum_kernel<mb200::UserRTargetCta, mb200::UserDenseMetric>")
    assert jit.RIEMANNIAN_RMETRIC_IDS["dense"] == USER_DENSE


# --------------------------------------------------------------------------------------- copies

def test_system_and_integrator_survive_deepcopy_and_pickle():
    t = _target(name="quad")
    m = _dense(params=(0.5,), aux=np.ones(72), name="had")
    integ = integrators.ImplicitLeapfrogIntegrator(systems.DenseRiemannianMetricSystem(t, m), 0.1)
    for clone in (copy.deepcopy(integ), pickle.loads(pickle.dumps(integ))):
        s = clone.system
        assert isinstance(s, systems.DenseRiemannianMetricSystem)
        assert s.target.source == t.source and s.metric_model.source == m.source
        assert s.metric_model.name == "had" and np.array_equal(s.metric_model.aux, m.aux)
        assert s._user_pair.metric.kind == "dense"
        assert s._rmetric_id == USER_DENSE and s._rmetric_params == (0.5,)


# ------------------------------------------------------------------------------- recorded calls

def test_every_dense_call_goes_to_the_user_twin_with_the_pair_image(rec):  # noqa: F811
    device = "cuda" if torch.cuda.is_available() else "cpu"
    r = rec(device)
    t = CudaTarget(hc.DIM, QUADRATIC, aux=np.identity(hc.DIM))
    system = systems.DenseRiemannianMetricSystem(t, _dense(params=(0.25,), aux=np.ones(4)))
    hc._watch(r, system)
    state = hc._state(r, device)
    integ = integrators.ImplicitLeapfrogIntegrator(system, 0.1)
    ops = [lambda: system.h(state), lambda: system.dh_dmom(state),
           lambda: integ.step_n(state, 2),
           lambda: transitions.MetropolisRandomIntegrationTransition(
               system, integ, (1, 3)).sample(state, np.random.default_rng(0)),
           lambda: transitions.MultinomialDynamicIntegrationTransition(
               system, integ, max_tree_depth=2).sample(state, np.random.default_rng(0))]
    if device == "cuda":
        ops.append(lambda: system.sample_momentum(state, np.random.default_rng(0)))
    calls = hc._run(r, ops)
    assert not [c for c in calls if c.startswith("raises")], calls
    rm_calls = [c for c in calls if "riemannian" in c and "workspace" not in c]
    symbols = {c.split("(")[0] for c in rm_calls}
    want = {"mb200_hamiltonian_riemannian_user", "mb200_dh_dmom_riemannian_user",
            "mb200_implicit_leapfrog_riemannian_user"}
    if device == "cuda":
        want.add("mb200_sample_momentum_riemannian_user")
    assert symbols == want, symbols
    for c in rm_calls:
        assert (f"Model(target=64/0 {{}} aux=@sys.target_aux "
                f"rmetric={USER_DENSE}/1 {{0: 0.25}} raux=@sys.rmetric_aux)") in c, c
        assert c.endswith(", @stream, @pair)"), c


# ------------------------------------------------------------------------------------ C entry

OPS = ("leapfrog", "midpoint", "hamiltonian", "sample_momentum", "dh_dmom")


@needs_no_gpu
@pytest.mark.parametrize("op", OPS)
def test_dense_image_refusals_launch_nothing(lib, op):  # noqa: F811
    cases = [
        (_model(1, USER_DENSE), _handle(USER_DENSE), "user-image entry point needs target_id"),
        (_model(64, USER_DIAG), _handle(USER_DENSE), "rmetric_id 32 does not match"),
        (_model(64, USER_DENSE), _handle(USER_DIAG), "rmetric_id 34 does not match"),
    ]
    for m, h, msg in cases:
        rc, err = _call(lib, op, m, h)
        assert rc == INVALID and err.startswith(msg), (op, rc, err)
    rc, err = _call(lib, op, _model(64, USER_DENSE), _handle(USER_DENSE), dim=577)
    if op == "midpoint":
        assert rc == -2 and err.startswith("implicit midpoint is not available"), (rc, err)
    else:
        assert rc == -2 and err == "dim 577: panel buffers exceed shared memory", (rc, err)


@needs_no_gpu
def test_midpoint_on_a_dense_image_is_unsupported(lib):  # noqa: F811
    rc, err = _call(lib, "midpoint", _model(64, USER_DENSE), _handle(USER_DENSE))
    assert rc == -2 and err == ("implicit midpoint is not available for the global-workspace "
                                "dense metric"), (rc, err)


@needs_no_gpu
@pytest.mark.parametrize("op", ("leapfrog", "hamiltonian", "sample_momentum", "dh_dmom"))
def test_routed_dense_calls_fail_only_at_their_first_cuda_call(lib, op):  # noqa: F811
    """The global-workspace launch plan: the implicit kernel's first CUDA call is its shared-memory
    attribute, the vector kernels' the workspace allocation."""
    rc, err = _call(lib, op, _model(64, USER_DENSE), _handle(USER_DENSE))
    first = "smem attr" if op in ("leapfrog", "hamiltonian") else "dense metric workspace"
    assert rc == CUDA and err.startswith(first), (op, rc, err)


@needs_no_gpu
@pytest.mark.parametrize("op", OPS)
def test_dense_id_stays_unknown_on_the_registry_entry_points(lib, op):  # noqa: F811
    from test_dispatch_routing import riemannian_call

    for target in (0, 1, 64):
        rc, err = riemannian_call(lib, op, _model(target, USER_DENSE), 8)
        assert rc == INVALID and err == f"unknown rmetric_id {USER_DENSE}", (rc, err)


@needs_no_gpu
def test_euclidean_entry_points_refuse_a_dense_handle(lib):  # noqa: F811
    m = _model(64, 0)
    h = _handle(USER_DENSE).ctypes.data
    rc = lib.mb200_hamiltonian_euclidean_user(PTR, PTR, 4, 8, 0, None, ctypes.byref(m), PTR, None, h)
    assert rc == INVALID and lib.mb200_last_error().decode().startswith("a Riemannian user image")


def test_workspace_query_for_the_dense_id(lib):  # noqa: F811
    """dense_global_workspace_bytes: one CTA per chain up to one per SM (4 chains take 4 on any
    GPU), each with L, X and M^-1 [np x np] and the W_kk blocks [np x 32], np = dim padded to 32."""
    ws = lib.mb200_implicit_workspace_bytes
    m = ctypes.byref(_model(64, USER_DENSE))

    def per_cta(np_):
        return 8 * (3 * np_ * np_ + np_ * 32)

    assert ws(4, 8, m) == 4 * per_cta(32)
    assert ws(4, 576, m) == 4 * per_cta(576)
    assert ws(4, 577, m) == 0
    for rmetric in (32, 33):
        assert ws(4, 8, ctypes.byref(_model(64, rmetric))) == 0


@needs_no_gpu
def test_loader_accepts_the_dense_id(lib):  # noqa: F811
    h = ctypes.c_void_p()
    names = (ctypes.c_char_p * 3)(b"a", b"b", b"c")
    # the arguments pass; loading the (not loadable) image is the first CUDA call
    assert lib.mb200_user_riemannian_load(b"x", 1, names, 3, USER_DENSE, ctypes.byref(h)) == CUDA
    assert lib.mb200_last_error().decode().startswith("cudaLibraryLoadData")
