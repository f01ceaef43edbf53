"""User-written targets (``CudaTarget``) without a GPU: NVRTC compilation, compile errors,
validation, the systems that refuse them, and pickling."""

import copy
import pickle

import numpy as np
import pytest

from mici_b200 import integrators, jit, systems
from mici_b200.errors import TargetCompileError
from mici_b200.targets import CudaTarget, QuadraticDiagonalMetric, Sphere

from user_target_sources import ALL_SOURCES, FUNNEL


def _elf_symbols(image):
    """Symbol names of an ELF64 image (the CUBIN), read from its .symtab."""
    import struct

    assert image[:4] == b"\x7fELF" and image[4] == 2
    shoff, = struct.unpack_from("<Q", image, 0x28)
    shentsize, shnum = struct.unpack_from("<HH", image, 0x3A)
    sections = [struct.unpack_from("<IIQQQQIIQQ", image, shoff + i * shentsize) for i in range(shnum)]
    names = set()
    for sh in sections:
        if sh[1] != 2:  # SHT_SYMTAB
            continue
        strtab = sections[sh[6]]
        for off in range(sh[4], sh[4] + sh[5], sh[9]):
            name_off, = struct.unpack_from("<I", image, off)
            end = image.index(b"\0", strtab[4] + name_off)
            names.add(image[strtab[4] + name_off:end].decode())
    return names


@pytest.mark.parametrize("name", list(ALL_SOURCES))
def test_example_sources_compile_to_sm90a_images_with_every_kernel(name):
    _, cubin, names = jit.compile_target(ALL_SOURCES[name], name)
    assert cubin[:4] == b"\x7fELF"
    e_flags = int.from_bytes(cubin[0x30:0x34], "little")
    assert e_flags & 0xFF == 90  # sm_90(a)
    assert len(names) == 10 and len(set(names)) == 10
    assert _elf_symbols(cubin) >= set(names)
    assert all("UserTarget" in n for n in names)


def test_syntax_error_reports_the_user_line():
    src = FUNNEL + "\n__device__ double broken(const mb200::Chain& c) {\n  return c.q[0] + q1;\n}\n"
    with pytest.raises(TargetCompileError) as e:
        jit.compile_target(src, "broken")
    line = FUNNEL.count("\n") + 3
    assert f"broken.cu({line})" in str(e.value)
    assert f"broken.cu({line})" in e.value.log


def test_missing_gradient_is_a_compile_error():
    src = FUNNEL[:FUNNEL.index("__device__ void grad_neg_log_dens")]
    with pytest.raises(TargetCompileError, match="grad_neg_log_dens"):
        jit.compile_target(src, "no_grad")


def test_constructor_validation():
    with pytest.raises(ValueError):
        CudaTarget(0, FUNNEL)
    with pytest.raises(ValueError):
        CudaTarget(1025, FUNNEL)
    with pytest.raises(ValueError):
        CudaTarget(4, FUNNEL, params=range(9))
    with pytest.raises(ValueError):
        CudaTarget(4, FUNNEL, aux=["a", "b"])
    with pytest.raises(ValueError):
        CudaTarget(4, FUNNEL, name="not an identifier")
    t = CudaTarget(1024, FUNNEL, params=range(8), aux=[[1, 2], [3, 4]])
    assert t.aux.dtype == np.float64 and t.params == tuple(float(i) for i in range(8))


def test_systems_without_user_target_support_refuse_it():
    t = CudaTarget(4, FUNNEL)
    for make in (
        lambda: systems.GaussianEuclideanMetricSystem(t),
        lambda: systems.DenseConstrainedEuclideanMetricSystem(t),
        lambda: systems.GaussianDenseConstrainedEuclideanMetricSystem(t),
        lambda: systems.SoftAbsRiemannianMetricSystem(t),
        lambda: systems.DiagonalRiemannianMetricSystem(t, QuadraticDiagonalMetric()),
    ):
        with pytest.raises(TypeError, match="EuclideanMetricSystem"):
            make()
    systems.EuclideanMetricSystem(t)  # accepted
    systems.DenseConstrainedEuclideanMetricSystem(Sphere(4))  # registry targets unchanged


def test_system_and_integrator_survive_deepcopy_and_pickle():
    t = CudaTarget(6, FUNNEL, params=(1.5,), aux=np.arange(3.0), name="funnel")
    system = systems.EuclideanMetricSystem(t, metric=np.linspace(1, 2, 6))
    integ = integrators.LeapfrogIntegrator(system, 0.1)
    for clone in (copy.deepcopy(integ), pickle.loads(pickle.dumps(integ))):
        ct = clone.system.target
        assert isinstance(ct, CudaTarget) and ct.source == t.source and ct.name == "funnel"
        assert ct.params == t.params and np.array_equal(ct.aux, t.aux)
        assert np.array_equal(clone.system.metric.array, system.metric.array)


def test_second_system_from_the_same_source_hits_the_cache():
    src = FUNNEL + "\n// cache probe\n"
    CudaTarget(8, src).compile()
    before = dict(jit.stats)
    CudaTarget(32, src).compile()  # another dimension: same kernels, same image
    assert jit.stats["hits"] == before["hits"] + 1
    assert jit.stats["compiles"] == before["compiles"]


def test_repeat_lookups_do_not_rehash_the_headers(monkeypatch):
    """A user target looks its image up before every launch: after the first compile that is a
    dictionary access, with no header hashing and no NVRTC call."""
    src = FUNNEL + "\n// repeat-lookup probe\n"
    first = jit.compile_target(src, "probe")
    calls = []

    def counted(*a, **k):
        calls.append(1)
        raise AssertionError("headers hashed again")

    monkeypatch.setattr(jit, "_headers_digest", counted)
    monkeypatch.setattr(jit, "_compile", counted)
    monkeypatch.setattr(jit, "version", counted)
    for _ in range(3):
        assert jit.compile_target(src, "probe") == first
    assert not calls


def test_params_from_any_iterable():
    t = CudaTarget(4, FUNNEL, params=(x for x in (1, 2)))
    assert t.params == (1.0, 2.0)
    with pytest.raises(ValueError):
        CudaTarget(4, FUNNEL, params=(x for x in range(9)))
    with pytest.raises(ValueError):
        CudaTarget(4, FUNNEL, params=3.0)
    with pytest.raises(ValueError):
        CudaTarget(4, 42)
