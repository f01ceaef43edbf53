"""User-written constraints (``CudaTarget(..., n_constr=...)``) without a GPU: NVRTC compilation
of the constrained image, compile errors, validation, the cache and pickling."""

import copy
import pickle
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from mici_b200 import integrators, jit, systems
from mici_b200.errors import TargetCompileError
from mici_b200.targets import CudaTarget

from test_user_target import _elf_symbols
from user_constraint_sources import GENERATOR, MULTI_SPHERE, SO3, SPHERE, TORUS

# (source, n_constr, kp, mhp_constr): every KP and several constraint counts
EXAMPLES = {
    "sphere_kp4": (SPHERE, 1, 4, True),
    "multi_sphere_c8_kp2": (MULTI_SPHERE, 8, 2, True),
    "multi_sphere_c3_kp1": (MULTI_SPHERE, 3, 1, False),
    "torus_kp1": (TORUS, 1, 1, True),
    "so3_c6_kp1": (SO3, 6, 1, False),
    "generator_c5_kp1": (GENERATOR, 5, 1, True),
}


def test_example_sources_compile_to_sm90a_images_with_every_kernel():
    def build(item):
        name, (src, nc, kp, mhp) = item
        return name, jit.compile_target(src, name, n_constr=nc, kp=kp, mhp_constr=mhp)

    with ThreadPoolExecutor(len(EXAMPLES)) as pool:
        images = dict(pool.map(build, EXAMPLES.items()))
    for name, (_, cubin, names) in images.items():
        kp = EXAMPLES[name][2]
        assert cubin[:4] == b"\x7fELF"
        assert int.from_bytes(cubin[0x30:0x34], "little") & 0xFF == 90  # sm_90(a)
        assert len(names) == 14 and len(set(names)) == 14
        assert _elf_symbols(cubin) >= set(names)
        assert all("UserTarget" in n for n in names[:10])
        assert all("UserConstrainedTarget" in n and f"Li{kp}E" in n for n in names[10:])
        assert sum("leapfrog" in n for n in names[10:]) == 2


def test_missing_jacobian_is_a_compile_error_naming_it():
    src = SPHERE.replace("jacob_constr(const mb200::Chain& c, double* J)",
                         "other_jacobian(const mb200::Chain& c, double* J)")
    with pytest.raises(TargetCompileError, match="jacob_constr"):
        jit.compile_target(src, "no_jacobian", n_constr=1, kp=1)


def test_lebesgue_density_and_gaussian_system_need_mhp_constr():
    t = CudaTarget(8, SPHERE, n_constr=1)
    systems.DenseConstrainedEuclideanMetricSystem(t)  # Hausdorff: accepted
    with pytest.raises(ValueError, match="mhp_constr"):
        systems.DenseConstrainedEuclideanMetricSystem(t, dens_wrt_hausdorff=False)
    with pytest.raises(ValueError, match="mhp_constr"):
        systems.ConstrainedEuclideanMetricSystem(t, dens_wrt_hausdorff=False)
    with pytest.raises(ValueError, match="mhp_constr"):
        systems.GaussianDenseConstrainedEuclideanMetricSystem(t)
    t = CudaTarget(8, SPHERE, n_constr=1, mhp_constr=True)
    systems.DenseConstrainedEuclideanMetricSystem(t, dens_wrt_hausdorff=False)
    systems.GaussianDenseConstrainedEuclideanMetricSystem(t)


def test_constructor_limits():
    for bad in (-1, 9, 1.5, True, "2"):
        with pytest.raises(ValueError):
            CudaTarget(8, SPHERE, n_constr=bad)
    CudaTarget(256, SPHERE, n_constr=1)
    with pytest.raises(ValueError):
        CudaTarget(257, SPHERE, n_constr=1)
    for nc in (2, 3, 5, 6, 7, 8):
        CudaTarget(128, MULTI_SPHERE, n_constr=nc)
        with pytest.raises(ValueError):
            CudaTarget(129, MULTI_SPHERE, n_constr=nc)
    CudaTarget(8, SPHERE, params=range(7), n_constr=1)
    with pytest.raises(ValueError):
        CudaTarget(8, SPHERE, params=range(8), n_constr=1)
    CudaTarget(1024, SPHERE, params=range(8))  # unconstrained limits unchanged
    t = CudaTarget(8, SPHERE, n_constr=2, mhp_constr=True)
    assert t.n_constr == 2 and t.mhp_constr
    assert not CudaTarget(8, SPHERE, mhp_constr=True).mhp_constr  # no constraint, no product


def test_kp_follows_the_registry_constrained_targets():
    assert [jit.constrained_kp(d, 1) for d in (3, 64, 65, 128, 129, 256)] == [1, 1, 2, 2, 4, 4]
    assert [jit.constrained_kp(d, 8) for d in (8, 64, 65, 128)] == [1, 1, 2, 2]
    assert jit.constrained_kp(257, 1) is None and jit.constrained_kp(129, 2) is None


def test_cache_hits_for_same_source_and_kp_and_misses_for_another_constraint_count(monkeypatch):
    """The key covers N_CONSTR, KP and mhp_constr; the unconstrained key is the one it always
    was.  NVRTC is replaced by a stub: only the cache logic is under test."""
    compiled = []

    def fake(source, name, constraint=()):
        compiled.append(constraint)
        return b"\x7fELF-stub", tuple(f"k{i}" for i in range(14 if constraint else 10))

    monkeypatch.setattr(jit, "_compile", fake)
    src = MULTI_SPHERE + "\n// cache probe\n"
    CudaTarget(16, src, n_constr=4).compile()
    before = dict(jit.stats)
    CudaTarget(40, src, n_constr=4).compile()  # another dim at the same KP: same image
    assert jit.stats["hits"] == before["hits"] + 1 and len(compiled) == 1
    CudaTarget(16, src, n_constr=2).compile()  # another N_CONSTR
    CudaTarget(100, src, n_constr=4).compile()  # another KP
    CudaTarget(16, src, n_constr=4, mhp_constr=True).compile()
    CudaTarget(16, src).compile()  # unconstrained
    assert compiled == [(4, 1, False), (2, 1, False), (4, 2, False), (4, 1, True), ()]
    keys = {jit.cache_key(src, "user_target", c) for c in compiled}
    assert len(keys) == 5 and jit.cache_key(src) in keys
    assert jit.cache_key(src) == jit.cache_key(src, "user_target", ())


def test_constrained_system_and_integrator_survive_deepcopy_and_pickle():
    t = CudaTarget(12, MULTI_SPHERE, aux=np.arange(3.0), name="multi", n_constr=3,
                   mhp_constr=True)
    system = systems.GaussianDenseConstrainedEuclideanMetricSystem(t, metric=np.linspace(1, 2, 12))
    integ = integrators.ConstrainedLeapfrogIntegrator(system, 0.1, n_inner_step=2)
    for clone in (copy.deepcopy(integ), pickle.loads(pickle.dumps(integ))):
        ct = clone.system.target
        assert isinstance(ct, CudaTarget) and ct.source == t.source and ct.name == "multi"
        assert ct.n_constr == 3 and ct.mhp_constr and np.array_equal(ct.aux, t.aux)
        assert isinstance(clone.system, systems.GaussianDenseConstrainedEuclideanMetricSystem)
        assert clone.n_inner_step == 2
        assert np.array_equal(clone.system.metric.array, system.metric.array)
