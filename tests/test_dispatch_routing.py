"""CPU tests of which models the Riemannian and constrained entry points accept.

Every call passes small host buffers and an ``mb200_model`` over a grid of metric, target,
dimension and operation. A rejected combination returns ``MB200_ERR_INVALID_ARG`` or
``MB200_ERR_UNSUPPORTED`` with its message. A combination routed to a launch fails at its first
CUDA call with ``MB200_ERR_CUDA``, because the machine has no device. The expectations below
state the rules each entry point applies, including the shared-memory sizes that decide between
shared memory, the per-CTA workspace and the global-workspace dense policy.

These tests tell "rejected" apart from "launched". They cannot tell which kernel was launched,
for example the rank-1 dense policy against the Sherman-Morrison one. The GPU parity tests and a
per-kernel comparison of the compiled code cover that.

On a machine with a GPU a routed call would start a kernel on host pointers, so the module skips
itself there.
"""

import ctypes

import numpy as np
import pytest
import torch

from mici_b200 import _lib

pytestmark = pytest.mark.skipif(
    torch.cuda.is_available(), reason="routed calls would launch kernels on host pointers"
)

INVALID, UNSUPPORTED, CUDA = -1, -2, -3
LAUNCHED = (CUDA, None)

SOFTABS, RANK1, HADAMARD, DIAG, FISHER, SCALAR, CHOL = range(7)
UNKNOWN_RMETRIC = 9
STD, FUNNEL, BANANA, QUADRATIC, TORUS, SPHERE, MULTI_SPHERE, QUARTIC = range(8)

SMEM = 227 * 1024  # opt-in shared memory per CTA on sm_90, bytes
DIMS = (2, 7, 64, 150, 160, 512, 600, 1100, 1300, 2100)

# a host buffer standing in for every array argument: nothing is read from it before the launch
BUF = np.zeros(16)
PTR = BUF.ctypes.data


@pytest.fixture(scope="module")
def lib():
    import os

    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge

        ge.build()
    return _lib.load()


def model(target, rmetric=0, tp=(), mp=(), taux=True, maux=True):
    m = _lib.Model()
    m.target_id, m.rmetric_id = target, rmetric
    for i, v in enumerate(tp):
        m.target_params[i] = v
    for i, v in enumerate(mp):
        m.rmetric_params[i] = v
    m.target_aux = PTR if taux else None
    m.rmetric_aux = PTR if maux else None
    return m


def call(lib, name, *args):
    rc = getattr(lib, name)(*args)
    return rc, lib.mb200_last_error().decode()


def check(got, want):
    """None when `got` = (rc, message) meets `want` = (rc, message prefix or None)."""
    rc, msg = got
    if rc == want[0] and (want[1] is None or msg.startswith(want[1])):
        return None
    return f"got {rc} {msg!r}, want {want[0]} {want[1]!r}"


# --- shared-memory sizes (doubles), as riemannian.cuh lays the per-chain buffers out --------------


def dpad(dim):
    return (dim + 1) & ~1


def rm_smem(dim, n_mats):
    dp = dpad(dim)
    return dim * (dim + 1) * n_mats + 27 * dp + 3 * (dp // 2 + 2) + 40


def rm_compact(dim, midpoint):
    return (24 if midpoint else 14) * dpad(dim) + 40


def dense_global_supported(dim):
    np_ = (dim + 31) & ~31
    return (12 * dpad(dim) + 40 + max(np_ - 32, 32) * 36 + 2 * 32 * 36) * 8 <= SMEM


# --- Riemannian entry points ----------------------------------------------------------------------

IMPLICIT_OPS = ("leapfrog", "midpoint", "hamiltonian")
RIEMANNIAN_OPS = IMPLICIT_OPS + ("sample_momentum", "dh_dmom")


def launch_plan(op, policy, target, dim):
    """Expected outcome of the launch helper for a policy that passed the route checks."""
    implicit = op in IMPLICIT_OPS
    if policy == "compact":
        if rm_compact(dim, op == "midpoint") * 8 > SMEM:
            return (UNSUPPORTED, f"dim {dim}: per-chain vectors" if implicit else f"dim {dim} too large")
        return LAUNCHED
    n_mats, ws_mats = {"softabs": (2, 3), "rank1": (1, 0), "woodbury": (0, 0), "chol": (1, 1)}[policy]
    if policy == "softabs" and implicit and (rm_smem(dim, 3) * 8 <= 113 * 1024 or target == QUARTIC):
        n_mats = 3
    if rm_smem(dim, n_mats) * 8 > SMEM:
        if ws_mats == 0:
            return (UNSUPPORTED, f"dim {dim}: per-chain metric" if implicit else f"dim {dim} too large")
        if rm_smem(dim, 0) * 8 > SMEM:
            return (UNSUPPORTED, f"dim {dim} too large")
    return LAUNCHED


def riemannian_expected(op, rmetric, target, dim, mp, taux, maux):
    fits = rm_smem(dim, 1) * 8 <= SMEM
    even_ok = not (target == BANANA and dim % 2)
    if rmetric == HADAMARD or (rmetric == RANK1 and not fits and mp[2] == 0 and target == QUADRATIC
                               and dense_global_supported(dim)):
        if op == "midpoint":
            return (UNSUPPORTED, "implicit midpoint is not available for the global-workspace")
        if not dense_global_supported(dim):
            return (UNSUPPORTED, f"dim {dim}: panel buffers exceed shared memory")
        if not maux:
            return (INVALID, "dense metric needs its matrices")
        if target != QUADRATIC:
            return (UNSUPPORTED, f"target {target} not compiled for the global-workspace dense")
        if not taux:
            return (INVALID, "quadratic target needs its precision matrix")
        return LAUNCHED
    if rmetric == SOFTABS:
        if not mp[0] > 0:
            return (INVALID, "softabs_coeff must be positive")
        if target == BANANA:
            return launch_plan(op, "softabs", target, dim) if even_ok else (
                INVALID, "banana target needs even dim")
        if target == QUARTIC:
            if not taux:
                return (INVALID, "quartic target needs its directions")
            if op == "midpoint":
                return (UNSUPPORTED, "implicit midpoint: quartic target not available")
            return launch_plan(op, "softabs", target, dim)
        return (UNSUPPORTED, f"target {target} has no device Hessian")
    if rmetric in (RANK1, CHOL) and not maux:
        return (INVALID, "rank-1 metric needs its base matrix" if rmetric == RANK1
                else "Cholesky-factored metric needs its base factor")
    if rmetric in (DIAG, SCALAR) and not (mp[0] > 0 and mp[1] >= 0):
        return (INVALID, "metric parameters need a > 0 and b >= 0")
    if rmetric not in (RANK1, DIAG, FISHER, SCALAR, CHOL):
        return (INVALID, f"unknown rmetric_id {rmetric}")
    if not even_ok:
        return (INVALID, "banana target needs even dim")
    if target == QUADRATIC and not taux:
        return (INVALID, "quadratic target needs its precision matrix")
    if rmetric == RANK1:
        woodbury = not fits or (mp[2] != 0 and op != "sample_momentum")
        if woodbury and op == "sample_momentum":
            return (UNSUPPORTED, f"dim {dim}: the Cholesky factor of M(q) does not fit")
        if target not in (STD, BANANA, QUADRATIC):
            return (UNSUPPORTED, f"target {target} not available")
        return launch_plan(op, "woodbury" if woodbury else "rank1", target, dim)
    if rmetric == FISHER and target != FUNNEL:
        return (UNSUPPORTED, f"the funnel Fisher metric needs the funnel target (got {target})")
    if target not in (STD, FUNNEL, BANANA, QUADRATIC):
        return (UNSUPPORTED, f"target {target} not available")
    return launch_plan(op, "chol" if rmetric == CHOL else "compact", target, dim)


def riemannian_call(lib, op, m, dim, fp_solver=0):
    n = 4
    if op in ("leapfrog", "midpoint"):
        args = [PTR, PTR, PTR, PTR, None, n, dim, 0.1, None, 1, None, ctypes.byref(m), fp_solver,
                1e-9, 1e10, 100, 2e-8, PTR, PTR, PTR, PTR]
        if op == "leapfrog":
            return call(lib, "mb200_implicit_leapfrog_riemannian", *args, None, 0, None)
        return call(lib, "mb200_implicit_midpoint_riemannian", *args, None)
    if op == "hamiltonian":
        return call(lib, "mb200_hamiltonian_riemannian", PTR, PTR, n, dim, ctypes.byref(m), PTR,
                    PTR, None, 0, None)
    name = "mb200_sample_momentum_riemannian" if op == "sample_momentum" else "mb200_dh_dmom_riemannian"
    return call(lib, name, PTR, PTR, PTR, n, dim, ctypes.byref(m), PTR, None)


# (metric parameters, target_aux set, rmetric_aux set): a valid model and one defect each
VARIANTS = {
    "valid": ((1.0, 0.5, 0.0), True, True),
    "no_target_aux": ((1.0, 0.5, 0.0), False, True),
    "no_metric_aux": ((1.0, 0.5, 0.0), True, False),
    "bad_params": ((0.0, 0.5, 0.0), True, True),
    "force_sherman_morrison": ((1.0, 0.5, 1.0), True, True),
}


@pytest.mark.parametrize("op", RIEMANNIAN_OPS)
def test_riemannian_routing(lib, op):
    failures = []
    for rmetric in (SOFTABS, RANK1, HADAMARD, DIAG, FISHER, SCALAR, CHOL, UNKNOWN_RMETRIC):
        for target in range(8):
            for dim in DIMS:
                for variant, (mp, taux, maux) in VARIANTS.items():
                    m = model(target, rmetric, tp=(1.0,), mp=mp, taux=taux, maux=maux)
                    want = riemannian_expected(op, rmetric, target, dim, mp, taux, maux)
                    err = check(riemannian_call(lib, op, m, dim), want)
                    if err:
                        failures.append(f"rmetric {rmetric} target {target} dim {dim} {variant}: {err}")
    assert not failures, f"{len(failures)} cases:\n" + "\n".join(failures[:40])


@pytest.mark.parametrize("op", ("leapfrog", "midpoint", "hamiltonian"))
def test_implicit_fixed_point_solver_is_checked(lib, op):
    m = model(BANANA, SOFTABS, mp=(1.0,))
    want = LAUNCHED if op == "hamiltonian" else (INVALID, "unknown fixed-point solver 7")
    assert check(riemannian_call(lib, op, m, 8, fp_solver=7), want) is None
    assert check(riemannian_call(lib, op, m, 8, fp_solver=1), LAUNCHED) is None


# --- constrained entry points ---------------------------------------------------------------------

CONSTRAINED_DIMS = (2, 3, 4, 7, 12, 64, 65, 100, 128, 130, 200, 256, 300)


def constrained_target_expected(target, dim, n_constr):
    if target == TORUS:
        return LAUNCHED if dim == 3 else (INVALID, "torus target needs dim == 3")
    if target == SPHERE:
        return LAUNCHED if dim <= 256 else (UNSUPPORTED, f"sphere target: dim {dim} > 256")
    if target == MULTI_SPHERE:
        if n_constr in (2, 4, 8) and dim % n_constr == 0 and dim <= 128:
            return LAUNCHED
        return (UNSUPPORTED, "multi-sphere target: n_constr must be 2, 4 or 8")
    return (UNSUPPORTED, f"target {target} defines no constraint")


def constrained_cases():
    for target in range(8):
        for n_constr in (2, 3, 4, 8) if target == MULTI_SPHERE else (0,):
            for dim in CONSTRAINED_DIMS:
                for lebesgue in (0.0, 1.0):
                    tp = [0.0] * _lib.MAX_PARAMS
                    tp[0] = n_constr if target == MULTI_SPHERE else 1.0
                    tp[-1] = lebesgue
                    yield target, n_constr, dim, model(target, tp=tp)


@pytest.mark.parametrize("gaussian", (False, True))
def test_constrained_leapfrog_routing(lib, gaussian):
    failures = []
    for target, n_constr, dim, m in constrained_cases():
        for metric_kind in (0, 1, 2, 3):
            for solver in (0, 1, 2, 3):
                args = [PTR, PTR, PTR, PTR, None, 4, dim, 0.1, None, 1, None, 2, metric_kind, PTR]
                tail = [ctypes.byref(m), solver, 1e-9, 1e-8, 1e10, 50, 10, 2e-8, PTR, PTR, PTR, PTR,
                        None]
                if gaussian:
                    got = call(lib, "mb200_constrained_leapfrog_gaussian_euclidean", *args, PTR, PTR,
                               PTR, *tail)
                else:
                    got = call(lib, "mb200_constrained_leapfrog_euclidean", *args, *tail)
                if solver > 2:
                    want = (INVALID, f"unknown projection solver {solver}")
                elif metric_kind > 2:
                    want = (INVALID, "bad metric_kind")
                else:
                    want = constrained_target_expected(target, dim, n_constr)
                err = check(got, want)
                if err:
                    failures.append(f"target {target} nc {n_constr} dim {dim} metric {metric_kind} "
                                    f"solver {solver}: {err}")
    assert not failures, f"{len(failures)} cases:\n" + "\n".join(failures[:40])


@pytest.mark.parametrize("gaussian", (False, True))
def test_constrained_null_metric_arrays_are_rejected(lib, gaussian):
    m = model(SPHERE)
    name = ("mb200_constrained_leapfrog_gaussian_euclidean" if gaussian
            else "mb200_constrained_leapfrog_euclidean")

    def run(metric_kind, minv, omega=PTR, eigvec=PTR):
        args = [PTR, PTR, PTR, PTR, None, 4, 10, 0.1, None, 1, None, 2, metric_kind, minv]
        extra = [omega, eigvec, eigvec] if gaussian else []
        return call(lib, name, *args, *extra, ctypes.byref(m), 0, 1e-9, 1e-8, 1e10, 50, 10, 2e-8,
                    PTR, PTR, PTR, PTR, None)

    assert check(run(1, None), (INVALID, "metric_inv is NULL")) is None
    assert check(run(0, None), LAUNCHED) is None
    if gaussian:
        assert check(run(0, None, omega=None), (INVALID, "metric_omega is NULL")) is None
        assert check(run(2, PTR, eigvec=None), (INVALID, "metric_eigvec")) is None
        assert check(run(1, PTR, eigvec=None), LAUNCHED) is None


@pytest.mark.parametrize("gaussian", (False, True))
def test_constrained_projection_routing(lib, gaussian):
    name = ("mb200_project_onto_cotangent_space_gaussian" if gaussian
            else "mb200_project_onto_cotangent_space")
    failures = []
    for target, n_constr, dim, m in constrained_cases():
        for metric_kind in (0, 1, 2, 3):
            for minv in (PTR, None):
                got = call(lib, name, PTR, PTR, PTR, 4, dim, metric_kind, minv, ctypes.byref(m), None)
                if metric_kind > 2:
                    want = (INVALID, "bad metric_kind")
                elif metric_kind != 0 and minv is None:
                    want = (INVALID, "metric_inv is NULL")
                else:
                    want = constrained_target_expected(target, dim, n_constr)
                err = check(got, want)
                if err:
                    failures.append(f"target {target} nc {n_constr} dim {dim} metric {metric_kind}: {err}")
    assert not failures, f"{len(failures)} cases:\n" + "\n".join(failures[:40])
