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


# --- Euclidean entry points -----------------------------------------------------------------------
#
# A routed Euclidean call fails at its first CUDA call with "<kernel>: <CUDA error>", so the message
# names the kernel that would have run: the tensor-core leapfrog K1 (leapfrog_dmma_kernel), the
# general-dimension leapfrog K1g (leapfrog_generic_kernel), the evaluation kernel, and fused NUTS in
# lock-step on the tensor pipe (nuts_dmma_kernel) or free-running (nuts_euclidean_kernel).

USER = 64
UNKNOWN_TARGET = 9
EUCLID_TARGETS = tuple(range(8)) + (UNKNOWN_TARGET,)
EUCLID_DIMS = (1, 2, 7, 8, 64, 65, 128, 129, 1024, 1025)
# (per-chain step sizes, per-chain lengths, coefficient schedule) of a leapfrog call
SCHEDULES = {
    "shared_eps": (False, False, False),
    "per_chain_eps": (True, False, False),
    "per_chain_lengths": (False, True, False),
    "coefficients": (False, False, True),
}
COEFS = np.array([0.25, 0.5, 0.5, 0.5, 0.25])
# a user-target handle whose kernel table is empty: calls that reach a launch fail there
FAKE_IMAGE = np.zeros(16, dtype=np.uint64)


def euclid_model_expected(target, dim, metric_kind, minv, user):
    """The model checks every Euclidean operation applies, in order; None when the model passes."""
    if metric_kind > 2:
        return (INVALID, "bad metric_kind")
    if metric_kind != 0 and minv is None:
        return (INVALID, "metric_inv is NULL")
    if target == BANANA and dim % 2:
        return (INVALID, "banana target needs even dim")
    if user and target != USER:
        return (INVALID, "user-target entry point needs target_id MB200_TARGET_USER")
    if not user and target not in (STD, FUNNEL, BANANA):
        return (UNSUPPORTED, f"target {target} not available")
    if dim > 1024:
        return (UNSUPPORTED, f"dim {dim} > 1024 not supported")
    return None


def k1_serves(target, dim, metric_kind, eps, per_chain_eps, n_steps, schedule):
    _, per_chain_lengths, coefficients = SCHEDULES[schedule]
    return (metric_kind == 2 and n_steps > 0 and 8 <= dim <= 128 and not per_chain_lengths
            and not coefficients and (per_chain_eps or (eps != 0 and np.isfinite(eps)))
            and target in (STD, FUNNEL, BANANA))


def leapfrog_call(lib, entry, m, dim, metric_kind, minv, schedule, eps=0.1, n_steps=1, user=None):
    per_chain_eps, per_chain_lengths, coefficients = SCHEDULES[schedule]
    args = [PTR, PTR, PTR, PTR, None, 4, dim, eps, PTR if per_chain_eps else None, n_steps,
            PTR if per_chain_lengths else None, len(COEFS) if coefficients else 0,
            COEFS.ctypes.data if coefficients else None, 1, metric_kind, minv, ctypes.byref(m),
            PTR, PTR, PTR, None]
    if entry == "user":
        return call(lib, "mb200_leapfrog_euclidean_user", *args, user)
    return call(lib, f"mb200_leapfrog_euclidean{'_generic' if entry == 'generic' else ''}", *args)


@pytest.mark.parametrize("entry", ("leapfrog", "generic", "user"))
def test_euclidean_leapfrog_routing(lib, entry):
    user = entry == "user"
    failures = []
    for target in EUCLID_TARGETS + ((USER,) if user else ()):
        for dim in EUCLID_DIMS:
            for metric_kind in (0, 1, 2, 3):
                for minv in (PTR, None):
                    for schedule in SCHEDULES:
                        m = model(target, tp=(1.0,))
                        got = leapfrog_call(lib, entry, m, dim, metric_kind, minv, schedule,
                                            user=FAKE_IMAGE.ctypes.data if user else None)
                        want = euclid_model_expected(target, dim, metric_kind, minv, user)
                        if want is None:
                            k1 = entry == "leapfrog" and k1_serves(
                                target, dim, metric_kind, 0.1, SCHEDULES[schedule][0], 1, schedule)
                            want = (CUDA, "leapfrog_dmma_kernel: " if k1 else "leapfrog_generic_kernel: ")
                        err = check(got, want)
                        if err:
                            failures.append(f"target {target} dim {dim} metric {metric_kind} "
                                            f"minv {minv is not None} {schedule}: {err}")
    assert not failures, f"{len(failures)} cases:\n" + "\n".join(failures[:40])


def test_euclidean_leapfrog_k1_needs_a_usable_step_size(lib):
    m = model(FUNNEL)
    for eps, n_steps in ((0.0, 1), (float("nan"), 1), (float("inf"), 1), (0.1, 0)):
        got = leapfrog_call(lib, "leapfrog", m, 64, 2, PTR, "shared_eps", eps=eps, n_steps=n_steps)
        assert check(got, (CUDA, "leapfrog_generic_kernel: ")) is None, (eps, n_steps, got)
        # per-chain step sizes: the scalar is not used
        got = leapfrog_call(lib, "leapfrog", m, 64, 2, PTR, "per_chain_eps", eps=eps, n_steps=n_steps)
        want = "leapfrog_dmma_kernel: " if n_steps > 0 else "leapfrog_generic_kernel: "
        assert check(got, (CUDA, want)) is None, (eps, n_steps, got)


def test_euclidean_bad_arguments_are_rejected(lib):
    m = model(STD)
    args = [PTR, PTR, PTR, PTR, None, 4, 8, 0.1, None, 1, None, 0, None, 1, 0, None,
            ctypes.byref(m), PTR, PTR, PTR, None]
    name = "mb200_leapfrog_euclidean"
    assert check(call(lib, name, *args[:3], None, *args[4:]), (INVALID, "null pointer")) is None
    assert check(call(lib, name, *args[:6], 0, *args[7:]), (INVALID, "bad sizes")) is None
    assert check(call(lib, name, *args[:9], -1, *args[10:]), (INVALID, "bad sizes")) is None
    assert check(call(lib, name, *args[:11], 2, COEFS.ctypes.data, *args[13:]),
                 (INVALID, "n_flows must be odd")) is None
    # an empty batch returns before any other check
    assert call(lib, name, *args[:5], 0, *args[6:])[0] == 0
    assert call(lib, name, None, *args[1:5], 0, *args[6:])[0] == 0
    assert call(lib, "mb200_euclidean_eval", None, PTR, 0, 8, 0, None, ctypes.byref(m), PTR, PTR,
                PTR, PTR, None)[0] == 0


@pytest.mark.parametrize("user", (False, True))
def test_euclidean_hamiltonian_routing(lib, user):
    failures = []
    for target in EUCLID_TARGETS + ((USER,) if user else ()):
        for dim in EUCLID_DIMS:
            for metric_kind in (0, 1, 2, 3):
                for minv in (PTR, None):
                    m = model(target, tp=(1.0,))
                    args = [PTR, PTR, 4, dim, metric_kind, minv, ctypes.byref(m)]
                    name = "mb200_hamiltonian_euclidean" + ("_user" if user else "")
                    tail = [None, FAKE_IMAGE.ctypes.data] if user else [None]
                    want = euclid_model_expected(target, dim, metric_kind, minv, user) or (
                        CUDA, "leapfrog_generic_kernel: ")
                    for h_out in (PTR, None):
                        got = call(lib, name, *args, h_out, *tail)
                        err = check(got, want if h_out else (INVALID, "h_out is NULL"))
                        if err:
                            failures.append(f"target {target} dim {dim} metric {metric_kind} "
                                            f"minv {minv is not None} h_out {h_out}: {err}")
    assert not failures, f"{len(failures)} cases:\n" + "\n".join(failures[:40])


@pytest.mark.parametrize("user", (False, True))
def test_euclidean_eval_routing(lib, user):
    failures = []
    for target in EUCLID_TARGETS + ((USER,) if user else ()):
        for dim in EUCLID_DIMS:
            for metric_kind in (0, 1, 2, 3):
                for minv in (PTR, None):
                    m = model(target, tp=(1.0,))
                    args = [PTR, PTR, 4, dim, metric_kind, minv, ctypes.byref(m), PTR, PTR, PTR, PTR,
                            None]
                    got = (call(lib, "mb200_euclidean_eval_user", *args, FAKE_IMAGE.ctypes.data)
                           if user else call(lib, "mb200_euclidean_eval", *args))
                    want = euclid_model_expected(target, dim, metric_kind, minv, user) or (
                        CUDA, "euclidean_eval_kernel: ")
                    err = check(got, want)
                    if err:
                        failures.append(f"target {target} dim {dim} metric {metric_kind} "
                                        f"minv {minv is not None}: {err}")
    assert not failures, f"{len(failures)} cases:\n" + "\n".join(failures[:40])


def test_euclidean_gaussian_leapfrog_routing(lib):
    failures = []
    for target in EUCLID_TARGETS:
        for dim in EUCLID_DIMS:
            for metric_kind in (0, 1, 2, 3):
                for minv in (PTR, None):
                    for rotation in (PTR, None):
                        for per_chain_eps in (False, True):
                            m = model(target, tp=(1.0,))
                            got = call(lib, "mb200_leapfrog_gaussian_euclidean", PTR, PTR, PTR, PTR,
                                       None, 4, dim, 0.1, PTR if per_chain_eps else None, 1, 0, None,
                                       1, metric_kind, minv, rotation, ctypes.byref(m), PTR, PTR, PTR,
                                       None)
                            if metric_kind != 0 and rotation is None:
                                want = (INVALID, "rotation is NULL")
                            elif metric_kind == 2 and per_chain_eps:
                                want = (UNSUPPORTED, "per-chain step sizes need per-chain rotation")
                            else:
                                want = euclid_model_expected(target, dim, metric_kind, minv, False) or (
                                    CUDA, "leapfrog_generic_kernel: ")
                            err = check(got, want)
                            if err:
                                failures.append(f"target {target} dim {dim} metric {metric_kind} "
                                                f"minv {minv is not None} rotation {rotation} "
                                                f"per-chain eps {per_chain_eps}: {err}")
    assert not failures, f"{len(failures)} cases:\n" + "\n".join(failures[:40])


@pytest.mark.parametrize("name", ("mb200_leapfrog_euclidean_user", "mb200_hamiltonian_euclidean_user",
                                  "mb200_euclidean_eval_user"))
def test_euclidean_null_user_target_is_rejected(lib, name):
    m = model(USER)
    if name == "mb200_leapfrog_euclidean_user":
        got = leapfrog_call(lib, "user", m, 8, 0, None, "shared_eps", user=None)
    elif name == "mb200_hamiltonian_euclidean_user":
        got = call(lib, name, PTR, PTR, 4, 8, 0, None, ctypes.byref(m), PTR, None, None)
    else:
        got = call(lib, name, PTR, PTR, 4, 8, 0, None, ctypes.byref(m), PTR, PTR, PTR, PTR, None, None)
    assert check(got, (INVALID, "user_target is NULL")) is None, got


def nuts_call(lib, m, dim, metric_kind, minv, workspace_bytes=1 << 40, depth=6, uniforms=PTR):
    return call(lib, "mb200_nuts_euclidean", PTR, PTR, PTR, PTR, 4, dim, 0.1, None, metric_kind,
                minv, ctypes.byref(m), 0, 0, 0, depth, 1000.0, uniforms, 8, PTR, workspace_bytes,
                PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, None)


def test_euclidean_nuts_routing(lib):
    failures = []
    for target in EUCLID_TARGETS:
        for dim in EUCLID_DIMS:
            for metric_kind in (0, 1, 2, 3):
                for minv in (PTR, None):
                    m = model(target, tp=(1.0,))
                    want = euclid_model_expected(target, dim, metric_kind, minv, False)
                    if want is None:
                        dmma = metric_kind == 2 and 8 <= dim <= 128
                        want = (CUDA, "nuts_dmma_kernel: " if dmma else "nuts_euclidean_kernel: ")
                    err = check(nuts_call(lib, m, dim, metric_kind, minv), want)
                    if err:
                        failures.append(f"target {target} dim {dim} metric {metric_kind} "
                                        f"minv {minv is not None}: {err}")
    assert not failures, f"{len(failures)} cases:\n" + "\n".join(failures[:40])


def test_euclidean_nuts_arguments_are_checked(lib):
    m = model(STD)
    assert check(nuts_call(lib, m, 8, 0, None, uniforms=None), (INVALID, "null pointer")) is None
    assert check(nuts_call(lib, m, 8, 0, None, depth=0), (INVALID, "max_tree_depth must be in")) is None
    assert check(nuts_call(lib, m, 8, 3, None, workspace_bytes=0), (INVALID, "bad metric_kind")) is None
    assert check(nuts_call(lib, m, 8, 0, None, workspace_bytes=0), (INVALID, "workspace too small")) is None
    # the workspace is checked before the model's target
    assert check(nuts_call(lib, model(UNKNOWN_TARGET), 8, 0, None, workspace_bytes=0),
                 (INVALID, "workspace too small")) is None
    assert check(nuts_call(lib, model(BANANA), 7, 0, None, workspace_bytes=0),
                 (INVALID, "workspace too small")) is None


NUTS_GENERIC_KERNELS = ("begin", "start", "leaf", "finish", "end")


def nuts_generic_call(lib, step, n, dim, opts, ws=PTR, cs=PTR, ws_bytes=1 << 40):
    o = ctypes.byref(opts) if opts is not None else None
    if step == "begin":
        return call(lib, "mb200_nuts_generic_begin", PTR, PTR, PTR, PTR, n, dim, o, ws, ws_bytes, cs,
                    1 << 40, None)
    if step == "start":
        return call(lib, "mb200_nuts_generic_start", n, dim, 2, o, ws, cs, PTR, PTR, PTR, PTR, None)
    if step == "leaf":
        return call(lib, "mb200_nuts_generic_leaf", PTR, PTR, PTR, PTR, PTR, n, dim, 0, 4, o, ws, cs,
                    PTR, None)
    if step == "finish":
        return call(lib, "mb200_nuts_generic_finish", n, dim, 2, o, ws, cs, None)
    return call(lib, "mb200_nuts_generic_end", n, dim, o, ws, cs, *[PTR] * 10, None)


@pytest.mark.parametrize("step", NUTS_GENERIC_KERNELS)
def test_nuts_generic_arguments_are_checked(lib, step):
    opts = _lib.NutsOptions(6, 0, 0, 0, 1000.0, PTR, 8)
    bad_depth = _lib.NutsOptions(0, 0, 0, 0, 1000.0, PTR, 8)
    no_uniforms = _lib.NutsOptions(6, 0, 0, 0, 1000.0, None, 8)
    failures = []
    for dim in EUCLID_DIMS:
        cases = [
            ((4, dim, opts), (INVALID, "bad sizes") if dim > 1024 else (CUDA, f"nuts_generic_{step}_kernel: ")),
            ((0, dim, None), (0, None)),
            ((4, dim, None), (INVALID, "null pointer")),
            ((4, dim, no_uniforms), (INVALID, "null pointer")),
            ((4, dim, bad_depth), (INVALID, "bad sizes") if dim > 1024 else (INVALID, "max_tree_depth")),
        ]
        for args, want in cases:
            err = check(nuts_generic_call(lib, step, *args), want)
            if err:
                failures.append(f"dim {dim} {args}: {err}")
        err = check(nuts_generic_call(lib, step, 4, dim, opts, ws=None), (INVALID, "null pointer"))
        if err:
            failures.append(f"dim {dim} null workspace: {err}")
    if step == "begin":
        err = check(nuts_generic_call(lib, step, 4, 8, opts, ws_bytes=0), (INVALID, "workspace / chain"))
        if err:
            failures.append(f"small workspace: {err}")
    assert not failures, f"{len(failures)} cases:\n" + "\n".join(failures[:40])
