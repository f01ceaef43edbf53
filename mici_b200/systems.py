"""Hamiltonian systems of the batched engine -- same class names, constructor keywords and
method meanings as ``mici.systems`` (reference ``src/mici/systems.py``) for the classes on the
hot path:

* ``EuclideanMetricSystem``                   systems.py:264-366
* ``DenseConstrainedEuclideanMetricSystem``   systems.py:619-873, 876-1031
* ``GaussianDenseConstrainedEuclideanMetricSystem``  systems.py:1034-1184
* ``DenseRiemannianMetricSystem``             systems.py:1187-1402, 1710-1760
* ``SoftAbsRiemannianMetricSystem``           systems.py:1763-1920
* ``ScalarRiemannianMetricSystem``            systems.py:1405-1490
* ``DiagonalRiemannianMetricSystem``          systems.py:1493-1571
* ``CholeskyFactoredRiemannianMetricSystem``  systems.py:1574-1653

Differences forced by the device: ``neg_log_dens`` is an instance of
``mici_b200.targets.Target`` (a model compiled into the library) instead of a Python callable,
its derivatives are implied, and states are batched ``mici_b200.states.ChainState`` s holding
``[n_chains, dim]`` fp64 CUDA tensors.  Methods return per-chain tensors.
"""

from __future__ import annotations

import ctypes

import numpy as np
import scipy.linalg as sla
import torch

from . import _lib
from .errors import LinAlgError
from .solvers import solve_projection_onto_manifold_newton
from .targets import (
    RMETRIC_SOFTABS,
    CudaCholeskyMetric,
    CudaDenseMetric,
    CudaDiagonalMetric,
    CudaRiemannianPair,
    CudaScalarMetric,
    CudaTarget,
    FunnelFisherMetric,
    HadamardMetric,
    NealFunnel,
    QuadraticCholeskyMetric,
    QuadraticDiagonalMetric,
    QuadraticScalarMetric,
    Rank1Metric,
    Target,
)

METRIC_IDENTITY, METRIC_DIAGONAL, METRIC_DENSE = 0, 1, 2


def _explicit_spd_inverse(array):
    """Dense explicit inverse built the way the reference builds ``metric.inv``: lower Cholesky
    factor (matrices.py:1161-1173) then two triangular solves against the identity
    (matrices.py:897-912, 1060-1061, 1183-1188).  Host side, once per metric assignment."""
    if not np.all(np.isfinite(array)):
        raise LinAlgError("Array is not finite.")
    try:
        chol = np.linalg.cholesky(array)
    except np.linalg.LinAlgError as e:
        raise LinAlgError("Cholesky factorisation failed.") from e
    inv_lt = sla.solve_triangular(chol.T, np.identity(array.shape[0]), lower=False, check_finite=False)
    inv = sla.solve_triangular(chol.T, inv_lt.T, lower=False, check_finite=False)
    return chol, inv


class _FixedMetric:
    """Host-side description of a fixed metric plus lazily uploaded device buffers."""

    def __init__(self, metric):
        if metric is None:
            self.kind, self.array, self.inv, self.sqrt = METRIC_IDENTITY, None, None, None
        else:
            if isinstance(metric, torch.Tensor):
                metric = metric.detach().cpu().numpy()
            metric = np.asarray(metric, dtype=np.float64)
            if metric.ndim == 1:
                if not np.all(metric > 0):
                    raise ValueError("Diagonal values must all be positive.")
                self.kind, self.array = METRIC_DIAGONAL, metric
                self.inv, self.sqrt = 1.0 / metric, metric**0.5
            elif metric.ndim == 2:
                self.kind, self.array = METRIC_DENSE, metric
                self.sqrt, self.inv = _explicit_spd_inverse(metric)
            else:
                msg = (
                    "If NumPy ndarray value is used for `metric` must be either 1D (diagonal "
                    "matrix) or 2D (dense positive definite matrix)."
                )
                raise ValueError(msg)
        self._dev = {}

    @classmethod
    def from_covariance(cls, covar):
        """The metric ``DensePositiveDefiniteMatrix(covar).inv`` that the covariance adapter
        assigns (adapters.py:642): with ``L = chol(covar)`` its array is the explicit inverse
        ``L^-T L^-1`` and its factor ``L^-T`` (matrices.py:1183-1188, 1209-1216), so ``metric.inv``
        multiplies by ``L L^T`` (matrices.py:1041-1046, 1060-1061) and ``metric.sqrt @ z`` solves
        ``L^T x = z`` (matrices.py:897-903) -- held here as the explicit upper-triangular factor."""
        covar = np.asarray(covar, dtype=np.float64)
        chol, explicit_inv = _explicit_spd_inverse(covar)
        self = cls.__new__(cls)
        self.kind, self.array = METRIC_DENSE, explicit_inv
        self.inv = chol @ chol.T
        self.sqrt = sla.solve_triangular(chol.T, np.identity(covar.shape[0]), lower=False,
                                         check_finite=False)
        self._dev = {}
        return self

    @property
    def shape(self):
        return (None, None) if self.array is None else (self.array.shape[0],) * 2

    def inv_device(self, device):
        """Device copy of 1/diag or of the explicit dense inverse (None for identity)."""
        if self.kind == METRIC_IDENTITY:
            return None
        key = ("inv", str(device))
        if key not in self._dev:
            self._dev[key] = torch.as_tensor(np.ascontiguousarray(self.inv), device=device)
        return self._dev[key]

    def sqrt_device(self, device):
        if self.kind == METRIC_IDENTITY:
            return None
        key = ("sqrt", str(device))
        if key not in self._dev:
            self._dev[key] = torch.as_tensor(np.ascontiguousarray(self.sqrt), device=device)
        return self._dev[key]

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_dev"] = {}
        return d


def _batched(state):
    """A state as (contiguous [n, D] pos, contiguous [n, D] mom, dir tensor-or-None, squeeze
    flag).

    NumPy arrays (the reference's own ``ChainState`` storage, states.py:160-305) are accepted
    and moved to the current CUDA device; callers convert results back (``_like_input``)."""
    pos, mom = state.pos, state.mom
    if isinstance(pos, np.ndarray):
        pos = torch.as_tensor(np.ascontiguousarray(pos, dtype=np.float64), device="cuda")
        mom = None if mom is None else torch.as_tensor(
            np.ascontiguousarray(mom, dtype=np.float64), device="cuda")
    single = pos.ndim == 1
    if single:
        pos, mom = pos[None], (None if mom is None else mom[None])
    d = state.dir if "dir" in state else 1
    return pos.contiguous(), None if mom is None else mom.contiguous(), d, single


def _on_batch(state, launch):
    """``launch(pos, mom, dir)`` on the batched view of ``state`` (``_batched``); its output
    tensor, or each tensor of its output tuple, is returned in the form of ``state.pos``: one
    row for a single chain, NumPy for NumPy."""
    pos, mom, d, single = _batched(state)
    out = launch(pos, mom, d)

    def back(x):
        return _like_input(state.pos, x[0] if single else x)

    return tuple(map(back, out)) if isinstance(out, tuple) else back(out)


def _check_metric_status(status, n):
    """Raise ``LinAlgError`` if the metric of any chain could not be factorised."""
    if bool((status != 0).any()):
        bad = int((status != 0).sum())
        raise LinAlgError(f"metric factorisation failed for {bad} of {n} chains")


def _like_input(ref, value):
    """Return ``value`` in the storage type of ``ref`` (NumPy in -> NumPy out)."""
    if isinstance(ref, np.ndarray) and isinstance(value, torch.Tensor):
        return value.cpu().numpy()
    return value


def _dir_tensor(d, n, device):
    """``dir`` as an int32 device tensor [n] (or None meaning all +1)."""
    if isinstance(d, torch.Tensor):
        return d.to(device=device, dtype=torch.int32).reshape(-1).contiguous()
    d = int(d)
    if d == 1:
        return None
    return torch.full((n,), d, dtype=torch.int32, device=device)


class System:
    """Base class (systems.py:39-229): holds the target model and builds ``mb200_model``."""

    # whether a user-written `CudaTarget` may drive the system (its kernels need only l and grad l);
    # a Riemannian system sets it on the instance when it is given a user metric
    _user_targets = False

    def __init__(self, neg_log_dens, *, grad_neg_log_dens=None, backend=None):
        if not isinstance(neg_log_dens, Target):
            msg = (
                "mici_b200 systems take a `mici_b200.targets.Target` instance as `neg_log_dens` "
                "(a registry model, or a `CudaTarget` written in CUDA C++); Python callables are "
                "not supported."
            )
            raise TypeError(msg)
        if isinstance(neg_log_dens, CudaTarget) and not self._user_targets:
            raise TypeError(f"{type(self).__name__} does not take a CudaTarget: user targets run "
                            "on EuclideanMetricSystem.")
        if grad_neg_log_dens is not None or backend is not None:
            raise ValueError("Derivatives are fused into the kernels; pass neither "
                             "`grad_neg_log_dens` nor `backend`.")
        self.target = neg_log_dens
        self._rmetric_id = 0
        self._rmetric_params = ()
        self._rmetric_aux = None
        self._dev = {}

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_dev"] = {}
        return d

    def _scratch(self, name, nbytes, device):
        """Device byte buffer ``name`` of at least ``nbytes``, kept and grown across calls."""
        key = (name, str(device))
        buf = self._dev.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=device)
            self._dev[key] = buf
        return buf

    def _aux_device(self, name, array, device):
        if array is None:
            return None
        key = (name, str(device))
        if key not in self._dev:
            self._dev[key] = torch.as_tensor(array, device=device).contiguous()
        return self._dev[key]

    def _model(self, device):
        m = _lib.Model()
        t = self.target
        m.target_id = t.target_id
        m.n_target_params = len(t.params)
        for i, v in enumerate(t.params):
            m.target_params[i] = v
        if not getattr(self, "dens_wrt_hausdorff", True):
            # constrained systems: density given with respect to the Lebesgue measure
            m.target_params[_lib.MAX_PARAMS - 1] = 1.0
        aux = self._aux_device("target_aux", t.aux, device)
        m.target_aux = None if aux is None else aux.data_ptr()
        m.rmetric_id = self._rmetric_id
        m.n_rmetric_params = len(self._rmetric_params)
        for i, v in enumerate(self._rmetric_params):
            m.rmetric_params[i] = v
        raux = self._aux_device("rmetric_aux", self._rmetric_aux, device)
        m.rmetric_aux = None if raux is None else raux.data_ptr()
        return m

    def dh_dmom(self, state):
        return self.dh2_dmom(state)


class TractableFlowSystem(System):
    """systems.py:232-261."""


class EuclideanMetricSystem(TractableFlowSystem):
    """Euclidean Hamiltonian system with a fixed metric (systems.py:264-366).

    ``metric``: ``None`` (identity), 1-D array (diagonal) or 2-D array (dense SPD), coerced as
    in systems.py:332-346.  Assignable (adapters set it: adapters.py:513, 642).
    """

    _user_targets = True

    def __init__(self, neg_log_dens, *, metric=None, grad_neg_log_dens=None, backend=None):
        super().__init__(neg_log_dens, grad_neg_log_dens=grad_neg_log_dens, backend=backend)
        self.metric = metric

    @property
    def metric(self):
        return self._metric

    @metric.setter
    def metric(self, value):
        self._metric = value if isinstance(value, _FixedMetric) else _FixedMetric(value)

    def _eval(self, state, what):
        """One output of ``mb200_euclidean_eval``: ``"nld"``, ``"grad"``, ``"vel"`` or ``"kin"``."""

        def launch(pos, mom, _):
            n, dim = pos.shape
            dev = pos.device
            mom = pos if mom is None else mom
            out = torch.empty(n, dtype=torch.float64, device=dev) if what in ("nld", "kin") \
                else torch.empty_like(pos)
            target = self.target if what in ("nld", "grad") else None
            if target is not None:
                model = self._model(dev)
            else:  # M^-1 p and p.M^-1 p do not involve the target (constrained targets have no
                model = _lib.Model()  # Euclidean-eval functor): neutral model
                model.target_id = 0
            outs = [_lib.ptr(out) if w == what else None for w in ("nld", "grad", "vel", "kin")]
            _lib.call("mb200_euclidean_eval", _lib.ptr(pos), _lib.ptr(mom), n, dim,
                      self._metric.kind, _lib.ptr(self._metric.inv_device(dev)),
                      ctypes.byref(model), *outs, _lib.current_stream_ptr(dev), target=target)
            return out

        return _on_batch(state, launch)

    def neg_log_dens(self, state):
        return self._eval(state, "nld")

    def grad_neg_log_dens(self, state):
        return self._eval(state, "grad")

    def h1(self, state):
        return self.neg_log_dens(state)

    def dh1_dpos(self, state):
        return self.grad_neg_log_dens(state)

    def h2(self, state):
        return self._eval(state, "kin")

    def dh2_dmom(self, state):
        return self._eval(state, "vel")

    def dh2_dpos(self, state):
        if isinstance(state.pos, np.ndarray):
            return np.zeros_like(state.pos)
        return torch.zeros_like(state.pos)

    def dh_dpos(self, state):
        return self.dh1_dpos(state)

    def h(self, state):
        """h = h1 + h2 (systems.py:187-196), one fused kernel."""

        def launch(pos, mom, _):
            n, dim = pos.shape
            dev = pos.device
            h = torch.empty(n, dtype=torch.float64, device=dev)
            model = self._model(dev)
            _lib.call("mb200_hamiltonian_euclidean", _lib.ptr(pos), _lib.ptr(mom), n, dim,
                      self._metric.kind, _lib.ptr(self._metric.inv_device(dev)),
                      ctypes.byref(model), _lib.ptr(h), _lib.current_stream_ptr(dev),
                      target=self.target)
            return h

        return _on_batch(state, launch)

    def h1_flow(self, state, dt):
        """p -= dt * grad l(q) (systems.py:143-152); ``dt`` scalar or per-chain tensor."""
        state.mom = state.mom - _col(dt) * self.dh1_dpos(state)

    def h2_flow(self, state, dt):
        """q += dt * M^-1 p (systems.py:362-363)."""
        state.pos = state.pos + _col(dt) * self.dh2_dmom(state)

    def sample_momentum(self, state, rng):
        """``metric.sqrt @ N(0, I)`` (systems.py:365-366).  The variates come from ``rng`` (a
        NumPy generator, a sequence of per-chain NumPy generators, or a device
        ``torch.Generator``: see ``mici_b200.transitions``); the product ``L z`` runs on the
        device through ``mb200_euclidean_eval`` with the transposed factor in the metric slot."""
        from .transitions import _normals  # noqa: PLC0415

        pos = state.pos if state.pos.ndim == 2 else state.pos[None]
        # NumPy-held states (the reference's own ChainState storage): device work on the current
        # CUDA device, NumPy back out
        dev = torch.device("cuda") if isinstance(pos, np.ndarray) else pos.device
        z = _normals(rng, tuple(pos.shape), dev).contiguous()
        m = self._metric
        if m.kind != METRIC_IDENTITY:
            n, dim = z.shape
            out = torch.empty_like(z)
            key = ("sqrt_t", str(z.device))
            if key not in m._dev:
                fac = m.sqrt if m.kind == METRIC_DIAGONAL else np.ascontiguousarray(m.sqrt.T)
                m._dev[key] = torch.as_tensor(fac, device=z.device).contiguous()
            model = _lib.Model()  # the product L z does not involve the target
            model.target_id = 0
            _lib.call("mb200_euclidean_eval", _lib.ptr(z), _lib.ptr(z), n, dim, m.kind,
                      _lib.ptr(m._dev[key]), ctypes.byref(model), None, None, _lib.ptr(out), None,
                      _lib.current_stream_ptr(z.device))
            z = out
        return _like_input(state.pos, z if state.pos.ndim == 2 else z[0])


class GaussianEuclideanMetricSystem(EuclideanMetricSystem):
    """Euclidean system whose target density is given relative to the standard Gaussian measure
    (systems.py:369-474) -- "next" row N4: ``h1 = l(q)``, ``h2 = q.q/2 + p.M^-1 p/2`` and
    ``h2_flow`` is the exact rotation of ``(q, p)`` in the eigenbasis of ``M``.  The tractable-
    flow integrators (leapfrog, symmetric compositions) drive it through
    ``mb200_leapfrog_gaussian_euclidean``."""

    _user_targets = False

    def h2(self, state):
        """``q.q/2 + p.M^-1 p/2`` (systems.py:450-453)."""
        pos = torch.as_tensor(state.pos)
        return super().h2(state) + _like_input(state.pos, 0.5 * (pos * pos).sum(-1))

    def dh2_dpos(self, state):
        """systems.py:460-462."""
        return state.pos

    def dh_dpos(self, state):
        return self.dh1_dpos(state) + state.pos

    def h(self, state):
        return self.h1(state) + self.h2(state)

    def _eig(self):
        """``(eigval, eigvec)`` of the metric as the reference obtains them: ``numpy.linalg.eigh``
        of the dense array (matrices.py:436-438); identity eigenvectors for identity / diagonal
        metrics (matrices.py:519-528, 743-749)."""
        m = self._metric
        if "eig" not in m._dev:
            m._dev["eig"] = np.linalg.eigh(m.array)
        return m._dev["eig"]

    def rotation_device(self, device, step_size, drift_coefficients):
        """Device operand ``rotation`` of ``mb200_leapfrog_gaussian_euclidean``."""
        m = self._metric
        if m.kind == METRIC_IDENTITY:
            return None
        if m.kind == METRIC_DIAGONAL:
            key = ("diag", str(device))
            if key not in m._dev:
                m._dev[key] = torch.as_tensor(np.ascontiguousarray(m.array), device=device)
            return m._dev[key]
        key = ("rot", str(device), float(step_size), tuple(float(c) for c in drift_coefficients))
        if key not in m._dev:
            # keep only the rotations of the most recent step sizes (adaptation visits many)
            stale = [k for k in m._dev if isinstance(k, tuple) and k and k[0] == "rot"]
            for k in stale[:-3]:
                del m._dev[k]
            eigval, u = self._eig()
            omega = 1.0 / eigval**0.5
            mats = []
            for c in drift_coefficients:
                t = float(c) * float(step_size)
                sn, cs = np.sin(omega * t), np.cos(omega * t)
                mats += [(u * cs) @ u.T, (u * (sn * omega)) @ u.T, -(u * (sn / omega)) @ u.T]
            m._dev[key] = torch.as_tensor(np.ascontiguousarray(np.stack(mats)), device=device)
        return m._dev[key]

    def h2_flow(self, state, dt):
        """Exact flow of ``h2`` over ``dt`` (systems.py:464-474), all chains in one launch."""
        from .integrators import _gaussian_flow  # noqa: PLC0415

        _gaussian_flow(self, state, dt)


def _registry_euclidean(system):
    """Whether ``system`` is a plain ``EuclideanMetricSystem`` (not constrained, not a Gaussian
    split) on a registry target: the systems the tensor-core leapfrog's host-buffer path and the
    fused dynamic transition serve."""
    return (isinstance(system, EuclideanMetricSystem)
            and not isinstance(system, (ConstrainedEuclideanMetricSystem,
                                        GaussianEuclideanMetricSystem))
            and not isinstance(system.target, CudaTarget))


def _col(dt):
    return dt[..., None] if isinstance(dt, torch.Tensor) and dt.ndim >= 1 else dt


class ConstrainedTractableFlowSystem(TractableFlowSystem):
    """systems.py:477-616."""

    def sample_momentum(self, state, rng):
        """Draw from N(0, M), then project onto the cotangent space (systems.py:613-616)."""
        mom = super().sample_momentum(state, rng)
        return self.project_onto_cotangent_space(mom, state)


class ConstrainedEuclideanMetricSystem(ConstrainedTractableFlowSystem, EuclideanMetricSystem):
    """Euclidean system subject to holonomic constraints (systems.py:619-873).

    ``constr`` must be the same ``Target`` instance as ``neg_log_dens`` (constrained targets
    carry their constraint function).  ``dens_wrt_hausdorff=False``: the target density is given
    with respect to the Lebesgue measure and ``h1`` / ``dh1_dpos`` carry ``log det gram / 2`` and
    its gradient through the constraint's matrix-Hessian product (systems.py:853-861, 1024-1031),
    fused into the kernels.

    A ``CudaTarget`` with ``n_constr >= 1`` brings its own constraint (user-written CUDA,
    ``csrc/user_constraint.cuh``); with ``dens_wrt_hausdorff=False`` it must define
    ``mhp_constr``.
    """

    _user_targets = True

    def __init__(self, neg_log_dens, constr=None, *, metric=None, dens_wrt_hausdorff=True,
                 grad_neg_log_dens=None, jacob_constr=None, backend=None):
        if isinstance(neg_log_dens, CudaTarget):
            if neg_log_dens.n_constr < 1:  # the TypeError of System for an unconstrained one
                raise TypeError(f"{type(self).__name__} does not take a CudaTarget: user targets "
                                "run on EuclideanMetricSystem.")
            if not dens_wrt_hausdorff and not neg_log_dens.mhp_constr:
                raise ValueError(f"{type(self).__name__} with a density with respect to the "
                                 "Lebesgue measure needs the constraint's matrix-Hessian "
                                 "product: define mhp_constr and pass mhp_constr=True to "
                                 "CudaTarget.")
        EuclideanMetricSystem.__init__(self, neg_log_dens, metric=metric,
                                       grad_neg_log_dens=grad_neg_log_dens, backend=backend)
        if constr is not None and constr is not neg_log_dens:
            raise ValueError("`constr` must be the target model passed as `neg_log_dens`.")
        if jacob_constr is not None:
            raise ValueError("The constraint Jacobian is fused into the kernels.")
        if neg_log_dens.n_constr < 1:
            raise ValueError(f"Target {neg_log_dens!r} defines no constraint function.")
        self.dens_wrt_hausdorff = bool(dens_wrt_hausdorff)

    def _leapfrog(self, pos, mom, pos_out, mom_out, dirs, eps, eps_t, max_n, ns, n_inner_step,
                  solver, solver_kw, reverse_check_tol, h, status, n_done, iters):
        """``mb200_constrained_leapfrog[_gaussian]_euclidean`` for this system, with the solver
        options ``solver_kw`` resolved; ``max_n = 0`` evaluates ``h`` only."""
        n, dim = pos.shape
        dev = pos.device
        m = self._metric
        metric = (m.kind, _lib.ptr(m.inv_device(dev)))
        entry = "mb200_constrained_leapfrog_euclidean"
        if isinstance(self, GaussianDenseConstrainedEuclideanMetricSystem):
            # exact h2 rotation with per-chain sin / cos, eigh-inverted Gram matrices
            entry = "mb200_constrained_leapfrog_gaussian_euclidean"
            metric += tuple(_lib.ptr(a) for a in self.rotation_args(dev))
        model = self._model(dev)
        _lib.call(
            entry, _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(pos_out), _lib.ptr(mom_out),
            _lib.ptr(dirs), n, dim, eps, _lib.ptr(eps_t), max_n, _lib.ptr(ns), int(n_inner_step),
            *metric, ctypes.byref(model), solver.kind, float(solver_kw["constraint_tol"]),
            float(solver_kw["position_tol"]), float(solver_kw["divergence_tol"]),
            int(solver_kw["max_iters"]), int(solver_kw.get("max_line_search_iters", 10)),
            float(reverse_check_tol), _lib.ptr(h), _lib.ptr(status), _lib.ptr(n_done),
            _lib.ptr(iters), _lib.current_stream_ptr(dev), target=self.target)

    def h(self, state):
        """``h1 + h2`` (systems.py:187-196, 451-454, 842-856), evaluated by a zero-step launch of
        the constrained kernel."""

        def launch(pos, mom, _):
            h = torch.empty(pos.shape[0], dtype=torch.float64, device=pos.device)
            solver = solve_projection_onto_manifold_newton
            # 2e-8: ConstrainedLeapfrogIntegrator's default reverse_check_tol
            self._leapfrog(pos, mom, torch.empty_like(pos), torch.empty_like(mom), None, 0.0, None,
                           0, None, 1, solver, solver.resolve_kwargs({}), 2e-8, h, None, None,
                           None)
            return h

        return _on_batch(state, launch)

    def project_onto_cotangent_space(self, mom, state):
        """``mom - J^T (J M^-1 J^T)^-1 J M^-1 mom`` at ``state.pos`` (systems.py:863-873) for all
        chains in one launch (``mb200_project_onto_cotangent_space``); on the Gaussian system
        ``J M^-1 J^T`` is inverted through its eigendecomposition (systems.py:1157-1169,
        ``mb200_project_onto_cotangent_space_gaussian``)."""
        pos = state.pos
        single = pos.ndim == 1
        ref = mom
        pos_t = torch.as_tensor(pos)
        if pos_t.device.type != "cuda":
            pos_t = pos_t.to("cuda")
        pos_t = (pos_t[None] if single else pos_t).contiguous()
        mom_t = torch.as_tensor(mom).to(pos_t.device)
        mom_t = (mom_t[None] if mom_t.ndim == 1 else mom_t).contiguous()
        n, dim = pos_t.shape
        dev = pos_t.device
        out = torch.empty_like(mom_t)
        m = self._metric
        minv = None if m.kind == METRIC_IDENTITY else m.inv_device(dev)
        model = self._model(dev)
        gaussian = isinstance(self, GaussianDenseConstrainedEuclideanMetricSystem)
        _lib.call("mb200_project_onto_cotangent_space" + ("_gaussian" if gaussian else ""),
                  _lib.ptr(pos_t), _lib.ptr(mom_t), _lib.ptr(out), n, dim, m.kind,
                  _lib.ptr(minv), ctypes.byref(model), _lib.current_stream_ptr(dev),
                  target=self.target)
        return _like_input(ref, out[0] if single else out)


class DenseConstrainedEuclideanMetricSystem(ConstrainedEuclideanMetricSystem):
    """systems.py:876-1031 (dense constraint Jacobian)."""

    def __init__(self, neg_log_dens, constr=None, *, metric=None, dens_wrt_hausdorff=True,
                 grad_neg_log_dens=None, jacob_constr=None, mhp_constr=None, backend=None):
        if mhp_constr is not None:
            raise ValueError("The constraint's matrix-Hessian product is fused into the kernels.")
        super().__init__(neg_log_dens, constr, metric=metric,
                         dens_wrt_hausdorff=dens_wrt_hausdorff,
                         grad_neg_log_dens=grad_neg_log_dens, jacob_constr=jacob_constr,
                         backend=backend)


class GaussianDenseConstrainedEuclideanMetricSystem(GaussianEuclideanMetricSystem,
                                                    DenseConstrainedEuclideanMetricSystem):
    """Gaussian Euclidean system subject to a dense set of constraints (systems.py:1034-1184):
    the target density is relative to the standard Gaussian measure on the ambient space and is
    conditioned on ``constr(q) == 0`` (always ``dens_wrt_hausdorff=False``).  ``h1 = l(q) +
    log det gram / 2``, ``h2 = q.q/2 + p.M^-1 p/2`` whose flow is the exact rotation in the
    eigenbasis of ``M``; the Gram matrices are inverted through their eigendecomposition.  The
    constrained leapfrog drives it through ``mb200_constrained_leapfrog_gaussian_euclidean``.
    A constrained ``CudaTarget`` must define ``mhp_constr``."""

    _user_targets = True  # GaussianEuclideanMetricSystem's False comes first in the MRO

    def __init__(self, neg_log_dens, constr=None, *, metric=None, grad_neg_log_dens=None,
                 jacob_constr=None, mhp_constr=None, backend=None):
        DenseConstrainedEuclideanMetricSystem.__init__(
            self, neg_log_dens, constr, metric=metric, dens_wrt_hausdorff=False,
            grad_neg_log_dens=grad_neg_log_dens, jacob_constr=jacob_constr,
            mhp_constr=mhp_constr, backend=backend)

    def rotation_args(self, device):
        """Device operands ``(metric_omega, metric_eigvec, metric_eigvec_t)`` of
        ``mb200_constrained_leapfrog_gaussian_euclidean``: ``w = 1 / eigval**0.5`` computed as
        the reference does (systems.py:1176), and ``U``, ``U^T`` for a dense metric."""
        m = self._metric
        key = ("gauss_constr", str(device))
        if key not in m._dev:
            dim = self.target.dim
            if m.kind == METRIC_IDENTITY:
                omega, u = 1.0 / np.ones(dim) ** 0.5, None
            elif m.kind == METRIC_DIAGONAL:
                omega, u = 1.0 / m.array**0.5, None
            else:
                eigval, u = self._eig()
                omega = 1.0 / eigval**0.5
            m._dev[key] = tuple(
                None if a is None else torch.as_tensor(np.ascontiguousarray(a), device=device)
                for a in (omega, u, None if u is None else u.T))
        return m._dev[key]

    # GaussianEuclideanMetricSystem's h1 + h2 comes first in the MRO
    h = ConstrainedEuclideanMetricSystem.h

    def h2(self, state):
        """``q.q/2 + p.M^-1 p/2`` (systems.py:451-454)."""
        return GaussianEuclideanMetricSystem.h2(self, state)

    def dh2_dpos(self, state):
        """systems.py:460-462."""
        return state.pos

    def h2_flow(self, state, dt):
        raise NotImplementedError(
            "The exact h2 flow of a constrained Gaussian system runs inside the constrained "
            "leapfrog kernel, followed by the projection onto the manifold.")


class RiemannianMetricSystem(System):
    """Riemannian Hamiltonian system with a position-dependent metric (systems.py:1187-1402)."""

    # the (CudaTarget, user metric) pair whose image the launches run, None for registry models
    _user_pair = None

    def _accept_user_metric(self, target, metric, cls):
        """Before ``System.__init__``: a user metric of class ``cls`` comes with an unconstrained
        ``CudaTarget``, which the system then takes."""
        if not isinstance(metric, cls):
            return
        if not isinstance(target, CudaTarget) or target.n_constr:
            raise TypeError(f"A {cls.__name__} needs an unconstrained CudaTarget as "
                            "`neg_log_dens`.")
        self._user_targets = True
        self._user_pair = CudaRiemannianPair(target, metric)

    def _workspace(self, n, dim, device):
        model = self._model(device)
        nbytes = int(_lib.load().mb200_implicit_workspace_bytes(n, dim, ctypes.byref(model)))
        return self._scratch("ws", nbytes, device)

    def h(self, state):
        """l(q) + log|M(q)|/2 + p^T M(q)^-1 p / 2 (systems.py:1375-1390)."""

        def launch(pos, mom, _):
            n, dim = pos.shape
            dev = pos.device
            h = torch.empty(n, dtype=torch.float64, device=dev)
            status = torch.empty(n, dtype=torch.int32, device=dev)
            ws = self._workspace(n, dim, dev)
            model = self._model(dev)
            _lib.call("mb200_hamiltonian_riemannian", _lib.ptr(pos), _lib.ptr(mom), n, dim,
                      ctypes.byref(model), _lib.ptr(h), _lib.ptr(status), _lib.ptr(ws),
                      ws.numel(), _lib.current_stream_ptr(dev), target=self._user_pair)
            return h

        return _on_batch(state, launch)

    def dh2_dmom(self, state):
        """``M(q)^-1 p`` (systems.py:1398-1399); not cached, as in the reference."""

        def launch(pos, mom, _):
            n, dim = pos.shape
            dev = pos.device
            vel = torch.empty((n, dim), dtype=torch.float64, device=dev)
            status = torch.empty(n, dtype=torch.int32, device=dev)
            model = self._model(dev)
            _lib.call("mb200_dh_dmom_riemannian", _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(vel), n,
                      dim, ctypes.byref(model), _lib.ptr(status), _lib.current_stream_ptr(dev),
                      target=self._user_pair)
            _check_metric_status(status, n)
            return vel

        return _on_batch(state, launch)

    def sample_momentum(self, state, rng):
        """``metric(state).sqrt @ N(0, I)`` (systems.py:1401-1402): the factor of M(q) is built
        per chain on the device (``mb200_sample_momentum_riemannian``).  Chains whose metric
        cannot be built raise ``LinAlgError`` as in the reference."""
        from .transitions import _normals  # noqa: PLC0415

        pos = torch.as_tensor(state.pos)
        single = pos.ndim == 1
        if pos.device.type != "cuda":
            pos = pos.to("cuda")
        pos = (pos[None] if single else pos).contiguous()
        n, dim = pos.shape
        dev = pos.device
        z = _normals(rng, (n, dim), dev).contiguous()
        out = torch.empty_like(z)
        status = torch.empty(n, dtype=torch.int32, device=dev)
        model = self._model(dev)
        _lib.call("mb200_sample_momentum_riemannian", _lib.ptr(pos), _lib.ptr(z), _lib.ptr(out),
                  n, dim, ctypes.byref(model), _lib.ptr(status), _lib.current_stream_ptr(dev),
                  target=self._user_pair)
        _check_metric_status(status, n)
        return _like_input(state.pos, out[0] if single else out)


class DenseRiemannianMetricSystem(RiemannianMetricSystem):
    """Dense position-dependent metric (systems.py:1710-1760): ``metric_func`` is a registered
    metric model -- ``mici_b200.targets.Rank1Metric`` (M(q) = B + c q q^T) or
    ``mici_b200.targets.HadamardMetric`` (M(q) = B + c (q q^T) o S, full rank).  Each chain's
    metric is factorised (Cholesky), inverted explicitly and differentiated through the model's
    VJP as the reference does (matrices.py:1161-1188, systems.py:1381-1399): in shared memory
    for D <= 160, in a per-CTA global workspace with DMMA-blocked routines beyond
    (csrc/dense_global.cuh).

    ``metric_func`` may also be a user-written ``mici_b200.targets.CudaDenseMetric`` with an
    unconstrained ``CudaTarget`` (``dim <= 576``): it runs on the global-workspace policy at every
    dimension, without the implicit midpoint integrator."""

    # the largest dimension whose panel buffers fit in shared memory (dense_global_supported)
    MAX_USER_DIM = 576

    def __init__(self, neg_log_dens, metric_func, *, vjp_metric_func=None,
                 grad_neg_log_dens=None, backend=None):
        self._accept_user_metric(neg_log_dens, metric_func, CudaDenseMetric)
        super().__init__(neg_log_dens, grad_neg_log_dens=grad_neg_log_dens, backend=backend)
        if not isinstance(metric_func, (Rank1Metric, HadamardMetric, CudaDenseMetric)):
            raise TypeError("`metric_func` must be a registered metric model "
                            "(Rank1Metric or HadamardMetric) or a CudaDenseMetric.")
        if vjp_metric_func is not None:
            raise ValueError("The metric VJP is fused into the kernels.")
        if isinstance(metric_func, CudaDenseMetric) and neg_log_dens.dim > self.MAX_USER_DIM:
            raise ValueError(f"A CudaDenseMetric needs dim <= {self.MAX_USER_DIM}, "
                             f"got {neg_log_dens.dim}.")
        self.metric_model = metric_func
        self._rmetric_id = metric_func.rmetric_id
        self._rmetric_params = metric_func.params
        self._rmetric_aux = metric_func.aux


class SoftAbsRiemannianMetricSystem(RiemannianMetricSystem):
    """SoftAbs-regularised Hessian metric (systems.py:1763-1920)."""

    def __init__(self, neg_log_dens, *, grad_neg_log_dens=None, hess_neg_log_dens=None,
                 mtp_neg_log_dens=None, softabs_coeff=1.0, backend=None):
        super().__init__(neg_log_dens, grad_neg_log_dens=grad_neg_log_dens, backend=backend)
        if hess_neg_log_dens is not None or mtp_neg_log_dens is not None:
            raise ValueError("Hessian and MTP of the target are fused into the kernels.")
        if softabs_coeff <= 0:
            raise ValueError("softabs_coeff must be positive.")
        self.softabs_coeff = float(softabs_coeff)
        self._rmetric_id = RMETRIC_SOFTABS
        self._rmetric_params = (self.softabs_coeff,)


class ScalarRiemannianMetricSystem(RiemannianMetricSystem):
    """Scaled-identity position-dependent metric ``s(q) I`` (systems.py:1405-1490) with
    ``PositiveScaledIdentityMatrix`` arithmetic (matrices.py:595-706): ``metric_scalar_func`` is a
    registered metric model, ``mici_b200.targets.QuadraticScalarMetric`` (s = a + b |q|^2), or a
    user-written ``mici_b200.targets.CudaScalarMetric`` with a ``CudaTarget``.

    A chain whose ``s(q)`` is not positive fails with status 3 (``LinAlgError``) outside a
    fixed-point solve and with ``ConvergenceError`` inside one; the reference raises
    ``ValueError`` in the first case (DESIGN.md section 1)."""

    def __init__(self, neg_log_dens, metric_scalar_func, *, vjp_metric_scalar_func=None,
                 grad_neg_log_dens=None, backend=None):
        self._accept_user_metric(neg_log_dens, metric_scalar_func, CudaScalarMetric)
        super().__init__(neg_log_dens, grad_neg_log_dens=grad_neg_log_dens, backend=backend)
        if not isinstance(metric_scalar_func, (QuadraticScalarMetric, CudaScalarMetric)):
            raise TypeError("`metric_scalar_func` must be a registered metric model "
                            "(QuadraticScalarMetric) or a CudaScalarMetric.")
        if vjp_metric_scalar_func is not None:
            raise ValueError("The metric VJP is fused into the kernels.")
        self.metric_model = metric_scalar_func
        self._rmetric_id = metric_scalar_func.rmetric_id
        self._rmetric_params = metric_scalar_func.params
        self._rmetric_aux = metric_scalar_func.aux


class DiagonalRiemannianMetricSystem(RiemannianMetricSystem):
    """Diagonal position-dependent metric ``diag(d(q))`` (systems.py:1493-1571) with
    ``PositiveDiagonalMatrix`` arithmetic (matrices.py:709-792): ``metric_diagonal_func`` is a
    registered metric model -- ``mici_b200.targets.QuadraticDiagonalMetric`` (d_i = a + b q_i^2)
    or ``mici_b200.targets.FunnelFisherMetric`` (the funnel's expected Fisher information, funnel
    target only) -- or a user-written ``mici_b200.targets.CudaDiagonalMetric`` with a
    ``CudaTarget``.  O(D) per metric: a chain's whole state lives in a small CTA's shared memory.

    A chain whose ``d(q)`` has an entry that is not positive fails with status 3
    (``LinAlgError``) outside a fixed-point solve and with ``ConvergenceError`` inside one; the
    reference raises ``ValueError`` in the first case (DESIGN.md section 1)."""

    def __init__(self, neg_log_dens, metric_diagonal_func, *, vjp_metric_diagonal_func=None,
                 grad_neg_log_dens=None, backend=None):
        self._accept_user_metric(neg_log_dens, metric_diagonal_func, CudaDiagonalMetric)
        super().__init__(neg_log_dens, grad_neg_log_dens=grad_neg_log_dens, backend=backend)
        if not isinstance(metric_diagonal_func,
                          (QuadraticDiagonalMetric, FunnelFisherMetric, CudaDiagonalMetric)):
            raise TypeError("`metric_diagonal_func` must be a registered metric model "
                            "(QuadraticDiagonalMetric or FunnelFisherMetric) or a "
                            "CudaDiagonalMetric.")
        if isinstance(metric_diagonal_func, FunnelFisherMetric) and not isinstance(
                neg_log_dens, NealFunnel):
            raise TypeError("FunnelFisherMetric is the metric of the NealFunnel target.")
        if vjp_metric_diagonal_func is not None:
            raise ValueError("The metric VJP is fused into the kernels.")
        self.metric_model = metric_diagonal_func
        self._rmetric_id = metric_diagonal_func.rmetric_id
        self._rmetric_params = metric_diagonal_func.params
        self._rmetric_aux = metric_diagonal_func.aux


class CholeskyFactoredRiemannianMetricSystem(RiemannianMetricSystem):
    """Position-dependent metric given by its lower-triangular Cholesky factor,
    ``M(q) = L(q) L(q)^T`` (systems.py:1574-1653), with ``TriangularFactoredPositiveDefiniteMatrix``
    arithmetic (matrices.py:795-1114): ``metric_chol_func`` is a registered metric model,
    ``mici_b200.targets.QuadraticCholeskyMetric`` (L = L0 + c tril(q q^T)).  No factorisation:
    each metric evaluation fills L and solves with it, O(D^2) per chain, with L in shared memory
    up to D of about 150 and in a per-CTA global workspace beyond.

    Failures follow the reference's matrix class: a non-finite entry of L fails when the metric
    is built -- status 3 (``LinAlgError``) outside a fixed-point solve, ``ConvergenceError``
    inside one.  A negative diagonal entry is legal.  A zero diagonal entry fails only where the
    metric is solved with: ``dh_dmom`` raises ``LinAlgError``, ``h`` is NaN, ``sample_momentum``
    succeeds, and an integrator step ends in ``ConvergenceError`` (DESIGN.md section 1).

    ``metric_chol_func`` may also be a user-written ``mici_b200.targets.CudaCholeskyMetric`` with
    an unconstrained ``CudaTarget`` (``dim <= 1016``), with the same failure rules; its factor and
    the matrix its VJP takes stay in shared memory up to D = 112."""

    # the largest dimension whose per-chain vectors fit in shared memory beside the workspace
    MAX_USER_DIM = 1016

    def __init__(self, neg_log_dens, metric_chol_func, *, vjp_metric_chol_func=None,
                 grad_neg_log_dens=None, backend=None):
        self._accept_user_metric(neg_log_dens, metric_chol_func, CudaCholeskyMetric)
        super().__init__(neg_log_dens, grad_neg_log_dens=grad_neg_log_dens, backend=backend)
        if not isinstance(metric_chol_func, (QuadraticCholeskyMetric, CudaCholeskyMetric)):
            raise TypeError("`metric_chol_func` must be a registered metric model "
                            "(QuadraticCholeskyMetric) or a CudaCholeskyMetric.")
        if vjp_metric_chol_func is not None:
            raise ValueError("The metric VJP is fused into the kernels.")
        if isinstance(metric_chol_func, CudaCholeskyMetric):
            if neg_log_dens.dim > self.MAX_USER_DIM:
                raise ValueError(f"A CudaCholeskyMetric needs dim <= {self.MAX_USER_DIM}, "
                                 f"got {neg_log_dens.dim}.")
        elif metric_chol_func.dim != neg_log_dens.dim:
            raise ValueError(f"The base factor is {metric_chol_func.dim} x {metric_chol_func.dim}; "
                             f"the target has dimension {neg_log_dens.dim}.")
        self.metric_model = metric_chol_func
        self._rmetric_id = metric_chol_func.rmetric_id
        self._rmetric_params = metric_chol_func.params
        self._rmetric_aux = metric_chol_func.aux
