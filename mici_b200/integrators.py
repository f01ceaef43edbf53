"""Batched symplectic integrators -- drop-in for the three ``mici.integrators`` classes on the
hot path (reference ``src/mici/integrators.py``):

* ``LeapfrogIntegrator``             integrators.py:134-173
* ``ImplicitLeapfrogIntegrator``     integrators.py:381-544
* ``ConstrainedLeapfrogIntegrator``  integrators.py:684-984

Same constructor signatures, keyword names and defaults; ``step(state)`` returns a NEW state and
leaves its argument untouched (integrators.py:63-80).  A state holds ``[n_chains, dim]`` tensors:
one call advances every chain by one step in a single kernel launch.  ``step_n(state, n)`` fuses
``n`` steps per launch (the loop ``for _ in range(n_step): state = integrator.step(state)`` of
transitions.py:289-291).

Failures: the reference raises ``IntegratorError`` subclasses from ``step``.  For a batched
state the per-chain outcome is returned in ``new_state.status`` (0 ok, 1 ConvergenceError,
2 NonReversibleStepError, 3 LinAlgError) and failed chains keep their pre-step state; for a
single-chain state (1-D ``pos``) the matching exception is raised, as in the reference.
"""

from __future__ import annotations

import ctypes
from abc import ABC, abstractmethod

import torch

from . import _lib
from .errors import AdaptationError, compatible, raise_for_status
from .solvers import (
    maximum_norm,
    solve_fixed_point_direct,
    solve_fixed_point_steffensen,
    solve_projection_onto_manifold_newton,
    solve_projection_onto_manifold_newton_with_line_search,
    solve_projection_onto_manifold_quasi_newton,
)

_FUSED_FIXED_POINT_SOLVERS = (solve_fixed_point_direct, solve_fixed_point_steffensen)
_FUSED_PROJECTION_SOLVERS = (
    solve_projection_onto_manifold_newton,
    solve_projection_onto_manifold_quasi_newton,
    solve_projection_onto_manifold_newton_with_line_search,
)
from .states import ChainState
from .systems import (
    ConstrainedEuclideanMetricSystem,
    EuclideanMetricSystem,
    GaussianEuclideanMetricSystem,
    RiemannianMetricSystem,
    _batched,
    _dir_tensor,
    _like_input,
    _on_batch,
    _registry_euclidean,
)


class Integrator(ABC):
    """Base class for integrators (integrators.py:30-89)."""

    COUNTER_NAMES = ("grad_neg_log_dens", "metric", "quad_form_vjp", "solver_iters")

    def __init__(self, system, step_size=None):
        self.system = system
        self.step_size = step_size
        self.call_counts = None  # int32 [n_chains, 4] device tensor once `count_calls()` is on
        self._counting = False

    def count_calls(self, enable=True):
        """Switch the kernel-side call counters on / off (``mb200_set_call_counters``; the
        per-chain counterpart of ``ChainState._call_counts``, states.py:44-72).  While on, every
        ``step_n`` adds to ``self.call_counts[chain]``: gradient evaluations, metric builds
        (Riemannian: factorisations / eigendecompositions; constrained: constraint-Jacobian
        evaluations), quadratic-form VJPs and solver iterations (``COUNTER_NAMES`` order)."""
        self._counting = bool(enable)
        self.call_counts = None
        return self

    def call_count_totals(self):
        """``{name: total over chains}`` of the counters gathered since ``count_calls()``."""
        if self.call_counts is None:
            return dict.fromkeys(self.COUNTER_NAMES, 0)
        tot = self.call_counts.sum(0).tolist()
        return dict(zip(self.COUNTER_NAMES, (int(v) for v in tot)))

    def step(self, state):
        """Perform a single integrator step from a supplied state; returns a new state."""
        return self.step_n(state, 1)

    def step_n(self, state, n_steps, *, return_h=False):
        """``n_steps`` integrator steps fused in one launch; returns a new state.

        With ``return_h=True`` the Hamiltonian of the new state is evaluated in the same launch
        and stored as ``new_state.h`` (callers evaluate ``system.h`` after every trajectory:
        transitions.py:300-301).
        """
        if self.step_size is None:
            msg = (
                "Integrator `step_size` is `None`. This value should only be used if a "
                "step size adapter is being used to set the step size."
            )
            raise compatible(AdaptationError)(msg)
        pos, mom, d, single = _batched(state)
        n, dim = pos.shape
        dev = pos.device
        pos_out = torch.empty_like(pos)
        mom_out = torch.empty_like(mom)
        status = torch.empty(n, dtype=torch.int32, device=dev)
        n_done = torch.empty(n, dtype=torch.int32, device=dev)
        h = torch.empty(n, dtype=torch.float64, device=dev) if return_h else None
        if not isinstance(n_steps, torch.Tensor):
            n_steps = int(n_steps)
        if self._counting:
            if self.call_counts is None or self.call_counts.shape[0] != n \
                    or self.call_counts.device != dev:
                self.call_counts = torch.zeros(n, 4, dtype=torch.int32, device=dev)
            _lib.load().mb200_set_call_counters(_lib.ptr(self.call_counts))
        try:
            aux = self._launch(pos, mom, pos_out, mom_out, _dir_tensor(d, n, dev), n_steps, h,
                               status, n_done)
        finally:
            if self._counting:
                _lib.load().mb200_set_call_counters(None)
        new = _new_state_like(state, _like_input(state.pos, pos_out[0] if single else pos_out),
                              _like_input(state.pos, mom_out[0] if single else mom_out))
        if not isinstance(new, ChainState):  # foreign (reference) state object: no extra slots
            if single:
                raise_for_status(int(status.item()), type(self).__name__ + ".step")
            return new
        new.status = status
        new.n_done = n_done
        if return_h:
            new.h = h[0] if single else h
        if aux is not None:
            new.solver_iters = aux
        if single:
            raise_for_status(int(status.item()), type(self).__name__ + ".step")
        return new

    def step_n_host(self, pos, mom, n_steps, *, dir=1, out_pos=None, out_mom=None,  # noqa: A002
                    out_status=None, device="cuda", n_chunks=6):
        """``step_n`` for states that live in HOST memory (the reference's ``ChainState`` arrays
        are NumPy: states.py:160-305).  ``pos`` / ``mom`` are CPU tensors ``[n_chains, dim]``
        (pinned memory makes the copies asynchronous); the batch is cut into ``n_chunks`` row
        blocks, each on its own stream, so that the host->device copy of block ``k+1`` and the
        device->host copy of block ``k-1`` overlap the kernel of block ``k`` (chains are
        independent: chunking changes results at most in the last bits -- the tensor-core kernel
        chooses its accumulation split by launch size).  Returns ``(pos, mom, status)`` CPU tensors
        (written into ``out_*`` when given) after synchronising the streams.
        """
        dev = torch.device(device)
        pos = torch.as_tensor(pos)
        mom = torch.as_tensor(mom)
        n = pos.shape[0]
        out_pos = torch.empty_like(pos) if out_pos is None else out_pos
        out_mom = torch.empty_like(mom) if out_mom is None else out_mom
        out_status = torch.empty(n, dtype=torch.int32) if out_status is None else out_status
        n_chunks = max(1, min(int(n_chunks), n))
        if self._host_fast_path(pos, mom, dir, out_pos, out_mom, out_status, n_steps, dev,
                                n_chunks):
            return out_pos, out_mom, out_status
        streams = _host_streams(dev, n_chunks)
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(dev))
        bounds = [(n * c) // n_chunks for c in range(n_chunks + 1)]
        for c in range(n_chunks):
            lo, hi = bounds[c], bounds[c + 1]
            if hi == lo:
                continue
            st = streams[c]
            st.wait_event(ready)
            with torch.cuda.stream(st):
                d = dir[lo:hi] if isinstance(dir, torch.Tensor) else dir
                blk = ChainState(pos=pos[lo:hi].to(dev, non_blocking=True),
                                 mom=mom[lo:hi].to(dev, non_blocking=True), dir=d)
                new = self.step_n(blk, n_steps)
                out_pos[lo:hi].copy_(new.pos, non_blocking=True)
                out_mom[lo:hi].copy_(new.mom, non_blocking=True)
                out_status[lo:hi].copy_(new.status, non_blocking=True)
        for st in streams:
            st.synchronize()
        return out_pos, out_mom, out_status

    def _host_fast_path(self, pos, mom, dir, out_pos, out_mom, out_status, n_steps, dev,  # noqa: A002
                        n_chunks):
        """Chunked host-buffer launch inside the library (``mb200_leapfrog_euclidean_host``) when
        the integrator has one; returns False to fall back to the Python chunk loop."""
        return False

    def _step(self, state, time_step):
        """In-place single step with an explicit signed time step (integrators.py:82-89)."""
        saved = self.step_size
        try:
            self.step_size = abs(float(time_step))
            tmp = state.copy()
            if "dir" in tmp:
                tmp.dir = 1 if time_step >= 0 else -1
            new = self.step_n(tmp, 1)
        finally:
            self.step_size = saved
        state.pos, state.mom = new.pos, new.mom
        state.status, state.n_done = new.status, new.n_done

    @abstractmethod
    def _launch(self, pos, mom, pos_out, mom_out, dirs, n_steps, h, status, n_done):
        """Enqueue the kernel(s); may return a tensor of solver iteration counts."""


_STREAMS = {}


def _host_streams(dev, n):
    """Per-device pool of side streams for the chunked host-buffer path."""
    key = (dev.type, dev.index if dev.index is not None else torch.cuda.current_device())
    pool = _STREAMS.setdefault(key, [])
    while len(pool) < n:
        pool.append(torch.cuda.Stream(device=dev))
    return pool[:n]


def _new_state_like(state, pos, mom):
    if isinstance(state, ChainState):
        extra = {k: v for k, v in state._variables.items() if k not in ("pos", "mom")}
        extra = {k: (v.clone() if hasattr(v, "clone") else v) for k, v in extra.items()}
        return ChainState(pos=pos, mom=mom, **extra)
    new = state.copy()  # duck-typed foreign state object
    new.pos, new.mom = pos, mom
    return new


class TractableFlowIntegrator(Integrator):
    """integrators.py:92-131."""

    def __init__(self, system, step_size=None):
        if not hasattr(system, "h1_flow") or not hasattr(system, "h2_flow"):
            msg = (
                f"{type(self)} can only be used for systems with explicit `h1_flow` "
                f"and `h2_flow` Hamiltonian component flow maps. For systems in which "
                f"only `h1_flow` is available the `ImplicitLeapfrogIntegrator` class "
                f"may be used instead."
            )
            raise ValueError(msg)
        super().__init__(system, step_size)

    def _launch(self, pos, mom, pos_out, mom_out, dirs, n_steps, h, status, n_done):
        """Leapfrog (``self.coefficients is None``) or symmetric composition steps on a Euclidean
        system, with scalar or per-chain step sizes and trajectory lengths."""
        sysm = self.system
        if isinstance(sysm, GaussianEuclideanMetricSystem):
            return _launch_gaussian(sysm, self.step_size, pos, mom, pos_out, mom_out, dirs,
                                    n_steps, h, status, n_done, self.coefficients,
                                    self.initial_h1_flow_step)
        n, dim = pos.shape
        dev = pos.device
        eps, eps_t, ns, max_n = _step_args(self.step_size, n_steps, n, dev)
        coefs, n_flows = _coefficients_arg(self.coefficients)
        model = sysm._model(dev)
        # a user-written target runs the general-dimension kernel of its run-time compiled image
        _lib.call(
            "mb200_leapfrog_euclidean", _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(pos_out),
            _lib.ptr(mom_out), _lib.ptr(dirs), n, dim, eps, _lib.ptr(eps_t), max_n, _lib.ptr(ns),
            n_flows, coefs, 1 if self.initial_h1_flow_step else 0, sysm.metric.kind,
            _lib.ptr(sysm.metric.inv_device(dev)), ctypes.byref(model), _lib.ptr(h),
            _lib.ptr(status), _lib.ptr(n_done), _lib.current_stream_ptr(dev), target=sysm.target)


def _step_args(step_size, n_steps, n, dev):
    """``(eps, eps_t, ns, max_n)`` of an integrator launch: the scalar step size and trajectory
    length, and the per-chain device arrays, ``None`` where the argument is a scalar.  A per-chain
    step size is a ``[n_chains]`` tensor (one dual-averaging state per chain during warm-up,
    adapters.py:262-283, 373), a per-chain length an integer tensor (transitions.py:355-412)."""
    if isinstance(step_size, torch.Tensor) and step_size.ndim == 1:
        if step_size.shape[0] != n:
            raise ValueError(f"per-chain step_size has {step_size.shape[0]} entries for {n} chains")
        eps, eps_t = 0.0, step_size.to(device=dev, dtype=torch.float64).contiguous()
    else:
        eps, eps_t = float(step_size), None
    if isinstance(n_steps, torch.Tensor):
        if n_steps.shape != (n,):
            raise ValueError("per-chain n_steps must have one entry per chain")
        ns = n_steps.to(device=dev, dtype=torch.int32).contiguous()
        return eps, eps_t, ns, (int(ns.max().item()) if n > 0 else 0)
    return eps, eps_t, None, int(n_steps)


def _coefficients_arg(coefficients):
    """``(HOST array pointer, n_flows)`` of a splitting schedule; ``(None, 0)`` for leapfrog."""
    if coefficients is None:
        return None, 0
    coefs = (ctypes.c_double * len(coefficients))(*coefficients)
    return ctypes.cast(coefs, ctypes.c_void_p), len(coefficients)


def _launch_gaussian(system, step_size, pos, mom, pos_out, mom_out, dirs, n_steps, h, status,
                     n_done, coefficients=None, initial_h1_flow_step=True):
    """``mb200_leapfrog_gaussian_euclidean``: leapfrog / composition over the flows of a
    ``GaussianEuclideanMetricSystem`` (systems.py:369-474)."""
    n, dim = pos.shape
    dev = pos.device
    if isinstance(n_steps, torch.Tensor):
        raise NotImplementedError("per-chain trajectory lengths: plain Euclidean systems only")
    model = system._model(dev)
    eps, eps_t, _, n_steps = _step_args(step_size, n_steps, n, dev)
    coefs, n_flows = _coefficients_arg(coefficients)
    if coefficients is None:
        drift = [1.0]
    else:
        first_drift = 1 if initial_h1_flow_step else 0
        drift = list(coefficients[first_drift::2])
    if eps_t is not None and system.metric.kind == 2:
        raise NotImplementedError("per-chain step sizes with a dense Gaussian-split metric")
    rot = system.rotation_device(dev, eps, drift)
    _lib.call(
        "mb200_leapfrog_gaussian_euclidean", _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(pos_out),
        _lib.ptr(mom_out), _lib.ptr(dirs), n, dim, eps, _lib.ptr(eps_t), n_steps, n_flows, coefs,
        1 if initial_h1_flow_step else 0, system.metric.kind,
        _lib.ptr(system.metric.inv_device(dev)), _lib.ptr(rot), ctypes.byref(model), _lib.ptr(h),
        _lib.ptr(status), _lib.ptr(n_done), _lib.current_stream_ptr(dev))


def _gaussian_flow(system, state, dt):
    """In-place ``h2_flow`` of a Gaussian-split system: a one-flow schedule {drift 1.0}."""

    def launch(pos, mom, _):
        n = pos.shape[0]
        pos_out, mom_out = torch.empty_like(pos), torch.empty_like(mom)
        if isinstance(dt, torch.Tensor) and dt.ndim == 1:
            dirs = torch.where(dt < 0, -1, 1).to(torch.int32)
            eps = dt.abs()
        else:
            dirs = None if float(dt) >= 0 else torch.full((n,), -1, dtype=torch.int32,
                                                          device=pos.device)
            eps = abs(float(dt))
        _launch_gaussian(system, eps, pos, mom, pos_out, mom_out, dirs, 1, None, None, None,
                         coefficients=[1.0], initial_h1_flow_step=False)
        return pos_out, mom_out

    state.pos, state.mom = _on_batch(state, launch)


def _is_per_chain(step_size, n_steps):
    return (isinstance(step_size, torch.Tensor) and step_size.ndim == 1) or isinstance(
        n_steps, torch.Tensor)


class LeapfrogIntegrator(TractableFlowIntegrator):
    """Explicit leapfrog Psi(t) = Phi_1(t/2) o Phi_2(t) o Phi_1(t/2) (integrators.py:134-173)
    for ``EuclideanMetricSystem`` s, target gradient and metric product fused in one kernel."""

    # splitting schedule of TractableFlowIntegrator._launch: None is leapfrog {0.5, 1, 0.5}
    coefficients = None
    initial_h1_flow_step = True

    def __init__(self, system, step_size=None):
        super().__init__(system, step_size)
        if not isinstance(system, EuclideanMetricSystem) or isinstance(
            system, ConstrainedEuclideanMetricSystem
        ):
            raise TypeError("LeapfrogIntegrator needs an (unconstrained) EuclideanMetricSystem.")

    def _host_fast_path(self, pos, mom, dir, out_pos, out_mom, out_status, n_steps, dev,  # noqa: A002
                        n_chunks):
        tensors = (pos, mom, out_pos, out_mom)
        if (not _registry_euclidean(self.system)
                or _is_per_chain(self.step_size, n_steps) or self.step_size is None
                or any(t.device.type != "cpu" or t.dtype != torch.float64 or not t.is_contiguous()
                       for t in tensors)
                or out_status.dtype != torch.int32 or not out_status.is_contiguous()):
            return False
        n, dim = pos.shape
        dir_t = None
        if isinstance(dir, torch.Tensor):
            if dir.device.type != "cpu":
                return False
            dir_t = dir.to(torch.int32).contiguous()
        elif int(dir) != 1:
            dir_t = torch.full((n,), int(dir), dtype=torch.int32)
        sysm = self.system
        scratch = sysm._scratch("host_scratch", int(_lib.load().mb200_host_scratch_bytes(n, dim)),
                                dev)
        n_streams = min(n_chunks, 8)
        streams = _host_streams(dev, n_streams)
        handles = (ctypes.c_void_p * n_streams)(*[s.cuda_stream for s in streams])
        model = sysm._model(dev)
        with torch.cuda.device(dev):
            torch.cuda.current_stream(dev).synchronize()  # inputs / scratch of earlier work
            _lib.call(
                "mb200_leapfrog_euclidean_host", _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(out_pos),
                _lib.ptr(out_mom), _lib.ptr(dir_t), n, dim, float(self.step_size), int(n_steps),
                sysm.metric.kind, _lib.ptr(sysm.metric.inv_device(dev)), ctypes.byref(model),
                _lib.ptr(out_status), n_chunks, ctypes.cast(handles, ctypes.c_void_p), n_streams,
                _lib.ptr(scratch), scratch.numel(), 1)
        return True


class SymmetricCompositionIntegrator(TractableFlowIntegrator):
    """Symmetric composition (splitting) integrator for ``EuclideanMetricSystem`` s
    (integrators.py:176-289) -- "next" row N4.  Same constructor as the reference: the full
    symmetric coefficient sequence is derived from ``free_coefficients`` exactly as in
    integrators.py:268-277; flows alternate ``a, b, ..., a`` with ``a = h1_flow`` if
    ``initial_h1_flow_step`` else ``h2_flow`` (:278-281)."""

    def __init__(self, system, free_coefficients, *, step_size=None, initial_h1_flow_step=True):
        super().__init__(system, step_size)
        if not isinstance(system, EuclideanMetricSystem) or isinstance(
            system, ConstrainedEuclideanMetricSystem
        ):
            raise TypeError("Composition integrators need an (unconstrained) EuclideanMetricSystem.")
        self.initial_h1_flow_step = initial_h1_flow_step
        n_free_coefficients = len(free_coefficients)
        coefficients = list(free_coefficients)
        coefficients.append(0.5 - sum(free_coefficients[(n_free_coefficients) % 2 :: 2]))
        coefficients.append(1 - 2 * sum(free_coefficients[(n_free_coefficients + 1) % 2 :: 2]))
        self.coefficients = coefficients + coefficients[-2::-1]


class BCSSTwoStageIntegrator(SymmetricCompositionIntegrator):
    """Blanes-Casas-Sanz-Serna two-stage integrator (integrators.py:292-316)."""

    def __init__(self, system, step_size=None):
        a_0 = (3 - 3**0.5) / 6
        super().__init__(system, (a_0,), step_size=step_size, initial_h1_flow_step=True)


class BCSSThreeStageIntegrator(SymmetricCompositionIntegrator):
    """Three-stage BCSS integrator (integrators.py:319-347)."""

    def __init__(self, system, step_size=None):
        a_0 = 0.11888010966548
        b_1 = 0.29619504261126
        super().__init__(system, (a_0, b_1), step_size=step_size, initial_h1_flow_step=True)


class BCSSFourStageIntegrator(SymmetricCompositionIntegrator):
    """Four-stage BCSS integrator (integrators.py:350-378)."""

    def __init__(self, system, step_size=None):
        a_0 = 0.071353913450279725904
        b_1 = 0.191667800000000000000
        a_1 = 0.268548791161230105820
        super().__init__(system, (a_0, b_1, a_1), step_size=step_size, initial_h1_flow_step=True)


class _ImplicitIntegrator(Integrator):
    """Implicit integrators on ``RiemannianMetricSystem`` s: the fixed-point solves and the
    reversibility check run inside the kernel."""

    _ENTRY = None  # C entry point
    _WORKSPACE = False  # whether the entry point takes the system's workspace

    def __init__(self, system, step_size=None, reverse_check_tol=2e-8,
                 reverse_check_norm=maximum_norm, fixed_point_solver=solve_fixed_point_direct,
                 fixed_point_solver_kwargs=None):
        super().__init__(system, step_size)
        if not isinstance(system, RiemannianMetricSystem):
            raise TypeError(f"{type(self).__name__} needs a RiemannianMetricSystem.")
        if reverse_check_norm is not maximum_norm:
            raise ValueError("Only `maximum_norm` is available for the reversibility check.")
        if fixed_point_solver not in _FUSED_FIXED_POINT_SOLVERS:
            raise ValueError("Only `solve_fixed_point_direct` and `solve_fixed_point_steffensen` "
                             "are fused into the kernels.")
        self.reverse_check_tol = reverse_check_tol
        self.reverse_check_norm = reverse_check_norm
        self.fixed_point_solver = fixed_point_solver
        self.fixed_point_solver_kwargs = dict(fixed_point_solver_kwargs or {})

    def _launch(self, pos, mom, pos_out, mom_out, dirs, n_steps, h, status, n_done):
        n, dim = pos.shape
        dev = pos.device
        sysm = self.system
        kw = self.fixed_point_solver.resolve_kwargs(self.fixed_point_solver_kwargs)
        model = sysm._model(dev)
        eps, eps_t, ns, max_n = _step_args(self.step_size, n_steps, n, dev)
        iters = torch.zeros((n, 4), dtype=torch.int32, device=dev)
        if self._WORKSPACE:
            ws = sysm._workspace(n, dim, dev)
            ws_args = (_lib.ptr(ws), ws.numel())
        else:
            ws_args = ()
        _lib.call(
            self._ENTRY, _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(pos_out), _lib.ptr(mom_out),
            _lib.ptr(dirs), n, dim, eps, _lib.ptr(eps_t), max_n, _lib.ptr(ns), ctypes.byref(model),
            self.fixed_point_solver.kind, float(kw["convergence_tol"]),
            float(kw["divergence_tol"]), int(kw["max_iters"]), float(self.reverse_check_tol),
            _lib.ptr(h), _lib.ptr(status), _lib.ptr(n_done), _lib.ptr(iters), *ws_args,
            _lib.current_stream_ptr(dev), target=sysm._user_pair)
        return iters


class ImplicitLeapfrogIntegrator(_ImplicitIntegrator):
    """Implicit generalised leapfrog for non-separable Hamiltonians (integrators.py:381-544),
    for ``RiemannianMetricSystem`` s.  Fixed-point solves and reversibility checks run inside
    the kernel.  NB: as in the reference at this commit every sub-map receives the full
    ``dir * step_size`` (integrators.py:538-544; SURVEY.md H3)."""

    _ENTRY = "mb200_implicit_leapfrog_riemannian"
    _WORKSPACE = True


class ImplicitMidpointIntegrator(_ImplicitIntegrator):
    """Implicit midpoint integrator for general Hamiltonians (integrators.py:547-681) --
    "next" row N4 -- for ``RiemannianMetricSystem`` s: a fixed-point solve in ``(q, p)`` for the
    forward half-step, an explicit Euler half-step and a reversibility check, all inside the
    kernel.  Same constructor as the reference."""

    _ENTRY = "mb200_implicit_midpoint_riemannian"


class ConstrainedLeapfrogIntegrator(TractableFlowIntegrator):
    """Leapfrog for constrained systems: RATTLE / geodesic integrator with Newton projection
    and reversibility check (integrators.py:684-984).  A
    ``GaussianDenseConstrainedEuclideanMetricSystem`` runs through its own entry point, whose
    drift is the exact rotation of the Gaussian split."""

    def __init__(self, system, step_size=None, n_inner_step=1, reverse_check_tol=2e-8,
                 reverse_check_norm=maximum_norm,
                 projection_solver=solve_projection_onto_manifold_newton,
                 projection_solver_kwargs=None):
        super().__init__(system, step_size)
        if not isinstance(system, ConstrainedEuclideanMetricSystem):
            raise TypeError("ConstrainedLeapfrogIntegrator needs a constrained Euclidean system.")
        if reverse_check_norm is not maximum_norm:
            raise ValueError("Only `maximum_norm` is available for the reversibility check.")
        if projection_solver not in _FUSED_PROJECTION_SOLVERS:
            raise ValueError("Only the Newton, quasi-Newton and Newton-with-line-search projection "
                             "solvers of `mici_b200.solvers` are fused into the kernels.")
        self.n_inner_step = n_inner_step
        self.reverse_check_tol = reverse_check_tol
        self.reverse_check_norm = reverse_check_norm
        self.projection_solver = projection_solver
        self.projection_solver_kwargs = dict(projection_solver_kwargs or {})

    def _launch(self, pos, mom, pos_out, mom_out, dirs, n_steps, h, status, n_done):
        n = pos.shape[0]
        dev = pos.device
        kw = self.projection_solver.resolve_kwargs(self.projection_solver_kwargs)
        eps, eps_t, ns, max_n = _step_args(self.step_size, n_steps, n, dev)
        iters = torch.zeros(n, dtype=torch.int32, device=dev)
        self.system._leapfrog(pos, mom, pos_out, mom_out, dirs, eps, eps_t, max_n, ns,
                              self.n_inner_step, self.projection_solver, kw,
                              self.reverse_check_tol, h, status, n_done, iters)
        return iters
