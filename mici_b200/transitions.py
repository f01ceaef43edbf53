"""Batched Markov transitions around the integrators -- "next" rows N1 / N4 of SURVEY.md 8(f).

Mirrors, for all chains at once, the reference's transitions:

* ``IndependentMomentumTransition``             transitions.py:129-142
* ``CorrelatedMomentumTransition``              transitions.py:145-198
* ``MetropolisStaticIntegrationTransition``     transitions.py:256-352
* ``MetropolisRandomIntegrationTransition``     transitions.py:355-402 (per-chain trajectory lengths)
* ``MultinomialDynamicIntegrationTransition``   transitions.py:487-809 (fused NUTS kernel)
* ``SliceDynamicIntegrationTransition``         transitions.py:812-858
* ``sample_hmc`` / ``sample_chains``            samplers.py:459-513, 1075-1141 (staged sampling)

so that a whole HMC iteration (momentum refresh, ``n_step`` fused integrator steps, energy,
accept / reject, direction flips) stays on the GPU: two kernel launches for the trajectory
(``system.h`` of the current state, then ``integrator.step_n(..., return_h=True)``) and one for
the Metropolis select (``mb200_metropolis_select``).

Random numbers.  ``rng`` is either a ``numpy.random.Generator`` (one stream for the whole batch),
a sequence of per-chain generators (each chain then consumes exactly the variates the reference
consumes from its own stream: ``standard_normal(dim)`` then one ``uniform()``, which is what the
parity tests use), or a ``torch.Generator`` on the device (variates generated on the GPU).
"""

from __future__ import annotations

import ctypes
from collections.abc import Sequence

import numpy as np
import torch

from . import _lib
from .states import ChainState
from .systems import _dir_tensor, _registry_euclidean


def _normals(rng, shape, device):
    if isinstance(rng, torch.Generator):
        return torch.randn(shape, dtype=torch.float64, device=device, generator=rng)
    if isinstance(rng, Sequence):
        z = np.stack([g.standard_normal(shape[1:]) for g in rng])
    else:
        z = rng.standard_normal(shape)
    return torch.as_tensor(z, device=device)


def _uniform_table(rng, n, n_uniforms, device):
    """The ``[n, n_uniforms]`` uniforms of one dynamic transition, and the state of each per-chain
    generator before the draw (``None`` unless ``rng`` is a sequence of generators)."""
    if isinstance(rng, torch.Generator):
        return torch.rand((n, n_uniforms), dtype=torch.float64, device=device, generator=rng), None
    if isinstance(rng, Sequence):
        saved = [g.bit_generator.state for g in rng]
        return torch.as_tensor(np.stack([g.uniform(size=n_uniforms) for g in rng]),
                               device=device), saved
    return torch.as_tensor(rng.uniform(size=(n, n_uniforms)), device=device), None


def _replay(rng, saved, used):
    """Leave every chain's generator advanced by exactly the ``used`` uniforms its chain
    consumed."""
    if saved is None:
        return
    for g, st, k in zip(rng, saved, used.cpu().tolist()):
        g.bit_generator.state = st
        if k:
            g.uniform(size=k)


def _uniforms(rng, n, device, mask=None):
    if isinstance(rng, torch.Generator):
        return torch.rand(n, dtype=torch.float64, device=device, generator=rng)
    if isinstance(rng, Sequence):
        # the reference draws `rng.uniform()` only for chains whose trajectory did not fail
        # (short-circuit in transitions.py:310); keep the per-chain streams in step with it
        u = np.array([g.uniform() if (mask is None or mask[i]) else 2.0 for i, g in enumerate(rng)])
    else:
        u = rng.uniform(size=n)
    return torch.as_tensor(u, device=device)


class IndependentMomentumTransition:
    """Resample every chain's momentum from N(0, M) (transitions.py:129-142)."""

    state_variables = frozenset({"mom"})
    statistic_types = None

    def __init__(self, system):
        self.system = system

    def sample(self, state, rng):
        state.mom = self.system.sample_momentum(state, rng)
        return state, None


def _integers(rng, lo, hi, n, device):
    """Per-chain ``rng.integers(lo, hi)`` (transitions.py:401)."""
    if isinstance(rng, torch.Generator):
        return torch.randint(lo, hi, (n,), dtype=torch.int32, device=device, generator=rng)
    if isinstance(rng, Sequence):
        k = np.array([g.integers(lo, hi) for g in rng], dtype=np.int32)
    else:
        k = rng.integers(lo, hi, size=n).astype(np.int32)
    return torch.as_tensor(k, device=device)


class CorrelatedMomentumTransition:
    """Partial momentum refresh ``mom <- sqrt(1 - c^2) mom + c * sample`` for every chain
    (transitions.py:145-198)."""

    state_variables = frozenset({"mom"})
    statistic_types = None

    def __init__(self, system, mom_resample_coeff=1.0):
        if not (mom_resample_coeff >= 0 and mom_resample_coeff <= 1):
            raise ValueError("mom_resample_coeff should have a value in the interval [0, 1].")
        self.system = system
        self.mom_resample_coeff = mom_resample_coeff

    def sample(self, state, rng):
        if state.mom is None or self.mom_resample_coeff == 1:
            state.mom = self.system.sample_momentum(state, rng)
        elif self.mom_resample_coeff != 0:
            mom_ind = self.system.sample_momentum(state, rng)
            state.mom = state.mom * (1.0 - self.mom_resample_coeff**2) ** 0.5 + (
                self.mom_resample_coeff * mom_ind)
        return state, None


class MetropolisIntegrationTransition:
    """Trajectory + Metropolis accept step for all chains (transitions.py:235-315).  ``sample``
    returns ``(state, stats)`` where ``stats`` holds per-chain tensors with the reference's
    statistic names (transitions.py:226-232, 273)."""

    state_variables = frozenset({"pos", "mom", "dir"})

    def __init__(self, system, integrator):
        self.system = system
        self.integrator = integrator

    def _sample_n_step(self, state, n_step, rng):
        """``n_step``: one integer for all chains or an integer tensor ``[n_chains]``."""
        n, dim = state.pos.shape
        dev = state.pos.device
        h_init = self.system.h(state)
        prop = self.integrator.step_n(state, n_step, return_h=True)
        status, n_done = prop.status, prop.n_done
        dirs = _dir_tensor(state.dir if "dir" in state else 1, n, dev)
        if dirs is None:
            dirs = torch.ones(n, dtype=torch.int32, device=dev)
        else:
            dirs = dirs.clone()
        mask = None
        if isinstance(rng, Sequence):
            mask = (status == 0).cpu().numpy()
        u = _uniforms(rng, n, dev, mask)
        pos, mom = state.pos.clone(), state.mom.clone()
        accept_prob = torch.empty(n, dtype=torch.float64, device=dev)
        accept_stat = torch.empty(n, dtype=torch.float64, device=dev)
        accepted = torch.empty(n, dtype=torch.int32, device=dev)
        _lib.call("mb200_metropolis_select", _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(prop.pos),
                  _lib.ptr(prop.mom), _lib.ptr(h_init), _lib.ptr(prop.h), _lib.ptr(status),
                  _lib.ptr(n_done), _lib.ptr(dirs), _lib.ptr(u), n, dim, _lib.ptr(accept_prob),
                  _lib.ptr(accept_stat), _lib.ptr(accepted), _lib.current_stream_ptr(dev))
        new = ChainState(pos=pos, mom=mom, dir=dirs)
        stats = {
            "n_step": n_done.to(torch.int64),
            "accept_stat": accept_stat,
            "metrop_accept_prob": accept_prob,
            "convergence_error": status == 1,
            "non_reversible_step": status == 2,
            "step_size": _step_size_stat(self.integrator.step_size, n, dev),
            "accepted": accepted.bool(),
        }
        return new, stats


def _step_size_stat(step_size, n, dev):
    if isinstance(step_size, torch.Tensor) and step_size.ndim == 1:
        return step_size.to(device=dev, dtype=torch.float64).clone()
    return torch.full((n,), float(step_size), dtype=torch.float64, device=dev)


class MetropolisStaticIntegrationTransition(MetropolisIntegrationTransition):
    """Static-trajectory HMC transition (transitions.py:318-352)."""

    def __init__(self, system, integrator, n_step):
        super().__init__(system, integrator)
        if n_step <= 0:
            raise ValueError("Number of integrator steps must be positive.")
        self.n_step = int(n_step)

    def sample(self, state, rng):
        return self._sample_n_step(state, self.n_step, rng)


class MetropolisRandomIntegrationTransition(MetropolisIntegrationTransition):
    """Trajectory length drawn per chain and per transition from ``rng.integers(lower, upper)``
    (transitions.py:355-402; NumPy's ``integers`` excludes ``upper``); all chains still advance
    in one launch (the ``n_steps_per_chain`` array of the integrator entry points)."""

    def __init__(self, system, integrator, n_step_range):
        super().__init__(system, integrator)
        n_step_lower, n_step_upper = n_step_range
        if not (n_step_lower > 0 and n_step_lower < n_step_upper):
            raise ValueError("Range bounds must be non-negative and first entry less than last.")
        self.n_step_range = (int(n_step_lower), int(n_step_upper))

    def sample(self, state, rng):
        n = state.pos.shape[0]
        n_step = _integers(rng, *self.n_step_range, n, state.pos.device)
        return self._sample_n_step(state, n_step, rng)


def euclidean_no_u_turn_criterion(system, state_1, state_2, _sum_mom):
    """transitions.py:405-436: terminate when either terminal velocity points against
    ``state_2.pos - state_1.pos``.  Passed to the dynamic transitions to select the fused test."""
    diff = state_2.pos - state_1.pos
    return ((system.dh_dmom(state_1) * diff).sum(-1) < 0) | (
        (system.dh_dmom(state_2) * diff).sum(-1) < 0)


def riemannian_no_u_turn_criterion(system, state_1, state_2, sum_mom):
    """transitions.py:439-470: the same test against the sum of the trajectory's momenta."""
    return ((system.dh_dmom(state_1) * sum_mom).sum(-1) < 0) | (
        (system.dh_dmom(state_2) * sum_mom).sum(-1) < 0)


class DynamicIntegrationTransition:
    """Dynamic-length integration transition (NUTS) for all chains (transitions.py:487-770).
    Same constructor as the reference; use the ``Multinomial...`` / ``Slice...`` subclasses.

    * ``LeapfrogIntegrator`` on an ``EuclideanMetricSystem`` (shared or per-chain step size):
      every chain builds its own binary trajectory tree inside ``mb200_nuts_euclidean`` (one warp
      per chain, ONE launch per transition).
    * Any other integrator / system (``ConstrainedLeapfrogIntegrator``,
      ``ImplicitLeapfrogIntegrator``, compositions ...): the chains grow their trees in lock-step,
      one batched ``integrator.step`` per leaf, with the tree bookkeeping (weights, binary-counter
      merges, no-U-turn tests, progressive sampling) in the ``mb200_nuts_generic_*`` kernels; a
      failed step terminates that chain's tree and sets ``convergence_error`` /
      ``non_reversible_step`` as transitions.py:670-676 does.

    Random numbers: the kernel consumes, per chain, exactly the uniform variates the reference
    draws from that chain's generator, in the same order.  With a sequence of per-chain NumPy
    generators each stream is left advanced by exactly the number its chain used."""

    state_variables = frozenset({"pos", "mom", "dir"})
    _slice = None

    def __init__(self, system, integrator, *, max_tree_depth=10, max_delta_h=1000.0,
                 termination_criterion=riemannian_no_u_turn_criterion,
                 do_extra_subtree_checks=True):
        from .integrators import LeapfrogIntegrator  # noqa: PLC0415

        if self._slice is None:
            raise TypeError("Use MultinomialDynamicIntegrationTransition or "
                            "SliceDynamicIntegrationTransition.")
        if max_tree_depth <= 0:
            raise ValueError("max_tree_depth must be non-negative.")
        if termination_criterion not in (euclidean_no_u_turn_criterion,
                                         riemannian_no_u_turn_criterion):
            raise ValueError("Only the two no-U-turn criteria of this module are fused.")
        # LeapfrogIntegrator on a plain EuclideanMetricSystem: whole transitions in ONE launch
        # (mb200_nuts_euclidean).  Every other pair (constrained, implicit, compositions,
        # Gaussian splitting, user-written targets): lock-step leaves through the integrator's own
        # kernels with the tree bookkeeping in the mb200_nuts_generic_* kernels.
        self._fused = type(integrator) is LeapfrogIntegrator and _registry_euclidean(system)
        self.system = system
        self.integrator = integrator
        self.max_tree_depth = int(max_tree_depth)
        self.max_delta_h = float(max_delta_h)
        self.termination_criterion = termination_criterion
        self.do_extra_subtree_checks = bool(do_extra_subtree_checks)

    @property
    def n_uniforms(self):
        """Upper bound on the ``rng.uniform()`` calls of one transition of one chain."""
        return 2 * self.max_tree_depth + 2**self.max_tree_depth + (1 if self._slice else 0)

    def sample(self, state, rng):
        from .errors import AdaptationError  # noqa: PLC0415

        if self.integrator.step_size is None:
            raise AdaptationError("Integrator `step_size` is `None`.")
        if not self._fused:
            return self._sample_generic(state, rng)
        pos, mom = state.pos.contiguous(), state.mom.contiguous()
        n, dim = pos.shape
        dev = pos.device
        n_uni = self.n_uniforms
        uni, saved = _uniform_table(rng, n, n_uni, dev)
        nbytes = int(_lib.load().mb200_nuts_workspace_bytes(n, dim, self.max_tree_depth))
        if nbytes < 0:
            raise ValueError("unsupported dim / max_tree_depth for the fused dynamic transition")
        ws = self.system._scratch("nuts_ws", nbytes, dev)
        eps = self.integrator.step_size
        per_chain = isinstance(eps, torch.Tensor) and eps.ndim == 1
        eps_t = eps.to(device=dev, dtype=torch.float64).contiguous() if per_chain else None
        pos_out, mom_out = torch.empty_like(pos), torch.empty_like(mom)
        f64 = {"dtype": torch.float64, "device": dev}
        i32 = {"dtype": torch.int32, "device": dev}
        h, av, rej = torch.empty(n, **f64), torch.empty(n, **f64), torch.empty(n, **f64)
        n_step, depth, div = torch.empty(n, **i32), torch.empty(n, **i32), torch.empty(n, **i32)
        used, status, dir_out = torch.empty(n, **i32), torch.empty(n, **i32), torch.empty(n, **i32)
        m = self.system.metric
        model = self.system._model(dev)
        _lib.call(
            "mb200_nuts_euclidean", _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(pos_out),
            _lib.ptr(mom_out), n, dim, 0.0 if per_chain else float(eps), _lib.ptr(eps_t), m.kind,
            _lib.ptr(m.inv_device(dev)), ctypes.byref(model), 1 if self._slice else 0,
            1 if self.termination_criterion is euclidean_no_u_turn_criterion else 0,
            1 if self.do_extra_subtree_checks else 0, self.max_tree_depth, self.max_delta_h,
            _lib.ptr(uni), n_uni, _lib.ptr(ws), ws.numel(), _lib.ptr(h), _lib.ptr(n_step),
            _lib.ptr(av), _lib.ptr(rej), _lib.ptr(depth), _lib.ptr(div), _lib.ptr(used),
            _lib.ptr(dir_out), _lib.ptr(status), _lib.current_stream_ptr(dev))
        _replay(rng, saved, used)
        if bool((status != 0).any()):
            raise RuntimeError("dynamic transition ran out of uniform variates")
        diverging = div.bool()
        no_failure = {"dtype": torch.bool, "device": dev}
        return _dynamic_result(pos_out, mom_out, dir_out, h, n_step, av, rej, depth, diverging,
                               torch.zeros(n, **no_failure), torch.zeros(n, **no_failure),
                               diverging, eps)

    def _sample_generic(self, state, rng):
        """Lock-step dynamic transition through the integrator's own step kernels."""
        pos, mom = state.pos.contiguous(), state.mom.contiguous()
        n, dim = pos.shape
        dev = pos.device
        n_uni = self.n_uniforms
        uni, saved = _uniform_table(rng, n, n_uni, dev)
        lib = _lib.load()
        system, integ = self.system, self.integrator
        ws_bytes = int(lib.mb200_nuts_workspace_bytes(n, dim, self.max_tree_depth))
        cs_bytes = int(lib.mb200_nuts_generic_state_bytes(n))
        if ws_bytes < 0:
            raise ValueError("unsupported dim / max_tree_depth for the dynamic transition")
        ws = system._scratch("nuts_ws", ws_bytes, dev)
        cs = torch.empty(max(cs_bytes, 8), dtype=torch.uint8, device=dev)
        opts = _lib.NutsOptions()
        opts.max_tree_depth = self.max_tree_depth
        opts.slice_variant = 1 if self._slice else 0
        opts.euclidean_criterion = (
            1 if self.termination_criterion is euclidean_no_u_turn_criterion else 0)
        opts.extra_subtree_checks = 1 if self.do_extra_subtree_checks else 0
        opts.max_delta_h = self.max_delta_h
        opts.uniforms = uni.data_ptr()
        opts.n_uniforms = n_uni
        o = ctypes.byref(opts)
        stream = _lib.current_stream_ptr(dev)
        f64 = {"dtype": torch.float64, "device": dev}
        i32 = {"dtype": torch.int32, "device": dev}
        init = ChainState(pos=pos, mom=mom, dir=1)
        h0 = system.h(init).contiguous()
        v0 = system.dh_dmom(init).contiguous()
        _lib.call("mb200_nuts_generic_begin", _lib.ptr(pos), _lib.ptr(mom), _lib.ptr(v0),
                  _lib.ptr(h0), n, dim, o, _lib.ptr(ws), ws.numel(), _lib.ptr(cs), cs.numel(),
                  stream)
        q_edge, p_edge = torch.empty_like(pos), torch.empty_like(mom)
        dirs, active = torch.empty(n, **i32), torch.empty(n, **i32)
        for depth in range(self.max_tree_depth):
            _lib.call("mb200_nuts_generic_start", n, dim, depth, o, _lib.ptr(ws), _lib.ptr(cs),
                      _lib.ptr(q_edge), _lib.ptr(p_edge), _lib.ptr(dirs), _lib.ptr(active), stream)
            if not bool(active.any()):
                break
            cur = ChainState(pos=q_edge, mom=p_edge, dir=dirs)
            n_leaves = 2**depth
            for k in range(1, n_leaves + 1):
                new = integ.step_n(cur, 1, return_h=True)
                vel = system.dh_dmom(_quiet(new)).contiguous()
                _lib.call("mb200_nuts_generic_leaf", _lib.ptr(new.pos), _lib.ptr(new.mom),
                          _lib.ptr(vel), _lib.ptr(new.h), _lib.ptr(new.status), n, dim, k,
                          n_leaves, o, _lib.ptr(ws), _lib.ptr(cs), _lib.ptr(active), stream)
                cur = ChainState(pos=new.pos, mom=new.mom, dir=dirs)
                # every chain's doubling may have terminated early: look now and then
                if k < n_leaves and (k & 7) == 0 and not bool(active.any()):
                    break
            _lib.call("mb200_nuts_generic_finish", n, dim, depth, o, _lib.ptr(ws), _lib.ptr(cs),
                      stream)
        pos_out, mom_out = torch.empty_like(pos), torch.empty_like(mom)
        h, av, rej = torch.empty(n, **f64), torch.empty(n, **f64), torch.empty(n, **f64)
        n_step, tdepth, flags = torch.empty(n, **i32), torch.empty(n, **i32), torch.empty(n, **i32)
        used, dir_out = torch.empty(n, **i32), torch.empty(n, **i32)
        _lib.call("mb200_nuts_generic_end", n, dim, o, _lib.ptr(ws), _lib.ptr(cs),
                  _lib.ptr(pos_out), _lib.ptr(mom_out), _lib.ptr(h), _lib.ptr(n_step), _lib.ptr(av),
                  _lib.ptr(rej), _lib.ptr(tdepth), _lib.ptr(flags), _lib.ptr(used),
                  _lib.ptr(dir_out), stream)
        _replay(rng, saved, used)
        if bool(((flags >> 3) & 1).any()):
            raise RuntimeError("dynamic transition ran out of uniform variates")
        diverging = (flags & 1).bool()
        conv = ((flags >> 1) & 1).bool()
        nonrev = ((flags >> 2) & 1).bool()
        return _dynamic_result(pos_out, mom_out, dir_out, h, n_step, av, rej, tdepth, diverging,
                               conv, nonrev, diverging | conv | nonrev, integ.step_size)


def _dynamic_result(pos, mom, dirs, h, n_step, av, rej, depth, diverging, conv, nonrev, failed,
                    step_size):
    """The next state and the statistics of a dynamic transition (transitions.py:758-769); a
    failed chain's ``accept_stat`` is 0."""
    n = pos.shape[0]
    new = ChainState(pos=pos, mom=mom, dir=dirs)
    new.h = h
    stats = {
        "n_step": n_step.to(torch.int64),
        "accept_stat": torch.where(failed, torch.zeros_like(av), av),
        "av_metrop_accept_prob": av,
        "reject_prob": rej,
        "tree_depth": depth.to(torch.int64),
        "diverging": diverging,
        "convergence_error": conv,
        "non_reversible_step": nonrev,
        "step_size": _step_size_stat(step_size, n, pos.device),
    }
    return new, stats


def _quiet(state):
    """A state whose ``dh_dmom`` is wanted for every chain although some chains may hold a
    failed step's (finite, pre-step) state: plain (pos, mom) copy without auxiliary slots."""
    return ChainState(pos=state.pos, mom=state.mom, dir=1)


class MultinomialDynamicIntegrationTransition(DynamicIntegrationTransition):
    """Progressive multinomial sampling of the next state (transitions.py:773-809)."""

    _slice = False


class SliceDynamicIntegrationTransition(DynamicIntegrationTransition):
    """Progressive slice sampling, NUTS as in Hoffman & Gelman (transitions.py:812-858)."""

    _slice = True


def _run_stage(mom_tr, int_tr, state, rng, n_iter, adapters, record, all_stats, trace, group,
               h_trace=None):
    """One sampling stage for every chain: the loop body of ``_sample_chain`` (samplers.py:459-513)
    then ``_finalize_adapters`` (samplers.py:1131-1138)."""
    adapters = adapters or []
    adapt_states = [a.initialize(state, int_tr) for a in adapters]
    for _ in range(n_iter):
        state, _ = mom_tr.sample(state, rng)
        state, st = int_tr.sample(state, rng)
        for a, a_state in zip(adapters, adapt_states):
            a.update(a_state, state, st, int_tr)
        if record:
            for k, v in st.items():
                all_stats.setdefault(k, []).append(v)
            if trace is not None:
                trace.append(state.pos.clone())
                if h_trace is not None:
                    # the reference's default trace function (samplers.py:1263-1269)
                    h_trace.append(state.h.clone() if "h" in state._aux and state.h is not None
                                   else int_tr.system.h(state))
    for a, a_state in zip(adapters, adapt_states):
        a.finalize(a_state, state, int_tr, rng, group=group)
    return state, adapt_states


def sample_hmc(system, integrator, state, rng, n_iter, n_step, trace_pos=False, adapters=None,
               group=None):
    """``n_iter`` static-HMC iterations (momentum refresh + Metropolis transition) for every
    chain of ``state`` -- the inner loop of ``samplers._sample_chain`` (samplers.py:479-513) with
    the chain axis on the device; ``adapters`` (``mici_b200.adapters``) are initialised before,
    updated after every transition and finalised after the last one, as in one reference
    sampling stage.  Returns ``(final_state, stats, traces)``: ``stats`` per-key tensors
    ``[n_iter, n_chains]``, ``traces`` the positions ``[n_iter, n_chains, dim]`` if requested."""
    mom_tr = IndependentMomentumTransition(system)
    int_tr = MetropolisStaticIntegrationTransition(system, integrator, n_step)
    all_stats, trace = {}, ([] if trace_pos else None)
    state, _ = _run_stage(mom_tr, int_tr, state, rng, n_iter, adapters, True, all_stats, trace,
                          group)
    stats = {k: torch.stack(v) for k, v in all_stats.items()}
    return state, stats, (torch.stack(trace) if trace_pos else None)


def sample_chains(system, integrator, state, rng, n_warm_up_iter, n_main_iter, *, n_step=None,
                  n_step_range=None, integration_transition=None, momentum_transition=None,
                  adapters=None, stager=None, trace_warm_up=False, trace_pos=True, trace_h=False,
                  group=None):
    """Staged sampling of all chains: ``HamiltonianMonteCarlo.sample_chains``
    (samplers.py:875-1141) for the static (``n_step``) or random (``n_step_range``) Metropolis
    HMC transitions or a given ``integration_transition`` (e.g. a dynamic one), with the stage schedule of ``mici_b200.stagers`` (default: one warm-up stage
    if all adapters are fast, else windowed: samplers.py:1075-1082).  Adapter states are
    re-initialised at the start of every stage and finalised at its end (across all chains and,
    with a process group, across all ranks).  Returns ``(final_state, stats, traces)`` over the
    recorded stages (the main stage; also the warm-up if ``trace_warm_up``); ``traces`` is the
    position tensor ``[n_iter, n_chains, dim]``, or with ``trace_h`` a dictionary
    ``{"pos", "hamiltonian"}`` like the reference's default trace function."""
    from .stagers import WarmUpStager, WindowedWarmUpStager  # noqa: PLC0415

    if (n_step is not None) + (n_step_range is not None) + (integration_transition is not None) != 1:
        raise ValueError(
            "Give exactly one of `n_step`, `n_step_range` and `integration_transition`.")
    adapters = list(adapters or [])
    mom_tr = (IndependentMomentumTransition(system) if momentum_transition is None
              else momentum_transition)
    if integration_transition is not None:
        int_tr = integration_transition
    elif n_step is not None:
        int_tr = MetropolisStaticIntegrationTransition(system, integrator, n_step)
    else:
        int_tr = MetropolisRandomIntegrationTransition(system, integrator, n_step_range)
    if stager is None:
        stager = WarmUpStager() if all(a.is_fast for a in adapters) else WindowedWarmUpStager()
    all_stats, trace = {}, ([] if trace_pos else None)
    h_trace = [] if (trace_pos and trace_h) else None
    for stage in stager.stages(n_warm_up_iter, n_main_iter, adapters,
                               trace_warm_up=trace_warm_up).values():
        state, _ = _run_stage(mom_tr, int_tr, state, rng, stage.n_iter, stage.adapters,
                              stage.record_stats, all_stats, trace if stage.trace else None,
                              group, h_trace if stage.trace else None)
    stats = {k: torch.stack(v) for k, v in all_stats.items()}
    if h_trace is not None:  # dictionary of traces keyed like the reference's default trace
        return state, stats, ({"pos": torch.stack(trace), "hamiltonian": torch.stack(h_trace)}
                              if trace else None)
    return state, stats, (torch.stack(trace) if trace_pos and trace else None)
