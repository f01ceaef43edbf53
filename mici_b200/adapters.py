"""Batched adapters -- "next" row N3 of SURVEY.md 8(f); mirror of ``mici.adapters``
(reference ``src/mici/adapters.py``) with the chain axis on the device.

The reference keeps one adapter state (a dict of Python floats / NumPy arrays) per chain and
combines them in ``finalize``.  Here ONE adapter state holds ``[n_chains]`` / ``[n_chains, dim]``
tensors, every ``update`` is a handful of elementwise device operations for all chains, and
``finalize`` is a reduction over the chain axis -- plus, when chains are sharded over GPUs, a
single ``all_gather`` of the per-rank partial statistics (the only collective of a warm-up
window; pass ``group=`` or rely on the default process group).

* ``DualAveragingStepSizeAdapter``   adapters.py:172-391: per-chain dual averaging; the integrator
  carries a per-chain step-size tensor while it runs (the ``step_sizes`` array of the integrator
  entry points),
  ``finalize`` reduces the smoothed log step sizes to the one shared step size of the main stage.
* ``OnlineVarianceMetricAdapter``    adapters.py:394-518: Welford per chain, Chan et al. merge.
* ``OnlineCovarianceMetricAdapter``  adapters.py:521-648: Welford per chain, Schubert-Gertz merge.
  The reference stores one ``[dim, dim]`` accumulator per chain; merging is linear in them, so
  only their SUM over chains is kept (one ``[dim, n_chains] x [n_chains, dim]`` product per
  update) next to the per-chain means -- O(n_chains dim + dim^2) memory instead of
  O(n_chains dim^2).
"""

from __future__ import annotations

from abc import ABC, abstractmethod
from math import exp, log

import torch
import torch.distributed as dist

from .errors import AdaptationError
from .systems import _FixedMetric


class Adapter(ABC):
    """adapters.py:31-124 with batched states."""

    @abstractmethod
    def initialize(self, chain_state, transition):
        """Return the initial adapter state for all chains of ``chain_state``."""

    @abstractmethod
    def update(self, adapt_state, chain_state, trans_stats, transition):
        """Update ``adapt_state`` in place after one transition of every chain."""

    @abstractmethod
    def finalize(self, adapt_state, chain_state, transition, rngs, group=None):
        """Set the transition parameters from the final adapter state (all chains, all ranks)."""

    @property
    @abstractmethod
    def is_fast(self):
        """Whether the adapter only needs local information (adapters.py:115-124)."""


def _any_rank(flag, device, group=None):
    """``flag`` OR-ed over the ranks of ``group`` (one tiny all-reduce), so that a failure seen by
    one rank's chains raises on EVERY rank instead of leaving the others waiting in the next
    collective (``finalize``)."""
    if group is False or not (dist.is_available() and dist.is_initialized()):
        return bool(flag)
    t = torch.tensor([1 if flag else 0], dtype=torch.int32, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return bool(t.item())


def _all_ranks(tensor, group=None):
    """List of ``tensor`` from every rank (just ``[tensor]`` without a process group, or with
    ``group=False``: adapt on this rank's chains only)."""
    if group is False or not (dist.is_available() and dist.is_initialized()):
        return [tensor]
    world = dist.get_world_size(group)
    if world == 1:
        return [tensor]
    sizes = [torch.zeros(1, dtype=torch.int64, device=tensor.device) for _ in range(world)]
    dist.all_gather(sizes, torch.tensor([tensor.shape[0]], dtype=torch.int64,
                                        device=tensor.device), group=group)
    sizes = [int(s.item()) for s in sizes]
    pad = max(sizes)
    buf = torch.zeros((pad, *tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
    buf[: tensor.shape[0]] = tensor
    out = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(out, buf, group=group)
    return [o[:s] for o, s in zip(out, sizes)]


def arithmetic_mean_log_step_size_reducer(log_step_sizes):
    """adapters.py:126-135."""
    x = torch.as_tensor(log_step_sizes, dtype=torch.float64)
    return float(torch.exp(x).sum() / x.numel())


def geometric_mean_log_step_size_reducer(log_step_sizes):
    """adapters.py:138-147."""
    x = torch.as_tensor(log_step_sizes, dtype=torch.float64)
    return exp(float(x.sum() / x.numel()))


def min_log_step_size_reducer(log_step_sizes):
    """adapters.py:150-159."""
    return exp(float(torch.as_tensor(log_step_sizes, dtype=torch.float64).min()))


def default_adapt_stat_func(stats):
    """adapters.py:162-171."""
    return stats["accept_stat"]


class DualAveragingStepSizeAdapter(Adapter):
    """Dual-averaging step-size adaptation (Hoffman & Gelman 2014) for all chains at once
    (adapters.py:172-391); same constructor arguments and defaults."""

    is_fast = True

    def __init__(self, adapt_stat_target=0.8, adapt_stat_func=None, log_step_size_reg_target=None,
                 log_step_size_reg_coefficient=0.05, iter_decay_coeff=0.75, iter_offset=10,
                 max_init_step_size_iters=100, log_step_size_reducer=None, group=None):
        # `group`: process group whose ranks share the chains (None = default group when
        # torch.distributed is initialised; False = this rank alone)
        self.group = group
        self.adapt_stat_target = adapt_stat_target
        self.adapt_stat_func = default_adapt_stat_func if adapt_stat_func is None else adapt_stat_func
        self.log_step_size_reg_target = log_step_size_reg_target
        self.log_step_size_reg_coefficient = log_step_size_reg_coefficient
        self.iter_decay_coeff = iter_decay_coeff
        self.iter_offset = iter_offset
        self.max_init_step_size_iters = max_init_step_size_iters
        self.log_step_size_reducer = (arithmetic_mean_log_step_size_reducer
                                      if log_step_size_reducer is None else log_step_size_reducer)

    def initialize(self, chain_state, transition):
        n = chain_state.pos.shape[0]
        dev = chain_state.pos.device
        init_step_size = self._find_and_set_init_step_size(chain_state, transition.system,
                                                           transition.integrator)
        if self.log_step_size_reg_target is None:
            reg_target = torch.log(10 * init_step_size)
        else:
            reg_target = torch.full((n,), float(self.log_step_size_reg_target),
                                    dtype=torch.float64, device=dev)
        return {
            "iter": 0,
            "smoothed_log_step_size": torch.zeros(n, dtype=torch.float64, device=dev),
            "adapt_stat_error": torch.zeros(n, dtype=torch.float64, device=dev),
            "log_step_size_reg_target": reg_target,
        }

    def _find_and_set_init_step_size(self, state, system, integrator):
        """Coarse search of adapters.py:285-352 with one step size per chain: every iteration
        steps ALL chains once from the initial state with their own candidate step size, then
        halves / doubles it chain by chain until the energy error crosses log 2."""
        init_state = state.copy()
        n = init_state.pos.shape[0]
        dev = init_state.pos.device
        h_init = system.h(init_state)
        if _any_rank(bool(torch.isnan(h_init).any()), dev, self.group):
            raise AdaptationError("Hamiltonian evaluating to NaN at initial state.")
        eps = torch.ones(n, dtype=torch.float64, device=dev)
        too_big = torch.zeros(n, dtype=torch.bool, device=dev)
        active = torch.ones(n, dtype=torch.bool, device=dev)
        threshold = log(2)
        for s in range(self.max_init_step_size_iters):
            integrator.step_size = eps
            new = integrator.step_n(init_state, 1, return_h=True)
            failed = new.status != 0
            delta_h = (h_init - new.h).abs()
            is_nan = torch.isnan(delta_h)
            over = delta_h > threshold  # False for NaN, as in Python
            if s == 0:
                flag = is_nan | over
            else:
                flag = too_big | is_nan
            flag = flag | failed  # except IntegratorError: step_size_too_big = True
            found = ~failed & ((flag & (delta_h <= threshold)) | (~flag & over))
            still = active & ~found
            eps = torch.where(still, torch.where(flag, eps / 2, eps * 2), eps)
            too_big = torch.where(active, flag, too_big)
            active = still
            # every rank runs the same number of search iterations (the slowest chain anywhere)
            if not _any_rank(bool(active.any()), dev, self.group):
                integrator.step_size = eps
                return eps
        integrator.step_size = eps
        bad = eps[active] if bool(active.any()) else eps
        msg = (
            f"Could not find reasonable initial step size in {self.max_init_step_size_iters} "
            f"iterations for {int(active.sum())} chains (final step sizes between "
            f"{float(bad.min())} and {float(bad.max())}). A very large final step size may "
            f"indicate that the target distribution is improper such that the negative log "
            f"density is flat in one or more directions while a very small final step size may "
            f"indicate that the density function is insufficiently smooth at the point "
            f"initialized at."
        )
        raise AdaptationError(msg)

    def update(self, adapt_state, chain_state, trans_stats, transition):  # noqa: ARG002
        adapt_state["iter"] += 1
        it = adapt_state["iter"]
        error_weight = 1 / (self.iter_offset + it)
        err = adapt_state["adapt_stat_error"]
        err *= 1 - error_weight
        err += error_weight * (self.adapt_stat_target - self.adapt_stat_func(trans_stats))
        smoothing_weight = (1 / it) ** self.iter_decay_coeff
        log_step_size = adapt_state["log_step_size_reg_target"] - (
            err * it**0.5 / self.log_step_size_reg_coefficient)
        sm = adapt_state["smoothed_log_step_size"]
        sm *= 1 - smoothing_weight
        sm += smoothing_weight * log_step_size
        transition.integrator.step_size = torch.exp(log_step_size)

    def finalize(self, adapt_state, chain_state, transition, rngs, group=None):  # noqa: ARG002
        logs = torch.cat(_all_ranks(adapt_state["smoothed_log_step_size"], group))
        transition.integrator.step_size = float(self.log_step_size_reducer(logs.cpu()))


def _merge_moments(parts, outer):
    """Chan et al. / Schubert-Gertz merge of ``(count, mean, m2)`` triples in order
    (adapters.py:487-505, 615-634)."""
    n_iter, mean_est, m2 = parts[0]
    mean_est, m2 = mean_est.clone(), m2.clone()
    for n_k, mean_k, m2_k in parts[1:]:
        n_prev = n_iter
        n_iter = n_iter + n_k
        mean_diff = mean_est - mean_k
        mean_est = (mean_est * n_prev + n_k * mean_k) / n_iter
        m2 = m2 + m2_k
        corr = torch.outer(mean_diff, mean_diff) if outer else mean_diff**2
        m2 = m2 + corr * (n_k * n_prev) / n_iter
    return n_iter, mean_est, m2


def _gather_moments(count, mean, m2, group):
    """Per-rank ``(count, mean, m2)`` -> merged over ranks (one all_gather)."""
    if (group is False or not (dist.is_available() and dist.is_initialized())
            or dist.get_world_size(group) == 1):
        return count, mean, m2
    flat = torch.cat([torch.tensor([float(count)], dtype=torch.float64, device=mean.device),
                      mean.reshape(-1), m2.reshape(-1)])[None]
    parts = []
    for f in _all_ranks(flat, group):
        f = f[0]
        parts.append((int(f[0].item()), f[1:1 + mean.numel()].reshape(mean.shape),
                      f[1 + mean.numel():].reshape(m2.shape)))
    return _merge_moments(parts, outer=m2.ndim == 2)


class OnlineVarianceMetricAdapter(Adapter):
    """Diagonal metric from online variance estimates (adapters.py:394-518)."""

    is_fast = False

    def __init__(self, reg_iter_offset=5, reg_scale=1e-3):
        self.reg_iter_offset = reg_iter_offset
        self.reg_scale = reg_scale

    def initialize(self, chain_state, transition):  # noqa: ARG002
        return {
            "iter": 0,
            "mean": torch.zeros_like(chain_state.pos),
            "sum_diff_sq": torch.zeros_like(chain_state.pos),
        }

    def update(self, adapt_state, chain_state, trans_stats, transition):  # noqa: ARG002
        # Welford (1962), all chains at once (adapters.py:446-458)
        adapt_state["iter"] += 1
        pos_minus_mean = chain_state.pos - adapt_state["mean"]
        adapt_state["mean"] += pos_minus_mean / adapt_state["iter"]
        adapt_state["sum_diff_sq"] += pos_minus_mean * (chain_state.pos - adapt_state["mean"])

    def _regularize_var_est(self, var_est, n_iter):
        """adapters.py:460-469."""
        if self.reg_iter_offset is not None and self.reg_iter_offset != 0:
            var_est *= n_iter / (self.reg_iter_offset + n_iter)
            var_est += self.reg_scale * (self.reg_iter_offset / (self.reg_iter_offset + n_iter))

    def finalize(self, adapt_state, chain_state, transition, rngs, group=None):
        m = adapt_state["iter"]
        means = adapt_state.pop("mean")
        n_chains = means.shape[0]
        # every chain of the batch has seen `m` samples, so the chain-by-chain Chan merge of
        # adapters.py:487-505 collapses to one reduction over the chain axis
        mean_est = means.mean(0)
        var_est = adapt_state.pop("sum_diff_sq").sum(0) + m * ((means - mean_est) ** 2).sum(0)
        n_iter, mean_est, var_est = _gather_moments(n_chains * m, mean_est, var_est, group)
        if n_iter < 2:  # noqa: PLR2004
            raise AdaptationError("At least two chain samples required to compute a variance estimates.")
        var_est = var_est / (n_iter - 1)
        self._regularize_var_est(var_est, n_iter)
        # PositiveDiagonalMatrix(var_est).inv (adapters.py:513)
        transition.system.metric = 1.0 / var_est.cpu().numpy()
        chain_state.mom = transition.system.sample_momentum(chain_state, rngs)


class OnlineCovarianceMetricAdapter(Adapter):
    """Dense metric from online covariance estimates (adapters.py:521-648)."""

    is_fast = False

    def __init__(self, reg_iter_offset=5, reg_scale=1e-3):
        self.reg_iter_offset = reg_iter_offset
        self.reg_scale = reg_scale

    def initialize(self, chain_state, transition):  # noqa: ARG002
        dim = chain_state.pos.shape[1]
        return {
            "iter": 0,
            "mean": torch.zeros_like(chain_state.pos),
            # sum over chains of the reference's per-chain `sum_diff_outer`
            "sum_diff_outer": torch.zeros((dim, dim), dtype=chain_state.pos.dtype,
                                          device=chain_state.pos.device),
        }

    def update(self, adapt_state, chain_state, trans_stats, transition):  # noqa: ARG002
        # per chain: S += (x - mean_old)[None, :] * (x - mean_new)[:, None] (adapters.py:583-590);
        # summed over chains that is (X - M_new)^T (X - M_old)
        adapt_state["iter"] += 1
        pos_minus_mean = chain_state.pos - adapt_state["mean"]
        adapt_state["mean"] += pos_minus_mean / adapt_state["iter"]
        adapt_state["sum_diff_outer"] += (chain_state.pos - adapt_state["mean"]).T @ pos_minus_mean

    def _regularize_covar_est(self, covar_est, n_iter):
        """adapters.py:592-601."""
        covar_est *= n_iter / (self.reg_iter_offset + n_iter)
        covar_est.diagonal().add_(
            self.reg_scale * (self.reg_iter_offset / (self.reg_iter_offset + n_iter)))

    def finalize(self, adapt_state, chain_state, transition, rngs, group=None):
        m = adapt_state["iter"]
        means = adapt_state.pop("mean")
        n_chains = means.shape[0]
        mean_est = means.mean(0)
        centred = means - mean_est
        covar_est = adapt_state.pop("sum_diff_outer") + m * (centred.T @ centred)
        n_iter, mean_est, covar_est = _gather_moments(n_chains * m, mean_est, covar_est, group)
        if n_iter < 2:  # noqa: PLR2004
            raise AdaptationError("At least two chain samples required to compute a variance estimates.")
        covar_est = covar_est / (n_iter - 1)
        self._regularize_covar_est(covar_est, n_iter)
        # DensePositiveDefiniteMatrix(covar_est).inv (adapters.py:642)
        transition.system.metric = _FixedMetric.from_covariance(covar_est.cpu().numpy())
        chain_state.mom = transition.system.sample_momentum(chain_state, rngs)


__all__ = [
    "Adapter",
    "DualAveragingStepSizeAdapter",
    "OnlineCovarianceMetricAdapter",
    "OnlineVarianceMetricAdapter",
    "arithmetic_mean_log_step_size_reducer",
    "default_adapt_stat_func",
    "geometric_mean_log_step_size_reducer",
    "min_log_step_size_reducer",
]
