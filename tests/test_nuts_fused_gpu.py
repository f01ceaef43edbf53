"""The fused dynamic (NUTS) transition kernels (``nuts_dmma_kernel``, ``nuts_dmma.cuh``: chains in
lock-step groups of 8 with the mat-vecs on the tensor pipe; ``nuts_euclidean_kernel``,
``nuts.cuh``: one free-running warp per chain) against the float64 oracle's transition
(``mici_oracle.nuts_transition``) and an extended-precision replay of the returned state, on
every target, layout (KP, GROUPS) and metric path they are built for, up to the deepest tree.

* Inputs: ``mb200_nuts_euclidean`` is called directly with an explicit per-chain table of
  uniform variates; the oracle reads the same row of it, steps each chain with its own step size,
  and records the signed leaf index ``j`` of every state it produces (the initial state is 0).
* Discrete outcomes (``n_step``, ``tree_depth``, ``diverging``, ``n_uniforms_used``, ``dir``,
  ``status``) equal the oracle's exactly.
* Continuous outcomes are measured against ``leapfrog_ext``: ``|j|`` long-double leapfrog steps
  from the initial state with ``dt = sign(j) eps_c`` and the float64 ``M^-1`` the kernel is given.
  The kernel's error in q, p and in h (at its own state) is bounded by the float64 oracle's
  error on the same chains with ``_check_ratio``: worst <= 4 F x oracle worst + 8 ulp, mean <=
  2 F x oracle mean + 2 ulp.  The rule comes from the two documented deviations.  (1) The
  velocity is tracked by linearity (``v -= dt/2 M^-1 grad``): v is rounded twice per step where
  the oracle rounds a fresh ``M^-1 p`` once, and (2) on the lock-step kernel ``M^-1 grad`` is
  summed in the tensor pipe's k-order (two interleaved accumulators per row); each at most
  doubles the oracle's roundings per step, so F = 2 for q and p.  The energy is formed the same
  way by both (F = 1), except that the kernel's kinetic term uses the tracked v, whose rounding
  accumulates over the |j| steps to the returned state: as a random walk of 2|j| roundings of
  half an ulp its size is about sqrt(|j|) ulp, which is added to the oracle's energy error per
  chain.  Measured on an H100 80GB HBM3 SXM (700 W power limit, 1980 MHz max SM clock), over
  all cases of this file, the largest shares of the bound used (worst / mean) are: q 0.31 / 0.58
  (free-running kernel, dense D = 512), p 0.40 / 0.40, h 0.08 / 0.11; the kernel/oracle ratio
  for q and p does not grow with |j| (deepest trees, |j| up to 3798: q 23 / 25 ulp, p 47 / 41
  ulp).  The energy's allowance is used: 16.5 ulp at |j| = 3798 on the lock-step kernel, where
  the oracle's own error is 0.7 ulp.
* ``av_metrop_accept_prob`` and ``reject_prob`` are functions of the leaf energies with
  derivative at most 1 per energy (``exp(min(0, h0 - h))``) and at most ``depth + 1`` factors
  (``prod (1 - a)``), so they agree with the oracle's to ``(depth + 2) x`` the energy discrepancy
  at the returned state, floored at 64 ulp of the energy scale (measured: at most 0.013 of it).
* Chains do not depend on each other (bitwise): poisoned neighbours in a lock-step group, and
  the whole batch rotated to other warp slots, groups, CTAs and passes.
* A chain that runs out of uniform variates reports status 1 and leaves every other chain as it
  was; the public ``sample()`` raises.
* The lock-step generic arm (``nuts_generic.cuh``, every KP) meets the same checks.
"""

import ctypes
import re
import zlib

import numpy as np
import pytest
import torch

from mici_b200 import _lib, problems, systems, transitions
from mici_b200 import integrators as minteg
from mici_b200 import targets as mtargets
from mici_b200.states import ChainState
from oracle import drivers as dr
from oracle import mici_oracle as mo

from extended_precision import (BANANA_B, ULP, L, _check_ratio, _GivenInverse, _h_terms,
                                _oracle_target, _rel_err, leapfrog_ext, need_extended)

DEV = "cuda:0"
NUTS_MAX_DEPTH = 12
TARGET_TYPE = {"std_gaussian": "StdGaussianTarget", "neal_funnel": "NealFunnelTarget",
               "banana": "BananaTarget"}
LEAF_BUDGET = 20_000  # oracle leaves per case (100-300 us each at D = 128)
F_QP = 2  # see the module docstring


def _kp(dim):
    return 1 if dim <= 64 else 2 if dim <= 128 else 4 if dim <= 256 else 8 if dim <= 512 else 16


def expected_kernel(target, dim, metric):
    """(name, template arguments) of the fused kernel eu_dispatch (api_common.cuh) picks."""
    kp = _kp(dim)
    if metric == "dense" and 8 <= dim <= 128:
        return "nuts_dmma_kernel", (TARGET_TYPE[target], kp, 2 if kp == 1 else 1)
    return "nuts_euclidean_kernel", (TARGET_TYPE[target], kp)


# ------------------------------------------------------------------------------------------------
# Inputs
# ------------------------------------------------------------------------------------------------


def _system(target, dim, metric, rng):
    """The system and its float64 M^-1 as the kernel receives it (array, vector or None)."""
    if metric == "dense":
        m = problems.dense_spd_metric(rng, dim)
    elif metric == "diagonal":
        m = rng.uniform(0.5, 2.0, dim)
    else:
        m = None
    params = {"dim": dim, "b": BANANA_B} if target == "banana" else {"dim": dim}
    system = systems.EuclideanMetricSystem(mtargets.make_target(target, **params), metric=m)
    return system, m, system.metric.inv


def _states(target, n, dim, m, rng):
    if target == "neal_funnel":
        v = rng.uniform(-2.0, 2.0, n)
        q = np.concatenate([v[:, None], rng.standard_normal((n, dim - 1)) * np.exp(v / 2)[:, None]],
                           axis=1)
    elif target == "banana":
        q = rng.standard_normal((n, dim))
        q[:, 0::2] *= 2.0
        q[:, 1::2] += BANANA_B * q[:, 0::2] ** 2
    else:
        q = rng.standard_normal((n, dim))
    return q, _refresh(rng, n, dim, m)


def _refresh(rng, n, dim, m):
    """p ~ N(0, M) for a dense (array), diagonal (vector) or identity (None) M."""
    z = rng.standard_normal((n, dim))
    if m is None:
        return z
    return z * np.sqrt(m) if m.ndim == 1 else z @ np.linalg.cholesky(m).T


# ------------------------------------------------------------------------------------------------
# The launch
# ------------------------------------------------------------------------------------------------

OUTPUTS = ("pos", "mom", "h", "n_step", "av_accept", "reject_prob", "tree_depth", "diverging",
           "n_used", "dir", "status")


def n_uniforms(opts):
    return 2 * opts["depth"] + 2 ** opts["depth"] + (1 if opts["slice"] else 0)


def run_fused(system, q, p, eps, eps_c, uni, opts, n_uni=None):
    """One mb200_nuts_euclidean launch -> dict of its 11 outputs as host arrays."""
    n, dim = q.shape
    n_uni = uni.shape[1] if n_uni is None else n_uni  # also the row stride of the table
    qt, pt = torch.as_tensor(q, device=DEV), torch.as_tensor(p, device=DEV)
    ut = torch.as_tensor(np.ascontiguousarray(uni[:, :n_uni]), device=DEV)
    et = None if eps_c is None else torch.as_tensor(eps_c, dtype=torch.float64, device=DEV)
    lib = _lib.load()
    nbytes = int(lib.mb200_nuts_workspace_bytes(n, dim, opts["depth"]))
    ws = torch.empty(nbytes // 8, dtype=torch.float64, device=DEV)
    f64 = {"dtype": torch.float64, "device": DEV}
    i32 = {"dtype": torch.int32, "device": DEV}
    out = {"pos": torch.empty_like(qt), "mom": torch.empty_like(pt)}
    for k in OUTPUTS[2:]:
        out[k] = (torch.full((n,), np.nan, **f64) if k in ("h", "av_accept", "reject_prob")
                  else torch.full((n,), -7, **i32))
    minv = system.metric.inv_device(qt.device)
    model = system._model(qt.device)
    rc = lib.mb200_nuts_euclidean(
        _lib.ptr(qt), _lib.ptr(pt), _lib.ptr(out["pos"]), _lib.ptr(out["mom"]), n, dim,
        0.0 if eps_c is not None else eps, _lib.ptr(et), system.metric.kind, _lib.ptr(minv),
        ctypes.byref(model), opts["slice"], opts["euclid"], opts["extra"], opts["depth"],
        opts["max_delta_h"], _lib.ptr(ut), n_uni, _lib.ptr(ws), nbytes,
        *[_lib.ptr(out[k]) for k in OUTPUTS[2:]], _lib.current_stream_ptr(qt.device))
    assert rc == 0, lib.mb200_last_error()
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


# ------------------------------------------------------------------------------------------------
# The oracle, per chain, with the leaf index of every state
# ------------------------------------------------------------------------------------------------


def _key(q, p):
    return np.asarray(q, dtype=np.float64).tobytes() + np.asarray(p, dtype=np.float64).tobytes()


def oracle_chain(q, p, row, eps, otarget, ometric, opts, n_uni=None):
    """mo.nuts_transition of one chain reading its uniforms from `row` (0.5 and `starved` past
    `n_uni`, as the kernels do) -> (q, p, stats, j, h, n_used, starved): j is the signed leaf
    index of the returned state."""
    n_uni = len(row) if n_uni is None else n_uni
    used = [0, False]

    def uniform():
        if used[0] >= n_uni:
            used[1] = True
            return 0.5
        used[0] += 1
        return float(row[used[0] - 1])

    index = {_key(q, p): 0}

    def step(qq, pp, d):
        q2, p2 = mo.leapfrog_steps(qq, pp, d * eps, 1, otarget, ometric)
        index.setdefault(_key(q2, p2), index[_key(qq, pp)] + d)
        return q2, p2

    def h_fn(qq, pp):
        return mo.euclidean_h(qq, pp, otarget, ometric)

    with np.errstate(all="ignore"):
        qn, pn, st = mo.nuts_transition(
            q, p, uniform, step, h_fn, lambda qq, pp: ometric.inv_matvec(pp),
            max_tree_depth=opts["depth"], max_delta_h=opts["max_delta_h"],
            criterion="euclidean" if opts["euclid"] else "riemannian",
            extra_checks=bool(opts["extra"]), variant="slice" if opts["slice"] else "multinomial")
        h = h_fn(qn, pn)
    return qn, pn, st, index[_key(qn, pn)], h, used[0], used[1]


# ------------------------------------------------------------------------------------------------
# Which chains the oracle checks
# ------------------------------------------------------------------------------------------------


def _subset(out, n, per_cta, rng, depth, budget=LEAF_BUDGET, extra=()):
    """Every chain of the first CTA, the last two groups of 8, flagged chains (diverged, at the
    maximum depth, starved: up to 40), then random others while the oracle's leaves stay within
    `budget`."""
    last = 8 * ((n - 1) // 8)
    must = set(range(min(per_cta, n))) | set(range(max(last - 8, 0), n)) | set(extra)
    flagged = np.flatnonzero((out["diverging"] != 0) | (out["tree_depth"] == depth - 1)
                             | (out["status"] != 0))
    flagged = np.setdiff1d(flagged, list(must))
    must |= set(rng.permutation(flagged)[:40].tolist())
    pick = sorted(must)
    leaves = int(out["n_step"][pick].sum())
    for c in rng.permutation(np.setdiff1d(np.arange(n), pick)):
        if len(pick) >= 600 or leaves + out["n_step"][c] > budget:
            break
        pick.append(int(c))
        leaves += int(out["n_step"][c])
    return np.array(sorted(pick))


# ------------------------------------------------------------------------------------------------
# The comparison
# ------------------------------------------------------------------------------------------------

MEASURED = {}  # label -> share of the bound used (worst, mean) for q, p, h


def _fraction(kern, orc, factor):
    """The share of _check_ratio's bound used: worst and mean."""
    return (kern.max() / (4 * factor * orc.max() + 8), kern.mean() / (2 * factor * orc.mean() + 2))


def check_against_oracle(label, target, q0, p0, eps_c, uni, opts, minv, out, idx, n_uni=None,
                         tracked_velocity=True):
    """The discrete outcomes of the chains `idx` equal the oracle's; q, p, h are within the
    module's bound of the oracle's error against the long-double replay; the accept statistics
    within their derived tolerance.  `tracked_velocity`: the kernel's h uses the velocity tracked
    by linearity (the fused kernels).  Returns the per-chain oracle leaf indices."""
    dim = q0.shape[1]
    otarget, ometric = _oracle_target(target, dim), _GivenInverse(minv)
    q_or, p_or = np.empty((idx.size, dim)), np.empty((idx.size, dim))
    h_or, j = np.empty(idx.size), np.empty(idx.size, dtype=np.int64)
    disc = {k: np.empty(idx.size, dtype=np.int64) for k in ("n_step", "tree_depth", "diverging",
                                                            "n_used", "dir", "status")}
    av_or, rej_or = np.empty(idx.size), np.empty(idx.size)
    for r, c in enumerate(idx):
        q_or[r], p_or[r], st, j[r], h_or[r], used, starved = oracle_chain(
            q0[c], p0[c], uni[c], float(eps_c[c]), otarget, ometric, opts, n_uni)
        disc["n_step"][r], disc["tree_depth"][r] = st["n_step"], st["tree_depth"]
        disc["diverging"][r], disc["dir"][r] = int(st["diverging"]), st["dir"]
        disc["n_used"][r], disc["status"][r] = used, int(starved)
        av_or[r], rej_or[r] = st["av_metrop_accept_prob"], st["reject_prob"]
    for k, v in disc.items():
        got = out[k][idx]
        bad = np.flatnonzero(got != v)
        assert bad.size == 0, (f"{label}: {k} differs from the oracle on chains {idx[bad][:8]}: "
                               f"kernel {got[bad][:8]}, oracle {v[bad][:8]}")
    # the state each method returned, against |j| long-double steps from the initial state
    with np.errstate(all="ignore"):
        q_ref, p_ref = leapfrog_ext(target, q0[idx], p0[idx], np.sign(j) * eps_c[idx],
                                    np.abs(j), minv)
    ok = np.isfinite(q_or).all(1) & np.isfinite(p_or).all(1) & (np.abs(q_ref).max(1) > 0)
    assert np.array_equal(ok, np.isfinite(out["pos"][idx]).all(1) & (np.abs(q_ref).max(1) > 0))
    sel, a = idx[ok], (None if minv is None else np.asarray(minv).astype(L))
    errs = {"q": (_rel_err(out["pos"][sel], q_ref[ok]), _rel_err(q_or[ok], q_ref[ok]), F_QP),
            "p": (_rel_err(out["mom"][sel], p_ref[ok]), _rel_err(p_or[ok], p_ref[ok]), F_QP)}
    hk, sk = _h_terms(target, out["pos"][sel].astype(L), out["mom"][sel].astype(L), a)
    ho, so = _h_terms(target, q_or[ok].astype(L), p_or[ok].astype(L), a)
    eh_k = (np.abs(out["h"][sel].astype(L) - hk) / sk / L(ULP)).astype(np.float64)
    eh_o = (np.abs(h_or[ok].astype(L) - ho) / so / L(ULP)).astype(np.float64)
    if tracked_velocity:  # the velocity's accumulated rounding (module docstring)
        eh_o = eh_o + np.sqrt(np.abs(j[ok]))
    errs["h"] = (eh_k, eh_o, 1)
    checks = [_check_ratio(k, *e) for k, e in errs.items()]
    fracs = {k: _fraction(*e) for k, e in errs.items()}
    # accept statistics: Lipschitz in the leaf energies (module docstring)
    dh = np.abs(out["h"][idx] - h_or)
    dh[~ok] = 0.0
    scale = np.zeros(idx.size)
    scale[ok] = np.maximum(sk, so).astype(np.float64)
    tol = (out["tree_depth"][idx] + 2) * np.maximum(dh, 64 * ULP * scale) + 1e-15
    d_av = np.abs(out["av_accept"][idx] - av_or)
    d_rej = np.abs(out["reject_prob"][idx] - rej_or)
    frac = max((d_av / tol).max(), (d_rej / tol).max())
    report = (f"{label}: {idx.size} chains, {int(disc['n_step'].sum())} leaves, |j| <= "
              f"{int(np.abs(j).max())}; kernel/oracle ulp " + "; ".join(r for _, r in checks)
              + "; share of bound " + " ".join(f"{k} {w:.2f}/{m:.2f}" for k, (w, m) in
                                               fracs.items())
              + f"; accept stats {frac:.3f} of tol")
    MEASURED[label] = fracs
    print("[nuts vs long double]", report)
    failures = [f for f, _ in checks if f is not None]
    assert not failures, (label, failures)
    assert frac <= 1.0, (label, "accept statistics", frac)
    return j


# ------------------------------------------------------------------------------------------------
# The case matrix
# ------------------------------------------------------------------------------------------------

STEP = {"std_gaussian": 0.1, "neal_funnel": 0.02, "banana": 0.05}


def _opts(depth, slice_=False, euclid=False, extra=True, max_delta_h=1000.0):
    return {"depth": depth, "slice": int(slice_), "euclid": int(euclid), "extra": int(extra),
            "max_delta_h": max_delta_h}


# name -> (target, dim, metric, n, opts, steps):  steps "shared", "decade" (per-chain over a
# decade inside every group, one chain with eps_c = 0), "divergent" (decade plus a few huge
# step sizes) or "coarse" (per-chain 1.2 .. 1.95 on the std Gaussian: neighbouring leaves point
# in very different directions, so the two-leaf no-U-turn tests decide the trees)
CASES = {
    # nuts_dmma KP 1 (GROUPS 2): ragged last group, a lone live chain, an empty second group,
    # more chains than one pass of the grid
    "dmma1_std_d8": ("std_gaussian", 8, "dense", 16 * 12 + 13, _opts(10), "decade"),
    "dmma1_funnel_d33": ("neal_funnel", 33, "dense", 8192 + 5, _opts(8, True, True), "shared"),
    "dmma1_banana_d64": ("banana", 64, "dense", 16 * 10 + 9, _opts(6, False, True, False),
                         "divergent"),
    "dmma1_funnel_d9": ("neal_funnel", 9, "dense", 16 * 6 + 8,
                        _opts(4, True, False, True, max_delta_h=0.5), "shared"),
    "dmma1_std_d63": ("std_gaussian", 63, "dense", 3, _opts(2), "shared"),
    "dmma1_banana_d10": ("banana", 10, "dense", 16 * 4 + 1, _opts(1, True), "decade"),
    "dmma1_std_d16_coarse": ("std_gaussian", 16, "dense", 16 * 40 + 6, _opts(6, False, True),
                             "coarse"),
    # nuts_dmma KP 2 (GROUPS 1)
    "dmma2_std_d65": ("std_gaussian", 65, "dense", 8 * 30 + 5, _opts(10, True, True), "decade"),
    "dmma2_funnel_d97": ("neal_funnel", 97, "dense", 8 * 30 + 1,
                         _opts(4, False, False, False, max_delta_h=0.5), "shared"),
    "dmma2_banana_d128": ("banana", 128, "dense", 8192 + 5, _opts(6), "divergent"),
    "dmma2_funnel_d127": ("neal_funnel", 127, "dense", 8 * 5 + 3, _opts(2, False, True), "decade"),
    "dmma2_std_d80_coarse": ("std_gaussian", 80, "dense", 8 * 60 + 7, _opts(6), "coarse"),
    # nuts_euclidean, dense metric: D < 8, the last staged D, the first streamed D, 512
    "warp1_dense_std_d5": ("std_gaussian", 5, "dense", 300, _opts(10, True), "decade"),
    "warp4_dense_funnel_d153": ("neal_funnel", 153, "dense", 160, _opts(6, False, True), "shared"),
    "warp4_dense_banana_d154": ("banana", 154, "dense", 160, _opts(5, False, False, False),
                                "divergent"),
    "warp8_dense_std_d512": ("std_gaussian", 512, "dense", 48, _opts(4, True), "shared"),
    # nuts_euclidean, identity and diagonal metrics
    "warp1_id_std_d1": ("std_gaussian", 1, "identity", 200, _opts(10, False, True), "decade"),
    "warp1_diag_funnel_d64": ("neal_funnel", 64, "diagonal", 200, _opts(6, True), "divergent"),
    "warp1_id_banana_d64": ("banana", 64, "identity", 200, _opts(6, False, False, False),
                            "shared"),
    "warp2_diag_std_d65": ("std_gaussian", 65, "diagonal", 150, _opts(6, False, True, False),
                           "shared"),
    "warp2_id_funnel_d128": ("neal_funnel", 128, "identity", 150,
                             _opts(6, False, False, True, max_delta_h=0.5), "shared"),
    "warp2_diag_banana_d128": ("banana", 128, "diagonal", 150, _opts(4, True, True), "decade"),
    "warp4_id_std_d256": ("std_gaussian", 256, "identity", 120, _opts(4), "divergent"),
    "warp8_diag_funnel_d257": ("neal_funnel", 257, "diagonal", 100, _opts(5, True, True),
                               "decade"),
    "warp8_id_banana_d258": ("banana", 258, "identity", 100, _opts(4), "shared"),
    "warp16_diag_std_d1024": ("std_gaussian", 1024, "diagonal", 64, _opts(4, False, True),
                              "shared"),
    "warp16_id_funnel_d513": ("neal_funnel", 513, "identity", 64, _opts(4, True), "divergent"),
    "warp16_diag_banana_d514": ("banana", 514, "diagonal", 64, _opts(3, False, False, False),
                                "decade"),
}


def _per_cta(target, dim, metric):
    name, args = expected_kernel(target, dim, metric)
    return 8 * args[2] if name == "nuts_dmma_kernel" else 8


def _step_sizes(kind, target, n, rng):
    """None (shared step size) or per-chain step sizes spread over a decade inside every group of
    8 chains; chain 3 has eps_c = 0; "divergent" adds step sizes 100 x the base on ~3% of the
    chains (they diverge within a few leaves, next to normal ones)."""
    if kind == "shared":
        return None
    if kind == "coarse":
        return rng.uniform(1.2, 1.95, n)
    eps_c = STEP[target] * 10.0 ** rng.uniform(-0.7, 0.3, n)
    if kind == "divergent":
        eps_c[rng.random(n) < 0.03] = 100.0 * STEP[target]
    eps_c[min(3, n - 1)] = 0.0
    return eps_c


def _case_inputs(name):
    target, dim, metric, n, opts, steps = CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    system, m, minv = _system(target, dim, metric, rng)
    q0, p0 = _states(target, n, dim, m, rng)
    eps_c = _step_sizes(steps, target, n, rng)
    uni = rng.uniform(size=(n, n_uniforms(opts)))
    return target, dim, metric, n, opts, system, minv, q0, p0, eps_c, uni, rng


@pytest.mark.gpu
@need_extended
@pytest.mark.parametrize("name", list(CASES))
def test_fused_nuts_matches_oracle(name):
    """Discrete outcomes equal the oracle's; q, p, h and the accept statistics within the bounds
    of the module docstring."""
    target, dim, metric, n, opts, system, minv, q0, p0, eps_c, uni, rng = _case_inputs(name)
    eps = STEP[target]
    out = run_fused(system, q0, p0, eps, eps_c, uni, opts)
    assert (out["status"] == 0).all()
    eps_all = np.full(n, eps) if eps_c is None else eps_c
    idx = _subset(out, n, _per_cta(target, dim, metric), rng, opts["depth"],
                  extra=[] if eps_c is None else [min(3, n - 1)])
    kname, args = expected_kernel(target, dim, metric)
    check_against_oracle(f"{name} {kname}<{', '.join(map(str, args))}>", target, q0, p0, eps_all,
                         uni, opts, minv, out, idx)
    c = min(3, n - 1)
    if eps_c is not None and eps_c[c] == 0:  # the chain never moves and runs to the maximum depth
        assert np.array_equal(out["pos"][c], q0[c]) and np.array_equal(out["mom"][c], p0[c])
        assert out["tree_depth"][c] == opts["depth"] - 1


# ------------------------------------------------------------------------------------------------
# Named cases: the benchmark shape, the deepest tree
# ------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@need_extended
@pytest.mark.parametrize("depth", [6, 8])
def test_benchmark_shape_two_transitions(depth):
    """C1 as the benchmark runs it (funnel D = 128, dense metric, 8192 chains, eps 0.01:
    nuts_dmma_kernel<NealFunnelTarget, 2, 1>): two consecutive transitions, momenta refreshed in
    between from a fixed table, each against the oracle from the kernel's own input."""
    prob = problems.make_problem("C1", seed=problems.BASE_SEED + 11)
    n, dim = prob.pos.shape
    system = systems.EuclideanMetricSystem(mtargets.make_target("neal_funnel", dim=dim),
                                           metric=prob.metric)
    minv = system.metric.inv
    opts = _opts(depth)
    rng = np.random.default_rng(1000 + depth)
    q, p = prob.pos, prob.mom
    for it in range(2):
        uni = rng.uniform(size=(n, n_uniforms(opts)))
        out = run_fused(system, q, p, prob.step_size, None, uni, opts)
        assert (out["status"] == 0).all()
        idx = _subset(out, n, 8, rng, depth)
        check_against_oracle(f"C1 depth {depth} transition {it + 1} "
                             "nuts_dmma_kernel<NealFunnelTarget, 2, 1>", "neal_funnel", q, p,
                             np.full(n, prob.step_size), uni, opts, minv, out, idx)
        q, p = out["pos"], _refresh(rng, n, dim, prob.metric)


@pytest.mark.gpu
@need_extended
@pytest.mark.parametrize("metric,dim,n", [("dense", 8, 16), ("identity", 64, 16)],
                         ids=["nuts_dmma_kp1_full_cta", "nuts_euclidean_kp1"])
def test_deepest_tree(metric, dim, n):
    """max_tree_depth = NUTS_MAX_DEPTH with a step small enough that every tree reaches it: 4095
    leaves, stack level 10, n_uniforms_used <= 2 x 12 + 2^12."""
    opts = _opts(NUTS_MAX_DEPTH)
    rng = np.random.default_rng(12 + dim)
    system, m, minv = _system("std_gaussian", dim, metric, rng)
    q0, p0 = _states("std_gaussian", n, dim, m, rng)
    eps = 4e-4  # 4095 steps span 1.64 < pi / 2: no mode turns (M^-1 <= I)
    uni = rng.uniform(size=(n, n_uniforms(opts)))
    out = run_fused(system, q0, p0, eps, None, uni, opts)
    assert (out["tree_depth"] == NUTS_MAX_DEPTH - 1).all()
    assert (out["n_step"] == 2**NUTS_MAX_DEPTH - 1).all()
    assert (out["n_used"] <= 2 * NUTS_MAX_DEPTH + 2**NUTS_MAX_DEPTH).all()
    kname, args = expected_kernel("std_gaussian", dim, metric)
    j = check_against_oracle(f"deepest {kname}<{', '.join(map(str, args))}> D {dim}",
                             "std_gaussian", q0, p0, np.full(n, eps), uni, opts, minv, out,
                             np.arange(n), )
    print(f"[deepest tree] |j| of the returned states: {sorted(np.abs(j).tolist())}")


# ------------------------------------------------------------------------------------------------
# Independence (bitwise)
# ------------------------------------------------------------------------------------------------

INDEP = {1: ("neal_funnel", 33), 2: ("banana", 100)}


def _indep_inputs(kp, n, depth):
    target, dim = INDEP[kp]
    rng = np.random.default_rng(500 + kp)
    system, m, minv = _system(target, dim, "dense", rng)
    q0, p0 = _states(target, n, dim, m, rng)
    eps_c = STEP[target] * 10.0 ** rng.uniform(-0.7, 0.3, n)
    opts = _opts(depth, extra=True)
    uni = rng.uniform(size=(n, n_uniforms(opts)))
    return target, system, q0, p0, eps_c, uni, opts, rng


def _assert_same(a, b, rows_a, rows_b, label):
    for k in OUTPUTS:
        x, y = a[k][rows_a], b[k][rows_b]
        bad = np.flatnonzero(~(x.view(np.uint8).reshape(len(rows_a), -1)
                               == y.view(np.uint8).reshape(len(rows_b), -1)).all(1))
        assert bad.size == 0, f"{label}: {k} differs on chains {np.asarray(rows_a)[bad][:8]}"


@pytest.mark.gpu
@pytest.mark.parametrize("kp", [1, 2], ids=["KP1", "KP2"])
def test_lockstep_poisoned_neighbours(kp):
    """In chosen lock-step groups every chain but one or two is replaced by a NaN position, a
    step size that diverges at the first leaf, eps_c = 0, or a chain that runs to the maximum
    depth; every untouched chain is bit-identical in all 11 outputs."""
    groups = 2 if kp == 1 else 1
    n = 8 * groups * 40 + 5
    target, system, q0, p0, eps_c, uni, opts, rng = _indep_inputs(kp, n, 6)
    clean = run_fused(system, q0, p0, 0.0, eps_c, uni, opts)
    q1, p1, e1 = q0.copy(), p0.copy(), eps_c.copy()
    kinds = ["nan", "diverge", "zero", "maxdepth"]
    touched = []
    for gi, g in enumerate(range(0, n // 8, 3)):
        rows = np.arange(8 * g, min(8 * g + 8, n))
        keep = rng.choice(rows, size=1 + gi % 2, replace=False)
        for r, c in enumerate(np.setdiff1d(rows, keep)):
            kind = kinds[(gi + r) % 4]
            if kind == "nan":
                q1[c, rng.integers(q0.shape[1])] = np.nan
            elif kind == "diverge":
                e1[c] = 1e3
            elif kind == "zero":
                e1[c] = 0.0
            else:
                e1[c] = 1e-6
            touched.append(c)
    dirty = run_fused(system, q1, p1, 0.0, e1, uni, opts)
    kept = np.setdiff1d(np.arange(n), touched)
    t = np.array(touched)
    assert (dirty["diverging"][t[e1[t] == 1e3]] == 1).all()
    assert (dirty["tree_depth"][t[(e1[t] == 1e-6) | (e1[t] == 0.0)]] == opts["depth"] - 1).all()
    _assert_same(clean, dirty, kept, kept, f"KP {kp} poisoned neighbours")


@pytest.mark.gpu
@pytest.mark.parametrize("kp", [1, 2], ids=["KP1", "KP2"])
def test_lockstep_placement(kp):
    """The batch rotated by 8 GROUPS m + 3 rows: every chain lands in another warp slot, group,
    CTA and pass of the grid, and its outputs are bit-identical (each row of U = G M^-1 comes
    from the same DMMA sequence whatever the row)."""
    groups = 2 if kp == 1 else 1
    n = 20_000
    target, system, q0, p0, eps_c, uni, opts, _ = _indep_inputs(kp, n, 5)
    a = run_fused(system, q0, p0, 0.0, eps_c, uni, opts)
    s = 8 * groups * 701 + 3
    perm = np.roll(np.arange(n), s)  # row r of the rotated batch is chain perm[r]
    b = run_fused(system, q0[perm], p0[perm], 0.0, eps_c[perm], uni[perm], opts)
    _assert_same(a, b, perm, np.arange(n), f"KP {kp} rotated by {s}")


# ------------------------------------------------------------------------------------------------
# Starvation
# ------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dmma1_std_d8", "warp2_diag_std_d65"])
def test_starvation(name):
    """n_uniforms smaller than some chains need: those report status 1 with every uniform
    used, match the oracle that draws 0.5 past the end, and every other chain is bit-identical
    to the full-table run."""
    target, dim, metric, n, opts, system, minv, q0, p0, eps_c, uni, rng = _case_inputs(name)
    eps = STEP[target]
    full = run_fused(system, q0, p0, eps, eps_c, uni, opts)
    counts = np.unique(full["n_used"])
    assert counts.size > 1
    short = int(counts[(counts.size - 1) // 2])  # some chains need more, some no more
    part = run_fused(system, q0, p0, eps, eps_c, uni, opts, n_uni=short)
    starved = part["status"] == 1
    assert starved.any() and not starved.all()
    assert np.array_equal(starved, full["n_used"] > short)
    assert (part["n_used"][starved] == short).all()
    rows = np.flatnonzero(~starved)
    _assert_same(full, part, rows, rows, f"{name} n_uniforms {short}")
    eps_all = np.full(n, eps) if eps_c is None else eps_c
    idx = rng.choice(np.flatnonzero(starved), size=min(20, int(starved.sum())), replace=False)
    check_against_oracle(f"{name} starved", target, q0, p0, eps_all, uni, opts, minv, part,
                         np.sort(idx), n_uni=short)


@pytest.mark.gpu
def test_starvation_raises_through_sample(monkeypatch):
    """The public transition raises when a chain runs out of uniform variates."""
    target, dim, metric, n, opts, system, minv, q0, p0, eps_c, uni, rng = _case_inputs(
        "dmma1_funnel_d9")
    integ = minteg.LeapfrogIntegrator(system, STEP[target])
    tr = transitions.SliceDynamicIntegrationTransition(
        system, integ, max_tree_depth=opts["depth"], max_delta_h=opts["max_delta_h"])
    assert tr._fused
    monkeypatch.setattr(type(tr), "n_uniforms", property(lambda self: 4))
    state = ChainState(pos=torch.as_tensor(q0, device=DEV), mom=torch.as_tensor(p0, device=DEV),
                       dir=1)
    with pytest.raises(RuntimeError, match="ran out of uniform variates"):
        tr.sample(state, [np.random.default_rng([9, c]) for c in range(n)])


# ------------------------------------------------------------------------------------------------
# The lock-step generic arm (nuts_generic.cuh), every KP
# ------------------------------------------------------------------------------------------------

GENERIC = {1: ("banana", 40, "diagonal", _opts(6, True, True)),
           2: ("neal_funnel", 100, "identity", _opts(5)),
           4: ("std_gaussian", 200, "diagonal", _opts(6, False, True, False)),
           8: ("banana", 400, "identity", _opts(4, True)),
           16: ("neal_funnel", 700, "diagonal", _opts(4, False, False, True, max_delta_h=0.5))}


@pytest.mark.gpu
@need_extended
@pytest.mark.parametrize("kp", list(GENERIC), ids=[f"KP{k}" for k in GENERIC])
def test_generic_arm_matches_oracle(kp):
    """transition._fused = False: the leaves through the leapfrog kernel, the tree bookkeeping in
    the nuts_generic_* kernels; per-chain generators, the same checks as the fused kernels."""
    target, dim, metric, opts = GENERIC[kp]
    n = 64
    rng = np.random.default_rng(900 + kp)
    system, m, minv = _system(target, dim, metric, rng)
    q0, p0 = _states(target, n, dim, m, rng)
    eps = STEP[target]
    cls = (transitions.SliceDynamicIntegrationTransition if opts["slice"]
           else transitions.MultinomialDynamicIntegrationTransition)
    crit = (transitions.euclidean_no_u_turn_criterion if opts["euclid"]
            else transitions.riemannian_no_u_turn_criterion)
    tr = cls(system, minteg.LeapfrogIntegrator(system, eps), max_tree_depth=opts["depth"],
             max_delta_h=opts["max_delta_h"], termination_criterion=crit,
             do_extra_subtree_checks=bool(opts["extra"]))
    tr._fused = False
    gens = [np.random.default_rng([77, kp, c]) for c in range(n)]
    # one more than the table, to find where each generator was left
    uni = np.stack([np.random.default_rng([77, kp, c]).uniform(size=n_uniforms(opts) + 1)
                    for c in range(n)])
    state = ChainState(pos=torch.as_tensor(q0, device=DEV), mom=torch.as_tensor(p0, device=DEV),
                       dir=1)
    new, st = tr.sample(state, gens)
    torch.cuda.synchronize()
    # the generators are left advanced by the uniforms each chain used
    used = np.array([int(np.flatnonzero(uni[c] == g.uniform())[0]) for c, g in enumerate(gens)])
    uni = uni[:, :-1]
    out = {"pos": new.pos.cpu().numpy(), "mom": new.mom.cpu().numpy(), "h": new.h.cpu().numpy(),
           "n_step": st["n_step"].cpu().numpy(), "av_accept":
           st["av_metrop_accept_prob"].cpu().numpy(), "reject_prob": st["reject_prob"].cpu().numpy(),
           "tree_depth": st["tree_depth"].cpu().numpy(), "diverging":
           st["diverging"].cpu().numpy().astype(np.int64), "n_used": used,
           "dir": np.broadcast_to(new.dir.cpu().numpy() if torch.is_tensor(new.dir) else new.dir,
                                  (n,)), "status": np.zeros(n, dtype=np.int64)}
    check_against_oracle(f"generic KP {kp} {target} D {dim} {metric}", target, q0, p0,
                         np.full(n, eps), uni, opts, minv, out, np.arange(n),
                         tracked_velocity=False)


# ------------------------------------------------------------------------------------------------
# Which kernel ran
# ------------------------------------------------------------------------------------------------


def _launched(fn):
    from torch.profiler import ProfilerActivity, profile  # noqa: PLC0415

    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"CUDA activity tracing not usable: {e}")
    names = [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]
    if not names:
        pytest.skip("CUDA activity tracing recorded no kernels (CUPTI not usable)")
    return names


def _matches(names, kname, args):
    pat = re.compile(re.escape(kname) + r"<(?:mb200::)?" + re.escape(args[0]) + "".join(
        r",\s*" + str(a) for a in args[1:]) + r">")
    return [s for s in names if pat.search(s)]


@pytest.mark.gpu
def test_expected_kernels_launch():
    """Every case of the matrix starts the fused kernel it is listed under (all 21 of them), and
    the generic arm starts the nuts_generic_* kernels of its KP."""
    seen = set()
    for name, (target, dim, metric, n, opts, steps) in CASES.items():
        rng = np.random.default_rng(1)
        system, m, _ = _system(target, dim, metric, rng)
        q0, p0 = _states(target, 9, dim, m, rng)
        o = _opts(1)
        uni = rng.uniform(size=(9, n_uniforms(o)))
        kname, args = expected_kernel(target, dim, metric)
        names = _launched(lambda: run_fused(system, q0, p0, 0.01, None, uni, o))
        assert _matches(names, kname, args), (name, kname, args, sorted(set(names)))
        seen.add((kname, args))
    assert len(seen) == 21, sorted(seen)
    for kp, (target, dim, metric, _) in GENERIC.items():
        rng = np.random.default_rng(2)
        system, m, _ = _system(target, dim, metric, rng)
        q0, p0 = _states(target, 4, dim, m, rng)
        tr = transitions.MultinomialDynamicIntegrationTransition(
            system, minteg.LeapfrogIntegrator(system, 0.01), max_tree_depth=1)
        tr._fused = False
        state = ChainState(pos=torch.as_tensor(q0, device=DEV),
                           mom=torch.as_tensor(p0, device=DEV), dir=1)
        names = _launched(lambda: tr.sample(state, np.random.default_rng(3)))
        for part in ("begin", "start", "leaf", "finish", "end"):
            assert [s for s in names if re.search(rf"nuts_generic_{part}_kernel<{kp}>", s)], (
                kp, part, sorted(set(names)))
        assert not [s for s in names if "nuts_euclidean_kernel" in s or "nuts_dmma_kernel" in s]


# ------------------------------------------------------------------------------------------------
# CPU self-checks of the harness
# ------------------------------------------------------------------------------------------------

FIXTURES = ["nuts_c1_multinomial_d10", "nuts_c1_slice_euclidean_d16",
            "nuts_c0_depth4_no_extra_checks", "nuts_c1_diag_divergent", "nuts_c1_identity_d70"]


def _fixture_opts(opts):
    return _opts(opts.get("max_tree_depth", 10), opts.get("variant") == "slice",
                 opts.get("criterion") == "euclidean", opts.get("extra_checks", True),
                 opts.get("max_delta_h", 1000.0))


@pytest.mark.parametrize("name", FIXTURES)
def test_harness_reproduces_nuts_fixture(name):
    """The harness's oracle plumbing (uniform table, per-chain step, leaf index) reproduces the
    fixture from its own seeds: per iteration the momentum, then a uniform table, then the
    generator rewound to the count used (as transitions._uniform_table / _replay do).  The leaf
    index of each returned state, replayed with mo.leapfrog_steps, gives that state bit for bit."""
    from golden_util import load_nuts_case  # noqa: PLC0415

    problem, n_iter, seed, fopts, g = load_nuts_case(name)
    opts = _fixture_opts(fopts)
    otarget = dr.build_target(problem)
    ometric = mo.coerce_metric(problem.metric)
    sample_mom = mo.euclidean_sample_momentum(ometric)
    ref = dr.oracle_nuts(problem, n_iter, seed, **fopts)
    n = problem.pos.shape[0]
    for c in range(n):
        rng = np.random.default_rng([seed, c])
        q = problem.pos[c].copy()
        for it in range(n_iter):
            p = sample_mom(q, rng)
            saved = rng.bit_generator.state
            row = rng.uniform(size=n_uniforms(opts))
            qn, pn, st, j, _, used, starved = oracle_chain(q, p, row, problem.step_size, otarget,
                                                           ometric, opts)
            rng.bit_generator.state = saved
            rng.uniform(size=used)
            assert not starved
            assert np.array_equal(qn, g["pos"][it, c])  # the reference's positions, bitwise
            for k in ("n_step", "tree_depth", "diverging", "dir"):
                assert st[k] == g[k][it, c], k
            for k in ("av_metrop_accept_prob", "reject_prob"):  # the oracle's, bitwise
                assert st[k] == ref[k][it, c], k
            qj, pj = mo.leapfrog_steps(q, p, np.sign(j) * problem.step_size, abs(int(j)),
                                       otarget, ometric)
            assert np.array_equal(qj, qn) and np.array_equal(pj, pn), (c, it, j)
            q = qn


@pytest.mark.parametrize("target", ["std_gaussian", "neal_funnel", "banana"])
@pytest.mark.parametrize("metric", ["diagonal", "identity"])
def test_extended_reference_metric_forms(target, metric):
    """leapfrog_ext with a diagonal (vector) or identity (None) M^-1 and per-row step counts
    equals the dense form with diag(M^-1) / I run row by row."""
    rng = np.random.default_rng(4)
    dim = 6
    _, m, minv = _system(target, dim, metric, rng)
    q0, p0 = _states(target, 3, dim, m, rng)
    dense = np.diag(minv) if metric == "diagonal" else np.identity(dim)
    steps = np.array([0, 3, 5])
    dt = np.array([0.05, -0.03, 0.04])
    q, p = leapfrog_ext(target, q0, p0, dt, steps, minv)
    for r in range(3):
        qr, pr = leapfrog_ext(target, q0[r:r + 1], p0[r:r + 1], dt[r:r + 1], int(steps[r]), dense)
        np.testing.assert_allclose(q[r].astype(np.float64), qr[0].astype(np.float64), rtol=1e-17)
        np.testing.assert_allclose(p[r].astype(np.float64), pr[0].astype(np.float64), rtol=1e-17)
