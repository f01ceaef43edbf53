"""The tensor-core leapfrog kernel (K1, ``leapfrog_dmma.cuh``) against an extended-precision
reference, on every target it is instantiated for, every dimension class, shared and per-chain
step sizes, and every tile layout that its launch can choose on this device.

* The reference is a batched NumPy leapfrog in ``np.longdouble`` (64-bit significand on x86,
  113 on aarch64) with the reference's schedule.  It takes exactly the kernel's float64 inputs,
  including the float64 ``M^-1`` the kernel is given.  A CPU test checks it against ``mpmath``.
* K1's error against it is bounded by the float64 oracle's (``oracle/mici_oracle.py``) error on
  the same chains: worst chain <= 4 x oracle's worst + 8 ulp, mean <= 2 x oracle's mean + 2 ulp
  for the energy; for q and p the oracle's error is first multiplied by the number of times K1
  rounds q per drift (its DMMA accumulator is q itself).  An accuracy loss of a few ulp per step
  would show up here, long before it would exceed the 1e-10 tolerances of the parity tests.
* ``exp_short_chain`` (the funnel's exp(-v) in K1) is checked on the device against the
  extended-precision exp, inside and outside its polynomial range, and for warps that mix both.
* A chain's result does not depend on its neighbours: poisoning one chain per group (NaN, inf,
  an exp(-v) outside the polynomial range) leaves every other chain bit-identical.
"""

import ctypes
import zlib

import numpy as np
import pytest
import torch

from mici_b200 import _lib, problems, systems
from mici_b200 import targets as mtargets
from oracle import mici_oracle as mo

from extended_precision import (BANANA_B, ULP, L, _check_ratio, _GivenInverse, _h_terms,
                                _oracle_target, _rel_err, leapfrog_ext, need_extended)

DEV = "cuda:0"

TARGETS = ["std_gaussian", "neal_funnel", "banana"]
STEP = {"std_gaussian": 0.1, "neal_funnel": 0.01, "banana": 0.05}
# dimensions on both sides of each class boundary of the kernel's padded width DP (even only for
# the banana, whose coordinates come in pairs)
DIMS = {32: [8, 9, 31, 32], 64: [33, 63, 64], 96: [65, 96], 128: [97, 127, 128]}
BANANA_DIMS = {32: [8, 32], 64: [34, 64], 96: [66, 96], 128: [98, 128]}


# ------------------------------------------------------------------------------------------------
# Tile layouts.  Restates the tiling of launch_dmma (leapfrog_dmma.cuh): T = ceil(n / 8) row tiles
# of 8 chains, tpc = min(ceil(T / S), 8) tiles per CTA and pass, blocks = min(ceil(T / tpc), S)
# persistent CTAs over the S SMs; the tiles of a pass are dealt to the 4 groups of a CTA as
# tiles / 4 + (g < tiles % 4).  A group with one tile runs the m8n8k4 path with its k-split
# (MT = 1), a group with two the m16n8k16 path (MT = 2).
# ------------------------------------------------------------------------------------------------


def _layout(n, sms):
    tiles = -(-n // 8)
    tpc = min(-(-tiles // sms), 8)
    blocks = min(-(-tiles // tpc), sms)
    return tiles, tpc, blocks


def _group_tiles(tiles):
    return [tiles // 4 + (g < tiles % 4) for g in range(4)]


def _passes(n, sms):
    """[(chain0, tiles)] of every CTA pass, in order of chain0."""
    tiles, tpc, _ = _layout(n, sms)
    rows = 8 * tpc
    return [(c0, min(tpc, -(-(n - c0) // 8))) for c0 in range(0, n, rows)]


LAYOUTS = ["tpc1", "tpc4", "tpc7", "tpc8", "over8S"]


def _batch(layout, sms):
    """Batch size that gives `layout` on `sms` SMs, always with a partial last tile (5 live
    chains): tpc1 one lone tile per CTA (three idle groups); tpc4 four lone-tile groups; tpc7
    groups of 2, 2, 2, 1; tpc8 eight tiles in every CTA; over8S more than 8 S tiles, so that CTA 0
    takes a second pass with 3 tiles (one idle group)."""
    tiles = {"tpc1": max(sms - 7, 1), "tpc4": 4 * sms - 2, "tpc7": 7 * sms - 3, "tpc8": 8 * sms,
             "over8S": 8 * sms + 3}[layout]
    n = 8 * tiles - 3
    t, tpc, blocks = _layout(n, sms)
    assert t == tiles
    if layout == "over8S":
        assert tpc == 8 and blocks == sms and _passes(n, sms)[-1][1] == 3
    else:
        assert tpc == int(layout[3:])
    return n


def _mts(n, sms):
    """Set of group tile counts (MT) that occur in a batch of n chains."""
    return {mt for _, t in _passes(n, sms) for mt in _group_tiles(t) if mt > 0}


# ------------------------------------------------------------------------------------------------
# Inputs and the launch
# ------------------------------------------------------------------------------------------------


def _inputs(target, n, dim, seed):
    """Seeded initial states and the float64 M^-1 that the system hands to the kernel."""
    rng = np.random.default_rng(seed)
    metric = problems.dense_spd_metric(rng, dim)
    if target == "neal_funnel":
        # per-chain v over [-8, 8] and x ~ N(0, exp(v)): every chain's exp(-v) is distinct and
        # its term is as large as the others
        v = rng.uniform(-8.0, 8.0, n)
        q = np.concatenate([v[:, None], rng.standard_normal((n, dim - 1)) * np.exp(v / 2)[:, None]],
                           axis=1)
    elif target == "banana":
        q = rng.standard_normal((n, dim))
        q[:, 0::2] *= 2.0
        q[:, 1::2] += BANANA_B * q[:, 0::2] ** 2
    else:
        q = rng.standard_normal((n, dim))
    p = rng.standard_normal((n, dim)) @ np.linalg.cholesky(metric).T
    params = {"dim": dim, "b": BANANA_B} if target == "banana" else {"dim": dim}
    system = systems.EuclideanMetricSystem(mtargets.make_target(target, **params), metric=metric)
    return q, p, system, rng


def _run_k1(system, q, p, dirs, eps, eps_c, n_steps):
    """One mb200_leapfrog_euclidean launch (dense metric, leapfrog schedule, no per-chain
    lengths: the tensor-core kernel) -> host arrays pos, mom, h, status, n_done."""
    n, dim = q.shape
    qt = torch.as_tensor(q, device=DEV)
    pt = torch.as_tensor(p, device=DEV)
    dt = torch.as_tensor(dirs.astype(np.int32), device=DEV)
    et = None if eps_c is None else torch.as_tensor(eps_c, dtype=torch.float64, device=DEV)
    qo, po = torch.empty_like(qt), torch.empty_like(pt)
    h = torch.empty(n, dtype=torch.float64, device=DEV)
    status = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    n_done = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    model = system._model(qt.device)
    minv = system.metric.inv_device(qt.device)
    rc = _lib.load().mb200_leapfrog_euclidean(
        _lib.ptr(qt), _lib.ptr(pt), _lib.ptr(qo), _lib.ptr(po), _lib.ptr(dt), n, dim,
        0.0 if eps_c is not None else eps, _lib.ptr(et), n_steps, None, 0, None, 0,
        system.metric.kind, _lib.ptr(minv), ctypes.byref(model), _lib.ptr(h), _lib.ptr(status),
        _lib.ptr(n_done), _lib.current_stream_ptr(qt.device))
    assert rc == 0, _lib.load().mb200_last_error()
    torch.cuda.synchronize()
    return (qo.cpu().numpy(), po.cpu().numpy(), h.cpu().numpy(), status.cpu().numpy(),
            n_done.cpu().numpy())


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------
# Accuracy cases: every target x DP class x {shared, per-chain step size} once on a layout with
# groups of one and of two tiles (tpc7 or over8S), plus every target on the single-MT layouts
# ------------------------------------------------------------------------------------------------


def _cases():
    cases = []
    k = 0
    for target in TARGETS:
        dims = BANANA_DIMS if target == "banana" else DIMS
        for dp, ds in dims.items():
            for pc in (False, True):
                cases.append((target, ds[k % len(ds)], ("tpc7", "over8S")[k % 2], pc,
                              (1, 2, 50)[k % 3], -1.0 if (k % 4) == 2 else 1.0))
                k += 1
    extra = [
        ("std_gaussian", 64, "tpc1", True, 50, 1.0), ("std_gaussian", 127, "tpc4", False, 2, -1.0),
        ("std_gaussian", 33, "tpc8", False, 50, 1.0), ("neal_funnel", 128, "tpc1", False, 50, 1.0),
        ("neal_funnel", 9, "tpc4", True, 50, 1.0), ("neal_funnel", 128, "tpc8", False, 50, 1.0),
        ("neal_funnel", 97, "tpc8", True, 2, 1.0), ("banana", 96, "tpc1", False, 2, -1.0),
        ("banana", 128, "tpc4", True, 50, 1.0), ("banana", 64, "tpc8", False, 50, 1.0),
    ]
    return cases + extra


CASES = _cases()


def _case_id(c):
    target, dim, layout, pc, n_steps, sign = c
    eps = "per_chain" if pc else ("neg_eps" if sign < 0 else "eps")
    return f"{target}-d{dim}-{layout}-{eps}-{n_steps}steps"


def _sample(n, sms, rng, extra=()):
    """All chains of the first and of the last CTA pass, ~250 random others: <= ~380 chains."""
    passes = _passes(n, sms)
    first = np.arange(0, min(8 * passes[0][1], n))
    last = np.arange(passes[-1][0], n)
    rest = np.setdiff1d(np.arange(n), np.concatenate([first, last]))
    pick = rng.choice(rest, size=min(250, rest.size), replace=False) if rest.size else rest
    return np.unique(np.concatenate([first, last, pick, np.asarray(extra, dtype=np.int64)]))


def _accumulation_roundings(dim):
    """Roundings of a position per drift inside K1 (documented deviation, DESIGN.md section 2):
    the drift accumulates into q itself, the DMMA accumulator, so q is rounded once per DMMA
    instruction, where the oracle rounds q + dt * (M^-1 p) once.  A lone row tile (m8n8k4 with
    its k-split) adds DP / 8 instructions into q plus the sum of the split; a two-tile group
    (m16n8k16) DP / 16."""
    dp = 32 * -(-dim // 32)
    return dp // 8 + 1


@pytest.mark.gpu
@need_extended
@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_k1_within_oracle_error_of_extended_reference(case):
    """q, p and the energy of K1 stay within a small multiple of the float64 oracle's own error
    against the long-double leapfrog, chain by chain (worst and mean over the sampled chains)."""
    target, dim, layout, pc, n_steps, sign = case
    sms = _sms()
    n = _batch(layout, sms)
    q0, p0, system, rng = _inputs(target, n, dim, seed=zlib.crc32(_case_id(case).encode()))
    dirs = rng.choice([-1, 1], n)
    eps = sign * STEP[target]
    eps_c = None
    if pc:
        eps_c = STEP[target] * rng.uniform(0.5, 1.5, n)
        eps_c[3] = 0.0  # in the first CTA: this chain does not move
    pos, mom, h, status, n_done = _run_k1(system, q0, p0, dirs, eps, eps_c, n_steps)
    assert (status == 0).all()
    assert (n_done == n_steps).all()

    idx = _sample(n, sms, rng, extra=[3])
    minv = system.metric.inv_device(DEV).cpu().numpy()
    a = minv.astype(L)
    step = dirs[idx] * (eps_c[idx] if pc else eps)
    q_ref, p_ref = leapfrog_ext(target, q0[idx], p0[idx], step, n_steps, minv)

    otarget, ometric = _oracle_target(target, dim), _GivenInverse(minv)
    q_or, p_or, h_or = np.empty((idx.size, dim)), np.empty((idx.size, dim)), np.empty(idx.size)
    for j, c in enumerate(idx):
        q_or[j], p_or[j] = mo.leapfrog_steps(q0[c], p0[c], float(step[j]), n_steps, otarget,
                                             ometric)
        h_or[j] = mo.euclidean_h(q_or[j], p_or[j], otarget, ometric)

    # q and p against R x the oracle's error, R the roundings of q per drift (the kicks carry q's
    # error into p).  Measured on an H100: K1's error reaches 0.32 R x the oracle's worst + 8 and
    # 0.52 R x its mean + 2 (R = 5 .. 17); the plain rule (R = 1) fails at every D >= 33.
    rq = _accumulation_roundings(dim)
    checks = [_check_ratio("q", _rel_err(pos[idx], q_ref), _rel_err(q_or, q_ref), rq),
              _check_ratio("p", _rel_err(mom[idx], p_ref), _rel_err(p_or, p_ref), rq)]
    # the energy in isolation: the exact h at each method's own output state, plain rule
    hk, sk = _h_terms(target, pos[idx].astype(L), mom[idx].astype(L), a)
    ho, so = _h_terms(target, q_or.astype(L), p_or.astype(L), a)
    eh_k1 = (np.abs(h[idx].astype(L) - hk) / sk / L(ULP)).astype(np.float64)
    eh_or = (np.abs(h_or.astype(L) - ho) / so / L(ULP)).astype(np.float64)
    checks.append(_check_ratio("h", eh_k1, eh_or))
    print(f"[k1 vs long double] {_case_id(case)} MT {sorted(_mts(n, sms))} R {rq} "
          f"({idx.size} of {n} chains; K1/oracle ulp): " + "; ".join(r for _, r in checks))
    failures = [f for f, _ in checks if f is not None]
    assert not failures, failures
    if pc:  # eps_c = 0: the unmoved state and its energy
        j = int(np.searchsorted(idx, 3))
        assert np.array_equal(pos[3], q0[3]) and np.array_equal(mom[3], p0[3])
        assert np.isfinite(h[3]) and eh_k1[j] <= 4


# ------------------------------------------------------------------------------------------------
# The reference itself against mpmath (CPU)
# ------------------------------------------------------------------------------------------------


def _mp_leapfrog(mp, target, q, p, dt, n_steps, a):
    dim = len(q)
    q = [mp.mpf(float(x)) for x in q]
    p = [mp.mpf(float(x)) for x in p]
    a = [[mp.mpf(float(x)) for x in row] for row in a]
    dt = mp.mpf(float(dt))

    def grad(q):
        if target == "std_gaussian":
            return list(q)
        if target == "neal_funnel":
            e = mp.exp(-q[0])
            xx = mp.fsum(x * x for x in q[1:])
            return [q[0] / 9 + mp.mpf(dim - 1) / 2 - e * xx / 2] + [e * x for x in q[1:]]
        g = [None] * dim
        for i in range(0, dim, 2):
            r = q[i + 1] - mp.mpf(BANANA_B) * q[i] ** 2
            g[i], g[i + 1] = q[i] / 4 - 2 * mp.mpf(BANANA_B) * q[i] * r, r
        return g

    g = grad(q)
    for _ in range(n_steps):
        p = [pi - dt / 2 * gi for pi, gi in zip(p, g)]
        q = [qi + dt * mp.fsum(a[i][k] * p[k] for k in range(dim)) for i, qi in enumerate(q)]
        g = grad(q)
        p = [pi - dt / 2 * gi for pi, gi in zip(p, g)]
    return q, p


@need_extended
@pytest.mark.parametrize("target", TARGETS)
@pytest.mark.parametrize("dim", [9, 33])
def test_extended_reference_agrees_with_mpmath(target, dim):
    """The long-double leapfrog agrees with a 50-digit one to below 0.01 x 2^-52 (relative,
    per chain) -- so it can stand in for the exact leapfrog when measuring float64 errors."""
    mp = pytest.importorskip("mpmath").mp
    if target == "banana" and dim % 2:
        dim += 1
    n, n_steps = 3, 3
    q0, p0, system, _ = _inputs(target, n, dim, seed=7 + dim)
    minv = system.metric.inv
    step = STEP[target] * np.array([1.0, -0.7, 1.3])
    q_ld, p_ld = leapfrog_ext(target, q0, p0, step, n_steps, minv)
    with mp.workdps(50):
        for c in range(n):
            q_mp, p_mp = _mp_leapfrog(mp, target, q0[c], p0[c], step[c], n_steps, minv)
            for got, ref in ((q_ld[c], q_mp), (p_ld[c], p_mp)):
                err = max(abs(mp.mpf(str(g)) - r) for g, r in zip(got, ref))
                scale = max(abs(r) for r in ref)
                assert err / scale < 0.01 * ULP, float(err / scale / ULP)


# ------------------------------------------------------------------------------------------------
# exp_short_chain on the device
# ------------------------------------------------------------------------------------------------


def _exp_dev(x):
    xt = torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64), device=DEV)
    yt = torch.empty_like(xt)
    rc = _lib.load().mb200_selftest_exp_short_chain(_lib.ptr(xt), _lib.ptr(yt), xt.numel(),
                                                    _lib.current_stream_ptr(xt.device))
    assert rc == 0, _lib.load().mb200_last_error()
    torch.cuda.synchronize()
    return yt.cpu().numpy()


def _ulp_err(y, x):
    """|y - exp(x)| in units of the spacing of float64 at exp(x) (long-double reference; the
    subnormal spacing 2^-1074 for subnormal results)."""
    ref = np.exp(x.astype(L))
    _, e = np.frexp(ref)
    spacing = np.ldexp(np.ones_like(ref), np.maximum(e, -1021) - 53)
    return (np.abs(y.astype(L) - ref) / spacing).astype(np.float64)


def _sweep(centres, k=64):
    """Every float64 within k ulp of each centre."""
    x = np.asarray(centres, dtype=np.float64)
    for _ in range(k):
        x = np.nextafter(x, -np.inf)
    pts = [x]
    for _ in range(2 * k):
        pts.append(np.nextafter(pts[-1], np.inf))
    return np.concatenate(pts)


def _in_range_points(rng):
    # the argument reduction's breakpoints (k + 1/2) ln 2, where k changes and |r| is largest
    centres = ((np.arange(-1011, 1011) + L(0.5)) * np.log(L(2))).astype(np.float64)
    tiny = np.array([5e-324, -5e-324, 2.2250738585072009e-308, -2.2250738585072009e-308,
                     1e-310, -1e-310, 1e-300, -1e-300, 1e-17, -1e-17])
    x = np.concatenate([rng.uniform(-700.0, 700.0, 1_000_000),
                        _sweep(np.concatenate([centres, [700.0, -700.0, 0.0, -0.0]])), tiny,
                        np.linspace(-30.0, 30.0, 200_001)])
    return x[np.abs(x) < 700.0]


@pytest.mark.gpu
@need_extended
def test_exp_short_chain_in_range():
    """|x| < 700, the polynomial: within 2.5 ulp of exp (its maximum is 2.1-2.2 ulp; one Taylor
    term fewer gives 3.6)."""
    x = _in_range_points(np.random.default_rng(3))
    err = _ulp_err(_exp_dev(x), x)
    worst = int(np.argmax(err))
    print(f"[exp_short_chain] {x.size} points in (-700, 700): max {err[worst]:.3f} ulp at "
          f"x = {x[worst]!r}, mean {err.mean():.3f}")
    assert err[worst] <= 2.5, (x[worst], err[worst])
    assert np.array_equal(_exp_dev(np.array([0.0, -0.0])), [1.0, 1.0])


@pytest.mark.gpu
@need_extended
def test_exp_short_chain_out_of_range():
    """|x| >= 700 and non-finite x take libm's exp: within 1 ulp of exp (the subnormal spacing
    for subnormal results), exactly 0 or inf where exp rounds to those, NaN for NaN."""
    hi = np.concatenate([np.linspace(700.0, 745.0, 450_001), _sweep([700.0, 709.782712893384])])
    hi = hi[hi >= 700.0]
    x = np.concatenate([hi, -hi, [np.inf, -np.inf]])
    y = _exp_dev(x)
    ref = np.exp(x.astype(L))
    with np.errstate(over="ignore"):
        ref64 = ref.astype(np.float64)
    zero_or_inf = (ref64 == 0) | np.isinf(ref64)
    assert np.array_equal(y[zero_or_inf], ref64[zero_or_inf])
    finite = ~zero_or_inf
    err = _ulp_err(y[finite], x[finite])
    assert err.max() <= 1.0, (x[finite][np.argmax(err)], err.max())
    assert np.isnan(_exp_dev(np.array([np.nan, -np.nan]))).all()


@pytest.mark.gpu
def test_exp_short_chain_warp_mixing():
    """A warp whose lanes are partly out of range sends only those lanes to libm: the in-range
    lanes are bit-identical to the same arguments in a warp that is entirely in range.  Lanes
    past the end of the array (a partial last warp) do not change the others either."""
    rng = np.random.default_rng(5)
    n_warps = 64
    base = rng.uniform(-700.0, 700.0, (n_warps, 32))
    out_pool = np.concatenate([rng.uniform(700.0, 745.0, 64), -rng.uniform(700.0, 745.0, 64),
                               [np.inf, -np.inf, np.nan, 700.0, -700.0]])
    mixed = base.copy()
    counts = [0, 1, 31, 32] * (n_warps // 4)
    for w, k in enumerate(counts):
        lanes = rng.choice(32, size=k, replace=False)
        mixed[w, lanes] = rng.choice(out_pool, size=k)
    y_base = _exp_dev(base.ravel()).reshape(n_warps, 32)
    y_mixed = _exp_dev(mixed.ravel()).reshape(n_warps, 32)
    in_range = np.abs(mixed) < 700.0
    assert in_range.sum() > 0
    assert np.array_equal(y_mixed[in_range].view(np.int64), y_base[in_range].view(np.int64))
    y_tail = _exp_dev(base.ravel()[:-7])
    assert np.array_equal(y_tail.view(np.int64), y_base.ravel()[:-7].view(np.int64))


# ------------------------------------------------------------------------------------------------
# Isolation: a chain's result does not depend on the other chains of its tile, group or CTA
# ------------------------------------------------------------------------------------------------

ISOLATION_DIMS = {"std_gaussian": 33, "neal_funnel": 64, "banana": 96}


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["tpc4", "tpc8"], ids=["MT1", "MT2"])
@pytest.mark.parametrize("pc", [False, True], ids=["shared_eps", "per_chain_eps"])
@pytest.mark.parametrize("target", TARGETS)
def test_k1_chains_do_not_affect_each_other(target, pc, layout):
    """One chain in every group of every CTA is poisoned: NaN in q, inf in p, or (funnel) a v
    whose exp(-v) is outside the polynomial's range (v in (700, 745): subnormal; v < -709.8:
    overflow).  Every other chain is bit-identical to the unpoisoned launch, and the poisoned
    chains are NaN exactly where the float64 oracle's are.  This catches a row-index slip in the
    per-chain exchanges (partial sums, exp(-v), energy partials), a 0 x NaN leak through padding,
    or a fallback that switches a whole warp to libm's exp."""
    sms = _sms()
    n = _batch(layout, sms)
    dim = ISOLATION_DIMS[target]
    n_steps = 3
    q0, p0, system, rng = _inputs(target, n, dim, seed=11 + dim)
    dirs = rng.choice([-1, 1], n)
    eps_c = STEP[target] * rng.uniform(0.5, 1.5, n) if pc else None
    clean = _run_k1(system, q0, p0, dirs, STEP[target], eps_c, n_steps)

    kinds = ["nan_q", "inf_p"] + (["v_big", "v_overflow"] if target == "neal_funnel" else [])
    q1, p1 = q0.copy(), p0.copy()
    poisoned = []
    k = 0
    for chain0, tiles in _passes(n, sms):
        row = 0
        for mt in _group_tiles(tiles):
            if mt == 0:
                continue
            c = chain0 + row + int(rng.integers(0, 8 * mt))
            row += 8 * mt
            if c >= n:
                continue
            kind = kinds[k % len(kinds)]
            k += 1
            j = int(rng.integers(0, dim))
            if kind == "nan_q":
                q1[c, j] = np.nan
            elif kind == "inf_p":
                p1[c, j] = np.inf if j % 2 else -np.inf
            elif kind == "v_big":
                q1[c, 0] = rng.uniform(700.5, 744.5)
            else:
                q1[c, 0] = -rng.uniform(709.9, 740.0)
            poisoned.append(c)
    poisoned = np.array(poisoned)
    assert poisoned.size >= 4
    dirty = _run_k1(system, q1, p1, dirs, STEP[target], eps_c, n_steps)

    others = np.setdiff1d(np.arange(n), poisoned)
    for a, b in zip(clean, dirty):
        assert np.array_equal(a[others].view(np.uint8), b[others].view(np.uint8))

    minv = system.metric.inv_device(DEV).cpu().numpy()
    otarget, ometric = _oracle_target(target, dim), _GivenInverse(minv)
    step = dirs * (eps_c if pc else STEP[target])
    with np.errstate(all="ignore"):
        for c in poisoned:
            q_or, p_or = mo.leapfrog_steps(q1[c], p1[c], float(step[c]), n_steps, otarget, ometric)
            assert np.array_equal(np.isnan(dirty[0][c]), np.isnan(q_or)), c
            assert np.array_equal(np.isnan(dirty[1][c]), np.isnan(p_or)), c
