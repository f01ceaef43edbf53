"""Extended-precision reference shared by the kernel accuracy tests: a batched NumPy leapfrog in
``np.longdouble`` (64-bit significand on x86, 113 on aarch64) with the reference's schedule, the
exact energy with the scale of its terms, and the rule that bounds a kernel's error by the float64
oracle's (``oracle/mici_oracle.py``) error on the same chains."""

import numpy as np
import pytest

from oracle import targets as otargets

L = np.longdouble
ULP = 2.0**-52  # float64 epsilon: errors below are reported in these units
EXTENDED = np.finfo(np.longdouble).nmant >= 63
need_extended = pytest.mark.skipif(
    not EXTENDED, reason=f"np.longdouble has a {np.finfo(np.longdouble).nmant}-bit mantissa, "
    "the extended-precision reference needs >= 63")

BANANA_B = 0.5


# ------------------------------------------------------------------------------------------------
# Formulas of oracle/targets.py; schedule of mici_oracle.leapfrog_steps: half kick, drift with
# M^-1, half kick with the memoised gradient, the two half kicks at a step boundary applied
# separately.  The metric is the float64 M^-1 a kernel is given: a D x D array (dense), a vector
# (diagonal) or None (identity).
# ------------------------------------------------------------------------------------------------


def _grad(target, q):
    dim = q.shape[1]
    if target == "std_gaussian":
        return q.copy()
    g = np.empty_like(q)
    if target == "neal_funnel":
        v, x = q[:, :1], q[:, 1:]
        e = np.exp(-v)
        g[:, :1] = v / L(9) + L(0.5) * (dim - 1) - L(0.5) * e * (x * x).sum(1, keepdims=True)
        g[:, 1:] = e * x
        return g
    b = L(BANANA_B)
    x, y = q[:, 0::2], q[:, 1::2]
    r = y - b * x * x
    g[:, 0::2] = x / L(4) - L(2) * b * x * r
    g[:, 1::2] = r
    return g


def _inv_apply(a, p):
    """M^-1 p per row for a dense (2-D), diagonal (1-D) or identity (None) M^-1."""
    if a is None:
        return p
    return p * a if a.ndim == 1 else p @ a.T


def _h_terms(target, q, p, a):
    """Per-chain h(q, p) = l(q) + p . M^-1 p / 2 and the sum of the absolute values of its terms
    (the scale its rounding error is measured against: the funnel's l cancels)."""
    dim = q.shape[1]
    kin = L(0.5) * np.einsum("ij,ij->i", p, _inv_apply(a, p))
    if target == "std_gaussian":
        terms = [L(0.5) * (q * q).sum(1)]
    elif target == "neal_funnel":
        v, x = q[:, 0], q[:, 1:]
        terms = [v * v / L(18), L(0.5) * (dim - 1) * v, L(0.5) * np.exp(-v) * (x * x).sum(1)]
    else:
        b = L(BANANA_B)
        x, y = q[:, 0::2], q[:, 1::2]
        r = y - b * x * x
        terms = [(x * x / L(8)).sum(1), (L(0.5) * r * r).sum(1)]
    h = sum(terms) + kin
    scale = sum(np.abs(t) for t in terms) + np.abs(kin)
    return h, scale


def leapfrog_ext(target, q, p, time_step, n_steps, minv):
    """n_steps leapfrog steps of every row of (q, p) in long double; time_step[c] = dir * eps_c.
    ``n_steps`` is one count for all rows or a count per row (a row stops after its own)."""
    q, p = q.astype(L), p.astype(L)
    a = None if minv is None else np.asarray(minv).astype(L)
    dt = np.asarray(time_step).astype(L)[:, None]
    counts = np.broadcast_to(np.asarray(n_steps), (q.shape[0],))
    g = _grad(target, q)
    for s in range(int(counts.max(initial=0))):
        live = (s < counts)[:, None]
        p1 = p - (dt / 2) * g
        q1 = q + dt * _inv_apply(a, p1)  # (M^-1 p) per row
        g1 = _grad(target, q1)
        p1 = p1 - (dt / 2) * g1
        if live.all():
            q, p, g = q1, p1, g1
        else:
            q, p, g = np.where(live, q1, q), np.where(live, p1, p), np.where(live, g1, g)
    return q, p


def _oracle_target(target, dim):
    if target == "banana":
        return otargets.Banana(dim, BANANA_B)
    return {"std_gaussian": otargets.StdGaussian, "neal_funnel": otargets.NealFunnel}[target](dim)


class _GivenInverse:
    """A fixed metric given by the explicit float64 M^-1 the kernel multiplies with: a D x D
    array (dense), a vector (diagonal) or None (identity)."""

    def __init__(self, minv):
        self.inv_array = minv
        self.kind = "identity" if minv is None else ("diagonal" if minv.ndim == 1 else "dense")

    def inv_matvec(self, v):
        if self.inv_array is None:
            return v
        return self.inv_array * v if self.inv_array.ndim == 1 else self.inv_array @ v

    def sqrt_matvec(self, v):  # not used by the leapfrog
        raise NotImplementedError


# ------------------------------------------------------------------------------------------------
# Errors and the bound
# ------------------------------------------------------------------------------------------------


def _rel_err(x, ref):
    """Per-chain max_i |x_i - ref_i| / max_i |ref_i| in units of 2^-52."""
    return (np.abs(x.astype(L) - ref).max(1) / np.abs(ref).max(1) / L(ULP)).astype(np.float64)


def _check_ratio(what, kern, orc, factor=1):
    """A kernel's per-chain errors against `factor` x the float64 oracle's on the same chains:
    worst chain <= 4 x factor x oracle's worst + 8 ulp, mean <= 2 x factor x oracle's mean + 2 ulp.
    Returns None or the failure message, and the report line."""
    kw, km, ow, om = kern.max(), kern.mean(), orc.max(), orc.mean()
    report = f"{what} worst {kw:.2f}/{ow:.2f} mean {km:.3f}/{om:.3f}"
    if kw > 4 * factor * ow + 8:
        return f"{what}: kernel worst {kw:.2f} ulp vs {factor} x oracle worst {ow:.2f}", report
    if km > 2 * factor * om + 2:
        return f"{what}: kernel mean {km:.3f} ulp vs {factor} x oracle mean {om:.3f}", report
    return None, report
