"""Target-model registry of the CUDA path.

The reference accepts arbitrary Python callables for ``neg_log_dens`` and its derivatives
(``src/mici/systems.py:88-95``).  A fused GPU gradient cannot, so the engine ships a closed
registry of models compiled into ``libmici_b200.so`` (``mici_b200/csrc/targets.cuh``); an
instance of one of these classes is what is passed as ``neg_log_dens=`` to the systems in
``mici_b200.systems``.  Instances only carry ids and parameters -- no host arithmetic.  Other
models are written by the user in CUDA C++ and compiled at run time (``CudaTarget``).
"""

from __future__ import annotations

import numpy as np

TARGET_STD_GAUSSIAN = 0
TARGET_NEAL_FUNNEL = 1
TARGET_BANANA = 2
TARGET_QUADRATIC = 3
TARGET_TORUS = 4
TARGET_SPHERE = 5
TARGET_MULTI_SPHERE = 6
TARGET_QUARTIC = 7
TARGET_USER = 64  # MB200_TARGET_USER: CudaTarget, compiled at run time

RMETRIC_SOFTABS = 0
RMETRIC_RANK1 = 1
RMETRIC_HADAMARD = 2
RMETRIC_DIAG_QUADRATIC = 3
RMETRIC_DIAG_FUNNEL_FISHER = 4
RMETRIC_SCALAR_QUADRATIC = 5
RMETRIC_CHOL_QUADRATIC = 6
RMETRIC_USER_DIAGONAL = 32  # MB200_RMETRIC_USER_DIAGONAL: CudaDiagonalMetric
RMETRIC_USER_SCALAR = 33  # MB200_RMETRIC_USER_SCALAR: CudaScalarMetric
RMETRIC_USER_DENSE = 34  # MB200_RMETRIC_USER_DENSE: CudaDenseMetric
RMETRIC_USER_CHOLESKY = 35  # MB200_RMETRIC_USER_CHOLESKY: CudaCholeskyMetric


class Target:
    """Base class: ``target_id``, scalar ``params`` and an optional dense ``aux`` array."""

    target_id: int = -1
    name: str = ""
    n_constr: int = 0

    def __init__(self, dim, params=(), aux=None):
        self.dim = int(dim)
        self.params = tuple(float(x) for x in params)
        self.aux = None if aux is None else np.ascontiguousarray(aux, dtype=np.float64)

    def __repr__(self):
        return f"{type(self).__name__}(dim={self.dim}, params={self.params})"


class StdGaussian(Target):
    """l(q) = |q|^2 / 2."""

    target_id = TARGET_STD_GAUSSIAN
    name = "std_gaussian"

    def __init__(self, dim):
        super().__init__(dim)


class MultiSphere(Target):
    """``n_constr`` (2, 4 or 8) unit spheres on consecutive blocks of ``dim / n_constr``
    coordinates, c_k(q) = |q_block_k|^2 - 1; l = |q|^2/2 + q[0]."""

    target_id = TARGET_MULTI_SPHERE
    name = "multi_sphere"

    def __init__(self, dim, n_constr):
        if n_constr not in (2, 4, 8) or dim % n_constr:
            raise ValueError("n_constr must be 2, 4 or 8 and divide dim.")
        self.n_constr = n_constr
        super().__init__(dim, (float(n_constr),))


class NealFunnel(Target):
    """v = q[0], x = q[1:]; l = v^2/18 + (D-1) v/2 + exp(-v) |x|^2 / 2."""

    target_id = TARGET_NEAL_FUNNEL
    name = "neal_funnel"

    def __init__(self, dim):
        super().__init__(dim)


class Banana(Target):
    """Pairs (x, y): l = sum x^2/8 + (y - b x^2)^2 / 2."""

    target_id = TARGET_BANANA
    name = "banana"

    def __init__(self, dim, b=0.5):
        if dim % 2:
            raise ValueError("Banana target needs an even dimension.")
        super().__init__(dim, (b,))


class Quadratic(Target):
    """l(q) = q^T P q / 2 with dense SPD ``prec``."""

    target_id = TARGET_QUADRATIC
    name = "quadratic"

    def __init__(self, prec):
        prec = np.asarray(prec, dtype=np.float64)
        super().__init__(prec.shape[0], (), prec)


class Quartic(Target):
    """l(q) = |q|^2/2 + (gamma/4) sum_m (a_m . q)^4 with ``directions`` A [D x D]: dense Hessian
    and third-derivative tensor (SoftAbs systems)."""

    target_id = TARGET_QUARTIC
    name = "quartic"

    def __init__(self, directions, gamma=1.0):
        a = np.ascontiguousarray(directions, dtype=np.float64)
        if a.ndim != 2 or a.shape[0] != a.shape[1]:
            raise ValueError("`directions` must be a square matrix (D directions in R^D).")
        super().__init__(a.shape[1], (float(gamma),), a)


class Torus(Target):
    """Density on a torus in R^3 with constraint c(q) = (rho - R)^2 + z^2 - r^2
    (reference README.md:315-337)."""

    target_id = TARGET_TORUS
    name = "torus"
    n_constr = 1

    def __init__(self, R=1.0, r=0.5, alpha=0.9):
        super().__init__(3, (R, r, alpha))


class Sphere(Target):
    """l = |q|^2/2 + q[0] on the unit sphere c(q) = |q|^2 - 1."""

    target_id = TARGET_SPHERE
    name = "sphere"
    n_constr = 1

    def __init__(self, dim):
        super().__init__(dim)


class CudaTarget(Target):
    """A user-written model: CUDA C++ source defining

        __device__ double neg_log_dens(const mb200::Chain& c);
        __device__ void grad_neg_log_dens(const mb200::Chain& c, double* g);

    (contract and rules: ``mici_b200/csrc/user_target.cuh``), compiled at run time with NVRTC
    together with the engine's general-dimension Euclidean kernels (``mici_b200.jit``).  ``params``
    (at most 8 scalars) reach the functions as ``c.params``, ``aux`` (any array convertible to
    fp64, e.g. a data matrix) as the device array ``c.aux``.  Runs on ``EuclideanMetricSystem``
    with any fixed metric, ``dim <= 1024``.

    The source compiles on first use (``compile()`` compiles now).  The instance holds only
    source, params and aux; the compiled image lives in a process-wide cache, so systems and
    integrators holding a ``CudaTarget`` survive ``deepcopy`` and pickling.

    ``n_constr >= 1`` makes it a constrained target: the source also defines ``constr`` and
    ``jacob_constr`` over ``mb200::N_CONSTR = n_constr`` constraints, and ``mhp_constr`` when
    ``mhp_constr=True`` (contract: ``mici_b200/csrc/user_constraint.cuh``).  It then runs on the
    constrained Euclidean systems with ``ConstrainedLeapfrogIntegrator``: ``n_constr <= 8``,
    ``dim <= 256`` with one constraint and ``dim <= 128`` with several, at most 7 params (the
    last slot carries the density's measure).  The Lebesgue density (``dens_wrt_hausdorff=False``)
    and ``GaussianDenseConstrainedEuclideanMetricSystem`` need ``mhp_constr``."""

    target_id = TARGET_USER

    def __init__(self, dim, source, params=(), aux=None, name=None, *, n_constr=0,
                 mhp_constr=False):
        if not isinstance(source, str):
            raise ValueError("`source` must be a string of CUDA C++.")
        dim = int(dim)
        if not 1 <= dim <= 1024:
            raise ValueError(f"CudaTarget dimension must be in [1, 1024], got {dim}.")
        try:
            params = tuple(float(x) for x in params)
        except (TypeError, ValueError) as e:
            raise ValueError(f"`params` must be an iterable of scalars: {e}") from e
        if len(params) > 8:
            raise ValueError(f"CudaTarget takes at most 8 params, got {len(params)}.")
        if (isinstance(n_constr, bool) or not isinstance(n_constr, (int, np.integer))
                or not 0 <= n_constr <= 8):
            raise ValueError(f"`n_constr` must be an integer in [0, 8], got {n_constr!r}.")
        n_constr = int(n_constr)
        if n_constr:
            max_dim = 256 if n_constr == 1 else 128
            if dim > max_dim:
                raise ValueError(f"A CudaTarget with {n_constr} constraint(s) needs dim <= "
                                 f"{max_dim}, got {dim}.")
            if len(params) > 7:
                raise ValueError("A constrained CudaTarget takes at most 7 params (the last slot "
                                 f"carries the density's measure), got {len(params)}.")
        if aux is not None:
            try:
                aux = np.ascontiguousarray(aux, dtype=np.float64)
            except (TypeError, ValueError) as e:
                raise ValueError(f"`aux` cannot be converted to a float64 array: {e}") from e
        super().__init__(dim, params, aux)
        self.source = source
        self.name = "user_target" if name is None else str(name)
        if not self.name.isidentifier():
            raise ValueError("`name` must be a valid identifier.")
        self.n_constr = n_constr
        self.mhp_constr = bool(mhp_constr) and n_constr > 0

    def _image_kwargs(self):
        """What the image depends on besides the source: constraint count, KP, mhp_constr."""
        if not self.n_constr:
            return {}
        from . import jit  # noqa: PLC0415

        return {"n_constr": self.n_constr, "kp": jit.constrained_kp(self.dim, self.n_constr),
                "mhp_constr": self.mhp_constr}

    def compile(self):
        """Compile now (raises ``mici_b200.errors.TargetCompileError``); returns ``self``."""
        from . import jit  # noqa: PLC0415

        jit.compile_target(self.source, self.name, **self._image_kwargs())
        return self

    def handle(self):
        """The loaded device image (``mb200_user_target_load``, or
        ``mb200_user_constraint_load`` when constrained) of this source, from the process
        cache."""
        from . import jit  # noqa: PLC0415

        return jit.load_target(self.source, self.name, **self._image_kwargs())

    def __repr__(self):
        extra = f", n_constr={self.n_constr}" if self.n_constr else ""
        return f"CudaTarget(dim={self.dim}, name={self.name!r}, params={self.params}{extra})"


class _CudaMetric:
    """A user-written diagonal, scalar, dense or Cholesky-factored metric (contract:
    ``mici_b200/csrc/user_riemannian.cuh``):
    CUDA C++ source, at most 8 ``params`` (``c.params`` inside the metric functions) and an
    optional ``aux`` array (``c.aux``).  It runs with a ``CudaTarget`` only, compiled with it into
    one image; like the target it holds only source, params and aux."""

    kind = ""
    rmetric_id = -1

    def __init__(self, source, params=(), aux=None, name=None):
        if not isinstance(source, str):
            raise ValueError("`source` must be a string of CUDA C++.")
        try:
            params = tuple(float(x) for x in params)
        except (TypeError, ValueError) as e:
            raise ValueError(f"`params` must be an iterable of scalars: {e}") from e
        if len(params) > 8:
            raise ValueError(f"{type(self).__name__} takes at most 8 params, got {len(params)}.")
        if aux is not None:
            try:
                aux = np.ascontiguousarray(aux, dtype=np.float64)
            except (TypeError, ValueError) as e:
                raise ValueError(f"`aux` cannot be converted to a float64 array: {e}") from e
        self.source = source
        self.params = params
        self.aux = aux
        self.name = "user_metric" if name is None else str(name)
        if not self.name.isidentifier():
            raise ValueError("`name` must be a valid identifier.")

    def __repr__(self):
        return f"{type(self).__name__}(name={self.name!r}, params={self.params})"


class CudaDiagonalMetric(_CudaMetric):
    """A user-written diagonal metric M(q) = diag(d(q)) for ``DiagonalRiemannianMetricSystem``:
    CUDA C++ source defining

        __device__ void metric_diagonal(const mb200::Chain& c, double* d);
        __device__ void vjp_metric_diagonal(const mb200::Chain& c, const double* w, double* out);

    with ``out[j] = sum_i w[i] dd_i/dq_j``."""

    kind = "diagonal"
    rmetric_id = RMETRIC_USER_DIAGONAL


class CudaScalarMetric(_CudaMetric):
    """A user-written scalar metric M(q) = s(q) I for ``ScalarRiemannianMetricSystem``: CUDA C++
    source defining

        __device__ double metric_scalar(const mb200::Chain& c);
        __device__ void vjp_metric_scalar(const mb200::Chain& c, double w, double* out);

    with ``out[j] = w ds/dq_j``."""

    kind = "scalar"
    rmetric_id = RMETRIC_USER_SCALAR


class CudaDenseMetric(_CudaMetric):
    """A user-written dense metric M(q), positive definite, for ``DenseRiemannianMetricSystem``:
    CUDA C++ source defining

        __device__ void metric_dense(const mb200::CtaChain& c, double* M, int ld);
        __device__ void vjp_metric_dense(const mb200::CtaChain& c, const double* V, int ld,
                                         double* out);

    with ``M[i * ld + j] = M_ij(q)`` for all ``i, j < dim`` and ``out[k] = sum_ij V[i * ld + j]
    dM_ij/dq_k`` for a symmetric ``V``, every ``out[k], k < dim`` written.  Both functions are
    called by the whole 256-thread CTA of the chain (``c.lane`` in ``[0, c.n_lanes)``, ``c.sum()``
    a CTA all-reduce), not by one warp; the target keeps its warp contract.  Every entry of the
    matrix must be finite and only its lower triangle is factored, as ``numpy.linalg.cholesky``
    does; a failure is a ``LinAlgError`` outside a fixed-point solve and a ``ConvergenceError``
    inside one.  ``dim <= 576``.  Contract: ``mici_b200/csrc/user_riemannian.cuh``."""

    kind = "dense"
    rmetric_id = RMETRIC_USER_DENSE


class CudaCholeskyMetric(_CudaMetric):
    """A user-written metric M(q) = L(q) L(q)^T given by its lower-triangular factor, for
    ``CholeskyFactoredRiemannianMetricSystem``: CUDA C++ source defining

        __device__ void metric_chol(const mb200::CtaChain& c, double* L, int ld);
        __device__ void vjp_metric_chol(const mb200::CtaChain& c, const double* V, int ld,
                                        double* out);

    with ``L[i * ld + j] = L_ij(q)`` for ``0 <= j <= i < dim`` (the upper triangle is never read)
    and ``out[k] = sum_{j <= i} V[i * ld + j] dL_ij/dq_k``, every ``out[k], k < dim`` written, for
    a lower-triangular ``V`` whose entries above the diagonal must not be read.  These are the
    reference's ``metric_chol_func`` and ``vjp_metric_chol_func(q)(V)``.  Both functions are
    called by the whole 256-thread CTA of the chain (``c.lane`` in ``[0, c.n_lanes)``,
    ``c.sum()`` a CTA all-reduce), as for ``CudaDenseMetric``; the target keeps its warp contract.
    No factorisation: O(D^2) per metric.  A non-finite entry of the lower triangle is a
    ``LinAlgError`` outside a fixed-point solve and a ``ConvergenceError`` inside one; a negative
    diagonal entry is legal; a zero one fails only where ``L`` is solved with.  ``dim <= 1016``.
    Contract: ``mici_b200/csrc/user_riemannian.cuh``."""

    kind = "cholesky"
    rmetric_id = RMETRIC_USER_CHOLESKY


class CudaRiemannianPair:
    """A ``CudaTarget`` with a user metric: what a Riemannian system with a user metric runs,
    compiled into one image (``mb200_user_riemannian_load``)."""

    def __init__(self, target, metric):
        self.target, self.metric = target, metric

    def _metric_key(self):
        return (self.metric.kind, self.metric.source, self.metric.name)

    def compile(self):
        """Compile now (raises ``mici_b200.errors.TargetCompileError``); returns ``self``."""
        from . import jit  # noqa: PLC0415

        jit.compile_target(self.target.source, self.target.name, metric=self._metric_key())
        return self

    def handle(self):
        """The loaded device image of this pair, from the process cache."""
        from . import jit  # noqa: PLC0415

        return jit.load_target(self.target.source, self.target.name, metric=self._metric_key())


def user_handle(target):
    """The loaded image of a ``CudaTarget`` or of a ``CudaRiemannianPair``, or ``None`` for a
    registry target."""
    return target.handle() if isinstance(target, (CudaTarget, CudaRiemannianPair)) else None


class Rank1Metric:
    """Position-dependent dense metric M(q) = B + c q q^T."""

    rmetric_id = RMETRIC_RANK1
    name = "rank1"

    def __init__(self, base, coeff, force_low_rank_form=False, generic_rank1_vjp=False):
        """``force_low_rank_form``: evaluate the metric through the Sherman-Morrison identities
        against the shared explicit ``B^-1`` (O(D^2) per metric, never factorises) instead of the
        reference's per-chain Cholesky path -- an OPTIONAL policy; by default the metric is
        factorised per chain exactly as a generic dense metric.  ``generic_rank1_vjp``: form
        ``-(M^-1 p)(M^-1 p)^T`` explicitly and hand it to the dense VJP (matrices.py:1179-1181)
        instead of using the model's rank-one VJP."""
        base = np.ascontiguousarray(base, dtype=np.float64)
        # shared explicit inverse and log-determinant of B, built once on the host the way the
        # reference builds a fixed dense metric's inverse (matrices.py:1161-1188, 982-984)
        import scipy.linalg as sla  # noqa: PLC0415

        chol = np.linalg.cholesky(base)
        inv_lt = sla.solve_triangular(chol.T, np.identity(base.shape[0]), lower=False)
        inv = sla.solve_triangular(chol.T, inv_lt.T, lower=False)
        self.base = base
        self.aux = np.ascontiguousarray(np.concatenate([base.ravel(), inv.ravel()]))
        self.params = (
            float(coeff),
            float(2.0 * np.log(np.abs(chol.diagonal())).sum()),
            1.0 if force_low_rank_form else 0.0,
            1.0 if generic_rank1_vjp else 0.0,
        )


class HadamardMetric:
    """Position-dependent dense metric M(q) = B + c (q q^T) o S, B and S symmetric positive
    definite: a full-rank perturbation of B (Schur product theorem keeps it SPD), so only the
    generic dense path -- per-chain Cholesky, explicit inverse, dense VJP -- applies."""

    rmetric_id = RMETRIC_HADAMARD
    name = "hadamard"

    def __init__(self, base, scale, coeff, generic_rank1_vjp=False):
        base = np.ascontiguousarray(base, dtype=np.float64)
        scale = np.ascontiguousarray(scale, dtype=np.float64)
        if base.shape != scale.shape or base.ndim != 2 or base.shape[0] != base.shape[1]:
            raise ValueError("`base` and `scale` must be square matrices of the same shape.")
        self.base, self.scale = base, scale
        self.aux = np.ascontiguousarray(np.concatenate([base.ravel(), scale.ravel()]))
        self.params = (float(coeff), 0.0, 0.0, 1.0 if generic_rank1_vjp else 0.0)


class QuadraticDiagonalMetric:
    """Position-dependent diagonal metric d_i(q) = a + b q_i^2 (``a > 0``, ``b >= 0``); with
    ``a = b = 1`` the metric ``1 + q**2`` of the reference's own integrator tests."""

    rmetric_id = RMETRIC_DIAG_QUADRATIC
    name = "diag_quadratic"
    aux = None

    def __init__(self, a=1.0, b=1.0):
        a, b = float(a), float(b)
        if not (a > 0 and b >= 0):
            raise ValueError("QuadraticDiagonalMetric needs a > 0 and b >= 0.")
        self.a, self.b = a, b
        self.params = (a, b)


class FunnelFisherMetric:
    """Diagonal metric of the funnel (``NealFunnel``): its expected Fisher information
    d(q) = [1/9 + (D-1)/2, e^-v, ..., e^-v] with v = q[0]."""

    rmetric_id = RMETRIC_DIAG_FUNNEL_FISHER
    name = "funnel_fisher"
    aux = None
    params = ()


class QuadraticScalarMetric:
    """Position-dependent scaled-identity metric s(q) I with s = a + b |q|^2 (``a > 0``,
    ``b >= 0``)."""

    rmetric_id = RMETRIC_SCALAR_QUADRATIC
    name = "scalar_quadratic"
    aux = None

    def __init__(self, a=1.0, b=1.0):
        a, b = float(a), float(b)
        if not (a > 0 and b >= 0):
            raise ValueError("QuadraticScalarMetric needs a > 0 and b >= 0.")
        self.a, self.b = a, b
        self.params = (a, b)


class QuadraticCholeskyMetric:
    """Position-dependent metric M(q) = L(q) L(q)^T given by its lower-triangular factor
    L(q) = L0 + c tril(q q^T) (``CholeskyFactoredRiemannianMetricSystem``).  Only the lower
    triangle of ``base_factor`` is used: its upper triangle is zeroed, as the reference does for
    every factor it is given.

    M(q) is positive definite wherever every diagonal entry L_ii(q) = (L0)_ii + c q_i^2 is
    non-zero; ``coeff >= 0`` with a positive diagonal of ``L0`` guarantees that at every finite
    q.  Any finite square ``L0`` and finite ``coeff`` are accepted, so that factors with
    negative or vanishing diagonal entries behave as in the reference: a negative entry is
    legal (only |L_ii| enters log|M|), a zero one fails wherever the metric is solved with."""

    rmetric_id = RMETRIC_CHOL_QUADRATIC
    name = "chol_quadratic"

    def __init__(self, base_factor, coeff):
        base = np.asarray(base_factor, dtype=np.float64)
        coeff = float(coeff)
        if base.ndim != 2 or base.shape[0] != base.shape[1]:
            raise ValueError("`base_factor` must be a square matrix.")
        if not np.all(np.isfinite(base)) or not np.isfinite(coeff):
            raise ValueError("`base_factor` and `coeff` must be finite.")
        self.base_factor = np.ascontiguousarray(np.tril(base))
        self.coeff = coeff
        self.dim = base.shape[0]
        self.aux = self.base_factor
        self.params = (coeff,)


REGISTRY = {
    cls.name: cls
    for cls in (StdGaussian, NealFunnel, Banana, Quadratic, Quartic, Torus, Sphere, MultiSphere)
}
METRIC_REGISTRY = {
    cls.name: cls
    for cls in (Rank1Metric, HadamardMetric, QuadraticDiagonalMetric, FunnelFisherMetric,
                QuadraticScalarMetric, QuadraticCholeskyMetric)
}


def make_target(name, **params):
    return REGISTRY[name](**params)


def make_metric_model(name, **params):
    return METRIC_REGISTRY[name](**params)
