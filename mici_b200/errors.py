"""Exception types -- same names and hierarchy as the reference (``src/mici/errors.py:6-35``)
so that callers catching ``IntegratorError`` (transitions.py:292, 670; adapters.py:338) work
unchanged.  If the reference package itself is importable its classes are re-used, so that
``except mici.errors.IntegratorError`` in reference code catches errors raised here."""

from __future__ import annotations

try:  # pragma: no cover - depends on environment
    from mici.errors import (  # type: ignore[import-not-found]
        AdaptationError,
        ConvergenceError,
        Error,
        HamiltonianDivergenceError,
        IntegratorError,
        LinAlgError,
        NonReversibleStepError,
        ReadOnlyStateError,
    )
except ImportError:

    class Error(RuntimeError):
        """Base class for errors."""

    class IntegratorError(Error):
        """Error raised when integrator step fails."""

    class NonReversibleStepError(IntegratorError):
        """Error raised when integrator step fails reversibility check."""

    class ConvergenceError(IntegratorError):
        """Error raised when solver fails to converge within allowed iterations."""

    class LinAlgError(Error):
        """Error raised when a matrix operation raises a linear algebra error."""

    class HamiltonianDivergenceError(IntegratorError):
        """Error raised when integration of Hamiltonian dynamics diverges."""

    class AdaptationError(Error):
        """Error raised when adaptation of transition parameters fails."""

    class ReadOnlyStateError(Error):
        """Error raised when writing to attributes of read-only chain state."""


class ExtensionNotBuiltError(Error):
    """libmici_b200.so is missing or cannot be loaded: there is no CPU fallback."""


class TargetCompileError(Error):
    """A user-written target (``mici_b200.targets.CudaTarget``) does not compile; ``log`` holds
    the NVRTC log, whose line numbers are the user source's."""

    def __init__(self, msg, log=""):
        super().__init__(msg)
        self.log = log


# per-chain status codes written by the kernels (include/mici_b200.h)
STATUS_OK = 0
STATUS_CONVERGENCE = 1
STATUS_NON_REVERSIBLE = 2
STATUS_LINALG = 3

STATUS_TO_ERROR = {
    STATUS_CONVERGENCE: ConvergenceError,
    STATUS_NON_REVERSIBLE: NonReversibleStepError,
    STATUS_LINALG: LinAlgError,
}


_DUAL = {}


def compatible(exc):
    """``exc`` itself, or -- when the reference package was imported AFTER this module, so that
    the classes above are this package's own -- a subclass of both ``exc`` and the reference's
    class of the same name: ``except mici.errors.IntegratorError`` in reference code
    (transitions.py:292, 670; adapters.py:338) and ``except mici_b200.errors.IntegratorError``
    both catch it."""
    import sys  # noqa: PLC0415

    ref_mod = sys.modules.get("mici.errors")
    ref = getattr(ref_mod, exc.__name__, None) if ref_mod is not None else None
    if ref is None or issubclass(exc, ref):
        return exc
    key = (exc, ref)
    if key not in _DUAL:
        _DUAL[key] = type(exc.__name__, (exc, ref), {})
    return _DUAL[key]


def raise_for_status(code: int, what: str = "integrator step") -> None:
    """Raise the reference exception matching a per-chain status code (single-chain shim)."""
    if code == STATUS_OK:
        return
    exc = compatible(STATUS_TO_ERROR.get(int(code), IntegratorError))
    raise exc(f"{what} failed with status {int(code)} ({exc.__name__}).")
