"""ctypes binding of ``libmici_b200.so`` (C ABI: ``include/mici_b200.h``).

The handle is held at module level and looked up lazily, never stored on system / integrator
objects, so those survive ``copy.deepcopy`` / pickling exactly like the reference's
(samplers.py:1124-1129 deep-copies the integrator per chain).  There is NO fallback: if the
shared library is missing every call raises ``ExtensionNotBuiltError``.
"""

from __future__ import annotations

import ctypes
import os
import threading

from .errors import Error, ExtensionNotBuiltError

MAX_PARAMS = 8
LIB_NAME = "libmici_b200.so"
# MICI_B200_LIB lets profiling experiments load an alternative build of the same C ABI
LIB_PATH = os.environ.get(
    "MICI_B200_LIB", os.path.join(os.path.dirname(os.path.abspath(__file__)), LIB_NAME)
)

c_double_p = ctypes.c_void_p  # device pointers travel as integers
c_int32_p = ctypes.c_void_p


class NutsOptions(ctypes.Structure):
    """``struct mb200_nuts_options``."""

    _fields_ = [
        ("max_tree_depth", ctypes.c_int32),
        ("slice_variant", ctypes.c_int32),
        ("euclidean_criterion", ctypes.c_int32),
        ("extra_subtree_checks", ctypes.c_int32),
        ("max_delta_h", ctypes.c_double),
        ("uniforms", ctypes.c_void_p),
        ("n_uniforms", ctypes.c_int32),
    ]


class Model(ctypes.Structure):
    """``struct mb200_model``."""

    _fields_ = [
        ("target_id", ctypes.c_int32),
        ("n_target_params", ctypes.c_int32),
        ("target_params", ctypes.c_double * MAX_PARAMS),
        ("target_aux", ctypes.c_void_p),
        ("rmetric_id", ctypes.c_int32),
        ("n_rmetric_params", ctypes.c_int32),
        ("rmetric_params", ctypes.c_double * MAX_PARAMS),
        ("rmetric_aux", ctypes.c_void_p),
    ]


_I64, _I32, _F64, _P = ctypes.c_int64, ctypes.c_int32, ctypes.c_double, ctypes.c_void_p
_MP = ctypes.POINTER(Model)
_NP = ctypes.POINTER(NutsOptions)

# mb200_leapfrog_euclidean and its general-kernel twin
_LEAPFROG_EUCLIDEAN_ARGS = [_P, _P, _P, _P, _P, _I64, _I32, _F64, _P, _I32, _P, _I32, _P, _I32, _I32,
                            _P, _MP, _P, _P, _P, _P]
# mb200_constrained_leapfrog[_gaussian]_euclidean: the Gaussian system's three rotation operands
# follow metric_inv
_CONSTRAINED_HEAD = [_P, _P, _P, _P, _P, _I64, _I32, _F64, _P, _I32, _P, _I32, _I32, _P]
_CONSTRAINED_TAIL = [_MP, _I32, _F64, _F64, _F64, _I32, _I32, _F64, _P, _P, _P, _P, _P]
_PROJECT_ARGS = [_P, _P, _P, _I64, _I32, _I32, _P, _MP, _P]

# symbol -> (restype, argtypes): every symbol declared in include/mici_b200.h
SIGNATURES = {
    "mb200_version": (ctypes.c_int, []),
    "mb200_last_error": (ctypes.c_char_p, []),
    "mb200_set_call_counters": (ctypes.c_int, [_P]),
    "mb200_leapfrog_euclidean": (ctypes.c_int, _LEAPFROG_EUCLIDEAN_ARGS),
    "mb200_leapfrog_euclidean_generic": (ctypes.c_int, _LEAPFROG_EUCLIDEAN_ARGS),
    "mb200_hamiltonian_euclidean": (ctypes.c_int, [_P, _P, _I64, _I32, _I32, _P, _MP, _P, _P]),
    "mb200_euclidean_eval": (ctypes.c_int, [_P, _P, _I64, _I32, _I32, _P, _MP, _P, _P, _P, _P, _P]),
    "mb200_user_target_load": (ctypes.c_int, [ctypes.c_char_p, _I64, _P, _I32, _P]),
    "mb200_user_target_unload": (ctypes.c_int, [_P]),
    "mb200_constrained_leapfrog_euclidean": (ctypes.c_int, _CONSTRAINED_HEAD + _CONSTRAINED_TAIL),
    "mb200_constrained_leapfrog_gaussian_euclidean": (
        ctypes.c_int, _CONSTRAINED_HEAD + [_P, _P, _P] + _CONSTRAINED_TAIL),
    "mb200_implicit_leapfrog_riemannian": (
        ctypes.c_int,
        [_P, _P, _P, _P, _P, _I64, _I32, _F64, _P, _I32, _P, _MP, _I32, _F64, _F64, _I32, _F64]
        + [_P, _P, _P, _P, _P, _I64, _P],
    ),
    "mb200_implicit_workspace_bytes": (_I64, [_I64, _I32, _MP]),
    "mb200_selftest_fixed_point": (
        ctypes.c_int,
        [_I32, _I32, _P, _P, _I64, _I32, _F64, _F64, _I32, _P, _P, _P, _P],
    ),
    "mb200_selftest_eigh": (ctypes.c_int, [_P, _I64, _I32, _I32, _P, _P, _P, _P]),
    "mb200_implicit_midpoint_riemannian": (
        ctypes.c_int,
        [_P, _P, _P, _P, _P, _I64, _I32, _F64, _P, _I32, _P, _MP, _I32, _F64, _F64, _I32, _F64]
        + [_P, _P, _P, _P, _P],
    ),
    "mb200_project_onto_cotangent_space": (ctypes.c_int, _PROJECT_ARGS),
    "mb200_project_onto_cotangent_space_gaussian": (ctypes.c_int, _PROJECT_ARGS),
    "mb200_user_constraint_load": (
        ctypes.c_int, [ctypes.c_char_p, _I64, _P, _I32, _I32, _I32, _I32, _P]),
    "mb200_sample_momentum_riemannian": (ctypes.c_int, [_P, _P, _P, _I64, _I32, _MP, _P, _P]),
    "mb200_dh_dmom_riemannian": (ctypes.c_int, [_P, _P, _P, _I64, _I32, _MP, _P, _P]),
    "mb200_selftest_dense_factor": (ctypes.c_int, [_P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P]),
    "mb200_selftest_exp_short_chain": (ctypes.c_int, [_P, _P, _I64, _P]),
    "mb200_nuts_generic_state_bytes": (ctypes.c_int64, [_I64]),
    "mb200_nuts_generic_begin": (
        ctypes.c_int, [_P, _P, _P, _P, _I64, _I32, _NP, _P, _I64, _P, _I64, _P]),
    "mb200_nuts_generic_start": (
        ctypes.c_int, [_I64, _I32, _I32, _NP, _P, _P, _P, _P, _P, _P, _P]),
    "mb200_nuts_generic_leaf": (
        ctypes.c_int, [_P, _P, _P, _P, _P, _I64, _I32, _I32, _I32, _NP, _P, _P, _P, _P]),
    "mb200_nuts_generic_finish": (ctypes.c_int, [_I64, _I32, _I32, _NP, _P, _P, _P]),
    "mb200_nuts_generic_end": (
        ctypes.c_int, [_I64, _I32, _NP, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "mb200_leapfrog_gaussian_euclidean": (
        ctypes.c_int,
        [_P, _P, _P, _P, _P, _I64, _I32, _F64, _P, _I32, _I32, _P, _I32, _I32, _P, _P, _MP, _P, _P,
         _P, _P],
    ),
    "mb200_nuts_workspace_bytes": (ctypes.c_int64, [_I64, _I32, _I32]),
    "mb200_nuts_euclidean": (
        ctypes.c_int,
        [_P, _P, _P, _P, _I64, _I32, _F64, _P, _I32, _P, _MP, _I32, _I32, _I32, _I32, _F64, _P,
         _I32, _P, _I64, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    ),
    "mb200_host_scratch_bytes": (ctypes.c_int64, [_I64, _I32]),
    "mb200_leapfrog_euclidean_host": (
        ctypes.c_int,
        [_P, _P, _P, _P, _P, _I64, _I32, _F64, _I32, _I32, _P, _MP, _P, _I32, _P, _I32, _P, _I64,
         _I32],
    ),
    "mb200_metropolis_select": (
        ctypes.c_int,
        [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I64, _I32, _P, _P, _P, _P],
    ),
    "mb200_hamiltonian_riemannian": (ctypes.c_int, [_P, _P, _I64, _I32, _MP, _P, _P, _P, _I64, _P]),
    "mb200_user_riemannian_load": (ctypes.c_int, [ctypes.c_char_p, _I64, _P, _I32, _I32, _P]),
}

# each `_user` twin takes its registry entry point's arguments plus the loaded image's handle
for _name in ("mb200_leapfrog_euclidean", "mb200_hamiltonian_euclidean", "mb200_euclidean_eval",
              "mb200_constrained_leapfrog_euclidean",
              "mb200_constrained_leapfrog_gaussian_euclidean",
              "mb200_project_onto_cotangent_space", "mb200_project_onto_cotangent_space_gaussian",
              "mb200_implicit_leapfrog_riemannian", "mb200_implicit_midpoint_riemannian",
              "mb200_hamiltonian_riemannian", "mb200_sample_momentum_riemannian",
              "mb200_dh_dmom_riemannian"):
    SIGNATURES[_name + "_user"] = (SIGNATURES[_name][0], SIGNATURES[_name][1] + [_P])

_lock = threading.Lock()
_lib = None


def load():
    """Return the loaded library (loading it on first use); raise if it has not been built."""
    global _lib  # noqa: PLW0603
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                msg = (
                    f"{LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; "
                    "g.build()'` or `make -C mici_b200/csrc`. mici_b200 has no CPU fallback."
                )
                raise ExtensionNotBuiltError(msg)
            try:
                lib = ctypes.CDLL(LIB_PATH)
            except OSError as e:
                raise ExtensionNotBuiltError(f"cannot load {LIB_PATH}: {e}") from e
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype = res
                fn.argtypes = args
            _lib = lib
    return _lib


def call(entry, *args, target=None):
    """Call the entry point ``entry`` and raise if it fails.  For a user-written ``CudaTarget``,
    or a ``CudaTarget`` paired with a user metric, it calls the ``_user`` twin instead, with the
    loaded image appended."""
    from .targets import user_handle  # noqa: PLC0415

    user = user_handle(target)
    if user is not None:
        entry, args = entry + "_user", (*args, user)
    check(getattr(load(), entry)(*args), entry)


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().mb200_last_error().decode("utf-8", "replace")
        raise Error(f"{what} failed (rc={rc}): {msg}")


def ptr(t):
    """Device pointer of a torch tensor (or None -> NULL)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def current_stream_ptr(device):
    import torch

    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)
