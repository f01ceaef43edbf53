"""Run-time compilation of user-written targets with NVRTC (``targets.CudaTarget``).

A user target is two CUDA device functions (contract: ``csrc/user_target.cuh``).  They are
compiled together with the engine's general-dimension Euclidean kernels
(``csrc/leapfrog_generic.cuh``) into one sm_90a CUBIN, which ``libmici_b200.so`` loads
(``mb200_user_target_load``).  NVRTC is driven through ``ctypes``; it needs no GPU, so compiling
works anywhere.  The library itself never links NVRTC.

Compiled images and loaded handles live in one process-wide cache keyed by a hash of the
headers, the user source, the options and the NVRTC version (nothing is written to disk), so
that system and integrator objects hold only the source and survive ``deepcopy`` / pickling.

A constrained user target (``n_constr >= 1``, contract: ``csrc/user_constraint.cuh``) also
carries the constrained leapfrog and projection kernels (``csrc/constrained.cuh``) for its
constraint count and KP; its cache key covers both and whether the source defines
``mhp_constr``.

A user target paired with a user diagonal, scalar, dense or Cholesky-factored metric (contract:
``csrc/user_riemannian.cuh``) compiles into an image of its own: the implicit-integrator, velocity
and momentum-refresh kernels of ``csrc/riemannian.cuh`` for that (target, metric) pair -- on the
global-workspace dense policy of ``csrc/dense_global.cuh`` for a dense metric -- keyed on both
sources and the metric kind.
"""

from __future__ import annotations

import ctypes
import glob
import hashlib
import os
import threading

from .errors import Error, TargetCompileError
from .targets import (
    RMETRIC_USER_CHOLESKY,
    RMETRIC_USER_DENSE,
    RMETRIC_USER_DIAGONAL,
    RMETRIC_USER_SCALAR,
)

_PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_PKG, "csrc")
INCLUDE = os.path.join(os.path.dirname(_PKG), "include")
ARCH = "sm_90a"
# -fmad=false as the library (csrc/Makefile): products and sums round as in NumPy.
# -default-device: the C prototypes of include/mici_b200.h become (unused) device declarations.
OPTIONS = ("-arch=" + ARCH, "-std=c++17", "-fmad=false", "-default-device")

# (KP, CPW) of the general-dimension kernel, in the kernel-table order of mb200_user_target_load:
# the order of EU_LAYOUTS in csrc/api_common.cuh, which this list must keep
LAYOUTS = ((1, 4), (2, 4), (4, 2), (8, 1), (16, 1))
NAME_EXPRESSIONS = tuple(
    [f"&mb200::leapfrog_generic_kernel<mb200::UserTarget, {kp}, {cpw}, false>" for kp, cpw in LAYOUTS]
    + [f"&mb200::euclidean_eval_kernel<mb200::UserTarget, {kp}>" for kp, _ in LAYOUTS]
)


def constrained_name_expressions(kp):
    """The kernels a constrained image carries after NAME_EXPRESSIONS, in the kernel-table order
    of ``mb200_user_constraint_load``: leapfrog then projection, each with GAUSS false then true
    (GaussianDenseConstrainedEuclideanMetricSystem)."""
    t = "mb200::UserConstrainedTarget"
    return tuple(f"&mb200::constrained_{k}_kernel<{t}, {kp}, {g}>"
                 for k in ("leapfrog", "project") for g in ("false", "true"))


# The kernels of a Riemannian image, in the kernel-table order of mb200_user_riemannian_load:
# implicit leapfrog / midpoint, velocity, momentum refresh
RIEMANNIAN_KINDS = ("diagonal", "scalar", "dense", "cholesky")
# the rmetric_id a Riemannian image serves, by metric kind
RIEMANNIAN_RMETRIC_IDS = {"diagonal": RMETRIC_USER_DIAGONAL, "scalar": RMETRIC_USER_SCALAR,
                          "dense": RMETRIC_USER_DENSE, "cholesky": RMETRIC_USER_CHOLESKY}
# the metric kinds whose policy runs a 256-thread CTA per chain: the metric functions see the
# whole CTA (mb200::CtaChain), the target's warp functions run on warp 0
CTA_KINDS = ("dense", "cholesky")


def riemannian_name_expressions(kind):
    m = "mb200::User%sMetric" % kind.capitalize()
    # the 256-thread CTA of the dense and Cholesky-factored policies calls the target's warp
    # functions from warp 0 only
    t = "mb200::UserRTargetCta" if kind in CTA_KINDS else "mb200::UserRTarget"
    return tuple(f"&mb200::{k}<{t}, {m}>"
                 for k in ("implicit_leapfrog_kernel", "riemannian_velocity_kernel",
                           "riemannian_sample_momentum_kernel"))


def constrained_kp(dim, n_constr):
    """KP (coordinates per lane / 2) of the constrained kernel for ``dim``, chosen as for the
    registry's sphere and multi-sphere targets; ``None`` outside dim <= 256 (one constraint) or
    dim <= 128 (several)."""
    if dim > (256 if n_constr == 1 else 128):
        return None
    return 1 if dim <= 64 else (2 if dim <= 128 else 4)

_lock = threading.Lock()
_nvrtc = None
_images = {}   # key -> (cubin bytes, lowered names)
_handles = {}  # key -> loaded library handle (ctypes.c_void_p)
# (source, name, constraint, metric) -> key / handle: a repeat lookup, once per launch of a user
# target, is one dict access; the headers are hashed and NVRTC's version read once per process
# (_static_key).  constraint: () for an unconstrained target, else (n_constr, kp, mhp_constr).
# metric: () for a Euclidean image, else (kind, metric source, metric name) of a Riemannian one.
_keys = {}
_loaded = {}
_static = None
stats = {"compiles": 0, "hits": 0}


def _candidates():
    """``libnvrtc.so.12`` locations in search order: the ``nvidia-cuda-nvrtc`` wheel that torch
    depends on, the default loader path, ``$CUDA_HOME/lib64``."""
    out = []
    try:
        import nvidia.cuda_nvrtc as pkg  # noqa: PLC0415

        for d in pkg.__path__:
            out.append(os.path.join(d, "lib", "libnvrtc.so.12"))
    except ImportError:
        out.append("<nvidia.cuda_nvrtc package not installed>")
    out.append("libnvrtc.so.12")
    cuda_home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    out.append(os.path.join(cuda_home, "lib64", "libnvrtc.so.12"))
    return out


def nvrtc():
    """The loaded NVRTC library (``ctypes.CDLL``); its path is ``nvrtc()._name``."""
    global _nvrtc  # noqa: PLW0603
    with _lock:
        if _nvrtc is None:
            tried = []
            for path in _candidates():
                if path.startswith("<"):
                    tried.append(path)
                    continue
                try:
                    lib = ctypes.CDLL(path)
                except OSError as e:
                    tried.append(f"{path}: {e}")
                    continue
                _declare(lib)
                _nvrtc = lib
                break
            else:
                raise Error("cannot load NVRTC (libnvrtc.so.12); tried:\n  " + "\n  ".join(tried))
    return _nvrtc


def _declare(lib):
    p, sz = ctypes.c_void_p, ctypes.c_size_t
    pp = ctypes.POINTER(ctypes.c_void_p)
    sigs = {
        "nvrtcVersion": [ctypes.POINTER(ctypes.c_int)] * 2,
        "nvrtcGetErrorString": [ctypes.c_int],
        "nvrtcCreateProgram": [pp, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, p, p],
        "nvrtcDestroyProgram": [pp],
        "nvrtcAddNameExpression": [p, ctypes.c_char_p],
        "nvrtcCompileProgram": [p, ctypes.c_int, p],
        "nvrtcGetProgramLogSize": [p, ctypes.POINTER(sz)],
        "nvrtcGetProgramLog": [p, ctypes.c_char_p],
        "nvrtcGetCUBINSize": [p, ctypes.POINTER(sz)],
        "nvrtcGetCUBIN": [p, ctypes.c_char_p],
        "nvrtcGetLoweredName": [p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_char_p)],
    }
    for name, args in sigs.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = ctypes.c_char_p if name == "nvrtcGetErrorString" else ctypes.c_int


def version():
    """``(major, minor)`` of the loaded NVRTC."""
    lib = nvrtc()
    major, minor = ctypes.c_int(), ctypes.c_int()
    _ok(lib.nvrtcVersion(ctypes.byref(major), ctypes.byref(minor)), "nvrtcVersion")
    return major.value, minor.value


def _ok(rc, what):
    if rc != 0:
        msg = nvrtc().nvrtcGetErrorString(rc).decode()
        raise Error(f"{what} failed: {msg}")


def _headers_digest():
    h = hashlib.sha256()
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [
            os.path.join(INCLUDE, "mici_b200.h")]:
        with open(path, "rb") as f:
            h.update(os.path.basename(path).encode() + b"\0" + f.read())
    return h.hexdigest()


def translation_unit(source, name="user_target", constraint=(), metric=()):
    """The program NVRTC compiles: the engine header, then the user source with its own line
    numbers (``#line``), so that compile errors point at the user's lines.  A Riemannian image
    adds the metric source, then binds the metric functions on the line after its last one."""
    if metric:
        _, msource, mname = metric
        end = len(msource.splitlines()) + 1
        return (f'#include "user_riemannian.cuh"\n#line 1 "{name}.cu"\n{source}\n'
                f'#line 1 "{mname}.cu"\n{msource}\n#line {end} "{mname}.cu"\n'
                "MB200_USER_METRIC_FUNCTIONS\n")
    header = "user_constraint.cuh" if constraint else "user_target.cuh"
    return f'#include "{header}"\n#line 1 "{name}.cu"\n{source}\n'


def _constraint(n_constr, kp, mhp_constr):
    if not n_constr:
        return ()
    if not 1 <= n_constr <= 8 or kp not in (1, 2, 4):
        raise ValueError(f"bad constrained image: n_constr={n_constr}, kp={kp}")
    return (int(n_constr), int(kp), bool(mhp_constr))


def _metric(metric):
    if not metric:
        return ()
    kind, msource, mname = metric
    if kind not in RIEMANNIAN_KINDS:
        raise ValueError(f"bad Riemannian image: metric kind {kind!r}")
    return (kind, str(msource), str(mname))


def _defines(constraint, metric=()):
    if metric:
        return ("-DMB200_USER_%s_METRIC" % metric[0].upper(),)
    if not constraint:
        return ()
    n_constr, _, mhp = constraint
    return (f"-DMB200_USER_N_CONSTR={n_constr}",) + (("-DMB200_USER_MHP_CONSTR",) if mhp else ())


def _name_expressions(constraint, metric=()):
    if metric:
        return riemannian_name_expressions(metric[0])
    return NAME_EXPRESSIONS + (constrained_name_expressions(constraint[1]) if constraint else ())


def _static_key():
    """The part of every cache key that is fixed for the process: the header contents, the
    options and the NVRTC version."""
    global _static  # noqa: PLW0603
    if _static is None:
        _static = "\0".join([_headers_digest(), *OPTIONS, "%d.%d" % version()])
    return _static


def cache_key(source, name="user_target", constraint=(), metric=()):
    parts = [_static_key(), name, source]
    if constraint:
        parts.append("n_constr=%d kp=%d mhp_constr=%d" % constraint)
    if metric:
        parts += ["riemannian metric=" + metric[0], metric[2], metric[1]]
    return hashlib.sha256("\0".join(parts).encode()).hexdigest()


def compile_target(source, name="user_target", *, n_constr=0, kp=0, mhp_constr=False,
                   metric=None):
    """Compile a user target; returns ``(key, cubin, lowered kernel names)``, from the process
    cache when the same source was compiled before.  ``n_constr >= 1``: a constrained target,
    whose image also carries the constrained kernels at ``kp``.  ``metric = (kind, source,
    name)``, kind ``"diagonal"``, ``"scalar"``, ``"dense"`` or ``"cholesky"``: the Riemannian image of the target
    with that user metric.  Raises ``TargetCompileError`` with the NVRTC log on failure."""
    constraint = _constraint(n_constr, kp, mhp_constr)
    metric = _metric(metric)
    lookup = (source, name, constraint, metric)
    with _lock:
        key = _keys.get(lookup)
        if key is not None:
            stats["hits"] += 1
            return key, *_images[key]
    key = cache_key(source, name, constraint, metric)
    with _lock:
        if key in _images:  # the same program under another (source, name) spelling
            stats["hits"] += 1
            _keys[lookup] = key
            return key, *_images[key]
    cubin, names = _compile(source, name, constraint, **({"metric": metric} if metric else {}))
    with _lock:
        _images.setdefault(key, (cubin, names))
        _keys[lookup] = key
        stats["compiles"] += 1
        return key, *_images[key]


def _compile(source, name, constraint=(), metric=()):
    lib = nvrtc()
    prog = ctypes.c_void_p()
    src = translation_unit(source, name, constraint, metric).encode()
    exprs = _name_expressions(constraint, metric)
    _ok(lib.nvrtcCreateProgram(ctypes.byref(prog), src, f"{name}_tu.cu".encode(), 0, None, None),
        "nvrtcCreateProgram")
    try:
        for expr in exprs:
            _ok(lib.nvrtcAddNameExpression(prog, expr.encode()), "nvrtcAddNameExpression")
        opts = [o.encode() for o in OPTIONS + _defines(constraint, metric)] + [
            f"-I{CSRC}".encode(), f"-I{INCLUDE}".encode()]
        argv = (ctypes.c_char_p * len(opts))(*opts)
        rc = lib.nvrtcCompileProgram(prog, len(opts), ctypes.cast(argv, ctypes.c_void_p))
        log_size = ctypes.c_size_t()
        _ok(lib.nvrtcGetProgramLogSize(prog, ctypes.byref(log_size)), "nvrtcGetProgramLogSize")
        log = ctypes.create_string_buffer(max(log_size.value, 1))
        _ok(lib.nvrtcGetProgramLog(prog, log), "nvrtcGetProgramLog")
        log = log.value.decode("utf-8", "replace")
        if rc != 0:
            err = lib.nvrtcGetErrorString(rc).decode()
            raise TargetCompileError(f"user target {name!r} does not compile ({err}):\n{log}",
                                     log=log)
        size = ctypes.c_size_t()
        _ok(lib.nvrtcGetCUBINSize(prog, ctypes.byref(size)), "nvrtcGetCUBINSize")
        cubin = ctypes.create_string_buffer(size.value)
        _ok(lib.nvrtcGetCUBIN(prog, cubin), "nvrtcGetCUBIN")
        names = []
        for expr in exprs:
            lowered = ctypes.c_char_p()
            _ok(lib.nvrtcGetLoweredName(prog, expr.encode(), ctypes.byref(lowered)),
                "nvrtcGetLoweredName")
            names.append(lowered.value.decode())
        return cubin.raw, tuple(names)
    finally:
        lib.nvrtcDestroyProgram(ctypes.byref(prog))


def load_target(source, name="user_target", *, n_constr=0, kp=0, mhp_constr=False, metric=None):
    """Handle of the loaded image of a user target (``mb200_user_target_load``,
    ``mb200_user_constraint_load`` for a constrained one, ``mb200_user_riemannian_load`` with a
    user metric), compiled and loaded once per process."""
    from . import _lib  # noqa: PLC0415

    constraint = _constraint(n_constr, kp, mhp_constr)
    metric = _metric(metric)
    lookup = (source, name, constraint, metric)
    with _lock:
        handle = _loaded.get(lookup)
    if handle is not None:
        return handle
    key, cubin, names = compile_target(source, name, n_constr=n_constr, kp=kp,
                                       mhp_constr=mhp_constr, metric=metric)
    with _lock:
        handle = _handles.get(key)
        if handle is None:
            arr = (ctypes.c_char_p * len(names))(*[n.encode() for n in names])
            handle = ctypes.c_void_p()
            if metric:
                _lib.call("mb200_user_riemannian_load", cubin, len(cubin), arr, len(names),
                          RIEMANNIAN_RMETRIC_IDS[metric[0]], ctypes.byref(handle))
            elif constraint:
                _lib.call("mb200_user_constraint_load", cubin, len(cubin), arr, len(names),
                          *constraint, ctypes.byref(handle))
            else:
                _lib.call("mb200_user_target_load", cubin, len(cubin), arr, len(names),
                          ctypes.byref(handle))
            _handles[key] = handle
        _loaded[lookup] = handle
    return handle
