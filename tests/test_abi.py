"""CPU tests of the drop-in boundary: the shared library builds/loads without a GPU and exports
exactly the symbols that include/mici_b200.h declares, with matching ctypes signatures."""

import ctypes
import os
import re

import pytest

from mici_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "mici_b200.h")


@pytest.fixture(scope="module")
def handle():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge

        ge.build()
    return ctypes.CDLL(_lib.LIB_PATH)


def declared_functions():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = re.findall(r"\b(mb200_[a-z0-9_]+)\s*\(", text)
    return sorted(set(names))


def test_header_declares_functions():
    names = declared_functions()
    assert "mb200_leapfrog_euclidean" in names
    assert "mb200_implicit_leapfrog_riemannian" in names
    assert "mb200_constrained_leapfrog_euclidean" in names
    assert len(names) >= 9


def test_library_exports_every_declared_symbol(handle):
    for name in declared_functions():
        assert hasattr(handle, name), f"{name} declared in mici_b200.h but not exported"


def test_ctypes_signatures_cover_the_header():
    assert sorted(_lib.SIGNATURES) == declared_functions()


def test_header_argument_counts_match_ctypes():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for name, (_, argtypes) in _lib.SIGNATURES.items():
        m = re.search(name + r"\s*\((.*?)\)\s*;", text, flags=re.S)
        assert m, name
        args = m.group(1).strip()
        n = 0 if args in ("", "void") else len(args.split(","))
        assert n == len(argtypes), (name, n, len(argtypes))


def test_abi_version_and_error_string_without_gpu(handle):
    handle.mb200_version.restype = ctypes.c_int
    assert handle.mb200_version() == 101
    handle.mb200_last_error.restype = ctypes.c_char_p
    assert isinstance(handle.mb200_last_error(), bytes)


def test_model_struct_layout_matches_header():
    # int32 x2, double[8], pointer, int32 x2, double[8], pointer (natural alignment)
    assert ctypes.sizeof(_lib.Model) == 8 + 64 + 8 + 8 + 64 + 8
    assert _lib.Model.target_params.offset == 8
    assert _lib.Model.target_aux.offset == 72
    assert _lib.Model.rmetric_id.offset == 80
    assert _lib.Model.rmetric_params.offset == 88
    assert _lib.Model.rmetric_aux.offset == 152


def test_missing_library_fails_loudly(monkeypatch):
    from mici_b200.errors import ExtensionNotBuiltError

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libmici_b200.so")
    with pytest.raises(ExtensionNotBuiltError):
        _lib.load()
