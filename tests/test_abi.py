"""The C-ABI library loads here (no GPU) and exports every symbol include/b200mol.h declares."""

import os
import re

from nvmolkit_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    names = set()
    for fn in os.listdir(os.path.join(ROOT, "include")):
        if fn.endswith(".h"):
            text = open(os.path.join(ROOT, "include", fn)).read()
            names |= set(re.findall(r"\b(b200mol_[a-z0-9_]+)\s*\(", text))
    return names


def test_every_declared_symbol_is_exported_and_bound(built_lib):
    declared = _declared()
    assert declared, "no declarations found"
    for name in sorted(declared):
        assert hasattr(built_lib, name), f"{name} declared in include/ but not exported"
    assert declared == set(_lib.SIGNATURES), sorted(declared ^ set(_lib.SIGNATURES))


def test_abi_version_and_error_string(built_lib):
    assert built_lib.b200mol_abi_version() >= 1
    assert isinstance(built_lib.b200mol_last_error(), bytes)


def test_no_cpu_fallback_without_device(built_lib):
    import torch

    if torch.cuda.is_available():
        return
    assert built_lib.b200mol_check_device(0) == _lib.ERR_NODEVICE
    assert b"no CPU fallback" in built_lib.b200mol_last_error() or b"sm_90a" in built_lib.b200mol_last_error()


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "nvmolkit_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(import|from)\s+oracle\b", text, re.M), f
                assert "liboracle" not in text, f


def test_pybind_host_module_exports_every_entry_point_and_translates_errors():
    """nvmolkit_b200._core (csrc_py/core.cpp): same names as the C-ABI, GIL released around the call, the reference's
    exception types (ValueError for invalid arguments)."""
    import numpy as np
    import pytest

    from nvmolkit_b200 import _lib

    mod = _lib.core()
    assert mod is not None and mod.abi_version() == _lib.load().b200mol_abi_version()
    skip = {"b200mol_last_error", "b200mol_abi_version", "b200mol_launch_count", "b200mol_profile_read", "b200mol_get_option"}
    for name in _lib.SIGNATURES:
        assert name in skip or hasattr(mod, name), name
    with pytest.raises(ValueError):
        _lib.call("b200mol_set_option", b"no_such_option", 1)
    with pytest.raises(ValueError):  # a host-only entry point with a bad argument, through the module
        _lib.call("b200mol_schedule_waves", 1, None, None, 99, None, None, None, None)
    assert mod.rows_of(np.array([0, 3, 3, 7, 9]), np.array([2, 0, 3, 1])).tolist() == [3, 4, 5, 6, 0, 1, 2, 7, 8]
    assert mod.running_index(np.array([5, 2, 5, 5, 2, 9])).tolist() == [0, 0, 1, 2, 1, 0]
