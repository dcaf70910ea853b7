"""ctypes binding of the C-ABI in ``include/b200mol.h`` (``nvmolkit_b200/lib/libb200mol.so``).

There is no CPU fallback: if the CUDA library is missing, or a call fails, this module raises.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200mol.so")

B200MOL_OK, ERR_INVALID, ERR_CUDA, ERR_NODEVICE = 0, 1, 2, 3
METRIC = {"tanimoto": 0, "cosine": 1}

_u32p = C.c_void_p  # device/host pointers travel as integers
_vp = C.c_void_p

# name -> (restype, argtypes); must list every symbol include/b200mol.h declares (tests/test_abi.py checks this).
SIGNATURES = {
    "b200mol_last_error": (C.c_char_p, []),
    "b200mol_abi_version": (C.c_int, []),
    "b200mol_launch_count": (C.c_uint64, []),
    "b200mol_check_device": (C.c_int, [C.c_int]),
    "b200mol_free_async": (C.c_int, [_vp, _vp]),
    "b200mol_set_option": (C.c_int, [C.c_char_p, C.c_longlong]),
    "b200mol_get_option": (C.c_int, [C.c_char_p, C.POINTER(C.c_longlong)]),
    "b200mol_profile_enable": (C.c_int, [C.c_int]),
    "b200mol_profile_read": (C.c_int, [C.c_char_p, C.POINTER(C.c_float)]),
    "b200mol_stats_read": (C.c_int, [_vp, C.c_int, _vp]),
    "b200mol_tanimoto_cross": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, _vp, _vp]),
    "b200mol_cosine_cross": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, _vp, _vp]),
    "b200mol_similarity_cross_host": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_int, _vp, C.c_size_t]),
    "b200mol_tanimoto_count_ge": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_int, C.c_double, C.c_int,
                                            _vp, _vp]),
    "b200mol_similarity_topk": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    "b200mol_similarity_threshold": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_int, C.c_double, _vp, _vp,
                                               _vp, C.c_uint64, C.POINTER(C.c_uint64), _vp]),
    "b200mol_tversky_cross": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_double, C.c_double, _vp, _vp]),
    "b200mol_tversky_cross_host": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_double, C.c_double, _vp,
                                             C.c_size_t]),
    "b200mol_tversky_topk": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_double, C.c_double, C.c_int, _vp,
                                       _vp, _vp]),
    "b200mol_tversky_threshold": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_double, C.c_double,
                                            C.c_double, _vp, _vp, _vp, C.c_uint64, C.POINTER(C.c_uint64), _vp]),
    "b200mol_count_cross": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_double, C.c_double, _vp, _vp]),
    "b200mol_count_topk": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_double, C.c_double, C.c_int, _vp,
                                     _vp, _vp]),
    "b200mol_count_threshold": (C.c_int, [_vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_double, C.c_double,
                                          C.c_double, _vp, _vp, _vp, C.c_uint64, C.POINTER(C.c_uint64), _vp]),
    "b200mol_count_neighbor_edges": (C.c_int, [_vp, C.c_size_t, C.c_int, C.c_double, C.c_double, C.c_double, _vp, _vp,
                                               C.c_uint64, C.POINTER(C.c_uint64), _vp]),
    "b200mol_count_butina_fused": (C.c_int, [_vp, C.c_size_t, C.c_int, C.c_double, C.c_double, C.c_double, _vp, _vp, _vp,
                                             _vp, _vp]),
    "b200mol_maxmin_pick": (C.c_int, [_vp, C.c_size_t, C.c_int, C.c_int, _vp, C.c_int, C.c_int, C.c_double, _vp, _vp,
                                      _vp]),
    "b200mol_leader_pick": (C.c_int, [_vp, C.c_size_t, C.c_int, C.c_int, C.c_double, _vp, C.c_int, C.c_int, _vp, _vp,
                                      _vp]),
    "b200mol_butina_fused": (C.c_int, [_vp, C.c_size_t, C.c_int, C.c_int, C.c_double, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_neighbor_edges": (C.c_int, [_vp, C.c_size_t, C.c_int, C.c_int, C.c_double, C.c_uint32, C.c_uint32, _vp,
                                         _vp, C.c_uint64, C.POINTER(C.c_uint64), _vp]),
    "b200mol_butina_from_edges": (C.c_int, [C.c_size_t, _vp, _vp, C.c_uint64, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_butina_dense": (C.c_int, [_vp, C.c_size_t, C.c_double, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_mmff_energy_grad": (C.c_int, [_vp, C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_uff_energy_grad": (C.c_int, [_vp, C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_uff_minimize": (C.c_int, [_vp, C.c_int32, _vp, _vp, C.c_int, _vp, C.c_int, C.c_double, _vp, _vp, _vp, _vp,
                                       _vp]),
    "b200mol_dg_energy_grad": (C.c_int, [_vp, C.c_int, C.c_double, C.c_double, C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_etk_energy_grad": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_mmff_minimize": (C.c_int, [_vp, C.c_int32, _vp, _vp, C.c_int, _vp, C.c_int, C.c_double, _vp, _vp, _vp, _vp,
                                        _vp]),
    "b200mol_dg_minimize": (C.c_int, [_vp, C.c_int, C.c_double, C.c_double, C.c_int32, _vp, _vp, C.c_int, _vp, C.c_int,
                                      C.c_double, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_etk_minimize": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int32, _vp, _vp, C.c_int, _vp, C.c_int, C.c_double, _vp, _vp,
                                       _vp, _vp, _vp]),
    "b200mol_poly_minimize": (C.c_int, [C.c_int32, _vp, C.c_int, C.c_int, _vp, _vp, _vp, C.c_int, C.c_double, C.c_int,
                                        C.c_int, _vp, _vp, _vp, _vp]),
    "b200mol_etkdg_embed": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int32, _vp, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_etkdg_initial_coords": (C.c_int, [_vp, _vp, C.c_int32, _vp, _vp, C.c_int, C.c_int32, _vp, _vp, _vp]),
    "b200mol_etkdg_check": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int32, _vp, _vp, C.c_int, _vp, _vp, _vp]),
    "b200mol_triangle_smooth": (C.c_int, [_vp, _vp, C.c_int32, C.c_double, _vp, _vp]),
    "b200mol_eig_topk": (C.c_int, [_vp, _vp, C.c_int32, C.c_int, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_metric_embed": (C.c_int, [_vp, _vp, _vp, C.c_int32, C.c_int, _vp, _vp, C.c_uint32, _vp, _vp, _vp]),
    "b200mol_schedule_waves": (C.c_int, [C.c_int32, _vp, _vp, C.c_int, _vp, _vp, _vp, C.POINTER(C.c_int64)]),
    "b200mol_dg_terms_from_bounds": (C.c_int, [C.c_int32, _vp, C.c_int32, _vp, _vp, C.c_int, C.c_double, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_etk_terms_from_details": (C.c_int, [C.c_int32, _vp, _vp, C.c_int, _vp, _vp, _vp]),
    "b200mol_allgather_counts": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, _vp, _vp]),
    "b200mol_allgather_results": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_rms_prune": (C.c_int, [C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp, C.c_double, _vp, _vp, _vp]),
    "b200mol_tfd_matrices": (C.c_int, [C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200mol_conformer_rmsd": (C.c_int, [C.c_int32, _vp, _vp, _vp, _vp, _vp, C.c_int32, _vp, _vp]),
    "b200mol_conformer_rmsd_mapped": (C.c_int, [C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int32, _vp,
                                                _vp]),
    "b200mol_align": (C.c_int, [C.c_int32, _vp, _vp, _vp, C.c_int32, _vp, _vp, _vp, C.c_int32, _vp, _vp, _vp, C.c_int32,
                                C.c_int32, C.c_int32, _vp, _vp, _vp]),
    "b200mol_best_align": (C.c_int, [C.c_int32, _vp, _vp, _vp, C.c_int32, _vp, _vp, _vp, C.c_int32, _vp, _vp, _vp, _vp,
                                     _vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _vp, _vp, _vp, _vp]),
    "b200mol_morgan": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, _vp,
                                 _vp]),
    "b200mol_morgan_counts": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int,
                                        _vp, _vp]),
}

_lib = None


class B200MolError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load libb200mol.so (once). Raises ImportError when it has not been built — there is no fallback path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). nvmolkit_b200 has no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(status: int) -> None:
    """Translate a C-ABI status into the exception types the reference's bindings raise."""
    if status == B200MOL_OK:
        return
    msg = load().b200mol_last_error().decode("utf-8", "replace")
    if status == ERR_INVALID:
        raise ValueError(msg)
    raise B200MolError(msg)


_core = None
_core_tried = False


def core():
    """The pybind11 host module nvmolkit_b200._core (C++ glue over the same C-ABI, built by `make pymodule`): native calls
    go through it so that the GIL is released while a kernel launch / synchronisation is in progress. None when it has not
    been built (the ctypes binding below then makes the calls itself, holding the GIL like the reference does)."""
    global _core, _core_tried
    if not _core_tried:
        _core_tried = True
        if os.environ.get("B200_NO_CORE"):  # (the instrumented builds of tools/ are separate .so files bound through ctypes)
            return None
        try:
            from nvmolkit_b200 import _core as mod  # noqa: PLC0415

            if mod.abi_version() == load().b200mol_abi_version():
                _core = mod
        except ImportError:
            _core = None
    return _core


def _plain(a):
    """ctypes argument -> what the pybind11 signatures take (addresses as integers)."""
    if a is None:
        return 0
    if isinstance(a, (int, float, str)):
        return a
    if isinstance(a, bytes):
        return a.decode()
    if isinstance(a, C._SimpleCData):
        return a.value or 0
    if hasattr(a, "_obj"):  # ctypes.byref(x)
        return C.addressof(a._obj)
    if isinstance(a, (C.Structure, C.Array)):
        return C.addressof(a)
    raise TypeError(f"cannot pass {type(a).__name__} to the native library")


def call(name: str, *args) -> None:
    mod = core()
    if mod is not None and hasattr(mod, name):
        try:
            getattr(mod, name)(*[_plain(a) for a in args])
        except mod.B200MolError as e:
            raise B200MolError(str(e)) from None
        return
    check(getattr(load(), name)(*args))


def launch_count() -> int:
    return int(load().b200mol_launch_count())


def profile_enable(on: bool) -> None:
    check(load().b200mol_profile_enable(1 if on else 0))


def profile_read(phase: str) -> float:
    ms = C.c_float(0.0)
    check(load().b200mol_profile_read(phase.encode(), C.byref(ms)))
    return float(ms.value)


def get_option(key: str) -> int:
    v = C.c_longlong(0)
    check(load().b200mol_get_option(key.encode(), C.byref(v)))
    return int(v.value)


def stats_read(reset: bool = True) -> dict:
    """Work counters of the conformer kernels on the current device (include/b200mol.h b200mol_stats_read)."""
    out = (C.c_uint64 * 16)()
    check(load().b200mol_stats_read(C.cast(out, C.c_void_p), 1 if reset else 0, None))
    keys = ("bfgs_iterations", "energy_evals", "gradient_evals", "algorithmic_bytes", "minimisations", "etkdg_attempts",
            "n2_iterations")
    return {bank: {k: int(out[8 * b + i]) for i, k in enumerate(keys)} for b, bank in enumerate(("embed", "minimize"))}


def set_option(key: str, value: int) -> None:
    check(load().b200mol_set_option(key.encode(), int(value)))


@contextlib.contextmanager
def options(**values):
    """Set library options for the body of a ``with`` block, then put back the values they had, also on an exception."""
    saved = {}
    try:
        for key, value in values.items():
            saved[key] = get_option(key)
            set_option(key, value)
        yield
    finally:
        for key, value in reversed(saved.items()):
            set_option(key, value)
