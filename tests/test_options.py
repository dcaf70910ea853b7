"""The library's options (b200mol_set_option / b200mol_get_option): every key's default, which values a write accepts,
how the two normalising keys store a value, the refusals, the documentation in include/b200mol.h, and option scopes.
Setting and reading a host option touches no CUDA API, so all but the device counters run without a GPU."""

import os
import re
import subprocess
import sys

import pytest

from nvmolkit_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BELOW_2_31 = (1 << 31) - 1

# key -> (default, probes): a probe is (value written, value read back) or (value written, error message it is refused with)
WRITABLE = {
    "similarity_tensor_min_pairs": (1 << 24, [(-5, -5), (0, 0), (123, 123), (1 << 40, 1 << 40), (-(1 << 40), -(1 << 40))]),
    "similarity_tensor_cluster": (1, [(0, 0), (3, 3), (-1, "similarity_tensor_cluster must be 0, 1, 2 or 3"),
                                      (4, "similarity_tensor_cluster must be 0, 1, 2 or 3")]),
    "similarity_superpose": (4, [(1, 1), (2, 2), (4, 4), (0, "similarity_superpose must be 1, 2 or 4"),
                                 (3, "similarity_superpose must be 1, 2 or 4"), (8, "similarity_superpose must be 1, 2 or 4")]),
    "similarity_superpose_cols": (4, [(1, 1), (2, 2), (4, 4), (0, "similarity_superpose_cols must be 1, 2 or 4"),
                                      (3, "similarity_superpose_cols must be 1, 2 or 4")]),
    "similarity_superpose_auto": (1, [(0, 0), (1, 1), (7, 1), (-3, 1)]),
    "similarity_pipeline_chunks": (4, [(1, 1), (8, 8), (0, "similarity_pipeline_chunks must be in [1, 8]"),
                                       (9, "similarity_pipeline_chunks must be in [1, 8]")]),
    "similarity_popcount_band": (1, [(0, 0), (1, 1), (2, 1)]),
    "topk_slab_cols": (0, [(0, 0), (128, 128), (BELOW_2_31, BELOW_2_31), (-1, "topk_slab_cols must be in [0, 2^31)"),
                           (1 << 31, "topk_slab_cols must be in [0, 2^31)")]),
    "maxmin_mode": (0, [(0, 0), (1, 1), (-1, "maxmin_mode must be 0 (dense) or 1 (deferred)"),
                        (2, "maxmin_mode must be 0 (dense) or 1 (deferred)")]),
    "maxmin_resident_rows": (-1, [(0, 0), (5, 5), (-1, -1), (-7, -1), (-(1 << 40), -1), (1 << 40, 1 << 40)]),
    "leader_window_rows": (0, [(0, 0), (300, 300), (BELOW_2_31, BELOW_2_31), (-1, "leader_window_rows must be in [0, 2^31)"),
                               (1 << 31, "leader_window_rows must be in [0, 2^31)")]),
    "butina_min_round_commits": (32, [(0, 0), (10 ** 9, 10 ** 9), (10 ** 9 + 1, 10 ** 9), (10 ** 12, 10 ** 9),
                                      (-1, "butina_min_round_commits must be >= 0")]),
    "bfgs_ctas_per_sm": (3, [(1, 1), (8, 8), (0, "bfgs_ctas_per_sm must be in [1, 8]"),
                             (9, "bfgs_ctas_per_sm must be in [1, 8]")]),
    "bfgs_l2_persist": (0, [(1, 1), (5, 1), (0, 0)]),
    "etkdg_hessian_fp64": (0, [(1, 1), (-1, 1), (0, 0)]),
}
# what the last call left: 0 until a call sets them
HOST_READ_ONLY = ["similarity_superpose_last", "similarity_candidates_last", "similarity_units_planned_last",
                  "topk_slabs_last", "maxmin_resident_last", "leader_windows_last", "leader_bulk_pairs_last"]
# device counters of the last call: reading one synchronises the device
DEVICE_READ_ONLY = ["similarity_units_last", "similarity_tiles_last", "topk_candidates_last", "topk_rows_redone_last",
                    "maxmin_distances_last", "maxmin_popcount_skips_last", "leader_window_pairs_last",
                    "leader_block_pairs_last"]


def test_defaults_on_a_fresh_load(built_lib):
    """In a process of its own, so that the values other tests' calls left behind cannot show."""
    keys = list(WRITABLE) + HOST_READ_ONLY
    code = ("import ctypes as C, sys\n"
            "lib = C.CDLL(sys.argv[1])\n"
            "for k in sys.argv[2:]:\n"
            "    v = C.c_longlong(-99)\n"
            "    assert lib.b200mol_get_option(k.encode(), C.byref(v)) == 0, k\n"
            "    print(v.value)\n")
    out = subprocess.run([sys.executable, "-c", code, _lib.LIB_PATH, *keys], check=True, capture_output=True, text=True)
    got = dict(zip(keys, map(int, out.stdout.split())))
    want = {k: d for k, (d, _) in WRITABLE.items()} | {k: 0 for k in HOST_READ_ONLY}
    assert got == want


@pytest.mark.parametrize("key", list(WRITABLE))
def test_writable_key_accepts_refuses_and_round_trips(built_lib, key):
    before = _lib.get_option(key)
    try:
        for value, want in WRITABLE[key][1]:
            if isinstance(want, str):
                current = _lib.get_option(key)
                with pytest.raises(ValueError, match=re.escape(want)):
                    _lib.set_option(key, value)
                assert _lib.get_option(key) == current, (key, value)  # a refused value changes nothing
            else:
                _lib.set_option(key, value)
                assert _lib.get_option(key) == want, (key, value)
                _lib.set_option(key, _lib.get_option(key))
                assert _lib.get_option(key) == want, (key, value)
    finally:
        _lib.set_option(key, before)
    assert _lib.get_option(key) == before


def test_every_writable_key_round_trips(built_lib):
    for key in WRITABLE:
        v = _lib.get_option(key)
        _lib.set_option(key, v)
        assert _lib.get_option(key) == v, key


@pytest.mark.parametrize("key", HOST_READ_ONLY + DEVICE_READ_ONLY)
def test_read_only_keys_refuse_writes(built_lib, key):
    with pytest.raises(ValueError):
        _lib.set_option(key, 0)


def test_unknown_keys_are_refused(built_lib):
    for key in ("no_such_option", "", "similarity_superpose ", "SIMILARITY_SUPERPOSE", "similarity"):
        with pytest.raises(ValueError, match=re.escape(f"unknown option '{key}'")):
            _lib.get_option(key)
        with pytest.raises(ValueError, match=re.escape(f"unknown option '{key}'")):
            _lib.set_option(key, 1)


def test_every_key_is_documented_in_the_header():
    text = open(os.path.join(ROOT, "include", "b200mol.h")).read()
    start = text.index("Tuning knobs")
    end = text.index("int b200mol_get_option(")
    doc = text[start:end]
    for key in list(WRITABLE) + HOST_READ_ONLY + DEVICE_READ_ONLY:
        assert f'"{key}"' in doc, key


@pytest.mark.gpu
@pytest.mark.parametrize("key", DEVICE_READ_ONLY)
def test_device_counters_read_as_non_negative_integers(cuda, key):
    v = _lib.get_option(key)
    assert isinstance(v, int) and v >= 0


# ------------------------------------------------------------------ _lib.options scopes
def test_scope_sets_and_restores(built_lib):
    before = {k: _lib.get_option(k) for k in ("maxmin_mode", "similarity_superpose", "topk_slab_cols")}
    with _lib.options(maxmin_mode=1, similarity_superpose=2, topk_slab_cols=512):
        assert [_lib.get_option(k) for k in before] == [1, 2, 512]
    assert {k: _lib.get_option(k) for k in before} == before


def test_scope_restores_on_an_exception(built_lib):
    before = _lib.get_option("similarity_pipeline_chunks")
    with pytest.raises(RuntimeError, match="inside"):
        with _lib.options(similarity_pipeline_chunks=1):
            raise RuntimeError("inside")
    assert _lib.get_option("similarity_pipeline_chunks") == before
    # a refused value on entry: what was already set is put back
    mode = _lib.get_option("maxmin_mode")
    with pytest.raises(ValueError):
        with _lib.options(maxmin_mode=1 - mode, similarity_superpose=3):
            pass
    assert _lib.get_option("maxmin_mode") == mode


def test_nested_scopes_unwind_in_order(built_lib):
    before = _lib.get_option("maxmin_resident_rows"), _lib.get_option("leader_window_rows")
    with _lib.options(maxmin_resident_rows=100):
        with _lib.options(maxmin_resident_rows=5, leader_window_rows=300):
            assert (_lib.get_option("maxmin_resident_rows"), _lib.get_option("leader_window_rows")) == (5, 300)
        assert (_lib.get_option("maxmin_resident_rows"), _lib.get_option("leader_window_rows")) == (100, before[1])
    assert (_lib.get_option("maxmin_resident_rows"), _lib.get_option("leader_window_rows")) == before
