"""Every C entry point that takes a B200MOL_METRIC_* code refuses an unknown one before it touches the device."""

import ctypes

import pytest

_NNZ = object()  # a host counter (uint64_t*)

# (entry point, its arguments with the metric as None), otherwise valid: 16-byte aligned dummy pointers, 128-bit rows
_CALLS = {
    "b200mol_similarity_cross_host": (16, 4, 16, 4, 4, None, 16, 0),
    "b200mol_tanimoto_count_ge": (16, 4, 16, 4, 4, None, 0.5, 1, 16, None),
    "b200mol_similarity_topk": (16, 4, 16, 100, 4, None, 5, 16, 16, None),
    "b200mol_similarity_threshold": (16, 4, 16, 4, 4, None, 0.5, 16, 16, 16, 16, _NNZ, None),
    "b200mol_neighbor_edges": (16, 4, 4, None, 0.5, 0, 1, 16, 16, 16, _NNZ, None),
    "b200mol_butina_fused": (16, 4, 4, None, 0.5, 16, 16, 16, 16, None),
    "b200mol_maxmin_pick": (16, 4, 4, None, 16, 1, 2, -1.0, 16, 16, None),
    "b200mol_leader_pick": (16, 4, 4, None, 0.5, 16, 0, 2, 16, 16, None),
}


@pytest.mark.parametrize("metric", [2, -1, 7])
@pytest.mark.parametrize("name", sorted(_CALLS))
def test_unknown_metric_is_refused(built_lib, name, metric):
    from nvmolkit_b200 import _lib

    metric_at = _CALLS[name].index(None)
    nnz = ctypes.c_uint64(0)
    args = [metric if i == metric_at else ctypes.byref(nnz) if a is _NNZ else a for i, a in enumerate(_CALLS[name])]
    assert getattr(built_lib, name)(*args) == _lib.ERR_INVALID
    assert b"unknown metric" in built_lib.b200mol_last_error()
