"""N x M fingerprint similarity on the GPU. API of ``nvmolkit/similarity.py`` (reference :34-184)."""

from __future__ import annotations

import numpy as np
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._interop import fingerprint_matrix, require_cuda, stream_ctx, stream_ptr
from nvmolkit_b200.types import AsyncGpuResult


def _cross(fn_name: str, one, two, stream) -> AsyncGpuResult:
    sptr = stream_ptr(stream)  # validates `stream` first, like the reference (TypeError)
    require_cuda()
    a = fingerprint_matrix(one, "fingerprint_group_one")
    b = a if two is None else fingerprint_matrix(two, "fingerprint_group_two")
    if a.shape[1] != b.shape[1]:
        raise ValueError(f"fingerprint widths differ: {a.shape[1]} vs {b.shape[1]} words")
    with stream_ctx(stream):
        out = torch.empty((a.shape[0], b.shape[0]), dtype=torch.float64, device=a.device)
        _lib.call(fn_name, a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], a.shape[1], out.data_ptr(), sptr)
        # keep inputs alive until the stream has consumed them
        a.record_stream(torch.cuda.current_stream())
        b.record_stream(torch.cuda.current_stream())
    return AsyncGpuResult(out)


def crossTanimotoSimilarity(fingerprint_group_one, fingerprint_group_two=None, stream=None) -> AsyncGpuResult:
    """(n, m) fp64 Tanimoto similarities; all-to-all within group one when group two is None. Asynchronous."""
    return _cross("b200mol_tanimoto_cross", fingerprint_group_one, fingerprint_group_two, stream)


def crossCosineSimilarity(fingerprint_group_one, fingerprint_group_two=None, stream=None) -> AsyncGpuResult:
    return _cross("b200mol_cosine_cross", fingerprint_group_one, fingerprint_group_two, stream)


TOPK_MAX = 256  # B200MOL_TOPK_MAX (include/b200mol.h): the largest k the search kernels are compiled for


def _check_k(k, library_size: int) -> int:
    if isinstance(k, bool) or not isinstance(k, int):
        raise ValueError(f"k must be an int, got {type(k).__name__}")
    if not 1 <= k <= min(library_size, TOPK_MAX):
        raise ValueError(f"k must be in [1, min(library size, {TOPK_MAX})] (got k={k}, library size {library_size})")
    return k


def _topk(metric: str, one, two, k, stream):
    sptr = stream_ptr(stream)  # validates `stream` first, like the matrix calls (TypeError)
    require_cuda()
    a = fingerprint_matrix(one, "fingerprint_group_one")
    b = a if two is None else fingerprint_matrix(two, "fingerprint_group_two")
    if a.shape[1] != b.shape[1]:
        raise ValueError(f"fingerprint widths differ: {a.shape[1]} vs {b.shape[1]} words")
    k = _check_k(k, b.shape[0])
    with stream_ctx(stream):
        values = torch.empty((a.shape[0], k), dtype=torch.float64, device=a.device)
        indices = torch.empty((a.shape[0], k), dtype=torch.int32, device=a.device)
        _lib.call("b200mol_similarity_topk", a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], a.shape[1],
                  _lib.METRIC[metric], k, values.data_ptr(), indices.data_ptr(), sptr)
        # keep inputs alive until the stream has consumed them
        a.record_stream(torch.cuda.current_stream())
        b.record_stream(torch.cuda.current_stream())
    return AsyncGpuResult(values), AsyncGpuResult(indices)


def topKTanimotoSimilarity(fingerprint_group_one, fingerprint_group_two=None, k=10, stream=None):
    """For each fingerprint of group one (the queries) its k most similar fingerprints of group two (the library; the
    queries themselves, self-matches included, when None): ``(values, indices)``, fp64 and int32 ``[Q, k]``. Row q is
    the first k columns of row q of ``crossTanimotoSimilarity`` ordered by (value descending, column ascending), the
    values bit-identical to the matrix entries, ties to the lowest index. The matrix is never stored.
    ``1 <= k <= min(len(library), TOPK_MAX)``, ``TOPK_MAX = 256``. Asynchronous on ``stream``."""
    return _topk("tanimoto", fingerprint_group_one, fingerprint_group_two, k, stream)


def topKCosineSimilarity(fingerprint_group_one, fingerprint_group_two=None, k=10, stream=None):
    """Cosine twin of ``topKTanimotoSimilarity``: rows of ``crossCosineSimilarity``."""
    return _topk("cosine", fingerprint_group_one, fingerprint_group_two, k, stream)


def _cross_host(metric: str, one, two, max_device_bytes: int = 0) -> np.ndarray:
    require_cuda()

    def host(x):
        if isinstance(x, AsyncGpuResult):
            x = x.torch()
        if isinstance(x, torch.Tensor):
            x = x.detach().cpu().numpy()
        x = np.ascontiguousarray(x)
        if x.dtype not in (np.int32, np.uint32) or x.ndim != 2:
            raise ValueError("fingerprints must be a 2D int32 array of packed 32-bit words")
        return x

    a = host(one)
    b = a if two is None else host(two)
    if a.shape[1] != b.shape[1]:
        raise ValueError(f"fingerprint widths differ: {a.shape[1]} vs {b.shape[1]} words")
    out = np.empty((a.shape[0], b.shape[0]), dtype=np.float64)
    _lib.call("b200mol_similarity_cross_host", a.ctypes.data, a.shape[0], b.ctypes.data, b.shape[0], a.shape[1],
              _lib.METRIC[metric], out.ctypes.data, int(max_device_bytes))
    return out


def crossTanimotoSimilarityMemoryConstrained(fingerprint_group_one, fingerprint_group_two=None) -> np.ndarray:
    """Host-in / host-out variant: result as a NumPy array, computed in row blocks with overlapped D2H."""
    return _cross_host("tanimoto", fingerprint_group_one, fingerprint_group_two)


def crossCosineSimilarityMemoryConstrained(fingerprint_group_one, fingerprint_group_two=None) -> np.ndarray:
    return _cross_host("cosine", fingerprint_group_one, fingerprint_group_two)
