"""N x M fingerprint similarity on the GPU. API of ``nvmolkit/similarity.py`` (reference :34-184)."""

from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._interop import as_tensor, check_stream, fingerprint_matrix, require_cuda, stream_ctx, stream_ptr
from nvmolkit_b200.types import AsyncGpuResult


def _entry(operation: str, measure, counts: bool = False):
    """The C entry point of an operation ("cross", "topk", "threshold" or "cross_host") for a measure (a key of
    _lib.METRIC, or the (alpha, beta) of Tversky), and the measure's arguments to it. counts: the entry point on count
    vectors ("cross", "topk" or "threshold"), which takes every measure as its (alpha, beta)."""
    if counts:
        return f"b200mol_count_{operation}", measure
    if not isinstance(measure, str):
        return f"b200mol_tversky_{operation}", measure
    if operation == "cross":  # (one entry point per metric)
        return f"b200mol_{measure}_cross", ()
    return f"b200mol_similarity_{operation}", (_lib.METRIC[measure],)


def _check_width(a, b, counts: bool = False) -> None:
    if b is not None and a.shape[1] != b.shape[1]:
        if counts:
            raise ValueError(f"count vector widths differ: {a.shape[1]} vs {b.shape[1]} bins")
        raise ValueError(f"fingerprint widths differ: {a.shape[1]} vs {b.shape[1]} words")


def _fingerprints(one, two, counts: bool = False):
    """CUDA, both matrices (packed bits, or count vectors when counts) and their widths; b is None for a search of
    group one against itself."""
    require_cuda()
    check = _count_matrix if counts else fingerprint_matrix
    a = check(one, "fingerprint_group_one")
    b = None if two is None else check(two, "fingerprint_group_two")
    _check_width(a, b, counts)
    return a, b


def _operands(one, two, stream, counts: bool):
    """The stream pointer and both matrices (b None for a self search), the stream checked first, like the reference
    (TypeError)."""
    sptr = stream_ptr(stream)
    return (sptr, *_fingerprints(one, two, counts))


def _prepare(x, counts: bool):
    """A checked matrix as the binding passes it (None stays None), on the call's stream: count vectors as int32."""
    return x.to(torch.int32).contiguous() if counts and x is not None else x


def _library(a, b, counts: bool):
    """The library a cross or top-k call passes: group two's, else for a self search group one's own (packed bits) or
    none (count vectors)."""
    if b is not None:
        return b.data_ptr()
    return None if counts else a.data_ptr()


def _keep_alive(*tensors) -> None:
    """keep inputs alive until the stream has consumed them"""
    for x in tensors:
        if x is not None:
            x.record_stream(torch.cuda.current_stream())


def _cross(measure, one, two, stream, counts: bool = False) -> AsyncGpuResult:
    sptr, a, b = _operands(one, two, stream, counts)
    n_b = (a if b is None else b).shape[0]
    fn, args = _entry("cross", measure, counts)
    with stream_ctx(stream):
        a, b = _prepare(a, counts), _prepare(b, counts)
        out = torch.empty((a.shape[0], n_b), dtype=torch.float64, device=a.device)
        _lib.call(fn, a.data_ptr(), a.shape[0], _library(a, b, counts), n_b, a.shape[1], *args, out.data_ptr(),
                  sptr)
        _keep_alive(a, b)
    return AsyncGpuResult(out)


def crossTanimotoSimilarity(fingerprint_group_one, fingerprint_group_two=None, stream=None) -> AsyncGpuResult:
    """(n, m) fp64 Tanimoto similarities; all-to-all within group one when group two is None. Asynchronous."""
    return _cross("tanimoto", fingerprint_group_one, fingerprint_group_two, stream)


def crossCosineSimilarity(fingerprint_group_one, fingerprint_group_two=None, stream=None) -> AsyncGpuResult:
    return _cross("cosine", fingerprint_group_one, fingerprint_group_two, stream)


TOPK_MAX = 256  # B200MOL_TOPK_MAX (include/b200mol.h): the largest k the search kernels are compiled for


def _check_k(k, library_size: int) -> int:
    if isinstance(k, bool) or not isinstance(k, int):
        raise ValueError(f"k must be an int, got {type(k).__name__}")
    if not 1 <= k <= min(library_size, TOPK_MAX):
        raise ValueError(f"k must be in [1, min(library size, {TOPK_MAX})] (got k={k}, library size {library_size})")
    return k


def _topk(measure, one, two, k, stream, counts: bool = False):
    sptr, a, b = _operands(one, two, stream, counts)
    n_lib = (a if b is None else b).shape[0]
    k = _check_k(k, n_lib)
    fn, args = _entry("topk", measure, counts)
    with stream_ctx(stream):
        a, b = _prepare(a, counts), _prepare(b, counts)
        values = torch.empty((a.shape[0], k), dtype=torch.float64, device=a.device)
        indices = torch.empty((a.shape[0], k), dtype=torch.int32, device=a.device)
        _lib.call(fn, a.data_ptr(), a.shape[0], _library(a, b, counts), n_lib, a.shape[1], *args, k,
                  values.data_ptr(), indices.data_ptr(), sptr)
        _keep_alive(a, b)
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


def _check_threshold(threshold) -> float:
    if isinstance(threshold, bool) or not isinstance(threshold, (int, float, np.integer, np.floating)):
        raise ValueError(f"threshold must be a real number, got {type(threshold).__name__}")
    t = float(threshold)
    if not 0.0 < t <= 1.0:  # (NaN fails too)
        raise ValueError(f"threshold must be in (0, 1] (got {threshold}); threshold 0 is the dense matrix: use the "
                         "cross*Similarity calls")
    return t


def _threshold(measure, one, two, threshold, stream, counts: bool = False):
    check_stream(stream)  # first, like the matrix calls (TypeError)
    t = _check_threshold(threshold)
    sptr = stream_ptr(stream)
    a, b = _fingerprints(one, two, counts)
    n_q, n_lib = a.shape[0], (a.shape[0] if b is None else b.shape[0])
    with stream_ctx(stream):
        a, b = _prepare(a, counts), _prepare(b, counts)
        if n_q == 0 or n_lib == 0:  # no pair (and an empty tensor's address may be 0, the C-ABI's "no library")
            return (AsyncGpuResult(torch.zeros(n_q + 1, dtype=torch.int64, device=a.device)),
                    AsyncGpuResult(torch.empty(0, dtype=torch.int32, device=a.device)),
                    AsyncGpuResult(torch.empty(0, dtype=torch.float64, device=a.device)))
        indptr = torch.empty(n_q + 1, dtype=torch.int64, device=a.device)
        # a first guess at the result size; a larger result is reported and the call is made once more with room for it
        cap = min(max(1 << 20, 64 * n_q), n_q * n_lib)
        fn, args = _entry("threshold", measure, counts)
        for _ in range(2):
            indices = torch.empty(cap, dtype=torch.int32, device=a.device)
            values = torch.empty(cap, dtype=torch.float64, device=a.device)
            nnz = C.c_uint64(0)
            _lib.call(fn, a.data_ptr(), n_q, None if b is None else b.data_ptr(), n_lib, a.shape[1], *args, t,
                      indptr.data_ptr(), indices.data_ptr(), values.data_ptr(), cap, C.byref(nnz), sptr)
            if nnz.value <= cap:
                break
            cap = int(nnz.value)
        _keep_alive(a, b)
    n = int(nnz.value)
    return AsyncGpuResult(indptr), AsyncGpuResult(indices[:n]), AsyncGpuResult(values[:n])


def thresholdTanimotoSimilarity(fingerprint_group_one, fingerprint_group_two=None, *, threshold, stream=None):
    """Every pair at or above a Tanimoto threshold, as CSR: ``(indptr, indices, values)``, int64 ``[Q + 1]``, int32
    ``[nnz]`` and fp64 ``[nnz]``. Row q (a fingerprint of group one) lists exactly the columns j (of group two; of group
    one itself, self-matches included, when None) whose ``crossTanimotoSimilarity`` entry is ``>= threshold``, in
    ascending column order, with values bit-identical to those matrix entries. The matrix is never stored.
    ``0 < threshold <= 1``. The result size is data-dependent, so the call synchronises ``stream`` (the arrays it returns
    are then written on ``stream``). As a sparse matrix::

        indptr, indices, values = (r.torch() for r in thresholdTanimotoSimilarity(q, lib, threshold=0.7))
        m = torch.sparse_csr_tensor(indptr, indices, values, size=(len(q), len(lib)))
        m = scipy.sparse.csr_matrix((values.cpu().numpy(), indices.cpu().numpy(), indptr.cpu().numpy()),
                                    shape=(len(q), len(lib)))
    """
    return _threshold("tanimoto", fingerprint_group_one, fingerprint_group_two, threshold, stream)


def thresholdCosineSimilarity(fingerprint_group_one, fingerprint_group_two=None, *, threshold, stream=None):
    """Cosine twin of ``thresholdTanimotoSimilarity``: the entries of ``crossCosineSimilarity`` that are
    ``>= threshold``."""
    return _threshold("cosine", fingerprint_group_one, fingerprint_group_two, threshold, stream)


def _cross_host(measure, one, two, max_device_bytes: int = 0) -> np.ndarray:
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
    _check_width(a, b)
    out = np.empty((a.shape[0], b.shape[0]), dtype=np.float64)
    fn, args = _entry("cross_host", measure)
    _lib.call(fn, a.ctypes.data, a.shape[0], b.ctypes.data, b.shape[0], a.shape[1], *args, out.ctypes.data,
              int(max_device_bytes))
    return out


def crossTanimotoSimilarityMemoryConstrained(fingerprint_group_one, fingerprint_group_two=None) -> np.ndarray:
    """Host-in / host-out variant: result as a NumPy array, computed in row blocks with overlapped D2H."""
    return _cross_host("tanimoto", fingerprint_group_one, fingerprint_group_two)


def crossCosineSimilarityMemoryConstrained(fingerprint_group_one, fingerprint_group_two=None) -> np.ndarray:
    return _cross_host("cosine", fingerprint_group_one, fingerprint_group_two)


# ---- Dice and Tversky ----
# tversky(c, a, b; alpha, beta) = 0 if c == 0, else c / ((alpha (a - c) + beta (b - c)) + c), a = |A| (group one, the row),
# b = |B|, c = |A & B|: each product, sum and the quotient one fp64 operation rounded to nearest, in that order. Dice,
# 2c / (a + b), is (1/2, 1/2); (1, 1) is Tanimoto bit for bit. alpha weights the bits only in group one's fingerprint, as
# in RDKit's TverskySimilarity(fp1, fp2, a, b), so cross(one, two, alpha, beta) is cross(two, one, beta, alpha).T.
# For dyadic weights (0, 1/4, 1/2, 1, 2, ...) the value does not depend on the order of evaluation; for others, such as
# (0.3, 0.7), an expanded form like alpha a + beta b + (1 - alpha - beta) c may differ from it by a few ulp, so bit parity
# with RDKit is not claimed there.
TVERSKY_MAX_WEIGHT = 1000.0  # the weights' range, 0 <= alpha, beta <= 1000 (the float tile filters are derived for it)
DICE = (0.5, 0.5)


def _check_weights(alpha, beta) -> tuple:
    out = []
    for name, w in (("alpha", alpha), ("beta", beta)):
        if isinstance(w, bool) or not isinstance(w, (int, float, np.integer, np.floating)):
            raise ValueError(f"Tversky {name} must be a real number, got {type(w).__name__}")
        w = float(w)
        if not 0.0 <= w <= TVERSKY_MAX_WEIGHT:  # (NaN fails too; so does inf)
            raise ValueError(f"Tversky {name} must be finite with 0 <= {name} <= {TVERSKY_MAX_WEIGHT:g} (got {w})")
        out.append(w)
    return tuple(out)


def crossDiceSimilarity(fingerprint_group_one, fingerprint_group_two=None, stream=None) -> AsyncGpuResult:
    """(n, m) fp64 Dice similarities 2|A & B| / (|A| + |B|) (0 for an empty intersection); all-to-all within group one
    when group two is None. Asynchronous. Bit-identical to ``crossTverskySimilarity(..., alpha=0.5, beta=0.5)``."""
    return _cross(DICE, fingerprint_group_one, fingerprint_group_two, stream)


def crossTverskySimilarity(fingerprint_group_one, fingerprint_group_two=None, *, alpha, beta, stream=None) -> AsyncGpuResult:
    """(n, m) fp64 Tversky similarities c / ((alpha (a - c) + beta (b - c)) + c), a the popcount of the row's fingerprint
    (group one), b the column's, c their intersection, 0 when c == 0; all-to-all within group one when group two is
    None. ``0 <= alpha, beta <= 1000``. Tversky(1, 0) = c / a is how much of the query a library fingerprint contains;
    (0.9, 0.1) is the usual fragment / scaffold setting. Asynchronous. See the module note on RDKit parity."""
    weights = _check_weights(alpha, beta)  # (before anything touches the device)
    return _cross(weights, fingerprint_group_one, fingerprint_group_two, stream)


def topKDiceSimilarity(fingerprint_group_one, fingerprint_group_two=None, k=10, stream=None):
    """Dice twin of ``topKTanimotoSimilarity``: rows of ``crossDiceSimilarity``. Dice orders pairs exactly as Tanimoto
    does, so the indices are those of ``topKTanimotoSimilarity`` on the same inputs."""
    return _topk(DICE, fingerprint_group_one, fingerprint_group_two, k, stream)


def topKTverskySimilarity(fingerprint_group_one, fingerprint_group_two=None, k=10, *, alpha, beta, stream=None):
    """Tversky twin of ``topKTanimotoSimilarity``: the first k columns of each row of ``crossTverskySimilarity`` by
    (value descending, column ascending). With an asymmetric measure a self search need not list the self-match first:
    under (alpha, beta) = (1, 0) every superset of the query also scores 1.0, and ties go to the lowest index."""
    weights = _check_weights(alpha, beta)  # (before anything touches the device)
    return _topk(weights, fingerprint_group_one, fingerprint_group_two, k, stream)


def thresholdDiceSimilarity(fingerprint_group_one, fingerprint_group_two=None, *, threshold, stream=None):
    """Dice twin of ``thresholdTanimotoSimilarity``: the entries of ``crossDiceSimilarity`` that are ``>= threshold``,
    as CSR. Synchronises ``stream``."""
    return _threshold(DICE, fingerprint_group_one, fingerprint_group_two, threshold, stream)


def thresholdTverskySimilarity(fingerprint_group_one, fingerprint_group_two=None, *, alpha, beta, threshold, stream=None):
    """Tversky twin of ``thresholdTanimotoSimilarity``: the entries of ``crossTverskySimilarity`` that are
    ``>= threshold``, as CSR; a self search (group two None) gives the same result as passing group one twice.
    Synchronises ``stream``."""
    weights = _check_weights(alpha, beta)  # (before anything touches the device)
    return _threshold(weights, fingerprint_group_one, fingerprint_group_two, threshold, stream)


def crossDiceSimilarityMemoryConstrained(fingerprint_group_one, fingerprint_group_two=None) -> np.ndarray:
    """Host-in / host-out Dice matrix as a NumPy array, computed in row blocks with overlapped D2H."""
    return _cross_host(DICE, fingerprint_group_one, fingerprint_group_two)


def crossTverskySimilarityMemoryConstrained(fingerprint_group_one, fingerprint_group_two=None, *, alpha,
                                            beta) -> np.ndarray:
    """Host-in / host-out Tversky matrix as a NumPy array, computed in row blocks with overlapped D2H."""
    weights = _check_weights(alpha, beta)
    return _cross_host(weights, fingerprint_group_one, fingerprint_group_two)


# ---- count vectors ----
# The measures above on count vectors (RDKit's SparseIntVect similarities, e.g. of GetCountFingerprint): with a the sum
# of the row's counts (group one), b the column's and c = sum over bins of min(row, column), the value is the Tversky
# expression above of (c, a, b). Tanimoto is (1, 1): c / (a + b - c); Dice (1/2, 1/2): 2c / (a + b); both bit for bit
# RDKit's, every intermediate an exact integer. The module's note on non-dyadic Tversky weights applies unchanged.
# Counts must lie in 0 .. 65535 (every sum then fits int32 and is exact in fp64); that is checked on the device and its
# flag read once, so every count call synchronises its stream, and a count out of range raises ValueError.
COUNT_MAX_BINS = 4096
COUNT_MAX = 65535
_COUNT_DTYPES = (torch.uint8, torch.int16, torch.int32)
TANIMOTO = (1.0, 1.0)


def _count_matrix(obj, name: str) -> torch.Tensor:
    t = as_tensor(obj)
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    if t.dtype not in _COUNT_DTYPES:
        raise ValueError(f"{name} must have dtype uint8, int16 or int32 (counts), got {t.dtype}")
    if t.ndim != 2:
        raise ValueError(f"{name} must be 2D, got shape={tuple(t.shape)}")
    if not 1 <= t.shape[1] <= COUNT_MAX_BINS:
        raise ValueError(f"{name} must have 1 to {COUNT_MAX_BINS} bins, got {t.shape[1]}")
    return t


def crossTanimotoCountSimilarity(fingerprint_group_one, fingerprint_group_two=None, stream=None) -> AsyncGpuResult:
    """(n, m) fp64 Tanimoto similarities of count vectors, c / (a + b - c) with a, b the row sums and c the sum of the
    bin-wise minima (0 when c == 0), RDKit's ``TanimotoSimilarity`` on count fingerprints bit for bit; all-to-all within
    group one when group two is None. Inputs: 2D uint8, int16 or int32 CUDA tensors (or ``AsyncGpuResult``) of counts in
    ``0 .. 65535``, 1 to 4096 bins, e.g. ``GetCountFingerprints``. Synchronises ``stream`` (the range check)."""
    return _cross(TANIMOTO, fingerprint_group_one, fingerprint_group_two, stream, counts=True)


def crossDiceCountSimilarity(fingerprint_group_one, fingerprint_group_two=None, stream=None) -> AsyncGpuResult:
    """Dice twin of ``crossTanimotoCountSimilarity``: 2c / (a + b), RDKit's ``DiceSimilarity`` on count fingerprints
    bit for bit. Synchronises ``stream``."""
    return _cross(DICE, fingerprint_group_one, fingerprint_group_two, stream, counts=True)


def crossTverskyCountSimilarity(fingerprint_group_one, fingerprint_group_two=None, *, alpha, beta,
                                stream=None) -> AsyncGpuResult:
    """Tversky twin of ``crossTanimotoCountSimilarity``: c / ((alpha (a - c) + beta (b - c)) + c), alpha weighting what
    only the row (group one) has. ``0 <= alpha, beta <= 1000``. See the module note on RDKit parity. Synchronises
    ``stream``."""
    weights = _check_weights(alpha, beta)  # (before anything touches the device)
    return _cross(weights, fingerprint_group_one, fingerprint_group_two, stream, counts=True)


def topKTanimotoCountSimilarity(fingerprint_group_one, fingerprint_group_two=None, k=10, stream=None):
    """For each count vector of group one its k most similar of group two (of group one itself, self-matches included,
    when None): ``(values, indices)``, fp64 and int32 ``[Q, k]``, the first k columns of each row of
    ``crossTanimotoCountSimilarity`` ordered by (value descending, column ascending), values bit-identical to the matrix.
    The matrix is never stored. ``1 <= k <= min(len(library), TOPK_MAX)``. Synchronises ``stream`` (the range check)."""
    return _topk(TANIMOTO, fingerprint_group_one, fingerprint_group_two, k, stream, counts=True)


def topKDiceCountSimilarity(fingerprint_group_one, fingerprint_group_two=None, k=10, stream=None):
    """Dice twin of ``topKTanimotoCountSimilarity``: rows of ``crossDiceCountSimilarity``."""
    return _topk(DICE, fingerprint_group_one, fingerprint_group_two, k, stream, counts=True)


def topKTverskyCountSimilarity(fingerprint_group_one, fingerprint_group_two=None, k=10, *, alpha, beta, stream=None):
    """Tversky twin of ``topKTanimotoCountSimilarity``: rows of ``crossTverskyCountSimilarity``."""
    weights = _check_weights(alpha, beta)
    return _topk(weights, fingerprint_group_one, fingerprint_group_two, k, stream, counts=True)


def thresholdTanimotoCountSimilarity(fingerprint_group_one, fingerprint_group_two=None, *, threshold, stream=None):
    """Every pair of count vectors at or above a Tanimoto threshold, as CSR ``(indptr, indices, values)``, int64
    ``[Q + 1]``, int32 and fp64 ``[nnz]``: row q lists exactly the columns whose ``crossTanimotoCountSimilarity`` entry
    is ``>= threshold``, ascending, with those values (group two None: group one against itself, self-matches
    included). ``0 < threshold <= 1``. The matrix is never stored. Synchronises ``stream``."""
    return _threshold(TANIMOTO, fingerprint_group_one, fingerprint_group_two, threshold, stream, counts=True)


def thresholdDiceCountSimilarity(fingerprint_group_one, fingerprint_group_two=None, *, threshold, stream=None):
    """Dice twin of ``thresholdTanimotoCountSimilarity``: entries of ``crossDiceCountSimilarity``."""
    return _threshold(DICE, fingerprint_group_one, fingerprint_group_two, threshold, stream, counts=True)


def thresholdTverskyCountSimilarity(fingerprint_group_one, fingerprint_group_two=None, *, alpha, beta, threshold,
                                    stream=None):
    """Tversky twin of ``thresholdTanimotoCountSimilarity``: entries of ``crossTverskyCountSimilarity``."""
    weights = _check_weights(alpha, beta)
    return _threshold(weights, fingerprint_group_one, fingerprint_group_two, threshold, stream, counts=True)
