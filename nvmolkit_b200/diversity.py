"""Diversity picking on fingerprints on the GPU. API of RDKit's ``rdkit.SimDivFilters.rdSimDivPickers.MaxMinPicker``
(``LazyBitVectorPick`` / ``LazyBitVectorPickWithThreshold``) and ``LeaderPicker`` (``LazyBitVectorPick``), plus
``metric`` and ``stream``."""

from __future__ import annotations

import ctypes
import secrets

import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._interop import fingerprint_matrix, require_cuda, stream_ctx, stream_ptr
from nvmolkit_b200.types import AsyncGpuResult


class MT19937:
    """The 32-bit Mersenne Twister (``std::mt19937`` / ``boost::mt19937``), seeded as both seed it from one integer."""

    def __init__(self, seed: int = 5489):
        mt = [0] * 624
        mt[0] = seed & 0xFFFFFFFF
        for i in range(1, 624):
            mt[i] = (1812433253 * (mt[i - 1] ^ (mt[i - 1] >> 30)) + i) & 0xFFFFFFFF
        self._mt, self._i = mt, 624

    def _twist(self) -> None:
        mt = self._mt
        for i in range(624):
            y = (mt[i] & 0x80000000) | (mt[(i + 1) % 624] & 0x7FFFFFFF)
            mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ (0x9908B0DF if y & 1 else 0)
        self._i = 0

    def __call__(self) -> int:
        if self._i >= 624:
            self._twist()
        y = self._mt[self._i]
        self._i += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9D2C5680
        y ^= (y << 15) & 0xEFC60000
        return y ^ (y >> 18)


def uniform_int(draw, pool_size: int) -> int:
    """``boost::uniform_int<>(0, pool_size - 1)`` over a 32-bit engine ``draw``: words are cut into pool_size buckets of
    ``0xFFFFFFFF // pool_size`` values (one more when ``0xFFFFFFFF % pool_size == pool_size - 1``), and a word past the
    last bucket is drawn again."""
    if pool_size == 1:
        return 0  # (boost returns the bound without drawing)
    bucket = 0xFFFFFFFF // pool_size
    if 0xFFFFFFFF % pool_size == pool_size - 1:
        bucket += 1
    while True:
        r = draw() // bucket
        if r < pool_size:
            return r


def seeded_first_pick(pool_size: int, seed: int) -> int:
    """RDKit's first pick when there are no first picks: ``boost::mt19937`` seeded with ``seed`` (a random seed when
    ``seed < 0``) through ``boost::uniform_int<>(0, pool_size - 1)``."""
    return uniform_int(MT19937(seed if seed >= 0 else secrets.randbits(32)), pool_size)


_WIDTHS = "a multiple of 4 words (128 bits) and at most 128 words (4096 bits)"


def _check_args(n: int, words: int, poolSize, pickSize, firstPicks, metric) -> list:
    """ValueError for any argument the picker refuses; returns the first picks as a list of ints."""
    if metric not in _lib.METRIC:
        raise ValueError(f"metric must be 'tanimoto' or 'cosine', got {metric!r}")
    if not (words > 0 and words % 4 == 0 and words <= 128):
        raise ValueError(f"fingerprint width must be {_WIDTHS}, got {words} words")
    for name, v in (("poolSize", poolSize), ("pickSize", pickSize)):
        if isinstance(v, bool) or not isinstance(v, int):
            raise ValueError(f"{name} must be an int, got {type(v).__name__}")
    if not 1 <= poolSize <= n:
        raise ValueError(f"poolSize must be in [1, {n}] (the fingerprint count), got {poolSize}")
    if not 1 <= pickSize <= poolSize:
        raise ValueError(f"pickSize must be in [1, poolSize = {poolSize}], got {pickSize}")
    first = []
    for f in firstPicks:
        if isinstance(f, bool) or not isinstance(f, int) and not hasattr(f, "__index__"):
            raise ValueError(f"firstPicks entries must be ints, got {type(f).__name__}")
        first.append(int(f))
    if len(first) > pickSize:
        raise ValueError(f"{len(first)} firstPicks for pickSize {pickSize}")
    for f in first:
        if not 0 <= f < poolSize:
            raise ValueError(f"first pick {f} is outside the pool [0, {poolSize})")
    if len(set(first)) != len(first):
        raise ValueError("firstPicks has a repeated entry")
    return first


def _pick(fingerprints, poolSize, pickSize, threshold, firstPicks, seed, metric, stream):
    sptr = stream_ptr(stream)  # validates `stream` first, like the other calls (TypeError)
    fp = fingerprint_matrix(fingerprints, "fingerprints")
    first = _check_args(fp.shape[0], fp.shape[1], poolSize, pickSize, firstPicks, metric)
    if not first:
        first = [seeded_first_pick(poolSize, int(seed))]
    require_cuda()
    h_first = torch.tensor(first, dtype=torch.int32)
    with stream_ctx(stream):
        picks = torch.empty(pickSize, dtype=torch.int32, device=fp.device)
        thr = torch.empty(1, dtype=torch.float64, device=fp.device)
        _lib.call("b200mol_maxmin_pick", fp.data_ptr(), poolSize, fp.shape[1], _lib.METRIC[metric], h_first.data_ptr(),
                  len(first), pickSize, float(threshold), picks.data_ptr(), thr.data_ptr(), sptr)
        fp.record_stream(torch.cuda.current_stream())  # keep the input alive until the stream has consumed it
    return AsyncGpuResult(picks), AsyncGpuResult(thr)


class MaxMinPicker:
    """MaxMin diversity picking of packed fingerprints on the GPU (RDKit's ``MaxMinPicker``).

    The pool is the first ``poolSize`` rows of ``fingerprints`` (anything ``crossTanimotoSimilarity`` takes: an int32
    ``(n, words)`` CUDA tensor, ``MorganFingerprintGenerator.GetFingerprints(...)``; 128 to 4096 bits, a multiple of 128).
    The distance of two items is ``1 - s``, s the fp64 value ``crossTanimotoSimilarity`` / ``crossCosineSimilarity``
    returns for the pair. Picks start with ``firstPicks`` in their order; without them the first pick is drawn as RDKit
    draws it from ``seed`` (``boost::mt19937`` + ``boost::uniform_int``, restated in Python here: the tests pin that
    restatement, not RDKit itself; ``seed < 0`` draws a random first pick). Every further pick is the unpicked item with
    the largest min distance to the picks, ties to the lowest index: exactly what RDKit's ``LazyBitVectorPick`` returns.

    Differences from RDKit: two empty fingerprints are at distance 1 here (similarity 0, the convention of the
    similarity calls), at 0 in RDKit; more ``firstPicks`` than ``pickSize``, or a repeated first pick, is a ValueError.

    Both methods are asynchronous on ``stream`` and do no host synchronisation."""

    def LazyBitVectorPick(self, fingerprints, poolSize, pickSize, firstPicks=(), seed=-1, metric="tanimoto",
                          stream=None) -> AsyncGpuResult:
        """int32 ``[pickSize]`` pool indices in pick order."""
        return _pick(fingerprints, poolSize, pickSize, -1.0, firstPicks, seed, metric, stream)[0]

    def LazyBitVectorPickWithThreshold(self, fingerprints, poolSize, pickSize, threshold, firstPicks=(), seed=-1,
                                       metric="tanimoto", stream=None) -> tuple[AsyncGpuResult, AsyncGpuResult]:
        """``(picks, threshold)``: picking stops before a pick whose max-min distance is ``<= threshold`` (a negative
        threshold never stops it); picks is int32 ``[pickSize]``, -1 past the stop; threshold is fp64 ``[1]``, the
        max-min distance of the last pick the loop added, -1.0 when it added none (the first picks filled
        ``pickSize``, or the first candidate was already within the threshold)."""
        return _pick(fingerprints, poolSize, pickSize, float(threshold), firstPicks, seed, metric, stream)


def _leader_args(n: int, words: int, poolSize, threshold, pickSize, firstPicks, metric) -> tuple[int, float, list]:
    """``MaxMinPicker``'s checks with ``pickSize = 0`` read as ``poolSize``, plus the threshold (in [0, 1], not NaN);
    returns (the pick cap, the threshold, the first picks)."""
    cap = poolSize if type(pickSize) is int and pickSize == 0 else pickSize
    first = _check_args(n, words, poolSize, cap, firstPicks, metric)
    try:
        thr = float(threshold)
    except (TypeError, ValueError):
        raise ValueError(f"threshold must be a number in [0, 1], got {threshold!r}") from None
    if not 0.0 <= thr <= 1.0:  # (also refuses NaN)
        raise ValueError(f"threshold must be in [0, 1], got {thr}")
    return cap, thr, first


class LeaderPicker:
    """Leader (sphere-exclusion) diversity picking of packed fingerprints on the GPU (RDKit's ``LeaderPicker``).

    The pool and the distance are ``MaxMinPicker``'s: the first ``poolSize`` rows of ``fingerprints``, and ``1 - s``
    with s the fp64 value ``crossTanimotoSimilarity`` / ``crossCosineSimilarity`` returns for the pair. Item j is covered
    by pick p when ``1 - s(p, j) <= threshold``. Picks start with ``firstPicks`` in their order, and every item that is a
    first pick or is covered by one leaves the pool; then, repeatedly, the lowest-index item left becomes the next pick,
    and it and every item it covers leave the pool, until the pool is empty or there are ``pickSize`` picks
    (``pickSize = 0``: no limit). Picks after the first ones therefore come in ascending index order. This restates
    RDKit's ``LeaderPicker::lazyPick`` (each pick is the head of the remaining list, which is compacted to the items with
    distance ``> threshold``); the tests pin this restatement, not RDKit itself.

    Differences from RDKit: two empty fingerprints are at distance 1 here (similarity 0, the convention of the
    similarity calls), at 0 in RDKit; a pick always leaves the pool itself, so an empty fingerprint is never picked twice.
    A threshold outside [0, 1] or NaN, more ``firstPicks`` than a non-zero ``pickSize``, or a repeated first pick is a
    ValueError. ``numThreads`` is accepted, so that RDKit call sites run unchanged, and ignored."""

    def LazyBitVectorPick(self, fingerprints, poolSize, threshold, pickSize=0, firstPicks=(), numThreads=1,
                          metric="tanimoto", stream=None) -> AsyncGpuResult:
        """int32 ``[nPicks]`` pool indices in pick order.

        The pick count is only known at the end, so this call synchronises ``stream``: it walks the pool in windows and
        reads back each window's survivor and pick counts to size the next one. The result is complete on return."""
        del numThreads  # (RDKit's thread count: the GPU call has none to set)
        sptr = stream_ptr(stream)  # validates `stream` first, like the other calls (TypeError)
        fp = fingerprint_matrix(fingerprints, "fingerprints")
        cap, thr, first = _leader_args(fp.shape[0], fp.shape[1], poolSize, threshold, pickSize, firstPicks, metric)
        require_cuda()
        h_first = torch.tensor(first, dtype=torch.int32)
        n = ctypes.c_int32(0)
        with stream_ctx(stream):
            picks = torch.empty(cap, dtype=torch.int32, device=fp.device)
            _lib.call("b200mol_leader_pick", fp.data_ptr(), poolSize, fp.shape[1], _lib.METRIC[metric], thr,
                      h_first.data_ptr() if first else None, len(first), cap, picks.data_ptr(), ctypes.addressof(n), sptr)
        return AsyncGpuResult(picks[:n.value])
