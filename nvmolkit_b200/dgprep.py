"""Distance-geometry preparation on the GPU: triangle smoothing, power-iteration eigenpairs, metric-matrix embedding."""

from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._interop import require_cuda, stream_ctx, stream_ptr


# The eigen kernel keeps its per-matrix vectors in 220 KB of shared memory even when the matrix itself is in global
# memory: 2 n doubles for eig_topk, (3 + dim) n + dim for metric_embed (include/b200mol.h).
_SMEM_DOUBLES = 220 * 1024 // 8


def _check_head(ns, per_atom: int, extra: int, what: str) -> None:
    big = [int(n) for n in ns if per_atom * int(n) + extra > _SMEM_DOUBLES]
    if big:
        raise ValueError(f"{what}: matrices of {max(big)} atoms exceed the largest supported size "
                         f"{(_SMEM_DOUBLES - extra) // per_atom}")


def _concat(mats: Sequence[np.ndarray], dev):
    sizes = np.array([m.shape[0] * m.shape[0] for m in mats], dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    flat = np.concatenate([np.ascontiguousarray(m, dtype=np.float64).ravel() for m in mats]) if len(mats) else np.zeros(0)
    return torch.from_numpy(flat).to(dev), torch.from_numpy(starts).to(dev), starts


def triangle_smooth(bounds: Sequence[np.ndarray], tol: float = 0.0, stream=None):
    """Smooth RDKit-layout bounds matrices. Returns (list of smoothed matrices, ok flags)."""
    sptr = stream_ptr(stream)
    require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    with stream_ctx(stream):
        d, st, starts = _concat(bounds, dev)
        ok = torch.zeros(len(bounds), dtype=torch.int8, device=dev)
        _lib.call("b200mol_triangle_smooth", d.data_ptr(), st.data_ptr(), len(bounds), float(tol), ok.data_ptr(), sptr)
        h = d.cpu().numpy()
    return [h[starts[i]:starts[i + 1]].reshape(bounds[i].shape) for i in range(len(bounds))], ok.cpu().numpy().astype(bool)


def eig_topk(mats: Sequence[np.ndarray], num_eigs: int, v0: Optional[Sequence[np.ndarray]] = None, seed: int = 42, stream=None):
    """Top eigenpairs of symmetric matrices. Returns (eigvals [n][k], list of eigvec arrays [k][n_m], n_converged)."""
    sptr = stream_ptr(stream)
    require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    ns = np.array([m.shape[0] for m in mats], dtype=np.int64)
    _check_head(ns, 2, 0, "eig_topk")
    with stream_ctx(stream):
        d, st, _ = _concat(mats, dev)
        vstarts = np.concatenate([[0], np.cumsum(ns * num_eigs)]).astype(np.int64)
        d_vs = torch.from_numpy(vstarts).to(dev)
        vals = torch.zeros((len(mats), num_eigs), dtype=torch.float64, device=dev)
        vecs = torch.zeros(int(vstarts[-1]), dtype=torch.float64, device=dev)
        conv = torch.zeros(len(mats), dtype=torch.int8, device=dev)
        d_v0 = torch.from_numpy(np.concatenate([np.ascontiguousarray(v, dtype=np.float64).ravel() for v in v0])).to(dev) if v0 is not None else None
        _lib.call("b200mol_eig_topk", d.data_ptr(), st.data_ptr(), len(mats), int(num_eigs),
                  d_v0.data_ptr() if d_v0 is not None else None, d_vs.data_ptr() if d_v0 is not None else None, int(seed),
                  vals.data_ptr(), vecs.data_ptr(), d_vs.data_ptr(), conv.data_ptr(), sptr)
        vh = vecs.cpu().numpy()
    return vals.cpu().numpy(), [vh[vstarts[i]:vstarts[i + 1]].reshape(num_eigs, ns[i]) for i in range(len(mats))], conv.cpu().numpy()


def metric_embed(dists: Sequence[np.ndarray], dim: int = 3, v0: Optional[Sequence[np.ndarray]] = None, seed: int = 42, stream=None):
    """Distance matrices -> coordinates (metric-matrix embedding). Returns (list of [n_m, dim] arrays, ok flags)."""
    sptr = stream_ptr(stream)
    require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    ns = np.array([m.shape[0] for m in dists], dtype=np.int64)
    _check_head(ns, 3 + dim, dim, "metric_embed")
    with stream_ctx(stream):
        d, st, _ = _concat(dists, dev)
        astarts = np.concatenate([[0], np.cumsum(ns)]).astype(np.int32)
        d_as = torch.from_numpy(astarts).to(dev)
        coords = torch.zeros((int(astarts[-1]), dim), dtype=torch.float64, device=dev)
        ok = torch.zeros(len(dists), dtype=torch.int8, device=dev)
        vstarts = np.concatenate([[0], np.cumsum(ns * dim)]).astype(np.int64)
        d_vs = torch.from_numpy(vstarts).to(dev)
        d_v0 = torch.from_numpy(np.concatenate([np.ascontiguousarray(v, dtype=np.float64).ravel() for v in v0])).to(dev) if v0 is not None else None
        _lib.call("b200mol_metric_embed", d.data_ptr(), st.data_ptr(), d_as.data_ptr(), len(dists), int(dim),
                  d_v0.data_ptr() if d_v0 is not None else None, d_vs.data_ptr() if d_v0 is not None else None, int(seed),
                  coords.data_ptr(), ok.data_ptr(), sptr)
        ch = coords.cpu().numpy()
    return [ch[astarts[i]:astarts[i + 1]] for i in range(len(dists))], ok.cpu().numpy().astype(bool)
