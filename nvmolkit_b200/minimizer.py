"""Batched BFGS minimisation / energy evaluation of conformer batches through the C-ABI (b200mol_*_minimize)."""

from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from nvmolkit_b200 import _lib
from nvmolkit_b200._interop import require_cuda, stream_ctx, stream_ptr
from nvmolkit_b200.forcefield import DIM, ConformerBatch, FlatSystem


@dataclass
class MinimizeResult:
    positions: torch.Tensor  # float64 [totalAtoms, dim] (device)
    energies: torch.Tensor  # float64 [nConf]
    status: torch.Tensor  # int8 [nConf], 0 = converged, 1 = maxIters reached
    iters: torch.Tensor  # int32 [nConf]


def _device_batch(batch: ConformerBatch, dev, positions: Optional[torch.Tensor] = None):
    conf_mol = torch.from_numpy(batch.conf_mol).to(dev, non_blocking=True)
    starts = torch.from_numpy(batch.atom_starts).to(dev, non_blocking=True)
    pos = positions if positions is not None else torch.from_numpy(batch.positions).to(dev, non_blocking=True)
    return conf_mol, starts, pos.contiguous()


def minimize(system: FlatSystem, batch: ConformerBatch, max_iters: int = 200, grad_tol: float = 1e-4, *,
             chiral_weight: float = 1.0, fourth_dim_weight: float = 0.1, dim: int = 0, plain: bool = False,
             recentre: bool = True, positions: Optional[torch.Tensor] = None,
             active: Optional[torch.Tensor] = None, stream=None) -> MinimizeResult:
    """Minimise every conformer of `batch` under `system` (kind mmff | dg | etk). Asynchronous on `stream`.

    `positions`: optional device tensor to use (and update in place) instead of uploading batch.positions."""
    sptr = stream_ptr(stream)
    require_cuda()
    kind = system.kind
    dim = dim or DIM[kind]
    dev = torch.device("cuda", torch.cuda.current_device())
    st, _keep = system.to_device(dev)
    with stream_ctx(stream):
        conf_mol, starts, pos = _device_batch(batch, dev, positions)
        if pos.shape[-1] != dim and pos.ndim == 2:
            raise ValueError(f"positions must have {dim} columns for kind '{kind}', got {pos.shape[-1]}")
        n = batch.n_conf
        energies = torch.empty(n, dtype=torch.float64, device=dev)
        status = torch.ones(n, dtype=torch.int8, device=dev)
        iters = torch.zeros(n, dtype=torch.int32, device=dev)
        act = active.data_ptr() if active is not None else None
        common = (n, conf_mol.data_ptr(), starts.data_ptr(), batch.max_atoms, pos.data_ptr(), int(max_iters),
                  float(grad_tol), act, energies.data_ptr(), status.data_ptr(), iters.data_ptr(), sptr)
        if kind == "mmff":
            _lib.call("b200mol_mmff_minimize", C.byref(st), *common)
        elif kind == "uff":
            _lib.call("b200mol_uff_minimize", C.byref(st), *common)
        elif kind == "dg":
            _lib.call("b200mol_dg_minimize", C.byref(st), int(dim), float(chiral_weight), float(fourth_dim_weight), *common)
        elif kind == "etk":
            _lib.call("b200mol_etk_minimize", C.byref(st), 1 if plain else 0, 1 if recentre else 0, *common)
        else:
            raise ValueError(f"unknown force field kind {kind}")
    return MinimizeResult(pos, energies, status, iters)


def energy_and_grad(system: FlatSystem, batch: ConformerBatch, want_grad: bool = True, *, chiral_weight: float = 1.0,
                    fourth_dim_weight: float = 0.1, dim: int = 0, plain: bool = False, recentre: bool = False,
                    stream=None):
    """(energies [nConf], gradients [totalAtoms, dim] | None) on the device."""
    sptr = stream_ptr(stream)
    require_cuda()
    kind = system.kind
    dim = dim or DIM[kind]
    dev = torch.device("cuda", torch.cuda.current_device())
    st, _keep = system.to_device(dev)
    with stream_ctx(stream):
        conf_mol, starts, pos = _device_batch(batch, dev)
        n = batch.n_conf
        energies = torch.empty(n, dtype=torch.float64, device=dev)
        grad = torch.zeros_like(pos) if want_grad else None
        gptr = grad.data_ptr() if want_grad else None
        if kind in ("mmff", "uff"):
            _lib.call(f"b200mol_{kind}_energy_grad", C.byref(st), n, conf_mol.data_ptr(), starts.data_ptr(), pos.data_ptr(),
                      energies.data_ptr(), gptr, sptr)
        elif kind == "dg":
            _lib.call("b200mol_dg_energy_grad", C.byref(st), int(dim), float(chiral_weight), float(fourth_dim_weight), n,
                      conf_mol.data_ptr(), starts.data_ptr(), pos.data_ptr(), energies.data_ptr(), gptr, sptr)
        elif kind == "etk":
            _lib.call("b200mol_etk_energy_grad", C.byref(st), 1 if plain else 0, 1 if recentre else 0, n, conf_mol.data_ptr(), starts.data_ptr(),
                      pos.data_ptr(), energies.data_ptr(), gptr, sptr)
        else:
            raise ValueError(f"unknown force field kind {kind}")
    return energies, grad


def poly_minimize(starts: np.ndarray, power: int, w: np.ndarray, c: np.ndarray, x0: np.ndarray, max_iters: int,
                  grad_tol: float, scale_grads: bool, stream=None, *, hessian_fp32: bool = False):
    """Analytic test systems E = sum w (x - c)^power driven through the same BFGS kernel (tests).

    `hessian_fp32`: keep the inverse Hessian in fp32, the embedder's default slab type (fp64 otherwise, like MMFF / UFF)."""
    sptr = stream_ptr(stream)
    require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    with stream_ctx(stream):
        d_starts = torch.from_numpy(np.ascontiguousarray(starts, dtype=np.int32)).to(dev)
        d_w = torch.from_numpy(np.ascontiguousarray(w, dtype=np.float64)).to(dev)
        d_c = torch.from_numpy(np.ascontiguousarray(c, dtype=np.float64)).to(dev)
        d_x = torch.from_numpy(np.ascontiguousarray(x0, dtype=np.float64)).to(dev)
        n = len(starts) - 1
        e = torch.empty(n, dtype=torch.float64, device=dev)
        status = torch.ones(n, dtype=torch.int8, device=dev)
        iters = torch.zeros(n, dtype=torch.int32, device=dev)
        _lib.call("b200mol_poly_minimize", n, d_starts.data_ptr(), int(np.diff(starts).max()), int(power), d_w.data_ptr(),
                  d_c.data_ptr(), d_x.data_ptr(), int(max_iters), float(grad_tol), 1 if scale_grads else 0,
                  1 if hessian_fp32 else 0, e.data_ptr(), status.data_ptr(), iters.data_ptr(), sptr)
    return d_x, e, status, iters
