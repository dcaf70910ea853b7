"""Tensor / stream plumbing between torch and the C-ABI (torch is plumbing only: memory, streams, distributed)."""

from __future__ import annotations

import torch

from nvmolkit_b200.types import AsyncGpuResult

_FP_DTYPES = (torch.int32, torch.uint32)


_checked_devices: set = set()


def require_cuda() -> None:
    if not torch.cuda.is_available():
        raise RuntimeError("nvmolkit_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.cuda.current_device()
    if dev not in _checked_devices:  # once per device: sm_90 check + keep the stream-ordered pool warm
        from nvmolkit_b200 import _lib

        _lib.check(_lib.load().b200mol_check_device(dev))
        _checked_devices.add(dev)


def as_tensor(obj) -> torch.Tensor:
    """AsyncGpuResult | torch.Tensor | anything with __cuda_array_interface__ -> CUDA tensor (no copy)."""
    if isinstance(obj, AsyncGpuResult):
        return obj.torch()
    if isinstance(obj, torch.Tensor):
        return obj
    if hasattr(obj, "__cuda_array_interface__"):
        return torch.as_tensor(obj, device="cuda")
    raise TypeError(f"expected a CUDA tensor or an object with __cuda_array_interface__, got {type(obj).__name__}")


def fingerprint_matrix(obj, name: str) -> torch.Tensor:
    t = as_tensor(obj)
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    if t.dtype not in _FP_DTYPES:
        raise ValueError(f"{name} must have dtype int32 (packed 32-bit words), got {t.dtype}")
    if t.ndim != 2:
        raise ValueError(f"{name} must be 2D, got shape={tuple(t.shape)}")
    return t.contiguous()


def stream_ptr(stream) -> int:
    if stream is not None and not isinstance(stream, torch.cuda.Stream):
        raise TypeError(f"stream must be a torch.cuda.Stream or None, got {type(stream).__name__}")
    return (stream if stream is not None else torch.cuda.current_stream()).cuda_stream


def stream_ctx(stream):
    return torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream())
