"""Shared plumbing of the mirror modules: fp32 master parameters (so reference checkpoints load
strict, utils/checkpoint.py:241-244) plus a lazily built pack of fp16/fp32 device tensors in the
layouts the kernels want.  The pack is dropped whenever parameters may have changed
(load_state_dict, .to()/.cuda())."""
from __future__ import annotations

import torch
import torch.nn as nn

from ... import _lib, ops


def half() -> torch.dtype:
    """The current 16-bit storage type (ops.set_storage_dtype)."""
    return ops.HALF


class PackedModule(nn.Module):
    def __init__(self):
        super().__init__()
        self._pk = None
        self._pk_epoch = -1

    # -- cache invalidation -----------------------------------------------------------------
    def _apply(self, fn, *a, **k):
        self._pk = None
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self._pk = None
        return super()._load_from_state_dict(*a, **k)

    def invalidate_pack(self):
        for m in self.modules():
            if isinstance(m, PackedModule):
                m._pk = None

    # -- pack access ------------------------------------------------------------------------
    def pk(self):
        if self._pk is None or self._pk_epoch != ops.STORAGE_EPOCH:  # (a storage-type switch re-packs)
            with torch.no_grad():
                self._pk_epoch = ops.STORAGE_EPOCH
                self._pk = self._pack()
        return self._pk

    def _pack(self):  # pragma: no cover - overridden
        return {}

    def lazy(self, name: str, make):
        """Pack entries only some call paths need (e.g. the un-folded QKV weights of the module-level API)."""
        p = self.pk()
        if name not in p:
            with torch.no_grad():
                p[name] = make()
        return p[name]


def dev_of(p: torch.Tensor) -> torch.device:
    if not p.is_cuda:
        raise _lib.IdiffError(
            "instancediffusion_b200 modules run only on a CUDA device (sm_90a); there is no CPU path. "
            "Move the module with .cuda() first.")
    return p.device


def w16(p: torch.Tensor) -> torch.Tensor:
    dev_of(p)
    return p.detach().to(half()).contiguous()


def f32(p: torch.Tensor) -> torch.Tensor:
    """fp32 *copy* for a pack.  (`.float()` of an fp32 parameter is the parameter itself: a pack entry aliasing it
    silently followed an in-place load_state_dict of a plain nn.Conv2d -- undo_first_conv_restore -- and the cached
    SD-first-conv pack carried the other conv's bias from the second sample() call on.)"""
    dev_of(p)
    return p.detach().to(dtype=torch.float32, copy=True).contiguous()


def to_tokens(x: torch.Tensor):
    """(B, N, C) any float dtype -> fp16 [B*N, C] contiguous."""
    B, N, C = x.shape
    return x.reshape(B * N, C).to(half()).contiguous(), B, N


def nchw_to_nhwc16(x: torch.Tensor):
    """(B, C, H, W) -> fp16 [B*H*W, C] (boundary glue of the module-level API; the UNet fast path
    converts once with idiff_nchw_f32_to_nhwc_f16)."""
    B, C, H, W = x.shape
    return x.permute(0, 2, 3, 1).reshape(B * H * W, C).to(half()).contiguous(), B, H, W


def nhwc16_to_nchw(y: torch.Tensor, B: int, H: int, W: int, dtype) -> torch.Tensor:
    C = y.shape[-1]
    return y.view(B, H, W, C).permute(0, 3, 1, 2).to(dtype).contiguous()
