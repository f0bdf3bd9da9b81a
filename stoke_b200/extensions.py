# -*- coding: utf-8 -*-
"""Optimizer-builder mixins and the data-parallel handler -- the plugin seam of
/root/reference/stoke/extensions.py (``BaseOptimizer.build_optimizer`` :53-78, ``FairscaleOSSExtension`` :109-141,
``BaseDDP.handle_ddp`` :179-216, ``FairscaleSDDPExtension`` :249-286) with the engine behind it."""
import os
from contextlib import contextmanager
from enum import Enum
from typing import Dict, Optional, Type

import torch

from . import _lib
from .configs import ClipGradConfig, ClipGradNormConfig
from .engine import ClipSpec
from .optim import B200FusedOptimizer, B200StockOptimizer, fused_supported


def clip_spec_from_config(grad_clip) -> ClipSpec:
    if grad_clip is None:
        return ClipSpec()
    if isinstance(grad_clip, ClipGradNormConfig):
        return ClipSpec(_lib.CLIP_NORM, max_norm=grad_clip.max_norm, norm_type=grad_clip.norm_type)
    if isinstance(grad_clip, ClipGradConfig):
        return ClipSpec(_lib.CLIP_VALUE, clip_value=grad_clip.clip_value)
    raise TypeError("Stoke -- grad_clip argument must be of type ClipGradConfig or ClipGradNormConfig")


class BaseOptimizer:
    _sharded_state = False

    def __init__(self, verbose: bool = True, **kwargs):
        self._verbose = verbose
        self._grad_accum = kwargs.get("grad_accum_steps", 1) or 1
        self._grad_clip = kwargs.get("grad_clip")

    def build_optimizer(self, optimizer: Type[torch.optim.Optimizer], optimizer_kwargs: Dict, model: torch.nn.Module):
        module = model.module if isinstance(model, B200DataParallel) else model
        fused = fused_supported(optimizer, optimizer_kwargs, module)
        if self._verbose:
            kind = "sharded (ZeRO-1) " if self._sharded_state else ""
            route = "fused optimizer" if fused else "stock optimizer behind the fused gradient path"
            self._print_device(f"Creating {kind}{route}: {optimizer.__name__}")
        cls = B200FusedOptimizer if fused else B200StockOptimizer   # any torch.optim class works (extensions.py:53-78)
        bucket_mb = None
        ddp_cfg = getattr(self, "_ddp_config", None)
        if ddp_cfg is not None and getattr(ddp_cfg, "bucket_cap_mb", None) and not os.environ.get("STK_BUCKET_MB"):
            bucket_mb = float(ddp_cfg.bucket_cap_mb)   # DDPConfig.bucket_cap_mb (stoke/configs.py:178-188); env overrides
        return cls(module, optimizer, optimizer_kwargs, engine=self._engine, grad_accum=self._grad_accum,
                   clip=clip_spec_from_config(self._grad_clip), sharded=self._sharded_state, lp_dtype=self._lp_dtype,
                   state_id=getattr(self, "_state_id", None), bucket_mb=bucket_mb)


class FairscaleOSSExtension(BaseOptimizer):
    """``fairscale_oss=True``: optimizer state (and fp32 master weights) sharded by element range; the fused step pushes
    the updated shard to every rank (parameter all-gather inside the kernel)."""
    _sharded_state = True

    def __init__(self, oss_config=None, verbose: bool = True, **kwargs):
        super().__init__(verbose=verbose, **kwargs)
        self._oss_config = oss_config


class RunnerOptimizerEnum(Enum):
    oss = FairscaleOSSExtension
    base = BaseOptimizer


class B200DataParallel(torch.nn.Module):
    """Thin wrapper returned by ``handle_ddp`` (what ``torch.nn.parallel.DistributedDataParallel`` is to the reference):
    exposes ``.module`` and ``.no_sync()``; with ``broadcast_buffers`` rank 0's module buffers (BatchNorm statistics) are
    pulled by every rank before each forward through one peer-copy kernel over a flat peer-visible buffer."""

    def __init__(self, module: torch.nn.Module, engine, broadcast_buffers: bool = True):
        super().__init__()
        self.module = module
        self._engine = engine
        self._broadcast_buffers = broadcast_buffers and engine.world > 1
        self._buf_flat = None
        self._buf_bytes = 0
        self.require_backward_grad_sync = True
        self._run = None

    def set_forward(self, fn):
        """Calls ``fn`` (``fuse.FusedForward`` over ``self.module``: not a module, so ``parameters()`` and
        ``state_dict()`` stay the user module's) in place of ``self.module``."""
        self._run = fn

    def _flatten_buffers(self):
        bufs = [b for b in self.module.buffers() if b is not None and b.numel() > 0]
        offs, off = [], 0
        for b in bufs:
            offs.append(off)
            off += (b.numel() * b.element_size() + 15) // 16 * 16
        self._buf_bytes = off
        if off == 0:
            self._broadcast_buffers = False
            return
        self._buf_flat = self._engine.alloc(off)
        raw = self._buf_flat.tensor(torch.uint8, off)
        for b, o in zip(bufs, offs):
            nb = b.numel() * b.element_size()
            view = raw[o: o + nb].view(b.dtype).view(b.shape)
            view.copy_(b.contiguous())
            b.data = view

    def forward(self, *args, **kwargs):
        if self._broadcast_buffers and self.require_backward_grad_sync and torch.is_grad_enabled():
            if self._buf_flat is None:
                self._flatten_buffers()
            if self._broadcast_buffers:
                self._engine.bcast(self._buf_flat, self._buf_bytes, root=0)
        return (self.module if self._run is None else self._run)(*args, **kwargs)

    @contextmanager
    def no_sync(self):
        prev = self.require_backward_grad_sync
        self.require_backward_grad_sync = False
        try:
            yield
        finally:
            self.require_backward_grad_sync = prev


class BaseDDP:
    def __init__(self, ddp_config=None, verbose: bool = True, **kwargs):
        self._verbose = verbose
        self._ddp_config = ddp_config

    def handle_ddp(self, model, optimizer, grad_accum: Optional[int], rank: int, engine=None):
        bb = self._ddp_config.broadcast_buffers if self._ddp_config is not None else True
        return B200DataParallel(model, engine, broadcast_buffers=bb), optimizer


class FairscaleSDDPExtension(BaseDDP):
    """``fairscale_sddp=True``: with OSS the gradient reduce is already a reduce-scatter to the owning rank, which is
    SDDP's reduce-to-owner; the wrapper only carries the SDDP config's ``broadcast_buffers``."""

    def __init__(self, sddp_config=None, verbose: bool = True, **kwargs):
        super().__init__(ddp_config=kwargs.get("ddp_config"), verbose=verbose)
        self._sddp_config = sddp_config

    def handle_ddp(self, model, optimizer, grad_accum: Optional[int], rank: int, engine=None):
        return B200DataParallel(model, engine, broadcast_buffers=self._sddp_config.broadcast_buffers), optimizer


class DistributedHandlerEnum(Enum):
    sddp = FairscaleSDDPExtension
    base = BaseDDP
