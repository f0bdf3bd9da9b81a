# -*- coding: utf-8 -*-
"""Flag/option validation for ``Stoke(...)`` -- the subset of /root/reference/stoke/status.py this package needs to keep
the constructor signature and its error behaviour (``ValueError`` / ``TypeError``) for the options on the hot path.

Differences from the reference, all deliberate (DESIGN.md "boundary"):
  * ``FP16Options.bf16`` is new: bf16 model/gradients + fp32 master weights (the reference has no bf16 mode; its closest
    semantics are Apex O2, stoke/fp16.py:582-635).
  * ``gpu=False`` is rejected: this package is the sm_90a engine, it has no CPU path.
  * horovod / deepspeed / apex / FSDP raise ``ValueError`` naming the option as out of scope instead of importing engines
    that do not exist here.
"""
import os
from enum import Enum
from typing import List, Optional, Union

import attr
import torch

from .configs import (AMPConfig, ClipGradConfig, ClipGradNormConfig, DDPConfig, FairscaleOSSConfig,
                      FairscaleSDDPConfig, WeightAverageConfig)


class DistributedOptions(Enum):
    horovod = "horovod"
    ddp = "ddp"
    deepspeed = "deepspeed"


class FP16Options(Enum):
    apex_O1 = "apex_O1"
    apex_O2 = "apex_O2"
    amp = "amp"
    deepspeed = "deepspeed"
    bf16 = "bf16"  # extension: bf16 params/grads, fp32 master weights, no loss scaling


def _cuda_available() -> bool:
    return torch.cuda.is_available()


def _value(opt):
    return opt.value if isinstance(opt, Enum) else opt


class StokeStatus:
    _CONFIG_NAMES = ("AMPConfig", "ApexConfig", "DDPConfig", "DeepspeedConfig", "FairscaleOSSConfig",
                     "FairscaleSDDPConfig", "FairscaleFSDPConfig", "HorovodConfig", "WeightAverageConfig")

    def __init__(self, batch_size_per_device: int, grad_accum: Optional[int],
                 grad_clip: Optional[Union[ClipGradConfig, ClipGradNormConfig]], gpu: bool, fp16, distributed,
                 fairscale_oss: bool, fairscale_sddp: bool, fairscale_fsdp: bool, configs: Optional[List]):
        self._configs = {type(c).__name__: c for c in (configs or [])}
        if grad_clip is not None and not isinstance(grad_clip, (ClipGradConfig, ClipGradNormConfig)):
            raise TypeError("Stoke -- grad_clip argument must be of type ClipGradConfig or ClipGradNormConfig")
        self._status = {
            "cuda": _cuda_available(),
            "nccl": torch.distributed.is_available() and torch.distributed.is_nccl_available(),
            "batch_size": batch_size_per_device,
            "grad_accum": grad_accum if grad_accum is not None else 1,
            "grad_clip": grad_clip,
            "gpu": gpu,
            "distributed": _value(distributed),
            "zero": None,
            "oss": fairscale_oss,
            "sharded": fairscale_sddp,
            "fully_sharded": fairscale_fsdp,
            "world_size": -1,
            "fp16": _value(fp16),
        }
        self._validate()

    def _validate(self):
        s = self._status
        if not s["gpu"]:
            raise ValueError("Stoke -- stoke_b200 is the H100 (sm_90a) engine and has no CPU path: pass gpu=True")
        if not s["cuda"]:
            raise ValueError("Stoke -- GPU(s) cannot be used as CUDA is not available")
        if s["distributed"] not in (None, "ddp"):
            raise ValueError(f"Stoke -- distributed backend '{s['distributed']}' is out of scope for stoke_b200 "
                             f"(supported: None, 'ddp')")
        if s["fp16"] not in (None, "amp", "bf16"):
            raise ValueError(f"Stoke -- mixed-precision backend '{s['fp16']}' is out of scope for stoke_b200 "
                             f"(supported: None, 'amp', 'bf16')")
        if s["fully_sharded"]:
            raise ValueError("Stoke -- Fairscale FSDP (ZeRO-3) is out of scope for stoke_b200")
        if s["distributed"] is not None and not s["nccl"]:
            raise ValueError(f"Stoke -- Distributed requires CUDA (currently: {s['cuda']}), GPU (currently: {s['gpu']}), "
                             f"and NCCL (currently: {s['nccl']})")
        if (s["oss"] or s["sharded"]) and s["distributed"] != "ddp":
            raise ValueError(f"Stoke -- Fairscale extensions (currently: oss: {s['oss']}, sddp: {s['sharded']}) "
                             f"requires CUDA, GPU, DDP (currently: {s['distributed'] == 'ddp'}) and NCCL")
        if s["sharded"] and not s["oss"]:
            raise ValueError(f"Stoke -- Fairscale SDDP requires OSS (currently: oss: {s['oss']}, sddp: {s['sharded']})")
        if s["oss"] and isinstance(s["grad_clip"], ClipGradConfig):
            raise ValueError("Stoke -- Fairscale OSS and FSDP do not currently support torch.nn.utils.clip_grad_value_ "
                             f"(currently: {type(s['grad_clip']).__name__})")
        for name in self._configs:
            if name not in self._CONFIG_NAMES:
                raise TypeError(f"Stoke -- unknown config object {name}")

    def set_post_init_values(self, world_size: int):
        self._status["world_size"] = world_size

    # ---- accessors (names follow the reference) ----
    status = property(lambda self: self._status)
    batch_size = property(lambda self: self._status["batch_size"])
    grad_clip = property(lambda self: self._status["grad_clip"])
    grad_accum = property(lambda self: self._status["grad_accum"])
    gpu = property(lambda self: self._status["gpu"])
    cuda = property(lambda self: self._status["cuda"])
    nccl = property(lambda self: self._status["nccl"])
    fp16 = property(lambda self: self._status["fp16"])
    oss = property(lambda self: self._status["oss"])
    sharded = property(lambda self: self._status["sharded"])
    fully_sharded = property(lambda self: self._status["fully_sharded"])
    world_size = property(lambda self: self._status["world_size"])
    zero = property(lambda self: self._status["zero"])
    distributed = property(lambda self: self._status["distributed"])
    is_fp16_apex = property(lambda self: False)
    is_fp16_amp = property(lambda self: self.fp16 == "amp")
    is_fp16_bf16 = property(lambda self: self.fp16 == "bf16")
    is_fp16_deepspeed = property(lambda self: False)
    is_fairscale = property(lambda self: self.oss or self.sharded or self.fully_sharded)
    is_distributed_ddp = property(lambda self: self.distributed == "ddp")
    is_distributed_horovod = property(lambda self: False)
    is_distributed_deepspeed = property(lambda self: False)

    @property
    def effective_batch_size(self):
        return self.batch_size * self.grad_accum * self._status["world_size"]

    @property
    def amp_config(self):
        return self._configs.get("AMPConfig") or AMPConfig()

    @property
    def ddp_config(self):
        cfg = self._configs.get("DDPConfig")
        if cfg is None or cfg.local_rank is None:
            if "LOCAL_RANK" not in os.environ:
                raise KeyError("Stoke -- Device local rank must be defined within the DDPConfig or as env variable "
                               "LOCAL_RANK (set by torchrun)")
            local_rank = int(os.environ["LOCAL_RANK"])
            cfg = DDPConfig(local_rank=local_rank) if cfg is None else attr.evolve(cfg, local_rank=local_rank)
        elif not isinstance(cfg.local_rank, int):
            cfg = attr.evolve(cfg, local_rank=int(cfg.local_rank))  # README passes os.getenv('LOCAL_RANK') (a str)
        return cfg

    @property
    def oss_config(self):
        return self._configs.get("FairscaleOSSConfig") or FairscaleOSSConfig()

    @property
    def sddp_config(self):
        return self._configs.get("FairscaleSDDPConfig") or FairscaleSDDPConfig()

    @property
    def weight_average_config(self) -> Optional[WeightAverageConfig]:
        return self._configs.get("WeightAverageConfig")

    def __repr__(self):
        clip = self.grad_clip
        clip_s = ", ".join(f"{k}: {v}" for k, v in attr.asdict(clip).items()) if clip is not None else "None"
        return (
            "STOKE STATE:\n"
            f"    CUDA AVAILABLE: {self.cuda}\n    NCCL AVAILABLE: {self.nccl}\n    GPU FLAG: {self.gpu}\n"
            f"    FP16 FLAG: {self.fp16}\n    DISTRIBUTED BACKEND: {self.distributed}\n    FAIRSCALE OSS: {self.oss}\n"
            f"    FAIRSCALE SDDP: {self.sharded}\n    FAIRSCALE FSDP: {self.fully_sharded}\n    DEEPSPEED ZeRO: False\n"
            f"    WORLD SIZE: {self.world_size}\n    GRAD ACCUMULATION STEPS: {self.grad_accum}\n"
            f"    BATCH SIZE (PER DEVICE): {self.batch_size}\n"
            f"    EFFECTIVE BATCH SIZE (ALL DEVICES): {self.effective_batch_size}\n    GRAD CLIP: ({clip_s})"
        )
