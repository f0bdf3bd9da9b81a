# -*- coding: utf-8 -*-
"""Checkpoint mixins: the reference's single-file 8-key format (/root/reference/stoke/io_ops.py:224-236, 290-322) and its
``stoke-{name}-backward-step-{n}.{ext}`` naming (:49-87), with the flat / sharded optimizer state exported through
``B200FusedOptimizer.state_dict()`` in torch's per-parameter layout (DDP flavour: barrier, rank-0 writes, barrier --
io_ops.py:551-653; sharded state is gathered first like OSS ``consolidate_state_dict``)."""
from enum import Enum
from typing import Callable, Optional

import torch

from .utils import make_folder


class BaseStokeIO:
    def __init__(self, save_rank: int = 0, verbose: bool = True, **kwargs):
        self._save_rank = save_rank
        self._prefix = "stoke"
        self._verbose = verbose

    def _make_tag(self, name: str, backward_step: int) -> str:
        return f"{self._prefix}-{name}-backward-step-{backward_step}"

    def _is_writer(self) -> bool:
        return self.rank in ("cpu", "gpu") or self.rank == self._save_rank

    def save(self, model, optimizer, path: str, backward_step: int, grad_accum_step: int, optimizer_step: int, name: str,
             status: dict, scaler_dict: Optional[dict] = None, extension: str = "pt", create_directory: bool = True,
             extras: Optional[dict] = None, weight_average: Optional[dict] = None):
        tag = f"{self._make_tag(name, backward_step)}.{extension}"
        full = f"{path}/{tag}"
        if self._verbose:
            self._print_device(f"Attempting to save model checkpoint to {full}")
        self.barrier()
        optimizer_dict = optimizer.state_dict()  # collective when the state is sharded: every rank calls it
        # parameters / buffers are typed views of the engine's flat buffers: detach them into ordinary per-tensor storages
        model_dict = {k: (v.detach().clone() if isinstance(v, torch.Tensor) else v) for k, v in model.state_dict().items()}
        if self._is_writer():
            try:
                if create_directory:
                    make_folder(path)
                ckpt = {"backward_step": backward_step, "grad_accum_step": grad_accum_step,
                        "optimizer_step": optimizer_step, "stoke_status": status, "model_state_dict": model_dict,
                        "optimizer_state_dict": optimizer_dict, "scaler_state_dict": scaler_dict, "extras": extras}
                if weight_average is not None:   # the one key averaging adds (WeightAverageConfig)
                    ckpt["weight_average_state_dict"] = weight_average
                torch.save(ckpt, full)
            except OSError as e:
                self._print_device(f"Unable to save model to given path: {full}")
                raise e
        self.barrier()
        return path, tag

    def load(self, model, optimizer, gpu: bool, path: str, tag: str, scaler_dict_fn: Optional[Callable] = None,
             strict: bool = True, weight_average_fn: Optional[Callable] = None):
        self.barrier()
        try:
            load_dict = torch.load(f"{path}/{tag}", map_location=f"cuda:{self.device_id}", weights_only=False)
        except OSError as e:
            self._print_device(f"Unable to load model from given path: {path}/{tag}")
            raise e
        # parameters are views of the flat bucket: load_state_dict copies in place, the views stay attached
        model.load_state_dict(state_dict=load_dict["model_state_dict"], strict=strict)
        optimizer.load_state_dict(load_dict["optimizer_state_dict"])
        if scaler_dict_fn is not None and load_dict["scaler_state_dict"] is not None:
            scaler_dict_fn(load_dict["scaler_state_dict"])
        if weight_average_fn is not None:   # None: a checkpoint without an average starts one afresh
            weight_average_fn(load_dict.get("weight_average_state_dict"))
        self.barrier()
        return load_dict["backward_step"], load_dict["grad_accum_step"], load_dict["optimizer_step"], load_dict["extras"]


class DDPIO(BaseStokeIO):
    pass


class RunnerIOEnum(Enum):
    base = BaseStokeIO
    ddp = DDPIO
