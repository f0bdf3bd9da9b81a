# -*- coding: utf-8 -*-
"""``Stoke`` -- the declarative training-step facade with the reference's public surface
(/root/reference/stoke/stoke.py: ``__init__`` :124-155, ``model`` :853, ``loss`` :872, ``backward`` :960, ``step`` :990,
``DataLoader`` :737, ``save``/``load`` :1060/:1108, ``zero_grads``/``reset``/``reset_tracking`` :1187-1224,
``detach_and_sync_loss`` :1164, ``barrier`` :1267, print helpers :371-520, properties :1271-1466), so an existing loop

    out = s.model(x); l = s.loss(out, y); s.backward(l); s.step()

runs unchanged.  The bookkeeping that is stoke's own (accumulation cadence ``(counter + 1) % (grad_accum + 1) == 0``
:326-334, loss tracking / EMA :872-958, wrap ordering :306-324) is restated here; everything below the runner seam is the
H100 engine (see distributed.py / fp16.py / extensions.py / optim.py and csrc/).
"""
from contextlib import nullcontext
from typing import Callable, List, Optional, Tuple, Union
from uuid import uuid4

import torch
from torch.utils.data import Dataset
from torch.utils.data.distributed import DistributedSampler

from .configs import ClipGradConfig, ClipGradNormConfig, StokeOptimizer
from .data import BucketedDistributedSampler, StokeDataLoader
from .distributed import RunnerDistEnum
from .extensions import B200DataParallel, RunnerOptimizerEnum
from .fp16 import RunnerFP16Enum
from .fuse import fuse_bn_act
from .io_ops import RunnerIOEnum
from .status import StokeStatus
from .utils import ParamNormalize, zero_optimizer_grads
from .weight_average import WeightAverage


def build_runner(status: StokeStatus, verbose: bool, info_rank, loss, configs: dict):
    """Composes the runner from four mixins chosen by option name, like ``Stoke._build_runner`` (stoke.py:599-657)."""
    dist_cls = RunnerDistEnum.ddp.value if status.is_distributed_ddp else RunnerDistEnum.gpu.value
    fp16_cls = RunnerFP16Enum[status.fp16].value if status.fp16 is not None else RunnerFP16Enum.full.value
    optim_cls = RunnerOptimizerEnum.oss.value if status.oss else RunnerOptimizerEnum.base.value
    io_cls = RunnerIOEnum.ddp.value if status.is_distributed_ddp else RunnerIOEnum.base.value

    def _init_all(self, *args, **kwargs):
        for cls in (dist_cls, fp16_cls, optim_cls, io_cls):
            cls.__init__(self, *args, **kwargs)

    runner = type("StokeRunner", (dist_cls, fp16_cls, optim_cls, io_cls), {"__init__": _init_all})(
        verbose=verbose, batch_size_per_device=status.batch_size, grad_accum_steps=status.grad_accum,
        grad_clip=status.grad_clip, info_rank=info_rank, loss=loss, **configs)
    info = [f"Distributed Mixin: {dist_cls.__name__}", f"Optimizer Mixin: {optim_cls.__name__}",
            f"FP16 Mixin: {fp16_cls.__name__}", f"IO Mixin: {io_cls.__name__}"]
    return runner, info


class Stoke:
    def __init__(self, model: torch.nn.Module, optimizer: StokeOptimizer,
                 loss: Union[Callable, List[Callable], Tuple[Callable]], batch_size_per_device: int,
                 grad_accum_steps: Optional[int] = 1,
                 grad_clip: Optional[Union[ClipGradConfig, ClipGradNormConfig]] = None, gpu: bool = False,
                 fp16=None, distributed=None, fairscale_oss: bool = False, fairscale_sddp: bool = False,
                 fairscale_fsdp: bool = False, configs: Optional[List] = None,
                 info_rank: Optional[Union[int, List[int]]] = 0, verbose: bool = True, ema_weight: float = 0.1):
        self._verbose = verbose
        self._info_rank = info_rank
        self._ema_weight = ema_weight
        self._status = StokeStatus(batch_size_per_device=batch_size_per_device, grad_accum=grad_accum_steps,
                                   grad_clip=grad_clip, gpu=gpu, fp16=fp16, distributed=distributed,
                                   fairscale_oss=fairscale_oss, fairscale_sddp=fairscale_sddp,
                                   fairscale_fsdp=fairscale_fsdp, configs=configs)
        self._model = self._check_model(model)
        self._optimizer = self._check_optimizer(optimizer)
        self._loss = self._check_loss(loss)
        self._runner, class_info = build_runner(self._status, self._verbose, self._info_rank, self._loss, {
            "amp_config": self.amp_config, "apex_config": None, "ddp_config": self.ddp_config,
            "deepspeed_config": None, "horovod_config": None, "oss_config": self.oss_config,
            "sharded_config": self.sddp_config, "fully_sharded_config": None})
        self._runner.setup_distributed()
        if self._verbose:
            dev_id = self.rank if self.rank in ("cpu", "gpu") else self._info_rank
            self.print(f"Printing verbose information on rank(s): {dev_id}")
            self.print(class_info)
            self.print("Automatically handling moving model to GPU(s)...")
        self._model.cuda()
        # wrap order (stoke.py:306-324): optimizer first only for SDDP+OSS
        if self.sharded and self.oss:
            self._optimizer = self._runner.build_optimizer(optimizer=optimizer["optimizer"],
                                                           optimizer_kwargs=optimizer["optimizer_kwargs"],
                                                           model=self._model)
            self._runner.wrap_fp16(model=self._model, optimizer=self._optimizer)
            self._model, self._optimizer = self._runner.wrap_distributed(model=self._model, grad_accum=self.grad_accum,
                                                                         optimizer=self._optimizer)
        else:
            self._model, _ = self._runner.wrap_distributed(model=self._model, grad_accum=self.grad_accum, optimizer=None)
            self._runner.wrap_fp16(model=self._model, optimizer=None)
            self._optimizer = self._runner.build_optimizer(optimizer=optimizer["optimizer"],
                                                           optimizer_kwargs=optimizer["optimizer_kwargs"],
                                                           model=self._model)
        self._forward = self._model
        if self._status.is_fp16_bf16:
            # BatchNorm2d -> [add] -> ReLU chains run as one kernel pass in training (fuse.py); the user's module is left
            # as it is and runs every call the rewritten graph does not apply to
            fused = fuse_bn_act(self.model_access, self._runner.engine)
            if fused is not None and isinstance(self._model, B200DataParallel):
                self._model.set_forward(fused)
            elif fused is not None:
                self._forward = fused
        wa = self._status.weight_average_config
        self._weight_average = WeightAverage(wa, self._optimizer.path, self.model_access) if wa is not None else None
        self.reset_tracking()
        self._status.set_post_init_values(world_size=self.world_size)
        if self._verbose:
            self.print(msg=self._status)

    # ---- checks ----------------------------------------------------------------------------------------------------
    @staticmethod
    def _check_model(model):
        if not isinstance(model, torch.nn.Module):
            raise TypeError(f"Stoke -- Model is not of type torch.nn.Module, currently {type(model)}")
        return model

    @staticmethod
    def _check_optimizer(optimizer):
        if not isinstance(optimizer, dict):
            raise TypeError(f"Stoke -- Optimizer is not of type torch.optim.Optimizer, currently {type(optimizer)}")
        return optimizer

    def _check_loss(self, loss):
        if isinstance(loss, (list, tuple)):
            return [self._check_loss(val) for val in loss]
        if callable(loss):
            return loss
        raise TypeError(f"Stoke -- Loss is not of type Callable, currently {type(loss)}")

    # ---- cadence ---------------------------------------------------------------------------------------------------
    def _check_accum(self) -> bool:
        return (self._grad_accum_counter + 1) % (self.grad_accum + 1) == 0

    def _check_pre_accum(self) -> bool:
        return (self._grad_accum_counter + 1) % (self.grad_accum + 1) == self.grad_accum

    def _set_loss_to_zero(self):
        return type(self._loss)([0.0] * len(self._loss)) if isinstance(self._loss, (list, tuple)) else 0.0

    def reset_ema(self):
        self._rolling_mean_loss = self._set_loss_to_zero()
        self._rolling_loss_steps = 0

    # ---- the four calls ----------------------------------------------------------------------------------------------
    def model(self, *args, **kwargs):
        with self._runner.model_context:
            return self._forward(*args, **kwargs)

    def loss(self, *args, **kwargs):
        with self._runner.loss_context:
            multi = isinstance(self._loss, (list, tuple))
            loss = type(self._loss)(fn(*args, **kwargs) for fn in self._loss) if multi else self._loss(*args, **kwargs)
            # The cross-rank mean is launched here and READ LATER: the value lands in a pinned ring and is folded into
            # step_loss / the accumulated loss / the EMA when one of them is looked at (reference: item() + barrier() +
            # all_reduce() + item() per micro-step, stoke/distributed.py:619-646).  No host synchronisation in the loop.
            begin = getattr(self._runner, "sync_loss_begin", None)
            if begin is not None:
                self._loss_queue.append(("loss", begin(loss)))
                if len(self._loss_queue) >= 128:   # far below the ring size; old entries completed long ago
                    self._fold_losses()
            elif multi:
                self._fold_one([self.detach_and_sync_loss(val) for val in loss])
            else:
                self._fold_one(self.detach_and_sync_loss(loss))
            if self.grad_accum > 1 and self.model_access.training:
                loss = type(loss)(val / self.grad_accum for val in loss) if multi else loss / self.grad_accum
            return loss

    def _fold_one(self, synced):
        if isinstance(self._loss, (list, tuple)):
            synced = type(self._loss)(synced)
            self._last = synced
            self._agg = type(self._loss)(a + s for a, s in zip(self._agg, synced))
        else:
            self._last = synced
            self._agg += synced
        self._handle_ema_loss(loss=synced)

    def _fold_losses(self):
        """Materialises the queued loss means in order (the only place the training loop can wait on the device)."""
        queue, self._loss_queue = self._loss_queue, []
        for kind, ticket in queue:
            if kind == "reset":
                self._agg = self._set_loss_to_zero()
            else:
                self._fold_one(self._runner.sync_loss_wait(ticket))

    def _lazy(name):  # noqa: N805 -- the three tracked values fold the queue before they are read
        def get(self):
            if self._loss_queue:
                self._fold_losses()
            return getattr(self, name)

        def put(self, value):
            if getattr(self, "_loss_queue", None):
                self._fold_losses()
            setattr(self, name, value)
        return property(get, put)

    _last_step_loss = _lazy("_last")
    _agg_loss = _lazy("_agg")
    _rolling_mean_loss = _lazy("_ema")
    del _lazy

    def _handle_ema_loss(self, loss):
        self._rolling_loss_steps += 1
        if isinstance(loss, (list, tuple)):
            self._ema = type(self._ema)(self._ema_loss(value=val, current_mean=self._ema[idx]) for idx, val in enumerate(loss))
        else:
            self._ema = self._ema_loss(value=loss, current_mean=self._ema)

    def _ema_loss(self, value: float, current_mean: float) -> float:
        if self._rolling_loss_steps == 1:
            return value
        return (self._ema_weight * value) + ((1.0 - self._ema_weight) * current_mean)

    def backward(self, loss):
        if self._weight_average is not None:
            self._weight_average._check_idle("backward")
        self._grad_accum_counter += 1
        ctx = nullcontext() if self._check_accum() else self._runner.grad_accum_context(self._model)
        with ctx:
            self._runner.backward_call(loss=loss, model=self.model_access, optimizer=self._optimizer)
        self._backward_steps += 1

    def step(self):
        if self._weight_average is not None:
            self._weight_average._check_idle("step")
        if not self._check_accum():
            return
        # a schedule-free optimizer in eval mode refuses the step before anything runs, the weight-average schedule included
        check_train_mode = getattr(self._optimizer, "check_train_mode", None)
        if check_train_mode is not None:
            check_train_mode()
        if self._verbose and self.grad_accum > 0:
            self.print(f"Gradient Accumulation Steps: {self.grad_accum}")
        if self.grad_clip is not None:
            self._runner.clip_grad(self.grad_clip, self.model_access, self._optimizer, oss=self.oss, horovod=False,
                                   deepspeed=False, fsdp=False)
        step_cm = self._runner.step_context(self._optimizer) if self.grad_clip is not None else nullcontext()
        if self._weight_average is not None:
            self._weight_average._schedule(self._optimizer_steps + 1)   # a due update rides in this step
        with step_cm:
            self._runner.step_call(model=self.model_access, optimizer=self._optimizer)
        self._reset()
        self._optimizer_steps += 1

    def _reset(self):
        if self._verbose:
            self.print("Resetting all grad/variables for next optimizer step")
        self.zero_grads()
        self._grad_accum_counter = 0
        if self._loss_queue:
            self._loss_queue.append(("reset", None))   # keeps its place in the order of the queued loss means
        else:
            self._agg = self._set_loss_to_zero()

    # ---- helpers with the reference's names ----------------------------------------------------------------------------
    def print(self, msg, single_line: bool = False):
        self._runner.print_device(msg=msg, rank=self._info_rank, single_line=single_line)

    def print_on_devices(self, msg, rank: Optional[Union[int, List[int]]] = 0):
        self._runner.print_device(msg=msg, rank=rank)

    @staticmethod
    def _fmt(prepend, loss, multiplier=None, single_line=False):
        fmt = (lambda v: f"{v * multiplier if multiplier is not None else v:.3f}")
        if isinstance(loss, (list, tuple)):
            return [f"{prepend} {idx}: {fmt(v)}" for idx, v in enumerate(loss)]
        return f"{prepend}: {fmt(loss)}"

    def print_ema_loss(self, prepend_msg: str = "Current EMA Loss", single_line: bool = False):
        self.print(self._fmt(prepend_msg, self._rolling_mean_loss), single_line=single_line)

    def print_mean_accumulated_synced_loss(self, prepend_msg: str = "Mean Accumulated & Synced Loss",
                                           pre_backwards: bool = True, single_line: bool = False):
        check_fn = self._check_pre_accum if pre_backwards else self._check_accum
        if check_fn():
            if isinstance(self._agg_loss, (list, tuple)):
                # the reference prints the bare scaled values for multiple losses (stoke.py:431-433)
                self.print([val / self.grad_accum for val in self._agg_loss], single_line=single_line)
            else:
                self.print(f"{prepend_msg}: {self._agg_loss / self.grad_accum:.3f}")

    def print_synced_loss(self, loss, prepend_msg: str = "Step Synced Loss", device=None, single_line: bool = False):
        self.print(self._fmt(prepend_msg, self.detach_and_sync_loss(loss, device), multiplier=self.grad_accum),
                   single_line=single_line)

    def print_num_model_parameters(self, normalize: ParamNormalize = ParamNormalize.MILLION):
        self.print(f"Total Trainable Model Parameters: {(self.num_model_parameters / normalize.value):.3f} {normalize.name}")

    def dump_model_parameter_info(self):
        self.print("Dumping all model parameter information to stdout....")
        for name, param in self.model_access.named_parameters():
            if param.requires_grad:
                self.print(f"Name: {name}, Shape: {param.shape}, Device: {param.device}, dtype: {param.dtype}")

    def DataLoader(self, dataset: Dataset, shuffle: bool = False, sampler=None, batch_sampler=None, num_workers: int = 0,
                   collate_fn=None, pin_memory: bool = False, drop_last: bool = False, timeout: float = 0,
                   worker_init_fn=None, multiprocessing_context=None, generator=None, *, prefetch_factor: Optional[int] = None,
                   persistent_workers: bool = False):
        # the reference rejects its own BucketedDistributedSampler here (stoke.py:822-826 vs data.py:111); accept both
        if self.distributed is not None and not isinstance(sampler, (DistributedSampler, BucketedDistributedSampler)):
            raise TypeError("Stoke -- Using a distributed backend requires passing an instance of a "
                            "DistributedSampler to the sampler argument")
        kwargs = dict(batch_size=self.batch_size, shuffle=shuffle, sampler=sampler, batch_sampler=batch_sampler,
                      num_workers=num_workers, collate_fn=collate_fn, pin_memory=pin_memory, drop_last=drop_last,
                      timeout=timeout, worker_init_fn=worker_init_fn, multiprocessing_context=multiprocessing_context,
                      generator=generator, persistent_workers=persistent_workers)
        if num_workers > 0:
            kwargs["prefetch_factor"] = 2 if prefetch_factor is None else prefetch_factor
        return StokeDataLoader(dataset, gpu=self.gpu, fp16=self.fp16, **kwargs)

    def save(self, path: str, name: str = None, extension: str = "pt", create_directory: bool = True,
             extras: Optional[dict] = None):
        name = uuid4() if name is None else name
        wa = self._weight_average._checkpoint() if self._weight_average is not None else None  # collective when sharded
        out_path, tag = self._runner.save(model=self.model_access, optimizer=self.optimizer, path=path,
                                          backward_step=self._backward_steps, grad_accum_step=self._grad_accum_counter,
                                          optimizer_step=self._optimizer_steps, name=name,
                                          scaler_dict=self.fp16_state_dict, extension=extension,
                                          create_directory=create_directory, extras=extras, status=self.status.status,
                                          weight_average=wa)
        self.print(f"Successfully saved model checkpoint to {out_path}/{tag}")
        return out_path, tag

    def load(self, path: str, tag: str, strict: bool = True):
        fn = self.scaler.load_state_dict if self.scaler is not None else None
        wa_fn = self._weight_average._load_checkpoint if self._weight_average is not None else None
        backward_step, grad_accum_step, optimizer_step, extras = self._runner.load(
            model=self.model_access, optimizer=self.optimizer, gpu=self.gpu, path=path, tag=tag, scaler_dict_fn=fn,
            strict=strict, weight_average_fn=wa_fn)
        self._backward_steps, self._grad_accum_counter, self._optimizer_steps = backward_step, grad_accum_step, optimizer_step
        self.print(f"Successfully loaded model checkpoint from {path}/{tag}")
        return extras

    def detach_and_sync_loss(self, loss, device=None):
        return self._runner.detach_and_sync_loss(loss=loss, device=device)

    def zero_grads(self):
        zero_optimizer_grads(optimizer=self._optimizer)

    def reset(self):
        self._reset()

    def reset_tracking(self):
        self._grad_accum_counter = 0
        self._optimizer_steps = 0
        self._backward_steps = 0
        self._loss_queue = []
        self._last = self._set_loss_to_zero()
        self._agg = self._set_loss_to_zero()
        self._ema = self._set_loss_to_zero()
        self._rolling_loss_steps = 0

    def barrier(self):
        self._runner.barrier()

    def close(self):
        """Releases the engine's flat buffers (peer mappings, multicast bindings, per-optimizer device state) and hands the
        model its parameters back in ordinary torch storage.  Under DDP call it on every rank at the same point."""
        if self._loss_queue:
            self._fold_losses()
        opt = getattr(self, "_optimizer", None)
        if opt is not None and hasattr(opt, "close"):
            if self.is_ddp:
                self._runner.barrier()
            opt.close()

    # ---- properties ----------------------------------------------------------------------------------------------------
    @property
    def model_access(self):
        return self._model.module if isinstance(self._model, (B200DataParallel, torch.nn.DataParallel)) else self._model

    step_loss = property(lambda self: self._last_step_loss)
    loss_access = property(lambda self: self._loss)
    optimizer = property(lambda self: self._optimizer)
    scaler = property(lambda self: self._runner.scaler)
    status = property(lambda self: self._status)
    batch_size = property(lambda self: self._status.batch_size)
    effective_batch_size = property(lambda self: self._status.effective_batch_size)
    grad_clip = property(lambda self: self._status.grad_clip)
    grad_accum = property(lambda self: self._status.grad_accum)
    gpu = property(lambda self: self._status.gpu)
    cuda = property(lambda self: self._status.cuda)
    nccl = property(lambda self: self._status.nccl)
    fp16 = property(lambda self: self._status.fp16)
    is_apex = property(lambda self: False)
    is_amp = property(lambda self: self._status.is_fp16_amp)
    distributed = property(lambda self: self._status.distributed)
    is_ddp = property(lambda self: self._status.is_distributed_ddp)
    is_horovod = property(lambda self: False)
    is_deepspeed = property(lambda self: False)
    oss = property(lambda self: self._status.oss)
    sharded = property(lambda self: self._status.sharded)
    fully_sharded = property(lambda self: False)
    world_size = property(lambda self: self._runner.world_size)
    rank = property(lambda self: self._runner.rank)
    ema_loss = property(lambda self: self._rolling_mean_loss)
    engine = property(lambda self: self._runner.engine)
    # the fp32 EMA / SWA of the weights (WeightAverageConfig), None when not configured
    weight_average = property(lambda self: self._weight_average)

    @property
    def fp16_state_dict(self):
        return self.scaler.state_dict() if self.scaler is not None else None

    @property
    def amp_config(self):
        return self._status.amp_config if self.is_amp else None

    @property
    def ddp_config(self):
        return self._status.ddp_config if self.is_ddp else None

    @property
    def oss_config(self):
        return self._status.oss_config if self.oss else None

    @property
    def sddp_config(self):
        return self._status.sddp_config if self.sharded else None

    apex_config = property(lambda self: None)
    deepspeed_config = property(lambda self: None)
    fsdp_config = property(lambda self: None)
    horovod_config = property(lambda self: None)

    @property
    def num_model_parameters(self):
        return sum(p.numel() for p in self.model_access.parameters() if p.requires_grad)
