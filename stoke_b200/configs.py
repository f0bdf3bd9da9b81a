# -*- coding: utf-8 -*-
"""Configuration objects of the ``Stoke(...)`` constructor -- same class names, fields and defaults as the reference
(/root/reference/stoke/configs.py) so existing user code constructs them unchanged.

Only the configs of the path this package implements carry behaviour (``AMPConfig`` :44-65, ``ClipGradConfig`` :99-110,
``ClipGradNormConfig`` :113-127, ``DDPConfig`` :130-188, ``FairscaleOSSConfig`` :576-593, ``FairscaleSDDPConfig`` :596-630).
The Horovod / Apex / DeepSpeed / FSDP configs are accepted for import compatibility and rejected at ``Stoke(...)`` time
with a clear error, because those engines are out of scope (SURVEY.md section 8).
"""
from enum import Enum
from typing import Dict, Optional, Type, TypedDict

import attr
import torch


class HorovodOps(Enum):
    Average = "Average"
    Sum = "Sum"
    Adasum = "Adasum"


class OffloadDevice(Enum):
    none = "none"
    cpu = "cpu"
    nvme = "nvme"


class BackendOptions(Enum):
    nccl = "nccl"
    mpi = " mpi"  # (sic) the reference's value has the leading space, configs.py:40
    gloo = "gloo"


def _cfg(cls):
    return attr.s(auto_attribs=True)(cls)


@_cfg
class AMPConfig:
    """Loss-scaler settings (torch GradScaler semantics, kept on the device by the engine)."""
    backoff_factor: float = 0.5
    growth_factor: float = 2.0
    growth_interval: int = 2000
    init_scale: float = 2.0**16


@_cfg
class ClipGradConfig:
    """Clip by value: ``g = clamp(g, -clip_value, clip_value)`` (applied in registers by the optimizer kernel)."""
    clip_value: float


@_cfg
class ClipGradNormConfig:
    """Clip by total norm: norm reduction fused into the gradient reduce, scaling fused into the optimizer kernel."""
    max_norm: float
    norm_type: float


@_cfg
class DDPConfig:
    """Data-parallel settings.  ``bucket_cap_mb`` sizes the gradient buckets whose reduce is launched from autograd hooks
    while backward is still running (reverse registration order, like torch DDP).  ``gradient_as_bucket_view``,
    ``find_unused_parameters`` and ``static_graph`` are accepted for compatibility: gradients always live in the flat
    peer-visible buffer (a bucket view), unused parameters are detected by the hooks, buckets not launched by a hook are
    flushed in order after backward.  ``no_sync=False`` is accepted with a warning (see distributed.py)."""
    local_rank: Optional[int]
    auto_mpi_discovery: bool = False
    convert_to_sync_batch_norm: bool = False
    backend: BackendOptions = "nccl"
    broadcast_buffers: bool = True
    bucket_cap_mb: int = 25
    find_unused_parameters: bool = False
    gradient_as_bucket_view: bool = False
    init_method: str = "env://"
    no_sync: bool = True
    static_graph: bool = False


@_cfg
class FairscaleOSSConfig:
    """Optimizer-state sharding (ZeRO-1).  ``broadcast_fp16`` is implied in mixed precision (the updated shard is pushed to
    the peers in the model dtype)."""
    broadcast_fp16: bool = False
    force_broadcast_object: bool = False


@_cfg
class FairscaleSDDPConfig:
    """Sharded DDP (ZeRO-2 flavour: gradients reduced to their owner only); requires OSS, like the reference."""
    auto_refresh_trainable: bool = True
    broadcast_buffers: bool = True
    reduce_buffer_size: int = 2**23
    reduce_fp16: bool = False
    sync_models_at_startup: bool = True
    warn_on_trainable_params_changed: bool = True


@_cfg
class WeightAverageConfig:
    """An fp32 moving average of the trainable weights kept by the engine (``Stoke.weight_average``), with the semantics of
    ``torch.optim.swa_utils.AveragedModel`` applied to fp32 copies of the master weights.  ``kind="ema"`` is
    ``multi_avg_fn=get_ema_multi_avg_fn(decay)``; ``kind="swa"`` is the default equal average.  After optimizer step s
    (1-based; accumulation micro-steps do not count) an update is due when ``s > start_step`` and
    ``(s - start_step) % every == 0``.  ``use_buffers`` averages the floating buffers too (AveragedModel's option);
    otherwise the average takes the model's current buffers.  Not in the reference: an extension of this engine."""
    kind: str = "ema"
    decay: float = 0.999
    every: int = 1
    start_step: int = 0
    use_buffers: bool = False

    def __attrs_post_init__(self):
        if self.kind not in ("ema", "swa"):
            raise ValueError(f"Stoke -- WeightAverageConfig kind must be 'ema' or 'swa', got {self.kind!r}")
        if not 0.0 <= float(self.decay) <= 1.0:
            raise ValueError(f"Stoke -- WeightAverageConfig decay must be in [0, 1], got {self.decay}")
        if int(self.every) != self.every or self.every < 1:
            raise ValueError(f"Stoke -- WeightAverageConfig every must be an integer >= 1, got {self.every}")
        if int(self.start_step) != self.start_step or self.start_step < 0:
            raise ValueError(f"Stoke -- WeightAverageConfig start_step must be an integer >= 0, got {self.start_step}")


# ---- accepted for import compatibility only (engines out of scope) -----------------------------------------------------
@_cfg
class ApexConfig:
    cast_model_outputs: Optional[torch.dtype] = None
    convert_to_sync_batch_norm: bool = False
    max_loss_scale: float = 2.0**24
    min_loss_scale: Optional[float] = None
    scaler_per_loss: bool = False
    verbosity: int = 0


@_cfg
class HorovodConfig:
    compression: bool = False
    convert_to_sync_batch_norm: bool = False
    gradient_predivide_factor: float = 1.0
    op: HorovodOps = "Average"
    use_fork_server: bool = False


@_cfg
class FairscaleFSDPConfig:
    bucket_cap_mb: int = 25
    buffer_dtype: Optional[torch.dtype] = None
    clear_autocast_cache: bool = False
    compute_dtype: Optional[torch.dtype] = None
    disable_reshard_on_root: bool = True
    flatten_parameters: bool = True
    force_input_to_fp32: bool = False
    fp32_reduce_scatter: bool = False
    gradient_predivide_factor: Optional[float] = None
    gradient_postdivide_factor: Optional[float] = None
    move_grads_to_cpu: Optional[bool] = None
    move_params_to_cpu: bool = False
    no_broadcast_optim_state: Optional[bool] = False
    reshard_after_forward: bool = True
    verbose: bool = False


@_cfg
class DeepspeedAIOConfig:
    block_size: int = 1048576
    ignore_unused_parameters: bool = True
    overlap_events: bool = True
    queue_depth: int = 8
    single_submit: bool = False
    thread_count: int = 1


@_cfg
class DeepspeedActivationCheckpointingConfig:
    contiguous_memory_optimization: bool = False
    cpu_checkpointing: bool = False
    number_checkpoints: Optional[int] = None
    partition_activations: bool = False
    profile: bool = False
    synchronize_checkpoint_boundary: bool = False


@_cfg
class DeepspeedFlopsConfig:
    detailed: bool = True
    module_depth: int = -1
    output_file: Optional[str] = None
    profile_step: int = 1
    top_modules: int = 1


@_cfg
class DeepspeedFP16Config:
    hysteresis: int = 2
    initial_scale_power: int = 32
    loss_scale: float = 0.0
    loss_scale_window: int = 1000
    min_loss_scale: int = 1000


@_cfg
class DeepspeedOffloadOptimizerConfig:
    buffer_count: int = 4
    device: OffloadDevice = "cpu"
    fast_init: bool = False
    nvme_path: str = "/local_nvme"
    pin_memory: bool = False
    pipeline: bool = False
    pipeline_read: bool = False
    pipeline_write: bool = False


@_cfg
class DeepspeedOffloadParamConfig:
    buffer_count: int = 5
    buffer_size: int = int(1e8)
    device: OffloadDevice = "cpu"
    max_in_cpu: int = int(1e9)
    nvme_path: str = "/local_nvme"
    pin_memory: bool = False


@_cfg
class DeepspeedPLDConfig:
    theta: float = 1.0
    gamma: float = 0.001


@_cfg
class DeepspeedTensorboardConfig:
    output_path: str = ""
    job_name: str = "DeepSpeedJobName"


@_cfg
class DeepspeedZeROConfig:
    allgather_bucket_size: int = int(5e8)
    allgather_partitions: bool = True
    contiguous_gradients: bool = False
    grad_hook: bool = True
    ignore_unused_parameters: bool = True
    legacy_stage1: bool = False
    offload_optimizer: Optional[DeepspeedOffloadOptimizerConfig] = None
    offload_param: Optional[DeepspeedOffloadParamConfig] = None
    overlap_comm: bool = False
    reduce_bucket_size: int = int(5e8)
    reduce_scatter: bool = True
    round_robin_gradients: bool = False
    stage: int = 0
    stage3_max_live_parameters: int = int(1e9)
    stage3_max_reuse_distance: int = int(1e9)
    stage3_prefetch_bucket_size: int = int(5e8)
    stage3_param_persistence_threshold: int = int(1e6)
    stage3_gather_fp16_weights_on_model_save: bool = False
    sub_group_size: int = int(1e12)


@_cfg
class DeepspeedConfig:
    activation_checkpointing: Optional[DeepspeedActivationCheckpointingConfig] = DeepspeedActivationCheckpointingConfig()
    aio: Optional[DeepspeedAIOConfig] = DeepspeedAIOConfig()
    auto_mpi_discovery: bool = True
    disable_allgather: bool = False
    dist_backend: BackendOptions = "nccl"
    distributed_port: int = 29500
    dump_state: bool = False
    flops_profiler: Optional[DeepspeedFlopsConfig] = None
    fp16: Optional[DeepspeedFP16Config] = None
    fp32_allreduce: bool = False
    gradient_predivide_factor: float = 1.0
    init_method: str = "env://"
    prescale_gradients: bool = False
    progressive_layer_drop: Optional[DeepspeedPLDConfig] = None
    sparse_gradients: bool = False
    steps_per_print: int = 10
    tensorboard: Optional[DeepspeedTensorboardConfig] = None
    verbose: bool = True
    wall_clock_breakdown: bool = False
    zero_optimization: Optional[DeepspeedZeROConfig] = DeepspeedZeROConfig()


class StokeOptimizer(TypedDict):
    """``{"optimizer": <uninstantiated torch.optim class>, "optimizer_kwargs": {...}}`` (reference configs.py:754-770)."""
    optimizer: Type[torch.optim.Optimizer]
    optimizer_kwargs: Dict


__all__ = [n for n, v in list(globals().items()) if isinstance(v, type) and v.__module__ == __name__]
