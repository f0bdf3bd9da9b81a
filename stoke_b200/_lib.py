# -*- coding: utf-8 -*-
"""ctypes binding of libstoke_b200.so (include/stoke_b200.h).  The library is the product: there is no Python or torch
fallback for any entry point -- a missing library or a failing call raises."""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libstoke_b200.so")

STK_MAX_WORLD = 8
STK_IPC_HANDLE_BYTES = 64
F32, BF16, F16 = 0, 1, 2
REDUCE_ALL, REDUCE_SCATTER = 0, 1
NORM_NONE, NORM_L2, NORM_INF, NORM_P = 0, 1, 2, 3
CLIP_NONE, CLIP_NORM, CLIP_VALUE = 0, 1, 2
OPT_ADAM, OPT_ADAMW, OPT_SGD, OPT_NADAM, OPT_RADAM, OPT_ADAMAX = 0, 1, 2, 3, 4, 5
OPT_ADADELTA, OPT_RPROP, OPT_ASGD, OPT_LION = 6, 7, 8, 9
OPT_SF_ADAMW, OPT_SF_SGD, OPT_ADEMAMIX, OPT_RMSPROP_TF, OPT_ADAN = 10, 11, 12, 13, 14
ACT_RELU, ACT_SILU, ACT_HARDSWISH, ACT_RELU6 = 0, 1, 2, 3
RF_FINAL, RF_ZERO_INPUT, RF_UNSCALE = 1, 2, 4
OPT_K1_ALGO, OPT_MEM_MODE, OPT_K1_MAX_BLOCKS, OPT_COOP_LAUNCH, OPT_NVLS_MAX_BLOCKS, OPT_K2_AG_MC = 1, 2, 3, 4, 5, 6
K1_ALGO_LDG, K1_ALGO_BULK, K1_ALGO_NVLS = 0, 1, 2
MAX_GROUPS, MAX_SEGMENTS, LOSS_RING = 8, 64, 256
ERR_INVALID, ERR_CUDA, ERR_STATE, ERR_PEER, ERR_UNSUPPORTED = -1, -2, -3, -4, -5


class StokeB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libstoke_b200: {msg} (status {code})")
        self.code = code


class Caps(C.Structure):
    _fields_ = [("sm_major", C.c_int), ("sm_minor", C.c_int), ("sm_count", C.c_int), ("rank", C.c_int),
                ("world", C.c_int), ("device", C.c_int), ("peer_access", C.c_int), ("multicast", C.c_int),
                ("hbm_bytes", C.c_size_t)]


class ScalerState(C.Structure):
    _fields_ = [("scale", C.c_float), ("growth_factor", C.c_float), ("backoff_factor", C.c_float),
                ("growth_interval", C.c_int32), ("growth_tracker", C.c_int32), ("enabled", C.c_int32),
                ("found_inf", C.c_int32), ("grad_norm", C.c_float), ("opt_steps", C.c_int64),
                ("skipped_steps", C.c_int64)]


class OptimHyper(C.Structure):
    _fields_ = [("kind", C.c_int), ("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double),
                ("eps", C.c_double), ("weight_decay", C.c_double), ("momentum", C.c_double),
                ("dampening", C.c_double), ("nesterov", C.c_int), ("maximize", C.c_int), ("clip_kind", C.c_int),
                ("clip_max_norm", C.c_double), ("clip_value", C.c_double)]


class OptimHyperExt(C.Structure):
    _fields_ = [("momentum_decay", C.c_double), ("decoupled_weight_decay", C.c_int), ("rho", C.c_double),
                ("etaminus", C.c_double), ("etaplus", C.c_double), ("step_size_min", C.c_double),
                ("step_size_max", C.c_double), ("lambd", C.c_double), ("alpha", C.c_double), ("t0", C.c_double)]


class OptimArgs(C.Structure):
    _fields_ = [("hyper", C.POINTER(OptimHyper)), ("n_groups", C.c_int), ("master", C.c_void_p), ("exp_avg", C.c_void_p),
                ("exp_avg_sq", C.c_void_p), ("grad", C.c_void_p), ("grad_dtype", C.c_int), ("grad_raw", C.c_int),
                ("acc", C.c_void_p), ("grad_mul", C.c_double), ("n_local", C.c_size_t),
                ("lp_ptrs", C.POINTER(C.c_void_p)), ("lp_world", C.c_int), ("lp_dtype", C.c_int), ("lp_offset", C.c_size_t),
                ("n_seg", C.c_int), ("seg_local", C.POINTER(C.c_size_t)), ("seg_global", C.POINTER(C.c_size_t)),
                ("n_ranges", C.c_int), ("range_end_vec", C.c_void_p), ("range_group", C.c_void_p),
                ("grid_n", C.c_size_t), ("range_bc", C.c_void_p), ("hyper_ext", C.POINTER(OptimHyperExt)),
                ("group_bc", C.c_void_p), ("exp_avg_slow", C.c_void_p)]


class SfHyper(C.Structure):
    _fields_ = [("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("r", C.c_double),
                ("weight_lr_power", C.c_double), ("warmup_steps", C.c_int64)]


class AdemamixHyper(C.Structure):
    _fields_ = [("alpha", C.c_double), ("beta3", C.c_double), ("alpha_warmup", C.c_int64), ("beta3_warmup", C.c_int64)]


class RmspropTfHyper(C.Structure):
    _fields_ = [("alpha", C.c_double), ("centered", C.c_int32), ("decoupled_decay", C.c_int32),
                ("lr_in_momentum", C.c_int32)]


class AdanHyper(C.Structure):
    _fields_ = [("beta3", C.c_double), ("no_prox", C.c_int32)]


class AdafactorParam(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("state", C.c_uint64), ("numel", C.c_int32), ("factored", C.c_int32),
                ("size", C.c_int32 * 4), ("stride", C.c_int32 * 4), ("contiguous", C.c_int32), ("tile0", C.c_int32),
                ("b0", C.c_int32), ("pad_", C.c_int32), ("line0", C.c_int64), ("out0", C.c_int64), ("rm0", C.c_int64)]


class AdafactorPlan(C.Structure):
    _fields_ = [("n_params", C.c_int32), ("n_tiles", C.c_int32), ("n_b", C.c_int32), ("pad_", C.c_int32),
                ("n_line", C.c_int64), ("n_out", C.c_int64), ("n_rm", C.c_int64), ("workspace_bytes", C.c_size_t)]


class AdafactorHyper(C.Structure):
    _fields_ = [("lr", C.c_double), ("beta2_decay", C.c_double), ("eps1", C.c_double), ("eps2", C.c_double),
                ("d", C.c_double), ("weight_decay", C.c_double), ("eps1_none", C.c_int), ("maximize", C.c_int)]


class AdafactorArgs(C.Structure):
    _fields_ = [("hyper", C.POINTER(AdafactorHyper)), ("n_groups", C.c_int), ("clip_kind", C.c_int),
                ("clip_max_norm", C.c_double), ("clip_value", C.c_double), ("params", C.c_void_p),
                ("plan", C.POINTER(AdafactorPlan)), ("param_group", C.c_void_p), ("steps", C.c_void_p),
                ("master", C.c_void_p), ("state", C.c_void_p), ("workspace", C.c_void_p), ("grad", C.c_void_p),
                ("grad_dtype", C.c_int), ("grad_raw", C.c_int), ("acc", C.c_void_p), ("grad_mul", C.c_double),
                ("lp", C.c_void_p), ("lp_dtype", C.c_int)]


LW_TILE = 8192
LW_LAMB, LW_LARS, LW_STABLE_ADAMW = 0, 1, 2


class LayerwiseParam(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("numel", C.c_int32), ("tile0", C.c_int32)]


class LayerwiseHyper(C.Structure):
    _fields_ = [("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double),
                ("weight_decay", C.c_double), ("momentum", C.c_double), ("dampening", C.c_double),
                ("trust_coefficient", C.c_double), ("bias_correction", C.c_int), ("nesterov", C.c_int),
                ("always_adapt", C.c_int), ("pad_", C.c_int)]


class LayerwiseArgs(C.Structure):
    _fields_ = [("kind", C.c_int), ("hyper", C.POINTER(LayerwiseHyper)), ("n_groups", C.c_int), ("clip_kind", C.c_int),
                ("clip_max_norm", C.c_double), ("clip_value", C.c_double), ("params", C.c_void_p),
                ("n_params", C.c_int), ("n_tiles", C.c_int), ("param_group", C.c_void_p), ("steps", C.c_void_p),
                ("master", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("workspace", C.c_void_p),
                ("grad", C.c_void_p), ("grad_dtype", C.c_int), ("grad_raw", C.c_int), ("acc", C.c_void_p),
                ("grad_mul", C.c_double), ("lp", C.c_void_p), ("lp_dtype", C.c_int)]


Q8_BLOCK = 256


class Adam8bitParam(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("numel", C.c_int32), ("block0", C.c_int32), ("small", C.c_int64)]


class Adam8bitHyper(C.Structure):
    _fields_ = [("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double),
                ("weight_decay", C.c_double)]


class Adam8bitArgs(C.Structure):
    _fields_ = [("hyper", C.POINTER(Adam8bitHyper)), ("n_groups", C.c_int), ("clip_kind", C.c_int),
                ("clip_max_norm", C.c_double), ("clip_value", C.c_double), ("params", C.c_void_p),
                ("block_param", C.c_void_p), ("n_params", C.c_int), ("n_blocks", C.c_int), ("param_group", C.c_void_p),
                ("steps", C.c_void_p), ("master", C.c_void_p), ("code1", C.c_void_p), ("code2", C.c_void_p),
                ("absmax1", C.c_void_p), ("absmax2", C.c_void_p), ("qmap1", C.c_void_p), ("qmap2", C.c_void_p),
                ("small", C.c_void_p), ("n_small", C.c_size_t), ("workspace", C.c_void_p), ("grad", C.c_void_p),
                ("grad_dtype", C.c_int), ("grad_raw", C.c_int), ("acc", C.c_void_p), ("grad_mul", C.c_double),
                ("lp", C.c_void_p), ("lp_dtype", C.c_int)]


class MuonParam(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("x_offset", C.c_uint64), ("a_offset", C.c_uint64), ("rows", C.c_int32),
                ("cols", C.c_int32), ("transposed", C.c_int32), ("param", C.c_int32), ("tile0", C.c_int32),
                ("tri0", C.c_int32), ("full0", C.c_int32), ("pad_", C.c_int32), ("lr_ratio", C.c_double)]


class MuonHyper(C.Structure):
    _fields_ = [("lr", C.c_double), ("weight_decay", C.c_double), ("momentum", C.c_double), ("eps", C.c_double),
                ("ns_a", C.c_double), ("ns_b", C.c_double), ("ns_c", C.c_double), ("nesterov", C.c_int),
                ("ns_steps", C.c_int)]


class MuonArgs(C.Structure):
    _fields_ = [("hyper", C.POINTER(MuonHyper)), ("n_groups", C.c_int), ("clip_kind", C.c_int),
                ("clip_max_norm", C.c_double), ("clip_value", C.c_double), ("params", C.c_void_p),
                ("n_params", C.c_int), ("n_tiles", C.c_int), ("n_tri", C.c_int), ("n_full", C.c_int),
                ("param_group", C.c_void_p), ("steps", C.c_void_p), ("master", C.c_void_p),
                ("momentum_buffer", C.c_void_p), ("x0", C.c_void_p), ("x1", C.c_void_p), ("a", C.c_void_p),
                ("b", C.c_void_p), ("workspace", C.c_void_p), ("grad", C.c_void_p), ("grad_dtype", C.c_int),
                ("grad_raw", C.c_int), ("acc", C.c_void_p), ("grad_mul", C.c_double), ("lp", C.c_void_p),
                ("lp_dtype", C.c_int)]


class SamplerPlan(C.Structure):
    _fields_ = [("n", C.c_int64), ("buckets", C.c_int64), ("batch_size", C.c_int64), ("world", C.c_int64),
                ("rank", C.c_int64), ("drop_last", C.c_int32), ("allow_bucket_overlap", C.c_int32),
                ("shuffle", C.c_int32), ("slice_size", C.c_int64), ("per_bucket", C.c_int64),
                ("slices_per_bucket", C.c_int64), ("rounded_per_bucket", C.c_int64),
                ("rounded_per_replica", C.c_int64), ("bucket_base", C.c_int64), ("bucket_rem", C.c_int64),
                ("n_bucket_batches", C.c_int64), ("n_overlap_batches", C.c_int64), ("n_batches", C.c_int64),
                ("needs_padding", C.c_int32)]


_P = C.c_void_p
_PP = C.POINTER(C.c_void_p)
_SIGNATURES = {
    "stk_version": (C.c_int, []),
    "stk_last_error": (C.c_char_p, [_P]),
    "stk_ctx_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_uint, _PP]),
    "stk_ctx_destroy": (C.c_int, [_P]),
    "stk_caps": (C.c_int, [_P, C.POINTER(Caps)]),
    "stk_mem_alloc_shared": (C.c_int, [_P, C.c_size_t, _PP, C.c_char_p]),
    "stk_mem_open_peers": (C.c_int, [_P, _P, C.c_char_p, _PP]),
    "stk_mem_free_shared": (C.c_int, [_P, _P]),
    "stk_comm_local": (C.c_int, [_P, C.c_char_p]),
    "stk_comm_connect": (C.c_int, [_P, C.c_char_p]),
    "stk_comm_check": (C.c_int, [_P, _P]),
    "stk_comm_poll": (C.c_int, [_P]),
    "stk_multicast_try_bind": (C.c_int, [_P, _P, _PP]),
    "stk_multicast_release": (C.c_int, [_P, _P]),
    "stk_state_create": (C.c_int, [_P, C.POINTER(C.c_int)]),
    "stk_state_select": (C.c_int, [_P, C.c_int]),
    "stk_state_destroy": (C.c_int, [_P, C.c_int]),
    "stk_option_set": (C.c_int, [_P, C.c_int, C.c_int]),
    "stk_option_get": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int)]),
    "stk_profile_enable": (C.c_int, [_P, C.c_int]),
    "stk_profile_read": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    "stk_profile_read_k1_device": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_double), _P]),
    "stk_profile_read_k2_device": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_int), _P]),
    "stk_scaler_set": (C.c_int, [_P, C.POINTER(ScalerState), _P]),
    "stk_scaler_get": (C.c_int, [_P, C.POINTER(ScalerState), _P]),
    "stk_scaler_scale_ptr": (_P, [_P]),
    "stk_grad_accumulate": (C.c_int, [_P, _P, C.c_int, _P, C.c_size_t, C.c_int, C.c_int, _P]),
    "stk_grad_reduce": (C.c_int, [_P, C.c_int, _PP, C.c_int, _PP, _PP, C.c_int, C.c_size_t, C.c_double, C.c_int,
                                  C.c_double, C.c_uint, _P]),
    "stk_grad_norm": (C.c_int, [_P, _P, C.c_int, _P, C.c_size_t, C.c_double, C.c_int, C.c_double, C.c_uint, _P]),
    "stk_grad_scale": (C.c_int, [_P, _P, C.c_size_t, C.c_int, C.c_double, C.c_double, _P]),
    "stk_shard_range": (C.c_int, [C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "stk_optim_step": (C.c_int, [_P, C.POINTER(OptimHyper), _P, _P, _P, _P, C.c_size_t, _PP, C.c_int, C.c_int,
                                 C.c_size_t, _P]),
    "stk_optim_step_ex": (C.c_int, [_P, C.POINTER(OptimArgs), _P]),
    "stk_optim_step_prologue": (C.c_int, [_P, C.POINTER(OptimHyper), C.POINTER(OptimHyperExt), C.c_int, C.c_int, _P, _P,
                                          _P, _P, _P]),
    "stk_sf_step_prologue": (C.c_int, [_P, C.POINTER(SfHyper), C.c_int, _P, _P, _P]),
    "stk_ademamix_step_prologue": (C.c_int, [_P, C.POINTER(OptimHyper), C.POINTER(AdemamixHyper), C.c_int, C.c_int, _P,
                                             _P, _P, _P]),
    "stk_rmsprop_tf_step": (C.c_int, [_P, C.POINTER(OptimArgs), C.POINTER(RmspropTfHyper), _P]),
    "stk_adan_step": (C.c_int, [_P, C.POINTER(OptimArgs), C.POINTER(AdanHyper), _P, _P]),
    "stk_adan_step_prologue": (C.c_int, [_P, C.POINTER(OptimHyper), C.POINTER(AdanHyper), C.c_int, C.c_int, _P, _P, _P,
                                         _P]),
    "stk_step_epilogue": (C.c_int, [_P, _P]),
    "stk_adafactor_plan": (C.c_int, [C.POINTER(AdafactorParam), C.c_int, C.POINTER(AdafactorPlan)]),
    "stk_adafactor_step": (C.c_int, [_P, C.POINTER(AdafactorArgs), _P]),
    "stk_layerwise_step": (C.c_int, [_P, C.POINTER(LayerwiseArgs), _P]),
    "stk_adam8bit_step": (C.c_int, [_P, C.POINTER(Adam8bitArgs), _P]),
    "stk_lion8bit_step": (C.c_int, [_P, C.POINTER(Adam8bitArgs), _P]),
    "stk_ademamix8bit_step": (C.c_int, [_P, C.POINTER(Adam8bitArgs), C.POINTER(AdemamixHyper), _P, _P, _P]),
    "stk_muon_step": (C.c_int, [_P, C.POINTER(MuonArgs), _P]),
    "stk_weight_avg": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_int, C.c_float, _P]),
    "stk_loss_sync": (C.c_int, [_P, _P, C.c_int, C.POINTER(C.c_double), _P]),
    "stk_loss_sync_begin": (C.c_int, [_P, _P, C.c_int, C.POINTER(C.c_int64), _P]),
    "stk_loss_sync_wait": (C.c_int, [_P, C.c_int64, C.POINTER(C.c_double)]),
    "stk_barrier": (C.c_int, [_P, _P]),
    "stk_bcast": (C.c_int, [_P, _PP, C.c_size_t, C.c_int, _P]),
    "stk_bn_act": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_double, _P, _P, C.c_size_t, C.c_size_t, _P]),
    "stk_bn_act_backward": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_size_t, C.c_size_t, _P]),
    "stk_bn_act_ex": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, C.c_double, _P, _P, C.c_size_t, C.c_size_t, _P]),
    "stk_bn_act_backward_ex": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_size_t,
                                         C.c_size_t, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "stk_bn_stats_act": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, C.c_int, C.c_double, C.c_double, _P, _P, _P, _P,
                                   C.c_size_t, C.c_size_t, _P, _P, _P, _P, _P, C.c_double, C.c_double, _P, _P]),
    "stk_randperm": (C.c_int, [C.c_uint64, C.POINTER(C.c_int64), C.c_int, _P]),
    "stk_sampler_plan": (C.c_int, [C.POINTER(SamplerPlan)]),
    "stk_sampler_last_slice": (C.c_int, [C.POINTER(SamplerPlan), C.c_int64, _P]),
    "stk_argsort_tmp_bytes": (C.c_size_t, [C.c_size_t]),
    "stk_argsort_u32": (C.c_int, [_P, _P, C.c_size_t, _P, _P, _P]),
    "stk_sampler_indices": (C.c_int, [_P, C.POINTER(SamplerPlan), _P, _P, _P, _P, _P, _P]),
}
EXPORTS = tuple(_SIGNATURES)

_lib = None
_lock = threading.Lock()


def load():
    """Loads libstoke_b200.so (built in-tree by ``stoke_b200/csrc/build.py`` / ``__graft_entry__.build()``)."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                # not a fallback: the only way forward is the CUDA library, so try to compile it in-tree (nvcc, sm_90a)
                try:
                    from .csrc.build import build as _build

                    _build()
                except Exception as e:  # noqa: BLE001
                    raise StokeB200Error(
                        ERR_STATE, f"{LIB_PATH} is missing and could not be built ({type(e).__name__}: {e}) -- build it "
                        f"with `python stoke_b200/csrc/build.py` (there is no non-CUDA fallback)") from e
            lib = C.CDLL(LIB_PATH)
            for name, (res, args) in _SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype = res
                fn.argtypes = args
            _lib = lib
    return _lib


def check(code, ctx=None):
    if code != 0:
        msg = load().stk_last_error(ctx)
        raise StokeB200Error(code, msg.decode() if msg else "unknown error")


def ptr_array(ptrs):
    arr = (C.c_void_p * len(ptrs))()
    for i, p in enumerate(ptrs):
        arr[i] = p
    return arr
