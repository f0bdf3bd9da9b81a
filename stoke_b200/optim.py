# -*- coding: utf-8 -*-
"""The optimizer objects ``Stoke.optimizer`` hands back.

``B200FusedOptimizer`` -- a ``torch.optim.Optimizer`` (so LR schedulers and ``param_groups`` edits work, README.md:241-250
of the reference) whose ``step()`` is the single fused K2 launch over the flat fp32 master / moment buffers; its sharded
flavour is the ZeRO-1 analogue of fairscale ``OSS`` (/root/reference/stoke/extensions.py:109-141): same ``clip_grad_norm`` /
``consolidate_state_dict`` surface.  Adam, AdamW, SGD(-momentum), NAdam, RAdam, Adamax, Adadelta, Rprop, ASGD and the
package's own ``Lion``, ``AdamWScheduleFree`` and ``SGDScheduleFree``, up to 8 parameter groups (per-group lr / betas / eps / weight decay / momentum ... selected inside
the kernel by element range).
NAdam, RAdam, Adamax, Adadelta and Rprop keep two fp32 state tensors per parameter like Adam (Adamax's ``exp_inf``,
Adadelta's ``acc_delta`` and Rprop's ``step_size`` in the second-moment buffer); ASGD keeps one (``ax``), as does Lion
(``exp_avg``, with no per-step scalars).  Their per-step
scalars, NAdam's ``mu_product`` and ASGD's ``eta`` / ``mu`` are formed on the device by ``stk_optim_step_prologue``, so
none of them reads a scalar back to the host (torch's single-tensor ASGD calls ``.item()`` three times per parameter).
Adadelta, Rprop, ASGD and Lion create their state lazily like torch: a parameter never stepped has no ``state_dict``
entry.  Lion is element-wise and independent of the partition, so under DDP / ``fairscale_oss`` it is sharded like the
other kinds.
``AdamWScheduleFree`` and ``SGDScheduleFree`` (defined here, after facebookresearch/schedule_free) are two more kinds:
``z`` in the first-moment buffer (AdamW's ``exp_avg_sq`` in the second), their per-group running state (``lr_max``,
``weight_sum``; ``k`` is the step count) on the device, advanced by ``stk_sf_step_prologue``, and lazy state without
``step``.  ``train()`` / ``eval()`` swap the master and the model between y and x; a step in eval mode raises.  They are
sharded like the other kinds.
``AdEMAMix`` (defined here, after apple/ml-ademamix) is the one kind with three fp32 state tensors: ``exp_avg_fast`` in
the first-moment buffer, ``exp_avg_sq`` in the second and ``exp_avg_slow`` in a third (``GradPath.M2``), with its
per-step scalars (bias corrections, the alpha and beta3 warm-ups) formed by ``stk_ademamix_step_prologue``.  It is
element-wise and sharded like Adam.
``RMSpropTF`` (defined here, after timm's TensorFlow-style RMSprop) keeps ``square_avg`` in the second-moment buffer
(filled with ones at construction), ``momentum_buffer`` in the first (only when some group has momentum) and ``grad_avg``
in the third (only when some group is centered).  Its per-group alpha and flags go to ``stk_rmsprop_tf_step``; it has no
per-step scalars.  It is element-wise and sharded like Adam.
``Adan`` (defined here, after the official Adan and timm's) is the one kind with four fp32 state tensors: ``exp_avg`` in
the first-moment buffer, ``exp_avg_sq`` in the second, ``exp_avg_diff`` in the third (M2) and ``neg_pre_grad`` in a
fourth (``GradPath.M3``).  Its step count lives in the group (``group["step"]``), like the schedule-free k;
``stk_adan_step_prologue`` forms the step sizes and each parameter's first-step flag, and ``stk_adan_step`` takes beta3,
no_prox and the fourth buffer.  It is element-wise and sharded like Adam.
``torch.optim.Adafactor`` takes its own fused entry point, ``stk_adafactor_step`` (per-parameter reductions: row / column
means of g^2, the parameter's RMS, the update's RMS), with per-parameter step counts on the device and torch's
state_dict layout (``row_var`` / ``col_var`` or ``variance``).  Its state is never sharded: the reductions need whole
parameters on one rank, so at world > 1 (``fairscale_oss=True`` included) it runs replicated on the all-reduce route,
every rank taking the same deterministic step on the same gradients, as the stock route is replicated too.
``LAMB`` and ``LARS`` (defined here; torch.optim has neither) take ``stk_layerwise_step``: per-parameter trust ratios from
two whole-parameter norms, per-parameter step counts on the device, the classes' own state_dict layout, and the same
replicated all-reduce route at world > 1.  ``StableAdamW`` (defined here) is a third kind of that step: its per-parameter
reduction is the RMS that scales its learning rate.
``AdamW8bit`` and ``Adam8bit`` (defined here, after bitsandbytes) take ``stk_adam8bit_step``: Adam's moments as 8-bit
codes, block-wise quantized over 256 elements, with per-parameter step counts on the device, bitsandbytes' state keys
and no fp32 moment buffers; replicated on the all-reduce route at world > 1 (the blocks do not follow shard boundaries).
``Lion8bit`` and ``AdEMAMix8bit`` keep Lion's momentum and AdEMAMix's three moments the same way, on
``stk_lion8bit_step`` and ``stk_ademamix8bit_step`` (one and three quantized states per element), with the same routes.
``torch.optim.Muon`` and ``MuonWithAuxAdamW`` (defined here) take ``stk_muon_step``: momentum, Newton-Schulz batched
over every matrix on bf16 tensor cores, the update; ``momentum_buffer`` in M, per-parameter step counts on the device
only to know which parameters have state.  MuonWithAuxAdamW's AdamW groups then take K2's AdamW with the Muon parameters
skipped through the range table.  Newton-Schulz needs whole matrices: replicated on the all-reduce route at world > 1.
Each fused kind's per-parameter state is one row of ``_STATE_LAYOUT``: torch's keys in order, the flat buffer that holds
each tensor (M, V, M2 or Adafactor's own), its initial value, the groups it exists in, and what a never-stepped
parameter exports.  The buffers ``GradPath`` allocates (``state_buffers``), ``state_dict`` (``export_state``) and
``load_state_dict`` (``import_state``) all follow from that row.  The per-group struct a kind's step takes besides
``OptimHyper`` (``_hyper_of``), or in its place for Adafactor, LAMB and LARS, is built by the kind's row of
``_GROUP_HYPER``; ``GradPath.optimizer_step`` chooses the prologues and the entry point of a K2 kind by its kind.  A new
kind therefore adds a state row, a struct builder and its ``_GROUP_HYPER`` row, and at most one case in that choice.

``B200StockOptimizer`` -- every other ``torch.optim`` class (the reference instantiates whatever class the user passes,
stoke/extensions.py:53-78) and the options the fused step does not cover (amsgrad, capturable, differentiable, more than 8
groups): the gradient path
is still the engine's (K1 reduce with fused cast / unscale / inf test / norm, the clip applied by ``k_grad_scale``); the
update itself is the stock optimizer stepping on per-parameter fp32 views of the flat master / main-grad buffers.
"""
import math
from typing import Callable, Dict, List, NamedTuple, Optional, Tuple, Type, Union

import torch

from . import _lib, layout
from .engine import ClipSpec, Engine, GradPath

_KINDS = {torch.optim.Adam: _lib.OPT_ADAM, torch.optim.AdamW: _lib.OPT_ADAMW, torch.optim.SGD: _lib.OPT_SGD,
          torch.optim.NAdam: _lib.OPT_NADAM, torch.optim.RAdam: _lib.OPT_RADAM, torch.optim.Adamax: _lib.OPT_ADAMAX,
          torch.optim.Adadelta: _lib.OPT_ADADELTA, torch.optim.Rprop: _lib.OPT_RPROP, torch.optim.ASGD: _lib.OPT_ASGD}
# per-step scalars from stk_optim_step_prologue, which takes their OptimHyperExt (_ext_hyper)
_EXT_KINDS = (_lib.OPT_NADAM, _lib.OPT_RADAM, _lib.OPT_ADAMAX, _lib.OPT_ADADELTA, _lib.OPT_RPROP, _lib.OPT_ASGD)
_STOCK_ONLY_TRUE = ("amsgrad", "capturable", "differentiable")
# torch.optim.Adafactor (torch >= 2.5) runs on its own entry point, stk_adafactor_step, not as a kind of K2
_ADAFACTOR = "adafactor"
if hasattr(torch.optim, "Adafactor"):
    _KINDS[torch.optim.Adafactor] = _ADAFACTOR


def _trust_where(cond_a: torch.Tensor, cond_b: torch.Tensor, value: torch.Tensor) -> torch.Tensor:
    """``value`` where both norms are positive, else 1 (torch.where: a NaN norm fails the comparison and gives 1)."""
    one = torch.ones_like(value)
    return torch.where(cond_a > 0, torch.where(cond_b > 0, value, one), one)


class LAMB(torch.optim.Optimizer):
    """LAMB (You et al., "Large Batch Optimization for Deep Learning: Training BERT in 76 minutes", 2019): Adam's update
    direction plus weight decay, scaled per parameter by the trust ratio ||w|| / ||r||.  For one parameter w with
    gradient g and its own step count t (after the increment)::

        m = m.lerp(g, 1 - beta1);  v = v * beta2 + (1 - beta2) * g * g
        bc1, bc2 = (1 - beta1 ** t, 1 - beta2 ** t) if bias_correction else (1, 1)
        r = (m / bc1) / (sqrt(v / bc2) + eps) + weight_decay * w
        trust = ||w|| / ||r|| if (weight_decay != 0 or always_adapt) and ||w|| > 0 and ||r|| > 0 else 1
        w = w - lr * (trust * r)

    ||w|| is taken before this step's update.  A group with ``weight_decay=0`` (biases, LayerNorm weights) therefore takes
    a plain bias-corrected Adam step unless ``always_adapt``.  State per parameter, created at its first step: ``step``
    (0-dim fp32 tensor), ``exp_avg``, ``exp_avg_sq``.  This ``step()`` is plain per-parameter torch: what runs outside the
    engine and on its stock route; inside ``Stoke`` the class runs on the fused sm_90a step (``stk_layerwise_step``)."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-6, weight_decay: float = 0.01,
                 bias_correction: bool = True, always_adapt: bool = False):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay,
                                      bias_correction=bias_correction, always_adapt=always_adapt))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            b1, b2 = group["betas"]
            lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                state = self.state[p]
                if not state:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                t = float(state["step"])
                m, v = state["exp_avg"], state["exp_avg_sq"]
                m.lerp_(g, 1 - b1)
                v.mul_(b2).addcmul_(g, g, value=1 - b2)
                bc1, bc2 = (1 - b1**t, 1 - b2**t) if group["bias_correction"] else (1.0, 1.0)
                r = (m / bc1) / ((v / bc2).sqrt() + eps)
                if wd != 0:
                    r = r + wd * p
                if wd != 0 or group["always_adapt"]:
                    wn, rn = torch.linalg.vector_norm(p), torch.linalg.vector_norm(r)
                    r = r * _trust_where(wn, rn, wn / rn)
                p.add_(r, alpha=-lr)
        return loss


class LARS(torch.optim.Optimizer):
    """LARS (You et al., "Large Batch Training of Convolutional Networks", 2017): SGD whose gradient, weight decay included,
    is scaled per parameter by the trust ratio trust_coefficient ||w|| / (||g|| + weight_decay ||w|| + eps).  For one
    parameter w with gradient g and its own step count t (after the increment)::

        if weight_decay != 0 or always_adapt:
            trust = tc * ||w|| / (||g|| + wd * ||w|| + eps) if ||w|| > 0 and ||g|| > 0 else 1   # g before weight decay
            g = (g + wd * w) * trust
        if momentum != 0:
            buf = g.clone() if t == 1 else buf * momentum + (1 - dampening) * g             # torch SGD's seeding
            g = g + momentum * buf if nesterov else buf
        w = w - lr * g

    A group with ``weight_decay=0`` (biases, BatchNorm weights) therefore takes a plain SGD step unless ``always_adapt``.
    State per parameter, created at its first step: ``step`` (0-dim fp32 tensor) and, with momentum, ``momentum_buffer``.
    Plain per-parameter torch here; inside ``Stoke`` the class runs on the fused sm_90a step (``stk_layerwise_step``)."""

    def __init__(self, params, lr: float = 1.0, momentum: float = 0.9, dampening: float = 0.0, weight_decay: float = 0.0,
                 nesterov: bool = False, trust_coefficient: float = 0.001, eps: float = 1e-8, always_adapt: bool = False):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay,
                                      nesterov=nesterov, trust_coefficient=trust_coefficient, eps=eps,
                                      always_adapt=always_adapt))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            lr, mom, damp, wd = group["lr"], group["momentum"], group["dampening"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                state = self.state[p]
                if not state:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                state["step"] += 1
                t = float(state["step"])
                if wd != 0 or group["always_adapt"]:
                    wn, gn = torch.linalg.vector_norm(p), torch.linalg.vector_norm(g)
                    trust = _trust_where(wn, gn, group["trust_coefficient"] * wn / (gn + wd * wn + group["eps"]))
                    g = g.add(p, alpha=wd).mul_(trust)
                if mom != 0:
                    buf = state.get("momentum_buffer")
                    if t == 1 or buf is None:
                        buf = state["momentum_buffer"] = torch.clone(g).detach()
                    else:
                        buf.mul_(mom).add_(g, alpha=1 - damp)
                    g = g.add(buf, alpha=mom) if group["nesterov"] else buf
                p.add_(g, alpha=-lr)
        return loss


class StableAdamW(torch.optim.Optimizer):
    """StableAdamW (Wortsman et al., "Stable and low-precision training for large-scale vision-language models", 2023,
    Algorithm 2): AdamW with debiased betas in place of bias correction, whose learning rate is scaled down per parameter
    by max(1, RMS), RMS = sqrt(mean(g^2 / v)), so that a rare large gradient meeting a decayed second moment cannot make
    a loss spike.  For one parameter w with gradient g and its own step count t (after the increment), exactly as this
    ``step()`` runs it (b1, b2 are python floats, both 0 at t = 1; every tensor op is one fp32 rounding)::

        b1 = beta1 * (1 - beta1 ** (t - 1)) / (1 - beta1 ** t)
        b2 = beta2 * (1 - beta2 ** (t - 1)) / (1 - beta2 ** t)
        m.lerp_(g, 1 - b1)                                         # exp_avg
        v.mul_(b2).addcmul_(g, g, value=1 - b2)                    # exp_avg_sq
        rms = (g * g).div_(v.clamp(min=eps * eps)).mean().sqrt()   # 0-dim on the parameter's device: no .item()
        lr_t = rms.clamp(min=1.0).reciprocal() * lr
        if weight_decay != 0:
            w.mul_(1 - lr_t * weight_decay)
        w.sub_(lr_t * (m / (v.sqrt() + eps)))

    A NaN anywhere in g gives a NaN RMS, which ``clamp`` keeps: the whole parameter becomes NaN.  State per parameter,
    created at its first step: ``step`` (0-dim fp32 tensor), ``exp_avg``, ``exp_avg_sq``.  This ``step()`` is plain
    per-parameter torch: what runs outside the engine and on its stock route; inside ``Stoke`` the class runs on the
    fused sm_90a step (``stk_layerwise_step``, kind ``STK_LW_STABLE_ADAMW``).  The defaults are this package's own."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.99), eps: float = 1e-6, weight_decay: float = 1e-2):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                state = self.state[p]
                if not state:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                t = float(state["step"])
                b1 = beta1 * (1 - beta1 ** (t - 1)) / (1 - beta1 ** t)
                b2 = beta2 * (1 - beta2 ** (t - 1)) / (1 - beta2 ** t)
                m, v = state["exp_avg"], state["exp_avg_sq"]
                m.lerp_(g, 1 - b1)
                v.mul_(b2).addcmul_(g, g, value=1 - b2)
                rms = (g * g).div_(v.clamp(min=eps * eps)).mean().sqrt()
                lr_t = rms.clamp(min=1.0).reciprocal() * lr
                if wd != 0:
                    p.mul_(1 - lr_t * wd)
                p.sub_(lr_t * (m / (v.sqrt() + eps)))
        return loss


class Lion(torch.optim.Optimizer):
    """Lion (Chen et al., "Symbolic Discovery of Optimization Algorithms", 2023): the sign of an interpolation between
    the momentum and the gradient, with decoupled weight decay applied before the update (as timm and lion-pytorch do).
    For one parameter w with gradient g::

        g = -g if maximize else g
        if weight_decay != 0: w = w * (1 - lr * weight_decay)
        w = w - lr * sign(beta1 * m + (1 - beta1) * g)
        m = beta2 * m + (1 - beta2) * g

    sign is ``torch.sign``: a NaN or a zero interpolation leaves w unchanged.  State per parameter, created at its first
    step: ``step`` (0-dim fp32 tensor; the update does not use it) and ``exp_avg``.  This ``step()`` is plain
    per-parameter torch: what runs outside the engine and on its stock route; inside ``Stoke`` the class runs on the fused
    sm_90a step (``k_optim_step``, kind ``STK_OPT_LION``)."""

    def __init__(self, params, lr: float = 1e-4, betas=(0.9, 0.99), weight_decay: float = 0.0, maximize: bool = False):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), weight_decay=weight_decay, maximize=maximize))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            b1, b2 = group["betas"]
            lr, wd = group["lr"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = -p.grad if group["maximize"] else p.grad
                state = self.state[p]
                if not state:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                m = state["exp_avg"]
                if wd != 0:
                    p.mul_(1 - lr * wd)
                u = m.mul(b1).add_(g, alpha=1 - b1).sign_()
                p.add_(u, alpha=-lr)
                m.mul_(b2).add_(g, alpha=1 - b2)
        return loss


_KINDS[Lion] = _lib.OPT_LION


def _sf_beta1(group) -> float:
    return group["betas"][0] if "betas" in group else group["momentum"]


def _check_train_mode(param_groups):
    if not all(g["train_mode"] for g in param_groups):
        raise RuntimeError("Stoke -- a schedule-free optimizer steps only in train mode: call optimizer.train() "
                           "before training steps and optimizer.eval() before evaluating or saving the evaluated weights")


def _sf_scheduled_lr(group, k: int) -> float:
    """The learning rate of step k + 1 (0-based k): the group's lr times the linear warmup."""
    warmup = group["warmup_steps"]
    return group["lr"] * ((k + 1) / warmup if k < warmup else 1.0)


class _ScheduleFree(torch.optim.Optimizer):
    """What AdamWScheduleFree and SGDScheduleFree share: the group scalars of a step, the y / x swap of ``train()`` and
    ``eval()``, and the refusal to step in eval mode.  Subclasses give ``_direction`` (the update direction d before
    weight decay) and ``_init_state``."""

    @torch.no_grad()
    def _swap(self, to_train: bool):
        for group in self.param_groups:
            if group["train_mode"] == to_train:
                continue
            beta1 = _sf_beta1(group)
            w = 1 - beta1 if to_train else 1 - 1 / beta1
            for p in group["params"]:
                if "z" in self.state[p]:
                    p.lerp_(self.state[p]["z"], w)
            group["train_mode"] = to_train

    def train(self):
        """Parameters to y, the point where gradients are taken: p = lerp(p, z, 1 - beta1)."""
        self._swap(True)

    def eval(self):
        """Parameters to x, the averaged point that is evaluated: p = lerp(p, z, 1 - 1 / beta1)."""
        self._swap(False)

    @torch.no_grad()
    def step(self, closure=None):
        _check_train_mode(self.param_groups)
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            k = group["k"]
            lr = group["scheduled_lr"] = _sf_scheduled_lr(group, k)
            lr_max = group["lr_max"] = max(lr, group["lr_max"])
            weight = ((k + 1) ** group["r"]) * (lr_max ** group["weight_lr_power"])
            weight_sum = group["weight_sum"] = group["weight_sum"] + weight
            ckp1 = weight / weight_sum if weight_sum != 0 else 0.0
            y_lr = lr * (_sf_beta1(group) * (1 - ckp1) - 1)
            wd = group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                state = self.state[p]
                if not state:
                    self._init_state(p, state)
                d = self._direction(p.grad, state, group, k)
                if wd != 0:
                    d = d.add(p, alpha=wd)
                p.lerp_(state["z"], ckp1)
                p.add_(d, alpha=y_lr)
                state["z"].sub_(d, alpha=lr)
            group["k"] = k + 1
        return loss


class AdamWScheduleFree(_ScheduleFree):
    """Schedule-free AdamW (Defazio et al., "The Road Less Scheduled", 2024; facebookresearch/schedule_free's
    ``AdamWScheduleFree``, same arguments, group keys and state keys, with the second-moment bias correction inside the
    denominator as its 1.3+ releases).  No learning-rate schedule and no stopping time: the evaluated weights x are an
    online average of the iterates z, and gradients are taken at y, an interpolation of the two.  Per group, with its
    step count k (0-based, python doubles)::

        lr = group_lr * ((k + 1) / warmup_steps if k < warmup_steps else 1)
        lr_max = max(lr, lr_max);  weight = (k + 1) ** r * lr_max ** weight_lr_power
        weight_sum = weight_sum + weight;  ckp1 = weight / weight_sum (0 if weight_sum == 0)
        bc2 = 1 - beta2 ** (k + 1)

    then for every parameter y with a gradient g::

        v = v * beta2 + (1 - beta2) * g * g;  d = g / (sqrt(v / bc2) + eps)
        if weight_decay != 0: d = d + weight_decay * y          # y before this step's update
        y = lerp(y, z, ckp1);  y = y + lr * (beta1 * (1 - ckp1) - 1) * d;  z = z - lr * d

    ``train()`` moves the parameters to y (lerp(p, z, 1 - beta1)), ``eval()`` to x (lerp(p, z, 1 - 1 / beta1)); a new
    optimizer is in eval mode and ``step()`` raises there, modifying nothing.  ``v / bc2`` is computed as
    ``v * (1 / bc2)``, one rounding the fused kernel reproduces.  State per parameter, created at its first gradient:
    ``z`` (a copy of the parameter) and ``exp_avg_sq``; no ``step``.  ``step()`` leaves ``p.grad`` unmodified.  This
    ``step()`` is plain per-parameter torch: what runs outside the engine and on its stock route; inside ``Stoke`` the
    class runs on the fused sm_90a step (``k_optim_step``, kind ``STK_OPT_SF_ADAMW``).  ``foreach`` is accepted and
    ignored.  BatchNorm running statistics are gathered at y: recompute them at x if the model has any."""

    def __init__(self, params, lr: float = 0.0025, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 warmup_steps: int = 0, r: float = 0.0, weight_lr_power: float = 2.0, foreach: Optional[bool] = None):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 < betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if warmup_steps < 0:
            raise ValueError(f"Invalid warmup_steps: {warmup_steps}")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, r=r, k=0, warmup_steps=int(warmup_steps),
                                      train_mode=False, weight_sum=0.0, lr_max=-1.0, scheduled_lr=0.0,
                                      weight_lr_power=weight_lr_power, weight_decay=weight_decay, foreach=foreach))

    @staticmethod
    def _init_state(p, state):
        state["z"] = torch.clone(p, memory_format=torch.preserve_format)
        state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)

    @staticmethod
    def _direction(g, state, group, k):
        beta2 = group["betas"][1]
        v = state["exp_avg_sq"]
        v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        bc2 = 1 - beta2 ** (k + 1)
        return g / v.mul(1 / bc2).sqrt_().add_(group["eps"])


class SGDScheduleFree(_ScheduleFree):
    """Schedule-free SGD (Defazio et al. 2024; facebookresearch/schedule_free's ``SGDScheduleFree``, same arguments,
    group keys and state keys).  The group scalars are AdamWScheduleFree's with beta1 = momentum (no bc2); for every
    parameter y with a gradient g::

        d = g + weight_decay * y if weight_decay != 0 else g   # y before this step's update
        y = lerp(y, z, ckp1);  y = y + lr * (momentum * (1 - ckp1) - 1) * d;  z = z - lr * d

    ``train()`` / ``eval()`` as AdamWScheduleFree's with beta1 = momentum; ``step()`` raises in eval mode, modifying
    nothing.  State per parameter, created at its first gradient: ``z`` (a copy of the parameter); no ``step``.
    ``step()`` leaves ``p.grad`` unmodified.  Plain per-parameter torch here; inside ``Stoke`` the class runs on the fused
    sm_90a step (``k_optim_step``, kind ``STK_OPT_SF_SGD``).  ``foreach`` is accepted and ignored."""

    def __init__(self, params, lr: float = 1.0, momentum: float = 0.9, weight_decay: float = 0.0, warmup_steps: int = 0,
                 r: float = 0.0, weight_lr_power: float = 2.0, foreach: Optional[bool] = None):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 < momentum < 1.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if warmup_steps < 0:
            raise ValueError(f"Invalid warmup_steps: {warmup_steps}")
        super().__init__(params, dict(lr=lr, momentum=momentum, r=r, k=0, warmup_steps=int(warmup_steps),
                                      train_mode=False, weight_sum=0.0, lr_max=-1.0, scheduled_lr=0.0,
                                      weight_lr_power=weight_lr_power, weight_decay=weight_decay, foreach=foreach))

    @staticmethod
    def _init_state(p, state):
        state["z"] = torch.clone(p, memory_format=torch.preserve_format)

    @staticmethod
    def _direction(g, state, group, k):
        return g


_KINDS[AdamWScheduleFree] = _lib.OPT_SF_ADAMW
_KINDS[SGDScheduleFree] = _lib.OPT_SF_SGD
_SF_KINDS = (_lib.OPT_SF_ADAMW, _lib.OPT_SF_SGD)


def ademamix_schedule(group, t: float) -> Tuple[float, float]:
    """AdEMAMix's ``(alpha_t, beta3_t)`` at step t (after the increment), in python doubles: the linear alpha warm-up
    from 0 and the beta3 warm-up that is linear in half-life from beta1 (apple/ml-ademamix's schedulers)."""
    b1, _, b3 = group["betas"]
    alpha, a_warm, b_warm = group["alpha"], group["alpha_warmup"], group["beta3_warmup"]
    alpha_t = (t / a_warm) * alpha if a_warm is not None and t < a_warm else alpha
    if b_warm is not None and t < b_warm:
        def f(b):
            return math.log(0.5) / math.log(b + 1e-8) - 1

        a = t / b_warm
        beta3_t = 0.5 ** (1 / ((1 - a) * f(b1) + a * f(b3) + 1))
    else:
        beta3_t = b3
    return alpha_t, beta3_t


def _check_ademamix_args(lr, betas, alpha, beta3_warmup, alpha_warmup, eps, weight_decay):
    if lr < 0.0:
        raise ValueError(f"Invalid learning rate: {lr}")
    if eps < 0.0:
        raise ValueError(f"Invalid epsilon value: {eps}")
    if len(betas) != 3 or not all(0.0 <= b < 1.0 for b in betas):
        raise ValueError(f"Invalid beta parameters: {betas}")
    if weight_decay < 0.0:
        raise ValueError(f"Invalid weight_decay value: {weight_decay}")
    if alpha < 0.0:
        raise ValueError(f"Invalid alpha value: {alpha}")
    for name, w in (("beta3_warmup", beta3_warmup), ("alpha_warmup", alpha_warmup)):
        if w is not None and (isinstance(w, bool) or not isinstance(w, int) or w <= 0):
            raise ValueError(f"Invalid {name}: {w} (None or a positive int)")


class AdEMAMix(torch.optim.Optimizer):
    """AdEMAMix (Pagliardini, Ablin and Grangier, "The AdEMAMix Optimizer: Better, Faster, Older", 2024;
    apple/ml-ademamix's arguments, group keys and state keys): Adam with a second, slow EMA of the gradient mixed into
    the numerator.  For one parameter p with gradient g and its own step count t (after the increment), in python
    doubles for the scalars::

        bc1 = 1 - beta1 ** t;  bc2 = 1 - beta2 ** t;  alpha_t, beta3_t = ademamix_schedule(group, t)
        m1 = lerp(m1, g, 1 - beta1)          (beta1 == 0: no exp_avg_fast state, m1 = g)
        m2 = lerp(m2, g, 1 - beta3_t)
        v = v * beta2 + (1 - beta2) * g * g
        u = (m1 * (1 / bc1) + alpha_t * m2) / (sqrt(v) * (1 / sqrt(bc2)) + eps)
        if weight_decay != 0: u = u + weight_decay * p
        p = p - lr * u

    alpha_t ramps linearly from 0 to alpha over ``alpha_warmup`` steps, and beta3_t from beta1 to beta3 over
    ``beta3_warmup`` steps, linearly in half-life; None means no warm-up.  The tensor ops are chosen so that the fused
    kernel can reproduce their CUDA rounding: ``lerp_`` for the two EMAs, multiplication by ``1 / bc1`` and
    ``1 / sqrt(bc2)``, ``add(alpha=)`` (one FFMA) and ``addcmul_`` (g * g rounded first).  State per parameter, created
    at its first step: ``step`` (0-dim fp32 tensor; ``load_state_dict`` also accepts upstream's python int),
    ``exp_avg_fast`` (None in a group with beta1 == 0), ``exp_avg_slow`` and ``exp_avg_sq``.  This ``step()`` is plain
    per-parameter torch: what runs outside the engine and on its stock route; inside ``Stoke`` the class runs on the
    fused sm_90a step (``k_optim_step``, kind ``STK_OPT_ADEMAMIX``)."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999, 0.9999), alpha: float = 2.0,
                 beta3_warmup: Optional[int] = None, alpha_warmup: Optional[int] = None, eps: float = 1e-8,
                 weight_decay: float = 0):
        _check_ademamix_args(lr, betas, alpha, beta3_warmup, alpha_warmup, eps, weight_decay)
        super().__init__(params, dict(lr=lr, betas=tuple(betas), alpha=alpha, beta3_warmup=beta3_warmup,
                                      alpha_warmup=alpha_warmup, eps=eps, weight_decay=weight_decay))

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        for st in self.state.values():   # upstream keeps step as a python int
            if "step" in st and not torch.is_tensor(st["step"]):
                st["step"] = torch.tensor(float(st["step"]), dtype=torch.float32)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            b1, b2, _ = group["betas"]
            lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                state = self.state[p]
                if not state:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["exp_avg_fast"] = torch.zeros_like(p, memory_format=torch.preserve_format) if b1 != 0 else None
                    state["exp_avg_slow"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                t = float(state["step"])
                bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
                alpha_t, beta3_t = ademamix_schedule(group, t)
                m1 = state["exp_avg_fast"]
                if m1 is None:
                    m1 = g
                else:
                    m1.lerp_(g, 1 - b1)
                m2, v = state["exp_avg_slow"], state["exp_avg_sq"]
                m2.lerp_(g, 1 - beta3_t)
                v.mul_(b2).addcmul_(g, g, value=1 - b2)
                denom = v.sqrt().mul_(1 / math.sqrt(bc2)).add_(eps)
                u = m1.mul(1 / bc1).add_(m2, alpha=alpha_t).div_(denom)
                if wd != 0:
                    u.add_(p, alpha=wd)
                p.add_(u, alpha=-lr)
        return loss


_KINDS[AdEMAMix] = _lib.OPT_ADEMAMIX


class RMSpropTF(torch.optim.Optimizer):
    """TensorFlow-style RMSprop (timm's ``RMSpropTF``: its arguments, group keys and state keys), the optimizer of the
    published EfficientNet and MobileNet recipes.  It differs from ``torch.optim.RMSprop`` in three ways: eps goes inside
    the square root, ``square_avg`` starts at ones, and (``lr_in_momentum``) the learning rate is accumulated into the
    momentum buffer.  For one parameter p with gradient g, in timm's order of ops::

        if weight_decay != 0:  p = p * (1 - lr * weight_decay) if decoupled_decay else g = g + weight_decay * p
        square_avg = square_avg + (1 - alpha) * (g * g - square_avg)
        centered:  grad_avg = grad_avg + (1 - alpha) * (g - grad_avg);  avg = sqrt(square_avg - grad_avg ** 2 + eps)
        else:      avg = sqrt(square_avg + eps)
        momentum > 0:  buf = buf * momentum + c * g / avg,  p = p - (1 if lr_in_momentum else lr) * buf,
                       with c = lr if lr_in_momentum else 1
        else:          p = p - lr * g / avg

    State per parameter, created at its first step: ``step`` (0-dim fp32 tensor; ``load_state_dict`` also accepts
    timm's python int), ``square_avg`` (ones), ``momentum_buffer`` (zeros, only in a group with momentum > 0) and
    ``grad_avg`` (zeros, only in a centered group).  This ``step()`` is plain per-parameter torch: what runs outside the
    engine and on its stock route; inside ``Stoke`` the class runs on the fused sm_90a step (``k_optim_step``, kind
    ``STK_OPT_RMSPROP_TF``), which rounds every element as this step does on CUDA."""

    def __init__(self, params, lr: float = 1e-2, alpha: float = 0.9, eps: float = 1e-10, weight_decay: float = 0,
                 momentum: float = 0.0, centered: bool = False, decoupled_decay: bool = False,
                 lr_in_momentum: bool = True):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if alpha < 0.0:
            raise ValueError(f"Invalid alpha value: {alpha}")
        super().__init__(params, dict(lr=lr, alpha=alpha, eps=eps, weight_decay=weight_decay, momentum=momentum,
                                      centered=centered, decoupled_decay=decoupled_decay,
                                      lr_in_momentum=lr_in_momentum))

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        for st in self.state.values():   # timm keeps step as a python int
            if "step" in st and not torch.is_tensor(st["step"]):
                st["step"] = torch.tensor(float(st["step"]), dtype=torch.float32)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            lr, alpha, eps, wd, mom = group["lr"], group["alpha"], group["eps"], group["weight_decay"], group["momentum"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                grad = p.grad
                state = self.state[p]
                if not state:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["square_avg"] = torch.ones_like(p, memory_format=torch.preserve_format)
                    if mom > 0:
                        state["momentum_buffer"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if group["centered"]:
                        state["grad_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                if wd != 0:
                    if group["decoupled_decay"]:
                        p.mul_(1 - lr * wd)
                    else:
                        grad = grad.add(p, alpha=wd)
                square_avg = state["square_avg"]
                square_avg.add_(grad.pow(2) - square_avg, alpha=1 - alpha)
                if group["centered"]:
                    grad_avg = state["grad_avg"]
                    grad_avg.add_(grad - grad_avg, alpha=1 - alpha)
                    avg = square_avg.addcmul(grad_avg, grad_avg, value=-1).add(eps).sqrt_()
                else:
                    avg = square_avg.add(eps).sqrt_()
                if mom > 0:
                    buf = state["momentum_buffer"]
                    buf.mul_(mom)
                    if group["lr_in_momentum"]:
                        buf.addcdiv_(grad, avg, value=lr)
                        p.add_(-buf)
                    else:
                        buf.addcdiv_(grad, avg)
                        p.add_(buf, alpha=-lr)
                else:
                    p.addcdiv_(grad, avg, value=-lr)
        return loss


_KINDS[RMSpropTF] = _lib.OPT_RMSPROP_TF


class Adan(torch.optim.Optimizer):
    """Adan (Xie, Zhou, Li, Lin and Yan, "Adan: Adaptive Nesterov Momentum Algorithm for Faster Optimizing Deep Models",
    2022; the official implementation's and timm's arguments, group keys and state keys): Adam-style moments of the
    gradient and of the gradient difference, with Nesterov momentum folded into the second moment.  With the code's
    convention (beta = 1 - the paper's beta), t = ``group["step"]`` after its increment and bc_i = 1 - beta_i ** t, for
    one parameter p with gradient g and previous gradient g_prev (g itself at the parameter's first step)::

        m = beta1 m + (1 - beta1) g;  d = beta2 d + (1 - beta2) (g - g_prev)
        n = beta3 n + (1 - beta3) (g + beta2 (g - g_prev)) ** 2;  den = sqrt(n) / sqrt(bc3) + eps
        no_prox:  p = p (1 - lr wd) - lr / bc1 * m / den - lr beta2 / bc2 * d / den
        else:     p = (p - lr / bc1 * m / den - lr beta2 / bc2 * d / den) / (1 + lr wd)

    That is the paper's Algorithm 1 with bias correction.  ``step()`` is plain per-parameter torch in the official
    single-tensor order of ops, which the fused kernel rounds like this step on CUDA.  The step count is a python int in
    the group, absent before the first step.  State per parameter, created at its first gradient: ``exp_avg``,
    ``exp_avg_sq``, ``exp_avg_diff`` (zeros) and ``neg_pre_grad`` (-g); no ``step``.  Upstream's ``max_grad_norm``
    (use Stoke's ``grad_clip``) and timm's ``caution`` are not arguments.  ``foreach`` is accepted and ignored.  Inside
    ``Stoke`` the class runs on the fused sm_90a step (``k_optim_step``, kind ``STK_OPT_ADAN``)."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.98, 0.92, 0.99), eps: float = 1e-8, weight_decay: float = 0.0,
                 no_prox: bool = False, foreach: Optional[bool] = None):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if len(betas) != 3 or not all(0.0 <= b < 1.0 for b in betas):
            raise ValueError(f"Invalid beta parameters: {betas}")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, no_prox=no_prox,
                                      foreach=foreach))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            group["step"] = t = group.get("step", 0) + 1
            b1, b2, b3 = group["betas"]
            lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
            bc1, bc2, bc3 = 1 - b1 ** t, 1 - b2 ** t, 1 - b3 ** t
            step_size, step_size_diff, bc3_sqrt = lr / bc1, lr * b2 / bc2, math.sqrt(bc3)
            for p in group["params"]:
                if p.grad is None:
                    continue
                grad = p.grad
                state = self.state[p]
                if not state:
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_diff"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                if "neg_pre_grad" not in state or t == 1:
                    state["neg_pre_grad"] = -grad   # so the first difference is 0
                exp_avg, exp_avg_sq, exp_avg_diff = state["exp_avg"], state["exp_avg_sq"], state["exp_avg_diff"]
                P = state["neg_pre_grad"]
                P.add_(grad)                                             # g - g_prev
                exp_avg.mul_(b1).add_(grad, alpha=1 - b1)
                exp_avg_diff.mul_(b2).add_(P, alpha=1 - b2)
                P.mul_(b2).add_(grad)                                    # g + beta2 (g - g_prev)
                exp_avg_sq.mul_(b3).addcmul_(P, P, value=1 - b3)
                denom = (exp_avg_sq.sqrt() / bc3_sqrt).add_(eps)
                if group["no_prox"]:
                    p.mul_(1 - lr * wd)
                    p.addcdiv_(exp_avg, denom, value=-step_size)
                    p.addcdiv_(exp_avg_diff, denom, value=-step_size_diff)
                else:
                    p.addcdiv_(exp_avg, denom, value=-step_size)
                    p.addcdiv_(exp_avg_diff, denom, value=-step_size_diff)
                    p.div_(1 + lr * wd)
                P.zero_().add_(grad, alpha=-1.0)
        return loss


_KINDS[Adan] = _lib.OPT_ADAN


def create_dynamic_map(signed: bool = True) -> torch.Tensor:
    """The 8-bit dynamic tree quantization map of Dettmers et al. (7 exponent bits, 8 bits in all): 256 ascending fp32
    entries in [-1, 1] (signed) or [0, 1] (unsigned), one of them 0.  For i in 0..6 the midpoints of
    ``linspace(0.1, 1, n_i)`` (fp32; n_i = 2 ** i + 1 signed, 2 ** (i + 1) + 1 unsigned) scaled by 10 ** (i - 6), with
    their negatives in the signed map, then 0 and 1."""
    data = []
    for i in range(7):
        b = torch.linspace(0.1, 1, 2 ** i + 1 if signed else 2 ** (i + 1) + 1)
        mid = (10 ** (i - 6)) * ((b[:-1] + b[1:]) / 2.0)
        data += mid.tolist() + ((-mid).tolist() if signed else [])
    data += [0.0, 1.0]
    return torch.tensor(sorted(data), dtype=torch.float32)


def _memory_view(t: torch.Tensor) -> torch.Tensor:
    """A 1-D view of a dense tensor in its memory order (a channels-last weight in its physical order)."""
    x = t.permute(sorted(range(t.dim()), key=lambda d: -t.stride(d)))
    if not x.is_contiguous():
        raise ValueError("AdamW8bit: parameters and their state must be dense")
    return x.view(-1)


def _sqrt_rn(x: torch.Tensor) -> torch.Tensor:
    """The correctly rounded fp32 square root on every device (taken in double, then rounded once: exact for fp32
    inputs).  torch's CPU ``sqrt`` of fp32 is not always correctly rounded; its CUDA ``sqrt`` and the kernel's are."""
    return x.double().sqrt_().float()


def quantize_blockwise(x: torch.Tensor, qmap: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(uint8 codes, fp32 absmax per block) of a 1-D fp32 tensor: see ``AdamW8bit``."""
    n = x.numel()
    nb = -(-n // _lib.Q8_BLOCK)
    absmax = torch.nn.functional.pad(x, (0, nb * _lib.Q8_BLOCK - n)).view(nb, _lib.Q8_BLOCK).abs().amax(1)
    inv = torch.where(absmax == 0, torch.zeros_like(absmax), absmax.reciprocal())
    y = x * inv.repeat_interleave(_lib.Q8_BLOCK)[:n]
    y = torch.where(torch.isnan(y), torch.zeros_like(y), y)
    hi = torch.searchsorted(qmap, y)   # the number of map entries below y
    lo = (hi - 1).clamp_(min=0)
    hi = hi.clamp_(max=qmap.numel() - 1)
    code = torch.where((y - qmap[lo]).abs() <= (y - qmap[hi]).abs(), lo, hi)
    return code.to(torch.uint8), absmax


def dequantize_blockwise(code: torch.Tensor, qmap: torch.Tensor, absmax: torch.Tensor) -> torch.Tensor:
    """qmap[code] * absmax of the code's block, fp32, 1-D."""
    return qmap[code.long()] * absmax.repeat_interleave(_lib.Q8_BLOCK)[: code.numel()]


def check_8bit_entries(entries: List[Dict], quantized: List[bool], states: Tuple[str, ...] = ("state1", "state2"),
                       maps: Tuple[str, ...] = ("qmap1", "qmap2"), name: str = "AdamW8bit"):
    """Refuses, with ValueError, 8-bit optimizer state a step could not continue from: a dtype of one of ``states``
    that does not match the parameter's ``min_8bit_size`` class (``quantized``: uint8, else fp32), ``maps`` that are not
    256 ascending entries, and maps that differ between parameters.  ``entries``: each parameter's state entry
    (``{}`` where it has none); ``states`` / ``maps``: the class's keys (AdamW8bit's by default; Lion8bit has
    ``state1`` and ``qmap1`` only); ``name``: the class named in the messages.  Returns the checkpoint's maps in the order
    of ``maps``, or None if it holds none."""
    found = None
    for i, (e, quant) in enumerate(zip(entries, quantized)):
        for key in states:
            s = e.get(key)
            want = torch.uint8 if quant else torch.float32
            if s is not None and s.dtype != want:
                raise ValueError(f"{name}: {key} of parameter {i} is {s.dtype}, expected {want} "
                                 f"({'at or above' if quant else 'below'} min_8bit_size)")
        if not quant or any(e.get(key) is None for key in maps):
            continue
        qm = tuple(e[key].detach().float().cpu() for key in maps)
        for key, q in zip(maps, qm):
            if q.numel() != 256 or not bool((q[1:] > q[:-1]).all()):
                raise ValueError(f"{name}: {key} must hold 256 ascending entries")
        if found is None:
            found = qm
        elif not all(torch.equal(a, b) for a, b in zip(found, qm)):
            raise ValueError(f"{name}: the quantization maps differ between parameters (the fused step keeps one "
                             f"{'pair' if len(maps) == 2 else 'map'})")
    return found


class AdamW8bit(torch.optim.Optimizer):
    """AdamW with 8-bit moments (bitsandbytes' ``AdamW8bit``: its arguments and state keys; Dettmers et al., "8-bit
    Optimizers via Block-wise Quantization", 2022), about 2 B of optimizer state per parameter instead of 8.  For one
    parameter w with gradient g and its own step count t (after the increment), every op one fp32 rounding in this order::

        c1 = 1 - beta1 ** t;  c2 = sqrt(1 - beta2 ** t)                     (python doubles)
        m = deq(m) * beta1 + g * (1 - beta1);  v = deq(v) * beta2 + (g * g) * (1 - beta2)
        if weight_decay != 0: w = w * (1 - lr * weight_decay)
        w = w - (m / (sqrt(v) + eps * c2)) * (lr * c2 / c1)
        m, v = quant(m), quant(v)                                            (the update uses the unquantized m, v)

    sqrt(v) is the correctly rounded fp32 square root on every device.  Quantization is block-wise over the parameter's
    elements in memory order (a channels-last weight in its physical
    order), 256 elements per block, the last one possibly short.  Per block absmax = amax(|x|) and
    n = x * (absmax == 0 ? 0 : 1 / absmax); the code is the index of the map entry nearest to n (fp32 distances
    |n - q|, equal distances to the lower index), and deq(code) = qmap[code] * absmax.  n is clamped into
    [qmap[0], qmap[255]] first, so an n beyond the map (+inf where 1 / absmax overflows, for a subnormal absmax at or
    below 2 ** -128) takes the code of its nearer end.  m takes the signed map
    ``qmap1``, v the unsigned ``qmap2`` (``create_dynamic_map``).

    Non-finite values: a NaN in a block makes its absmax NaN, an inf (and no NaN) makes it inf.  A NaN n -- a NaN or inf
    element, or any element of a block whose absmax is NaN -- takes the code of 0 (the entry nearest to 0), and every
    element of a block whose absmax is not finite decodes to NaN at the next step (qmap[code] * inf is NaN for the code
    of 0 and +-inf otherwise; a finite element of an inf block has n = 0).

    A parameter with fewer than ``min_8bit_size`` elements keeps fp32 ``state1`` / ``state2`` and takes the same update
    without quantization.  State per parameter, created at its first step: ``step`` (0-dim fp32 tensor;
    ``load_state_dict`` also accepts upstream's python int), ``state1``, ``qmap1``, ``state2``, ``qmap2``, ``absmax1``,
    ``absmax2`` (no maps or absmax for a small parameter).  ``optim_bits`` is accepted and ignored; ``amsgrad``,
    ``percentile_clipping != 100``, ``block_wise=False``, ``is_paged`` and ``args`` raise ValueError.  This ``step()``
    is plain per-parameter torch: what runs outside the engine and on its stock route; inside ``Stoke`` the class runs
    on the fused sm_90a step (``stk_adam8bit_step``)."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 amsgrad: bool = False, optim_bits: int = 32, args=None, min_8bit_size: int = 4096,
                 percentile_clipping: int = 100, block_wise: bool = True, is_paged: bool = False):
        _refuse_8bit_options(type(self).__name__, amsgrad=(amsgrad, amsgrad), args=(args, args is not None),
                             percentile_clipping=(percentile_clipping, percentile_clipping != 100),
                             block_wise=(block_wise, not block_wise), is_paged=(is_paged, is_paged))
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay,
                                      min_8bit_size=int(min_8bit_size)))
        self._maps: Dict[torch.device, Tuple[torch.Tensor, torch.Tensor]] = {}

    def _init_state(self, p, state, quant: bool):
        state["step"] = torch.tensor(0.0, dtype=torch.float32)
        if not quant:
            state["state1"] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
            state["state2"] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
            return
        if p.device not in self._maps:
            self._maps[p.device] = (create_dynamic_map(True).to(p.device), create_dynamic_map(False).to(p.device))
        q1, q2 = self._maps[p.device]
        nb = -(-p.numel() // _lib.Q8_BLOCK)
        state["state1"] = torch.zeros_like(p, dtype=torch.uint8, memory_format=torch.preserve_format)
        state["qmap1"] = q1
        state["state2"] = torch.zeros_like(p, dtype=torch.uint8, memory_format=torch.preserve_format)
        state["qmap2"] = q2
        state["absmax1"] = torch.zeros(nb, dtype=torch.float32, device=p.device)
        state["absmax2"] = torch.zeros(nb, dtype=torch.float32, device=p.device)

    def load_state_dict(self, state_dict):
        ids = [i for g in state_dict["param_groups"] for i in g["params"]]
        quantized = [p.numel() >= sg.get("min_8bit_size", g["min_8bit_size"])
                     for sg, g in zip(state_dict["param_groups"], self.param_groups) for p in g["params"]]
        params = [p for g in self.param_groups for p in g["params"]]
        check_8bit_entries([state_dict["state"].get(i, {}) for i in ids], quantized)
        super().load_state_dict(state_dict)
        for p in params:   # torch casts floating-point state to the parameter's dtype; the codes stay uint8
            st = self.state.get(p)
            if not st:
                continue
            if "step" in st and not torch.is_tensor(st["step"]):   # upstream keeps step as a python int
                st["step"] = torch.tensor(float(st["step"]), dtype=torch.float32)
            if "qmap1" in st:
                st["state1"], st["state2"] = st["state1"].to(torch.uint8), st["state2"].to(torch.uint8)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            b1, b2 = group["betas"]
            lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                state = self.state[p]
                if not state:
                    self._init_state(p, state, p.numel() >= group["min_8bit_size"])
                state["step"] += 1
                t = float(state["step"])
                c1, c2 = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
                g = p.grad if p.grad.stride() == p.stride() else torch.empty_like(p).copy_(p.grad)
                g, w = _memory_view(g), _memory_view(p)
                quant = "qmap1" in state
                s1, s2 = _memory_view(state["state1"]), _memory_view(state["state2"])
                if quant:
                    m = dequantize_blockwise(s1, state["qmap1"], state["absmax1"])
                    v = dequantize_blockwise(s2, state["qmap2"], state["absmax2"])
                else:
                    m, v = s1, s2
                m.mul_(b1).add_(g * (1 - b1))
                v.mul_(b2).add_(g.mul(g).mul_(1 - b2))
                if wd != 0:
                    w.mul_(1 - lr * wd)
                w.sub_(m.div(_sqrt_rn(v).add_(eps * c2)).mul_(lr * c2 / c1))
                if quant:
                    for s, x, q, a in ((s1, m, state["qmap1"], state["absmax1"]), (s2, v, state["qmap2"], state["absmax2"])):
                        code, absmax = quantize_blockwise(x, q)
                        s.copy_(code)
                        a.copy_(absmax)
        return loss


class Adam8bit(AdamW8bit):
    """bitsandbytes' ``Adam8bit``: ``AdamW8bit`` with ``weight_decay=0`` by default (the decay, when given, is decoupled
    as in AdamW8bit)."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 amsgrad: bool = False, optim_bits: int = 32, args=None, min_8bit_size: int = 4096,
                 percentile_clipping: int = 100, block_wise: bool = True, is_paged: bool = False):
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                         optim_bits=optim_bits, args=args, min_8bit_size=min_8bit_size,
                         percentile_clipping=percentile_clipping, block_wise=block_wise, is_paged=is_paged)


def _refuse_8bit_options(cls_name: str, **bad):
    """ValueError for the first bitsandbytes option given as ``name=(value, refused)`` with ``refused`` true."""
    for name, (value, refused) in bad.items():
        if refused:
            raise ValueError(f"{cls_name}: {name}={value!r} is not supported")


def _q8_zeros(p: torch.Tensor, dtype: torch.dtype, lead: int = 0) -> torch.Tensor:
    """Zero state for p: shaped and strided like p, or with ``lead`` > 0 shaped ``(lead, *p.shape)``, each ``[k]`` laid
    out like p (so ``_memory_view`` of it walks p's memory order)."""
    if not lead:
        return torch.zeros_like(p, dtype=dtype, memory_format=torch.preserve_format)
    flat = torch.zeros(lead * p.numel(), dtype=dtype, device=p.device)
    return flat.as_strided((lead, *p.shape), (p.numel(), *p.stride()))


class _Blockwise8bit(torch.optim.Optimizer):
    """What Lion8bit and AdEMAMix8bit share: the maps cached per device, state creation from ``_STATES`` and loading.
    ``_STATES``: per state key, (its map key, its absmax key, its leading dimension: 0 or the number of tensors it
    stacks); ``_MAPS``: the map keys with their signedness, in order."""
    _STATES: Tuple[Tuple[str, str, str, int], ...] = ()
    _MAPS: Tuple[Tuple[str, bool], ...] = ()

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._maps: Dict[torch.device, Dict[str, torch.Tensor]] = {}

    def _init_state(self, p, state, quant: bool):
        state["step"] = torch.tensor(0.0, dtype=torch.float32)
        if not quant:
            for key, _, _, lead in self._STATES:
                state[key] = _q8_zeros(p, torch.float32, lead)
            return
        if p.device not in self._maps:
            self._maps[p.device] = {k: create_dynamic_map(signed).to(p.device) for k, signed in self._MAPS}
        nb = -(-p.numel() // _lib.Q8_BLOCK)
        for key, qkey, _, lead in self._STATES:
            state[key] = _q8_zeros(p, torch.uint8, lead)
            state[qkey] = self._maps[p.device][qkey]
        for _, _, akey, lead in self._STATES:
            state[akey] = torch.zeros((lead, nb) if lead else (nb,), dtype=torch.float32, device=p.device)

    def load_state_dict(self, state_dict):
        ids = [i for g in state_dict["param_groups"] for i in g["params"]]
        quantized = [p.numel() >= sg.get("min_8bit_size", g["min_8bit_size"])
                     for sg, g in zip(state_dict["param_groups"], self.param_groups) for p in g["params"]]
        params = [p for g in self.param_groups for p in g["params"]]
        check_8bit_entries([state_dict["state"].get(i, {}) for i in ids], quantized,
                           tuple(s[0] for s in self._STATES), tuple(m[0] for m in self._MAPS), type(self).__name__)
        super().load_state_dict(state_dict)
        for p in params:
            st = self.state.get(p)
            if not st:
                continue
            if "step" in st and not torch.is_tensor(st["step"]):   # upstream keeps step as a python int
                st["step"] = torch.tensor(float(st["step"]), dtype=torch.float32)
            # torch casts floating-point state to the parameter's dtype (the codes back to uint8 here), and a checkpoint
            # may hold the tensors in any strides: each goes back to the layout _init_state gives it
            for key, _, _, lead in self._STATES:
                if key in st:
                    src = st[key]
                    st[key] = _q8_zeros(p, torch.uint8 if "qmap1" in st else torch.float32, lead)
                    st[key].copy_(src.reshape(st[key].shape))

    def _views(self, p, state):
        """(quantized, per state key: its memory-order views, one per stacked tensor)"""
        return "qmap1" in state, {key: [_memory_view(state[key][k]) for k in range(lead)] if lead else
                                  [_memory_view(state[key])] for key, _, _, lead in self._STATES}

    @staticmethod
    def _deq(state, key, qkey, akey, lead, views):
        absmax = state[akey]
        return [dequantize_blockwise(v, state[qkey], absmax[k] if lead else absmax) for k, v in enumerate(views)]

    def _store(self, state, key, qkey, akey, lead, views, xs):
        absmax = state[akey]
        for k, (v, x) in enumerate(zip(views, xs)):
            code, a = quantize_blockwise(x, state[qkey])
            v.copy_(code)
            (absmax[k] if lead else absmax).copy_(a)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                state = self.state[p]
                if not state:
                    self._init_state(p, state, p.numel() >= group["min_8bit_size"])
                state["step"] += 1
                g = p.grad if p.grad.stride() == p.stride() else torch.empty_like(p).copy_(p.grad)
                g, w = _memory_view(g), _memory_view(p)
                quant, views = self._views(p, state)
                # the unquantized state of this step: dequantized copies, or the fp32 state itself (updated in place)
                xs = {s[0]: self._deq(state, *s, views[s[0]]) if quant else views[s[0]] for s in self._STATES}
                self._update(group, float(state["step"]), w, g, xs)
                if quant:
                    for s in self._STATES:
                        self._store(state, *s, views[s[0]], xs[s[0]])
        return loss

    def _update(self, group, t: float, w, g, xs):
        raise NotImplementedError


class Lion8bit(_Blockwise8bit):
    """Lion with 8-bit momentum (bitsandbytes' ``Lion8bit``: its arguments and state keys), about 1 B of optimizer state
    per parameter instead of 4.  For one parameter w with gradient g, every op one fp32 rounding in this order::

        if weight_decay != 0: w = w * (1 - lr * weight_decay)
        c = deq(m) * beta1 + g * (1 - beta1);  s = (c > 0) - (c < 0)       (torch.sign: NaN and +-0 give 0)
        w = w - s * lr
        m = deq(m) * beta2 + g * (1 - beta2);  m = quant(m)

    Quantization is ``AdamW8bit``'s (block-wise over 256 elements in memory order, its clamping, tie and NaN rules) on
    the signed map ``qmap1``.  A parameter with fewer than ``min_8bit_size`` elements keeps an fp32 ``state1`` and takes
    the same update without quantization.  State per parameter, created at its first step: ``step`` (0-dim fp32 tensor;
    the update does not use it; ``load_state_dict`` also accepts a python int), ``state1`` (uint8 codes of exp_avg),
    ``qmap1``, ``absmax1``.  ``args``, ``percentile_clipping != 100``, ``block_wise=False`` and ``is_paged`` raise
    ValueError.  No parity with bitsandbytes is claimed.  This ``step()`` is plain per-parameter torch: what runs
    outside the engine and on its stock route; inside ``Stoke`` the class runs on the fused sm_90a step
    (``stk_lion8bit_step``)."""
    _STATES = (("state1", "qmap1", "absmax1", 0),)
    _MAPS = (("qmap1", True),)

    def __init__(self, params, lr: float = 1e-4, betas=(0.9, 0.99), weight_decay: float = 0.0, args=None,
                 min_8bit_size: int = 4096, percentile_clipping: int = 100, block_wise: bool = True,
                 is_paged: bool = False):
        _refuse_8bit_options(type(self).__name__, args=(args, args is not None),
                             percentile_clipping=(percentile_clipping, percentile_clipping != 100),
                             block_wise=(block_wise, not block_wise), is_paged=(is_paged, is_paged))
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), weight_decay=weight_decay,
                                      min_8bit_size=int(min_8bit_size)))

    def _update(self, group, t, w, g, xs):
        b1, b2 = group["betas"]
        lr, wd = group["lr"], group["weight_decay"]
        m = xs["state1"][0]
        if wd != 0:
            w.mul_(1 - lr * wd)
        w.sub_(m.mul(b1).add_(g.mul(1 - b1)).sign_().mul_(lr))
        m.mul_(b2).add_(g.mul(1 - b2))


def ademamix8bit_scalars(group, t: float) -> Tuple[float, float, float, float]:
    """AdEMAMix8bit's per-step scalars at step t (after the increment), in python doubles: ``(1 / bc1, 1 / sqrt(bc2),
    alpha_t, beta3_t)``, the numbers ``AdEMAMix.step`` uses."""
    b1, b2, _ = group["betas"]
    alpha_t, beta3_t = ademamix_schedule(group, t)
    return 1 / (1 - b1 ** t), 1 / math.sqrt(1 - b2 ** t), alpha_t, beta3_t


class AdEMAMix8bit(_Blockwise8bit):
    """AdEMAMix with 8-bit state: ``AdEMAMix``'s arguments and warm-ups, with its three moments stored as 8-bit codes,
    about 3 B of optimizer state per parameter instead of 12.  For one parameter w with gradient g and its own step count
    t (after the increment), the scalars ``ademamix8bit_scalars`` in python doubles, then every op one fp32 rounding in
    this order::

        m1 = deq(m1) * beta1 + g * (1 - beta1)
        m2 = deq(m2) * beta3_t + g * (1 - beta3_t)
        nu = deq(nu) * beta2 + (g * g) * (1 - beta2)
        den = sqrt(nu) * (1 / sqrt(bc2)) + eps
        u = (m1 * (1 / bc1) + m2 * alpha_t) / den
        if weight_decay != 0: u = u + w * weight_decay
        w = w - u * lr
        m1, m2, nu = quant(m1), quant(m2), quant(nu)                     (the update uses the unquantized state)

    sqrt is the correctly rounded fp32 square root on every device.  Quantization is ``AdamW8bit``'s (block-wise over
    256 elements in memory order, its clamping, tie and NaN rules): m1 (fast) and m2 (slow) on the signed map ``qmap1``,
    nu on the unsigned ``qmap2``.  A parameter with fewer than ``min_8bit_size`` elements keeps fp32 state and takes the
    same update without quantization.  State per parameter, created at its first step: ``step`` (0-dim fp32 tensor;
    ``load_state_dict`` also accepts a python int), ``state1`` (uint8, shaped ``(2, *p.shape)``: the codes of m1 then
    m2), ``qmap1``, ``state2`` (the codes of nu), ``qmap2``, ``absmax1`` (shaped ``(2, n_blocks)``) and ``absmax2``; a
    small parameter has fp32 ``state1`` ``(2, *p.shape)`` and ``state2``.  ``betas[0] == 0`` raises ValueError.  This
    ``step()`` is plain per-parameter torch: what runs outside the engine and on its stock route; inside ``Stoke`` the
    class runs on the fused sm_90a step (``stk_ademamix8bit_step``)."""
    _STATES = (("state1", "qmap1", "absmax1", 2), ("state2", "qmap2", "absmax2", 0))
    _MAPS = (("qmap1", True), ("qmap2", False))

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999, 0.9999), alpha: float = 2.0,
                 beta3_warmup: Optional[int] = None, alpha_warmup: Optional[int] = None, eps: float = 1e-8,
                 weight_decay: float = 0, min_8bit_size: int = 4096):
        _check_ademamix_args(lr, betas, alpha, beta3_warmup, alpha_warmup, eps, weight_decay)
        if betas[0] == 0:
            raise ValueError(f"{type(self).__name__}: betas[0] = 0 is not supported")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), alpha=alpha, beta3_warmup=beta3_warmup,
                                      alpha_warmup=alpha_warmup, eps=eps, weight_decay=weight_decay,
                                      min_8bit_size=int(min_8bit_size)))

    def _update(self, group, t, w, g, xs):
        b1, b2, _ = group["betas"]
        lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
        c1, c2, alpha_t, beta3_t = ademamix8bit_scalars(group, t)
        (m1, m2), (nu,) = xs["state1"], xs["state2"]
        m1.mul_(b1).add_(g.mul(1 - b1))
        m2.mul_(beta3_t).add_(g.mul(1 - beta3_t))
        nu.mul_(b2).add_(g.mul(g).mul_(1 - b2))
        den = _sqrt_rn(nu).mul_(c2).add_(eps)
        u = m1.mul(c1).add_(m2.mul(alpha_t)).div_(den)
        if wd != 0:
            u.add_(w.mul(wd))
        w.sub_(u.mul_(lr))


# The 8-bit classes run on their own entry points (block-wise quantized state), not as kinds of K2: AdamW8bit and
# Adam8bit on stk_adam8bit_step, Lion8bit on stk_lion8bit_step, AdEMAMix8bit on stk_ademamix8bit_step
_ADAM8BIT, _LION8BIT, _ADEMAMIX8BIT = "adam8bit", "lion8bit", "ademamix8bit"
_KINDS[AdamW8bit] = _ADAM8BIT
_KINDS[Adam8bit] = _ADAM8BIT
_KINDS[Lion8bit] = _LION8BIT
_KINDS[AdEMAMix8bit] = _ADEMAMIX8BIT
_Q8_KINDS = {_ADAM8BIT: 2, _LION8BIT: 1, _ADEMAMIX8BIT: 3}   # kind -> quantized states per element

# LAMB, LARS and StableAdamW run on their own entry point, stk_layerwise_step (per-parameter trust ratios or RMS), not
# as kinds of K2
_LAMB, _LARS, _STABLE_ADAMW = "lamb", "lars", "stable_adamw"
_KINDS[LAMB] = _LAMB
_KINDS[LARS] = _LARS
_KINDS[StableAdamW] = _STABLE_ADAMW
_LAYERWISE = {_LAMB: _lib.LW_LAMB, _LARS: _lib.LW_LARS, _STABLE_ADAMW: _lib.LW_STABLE_ADAMW}


def muon_lr_ratio(adjust_lr_fn: Optional[str], rows: int, cols: int) -> float:
    """torch.optim.Muon's ``_adjust_lr`` factor for a rows x cols matrix: the step is ``lr`` times it (double)."""
    if adjust_lr_fn is None or adjust_lr_fn == "original":
        return math.sqrt(max(1, rows / cols))
    if adjust_lr_fn == "match_rms_adamw":
        return 0.2 * math.sqrt(max(rows, cols))
    return 1.0


_MUON_DEFAULTS = dict(lr=1e-3, weight_decay=0.1, momentum=0.95, nesterov=True, ns_coefficients=(3.4445, -4.7750, 2.0315),
                      eps=1e-7, ns_steps=5, adjust_lr_fn=None)   # torch.optim.Muon's
_AUX_ADAMW_DEFAULTS = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)   # torch.optim.AdamW's


class MuonWithAuxAdamW(torch.optim.Optimizer):
    """Muon for the matrices of a model and AdamW for everything else, in one optimizer, so that a whole model (biases,
    norms, embeddings, conv weights) can train with Muon.  Every parameter group carries ``use_muon``:

    * ``use_muon=True``: torch.optim.Muon's keys and defaults (``lr``, ``weight_decay``, ``momentum``, ``nesterov``,
      ``ns_coefficients``, ``eps``, ``ns_steps``, ``adjust_lr_fn``) and state (``momentum_buffer``, no ``step``).
      Parameters of 2 or more dims, each treated as the ``(shape[0], numel / shape[0])`` matrix (a conv weight
      ``(out, in, kh, kw)`` as ``(out, in kh kw)``).  For one parameter w with gradient g, as R x C matrices, this is
      torch.optim.Muon's ``_single_tensor_muon``::

          buf.lerp_(g, 1 - momentum)
          u = g.lerp(buf, momentum) if nesterov else buf
          X = u.bfloat16();  X = X.T if R > C
          X.div_(X.norm().clamp(min=eps))
          ns_steps times:  A = X @ X.T;  B = torch.addmm(A, A, A, beta=b, alpha=c);  X = torch.addmm(X, B, X, beta=a)
          X = X.T if R > C
          w.mul_(1 - lr * weight_decay)
          w.add_(X, alpha=-(lr * ratio))        # ratio: muon_lr_ratio(adjust_lr_fn, R, C), torch's _adjust_lr

    * ``use_muon=False``: torch.optim.AdamW's keys and defaults (``lr``, ``betas``, ``eps``, ``weight_decay``) and state
      (``step`` as a 0-dim fp32 tensor, ``exp_avg``, ``exp_avg_sq``), in torch's single-tensor op order, t the
      parameter's step count after the increment::

          w.mul_(1 - lr * weight_decay)         # when weight_decay != 0
          m.lerp_(g, 1 - beta1)
          v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
          w.addcdiv_(m, (v.sqrt() / (1 - beta2 ** t) ** 0.5).add_(eps), value=-(lr / (1 - beta1 ** t)))

    State is created at a parameter's first step; a parameter without a gradient is not touched.  ``step()`` is plain
    per-parameter torch with no ``.item()``: what runs outside the engine and on its stock route; inside ``Stoke`` the
    Muon groups run on the fused sm_90a Muon step (``stk_muon_step``) and the AdamW groups on the fused AdamW step.  No
    parity with any third-party package is claimed."""

    def __init__(self, params):
        super().__init__(params, {})

    def add_param_group(self, param_group):
        if "use_muon" not in param_group:
            raise ValueError("MuonWithAuxAdamW -- every parameter group needs use_muon=True or False")
        muon = bool(param_group["use_muon"])
        for k, v in (_MUON_DEFAULTS if muon else _AUX_ADAMW_DEFAULTS).items():
            param_group.setdefault(k, v)
        g = param_group
        if not 0.0 <= g["lr"]:
            raise ValueError(f"Invalid learning rate: {g['lr']}")
        if not 0.0 <= g["weight_decay"]:
            raise ValueError(f"Invalid weight_decay value: {g['weight_decay']}")
        if not 0.0 <= g["eps"]:
            raise ValueError(f"Invalid epsilon value: {g['eps']}")
        if muon:
            if not 0.0 <= g["momentum"]:
                raise ValueError(f"Invalid momentum value: {g['momentum']}")
            if g["adjust_lr_fn"] not in (None, "original", "match_rms_adamw"):
                raise ValueError(f"Adjust learning rate function {g['adjust_lr_fn']} is not supported")
            if len(g["ns_coefficients"]) != 3:
                raise ValueError("ns_coefficients must be a tuple of exactly 3 values")
            if not 0 <= int(g["ns_steps"]) < 100:
                raise ValueError(f"ns_steps must be in [0, 100), got {g['ns_steps']}")
        elif not 0.0 <= g["betas"][0] < 1.0 or not 0.0 <= g["betas"][1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {g['betas']}")
        super().add_param_group(param_group)
        if muon:
            for p in self.param_groups[-1]["params"]:
                if p.ndim < 2:
                    raise ValueError(f"MuonWithAuxAdamW -- a use_muon group holds a parameter of size {tuple(p.shape)}; "
                                     "Muon takes parameters of 2 or more dims")

    @staticmethod
    def _muon(p, g, state, group):
        if "momentum_buffer" not in state:
            state["momentum_buffer"] = torch.zeros_like(g, memory_format=torch.preserve_format)
        rows = p.shape[0]
        # views of contiguous tensors; copies (written back below) of strided ones, e.g. a channels-last conv weight
        w, g2, buf = (t.reshape(rows, -1) for t in (p, g, state["momentum_buffer"]))
        a, b, c = group["ns_coefficients"]
        momentum = group["momentum"]
        buf.lerp_(g2, 1 - momentum)
        update = g2.lerp(buf, momentum) if group["nesterov"] else buf
        x = update.bfloat16()
        tall = x.size(0) > x.size(1)
        if tall:
            x = x.T
        x.div_(x.norm().clamp(min=group["eps"]))
        for _ in range(group["ns_steps"]):
            gram = x @ x.T
            gram_update = torch.addmm(gram, gram, gram, beta=b, alpha=c)
            x = torch.addmm(x, gram_update, x, beta=a)
        if tall:
            x = x.T
        lr = group["lr"]
        w.mul_(1 - lr * group["weight_decay"])
        w.add_(x, alpha=-(lr * muon_lr_ratio(group["adjust_lr_fn"], rows, w.size(1))))
        for dst, src in ((p, w), (state["momentum_buffer"], buf)):
            if dst.data_ptr() != src.data_ptr() or not dst.is_contiguous():
                dst.copy_(src.reshape(dst.shape))

    @staticmethod
    def _adamw(p, g, state, group):
        if not state:
            state["step"] = torch.tensor(0.0, dtype=torch.float32)
            state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        state["step"] += 1
        t = float(state["step"])
        beta1, beta2 = group["betas"]
        lr, wd = group["lr"], group["weight_decay"]
        m, v = state["exp_avg"], state["exp_avg_sq"]
        if wd != 0:
            p.mul_(1 - lr * wd)
        m.lerp_(g, 1 - beta1)
        v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        denom = (v.sqrt() / (1 - beta2 ** t) ** 0.5).add_(group["eps"])
        p.addcdiv_(m, denom, value=-(lr / (1 - beta1 ** t)))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            update = self._muon if group["use_muon"] else self._adamw
            for p in group["params"]:
                if p.grad is not None:
                    update(p, p.grad, self.state[p], group)
        return loss


# torch.optim.Muon (torch >= 2.9) and MuonWithAuxAdamW run on their own entry point, stk_muon_step (batched
# Newton-Schulz on tensor cores), not as kinds of K2; MuonWithAuxAdamW's AdamW groups then take K2's AdamW
_MUON = "muon"
if hasattr(torch.optim, "Muon"):
    _KINDS[torch.optim.Muon] = _MUON
_KINDS[MuonWithAuxAdamW] = _MUON


def _use_muon(g) -> bool:
    """A group of torch.optim.Muon (no ``use_muon`` key) or a Muon group of MuonWithAuxAdamW."""
    return bool(g.get("use_muon", True))


def muon_matrices(params, group_of: List[int], groups: List[Dict]) -> List[Optional[Tuple[int, int, float]]]:
    """Per parameter, the (rows, cols) of its Muon matrix and torch's ``_adjust_lr`` factor of that shape, or None in
    an AdamW group."""
    out = []
    for p, gi in zip(params, group_of):
        g = groups[gi]
        if not _use_muon(g):
            out.append(None)
            continue
        rows = p.shape[0]
        cols = p.numel() // rows
        out.append((rows, cols, muon_lr_ratio(g["adjust_lr_fn"], rows, cols)))
    return out


def _muon_flat_matrix(p: torch.Tensor) -> bool:
    """The fused Muon step reads a parameter's flat elements as its (shape[0], numel / shape[0]) matrix: every row one
    contiguous run of the flat layout, dim 0 outermost and the tensor dense (contiguous or channels-last).  The column
    order within a row may differ from the logical one (channels-last); Newton-Schulz commutes with that permutation."""
    if p.ndim < 2 or p.numel() == 0:
        return False
    dense = p.is_contiguous() or (p.ndim == 4 and p.is_contiguous(memory_format=torch.channels_last))
    return dense and p.stride(0) == p.numel() // p.shape[0]


class StateTensor(NamedTuple):
    """One per-parameter state tensor of a fused kind."""
    key: str                                         # torch's state key
    buf: str                                         # the flat fp32 buffer: "M", "V", "M2" or "M3"; "af": Adafactor's;
                                                     # "q8": the 8-bit step's codes, maps, absmax and fp32 state
    init: Union[float, str] = 0.0                    # its value before the first step: 0.0, 1.0 or "master"
    where: Optional[Callable[[Dict], bool]] = None   # the group condition under which it exists (None: every group)
    none: bool = False                               # where it does not exist, a parameter exports None (else no key)
    alloc: Optional[Callable[[Dict], bool]] = None   # the buffer exists iff some group satisfies this (None: `where`)


class StateLayout(NamedTuple):
    """What a fused kind keeps per parameter, in torch's ``state_dict`` format."""
    step: bool                          # entries carry ``step`` (a 0-dim fp32 tensor)
    scalars: Tuple[str, ...]            # scalar state, 0-dim fp32 tensors after ``step``
    unstepped: str                      # a never-stepped parameter: "omit" (no entry, torch's lazy state), "same"
                                        # (exported like a stepped one, at step 0) or "none" (every tensor None)
    tensors: Tuple[StateTensor, ...]    # in torch's key order
    # the step count lives in the parameter groups, not in ``state``: (the group key, the state key whose presence marks
    # a parameter that has stepped); None: per-parameter ``step`` (or SGD's momentum_buffer rule)
    group_count: Optional[Tuple[str, str]] = None


def _momentum(g):
    return g["momentum"] != 0


_ADAM_STATE = (StateTensor("exp_avg", "M"), StateTensor("exp_avg_sq", "V"))
# Every fused kind's state.  A new kind adds one row; allocation (state_buffers), state_dict (export_state) and
# load_state_dict (import_state) follow from it.  SGD exports its momentum buffer in every group once some group has
# momentum: M exists for all of them.
_STATE_LAYOUT: Dict[object, StateLayout] = {
    _lib.OPT_SGD: StateLayout(False, (), "none", (StateTensor("momentum_buffer", "M", none=True, alloc=_momentum),)),
    _lib.OPT_ADAM: StateLayout(True, (), "same", _ADAM_STATE),
    _lib.OPT_ADAMW: StateLayout(True, (), "same", _ADAM_STATE),
    _lib.OPT_RADAM: StateLayout(True, (), "same", _ADAM_STATE),
    _lib.OPT_NADAM: StateLayout(True, ("mu_product",), "same", _ADAM_STATE),
    _lib.OPT_ADAMAX: StateLayout(True, (), "same", (StateTensor("exp_avg", "M"), StateTensor("exp_inf", "V"))),
    _lib.OPT_ADADELTA: StateLayout(True, (), "omit", (StateTensor("square_avg", "M"), StateTensor("acc_delta", "V"))),
    _lib.OPT_RPROP: StateLayout(True, (), "omit", (StateTensor("prev", "M"), StateTensor("step_size", "V"))),
    _lib.OPT_ASGD: StateLayout(True, ("eta", "mu"), "omit", (StateTensor("ax", "M"),)),
    _lib.OPT_LION: StateLayout(True, (), "omit", (StateTensor("exp_avg", "M"),)),
    _lib.OPT_SF_ADAMW: StateLayout(False, (), "omit", (StateTensor("z", "M", "master"),
                                                       StateTensor("exp_avg_sq", "V")), ("k", "z")),
    _lib.OPT_SF_SGD: StateLayout(False, (), "omit", (StateTensor("z", "M", "master"),), ("k", "z")),
    _lib.OPT_ADEMAMIX: StateLayout(True, (), "omit", (
        StateTensor("exp_avg_fast", "M", where=lambda g: g["betas"][0] != 0, none=True),
        StateTensor("exp_avg_slow", "M2"), StateTensor("exp_avg_sq", "V"))),
    _lib.OPT_RMSPROP_TF: StateLayout(True, (), "omit", (
        StateTensor("square_avg", "V", 1.0), StateTensor("momentum_buffer", "M", where=lambda g: g["momentum"] > 0),
        StateTensor("grad_avg", "M2", where=lambda g: g["centered"]))),
    _lib.OPT_ADAN: StateLayout(False, (), "omit", (
        StateTensor("exp_avg", "M"), StateTensor("exp_avg_sq", "V"), StateTensor("exp_avg_diff", "M2"),
        StateTensor("neg_pre_grad", "M3")), ("step", "exp_avg")),
    _LAMB: StateLayout(True, (), "omit", _ADAM_STATE),
    _LARS: StateLayout(True, (), "omit", (StateTensor("momentum_buffer", "M", where=_momentum),)),
    _STABLE_ADAMW: StateLayout(True, (), "omit", _ADAM_STATE),
    # row_var / col_var of a factored parameter, variance of the others: views of GradPath.af_state
    _ADAFACTOR: StateLayout(True, (), "omit", (StateTensor("row_var", "af"), StateTensor("col_var", "af"),
                                               StateTensor("variance", "af"))),
    # uint8 codes (fp32 for a parameter below min_8bit_size), the maps and the block absmax: views of GradPath's 8-bit
    # state (q8_state_views); no fp32 moment buffers
    _ADAM8BIT: StateLayout(True, (), "omit", tuple(StateTensor(k, "q8") for k in (
        "state1", "qmap1", "state2", "qmap2", "absmax1", "absmax2"))),
    _LION8BIT: StateLayout(True, (), "omit", tuple(StateTensor(k, "q8") for k in ("state1", "qmap1", "absmax1"))),
    # state1 / absmax1 stack m1 and m2: shaped (2, *p.shape) / (2, n_blocks)
    _ADEMAMIX8BIT: StateLayout(True, (), "omit", tuple(StateTensor(k, "q8") for k in (
        "state1", "qmap1", "state2", "qmap2", "absmax1", "absmax2"))),
    # Muon groups: momentum_buffer (no step: state_dict drops it from their entries); MuonWithAuxAdamW's AdamW groups:
    # step, exp_avg, exp_avg_sq.  M holds both kinds of first tensor, each at its parameters' offsets.
    _MUON: StateLayout(True, (), "omit", (
        StateTensor("momentum_buffer", "M", where=_use_muon),
        StateTensor("exp_avg", "M", where=lambda g: not _use_muon(g)),
        StateTensor("exp_avg_sq", "V", where=lambda g: not _use_muon(g)))),
}


def _ext_hyper(g) -> _lib.OptimHyperExt:
    x = _lib.OptimHyperExt()
    x.momentum_decay = float(g.get("momentum_decay", 0.0))
    x.decoupled_weight_decay = int(bool(g.get("decoupled_weight_decay", False)))
    x.rho = float(g.get("rho", 0.0))
    x.etaminus, x.etaplus = (float(e) for e in g.get("etas", (0.0, 0.0)))
    x.step_size_min, x.step_size_max = (float(e) for e in g.get("step_sizes", (0.0, 0.0)))
    x.lambd, x.alpha, x.t0 = float(g.get("lambd", 0.0)), float(g.get("alpha", 0.0)), float(g.get("t0", 0.0))
    return x


def _sf_hyper(g) -> _lib.SfHyper:
    x = _lib.SfHyper()
    x.lr, x.beta1, x.r = float(g["lr"]), float(_sf_beta1(g)), float(g["r"])
    x.weight_lr_power = float(g["weight_lr_power"])
    x.beta2 = float(g["betas"][1]) if "betas" in g else 0.0
    x.warmup_steps = int(g["warmup_steps"])
    return x


def _ademamix_hyper(g) -> _lib.AdemamixHyper:
    x = _lib.AdemamixHyper()
    x.alpha, x.beta3 = float(g["alpha"]), float(g["betas"][2])
    x.alpha_warmup = int(g["alpha_warmup"] or 0)   # 0: none
    x.beta3_warmup = int(g["beta3_warmup"] or 0)
    return x


def _rmsprop_tf_hyper(g) -> _lib.RmspropTfHyper:
    x = _lib.RmspropTfHyper()
    x.alpha = float(g["alpha"])
    x.centered, x.decoupled_decay = int(bool(g["centered"])), int(bool(g["decoupled_decay"]))
    x.lr_in_momentum = int(bool(g["lr_in_momentum"]))
    return x


def _adan_hyper(g) -> _lib.AdanHyper:
    x = _lib.AdanHyper()
    x.beta3, x.no_prox = float(g["betas"][2]), int(bool(g["no_prox"]))
    return x


def _adafactor_hyper(g) -> _lib.AdafactorHyper:
    h = _lib.AdafactorHyper()
    eps1, eps2 = g["eps"]
    h.lr, h.beta2_decay, h.eps2, h.d = float(g["lr"]), float(g["beta2_decay"]), float(eps2), float(g["d"])
    h.weight_decay = float(g["weight_decay"])
    h.eps1_none, h.eps1 = int(eps1 is None), float(eps1 if eps1 is not None else 0.0)
    h.maximize = int(bool(g.get("maximize", False)))
    return h


def _adam8bit_hyper(g) -> _lib.Adam8bitHyper:
    """The per-group struct of every 8-bit step: AdamW8bit's fields; Lion8bit has no eps (0), AdEMAMix8bit's third beta
    goes in its AdemamixHyper."""
    h = _lib.Adam8bitHyper()
    h.lr, h.eps, h.weight_decay = float(g["lr"]), float(g.get("eps", 0.0)), float(g["weight_decay"])
    h.beta1, h.beta2 = (float(b) for b in g["betas"][:2])
    return h


def _ademamix8bit_hyper(g) -> Tuple[_lib.Adam8bitHyper, _lib.AdemamixHyper]:
    return _adam8bit_hyper(g), _ademamix_hyper(g)


def _muon_hyper(g) -> Tuple[_lib.MuonHyper, _lib.OptimHyper]:
    """(the Muon step's struct, K2's AdamW struct) of one group; the one its ``use_muon`` does not select is left
    neutral (the step skips its parameters)."""
    m, h = _lib.MuonHyper(), _lib.OptimHyper()
    h.kind, h.beta1, h.beta2 = _lib.OPT_ADAMW, 0.9, 0.999
    if _use_muon(g):
        m.lr, m.weight_decay, m.momentum, m.eps = float(g["lr"]), float(g["weight_decay"]), float(g["momentum"]), float(g["eps"])
        m.ns_a, m.ns_b, m.ns_c = (float(x) for x in g["ns_coefficients"])
        m.nesterov, m.ns_steps = int(bool(g["nesterov"])), int(g["ns_steps"])
    else:
        h.lr, h.eps, h.weight_decay = float(g["lr"]), float(g["eps"]), float(g["weight_decay"])
        h.beta1, h.beta2 = (float(b) for b in g["betas"])
    return m, h


def _layerwise_hyper(g) -> _lib.LayerwiseHyper:
    h = _lib.LayerwiseHyper()
    h.lr, h.eps, h.weight_decay = float(g["lr"]), float(g["eps"]), float(g["weight_decay"])
    h.always_adapt = int(bool(g["always_adapt"]))
    if "betas" in g:   # LAMB
        h.beta1, h.beta2 = (float(b) for b in g["betas"])
        h.bias_correction = int(bool(g["bias_correction"]))
    else:              # LARS
        h.momentum, h.dampening = float(g["momentum"]), float(g["dampening"])
        h.trust_coefficient, h.nesterov = float(g["trust_coefficient"]), int(bool(g["nesterov"]))
    return h


def _stable_adamw_hyper(g) -> _lib.LayerwiseHyper:
    h = _lib.LayerwiseHyper()
    h.lr, h.eps, h.weight_decay = float(g["lr"]), float(g["eps"]), float(g["weight_decay"])
    h.beta1, h.beta2 = (float(b) for b in g["betas"])
    return h


# The per-group struct each fused kind's step takes, built from one param group.  The K2 kinds pass it beside their
# OptimHyper array (GradPath.optimizer_step chooses the prologues and the entry point by kind); a K2 kind without a row
# passes OptimHyper alone.  Adafactor, LAMB, LARS and the 8-bit kinds pass it alone to their own entry points
# (AdEMAMix8bit: an (Adam8bitHyper, AdemamixHyper) pair; Muon: a (MuonHyper, OptimHyper) pair).
_GROUP_HYPER: Dict[object, Callable[[Dict], object]] = {
    **{k: _ext_hyper for k in _EXT_KINDS},
    _lib.OPT_SF_ADAMW: _sf_hyper, _lib.OPT_SF_SGD: _sf_hyper,
    _lib.OPT_ADEMAMIX: _ademamix_hyper,
    _lib.OPT_RMSPROP_TF: _rmsprop_tf_hyper,
    _lib.OPT_ADAN: _adan_hyper,
    _ADAFACTOR: _adafactor_hyper,
    _LAMB: _layerwise_hyper, _LARS: _layerwise_hyper, _STABLE_ADAMW: _stable_adamw_hyper,
    _ADAM8BIT: _adam8bit_hyper, _LION8BIT: _adam8bit_hyper,
    _ADEMAMIX8BIT: _ademamix8bit_hyper,
    _MUON: _muon_hyper,
}


def state_buffers(layout: StateLayout, groups: List[Dict]) -> Dict[str, object]:
    """The flat fp32 buffers a kind needs for these parameter groups: ``{"M", "V", "M2"} -> initial value`` (0.0, 1.0
    or "master"), None for a buffer that is not allocated, plus ``"M3"`` for a kind that keeps a tensor there."""
    out = {"M": None, "V": None, "M2": None}
    if any(t.buf == "M3" for t in layout.tensors):
        out["M3"] = None
    for t in layout.tensors:
        cond = t.alloc or t.where
        if t.buf in out and (cond is None or any(cond(g) for g in groups)):
            out[t.buf] = t.init
    return out


def export_state(layout: StateLayout, groups: List[Dict], group_of: List[int], sd_index: Dict[int, int],
                 steps: List[int], scalars: Optional[List[List[float]]],
                 views: Dict[str, List[Optional[torch.Tensor]]]) -> Dict[int, Dict]:
    """torch's ``state`` mapping.  ``steps`` / ``scalars``: every parameter's step count and scalar state (flat order);
    ``views``: per state key, every parameter's view of the full-length vector that holds it (None, or no key, where it
    has none).  A tensor is exported as a clone where the parameter has a view and its group meets ``where``."""
    state = {}
    for i, gi in enumerate(group_of):
        if steps[i] == 0 and layout.unstepped == "omit":
            continue
        if steps[i] == 0 and layout.unstepped == "none":
            state[sd_index[i]] = {t.key: None for t in layout.tensors}
            continue
        d = {"step": torch.tensor(float(steps[i]))} if layout.step else {}
        for key, val in zip(layout.scalars, scalars[i] if layout.scalars else ()):
            d[key] = torch.tensor(val, dtype=torch.float32)
        for t in layout.tensors:
            view = views[t.key][i] if t.key in views else None
            if view is not None and (t.where is None or t.where(groups[gi])):
                d[t.key] = view.clone()
            elif t.none:
                d[t.key] = None
        state[sd_index[i]] = d
    return state


def import_state(layout: StateLayout, entries: List[Dict], views: Dict[str, List[Optional[torch.Tensor]]]):
    """Copies a state dict's tensors into ``views`` (as ``export_state``'s, already at their initial values).
    ``entries``: torch's state entry of every parameter in flat order (``{}`` where it has none); a key that is missing
    or None leaves the parameter at the initial value."""
    for t in layout.tensors:
        for src, view in zip(entries, views.get(t.key, ())):
            if view is not None and src.get(t.key) is not None:
                view.copy_(src[t.key].reshape(view.shape))


def _module_params(module: torch.nn.Module):
    return [p for p in module.parameters() if p.requires_grad]


def _group_layout(module: torch.nn.Module, optim_kwargs: Dict):
    """(params in registration order, group index per param, per-group kwargs).  ``optimizer_kwargs["params"]`` may carry
    torch-style parameter groups (list of dicts); the reference itself passes ``model.parameters()``."""
    params = _module_params(module)
    kw = dict(optim_kwargs)
    groups = kw.pop("params", None)
    if groups is None:
        return params, [0] * len(params), [{}], kw
    groups = list(groups)
    if groups and not isinstance(groups[0], dict):
        groups = [{"params": groups}]
    index = {id(p): i for i, p in enumerate(params)}
    group_of = [-1] * len(params)
    extra = []
    for gi, g in enumerate(groups):
        extra.append({k: v for k, v in g.items() if k != "params"})
        for p in g["params"]:
            if id(p) not in index:
                raise ValueError("Stoke -- a parameter group holds a tensor that is not a trainable parameter of the model")
            group_of[index[id(p)]] = gi
    if any(g < 0 for g in group_of):
        raise ValueError("Stoke -- every trainable parameter must belong to a parameter group")
    return params, group_of, extra, kw


def state_dict_index(group_of: List[int], n_groups: int) -> Dict[int, int]:
    """flat parameter position -> torch's ``state_dict()`` parameter id (torch numbers parameters group by group, in group
    order: torch/optim/optimizer.py ``state_dict``)."""
    order = [i for gi in range(n_groups) for i, g in enumerate(group_of) if g == gi]
    return {flat_i: sd_i for sd_i, flat_i in enumerate(order)}


def load_step_counts(kind, entries: List[Dict], group_of: List[int], opt_steps: Optional[int], per_param_on: bool,
                     momentum: Optional[List[float]] = None, group_k: Optional[List[int]] = None):
    """How a loaded state dict's step counts and scalar state (NAdam's ``mu_product``, ASGD's ``eta`` / ``mu``) go onto
    the fused step.  ``entries``: torch's state entry of every parameter in flat order (``{}`` where it has none);
    ``opt_steps``: the checkpoint's ``b200_opt_steps`` (None in a torch-written one); ``per_param_on``: the step already
    keeps per-parameter counts; ``momentum``: SGD's per-group momentum; ``group_k``: every group's count, for the kinds
    that keep it in the group (``StateLayout.group_count``: the schedule-free ``k``, Adan's ``step``).

    torch creates a parameter's state at its first step, so a parameter without an entry has taken 0 steps and has the
    initial scalar state (1.0).  torch's SGD keeps no ``step``: a parameter with a ``momentum_buffer`` has taken
    ``opt_steps`` steps (1 in a torch-written checkpoint), one without it 0; in a group without momentum the count has no
    effect and is the optimizer-wide one.  Muon keeps no ``step`` either: its parameters follow SGD's rule (a Muon group
    always has the buffer), MuonWithAuxAdamW's AdamW parameters carry ``step``.

    Returns ``(opt_steps, steps, scalars)``: the optimizer-wide count, then either per-parameter counts and per-parameter
    scalar state (``steps`` a list) or ``steps = None`` and per-group scalar state.  Counts go per parameter when they
    are not all the optimizer-wide count, when the scalar state differs within a group, or when ``per_param_on``.
    ``scalars`` is None for the kinds without scalar state.

    The kinds with ``group_count`` keep no per-parameter ``step``: the count is the checkpoint's ``b200_opt_steps``, else
    the groups' common count (groups whose counts differ raise ValueError), and a parameter has taken that many steps if
    its entry has the marker tensor (schedule-free ``z``, Adan's ``exp_avg``), 0 if not."""
    group_count = _STATE_LAYOUT[kind].group_count
    if group_count is not None:
        key, marker = group_count
        if opt_steps is None:
            ks = set(int(k) for k in (group_k or []))
            if len(ks) > 1:
                raise ValueError(f"Stoke -- parameter groups with different step counts {key}: {sorted(ks)}")
            opt_steps = ks.pop() if ks else 0
        steps = [opt_steps if marker in e else 0 for e in entries]
        if per_param_on or any(s != opt_steps for s in steps):
            return opt_steps, steps, None
        return opt_steps, None, None

    def count(e, g):
        if kind == _MUON and "step" not in e:
            return 0 if e.get("momentum_buffer") is None else 1 if opt_steps is None else opt_steps
        if kind != _lib.OPT_SGD:
            return int(float(e["step"])) if "step" in e else 0
        if momentum[g] == 0:
            return None
        if e.get("momentum_buffer") is None:
            return 0
        return 1 if opt_steps is None else opt_steps

    keys = _STATE_LAYOUT[kind].scalars
    steps = [count(e, g) for e, g in zip(entries, group_of)]
    if opt_steps is None:
        opt_steps = max([s for s in steps if s is not None], default=0)
    steps = [opt_steps if s is None else s for s in steps]
    scal = [[float(e[k]) if k in e else 1.0 for k in keys] for e in entries]
    n_groups = max(group_of, default=-1) + 1
    # only stepped parameters' scalars count: an unstepped one forces per-parameter counts through its count of 0
    groups_differ = any(len({tuple(scal[i]) for i, g in enumerate(group_of) if g == gi and steps[i] > 0}) > 1
                        for gi in range(n_groups))
    if per_param_on or groups_differ or any(s != opt_steps for s in steps):
        return opt_steps, steps, scal if keys else None
    if not keys:
        return opt_steps, None, None
    first = {}
    for i, g in enumerate(group_of):
        first.setdefault(g, scal[i])
    return opt_steps, None, [first.get(gi, [1.0] * len(keys)) for gi in range(n_groups)]


def fused_supported(optim_cls, optim_kwargs: Dict, module: torch.nn.Module) -> bool:
    if optim_cls not in _KINDS:
        return False
    _, _, extra, kw = _group_layout(module, optim_kwargs)
    if len(extra) > _lib.MAX_GROUPS:
        return False
    for g in extra:
        merged = dict(kw, **g)
        if any(merged.get(k) for k in _STOCK_ONLY_TRUE):
            return False
    if _KINDS[optim_cls] == _MUON:   # every Muon parameter's flat elements must form its matrix
        params, group_of, _, _ = _group_layout(module, optim_kwargs)
        if not all(_muon_flat_matrix(p) for p, gi in zip(params, group_of) if _use_muon(extra[gi])):
            return False
    if _KINDS[optim_cls] == _ADAFACTOR:
        try:   # up to four dims, dense (channels-last included)
            for p in _module_params(module):
                layout.adafactor_layout(p.shape, p.stride())
        except ValueError:
            return False
    return True


class B200FusedOptimizer(torch.optim.Optimizer):
    def __init__(self, module: torch.nn.Module, optim_cls: Type[torch.optim.Optimizer], optim_kwargs: Dict,
                 engine: Engine, grad_accum: int = 1, clip: Optional[ClipSpec] = None, sharded: bool = False,
                 lp_dtype: Optional[torch.dtype] = None, state_id: Optional[int] = None, route: Optional[str] = None,
                 bucket_mb: Optional[float] = None):
        if optim_cls not in _KINDS:
            raise NotImplementedError(
                f"Stoke -- the fused step covers torch.optim.Adam, AdamW, SGD, NAdam, RAdam, Adamax, Adadelta, Rprop, ASGD and Adafactor and stoke_b200.optim.LAMB, LARS, StableAdamW, Lion, AdamWScheduleFree, SGDScheduleFree, AdEMAMix, RMSpropTF, Adan, AdamW8bit, Adam8bit, Lion8bit, AdEMAMix8bit, torch.optim.Muon and MuonWithAuxAdamW; got {getattr(optim_cls, '__name__', optim_cls)}"
                f" (use B200StockOptimizer / build_optimizer, which routes other classes to the stock-optimizer path)")
        params, group_of, extra, kw = _group_layout(module, optim_kwargs)
        if len(extra) > _lib.MAX_GROUPS:
            raise NotImplementedError(f"Stoke -- the fused step handles up to {_lib.MAX_GROUPS} parameter groups")
        # let torch validate the kwargs exactly as the reference would (optimizer(params=..., **kwargs)); Muon takes
        # matrices only
        shape = (1, 1) if _KINDS[optim_cls] == _MUON else (1,)
        probe = optim_cls([dict(g, params=[torch.nn.Parameter(torch.zeros(shape))]) for g in extra], **kw)
        for g in probe.param_groups:
            for k in _STOCK_ONLY_TRUE:
                if g.get(k):
                    raise NotImplementedError(f"Stoke -- optimizer option {k}=True is not covered by the fused step")
        self._kind = _KINDS[optim_cls]
        # torch >= 2.6: AdamW is Adam(decoupled_weight_decay=True).  NAdam and RAdam carry the same flag as a per-group option
        # of their own update (hyper_ext), so it does not change their kind.
        if self._kind == _lib.OPT_ADAM and probe.defaults.get("decoupled_weight_decay"):
            self._kind = _lib.OPT_ADAMW
        self._torch_cls = optim_cls
        self._layout = _STATE_LAYOUT[self._kind]
        self._buffers = state_buffers(self._layout, probe.param_groups)
        ada = self._kind == _ADAFACTOR
        lw = self._kind in _LAYERWISE
        q8 = None
        if self._kind in _Q8_KINDS:   # which parameters keep 8-bit state (the others: fp32, below min_8bit_size)
            q8 = [p.numel() >= probe.param_groups[gi]["min_8bit_size"] for p, gi in zip(params, group_of)]
        muon = None
        if self._kind == _MUON:
            # MuonWithAuxAdamW has no optimizer-wide defaults: each group takes Muon's or AdamW's, as the probe filled them
            extra = [{k: v for k, v in g.items() if k != "params"} for g in probe.param_groups]
            # the class's own checks on the real parameters (torch.optim.Muon: 2-D only; MuonWithAuxAdamW: 2 or more dims)
            optim_cls([dict(g, params=[p for p, gi in zip(params, group_of) if gi == k]) for k, g in enumerate(extra)],
                      **kw)
            if not all(_muon_flat_matrix(p) for p, gi in zip(params, group_of) if _use_muon(probe.param_groups[gi])):
                raise NotImplementedError("Stoke -- the fused Muon step needs every Muon parameter dense with dim 0 "
                                          "outermost (contiguous or channels-last)")
            muon = muon_matrices(params, group_of, probe.param_groups)
        if (ada or lw or q8 is not None or muon is not None) and engine.world > 1:
            # Adafactor's per-parameter reductions, LAMB's / LARS's trust ratios and Muon's Newton-Schulz need whole
            # parameters on one rank, and the 8-bit state's 256-element blocks do not follow the shard boundaries: their
            # state is replicated (also under fairscale_oss) and every rank runs the same deterministic step on the same
            # all-reduced fp32 gradients
            route = "allreduce"
        self.path = GradPath(engine, params, grad_accum=grad_accum, clip=clip, sharded=sharded, lp_dtype=lp_dtype,
                             module=module, state=self._buffers, state_id=state_id, route=route,
                             group_of=group_of, bucket_mb=bucket_mb, scalar_state=len(self._layout.scalars),
                             adafactor=ada, layerwise=lw, schedule_free=self._kind in _SF_KINDS, adam8bit=q8,
                             q8_states=_Q8_KINDS.get(self._kind, 2), muon=muon)
        by_group: List[List[torch.nn.Parameter]] = [[] for _ in extra]
        for p, gi in zip(params, group_of):
            by_group[gi].append(p)
        super().__init__([dict(g, params=ps) for g, ps in zip(extra, by_group)], dict(probe.defaults))
        self._group_of = group_of
        # position of every parameter inside torch's state_dict numbering (group by group, in group order)
        self._sd_index = state_dict_index(group_of, len(extra))
        engine.scaler_set(state=self.path.state_id, opt_steps=0, skipped_steps=0, found_inf=0, growth_tracker=0)

    # -- the step -------------------------------------------------------------------------------------------------------
    def _hyper_of(self, g) -> _lib.OptimHyper:
        h = _lib.OptimHyper()
        h.kind = self._kind
        h.lr = float(g["lr"])
        h.weight_decay = float(g.get("weight_decay", 0.0))
        h.maximize = int(bool(g.get("maximize", False)))
        if self._kind == _lib.OPT_SGD:
            h.momentum = float(g.get("momentum", 0.0))
            h.dampening = float(g.get("dampening", 0.0))
            h.nesterov = int(bool(g.get("nesterov", False)))
        elif self._kind == _lib.OPT_RMSPROP_TF:   # alpha and the flags go in RmspropTfHyper
            h.eps, h.momentum = float(g["eps"]), float(g["momentum"])
        elif "betas" in g:   # AdEMAMix and Adan have a third beta, which goes in AdemamixHyper / AdanHyper
            h.beta1, h.beta2 = float(g["betas"][0]), float(g["betas"][1])
            h.eps = float(g.get("eps", 0.0))   # Lion has no eps
        elif "eps" in g:   # Adadelta
            h.eps = float(g["eps"])
        return h

    @torch.no_grad()
    def step(self, closure=None):
        if closure is not None:
            raise NotImplementedError("Stoke -- closures are not supported by the fused step")
        self.check_train_mode()
        build = _GROUP_HYPER.get(self._kind)
        per_group = [build(g) for g in self.param_groups] if build is not None else None
        if self._kind == _ADAFACTOR:
            self.path.adafactor_step(per_group)
        elif self._kind in _LAYERWISE:
            self.path.layerwise_step(_LAYERWISE[self._kind], per_group)
        elif self._kind == _ADAM8BIT:
            self.path.adam8bit_step(per_group)
        elif self._kind == _LION8BIT:
            self.path.lion8bit_step(per_group)
        elif self._kind == _ADEMAMIX8BIT:
            self.path.ademamix8bit_step(*zip(*per_group))
        elif self._kind == _MUON:
            muon, adamw = zip(*per_group)
            mats = muon_matrices(self.path.params, self._group_of, self.param_groups)
            aux = not all(_use_muon(g) for g in self.param_groups)
            self.path.muon_step(muon, [m[2] for m in mats if m is not None], adamw if aux else None)
        else:
            self.path.optimizer_step([self._hyper_of(g) for g in self.param_groups], per_group)

    # -- schedule-free: train() / eval() ------------------------------------------------------------------------------------
    def check_train_mode(self):
        """Raises RuntimeError if a schedule-free optimizer is in eval mode (``Stoke.step`` asks before it runs anything)."""
        if self._kind in _SF_KINDS:
            _check_train_mode(self.param_groups)

    def _sf_swap(self, to_train: bool):
        if self._kind not in _SF_KINDS:
            raise NotImplementedError("Stoke -- optimizer.train() / eval() swap the weights of AdamWScheduleFree and "
                                      "SGDScheduleFree only")
        path = self.path
        if path.avg_owner is not None:
            path.avg_owner._check_idle(f"optimizer.{'train' if to_train else 'eval'}()")
        weights = {}
        for gi, g in enumerate(self.param_groups):
            if g["train_mode"] != to_train:
                beta1 = _sf_beta1(g)
                weights[gi] = 1 - beta1 if to_train else 1 - 1 / beta1
        if weights:
            path.schedule_free_swap([weights.get(gi) for gi in self._group_of])
        for g in self.param_groups:
            g["train_mode"] = to_train

    def train(self):
        """Schedule-free: the master (and the model's parameters) to y, where gradients are taken."""
        self._sf_swap(True)

    def eval(self):
        """Schedule-free: the master (and the model's parameters) to x, the averaged point that is evaluated."""
        self._sf_swap(False)

    def zero_grad(self, set_to_none: bool = True):
        """No-op: the gradient bucket is zeroed by the kernel that consumes it, and ``param.grad`` must stay a view of that
        bucket (reference: zero_optimizer_grads, stoke/utils.py:83-106).  ``set_to_none`` semantics -- a parameter that
        receives no gradient in a step is not touched by the optimizer -- are kept by the engine's unused-parameter
        detection (autograd hooks + the range table of the fused step)."""
        return None

    # -- fairscale OSS surface (stoke/fp16.py:227-228, stoke/io_ops.py:596-600) ------------------------------------------
    def clip_grad_norm(self, max_norm: float, norm_type: float = 2.0):
        self.path.clip = ClipSpec(_lib.CLIP_NORM, max_norm=max_norm, norm_type=norm_type)

    def consolidate_state_dict(self, recipient_rank: int = 0):
        """fairscale OSS gathers the shards on ``recipient_rank`` before ``state_dict()``; here ``state_dict()`` itself
        all-gathers the sharded buffers on every rank, so this only exists for call-compatibility."""
        return None

    # -- state dict in torch's per-parameter format ----------------------------------------------------------------------
    def _flats(self) -> Dict[str, torch.Tensor]:
        """This rank's allocated state buffers, by name."""
        path = self.path
        flats = {"M": path.m_flat, "V": path.v_flat, "M2": path.m2_flat, "M3": path.m3_flat}
        return {b: f for b, f in flats.items() if f is not None}

    def _views(self, full: Dict[str, torch.Tensor]) -> Dict[str, List[Optional[torch.Tensor]]]:
        """Per state key, every parameter's view of it: into the full-length vectors ``full`` (by buffer), or for
        Adafactor into its own state buffer (row_var / col_var of a factored parameter, variance of the others)."""
        if self._kind == _ADAFACTOR:
            per_param = [dict(zip(("row_var", "col_var") if len(vs) == 2 else ("variance",), vs))
                         for vs in self.path.adafactor_state_views()]
            return {t.key: [d.get(t.key) for d in per_param] for t in self._layout.tensors}
        if self._kind in _Q8_KINDS:
            per_param = self.path.q8_state_views()
            return {t.key: [d.get(t.key) for d in per_param] for t in self._layout.tensors}
        return {t.key: self.path.unflatten(full[t.buf]) for t in self._layout.tensors if t.buf in full}

    def _groups_sd(self):
        groups, start = [], 0
        for g in self.param_groups:
            d = {k: val for k, val in g.items() if k != "params"}
            d["params"] = list(range(start, start + len(g["params"])))
            start += len(g["params"])
            groups.append(d)
        return groups

    def _export(self, state):
        path = self.path
        return {"state": state, "param_groups": self._groups_sd(), "b200_master": path.gather_master(),
                "b200_opt_steps": int(path.engine.scaler_get(path.state_id).opt_steps)}

    def state_dict(self):
        """torch's per-parameter format, as ``_STATE_LAYOUT`` describes this kind: ``step``, the scalar state (NAdam's
        ``mu_product``, ASGD's ``eta`` and ``mu``) as 0-dim fp32 tensors, then the class's state tensors.  Sharded
        buffers are all-gathered (collective)."""
        path = self.path
        full = {b: path._gather_shards(f) if path.sharded else f for b, f in self._flats().items()}
        scalars = path.param_scalars() if self._layout.scalars else None
        out = self._export(export_state(self._layout, self.param_groups, self._group_of, self._sd_index,
                                        path.param_steps(), scalars, self._views(full)))
        if self._kind in _SF_KINDS:   # the running group state, read back from the device (one synchronisation)
            k = out["b200_opt_steps"]
            for g, src, (lr_max, weight_sum) in zip(out["param_groups"], self.param_groups, path._sf_state.tolist()):
                vals = dict(k=k, lr_max=lr_max, weight_sum=weight_sum,
                            scheduled_lr=_sf_scheduled_lr(src, k - 1) if k > 0 else src["scheduled_lr"])
                g.update(vals)
                src.update(vals)   # param_groups as of this state_dict(); reading them every step would synchronise
        if self._kind == _MUON:   # Muon keeps no step
            for i, gi in enumerate(self._group_of):
                if _use_muon(self.param_groups[gi]) and self._sd_index[i] in out["state"]:
                    out["state"][self._sd_index[i]].pop("step", None)
        if self._kind == _lib.OPT_ADAN and out["b200_opt_steps"] > 0:   # the class creates group["step"] at its first step
            for g, src in zip(out["param_groups"], self.param_groups):
                g["step"] = src["step"] = out["b200_opt_steps"]
        return out

    def load_state_dict(self, sd):
        """Accepts this class's own export and a plain ``torch.optim`` state dict written by the reference
        (stoke/io_ops.py:224-236): without ``b200_master`` the fp32 master weights are rebuilt from the model parameters
        that ``model.load_state_dict`` has just filled (load order of BaseStokeIO.load).  A state tensor the checkpoint
        lacks starts at its initial value.  Step counts and scalar state follow torch's lazy state creation
        (``load_step_counts``)."""
        path = self.path
        for g, src in zip(self.param_groups, sd["param_groups"]):
            for k, val in src.items():
                if k != "params":
                    g[k] = val
        dev = path.p_flat.device
        entries = [sd["state"].get(self._sd_index[i], {}) for i in range(len(path.params))]
        # the master this checkpoint continues from: its own, or (reference-written) the model weights already in P
        master = sd["b200_master"].to(device=dev, dtype=torch.float32) if "b200_master" in sd else path.p_flat.float()
        full = {b: master.clone() if self._buffers[b] == "master" else
                torch.full((path.n,), float(self._buffers[b]), dtype=torch.float32, device=dev) for b in self._flats()}
        if self._kind == _ADAFACTOR:
            path.af_state.zero_()
        if self._kind in _Q8_KINDS:   # refuses what the step could not continue from, then starts from the initial state
            keys = [t.key for t in self._layout.tensors]
            check_8bit_entries(entries, path.q8_quantized, tuple(k for k in keys if k.startswith("state")),
                               tuple(k for k in keys if k.startswith("qmap")), self._torch_cls.__name__)
            path.adam8bit_reset()
        import_state(self._layout, entries, self._views(full))
        for b, local in self._flats().items():
            path.scatter_local(full[b], local)
        steps, per_param, scalars = load_step_counts(self._kind, entries, self._group_of, sd.get("b200_opt_steps"),
                                                     path._range_steps is not None,
                                                     [g.get("momentum", 0.0) for g in self.param_groups],
                                                     [g.get(self._layout.group_count[0], 0) for g in self.param_groups]
                                                     if self._layout.group_count else None)
        if self._kind in _SF_KINDS:
            path._sf_state.copy_(torch.tensor([[float(g["lr_max"]), float(g["weight_sum"])] for g in self.param_groups],
                                              dtype=torch.float64))
        if per_param is not None:
            path.enable_per_param_steps(per_param, scalars)
        elif scalars is not None:
            path.set_group_scalars(scalars)
        if "b200_master" in sd:
            if path.master_flat is not path.p_flat:
                path.scatter_local(master, path.master_flat)
            path.p_flat.copy_(master)
        elif path.master_flat is not path.p_flat:
            # reference-written checkpoint: the model weights are already in P (model dtype); they are the best master
            path.scatter_local(master, path.master_flat)
        path.engine.scaler_set(state=path.state_id, opt_steps=steps)

    def close(self):
        self.path.close()


class B200StockOptimizer(torch.optim.Optimizer):
    """Any ``torch.optim`` class behind the engine's gradient path (see the module docstring).  Replicated optimizer state:
    ``route="allreduce"`` (world > 1) or ``"main"`` (world == 1) materialises fp32 main grads on every rank."""

    def __init__(self, module: torch.nn.Module, optim_cls: Type[torch.optim.Optimizer], optim_kwargs: Dict,
                 engine: Engine, grad_accum: int = 1, clip: Optional[ClipSpec] = None, sharded: bool = False,
                 lp_dtype: Optional[torch.dtype] = None, state_id: Optional[int] = None, bucket_mb: Optional[float] = None):
        params, group_of, extra, kw = _group_layout(module, optim_kwargs)
        self.path = GradPath(engine, params, grad_accum=grad_accum, clip=clip, sharded=False, lp_dtype=lp_dtype,
                             module=module, state_id=state_id, route="allreduce" if engine.world > 1 else "main",
                             group_of=None, bucket_mb=bucket_mb)
        path = self.path
        self.user_sharded = bool(sharded)
        # fp32 master parameters: per-parameter views of the flat master buffer, their .grad views of the main grads
        self._masters = [torch.nn.Parameter(v, requires_grad=True) for v in path.unflatten(path.master_flat)]
        for mp, gv in zip(self._masters, path.unflatten(path.main_flat)):
            mp.grad = gv
        self._main_views = path.unflatten(path.main_flat)
        by_group: List[List[torch.nn.Parameter]] = [[] for _ in extra]
        for mp, gi in zip(self._masters, group_of):
            by_group[gi].append(mp)
        self.inner = optim_cls([dict(g, params=ps) for g, ps in zip(extra, by_group)], **kw)
        torch.optim.Optimizer.__init__(self, [dict(g, params=ps) for g, ps in zip(extra, by_group)], dict(self.inner.defaults))
        self.param_groups = self.inner.param_groups  # schedulers edit the inner optimizer's groups
        self.state = self.inner.state
        engine.scaler_set(state=path.state_id, opt_steps=0, skipped_steps=0, found_inf=0, growth_tracker=0)

    def check_train_mode(self):
        """Raises RuntimeError if a schedule-free optimizer is in eval mode (``Stoke.step`` asks before it runs anything)."""
        if isinstance(self.inner, _ScheduleFree):
            _check_train_mode(self.inner.param_groups)

    def _sf_swap(self, to_train: bool):
        if not isinstance(self.inner, _ScheduleFree):
            raise NotImplementedError("Stoke -- optimizer.train() / eval() swap the weights of AdamWScheduleFree and "
                                      "SGDScheduleFree only")
        path = self.path
        if path.avg_owner is not None:
            path.avg_owner._check_idle(f"optimizer.{'train' if to_train else 'eval'}()")
        self.inner.train() if to_train else self.inner.eval()
        if path.master_flat is not path.p_flat:
            path.p_flat.copy_(path.master_flat)   # fp32 -> model dtype, round-to-nearest-even

    def train(self):
        """Schedule-free: the inner optimizer's ``train()`` on the master, then the model's parameters from it."""
        self._sf_swap(True)

    def eval(self):
        """Schedule-free: the inner optimizer's ``eval()`` on the master, then the model's parameters from it."""
        self._sf_swap(False)

    @torch.no_grad()
    def step(self, closure=None):
        self.check_train_mode()   # before the clip touches the gradients
        path, e = self.path, self.path.engine
        e.state_select(path.state_id)
        skip = False
        st = None
        if path.clip.kind != _lib.CLIP_NONE:
            e.grad_scale(path.MAIN.ptr, path.n, path.clip.kind, path.clip.max_norm, path.clip.clip_value)
        st = e.scaler_get()        # one synchronisation, like GradScaler.step's found_inf.item()
        skip = bool(st.found_inf)
        if not skip:
            for mp, gv in zip(self._masters, self._main_views):
                if mp.grad is not gv:
                    mp.grad = gv
            self.inner.step(closure) if closure is not None else self.inner.step()
            if path.master_flat is not path.p_flat:
                path.p_flat.copy_(path.master_flat)   # fp32 -> model dtype, round-to-nearest-even
        path.weight_avg_after_step()
        e.step_epilogue()
        e.comm_poll()

    def zero_grad(self, set_to_none: bool = True):
        return None

    def clip_grad_norm(self, max_norm: float, norm_type: float = 2.0):
        self.path.clip = ClipSpec(_lib.CLIP_NORM, max_norm=max_norm, norm_type=norm_type)

    def consolidate_state_dict(self, recipient_rank: int = 0):
        return None

    def state_dict(self):
        sd = self.inner.state_dict()
        sd["b200_master"] = self.path.gather_master()
        sd["b200_opt_steps"] = int(self.path.engine.scaler_get(self.path.state_id).opt_steps)
        return sd

    def load_state_dict(self, sd):
        path = self.path
        inner = {k: v for k, v in sd.items() if not k.startswith("b200_")}
        self.inner.load_state_dict(inner)
        self.param_groups = self.inner.param_groups
        self.state = self.inner.state
        if "b200_master" in sd:
            master = sd["b200_master"].to(device=path.p_flat.device, dtype=torch.float32)
            if path.master_flat is not path.p_flat:
                path.master_flat.copy_(master)
            path.p_flat.copy_(master)
        elif path.master_flat is not path.p_flat:
            path.master_flat.copy_(path.p_flat.float())
        path.engine.scaler_set(state=path.state_id, opt_steps=int(sd.get("b200_opt_steps", 0)))

    def close(self):
        self.path.close()
