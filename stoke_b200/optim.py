# -*- coding: utf-8 -*-
"""The optimizer objects ``Stoke.optimizer`` hands back.

``B200FusedOptimizer`` -- a ``torch.optim.Optimizer`` (so LR schedulers and ``param_groups`` edits work, README.md:241-250
of the reference) whose ``step()`` is the single fused K2 launch over the flat fp32 master / moment buffers; its sharded
flavour is the ZeRO-1 analogue of fairscale ``OSS`` (/root/reference/stoke/extensions.py:109-141): same ``clip_grad_norm`` /
``consolidate_state_dict`` surface.  Adam, AdamW, SGD(-momentum), NAdam, RAdam, Adamax, Adadelta, Rprop and ASGD, up to 8
parameter groups (per-group lr / betas / eps / weight decay / momentum ... selected inside the kernel by element range).
NAdam, RAdam, Adamax, Adadelta and Rprop keep two fp32 state tensors per parameter like Adam (Adamax's ``exp_inf``,
Adadelta's ``acc_delta`` and Rprop's ``step_size`` in the second-moment buffer); ASGD keeps one (``ax``).  Their per-step
scalars, NAdam's ``mu_product`` and ASGD's ``eta`` / ``mu`` are formed on the device by ``stk_optim_step_prologue``, so
none of them reads a scalar back to the host (torch's single-tensor ASGD calls ``.item()`` three times per parameter).
Adadelta, Rprop and ASGD create their state lazily like torch: a parameter never stepped has no ``state_dict`` entry.
``torch.optim.Adafactor`` takes its own fused entry point, ``stk_adafactor_step`` (per-parameter reductions: row / column
means of g^2, the parameter's RMS, the update's RMS), with per-parameter step counts on the device and torch's
state_dict layout (``row_var`` / ``col_var`` or ``variance``).  Its state is never sharded: the reductions need whole
parameters on one rank, so at world > 1 (``fairscale_oss=True`` included) it runs replicated on the all-reduce route,
every rank taking the same deterministic step on the same gradients, as the stock route is replicated too.
``LAMB`` and ``LARS`` (defined here; torch.optim has neither) take ``stk_layerwise_step``: per-parameter trust ratios from
two whole-parameter norms, per-parameter step counts on the device, the classes' own state_dict layout, and the same
replicated all-reduce route at world > 1.

``B200StockOptimizer`` -- every other ``torch.optim`` class (the reference instantiates whatever class the user passes,
stoke/extensions.py:53-78) and the options the fused step does not cover (amsgrad, capturable, differentiable, more than 8
groups): the gradient path
is still the engine's (K1 reduce with fused cast / unscale / inf test / norm, the clip applied by ``k_grad_scale``); the
update itself is the stock optimizer stepping on per-parameter fp32 views of the flat master / main-grad buffers.
"""
from typing import Dict, List, Optional, Type

import torch

from . import _lib, layout
from .engine import ClipSpec, Engine, GradPath

_KINDS = {torch.optim.Adam: _lib.OPT_ADAM, torch.optim.AdamW: _lib.OPT_ADAMW, torch.optim.SGD: _lib.OPT_SGD,
          torch.optim.NAdam: _lib.OPT_NADAM, torch.optim.RAdam: _lib.OPT_RADAM, torch.optim.Adamax: _lib.OPT_ADAMAX,
          torch.optim.Adadelta: _lib.OPT_ADADELTA, torch.optim.Rprop: _lib.OPT_RPROP, torch.optim.ASGD: _lib.OPT_ASGD}
# per-step scalars from stk_optim_step_prologue
_EXT_KINDS = (_lib.OPT_NADAM, _lib.OPT_RADAM, _lib.OPT_ADAMAX, _lib.OPT_ADADELTA, _lib.OPT_RPROP, _lib.OPT_ASGD)
# element-wise classes whose state torch creates at a parameter's first step (no state_dict entry before it)
_LAZY_KINDS = (_lib.OPT_ADADELTA, _lib.OPT_RPROP, _lib.OPT_ASGD)
# torch's per-parameter state keys of the two fp32 buffers M and V (None: no V buffer)
_STATE_KEYS = {_lib.OPT_SGD: ("momentum_buffer", None),
               _lib.OPT_ADAM: ("exp_avg", "exp_avg_sq"), _lib.OPT_ADAMW: ("exp_avg", "exp_avg_sq"),
               _lib.OPT_NADAM: ("exp_avg", "exp_avg_sq"), _lib.OPT_RADAM: ("exp_avg", "exp_avg_sq"),
               _lib.OPT_ADAMAX: ("exp_avg", "exp_inf"), _lib.OPT_ADADELTA: ("square_avg", "acc_delta"),
               _lib.OPT_RPROP: ("prev", "step_size"), _lib.OPT_ASGD: ("ax", None)}
# per-entry scalar state carried by the step prologue: NAdam's mu_product, ASGD's (eta, mu), torch's 0-dim fp32 tensors
_SCALAR_KEYS = {_lib.OPT_NADAM: ("mu_product",), _lib.OPT_ASGD: ("eta", "mu")}
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


# LAMB and LARS run on their own entry point, stk_layerwise_step (per-parameter trust ratios), not as kinds of K2
_LAMB, _LARS = "lamb", "lars"
_KINDS[LAMB] = _LAMB
_KINDS[LARS] = _LARS
_LAYERWISE = {_LAMB: _lib.LW_LAMB, _LARS: _lib.LW_LARS}


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
                     momentum: Optional[List[float]] = None):
    """How a loaded state dict's step counts and scalar state (NAdam's ``mu_product``, ASGD's ``eta`` / ``mu``) go onto
    the fused step.  ``entries``: torch's state entry of every parameter in flat order (``{}`` where it has none);
    ``opt_steps``: the checkpoint's ``b200_opt_steps`` (None in a torch-written one); ``per_param_on``: the step already
    keeps per-parameter counts; ``momentum``: SGD's per-group momentum.

    torch creates a parameter's state at its first step, so a parameter without an entry has taken 0 steps and has the
    initial scalar state (1.0).  torch's SGD keeps no ``step``: a parameter with a ``momentum_buffer`` has taken
    ``opt_steps`` steps (1 in a torch-written checkpoint), one without it 0; in a group without momentum the count has no
    effect and is the optimizer-wide one.

    Returns ``(opt_steps, steps, scalars)``: the optimizer-wide count, then either per-parameter counts and per-parameter
    scalar state (``steps`` a list) or ``steps = None`` and per-group scalar state.  Counts go per parameter when they
    are not all the optimizer-wide count, when the scalar state differs within a group, or when ``per_param_on``.
    ``scalars`` is None for the kinds without scalar state."""
    def count(e, g):
        if kind != _lib.OPT_SGD:
            return int(float(e["step"])) if "step" in e else 0
        if momentum[g] == 0:
            return None
        if e.get("momentum_buffer") is None:
            return 0
        return 1 if opt_steps is None else opt_steps

    keys = _SCALAR_KEYS.get(kind, ())
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
                f"Stoke -- the fused step covers torch.optim.Adam, AdamW, SGD, NAdam, RAdam, Adamax, Adadelta, Rprop, ASGD and Adafactor and stoke_b200.optim.LAMB and LARS; got {getattr(optim_cls, '__name__', optim_cls)}"
                f" (use B200StockOptimizer / build_optimizer, which routes other classes to the stock-optimizer path)")
        params, group_of, extra, kw = _group_layout(module, optim_kwargs)
        if len(extra) > _lib.MAX_GROUPS:
            raise NotImplementedError(f"Stoke -- the fused step handles up to {_lib.MAX_GROUPS} parameter groups")
        # let torch validate the kwargs exactly as the reference would (optimizer(params=..., **kwargs))
        probe = optim_cls([dict(g, params=[torch.nn.Parameter(torch.zeros(1))]) for g in extra], **kw)
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
        sgd = self._kind == _lib.OPT_SGD
        any_mom = any(g.get("momentum", 0) != 0 for g in probe.param_groups)
        ada = self._kind == _ADAFACTOR
        lw = self._kind in _LAYERWISE
        lars = self._kind == _LARS
        if (ada or lw) and engine.world > 1:
            # Adafactor's per-parameter reductions and LAMB's / LARS's trust ratios need whole parameters on one rank: their
            # state is replicated (also under fairscale_oss) and every rank runs the same deterministic step on the same
            # all-reduced fp32 gradients
            route = "allreduce"
        self.path = GradPath(engine, params, grad_accum=grad_accum, clip=clip, sharded=sharded, lp_dtype=lp_dtype,
                             module=module, needs_second_moment=not (sgd or ada or lars or self._kind == _lib.OPT_ASGD),
                             needs_first_moment=not (sgd or ada or lars) or any_mom, state_id=state_id, route=route,
                             group_of=group_of, bucket_mb=bucket_mb, scalar_state=len(_SCALAR_KEYS.get(self._kind, ())),
                             adafactor=ada, layerwise=lw)
        by_group: List[List[torch.nn.Parameter]] = [[] for _ in extra]
        for p, gi in zip(params, group_of):
            by_group[gi].append(p)
        super().__init__([dict(g, params=ps) for g, ps in zip(extra, by_group)], dict(probe.defaults))
        self._group_of = group_of
        # position of every parameter inside torch's state_dict numbering (group by group, in group order)
        self._sd_index = state_dict_index(group_of, len(extra))
        engine.scaler_set(state=self.path.state_id, opt_steps=0, skipped_steps=0, found_inf=0, growth_tracker=0)

    # -- the step -------------------------------------------------------------------------------------------------------
    @staticmethod
    def _adafactor_hyper_of(g) -> _lib.AdafactorHyper:
        h = _lib.AdafactorHyper()
        eps1, eps2 = g["eps"]
        h.lr, h.beta2_decay, h.eps2, h.d = float(g["lr"]), float(g["beta2_decay"]), float(eps2), float(g["d"])
        h.weight_decay = float(g["weight_decay"])
        h.eps1_none, h.eps1 = int(eps1 is None), float(eps1 if eps1 is not None else 0.0)
        h.maximize = int(bool(g.get("maximize", False)))
        return h

    @staticmethod
    def _layerwise_hyper_of(g) -> _lib.LayerwiseHyper:
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
        elif "betas" in g:
            h.beta1, h.beta2 = (float(b) for b in g["betas"])
            h.eps = float(g["eps"])
        elif "eps" in g:   # Adadelta
            h.eps = float(g["eps"])
        return h

    def _hyper(self) -> _lib.OptimHyper:
        return self._hyper_of(self.param_groups[0])

    def _hypers(self) -> List[_lib.OptimHyper]:
        return [self._hyper_of(g) for g in self.param_groups]

    def _exts(self) -> Optional[List[_lib.OptimHyperExt]]:
        if self._kind not in _EXT_KINDS:
            return None
        out = []
        for g in self.param_groups:
            x = _lib.OptimHyperExt()
            x.momentum_decay = float(g.get("momentum_decay", 0.0))
            x.decoupled_weight_decay = int(bool(g.get("decoupled_weight_decay", False)))
            x.rho = float(g.get("rho", 0.0))
            x.etaminus, x.etaplus = (float(e) for e in g.get("etas", (0.0, 0.0)))
            x.step_size_min, x.step_size_max = (float(e) for e in g.get("step_sizes", (0.0, 0.0)))
            x.lambd, x.alpha, x.t0 = float(g.get("lambd", 0.0)), float(g.get("alpha", 0.0)), float(g.get("t0", 0.0))
            out.append(x)
        return out

    @torch.no_grad()
    def step(self, closure=None):
        if closure is not None:
            raise NotImplementedError("Stoke -- closures are not supported by the fused step")
        if self._kind == _ADAFACTOR:
            self.path.adafactor_step([self._adafactor_hyper_of(g) for g in self.param_groups])
            return
        if self._kind in _LAYERWISE:
            self.path.layerwise_step(_LAYERWISE[self._kind], [self._layerwise_hyper_of(g) for g in self.param_groups])
            return
        self.path.optimizer_step(self._hypers(), self._exts())

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
    def _full(self, flat: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        if flat is None:
            return None
        return self.path._gather_shards(flat) if self.path.sharded else flat

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

    def _adafactor_state_dict(self):
        """torch's format: a parameter that was never stepped has no entry (torch creates its state at its first gradient)."""
        path = self.path
        steps = path.param_steps()
        state = {}
        for i, views in enumerate(path.adafactor_state_views()):
            if steps[i] == 0:
                continue
            keys = ("row_var", "col_var") if len(views) == 2 else ("variance",)
            state[self._sd_index[i]] = dict({"step": torch.tensor(float(steps[i]))},
                                            **{k: v.clone() for k, v in zip(keys, views)})
        return self._export(state)

    def _layerwise_state_dict(self):
        """The classes' own format: a parameter that was never stepped has no entry; ``step``, then LAMB's ``exp_avg`` /
        ``exp_avg_sq`` or, in a LARS group with momentum, ``momentum_buffer``."""
        path = self.path
        steps = path.param_steps()
        ms = path.unflatten(path.m_flat) if path.m_flat is not None else None
        vs = path.unflatten(path.v_flat) if path.v_flat is not None else None
        state = {}
        for i in range(len(path.params)):
            if steps[i] == 0:
                continue
            d = {"step": torch.tensor(float(steps[i]))}
            if self._kind == _LAMB:
                d["exp_avg"], d["exp_avg_sq"] = ms[i].clone(), vs[i].clone()
            elif self.param_groups[self._group_of[i]]["momentum"] != 0:
                d["momentum_buffer"] = ms[i].clone()
            state[self._sd_index[i]] = d
        return self._export(state)

    def state_dict(self):
        """torch's per-parameter format: ``step``, the scalar state (NAdam's ``mu_product``, ASGD's ``eta`` and ``mu``) as
        0-dim fp32 tensors, then the class's state tensors.  Adadelta, Rprop and ASGD omit a parameter that was never
        stepped (torch creates their state at its first gradient); the other kinds emit it.  SGD emits only
        ``momentum_buffer``, None before a parameter's first step or without momentum."""
        path = self.path
        if self._kind == _ADAFACTOR:
            return self._adafactor_state_dict()
        if self._kind in _LAYERWISE:
            return self._layerwise_state_dict()
        k_m, k_v = _STATE_KEYS[self._kind]
        ms = path.unflatten(self._full(path.m_flat)) if path.m_flat is not None else None
        vs = path.unflatten(self._full(path.v_flat)) if k_v is not None else None
        steps = path.param_steps()
        scal = path.param_scalars() if self._kind in _SCALAR_KEYS else None
        state = {}
        for i in range(len(path.params)):
            j = self._sd_index[i]
            if self._kind == _lib.OPT_SGD:
                state[j] = {k_m: ms[i].clone() if ms is not None and steps[i] > 0 else None}
                continue
            if steps[i] == 0 and self._kind in _LAZY_KINDS:
                continue
            d = {"step": torch.tensor(float(steps[i]))}
            if scal is not None:
                for key, val in zip(_SCALAR_KEYS[self._kind], scal[i]):
                    d[key] = torch.tensor(val, dtype=torch.float32)
            d[k_m] = ms[i].clone()
            if k_v is not None:
                d[k_v] = vs[i].clone()
            state[j] = d
        return self._export(state)

    def load_state_dict(self, sd):
        """Accepts this class's own export and a plain ``torch.optim`` state dict written by the reference
        (stoke/io_ops.py:224-236): without ``b200_master`` the fp32 master weights are rebuilt from the model parameters
        that ``model.load_state_dict`` has just filled (load order of BaseStokeIO.load).  Step counts and scalar state
        follow torch's lazy state creation (``load_step_counts``)."""
        path = self.path
        for g, src in zip(self.param_groups, sd["param_groups"]):
            for k, val in src.items():
                if k != "params":
                    g[k] = val
        dev = path.p_flat.device
        entries = [sd["state"].get(self._sd_index[i], {}) for i in range(len(path.params))]
        if self._kind == _ADAFACTOR:
            for src, views in zip(entries, path.adafactor_state_views()):
                keys = ("row_var", "col_var") if len(views) == 2 else ("variance",)
                for k, v in zip(keys, views):
                    if k in src:
                        v.copy_(src[k].to(device=dev, dtype=torch.float32).reshape(v.shape))
                    else:
                        v.zero_()
        else:
            keys = _STATE_KEYS[self._kind] if self._kind not in _LAYERWISE else \
                (("exp_avg", "exp_avg_sq") if self._kind == _LAMB else ("momentum_buffer", None))
            for local_dst, key in zip((path.m_flat, path.v_flat), keys):
                if local_dst is None:
                    continue
                full = torch.zeros(path.n, dtype=torch.float32, device=dev)
                for view, src in zip(path.unflatten(full), entries):
                    if src.get(key) is not None:
                        view.copy_(src[key].to(device=dev, dtype=torch.float32))
                path.scatter_local(full, local_dst)
        steps, per_param, scalars = load_step_counts(self._kind, entries, self._group_of, sd.get("b200_opt_steps"),
                                                     path._range_steps is not None,
                                                     [g.get("momentum", 0.0) for g in self.param_groups])
        if per_param is not None:
            path.enable_per_param_steps(per_param, scalars)
        elif scalars is not None:
            path.set_group_scalars(scalars)
        if "b200_master" in sd:
            master = sd["b200_master"].to(device=dev, dtype=torch.float32)
            if path.master_flat is not path.p_flat:
                path.scatter_local(master, path.master_flat)
            path.p_flat.copy_(master)
        elif path.master_flat is not path.p_flat:
            # reference-written checkpoint: the model weights are already in P (model dtype); they are the best master
            path.scatter_local(path.p_flat.float(), path.master_flat)
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
                             module=module, needs_second_moment=False, needs_first_moment=False, state_id=state_id,
                             route="allreduce" if engine.world > 1 else "main", group_of=None, bucket_mb=bucket_mb)
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

    @torch.no_grad()
    def step(self, closure=None):
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
