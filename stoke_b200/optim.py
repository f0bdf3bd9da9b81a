# -*- coding: utf-8 -*-
"""The optimizer objects ``Stoke.optimizer`` hands back.

``B200FusedOptimizer`` -- a ``torch.optim.Optimizer`` (so LR schedulers and ``param_groups`` edits work, README.md:241-250
of the reference) whose ``step()`` is the single fused K2 launch over the flat fp32 master / moment buffers; its sharded
flavour is the ZeRO-1 analogue of fairscale ``OSS`` (/root/reference/stoke/extensions.py:109-141): same ``clip_grad_norm`` /
``consolidate_state_dict`` surface.  Adam, AdamW, SGD(-momentum), NAdam, RAdam and Adamax, up to 8 parameter groups
(per-group lr / betas / eps / weight decay / momentum ... selected inside the kernel by element range).  NAdam, RAdam and
Adamax keep two fp32 state tensors per parameter like Adam (Adamax's ``exp_inf`` in the second-moment buffer); their
per-step scalars, and NAdam's ``mu_product``, are formed on the device by ``stk_optim_step_prologue``.
``torch.optim.Adafactor`` takes its own fused entry point, ``stk_adafactor_step`` (per-parameter reductions: row / column
means of g^2, the parameter's RMS, the update's RMS), with per-parameter step counts on the device and torch's
state_dict layout (``row_var`` / ``col_var`` or ``variance``).  Its state is never sharded: the reductions need whole
parameters on one rank, so at world > 1 (``fairscale_oss=True`` included) it runs replicated on the all-reduce route,
every rank taking the same deterministic step on the same gradients, as the stock route is replicated too.

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
          torch.optim.NAdam: _lib.OPT_NADAM, torch.optim.RAdam: _lib.OPT_RADAM, torch.optim.Adamax: _lib.OPT_ADAMAX}
_EXT_KINDS = (_lib.OPT_NADAM, _lib.OPT_RADAM, _lib.OPT_ADAMAX)   # per-step scalars from stk_optim_step_prologue
# torch's per-parameter state keys of the two fp32 buffers M and V
_STATE_KEYS = {_lib.OPT_ADAM: ("exp_avg", "exp_avg_sq"), _lib.OPT_ADAMW: ("exp_avg", "exp_avg_sq"),
               _lib.OPT_NADAM: ("exp_avg", "exp_avg_sq"), _lib.OPT_RADAM: ("exp_avg", "exp_avg_sq"),
               _lib.OPT_ADAMAX: ("exp_avg", "exp_inf")}
_STOCK_ONLY_TRUE = ("amsgrad", "capturable", "differentiable")
# torch.optim.Adafactor (torch >= 2.5) runs on its own entry point, stk_adafactor_step, not as a kind of K2
_ADAFACTOR = "adafactor"
if hasattr(torch.optim, "Adafactor"):
    _KINDS[torch.optim.Adafactor] = _ADAFACTOR


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
                f"Stoke -- the fused step covers torch.optim.Adam, AdamW, SGD, NAdam, RAdam, Adamax and Adafactor; got {getattr(optim_cls, '__name__', optim_cls)}"
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
        if ada and engine.world > 1:
            # Adafactor's per-parameter reductions need whole parameters on one rank: its state is replicated (also under
            # fairscale_oss) and every rank runs the same deterministic step on the same all-reduced fp32 gradients
            route = "allreduce"
        self.path = GradPath(engine, params, grad_accum=grad_accum, clip=clip, sharded=sharded, lp_dtype=lp_dtype,
                             module=module, needs_second_moment=not (sgd or ada),
                             needs_first_moment=not (sgd or ada) or any_mom, state_id=state_id, route=route,
                             group_of=group_of, bucket_mb=bucket_mb, mu_product=self._kind == _lib.OPT_NADAM,
                             adafactor=ada)
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
        else:
            h.beta1, h.beta2 = (float(b) for b in g["betas"])
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
            out.append(x)
        return out

    @torch.no_grad()
    def step(self, closure=None):
        if closure is not None:
            raise NotImplementedError("Stoke -- closures are not supported by the fused step")
        if self._kind == _ADAFACTOR:
            self.path.adafactor_step([self._adafactor_hyper_of(g) for g in self.param_groups])
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

    def _adafactor_state_dict(self):
        """torch's format: a parameter that was never stepped has no entry (torch creates its state at its first gradient)."""
        path = self.path
        st = path.engine.scaler_get(path.state_id)
        steps = path.param_steps()
        state = {}
        for i, views in enumerate(path.adafactor_state_views()):
            if steps[i] == 0:
                continue
            keys = ("row_var", "col_var") if len(views) == 2 else ("variance",)
            state[self._sd_index[i]] = dict({"step": torch.tensor(float(steps[i]))},
                                            **{k: v.clone() for k, v in zip(keys, views)})
        return {"state": state, "param_groups": self._groups_sd(), "b200_master": path.gather_master(),
                "b200_opt_steps": int(st.opt_steps)}

    def _adafactor_load_state_dict(self, sd):
        path = self.path
        dev = path.p_flat.device
        state = sd["state"]
        steps = []
        for i, views in enumerate(path.adafactor_state_views()):
            src = state.get(self._sd_index[i], {})
            keys = ("row_var", "col_var") if len(views) == 2 else ("variance",)
            for k, v in zip(keys, views):
                if k in src:
                    v.copy_(src[k].to(device=dev, dtype=torch.float32).reshape(v.shape))
                else:
                    v.zero_()
            steps.append(int(float(src["step"])) if "step" in src else 0)
        path._range_steps.copy_(torch.tensor(steps, dtype=torch.int32))
        return int(sd.get("b200_opt_steps", max(steps)))

    def state_dict(self):
        path = self.path
        if self._kind == _ADAFACTOR:
            return self._adafactor_state_dict()
        st = path.engine.scaler_get(path.state_id)
        m, v, master = self._full(path.m_flat), self._full(path.v_flat), path.gather_master()
        state = {}
        ms = path.unflatten(m) if m is not None else None
        vs = path.unflatten(v) if v is not None else None
        steps = path.param_steps() if path._range_steps is not None else [int(st.opt_steps)] * len(path.params)
        mus = path.param_mu_products() if self._kind == _lib.OPT_NADAM else None
        for i in range(len(path.params)):
            j = self._sd_index[i]
            if self._kind == _lib.OPT_SGD:
                # torch creates the buffer on the first step; before that (or without momentum) it is None
                state[j] = {"momentum_buffer": ms[i].clone() if ms is not None and steps[i] > 0 else None}
            else:
                k_m, k_v = _STATE_KEYS[self._kind]
                state[j] = {"step": torch.tensor(float(steps[i]))}
                if mus is not None:   # torch/optim/nadam.py: a 0-dim fp32 tensor
                    state[j]["mu_product"] = torch.tensor(mus[i], dtype=torch.float32)
                state[j][k_m] = ms[i].clone()
                state[j][k_v] = vs[i].clone()
        return {"state": state, "param_groups": self._groups_sd(), "b200_master": master,
                "b200_opt_steps": int(st.opt_steps)}

    def load_state_dict(self, sd):
        """Accepts this class's own export and a plain ``torch.optim`` state dict written by the reference
        (stoke/io_ops.py:224-236): without ``b200_master`` the fp32 master weights are rebuilt from the model parameters
        that ``model.load_state_dict`` has just filled (load order of BaseStokeIO.load)."""
        path = self.path
        for g, src in zip(self.param_groups, sd["param_groups"]):
            for k, val in src.items():
                if k != "params":
                    g[k] = val
        steps = int(sd.get("b200_opt_steps", 0))
        dev = path.p_flat.device
        n = len(path.params)
        state = sd["state"]
        if self._kind == _ADAFACTOR:
            steps = self._adafactor_load_state_dict(sd)

        def put(local_dst, key):
            if local_dst is None:
                return
            full = torch.zeros(path.n, dtype=torch.float32, device=dev)
            views = path.unflatten(full)
            for i in range(n):
                src = state.get(self._sd_index[i], {}).get(key)
                if src is not None:
                    views[i].copy_(src.to(device=dev, dtype=torch.float32))
            path.scatter_local(full, local_dst)

        if self._kind == _ADAFACTOR:
            pass
        elif self._kind == _lib.OPT_SGD:
            put(path.m_flat, "momentum_buffer")
        else:
            k_m, k_v = _STATE_KEYS[self._kind]
            put(path.m_flat, k_m)
            put(path.v_flat, k_v)
            per_param = [int(float(state[self._sd_index[i]]["step"])) if self._sd_index[i] in state and "step" in state[self._sd_index[i]]
                         else None for i in range(n)]
            known = [v for v in per_param if v is not None]
            if "b200_opt_steps" not in sd and known:
                steps = max(known)
            mus = None
            if self._kind == _lib.OPT_NADAM:
                # a parameter torch never stepped has no state yet: its mu_product is torch's initial 1.0
                mus = [float(state[self._sd_index[i]]["mu_product"]) if "mu_product" in state.get(self._sd_index[i], {})
                       else 1.0 for i in range(n)]
            groups_differ = mus is not None and any(
                len({mus[i] for i in range(n) if self._group_of[i] == gi}) > 1 for gi in range(len(self.param_groups)))
            if known and (len(set(known)) > 1 or len(known) < n) or groups_differ or (
                    mus is not None and path._range_steps is not None):
                # parameters stepped a different number of times (some were unused for a while): keep torch's per-parameter counts
                path.enable_per_param_steps([steps if v is None else v for v in per_param], mu_products=mus)
            elif mus is not None:
                first = {}
                for i in range(n):
                    first.setdefault(self._group_of[i], mus[i])
                path.set_group_mu_products([first.get(gi, 1.0) for gi in range(len(self.param_groups))])
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
