# -*- coding: utf-8 -*-
"""BatchNorm2d -> [add] -> activation in one pass for bf16 channels-last training (``stk_bn_act_ex``, csrc/bn_act.cu).

``fuse_bn_act(module, engine)`` traces ``module`` with ``torch.fx`` into a ``GraphModule`` that shares every submodule,
parameter and buffer with ``module``, in which each ``BatchNorm2d -> act`` and ``BatchNorm2d -> add -> ReLU`` chain
(every intermediate with that single user) is one ``BnAct`` call.  ``act`` is ReLU, SiLU, Hardswish or ReLU6, as a module
(``nn.ReLU``, ``nn.SiLU``, ``nn.Hardswish``, ``nn.ReLU6``) or a function (``F.relu`` / ``torch.relu``, ``F.silu``,
``F.hardswish``, ``F.relu6``), in place or not; a residual add is fused only before a ReLU.  It returns a
``FusedForward``, which runs that graph only for calls it is a faithful trace of (training mode, required arguments
only, no hooks) and ``module`` itself for every other call, or None when tracing or rewriting fails or nothing matches;
the caller then keeps running ``module``.

The forward is one kernel (``stk_bn_stats_act``): the batch statistics and the running-statistics update, merged in the
order of torch's ``batch_norm_update_stats`` (the reduction the native training forward runs), then the apply / add /
activation, which rounds every intermediate as the unfused ops do.  The backward (``stk_bn_act_backward_ex``) folds the activation's
backward op (``threshold_backward``, ``silu_backward``, ``hardswish_backward``, ``hardtanh_backward``) into the two
passes of torch's channels-last ``native_batch_norm_backward`` and adds its per-channel sums in torch's order, so every
result is bit-identical to the calls autograd makes for the unfused chain.  It takes the gradient when torch's BatchNorm
backward would run its channels-last kernels on it (the activation backward's output is channels-last; another layout
is made channels-last first) and it is bf16 and aligned; otherwise it runs those calls.  A residual that is itself a
single-use BatchNorm2d output (a ResNet downsample) joins the site (``BnAct.residual_bn``): both BatchNorms' statistics,
applies, add and ReLU in the one forward launch, both backwards in its kernels.  A residual site whose output
has two users that only read it (a ResNet block output) returns it once per user (``BnAct.fork``), so that its backward
adds the two gradients in its reduce kernel, with the rounding of the bf16 add autograd would otherwise run.
Each call falls back to the unfused torch ops when the kernel does not cover its inputs (eval mode, no running statistics,
running statistics neither fp32 nor bf16, not bf16, not channels-last, misaligned, C % 8 != 0, 2^31 elements or more, a CPU tensor), so the same inputs give the
same results whether or not the model was rewritten.
"""
import functools
import inspect
import operator
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from ._lib import ACT_HARDSWISH, ACT_RELU, ACT_RELU6, ACT_SILU

_RELU_FNS = (F.relu, torch.relu)
_ADD_FNS = (operator.add, operator.iadd, torch.add)
# the activations other than ReLU, as modules and as functions (whose only other argument is ``inplace``)
_ACT_MODULES = {torch.nn.SiLU: ACT_SILU, torch.nn.Hardswish: ACT_HARDSWISH, torch.nn.ReLU6: ACT_RELU6}
_ACT_FNS = {F.silu: ACT_SILU, F.hardswish: ACT_HARDSWISH, F.relu6: ACT_RELU6}
# the unfused activation of a BnAct built without one
_DEFAULT_ACT_FN = {ACT_RELU: torch.relu, ACT_SILU: F.silu, ACT_HARDSWISH: F.hardswish, ACT_RELU6: F.relu6}
# the backward op autograd runs for each activation, as a function of (grad, activation input or ReLU output)
_ACT_BACKWARD = {
    ACT_RELU: lambda g, y: torch.ops.aten.threshold_backward(g, y, 0),
    ACT_SILU: lambda g, y: torch.ops.aten.silu_backward(g, y),
    ACT_HARDSWISH: lambda g, y: torch.ops.aten.hardswish_backward(g, y),
    ACT_RELU6: lambda g, y: torch.ops.aten.hardtanh_backward(g, y, 0, 6),
}


def _momentum(bn: torch.nn.BatchNorm2d) -> float:
    """The running-statistics bookkeeping of ``_BatchNorm.forward`` in training mode: bumps ``num_batches_tracked`` and
    returns the averaging factor (a cumulative average when ``momentum`` is None)."""
    factor = 0.0 if bn.momentum is None else bn.momentum
    if bn.num_batches_tracked is not None:
        bn.num_batches_tracked.add_(1)
        factor = 1.0 / float(bn.num_batches_tracked) if bn.momentum is None else bn.momentum
    return factor


def _aligned(*ts) -> bool:
    return all(t.data_ptr() % 16 == 0 for t in ts)


def _covered(bn: torch.nn.BatchNorm2d, x: torch.Tensor, r: Optional[torch.Tensor]) -> bool:
    if not (bn.training and bn.track_running_stats and bn.running_mean is not None and bn.running_var is not None):
        return False
    w, b = bn.weight, bn.bias
    if w is None or b is None or w.dtype != torch.bfloat16 or b.dtype != torch.bfloat16:
        return False
    rm, rv = bn.running_mean, bn.running_var
    if not (rm.dtype in (torch.float32, torch.bfloat16) and rv.dtype == rm.dtype and rm.device == x.device
            and rv.device == x.device and rm.is_contiguous() and rv.is_contiguous()):
        return False
    if not (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and x.is_contiguous(memory_format=torch.channels_last)):
        return False
    n, c = x.numel(), x.shape[1]
    if c % 8 or n // c < 2 or n >= 2 ** 31 or not (w.is_contiguous() and b.is_contiguous() and _aligned(x, w, b)):
        return False
    if r is not None and not (r.shape == x.shape and r.dtype == x.dtype and r.device == x.device
                              and r.is_contiguous(memory_format=torch.channels_last) and _aligned(r)):
        return False
    return True


def _grad_covered(grad: torch.Tensor, x: torch.Tensor) -> bool:
    """The backward kernel takes ``grad`` when torch would run its channels-last BatchNorm backward on it."""
    return (grad.dtype == torch.bfloat16 and grad.device == x.device and grad.shape == x.shape
            and grad.is_contiguous(memory_format=torch.channels_last) and _aligned(grad))


def _mask_output_channels_last(grad: torch.Tensor, x: torch.Tensor, act: int = ACT_RELU) -> bool:
    """Whether the activation's backward op (``threshold_backward(grad, out)``, ``silu_backward(grad, y)``, ...; ``out``
    and ``y`` laid out like ``x``) returns a channels-last tensor, which is what decides whether torch's BatchNorm
    backward runs its channels-last kernels.  Asked of a structured op's meta kernel, which is TensorIterator's own
    layout logic: ``threshold_backward``'s for ReLU (its iterator takes ``out`` first, so an NCHW gradient gives a
    channels-last output), ``silu_backward``'s for the others.  ``silu_backward``, ``hardswish_backward`` and
    ``hardtanh_backward`` are all binary TensorIterator ops over (grad, y), so an NCHW gradient gives an NCHW output;
    the Python meta functions of the latter two lay it out differently from their CUDA kernels, so they are not asked.
    A gradient arriving expanded (the average pool's backward) gets a channels-last output from all of them."""
    def meta(t):
        return torch.empty_strided(t.shape, t.stride(), dtype=t.dtype, device="meta")

    op = _ACT_BACKWARD[ACT_RELU if act == ACT_RELU else ACT_SILU]
    return op(meta(grad), meta(x)).is_contiguous(memory_format=torch.channels_last)


class _BnActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, residual, bn, engine, act, fork, weight2, bias2, rbn):
        momentum = _momentum(bn)
        out = torch.empty_like(x)
        mean = torch.empty(x.shape[1], dtype=torch.float32, device=x.device)
        invstd = torch.empty_like(mean)
        second, saved2 = None, ()
        if rbn is not None:   # the residual is rbn's input: relu(bn(x) + rbn(residual))
            mean2, invstd2 = torch.empty_like(mean), torch.empty_like(mean)
            second = (weight2, bias2, rbn.running_mean, rbn.running_var, _momentum(rbn), rbn.eps, mean2, invstd2)
            saved2 = (residual, weight2, mean2, invstd2)
        engine.bn_stats_act(x, residual, weight, bias, bn.running_mean, bn.running_var, momentum, bn.eps, out, mean,
                            invstd, act, residual_bn=second)
        # the ReLU mask: out at a site with a residual; otherwise the activation's input is recomputed from x and the
        # parameters (bias saved instead)
        ctx.save_for_backward(x, weight, out if residual is not None else bias, mean, invstd, *saved2)
        ctx.bn, ctx.engine, ctx.act, ctx.rbn = bn, engine, act, rbn
        ctx.has_residual = residual is not None
        if not fork:
            return out
        # two outputs over one storage, one per user: autograd hands their gradients to backward separately, which adds
        # them inside the reduce kernel instead of in a bf16 add of its own
        ctx.set_materialize_grads(False)
        return out, out.detach()

    @staticmethod
    def backward(ctx, grad_out, grad2=None):
        x, weight, out_or_bias, mean, invstd, *saved2 = ctx.saved_tensors
        bn, res, act, rbn = ctx.bn, ctx.has_residual, ctx.act, ctx.rbn
        need_x, need_w, need_b, need_r = ctx.needs_input_grad[:4]
        need_w2, need_b2 = ctx.needs_input_grad[8:10]
        if grad_out is None:
            grad_out, grad2 = grad2, None
        if grad_out is None:
            return (None,) * 11
        if grad2 is not None and not (_grad_covered(grad_out, x) and _grad_covered(grad2, x)):
            grad_out, grad2 = grad_out + grad2, None   # the add autograd runs for an output with two users
        if (grad_out.dtype == torch.bfloat16 and grad_out.shape == x.shape
                and not grad_out.is_contiguous(memory_format=torch.channels_last)
                and _mask_output_channels_last(grad_out, x, act)):
            grad_out = grad_out.contiguous(memory_format=torch.channels_last)   # same values, so the same g
        if _grad_covered(grad_out, x):
            dw, db = torch.empty_like(weight), torch.empty_like(weight)
            dr = torch.empty_like(x) if res else None   # g at a site whose residual has its own BatchNorm
            if rbn is not None:
                x2, w2, mean2, invstd2 = saved2
                dx = torch.empty_like(x) if need_x or need_r else None
                dx2 = torch.empty_like(x2) if dx is not None else None
                dw2, db2 = torch.empty_like(w2), torch.empty_like(w2)
                ctx.engine.bn_act_backward(grad_out, x, out_or_bias, mean, invstd, weight, None, dx, dw, db, dr, act,
                                           grad2=grad2, residual_bn=(x2, mean2, invstd2, w2, dx2, dw2, db2))
                return (dx if need_x else None, dw if need_w else None, db if need_b else None,
                        dx2 if need_r else None, None, None, None, None,
                        dw2 if need_w2 else None, db2 if need_b2 else None, None)
            dx = torch.empty_like(x) if need_x else None
            ctx.engine.bn_act_backward(grad_out, x, out_or_bias if res else None, mean, invstd, weight,
                                       None if res else out_or_bias, dx, dw, db, dr, act, grad2=grad2)
            return (dx, dw if need_w else None, db if need_b else None, dr if need_r else None) + (None,) * 7
        # without a residual y = batch_norm_elemt(x) (the transform the forward kernel reproduces) is the activation's
        # input, which its backward op takes (threshold_backward takes relu's output, but relu(y) <= 0 exactly when y <= 0)
        out = out_or_bias if res else torch.batch_norm_elemt(x, weight, out_or_bias, mean, invstd, bn.eps)
        g = _ACT_BACKWARD[act](grad_out, out)
        mask = [need_x, need_w, need_b]
        dx, dw, db = torch.ops.aten.native_batch_norm_backward(g, x, weight, bn.running_mean, bn.running_var, mean, invstd,
                                                              True, bn.eps, mask)
        if rbn is not None:   # the residual BatchNorm's backward of the same g
            x2, w2, mean2, invstd2 = saved2
            dx2, dw2, db2 = torch.ops.aten.native_batch_norm_backward(g, x2, w2, rbn.running_mean, rbn.running_var, mean2,
                                                                     invstd2, True, rbn.eps, [need_r, need_w2, need_b2])
            return dx, dw, db, dx2, None, None, None, None, dw2, db2, None
        dr = g if res and need_r else None
        return (dx, dw, db, dr) + (None,) * 7


class BnAct(torch.nn.Module):
    """``act(bn(x) [+ residual])``: one ``stk_bn_stats_act`` launch when the kernel covers the inputs, the unfused torch
    ops otherwise (``inplace``: the add was ``out += residual``, which keeps ``out``'s dtype).  ``act`` is one of
    ``_lib.ACT_*``; only ReLU takes a residual.  ``act_fn`` is the unfused activation (the user's module or function),
    by default ``torch.relu``, ``F.silu``, ``F.hardswish`` or ``F.relu6``.  Holds a reference to the user's BatchNorm2d
    (shared, not copied).  ``fork`` (a site with a residual whose output has two users that do not mutate it): returns
    the output twice, as two tensors over one storage, so that the backward receives the two users' gradients apart
    and adds them in its reduce kernel; the unfused fallback returns the same tensor twice, which autograd sums.
    ``residual_bn`` (a ReLU site; shared with the user's model, not copied): the residual passes through this second
    BatchNorm2d first, ``relu(bn(x) + residual_bn(residual))``, in the same launch when the kernel covers both; when it
    covers only the first, ``residual_bn`` runs in torch and its output is the residual."""

    def __init__(self, bn: torch.nn.BatchNorm2d, engine, inplace: bool = False, act: int = ACT_RELU, act_fn=None,
                 fork: bool = False, residual_bn: Optional[torch.nn.BatchNorm2d] = None):
        super().__init__()
        if act not in _DEFAULT_ACT_FN:
            raise ValueError(f"unknown activation kind {act}")
        if residual_bn is not None and (act != ACT_RELU or residual_bn is bn):
            raise ValueError("BnAct: residual_bn needs a ReLU site and a BatchNorm2d of its own")
        self.bn = bn
        self.residual_bn = residual_bn
        self.act = act
        self.fork = fork
        self._engine = engine
        self._inplace = inplace
        self._act_fn = act_fn if act_fn is not None else _DEFAULT_ACT_FN[act]

    def forward(self, x, residual=None):
        if residual is not None and self.act != ACT_RELU:
            raise ValueError("BnAct: only a ReLU site takes a residual")
        if self.fork and residual is None:
            raise ValueError("BnAct: only a site with a residual forks")
        rbn = self.residual_bn
        if rbn is not None:
            if residual is None:
                raise ValueError("BnAct: a site with residual_bn takes a residual")
            if (_covered(self.bn, x, residual) and _covered(rbn, residual, None)
                    and rbn.running_mean.dtype == self.bn.running_mean.dtype):
                return _BnActFn.apply(x, self.bn.weight, self.bn.bias, residual, self.bn, self._engine, self.act,
                                      self.fork, rbn.weight, rbn.bias, rbn)
            residual = rbn(residual)
        if _covered(self.bn, x, residual):
            return _BnActFn.apply(x, self.bn.weight, self.bn.bias, residual, self.bn, self._engine, self.act, self.fork,
                                  None, None, None)
        y = self.bn(x)
        if residual is not None:
            if self._inplace:
                y += residual
            else:
                y = y + residual
        y = self._act_fn(y)
        return (y, y) if self.fork else y


class _InplaceProxy(torch.fx.Proxy):
    """Records ``a += b`` as ``operator.iadd`` (plain fx rebinds the name to ``a + b``, which drops the mutation and, for
    mixed dtypes, changes the result's dtype)."""


for _op in ("iadd", "isub", "imul", "itruediv"):
    setattr(_InplaceProxy, f"__{_op}__",
            lambda self, other, _f=getattr(operator, _op): self.tracer.create_proxy("call_function", _f, (self, other), {}))


class _Tracer(torch.fx.Tracer):
    def proxy(self, node):
        return _InplaceProxy(node, self)


class FusedForward:
    """Calls the rewritten graph in place of ``module`` when the call is one the graph is a faithful trace of, and
    ``module`` itself otherwise.  The graph was traced in training mode with every optional argument at its default, and
    it inlines containers, so it is used only when every submodule is in training mode, the call passes exactly the
    required arguments positionally, and no module or global hook is registered."""

    def __init__(self, module: torch.nn.Module, gm: torch.fx.GraphModule, n_required: int, sites: int):
        self.module, self.graph_module, self.fused_sites = module, gm, sites
        self._n_required = n_required
        self._modules = list(module.modules())

    def _graph_applies(self, args, kwargs) -> bool:
        if kwargs or len(args) != self._n_required:
            return False
        g = torch.nn.modules.module
        if any(getattr(g, h, None) for h in _GLOBAL_HOOKS):
            return False
        return all(m.training and not (m._forward_hooks or m._forward_pre_hooks or m._backward_hooks
                                       or m._backward_pre_hooks) for m in self._modules)

    def __call__(self, *args, **kwargs):
        if self._graph_applies(args, kwargs):
            return self.graph_module(*args)
        return self.module(*args, **kwargs)


_GLOBAL_HOOKS = ("_global_forward_hooks", "_global_forward_pre_hooks", "_global_backward_hooks",
                 "_global_backward_pre_hooks")


def _is_relu(gm: torch.fx.GraphModule, node: torch.fx.Node) -> bool:
    if node.op == "call_module":
        return type(gm.get_submodule(node.target)) is torch.nn.ReLU
    return node.op == "call_function" and node.target in _RELU_FNS


def _other_act(gm: torch.fx.GraphModule, node: torch.fx.Node):
    """(kind, unfused activation) when ``node`` is a SiLU, Hardswish or ReLU6 module call, or a call of its function
    whose only other argument is a constant ``inplace``; None otherwise."""
    if node.op == "call_module":
        m = gm.get_submodule(node.target)
        return (_ACT_MODULES[type(m)], m) if type(m) in _ACT_MODULES else None
    if node.op != "call_function" or node.target not in _ACT_FNS:
        return None
    kwargs = dict(node.kwargs)
    if len(node.args) == 2 and "inplace" not in kwargs:   # f(input, inplace): bound by name, after the input
        kwargs["inplace"] = node.args[1]
    elif len(node.args) != 1:
        return None
    if set(kwargs) - {"inplace"} or any(isinstance(a, torch.fx.Node) for a in kwargs.values()):
        return None
    return _ACT_FNS[node.target], functools.partial(node.target, **kwargs)


def _single_bn_input(gm: torch.fx.GraphModule, node) -> bool:
    """``node`` is a BatchNorm2d call on one tensor whose only user is the next node of the chain."""
    return (isinstance(node, torch.fx.Node) and node.op == "call_module" and len(node.users) == 1
            and type(gm.get_submodule(node.target)) is torch.nn.BatchNorm2d and len(node.args) == 1 and not node.kwargs)


def _trace(module: torch.nn.Module):
    """(graph module traced in training mode with every optional argument at its default, number of required
    arguments); the module's training flags are restored afterwards."""
    params = list(inspect.signature(module.forward).parameters.values())
    if any(p.kind in (p.VAR_POSITIONAL, p.VAR_KEYWORD, p.KEYWORD_ONLY) for p in params):
        raise TypeError("only positional forward arguments are traced")
    required = [p for p in params if p.default is p.empty]   # positional: the ones with defaults come last
    flags = [(m, m.training) for m in module.modules()]
    module.train()
    try:
        graph = _Tracer().trace(module, concrete_args={p.name: p.default for p in params[len(required):]})
    finally:
        for m, t in flags:
            m.training = t
    return torch.fx.GraphModule(module, graph), len(required)


def _rewrite(gm: torch.fx.GraphModule, engine) -> int:
    sites = 0
    for relu in list(gm.graph.nodes):   # the activation node (a ReLU, or another kind when `other` is set)
        is_relu = _is_relu(gm, relu)
        other = None if is_relu else _other_act(gm, relu)
        if not (is_relu or other) or not relu.args:
            continue
        src, residual, inplace = relu.args[0], None, False
        # a residual add is fused only before a ReLU
        if (other is None and isinstance(src, torch.fx.Node) and src.op == "call_function" and src.target in _ADD_FNS
                and len(src.users) == 1 and len(src.args) == 2 and not src.kwargs
                and all(isinstance(a, torch.fx.Node) for a in src.args)):
            a, b = src.args
            inplace = src.target is operator.iadd
            # an out-of-place add takes the BatchNorm on either side (two-operand float addition is commutative); `+=`
            # only on the left, where the tensor it mutates is the BatchNorm output nothing else sees
            bn_node, residual = (a, b) if _single_bn_input(gm, a) or inplace else (b, a)
            if bn_node is residual:
                continue
            chain = [relu, src]
        else:
            bn_node, chain = src, [relu]
        if not _single_bn_input(gm, bn_node):
            continue
        name = bn_node.target.replace(".", "_") + "_act"
        bn = gm.get_submodule(bn_node.target)
        # a residual that is itself a BatchNorm's single-use output (a ResNet downsample) joins the site
        rbn_node = None
        if (residual is not None and _single_bn_input(gm, residual)
                and gm.get_submodule(residual.target) is not bn):
            rbn_node, residual = residual, residual.args[0]
        gm.add_submodule(name, BnAct(bn, engine, inplace, residual_bn=rbn_node and gm.get_submodule(rbn_node.target))
                         if other is None else BnAct(bn, engine, act=other[0], act_fn=other[1]))
        with gm.graph.inserting_before(relu):
            fused = gm.graph.call_module(name, (bn_node.args[0],) + ((residual,) if residual is not None else ()))
        relu.replace_all_uses_with(fused)
        for n in chain + [bn_node] + ([rbn_node] if rbn_node is not None else []):
            gm.graph.erase_node(n)
        sites += 1
    return sites


def _reads_only(gm: torch.fx.GraphModule, user: torch.fx.Node, node: torch.fx.Node) -> bool:
    """``user`` takes ``node`` once and does not mutate it: a Conv2d, or a BnAct (which never writes its inputs)."""
    if user.op != "call_module" or user.kwargs or list(user.args).count(node) != 1:
        return False
    m = gm.get_submodule(user.target)
    return type(m) is torch.nn.Conv2d or isinstance(m, BnAct)


def _fork(gm: torch.fx.GraphModule) -> int:
    """Sets ``fork`` on each residual-site BnAct whose output has exactly two users that only read it (a ResNet block
    output: the next block's conv1, and its identity or downsample conv), and gives each user its own output."""
    forks = 0
    for node in list(gm.graph.nodes):
        if not (node.op == "call_module" and len(node.args) == 2 and isinstance(gm.get_submodule(node.target), BnAct)):
            continue
        users = list(node.users)
        if len(users) != 2 or not all(_reads_only(gm, u, node) for u in users):
            continue
        gm.get_submodule(node.target).fork = True
        prev = node
        for i, user in enumerate(users):
            with gm.graph.inserting_after(prev):
                prev = gm.graph.call_function(operator.getitem, (node, i))
            user.replace_input_with(node, prev)
        forks += 1
    return forks


def site_shapes(fwd: FusedForward, *example) -> Dict[tuple, int]:
    """{(act, C, H, W, eps, momentum): number of sites} of a rewritten model: runs its graph once on ``example`` (meta
    tensors of a model built on the meta device work, and cost no arithmetic) with hooks on the ``BnAct`` modules."""
    sites: Dict[tuple, int] = {}

    def hook(mod, args, out):
        _, c, h, w = args[0].shape
        key = (mod.act, c, h, w, mod.bn.eps, mod.bn.momentum)
        sites[key] = sites.get(key, 0) + 1

    handles = [m.register_forward_hook(hook) for m in fwd.graph_module.modules() if isinstance(m, BnAct)]
    try:
        with torch.no_grad():
            fwd.graph_module(*example)
    finally:
        for h in handles:
            h.remove()
    return sites


def fuse_bn_act(module: torch.nn.Module, engine) -> Optional[FusedForward]:
    try:
        gm, n_required = _trace(module)
        sites = _rewrite(gm, engine)
        if sites == 0:
            return None
        _fork(gm)
        gm.graph.lint()
        gm.recompile()
    except Exception:  # noqa: BLE001 -- a model fx cannot trace or rewrite runs unchanged
        return None
    return FusedForward(module, gm, n_required, sites)
