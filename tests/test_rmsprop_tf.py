"""CPU tests of stoke_b200.RMSpropTF: the class against an independent float64 transcription of TensorFlow-style RMSprop,
argument validation, the state-dict layout, and the pieces the fused step relies on (constants, routing, the ABI struct,
step counts)."""
import copy
import ctypes as C
import os

import pytest
import torch

import stoke_b200 as sb
from stoke_b200 import _lib
from stoke_b200.optim import RMSpropTF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Ref64:
    """The RMSpropTF update in float64, written from the formulas (not from the class)."""

    def __init__(self, params, groups):
        self.p = [p.detach().double().clone() for p in params]
        self.groups = groups
        self.t = [0] * len(params)
        self.sq = [torch.ones_like(x) for x in self.p]
        self.buf = [torch.zeros_like(x) for x in self.p]
        self.ga = [torch.zeros_like(x) for x in self.p]

    def step(self, grads, group_of):
        for i, g in enumerate(grads):
            if g is None:
                continue
            h = self.groups[group_of[i]]
            lr, a, eps, wd, mom = h["lr"], h["alpha"], h["eps"], h["weight_decay"], h["momentum"]
            g = g.double()
            self.t[i] += 1
            if wd != 0:
                if h["decoupled_decay"]:
                    self.p[i] = self.p[i] * (1 - lr * wd)
                else:
                    g = g + wd * self.p[i]
            self.sq[i] = a * self.sq[i] + (1 - a) * g * g
            if h["centered"]:
                self.ga[i] = a * self.ga[i] + (1 - a) * g
                avg = torch.sqrt(self.sq[i] - self.ga[i] ** 2 + eps)
            else:
                avg = torch.sqrt(self.sq[i] + eps)
            if mom > 0:
                if h["lr_in_momentum"]:
                    self.buf[i] = mom * self.buf[i] + lr * g / avg
                    self.p[i] = self.p[i] - self.buf[i]
                else:
                    self.buf[i] = mom * self.buf[i] + g / avg
                    self.p[i] = self.p[i] - lr * self.buf[i]
            else:
                self.p[i] = self.p[i] - lr * g / avg


def _group(**kw):
    return dict(dict(lr=1e-2, alpha=0.9, eps=1e-3, weight_decay=0.0, momentum=0.0, centered=False,
                     decoupled_decay=False, lr_in_momentum=True), **kw)


# every flag both ways across five groups: momentum 0 / > 0, centered, decoupled or L2 decay, lr_in_momentum both ways
GROUPS = [_group(momentum=0.9, weight_decay=1e-2),                                       # the EfficientNet recipe
          _group(lr=3e-3, alpha=0.95, eps=1e-8, centered=True, weight_decay=5e-2, decoupled_decay=True),
          _group(lr=5e-3, momentum=0.8, centered=True, lr_in_momentum=False, weight_decay=1e-2),
          _group(lr=2e-2, alpha=0.99, eps=1e-6, momentum=0.5, lr_in_momentum=False, decoupled_decay=True,
                 weight_decay=0.1),
          _group(lr=1e-3, eps=1e-10)]


def test_class_follows_the_float64_formulas():
    """50 steps over five groups; parameter 1 gets no gradient on every third step."""
    gen = torch.Generator().manual_seed(0)
    shapes = ((7, 5), (11,), (3, 2, 2), (4,), (6,), (2, 3), (5,))
    params = [torch.nn.Parameter(torch.randn(*s, generator=gen) * 0.5) for s in shapes]
    group_of = [0, 0, 1, 2, 3, 3, 4]
    opt = RMSpropTF([dict(g, params=[p for p, gi in zip(params, group_of) if gi == j]) for j, g in enumerate(GROUPS)])
    ref = Ref64(params, GROUPS)
    for step in range(50):
        grads = [None if (i == 1 and step % 3 == 2) else torch.randn(p.shape, generator=gen) for i, p in enumerate(params)]
        for p, gr in zip(params, grads):
            p.grad = None if gr is None else gr.clone()
        opt.step()
        ref.step(grads, group_of)
        for i, p in enumerate(params):
            assert torch.allclose(p.detach().double(), ref.p[i], rtol=1e-5, atol=1e-6), (step, i)
    assert [int(opt.state[p]["step"]) for p in params] == ref.t and ref.t[1] == 34
    for i, p in enumerate(params):
        st, h = opt.state[p], GROUPS[group_of[i]]
        assert torch.allclose(st["square_avg"].double(), ref.sq[i], rtol=1e-5, atol=1e-7)
        if h["momentum"] > 0:
            assert torch.allclose(st["momentum_buffer"].double(), ref.buf[i], rtol=1e-5, atol=1e-6)
        if h["centered"]:
            assert torch.allclose(st["grad_avg"].double(), ref.ga[i], rtol=1e-5, atol=1e-7)


def test_validation():
    p = [torch.nn.Parameter(torch.zeros(2))]
    for kw in ({"lr": -1.0}, {"eps": -1.0}, {"momentum": -0.1}, {"weight_decay": -0.1}, {"alpha": -0.5}):
        with pytest.raises(ValueError):
            RMSpropTF(p, **kw)
    d = RMSpropTF(p).defaults
    assert d == dict(lr=1e-2, alpha=0.9, eps=1e-10, weight_decay=0, momentum=0.0, centered=False,
                     decoupled_decay=False, lr_in_momentum=True)
    RMSpropTF(p, lr=0.0, alpha=0.0, eps=0.0, weight_decay=0.0, momentum=0.0)


def test_state_layout_and_int_step():
    p = [torch.nn.Parameter(torch.ones(3)), torch.nn.Parameter(torch.ones(2)), torch.nn.Parameter(torch.ones(2))]

    def make(ps):
        return RMSpropTF([dict(params=ps[:1], momentum=0.9), dict(params=ps[1:], centered=True)], lr=0.1)

    opt = make(p)
    # square_avg starts at ones: one zero-gradient step moves it to alpha exactly and leaves the parameter alone
    p[0].grad, p[1].grad = torch.zeros(3), torch.zeros(2)
    opt.step()
    assert list(opt.state[p[0]]) == ["step", "square_avg", "momentum_buffer"]
    assert list(opt.state[p[1]]) == ["step", "square_avg", "grad_avg"]
    assert p[2] not in opt.state
    assert torch.equal(opt.state[p[0]]["square_avg"], torch.full((3,), 0.9))
    assert torch.equal(p[0].detach(), torch.ones(3))
    assert opt.state[p[0]]["step"].dtype == torch.float32 and opt.state[p[0]]["step"].dim() == 0
    sd = opt.state_dict()
    assert set(sd["state"]) == {0, 1}
    assert set(sd["param_groups"][0]) == {"lr", "alpha", "eps", "weight_decay", "momentum", "centered",
                                          "decoupled_decay", "lr_in_momentum", "params"}
    # timm keeps step as a python int: loading converts it, and the run continues the same
    sd_int = copy.deepcopy(dict(sd, state={i: dict(e, step=int(e["step"])) for i, e in sd["state"].items()}))
    q = [torch.nn.Parameter(x.detach().clone()) for x in p]
    opt2 = make(q)
    opt2.load_state_dict(sd_int)
    assert opt2.state[q[0]]["step"].dtype == torch.float32 and float(opt2.state[q[0]]["step"]) == 1.0
    for x, y in zip(p, q):
        x.grad = torch.full_like(x, 0.5)
        y.grad = torch.full_like(y, 0.5)
    opt.step()
    opt2.step()
    for x, y in zip(p, q):
        assert torch.equal(x.detach(), y.detach())


def test_constants_struct_routing_and_state_layout():
    from stoke_b200.optim import _EXT_KINDS, _KINDS, _STATE_LAYOUT, fused_supported

    assert _lib.OPT_RMSPROP_TF == 13
    with open(os.path.join(ROOT, "include", "stoke_b200.h")) as f:
        header = f.read()
    assert "STK_OPT_RMSPROP_TF = 13" in header and "int stk_rmsprop_tf_step(" in header
    assert sb.RMSpropTF is RMSpropTF and "RMSpropTF" in sb.__all__
    assert _KINDS[RMSpropTF] == _lib.OPT_RMSPROP_TF
    lay = _STATE_LAYOUT[_lib.OPT_RMSPROP_TF]
    assert [(t.key, t.buf, t.init) for t in lay.tensors] == \
        [("square_avg", "V", 1.0), ("momentum_buffer", "M", 0.0), ("grad_avg", "M2", 0.0)]
    assert lay.unstepped == "omit" and _lib.OPT_RMSPROP_TF not in _EXT_KINDS
    assert lay.scalars == ()
    # stk_rmsprop_tf_hyper_t: one double, three int32 (and 4 bytes of tail padding)
    assert C.sizeof(_lib.RmspropTfHyper) == 24
    assert [(n, getattr(_lib.RmspropTfHyper, n).offset) for n, _ in _lib.RmspropTfHyper._fields_] == \
        [("alpha", 0), ("centered", 8), ("decoupled_decay", 12), ("lr_in_momentum", 16)]
    net = torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(9)])
    ps = list(net.parameters())
    assert fused_supported(RMSpropTF, {"lr": 1e-2, "momentum": 0.9}, net)
    eight = [{"params": [q]} for q in ps[:8]]
    eight[7]["params"].append(ps[8])
    assert fused_supported(RMSpropTF, {"params": eight}, net)
    assert not fused_supported(RMSpropTF, {"params": [{"params": [q]} for q in ps]}, net)


def test_load_step_counts_for_rmsprop_tf_state():
    from stoke_b200.optim import load_step_counts

    kind = _lib.OPT_RMSPROP_TF
    e3 = {"step": torch.tensor(3.0), "square_avg": torch.ones(2)}
    e3_int = dict(e3, step=3)
    assert load_step_counts(kind, [e3, {}, e3_int], [0, 0, 1], None, False) == (3, [3, 0, 3], None)
    assert load_step_counts(kind, [e3_int, e3], [0, 1], None, False) == (3, None, None)
    assert load_step_counts(kind, [e3_int, e3], [0, 1], 3, True) == (3, [3, 3], None)


def test_hypers_without_a_gpu():
    """What the fused optimizer hands stk_rmsprop_tf_step."""
    from stoke_b200.optim import _GROUP_HYPER, B200FusedOptimizer

    obj = B200FusedOptimizer.__new__(B200FusedOptimizer)
    obj._kind = _lib.OPT_RMSPROP_TF
    p = [torch.nn.Parameter(torch.zeros(1))]
    obj.param_groups = [dict(RMSpropTF(p, lr=0.3, alpha=0.95, eps=1e-3, weight_decay=1e-5, momentum=0.9).defaults),
                        dict(RMSpropTF(p, centered=True, decoupled_decay=True, lr_in_momentum=False).defaults)]
    h = obj._hyper_of(obj.param_groups[0])
    assert (h.kind, h.lr, h.eps, h.weight_decay, h.momentum, h.maximize) == (13, 0.3, 1e-3, 1e-5, 0.9, 0)
    assert obj._hyper_of(obj.param_groups[1]).momentum == 0.0
    x, y = (_GROUP_HYPER[_lib.OPT_RMSPROP_TF](g) for g in obj.param_groups)
    assert (x.alpha, x.centered, x.decoupled_decay, x.lr_in_momentum) == (0.95, 0, 0, 1)
    assert (y.alpha, y.centered, y.decoupled_decay, y.lr_in_momentum) == (0.9, 1, 1, 0)
