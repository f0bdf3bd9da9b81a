"""CPU tests of stoke_b200.AdamWScheduleFree and SGDScheduleFree: the classes against an independent float64
transcription of the schedule-free formulas, the train() / eval() swap, the refused step in eval mode, a state dict in
the upstream key layout, and the pieces the fused step relies on (constants, routing, the ABI struct, step counts)."""
import ctypes as C
import math
import os

import pytest
import torch

import stoke_b200 as sb
from stoke_b200 import _lib
from stoke_b200.optim import AdamWScheduleFree, SGDScheduleFree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Ref64:
    """The schedule-free update in float64, written from the formulas (not from the classes)."""

    def __init__(self, params, kind, **h):
        self.kind, self.h = kind, h
        self.y = [p.detach().double().clone() for p in params]
        self.z, self.v = [None] * len(params), [None] * len(params)
        self.k, self.lr_max, self.weight_sum = 0, -1.0, 0.0

    def step(self, grads, lr):
        h, k = self.h, self.k
        beta1 = h["betas"][0] if self.kind == "adamw" else h["momentum"]
        warm = h.get("warmup_steps", 0)
        sched = (k + 1) / warm if k < warm else 1.0
        lr_t = lr * sched
        self.lr_max = max(self.lr_max, lr_t)
        weight = (k + 1) ** h.get("r", 0.0) * self.lr_max ** h.get("weight_lr_power", 2.0)
        self.weight_sum += weight
        c = weight / self.weight_sum if self.weight_sum != 0 else 0.0
        for i, g in enumerate(grads):
            if g is None:
                continue
            g = g.double()
            if self.z[i] is None:
                self.z[i] = self.y[i].clone()
                self.v[i] = torch.zeros_like(self.y[i])
            if self.kind == "adamw":
                b2 = h["betas"][1]
                self.v[i] = b2 * self.v[i] + (1 - b2) * g * g
                d = g / (torch.sqrt(self.v[i] / (1 - b2 ** (k + 1))) + h.get("eps", 1e-8))
            else:
                d = g
            d = d + h.get("weight_decay", 0.0) * self.y[i]
            y = (1 - c) * self.y[i] + c * self.z[i]
            self.y[i] = y + lr_t * (beta1 * (1 - c) - 1) * d
            self.z[i] = self.z[i] - lr_t * d
        self.k += 1


def _params(seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(*s, generator=g) * 0.5) for s in ((7, 5), (11,), (3, 2, 2))]


RUNS = {
    "adamw_warmup_wd": ("adamw", {"lr": 0.02, "betas": (0.9, 0.999), "weight_decay": 0.05, "warmup_steps": 6}),
    "adamw_r_power": ("adamw", {"lr": 0.01, "betas": (0.8, 0.99), "eps": 1e-6, "r": 0.5, "weight_lr_power": 1.0}),
    "sgd_warmup_wd": ("sgd", {"lr": 0.2, "momentum": 0.9, "weight_decay": 0.01, "warmup_steps": 4}),
    "sgd_r": ("sgd", {"lr": 0.1, "momentum": 0.75, "r": 1.0}),
}


@pytest.mark.parametrize("name", list(RUNS))
def test_classes_follow_the_float64_formulas(name):
    """20 steps with a learning rate changed at step 8, a parameter that gets its first gradient at step 5 and
    steps with lr = 0 at the start (ckp1 = 0 while the weight sum is 0)."""
    kind, kw = RUNS[name]
    params = _params()
    cls = AdamWScheduleFree if kind == "adamw" else SGDScheduleFree
    opt = cls(params, **kw)
    ref = Ref64(params, kind, **kw)
    opt.train()
    for p, y in zip(params, ref.y):   # train() from a fresh optimizer moves nothing: no parameter has z yet
        assert torch.equal(p.detach().double(), y)
    gen = torch.Generator().manual_seed(1)
    for step in range(20):
        lr = 0.0 if step < 2 else (kw["lr"] if step < 8 else kw["lr"] * 0.5)
        for g in opt.param_groups:
            g["lr"] = lr
        grads = [None if (i == 1 and step < 5) else torch.randn(p.shape, generator=gen) for i, p in enumerate(params)]
        for p, gr in zip(params, grads):
            p.grad = None if gr is None else gr.clone()
        opt.step()
        ref.step(grads, lr)
        for p, gr in zip(params, grads):   # step() leaves the gradient as it was
            assert (p.grad is None) == (gr is None) and (gr is None or torch.equal(p.grad, gr))
        if step < 2:
            assert opt.param_groups[0]["weight_sum"] == 0.0
        for p, y in zip(params, ref.y):
            assert torch.allclose(p.detach().double(), y, rtol=1e-5, atol=1e-6), (step, (p.detach().double() - y).abs().max())
    assert params[1] in opt.state and opt.param_groups[0]["k"] == 20
    g = opt.param_groups[0]
    assert g["lr_max"] == ref.lr_max and math.isclose(g["weight_sum"], ref.weight_sum, rel_tol=1e-12)
    assert g["scheduled_lr"] == kw["lr"] * 0.5


@pytest.mark.parametrize("cls,kw,beta1", [(AdamWScheduleFree, {"betas": (0.9, 0.999)}, 0.9),
                                          (SGDScheduleFree, {"momentum": 0.8}, 0.8)])
def test_eval_train_lerps_and_refused_step(cls, kw, beta1):
    params = _params()
    opt = cls(params, lr=0.05, **kw)
    with pytest.raises(RuntimeError):   # a new optimizer is in eval mode
        opt.step()
    opt.train()
    for p in params:
        p.grad = torch.ones_like(p)
    opt.step()
    opt.step()
    y = [p.detach().clone() for p in params]
    z = [opt.state[p]["z"].clone() for p in params]
    opt.eval()
    assert not opt.param_groups[0]["train_mode"]
    for p, a, b in zip(params, y, z):
        assert torch.equal(p.detach(), torch.lerp(a, b, 1 - 1 / beta1))
    x = [p.detach().clone() for p in params]
    state = {p: {k: v.clone() for k, v in opt.state[p].items()} for p in params}
    groups = [dict(g) for g in opt.param_groups]
    opt.eval()   # already in eval mode: nothing moves
    with pytest.raises(RuntimeError):
        opt.step()
    for p, a in zip(params, x):
        assert torch.equal(p.detach(), a)
        for k, v in state[p].items():
            assert torch.equal(opt.state[p][k], v)
    assert [dict(g) for g in opt.param_groups] == groups
    opt.train()
    for p, a, b in zip(params, x, z):
        assert torch.equal(p.detach(), torch.lerp(a, b, 1 - beta1))


def test_upstream_layout_state_dict_loads_and_continues():
    """A state dict written by hand in facebookresearch/schedule_free's layout (z / exp_avg_sq, no step; k, lr_max,
    weight_sum, train_mode ... in the groups) loads into the class and continues exactly like the optimizer it
    describes."""
    params = _params()
    opt = AdamWScheduleFree(params, lr=0.01, warmup_steps=3, weight_decay=0.01)
    opt.train()
    gen = torch.Generator().manual_seed(2)
    for _ in range(4):
        for p in params:
            p.grad = torch.randn(p.shape, generator=gen)
        opt.step()
    g = opt.param_groups[0]
    hand = {"state": {i: {"z": opt.state[p]["z"].clone(), "exp_avg_sq": opt.state[p]["exp_avg_sq"].clone()}
                      for i, p in enumerate(params)},
            "param_groups": [{"lr": 0.01, "betas": (0.9, 0.999), "eps": 1e-8, "r": 0.0, "k": g["k"], "warmup_steps": 3,
                              "train_mode": True, "weight_sum": g["weight_sum"], "lr_max": g["lr_max"],
                              "scheduled_lr": g["scheduled_lr"], "weight_lr_power": 2.0, "weight_decay": 0.01,
                              "foreach": True, "params": [0, 1, 2]}]}
    assert set(opt.state_dict()["param_groups"][0]) == set(hand["param_groups"][0])
    params2 = [torch.nn.Parameter(p.detach().clone()) for p in params]
    opt2 = AdamWScheduleFree(params2)
    opt2.load_state_dict(hand)
    for _ in range(3):
        for p, q in zip(params, params2):
            p.grad = torch.randn(p.shape, generator=gen)
            q.grad = p.grad.clone()
        opt.step()
        opt2.step()
    opt.eval()
    opt2.eval()
    for p, q in zip(params, params2):
        assert torch.equal(p.detach(), q.detach())


def test_validation():
    p = [torch.nn.Parameter(torch.zeros(2))]
    for kw in ({"lr": -1.0}, {"betas": (0.0, 0.9)}, {"betas": (0.9, 1.0)}, {"eps": -1.0}, {"weight_decay": -0.1},
               {"warmup_steps": -1}):
        with pytest.raises(ValueError):
            AdamWScheduleFree(p, **kw)
    for kw in ({"lr": -1.0}, {"momentum": 0.0}, {"momentum": 1.0}, {"weight_decay": -0.1}, {"warmup_steps": -1}):
        with pytest.raises(ValueError):
            SGDScheduleFree(p, **kw)
    d = AdamWScheduleFree(p).defaults
    assert (d["lr"], d["betas"], d["eps"], d["weight_decay"], d["warmup_steps"], d["r"], d["weight_lr_power"]) == \
        (0.0025, (0.9, 0.999), 1e-8, 0.0, 0, 0.0, 2.0)
    assert (d["k"], d["train_mode"], d["weight_sum"], d["lr_max"], d["scheduled_lr"]) == (0, False, 0.0, -1.0, 0.0)
    d = SGDScheduleFree(p).defaults
    assert (d["lr"], d["momentum"], d["weight_decay"], d["warmup_steps"], d["r"], d["weight_lr_power"]) == \
        (1.0, 0.9, 0.0, 0, 0.0, 2.0)


def test_constants_struct_routing_and_state_layout():
    from stoke_b200.optim import _EXT_KINDS, _KINDS, _STATE_LAYOUT, fused_supported

    assert (_lib.OPT_SF_ADAMW, _lib.OPT_SF_SGD) == (10, 11)
    assert sb.AdamWScheduleFree is AdamWScheduleFree and sb.SGDScheduleFree is SGDScheduleFree
    assert "AdamWScheduleFree" in sb.__all__ and "SGDScheduleFree" in sb.__all__
    assert _KINDS[AdamWScheduleFree] == _lib.OPT_SF_ADAMW and _KINDS[SGDScheduleFree] == _lib.OPT_SF_SGD
    def tensors(k):
        return [(t.key, t.buf, t.init) for t in _STATE_LAYOUT[k].tensors]

    assert tensors(_lib.OPT_SF_ADAMW) == [("z", "M", "master"), ("exp_avg_sq", "V", 0.0)]
    assert tensors(_lib.OPT_SF_SGD) == [("z", "M", "master")]
    for k in (_lib.OPT_SF_ADAMW, _lib.OPT_SF_SGD):
        lay = _STATE_LAYOUT[k]
        assert lay.unstepped == "omit" and not lay.step and k not in _EXT_KINDS and lay.scalars == ()
    with open(os.path.join(ROOT, "include", "stoke_b200.h")) as f:
        header = f.read()
    assert "STK_OPT_SF_ADAMW = 10" in header and "STK_OPT_SF_SGD = 11" in header
    # stk_sf_hyper_t: five doubles and an int64
    assert C.sizeof(_lib.SfHyper) == 48
    assert [(n, getattr(_lib.SfHyper, n).offset) for n, _ in _lib.SfHyper._fields_] == \
        [("lr", 0), ("beta1", 8), ("beta2", 16), ("r", 24), ("weight_lr_power", 32), ("warmup_steps", 40)]
    net = torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(9)])
    ps = list(net.parameters())
    for cls in (AdamWScheduleFree, SGDScheduleFree):
        assert fused_supported(cls, {"lr": 1e-3}, net)
        eight = [{"params": [q]} for q in ps[:8]]
        eight[7]["params"].append(ps[8])
        assert fused_supported(cls, {"params": eight}, net)
        assert not fused_supported(cls, {"params": [{"params": [q]} for q in ps]}, net)


def test_load_step_counts_for_schedule_free_state():
    from stoke_b200.optim import load_step_counts

    z = {"z": torch.zeros(2)}
    kind = _lib.OPT_SF_SGD
    # no b200_opt_steps: k from the groups; an entry without z has taken 0 steps
    assert load_step_counts(kind, [z, {}, z], [0, 0, 1], None, False, group_k=[5, 5]) == (5, [5, 0, 5], None)
    assert load_step_counts(kind, [z, z], [0, 1], None, False, group_k=[5, 5]) == (5, None, None)
    assert load_step_counts(_lib.OPT_SF_ADAMW, [z, z], [0, 1], 7, False, group_k=[5, 5]) == (7, None, None)
    assert load_step_counts(kind, [z, z], [0, 1], 7, True, group_k=[7, 7]) == (7, [7, 7], None)
    with pytest.raises(ValueError):
        load_step_counts(kind, [z, z], [0, 1], None, False, group_k=[4, 5])


def test_sf_hypers_and_swap_guard_without_a_gpu():
    """What the fused optimizer hands stk_sf_step_prologue; train() / eval() on another kind is refused."""
    from stoke_b200.optim import _GROUP_HYPER, B200FusedOptimizer

    obj = B200FusedOptimizer.__new__(B200FusedOptimizer)
    obj._kind = _lib.OPT_SF_SGD
    obj.param_groups = [dict(SGDScheduleFree([torch.nn.Parameter(torch.zeros(1))], lr=0.3, momentum=0.8, r=0.5,
                                             warmup_steps=7, weight_decay=0.1).defaults)]
    x = _GROUP_HYPER[_lib.OPT_SF_SGD](obj.param_groups[0])
    assert (x.lr, x.beta1, x.beta2, x.r, x.weight_lr_power, x.warmup_steps) == (0.3, 0.8, 0.0, 0.5, 2.0, 7)
    h = obj._hyper_of(obj.param_groups[0])
    assert (h.kind, h.lr, h.weight_decay) == (11, 0.3, 0.1)
    with pytest.raises(RuntimeError):
        obj.check_train_mode()
    obj._kind = _lib.OPT_ADAM
    obj.check_train_mode()   # other kinds have no eval mode
    with pytest.raises(NotImplementedError):
        obj.eval()
