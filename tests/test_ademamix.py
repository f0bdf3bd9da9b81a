"""CPU tests of stoke_b200.AdEMAMix: the class against an independent float64 transcription of the AdEMAMix formulas,
the alpha and beta3 warm-up schedules at their ends, argument validation, the state-dict layout, and the pieces the
fused step relies on (constants, routing, the ABI structs, step counts)."""
import copy
import ctypes as C
import math
import os

import pytest
import torch

import stoke_b200 as sb
from stoke_b200 import _lib
from stoke_b200.optim import AdEMAMix, ademamix_schedule

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _f(b):
    return math.log(0.5) / math.log(b + 1e-8) - 1


def _f_inv(x):
    return 0.5 ** (1 / (x + 1))


def _schedule64(h, t):
    """(alpha_t, beta3_t) written from the paper's schedulers (not from the class)."""
    b1, _, b3 = h["betas"]
    aw, bw = h.get("alpha_warmup"), h.get("beta3_warmup")
    alpha_t = h["alpha"] * t / aw if aw is not None and t < aw else h["alpha"]
    if bw is not None and t < bw:
        a = t / bw
        beta3_t = _f_inv((1 - a) * _f(b1) + a * _f(b3))
    else:
        beta3_t = b3
    return alpha_t, beta3_t


class Ref64:
    """The AdEMAMix update in float64, one step count per parameter."""

    def __init__(self, params, groups):
        self.p = [p.detach().double().clone() for p in params]
        self.groups = groups
        self.t = [0] * len(params)
        self.m1 = [torch.zeros_like(x) for x in self.p]
        self.m2 = [torch.zeros_like(x) for x in self.p]
        self.v = [torch.zeros_like(x) for x in self.p]

    def step(self, grads, group_of):
        for i, g in enumerate(grads):
            if g is None:
                continue
            h = self.groups[group_of[i]]
            b1, b2, _ = h["betas"]
            g = g.double()
            self.t[i] += 1
            t = self.t[i]
            alpha_t, beta3_t = _schedule64(h, t)
            self.m1[i] = b1 * self.m1[i] + (1 - b1) * g
            self.m2[i] = beta3_t * self.m2[i] + (1 - beta3_t) * g
            self.v[i] = b2 * self.v[i] + (1 - b2) * g * g
            bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
            u = (self.m1[i] / bc1 + alpha_t * self.m2[i]) / (torch.sqrt(self.v[i]) / math.sqrt(bc2) + h["eps"])
            u = u + h["weight_decay"] * self.p[i]
            self.p[i] = self.p[i] - h["lr"] * u


GROUPS = [dict(lr=1e-2, betas=(0.9, 0.999, 0.9999), alpha=4.0, alpha_warmup=20, beta3_warmup=35, eps=1e-8,
               weight_decay=0.05),
          dict(lr=5e-3, betas=(0.0, 0.99, 0.999), alpha=2.0, alpha_warmup=None, beta3_warmup=12, eps=1e-6,
               weight_decay=0.0)]


def test_class_follows_the_float64_formulas():
    """60 steps across both warm-ups, two groups (the second with beta1 == 0) and weight decay; parameter 1 gets no
    gradient on every third step, so its step count (and its schedules) fall behind the others'."""
    gen = torch.Generator().manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(*s, generator=gen) * 0.5) for s in ((7, 5), (11,), (3, 2, 2), (4,))]
    group_of = [0, 0, 1, 1]
    opt = AdEMAMix([dict(GROUPS[0], params=params[:2]), dict(GROUPS[1], params=params[2:])])
    ref = Ref64(params, GROUPS)
    for step in range(60):
        grads = [None if (i == 1 and step % 3 == 2) else torch.randn(p.shape, generator=gen) for i, p in enumerate(params)]
        for p, gr in zip(params, grads):
            p.grad = None if gr is None else gr.clone()
        opt.step()
        ref.step(grads, group_of)
        for i, p in enumerate(params):
            assert torch.allclose(p.detach().double(), ref.p[i], rtol=1e-5, atol=1e-6), (step, i)
    assert [int(opt.state[p]["step"]) for p in params] == ref.t == [60, 40, 60, 60]
    for i, p in enumerate(params):
        st = opt.state[p]
        assert torch.allclose(st["exp_avg_slow"].double(), ref.m2[i], rtol=1e-5, atol=1e-7)
        assert torch.allclose(st["exp_avg_sq"].double(), ref.v[i], rtol=1e-5, atol=1e-9)
        if group_of[i] == 0:
            assert torch.allclose(st["exp_avg_fast"].double(), ref.m1[i], rtol=1e-5, atol=1e-7)
        else:
            assert st["exp_avg_fast"] is None


@pytest.mark.parametrize("T", [2, 7, 100, 256_000])
def test_schedules_at_the_warmup_ends(T):
    h = dict(betas=(0.9, 0.999, 0.9999), alpha=8.0, alpha_warmup=T, beta3_warmup=T)
    a1, b1 = ademamix_schedule(h, 1.0)
    assert a1 == 8.0 / T and b1 == _schedule64(h, 1)[1]
    assert 0.9 < b1 < 0.9999 or T == 2
    aT1, bT1 = ademamix_schedule(h, float(T - 1))
    assert aT1 == pytest.approx(8.0 * (T - 1) / T, rel=1e-15) and aT1 < 8.0
    assert bT1 == _schedule64(h, T - 1)[1]   # just above beta3 for long warm-ups: f has the 1e-8, f_inv has not
    for t in (T, T + 1):
        assert ademamix_schedule(h, float(t)) == (8.0, 0.9999)
    # the half-life of beta3_t moves linearly from beta1's to beta3's (f's half-lives carry its 1e-8, f_inv's do not)
    a = (T - 1) / T
    assert math.log(0.5) / math.log(bT1) == pytest.approx((1 - a) * (_f(0.9) + 1) + a * (_f(0.9999) + 1), rel=1e-9)
    # no warm-up: alpha and beta3 from the first step
    assert ademamix_schedule(dict(h, alpha_warmup=None, beta3_warmup=None), 1.0) == (8.0, 0.9999)


def test_validation():
    p = [torch.nn.Parameter(torch.zeros(2))]
    for kw in ({"lr": -1.0}, {"eps": -1.0}, {"weight_decay": -0.1}, {"alpha": -1.0}, {"betas": (1.0, 0.999, 0.9999)},
               {"betas": (0.9, 1.0, 0.9999)}, {"betas": (0.9, 0.999, 1.0)}, {"betas": (-0.1, 0.999, 0.9999)},
               {"betas": (0.9, 0.999)}, {"beta3_warmup": 0}, {"beta3_warmup": -5}, {"alpha_warmup": 2.5},
               {"alpha_warmup": 0}, {"alpha_warmup": True}):
        with pytest.raises(ValueError):
            AdEMAMix(p, **kw)
    d = AdEMAMix(p).defaults
    assert (d["lr"], d["betas"], d["alpha"], d["beta3_warmup"], d["alpha_warmup"], d["eps"], d["weight_decay"]) == \
        (1e-3, (0.9, 0.999, 0.9999), 2.0, None, None, 1e-8, 0)
    AdEMAMix(p, betas=(0.0, 0.0, 0.0), alpha=0.0, alpha_warmup=1, beta3_warmup=1, weight_decay=0.0)


def test_state_layout_and_int_step():
    p = [torch.nn.Parameter(torch.ones(3)), torch.nn.Parameter(torch.ones(2)), torch.nn.Parameter(torch.ones(2))]
    opt = AdEMAMix([dict(params=p[:1]), dict(params=p[1:], betas=(0.0, 0.9, 0.99))], alpha_warmup=5)
    p[0].grad, p[1].grad = torch.ones(3), torch.ones(2)
    opt.step()
    assert list(opt.state[p[0]]) == ["step", "exp_avg_fast", "exp_avg_slow", "exp_avg_sq"]
    assert opt.state[p[0]]["step"].dtype == torch.float32 and opt.state[p[0]]["step"].dim() == 0
    assert opt.state[p[1]]["exp_avg_fast"] is None and p[2] not in opt.state
    sd = opt.state_dict()
    assert set(sd["state"]) == {0, 1}
    assert set(sd["param_groups"][0]) == {"lr", "betas", "alpha", "beta3_warmup", "alpha_warmup", "eps",
                                          "weight_decay", "params"}
    # upstream keeps step as a python int: loading converts it, and the run continues the same
    sd_int = copy.deepcopy(dict(sd, state={i: dict(e, step=int(e["step"])) for i, e in sd["state"].items()}))
    q = [torch.nn.Parameter(x.detach().clone()) for x in p]
    opt2 = AdEMAMix([dict(params=q[:1]), dict(params=q[1:], betas=(0.0, 0.9, 0.99))], alpha_warmup=5)
    opt2.load_state_dict(sd_int)
    assert opt2.state[q[0]]["step"].dtype == torch.float32 and float(opt2.state[q[0]]["step"]) == 1.0
    for x, y in zip(p, q):
        x.grad = torch.full_like(x, 0.5)
        y.grad = torch.full_like(y, 0.5)
    opt.step()
    opt2.step()
    for x, y in zip(p, q):
        assert torch.equal(x.detach(), y.detach())


def test_constants_structs_routing_and_state_layout():
    from stoke_b200.optim import _EXT_KINDS, _KINDS, _STATE_LAYOUT, fused_supported

    assert _lib.OPT_ADEMAMIX == 12
    with open(os.path.join(ROOT, "include", "stoke_b200.h")) as f:
        header = f.read()
    assert "STK_OPT_ADEMAMIX = 12" in header
    assert sb.AdEMAMix is AdEMAMix and "AdEMAMix" in sb.__all__
    assert _KINDS[AdEMAMix] == _lib.OPT_ADEMAMIX
    lay = _STATE_LAYOUT[_lib.OPT_ADEMAMIX]
    assert [(t.key, t.buf) for t in lay.tensors] == [("exp_avg_fast", "M"), ("exp_avg_slow", "M2"), ("exp_avg_sq", "V")]
    assert lay.tensors[0].none and not lay.tensors[0].where({"betas": (0.0, 0.9, 0.99)})   # None where beta1 == 0
    assert lay.unstepped == "omit" and _lib.OPT_ADEMAMIX not in _EXT_KINDS
    assert lay.scalars == ()
    # stk_ademamix_hyper_t: two doubles, two int64
    assert C.sizeof(_lib.AdemamixHyper) == 32
    assert [(n, getattr(_lib.AdemamixHyper, n).offset) for n, _ in _lib.AdemamixHyper._fields_] == \
        [("alpha", 0), ("beta3", 8), ("alpha_warmup", 16), ("beta3_warmup", 24)]
    # stk_optim_args_t: exp_avg_slow appended, every earlier field where it was
    names = [n for n, _ in _lib.OptimArgs._fields_]
    assert names[-2:] == ["group_bc", "exp_avg_slow"]
    assert _lib.OptimArgs.exp_avg_slow.offset == _lib.OptimArgs.group_bc.offset + 8
    assert C.sizeof(_lib.OptimArgs) == _lib.OptimArgs.exp_avg_slow.offset + 8
    net = torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(9)])
    ps = list(net.parameters())
    assert fused_supported(AdEMAMix, {"lr": 1e-3}, net)
    eight = [{"params": [q]} for q in ps[:8]]
    eight[7]["params"].append(ps[8])
    assert fused_supported(AdEMAMix, {"params": eight}, net)
    assert not fused_supported(AdEMAMix, {"params": [{"params": [q]} for q in ps]}, net)
    assert not fused_supported(AdEMAMix, {"lr": 1e-3, "differentiable": True}, net)


def test_load_step_counts_for_ademamix_state():
    from stoke_b200.optim import load_step_counts

    kind = _lib.OPT_ADEMAMIX
    e3 = {"step": torch.tensor(3.0), "exp_avg_fast": None, "exp_avg_slow": torch.zeros(2), "exp_avg_sq": torch.zeros(2)}
    e3_int = dict(e3, step=3)
    # a missing entry: that parameter has taken no step, so counts go per parameter
    assert load_step_counts(kind, [e3, {}, e3_int], [0, 0, 1], None, False) == (3, [3, 0, 3], None)
    assert load_step_counts(kind, [e3_int, e3], [0, 1], None, False) == (3, None, None)
    assert load_step_counts(kind, [e3_int, e3], [0, 1], 3, True) == (3, [3, 3], None)


def test_hypers_without_a_gpu():
    """What the fused optimizer hands stk_optim_step_ex and stk_ademamix_step_prologue."""
    from stoke_b200.optim import _GROUP_HYPER, B200FusedOptimizer

    obj = B200FusedOptimizer.__new__(B200FusedOptimizer)
    obj._kind = _lib.OPT_ADEMAMIX
    p = [torch.nn.Parameter(torch.zeros(1))]
    obj.param_groups = [dict(AdEMAMix(p, lr=0.3, betas=(0.8, 0.95, 0.999), alpha=6.0, alpha_warmup=7, eps=1e-6,
                                      weight_decay=0.1).defaults),
                        dict(AdEMAMix(p, betas=(0.0, 0.9, 0.99), beta3_warmup=11).defaults)]
    h = obj._hyper_of(obj.param_groups[0])
    assert (h.kind, h.lr, h.beta1, h.beta2, h.eps, h.weight_decay) == (12, 0.3, 0.8, 0.95, 1e-6, 0.1)
    x, y = (_GROUP_HYPER[_lib.OPT_ADEMAMIX](g) for g in obj.param_groups)
    assert (x.alpha, x.beta3, x.alpha_warmup, x.beta3_warmup) == (6.0, 0.999, 7, 0)
    assert (y.alpha, y.beta3, y.alpha_warmup, y.beta3_warmup) == (2.0, 0.99, 0, 11)
    assert obj._hyper_of(obj.param_groups[1]).beta1 == 0.0
