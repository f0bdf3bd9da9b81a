"""CPU tests of stoke_b200.Adan: the class against an independent float64 transcription of the paper's Algorithm 1 with
bias correction, argument validation, the group-held step count, the state-dict layout, and the pieces the fused step
relies on (constants, routing, the ABI structs, buffers, step counts)."""
import ctypes as C
import os

import pytest
import torch

import stoke_b200 as sb
from stoke_b200 import _lib, layout
from stoke_b200.optim import Adan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Paper64:
    """Xie et al.'s Algorithm 1 in float64, in the paper's convention (its beta_i is 1 - the code's), with the bias
    corrections 1 - (1 - beta_i)^t of the group's step count t.  Written from the paper, not from the class: the
    previous gradient is kept as such, and a parameter's first difference is 0."""

    def __init__(self, params, groups):
        self.p = [p.detach().double().clone() for p in params]
        self.groups = groups
        self.t = 0
        self.m = [torch.zeros_like(x) for x in self.p]
        self.v = [torch.zeros_like(x) for x in self.p]
        self.n = [torch.zeros_like(x) for x in self.p]
        self.prev = [None] * len(self.p)

    def step(self, grads, group_of):
        self.t += 1
        for i, g in enumerate(grads):
            if g is None:
                continue
            h = self.groups[group_of[i]]
            c1, c2, c3 = h["betas"]
            b1, b2, b3 = 1 - c1, 1 - c2, 1 - c3   # the paper's betas
            eta, eps, lam = h["lr"], h["eps"], h["weight_decay"]
            g = g.double()
            diff = torch.zeros_like(g) if self.prev[i] is None else g - self.prev[i]
            self.m[i] = (1 - b1) * self.m[i] + b1 * g
            self.v[i] = (1 - b2) * self.v[i] + b2 * diff
            self.n[i] = (1 - b3) * self.n[i] + b3 * (g + (1 - b2) * diff) ** 2
            bc1, bc2, bc3 = (1 - c ** self.t for c in (c1, c2, c3))
            eta_k = eta / (torch.sqrt(self.n[i] / bc3) + eps)
            upd = eta_k * (self.m[i] / bc1 + (1 - b2) * self.v[i] / bc2)
            if h["no_prox"]:
                self.p[i] = self.p[i] * (1 - lam * eta) - upd
            else:
                self.p[i] = (self.p[i] - upd) / (1 + lam * eta)
            self.prev[i] = g


def _group(**kw):
    return dict(dict(lr=1e-2, betas=(0.98, 0.92, 0.99), eps=1e-8, weight_decay=0.0, no_prox=False), **kw)


GROUPS = [_group(weight_decay=0.02),
          _group(lr=3e-3, betas=(0.9, 0.9, 0.999), eps=1e-6, weight_decay=0.05, no_prox=True),
          _group(lr=5e-3, no_prox=True),
          _group(lr=2e-2, betas=(0.95, 0.8, 0.98))]
SHAPES = ((7, 5), (11,), (3, 2, 2), (4,), (6,), (2, 3))
GROUP_OF = [0, 0, 1, 2, 3, 3]


def _grads(step, gen, params):
    """Parameter 1 gets its first gradient at t = 3; parameter 4 none at t = 5 and 6 (its next difference is against
    t = 4's gradient)."""
    out = []
    for i, p in enumerate(params):
        if (i == 1 and step < 2) or (i == 4 and step in (4, 5)):
            out.append(None)
        else:
            out.append(torch.randn(p.shape, generator=gen, dtype=p.dtype))
    return out


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_class_follows_the_paper(dtype):
    """The class's in-place op order is the paper's Algorithm 1: to rounding in float64, to fp32 tolerance in fp32, over
    20 steps with no_prox both ways, with and without weight decay, and a parameter first stepped at t = 3."""
    gen = torch.Generator().manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(*s, generator=gen, dtype=dtype) * 0.5) for s in SHAPES]
    opt = Adan([dict(g, params=[p for p, gi in zip(params, GROUP_OF) if gi == j]) for j, g in enumerate(GROUPS)])
    ref = Paper64(params, GROUPS)
    tol = dict(rtol=1e-12, atol=1e-14) if dtype == torch.float64 else dict(rtol=1e-5, atol=1e-6)
    for step in range(20):
        grads = _grads(step, gen, params)
        for p, gr in zip(params, grads):
            p.grad = None if gr is None else gr.clone()
        opt.step()
        ref.step(grads, GROUP_OF)
        for i, p in enumerate(params):
            assert torch.allclose(p.detach().double(), ref.p[i], **tol), (step, i)
            if i == 1 and step < 2:
                assert p not in opt.state and torch.equal(p.detach().double(), ref.p[i])
        assert [g["step"] for g in opt.param_groups] == [step + 1] * 4
    for i, p in enumerate(params):
        st = opt.state[p]
        for key, want in (("exp_avg", ref.m[i]), ("exp_avg_diff", ref.v[i]), ("exp_avg_sq", ref.n[i])):
            assert torch.allclose(st[key].double(), want, **tol), (i, key)
        assert torch.equal(st["neg_pre_grad"].double(), -ref.prev[i])


def test_validation_and_defaults():
    p = [torch.nn.Parameter(torch.zeros(2))]
    for kw in ({"lr": -1.0}, {"eps": -1.0}, {"betas": (0.9, 0.9)}, {"betas": (0.9, 0.9, 0.9, 0.9)},
               {"betas": (1.0, 0.9, 0.9)}, {"betas": (0.9, -0.1, 0.9)}, {"betas": (0.9, 0.9, 1.5)}):
        with pytest.raises(ValueError):
            Adan(p, **kw)
    assert Adan(p).defaults == dict(lr=1e-3, betas=(0.98, 0.92, 0.99), eps=1e-8, weight_decay=0.0, no_prox=False,
                                    foreach=None)
    Adan(p, lr=0.0, betas=(0.0, 0.0, 0.0), eps=0.0, foreach=True)   # foreach is accepted and ignored


def test_group_step_and_state_keys():
    p = [torch.nn.Parameter(torch.ones(3)), torch.nn.Parameter(torch.ones(2)), torch.nn.Parameter(torch.ones(2))]
    opt = Adan([dict(params=p[:2]), dict(params=p[2:], no_prox=True)], lr=0.1, weight_decay=0.1)
    assert all("step" not in g for g in opt.param_groups)
    g0 = torch.tensor([0.5, -1.0, 0.0])
    p[0].grad = g0.clone()
    opt.step()
    # the count is in the group, a python int, advanced in every group (the second one had no gradient)
    assert [g["step"] for g in opt.param_groups] == [1, 1] and type(opt.param_groups[0]["step"]) is int
    st = opt.state[p[0]]
    assert list(st) == ["exp_avg", "exp_avg_sq", "exp_avg_diff", "neg_pre_grad"]
    assert torch.equal(st["neg_pre_grad"], -g0) and torch.equal(st["exp_avg_diff"], torch.zeros(3))
    assert p[1] not in opt.state and p[2] not in opt.state
    opt.step()   # no gradient anywhere: the count still advances, nothing else moves
    assert [g["step"] for g in opt.param_groups] == [2, 2] and torch.equal(opt.state[p[0]]["neg_pre_grad"], -g0)
    sd = opt.state_dict()
    assert set(sd["state"]) == {0} and sd["param_groups"][0]["step"] == 2
    assert set(sd["param_groups"][0]) == {"lr", "betas", "eps", "weight_decay", "no_prox", "foreach", "step", "params"}


def test_constants_structs_and_routing():
    from stoke_b200.optim import _EXT_KINDS, _KINDS, fused_supported

    assert _lib.OPT_ADAN == 14
    with open(os.path.join(ROOT, "include", "stoke_b200.h")) as f:
        header = f.read()
    assert "STK_OPT_ADAN = 14" in header
    for fn in ("int stk_adan_step(", "int stk_adan_step_prologue("):
        assert fn in header
    assert "stk_adan_step" in _lib._SIGNATURES and "stk_adan_step_prologue" in _lib._SIGNATURES
    assert sb.Adan is Adan and "Adan" in sb.__all__
    assert _KINDS[Adan] == _lib.OPT_ADAN and _lib.OPT_ADAN not in _EXT_KINDS
    # stk_adan_hyper_t: one double, one int32 (and 4 bytes of tail padding)
    assert C.sizeof(_lib.AdanHyper) == 16
    assert [(n, getattr(_lib.AdanHyper, n).offset) for n, _ in _lib.AdanHyper._fields_] == [("beta3", 0), ("no_prox", 8)]
    net = torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(9)])
    ps = list(net.parameters())
    assert fused_supported(Adan, {"lr": 1e-3, "no_prox": True}, net)
    eight = [{"params": [q]} for q in ps[:8]]
    eight[7]["params"].append(ps[8])
    assert fused_supported(Adan, {"params": eight}, net)
    assert not fused_supported(Adan, {"params": [{"params": [q]} for q in ps]}, net)


def test_state_layout_buffers_and_round_trip():
    """The layout row against the class's own state dict: import -> export gives back the class's entries (key order,
    values, no entry for a parameter that never had a gradient), and the four buffers are allocated at zero."""
    from stoke_b200.optim import (_STATE_LAYOUT, export_state, import_state, state_buffers, state_dict_index)

    lay = _STATE_LAYOUT[_lib.OPT_ADAN]
    assert [(t.key, t.buf, t.init, t.where) for t in lay.tensors] == [
        ("exp_avg", "M", 0.0, None), ("exp_avg_sq", "V", 0.0, None), ("exp_avg_diff", "M2", 0.0, None),
        ("neg_pre_grad", "M3", 0.0, None)]
    assert (lay.step, lay.scalars, lay.unstepped, lay.group_count) == (False, (), "omit", ("step", "exp_avg"))
    groups_cfg = [dict(params=None), dict(params=None, no_prox=True, weight_decay=0.1)]
    assert state_buffers(lay, groups_cfg) == {"M": 0.0, "V": 0.0, "M2": 0.0, "M3": 0.0}
    # the other kinds keep their three buffers
    assert set(state_buffers(_STATE_LAYOUT[_lib.OPT_ADEMAMIX], [{"betas": (0.9, 0.9, 0.9)}])) == {"M", "V", "M2"}

    gen = torch.Generator().manual_seed(3)
    params = [torch.nn.Parameter(torch.randn(*s, generator=gen)) for s in ((3, 4), (5,), (2, 2), (7,))]
    group_of = [0, 1, 0, 1]
    opt = Adan([dict(params=[params[0], params[2]]), dict(params=[params[1], params[3]], no_prox=True,
                                                         weight_decay=0.1)], lr=1e-2)
    for _ in range(2):
        for i, p in enumerate(params):
            p.grad = None if i == 2 else torch.randn(p.shape, generator=gen)
        opt.step()
    sd = opt.state_dict()
    sd_index = state_dict_index(group_of, 2)
    entries = [sd["state"].get(sd_index[i], {}) for i in range(len(params))]
    offsets, _, n = layout.param_offsets([p.numel() for p in params])
    full = {b: torch.zeros(n) for b in ("M", "V", "M2", "M3")}
    views = {t.key: [full[t.buf][o: o + p.numel()].view(p.shape) for p, o in zip(params, offsets)] for t in lay.tensors}
    import_state(lay, entries, views)
    steps = [0 if i == 2 else 2 for i in range(len(params))]
    got = export_state(lay, sd["param_groups"], group_of, sd_index, steps, None, views)
    assert set(got) == set(sd["state"]) and sd_index[2] not in got
    for j, e in sd["state"].items():
        assert list(got[j]) == list(e)
        for k in e:
            assert torch.equal(got[j][k], e[k]), (j, k)


def test_load_step_counts_from_the_groups():
    from stoke_b200.optim import load_step_counts

    kind = _lib.OPT_ADAN
    e = {"exp_avg": torch.zeros(2), "exp_avg_sq": torch.zeros(2), "exp_avg_diff": torch.zeros(2),
         "neg_pre_grad": torch.zeros(2)}
    # no b200_opt_steps: the count from the groups; an entry without exp_avg has taken 0 steps
    assert load_step_counts(kind, [e, {}, e], [0, 0, 1], None, False, group_k=[5, 5]) == (5, [5, 0, 5], None)
    assert load_step_counts(kind, [e, e], [0, 1], None, False, group_k=[5, 5]) == (5, None, None)
    assert load_step_counts(kind, [e, e], [0, 1], 7, False, group_k=[5, 5]) == (7, None, None)
    assert load_step_counts(kind, [e, e], [0, 1], 7, True, group_k=[7, 7]) == (7, [7, 7], None)
    assert load_step_counts(kind, [{}, {}], [0, 1], None, False, group_k=[0, 0]) == (0, None, None)
    with pytest.raises(ValueError):
        load_step_counts(kind, [e, e], [0, 1], None, False, group_k=[4, 5])


def test_hypers_without_a_gpu():
    """What the fused optimizer hands stk_adan_step_prologue and stk_adan_step."""
    from stoke_b200.optim import _GROUP_HYPER, B200FusedOptimizer

    obj = B200FusedOptimizer.__new__(B200FusedOptimizer)
    obj._kind = _lib.OPT_ADAN
    p = [torch.nn.Parameter(torch.zeros(1))]
    obj.param_groups = [dict(Adan(p, lr=0.3, betas=(0.9, 0.8, 0.7), eps=1e-6, weight_decay=0.02).defaults),
                        dict(Adan(p, no_prox=True).defaults)]
    h = obj._hyper_of(obj.param_groups[0])
    assert (h.kind, h.lr, h.beta1, h.beta2, h.eps, h.weight_decay, h.maximize) == (14, 0.3, 0.9, 0.8, 1e-6, 0.02, 0)
    x, y = (_GROUP_HYPER[_lib.OPT_ADAN](g) for g in obj.param_groups)
    assert (x.beta3, x.no_prox) == (0.7, 0) and (y.beta3, y.no_prox) == (0.99, 1)
