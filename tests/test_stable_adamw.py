"""CPU tests of stoke_b200.StableAdamW: the class against an independent float64 transcription of its formula, the RMS
clip, NaN propagation, argument validation, the float64 reference's bounds (they accept the class's fp32 step and reject
deliberately wrong references), and the pieces the fused step relies on (constants, routing, the hyper struct, the
state layout and step counts)."""
import math
import os

import numpy as np
import pytest
import torch

import stable_adamw_ref as sr
import stoke_b200 as sb
from stoke_b200 import _lib, layout
from stoke_b200.optim import StableAdamW

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Formula64:
    """Wortsman et al.'s Algorithm 2 with this package's debiased betas and RMS clip, in numpy float64, written from the
    formula (not the class): per parameter its own step count, lazily created moments."""

    def __init__(self, params, groups):
        self.p = [p.detach().double().numpy().copy() for p in params]
        self.groups = groups
        self.t = [0] * len(self.p)
        self.m = [np.zeros_like(x) for x in self.p]
        self.v = [np.zeros_like(x) for x in self.p]
        self.lr_t = [None] * len(self.p)

    def step(self, grads, group_of):
        for i, g in enumerate(grads):
            if g is None:
                continue
            h = self.groups[group_of[i]]
            beta1, beta2 = h["betas"]
            g = g.double().numpy()
            self.t[i] += 1
            t = self.t[i]
            b1 = beta1 * (1 - beta1 ** (t - 1)) / (1 - beta1 ** t)
            b2 = beta2 * (1 - beta2 ** (t - 1)) / (1 - beta2 ** t)
            self.m[i] = b1 * self.m[i] + (1 - b1) * g
            self.v[i] = b2 * self.v[i] + (1 - b2) * g * g
            rms = math.sqrt(float(np.mean(g * g / np.maximum(self.v[i], h["eps"] ** 2))))
            lr_t = h["lr"] / max(1.0, rms)
            self.lr_t[i] = lr_t
            self.p[i] = self.p[i] * (1 - lr_t * h["weight_decay"]) - lr_t * self.m[i] / (np.sqrt(self.v[i]) + h["eps"])


def _params(shapes, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(*s, generator=gen, dtype=torch.float64) * 0.1) for s in shapes]


def test_class_follows_the_formula():
    """Two groups (weight_decay 0 and != 0), per-parameter counts through a parameter without a gradient, steps whose RMS
    stays below 1 and steps where it exceeds 1."""
    shapes = [(5, 7), (13,), (3, 2, 2), (40,)]
    params = _params(shapes)
    groups = [dict(sr.DEFAULTS, lr=1e-2, weight_decay=0.1), dict(sr.DEFAULTS, lr=3e-3, betas=(0.8, 0.95), eps=1e-8,
                                                                weight_decay=0.0)]
    group_of = [0, 1, 0, 1]
    opt = StableAdamW([dict(params=[params[0], params[2]], lr=1e-2, weight_decay=0.1),
                       dict(params=[params[1], params[3]], lr=3e-3, betas=(0.8, 0.95), eps=1e-8, weight_decay=0.0)])
    ref = Formula64(params, groups)
    gen = torch.Generator().manual_seed(1)
    base = [torch.randn(*s, generator=gen, dtype=torch.float64) * 1e-2 for s in shapes]
    scales = [1.0, 0.5, 3.0, 0.1, 5.0, 1.0]
    for k, sc in enumerate(scales):
        grads = [None if (i == 3 and k in (1, 2)) else base[i] * sc + 1e-3 * k for i in range(len(params))]
        for p, g in zip(params, grads):
            p.grad = None if g is None else g.clone()
        opt.step()
        ref.step(grads, group_of)
        for i, p in enumerate(params):
            np.testing.assert_allclose(p.detach().numpy(), ref.p[i], rtol=1e-12, atol=1e-15)
            st = opt.state[p]
            assert float(st["step"]) == ref.t[i]
            np.testing.assert_allclose(st["exp_avg"].numpy(), ref.m[i], rtol=1e-12, atol=1e-18)
            np.testing.assert_allclose(st["exp_avg_sq"].numpy(), ref.v[i], rtol=1e-12, atol=1e-20)
    assert ref.t == [6, 6, 6, 4]
    assert list(opt.state[params[0]]) == ["step", "exp_avg", "exp_avg_sq"]
    assert opt.state[params[0]]["step"].dtype == torch.float32 and opt.state[params[0]]["step"].dim() == 0


def test_first_step_moments_and_lr():
    """At t = 1 both debiased betas are 0: m = g, v = g^2, every g^2 / v is 1 (or 0 where g = 0), so RMS <= 1 and
    lr_t = lr."""
    p = _params([(64,)])[0]
    w0 = p.detach().clone()
    g = torch.linspace(-1, 1, 64, dtype=torch.float64)
    g[10] = 0.0
    opt = StableAdamW([p], lr=0.1, weight_decay=0.2, eps=1e-8)
    p.grad = g.clone()
    opt.step()
    st = opt.state[p]
    assert torch.equal(st["exp_avg"], g) and torch.equal(st["exp_avg_sq"], g * g)
    assert sr.debiased(0.9, 1) == 0.0 and sr.debiased(0.99, 1) == 0.0
    lr_t = 0.1
    want = w0 * (1 - lr_t * 0.2) - lr_t * g / (g.abs() + 1e-8)
    torch.testing.assert_close(p.detach(), want, rtol=1e-14, atol=1e-15)


def test_rms_above_one_scales_lr_down():
    """A gradient three times the first meets a second moment that still remembers the first: RMS ~ 1.34, lr_t < lr."""
    p = _params([(1000,)])[0]
    gen = torch.Generator().manual_seed(5)
    g1 = torch.randn(1000, generator=gen, dtype=torch.float64) * 1e-2
    opt = StableAdamW([p], lr=1e-2, weight_decay=0.0)
    p.grad = g1.clone()
    opt.step()
    st = {k: opt.state[p][k].clone() for k in sr.KEYS}
    w1 = p.detach().clone()
    p.grad = 3 * g1
    opt.step()
    lr_t = sr.lr_t_of(st, 3 * g1, 1, dict(lr=1e-2, weight_decay=0.0))
    assert 1e-2 / 1.4 < lr_t < 1e-2 / 1.3
    m, v = opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"]
    torch.testing.assert_close(p.detach(), w1 - lr_t * m / (v.sqrt() + 1e-6), rtol=1e-13, atol=1e-16)
    # the unclipped update would have been lr / lr_t times larger
    full = (1e-2 * m / (v.sqrt() + 1e-6)).abs().sum()
    assert float((w1 - p.detach()).abs().sum()) < 0.8 * float(full)


@pytest.mark.parametrize("wd", [0.0, 0.1])
def test_nan_gradient_makes_its_parameter_nan(wd):
    a, b = _params([(8, 8), (17,)])
    opt = StableAdamW([a, b], lr=1e-2, weight_decay=wd)
    ga = torch.full((8, 8), 1e-3, dtype=torch.float64)
    ga[3, 4] = float("nan")
    a.grad, b.grad = ga, torch.full((17,), 1e-3, dtype=torch.float64)
    opt.step()
    assert bool(a.detach().isnan().all())
    assert bool(b.detach().isfinite().all())


def test_validation_and_defaults():
    p = [torch.nn.Parameter(torch.zeros(2))]
    assert StableAdamW(p).defaults == dict(lr=1e-3, betas=(0.9, 0.99), eps=1e-6, weight_decay=1e-2)
    for kw in (dict(lr=-1.0), dict(eps=-1e-8), dict(weight_decay=-0.1), dict(betas=(1.0, 0.9)), dict(betas=(0.9, 1.0)),
               dict(betas=(-0.1, 0.9)), dict(betas=(0.9, -0.5))):
        with pytest.raises(ValueError):
            StableAdamW(p, **kw)
    StableAdamW(p, lr=0.0, eps=0.0, weight_decay=0.0, betas=(0.0, 0.0))


# ---- the float64 reference's bounds -----------------------------------------------------------------------------------
BOUND_CASES = [((8193,), dict(lr=1e-2, weight_decay=0.1), [1.0, 0.5, 3.0]),
               ((64, 16, 3, 3), dict(lr=1e-3, weight_decay=0.0, eps=1e-8, betas=(0.8, 0.95)), [1.0, 3.0, 0.25]),
               ((37, 23), dict(lr=5e-2, weight_decay=0.3), [1.0, 5.0, 1.0])]


@pytest.mark.parametrize("shape,h,scales", BOUND_CASES)
def test_reference_bounds_accept_the_fp32_class(shape, h, scales):
    """The class's own fp32 step, restarted every step from its fp32 state, lies inside the bounds of the float64
    reference, RMS clip engaged or not."""
    gen = torch.Generator().manual_seed(7)
    w = torch.randn(*shape, generator=gen) * 0.1
    g0 = torch.randn(*shape, generator=gen) * 1e-3
    state = sr.zero_state(shape)
    clipped = 0
    for step, sc in enumerate(scales):
        G = g0 * sc
        w32, st32 = sr.step_ref(w, state, G, step, h, dtype=torch.float32)
        rw, rst = sr.step_ref(w, state, G, step, h)
        ew, est = sr.step_bound(w, state, G, step, h, rw, rst)
        assert not bool(sr.outside(w32, rw, ew).any()), step
        for k in sr.KEYS:
            assert not bool(sr.outside(st32[k], rst[k], est[k]).any()), (step, k)
        clipped += sr.lr_t_of(state, G, step, h) < sr.hyper(h)["lr"]
        w, state = w32, st32
    assert clipped >= 1


@pytest.mark.parametrize("mutation", sr.MUTATIONS)
def test_reference_bounds_reject_wrong_references(mutation):
    gen = torch.Generator().manual_seed(11)
    shape = (300,)
    h = dict(lr=1e-2, weight_decay=0.1)
    w = torch.randn(*shape, generator=gen) * 0.1
    g0 = torch.randn(*shape, generator=gen) * 1e-3
    state = sr.zero_state(shape)
    caught = False
    for step, sc in enumerate([1.0, 3.0, 0.5]):
        G = g0 * sc
        if mutation == "fmax_clamp" and step == 2:
            G = G.clone()
            G[17] = float("nan")
        rw, rst = sr.step_ref(w, state, G, step, h)
        ew, _ = sr.step_bound(w, state, G, step, h, rw, rst)
        caught |= bool(sr.outside(sr.step_mutant(w, state, G, step, h, mutation), rw, ew).any())
        # the correct transcription stays inside
        assert not bool(sr.outside(sr.step_mutant(w, state, G, step, h, "none"), rw, ew).any()), step
        w32, state = sr.step_ref(w, state, G, step, h, dtype=torch.float32)
        w = w32
    assert caught, mutation


# ---- what the fused step relies on --------------------------------------------------------------------------------------
def test_constants_routing_and_export():
    from stoke_b200.optim import _GROUP_HYPER, _KINDS, _LAYERWISE, fused_supported

    assert _lib.LW_STABLE_ADAMW == 2
    with open(os.path.join(ROOT, "include", "stoke_b200.h")) as f:
        assert "STK_LW_STABLE_ADAMW = 2" in f.read()
    assert sb.StableAdamW is StableAdamW and "StableAdamW" in sb.__all__
    kind = _KINDS[StableAdamW]
    assert _LAYERWISE[kind] == _lib.LW_STABLE_ADAMW
    h = _GROUP_HYPER[kind](dict(StableAdamW([torch.nn.Parameter(torch.zeros(1))], lr=0.3, betas=(0.8, 0.7), eps=1e-7,
                                            weight_decay=0.02).defaults))
    assert (h.lr, h.beta1, h.beta2, h.eps, h.weight_decay) == (0.3, 0.8, 0.7, 1e-7, 0.02)
    assert (h.momentum, h.dampening, h.trust_coefficient, h.bias_correction, h.nesterov, h.always_adapt) == (0, 0, 0, 0, 0, 0)
    net = torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(9)])
    ps = list(net.parameters())
    assert fused_supported(StableAdamW, {"lr": 1e-3}, net)
    eight = [{"params": [q]} for q in ps[:8]]
    eight[7]["params"].append(ps[8])
    assert fused_supported(StableAdamW, {"params": eight}, net)
    assert not fused_supported(StableAdamW, {"params": [{"params": [q]} for q in ps]}, net)


def test_state_layout_buffers_and_round_trip():
    from stoke_b200.optim import (_KINDS, _STATE_LAYOUT, export_state, import_state, state_buffers, state_dict_index)

    lay = _STATE_LAYOUT[_KINDS[StableAdamW]]
    assert [(t.key, t.buf, t.init, t.where) for t in lay.tensors] == [("exp_avg", "M", 0.0, None),
                                                                     ("exp_avg_sq", "V", 0.0, None)]
    assert (lay.step, lay.scalars, lay.unstepped, lay.group_count) == (True, (), "omit", None)
    assert state_buffers(lay, [{}, {"weight_decay": 0.0}]) == {"M": 0.0, "V": 0.0, "M2": None}

    gen = torch.Generator().manual_seed(3)
    params = [torch.nn.Parameter(torch.randn(*s, generator=gen)) for s in ((3, 4), (5,), (2, 2), (7,))]
    group_of = [0, 1, 0, 1]
    opt = StableAdamW([dict(params=[params[0], params[2]]), dict(params=[params[1], params[3]], weight_decay=0.0)])
    for k in range(3):
        for i, p in enumerate(params):
            p.grad = None if i == 2 or (i == 3 and k == 0) else torch.randn(p.shape, generator=gen)
        opt.step()
    sd = opt.state_dict()
    sd_index = state_dict_index(group_of, 2)
    entries = [sd["state"].get(sd_index[i], {}) for i in range(len(params))]
    offsets, _, n = layout.param_offsets([p.numel() for p in params])
    full = {b: torch.zeros(n) for b in ("M", "V")}
    views = {t.key: [full[t.buf][o: o + p.numel()].view(p.shape) for p, o in zip(params, offsets)] for t in lay.tensors}
    import_state(lay, entries, views)
    steps = [3, 3, 0, 2]
    got = export_state(lay, sd["param_groups"], group_of, sd_index, steps, None, views)
    assert set(got) == set(sd["state"]) and sd_index[2] not in got
    for j, e in sd["state"].items():
        assert list(got[j]) == list(e)
        for k in e:
            assert torch.equal(got[j][k], e[k]), (j, k)


def test_load_step_counts_per_parameter():
    from stoke_b200.optim import _KINDS, load_step_counts

    kind = _KINDS[StableAdamW]
    e = lambda t: {"step": torch.tensor(float(t)), "exp_avg": torch.zeros(2), "exp_avg_sq": torch.zeros(2)}  # noqa: E731
    assert load_step_counts(kind, [e(4), e(4)], [0, 1], None, False) == (4, None, None)
    assert load_step_counts(kind, [e(4), {}, e(2)], [0, 0, 1], None, False) == (4, [4, 0, 2], None)
    assert load_step_counts(kind, [e(4), e(4)], [0, 1], None, True) == (4, [4, 4], None)
