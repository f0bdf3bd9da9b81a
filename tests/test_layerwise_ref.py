"""CPU checks of the LAMB / LARS classes, the fused step's reference and bounds, routing and checkpoint state (no GPU).

fp32 runs of the classes' own step lie inside the per-element bounds of tests/layerwise_ref.py around float64 runs over
several steps; deliberately wrong references lie outside them somewhere; the edge cases of the trust ratio follow the
written formulas; fused_supported routes up to 8 groups to the fused step; state is created lazily in the classes' own
layout and load_step_counts reads it."""
import copy
import math
import zlib

import pytest
import torch

import layerwise_ref as lr_
from stoke_b200 import LAMB, LARS
from stoke_b200.optim import _LAMB, _LARS, fused_supported, load_step_counts

SHAPES = {"matrix": (37, 23), "conv3x3": (8, 6, 3, 3), "vector": (100,), "big": (3, 9000), "one": (1,)}
HYPERS = {
    "lamb": {
        "default": {"lr": 1e-2},
        "no_bc_adapt": {"lr": 1e-2, "bias_correction": False, "always_adapt": True, "weight_decay": 0.0},
        "wd0_plain": {"lr": 1e-2, "weight_decay": 0.0},
        "big_wd": {"lr": 5e-3, "weight_decay": 0.1, "betas": (0.8, 0.99), "eps": 1e-4},
    },
    "lars": {
        "default": {"lr": 0.5, "weight_decay": 1e-4},
        "nesterov": {"lr": 0.5, "weight_decay": 5e-4, "nesterov": True, "trust_coefficient": 0.02},
        "damp": {"lr": 1.0, "weight_decay": 1e-3, "dampening": 0.5, "trust_coefficient": 0.02},
        "no_momentum_adapt": {"lr": 0.1, "momentum": 0.0, "always_adapt": True},
        "wd0_plain": {"lr": 0.1},
    },
}
CASES = [(k, h, s) for k in HYPERS for h in HYPERS[k] for s in SHAPES]


def _grad(shape, gen):
    return torch.randn(shape, generator=gen) * 1e-2


@pytest.mark.parametrize("kind,hname,sname", CASES)
def test_fp32_class_inside_bounds(kind, hname, sname):
    shape, h = SHAPES[sname], HYPERS[kind][hname]
    gen = torch.Generator().manual_seed(zlib.crc32(f"{kind}{hname}{sname}".encode()))
    w = torch.randn(shape, generator=gen) * 0.1
    state = lr_.zero_state(kind, shape, h)
    for step in range(5):
        g = _grad(shape, gen)
        rw, rst = lr_.step_ref(kind, w, state, g, step, h)
        fw, fst = lr_.step_ref(kind, w, state, g, step, h, dtype=torch.float32)
        ew, est = lr_.step_bound(kind, w, state, g, step, h, rw, rst)
        assert not bool(lr_.outside(fw, rw, ew).any()), (kind, hname, sname, step)
        for k in rst:
            assert not bool(lr_.outside(fst[k], rst[k], est[k]).any()), (kind, hname, sname, step, k)
        # the bound says something: far below the update itself
        assert float(ew.max()) < 1e-2 * float((rw - w.double()).abs().max()) + 1e-9
        w, state = fw, {k: v.float() for k, v in fst.items()}


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_reference_written_out_agrees_with_class(kind):
    """step_mutant with no mutation is the written formula: it agrees with the class's float64 step."""
    for hname, h in HYPERS[kind].items():
        gen = torch.Generator().manual_seed(5)
        w = torch.randn(40, 7, generator=gen) * 0.1
        state = lr_.zero_state(kind, w.shape, h)
        for step in range(3):
            g = _grad(w.shape, gen)
            rw, rst = lr_.step_ref(kind, w, state, g, step, h)
            mw = lr_.step_mutant(kind, w, state, g, step, h, "none")
            assert torch.allclose(rw, mw, rtol=1e-12, atol=1e-15), (kind, hname, step)
            w, state = rw.float(), {k: v.float() for k, v in rst.items()}


@pytest.mark.parametrize("kind,mutation", [(k, m) for k in lr_.MUTATIONS for m in lr_.MUTATIONS[k]])
def test_mutations_fall_outside_bounds(kind, mutation):
    caught = False
    for hname, h in HYPERS[kind].items():
        gen = torch.Generator().manual_seed(zlib.crc32(f"{kind}{mutation}{hname}".encode()))
        w = torch.randn(37, 23, generator=gen) * 0.1
        state = lr_.zero_state(kind, w.shape, h)
        for step in range(3):
            g = _grad(w.shape, gen)
            rw, rst = lr_.step_ref(kind, w, state, g, step, h)
            ew, _ = lr_.step_bound(kind, w, state, g, step, h, rw, rst)
            if bool(lr_.outside(lr_.step_mutant(kind, w, state, g, step, h, mutation), rw, ew).any()):
                caught = True
            w, state = rw.float(), {k: v.float() for k, v in rst.items()}
    assert caught, (kind, mutation)


# ---- edge cases of the trust ratio ---------------------------------------------------------------------------------------
def _one_step(cls, w, g, state=None, **kw):
    p = torch.nn.Parameter(w.clone().double())
    opt = cls([p], **kw)
    if state is not None:
        opt.state[p] = state
    p.grad = g.clone().double()
    opt.step()
    return p.detach(), opt


def test_lamb_zero_weight_norm_gives_trust_one():
    g = torch.tensor([0.5, -1.0, 2.0])
    w1, _ = _one_step(LAMB, torch.zeros(3), g, lr=0.1, weight_decay=0.01)
    # t = 1: m / bc1 = g, sqrt(v / bc2) = |g|: r = sign(g) / (1 + eps / |g|), trust 1
    r = g.double() / (g.double().abs() + 1e-6)
    assert torch.allclose(w1, -0.1 * r, rtol=1e-12)


def test_lamb_zero_update_norm_gives_trust_one():
    """rn == 0: zero gradient and zero moments with weight decay 0 and always_adapt; the update is 0, not NaN."""
    w = torch.tensor([1.0, 2.0])
    w1, _ = _one_step(LAMB, w, torch.zeros(2), lr=0.1, weight_decay=0.0, always_adapt=True)
    assert torch.equal(w1, w.double())


def test_lars_zero_norms_give_trust_one():
    g = torch.tensor([0.5, -1.0])
    w1, _ = _one_step(LARS, torch.zeros(2), g, lr=0.1, momentum=0.0, weight_decay=0.1)   # wn == 0: g + wd w = g
    assert torch.allclose(w1, -0.1 * g.double())
    w = torch.tensor([1.0, -2.0])
    w1, _ = _one_step(LARS, w, torch.zeros(2), lr=0.1, momentum=0.0, weight_decay=0.1)   # gn == 0: trust 1
    assert torch.allclose(w1, w.double() - 0.1 * 0.1 * w.double())


def test_nan_norm_gives_trust_one():
    """A NaN gradient makes ||g|| (LARS) or ||r|| (LAMB) NaN; the comparison fails and the trust ratio is 1, so only the
    NaN element's own update is NaN."""
    w = torch.tensor([1.0, -2.0, 3.0])
    g = torch.tensor([0.1, float("nan"), 0.2])
    w1, _ = _one_step(LARS, w, g, lr=0.1, momentum=0.0, weight_decay=0.1)
    exp = w.double() - 0.1 * (g.double() + 0.1 * w.double())
    assert torch.equal(w1.isnan(), exp.isnan()) and torch.allclose(w1[~exp.isnan()], exp[~exp.isnan()])
    w1, _ = _one_step(LAMB, w, g, lr=0.1, weight_decay=0.1)
    r = g.double() / (g.double().abs() + 1e-6) + 0.1 * w.double()
    exp = w.double() - 0.1 * r
    assert torch.equal(w1.isnan(), exp.isnan()) and torch.allclose(w1[~exp.isnan()], exp[~exp.isnan()])


def test_weight_decay_zero_with_and_without_always_adapt():
    w = torch.tensor([1.0, -2.0, 3.0])
    g = torch.tensor([0.3, -0.1, 0.2])
    # LARS, no momentum: plain SGD without always_adapt; trust tc ||w|| / (||g|| + eps) with it
    w1, _ = _one_step(LARS, w, g, lr=0.5, momentum=0.0)
    assert torch.allclose(w1, w.double() - 0.5 * g.double())
    w1, _ = _one_step(LARS, w, g, lr=0.5, momentum=0.0, always_adapt=True, trust_coefficient=0.01)
    trust = 0.01 * w.double().norm() / (g.double().norm() + 1e-8)
    assert torch.allclose(w1, w.double() - 0.5 * trust * g.double())
    # LAMB at t = 1: r = g / (|g| + eps); with always_adapt scaled to ||w|| / ||r||
    r = g.double() / (g.double().abs() + 1e-6)
    w1, _ = _one_step(LAMB, w, g, lr=0.1, weight_decay=0.0)
    assert torch.allclose(w1, w.double() - 0.1 * r)
    w1, _ = _one_step(LAMB, w, g, lr=0.1, weight_decay=0.0, always_adapt=True)
    assert torch.allclose(w1, w.double() - 0.1 * (w.double().norm() / r.norm()) * r)


def test_lars_nesterov_and_momentum_seeding():
    w = torch.tensor([1.0, -2.0])
    g1, g2 = torch.tensor([0.3, -0.1]), torch.tensor([-0.2, 0.4])
    p = torch.nn.Parameter(w.clone().double())
    opt = LARS([p], lr=0.1, momentum=0.9, nesterov=True)
    p.grad = g1.double()
    opt.step()
    buf = g1.double()                                   # t == 1: buf = g
    exp = w.double() - 0.1 * (g1.double() + 0.9 * buf)
    assert torch.allclose(p.detach(), exp)
    p.grad = g2.double()
    opt.step()
    buf = buf * 0.9 + g2.double()
    exp = exp - 0.1 * (g2.double() + 0.9 * buf)
    assert torch.allclose(p.detach(), exp)
    assert torch.allclose(opt.state[p]["momentum_buffer"], buf)
    with pytest.raises(ValueError):
        LARS([p], momentum=0.0, nesterov=True)


def test_closure_is_called():
    for cls in (LAMB, LARS):
        p = torch.nn.Parameter(torch.ones(3))
        opt = cls([p])

        def closure():
            opt.zero_grad()
            loss = (p * p).sum()
            loss.backward()
            return loss

        assert float(opt.step(closure).detach()) == 3.0
        assert not torch.equal(p.detach(), torch.ones(3))


# ---- routing and checkpoint state ------------------------------------------------------------------------------------------
def _groups(n):
    net = torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(n)])
    return net, {"params": [{"params": [m.weight], "weight_decay": 0.0 if i % 2 else 0.01} for i, m in enumerate(net)]}


@pytest.mark.parametrize("cls", [LAMB, LARS])
def test_fused_supported_up_to_eight_groups(cls):
    for n in (1, 8):
        net, kw = _groups(n)
        assert fused_supported(cls, kw, net), n
    net, kw = _groups(9)
    assert not fused_supported(cls, kw, net)
    assert fused_supported(cls, {"lr": 0.1}, torch.nn.Linear(3, 3))


def test_state_is_created_lazily_in_the_classes_layout():
    a, b = torch.nn.Parameter(torch.randn(4)), torch.nn.Parameter(torch.randn(3))
    for cls, kw, keys in ((LAMB, {}, {"step", "exp_avg", "exp_avg_sq"}), (LARS, {}, {"step", "momentum_buffer"}),
                          (LARS, {"momentum": 0.0}, {"step"})):
        opt = cls([a, b], **kw)
        assert opt.state_dict()["state"] == {}
        a.grad, b.grad = torch.randn(4), None
        opt.step()
        sd = opt.state_dict()["state"]
        assert set(sd) == {0} and set(sd[0]) == keys, (cls, kw)
        assert sd[0]["step"].dtype == torch.float32 and sd[0]["step"].dim() == 0 and float(sd[0]["step"]) == 1.0
        a.grad = None


def test_load_step_counts_reads_the_classes_state():
    """Per-parameter counts come from ``step``; a parameter without an entry has taken 0 steps; there is no scalar state."""
    for kind in (_LAMB, _LARS):
        entries = [{"step": torch.tensor(3.0)}, {}, {"step": torch.tensor(2.0)}]
        opt_steps, steps, scal = load_step_counts(kind, entries, [0, 0, 1], None, True)
        assert (opt_steps, steps, scal) == (3, [3, 0, 2], None)
        opt_steps, steps, scal = load_step_counts(kind, entries, [0, 0, 1], 5, True)
        assert (opt_steps, steps, scal) == (5, [3, 0, 2], None)


def test_checkpoint_round_trip_between_class_instances():
    """A state dict of one instance continues identically in another (torch's load_state_dict of the classes)."""
    torch.manual_seed(0)
    for cls, kw in ((LAMB, {"lr": 1e-2}), (LARS, {"lr": 0.1, "weight_decay": 1e-3})):
        m1 = torch.nn.Linear(5, 3)
        m2 = torch.nn.Linear(5, 3)
        o1 = cls(m1.parameters(), **kw)
        xs = [torch.randn(4, 5) for _ in range(6)]
        for x in xs[:3]:
            o1.zero_grad()
            m1(x).pow(2).sum().backward()
            o1.step()
        m2.load_state_dict(m1.state_dict())
        o2 = cls(m2.parameters(), **kw)
        o2.load_state_dict(copy.deepcopy(o1.state_dict()))   # torch's load keeps same-device tensors as they are
        for x in xs[3:]:
            for m, o in ((m1, o1), (m2, o2)):
                o.zero_grad()
                m(x).pow(2).sum().backward()
                o.step()
        for a, b in zip(m1.parameters(), m2.parameters()):
            assert torch.equal(a, b)
        assert not math.isnan(float(m1.weight.sum()))
