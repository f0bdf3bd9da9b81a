"""CPU checks of the NAdam / RAdam / Adamax reference (tests/optim_family_ref.py) and of the routing of those classes to the
fused step.

torch's own fp32 single-tensor step must stay inside the per-element bounds over a run of steps, every step compared with
the float64 reference restarted from the fp32 state, and every deliberately wrong reference must fall outside them: the same
check the GPU tests apply to the kernel.  NAdam's fp32 ``mu_product`` must follow ``mu_product_f32`` (the formula the step
prologue uses) bit for bit."""
import pytest
import torch

import optim_family_ref as ofr
from kernel_ref import U

BASE = {"lr": 2.0**-7, "beta1": 0.875, "beta2": 0.999, "eps": 2.0**-20, "momentum_decay": 4e-3}
CASES = {
    "nadam": BASE,
    "nadam_l2_max": dict(BASE, weight_decay=0.25, maximize=True),
    "nadam_decoupled": dict(BASE, weight_decay=0.25, decoupled_weight_decay=True, momentum_decay=0.05),
    "radam": BASE,
    "radam_l2": dict(BASE, weight_decay=0.25, maximize=True),
    "radam_decoupled": dict(BASE, weight_decay=0.25, decoupled_weight_decay=True),
    "adamax": dict(BASE, eps=2.0**-12),
    "adamax_l2_max": dict(BASE, eps=2.0**-12, weight_decay=0.25, maximize=True),
}
STEPS = 12
# the first step torch's RAdam takes rectified (rho_t > 5) with beta2 = 0.999: found from torch's own update (the test below
# checks that steps 1..5 match the plain update and step 6 the rectified one)
RADAM_FIRST_RECTIFIED = 6


def _mutations(kind, h):
    return [mu for mu in ofr.MUTATIONS[kind] if mu != "decoupled_as_l2" or h.get("decoupled_weight_decay")]


def _same_by_construction(kind, mutation, h, t):
    """Steps at which a wrong reference computes the same formula as torch: the threshold moved by one step differs only
    at the crossing, rect only matters on rectified steps, and eps after the max equals eps inside it while exp_inf is 0."""
    if mutation == "threshold_late":
        return t != RADAM_FIRST_RECTIFIED
    if mutation == "threshold_early":
        return t != RADAM_FIRST_RECTIFIED - 1
    if mutation == "no_rect":
        return not ofr.radam_rectified(h, t)
    if mutation == "eps_after_max":
        return t == 1
    if mutation == "decoupled_as_l2":   # RAdam's plain first step: w (1 - lr wd) - lr g either way (bc1 = 1 - b1)
        return kind == "radam" and t == 1
    return False


@pytest.mark.parametrize("name", list(CASES))
def test_fp32_torch_inside_bounds_and_mutants_outside(name):
    kind = name.split("_")[0]
    h = CASES[name]
    n = 4096
    gen = torch.Generator().manual_seed(len(name))
    p = torch.nn.Parameter(torch.randn(n, generator=gen) * 1e-3)
    opt = ofr.make_optimizer(kind, [p], h)
    hit = set()
    for step in range(STEPS):
        g = torch.randn(n, generator=gen) * 1e-3
        st = opt.state.get(p)
        w = p.detach().clone()
        if st:
            m, v = st["exp_avg"].clone(), st[ofr.second_key(kind)].clone()
            mu0 = float(st["mu_product"]) if kind == "nadam" else None
        else:
            m, v, mu0 = torch.zeros(n), torch.zeros(n), 1.0
        p.grad = g.clone()
        opt.step()
        st = opt.state[p]
        got_w, got_m, got_v = p.detach(), st["exp_avg"], st[ofr.second_key(kind)]
        rw, rm, rv, rmu = ofr.step_ref(kind, w, m, v, g, step, h, mu0)
        ew, em, ev = ofr.step_bound(kind, w, m, v, g.double(), torch.zeros(n, dtype=torch.float64), step, h, rm, rv, mu0)
        for what, got, ref, b in (("w", got_w, rw, ew), ("m", got_m, rm, em), ("v", got_v, rv, ev)):
            bad = (got.double() - ref).abs() > b
            assert not bool(bad.any()), f"{name} step {step + 1}: {what} outside the bound at {bad.nonzero()[:4].flatten()}"
        if kind == "nadam":
            got_mu = float(st["mu_product"])
            assert st["mu_product"].dtype == torch.float32 and st["mu_product"].dim() == 0
            assert got_mu == ofr.mu_product_f32(mu0, h, step + 1)
            assert abs(got_mu - rmu) <= 2 * U * rmu
        for mu in _mutations(kind, h):
            if mu == "mu_not_advanced" and step == 0:   # the product before step 1 is 1: that coefficient is infinite
                continue
            mw = ofr.step_mutant(kind, w, m, v, g, step, h, mu, mu0)
            if bool(((got_w.double() - mw).abs() > ew).any()):
                hit.add(mu)
            elif not _same_by_construction(kind, mu, h, step + 1):
                pytest.fail(f"{name}: negative control {mu} passed at step {step + 1}")
    assert hit == set(_mutations(kind, h)), hit


def test_radam_crossing_step():
    h = CASES["radam"]
    assert [ofr.radam_rectified(h, t) for t in range(1, 9)] == [t >= RADAM_FIRST_RECTIFIED for t in range(1, 9)]


def test_nadam_mu_product_follows_fp32_formula_over_many_steps():
    h = dict(BASE, momentum_decay=0.05)
    p = torch.nn.Parameter(torch.zeros(8))
    opt = ofr.make_optimizer("nadam", [p], h)
    mu = 1.0
    for t in range(1, 301):
        p.grad = torch.ones(8)
        opt.step()
        mu = ofr.mu_product_f32(mu, h, t)
        assert float(opt.state[p]["mu_product"]) == mu, t


# ---- routing ----------------------------------------------------------------------------------------------------------------
def _net():
    return torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.Linear(4, 2))


def test_fused_supported_routing():
    from stoke_b200.optim import fused_supported

    net = _net()
    for cls in (torch.optim.NAdam, torch.optim.RAdam, torch.optim.Adamax):
        assert fused_supported(cls, {"lr": 1e-3}, net)
        assert fused_supported(cls, {"lr": 1e-3, "weight_decay": 0.1, "maximize": True}, net)
        assert not fused_supported(cls, {"lr": 1e-3, "capturable": True}, net)
        assert not fused_supported(cls, {"lr": 1e-3, "differentiable": True}, net)
        params = list(net.parameters())
        assert fused_supported(cls, {"lr": 1e-3, "params": [{"params": [q]} for q in params]}, net)
    for cls in (torch.optim.NAdam, torch.optim.RAdam):
        assert fused_supported(cls, {"lr": 1e-3, "weight_decay": 0.1, "decoupled_weight_decay": True}, net)
    assert not fused_supported(torch.optim.RMSprop, {"lr": 1e-3}, net)
    assert not fused_supported(torch.optim.Adagrad, {"lr": 1e-3}, net)
    assert not fused_supported(torch.optim.Adam, {"lr": 1e-3, "amsgrad": True}, net)
    # 9 groups: one more than the kernel's group table
    big = torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(9)])
    nine = {"lr": 1e-3, "params": [{"params": [q]} for q in big.parameters()]}
    for cls in (torch.optim.NAdam, torch.optim.RAdam, torch.optim.Adamax, torch.optim.Adam):
        assert not fused_supported(cls, nine, big)


def test_kind_of_each_class():
    """NAdam and RAdam carry decoupled_weight_decay as an option of their own update: it must not turn them into AdamW
    (only Adam(decoupled_weight_decay=True) is AdamW).  Checked on the kind selection alone (no GPU needed)."""
    from stoke_b200 import _lib
    from stoke_b200.optim import _KINDS

    assert _KINDS[torch.optim.NAdam] == _lib.OPT_NADAM
    assert _KINDS[torch.optim.RAdam] == _lib.OPT_RADAM
    assert _KINDS[torch.optim.Adamax] == _lib.OPT_ADAMAX
    from stoke_b200.optim import B200FusedOptimizer

    class FakeEngine:   # stops construction right after the kind is chosen
        pass

    for cls, kw, want in ((torch.optim.NAdam, {"decoupled_weight_decay": True, "weight_decay": 0.1}, _lib.OPT_NADAM),
                          (torch.optim.RAdam, {"decoupled_weight_decay": True, "weight_decay": 0.1}, _lib.OPT_RADAM),
                          (torch.optim.Adam, {"decoupled_weight_decay": True, "weight_decay": 0.1}, _lib.OPT_ADAMW),
                          (torch.optim.Adamax, {}, _lib.OPT_ADAMAX)):
        obj = B200FusedOptimizer.__new__(B200FusedOptimizer)
        with pytest.raises(Exception):
            B200FusedOptimizer.__init__(obj, _net(), cls, dict(kw, lr=1e-3), engine=FakeEngine())
        assert obj._kind == want, cls
