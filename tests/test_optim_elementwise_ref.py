"""CPU checks of the Adadelta / Rprop / ASGD reference (tests/optim_elementwise_ref.py), of the routing of those classes to
the fused step, and of their state_dict layout.

torch's own fp32 single-tensor step must stay inside the per-element bounds (Adadelta, ASGD) or reproduce the fp32
reference bit for bit (Rprop) over a run of steps, every step compared with the reference restarted from the fp32 state,
and every deliberately wrong reference must fall outside them: the same check the GPU tests apply to the kernel.  ASGD's
fp32 ``eta`` / ``mu`` must follow ``asgd_next`` (the formulas the step prologue uses) bit for bit."""
import pytest
import torch

import optim_elementwise_ref as oer

ADADELTA = {"lr": 0.5, "rho": 0.875, "eps": 1e-6}
RPROP = {"lr": 2.0**-7, "etas": (0.5, 1.2), "step_sizes": (1e-6, 50.0)}
ASGD = {"lr": 2.0**-4, "lambd": 1e-2, "alpha": 0.75, "t0": 1e6}
CASES = {
    "adadelta": ADADELTA,
    "adadelta_l2_max": dict(ADADELTA, weight_decay=0.25, maximize=True),
    "rprop": RPROP,
    "rprop_max_tight": dict(RPROP, maximize=True, step_sizes=(2.0**-9, 2.0**-6)),
    "rprop_etaminus_one": dict(RPROP, etas=(1.0, 1.2)),
    "rprop_etas_equal": dict(RPROP, etas=(1.2, 1.2)),
    "asgd": ASGD,
    "asgd_l2_max_t0": dict(ASGD, weight_decay=0.25, maximize=True, t0=3.0),
}
STEPS = 10


def _mutations(name, h):
    kind = name.split("_")[0]
    out = list(oer.MUTATIONS[kind])
    if kind == "rprop" and h["etas"][0] != 1.0 and h["etas"][0] != h["etas"][1]:
        out.remove("no_mask_quirk")   # the quirk only shows with etaminus == 1 or etaplus == etaminus
    if kind == "rprop" and h["etas"][0] == 1.0:
        out.remove("sign_per_factor")   # etaminus == 1 masks every s == 0 element, so prev stays 0 for good
    if kind == "asgd":   # with t0 = 1e6 mu stays 1: "never_average" is the right update; with a small t0 averaging is due
        out.remove("never_average" if h["t0"] > 100 else "always_average")
    return out


def _grad(kind, n, gen, step):
    g = torch.randn(n, generator=gen) * 1e-3
    if kind == "rprop":   # a band of tiny gradients whose fp32 product with prev underflows to 0, both factors non-zero
        g[: n // 8] *= 1e-22
    if step % 3 == 2:   # some exact zeros and sign flips
        g[n // 8: n // 8 + 64] = 0.0
    return g


def _same_by_construction(kind, mutation, t, h):
    if mutation == "always_average":   # mu = 1 / t is 1 at the first step
        return t == 1
    if mutation == "sign_per_factor":  # prev = 0 at the first step: both signs are 0
        return t == 1
    if mutation == "no_mask_quirk":
        # prev = 0 at the first step: s == 0 elements are masked only when etaminus == 1.  With etaplus == etaminus every
        # s != 0 element is masked at even steps, so prev is 0 there at the odd steps that follow
        return h["etas"][0] != 1.0 and t % 2 == 1
    if mutation == "never_average":    # mu = 1 / max(1, t - 1 - t0) while t - 1 - t0 <= 1
        return t - 1 - h["t0"] <= 1
    return False


@pytest.mark.parametrize("name", list(CASES))
def test_fp32_torch_inside_bounds_and_mutants_outside(name):
    kind = name.split("_")[0]
    h = CASES[name]
    n = 4096
    gen = torch.Generator().manual_seed(len(name))
    p = torch.nn.Parameter(torch.randn(n, generator=gen) * 1e-3)
    opt = oer.make_optimizer(kind, [p], h)
    keys = oer.STATE_KEYS[kind]
    hit = set()
    for step in range(STEPS):
        g = _grad(kind, n, gen, step)
        st = opt.state.get(p)
        w = p.detach().clone()
        m = st[keys[0]].clone() if st else torch.zeros(n)
        v = (st[keys[1]].clone() if st else torch.zeros(n)) if len(keys) > 1 else None
        eta = float(st["eta"]) if kind == "asgd" and st else None
        mu = float(st["mu"]) if kind == "asgd" and st else None
        p.grad = g.clone()
        opt.step()
        st = opt.state[p]
        got_w, got_m = p.detach(), st[keys[0]]
        got_v = st[keys[1]] if len(keys) > 1 else None
        if kind == "rprop":
            rw, rm, rv = oer.rprop_fp32(w, m, v, g, step, h)
            for what, got, ref in (("w", got_w, rw), ("prev", got_m, rm), ("step_size", got_v, rv)):
                assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), f"{name} step {step + 1}: {what}"
            base = (got_w, got_m, got_v)
        else:
            e_use, m_use = oer.asgd_used(h, step, eta, mu) if kind == "asgd" else (None, None)
            rw, rm, rv, reta, rmu = oer.torch_step(kind, w, m, v, g, step, h, eta, mu)
            ew, em, ev = oer.step_bound(kind, w, m, v, g.double(), torch.zeros(n, dtype=torch.float64), h, rw, rm, rv,
                                        e_use, m_use)
            outs = [("w", got_w, rw, ew), ("m", got_m, rm, em)] + ([("v", got_v, rv, ev)] if v is not None else [])
            for what, got, ref, b in outs:
                bad = (got.double() - ref).abs() > b
                assert not bool(bad.any()), f"{name} step {step + 1}: {what} outside the bound at {bad.nonzero()[:4].flatten()}"
            if kind == "asgd":
                assert st["eta"].dtype == torch.float32 and st["eta"].dim() == 0 and st["mu"].dim() == 0
                assert (float(st["eta"]), float(st["mu"])) == oer.asgd_next(h, step + 1) == (reta, rmu)
        for mut in _mutations(name, h):
            mw, mm, mv = oer.step_mutant(kind, w, m, v, g, step, h, mut, eta, mu)
            if kind == "rprop":
                caught = not all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(base, (mw, mm, mv)))
            else:
                caught = bool(((got_w.double() - mw).abs() > ew).any()) or bool(((got_m.double() - mm).abs() > em).any())
            if caught:
                hit.add(mut)
            elif not _same_by_construction(kind, mut, step + 1, h):
                pytest.fail(f"{name}: negative control {mut} passed at step {step + 1}")
    assert hit == set(_mutations(name, h)), hit


def test_asgd_scalars_follow_fp32_formulas_over_many_steps():
    h = dict(ASGD, t0=50.0, lambd=1e-3)
    p = torch.nn.Parameter(torch.zeros(8))
    opt = oer.make_optimizer("asgd", [p], h)
    for t in range(1, 301):
        eta_before = float(opt.state[p]["eta"]) if t > 1 else None
        p.grad = torch.ones(8)
        opt.step()
        assert (float(opt.state[p]["eta"]), float(opt.state[p]["mu"])) == oer.asgd_next(h, t), t
        if eta_before is not None:   # the hand-off uses the stored value, not this step's
            assert oer.asgd_handoff(h, t - 1, eta_before, 1.0)[0] == -eta_before


def test_rprop_first_step_seeds_step_size_with_current_lr():
    """torch creates step_size = full_like(p, lr) at the first step with the group's lr at that moment."""
    p = torch.nn.Parameter(torch.ones(4))
    opt = oer.make_optimizer("rprop", [p], RPROP)
    opt.param_groups[0]["lr"] = 0.125   # a scheduler edit before the first step
    p.grad = torch.tensor([1.0, -1.0, 0.0, 2.0])
    opt.step()
    assert torch.equal(opt.state[p]["step_size"], torch.full((4,), 0.125))
    w, prev, ss = oer.rprop_fp32(torch.ones(4), torch.zeros(4), torch.zeros(4), torch.tensor([1.0, -1.0, 0.0, 2.0]), 0,
                                 dict(RPROP, lr=0.125))
    assert torch.equal(ss, opt.state[p]["step_size"]) and torch.equal(w, p.detach())


# ---- routing and state_dict layout ---------------------------------------------------------------------------------------
def _net():
    return torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.Linear(4, 2))


ELEMENTWISE = (torch.optim.Adadelta, torch.optim.Rprop, torch.optim.ASGD)


def test_fused_supported_routing():
    from stoke_b200.optim import fused_supported

    net = _net()
    for cls in ELEMENTWISE:
        assert fused_supported(cls, {"lr": 1e-3}, net)
        assert fused_supported(cls, {"lr": 1e-3, "maximize": True}, net)
        assert fused_supported(cls, {"lr": 1e-3, "foreach": True}, net)
        assert not fused_supported(cls, {"lr": 1e-3, "capturable": True}, net)
        assert not fused_supported(cls, {"lr": 1e-3, "differentiable": True}, net)
        params = list(net.parameters())
        assert fused_supported(cls, {"lr": 1e-3, "params": [{"params": [q]} for q in params]}, net)
    big = torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(9)])
    nine = {"lr": 1e-3, "params": [{"params": [q]} for q in big.parameters()]}
    eight = {"lr": 1e-3, "params": [{"params": [q]} for q in list(big.parameters())[:8]] +
             [{"params": [list(big.parameters())[8]], "lr": 2e-3}]}
    for cls in ELEMENTWISE:
        assert not fused_supported(cls, nine, big)
    eight["params"][7]["params"].append(eight["params"].pop()["params"][0])
    for cls in ELEMENTWISE:
        assert fused_supported(cls, eight, big)
    # the classes this change leaves on the stock route
    for cls in (torch.optim.RMSprop, torch.optim.Adagrad, torch.optim.LBFGS, torch.optim.SparseAdam):
        assert not fused_supported(cls, {"lr": 1e-3}, net)


def test_kind_and_state_layout_of_each_class():
    from stoke_b200 import _lib
    from stoke_b200.optim import _KINDS, _STATE_LAYOUT

    assert (_lib.OPT_ADADELTA, _lib.OPT_RPROP, _lib.OPT_ASGD) == (6, 7, 8)
    assert _KINDS[torch.optim.Adadelta] == _lib.OPT_ADADELTA
    assert _KINDS[torch.optim.Rprop] == _lib.OPT_RPROP
    assert _KINDS[torch.optim.ASGD] == _lib.OPT_ASGD
    # the state torch's single-tensor classes keep, per parameter
    for cls, kind in ((torch.optim.Adadelta, _lib.OPT_ADADELTA), (torch.optim.Rprop, _lib.OPT_RPROP),
                      (torch.optim.ASGD, _lib.OPT_ASGD)):
        p = torch.nn.Parameter(torch.ones(3))
        opt = cls([p], lr=1e-2, foreach=False)
        p.grad = torch.ones(3)
        opt.step()
        lay = _STATE_LAYOUT[kind]
        want = {t.key for t in lay.tensors} | set(lay.scalars) | {"step"}
        assert set(opt.state[p]) == want, cls
    assert [t.buf for t in _STATE_LAYOUT[_lib.OPT_ASGD].tensors] == ["M"]   # ASGD has no V


def test_ext_struct_appends_fields():
    """The new hyper-parameters are appended to stk_optim_hyper_ext_t: the NAdam / RAdam fields keep their offsets."""
    import ctypes as C

    from stoke_b200 import _lib

    X = _lib.OptimHyperExt
    assert X.momentum_decay.offset == 0 and X.decoupled_weight_decay.offset == 8
    names = [f[0] for f in X._fields_]
    assert names == ["momentum_decay", "decoupled_weight_decay", "rho", "etaminus", "etaplus", "step_size_min",
                     "step_size_max", "lambd", "alpha", "t0"]
    assert C.sizeof(X) == 16 + 8 * 8
    assert C.sizeof(_lib.OptimHyper) == 8 + 8 * 7 + 4 * 3 + 4 + 16


def test_exts_and_hypers_per_group():
    """_hyper_of and the OptimHyperExt builder fill each class's fields from its param_groups (no GPU: the optimizer
    object is not built)."""
    from stoke_b200 import _lib
    from stoke_b200.optim import _EXT_KINDS, _GROUP_HYPER, B200FusedOptimizer, _ext_hyper

    obj = B200FusedOptimizer.__new__(B200FusedOptimizer)
    groups = {
        _lib.OPT_ADADELTA: {"lr": 0.5, "rho": 0.8, "eps": 1e-5, "weight_decay": 0.1, "maximize": True},
        _lib.OPT_RPROP: {"lr": 0.01, "etas": (0.4, 1.3), "step_sizes": (1e-5, 10.0), "maximize": False},
        _lib.OPT_ASGD: {"lr": 0.02, "lambd": 1e-3, "alpha": 0.5, "t0": 100.0, "weight_decay": 0.2, "maximize": False},
    }
    for kind, g in groups.items():
        obj._kind = kind
        obj.param_groups = [g]
        h, x = obj._hyper_of(g), _GROUP_HYPER[kind](g)
        assert h.kind == kind and h.lr == g["lr"] and h.maximize == int(g["maximize"])
        assert h.weight_decay == g.get("weight_decay", 0.0)
        if kind == _lib.OPT_ADADELTA:
            assert (h.eps, x.rho) == (1e-5, 0.8)
        if kind == _lib.OPT_RPROP:
            assert (x.etaminus, x.etaplus, x.step_size_min, x.step_size_max) == (0.4, 1.3, 1e-5, 10.0)
        if kind == _lib.OPT_ASGD:
            assert (x.lambd, x.alpha, x.t0) == (1e-3, 0.5, 100.0)
    assert {k for k, f in _GROUP_HYPER.items() if f is _ext_hyper} == set(_EXT_KINDS)
