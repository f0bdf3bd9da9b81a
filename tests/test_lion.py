"""stoke_b200.Lion on the CPU: argument validation, known answers on hand-picked fp32 values (every value below is exact in
fp32, so each expected number is exact), lazy state, and the routing / ABI constants of the fused step."""
import os

import pytest
import torch

import stoke_b200 as sb
from stoke_b200 import _lib
from stoke_b200.optim import Lion

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _one(values, grad, **kw):
    p = torch.nn.Parameter(torch.tensor(values, dtype=torch.float32))
    opt = Lion([p], **kw)
    p.grad = torch.tensor(grad, dtype=torch.float32)
    return p, opt


@pytest.mark.parametrize("kw", [{"lr": -1e-4}, {"betas": (1.0, 0.99)}, {"betas": (0.9, 1.0)}, {"betas": (-0.1, 0.99)},
                                {"betas": (0.9, -0.5)}, {"weight_decay": -0.1}])
def test_validation(kw):
    with pytest.raises(ValueError):
        Lion([torch.nn.Parameter(torch.zeros(2))], **kw)


def test_defaults():
    opt = Lion([torch.nn.Parameter(torch.zeros(2))])
    assert opt.defaults == {"lr": 1e-4, "betas": (0.9, 0.99), "weight_decay": 0.0, "maximize": False}
    Lion([torch.nn.Parameter(torch.zeros(2))], lr=0.0, betas=(0.0, 0.0), weight_decay=0.0)   # the closed ends are valid


def test_first_step_signs_zero_and_nan():
    """m = 0 at the first step, so c = (1 - beta1) g and the update is -lr sign(g).  c == 0 (a +-0 gradient) and a NaN
    gradient leave the parameter bit-unchanged (+-0 parameters keep their sign bit); the NaN lands in exp_avg."""
    nan = float("nan")
    p, opt = _one([1.0, -2.0, 0.0, -0.0, 0.0, -0.0, 4.0, 3.0],
                  [1.0, 1.0, -1.0, 2.0, 0.0, -0.0, -0.0, nan], lr=0.5, betas=(0.5, 0.75))
    before = p.detach().clone()
    opt.step()
    want = torch.tensor([0.5, -2.5, 0.5, -0.5, 0.0, -0.0, 4.0, 3.0])
    assert torch.equal(_bits(p), _bits(want))
    assert torch.equal(_bits(p[4:7]), _bits(before[4:7]))
    m = opt.state[p]["exp_avg"]
    assert torch.equal(m[:7], torch.tensor([0.25, 0.25, -0.25, 0.5, 0.0, 0.0, 0.0]))
    assert bool(torch.isnan(m[7]))


def test_second_step_uses_beta1_for_the_update_and_beta2_for_the_state():
    """c = beta1 m + (1 - beta1) g decides the sign; exp_avg moves with beta2.  With m = 0.25 (from g = 1) and g = -1:
    c = 0.5 * 0.25 - 0.5 = -0.375 (update +lr) and m = 0.75 * 0.25 - 0.25 = -0.0625.  For the second element g = -0.25:
    c = 0.125 - 0.125 = 0 (no update) while the new exp_avg is 0.125 > 0, so taking the sign of the new exp_avg, or
    swapping the betas (c = 0.1875 - 0.0625 > 0), would move it."""
    p, opt = _one([1.0, 1.0], [1.0, 1.0], lr=0.5, betas=(0.5, 0.75))
    opt.step()
    assert torch.equal(p.detach(), torch.tensor([0.5, 0.5]))
    p.grad = torch.tensor([-1.0, -0.25])
    opt.step()
    assert torch.equal(p.detach(), torch.tensor([1.0, 0.5]))
    assert torch.equal(opt.state[p]["exp_avg"], torch.tensor([-0.0625, 0.125]))
    assert float(opt.state[p]["step"]) == 2.0


def test_maximize_flips_the_gradient():
    p, opt = _one([1.0, 1.0], [1.0, -1.0], lr=0.5, betas=(0.5, 0.75), maximize=True)
    opt.step()
    assert torch.equal(p.detach(), torch.tensor([1.5, 0.5]))
    assert torch.equal(opt.state[p]["exp_avg"], torch.tensor([-0.25, 0.25]))


def test_weight_decay_is_decoupled_and_applied_before_the_update():
    """w = 2, lr = 0.5, wd = 0.5: w (1 - 0.25) - 0.5 = 1.0.  Decay after the update would give (2 - 0.5) 0.75 = 1.125;
    decay added to the gradient would change nothing here (the sign stays +1) but also move exp_avg."""
    p, opt = _one([2.0, 2.0], [1.0, 0.0], lr=0.5, betas=(0.5, 0.75), weight_decay=0.5)
    opt.step()
    assert torch.equal(p.detach(), torch.tensor([1.0, 1.5]))
    assert torch.equal(opt.state[p]["exp_avg"], torch.tensor([0.25, 0.0]))


def test_lazy_state_and_step_counter():
    a, b = torch.nn.Parameter(torch.ones(3)), torch.nn.Parameter(torch.ones(2))
    opt = Lion([a, b], lr=0.1)
    assert opt.state_dict()["state"] == {}
    a.grad = torch.ones(3)
    opt.step()
    assert b not in opt.state
    sd = opt.state_dict()
    assert set(sd["state"]) == {0}
    st = sd["state"][0]
    assert set(st) == {"step", "exp_avg"}
    assert st["step"].dtype == torch.float32 and st["step"].dim() == 0 and float(st["step"]) == 1.0
    b.grad = torch.ones(2)
    opt.step()
    assert float(opt.state[a]["step"]) == 2.0 and float(opt.state[b]["step"]) == 1.0
    # a plain Lion continues from its own state dict
    a2, b2 = torch.nn.Parameter(a.detach().clone()), torch.nn.Parameter(b.detach().clone())
    opt2 = Lion([a2, b2], lr=0.1)
    opt2.load_state_dict(opt.state_dict())
    for x, y in ((a, a2), (b, b2)):
        x.grad = torch.full_like(x, -0.5)
        y.grad = torch.full_like(y, -0.5)
    opt.step()
    opt2.step()
    assert torch.equal(a.detach(), a2.detach()) and torch.equal(b.detach(), b2.detach())


def test_constants_and_state_layout():
    from stoke_b200.optim import _EXT_KINDS, _KINDS, _STATE_LAYOUT

    assert _lib.OPT_LION == 9
    assert "Lion" in sb.__all__ and sb.Lion is Lion
    assert _KINDS[Lion] == _lib.OPT_LION
    lay = _STATE_LAYOUT[_lib.OPT_LION]
    assert [(t.key, t.buf) for t in lay.tensors] == [("exp_avg", "M")]   # one state tensor: no V
    assert lay.step and lay.unstepped == "omit" and lay.scalars == ()
    assert _lib.OPT_LION not in _EXT_KINDS   # no per-step scalars: the prologue runs only for per-parameter counts
    with open(os.path.join(ROOT, "include", "stoke_b200.h")) as f:
        assert "STK_OPT_LION = 9" in f.read()


def _net(n=3):
    return torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(n)])


def test_fused_supported():
    from stoke_b200.optim import fused_supported

    net = _net()
    assert fused_supported(Lion, {"lr": 1e-4}, net)
    assert fused_supported(Lion, {"lr": 1e-4, "weight_decay": 0.1, "maximize": True}, net)
    assert not fused_supported(Lion, {"lr": 1e-4, "differentiable": True}, net)
    big = _net(9)
    ps = list(big.parameters())
    assert not fused_supported(Lion, {"params": [{"params": [q]} for q in ps]}, big)
    eight = [{"params": [q], "lr": 1e-4 * (i + 1)} for i, q in enumerate(ps[:8])]
    eight[7]["params"].append(ps[8])
    assert fused_supported(Lion, {"params": eight}, big)
    # these stay on the stock route
    for cls, kw in ((torch.optim.RMSprop, {}), (torch.optim.Adagrad, {}), (torch.optim.Adam, {"amsgrad": True}),
                    (torch.optim.AdamW, {"amsgrad": True})):
        assert not fused_supported(cls, dict(kw, lr=1e-3), net)


def test_hyper_of_lion_and_the_existing_classes():
    """Lion's betas, weight decay and maximize reach stk_optim_hyper_t (Lion has no eps); the classes with betas and eps
    keep theirs."""
    from stoke_b200.optim import _GROUP_HYPER, B200FusedOptimizer

    obj = B200FusedOptimizer.__new__(B200FusedOptimizer)
    obj._kind = _lib.OPT_LION
    g = {"lr": 3e-4, "betas": (0.95, 0.98), "weight_decay": 0.1, "maximize": True}
    obj.param_groups = [g]
    h = obj._hyper_of(g)
    assert (h.kind, h.lr, h.beta1, h.beta2, h.weight_decay, h.maximize, h.eps) == (9, 3e-4, 0.95, 0.98, 0.1, 1, 0.0)
    assert _lib.OPT_LION not in _GROUP_HYPER   # OptimHyper alone
    obj._kind = _lib.OPT_ADAM
    g = {"lr": 1e-3, "betas": (0.8, 0.9), "eps": 1e-7, "weight_decay": 0.0, "maximize": False}
    h = obj._hyper_of(g)
    assert (h.beta1, h.beta2, h.eps) == (0.8, 0.9, 1e-7)


def test_load_step_counts_for_lazy_lion_state():
    """A Lion state dict without an entry for a parameter (never stepped) puts step counts per parameter: 0 for it."""
    from stoke_b200.optim import load_step_counts

    entries = [{"step": torch.tensor(3.0), "exp_avg": torch.zeros(2)}, {}, {"step": torch.tensor(3.0), "exp_avg": torch.zeros(2)}]
    opt_steps, steps, scal = load_step_counts(_lib.OPT_LION, entries, [0, 0, 1], None, False)
    assert (opt_steps, steps, scal) == (3, [3, 0, 3], None)
    opt_steps, steps, scal = load_step_counts(_lib.OPT_LION, [entries[0], entries[2]], [0, 1], 3, False)
    assert (opt_steps, steps, scal) == (3, None, None)
