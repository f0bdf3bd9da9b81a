"""LAMB, LARS and Adafactor at the edges of their per-parameter scalars, element by element (GPU).

The trust ratio of LAMB / LARS (k_lw_fold) and Adafactor's alpha and update clip (k_af_prologue, k_af_coef) each have a
second branch that random weights and gradients never reach:
  * all-zero weights (BatchNorm biases start at zero; zero_init_residual zeroes a BatchNorm weight in every ResNet block):
    ||w|| = 0 gives LAMB / LARS a trust ratio of 1 and Adafactor alpha = eps2 * rho, with weight decay and (LAMB / LARS)
    with always_adapt and no weight decay;
  * an all-zero gradient window on a parameter that is still stepped: LARS's ||g|| = 0 gives a trust ratio of 1 (also at
    the first step, which seeds the momentum buffer), LAMB's r comes from its moments and wd * w, Adafactor's u = 0 so
    max(1, 0) = 1 and only the weight decay acts;
  * one NaN or +inf gradient element without a loss scaler, under no clip and clip by value: a NaN norm gives a trust
    ratio of 1 (torch.where), an inf one 0 (LARS), Adafactor's max(1, NaN) is 1.  The element sits in the last, partial
    tile of a multi-tile parameter, in a parameter of one element, or in one of five (padding inside one vector).
Every element of every parameter is checked against the float64 references (tests/layerwise_ref.py,
tests/adafactor_ref.py: the classes' and torch's own semantics) restarted from the kernel's own state each step, on the
raw bf16 route and the main fp32 route.  NaN patterns must match exactly and the other parameters stay finite."""
import pytest
import torch

import adafactor_ref as ar
import layerwise_ref as lr_
from test_gpu_engine import _inject
from test_gpu_layerwise import _state_views

pytestmark = pytest.mark.gpu

# 0: three tiles of 8192, the last partial; 1: one element; 2: five elements; 3-4: ordinary; 5, 6: all-zero weights;
# 7, 8: all-zero gradient windows
SHAPES = [((20000,), False), ((1,), False), ((5,), False), ((37, 23), False), ((16, 8, 3, 3), True), ((300,), False),
          ((7, 9), False), ((40, 50), False), ((33,), False)]
GROUP1 = [1, 3, 6, 8]
ZERO_W = (5, 6)
ZERO_G = (7, 8)
SPECIAL_AT = {"last_tile": (0, 20000 - 3), "numel1": (1, 0), "numel5": (2, 4)}

HYPER = {   # (first group, second group's overrides)
    "lamb": ({"lr": 1e-2, "weight_decay": 0.01}, {"lr": 5e-3, "weight_decay": 0.0, "always_adapt": True}),
    "lars": ({"lr": 0.5, "weight_decay": 5e-4}, {"lr": 0.2, "weight_decay": 0.0, "always_adapt": True}),
    "adafactor": ({"lr": 1e-2, "weight_decay": 0.1}, {"lr": 5e-3, "weight_decay": 0.0, "eps": (None, 1e-2)}),
}
ROUTES = {"raw_bf16": (torch.bfloat16, "local"), "main_f32": (None, "main")}


class Shapes(torch.nn.Module):
    def __init__(self, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        ps = []
        for i, (s, cl) in enumerate(SHAPES):
            t = torch.randn(s, generator=g) * 0.1
            if i in ZERO_W:
                t.zero_()
            if cl:
                t = t.contiguous(memory_format=torch.channels_last)
            ps.append(torch.nn.Parameter(t))
        self.ps = torch.nn.ParameterList(ps)


def _hyp(kind, i):
    base, extra = HYPER[kind]
    return dict(base, **extra) if i in GROUP1 else dict(base)


def _build(kind, route, clip):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import LAMB, LARS, B200FusedOptimizer

    lp, r = ROUTES[route]
    cls = {"lamb": LAMB, "lars": LARS, "adafactor": torch.optim.Adafactor}[kind]
    torch.cuda.set_device(0)
    net = Shapes().cuda()
    ps = list(net.parameters())
    base, extra = HYPER[kind]
    kw = dict(base, params=[{"params": [p for i, p in enumerate(ps) if i not in GROUP1]},
                            dict(extra, params=[ps[i] for i in GROUP1])])
    spec = ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1]) if clip is not None else None
    opt = B200FusedOptimizer(net, cls, kw, engine=get_engine(0), clip=spec, lp_dtype=lp, route=r)
    assert opt.path.route == r
    return opt, lp


def _states(kind, path):
    if kind == "adafactor":
        views = [tuple(v.cpu().clone() for v in vs) for vs in path.adafactor_state_views()]
        return [dict(zip(ar.state_keys(p.shape), vs)) for p, vs in zip(path.params, views)]
    views = _state_views(kind, path)
    return [{k: views[k][i] for k in views} for i in range(len(path.params))]


def _outside(got, ref, bound):
    """layerwise_ref.outside, and an element equal to its reference (an infinity in the state) is inside."""
    return lr_.outside(got, ref, bound) & ~(got.double() == ref.double())


def _check(kind, path, grads, clip, w0, s0, steps0, special, tag):
    w1 = [t.detach().cpu() for t in path.unflatten(path.gather_master())]
    s1 = _states(kind, path)
    for i, p in enumerate(path.params):
        G = grads[i].float().reshape(p.shape)
        if clip is not None:
            G = G.clamp(-clip[1], clip[1])
        h = _hyp(kind, i)
        if kind == "adafactor":
            rw, rst = ar.step_ref(w0[i], s0[i], G, steps0[i], h)
            ew, est = ar.step_bound(w0[i], s0[i], G, steps0[i], h, rw, rst)
            keys = ar.state_keys(p.shape)
        else:
            keys = lr_.state_keys(kind, h)
            state = {k: s0[i][k] for k in keys} if steps0[i] > 0 else lr_.zero_state(kind, p.shape, h)
            rw, rst = lr_.step_ref(kind, w0[i], state, G, steps0[i], h)
            ew, est = lr_.step_bound(kind, w0[i], state, G, steps0[i], h, rw, rst)
        assert torch.equal(w1[i].isnan(), rw.isnan()), (tag, i, "NaN pattern", int(w1[i].isnan().sum()),
                                                        int(rw.isnan().sum()))
        bad = _outside(w1[i], rw, ew)
        assert not bool(bad.any()), (tag, i, p.shape, torch.nonzero(bad.reshape(-1))[:5].flatten().tolist())
        for k in keys:
            assert torch.equal(s1[i][k].isnan(), rst[k].isnan()), (tag, i, k, "NaN pattern")
            assert not bool(_outside(s1[i][k], rst[k], est[k]).any()), (tag, i, k)
        if special is None or i != special[0]:
            assert bool(torch.isfinite(w1[i]).all()), (tag, i, "a parameter without the special element")


def _step(kind, opt, lp, step, clip, special, tag):
    path = opt.path
    grads = _inject(path, step, 0, lp or torch.float32, scale=1e-3)
    for i in ZERO_G:   # a whole window of zeros on a parameter that still steps
        grads[i].zero_()
        path.grad_views[i].zero_()
    if special is not None:
        (i, e), val = SPECIAL_AT[special[0]], special[1]
        grads[i].view(-1)[e] = val
        path.grad_views[i].view(-1)[e] = val
    w0 = [t.detach().cpu().clone() for t in path.unflatten(path.gather_master())]
    s0 = _states(kind, path)
    steps0 = path.param_steps()
    path.after_backward(sync=True, unscale=False)
    opt.step()
    _check(kind, path, grads, clip, w0, s0, steps0, None if special is None else SPECIAL_AT[special[0]], tag)
    assert path.param_steps() == [s + 1 for s in steps0], tag
    if lp is not None:   # the low-precision copy is the master rounded, a NaN element a NaN
        got, want = path.p_flat.cpu(), path.gather_master().cpu().to(lp)
        assert torch.equal(got.isnan(), want.isnan()), tag
        assert torch.equal(got[~got.isnan()], want[~want.isnan()]), tag
    assert float(path.g_flat.float().abs().max()) == 0.0, tag


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("kind", list(HYPER))
def test_zero_weights_and_zero_gradient_windows(kind, route):
    """Steps 1-3: parameters 5 and 6 start at zero weights (one with weight decay, one without: always_adapt for LAMB /
    LARS); 7 and 8 get an all-zero gradient every step, from the first (LARS: the momentum buffer is seeded with 0)."""
    opt, lp = _build(kind, route, None)
    try:
        w = [t.cpu() for t in opt.path.unflatten(opt.path.gather_master())]
        assert all(float(w[i].abs().max()) == 0.0 for i in ZERO_W)
        for step in range(3):
            _step(kind, opt, lp, step, None, None, (kind, route, step))
        if kind == "adafactor":   # no gradient, so only the weight decay moved parameter 7 (group 0); 8 stays put
            w1 = [t.cpu() for t in opt.path.unflatten(opt.path.gather_master())]
            assert bool(((w1[7].abs() < w[7].abs()) | (w[7] == 0)).all())
            assert torch.equal(w1[8], w[8])
    finally:
        opt.close()


SPECIAL_CASES = [(k, r, v, c, at) for k in HYPER for r in ROUTES for v in ("nan", "inf") for c in ("none", "value")
                 for at in SPECIAL_AT]


@pytest.mark.parametrize("kind,route,value,clip,at", SPECIAL_CASES,
                         ids=["-".join(c) for c in SPECIAL_CASES])
def test_one_nonfinite_gradient_element(kind, route, value, clip, at):
    """Two ordinary steps, then one whose gradient has a single NaN / +inf element (no loss scaler: the step runs)."""
    clip_ = ("value", 2e-3) if clip == "value" else None
    opt, lp = _build(kind, route, clip_)
    try:
        for step in range(3):
            special = (at, float(value)) if step == 2 else None
            _step(kind, opt, lp, step, clip_, special, (kind, route, value, clip, at, step))
        w1 = [t.cpu() for t in opt.path.unflatten(opt.path.gather_master())]
        i = SPECIAL_AT[at][0]
        # the element reaches its parameter's weights unless the clip by value turned it finite (+inf)
        assert bool(torch.isfinite(w1[i]).all()) == (value == "inf" and clip == "value"), (kind, route, value, clip, at)
    finally:
        opt.close()
