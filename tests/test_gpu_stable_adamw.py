"""StableAdamW on the fused layer-wise step (GPU).

Where the RMS clip does not engage (every parameter's RMS below 1), lr_t is exactly lr and the fused master, exp_avg,
exp_avg_sq and bf16 copy are bit-identical to the class's own step() on CUDA fp32 tensors with the same gradient.  Where
it engages, every element lies inside the float64 bounds of tests/stable_adamw_ref.py, restarted from the kernel's own
state, and the update is really smaller.  Also: found_inf and per-parameter skips, the gradient forms through Stoke
(accumulation, AMP loss scaling, both clips) against the stock route, NaN propagation, determinism, no host
synchronisation, and checkpoints carried through the fused step, the plain class and the stock route."""
import numpy as np
import pytest
import torch

import stable_adamw_ref as sr
from test_gpu_engine import OddNet, _inject, _rel
from test_gpu_layerwise import BIG, SMALL, Shapes, _spec

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _cls():
    from stoke_b200.optim import StableAdamW

    return StableAdamW


def _groups8(n):
    """8 groups over n parameters, alternating weight_decay == 0 and != 0, each with its own lr, betas and eps."""
    out = []
    for gi in range(8):
        extra = {"lr": 1e-2 * (1 + 0.25 * gi), "weight_decay": 0.0 if gi % 2 else 0.01 * (1 + gi),
                 "betas": (0.9 - 0.02 * gi, 0.99 - 0.001 * gi), "eps": 1e-6 if gi < 4 else 1e-8}
        out.append(([i for i in range(n) if i % 8 == gi], extra))
    return out


def _build(shapes, kw, lp, route, groups=None, clip=None):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    net = Shapes(shapes).cuda()
    kwargs = dict(kw)
    if groups is not None:
        ps = list(net.parameters())
        kwargs["params"] = [dict(extra, params=[ps[i] for i in idx]) for idx, extra in groups]
    opt = B200FusedOptimizer(net, _cls(), kwargs, engine=get_engine(0), clip=_spec(clip), lp_dtype=lp, route=route)
    assert opt.path.route == route
    return net, opt


def _hypers(path, kw, groups):
    hyp = [dict(kw)] * len(path.params)
    if groups is not None:
        for idx, extra in groups:
            for i in idx:
                hyp[i] = dict(kw, **extra)
    return hyp


def _base_grads(path, dtype, scale=1e-3):
    """Seeded gradients with every 64th element zero: at the first step each g^2 / v is 1 or 0, so the RMS is at most
    sqrt(63 / 64) < 1 - 1e-3."""
    out = []
    for i, gv in enumerate(path.grad_views):
        from stoke_b200 import synthetic

        g = synthetic.injected_grad(gv.numel(), 0, 100 + i, dtype=dtype, scale=scale).view(-1).clone()
        g[::64] = 0
        out.append(g.view(gv.shape))
    return out


def _write(path, grads):
    for gv, g in zip(path.grad_views, grads):
        gv.copy_(g.cuda())


def _views(path):
    w = [t.detach().cpu().clone() for t in path.unflatten(path.gather_master())]
    m = [t.cpu().clone() for t in path.unflatten(path.m_flat)]
    v = [t.cpu().clone() for t in path.unflatten(path.v_flat)]
    return w, m, v


def _bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    if a.dtype == torch.bfloat16:
        return torch.equal(a.view(torch.int16), b.view(torch.int16))
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _same(a, b):
    """Bit for bit; a NaN matches a NaN."""
    a, b = a.cpu(), b.cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def _fma(a, b, c):
    """fp32 fma(a, b, c) through float64: the product of two fp32 values is exact there."""
    return (a.double() * b.double() + c.double()).float()


def test_probe_cuda_rounding_of_the_class_ops():
    """What k_lw_tiles<STK_LW_STABLE_ADAMW> relies on, on this GPU: ``lerp_`` with a python weight w is
    FFMA(w, g - m, m) for w < 0.5 and FFMA(-(g - m), 1 - w, g) otherwise; ``mul_(b2).addcmul_(g, g, value=a)`` rounds
    v * b2 and g * g, then one FFMA(a, g * g, v * b2), which differs from K2's foreach form FFMA(a * g, g, v * b2);
    ``(g * g).div_(v.clamp(min=e))`` is IEEE."""
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(3)
    n = 1 << 16
    m = torch.randn(n, device="cuda", generator=gen) * 1e-3
    g = torch.randn(n, device="cuda", generator=gen) * 1e-3
    v = torch.rand(n, device="cuda", generator=gen) * 1e-6
    for b1 in (sr.debiased(0.9, 2), sr.debiased(0.9, 3), sr.debiased(0.8, 7)):
        w = torch.tensor(1 - b1, dtype=torch.float32, device="cuda")
        d = g - m
        want = _fma(w, d, m) if float(w) < 0.5 else _fma(-d, 1 - w, g)
        assert _same(m.clone().lerp_(g, 1 - b1), want), b1
    for b2 in (sr.debiased(0.99, 2), sr.debiased(0.99, 5), sr.debiased(0.95, 3)):
        a = torch.tensor(1 - b2, dtype=torch.float32, device="cuda")
        vb = v * torch.tensor(b2, dtype=torch.float32, device="cuda")
        got = v.clone().mul_(b2).addcmul_(g, g, value=1 - b2)
        assert _same(got, _fma(a, g * g, vb)), b2
        assert not _same(got, _fma(a * g, g, vb)), b2
    e2 = 1e-6 * 1e-6
    q = (g * g).div_(v.clamp(min=e2))
    assert _same(q, ((g * g).double() / v.clamp(min=e2).double()).float())


BITWISE = {
    "raw_bf16": (SMALL, {"lr": 1e-2, "weight_decay": 0.05}, torch.bfloat16, "local", None),
    "raw_f32_8groups": (SMALL * 2, {"lr": 1e-2}, None, "local", "g8"),
    "main_f32": (SMALL, {"lr": 5e-3, "weight_decay": 0.0, "eps": 1e-8}, None, "main", None),
    "raw_bf16_8groups": (SMALL * 2, {"lr": 1e-2}, torch.bfloat16, "local", "g8"),
    "raw_bf16_big": (BIG, {"lr": 1e-3}, torch.bfloat16, "local", None),
}


@pytest.mark.parametrize("name", list(BITWISE))
def test_bit_exact_where_the_clip_does_not_engage(name):
    """g_k = 0.5^(k-1) g_1 over four steps: every RMS stays below 1, so the fused step equals the class bit for bit.
    Step 2 takes lerp_'s weight >= 0.5 branch (1 - b1 ~ 0.53), the later steps the other one."""
    shapes, kw, lp, route, groups = BITWISE[name]
    groups = _groups8(len(shapes)) if groups == "g8" else None
    net, opt = _build(shapes, kw, lp, route, groups)
    path = opt.path
    hyp = _hypers(path, kw, groups)
    plain = [torch.nn.Parameter(w.cuda().clone()) for w in path.unflatten(path.gather_master())]
    if groups is None:
        topt = _cls()(plain, **kw)
    else:
        topt = _cls()([dict(extra, params=[plain[i] for i in idx]) for idx, extra in groups], **kw)
    base = _base_grads(path, lp or torch.float32)
    for step in range(4):
        grads = [g * 0.5**step for g in base]   # exact in bf16 and fp32
        state = None
        if step > 0:
            state = [{k: topt.state[p][k].cpu() for k in sr.KEYS} for p in plain]
        for i, (p, g) in enumerate(zip(plain, grads)):
            p.grad = g.float().cuda().reshape(p.shape)
            if state is not None:   # the premise: the clip does not engage
                assert sr.lr_t_of(state[i], p.grad.cpu(), step, hyp[i]) == hyp[i]["lr"]
        _write(path, grads)
        path.after_backward(sync=True, unscale=False)
        opt.step()
        topt.step()
        w, m, v = _views(path)
        for i, p in enumerate(plain):
            st = topt.state[p]
            assert _bits(w[i], p.detach().cpu()), (name, step, i)
            assert _bits(m[i], st["exp_avg"].cpu()), (name, step, i)
            assert _bits(v[i], st["exp_avg_sq"].cpu()), (name, step, i)
        if lp is not None:
            assert _bits(path.p_flat.cpu(), path.gather_master().cpu().to(lp))
        assert path.param_steps() == [step + 1] * len(path.params)
        assert float(path.g_flat.float().abs().max()) == 0.0
    opt.close()


def _check_bounds(path, hyp, grads, w0, m0, v0, steps0, stepped, tag):
    """Every stepped parameter inside the float64 bounds, restarted from the kernel's pre-step state; every other one
    unchanged.  Returns the stepped parameters' float64 lr_t."""
    w1, m1, v1 = _views(path)
    lrs = []
    for i, p in enumerate(path.params):
        if not stepped[i]:
            assert torch.equal(w1[i], w0[i]) and torch.equal(m1[i], m0[i]) and torch.equal(v1[i], v0[i]), (tag, i)
            continue
        G = grads[i].float().reshape(p.shape)
        state = {"exp_avg": m0[i], "exp_avg_sq": v0[i]} if steps0[i] > 0 else sr.zero_state(p.shape)
        rw, rst = sr.step_ref(w0[i], state, G, steps0[i], hyp[i])
        ew, est = sr.step_bound(w0[i], state, G, steps0[i], hyp[i], rw, rst)
        bad = sr.outside(w1[i], rw, ew)
        assert not bool(bad.any()), (tag, i, p.shape, torch.nonzero(bad.reshape(-1))[:5].flatten().tolist())
        assert not bool(sr.outside(m1[i], rst["exp_avg"], est["exp_avg"]).any()), (tag, i)
        assert not bool(sr.outside(v1[i], rst["exp_avg_sq"], est["exp_avg_sq"]).any()), (tag, i)
        lrs.append((i, sr.lr_t_of(state, G, steps0[i], hyp[i])))
    return lrs


@pytest.mark.parametrize("lp,route", [(torch.bfloat16, "local"), (None, "main")], ids=["raw_bf16", "main_f32"])
def test_bounds_where_the_clip_engages(lp, route):
    """Step 2 with g_2 = 3 g_1: RMS ~ 1.34 in every parameter.  Every element lies inside the float64 bounds, and the
    update is smaller than the one lr would have made."""
    shapes = SMALL * 2
    kw = {"lr": 1e-2}
    groups = _groups8(len(shapes))
    net, opt = _build(shapes, kw, lp, route, groups)
    path = opt.path
    hyp = _hypers(path, kw, groups)
    base = _base_grads(path, lp or torch.float32)
    for step, sc in enumerate([1.0, 3.0]):
        grads = [g * sc for g in base]
        w0, m0, v0 = _views(path)
        steps0 = path.param_steps()
        _write(path, grads)
        path.after_backward(sync=True, unscale=False)
        opt.step()
        lrs = _check_bounds(path, hyp, grads, w0, m0, v0, steps0, [True] * len(path.params), step)
        if step == 1:
            w1, m1, v1 = _views(path)
            for i, lr_t in lrs:
                assert lr_t < 0.8 * hyp[i]["lr"], (i, lr_t)
                h = sr.hyper(hyp[i])
                q = m1[i].double() / (v1[i].double().sqrt() + h["eps"])
                full = (w0[i].double() * h["lr"] * h["weight_decay"] + h["lr"] * q).abs().sum()
                assert float((w1[i].double() - w0[i].double()).abs().sum()) < 0.85 * float(full), i
    opt.close()


def test_found_inf_and_skipped_parameters_leave_state():
    """A parameter without a gradient keeps its master, state and count while the others step inside the bounds; an inf
    gradient under the loss scaler skips every parameter; per-parameter counts apply afterwards.  The raw bucket is
    zeroed in every case."""
    from stoke_b200.fp16 import DeviceGradScaler

    kw = {"lr": 1e-2}
    shapes = SMALL * 2
    groups = _groups8(len(shapes))
    net, opt = _build(shapes, kw, torch.bfloat16, "local", groups)
    path = opt.path
    hyp = _hypers(path, kw, groups)
    scaler = DeviceGradScaler(path.engine, init_scale=2.0**4, growth_interval=1000, state_id=path.state_id)
    for step, (skip, bad) in enumerate([((), False), ((1, 4, 9), False), ((), True), ((4,), False), ((), False)]):
        scale = scaler.get_scale()
        grads = _inject(path, step, 0, torch.bfloat16, scale=1e-3 * scale * (3.0 if step == 3 else 1.0))
        if bad:
            path.grad_views[2].view(-1)[5] = float("inf")
        path._track_touched = True
        path._touched = np.array([i not in skip for i in range(len(path.params))])
        w0, m0, v0 = _views(path)
        steps0 = path.param_steps()
        path.after_backward(sync=True, unscale=True)
        opt.step()
        stepped = [not bad and i not in skip for i in range(len(path.params))]
        grads = [g / scale for g in grads]   # exact: the scale is a power of two
        _check_bounds(path, hyp, grads, w0, m0, v0, steps0, stepped, step)
        assert path.param_steps() == [s + int(d) for s, d in zip(steps0, stepped)]
        assert float(path.g_flat.float().abs().max()) == 0.0
    assert path.param_steps()[1] == 3 and path.param_steps()[4] == 2 and path.param_steps()[0] == 4
    opt.close()


def test_nan_gradient_makes_only_its_parameter_nan():
    """fp32, no loss scaler, no clip: one NaN element makes its whole parameter NaN (the RMS is NaN and clamp keeps
    it), as the class does; the other parameters stay finite and equal the class bit for bit."""
    shapes = SMALL
    kw = {"lr": 1e-2, "weight_decay": 0.1}
    net, opt = _build(shapes, kw, None, "local")
    path = opt.path
    plain = [torch.nn.Parameter(w.cuda().clone()) for w in path.unflatten(path.gather_master())]
    topt = _cls()(plain, **kw)
    grads = _base_grads(path, torch.float32)
    grads[2].view(-1)[7] = float("nan")
    for p, g in zip(plain, grads):
        p.grad = g.cuda().reshape(p.shape)
    _write(path, grads)
    path.after_backward(sync=True, unscale=False)
    opt.step()
    topt.step()
    w, _, _ = _views(path)
    assert bool(plain[2].detach().isnan().all()) and bool(w[2].isnan().all())
    for i, p in enumerate(plain):
        if i != 2:
            assert bool(w[i].isfinite().all()) and _bits(w[i], p.detach().cpu()), i
    assert float(path.g_flat.float().abs().max()) == 0.0
    opt.close()


def test_deterministic_and_no_host_sync():
    """Two identical runs with the clip engaged give bit-identical masters, state and bf16 copies; a step runs under
    torch.cuda.set_sync_debug_mode("error")."""
    outs = []
    for _ in range(2):
        net, opt = _build(SMALL + BIG[:1], {"lr": 1e-2}, torch.bfloat16, "local", clip=("norm", 0.5))
        path = opt.path
        base = _base_grads(path, torch.bfloat16)
        for step, sc in enumerate([1.0, 3.0, 2.0]):
            _write(path, [g * sc for g in base])
            path.after_backward(sync=True, unscale=False)
            if step == 2:
                torch.cuda.synchronize()
                torch.cuda.set_sync_debug_mode("error")
                try:
                    opt.step()
                finally:
                    torch.cuda.set_sync_debug_mode("default")
            else:
                opt.step()
        outs.append((path.gather_master().cpu(), path.m_flat.cpu(), path.v_flat.cpu(), path.p_flat.cpu()))
        opt.close()
    for a, b in zip(*outs):
        assert _bits(a, b)


# ---- through Stoke ------------------------------------------------------------------------------------------------------
FACADE_KW = {"lr": 5e-3, "betas": (0.9, 0.99), "weight_decay": 0.02}


def _stoke(fp16, clip, accum, stock):
    import stoke_b200 as sb
    from test_gpu_adan import Net, _mse

    model = Net()
    used = [p for m in model.layers for p in m.parameters()]
    unused = dict(params=list(model.unused.parameters()), weight_decay=0.0)
    groups = [dict(params=[p]) for p in used] + [unused] if stock else [dict(params=used), unused]
    grad_clip = None
    if clip is not None:
        grad_clip = sb.ClipGradNormConfig(max_norm=clip[1], norm_type=2.0) if clip[0] == "norm" else \
            sb.ClipGradConfig(clip_value=clip[1])
    return sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=_cls(), optimizer_kwargs=dict(FACADE_KW,
                                                                                                     params=groups)),
                    loss=_mse, batch_size_per_device=8, grad_accum_steps=accum, grad_clip=grad_clip, gpu=True, fp16=fp16,
                    verbose=False)


@pytest.mark.parametrize("fp16,clip,accum", [(None, None, 2), ("amp", None, 1), ("amp", ("norm", 0.5), 2),
                                             ("bf16", ("norm", 0.5), 1), ("bf16", ("value", 0.05), 2),
                                             (None, ("value", 0.05), 1)])
def test_stoke_gradient_forms_match_the_stock_route(fp16, clip, accum):
    """Accumulated, loss-scaled and clipped gradients through Stoke: the fused step (2 groups) and the class's own step
    on the stock route (9 groups) agree within 1e-5 relative L2 on the master and both moments after 8 steps (the RMS
    sums add in different orders on the two routes); the unused Linear keeps its weights and has no state entry."""
    from test_gpu_adan import _drive
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    torch.cuda.set_device(0)
    runs = []
    for stock in (False, True):
        s = _stoke(fp16, clip, accum, stock)
        assert isinstance(s.optimizer, B200StockOptimizer if stock else B200FusedOptimizer)
        _drive(s, 8, fp16, accum)
        runs.append((s, s.optimizer.path.gather_master().cpu(), s.optimizer.state_dict()))
    (fs, fw, fsd), (ss, sw, ssd) = runs
    assert _rel(fw, sw) < TOL
    for i in range(8):
        assert list(fsd["state"][i]) == ["step", "exp_avg", "exp_avg_sq"] == list(ssd["state"][i])
        # AMP's scaler skips the steps whose scaled gradients overflow, on both routes alike
        assert float(fsd["state"][i]["step"]) == float(ssd["state"][i]["step"]) > 0
        for k in sr.KEYS:
            assert _rel(fsd["state"][i][k].cpu(), ssd["state"][i][k].cpu()) < TOL, (i, k)
    assert 8 not in fsd["state"] and 9 not in fsd["state"]
    for s in (fs, ss):
        s.optimizer.close()


# ---- checkpoints ------------------------------------------------------------------------------------------------------------
def _opt(net, kw, stock=False):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    return (B200StockOptimizer if stock else B200FusedOptimizer)(net, _cls(), kw, engine=get_engine(0))


def _ckpt_kw(net):
    ps = list(net.parameters())
    return dict(lr=1e-2, weight_decay=0.05, params=[dict(params=ps[:4]), dict(params=ps[4:], weight_decay=0.0,
                                                                               betas=(0.8, 0.95))])


def test_checkpoint_through_class_and_stock_route():
    """fused (4 steps) -> plain class on CUDA (4) -> stock route (4) -> fused (4) against the class's uninterrupted
    16-step run: the master within 1e-5 relative L2, state_dict in the class's format at every hand-over."""
    torch.cuda.set_device(0)
    net = OddNet().cuda()
    ref = [torch.nn.Parameter(p.detach().clone()) for p in net.parameters()]
    ropt = _cls()(**_ckpt_kw(torch.nn.ParameterList(ref)))
    a = _opt(net, _ckpt_kw(net))
    grads_of = {}

    def run(opt, steps, plain=None, popt=None):
        for step in steps:
            if opt is not None:
                grads_of[step] = _inject(opt.path, step, 0, torch.float32)
                opt.path.after_backward(sync=True, unscale=False)
                opt.step()
            else:
                for p, g in zip(plain, grads_of[step]):
                    p.grad = g.reshape(p.shape).cuda()
                popt.step()

    def fmt(sd, steps):
        for e in sd["state"].values():
            assert list(e) == ["step", "exp_avg", "exp_avg_sq"] and float(e["step"]) == steps
            assert e["step"].dtype == torch.float32 and e["step"].dim() == 0

    run(a, range(4))
    sd = a.state_dict()
    fmt(sd, 4)
    plain = [torch.nn.Parameter(w.cuda().clone()) for w in a.path.unflatten(a.path.gather_master())]
    popt = _cls()(**_ckpt_kw(torch.nn.ParameterList(plain)))
    popt.load_state_dict({k: v for k, v in sd.items() if not k.startswith("b200_")})
    for step in range(4, 8):
        grads_of[step] = _inject(a.path, step, 0, torch.float32)
    run(None, range(4, 8), plain, popt)
    fmt(popt.state_dict(), 8)
    a.close()
    net_b = OddNet().cuda()
    with torch.no_grad():
        for p, q in zip(net_b.parameters(), plain):
            p.copy_(q.detach())
    b = _opt(net_b, _ckpt_kw(net_b), stock=True)
    b.load_state_dict(popt.state_dict())
    run(b, range(8, 12))
    sd_b = b.state_dict()
    fmt(sd_b, 12)
    net_c = OddNet().cuda()
    with torch.no_grad():
        for p, q in zip(net_c.parameters(), b.path.unflatten(b.path.gather_master())):
            p.copy_(q)
    c = _opt(net_c, _ckpt_kw(net_c))
    c.load_state_dict(sd_b)
    run(c, range(12, 16))
    fmt(c.state_dict(), 16)
    run(None, range(16), ref, ropt)
    got = [t.reshape(-1) for t in c.path.unflatten(c.path.gather_master().cpu())]
    want = torch.cat([p.detach().cpu().reshape(-1) for p in ref])
    assert _rel(torch.cat(got), want) < TOL
    for o in (b, c):
        o.close()
