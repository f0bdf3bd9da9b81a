"""stoke_b200.AdamW8bit / Adam8bit on the fused step (GPU).

Rounding probe: the CUDA ops the class relies on (sqrt, reciprocal) against correctly rounded fp32.  Engine level: the
fused step (``stk_adam8bit_step``) against the class's ``step()`` on CUDA fp32 tensors, bit for bit over several steps:
master, codes, absmax, the fp32 state of the parameters below min_8bit_size and the step counts, on the raw bf16 route,
the raw fp32 route with an accumulator and the main route, with clip by norm and by value and a NaN gradient; an fp16
AMP step the scaler skips and per-parameter skips; the weight average; a step without host synchronisation; a
checkpoint carried fused -> class -> stock route -> fused; no fp32 moment buffers.  The W = 2 replicated route is
covered by tests/optim8bit_mgpu_worker.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same(a, b):
    """Bit for bit; a NaN matches a NaN."""
    a, b = a.detach().cpu(), b.detach().cpu()
    if a.dtype == torch.uint8:
        return torch.equal(a, b)
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def test_probe_cuda_rounding():
    """The class's sqrt (``_sqrt_rn``) and torch's CUDA sqrt and reciprocal are correctly rounded fp32, as the kernel's
    __fsqrt_rn and __frcp_rn are."""
    from stoke_b200.optim import _sqrt_rn

    torch.cuda.set_device(0)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.rand(1 << 20, device="cuda", generator=g) * torch.logspace(-30, 30, 1 << 20, device="cuda")
    cr = x.double().sqrt().float()
    assert _same(x.sqrt(), cr) and _same(_sqrt_rn(x), cr)
    assert _same(x.reciprocal(), (1 / x.double()).float())


class Shapes(torch.nn.Module):
    def __init__(self, shapes, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        ps = []
        for s, cl in shapes:
            t = torch.randn(s, generator=g) * 0.1
            if cl:
                t = t.contiguous(memory_format=torch.channels_last)
            ps.append(torch.nn.Parameter(t))
        self.ps = torch.nn.ParameterList(ps)


# a channels-last conv weight, parameters below / at / above min_8bit_size (4096), a short last block (21000 = 82 blocks
# + 8), small parameters whose numel is not a multiple of 16
SHAPES = [((64, 32, 3, 3), True), ((1000,), False), ((37, 23), False), ((4095,), False), ((4096,), False),
          ((4097,), False), ((300, 70), False), ((3, 5, 7), False)]
GROUPS = [([0, 2, 4, 6], dict(weight_decay=0.01)), ([1, 3, 5, 7], dict(lr=3e-3, betas=(0.8, 0.99), weight_decay=0.0))]
KW = dict(lr=1e-2)


def _kwargs(net, kw=KW, groups=GROUPS):
    ps = list(net.parameters())
    return dict(kw, params=[dict(extra, params=[ps[i] for i in idx]) for idx, extra in groups])


def _spec(clip):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec

    if clip is None:
        return None
    if clip[0] == "norm":
        return ClipSpec(_lib.CLIP_NORM, max_norm=clip[1], norm_type=2.0)
    return ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1])


def _fused(net, lp, route, accum=1, clip=None, cls=None, groups=GROUPS):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import AdamW8bit, B200FusedOptimizer

    opt = B200FusedOptimizer(net, cls or AdamW8bit, _kwargs(net, groups=groups), engine=get_engine(0), grad_accum=accum,
                             clip=_spec(clip), lp_dtype=lp, route=route)
    assert opt.path.route == route
    return opt


def _reference(path, cls=None, groups=GROUPS):
    """The class on CUDA fp32 copies of the master, laid out like the parameters (channels-last kept)."""
    from stoke_b200.optim import AdamW8bit

    ref = [torch.nn.Parameter(torch.empty_like(v).copy_(v)) for v in path.unflatten(path.gather_master())]
    return ref, (cls or AdamW8bit)([dict(KW, **extra, params=[ref[i] for i in idx]) for idx, extra in groups])


def _inject(path, step, dtype, scale=1.0):
    from stoke_b200 import synthetic

    out = []
    for i, gv in enumerate(path.grad_views):
        g = synthetic.injected_grad(gv.numel(), 0, step * 100 + i, dtype=dtype, scale=scale).view(gv.shape)
        gv.copy_(g.cuda())
        out.append(g.float().cuda())
    return out


def _clip(grads, clip, path):
    """The gradient the kernel forms: clip_grad_norm_'s coefficient from the engine's norm, or the value clamp."""
    if clip is None:
        return grads
    if clip[0] == "value":
        return [g.clamp(-clip[1], clip[1]) for g in grads]
    norm = np.float32(path.engine.scaler_get(path.state_id).grad_norm)
    coef = min(np.float32(clip[1]) / (norm + np.float32(1e-6)), np.float32(1.0))
    return [g * torch.tensor(coef, dtype=torch.float32, device="cuda") for g in grads]


def _check(path, ref, ropt, tag):
    """Master, codes, absmax, fp32 state and counts of the fused step against the class, bit for bit."""
    for i, (a, b) in enumerate(zip(path.unflatten(path.gather_master()), ref)):
        assert _same(a, b), (tag, "master", i)
    steps = path.param_steps()
    for i, (views, p) in enumerate(zip(path.adam8bit_state_views(), ref)):
        st = ropt.state.get(p, {})
        if not st:
            assert steps[i] == 0, (tag, i)
            continue
        assert steps[i] == int(st["step"]), (tag, "step", i)
        assert set(views) == set(st) - {"step"}, (tag, i)
        for k, v in views.items():
            assert v.dtype == st[k].dtype and v.shape == st[k].shape, (tag, k, i)
            assert _same(v, st[k]), (tag, k, i)


ROUTES = [
    ("raw-bf16", torch.bfloat16, "local", 1, None),
    ("raw-fp32-acc2", None, "local", 2, ("value", 0.02)),
    ("main", torch.bfloat16, "main", 1, ("norm", 1.0)),
    ("raw-bf16-clipnorm", torch.bfloat16, "local", 1, ("norm", 0.5)),
]


@pytest.mark.parametrize("name,lp,route,accum,clip", ROUTES, ids=[r[0] for r in ROUTES])
def test_fused_matches_class(name, lp, route, accum, clip):
    torch.cuda.set_device(0)
    net = Shapes(SHAPES).cuda()
    opt = _fused(net, lp, route, accum, clip)
    path = opt.path
    ref, ropt = _reference(path)
    for step in range(6):
        grads = None
        for micro in range(accum):
            g = _inject(path, step * accum + micro, lp or torch.float32, scale=1e-2)
            if name == "raw-fp32-acc2" and step == 3 and micro == accum - 1:
                path.grad_views[6].view(-1)[300] = float("nan")   # clip by value passes it through: block 1 goes NaN
                g[6].view(-1)[300] = float("nan")
            grads = g if grads is None else [a + b for a, b in zip(g, grads)]
            path.after_backward(sync=(micro == accum - 1), unscale=False)
        opt.step()
        for p, g in zip(ref, _clip(grads, clip, path)):
            p.grad = g
        ropt.step()
        _check(path, ref, ropt, (name, step))
        assert float(path.g_flat.float().abs().max()) == 0.0   # the raw bucket is consumed
        if lp is not None:
            assert torch.equal(path.p_flat, path.gather_master().to(lp))
    if name == "raw-fp32-acc2":
        assert bool(torch.isnan(path.adam8bit_state_views()[6]["absmax1"][1]))
    opt.close()


def test_adam8bit_class_on_the_fused_step():
    from stoke_b200.optim import Adam8bit

    torch.cuda.set_device(0)
    groups = [(list(range(8)), {})]
    net = Shapes(SHAPES).cuda()
    opt = _fused(net, torch.bfloat16, "local", cls=Adam8bit, groups=groups)
    ref, ropt = _reference(opt.path, cls=Adam8bit, groups=groups)
    assert opt.param_groups[0]["weight_decay"] == 0.0
    for step in range(3):
        grads = _inject(opt.path, step, torch.bfloat16, scale=1e-2)
        opt.path.after_backward(sync=True, unscale=False)
        opt.step()
        for p, g in zip(ref, grads):
            p.grad = g
        ropt.step()
        _check(opt.path, ref, ropt, step)
    opt.close()


def test_skipped_steps_and_parameters():
    """fp16 AMP (fp32 model, loss scaler): an inf gradient skips every parameter and a parameter without a gradient is
    skipped alone -- codes, absmax, fp32 state, master and count stay as they are -- and the raw bucket is zeroed either
    way; the other parameters step as the class does."""
    from stoke_b200.fp16 import DeviceGradScaler

    torch.cuda.set_device(0)
    net = Shapes(SHAPES).cuda()
    opt = _fused(net, None, "local")
    path = opt.path
    ref, ropt = _reference(path)
    scaler = DeviceGradScaler(path.engine, init_scale=2.0**4, growth_interval=1000, state_id=path.state_id)
    for step, (skip, bad) in enumerate([((), False), ((1, 4, 6), False), ((), True), ((4,), False), ((), False)]):
        scale = scaler.get_scale()
        grads = _inject(path, step, torch.float32, scale=1e-2 * scale)
        if bad:
            path.grad_views[2].view(-1)[5] = float("inf")
        path._track_touched = True
        path._touched = np.array([i not in skip for i in range(len(path.params))])
        before = [{k: v.clone() for k, v in d.items()} for d in path.adam8bit_state_views()]
        master0 = path.gather_master()
        path.after_backward(sync=True, unscale=True)
        opt.step()
        assert float(path.g_flat.float().abs().max()) == 0.0
        if bad:
            assert torch.equal(path.gather_master(), master0)
            for d0, d1 in zip(before, path.adam8bit_state_views()):
                assert all(_same(d0[k], d1[k]) for k in d0)
        else:
            for i, p in enumerate(ref):
                p.grad = None if i in skip else grads[i] * torch.tensor(np.float32(1.0 / scale), device="cuda")
            ropt.step()
            for i in skip:
                assert all(_same(before[i][k], v) for k, v in path.adam8bit_state_views()[i].items())
        _check(path, ref, ropt, step)
    opt.close()


def test_weight_average_after_the_step():
    from stoke_b200.weight_average import LERP

    torch.cuda.set_device(0)
    net = Shapes(SHAPES).cuda()
    opt = _fused(net, torch.bfloat16, "local")
    path = opt.path
    path.enable_weight_average()
    avg = path.gather_master()
    for step in range(3):
        _inject(path, step, torch.bfloat16, scale=1e-2)
        path.after_backward(sync=True, unscale=False)
        path.avg_due = (LERP, float(np.float32(0.1)))
        opt.step()
        avg = torch.lerp(avg, path.gather_master(), float(np.float32(0.1)))
        assert _same(path.gather_avg(), avg)
    opt.close()


def test_deterministic_and_no_host_sync():
    outs = []
    for _ in range(2):
        torch.cuda.set_device(0)
        net = Shapes(SHAPES).cuda()
        opt = _fused(net, torch.bfloat16, "local", clip=("norm", 0.5))
        path = opt.path
        for step in range(3):
            _inject(path, step, torch.bfloat16, scale=1e-2)
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
        outs.append((path.gather_master(), path.q8_code1.clone(), path.q8_code2.clone(), path.q8_absmax1.clone(),
                     path.q8_absmax2.clone(), path.q8_small.clone(), path.p_flat.float()))
        opt.close()
    for a, b in zip(*outs):
        assert _same(a, b)


def test_no_fp32_moment_buffers():
    torch.cuda.set_device(0)
    net = Shapes(SHAPES).cuda()
    opt = _fused(net, torch.bfloat16, "local")
    path = opt.path
    assert path.M is None and path.V is None and path.M2 is None and path.M3 is None
    assert path.m_flat is None and path.v_flat is None
    assert path.q8_code1.dtype == torch.uint8 and path.q8_code1.numel() == path.n
    small = sum(p.numel() for p in path.params if p.numel() < 4096)
    assert 2 * small <= path.q8_small.numel() < 2 * small + 16 * 2 * len(path.params)
    assert path.q8_absmax1.numel() == sum(-(-p.numel() // 256) for p in path.params)
    opt.close()


def test_checkpoint_fused_class_stock_fused():
    """A run carried through four owners -- fused step, the plain class, the stock route (B200StockOptimizer running the
    class on the fp32 masters), fused step again -- ends bit-identical to the class alone."""
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import AdamW8bit, B200StockOptimizer

    torch.cuda.set_device(0)
    net = Shapes(SHAPES).cuda()
    opt = _fused(net, None, "local")
    ref, ropt = _reference(opt.path)

    def ref_step(grads):
        for p, g in zip(ref, grads):
            p.grad = g
        ropt.step()

    def path_step(o, step):
        grads = _inject(o.path, step, torch.float32, scale=1e-2)
        o.path.after_backward(sync=True, unscale=False)
        o.step()
        ref_step(grads)
        return grads

    for step in range(3):
        path_step(opt, step)
    sd = opt.state_dict()
    assert all(torch.is_tensor(st["step"]) and st["step"].dtype == torch.float32 for st in sd["state"].values())
    # fused -> class
    cls_params = [torch.nn.Parameter(torch.empty_like(v).copy_(v)) for v in opt.path.unflatten(opt.path.gather_master())]
    copt = AdamW8bit([dict(KW, **extra, params=[cls_params[i] for i in idx]) for idx, extra in GROUPS])
    copt.load_state_dict({k: v for k, v in sd.items() if not k.startswith("b200_")})
    opt.close()
    for step in range(3, 5):
        grads = [torch.randn(p.shape, generator=torch.Generator().manual_seed(step * 10 + i)).cuda() * 1e-2
                 for i, p in enumerate(cls_params)]
        for p, g in zip(cls_params, grads):
            p.grad = g.clone()
        copt.step()
        ref_step(grads)
    # class -> stock route (9 groups would pick it; built directly here), the model weights loaded first
    net2 = Shapes(SHAPES).cuda()
    with torch.no_grad():
        for p, q in zip(net2.parameters(), cls_params):
            p.copy_(q)
    stock = B200StockOptimizer(net2, AdamW8bit, _kwargs(net2), engine=get_engine(0))
    stock.load_state_dict(copt.state_dict())
    for step in range(5, 7):
        path_step(stock, step)
    sd3 = stock.state_dict()
    # stock -> fused
    net3 = Shapes(SHAPES).cuda()
    opt3 = _fused(net3, None, "local")
    opt3.load_state_dict(sd3)
    stock.close()
    for step in range(7, 9):
        path_step(opt3, step)
    _check(opt3.path, ref, ropt, "final")
    opt3.close()


@pytest.mark.multigpu
def test_replicated_matches_world1_w2(tmp_path):
    """W = 2 with fairscale_oss asked for: the 8-bit state is replicated on the all-reduce route, both replicas are
    bit-identical and equal to the class stepping on the mean gradient."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "optim8bit_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29583", os.path.join(ROOT, "tests", "optim8bit_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    assert res["route"] == "allreduce" and res["replicas_identical"] and res["matches_world1"], res
