"""stoke_b200.Lion8bit and AdEMAMix8bit on the fused step (GPU).

The fused steps (``stk_lion8bit_step``, ``stk_ademamix8bit_step``) against the class's ``step()`` on CUDA fp32 tensors,
bit for bit after every step: master, codes, absmax, the fp32 state of the parameters below min_8bit_size and the step
counts.  On the raw bf16 route, the raw fp32 route with an accumulator and the main route; with clip by norm and by
value, a NaN gradient, an fp16 loss-scaler skip and per-parameter skips; AdEMAMix through its alpha and beta3 warm-ups;
at the quantizer's edges (an all-zero block, subnormal absmax, an inf gradient, n beyond a loaded map); two runs
bit-identical and without host synchronisation; a checkpoint carried fused -> class -> stock route -> fused; the
``Stoke`` facade in bf16; the weight average on top.  The W = 2 replicated route is covered by
tests/optim8bit_more_mgpu_worker.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import optim8bit_edges_ref as er
from test_gpu_optim8bit import SHAPES, Shapes, _clip, _inject, _same, _spec

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(lr=1e-2)
# two groups; AdEMAMix's first is inside both warm-ups for the first steps
GROUPS = {"Lion8bit": [([0, 2, 4, 6], dict(weight_decay=0.01)), ([1, 3, 5, 7], dict(lr=3e-3, betas=(0.8, 0.99)))],
          "AdEMAMix8bit": [([0, 2, 4, 6], dict(weight_decay=0.01, alpha_warmup=4, beta3_warmup=3)),
                           ([1, 3, 5, 7], dict(lr=3e-3, betas=(0.8, 0.99, 0.999), alpha=5.0, eps=1e-6))]}
NAMES = sorted(GROUPS)


def _cls(name):
    from stoke_b200 import optim

    return getattr(optim, name)


def _kwargs(net, groups):
    ps = list(net.parameters())
    return dict(KW, params=[dict(extra, params=[ps[i] for i in idx]) for idx, extra in groups])


def _fused(name, net, lp, route, accum=1, clip=None, groups=None):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer

    opt = B200FusedOptimizer(net, _cls(name), _kwargs(net, groups or GROUPS[name]), engine=get_engine(0),
                             grad_accum=accum, clip=_spec(clip), lp_dtype=lp, route=route)
    assert opt.path.route == route
    return opt


def _reference(name, path, groups=None):
    """The class on CUDA fp32 copies of the master, laid out like the parameters (channels-last kept)."""
    ref = [torch.nn.Parameter(torch.empty_like(v).copy_(v)) for v in path.unflatten(path.gather_master())]
    return ref, _cls(name)([dict(KW, **extra, params=[ref[i] for i in idx]) for idx, extra in groups or GROUPS[name]])


def _check(path, ref, ropt, tag):
    """Master, codes, absmax, fp32 state and counts of the fused step against the class, bit for bit."""
    for i, (a, b) in enumerate(zip(path.unflatten(path.gather_master()), ref)):
        assert _same(a, b), (tag, "master", i)
    steps = path.param_steps()
    for i, (views, p) in enumerate(zip(path.q8_state_views(), ref)):
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


@pytest.mark.parametrize("route_case", ROUTES, ids=[r[0] for r in ROUTES])
@pytest.mark.parametrize("name", NAMES)
def test_fused_matches_class(name, route_case):
    route_name, lp, route, accum, clip = route_case
    torch.cuda.set_device(0)
    net = Shapes(SHAPES).cuda()
    opt = _fused(name, net, lp, route, accum, clip)
    path = opt.path
    ref, ropt = _reference(name, path)
    for step in range(6):
        grads = None
        for micro in range(accum):
            g = _inject(path, step * accum + micro, lp or torch.float32, scale=1e-2)
            if route_name == "raw-fp32-acc2" and step == 3 and micro == accum - 1:
                path.grad_views[6].view(-1)[300] = float("nan")   # clip by value passes it through
                g[6].view(-1)[300] = float("nan")
            grads = g if grads is None else [a + b for a, b in zip(g, grads)]
            path.after_backward(sync=(micro == accum - 1), unscale=False)
        opt.step()
        for p, g in zip(ref, _clip(grads, clip, path)):
            p.grad = g
        ropt.step()
        _check(path, ref, ropt, (route_name, step))
        assert float(path.g_flat.float().abs().max()) == 0.0   # the raw bucket is consumed
        if lp is not None:
            assert torch.equal(path.p_flat, path.gather_master().to(lp))
    if route_name == "raw-fp32-acc2":
        assert bool(torch.isnan(path.q8_state_views()[6]["absmax1"].reshape(-1, path.q8_state_views()[6]["absmax1"]
                                                                             .shape[-1])[:, 1]).any())
    opt.close()


@pytest.mark.parametrize("name", NAMES)
def test_state_buffers(name):
    """Only the buffers the kind needs: codes per state, absmax per block and state, the compact fp32 buffer sized by
    the number of states; no fp32 moment buffers."""
    torch.cuda.set_device(0)
    net = Shapes(SHAPES).cuda()
    opt = _fused(name, net, torch.bfloat16, "local")
    path = opt.path
    states = 1 if name == "Lion8bit" else 3
    assert path.M is None and path.V is None and path.M2 is None and path.M3 is None
    assert path.q8_code1.numel() == path.n and path.q8_codes.numel() == (2 if states == 3 else 1) * path.n
    assert (path.q8_code2 is None) == (states == 1) and (path.q8_code3 is None) == (states != 3)
    assert (path.q8_qmap2 is None) == (states == 1)
    small = sum(p.numel() for p in path.params if p.numel() < 4096)
    assert states * small <= path.q8_small.numel() < states * (small + 16 * len(path.params))
    assert path.q8_absmax1.numel() == sum(-(-p.numel() // 256) for p in path.params)
    opt.close()


@pytest.mark.parametrize("name", NAMES)
def test_skipped_steps_and_parameters(name):
    """fp16 AMP (fp32 model, loss scaler): an inf gradient skips every parameter and a parameter without a gradient is
    skipped alone -- codes, absmax, fp32 state, master and count stay as they are -- and the raw bucket is zeroed either
    way; the other parameters step as the class does."""
    from stoke_b200.fp16 import DeviceGradScaler

    torch.cuda.set_device(0)
    net = Shapes(SHAPES).cuda()
    opt = _fused(name, net, None, "local")
    path = opt.path
    ref, ropt = _reference(name, path)
    scaler = DeviceGradScaler(path.engine, init_scale=2.0**4, growth_interval=1000, state_id=path.state_id)
    for step, (skip, bad) in enumerate([((), False), ((1, 4, 6), False), ((), True), ((4,), False), ((), False)]):
        scale = scaler.get_scale()
        grads = _inject(path, step, torch.float32, scale=1e-2 * scale)
        if bad:
            path.grad_views[2].view(-1)[5] = float("inf")
        path._track_touched = True
        path._touched = np.array([i not in skip for i in range(len(path.params))])
        before = [{k: v.clone() for k, v in d.items()} for d in path.q8_state_views()]
        master0 = path.gather_master()
        path.after_backward(sync=True, unscale=True)
        opt.step()
        assert float(path.g_flat.float().abs().max()) == 0.0
        if bad:
            assert torch.equal(path.gather_master(), master0)
            for d0, d1 in zip(before, path.q8_state_views()):
                assert all(_same(d0[k], d1[k]) for k in d0)
        else:
            for i, p in enumerate(ref):
                p.grad = None if i in skip else grads[i] * torch.tensor(np.float32(1.0 / scale), device="cuda")
            ropt.step()
            for i in skip:
                assert all(_same(before[i][k], v) for k, v in path.q8_state_views()[i].items())
        _check(path, ref, ropt, step)
    opt.close()


# ---- the quantizer's edges ----------------------------------------------------------------------------------------------
def _pad(b):
    return np.pad(b, (0, er.BLOCK - b.size))


def _other_maps():
    """A signed map and an unsigned one that both top out below 1, their two top entries 2 ** -25 apart (n = 1 is
    equally far from both in fp32): n = 1 lies beyond the map."""
    q1 = torch.cat([torch.linspace(-1, 0.25, 255, dtype=torch.float32), torch.tensor([0.25 + 2.0 ** -25])])
    q2 = torch.linspace(2.0 ** -10, 0.25, 255, dtype=torch.float32)
    q2 = torch.cat([q2, torch.tensor([0.25 + 2.0 ** -25])])
    for q in (q1, q2):
        assert bool((q[1:] > q[:-1]).all()) and float(q[-1]) - float(q[-2]) == 2.0 ** -25
    return q1, q2


@pytest.mark.parametrize("name", NAMES)
def test_quantizer_edges(name):
    """fp32 model on the raw route, the class beside it, bit for bit after every step:
    step 0: an all-zero block (absmax 0, every code the code of 0);
    step 1: blocks of subnormal absmax (1 / absmax overflows, n = +-inf) and an inf gradient (its block's absmax inf);
    step 2: the inf block decodes to NaN (AdEMAMix's weights there go NaN, Lion's stay: sign(NaN) = 0); then maps from a class checkpoint that top out below 1, so n = 1 lies beyond
    them and takes code 255, on crafted and random gradients."""
    torch.cuda.set_device(0)
    shapes = [((4096,), False), ((4096 + 100,), False), ((1000,), False)]
    groups = [([0, 1, 2], {})]
    net = Shapes(shapes).cuda()
    opt = _fused(name, net, None, "local", groups=groups)
    path = opt.path
    ref, ropt = _reference(name, path, groups)
    rng = np.random.default_rng(7)
    sub = np.concatenate([_pad(er.subnormal_block(a)) for _, a in er.SUBNORMAL_ABSMAX])
    for step in range(6):
        if step == 3:
            q1, q2 = _other_maps()
            sd = ropt.state_dict()
            maps = dict(qmap1=q1.cuda()) if name == "Lion8bit" else dict(qmap1=q1.cuda(), qmap2=q2.cuda())
            ck = {"state": {k: dict(v, **maps) if "qmap1" in v else dict(v) for k, v in sd["state"].items()},
                  "param_groups": sd["param_groups"]}
            ropt.load_state_dict(ck)
            opt.load_state_dict(ck)
            assert torch.equal(path.q8_qmap1.cpu(), q1)
            _check(path, ref, ropt, "loaded")
        g0 = (rng.standard_normal(4096) * 1e-2).astype(np.float32)
        if step == 0:
            g0[er.BLOCK: 2 * er.BLOCK] = 0
        elif step in (1, 4):
            g0[: sub.size] = sub
        g1 = (rng.standard_normal(4196) * 1e-2).astype(np.float32)
        if step == 1:
            g1[2 * er.BLOCK + 7] = np.inf
        g2 = (rng.standard_normal(1000) * 1e-2).astype(np.float32)
        grads = [torch.from_numpy(g).cuda() for g in (g0, g1, g2)]
        for gv, g in zip(path.grad_views, grads):
            gv.copy_(g)
        path.after_backward(sync=True, unscale=False)
        opt.step()
        for p, g in zip(ref, grads):
            p.grad = g
        ropt.step()
        _check(path, ref, ropt, (name, step))
        v0, v1 = path.q8_state_views()[0], path.q8_state_views()[1]
        a0 = v0["absmax1"].reshape(-1, v0["absmax1"].shape[-1])[0]
        codes0 = v0["state1"].reshape(-1, 4096)[0]
        if step == 0:
            assert float(a0[1]) == 0.0 and bool((codes0[er.BLOCK: 2 * er.BLOCK] == 127).all())
        if step == 1:
            assert er.overflows(a0.cpu().numpy()).any()
            assert float(v1["absmax1"].reshape(-1, v1["absmax1"].shape[-1])[0, 2]) == float("inf")
        if step == 2:   # the inf block decoded to NaN: its new absmax is NaN
            assert torch.isnan(v1["absmax1"].reshape(-1, v1["absmax1"].shape[-1])[0, 2])
            w1 = path.unflatten(path.gather_master())[1]
            if name == "AdEMAMix8bit":
                assert bool(torch.isnan(w1[2 * er.BLOCK: 3 * er.BLOCK]).all())
            else:   # Lion: sign(NaN) = 0 leaves those weights where they were
                assert not bool(torch.isnan(w1).any())
        if step >= 3:
            assert bool((path.q8_code1 == 255).any())
    opt.close()


@pytest.mark.parametrize("name", NAMES)
def test_deterministic_and_no_host_sync(name):
    outs = []
    for _ in range(2):
        torch.cuda.set_device(0)
        net = Shapes(SHAPES).cuda()
        opt = _fused(name, net, torch.bfloat16, "local", clip=("norm", 0.5))
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
        outs.append([path.gather_master(), path.q8_codes.clone(), path.q8_absmaxes.clone(), path.q8_small.clone(),
                     path.p_flat.float()] + ([path.q8_code2.clone(), path.q8_absmax2.clone()]
                                             if path.q8_code2 is not None else []))
        opt.close()
    for a, b in zip(*outs):
        assert _same(a, b)


@pytest.mark.parametrize("name", NAMES)
def test_weight_average_after_the_step(name):
    from stoke_b200.weight_average import LERP

    torch.cuda.set_device(0)
    net = Shapes(SHAPES).cuda()
    opt = _fused(name, net, torch.bfloat16, "local")
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


@pytest.mark.parametrize("name", NAMES)
def test_checkpoint_fused_class_stock_fused(name):
    """A run carried through four owners -- fused step, the plain class, the stock route (B200StockOptimizer running the
    class on the fp32 masters), fused step again -- ends bit-identical to the class alone."""
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200StockOptimizer

    torch.cuda.set_device(0)
    groups = GROUPS[name]
    net = Shapes(SHAPES).cuda()
    opt = _fused(name, net, None, "local")
    ref, ropt = _reference(name, opt.path)

    def ref_step(grads):
        for p, g in zip(ref, grads):
            p.grad = g
        ropt.step()

    def path_step(o, step):
        grads = _inject(o.path, step, torch.float32, scale=1e-2)
        o.path.after_backward(sync=True, unscale=False)
        o.step()
        ref_step(grads)

    for step in range(3):
        path_step(opt, step)
    sd = opt.state_dict()
    assert all(torch.is_tensor(st["step"]) and st["step"].dtype == torch.float32 for st in sd["state"].values())
    # fused -> class
    cls_params = [torch.nn.Parameter(torch.empty_like(v).copy_(v)) for v in opt.path.unflatten(opt.path.gather_master())]
    copt = _cls(name)([dict(KW, **extra, params=[cls_params[i] for i in idx]) for idx, extra in groups])
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
    stock = B200StockOptimizer(net2, _cls(name), _kwargs(net2, groups), engine=get_engine(0))
    stock.load_state_dict(copt.state_dict())
    for step in range(5, 7):
        path_step(stock, step)
    sd3 = stock.state_dict()
    # stock -> fused
    net3 = Shapes(SHAPES).cuda()
    opt3 = _fused(name, net3, None, "local")
    opt3.load_state_dict(sd3)
    stock.close()
    for step in range(7, 9):
        path_step(opt3, step)
    _check(opt3.path, ref, ropt, "final")
    opt3.close()


class TwoHeads(torch.nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(3)
        self.body = torch.nn.Linear(16, 24)
        self.a = torch.nn.Linear(24, 1)
        self.b = torch.nn.Linear(24, 1)
        self.use_b = True

    def forward(self, x):
        h = torch.tanh(self.body(x))
        return self.a(h) + (self.b(h) if self.use_b else 0.0)


@pytest.mark.parametrize("name", NAMES)
def test_stoke_facade_bf16(name):
    """Through the public Stoke calls in bf16: the class is routed to its fused step, head b receives no gradient on some
    steps (its count stays behind), and master and state follow the class stepping on the same bf16 gradients, bit for
    bit."""
    import stoke_b200 as sb
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    model = TwoHeads()
    kw = dict(lr=5e-3, weight_decay=0.1, min_8bit_size=64)
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=_cls(name), optimizer_kwargs=kw),
                 loss=lambda out, y: (out.float() - y).pow(2).mean(), batch_size_per_device=8, gpu=True, fp16="bf16",
                 verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    path = s.optimizer.path
    assert path.q8_quantized == [True, False, False, False, False, False]   # body.weight: 384 elements
    ref = [torch.nn.Parameter(torch.empty_like(v).copy_(v)) for v in path.unflatten(path.gather_master())]
    ropt = _cls(name)(ref, **kw)
    g = torch.Generator().manual_seed(0)
    x, y = torch.randn(8, 16, generator=g).cuda().bfloat16(), torch.randn(8, 1, generator=g).cuda()
    losses = []
    for step in range(8):
        model.use_b = step % 3 != 1
        loss = s.loss(s.model(x), y)
        grads = torch.autograd.grad(loss, path.params, retain_graph=True, allow_unused=True)
        s.backward(loss)
        s.step()
        for p, gr in zip(ref, grads):
            p.grad = None if gr is None else gr.detach().float()
        ropt.step()
        losses.append(float(loss.detach()))
        _check(path, ref, ropt, ("facade", step))
    assert torch.equal(path.p_flat, path.gather_master().to(torch.bfloat16))
    assert path.param_steps() == [8, 8, 8, 8, 5, 5]
    assert losses[-1] < losses[0]
    s.optimizer.close()


@pytest.mark.multigpu
@pytest.mark.parametrize("name", NAMES)
def test_replicated_matches_world1_w2(tmp_path, name):
    """W = 2 with fairscale_oss asked for: the 8-bit state is replicated on the all-reduce route, both replicas are
    bit-identical and equal to the class stepping on the mean gradient."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "optim8bit_more_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29587", os.path.join(ROOT, "tests", "optim8bit_more_mgpu_worker.py"), name, str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    res = json.loads(out.read_text())
    assert res["route"] == "allreduce" and res["replicas_identical"] and res["matches_world1"], res
