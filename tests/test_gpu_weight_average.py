"""Weight averaging (EMA / SWA) on the engine (GPU).

The reference throughout is torch.optim.swa_utils.AveragedModel (get_ema_multi_avg_fn, or the default equal average for
SWA) over an fp32 module whose parameters are clones of the engine's fp32 master after each step; "bit-identical" is
torch.equal on the bits.  Every optimizer route (the K2 kinds, Adafactor, LAMB / LARS, the stock route) is followed by
stk_weight_avg when an update is due.  Turning averaging on changes nothing else the step computes."""
import json
import os
import subprocess
import sys

import pytest
import torch
from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

import stoke_b200 as sb
from stoke_b200.weight_average import WeightAverage

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

OPTS = {
    "adam": (torch.optim.Adam, {"lr": 1e-2, "weight_decay": 0.01}),
    "adamw": (torch.optim.AdamW, {"lr": 1e-2, "weight_decay": 0.05}),
    "sgd": (torch.optim.SGD, {"lr": 0.05, "momentum": 0.9}),
    "nadam": (torch.optim.NAdam, {"lr": 1e-2}),
    "radam": (torch.optim.RAdam, {"lr": 1e-2}),
    "adamax": (torch.optim.Adamax, {"lr": 1e-2}),
    "adadelta": (torch.optim.Adadelta, {"lr": 1.0}),
    "rprop": (torch.optim.Rprop, {"lr": 1e-2}),
    "asgd": (torch.optim.ASGD, {"lr": 1e-2, "t0": 2}),
    "adafactor": (getattr(torch.optim, "Adafactor", None), {"lr": 1e-2}),
    "lamb": (sb.LAMB, {"lr": 1e-2}),
    "lars": (sb.LARS, {"lr": 0.5, "weight_decay": 1e-4}),
    "rmsprop": (torch.optim.RMSprop, {"lr": 1e-3}),   # no fused step: the stock route
}
# (kind, decay): 0.999 takes lerp's |w| < 0.5 branch, 0.3 the other; SWA takes both (w = 1/2, then 1/3, 1/4 ...)
AVGS = {"ema0.999": ("ema", 0.999), "ema0.3": ("ema", 0.3), "swa": ("swa", 0.0)}


def _bits(t):
    if not t.is_floating_point():
        return t.detach()
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _equal(a, b):
    return torch.equal(_bits(a), _bits(b))


class Net(torch.nn.Module):
    """Odd numels, and a parameter that never receives a gradient."""

    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(37, 29)
        self.b = torch.nn.Linear(29, 13)
        self.unused = torch.nn.Parameter(torch.randn(11))

    def forward(self, x):
        return self.b(torch.relu(self.a(x)))


class Reference:
    """AveragedModel over fp32 clones of the master, updated whenever the engine's average took an update."""

    def __init__(self, path, kind, decay):
        self.path = path
        self.holder = torch.nn.ParameterList([torch.nn.Parameter(v.clone()) for v in path.unflatten(path.gather_master())])
        self.avg = (AveragedModel(self.holder, multi_avg_fn=get_ema_multi_avg_fn(decay)) if kind == "ema"
                    else AveragedModel(self.holder))

    def update(self):
        with torch.no_grad():
            for p, v in zip(self.holder, self.path.unflatten(self.path.gather_master())):
                p.copy_(v)
        self.avg.update_parameters(self.holder)

    def check(self):
        got = self.path.unflatten(self.path.gather_avg())
        for a, r in zip(got, self.avg.module.parameters()):
            assert _equal(a, r)


def _build(name, lp):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer, fused_supported

    cls, kw = OPTS[name]
    if cls is None:
        pytest.skip("torch without Adafactor")
    torch.manual_seed(0)
    net = Net().cuda()
    kwargs = dict(kw, params=[{"params": [net.a.weight, net.b.weight, net.unused]},
                              {"params": [net.a.bias, net.b.bias], "lr": kw["lr"] * 0.5}])
    stock = not fused_supported(cls, kwargs, net)
    assert stock == (name == "rmsprop")
    opt_cls = B200StockOptimizer if stock else B200FusedOptimizer
    opt = opt_cls(net, cls, kwargs, engine=get_engine(0), clip=ClipSpec(_lib.CLIP_NORM, max_norm=0.5), lp_dtype=lp)
    return net, opt


def _state(opt):
    path = opt.path
    out = [path.gather_master(), path.p_flat.clone(), path.g_flat.clone()]
    out += [t.clone() for t in (path.m_flat, path.v_flat, getattr(path, "af_state", None)) if t is not None]
    inner = getattr(opt, "inner", None)
    if inner is not None:
        out += [v.clone() for st in inner.state.values() for v in st.values() if torch.is_tensor(v)]
    return out


def _run(name, lp, avg, steps=6, inf_step=4):
    """``steps`` optimizer steps from real backward passes; at ``inf_step`` the scaler reports an inf (the step is
    skipped, the average still moves toward the unchanged master)."""
    net, opt = _build(name, lp)
    path = opt.path
    wa = ref = None
    if avg is not None:
        kind, decay = AVGS[avg]
        wa = WeightAverage(sb.WeightAverageConfig(kind=kind, decay=decay), path, net)
        ref = Reference(path, kind, decay)
    g = torch.Generator(device="cuda").manual_seed(1)
    for step in range(1, steps + 1):
        x = torch.randn(16, 37, generator=g, device="cuda").to(lp or torch.float32)
        path.begin_backward(sync=True, unscale=False)
        net(x).float().pow(2).mean().backward()
        path.after_backward(sync=True, unscale=False)
        if step == inf_step:
            path.engine.scaler_set(state=path.state_id, found_inf=1)
        if wa is not None:
            wa._schedule(step)
        opt.step()
        if ref is not None:
            ref.update()
            ref.check()
    if wa is not None:
        assert wa.n_averaged == steps
    state = _state(opt)
    opt.close()
    return state


@pytest.mark.parametrize("avg", list(AVGS))
@pytest.mark.parametrize("lp", [torch.bfloat16, None], ids=["bf16", "fp32"])
@pytest.mark.parametrize("name", list(OPTS))
def test_average_matches_averaged_model_and_changes_nothing_else(name, lp, avg):
    with_avg = _run(name, lp, avg)
    without = _run(name, lp, None)
    assert len(with_avg) == len(without)
    for a, b in zip(with_avg, without):
        assert _equal(a, b)


def test_due_step_adds_no_host_sync():
    """A step with an update due (schedule included) runs under torch.cuda.set_sync_debug_mode("error").  Gradients are
    written into the bucket directly, so every parameter has one and no skip table is uploaded."""
    net, opt = _build("adam", torch.bfloat16)
    path = opt.path
    wa = WeightAverage(sb.WeightAverageConfig(decay=0.9), path, net)
    ref = Reference(path, "ema", 0.9)
    g = torch.Generator(device="cuda").manual_seed(2)
    for step in range(1, 4):
        for gv in path.grad_views:
            gv.copy_(torch.randn(gv.shape, generator=g, device="cuda") * 1e-2)
        path.after_backward(sync=True, unscale=False)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            wa._schedule(step)
            opt.step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        ref.update()
        ref.check()
    opt.close()


class SmallCNN(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 16, 3, padding=1, bias=False)
        self.bn = torch.nn.BatchNorm2d(16)
        self.fc = torch.nn.Linear(16, 10)

    def forward(self, x):
        return self.fc(torch.relu(self.bn(self.conv(x))).mean((2, 3)))


def _stoke(model, cfg, fp16="bf16", accum=1, opt=(torch.optim.Adam, {"lr": 1e-2})):
    return sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=opt[0], optimizer_kwargs=opt[1]),
                    loss=torch.nn.CrossEntropyLoss(), batch_size_per_device=8, grad_accum_steps=accum,
                    grad_clip=sb.ClipGradNormConfig(max_norm=1.0, norm_type=2.0), gpu=True, fp16=fp16,
                    configs=[cfg] if cfg is not None else None, verbose=False)


def _batch(i, n=8, hw=8):
    g = torch.Generator().manual_seed(100 + i)
    return torch.randn(n, 3, hw, hw, generator=g).cuda(), torch.randint(0, 10, (n,), generator=g).cuda()


def _micro(s, i):
    x, y = _batch(i)
    s.backward(s.loss(s.model(x), y))
    s.step()


def test_stoke_schedule_and_launches():
    """every=3, start_step=2, grad_accum=2: updates after optimizer steps 5 and 8 only; a micro-step launches what it
    launches without averaging, plus the one stk_weight_avg of a step with an update due; the average is
    AveragedModel's."""
    runs = {}
    for cfg in (None, sb.WeightAverageConfig(decay=0.9, every=3, start_step=2)):
        torch.manual_seed(0)
        s = _stoke(SmallCNN(), cfg, accum=2)
        ref = Reference(s.optimizer.path, "ema", 0.9) if cfg is not None else None
        launches, counts = [], []
        for i in range(20):
            before = s.engine.launches
            _micro(s, i)
            launches.append(s.engine.launches - before)
            if i % 2 == 1 and cfg is not None:
                counts.append(s.weight_average.n_averaged)
                if s.weight_average.n_averaged != (counts[-2] if len(counts) > 1 else 0):
                    ref.update()
                ref.check()
        runs[cfg is None] = (launches, counts, s.optimizer.path.gather_master())
        s.close()
    due_micro = {2 * 5 - 1, 2 * 8 - 1}   # the micro-steps that take optimizer steps 5 and 8
    assert runs[False][0] == [n + (i in due_micro) for i, n in enumerate(runs[True][0])]
    assert _equal(runs[True][2], runs[False][2])
    assert runs[False][1] == [0, 0, 0, 0, 1, 1, 1, 2, 2, 2]


@pytest.mark.parametrize("fp16", ["bf16", None])
@pytest.mark.parametrize("use_buffers", [True, False])
def test_applied_swaps_in_and_restores(fp16, use_buffers):
    torch.manual_seed(0)
    s = _stoke(SmallCNN(), sb.WeightAverageConfig(decay=0.5, use_buffers=use_buffers), fp16=fp16)
    for i in range(4):
        _micro(s, i)
    model, wa, path = s.model_access, s.weight_average, s.optimizer.path
    before = {k: v.detach().clone() for k, v in model.state_dict().items()}
    avg = wa.state_dict()
    with wa.applied():
        for name, p in model.named_parameters():
            assert _equal(p, avg[name].to(p.dtype))
        for name, b in model.named_buffers():
            expect = avg[name].to(b.dtype) if use_buffers else before[name]
            assert _equal(b, expect)
        if use_buffers:
            assert not _equal(model.bn.running_mean, before["bn.running_mean"])
        with pytest.raises(RuntimeError):
            s.backward(torch.zeros((), requires_grad=True, device="cuda"))
        with pytest.raises(RuntimeError):
            s.step()
        model.eval()
        s.model(_batch(9)[0])
        model.train()
    for k, v in model.state_dict().items():
        assert _equal(v, before[k]), k
    assert _equal(path.p_flat, path.master_flat.to(path.p_flat.dtype)) or path.master_flat is path.p_flat
    _micro(s, 5)   # training continues after the context
    s.close()


def test_state_dict_loads_into_plain_fp32_resnet18():
    import torchvision

    torch.manual_seed(0)
    s = _stoke(torchvision.models.resnet18(num_classes=10), sb.WeightAverageConfig(decay=0.9, use_buffers=True))
    for i in range(3):
        x, y = _batch(i, hw=32)
        s.backward(s.loss(s.model(x), y))
        s.step()
    sd = s.weight_average.state_dict()
    plain = torchvision.models.resnet18(num_classes=10)
    plain.load_state_dict(sd, strict=True)
    path = s.optimizer.path
    for p, v in zip(path.params, path.unflatten(path.gather_avg())):
        name = s.weight_average._name_of[id(p)]
        assert _equal(dict(plain.named_parameters())[name], v.cpu())
        assert sd[name].dtype == torch.float32
    assert _equal(plain.bn1.running_var, s.weight_average._buffers["bn1.running_var"].cpu())
    s.close()


def test_checkpoint_resume_is_bit_identical(tmp_path):
    """4 steps, save, load into a fresh Stoke, 4 more == 8 continuous, with the decay the loop set after step 2 restored
    from the checkpoint; a checkpoint without the key starts afresh."""
    cfg = sb.WeightAverageConfig(decay=0.9, use_buffers=True)

    torch.manual_seed(0)
    cont = _stoke(SmallCNN(), cfg)
    for i in range(8):
        if i == 2:
            cont.weight_average.decay = 0.7
        _micro(cont, i)
    want = cont.weight_average.state_dict()
    n_want = cont.weight_average.n_averaged
    cont.close()

    torch.manual_seed(0)
    first = _stoke(SmallCNN(), cfg)
    for i in range(4):
        if i == 2:
            first.weight_average.decay = 0.7
        _micro(first, i)
    out, tag = first.save(str(tmp_path), name="wa")
    first.close()
    torch.manual_seed(1)
    second = _stoke(SmallCNN(), cfg)
    second.load(out, tag)
    assert second.weight_average.n_averaged == 4 and second.weight_average.decay == 0.7
    for i in range(4, 8):
        _micro(second, i)
    got = second.weight_average.state_dict()
    assert second.weight_average.n_averaged == n_want
    assert set(got) == set(want)
    for k in want:
        assert _equal(got[k], want[k]), k
    second.close()

    torch.manual_seed(0)
    plain = _stoke(SmallCNN(), None)
    _micro(plain, 0)
    out, tag = plain.save(str(tmp_path), name="plain")
    assert "weight_average_state_dict" not in torch.load(f"{out}/{tag}", weights_only=False)
    plain.close()
    fresh = _stoke(SmallCNN(), cfg)
    _micro(fresh, 0)
    fresh.load(out, tag)
    assert fresh.weight_average.n_averaged == 0
    path = fresh.optimizer.path
    assert _equal(path.gather_avg(), path.gather_master())
    _micro(fresh, 1)
    assert fresh.weight_average.n_averaged == 1 and _equal(path.gather_avg(), path.gather_master())
    fresh.close()


def test_resnet50_bf16_channels_last_average_bit_identical():
    """ResNet-50, bf16 channels-last with its fused BatchNorm sites, Adam, clip 1.0, 5 steps."""
    from stoke_b200 import synthetic

    model = synthetic.resnet50().to(memory_format=torch.channels_last)
    s = _stoke(model, sb.WeightAverageConfig(decay=0.999), opt=(torch.optim.Adam, {"lr": 1e-3}))
    ref = Reference(s.optimizer.path, "ema", 0.999)
    x, y = synthetic.resnet50_batch(16, size=64)
    x, y = x.contiguous(memory_format=torch.channels_last).cuda(), y.cuda()
    for _ in range(5):
        s.backward(s.loss(s.model(x), y))
        s.step()
        ref.update()
    ref.check()
    assert s.weight_average.n_averaged == 5
    s.close()


def test_stoke_due_step_adds_no_host_sync():
    """Through Stoke: an optimizer step with an update due, the buffer average of use_buffers included, runs under
    torch.cuda.set_sync_debug_mode("error")."""
    torch.manual_seed(0)
    s = _stoke(SmallCNN(), sb.WeightAverageConfig(decay=0.9, use_buffers=True))
    ref = Reference(s.optimizer.path, "ema", 0.9)
    for i in range(4):
        x, y = _batch(i)
        s.backward(s.loss(s.model(x), y))
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error" if i > 0 else "default")
        try:
            s.step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        ref.update()
        ref.check()
    assert s.weight_average.n_averaged == 4
    s.close()


def test_amp_inf_step_averages_toward_unchanged_master():
    """fp16="amp": a step whose gradients are not finite is skipped by the scaler; the average still takes its update,
    toward the unchanged master, as AveragedModel does after a skipped scaler.step."""
    torch.manual_seed(0)
    s = _stoke(SmallCNN(), sb.WeightAverageConfig(decay=0.5), fp16="amp")
    path = s.optimizer.path
    ref = Reference(path, "ema", 0.5)
    for i in range(5):
        x, y = _batch(i)
        loss = s.loss(s.model(x), y)
        if i == 2:
            loss = loss * float("inf")
        before = path.gather_master()
        s.backward(loss)
        s.step()
        if i == 2:
            assert _equal(path.gather_master(), before)
        ref.update()
        ref.check()
    assert s.engine.scaler_get(path.state_id).skipped_steps == 1
    assert s.weight_average.n_averaged == 5
    s.close()


@pytest.mark.multigpu
def test_sharded_and_allreduce_routes_w2(tmp_path):
    """W = 2, sharded and all-reduce routes: the gathered average equals AveragedModel over the gathered master after
    every step; state_dict() on every rank, applied() and its restore of P, checkpoint load (tests/
    weight_average_mgpu_worker.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "weight_average_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29571", os.path.join(ROOT, "tests", "weight_average_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    res = json.loads(out.read_text())
    for route in ("sharded", "allreduce"):
        r = res[route]
        assert r["route"] == route, r
        assert r["n_local"] < r["n"] if route == "sharded" else r["n_local"] == r["n"], r
        assert all(r[k] for k in ("avg_each_step", "state_dict", "applied", "restored", "load")), (route, r)
