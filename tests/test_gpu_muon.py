"""torch.optim.Muon and MuonWithAuxAdamW on the fused sm_90a Muon step (GPU).

* Newton-Schulz: the kernel's bf16 iteration, torch's ``_zeropower_via_newtonschulz`` on CUDA (cuBLAS) and a float64
  run, all on the same normalised bf16 input: the kernel's distance to float64 is at most twice cuBLAS's plus 2^-10
  (a chosen tolerance, not a measured one), on square, wide, tall (transposed), non-tile-multiple, 1 x n and
  30522 x 768 matrices.
* Given the kernel's own bf16 X, the momentum buffers and the masters are bit-identical to the class's operations on
  CUDA fp32, on the raw bf16 route and the fp32 main route; the AdamW half is bit-identical to the fused AdamW step.
* found_inf and per-parameter skips; clip by norm and by value, accumulation, AMP loss scaling and unused parameters
  through Stoke against the stock route; determinism and no host synchronisation; checkpoints carried fused -> class ->
  stock -> fused, and plain torch.optim.Muon state dicts; a ResNet-50 and a BERT training through Stoke in bf16.
* The W = 2 replicated route is covered by tests/muon_mgpu_worker.py (needs two GPUs)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import muon_ref as mr
from test_gpu_engine import _inject, _rel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Mats(torch.nn.Module):
    def __init__(self, shapes, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.w = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(s, generator=g) * 0.05) for s in shapes])


def _fused(net, kw, lp=None, route=None, clip=None, cls=None):
    from stoke_b200 import MuonWithAuxAdamW
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    opt = B200FusedOptimizer(net, cls or MuonWithAuxAdamW, kw, engine=get_engine(0), lp_dtype=lp, route=route,
                             clip=clip)
    if route is not None:
        assert opt.path.route == route
    return opt


def _bits(a, b):
    a, b = a.detach().contiguous().cpu(), b.detach().contiguous().cpu()
    if a.dtype == torch.bfloat16:
        return torch.equal(a.view(torch.int16), b.view(torch.int16))
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- Newton-Schulz -------------------------------------------------------------------------------------------------------
NS_SHAPES = {"square": (256, 256), "wide": (128, 320), "tall": (300, 100), "odd": (70, 130), "row": (1, 257),
             "embedding": (30522, 768)}


@pytest.mark.parametrize("name", list(NS_SHAPES))
def test_newton_schulz_against_float64(name):
    """momentum 0 and no nesterov make u = g; g is a bf16 matrix whose norm rounds to 1 in bf16, so the kernel's and
    torch's normalisations both leave it as it is and all three computations start from the same input."""
    from torch.optim._muon import _zeropower_via_newtonschulz

    R, C = NS_SHAPES[name]
    net = Mats([(R, C)]).cuda()
    kw = {"params": [dict(params=list(net.parameters()), use_muon=True, momentum=0.0, nesterov=False)]}
    opt = _fused(net, kw)
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(min(R, C), max(R, C), device="cuda", generator=gen, dtype=torch.float64)
    x = (x / x.norm()).bfloat16()
    assert float(x.norm().clamp(min=1e-7)) == 1.0
    g = x.T if R > C else x
    path = opt.path
    path.grad_views[0].copy_(g.float())
    path.after_backward(sync=True, unscale=False)
    opt.step()
    fused = path.muon_x_views([5])[0].double()
    cub = _zeropower_via_newtonschulz(g, mr.COEFFS, 5, 1e-7)
    cub = (cub.T if R > C else cub).double()
    o64 = mr.ns64(x.double(), mr.COEFFS, 5)
    e_fused = float((fused - o64).norm() / o64.norm())
    e_cublas = float((cub - o64).norm() / o64.norm())
    assert e_fused <= 2 * e_cublas + 2 ** -10, (name, e_fused, e_cublas)
    opt.close()


# ---- the bit-exact parts -------------------------------------------------------------------------------------------------
SHAPES = [(64, 96), (96, 64), (8, 4, 3, 3), (33, 70), (1, 40), (100, 1), (96,), (33,)]
MUON_GROUPS = [dict(lr=0.02, weight_decay=0.1, momentum=0.95, nesterov=True, ns_steps=5),
               dict(lr=0.01, weight_decay=0.0, momentum=0.9, nesterov=False, ns_steps=4, adjust_lr_fn="match_rms_adamw")]
AUX = dict(lr=1e-2, weight_decay=0.01, betas=(0.9, 0.99))


def _aux_kw(net):
    ps = list(net.parameters())
    return {"params": [dict(params=ps[0:6:2], use_muon=True, **MUON_GROUPS[0]),
                       dict(params=ps[1:6:2], use_muon=True, **MUON_GROUPS[1]),
                       dict(params=ps[6:], use_muon=False, **AUX)]}


def _ns_steps(opt):
    return [g.get("ns_steps", 0) for g in opt.param_groups]


@pytest.mark.parametrize("lp,route", [(torch.bfloat16, "local"), (None, "main")], ids=["raw_bf16", "main_f32"])
def test_bit_exact_given_the_kernels_x(lp, route):
    """Three steps: the momentum buffers equal buf.lerp_(g, 1 - momentum) bit for bit, and the masters equal
    w.mul_(1 - lr wd).add_(X, alpha=-lr ratio) on CUDA fp32 with the kernel's X; that X is Newton-Schulz of u to within
    bf16 error; the bf16 copy is the master's cast; the raw bucket is zero."""
    from torch.optim._muon import _zeropower_via_newtonschulz

    from stoke_b200.optim import muon_lr_ratio

    net = Mats(SHAPES).cuda()
    opt = _fused(net, _aux_kw(net), lp, route)
    path = opt.path
    groups = opt.param_groups
    ws = [w.clone() for w in path.unflatten(path.gather_master())]
    bufs = [torch.zeros_like(w) for w in ws]
    for step in range(3):
        grads = _inject(path, step, 0, lp or torch.float32, scale=1e-2)
        path.after_backward(sync=True, unscale=False)
        opt.step()
        xs = path.muon_x_views(_ns_steps(opt))
        master = path.unflatten(path.gather_master())
        mom = path.unflatten(path.m_flat)
        for k, i in enumerate(path.mu_index):
            gp = groups[path.group_of[i]]
            g = grads[i].cuda()
            bufs[i].lerp_(g, 1 - gp["momentum"])
            assert _bits(mom[i], bufs[i]), (step, i)
            R = ws[i].shape[0]
            w2 = ws[i].view(R, -1)
            x = xs[k].T if R > w2.shape[1] else xs[k]
            w2.mul_(1 - gp["lr"] * gp["weight_decay"])
            w2.add_(x, alpha=-(gp["lr"] * muon_lr_ratio(gp.get("adjust_lr_fn"), R, w2.shape[1])))
            assert _bits(master[i], ws[i]), (step, i)
            u = g.lerp(bufs[i], gp["momentum"]) if gp["nesterov"] else bufs[i]
            want = _zeropower_via_newtonschulz(u.view(R, -1), mr.COEFFS, gp["ns_steps"], 1e-7).float()
            assert _rel(x.float(), want) < 0.05, (step, i)
        for i in range(6, 8):
            ws[i] = master[i].clone()
        if lp is not None:
            assert _bits(path.p_flat, path.gather_master().to(lp))
        assert float(path.g_flat.float().abs().max()) == 0.0
    assert path.param_steps() == [3] * len(SHAPES)
    opt.close()


def test_adamw_half_equals_the_fused_adamw_step():
    """The AdamW groups of MuonWithAuxAdamW (K2 with the Muon parameters skipped through the range table) against the
    fused torch.optim.AdamW step over the same parameters alone: master, exp_avg, exp_avg_sq and step counts bit for bit
    over three bf16 steps."""
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer

    net = Mats(SHAPES).cuda()
    aux = Mats(SHAPES[6:]).cuda()
    with torch.no_grad():
        for p, q in zip(aux.parameters(), list(net.parameters())[6:]):
            p.copy_(q)
    opt = _fused(net, _aux_kw(net), torch.bfloat16, "local")
    ref = B200FusedOptimizer(aux, torch.optim.AdamW, dict(AUX), engine=get_engine(0), lp_dtype=torch.bfloat16)
    for step in range(3):
        grads = _inject(opt.path, step, 0, torch.bfloat16, scale=1e-2)
        for gv, g in zip(ref.path.grad_views, grads[6:]):
            gv.copy_(g.to(torch.bfloat16).cuda())
        for o in (opt, ref):
            o.path.after_backward(sync=True, unscale=False)
            o.step()
        a, b = opt.path, ref.path
        for x, y in ((a.gather_master(), b.gather_master()), (a.m_flat, b.m_flat), (a.v_flat, b.v_flat)):
            for u, v in zip(a.unflatten(x)[6:], b.unflatten(y)):
                assert _bits(u, v), step
        assert a.param_steps()[6:] == b.param_steps() == [step + 1] * 2
    for o in (opt, ref):
        o.close()


def test_found_inf_and_skipped_parameters():
    """A parameter without a gradient keeps its master, state and count; an inf gradient under the loss scaler skips
    every parameter; the raw bucket is zeroed every time."""
    from stoke_b200.fp16 import DeviceGradScaler

    net = Mats(SHAPES).cuda()
    opt = _fused(net, _aux_kw(net), torch.bfloat16, "local")
    path = opt.path
    scaler = DeviceGradScaler(path.engine, init_scale=2.0 ** 4, growth_interval=1000, state_id=path.state_id)
    for step, (skip, bad) in enumerate([((), False), ((0, 3, 7), False), ((), True), ((3,), False)]):
        w0 = [t.clone() for t in path.unflatten(path.gather_master())]
        m0 = [t.clone() for t in path.unflatten(path.m_flat)]
        steps0 = path.param_steps()
        _inject(path, step, 0, torch.bfloat16, scale=1e-3 * scaler.get_scale())
        if bad:
            path.grad_views[1].view(-1)[5] = float("inf")
        path._track_touched = True
        path._touched = np.array([i not in skip for i in range(len(SHAPES))])
        path.after_backward(sync=True, unscale=True)
        opt.step()
        w1, m1 = path.unflatten(path.gather_master()), path.unflatten(path.m_flat)
        stepped = [not bad and i not in skip for i in range(len(SHAPES))]
        for i, s in enumerate(stepped):
            assert torch.equal(w1[i], w0[i]) != s and torch.equal(m1[i], m0[i]) != s, (step, i)
        assert path.param_steps() == [a + int(s) for a, s in zip(steps0, stepped)]
        assert float(path.g_flat.float().abs().max()) == 0.0
    assert path.param_steps()[0] == 2 and path.param_steps()[3] == 1 and path.param_steps()[1] == 3
    sd = opt.state_dict()
    assert list(sd["state"][0]) == ["momentum_buffer"] and list(sd["state"][6]) == ["step", "exp_avg", "exp_avg_sq"]
    opt.close()


def test_deterministic_and_no_host_sync():
    """Two identical runs give bit-identical masters, state and bf16 copies; a step runs under
    torch.cuda.set_sync_debug_mode("error")."""
    from stoke_b200.engine import ClipSpec
    from stoke_b200 import _lib

    outs = []
    for _ in range(2):
        net = Mats(SHAPES).cuda()
        opt = _fused(net, _aux_kw(net), torch.bfloat16, "local", clip=ClipSpec(_lib.CLIP_NORM, max_norm=0.05))
        path = opt.path
        for step in range(3):
            _inject(path, step, 0, torch.bfloat16, scale=1e-2)
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
        outs.append((path.gather_master().cpu(), path.m_flat.cpu(), path.v_flat.cpu(), path.p_flat.cpu(),
                     path.mu_x.cpu()))
        opt.close()
    for a, b in zip(*outs):
        assert _bits(a, b)


# ---- through Stoke ------------------------------------------------------------------------------------------------------
MK = dict(lr=0.02, weight_decay=0.01)
AK = dict(lr=5e-3, weight_decay=0.02)


def _stoke(fp16, clip, accum, stock):
    import stoke_b200 as sb
    from test_gpu_adan import Net, _mse

    model = Net()
    ws, bs = [m.weight for m in model.layers], [m.bias for m in model.layers]
    uw = [dict(params=[model.unused.weight], use_muon=True, **MK), dict(params=[model.unused.bias], use_muon=False, **AK)]
    if stock:   # 10 groups: more than the fused step takes
        groups = [dict(params=[p], use_muon=p.ndim > 1, **(MK if p.ndim > 1 else AK)) for p in ws + bs] + uw
    else:
        groups = [dict(params=ws, use_muon=True, **MK), dict(params=bs, use_muon=False, **AK)] + uw
    grad_clip = None
    if clip is not None:
        grad_clip = sb.ClipGradNormConfig(max_norm=clip[1], norm_type=2.0) if clip[0] == "norm" else \
            sb.ClipGradConfig(clip_value=clip[1])
    return sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=sb.MuonWithAuxAdamW,
                                                             optimizer_kwargs={"params": groups}),
                    loss=_mse, batch_size_per_device=8, grad_accum_steps=accum, grad_clip=grad_clip, gpu=True, fp16=fp16,
                    verbose=False)


@pytest.mark.parametrize("fp16,clip,accum,inf_at", [(None, None, 2, None), ("amp", None, 1, 3),
                                                    ("amp", ("norm", 0.5), 2, None), ("bf16", ("norm", 0.5), 1, None),
                                                    ("bf16", ("value", 0.05), 2, None), (None, ("value", 0.05), 1, None)])
def test_stoke_gradient_forms_match_the_stock_route(fp16, clip, accum, inf_at):
    """Accumulated, loss-scaled (one overflowing step skipped) and clipped gradients through Stoke: the fused step
    (4 groups) and the class's own step on the stock route (10 groups) after 8 steps.  Newton-Schulz output does not
    change when every gradient is scaled alike, so the momentum buffers, which do, are compared as well as the weights.
    The two routes' Newton-Schulz round differently in bf16 (each within its tested distance of float64), and the
    forward feeds that back for 8 steps: the used parameters' displacement, momentum buffers and exp_avg agree within
    10 %.  State entries are in the class's format; the fused route has none for the unused Linear and leaves its
    weights as they are (the stock route's masters always carry a gradient, zero for an unused parameter)."""
    from test_gpu_adan import _drive

    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    torch.cuda.set_device(0)
    runs = []
    for stock in (False, True):
        s = _stoke(fp16, clip, accum, stock)
        assert isinstance(s.optimizer, B200StockOptimizer if stock else B200FusedOptimizer)
        w0 = s.optimizer.path.gather_master().cpu()
        _drive(s, 8, fp16, accum, inf_at=inf_at)
        runs.append((s, w0, s.optimizer.path.gather_master().cpu(), s.optimizer.state_dict()))
    (fs, fw0, fw, fsd), (ss, sw0, sw, ssd) = runs
    assert torch.equal(fw0, sw0)
    path = fs.optimizer.path
    used = slice(0, path.offsets[8])   # the 8 parameters in use come first in the flat layout
    assert _rel(fw[used] - fw0[used], sw[used] - sw0[used]) < 0.1
    assert sorted(fsd["state"]) == list(range(8))
    for i in range(8):
        want = ["momentum_buffer"] if i < 4 else ["step", "exp_avg", "exp_avg_sq"]
        assert list(fsd["state"][i]) == want == list(ssd["state"][i]), i
        key = "momentum_buffer" if i < 4 else "exp_avg"
        assert _rel(fsd["state"][i][key].cpu(), ssd["state"][i][key].cpu()) < 0.1, i
        if i >= 4:
            assert float(fsd["state"][i]["step"]) == float(ssd["state"][i]["step"]) == 8 - (inf_at is not None)
    assert all(torch.equal(a, b) for a, b in zip(path.unflatten(fw)[8:], path.unflatten(fw0)[8:]))
    for s in (fs, ss):
        s.optimizer.close()


# ---- checkpoints ------------------------------------------------------------------------------------------------------------
def test_checkpoint_through_class_and_stock_route():
    """fused (3 steps) -> plain class on CUDA (3) -> stock route (3) -> fused (3) against the class's uninterrupted
    12-step run: the displacement within 3 %; state_dict in the class's format at every hand-over."""
    from stoke_b200 import MuonWithAuxAdamW
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200StockOptimizer

    torch.cuda.set_device(0)
    net = Mats(SHAPES).cuda()
    w_init = [p.detach().clone() for p in net.parameters()]
    ref = [torch.nn.Parameter(p.detach().clone()) for p in net.parameters()]
    ropt = MuonWithAuxAdamW(**_aux_kw(torch.nn.ParameterList(ref)))
    grads_of = {}

    def run(opt, steps, plain=None, popt=None):
        for step in steps:
            if opt is not None:
                grads_of[step] = _inject(opt.path, step, 0, torch.float32, scale=1e-2)
                opt.path.after_backward(sync=True, unscale=False)
                opt.step()
            else:
                for p, g in zip(plain, grads_of[step]):
                    p.grad = g.reshape(p.shape).cuda()
                popt.step()

    def fmt(sd, steps):
        for i, e in sd["state"].items():
            if i < 6:
                assert list(e) == ["momentum_buffer"], i
            else:
                assert list(e) == ["step", "exp_avg", "exp_avg_sq"] and float(e["step"]) == steps, i

    a = _fused(net, _aux_kw(net))
    run(a, range(3))
    sd = a.state_dict()
    fmt(sd, 3)
    plain = [torch.nn.Parameter(w.clone()) for w in a.path.unflatten(a.path.gather_master())]
    popt = MuonWithAuxAdamW(**_aux_kw(torch.nn.ParameterList(plain)))
    popt.load_state_dict({k: v for k, v in sd.items() if not k.startswith("b200_")})
    for step in range(3, 6):
        grads_of[step] = [g.clone() for g in _inject(a.path, step, 0, torch.float32, scale=1e-2)]
    run(None, range(3, 6), plain, popt)
    fmt(popt.state_dict(), 6)
    a.close()
    net_b = Mats(SHAPES).cuda()
    with torch.no_grad():
        for p, q in zip(net_b.parameters(), plain):
            p.copy_(q)
    b = B200StockOptimizer(net_b, MuonWithAuxAdamW, _aux_kw(net_b), engine=get_engine(0))
    b.load_state_dict(popt.state_dict())
    run(b, range(6, 9))
    sd_b = b.state_dict()
    fmt(sd_b, 9)
    net_c = Mats(SHAPES).cuda()
    with torch.no_grad():
        for p, q in zip(net_c.parameters(), b.path.unflatten(b.path.gather_master())):
            p.copy_(q)
    c = _fused(net_c, _aux_kw(net_c))
    c.load_state_dict(sd_b)
    # Muon keeps no count: its parameters' counts only mark that they have state
    assert c.path.param_steps()[6:] == [9, 9] and min(c.path.param_steps()) > 0
    run(c, range(9, 12))
    fmt(c.state_dict(), 12)
    run(None, range(12), ref, ropt)
    got = torch.cat([t.reshape(-1) for t in c.path.unflatten(c.path.gather_master().cpu())])
    want = torch.cat([p.detach().cpu().reshape(-1) for p in ref])
    init = torch.cat([p.cpu().reshape(-1) for p in w_init])
    assert _rel(got - init, want - init) < 0.03
    for o in (b, c):
        o.close()


def test_plain_torch_muon_state_dicts_load():
    """torch.optim.Muon on the fused step: its state_dict is torch's (momentum_buffer only, a never-stepped parameter
    without an entry); a state dict written by the plain class loads, as one torch would write."""
    shapes = [(32, 48), (48, 32), (5, 7)]
    net = Mats(shapes).cuda()
    kw = dict(lr=0.02)
    opt = _fused(net, kw, cls=torch.optim.Muon)
    path = opt.path
    for step in range(2):
        _inject(path, step, 0, torch.float32, scale=1e-2)
        path._track_touched = True
        path._touched = np.array([True, True, step > 0])
        path.after_backward(sync=True, unscale=False)
        opt.step()
    sd = opt.state_dict()
    assert sorted(sd["state"]) == [0, 1, 2] and all(list(e) == ["momentum_buffer"] for e in sd["state"].values())
    plain = [torch.nn.Parameter(w.clone()) for w in path.unflatten(path.gather_master())]
    tm = torch.optim.Muon(plain, **kw)
    tm.load_state_dict({k: v for k, v in sd.items() if not k.startswith("b200_")})
    for p, g in zip(plain, _inject(path, 2, 0, torch.float32, scale=1e-2)):
        p.grad = g.cuda()
    tm.step()
    opt.close()
    net2 = Mats(shapes).cuda()
    with torch.no_grad():
        for p, q in zip(net2.parameters(), plain):
            p.copy_(q)
    opt2 = _fused(net2, kw, cls=torch.optim.Muon)
    opt2.load_state_dict(tm.state_dict())
    assert opt2.path.param_steps() == [1, 1, 1]
    for i, p in enumerate(plain):
        assert torch.equal(opt2.path.unflatten(opt2.path.m_flat)[i], tm.state[p]["momentum_buffer"])
        assert torch.equal(opt2.path.unflatten(opt2.path.gather_master())[i], p.detach())
    opt2.close()


# ---- training ------------------------------------------------------------------------------------------------------------------
def _muon_groups(model):
    mats = [p for p in model.parameters() if p.dim() > 1]
    rest = [p for p in model.parameters() if p.dim() <= 1]
    return [dict(params=mats, use_muon=True, lr=0.02, weight_decay=0.01),
            dict(params=rest, use_muon=False, lr=1e-3, weight_decay=0.0)]


def test_stoke_bf16_resnet50_trains():
    import torchvision

    import stoke_b200 as sb
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    torch.manual_seed(0)
    model = torchvision.models.resnet50(num_classes=10).to(memory_format=torch.channels_last)
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=sb.MuonWithAuxAdamW,
                                                          optimizer_kwargs={"params": _muon_groups(model)}),
                 loss=torch.nn.CrossEntropyLoss(), batch_size_per_device=32, gpu=True, fp16="bf16", verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    assert len(s.optimizer.path.mu_index) == 54   # 53 convs and the classifier
    g = torch.Generator().manual_seed(1)
    x = torch.randn(32, 3, 64, 64, generator=g).cuda().to(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (32,), generator=g).cuda()
    losses = []
    for _ in range(25):
        loss = s.loss(s.model(x), y)
        s.backward(loss)
        s.step()
        losses.append(float(loss))
    assert all(np.isfinite(losses)) and losses[-1] < 0.5 * losses[0], losses
    s.optimizer.close()


def test_stoke_bf16_bert_trains():
    from transformers import BertConfig, BertForSequenceClassification

    import stoke_b200 as sb
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size=500, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128,
                     max_position_embeddings=64, num_labels=3, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)

    class Wrap(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, ids):
            return self.m(input_ids=ids).logits

    wrap = Wrap(BertForSequenceClassification(cfg))
    s = sb.Stoke(model=wrap, optimizer=sb.StokeOptimizer(optimizer=sb.MuonWithAuxAdamW,
                                                         optimizer_kwargs={"params": _muon_groups(wrap)}),
                 loss=torch.nn.CrossEntropyLoss(), batch_size_per_device=16, gpu=True, fp16="bf16", verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(0, 500, (16, 32), generator=g).cuda()
    y = torch.randint(0, 3, (16,), generator=g).cuda()
    losses = []
    for _ in range(30):
        loss = s.loss(s.model(ids), y)
        s.backward(loss)
        s.step()
        losses.append(float(loss))
    assert all(np.isfinite(losses)) and losses[-1] < 0.5 * losses[0], losses
    s.optimizer.close()


@pytest.mark.multigpu
def test_two_ranks_replicated_route(tmp_path):
    """W = 2 (fairscale_oss asked for): the Muon state is replicated on the all-reduce route; both replicas are
    bit-identical and match a world-1 fused step on the mean gradient."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "muon_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29591", os.path.join(ROOT, "tests", "muon_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    res = json.loads(out.read_text())
    assert res["route"] == "allreduce" and res["replicas_identical"], res
