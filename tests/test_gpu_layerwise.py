"""LAMB and LARS on the fused step (GPU).

Element level: one B200FusedOptimizer step at a time over parameters between guard bands (the flat buffers' padding and
the neighbouring parameters), compared element by element (master and state) with the float64 reference of
tests/layerwise_ref.py, restarted from the kernel's own state every step: every gradient source, every clip, tile
boundaries, 8 groups mixing weight_decay == 0 and != 0.  Engine level: found_inf and per-parameter skips, gradient-injection
parity with the CPU oracle (the class itself), the stock route at 9 groups, unused parameters, determinism, no host
synchronisation, the Stoke facade on ResNet-18 and BERT, checkpoints exchanged with the classes' plain step, W = 2."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import layerwise_ref as lr_
from test_gpu_engine import OddNet, _inject, _oracle_flat, _rel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-5


def _cls(kind):
    from stoke_b200.optim import LAMB, LARS

    return LAMB if kind == "lamb" else LARS


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


# a channels-last 3x3 conv, a 1-D bias, numel not a multiple of 16 (851), sizes at a tile boundary -1 / 0 / +1
SMALL = [((64, 64, 3, 3), True), ((1000,), False), ((37, 23), False), ((8191,), False), ((8192,), False),
         ((8193,), False), ((3, 5, 7), False)]
BIG = [((30522, 768), False), ((768,), False)]


def _spec(clip):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec

    if clip is None:
        return None
    if clip[0] == "norm":
        return ClipSpec(_lib.CLIP_NORM, max_norm=clip[1], norm_type=2.0)
    return ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1])


def _build(kind, shapes, kw, lp, route, clip=None, groups=None, seed=0):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    net = Shapes(shapes, seed).cuda()
    kwargs = dict(kw)
    if groups is not None:
        ps = list(net.parameters())
        kwargs["params"] = [dict(extra, params=[ps[i] for i in idx]) for idx, extra in groups]
    opt = B200FusedOptimizer(net, _cls(kind), kwargs, engine=get_engine(0), clip=_spec(clip), lp_dtype=lp, route=route)
    assert opt.path.route == route
    return net, opt


def _groups8(n, kind):
    """8 groups over n parameters, alternating weight_decay == 0 and != 0, with their own lr and hyper-parameters."""
    out = []
    for gi in range(8):
        extra = {"lr": (1e-2 if kind == "lamb" else 0.5) * (1 + 0.25 * gi),
                 "weight_decay": 0.0 if gi % 2 else (0.01 if kind == "lamb" else 5e-4) * (1 + gi)}
        if kind == "lamb":
            extra["betas"] = (0.9 - 0.01 * gi, 0.999)
            extra["bias_correction"] = gi != 2
            extra["always_adapt"] = gi == 3
        else:
            extra["momentum"] = 0.0 if gi == 5 else 0.9
            extra["nesterov"] = gi == 4
            extra["always_adapt"] = gi == 3
            extra["trust_coefficient"] = 0.001 * (1 + gi)
        out.append(([i for i in range(n) if i % 8 == gi], extra))
    return out


ELEM_CASES = {
    "lamb_raw_bf16_clipnorm": ("lamb", SMALL, {"lr": 1e-2, "weight_decay": 0.01}, torch.bfloat16, "local",
                               ("norm", 0.05), None),
    "lamb_raw_f32_clipvalue": ("lamb", SMALL, {"lr": 1e-2, "weight_decay": 0.1, "eps": 1e-4}, None, "local",
                               ("value", 2e-3), None),
    "lamb_main_f32_adapt_nobc": ("lamb", SMALL, {"lr": 1e-2, "weight_decay": 0.0, "always_adapt": True,
                                                 "bias_correction": False}, None, "main", None, None),
    "lars_raw_bf16": ("lars", SMALL, {"lr": 0.5, "weight_decay": 1e-4}, torch.bfloat16, "local", None, None),
    "lars_raw_f32_clipnorm_damp": ("lars", SMALL, {"lr": 1.0, "weight_decay": 1e-3, "dampening": 0.3}, None, "local",
                                   ("norm", 0.5), None),
    "lars_main_f32_clipvalue_nesterov": ("lars", SMALL, {"lr": 0.5, "weight_decay": 5e-4, "nesterov": True}, None,
                                         "main", ("value", 3e-3), None),
    "lamb_8groups_raw_bf16": ("lamb", SMALL * 2, {"lr": 1e-2}, torch.bfloat16, "local", ("norm", 1.0), "g8"),
    "lars_8groups_raw_bf16": ("lars", SMALL * 2, {"lr": 0.5}, torch.bfloat16, "local", None, "g8"),
    "lamb_big_raw_bf16": ("lamb", BIG, {"lr": 1e-3, "weight_decay": 0.01}, torch.bfloat16, "local", None, None),
    "lars_big_main_f32": ("lars", BIG, {"lr": 1.0, "weight_decay": 1e-4}, None, "main", ("norm", 1.0), None),
}


def _state_views(kind, path):
    views = {}
    if path.m_flat is not None:
        views["exp_avg" if kind == "lamb" else "momentum_buffer"] = [v.cpu().clone() for v in path.unflatten(path.m_flat)]
    if path.v_flat is not None:
        views["exp_avg_sq"] = [v.cpu().clone() for v in path.unflatten(path.v_flat)]
    return views


def _check_step(kind, path, hyp, grads, coef, clip, step, w0, s0, steps0, stepped, tag):
    """Every stepped parameter inside the bounds of the float64 reference; every other one unchanged."""
    w1 = [t.detach().cpu() for t in path.unflatten(path.gather_master())]
    s1 = _state_views(kind, path)
    for i, p in enumerate(path.params):
        if not stepped[i]:
            assert torch.equal(w1[i], w0[i]), (tag, step, i)
            for k in s1:
                assert torch.equal(s1[k][i], s0[k][i]), (tag, step, i, k)
            continue
        G = grads[i].float().reshape(p.shape)
        if clip is not None:
            G = G * coef if clip[0] == "norm" else G.clamp(-clip[1], clip[1])
        keys = lr_.state_keys(kind, hyp[i])
        state = {k: s0[k][i] for k in keys} if steps0[i] > 0 else lr_.zero_state(kind, p.shape, hyp[i])
        rw, rst = lr_.step_ref(kind, w0[i], state, G, steps0[i], hyp[i])
        ew, est = lr_.step_bound(kind, w0[i], state, G, steps0[i], hyp[i], rw, rst)
        bad = lr_.outside(w1[i], rw, ew)
        assert not bool(bad.any()), (tag, step, i, p.shape, torch.nonzero(bad.reshape(-1))[:5].flatten().tolist())
        for k in keys:
            assert not bool(lr_.outside(s1[k][i], rst[k], est[k]).any()), (tag, step, i, k)


@pytest.mark.parametrize("name", list(ELEM_CASES))
def test_step_matches_float64_reference(name):
    kind, shapes, kw, lp, route, clip, groups = ELEM_CASES[name]
    groups = _groups8(len(shapes), kind) if groups == "g8" else None
    net, opt = _build(kind, shapes, kw, lp, route, clip, groups=groups)
    path = opt.path
    hyp = [dict(kw)] * len(path.params)
    if groups is not None:
        for idx, extra in groups:
            for i in idx:
                hyp[i] = dict(kw, **extra)
    guard = torch.full((path.n,), True)   # guard bands: the padding after every parameter stays exactly as it was
    for v in path.unflatten(guard):
        v.fill_(False)
    steps = 2 if "big" in name else 3
    for step in range(steps):
        grads = _inject(path, step, 0, lp or torch.float32, scale=1e-3 * (1 + step))
        w0 = [t.detach().cpu().clone() for t in path.unflatten(path.gather_master())]
        s0 = _state_views(kind, path)
        flat0 = (path.gather_master().cpu(), path.m_flat.cpu().clone() if path.m_flat is not None else None)
        steps0 = path.param_steps()
        path.after_backward(sync=True, unscale=False)
        opt.step()
        st = path.engine.scaler_get(path.state_id)
        coef = torch.tensor(1.0)
        if clip is not None and clip[0] == "norm":
            coef = torch.clamp(torch.tensor(clip[1], dtype=torch.float32) / (torch.tensor(st.grad_norm) + 1e-6), max=1.0)
        _check_step(kind, path, hyp, grads, coef, clip, step, w0, s0, steps0, [True] * len(path.params), name)
        assert torch.equal(path.gather_master().cpu()[guard], flat0[0][guard])
        if flat0[1] is not None:
            assert torch.equal(path.m_flat.cpu()[guard], flat0[1][guard])
        assert path.param_steps() == [step + 1] * len(path.params)
        if lp is not None:
            assert torch.equal(path.p_flat.cpu(), path.gather_master().cpu().to(lp))
        assert float(path.g_flat.float().abs().max()) == 0.0
    opt.close()


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_found_inf_and_skipped_parameters_leave_state(kind):
    """A skipped parameter (no gradient this step) keeps its master, state and count while the others step inside the
    bounds; an inf gradient under the loss scaler skips every parameter.  The raw bucket is zeroed either way."""
    from stoke_b200.fp16 import DeviceGradScaler

    kw = {"lr": 1e-2} if kind == "lamb" else {"lr": 0.5}
    shapes = SMALL * 2
    groups = _groups8(len(shapes), kind)
    net, opt = _build(kind, shapes, kw, torch.bfloat16, "local", groups=groups)
    path = opt.path
    hyp = [dict(kw)] * len(path.params)
    for idx, extra in groups:
        for i in idx:
            hyp[i] = dict(kw, **extra)
    scaler = DeviceGradScaler(path.engine, init_scale=2.0**4, growth_interval=1000, state_id=path.state_id)
    for step, (skip, bad) in enumerate([((), False), ((1, 4, 9), False), ((), True), ((4,), False)]):
        scale = scaler.get_scale()
        grads = _inject(path, step, 0, torch.bfloat16, scale=1e-3 * scale)
        if bad:
            path.grad_views[2].view(-1)[5] = float("inf")
        path._track_touched = True
        path._touched = np.array([i not in skip for i in range(len(path.params))])
        w0 = [t.detach().cpu().clone() for t in path.unflatten(path.gather_master())]
        s0 = _state_views(kind, path)
        steps0 = path.param_steps()
        path.after_backward(sync=True, unscale=True)
        opt.step()
        stepped = [not bad and i not in skip for i in range(len(path.params))]
        grads = [g / scale for g in grads]   # exact: the scale is a power of two
        _check_step(kind, path, hyp, grads, None, None, step, w0, s0, steps0, stepped, kind)
        assert path.param_steps() == [s + int(d) for s, d in zip(steps0, stepped)]
        assert float(path.g_flat.float().abs().max()) == 0.0
    opt.close()


# ---- engine level ------------------------------------------------------------------------------------------------------------
PARITY = [
    ("lamb", {"lr": 1e-2, "weight_decay": 0.01}, torch.bfloat16, ("norm", 1.0, 2.0), 1, "local"),
    ("lamb", {"lr": 5e-3, "weight_decay": 0.0, "always_adapt": True}, None, ("value", 0.3), 2, "local"),
    ("lamb", {"lr": 1e-2, "bias_correction": False}, None, None, 2, "main"),
    ("lars", {"lr": 0.5, "weight_decay": 1e-4}, torch.bfloat16, ("norm", 1.0, 2.0), 1, "local"),
    ("lars", {"lr": 0.5, "weight_decay": 5e-4, "nesterov": True}, None, None, 2, "local"),
    ("lars", {"lr": 0.2, "momentum": 0.0, "always_adapt": True}, None, ("value", 0.3), 1, "main"),
]


def _fused(net, kind, kw, lp, clip=None, accum=1, route=None):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import B200FusedOptimizer

    spec = None
    if clip is not None:
        spec = ClipSpec(_lib.CLIP_NORM, max_norm=clip[1], norm_type=clip[2]) if clip[0] == "norm" else \
            ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1])
    return B200FusedOptimizer(net, _cls(kind), kw, engine=get_engine(0), grad_accum=accum, clip=spec, lp_dtype=lp,
                              route=route)


def _check_state(sd, oracle):
    for i, p in enumerate(oracle.params):
        st = oracle.optimizer.state[p]
        assert set(sd["state"].get(i, {})) == set(st), (i, set(sd["state"].get(i, {})), set(st))
        if not st:
            continue
        assert float(sd["state"][i]["step"]) == float(st["step"])
        for k in st:
            if k != "step":
                assert sd["state"][i][k].shape == st[k].shape
                assert _rel(sd["state"][i][k].cpu(), st[k]) < TOL, (i, k)


@pytest.mark.parametrize("kind,kw,lp,clip,accum,route", PARITY)
def test_gradient_injection_parity(kind, kw, lp, clip, accum, route):
    from engine_oracle import OracleEngine

    torch.cuda.set_device(0)
    net = OddNet().cuda()
    init = [p.detach().cpu().clone() for p in net.parameters()]
    opt = _fused(net, kind, kw, lp, clip, accum, route=route)
    path = opt.path
    oracle = OracleEngine(init, 1, _cls(kind), kw, grad_accum=accum, clip=clip)
    for step in range(10):
        for micro in range(accum):
            oracle.micro_step([_inject(path, step * accum + micro, 0, lp or torch.float32)])
            path.after_backward(sync=(micro == accum - 1), unscale=False)
        opt.step()
        oracle.step()
        assert float(path.g_flat.float().abs().max()) == 0.0
    got = path.gather_master().cpu()
    assert _rel(got, _oracle_flat(path, oracle.weights())) < TOL
    if lp is not None:
        assert torch.equal(path.p_flat.cpu(), got.to(lp))
    _check_state(opt.state_dict(), oracle)
    opt.close()


class NineParams(torch.nn.Module):
    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(4)
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(17 + 5 * i, 3, generator=g) * 0.1)
                                          for i in range(9)])


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_nine_groups_take_the_stock_route(kind):
    """More than 8 groups: build_optimizer picks B200StockOptimizer, which runs the class's own step on the fp32 masters."""
    from engine_oracle import OracleEngine
    from stoke_b200.engine import get_engine
    from stoke_b200.extensions import BaseOptimizer
    from stoke_b200.optim import B200StockOptimizer, fused_supported

    torch.cuda.set_device(0)
    net = NineParams().cuda()
    init = [p.detach().cpu().clone() for p in net.parameters()]
    base = {"lr": 1e-2} if kind == "lamb" else {"lr": 0.5}
    groups = [([i], {"weight_decay": 0.0 if i % 2 else (0.01 if kind == "lamb" else 1e-3), "lr": base["lr"] * (1 + i / 8)})
              for i in range(9)]
    kw = dict(base, params=[dict(extra, params=[list(net.parameters())[i] for i in idx]) for idx, extra in groups])
    assert not fused_supported(_cls(kind), kw, net)
    b = BaseOptimizer(verbose=False)
    b._engine, b._lp_dtype = get_engine(0), torch.bfloat16
    opt = b.build_optimizer(_cls(kind), kw, net)
    assert isinstance(opt, B200StockOptimizer)
    path = opt.path
    oracle = OracleEngine(init, 1, _cls(kind), base, groups=groups)
    for step in range(6):
        oracle.micro_step([_inject(path, step, 0, torch.bfloat16)])
        path.after_backward(sync=True, unscale=False)
        opt.step()
        oracle.step()
    assert _rel(path.gather_master().cpu(), _oracle_flat(path, oracle.weights())) < TOL
    opt.close()


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


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_unused_parameter_keeps_its_step_and_state(kind):
    """Through Stoke (fp32): head b is unused on some steps; its step count and state stay put like the class's, and a
    parameter never stepped has no state entry."""
    from engine_oracle import OracleEngine
    import stoke_b200 as sb
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    kw = {"lr": 1e-2, "weight_decay": 0.1} if kind == "lamb" else {"lr": 0.5, "weight_decay": 1e-3}
    model = TwoHeads()
    init = [p.detach().clone() for p in model.parameters()]
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=_cls(kind), optimizer_kwargs=kw),
                 loss=torch.nn.MSELoss(), batch_size_per_device=8, gpu=True, verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    oracle = OracleEngine(init, 1, _cls(kind), kw)
    path = s.optimizer.path
    g = torch.Generator().manual_seed(0)
    for step in range(9):
        model.use_b = step % 3 != 1 and step != 0
        x, y = torch.randn(8, 16, generator=g).cuda(), torch.randn(8, 1, generator=g).cuda()
        loss = s.loss(s.model(x), y)
        path.begin_backward(sync=True, unscale=False)
        loss.backward()
        grads = [gv.detach().float().cpu().clone() if path._touched[i] else None for i, gv in enumerate(path.grad_views)]
        oracle.micro_step([grads])
        s._grad_accum_counter += 1
        path.after_backward(sync=True, unscale=False)
        s._backward_steps += 1
        s.step()
        oracle.step()
        if step == 0:
            assert set(s.optimizer.state_dict()["state"]) == {0, 1, 2, 3}   # head b never stepped: no state
    for a, b in zip(model.parameters(), oracle.weights()):
        assert _rel(a.detach().float().cpu().reshape(-1), b.reshape(-1)) < TOL
    sd = s.optimizer.state_dict()
    _check_state(sd, oracle)
    assert [float(sd["state"][j]["step"]) for j in range(6)] == [9.0, 9.0, 9.0, 9.0, 5.0, 5.0]
    s.optimizer.close()


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_deterministic_and_no_host_sync(kind):
    """Two identical runs give bit-identical masters, state and bf16 copies; a step runs under
    torch.cuda.set_sync_debug_mode("error")."""
    kw = {"lr": 1e-2, "weight_decay": 0.01} if kind == "lamb" else {"lr": 0.5, "weight_decay": 1e-4}
    outs = []
    for _ in range(2):
        net, opt = _build(kind, SMALL + BIG[:1], kw, torch.bfloat16, "local", ("norm", 0.5))
        path = opt.path
        for step in range(3):
            _inject(path, step, 0, torch.bfloat16, scale=1e-3)
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
        outs.append((path.gather_master().cpu(), path.m_flat.cpu(),
                     path.v_flat.cpu() if path.v_flat is not None else torch.zeros(1), path.p_flat.cpu()))
        opt.close()
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                           b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))


def _no_decay_groups(model, wd, **plain_extra):
    """The recipes' split: weight decay on weight matrices / kernels, none on biases and norm weights."""
    decay = [p for p in model.parameters() if p.dim() > 1]
    plain = [p for p in model.parameters() if p.dim() <= 1]
    return [{"params": decay, "weight_decay": wd}, dict({"params": plain, "weight_decay": 0.0}, **plain_extra)]


def test_stoke_bf16_lars_resnet18_trains():
    import torchvision

    import stoke_b200 as sb
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    torch.manual_seed(0)
    model = torchvision.models.resnet18(num_classes=10).to(memory_format=torch.channels_last)
    kw = {"lr": 5.0, "momentum": 0.9, "params": _no_decay_groups(model, 5e-5, lr=0.05)}
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=sb.LARS, optimizer_kwargs=kw),
                 loss=torch.nn.CrossEntropyLoss(), batch_size_per_device=32, gpu=True, fp16="bf16", verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(32, 3, 64, 64, generator=g).cuda().to(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (32,), generator=g).cuda()
    losses = []
    for _ in range(25):
        loss = s.loss(s.model(x), y)
        s.backward(loss)
        s.step()
        losses.append(float(loss))
    assert losses[-1] < 0.5 * losses[0], losses
    s.optimizer.close()


def test_stoke_bf16_lamb_bert_trains_and_scheduler():
    """LAMB on a small BertForSequenceClassification through the facade; an LR scheduler's edit of param_groups takes
    effect at the next step (lr = 0 freezes the weights)."""
    from transformers import BertConfig, BertForSequenceClassification

    import stoke_b200 as sb
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size=500, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128,
                     max_position_embeddings=64, num_labels=3, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    model = BertForSequenceClassification(cfg)

    class Wrap(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, ids):
            return self.m(input_ids=ids).logits

    wrap = Wrap(model)
    kw = {"lr": 2e-2, "params": _no_decay_groups(wrap, 0.01)}
    s = sb.Stoke(model=wrap, optimizer=sb.StokeOptimizer(optimizer=sb.LAMB, optimizer_kwargs=kw),
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
    assert losses[-1] < 0.5 * losses[0], losses
    sched = torch.optim.lr_scheduler.LambdaLR(s.optimizer, lambda e: 0.0)
    assert all(gr["lr"] == 0.0 for gr in s.optimizer.param_groups)
    before = s.optimizer.path.gather_master().clone()
    loss = s.loss(s.model(ids), y)
    s.backward(loss)
    s.step()
    assert torch.equal(before, s.optimizer.path.gather_master())
    del sched
    s.optimizer.close()


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_checkpoint_round_trip_with_plain_step(kind):
    """Fused -> class: the fused state_dict loaded into the class continues to the fused run's weights.  Class -> fused:
    a state dict written by the class's plain step (the model weights loaded first) continues the same way."""
    torch.cuda.set_device(0)
    kw = {"lr": 1e-2, "weight_decay": 0.01} if kind == "lamb" else {"lr": 0.5, "weight_decay": 1e-3, "nesterov": True}
    net = OddNet().cuda()
    opt = _fused(net, kind, kw, None)
    path = opt.path
    for step in range(4):
        _inject(path, step, 0, torch.float32)
        path.after_backward(sync=True, unscale=False)
        opt.step()
    sd = opt.state_dict()
    cpu_params = [torch.nn.Parameter(w.cpu().clone()) for w in path.unflatten(path.gather_master())]
    topt = _cls(kind)(cpu_params, **kw)
    topt.load_state_dict({k: (v if k != "state" else {i: {kk: vv.cpu().clone() for kk, vv in s_.items()}
                                                      for i, s_ in v.items()})
                          for k, v in sd.items() if not k.startswith("b200_")})
    for step in range(4, 8):
        for p, gr in zip(cpu_params, _inject(path, step, 0, torch.float32)):
            p.grad = gr.reshape(p.shape).clone()
        path.after_backward(sync=True, unscale=False)
        opt.step()
        topt.step()
    for a, b in zip(path.unflatten(path.gather_master().cpu()), cpu_params):
        assert _rel(a.reshape(-1), b.detach().reshape(-1)) < TOL
    net2 = OddNet().cuda()
    with torch.no_grad():
        for p, q in zip(net2.parameters(), cpu_params):
            p.copy_(q.detach())
    opt2 = _fused(net2, kind, kw, None)
    opt2.load_state_dict(topt.state_dict())
    for step in range(8, 12):
        grads = _inject(opt2.path, step, 0, torch.float32)
        for p, gr in zip(cpu_params, grads):
            p.grad = gr.reshape(p.shape).clone()
        opt2.path.after_backward(sync=True, unscale=False)
        opt2.step()
        topt.step()
    for a, b in zip(opt2.path.unflatten(opt2.path.gather_master().cpu()), cpu_params):
        assert _rel(a.reshape(-1), b.detach().reshape(-1)) < TOL
    sd2 = opt2.state_dict()
    for i, p in enumerate(cpu_params):
        assert float(sd2["state"][i]["step"]) == float(topt.state[p]["step"])
    opt.close()
    opt2.close()


@pytest.mark.multigpu
def test_replicas_bit_identical_w2(tmp_path):
    """W = 2 (fairscale_oss asked for, state replicated): both replicas bit-identical, and within the bar of the
    W = 1 oracle."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "layerwise_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29567", os.path.join(ROOT, "tests", "layerwise_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    for kind in ("lamb", "lars"):
        r = res[kind]
        assert r["route"] == "allreduce" and r["replicas_identical"] and r["rel_vs_oracle"] < TOL, (kind, r)
