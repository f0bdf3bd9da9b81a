"""torch.optim.Adafactor on the fused step (GPU).

Element level: one B200FusedOptimizer step at a time over parameters of every layout the kernel distinguishes, compared
element by element (master and state) with the float64 reference of tests/adafactor_ref.py, restarted from the kernel's
own state every step.  Engine level: gradient-injection parity with the CPU oracle (fp32 torch) on both world-1 routes,
the loss scaler's skipped step, NaN without a scaler, unused parameters, determinism, no host synchronisation, the Stoke
facade, checkpoints exchanged with plain torch and LR schedulers."""
import os
import subprocess
import sys

import pytest
import torch

import adafactor_ref as ar
from test_gpu_engine import OddNet, _inject, _oracle_flat, _rel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-5
ADA = torch.optim.Adafactor


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


SMALL = [((64, 64, 3, 3), True), ((256, 64, 1, 1), True), ((5, 7, 11), False), ((37, 23), False), ((1000,), False),
         ((), False)]
BIG = [((1000, 2048), False), ((30522, 768), False)]


def _build(shapes, kw, lp, route, clip=None, seed=0, groups=None):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    net = Shapes(shapes, seed).cuda()
    spec = None
    if clip is not None:
        spec = ClipSpec(_lib.CLIP_NORM, max_norm=clip[1], norm_type=2.0) if clip[0] == "norm" else \
            ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1])
    kwargs = dict(kw)
    if groups is not None:
        ps = list(net.parameters())
        kwargs["params"] = [dict(extra, params=[ps[i] for i in idx]) for idx, extra in groups]
    opt = B200FusedOptimizer(net, ADA, kwargs, engine=get_engine(0), clip=spec, lp_dtype=lp, route=route)
    assert opt.path.route == route
    return net, opt


ELEM_CASES = {
    "small_raw_bf16_clipnorm": (SMALL, {"lr": 1e-2}, torch.bfloat16, "local", ("norm", 0.05), None),
    "small_main_f32_clipvalue_decay_max": (SMALL, {"lr": 2e-2, "weight_decay": 0.5, "maximize": True}, None, "main",
                                           ("value", 2e-3), None),
    "small_raw_bf16_eps_d_2groups": (SMALL, {"lr": 1e-2, "eps": (1e-4, 1e-3), "d": 2.0}, torch.bfloat16, "local", None,
                                     [([0, 2, 4], {}), ([1, 3, 5], {"lr": 3e-3, "beta2_decay": -0.5,
                                                                    "eps": (None, 1e-2)})]),
    "big_raw_bf16": (BIG, {"lr": 1e-2, "weight_decay": 0.1}, torch.bfloat16, "local", None, None),
    "big_main_f32": (BIG, {"lr": 1e-2}, None, "main", ("norm", 1.0), None),
}


@pytest.mark.parametrize("name", list(ELEM_CASES))
def test_step_matches_torch_float64(name):
    shapes, kw, lp, route, clip, groups = ELEM_CASES[name]
    net, opt = _build(shapes, kw, lp, route, clip, groups=groups)
    path = opt.path
    hyp = [dict(kw)] * len(path.params)
    if groups is not None:
        for idx, extra in groups:
            for i in idx:
                hyp[i] = dict(kw, **extra)
    steps = 2 if name.startswith("big") else 3
    for step in range(steps):
        grads = _inject(path, step, 0, lp or torch.float32, scale=1e-3 * (1 + step))
        if step == 1:
            row = (0,) * (grads[0].dim() - 1)   # a zero row: v = 0 there, clamped at eps1^2
            grads[0][row] = 0.0
            path.grad_views[0][row] = 0.0
        w0 = [t.detach().cpu().clone() for t in path.unflatten(path.gather_master())]
        s0 = [tuple(v.cpu().clone() for v in vs) for vs in path.adafactor_state_views()]
        path.after_backward(sync=True, unscale=False)
        opt.step()
        st = path.engine.scaler_get(path.state_id)
        coef = torch.tensor(1.0)
        if clip is not None and clip[0] == "norm":
            coef = torch.clamp(torch.tensor(clip[1], dtype=torch.float32) / (torch.tensor(st.grad_norm) + 1e-6), max=1.0)
        w1 = [t.detach().cpu() for t in path.unflatten(path.gather_master())]
        s1 = [tuple(v.cpu() for v in vs) for vs in path.adafactor_state_views()]
        for i, p in enumerate(path.params):
            G = grads[i].float().reshape(p.shape)
            if clip is not None:
                G = G * coef if clip[0] == "norm" else G.clamp(-clip[1], clip[1])
            keys = ar.state_keys(p.shape)
            state = dict(zip(keys, s0[i]))
            rw, rst = ar.step_ref(w0[i], state, G, step, hyp[i])
            ew, est = ar.step_bound(w0[i], state, G, step, hyp[i], rw, rst)
            bad = ar.outside(w1[i], rw, ew)
            assert not bool(bad.any()), (name, step, i, p.shape, torch.nonzero(bad.reshape(-1))[:5].flatten().tolist())
            for k, got in zip(keys, s1[i]):
                assert not bool(ar.outside(got, rst[k], est[k]).any()), (name, step, i, k)
        assert path.param_steps() == [step + 1] * len(path.params)
        if lp is not None:
            assert torch.equal(path.p_flat.cpu(), path.gather_master().cpu().to(lp))
        assert float(path.g_flat.float().abs().max()) == 0.0
    opt.close()


# ---- engine level ------------------------------------------------------------------------------------------------------------
PARITY = [
    ({"lr": 1e-2}, torch.bfloat16, ("norm", 1.0, 2.0), 1),
    ({"lr": 1e-2, "weight_decay": 0.05, "maximize": True}, None, ("value", 0.3), 2),
    ({"lr": 5e-3, "eps": (1e-5, 1e-3), "d": 1.5, "beta2_decay": -0.6}, torch.bfloat16, None, 2),
]


def _fused(net, kw, lp, clip=None, accum=1, route=None):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import B200FusedOptimizer

    spec = None
    if clip is not None:
        spec = ClipSpec(_lib.CLIP_NORM, max_norm=clip[1], norm_type=clip[2]) if clip[0] == "norm" else \
            ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1])
    return B200FusedOptimizer(net, ADA, kw, engine=get_engine(0), grad_accum=accum, clip=spec, lp_dtype=lp, route=route)


def _check_state(sd, oracle):
    for i, p in enumerate(oracle.params):
        st = oracle.optimizer.state[p]
        assert set(sd["state"][i]) == set(st), (set(sd["state"][i]), set(st))
        assert float(sd["state"][i]["step"]) == float(st["step"])
        for k in st:
            if k != "step":
                assert sd["state"][i][k].shape == st[k].shape
                assert _rel(sd["state"][i][k].cpu(), st[k]) < TOL, (i, k)


@pytest.mark.parametrize("route", ["local", "main"])
@pytest.mark.parametrize("kw,lp,clip,accum", PARITY)
def test_gradient_injection_parity(kw, lp, clip, accum, route):
    from engine_oracle import OracleEngine

    torch.cuda.set_device(0)
    net = OddNet().cuda()
    init = [p.detach().cpu().clone() for p in net.parameters()]
    opt = _fused(net, kw, lp, clip, accum, route=route)
    path = opt.path
    oracle = OracleEngine(init, 1, ADA, kw, grad_accum=accum, clip=clip)
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


@pytest.mark.parametrize("route", ["local", "main"])
def test_scaler_skip_and_nan_without_scaler(route):
    """Loss scaler: an inf gradient skips the step (master, state and step counts unchanged, bucket zeroed), as
    GradScaler.step does.  No scaler: a NaN gradient gives torch's NaN pattern (python's max(1.0, nan) is 1.0)."""
    from engine_oracle import OracleEngine
    from stoke_b200.fp16 import DeviceGradScaler

    torch.cuda.set_device(0)
    kw = {"lr": 1e-2}
    net = OddNet().cuda()
    init = [p.detach().cpu().clone() for p in net.parameters()]
    opt = _fused(net, kw, None, ("norm", 1.0, 2.0), route=route)
    path = opt.path
    scaler = DeviceGradScaler(path.engine, init_scale=2.0**10, growth_interval=3, state_id=path.state_id)
    oracle = OracleEngine(init, 1, ADA, kw, clip=("norm", 1.0, 2.0), amp=dict(init_scale=2.0**10, growth_interval=3))
    for step, bad in enumerate([False, True, False, False]):
        grads = _inject(path, step, 0, torch.float32, scale=scaler.get_scale())
        if bad:
            path.grad_views[2].view(-1)[5] = float("inf")
            grads[2].view(-1)[5] = float("inf")
        oracle.micro_step([grads])
        before = (path.gather_master().clone(), path.af_state.clone(), path.param_steps())
        path.after_backward(sync=True, unscale=True)
        opt.step()
        assert oracle.step() == (not bad)
        if bad:
            assert torch.equal(before[0], path.gather_master()) and torch.equal(before[1], path.af_state)
            assert before[2] == path.param_steps()
        assert float(path.g_flat.float().abs().max()) == 0.0
    assert _rel(path.gather_master().cpu(), _oracle_flat(path, oracle.weights())) < TOL
    _check_state(opt.state_dict(), oracle)
    opt.close()
    # NaN without a scaler
    net = OddNet().cuda()
    init = [p.detach().cpu().clone() for p in net.parameters()]
    opt = _fused(net, kw, None, None, route=route)
    path = opt.path
    oracle = OracleEngine(init, 1, ADA, kw)
    for step in range(3):
        grads = _inject(path, step, 0, torch.float32)
        if step == 1:
            path.grad_views[4].view(-1)[9] = float("nan")
            grads[4].view(-1)[9] = float("nan")
        oracle.micro_step([grads])
        path.after_backward(sync=True, unscale=False)
        opt.step()
        oracle.step()
        got = torch.cat([t.reshape(-1) for t in path.unflatten(path.gather_master().cpu())])
        ref = torch.cat([w.reshape(-1) for w in oracle.weights()])
        assert torch.equal(got.isnan(), ref.isnan()), step
        fin = ~ref.isnan()
        assert _rel(got[fin], ref[fin]) < TOL
    opt.close()


def test_deterministic_and_no_host_sync():
    """Two identical runs give bit-identical masters and state; a step in which every parameter has a gradient runs
    under torch.cuda.set_sync_debug_mode("error")."""
    outs = []
    for _ in range(2):
        net, opt = _build(SMALL + BIG[:1], {"lr": 1e-2, "weight_decay": 0.01}, torch.bfloat16, "local", ("norm", 0.5))
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
        outs.append((path.gather_master().cpu(), path.af_state.cpu(), path.p_flat.cpu()))
        opt.close()
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int8) if a.dtype != torch.float32 else a.view(torch.int32),
                           b.view(torch.int8) if b.dtype != torch.float32 else b.view(torch.int32))


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


def test_unused_parameter_keeps_its_step():
    """Through Stoke (fp32): head b is unused on some steps; its step count and state stay put like torch's, and a
    parameter never stepped has no state entry."""
    from engine_oracle import OracleEngine
    import stoke_b200 as sb
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    kw = {"lr": 1e-2, "weight_decay": 0.1}
    model = TwoHeads()
    init = [p.detach().clone() for p in model.parameters()]
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=ADA, optimizer_kwargs=kw), loss=torch.nn.MSELoss(),
                 batch_size_per_device=8, gpu=True, verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    oracle = OracleEngine(init, 1, ADA, kw)
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


def test_stoke_bf16_facade_loss_decreases_and_scheduler():
    """Stoke with fp16="bf16" builds a B200FusedOptimizer for Adafactor and trains; an LR scheduler's edit of
    param_groups takes effect at the next step (lr = 0 freezes the weights)."""
    import stoke_b200 as sb
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.ReLU(), torch.nn.Flatten(),
                                torch.nn.Linear(8 * 8 * 8, 4)).to(memory_format=torch.channels_last)
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=ADA, optimizer_kwargs={"lr": 3e-2}),
                 loss=torch.nn.CrossEntropyLoss(), batch_size_per_device=16, gpu=True, fp16="bf16", verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(16, 3, 8, 8, generator=g).cuda().to(memory_format=torch.channels_last)
    y = torch.randint(0, 4, (16,), generator=g).cuda()
    losses = []
    for _ in range(30):
        loss = s.loss(s.model(x), y)
        s.backward(loss)
        s.step()
        losses.append(float(loss))
    assert losses[-1] < 0.5 * losses[0], losses
    sched = torch.optim.lr_scheduler.LambdaLR(s.optimizer, lambda e: 0.0)
    assert s.optimizer.param_groups[0]["lr"] == 0.0
    before = s.optimizer.path.gather_master().clone()
    loss = s.loss(s.model(x), y)
    s.backward(loss)
    s.step()
    assert torch.equal(before, s.optimizer.path.gather_master())
    del sched
    s.optimizer.close()


def test_checkpoint_round_trip_with_plain_torch():
    """Engine -> torch: the engine's state_dict loaded into torch.optim.Adafactor continues to the engine's weights.
    torch -> engine: a plain torch state dict (the model weights loaded first) continues the same way."""
    torch.cuda.set_device(0)
    kw = {"lr": 1e-2, "weight_decay": 0.01}
    net = OddNet().cuda()
    opt = _fused(net, kw, None)
    path = opt.path
    for step in range(4):
        _inject(path, step, 0, torch.float32)
        path.after_backward(sync=True, unscale=False)
        opt.step()
    sd = opt.state_dict()
    cpu_params = [torch.nn.Parameter(w.cpu().clone()) for w in path.unflatten(path.gather_master())]
    topt = ADA(cpu_params, **kw, foreach=False)
    topt.load_state_dict({k: (v if k != "state" else {i: {kk: vv.cpu() for kk, vv in s_.items()} for i, s_ in v.items()})
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
    opt2 = _fused(net2, kw, None)
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
    out = tmp_path / "adafactor_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29563", os.path.join(ROOT, "tests", "adafactor_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    assert res["route"] == "allreduce" and res["replicas_identical"] and res["rel_vs_oracle"] < TOL, res
