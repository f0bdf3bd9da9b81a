"""stoke_b200.Lion on the fused step (GPU).

Kernel level: stk_optim_step_ex (with stk_optim_step_prologue where step counts are per parameter) called directly, the
buffers between guard bands (see test_gpu_kernels.py), and compared bit for bit with ``Lion.step()`` on CUDA fp32 tensors
holding the same formed gradient, restarted from the kernel's own state every step.  Three deliberately wrong updates
must fail the same comparison.  Engine level: gradient-injection parity with the CPU oracle, the Stoke facade with an
unused parameter, checkpoints exchanged with a plain Lion and with the stock route, a step without host
synchronisation, weight averaging, and the sharded W = 2 run."""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import stoke_b200 as sb
from stoke_b200.optim import Lion
from test_gpu_kernels import BF16, F32, INT_VIEW, Buf, _dt, _layout

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-5
BASE = {"lr": 2.0**-7, "betas": (0.875, 0.9921875), "weight_decay": 0.0, "maximize": False}
GROUPS8 = [BASE, dict(BASE, lr=2.0**-5), dict(BASE, betas=(0.9, 0.99)), dict(BASE, maximize=True),
           dict(BASE, weight_decay=0.25), dict(BASE, betas=(0.5, 0.75), weight_decay=1.5), dict(BASE, lr=0.0),
           dict(BASE, lr=1e-3, weight_decay=0.1, maximize=True)]
MUTANTS = ("decay_after", "sign_of_new", "swap_betas")


def _L():
    from stoke_b200 import _lib

    return _lib


def _hyper(h):
    L = _L()
    o = L.OptimHyper()
    o.kind = L.OPT_LION
    o.lr = h["lr"]
    o.beta1, o.beta2 = h["betas"]
    o.weight_decay = h["weight_decay"]
    o.maximize = int(h["maximize"])
    o.clip_kind = L.CLIP_NONE
    return o


@pytest.fixture
def eng():
    from stoke_b200.engine import get_engine

    torch.cuda.set_device(0)
    e = get_engine(0)
    sid = e.state_create()
    e.state_select(sid)
    yield e
    torch.cuda.synchronize()
    e.state_destroy(sid)


def _torch_lion(w, m, g, h, done):
    """Lion.step() on CUDA fp32 tensors, restarted from (w, m) after ``done`` steps."""
    p = torch.nn.Parameter(w.clone())
    opt = Lion([p], **h)
    opt.state[p] = {"step": torch.tensor(float(done)), "exp_avg": m.clone()}
    p.grad = g.clone()
    opt.step()
    return p.detach(), opt.state[p]["exp_avg"]


def _mutant(w, m, g, h, mut):
    """The same update with one deliberate mistake: weight decay after the update, the sign of the NEW exp_avg, or
    beta1 and beta2 swapped."""
    lr, (b1, b2), wd = h["lr"], h["betas"], h["weight_decay"]
    g = -g if h["maximize"] else g
    if mut == "swap_betas":
        b1, b2 = b2, b1
    w, m = w.clone(), m.clone()
    if wd != 0 and mut != "decay_after":
        w.mul_(1 - lr * wd)
    if mut == "sign_of_new":
        m.mul_(b2).add_(g, alpha=1 - b2)
        u = m.sign()
    else:
        u = m.mul(b1).add_(g, alpha=1 - b1).sign_()
        m.mul_(b2).add_(g, alpha=1 - b2)
    w.add_(u, alpha=-lr)
    if wd != 0 and mut == "decay_after":
        w.mul_(1 - lr * wd)
    return w, m


def _same(a, b):
    """Bit for bit; a NaN matches a NaN."""
    a, b = a.cpu(), b.cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


SPECIALS = [0.0, -0.0, 1e-40, -1e-40, 1e-45, float("inf"), float("-inf"), float("nan"), 3e-39, -2.5e-39]

# name: gradient source, model copy, n_local, segments, groups, range table, skip bits, per-parameter counts,
#       fp32 accumulator (raw fp32 route), found_inf step
CASES = {
    "raw_bf16": ("raw_bf16", "bf16", 2_056, 0, [dict(BASE, weight_decay=0.125)], False, False, False, False, None),
    "raw_f32_acc_inf": ("raw_f32", None, 2_040, 3, [dict(BASE, weight_decay=0.25)], False, False, False, True, 2),
    "main_max": ("main", "f32", 2_056, 0, [dict(BASE, maximize=True, weight_decay=0.5)], False, False, False, False, None),
    "seg64_8groups_steps": ("raw_bf16", "bf16", 2_048, 64, GROUPS8, True, True, True, False, 4),
    "raw_f32_acc_8groups": ("raw_f32", None, 2_056, 5, GROUPS8, True, True, True, True, None),
    "main_8groups_ranges": ("main", "bf16", 2_048, 7, GROUPS8, True, True, False, False, 3),
}
STEPS = 7


@pytest.mark.parametrize("name", list(CASES))
def test_lion_kernel_matches_cuda_torch_bit_for_bit(eng, name):
    L = _L()
    src, lp, n_local, n_seg, groups, use_ranges, use_skip, per_range, use_acc, inf_at = CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    pieces, N = _layout(n_local, n_seg, rng, base=64)
    N = -(-N // 16) * 16
    gidx = np.concatenate([np.arange(g0, g0 + (l1 - l0)) for l0, l1, g0 in pieces])
    if use_ranges:
        nr = 12
        ends = sorted(rng.choice(np.arange(1, N // 16), nr - 1, replace=False).tolist()) + [N // 16]
        ends = [e * 16 for e in ends]
        rgroup = [j % len(groups) for j in range(nr)]
        rskip = [bool(use_skip and j % 4 == 1) for j in range(nr)]
    else:
        ends, rgroup, rskip = [N], [0], [False]
    elem_range = np.searchsorted(np.asarray(ends), gidx, side="right")
    ng = len(groups)
    hyp = (L.OptimHyper * ng)(*[_hyper(h) for h in groups])
    w0 = rng.standard_normal(n_local).astype(np.float32) * 1e-2
    w0[:32] = np.tile([0.0, -0.0], 16)          # +-0 parameters; their gradient is zero on every step (c == 0)
    MB = Buf(n_local, F32, torch.from_numpy(w0).cuda())
    MM = Buf(n_local, F32, torch.zeros(n_local).cuda())
    LPB = None if lp is None else Buf(N, BF16 if lp == "bf16" else F32, torch.full((N,), -5.0))
    gdt = {"raw_bf16": BF16, "raw_f32": F32, "main": F32}[src]
    GB = Buf(N if src != "main" else n_local, gdt)
    AB = Buf(N, F32) if use_acc else None
    BC = Buf(len(ends) * 4, F32, torch.full((len(ends) * 4,), float("nan")).cuda()) if per_range else None
    if use_ranges:
        rend = torch.tensor([e // 8 for e in ends], dtype=torch.int32).cuda()
        rgrp = torch.tensor([g | (0x80 if s else 0) for g, s in zip(rgroup, rskip)], dtype=torch.uint8).cuda()
    rsteps = torch.zeros(len(ends), dtype=torch.int32).cuda()
    sl = (C.c_size_t * (len(pieces) + 1))(*([p[0] for p in pieces] + [n_local]))
    sg = (C.c_size_t * len(pieces))(*[p[2] for p in pieces])
    lpp = L.ptr_array([LPB.ptr()]) if lp is not None else None
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0)
    live = {rgroup[j] for j in range(len(ends)) if not rskip[j] and bool((elem_range == j).any())}
    muts = set(MUTANTS)
    if all(groups[gi]["weight_decay"] == 0 for gi in live):
        muts.discard("decay_after")
    hit = set()
    g32 = rng.standard_normal(n_local).astype(np.float32)

    for step in range(STEPS):
        g = np.roll(g32, step * 37) * 1e-3
        pos = 40 + (step * 13) % 200
        g[pos:pos + len(SPECIALS)] = SPECIALS      # +-0, subnormals, +-inf and NaN at moving positions
        g[:32] = 0.0
        g[32:48] *= 1e-36                           # gradients in the fp32 subnormal range once the betas scale them
        g = torch.from_numpy(g.astype(np.float32)).to(gdt)
        gfull = torch.zeros(GB.n, dtype=gdt)
        if src == "main":
            gfull[:] = g
        else:
            gfull[:] = torch.from_numpy(rng.standard_normal(GB.n).astype(np.float32)).to(gdt)
            gfull[torch.from_numpy(gidx)] = g
        GB.t.copy_(gfull.cuda())
        acc_local = None
        if AB is not None:
            afull = torch.from_numpy(rng.standard_normal(N).astype(np.float32) * 1e-3)
            AB.t.copy_(afull.cuda())
            acc_local = afull[torch.from_numpy(gidx)]
        found_inf = inf_at == step
        eng.scaler_set(found_inf=int(found_inf))
        w, m = MB.t.clone(), MM.t.clone()
        snap = {k: b.bits() for k, b in (("G", GB), ("M", MB), ("MM", MM), ("LP", LPB), ("A", AB)) if b}
        steps_before = rsteps.cpu().clone()
        if per_range:
            eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, None, ng, len(ends), rgrp.data_ptr(),
                                                       rsteps.data_ptr(), None, BC.ptr(), eng._stream()))
        a = L.OptimArgs()
        a.hyper, a.n_groups = hyp, ng
        a.master, a.exp_avg, a.exp_avg_sq = MB.ptr(), MM.ptr(), None
        a.grad, a.grad_dtype, a.grad_raw, a.grad_mul = GB.ptr(), _dt(gdt), int(src != "main"), 1.0
        a.acc = AB.ptr() if AB is not None else None
        a.n_local = n_local
        a.lp_ptrs, a.lp_world, a.lp_dtype = lpp, (1 if lp else 0), (L.BF16 if lp == "bf16" else L.F32)
        a.n_seg = n_seg
        a.seg_local, a.seg_global = (sl, sg) if n_seg else (None, None)
        a.lp_offset = pieces[0][2] if n_seg == 0 else 0
        if use_ranges:
            a.n_ranges, a.range_end_vec, a.range_group = len(ends), rend.data_ptr(), rgrp.data_ptr()
        if per_range:
            a.range_bc = BC.ptr()
        eng.optim_step_ex(a)   # without per-parameter counts Lion needs no prologue scalars at all
        eng.step_epilogue()
        got_w, got_m = MB.t.clone(), MM.t.clone()
        if per_range:   # Lion's row of the prologue is all zero; the counts advance like every kind's
            assert torch.equal(BC.t.cpu(), torch.zeros(len(ends) * 4))
            for j in range(len(ends)):
                assert int(rsteps[j]) == int(steps_before[j]) + (0 if rskip[j] or found_inf else 1)
            BC.check_guards()

        skip_elem = torch.from_numpy(np.asarray(rskip)[elem_range]) | found_inf
        gl = g.float()
        if acc_local is not None:
            gl = gl + acc_local                       # the kernel's raw + accumulator sum, one fp32 add
        gl = gl.cuda()
        ref_w, ref_m = w.clone(), m.clone()
        mut_w = {mu: w.clone() for mu in muts}
        mut_m = {mu: m.clone() for mu in muts}
        for j in range(len(ends)):
            s = torch.from_numpy(elem_range == j).cuda()
            if rskip[j] or found_inf or not bool(s.any()):
                continue
            h = groups[rgroup[j]]
            done = int(steps_before[j]) if per_range else step   # Lion's update does not read the count
            ref_w[s], ref_m[s] = _torch_lion(w[s], m[s], gl[s], h, done)
            for mu in muts:
                mut_w[mu][s], mut_m[mu][s] = _mutant(w[s], m[s], gl[s], h, mu)
        assert _same(got_w, ref_w), f"step {step}: master"
        assert _same(got_m, ref_m), f"step {step}: exp_avg"
        for mu in muts:
            if not (_same(got_w, mut_w[mu]) and _same(got_m, mut_m[mu])):
                hit.add(mu)
        # ---- where the kernel wrote ----
        MB.check_unchanged_except(snap["M"], ~skip_elem)
        MM.check_unchanged_except(snap["MM"], ~skip_elem)
        assert torch.equal(got_w[skip_elem.cuda()].view(torch.int32), w[skip_elem.cuda()].view(torch.int32))
        if src != "main":   # the raw bucket is consumed, also on a skipped step; the accumulator is only read
            seg = torch.zeros(GB.n, dtype=torch.bool)
            seg[torch.from_numpy(gidx)] = True
            GB.check_unchanged_except(snap["G"], seg)
            assert float(GB.t[torch.from_numpy(gidx).cuda()].float().abs().max()) == 0.0
            if AB is not None:
                AB.check_unchanged_except(snap["A"], torch.zeros(N, dtype=torch.bool))
        else:
            GB.check_unchanged_except(snap["G"], torch.zeros(GB.n, dtype=torch.bool))
        if LPB is not None:
            stepped = ~skip_elem
            mask = torch.zeros(LPB.n, dtype=torch.bool)
            mask[torch.from_numpy(gidx)[stepped]] = True
            LPB.check_unchanged_except(snap["LP"], mask)
            if bool(stepped.any()):
                glp = LPB.t[torch.from_numpy(gidx)[stepped].cuda()].cpu()
                want = got_w.cpu()[stepped].to(LPB.dtype)
                assert torch.equal(glp.view(INT_VIEW[LPB.dtype]), want.view(INT_VIEW[LPB.dtype]))
        if found_inf:   # a skipped step: master and state bit-identical
            assert torch.equal(MB.bits(), snap["M"]) and torch.equal(MM.bits(), snap["MM"])
    assert hit == muts, f"deliberately wrong updates that passed every step: {muts - hit}"


def test_lion_kernel_rejects_a_missing_exp_avg(eng):
    from stoke_b200.engine import StokeB200Error

    L = _L()
    MB, GB = Buf(64, F32, torch.zeros(64).cuda()), Buf(64, F32)
    hyp = (L.OptimHyper * 1)(_hyper(BASE))
    a = L.OptimArgs()
    a.hyper, a.n_groups = hyp, 1
    a.master, a.exp_avg, a.exp_avg_sq = MB.ptr(), None, None
    a.grad, a.grad_dtype, a.grad_raw, a.grad_mul = GB.ptr(), L.F32, 0, 1.0
    a.n_local = 64
    with pytest.raises(StokeB200Error):
        eng.optim_step_ex(a)


# ---- engine level ------------------------------------------------------------------------------------------------------------
from test_gpu_engine import OddNet, _inject, _oracle_flat, _rel  # noqa: E402

ENGINE_CASES = [
    ({"lr": 1e-3}, torch.bfloat16, ("norm", 1.0, 2.0), 1),
    ({"lr": 1e-3, "betas": (0.95, 0.98), "weight_decay": 0.1}, None, ("value", 0.3), 2),
    ({"lr": 3e-4, "weight_decay": 0.5, "maximize": True}, torch.bfloat16, None, 2),
    ({"lr": 1e-3, "betas": (0.9, 0.99)}, None, ("norm", 0.5, float("inf")), 1),
]


def _fused(net, kw, lp, clip=None, accum=1, route=None, stock=False):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    spec = None
    if clip is not None:
        spec = ClipSpec(_lib.CLIP_NORM, max_norm=clip[1], norm_type=clip[2]) if clip[0] == "norm" else \
            ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1])
    if stock:
        return B200StockOptimizer(net, Lion, kw, engine=get_engine(0), grad_accum=accum, clip=spec, lp_dtype=lp)
    return B200FusedOptimizer(net, Lion, kw, engine=get_engine(0), grad_accum=accum, clip=spec, lp_dtype=lp, route=route)


def _check_state(sd, oracle):
    for i, p in enumerate(oracle.params):
        st = oracle.optimizer.state.get(p, {})
        if not st:
            assert i not in sd["state"], i   # never stepped: no entry
            continue
        got = sd["state"][i]
        assert set(got) == {"step", "exp_avg"} == set(st)
        assert got["step"].dtype == torch.float32 and got["step"].dim() == 0 and float(got["step"]) == float(st["step"])
        assert _rel(got["exp_avg"].cpu(), st["exp_avg"]) < TOL


@pytest.mark.parametrize("route", ["local", "main"])
@pytest.mark.parametrize("kw,lp,clip,accum", ENGINE_CASES)
def test_gradient_injection_parity(kw, lp, clip, accum, route):
    from engine_oracle import OracleEngine
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    net = OddNet().cuda()
    init = [p.detach().cpu().clone() for p in net.parameters()]
    opt = _fused(net, kw, lp, clip, accum, route=route)
    assert isinstance(opt, B200FusedOptimizer) and opt.path.route == route and opt.path.v_flat is None
    path = opt.path
    oracle = OracleEngine(init, 1, Lion, kw, grad_accum=accum, clip=clip)
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


def _mse(out, y):
    return (out.float() - y).pow(2).mean()


@pytest.mark.parametrize("accum", [1, 2])
@pytest.mark.parametrize("clip", [None, ("norm", 1.0, 2.0), ("value", 0.2)], ids=["noclip", "norm", "value"])
@pytest.mark.parametrize("fp16", [None, "bf16"], ids=["fp32", "bf16"])
def test_stoke_facade_with_unused_parameter(fp16, clip, accum):
    """Through the public Stoke calls (model / loss / backward / step).  Head b receives no gradient on the first two
    steps and on some later ones, so step counts go per parameter as torch keeps them; a parameter not yet stepped has no
    state entry; master weights and state follow the CPU oracle fed with the same gradients."""
    from engine_oracle import OracleEngine
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    model = TwoHeads()
    kw = {"lr": 5e-3, "weight_decay": 0.1}
    grad_clip = None
    if clip is not None:
        grad_clip = sb.ClipGradNormConfig(max_norm=clip[1], norm_type=clip[2]) if clip[0] == "norm" else \
            sb.ClipGradConfig(clip_value=clip[1])
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=Lion, optimizer_kwargs=kw), loss=_mse,
                 batch_size_per_device=8, grad_accum_steps=accum, grad_clip=grad_clip, gpu=True, fp16=fp16, verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    path = s.optimizer.path
    dt = torch.bfloat16 if fp16 else torch.float32
    oracle = OracleEngine(path.unflatten(path.gather_master().cpu()), 1, Lion, kw, grad_accum=accum, clip=clip)
    g = torch.Generator().manual_seed(0)
    batches = [(torch.randn(8, 16, generator=g).cuda().to(dt), torch.randn(8, 1, generator=g).cuda()) for _ in range(accum)]
    losses = []
    for step in range(12):
        model.use_b = step >= 2 and step % 4 != 1
        for x, y in batches:
            loss = s.loss(s.model(x), y)
            grads = torch.autograd.grad(loss, path.params, retain_graph=True, allow_unused=True)
            oracle.micro_step([[None if gr is None else gr.detach().float().cpu() for gr in grads]])
            s.backward(loss)
            s.step()
            losses.append(float(loss.detach()))
        oracle.step()
        if step == 1:   # head b never stepped yet: no state entry
            sd = s.optimizer.state_dict()
            assert 4 not in sd["state"] and 5 not in sd["state"] and 0 in sd["state"]
    got = path.gather_master().cpu()
    assert _rel(got, _oracle_flat(path, oracle.weights())) < TOL
    if fp16:
        assert torch.equal(path.p_flat.cpu(), got.to(torch.bfloat16))
    sd = s.optimizer.state_dict()
    _check_state(sd, oracle)
    assert [float(sd["state"][j]["step"]) for j in range(6)] == [12.0] * 4 + [8.0, 8.0]
    assert losses[-1] < losses[2 * accum]
    s.optimizer.close()


def _run_injected(opt, steps, cpu_params=None, topt=None):
    path = opt.path
    for step in steps:
        grads = _inject(path, step, 0, torch.float32)
        if topt is not None:
            for p, gr in zip(cpu_params, grads):
                p.grad = gr.reshape(p.shape).clone()
            topt.step()
        path.after_backward(sync=True, unscale=False)
        opt.step()


def test_checkpoints_fused_plain_fused_match_continuous_runs():
    """Fused (4 steps) -> plain Lion (4 steps, the fused run alongside) -> fused again (4 steps, plain alongside): every
    leg matches its partner, and the final weights match one continuous fused run and one continuous plain run."""
    torch.cuda.set_device(0)
    kw = {"lr": 1e-3, "betas": (0.9, 0.95), "weight_decay": 0.1}
    # continuous runs
    net_c = OddNet().cuda()
    cont_plain = [torch.nn.Parameter(p.detach().cpu().clone()) for p in net_c.parameters()]
    topt_c = Lion(cont_plain, **kw)
    opt_c = _fused(net_c, kw, None)
    _run_injected(opt_c, range(12), cont_plain, topt_c)
    cont_fused = opt_c.path.unflatten(opt_c.path.gather_master().cpu())
    opt_c.close()
    # fused -> plain
    net = OddNet().cuda()
    opt = _fused(net, kw, None)
    _run_injected(opt, range(4))
    sd = opt.state_dict()
    assert set(sd["state"][0]) == {"step", "exp_avg"} and float(sd["state"][0]["step"]) == 4.0
    cpu_params = [torch.nn.Parameter(w.cpu().clone()) for w in opt.path.unflatten(opt.path.gather_master())]
    topt = Lion(cpu_params, **kw)
    topt.load_state_dict({k: v for k, v in sd.items() if not k.startswith("b200_")})
    _run_injected(opt, range(4, 8), cpu_params, topt)
    for a, b in zip(opt.path.unflatten(opt.path.gather_master().cpu()), cpu_params):
        assert _rel(a.reshape(-1), b.detach().reshape(-1)) < TOL
    opt.close()
    # plain -> fused (a plain state dict: no b200_* keys, the model weights loaded first)
    net2 = OddNet().cuda()
    with torch.no_grad():
        for p, q in zip(net2.parameters(), cpu_params):
            p.copy_(q.detach())
    opt2 = _fused(net2, kw, None)
    opt2.load_state_dict(topt.state_dict())
    _run_injected(opt2, range(8, 12), cpu_params, topt)
    final = opt2.path.unflatten(opt2.path.gather_master().cpu())
    for a, b, c, d in zip(final, cpu_params, cont_fused, cont_plain):
        assert _rel(a.reshape(-1), b.detach().reshape(-1)) < TOL
        assert _rel(a.reshape(-1), c.reshape(-1)) < TOL
        assert _rel(a.reshape(-1), d.detach().reshape(-1)) < TOL
    sd2 = opt2.state_dict()
    for i, p in enumerate(cpu_params):
        assert float(sd2["state"][i]["step"]) == float(topt.state[p]["step"]) == 12.0
        assert _rel(sd2["state"][i]["exp_avg"].cpu(), topt.state[p]["exp_avg"]) < TOL
    opt2.close()


def test_checkpoints_between_fused_and_stock_routes():
    """The stock route (the class's own step on fp32 views of the master) and the fused step read each other's
    checkpoints: fused -> stock and stock -> fused both continue to the weights and state of one continuous plain Lion."""
    torch.cuda.set_device(0)
    kw = {"lr": 1e-3, "betas": (0.9, 0.95), "weight_decay": 0.05}
    net_c = OddNet().cuda()
    plain = [torch.nn.Parameter(p.detach().cpu().clone()) for p in net_c.parameters()]
    topt = Lion(plain, **kw)
    for step in range(6):
        for p, gr in zip(plain, _grads_for(net_c, step)):
            p.grad = gr.reshape(p.shape).clone()
        topt.step()
    for first_stock in (False, True):
        a = _fused(OddNet().cuda(), kw, None, stock=first_stock)
        _run_injected(a, range(3))
        sd = a.state_dict()
        assert set(sd["state"][0]) == {"step", "exp_avg"}
        b = _fused(OddNet().cuda(), kw, None, stock=not first_stock)
        b.load_state_dict(sd)
        _run_injected(b, range(3, 6))
        for x, y in zip(b.path.unflatten(b.path.gather_master().cpu()), plain):
            assert _rel(x.reshape(-1), y.detach().reshape(-1)) < TOL
        sd_b = b.state_dict()
        for i, p in enumerate(plain):
            assert float(sd_b["state"][i]["step"]) == float(topt.state[p]["step"]) == 6.0
            assert _rel(sd_b["state"][i]["exp_avg"].cpu().reshape(-1), topt.state[p]["exp_avg"].reshape(-1)) < TOL
        a.close()
        b.close()


def _grads_for(net, step):
    """The fp32 gradients _inject writes for ``step`` (same seeds), without an engine."""
    from stoke_b200 import synthetic

    return [synthetic.injected_grad(p.numel(), 0, step * 100 + i, dtype=torch.float32).float()
            for i, p in enumerate(net.parameters())]


def test_plain_checkpoint_with_unstepped_parameter():
    """A plain Lion state where parameter 0 was never stepped (no entry) and parameter 1 took fewer steps: the fused
    optimizer goes per parameter, creates parameter 0's state at its first gradient like Lion, and continues exactly
    like the plain class."""
    torch.cuda.set_device(0)
    kw = {"lr": 1e-3, "weight_decay": 0.1}
    net = OddNet().cuda()
    cpu_params = [torch.nn.Parameter(p.detach().cpu().clone()) for p in net.parameters()]
    topt = Lion(cpu_params, **kw)
    gen = torch.Generator().manual_seed(4)
    for step in range(5):
        for i, p in enumerate(cpu_params):
            p.grad = None if (i == 0 or (i == 1 and step < 3)) else torch.randn(p.shape, generator=gen) * 1e-2
        topt.step()
    assert cpu_params[0] not in topt.state
    with torch.no_grad():
        for p, q in zip(net.parameters(), cpu_params):
            p.copy_(q.detach())
    opt = _fused(net, kw, None)
    opt.load_state_dict(topt.state_dict())
    assert opt.path._range_steps is not None
    _run_injected(opt, range(5, 9), cpu_params, topt)
    for a, b in zip(opt.path.unflatten(opt.path.gather_master().cpu()), cpu_params):
        assert _rel(a.reshape(-1), b.detach().reshape(-1)) < TOL
    sd = opt.state_dict()
    for i, p in enumerate(cpu_params):
        assert float(sd["state"][i]["step"]) == float(topt.state[p]["step"])
    assert [float(sd["state"][i]["step"]) for i in range(3)] == [4.0, 6.0, 9.0]
    opt.close()


def test_step_makes_no_host_sync():
    net = OddNet().cuda()
    opt = _fused(net, {"lr": 1e-3, "weight_decay": 0.1}, torch.bfloat16, ("norm", 0.5, 2.0))
    path = opt.path
    for step in range(3):
        _inject(path, step, 0, torch.bfloat16)
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
    assert bool(torch.isfinite(path.gather_master()).all())
    opt.close()


@pytest.mark.parametrize("avg", ["ema0.999", "ema0.3", "swa"])
@pytest.mark.parametrize("lp", [torch.bfloat16, None], ids=["bf16", "fp32"])
def test_weight_average_matches_averaged_model(monkeypatch, lp, avg):
    """Lion with WeightAverageConfig: the average equals AveragedModel over the master bit for bit, and averaging changes
    nothing else the step computes (the harness of test_gpu_weight_average.py, with Lion added to its classes)."""
    import test_gpu_weight_average as twa

    monkeypatch.setitem(twa.OPTS, "lion", (Lion, {"lr": 1e-3, "weight_decay": 0.1}))
    with_avg = twa._run("lion", lp, avg)
    without = twa._run("lion", lp, None)
    assert len(with_avg) == len(without)
    for a, b in zip(with_avg, without):
        assert twa._equal(a, b)


@pytest.mark.multigpu
def test_sharded_matches_replicated_w2(tmp_path):
    """fairscale_oss at W = 2: Lion sharded (ZeRO-1, in-kernel parameter all-gather) against Lion replicated (all-reduce
    route): final weights and the gathered state_dict bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "lion_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29567", os.path.join(ROOT, "tests", "lion_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    assert set(res) == {"lion", "lion_wd_max"}
    for name, r in res.items():
        assert r["sharded_route"] == "sharded" and r["replicated_route"] == "allreduce", (name, r)
        assert r["weights_identical"] and r["state_identical"], (name, r)
