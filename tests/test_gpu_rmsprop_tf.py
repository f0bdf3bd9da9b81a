"""stoke_b200.RMSpropTF on the fused step (GPU).

Rounding probe: the CUDA ops the class is written with, pinned against explicit fp32 formulas.  Kernel level:
stk_rmsprop_tf_step called directly, the buffers between guard bands (see test_gpu_kernels.py), compared bit for bit
with the class's ``step()`` on CUDA fp32 tensors restarted from the kernel's own state every step.  Engine level: the
Stoke facade against the same class on the stock route (9 groups), with clip and gradient accumulation; checkpoints
continued on the fused step, the plain class and the stock route; the weight average on top; a step without host
synchronisation; the EfficientNet recipe end to end on a bf16 channels-last MBConv model; the sharded W = 2 run."""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import stoke_b200 as sb
from stoke_b200.optim import RMSpropTF
from test_gpu_kernels import BF16, F32, INT_VIEW, Buf, _dt, _layout

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _L():
    from stoke_b200 import _lib

    return _lib


def _same(a, b):
    """Bit for bit; a NaN matches a NaN."""
    a, b = a.cpu(), b.cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def _fma(a, b, c):
    """fp32 fma(a, b, c) through float64: the product of two fp32 values is exact there."""
    return (a.double() * b.double() + c.double()).float()


def test_probe_cuda_rounding_of_the_class_ops():
    """What the kernel relies on, on this GPU: ``pow(2)`` is g * g; ``add_(x, alpha=a)`` and ``addcdiv_`` contract to one
    FFMA (on the rounded quotient); ``addcmul(t, t, value=-1)`` rounds t * t first; ``add(eps).sqrt_()`` and ``/`` are
    IEEE.  Each contracted form must also differ from the uncontracted one somewhere, so the probe can tell them apart."""
    torch.cuda.set_device(0)
    g = torch.Generator(device="cuda").manual_seed(3)
    n = 1 << 16
    x = torch.randn(n, device="cuda", generator=g)
    s = torch.rand(n, device="cuda", generator=g) + 0.5
    t = torch.randn(n, device="cuda", generator=g) * 0.3
    a = 1 - 0.9   # python double, rounded to fp32 by torch
    a32 = torch.tensor(a, dtype=torch.float32, device="cuda")
    assert torch.equal(x.pow(2).view(torch.int32), (x * x).view(torch.int32))
    d = x * x - s
    got = s.clone().add_(d, alpha=a)
    assert _same(got, _fma(a32, d, s)) and not _same(got, s + a32 * d)
    q = x / s
    assert _same(q, (x.double() / s.double()).float())
    for c in (0.016, 1.0, -0.016):
        c32 = torch.tensor(c, dtype=torch.float32, device="cuda")
        got = t.clone().addcdiv_(x, s, value=c)
        assert _same(got, _fma(c32, q, t)), c
        if c != 1.0:
            assert not _same(got, t + c32 * q), c
    got = s.addcmul(t, t, value=-1)
    assert _same(got, s - t * t) and not _same(got, _fma(-t, t, s))
    eps = torch.tensor(1e-3, dtype=torch.float32, device="cuda")
    got = s.add(1e-3).sqrt_()
    assert _same(got, (s + eps).double().sqrt().float())


def _hyper(h, clip=None):
    L = _L()
    o = L.OptimHyper()
    o.kind = L.OPT_RMSPROP_TF
    o.lr, o.eps, o.weight_decay, o.momentum = h["lr"], h["eps"], h["weight_decay"], h["momentum"]
    o.clip_kind = L.CLIP_NONE
    if clip is not None:
        o.clip_kind = L.CLIP_NORM if clip[0] == "norm" else L.CLIP_VALUE
        o.clip_max_norm = clip[1] if clip[0] == "norm" else 0.0
        o.clip_value = clip[1] if clip[0] == "value" else 0.0
    return o


def _rhyper(h):
    x = _L().RmspropTfHyper()
    x.alpha = h["alpha"]
    x.centered, x.decoupled_decay = int(h["centered"]), int(h["decoupled_decay"])
    x.lr_in_momentum = int(h["lr_in_momentum"])
    return x


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


def _g(**kw):
    return dict(dict(lr=1e-2, alpha=0.9, eps=1e-3, weight_decay=0.0, momentum=0.0, centered=False,
                     decoupled_decay=False, lr_in_momentum=True), **kw)


RECIPE = _g(lr=0.016, momentum=0.9, weight_decay=1e-5)
# eight groups: every flag both ways
G8 = [RECIPE,
      _g(lr=3e-3, alpha=0.95, eps=1e-8, centered=True, weight_decay=5e-2, decoupled_decay=True),
      _g(lr=5e-3, momentum=0.8, centered=True, lr_in_momentum=False, weight_decay=1e-2),
      _g(lr=2e-2, alpha=0.99, eps=1e-6, momentum=0.5, lr_in_momentum=False, decoupled_decay=True, weight_decay=0.1),
      _g(lr=1e-3, eps=1e-10),
      _g(lr=1e-2, momentum=0.9, centered=True, weight_decay=1e-4),
      _g(lr=4e-3, alpha=0.5, eps=0.0, momentum=0.7, lr_in_momentum=False),
      _g(lr=6e-3, alpha=0.8, centered=True, decoupled_decay=True, weight_decay=1e-3)]
G3 = [G8[2], G8[4], G8[1]]

# name: gradient source, model copy, n_local, segments, groups, range table, per-parameter counts (with skip bits),
#       fp32 accumulator, found_inf step, clip, special gradient elements (zero, +-inf, NaN)
CASES = {
    "raw_bf16_recipe": ("raw_bf16", "bf16", 2_056, 0, [RECIPE], False, False, False, 7, None, False),
    "main_8groups_per_param_clip_norm": ("main", "f32", 2_048, 7, G8, True, True, False, 11, ("norm", 0.05), False),
    "raw_bf16_8groups_per_param_clip_value": ("raw_bf16", "bf16", 2_048, 64, G8, True, True, False, None,
                                              ("value", 4e-3), False),
    "raw_f32_acc_3groups": ("raw_f32", None, 2_056, 5, G3, True, False, True, 3, None, False),
    "main_plain_no_m_no_m2": ("main", None, 2_040, 3, [G8[4]], False, False, False, None, ("norm", 10.0), False),
    "main_centered_momentum_only": ("main", None, 2_040, 2, [G8[5], G8[2]], True, False, False, None, None, False),
    "raw_bf16_8groups_specials_eps0": ("raw_bf16", "bf16", 2_048, 4, [dict(h, eps=0.0) for h in G8], True, True, False,
                                       None, None, True),
}
STEPS = 24


@pytest.mark.parametrize("name", list(CASES))
def test_rmsprop_tf_kernel_matches_cuda_class_bit_for_bit(eng, name):
    L = _L()
    src, lp, n_local, n_seg, groups, use_ranges, per_range, use_acc, inf_at, clip, specials = CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    pieces, N = _layout(n_local, n_seg, rng, base=64)
    N = -(-N // 16) * 16
    gidx = np.concatenate([np.arange(g0, g0 + (l1 - l0)) for l0, l1, g0 in pieces])
    ng = len(groups)
    if use_ranges:
        nr = 12
        ends = sorted(rng.choice(np.arange(1, N // 16), nr - 1, replace=False).tolist()) + [N // 16]
        ends = [e * 16 for e in ends]
        rgroup = [j % ng for j in range(nr)]
    else:
        ends, rgroup = [N], [0]
    elem_range = np.searchsorted(np.asarray(ends), gidx, side="right")
    ranges = [j for j in range(len(ends)) if bool((elem_range == j).any())]
    hyp = (L.OptimHyper * ng)(*[_hyper(h, clip) for h in groups])
    rhyp = (L.RmspropTfHyper * ng)(*[_rhyper(h) for h in groups])
    has_m, has_m2 = any(h["momentum"] > 0 for h in groups), any(h["centered"] for h in groups)
    w0 = torch.from_numpy(rng.standard_normal(n_local).astype(np.float32) * 1e-1)
    MB = Buf(n_local, F32, w0.cuda())
    VB = Buf(n_local, F32, torch.ones(n_local).cuda())
    BUF = Buf(n_local, F32, torch.zeros(n_local).cuda()) if has_m else None
    GA = Buf(n_local, F32, torch.zeros(n_local).cuda()) if has_m2 else None
    LPB = None if lp is None else Buf(N, BF16 if lp == "bf16" else F32, torch.full((N,), -5.0))
    gdt = {"raw_bf16": BF16, "raw_f32": F32, "main": F32}[src]
    GB = Buf(N if src != "main" else n_local, gdt)
    AB = Buf(N, F32) if use_acc else None
    BC = Buf(len(ends) * 4, F32, torch.full((len(ends) * 4,), float("nan")).cuda()) if per_range else None
    rend = torch.tensor([e // 8 for e in ends], dtype=torch.int32).cuda()
    rsteps = torch.zeros(len(ends), dtype=torch.int32).cuda()
    sl = (C.c_size_t * (len(pieces) + 1))(*([p[0] for p in pieces] + [n_local]))
    sg = (C.c_size_t * len(pieces))(*[p[2] for p in pieces])
    lpp = L.ptr_array([LPB.ptr()]) if lp is not None else None
    grad_norm = 1.5
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0, grad_norm=grad_norm)
    masks = {j: torch.from_numpy(elem_range == j).cuda() for j in ranges}
    ref_params = {j: torch.nn.Parameter(w0.cuda()[masks[j]].clone()) for j in ranges}
    ref = RMSpropTF([dict(h, params=[ref_params[j] for j in ranges if rgroup[j] == gi]) for gi, h in enumerate(groups)])
    coef = None
    if clip is not None and clip[0] == "norm":
        coef = min(np.float32(clip[1]) / (np.float32(grad_norm) + np.float32(1e-6)), np.float32(1.0))
    g32 = rng.standard_normal(n_local).astype(np.float32)
    if specials:   # exact zeros, +-inf and NaN in a few elements of every step's gradient
        sp = rng.choice(n_local, 12, replace=False)
        g32[sp[:6]] = 0.0
        g32[sp[6:8]] = np.inf
        g32[sp[8:10]] = -np.inf
        g32[sp[10:]] = np.nan
    done, entry_done = 0, [0] * len(ends)
    grp_of_range = np.asarray(rgroup)
    no_mom = torch.from_numpy(np.asarray([not (groups[g]["momentum"] > 0) for g in grp_of_range])[elem_range])
    plain = torch.from_numpy(np.asarray([not groups[g]["centered"] for g in grp_of_range])[elem_range])
    for step in range(STEPS):
        skip = {j for j in ranges if (j + step) % 5 == 1} if per_range else set()
        rgrp = torch.tensor([g | (0x80 if j in skip else 0) for j, g in enumerate(rgroup)], dtype=torch.uint8).cuda()
        g = torch.from_numpy((np.roll(g32, step * 37) * 1e-2).astype(np.float32)).to(gdt)
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
        w, v = MB.t.clone(), VB.t.clone()
        buf = BUF.t.clone() if BUF is not None else None
        ga = GA.t.clone() if GA is not None else None
        snap = {k: b.bits() for k, b in (("W", MB), ("V", VB), ("BUF", BUF), ("GA", GA), ("LP", LPB)) if b}
        if per_range:   # per-parameter step counts: the shared prologue keeps them (an all-zero row for this kind)
            eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, None, ng, len(ends), rgrp.data_ptr(),
                                                       rsteps.data_ptr(), None, BC.ptr(), eng._stream()))
        a = L.OptimArgs()
        a.hyper, a.n_groups = hyp, ng
        a.master, a.exp_avg_sq = MB.ptr(), VB.ptr()
        a.exp_avg = BUF.ptr() if BUF is not None else None
        a.exp_avg_slow = GA.ptr() if GA is not None else None
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
        eng.rmsprop_tf_step(a, rhyp)
        eng.step_epilogue()
        got = {"W": MB.t.clone(), "V": VB.t.clone()}
        if BUF is not None:
            got["BUF"] = BUF.t.clone()
        if GA is not None:
            got["GA"] = GA.t.clone()
        if per_range:
            BC.check_guards()
            assert float(BC.t.abs().max()) == 0.0   # the prologue's row for this kind: no per-step scalars
            for k in range(len(ends)):
                if not found_inf and k not in skip:
                    entry_done[k] += 1
            assert rsteps.cpu().tolist() == entry_done
        # ---- the reference step (not taken at all on a found_inf step, like GradScaler.step) ----
        gl = g.float()
        if acc_local is not None:
            gl = gl + acc_local                       # the kernel's raw + accumulator sum, one fp32 add
        gl = gl.cuda()
        if coef is not None:
            gl = gl * torch.tensor(coef, dtype=torch.float32, device="cuda")
        elif clip is not None:
            gl = gl.clamp(-clip[1], clip[1])
        for j in ranges:
            p = ref_params[j]
            p.data.copy_(w[masks[j]])
            p.grad = None if j in skip else gl[masks[j]].clone()
            st = ref.state[p]
            if st:   # restart from the kernel's state
                st["square_avg"] = v[masks[j]].clone()
                if "momentum_buffer" in st:
                    st["momentum_buffer"] = buf[masks[j]].clone()
                if "grad_avg" in st:
                    st["grad_avg"] = ga[masks[j]].clone()
        if not found_inf:
            ref.step()
            done += 1
        assert int(eng.scaler_get().opt_steps) == done
        want = {"W": w.clone(), "V": v.clone()}
        if buf is not None:
            want["BUF"] = buf.clone()
        if ga is not None:
            want["GA"] = ga.clone()
        for j in ranges:
            p, s = ref_params[j], masks[j]
            want["W"][s] = p.detach()
            st = ref.state[p]
            if not st:
                continue
            want["V"][s] = st["square_avg"]
            h = groups[rgroup[j]]
            assert ("momentum_buffer" in st) == (h["momentum"] > 0) and ("grad_avg" in st) == h["centered"]
            if "momentum_buffer" in st:
                want["BUF"][s] = st["momentum_buffer"]
            if "grad_avg" in st:
                want["GA"][s] = st["grad_avg"]
        for key in got:
            assert _same(got[key], want[key]), f"step {step}: {key}"
        # ---- where the kernel wrote: nothing for skipped ranges, a found_inf step, or a buffer the group lacks ----
        skip_elem = torch.from_numpy(np.isin(elem_range, list(skip))) | found_inf
        for key, b in (("W", MB), ("V", VB)):
            b.check_unchanged_except(snap[key], ~skip_elem)
        if BUF is not None:
            BUF.check_unchanged_except(snap["BUF"], ~skip_elem & ~no_mom)
        if GA is not None:
            GA.check_unchanged_except(snap["GA"], ~skip_elem & ~plain)
        if src != "main":
            assert float(GB.t[torch.from_numpy(gidx).cuda()].float().abs().max()) == 0.0
        if LPB is not None:
            stepped = ~skip_elem
            mask = torch.zeros(LPB.n, dtype=torch.bool)
            mask[torch.from_numpy(gidx)[stepped]] = True
            LPB.check_unchanged_except(snap["LP"], mask)
            if bool(stepped.any()):
                glp = LPB.t[torch.from_numpy(gidx)[stepped].cuda()].cpu()
                wl = got["W"].cpu()[stepped].to(LPB.dtype)
                # a NaN master element is a NaN in the copy (the kernel's cast writes the canonical bf16 NaN, 0x7fff)
                nan = torch.isnan(wl)
                assert torch.equal(torch.isnan(glp), nan)
                assert torch.equal(glp[~nan].view(INT_VIEW[LPB.dtype]), wl[~nan].view(INT_VIEW[LPB.dtype]))
        if found_inf:
            assert all(torch.equal(b.bits(), snap[k]) for k, b in (("W", MB), ("V", VB)))
    assert done == STEPS - (inf_at is not None)
    if specials:
        assert bool(torch.isnan(MB.t).any()) and bool(torch.isfinite(MB.t).any())


def test_entry_points_require_their_buffers(eng):
    from stoke_b200.engine import StokeB200Error

    L = _L()
    bufs = [Buf(64, F32, torch.zeros(64).cuda()) for _ in range(5)]
    mom_centered = _g(momentum=0.9, centered=True)

    def args(h, m, m2, v):
        a = L.OptimArgs()
        a.hyper, a.n_groups = (L.OptimHyper * 1)(_hyper(h)), 1
        a.master, a.grad, a.grad_dtype, a.n_local = bufs[0].ptr(), bufs[1].ptr(), L.F32, 64
        a.exp_avg = bufs[2].ptr() if m else None
        a.exp_avg_slow = bufs[3].ptr() if m2 else None
        a.exp_avg_sq = bufs[4].ptr() if v else None
        return a

    rh = (L.RmspropTfHyper * 1)(_rhyper(mom_centered))
    for m, m2, v in ((False, True, True), (True, False, True), (True, True, False)):
        with pytest.raises(StokeB200Error):
            eng.rmsprop_tf_step(args(mom_centered, m, m2, v), rh)
    with pytest.raises(StokeB200Error, match="stk_rmsprop_tf_step"):   # the kind's hyper-parameters have one entry point
        eng.optim_step_ex(args(mom_centered, True, True, True))
    adam = args(mom_centered, True, True, True)
    adam.hyper[0].kind = L.OPT_ADAM
    with pytest.raises(StokeB200Error):
        eng.rmsprop_tf_step(adam, rh)
    # no momentum, not centered: square_avg alone is enough, and no group_bc is needed
    eng.rmsprop_tf_step(args(_g(), False, False, True), (L.RmspropTfHyper * 1)(_rhyper(_g())))
    torch.cuda.synchronize()


# ---- engine level ------------------------------------------------------------------------------------------------------------
from test_gpu_engine import OddNet, _inject, _rel  # noqa: E402


class Net(torch.nn.Module):
    """Eight parameters in use and one Linear the forward never calls."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(5)
        self.layers = torch.nn.ModuleList([torch.nn.Linear(16, 24), torch.nn.Linear(24, 24), torch.nn.Linear(24, 24),
                                           torch.nn.Linear(24, 1)])
        self.unused = torch.nn.Linear(4, 4)

    def forward(self, x):
        for i, m in enumerate(self.layers):
            x = m(x)
            if i < 3:
                x = torch.tanh(x)
        return x


def _mse(out, y):
    return (out.float() - y).pow(2).mean()


FACADE_KW = {"lr": 5e-3, "alpha": 0.9, "eps": 1e-3, "momentum": 0.9, "centered": True, "weight_decay": 1e-2}


def _stoke(fp16, clip, accum, stock, wa=None, kw=FACADE_KW):
    model = Net()
    used = [p for m in model.layers for p in m.parameters()]
    unused = dict(params=list(model.unused.parameters()), weight_decay=0.0, momentum=0.0, centered=False)
    if stock:   # 9 groups: more than the fused step takes, so Stoke builds the stock route
        groups = [dict(params=[p]) for p in used] + [unused]
    else:
        groups = [dict(params=used), unused]
    grad_clip = None
    if clip is not None:
        grad_clip = sb.ClipGradNormConfig(max_norm=clip[1], norm_type=2.0) if clip[0] == "norm" else \
            sb.ClipGradConfig(clip_value=clip[1])
    return sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=RMSpropTF, optimizer_kwargs=dict(kw, params=groups)),
                    loss=_mse, batch_size_per_device=8, grad_accum_steps=accum, grad_clip=grad_clip, gpu=True, fp16=fp16,
                    verbose=False, configs=[wa] if wa is not None else None)


def _drive(s, steps, fp16, accum, seed=0, each=None):
    dt = torch.bfloat16 if fp16 else torch.float32
    g = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for _ in range(accum):
            x, y = torch.randn(8, 16, generator=g).cuda().to(dt), torch.randn(8, 1, generator=g).cuda()
            s.backward(s.loss(s.model(x), y))
            s.step()
        if each is not None:
            each(s)


@pytest.mark.parametrize("accum", [1, 2])
@pytest.mark.parametrize("clip", [None, ("value", 0.05), ("norm", 0.5)], ids=["noclip", "value", "norm"])
@pytest.mark.parametrize("fp16", [None, "bf16"], ids=["fp32", "bf16"])
def test_stoke_facade_matches_stock_route(fp16, clip, accum):
    """The fused step and the class's own step on the stock route (9 groups) give the same master and the same three
    state tensors bit for bit over 9 steps; the never-used parameter keeps its weights, has no state entry, and its
    square_avg stays at ones.  Clip by norm takes its norm from different kernels on the two routes, so there the bar is
    fp32 tolerance."""
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    torch.cuda.set_device(0)
    runs = []
    for stock in (False, True):
        s = _stoke(fp16, clip, accum, stock)
        assert isinstance(s.optimizer, B200StockOptimizer if stock else B200FusedOptimizer)
        _drive(s, 9, fp16, accum)
        runs.append((s, s.optimizer.path.gather_master().cpu(), s.optimizer.state_dict()))
    (fs, fw, fsd), (ss, sw, ssd) = runs
    exact = clip is None or clip[0] == "value"
    assert _same(fw, sw) if exact else _rel(fw, sw) < 1e-5
    keys = ("square_avg", "momentum_buffer", "grad_avg")
    for i in range(8):
        assert set(fsd["state"][i]) == set(keys) | {"step"} == set(ssd["state"][i])
        assert float(fsd["state"][i]["step"]) == 9 == float(ssd["state"][i]["step"])
        for k in keys:
            a, b = fsd["state"][i][k].cpu(), ssd["state"][i][k].cpu()
            assert _same(a, b) if exact else _rel(a, b) < 1e-5, (i, k)
    assert 8 not in fsd["state"] and 9 not in fsd["state"]   # the unused Linear: never stepped
    path = fs.optimizer.path
    init = Net().unused
    got = path.unflatten(path.gather_master().cpu())
    assert torch.equal(got[8], init.weight.detach()) and torch.equal(got[9], init.bias.detach())
    sq = path.unflatten(path.v_flat.cpu())
    assert bool((sq[8] == 1).all()) and bool((sq[9] == 1).all())
    for s in (fs, ss):
        s.optimizer.close()


def _fused(net, kw, lp=None, stock=False, accum=1):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    cls = B200StockOptimizer if stock else B200FusedOptimizer
    return cls(net, RMSpropTF, kw, engine=get_engine(0), grad_accum=accum, lp_dtype=lp)


def _run_injected(opt, steps, plain=None, topt=None):
    path = opt.path
    for step in steps:
        grads = _inject(path, step, 0, torch.float32)
        if topt is not None:
            for p, gr in zip(plain, grads):
                p.grad = gr.reshape(p.shape).cuda()
            topt.step()
        path.after_backward(sync=True, unscale=False)
        opt.step()


def _masters(opt):
    return [t.reshape(-1) for t in opt.path.unflatten(opt.path.gather_master().cpu())]


def _ckpt_kw(net):
    """Two groups: the recipe with centered, and a plain one (no momentum, decoupled decay)."""
    ps = list(net.parameters())
    return dict(lr=1e-2, alpha=0.9, eps=1e-3, weight_decay=1e-4,
                params=[dict(params=ps[:4], momentum=0.9, centered=True),
                        dict(params=ps[4:], momentum=0.0, decoupled_decay=True, weight_decay=0.05, alpha=0.95)])


def _int_steps(sd):
    """The state dict as timm writes it: ``step`` a python int."""
    return dict(sd, state={i: dict(e, step=int(float(e["step"]))) for i, e in sd["state"].items()})


def test_checkpoints_continue_bit_for_bit():
    """A checkpoint saved after 4 steps continues like the uninterrupted 12-step run, bit for bit: fused -> fused (with
    timm's int ``step``), fused -> plain class (4 steps) -> fused (4 steps), and fused -> stock -> fused.  The second
    group has neither momentum_buffer nor grad_avg in its entries."""
    torch.cuda.set_device(0)

    def make(stock=False, net=None):
        net = net if net is not None else OddNet().cuda()
        return _fused(net, _ckpt_kw(net), stock=stock)

    cont = make()
    _run_injected(cont, range(12))
    want = _masters(cont)
    want_sd = cont.state_dict()
    cont.close()

    first = make()
    _run_injected(first, range(4))
    sd = first.state_dict()
    for i, e in sd["state"].items():
        assert list(e) == (["step", "square_avg", "momentum_buffer", "grad_avg"] if i < 4 else ["step", "square_avg"])
        assert float(e["step"]) == 4
    again = make()
    again.load_state_dict(_int_steps(sd))
    _run_injected(again, range(4, 12))
    assert all(_same(a, b) for a, b in zip(_masters(again), want))
    again.close()
    # fused -> plain class -> fused
    plain = [torch.nn.Parameter(w.cuda().clone()) for w in first.path.unflatten(first.path.gather_master())]
    topt = RMSpropTF(**_ckpt_kw(torch.nn.ParameterList(plain)))
    topt.load_state_dict(_int_steps({k: v for k, v in sd.items() if not k.startswith("b200_")}))
    assert all(torch.is_tensor(e["step"]) and e["step"].dtype == torch.float32 for e in topt.state.values())
    _run_injected(first, range(4, 8), plain, topt)   # the fused run alongside: the same gradients
    for a, b in zip(_masters(first), plain):
        assert _same(a, b.detach().reshape(-1))
    first.close()
    net = OddNet().cuda()
    with torch.no_grad():
        for p, q in zip(net.parameters(), plain):
            p.copy_(q.detach())
    last = make(net=net)
    last.load_state_dict(topt.state_dict())   # a plain state dict: no b200_* keys, the model weights loaded first
    _run_injected(last, range(8, 12))
    assert all(_same(a, b) for a, b in zip(_masters(last), want))
    got_sd = last.state_dict()
    for i, e in want_sd["state"].items():
        assert list(got_sd["state"][i]) == list(e)
        for k in e:
            assert _same(got_sd["state"][i][k], e[k]), (i, k)
    last.close()
    # fused -> stock -> fused
    a = make()
    _run_injected(a, range(4))
    b = make(stock=True)
    b.load_state_dict(a.state_dict())
    _run_injected(b, range(4, 8))
    c = make()
    c.load_state_dict(b.state_dict())
    _run_injected(c, range(8, 12))
    assert all(_same(x, y) for x, y in zip(_masters(c), want))
    for o in (a, b, c):
        o.close()


def test_load_fills_square_avg_with_ones():
    """An entry without ``square_avg`` (or a parameter without an entry) loads as timm's initial state: ones, and zeros
    for the other buffers; the next step equals the plain class's first step there."""
    torch.cuda.set_device(0)
    net = OddNet().cuda()
    opt = _fused(net, _ckpt_kw(net))
    _run_injected(opt, range(2))
    sd = opt.state_dict()
    del sd["state"][1]                            # parameter 1: never stepped as far as the checkpoint knows
    sd["state"][0] = {"step": sd["state"][0]["step"]}   # parameter 0: stepped, buffers missing
    opt.load_state_dict(sd)
    path = opt.path
    sq, buf, ga = (path.unflatten(f.cpu()) for f in (path.v_flat, path.m_flat, path.m2_flat))
    for i in (0, 1):
        assert bool((sq[i] == 1).all()) and bool((buf[i] == 0).all()) and bool((ga[i] == 0).all())
    assert path.param_steps()[:3] == [2, 0, 2]
    opt.close()


def test_weight_average_on_top():
    """An EMA of the weights over the fused RMSpropTF step: the master is the run's without averaging, bit for bit, and
    the average is AveragedModel's update (copy, then torch's fp32 lerp with 1 - decay) applied to every step's master."""
    torch.cuda.set_device(0)
    out = []
    for wa in (None, sb.WeightAverageConfig(kind="ema", decay=0.9)):
        s = _stoke("bf16", None, 2, False, wa=wa)
        ref = []

        def each(s_):
            m = s_.optimizer.path.gather_master()
            if not ref:
                ref.append(m.clone())
            else:
                torch._foreach_lerp_(ref, [m], 1 - 0.9)

        _drive(s, 8, "bf16", 2, each=each)
        path = s.optimizer.path
        out.append(path.gather_master().cpu())
        if wa is not None:
            assert s.weight_average.n_averaged == 8
            assert _same(path.gather_avg().cpu(), ref[0].cpu())
        s.optimizer.close()
    assert _same(out[0], out[1])


def test_step_makes_no_host_sync():
    net = OddNet().cuda()
    opt = _fused(net, _ckpt_kw(net), torch.bfloat16)
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


# ---- the EfficientNet recipe end to end ------------------------------------------------------------------------------------
class MBConv(torch.nn.Module):
    """EfficientNet's inverted residual without squeeze-excitation: expand Conv-BN-SiLU, depthwise Conv-BN-SiLU, projection
    Conv-BN, residual add."""

    def __init__(self, c, e=4):
        super().__init__()
        h = c * e
        self.expand = torch.nn.Sequential(torch.nn.Conv2d(c, h, 1, bias=False), torch.nn.BatchNorm2d(h, eps=1e-3),
                                          torch.nn.SiLU(inplace=True))
        self.dw = torch.nn.Sequential(torch.nn.Conv2d(h, h, 3, padding=1, groups=h, bias=False),
                                      torch.nn.BatchNorm2d(h, eps=1e-3), torch.nn.SiLU(inplace=True))
        self.proj = torch.nn.Sequential(torch.nn.Conv2d(h, c, 1, bias=False), torch.nn.BatchNorm2d(c, eps=1e-3))

    def forward(self, x):
        return x + self.proj(self.dw(self.expand(x)))


class MBNet(torch.nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(21)
        self.stem = torch.nn.Sequential(torch.nn.Conv2d(3, 16, 3, stride=2, padding=1, bias=False),
                                        torch.nn.BatchNorm2d(16, eps=1e-3), torch.nn.SiLU(inplace=True))
        self.blocks = torch.nn.Sequential(MBConv(16), MBConv(16))
        self.head = torch.nn.Linear(16, 10)

    def forward(self, x):
        return self.head(self.blocks(self.stem(x)).mean((2, 3)))


def test_efficientnet_recipe_end_to_end(monkeypatch):
    """A bf16 channels-last MBConv model through Stoke with its BatchNorm sites fused, RMSpropTF with timm's EfficientNet
    settings (weight decay on conv / linear weights only) and an fp32 EMA of the weights: the fused step (2 groups) and
    the class on the stock route (the same settings over 10 groups) give the same master, state and average bit for bit."""
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    torch.cuda.set_device(0)
    try:
        runs = []
        for stock in (False, True):
            model = MBNet().to(memory_format=torch.channels_last)
            decay = [p for p in model.parameters() if p.dim() > 1]
            no_decay = [p for p in model.parameters() if p.dim() <= 1]
            if stock:
                groups = [dict(params=decay[i::5]) for i in range(5)] + \
                    [dict(params=no_decay[i::5], weight_decay=0.0) for i in range(5)]
            else:
                groups = [dict(params=decay), dict(params=no_decay, weight_decay=0.0)]
            kw = dict(lr=0.016, alpha=0.9, eps=1e-3, momentum=0.9, weight_decay=1e-5, params=groups)
            s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=RMSpropTF, optimizer_kwargs=kw),
                         loss=torch.nn.CrossEntropyLoss(), batch_size_per_device=16, gpu=True, fp16="bf16",
                         configs=[sb.WeightAverageConfig(kind="ema", decay=0.99)], verbose=False)
            assert s._forward is not s._model and s._forward.fused_sites > 0, "the BatchNorm sites were not fused"
            g = torch.Generator().manual_seed(9)
            for _ in range(6):
                x = torch.randn(16, 3, 32, 32, generator=g).cuda().contiguous(memory_format=torch.channels_last)
                y = torch.randint(0, 10, (16,), generator=g).cuda()
                s.backward(s.loss(s.model(x), y))
                s.step()
            path = s.optimizer.path
            # state by parameter: torch numbers the state dict's parameters group by group, so the runs differ there
            order = {id(p): i for i, p in enumerate(model.parameters())}
            sd_to_flat = [order[id(p)] for grp in groups for p in grp["params"]]
            state = {sd_to_flat[j]: e for j, e in s.optimizer.state_dict()["state"].items()}
            runs.append((path.params, path.unflatten(path.gather_master().cpu()), state,
                         path.unflatten(path.gather_avg().cpu())))
            s.optimizer.close()
        (pf, wf, sf, af), (ps, ws, ss, as_) = runs
        # both runs register the model's parameters in the same order
        assert [tuple(p.shape) for p in pf] == [tuple(p.shape) for p in ps]
        for i in range(len(pf)):
            assert _same(wf[i], ws[i]), i
            assert _same(af[i], as_[i]), i
            assert set(sf[i]) == {"step", "square_avg", "momentum_buffer"} == set(ss[i])
            for k in ("square_avg", "momentum_buffer"):
                assert _same(sf[i][k], ss[i][k]), (i, k)
    finally:
        torch.use_deterministic_algorithms(det)


@pytest.mark.multigpu
def test_sharded_matches_replicated_w2(tmp_path):
    """fairscale_oss at W = 2: RMSpropTF sharded (ZeRO-1, in-kernel parameter all-gather) against the replicated
    all-reduce route: final weights and the gathered state_dict bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "rmsprop_tf_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29577", os.path.join(ROOT, "tests", "rmsprop_tf_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    assert res["sharded_route"] == "sharded" and res["replicated_route"] == "allreduce", res
    assert res["weights_identical"] and res["state_identical"], res
