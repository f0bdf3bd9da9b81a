"""stoke_b200.AdEMAMix on the fused step (GPU).

Kernel level: stk_ademamix_step_prologue + stk_optim_step_ex called directly, the buffers between guard bands (see
test_gpu_kernels.py), compared bit for bit with the class's ``step()`` on CUDA fp32 tensors restarted from the kernel's
own state every step; the prologue's fp32 scalars against the class's, at every step of the tested warm-ups.  Engine
level: the Stoke facade against the same class on the stock route (9 groups), with gradient accumulation; checkpoints
continued on the fused step, the plain class and the stock route; the weight average on top; a step without host
synchronisation; the sharded W = 2 run."""
import ctypes as C
import math
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import stoke_b200 as sb
from stoke_b200.optim import AdEMAMix, ademamix_schedule
from test_gpu_kernels import BF16, F32, INT_VIEW, Buf, _dt, _layout

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# three groups with different betas, alpha and warm-ups; the second has beta1 == 0 (no exp_avg_fast)
G3 = [dict(lr=2e-2, betas=(0.9, 0.999, 0.9999), alpha=2.0, alpha_warmup=12, beta3_warmup=20, eps=1e-8, weight_decay=0.0),
      dict(lr=1e-2, betas=(0.0, 0.99, 0.999), alpha=5.0, alpha_warmup=None, beta3_warmup=9, eps=1e-6, weight_decay=0.05),
      dict(lr=5e-3, betas=(0.8, 0.95, 0.995), alpha=0.5, alpha_warmup=25, beta3_warmup=None, eps=1e-8, weight_decay=0.1)]


def _L():
    from stoke_b200 import _lib

    return _lib


def _hyper(h, clip=None):
    L = _L()
    o = L.OptimHyper()
    o.kind = L.OPT_ADEMAMIX
    o.lr, o.eps, o.weight_decay = h["lr"], h["eps"], h["weight_decay"]
    o.beta1, o.beta2 = h["betas"][0], h["betas"][1]
    o.clip_kind = L.CLIP_NONE
    if clip is not None:
        o.clip_kind = L.CLIP_NORM if clip[0] == "norm" else L.CLIP_VALUE
        o.clip_max_norm = clip[1] if clip[0] == "norm" else 0.0
        o.clip_value = clip[1] if clip[0] == "value" else 0.0
    return o


def _ahyper(h):
    x = _L().AdemamixHyper()
    x.alpha, x.beta3 = h["alpha"], h["betas"][2]
    x.alpha_warmup, x.beta3_warmup = h["alpha_warmup"] or 0, h["beta3_warmup"] or 0
    return x


def _want_scalars(h, t):
    """The class's per-step scalars at step t, cast to fp32 (what the kernel must read)."""
    b1, b2, _ = h["betas"]
    alpha_t, beta3_t = ademamix_schedule(h, float(t))
    return torch.tensor([1 / (1 - b1 ** t), 1 / math.sqrt(1 - b2 ** t), alpha_t, 1 - beta3_t], dtype=torch.float32)


def _same(a, b):
    """Bit for bit; a NaN matches a NaN."""
    a, b = a.cpu(), b.cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


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


# name: gradient source, model copy, n_local, segments, groups, range table, per-parameter counts (with skip bits),
#       fp32 accumulator, found_inf step, clip
CASES = {
    "raw_bf16_one_group": ("raw_bf16", "bf16", 2_056, 0, [G3[0]], False, False, False, 7, None),
    "main_3groups_per_param_clip_norm": ("main", "f32", 2_048, 7, G3, True, True, False, 11, ("norm", 0.05)),
    "raw_bf16_3groups_per_param_clip_value": ("raw_bf16", "bf16", 2_048, 64, G3, True, True, False, None,
                                              ("value", 4e-3)),
    "raw_f32_acc_3groups": ("raw_f32", None, 2_056, 5, G3, True, False, True, 3, None),
    "main_beta1_zero_no_exp_avg": ("main", None, 2_040, 3, [G3[1]], False, False, False, None, ("norm", 10.0)),
}
STEPS = 32


@pytest.mark.parametrize("name", list(CASES))
def test_ademamix_kernel_matches_cuda_class_bit_for_bit(eng, name):
    L = _L()
    src, lp, n_local, n_seg, groups, use_ranges, per_range, use_acc, inf_at, clip = CASES[name]
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
    ahyp = (L.AdemamixHyper * ng)(*[_ahyper(h) for h in groups])
    has_m = any(h["betas"][0] != 0 for h in groups)
    w0 = torch.from_numpy(rng.standard_normal(n_local).astype(np.float32) * 1e-1)
    MB = Buf(n_local, F32, w0.cuda())
    M1 = Buf(n_local, F32, torch.zeros(n_local).cuda()) if has_m else None
    M2 = Buf(n_local, F32, torch.zeros(n_local).cuda())
    VB = Buf(n_local, F32, torch.zeros(n_local).cuda())
    LPB = None if lp is None else Buf(N, BF16 if lp == "bf16" else F32, torch.full((N,), -5.0))
    gdt = {"raw_bf16": BF16, "raw_f32": F32, "main": F32}[src]
    GB = Buf(N if src != "main" else n_local, gdt)
    AB = Buf(N, F32) if use_acc else None
    n_entries = len(ends) if per_range else ng
    BC = Buf(n_entries * 4, F32, torch.full((n_entries * 4,), float("nan")).cuda())
    rend = torch.tensor([e // 8 for e in ends], dtype=torch.int32).cuda()
    rsteps = torch.zeros(len(ends), dtype=torch.int32).cuda()
    sl = (C.c_size_t * (len(pieces) + 1))(*([p[0] for p in pieces] + [n_local]))
    sg = (C.c_size_t * len(pieces))(*[p[2] for p in pieces])
    lpp = L.ptr_array([LPB.ptr()]) if lp is not None else None
    grad_norm = 1.5
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0, grad_norm=grad_norm)
    masks = {j: torch.from_numpy(elem_range == j).cuda() for j in ranges}
    ref_params = {j: torch.nn.Parameter(w0.cuda()[masks[j]].clone()) for j in ranges}
    ref = AdEMAMix([dict(h, params=[ref_params[j] for j in ranges if rgroup[j] == gi]) for gi, h in enumerate(groups)])
    # the kernel's clip coefficient, fp32 (k1_common.cuh clip_coef), applied to the gradient the class sees
    coef = None
    if clip is not None and clip[0] == "norm":
        coef = min(np.float32(clip[1]) / (np.float32(grad_norm) + np.float32(1e-6)), np.float32(1.0))
    g32 = rng.standard_normal(n_local).astype(np.float32)
    done, entry_done = 0, [0] * n_entries
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
        w, v, s2 = MB.t.clone(), VB.t.clone(), M2.t.clone()
        m1 = M1.t.clone() if M1 is not None else None
        snap = {k: b.bits() for k, b in (("W", MB), ("M1", M1), ("M2", M2), ("V", VB), ("LP", LPB)) if b}
        eng._check(eng.lib.stk_ademamix_step_prologue(eng.ctx, hyp, ahyp, ng, len(ends) if per_range else 0,
                                                      rgrp.data_ptr() if per_range else None,
                                                      rsteps.data_ptr() if per_range else None, BC.ptr(),
                                                      eng._stream()))
        a = L.OptimArgs()
        a.hyper, a.n_groups = hyp, ng
        a.master, a.exp_avg, a.exp_avg_sq = MB.ptr(), M1.ptr() if M1 is not None else None, VB.ptr()
        a.exp_avg_slow = M2.ptr()
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
        else:
            a.group_bc = BC.ptr()
        eng.optim_step_ex(a)
        eng.step_epilogue()
        got = {"W": MB.t.clone(), "M2": M2.t.clone(), "V": VB.t.clone()}
        if M1 is not None:
            got["M1"] = M1.t.clone()
        BC.check_guards()

        # ---- the prologue: this step's scalars of every entry, and its step counts ----
        bc = BC.t.cpu().view(n_entries, 4)
        for k in range(n_entries):
            h = groups[rgroup[k]] if per_range else groups[k]
            want = _want_scalars(h, entry_done[k] + 1)
            assert torch.equal(bc[k].view(torch.int32), want.view(torch.int32)), (step, k, bc[k], want)
            if not found_inf and not (per_range and k in skip):
                entry_done[k] += 1
        if per_range:
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
                if st["exp_avg_fast"] is not None:
                    st["exp_avg_fast"] = m1[masks[j]].clone()
                st["exp_avg_slow"], st["exp_avg_sq"] = s2[masks[j]].clone(), v[masks[j]].clone()
        if not found_inf:
            ref.step()
            done += 1
        assert int(eng.scaler_get().opt_steps) == done
        want = {"W": w.clone(), "M2": s2.clone(), "V": v.clone()}
        if m1 is not None:
            want["M1"] = m1.clone()
        for j in ranges:
            p, s = ref_params[j], masks[j]
            want["W"][s] = p.detach()
            st = ref.state[p]
            if not st:
                continue
            want["M2"][s], want["V"][s] = st["exp_avg_slow"], st["exp_avg_sq"]
            if st["exp_avg_fast"] is not None:
                want["M1"][s] = st["exp_avg_fast"]
            assert (st["exp_avg_fast"] is None) == (groups[rgroup[j]]["betas"][0] == 0)
        for key in got:
            assert _same(got[key], want[key]), f"step {step}: {key}"
        # ---- where the kernel wrote: nothing for skipped ranges, a found_inf step or a beta1 == 0 group's M ----
        skip_elem = torch.from_numpy(np.isin(elem_range, list(skip))) | found_inf
        b1_zero = torch.from_numpy(np.asarray([groups[rgroup[j]]["betas"][0] == 0 for j in range(len(ends))])[elem_range])
        for key, b in (("W", MB), ("M2", M2), ("V", VB)):
            b.check_unchanged_except(snap[key], ~skip_elem)
        if M1 is not None:
            M1.check_unchanged_except(snap["M1"], ~skip_elem & ~b1_zero)
        if src != "main":
            seg = torch.zeros(GB.n, dtype=torch.bool)
            seg[torch.from_numpy(gidx)] = True
            assert float(GB.t[torch.from_numpy(gidx).cuda()].float().abs().max()) == 0.0
        if LPB is not None:
            stepped = ~skip_elem
            mask = torch.zeros(LPB.n, dtype=torch.bool)
            mask[torch.from_numpy(gidx)[stepped]] = True
            LPB.check_unchanged_except(snap["LP"], mask)
            if bool(stepped.any()):
                glp = LPB.t[torch.from_numpy(gidx)[stepped].cuda()].cpu()
                wl = got["W"].cpu()[stepped].to(LPB.dtype)
                assert torch.equal(glp.view(INT_VIEW[LPB.dtype]), wl.view(INT_VIEW[LPB.dtype]))
        if found_inf:
            assert all(torch.equal(b.bits(), snap[k]) for k, b in (("W", MB), ("M2", M2), ("V", VB)))
    assert done == STEPS - (inf_at is not None)


# group configurations whose schedules the prologue must reproduce at every step of their warm-ups
PROLOGUE_GROUPS = [
    dict(lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, alpha_warmup=4000, beta3_warmup=4000, eps=1e-8, weight_decay=0),
    dict(lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=8.0, alpha_warmup=256_000, beta3_warmup=256_000, eps=1e-8,
         weight_decay=0),
    dict(lr=1e-3, betas=(0.0, 0.99, 0.999), alpha=2.0, alpha_warmup=3, beta3_warmup=1777, eps=1e-8, weight_decay=0),
    dict(lr=1e-3, betas=(0.8, 0.95, 0.99999), alpha=0.3, alpha_warmup=None, beta3_warmup=5000, eps=1e-8, weight_decay=0),
]


def test_prologue_scalars_equal_the_class_at_every_warmup_step(eng):
    """One prologue launch per group with one range per step count: the fp32 scalars of every step t = 1 .. T + 1 of the
    longest warm-up equal the class's (python doubles cast to fp32) bit for bit; 256 000 steps for the paper's schedule.
    The step counts advance by one and a found_inf launch leaves them where they were."""
    L = _L()
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0)
    for h in PROLOGUE_GROUPS:
        T = max(x for x in (h["alpha_warmup"], h["beta3_warmup"]) if x is not None)
        n = T + 1
        steps = torch.arange(n, dtype=torch.int32)          # entry j holds j steps: it forms the scalars of t = j + 1
        rsteps = steps.cuda()
        rgrp = torch.zeros(n, dtype=torch.uint8).cuda()
        bc = torch.full((n, 4), float("nan"), dtype=torch.float32, device="cuda")
        hyp = (L.OptimHyper * 1)(_hyper(h))
        ahyp = (L.AdemamixHyper * 1)(_ahyper(h))
        eng._check(eng.lib.stk_ademamix_step_prologue(eng.ctx, hyp, ahyp, 1, n, rgrp.data_ptr(), rsteps.data_ptr(),
                                                      bc.data_ptr(), eng._stream()))
        got = bc.cpu()
        want = torch.stack([_want_scalars(h, t) for t in range(1, n + 1)])
        bad = (got.view(torch.int32) != want.view(torch.int32)).any(dim=1).nonzero().flatten().tolist()
        assert not bad, f"steps whose fp32 scalars differ: {[t + 1 for t in bad[:20]]} ({len(bad)} of {n})"
        assert torch.equal(rsteps.cpu(), steps + 1)
        eng.scaler_set(found_inf=1)
        eng._check(eng.lib.stk_ademamix_step_prologue(eng.ctx, hyp, ahyp, 1, n, rgrp.data_ptr(), rsteps.data_ptr(),
                                                      bc.data_ptr(), eng._stream()))
        assert torch.equal(rsteps.cpu(), steps + 1)
        eng.scaler_set(found_inf=0)


def test_kernel_requires_its_buffers_and_scalars(eng):
    from stoke_b200.engine import StokeB200Error

    L = _L()
    bufs = [Buf(64, F32, torch.zeros(64).cuda()) for _ in range(5)]
    BC = Buf(4, F32, torch.zeros(4).cuda())
    for h, m1, m2, v, bc in ((G3[0], True, False, True, True), (G3[0], False, True, True, True),
                             (G3[0], True, True, False, True), (G3[0], True, True, True, False)):
        a = L.OptimArgs()
        hyp = (L.OptimHyper * 1)(_hyper(h))
        a.hyper, a.n_groups = hyp, 1
        a.master, a.grad, a.grad_dtype, a.n_local = bufs[0].ptr(), bufs[1].ptr(), L.F32, 64
        a.exp_avg = bufs[2].ptr() if m1 else None
        a.exp_avg_slow = bufs[3].ptr() if m2 else None
        a.exp_avg_sq = bufs[4].ptr() if v else None
        a.group_bc = BC.ptr() if bc else None
        with pytest.raises(StokeB200Error):
            eng.optim_step_ex(a)
    with pytest.raises(StokeB200Error):   # stk_optim_step_prologue does not form AdEMAMix's scalars
        eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, (L.OptimHyper * 1)(_hyper(G3[0])), None, 1, 0, None, None,
                                                   None, BC.ptr(), eng._stream()))


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


FACADE_KW = {"lr": 5e-3, "betas": (0.9, 0.99, 0.999), "alpha": 4.0, "alpha_warmup": 4, "beta3_warmup": 6,
             "weight_decay": 0.01}


def _stoke(fp16, clip, accum, stock, wa=None, kw=FACADE_KW):
    model = Net()
    used = [p for m in model.layers for p in m.parameters()]
    if stock:   # 9 groups: more than the fused step takes, so Stoke builds the stock route
        groups = [dict(params=[p]) for p in used] + [dict(params=list(model.unused.parameters()), weight_decay=0.0)]
    else:
        groups = [dict(params=used), dict(params=list(model.unused.parameters()), weight_decay=0.0)]
    grad_clip = None
    if clip is not None:
        grad_clip = sb.ClipGradNormConfig(max_norm=clip[1], norm_type=2.0) if clip[0] == "norm" else \
            sb.ClipGradConfig(clip_value=clip[1])
    return sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=AdEMAMix, optimizer_kwargs=dict(kw, params=groups)),
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
    state tensors bit for bit over 9 steps that cross both warm-ups; the never-used parameter keeps its weights and has
    no fused state entry.  Clip by norm takes its norm from different kernels on the two routes, so there the bar is fp32
    tolerance."""
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
    keys = ("exp_avg_fast", "exp_avg_slow", "exp_avg_sq")
    for i in range(8):
        assert set(fsd["state"][i]) == set(keys) | {"step"}
        assert float(fsd["state"][i]["step"]) == 9 == float(ssd["state"][i]["step"])
        for k in keys:
            a, b = fsd["state"][i][k].cpu(), ssd["state"][i][k].cpu()
            assert _same(a, b) if exact else _rel(a, b) < 1e-5, (i, k)
    assert 8 not in fsd["state"] and 9 not in fsd["state"]   # the unused Linear: never stepped
    init = Net().unused
    got = fs.optimizer.path.unflatten(fs.optimizer.path.gather_master().cpu())
    assert torch.equal(got[8], init.weight.detach()) and torch.equal(got[9], init.bias.detach())
    for s in (fs, ss):
        s.optimizer.close()


def _fused(net, kw, lp=None, stock=False, accum=1):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    cls = B200StockOptimizer if stock else B200FusedOptimizer
    return cls(net, AdEMAMix, kw, engine=get_engine(0), grad_accum=accum, lp_dtype=lp)


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


CKPT_KW = {"params": None, "lr": 1e-2, "betas": (0.9, 0.99, 0.999), "alpha": 3.0, "alpha_warmup": 6,
           "beta3_warmup": 10, "weight_decay": 0.05}


def _ckpt_kw(net):
    """Two groups, the second with beta1 == 0."""
    ps = list(net.parameters())
    return dict({k: v for k, v in CKPT_KW.items() if k != "params"},
                params=[dict(params=ps[:4]), dict(params=ps[4:], betas=(0.0, 0.95, 0.99), alpha=1.5)])


def _int_steps(sd):
    """The state dict as upstream writes it: ``step`` a python int."""
    return dict(sd, state={i: dict(e, step=int(float(e["step"]))) for i, e in sd["state"].items()})


def test_checkpoints_continue_bit_for_bit():
    """A checkpoint saved after 4 steps continues like the uninterrupted 12-step run (both warm-ups crossed), bit for
    bit: fused -> fused (with upstream's int ``step``), fused -> plain class (4 steps) -> fused (4 steps), and fused ->
    stock -> fused.  The second group has beta1 == 0: its entries carry ``exp_avg_fast = None``."""
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
        assert list(e) == ["step", "exp_avg_fast", "exp_avg_slow", "exp_avg_sq"] and float(e["step"]) == 4
        assert (e["exp_avg_fast"] is None) == (i >= 4)
    # fused -> fused, from upstream's int steps
    again = make()
    again.load_state_dict(_int_steps(sd))
    _run_injected(again, range(4, 12))
    assert all(_same(a, b) for a, b in zip(_masters(again), want))
    again.close()
    # fused -> plain class -> fused
    plain = [torch.nn.Parameter(w.cuda().clone()) for w in first.path.unflatten(first.path.gather_master())]
    topt = AdEMAMix(**_ckpt_kw(torch.nn.ParameterList(plain)))
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
        for k in e:
            assert (e[k] is None and got_sd["state"][i][k] is None) or _same(got_sd["state"][i][k], e[k]), (i, k)
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


def test_weight_average_on_top():
    """An EMA of the weights over the fused AdEMAMix step: the master is the run's without averaging, bit for bit, and
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


@pytest.mark.multigpu
def test_sharded_matches_replicated_w2(tmp_path):
    """fairscale_oss at W = 2: AdEMAMix sharded (ZeRO-1, in-kernel parameter all-gather) against the replicated
    all-reduce route: final weights and the gathered state_dict bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "ademamix_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29573", os.path.join(ROOT, "tests", "ademamix_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    assert res["sharded_route"] == "sharded" and res["replicated_route"] == "allreduce", res
    assert res["weights_identical"] and res["state_identical"], res
