"""stoke_b200.AdamWScheduleFree and SGDScheduleFree on the fused step (GPU).

Kernel level: stk_sf_step_prologue + stk_optim_step_ex called directly, the buffers between guard bands (see
test_gpu_kernels.py), compared bit for bit with the class's ``step()`` on CUDA fp32 tensors restarted from the kernel's
own state every step; the prologue's scalars against the class's, cast to fp32.  Three deliberately wrong updates must
fail the same comparison.  Engine level: the Stoke facade against the same class on the stock route (9 groups), with
train() / eval() between steps; checkpoints saved in train and eval mode, continued on the fused step, the plain class
and the stock route; a step without host synchronisation; the refused step in eval mode; the sharded W = 2 run."""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import stoke_b200 as sb
from stoke_b200.optim import AdamWScheduleFree, SGDScheduleFree
from test_gpu_kernels import BF16, F32, INT_VIEW, Buf, _dt, _layout

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLS = {"adamw": AdamWScheduleFree, "sgd": SGDScheduleFree}
BASE = {"adamw": {"lr": 2e-2, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0.0, "warmup_steps": 0, "r": 0.0,
                  "weight_lr_power": 2.0},
        "sgd": {"lr": 0.5, "momentum": 0.9, "weight_decay": 0.0, "warmup_steps": 0, "r": 0.0, "weight_lr_power": 2.0}}


def _groups8(kind):
    b = BASE[kind]
    out = [dict(b), dict(b, warmup_steps=5), dict(b, weight_decay=0.125), dict(b, r=0.5, warmup_steps=3),
           dict(b, lr=0.0), dict(b, weight_lr_power=1.0, weight_decay=0.01), dict(b, lr=b["lr"] * 4, r=1.0)]
    out.append(dict(b, betas=(0.8, 0.99)) if kind == "adamw" else dict(b, momentum=0.75))
    return out


def _L():
    from stoke_b200 import _lib

    return _lib


def _beta1(h):
    return h["betas"][0] if "betas" in h else h["momentum"]


def _hyper(kind, h):
    L = _L()
    o = L.OptimHyper()
    o.kind = L.OPT_SF_ADAMW if kind == "adamw" else L.OPT_SF_SGD
    o.lr = h["lr"]
    if kind == "adamw":
        o.beta1, o.beta2 = h["betas"]
        o.eps = h["eps"]
    o.weight_decay = h["weight_decay"]
    o.clip_kind = L.CLIP_NONE
    return o


def _sf_hyper(h):
    L = _L()
    x = L.SfHyper()
    x.lr, x.beta1, x.r, x.weight_lr_power = h["lr"], _beta1(h), h["r"], h["weight_lr_power"]
    x.beta2 = h["betas"][1] if "betas" in h else 0.0
    x.warmup_steps = h["warmup_steps"]
    return x


def _scalars(h, k, lr_max, weight_sum, shift=1):
    """The group scalars of step k + 1 from the state before it (python doubles, the class's formulas); ``shift=0`` is the
    deliberately wrong count k in place of k + 1."""
    kk = k + shift
    lr = h["lr"] * (kk / h["warmup_steps"] if k < h["warmup_steps"] else 1.0)
    lr_max = max(lr, lr_max)
    weight = (kk ** h["r"]) * (lr_max ** h["weight_lr_power"])
    weight_sum = weight_sum + weight
    ckp1 = weight / weight_sum if weight_sum != 0 else 0.0
    bc2 = 1 - h["betas"][1] ** (k + 1) if "betas" in h else 1.0
    return lr, ckp1, lr * (_beta1(h) * (1 - ckp1) - 1), bc2, lr_max, weight_sum


def _mutant(kind, w, z, v, g, h, k, lr_max, weight_sum, mut):
    """One step with a deliberate mistake: the lerp after the add, the count k instead of k + 1 in the group scalars, or
    AdamW's bias correction applied to the learning rate instead of the second moment."""
    lr, ckp1, y_lr, bc2, _, _ = _scalars(h, k, lr_max, weight_sum, shift=0 if mut == "k_not_kp1" else 1)
    w, z, v = w.clone(), z.clone(), v.clone() if v is not None else None
    d = g
    if kind == "adamw":
        b2 = h["betas"][1]
        v.mul_(b2).addcmul_(g, g, value=1 - b2)
        if mut == "bc_on_lr":
            d = g / v.sqrt().add_(h["eps"])
            lr, y_lr = lr * bc2 ** 0.5, y_lr * bc2 ** 0.5
        else:
            d = g / v.mul(1 / bc2).sqrt_().add_(h["eps"])
    if h["weight_decay"] != 0:
        d = d.add(w, alpha=h["weight_decay"])
    if mut == "lerp_after_add":
        w.add_(d, alpha=y_lr)
        w.lerp_(z, ckp1)
    else:
        w.lerp_(z, ckp1)
        w.add_(d, alpha=y_lr)
    z.sub_(d, alpha=lr)
    return w, z, v


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


# name: kind, gradient source, model copy, n_local, segments, groups (None: one), range table with skip bits,
#       per-parameter counts (range_bc handed over and ignored), fp32 accumulator, found_inf step
CASES = {
    "adamw_raw_bf16_warmup": ("adamw", "raw_bf16", "bf16", 2_056, 0, [dict(BASE["adamw"], warmup_steps=4,
                                                                           weight_decay=0.05)], False, False, False, 6),
    "adamw_main_8groups_ranges": ("adamw", "main", "f32", 2_048, 7, "g8", True, True, False, 9),
    "adamw_raw_f32_acc_8groups": ("adamw", "raw_f32", None, 2_056, 5, "g8", True, False, True, None),
    "sgd_raw_bf16_8groups_ranges": ("sgd", "raw_bf16", "bf16", 2_048, 64, "g8", True, True, False, 3),
    "sgd_main_wd_r": ("sgd", "main", None, 2_040, 3, [dict(BASE["sgd"], weight_decay=0.1, r=0.25, warmup_steps=2)],
                      False, False, False, None),
}
STEPS = 20


@pytest.mark.parametrize("name", list(CASES))
def test_sf_kernel_matches_cuda_class_bit_for_bit(eng, name):
    L = _L()
    kind, src, lp, n_local, n_seg, groups, use_ranges, per_range, use_acc, inf_at = CASES[name]
    groups = _groups8(kind) if groups == "g8" else groups
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
    hyp = (L.OptimHyper * ng)(*[_hyper(kind, h) for h in groups])
    sfh = (L.SfHyper * ng)(*[_sf_hyper(h) for h in groups])
    w0 = torch.from_numpy(rng.standard_normal(n_local).astype(np.float32) * 1e-1)
    MB = Buf(n_local, F32, w0.cuda())
    ZB = Buf(n_local, F32, w0.cuda())   # z starts as the parameter
    VB = Buf(n_local, F32, torch.zeros(n_local).cuda()) if kind == "adamw" else None
    LPB = None if lp is None else Buf(N, BF16 if lp == "bf16" else F32, torch.full((N,), -5.0))
    gdt = {"raw_bf16": BF16, "raw_f32": F32, "main": F32}[src]
    GB = Buf(N if src != "main" else n_local, gdt)
    AB = Buf(N, F32) if use_acc else None
    BC = Buf(ng * 4, F32, torch.full((ng * 4,), float("nan")).cuda())
    RBC = Buf(len(ends) * 4, F32, torch.full((len(ends) * 4,), float("nan")).cuda()) if per_range else None
    state = torch.tensor([[-1.0, 0.0]] * ng, dtype=torch.float64).cuda()
    rend = torch.tensor([e // 8 for e in ends], dtype=torch.int32).cuda()
    rsteps = torch.zeros(len(ends), dtype=torch.int32).cuda()
    sl = (C.c_size_t * (len(pieces) + 1))(*([p[0] for p in pieces] + [n_local]))
    sg = (C.c_size_t * len(pieces))(*[p[2] for p in pieces])
    lpp = L.ptr_array([LPB.ptr()]) if lp is not None else None
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0)
    # the reference: one class instance, one group per kernel group, one parameter per (range, group) slice
    masks = {j: torch.from_numpy(elem_range == j).cuda() for j in ranges}
    ref_params = {j: torch.nn.Parameter(w0.cuda()[masks[j]].clone()) for j in ranges}
    ref = CLS[kind]([dict(h, params=[ref_params[j] for j in ranges if rgroup[j] == gi]) for gi, h in enumerate(groups)])
    ref.train()
    muts = {"lerp_after_add", "k_not_kp1"} | ({"bc_on_lr"} if kind == "adamw" else set())
    hit = set()
    g32 = rng.standard_normal(n_local).astype(np.float32)
    done = 0
    for step in range(STEPS):
        skip = {j for j in ranges if use_ranges and (j + step) % 5 == 1} if per_range else set()
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
        w, z = MB.t.clone(), ZB.t.clone()
        v = VB.t.clone() if VB is not None else None
        snap = {k: b.bits() for k, b in (("G", GB), ("M", MB), ("Z", ZB), ("V", VB), ("LP", LPB), ("A", AB)) if b}
        before = [(g_["k"], g_["lr_max"], g_["weight_sum"]) for g_ in ref.param_groups]
        if per_range:   # per-parameter counts: their prologue writes range_bc, which the schedule-free kinds ignore
            eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, None, ng, len(ends), rgrp.data_ptr(),
                                                       rsteps.data_ptr(), None, RBC.ptr(), eng._stream()))
        eng._check(eng.lib.stk_sf_step_prologue(eng.ctx, sfh, ng, state.data_ptr(), BC.ptr(), eng._stream()))
        a = L.OptimArgs()
        a.hyper, a.n_groups = hyp, ng
        a.master, a.exp_avg, a.exp_avg_sq = MB.ptr(), ZB.ptr(), VB.ptr() if VB is not None else None
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
            a.range_bc = RBC.ptr()
        a.group_bc = BC.ptr()
        eng.optim_step_ex(a)
        eng.step_epilogue()
        got_w, got_z = MB.t.clone(), ZB.t.clone()
        got_v = VB.t.clone() if VB is not None else None
        BC.check_guards()

        # ---- the reference step (not taken at all on a found_inf step, like GradScaler.step) ----
        gl = g.float()
        if acc_local is not None:
            gl = gl + acc_local                       # the kernel's raw + accumulator sum, one fp32 add
        gl = gl.cuda()
        for j in ranges:
            p = ref_params[j]
            p.data.copy_(w[masks[j]])
            p.grad = None if j in skip else gl[masks[j]].clone()
            ref.state[p]["z"] = z[masks[j]].clone()
            if kind == "adamw":
                ref.state[p]["exp_avg_sq"] = v[masks[j]].clone()
        grads_before = {j: ref_params[j].grad.clone() for j in ranges if j not in skip}
        if not found_inf:
            ref.step()
            done += 1
        assert int(eng.scaler_get().opt_steps) == done
        # prologue: the scalars of this step, cast to fp32, are the class's; lr_max / weight_sum advance unless found_inf
        bc = BC.t.cpu().view(ng, 4)
        st = state.cpu()
        for gi, h in enumerate(groups):
            lr, ckp1, y_lr, bc2, lr_max, wsum = _scalars(h, *before[gi])
            want = torch.tensor([ckp1, y_lr, lr, 1 / bc2], dtype=torch.float32)
            assert torch.equal(bc[gi].view(torch.int32), want.view(torch.int32)), (step, gi, bc[gi], want)
            grp = ref.param_groups[gi]
            assert grp["k"] == done
            assert st[gi].tolist() == pytest.approx([grp["lr_max"], grp["weight_sum"]], rel=1e-14, abs=0)
            if found_inf:
                assert (grp["lr_max"], grp["weight_sum"]) == before[gi][1:]
        ref_w, ref_z = w.clone(), z.clone()
        ref_v = v.clone() if v is not None else None
        mut_out = {mu: (w.clone(), z.clone(), v.clone() if v is not None else None) for mu in muts}
        for j in ranges:
            p, s = ref_params[j], masks[j]
            ref_w[s] = p.detach()
            ref_z[s] = ref.state[p]["z"]
            if kind == "adamw":
                ref_v[s] = ref.state[p]["exp_avg_sq"]
            if j in skip or found_inf:
                continue
            assert torch.equal(p.grad, grads_before[j])   # step() leaves p.grad as it was
            h = groups[rgroup[j]]
            for mu in muts:
                mw, mz, mv = _mutant(kind, w[s], z[s], v[s] if v is not None else None, gl[s], h, *before[rgroup[j]], mu)
                mut_out[mu][0][s], mut_out[mu][1][s] = mw, mz
                if mv is not None:
                    mut_out[mu][2][s] = mv
        assert _same(got_w, ref_w), f"step {step}: master"
        assert _same(got_z, ref_z), f"step {step}: z"
        if kind == "adamw":
            assert _same(got_v, ref_v), f"step {step}: exp_avg_sq"
        for mu in muts:
            mw, mz, mv = mut_out[mu]
            if not (_same(got_w, mw) and _same(got_z, mz) and (mv is None or _same(got_v, mv))):
                hit.add(mu)
        # ---- where the kernel wrote ----
        skip_elem = torch.from_numpy(np.isin(elem_range, list(skip))) | found_inf
        MB.check_unchanged_except(snap["M"], ~skip_elem)
        ZB.check_unchanged_except(snap["Z"], ~skip_elem)
        if VB is not None:
            VB.check_unchanged_except(snap["V"], ~skip_elem)
        if src != "main":
            seg = torch.zeros(GB.n, dtype=torch.bool)
            seg[torch.from_numpy(gidx)] = True
            GB.check_unchanged_except(snap["G"], seg)
            assert float(GB.t[torch.from_numpy(gidx).cuda()].float().abs().max()) == 0.0
        if LPB is not None:
            stepped = ~skip_elem
            mask = torch.zeros(LPB.n, dtype=torch.bool)
            mask[torch.from_numpy(gidx)[stepped]] = True
            LPB.check_unchanged_except(snap["LP"], mask)
            if bool(stepped.any()):
                glp = LPB.t[torch.from_numpy(gidx)[stepped].cuda()].cpu()
                want = got_w.cpu()[stepped].to(LPB.dtype)
                assert torch.equal(glp.view(INT_VIEW[LPB.dtype]), want.view(INT_VIEW[LPB.dtype]))
        if found_inf:
            assert torch.equal(MB.bits(), snap["M"]) and torch.equal(ZB.bits(), snap["Z"])
    assert hit == muts, f"deliberately wrong updates that passed every step: {muts - hit}"


def test_sf_kernel_requires_group_scalars(eng):
    from stoke_b200.engine import StokeB200Error

    L = _L()
    MB, ZB, GB = Buf(64, F32, torch.zeros(64).cuda()), Buf(64, F32, torch.zeros(64).cuda()), Buf(64, F32)
    hyp = (L.OptimHyper * 1)(_hyper("sgd", BASE["sgd"]))
    a = L.OptimArgs()
    a.hyper, a.n_groups = hyp, 1
    a.master, a.exp_avg, a.exp_avg_sq = MB.ptr(), ZB.ptr(), None
    a.grad, a.grad_dtype, a.grad_raw, a.grad_mul = GB.ptr(), L.F32, 0, 1.0
    a.n_local = 64
    with pytest.raises(StokeB200Error):
        eng.optim_step_ex(a)


def test_lerp_forms_round_alike():
    """Tensor.lerp_ and torch._foreach_lerp_ (AveragedModel's, which stk_weight_avg reproduces) round alike on CUDA fp32
    at the weights the classes use, so the classes' per-parameter lerp_ is the swap's lerp."""
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.randn(1 << 16, device="cuda", generator=g)
    z = y + 1e-2 * torch.randn(1 << 16, device="cuda", generator=g)
    for w in (0.1, 1 - 1 / 0.9, 0.25, 0.75, 1.0, 1 - 1 / 0.75, 0.37):
        a = y.clone().lerp_(z, w)
        b = [y.clone()]
        torch._foreach_lerp_(b, [z], w)
        assert torch.equal(a.view(torch.int32), b[0].view(torch.int32)), w


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


def _stoke(kind, kw, fp16, clip, accum, stock, wa=None):
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
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=CLS[kind], optimizer_kwargs=dict(kw, params=groups)),
                 loss=_mse, batch_size_per_device=8, grad_accum_steps=accum, grad_clip=grad_clip, gpu=True, fp16=fp16,
                 verbose=False, configs=[wa] if wa is not None else None)
    return s


def _drive(s, steps, fp16, accum, swap_at=(), seed=0):
    """Training steps through the public calls, with eval() / train() after the steps in ``swap_at``; returns P after
    every swap (checked against the master's cast)."""
    path = s.optimizer.path
    dt = torch.bfloat16 if fp16 else torch.float32
    g = torch.Generator().manual_seed(seed)
    for step in range(steps):
        for _ in range(accum):
            x, y = torch.randn(8, 16, generator=g).cuda().to(dt), torch.randn(8, 1, generator=g).cuda()
            loss = s.loss(s.model(x), y)
            s.backward(loss)
            s.step()
        if step in swap_at:
            for mode in ("eval", "train"):
                getattr(s.optimizer, mode)()
                assert torch.equal(path.p_flat.cpu(), path.gather_master().cpu().to(path.p_flat.dtype)), mode


FACADE = [("adamw", {"lr": 5e-3, "weight_decay": 0.01, "warmup_steps": 3}),
          ("sgd", {"lr": 0.2, "momentum": 0.9, "weight_decay": 1e-3, "r": 0.5})]


@pytest.mark.parametrize("accum", [1, 2])
@pytest.mark.parametrize("clip", [None, ("value", 0.05), ("norm", 0.5)], ids=["noclip", "value", "norm"])
@pytest.mark.parametrize("fp16", [None, "bf16"], ids=["fp32", "bf16"])
@pytest.mark.parametrize("kind,kw", FACADE, ids=["adamw", "sgd"])
def test_stoke_facade_matches_stock_route(kind, kw, fp16, clip, accum):
    """The fused step and the class's own step on the stock route (9 groups) give the same master, z and exp_avg_sq bit
    for bit, with eval() / train() between steps; the never-used parameter keeps its weights and has no fused state
    entry.  Clip by norm takes its norm from different kernels on the two routes, so there the bar is fp32 tolerance."""
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    torch.cuda.set_device(0)
    runs = []
    for stock in (False, True):
        s = _stoke(kind, kw, fp16, clip, accum, stock)
        assert isinstance(s.optimizer, B200StockOptimizer if stock else B200FusedOptimizer)
        s.optimizer.train()
        _drive(s, 8, fp16, accum, swap_at=(2, 5))
        runs.append((s, s.optimizer.path.gather_master().cpu(), s.optimizer.state_dict()))
    (fs, fw, fsd), (ss, sw, ssd) = runs
    exact = clip is None or clip[0] == "value"
    assert _same(fw, sw) if exact else _rel(fw, sw) < 1e-5
    keys = ("z", "exp_avg_sq") if kind == "adamw" else ("z",)
    for i in range(8):
        assert set(fsd["state"][i]) == set(keys)
        for k in keys:
            a, b = fsd["state"][i][k].cpu(), ssd["state"][i][k].cpu()
            assert _same(a, b) if exact else _rel(a, b) < 1e-5, (i, k)
    assert 8 not in fsd["state"] and 9 not in fsd["state"]   # the unused Linear: never stepped
    init = Net().unused
    got = fs.optimizer.path.unflatten(fs.optimizer.path.gather_master().cpu())
    assert torch.equal(got[8], init.weight.detach()) and torch.equal(got[9], init.bias.detach())
    assert fsd["param_groups"][0]["k"] == 8 == ssd["param_groups"][0]["k"]
    assert fsd["param_groups"][0]["weight_sum"] == pytest.approx(ssd["param_groups"][0]["weight_sum"], rel=1e-14)
    for s in (fs, ss):
        s.optimizer.close()


def _fused(net, kind, kw, lp=None, stock=False, accum=1):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    cls = B200StockOptimizer if stock else B200FusedOptimizer
    return cls(net, CLS[kind], kw, engine=get_engine(0), grad_accum=accum, lp_dtype=lp)


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


CKPT_KW = {"adamw": {"lr": 1e-2, "weight_decay": 0.05, "warmup_steps": 3, "r": 0.5},
           "sgd": {"lr": 0.3, "weight_decay": 0.01, "warmup_steps": 2}}


@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("kind", ["adamw", "sgd"])
def test_checkpoints_continue_bit_for_bit(kind, mode):
    """A checkpoint saved in train or eval mode after 4 steps continues like the uninterrupted run, bit for bit:
    fused -> fused, fused -> plain class (4 steps) -> fused (4 steps), and fused -> stock -> fused.  Every run makes the
    same eval() (/ train()) calls at the same points."""
    torch.cuda.set_device(0)
    kw = CKPT_KW[kind]

    def pause(o):   # the calls around the save point, identical in every run
        o.eval()
        if mode == "train":
            o.train()

    def resume(o):
        if mode == "eval":
            o.train()

    cont = _fused(OddNet().cuda(), kind, kw)
    cont.train()
    _run_injected(cont, range(4))
    pause(cont)
    resume(cont)
    _run_injected(cont, range(4, 12))
    want = _masters(cont)
    want_sd = cont.state_dict()
    cont.close()

    first = _fused(OddNet().cuda(), kind, kw)
    first.train()
    _run_injected(first, range(4))
    pause(first)
    sd = first.state_dict()
    assert all(set(e) == ({"z", "exp_avg_sq"} if kind == "adamw" else {"z"}) for e in sd["state"].values())
    assert sd["param_groups"][0]["train_mode"] == (mode == "train") and sd["param_groups"][0]["k"] == 4
    # fused -> fused
    again = _fused(OddNet().cuda(), kind, kw)
    again.load_state_dict(sd)
    resume(again)
    _run_injected(again, range(4, 12))
    assert all(_same(a, b) for a, b in zip(_masters(again), want))
    again.close()
    # fused -> plain class -> fused
    plain = [torch.nn.Parameter(w.cuda().clone()) for w in first.path.unflatten(first.path.gather_master())]
    topt = CLS[kind](plain, **kw)
    topt.load_state_dict({k: v for k, v in sd.items() if not k.startswith("b200_")})
    resume(topt)
    resume(first)
    _run_injected(first, range(4, 8), plain, topt)   # the fused run alongside: the same gradients
    for a, b in zip(_masters(first), plain):
        assert _same(a, b.detach().reshape(-1))
    first.close()
    net = OddNet().cuda()
    with torch.no_grad():
        for p, q in zip(net.parameters(), plain):
            p.copy_(q.detach())
    last = _fused(net, kind, kw)
    last.load_state_dict(topt.state_dict())   # a plain state dict: no b200_* keys, the model weights loaded first
    _run_injected(last, range(8, 12))
    assert all(_same(a, b) for a, b in zip(_masters(last), want))
    got_sd = last.state_dict()
    for i, e in want_sd["state"].items():
        for k in e:
            assert _same(got_sd["state"][i][k], e[k]), (i, k)
    for key in ("k", "scheduled_lr", "train_mode"):
        assert got_sd["param_groups"][0][key] == want_sd["param_groups"][0][key], key
    for key in ("lr_max", "weight_sum"):   # python's pow and the device's may differ in the last bit of a double
        assert got_sd["param_groups"][0][key] == pytest.approx(want_sd["param_groups"][0][key], rel=1e-14), key
    last.close()
    # fused -> stock -> fused
    a = _fused(OddNet().cuda(), kind, kw)
    a.train()
    _run_injected(a, range(4))
    pause(a)
    b = _fused(OddNet().cuda(), kind, kw, stock=True)
    b.load_state_dict(a.state_dict())
    resume(b)
    _run_injected(b, range(4, 8))
    c = _fused(OddNet().cuda(), kind, kw)
    c.load_state_dict(b.state_dict())
    _run_injected(c, range(8, 12))
    assert all(_same(x, y) for x, y in zip(_masters(c), want))
    for o in (a, b, c):
        o.close()


def test_step_makes_no_host_sync():
    net = OddNet().cuda()
    opt = _fused(net, "adamw", {"lr": 1e-3, "weight_decay": 0.1, "warmup_steps": 5}, torch.bfloat16)
    opt.train()
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


def test_found_inf_under_amp_leaves_the_group_state():
    """bf16 with the device loss scaler and an inf injected into one gradient: the step is skipped, and k, lr_max and weight_sum stay where they
    were; the next step continues like a run in which the bad step never happened."""
    from stoke_b200.fp16 import DeviceGradScaler

    torch.cuda.set_device(0)
    kw = {"lr": 1e-2, "warmup_steps": 4, "r": 1.0}
    res = []
    for bad_step in (None, 2):
        opt = _fused(OddNet().cuda(), "sgd", kw, torch.bfloat16)
        opt.train()
        path = opt.path
        scaler = DeviceGradScaler(path.engine, init_scale=2.0**4, growth_interval=1000, state_id=path.state_id)
        seq = [0, 1, 2, 2, 3] if bad_step is not None else [0, 1, 2, 3]
        for n, step in enumerate(seq):
            _inject(path, step, 0, torch.bfloat16, scale=scaler.get_scale())
            bad = bad_step is not None and n == bad_step
            if bad:
                path.grad_views[2].view(-1)[5] = float("inf")
                before = path._sf_state.cpu().clone()
            path.after_backward(sync=True, unscale=True)
            opt.step()
            if bad:
                assert torch.equal(path._sf_state.cpu(), before)
                assert int(path.engine.scaler_get(path.state_id).opt_steps) == 2
        res.append((path.gather_master().cpu(), path._sf_state.cpu(), opt.state_dict()["param_groups"][0]["k"]))
        opt.close()
    assert _same(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]) and res[0][2] == res[1][2] == 4


def test_refused_step_in_eval_mode():
    """Stoke.step raises in eval mode before anything runs: after train(), the run matches bit for bit one that makes
    the same eval() / train() calls without the refused step, weight average included.  train() / eval() raise inside
    weight_average.applied()."""
    torch.cuda.set_device(0)
    kw = {"lr": 5e-3, "weight_decay": 0.01}
    wa = sb.WeightAverageConfig(kind="ema", decay=0.9)
    out = []
    for refuse in (False, True):
        s = _stoke("adamw", kw, "bf16", None, 1, False, wa=wa)
        s.optimizer.train()
        g = torch.Generator().manual_seed(1)
        for step in range(6):
            x, y = torch.randn(8, 16, generator=g).cuda().bfloat16(), torch.randn(8, 1, generator=g).cuda()
            s.backward(s.loss(s.model(x), y))
            if step == 3:
                s.optimizer.eval()
                if refuse:
                    with pytest.raises(RuntimeError):
                        s.step()
                s.optimizer.train()
            s.step()
        with s.weight_average.applied():
            with pytest.raises(RuntimeError):
                s.optimizer.eval()
        p = s.optimizer.path
        out.append((p.gather_master().cpu(), p.gather_avg().cpu(), s.weight_average.n_averaged))
        s.optimizer.close()
    assert out[0][2] == out[1][2] == 6
    assert _same(out[0][0], out[1][0]) and _same(out[0][1], out[1][1])


def test_swap_on_other_kinds_is_refused():
    net = OddNet().cuda()
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer

    opt = B200FusedOptimizer(net, torch.optim.Adam, {"lr": 1e-3}, engine=get_engine(0))
    with pytest.raises(NotImplementedError):
        opt.eval()
    opt.close()


@pytest.mark.multigpu
def test_sharded_matches_replicated_w2(tmp_path):
    """fairscale_oss at W = 2: both classes sharded (ZeRO-1, in-kernel parameter all-gather, collective swap) against the
    replicated all-reduce route: final weights and the gathered state_dict bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "sf_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29571", os.path.join(ROOT, "tests", "schedule_free_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    assert set(res) == {"adamw", "sgd"}
    for name, r in res.items():
        assert r["sharded_route"] == "sharded" and r["replicated_route"] == "allreduce", (name, r)
        assert r["weights_identical"] and r["state_identical"], (name, r)
