"""stoke_b200.Adan on the fused step (GPU).

Rounding probe: the CUDA ops the class is written with, pinned against explicit fp32 formulas, including true division by
a python scalar.  Kernel level: stk_adan_step_prologue's scalars against the class's python formulas, and stk_adan_step
called directly, the buffers between guard bands (see test_gpu_kernels.py), compared bit for bit with the class's
``step()`` on CUDA fp32 tensors restarted from the kernel's own state every step.  The sharded form needs peers (world
> 1): the W = 2 test covers it.  Engine level: the Stoke facade against the same class on the stock route (9 groups),
with clip, gradient accumulation and an fp16 AMP step the scaler skips; checkpoints continued on the fused step, the
plain class and the stock route; the weight average on top; a step without host synchronisation."""
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
from stoke_b200.optim import Adan
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


def _f32(x):
    return torch.tensor(x, dtype=torch.float32, device="cuda")


def test_probe_cuda_rounding_of_the_class_ops():
    """What the kernel relies on, on this GPU: true division by a python scalar b is a multiplication by fp32(1 / b),
    the reciprocal taken in double -- not x / b, and not fp32(1 / fp32(b)), which differs for sqrt(bc3) at t = 2 and 5;
    ``mul_(b).add_(x, alpha=a)`` is one FFMA on the rounded product; ``addcmul_(t, t)`` rounds t * t first;
    ``addcdiv_`` is one FFMA on the rounded quotient."""
    torch.cuda.set_device(0)
    g = torch.Generator(device="cuda").manual_seed(5)
    n = 1 << 16
    x = torch.rand(n, device="cuda", generator=g) + 0.5
    s = torch.rand(n, device="cuda", generator=g) + 0.5
    t = torch.randn(n, device="cuda", generator=g) * 0.3
    for b in (math.sqrt(1 - 0.99 ** 2), math.sqrt(1 - 0.99 ** 5), 1 + 1e-2 * 0.02, 0.7):
        got = x / b
        assert _same(got, x * _f32(1 / b)), b
        assert not _same(got, (x.double() / b).float()), b
        if np.float32(1 / b) != np.float32(1) / np.float32(b):
            assert not _same(got, x * _f32(float(np.float32(1) / np.float32(b)))), b
    a, beta = 1 - 0.92, 0.92
    got = s.clone().mul_(beta).add_(t, alpha=a)
    assert _same(got, _fma(t, _f32(a), s * _f32(beta))) and not _same(got, s * _f32(beta) + _f32(a) * t)
    got = s.clone().addcmul_(t, t, value=a)
    assert _same(got, _fma(_f32(a), t * t, s)) and not _same(got, _fma(_f32(a) * t, t, s))
    q = t / s
    got = x.clone().addcdiv_(t, s, value=-0.0123)
    assert _same(got, _fma(_f32(-0.0123), q, x)) and not _same(got, x + _f32(-0.0123) * q)


def _hyper(h, clip=None):
    L = _L()
    o = L.OptimHyper()
    o.kind = L.OPT_ADAN
    o.lr, o.eps, o.weight_decay = h["lr"], h["eps"], h["weight_decay"]
    o.beta1, o.beta2 = h["betas"][0], h["betas"][1]
    o.clip_kind = L.CLIP_NONE
    if clip is not None:
        o.clip_kind = L.CLIP_NORM if clip[0] == "norm" else L.CLIP_VALUE
        o.clip_max_norm = clip[1] if clip[0] == "norm" else 0.0
        o.clip_value = clip[1] if clip[0] == "value" else 0.0
    return o


def _ahyper(h):
    x = _L().AdanHyper()
    x.beta3, x.no_prox = h["betas"][2], int(h["no_prox"])
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
    return dict(dict(lr=1e-2, betas=(0.98, 0.92, 0.99), eps=1e-8, weight_decay=0.0, no_prox=False), **kw)


DEFAULT = _g(weight_decay=0.02)
G4 = [DEFAULT,
      _g(lr=3e-3, betas=(0.9, 0.9, 0.999), eps=1e-6, weight_decay=0.05, no_prox=True),
      _g(lr=5e-3, no_prox=True),
      _g(lr=2e-2, betas=(0.95, 0.8, 0.98))]

# name: gradient source, model copy, n_local, segments, groups, range table, per-parameter counts (with skip bits),
#       fp32 accumulator, found_inf step, clip
CASES = {
    "raw_bf16_default": ("raw_bf16", "bf16", 2_056, 0, [DEFAULT], False, False, False, 7, None),
    "main_4groups_per_param_clip_norm": ("main", "f32", 2_048, 7, G4, True, True, False, 11, ("norm", 0.05)),
    "raw_bf16_4groups_per_param_clip_value": ("raw_bf16", "bf16", 2_048, 64, G4, True, True, False, None,
                                              ("value", 4e-3)),
    "raw_f32_acc_2groups": ("raw_f32", None, 2_056, 5, G4[:2], True, False, True, 3, None),
    "main_wd0_no_prox": ("main", None, 2_040, 3, [G4[2]], False, False, False, None, ("norm", 10.0)),
}
STEPS = 16
KEYS = ("W", "M", "V", "D", "P")   # master, exp_avg, exp_avg_sq, exp_avg_diff, neg_pre_grad
STATE_KEY = {"M": "exp_avg", "V": "exp_avg_sq", "D": "exp_avg_diff", "P": "neg_pre_grad"}


@pytest.mark.parametrize("name", list(CASES))
def test_adan_kernel_matches_cuda_class_bit_for_bit(eng, name):
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
    ahyp = (L.AdanHyper * ng)(*[_ahyper(h) for h in groups])
    w0 = torch.from_numpy(rng.standard_normal(n_local).astype(np.float32) * 1e-1)
    B = {"W": Buf(n_local, F32, w0.cuda())}
    for k in ("M", "V", "D", "P"):
        B[k] = Buf(n_local, F32, torch.zeros(n_local).cuda())
    LPB = None if lp is None else Buf(N, BF16 if lp == "bf16" else F32, torch.full((N,), -5.0))
    gdt = {"raw_bf16": BF16, "raw_f32": F32, "main": F32}[src]
    GB = Buf(N if src != "main" else n_local, gdt)
    AB = Buf(N, F32) if use_acc else None
    nbc = len(ends) if per_range else ng
    BC = Buf(nbc * 4, F32, torch.full((nbc * 4,), float("nan")).cuda())
    rend = torch.tensor([e // 8 for e in ends], dtype=torch.int32).cuda()
    rsteps = torch.zeros(len(ends), dtype=torch.int32).cuda()
    sl = (C.c_size_t * (len(pieces) + 1))(*([p[0] for p in pieces] + [n_local]))
    sg = (C.c_size_t * len(pieces))(*[p[2] for p in pieces])
    lpp = L.ptr_array([LPB.ptr()]) if lp is not None else None
    grad_norm = 1.5
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0, grad_norm=grad_norm)
    masks = {j: torch.from_numpy(elem_range == j).cuda() for j in ranges}
    ref_params = {j: torch.nn.Parameter(w0.cuda()[masks[j]].clone()) for j in ranges}
    ref = Adan([dict(h, params=[ref_params[j] for j in ranges if rgroup[j] == gi]) for gi, h in enumerate(groups)])
    coef = None
    if clip is not None and clip[0] == "norm":
        coef = min(np.float32(clip[1]) / (np.float32(grad_norm) + np.float32(1e-6)), np.float32(1.0))
    g32 = rng.standard_normal(n_local).astype(np.float32)
    done, entry_done, late_first = 0, [0] * len(ends), set()
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
        before = {k: b.t.clone() for k, b in B.items()}
        snap = {k: b.bits() for k, b in B.items()}
        if LPB is not None:
            snap["LP"] = LPB.bits()
        eng._check(eng.lib.stk_adan_step_prologue(eng.ctx, hyp, ahyp, ng, len(ends) if per_range else 0,
                                                  rgrp.data_ptr() if per_range else None,
                                                  rsteps.data_ptr() if per_range else None, BC.ptr(), eng._stream()))
        a = L.OptimArgs()
        a.hyper, a.n_groups = hyp, ng
        a.master, a.exp_avg, a.exp_avg_sq, a.exp_avg_slow = B["W"].ptr(), B["M"].ptr(), B["V"].ptr(), B["D"].ptr()
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
        eng.adan_step(a, ahyp, B["P"].ptr())
        eng.step_epilogue()
        got = {k: b.t.clone() for k, b in B.items()}
        BC.check_guards()
        if per_range:
            bc = BC.t.view(-1, 4).cpu()
            for k in range(len(ends)):
                assert float(bc[k, 3]) == float(done == 0 or entry_done[k] == 0), (step, k)
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
        for grp in ref.param_groups:
            grp["step"] = done                        # the count lives in the group; the class advances it
        for j in ranges:
            p = ref_params[j]
            p.data.copy_(before["W"][masks[j]])
            p.grad = None if j in skip else gl[masks[j]].clone()
            st = ref.state[p]
            for k, key in STATE_KEY.items():          # restart from the kernel's state
                if key in st:
                    st[key] = before[k][masks[j]].clone()
        had = {j for j in ranges if ref.state[ref_params[j]]}
        if not found_inf:
            ref.step()
            done += 1
        late_first |= {j for j in ranges if ref.state[ref_params[j]] and j not in had and done > 1}
        assert int(eng.scaler_get().opt_steps) == done
        want = {k: before[k].clone() for k in KEYS}
        for j in ranges:
            p, s = ref_params[j], masks[j]
            want["W"][s] = p.detach()
            st = ref.state[p]
            if not st:
                continue
            for k, key in STATE_KEY.items():
                want[k][s] = st[key]
        for key in KEYS:
            assert _same(got[key], want[key]), f"step {step}: {key}"
        # ---- where the kernel wrote: nothing for skipped ranges or a found_inf step ----
        skip_elem = torch.from_numpy(np.isin(elem_range, list(skip))) | found_inf
        for key, b in B.items():
            b.check_unchanged_except(snap[key], ~skip_elem)
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
                assert torch.equal(glp.view(INT_VIEW[LPB.dtype]), wl.view(INT_VIEW[LPB.dtype]))
        if found_inf:
            assert all(torch.equal(b.bits(), snap[k]) for k, b in B.items())
    assert done == STEPS - (inf_at is not None)
    assert [grp["step"] for grp in ref.param_groups] == [done] * ng
    if per_range:   # some range first stepped after t = 1: a zero first difference under the group's t
        assert late_first


def _class_scalars(h, t):
    b1, b2, b3 = h["betas"]
    bc1, bc2, bc3 = 1 - b1 ** t, 1 - b2 ** t, 1 - b3 ** t
    return [float(np.float32(h["lr"] / bc1)), float(np.float32(h["lr"] * b2 / bc2)),
            float(np.float32(1 / math.sqrt(bc3)))]


def test_prologue_scalars_match_the_class(eng):
    """Per group at steps 1..40 (the optimizer-wide count); per range with its own counts: the bias corrections still
    use the optimizer-wide count, `first` follows the range's count, and a skipped range or a found_inf step does not
    advance it."""
    L = _L()
    groups = [G4[0], G4[1], _g(lr=0.3, betas=(0.5, 0.6, 0.7))]
    hyp = (L.OptimHyper * 3)(*[_hyper(h) for h in groups])
    ahyp = (L.AdanHyper * 3)(*[_ahyper(h) for h in groups])
    bc = torch.full((8, 4), float("nan"), device="cuda")
    for t in range(1, 41):
        eng.scaler_set(opt_steps=t - 1, found_inf=0)
        eng._check(eng.lib.stk_adan_step_prologue(eng.ctx, hyp, ahyp, 3, 0, None, None, bc.data_ptr(), eng._stream()))
        got = bc[:3].cpu()
        for gi, h in enumerate(groups):
            assert got[gi].tolist() == _class_scalars(h, t) + [float(t == 1)], (t, gi)
    rgroup = torch.tensor([0, 1, 2 | 0x80, 0], dtype=torch.uint8, device="cuda")
    rsteps = torch.tensor([0, 3, 0, 5], dtype=torch.int32, device="cuda")
    for found_inf in (1, 0):
        eng.scaler_set(opt_steps=5, found_inf=found_inf)
        eng._check(eng.lib.stk_adan_step_prologue(eng.ctx, hyp, ahyp, 3, 4, rgroup.data_ptr(), rsteps.data_ptr(),
                                                  bc.data_ptr(), eng._stream()))
        got = bc[:4].cpu()
        for j, (gi, first) in enumerate(((0, 1.0), (1, 0.0), (2, 1.0), (0, 0.0))):
            assert got[j].tolist() == _class_scalars(groups[gi], 6) + [first], (found_inf, j)
        assert rsteps.cpu().tolist() == ([0, 3, 0, 5] if found_inf else [1, 4, 0, 6])
    eng.scaler_set(found_inf=0)


def test_entry_points_require_their_buffers_and_scalars(eng):
    from stoke_b200.engine import StokeB200Error

    L = _L()
    bufs = [Buf(64, F32, torch.zeros(64).cuda()) for _ in range(7)]
    bc = torch.zeros(4, device="cuda")
    ah = (L.AdanHyper * 1)(_ahyper(DEFAULT))
    eng.scaler_set(opt_steps=0, found_inf=0)
    eng._check(eng.lib.stk_adan_step_prologue(eng.ctx, (L.OptimHyper * 1)(_hyper(DEFAULT)), ah, 1, 0, None, None,
                                              bc.data_ptr(), eng._stream()))

    def args(m=True, v=True, d=True, scalars=True):
        a = L.OptimArgs()
        a.hyper, a.n_groups = (L.OptimHyper * 1)(_hyper(DEFAULT)), 1
        a.master, a.grad, a.grad_dtype, a.n_local = bufs[0].ptr(), bufs[1].ptr(), L.F32, 64
        a.exp_avg = bufs[2].ptr() if m else None
        a.exp_avg_sq = bufs[3].ptr() if v else None
        a.exp_avg_slow = bufs[4].ptr() if d else None
        a.group_bc = bc.data_ptr() if scalars else None
        return a

    for kw in ({"m": False}, {"v": False}, {"d": False}, {"scalars": False}):
        with pytest.raises(StokeB200Error, match="stk_adan_step"):
            eng.adan_step(args(**kw), ah, bufs[5].ptr())
    with pytest.raises(StokeB200Error, match="neg_pre_grad"):
        eng.adan_step(args(), ah, None)
    with pytest.raises(StokeB200Error, match="stk_adan_step"):   # the kind's hyper-parameters have one entry point
        eng.optim_step_ex(args())
    adam = args()
    adam.hyper[0].kind = L.OPT_ADAM
    with pytest.raises(StokeB200Error, match="STK_OPT_ADAN"):
        eng.adan_step(adam, ah, bufs[5].ptr())
    eng.adan_step(args(), ah, bufs[5].ptr())
    torch.cuda.synchronize()
    for b in bufs:
        b.check_guards()


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


FACADE_KW = {"lr": 5e-3, "betas": (0.98, 0.92, 0.99), "weight_decay": 0.02}
STATE_KEYS = ("exp_avg", "exp_avg_sq", "exp_avg_diff", "neg_pre_grad")


def _stoke(fp16, clip, accum, stock, wa=None, kw=FACADE_KW):
    model = Net()
    used = [p for m in model.layers for p in m.parameters()]
    unused = dict(params=list(model.unused.parameters()), weight_decay=0.0, no_prox=True)
    if stock:   # 9 groups: more than the fused step takes, so Stoke builds the stock route
        groups = [dict(params=[p]) for p in used] + [unused]
    else:
        groups = [dict(params=used), unused]
    grad_clip = None
    if clip is not None:
        grad_clip = sb.ClipGradNormConfig(max_norm=clip[1], norm_type=2.0) if clip[0] == "norm" else \
            sb.ClipGradConfig(clip_value=clip[1])
    return sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=Adan, optimizer_kwargs=dict(kw, params=groups)),
                    loss=_mse, batch_size_per_device=8, grad_accum_steps=accum, grad_clip=grad_clip, gpu=True, fp16=fp16,
                    verbose=False, configs=[wa] if wa is not None else None)


def _drive(s, steps, fp16, accum, seed=0, each=None, inf_at=None):
    dt = torch.float32 if fp16 in (None, "amp") else torch.bfloat16
    g = torch.Generator().manual_seed(seed)
    for step in range(steps):
        for _ in range(accum):
            x, y = torch.randn(8, 16, generator=g).cuda().to(dt), torch.randn(8, 1, generator=g).cuda()
            loss = s.loss(s.model(x), y)
            if step == inf_at:
                loss = loss * float("inf")
            s.backward(loss)
            s.step()
        if each is not None:
            each(s)


def _compare_runs(fp16, clip, accum, steps, inf_at=None):
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    torch.cuda.set_device(0)
    runs = []
    for stock in (False, True):
        s = _stoke(fp16, clip, accum, stock)
        assert isinstance(s.optimizer, B200StockOptimizer if stock else B200FusedOptimizer)
        _drive(s, steps, fp16, accum, inf_at=inf_at)
        runs.append((s, s.optimizer.path.gather_master().cpu(), s.optimizer.state_dict()))
    (fs, fw, fsd), (ss, sw, ssd) = runs
    taken = steps - (inf_at is not None)
    exact = clip is None or clip[0] == "value"
    assert _same(fw, sw) if exact else _rel(fw, sw) < 1e-5
    assert [g["step"] for g in fsd["param_groups"]] == [taken] * 2
    assert [g["step"] for g in ssd["param_groups"]] == [taken] * 9
    for i in range(8):
        assert list(fsd["state"][i]) == list(STATE_KEYS) == list(ssd["state"][i])
        for k in STATE_KEYS:
            a, b = fsd["state"][i][k].cpu(), ssd["state"][i][k].cpu()
            assert _same(a, b) if exact else _rel(a, b) < 1e-5, (i, k)
    assert 8 not in fsd["state"] and 9 not in fsd["state"]   # the unused Linear: never stepped
    path = fs.optimizer.path
    init = Net().unused
    got = path.unflatten(path.gather_master().cpu())
    assert torch.equal(got[8], init.weight.detach()) and torch.equal(got[9], init.bias.detach())
    for s in (fs, ss):
        if inf_at is not None:
            assert s.engine.scaler_get(s.optimizer.path.state_id).skipped_steps == 1
        s.optimizer.close()


@pytest.mark.parametrize("accum", [1, 2])
@pytest.mark.parametrize("clip", [None, ("value", 0.05), ("norm", 0.5)], ids=["noclip", "value", "norm"])
@pytest.mark.parametrize("fp16", [None, "bf16"], ids=["fp32", "bf16"])
def test_stoke_facade_matches_stock_route(fp16, clip, accum):
    """The fused step and the class's own step on the stock route (9 groups) give the same master, the same four state
    tensors and the same group step counts bit for bit over 9 steps; the never-used parameter keeps its weights and has
    no state entry.  Clip by norm takes its norm from different kernels on the two routes, so there the bar is fp32
    tolerance."""
    _compare_runs(fp16, clip, accum, 9)


def test_stoke_facade_amp_with_a_skipped_step():
    """fp16 AMP with a step whose loss is infinite: the scaler skips it on both routes, the group count does not
    advance and neg_pre_grad keeps the last applied step's gradient, so the runs still agree bit for bit."""
    _compare_runs("amp", None, 1, 7, inf_at=3)


def _fused(net, kw, lp=None, stock=False, accum=1):
    from stoke_b200.engine import get_engine
    from stoke_b200.optim import B200FusedOptimizer, B200StockOptimizer

    cls = B200StockOptimizer if stock else B200FusedOptimizer
    return cls(net, Adan, kw, engine=get_engine(0), grad_accum=accum, lp_dtype=lp)


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
    """Two groups: proximal weight decay, and no_prox with other betas."""
    ps = list(net.parameters())
    return dict(lr=1e-2, betas=(0.98, 0.92, 0.99), weight_decay=0.02,
                params=[dict(params=ps[:4]), dict(params=ps[4:], no_prox=True, betas=(0.9, 0.9, 0.999))])


def test_checkpoints_continue_bit_for_bit():
    """A checkpoint saved after 4 steps continues like the uninterrupted 12-step run, bit for bit: fused -> fused,
    fused -> plain class (4 steps) -> fused (4 steps), and fused -> stock -> fused.  The group count travels as
    ``param_groups[*]["step"]``."""
    torch.cuda.set_device(0)

    def make(stock=False, net=None):
        net = net if net is not None else OddNet().cuda()
        return _fused(net, _ckpt_kw(net), stock=stock)

    cont = make()
    _run_injected(cont, range(12))
    want = _masters(cont)
    want_sd = cont.state_dict()
    assert [g["step"] for g in want_sd["param_groups"]] == [12, 12]
    cont.close()

    first = make()
    assert all("step" not in g for g in first.state_dict()["param_groups"])   # absent before the first step
    _run_injected(first, range(4))
    sd = first.state_dict()
    assert [g["step"] for g in sd["param_groups"]] == [4, 4]
    for e in sd["state"].values():
        assert list(e) == list(STATE_KEYS)
    again = make()
    again.load_state_dict(sd)
    _run_injected(again, range(4, 12))
    assert all(_same(a, b) for a, b in zip(_masters(again), want))
    again.close()
    # fused -> plain class -> fused
    plain = [torch.nn.Parameter(w.cuda().clone()) for w in first.path.unflatten(first.path.gather_master())]
    topt = Adan(**_ckpt_kw(torch.nn.ParameterList(plain)))
    topt.load_state_dict({k: v for k, v in sd.items() if not k.startswith("b200_")})
    assert [g["step"] for g in topt.param_groups] == [4, 4]
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
    assert [g["step"] for g in got_sd["param_groups"]] == [12, 12]
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


def test_weight_average_on_top():
    """An EMA of the weights over the fused Adan step: the master is the run's without averaging, bit for bit, and the
    average is AveragedModel's update (copy, then torch's fp32 lerp with 1 - decay) applied to every step's master."""
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
    """fairscale_oss at W = 2: Adan sharded (ZeRO-1, in-kernel parameter all-gather, all four state streams split) against
    the replicated all-reduce route: final weights, the gathered state_dict and the group counts bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "adan_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29579", os.path.join(ROOT, "tests", "adan_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    assert res["sharded_route"] == "sharded" and res["replicated_route"] == "allreduce", res
    assert res["weights_identical"] and res["state_identical"], res
