"""NAdam, RAdam and Adamax on the fused step (GPU).

Kernel level: stk_optim_step_prologue + stk_optim_step_ex called directly and compared element by element with the float64
reference of tests/optim_family_ref.py, restarted from the kernel's own state every step, with the buffers between guard
bands (see test_gpu_kernels.py).  Engine level: gradient-injection parity of B200FusedOptimizer with the CPU oracle,
unused parameters, the Stoke facade, and checkpoints exchanged with plain torch."""
import ctypes as C
import math
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import kernel_ref as kr
import optim_family_ref as ofr
from test_gpu_kernels import BF16, F32, INT_VIEW, Buf, _dt, _layout

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-5
BASE = {"lr": 2.0**-7, "beta1": 0.875, "beta2": 0.999, "eps": 2.0**-20, "momentum_decay": 4e-3}
KIND_BASE = {"nadam": BASE, "radam": BASE, "adamax": dict(BASE, eps=2.0**-12)}
CLS = {"nadam": torch.optim.NAdam, "radam": torch.optim.RAdam, "adamax": torch.optim.Adamax}


def _L():
    from stoke_b200 import _lib

    return _lib


def _hyper(kind, h):
    L = _L()
    o = L.OptimHyper()
    o.kind = {"nadam": L.OPT_NADAM, "radam": L.OPT_RADAM, "adamax": L.OPT_ADAMAX}[kind]
    o.lr, o.beta1, o.beta2, o.eps = h["lr"], h["beta1"], h["beta2"], h["eps"]
    o.weight_decay = h.get("weight_decay", 0.0)
    o.maximize = int(h.get("maximize", False))
    o.clip_kind = L.CLIP_NONE
    return o


def _ext(h):
    x = _L().OptimHyperExt()
    x.momentum_decay = h.get("momentum_decay", 4e-3)
    x.decoupled_weight_decay = int(bool(h.get("decoupled_weight_decay", False)))
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


def _groups8(kind):
    b = KIND_BASE[kind]
    return [b, dict(b, lr=2.0**-6, beta2=0.99), dict(b, weight_decay=0.25), dict(b, maximize=True),
            dict(b, weight_decay=0.25, decoupled_weight_decay=True), dict(b, momentum_decay=0.05, beta1=0.75),
            dict(b, lr=0.0), dict(b, lr=2.0**-8, eps=1e-8)]


def _cases():
    out = {}
    for kind in ofr.KINDS:
        b = KIND_BASE[kind]
        out[f"{kind}_raw_bf16"] = (kind, "raw_bf16", "bf16", 2_048, 0, [b], False, False, {})
        out[f"{kind}_raw_f32_l2_inf"] = (kind, "raw_f32", None, 2_056, 3, [dict(b, weight_decay=0.25)], False, False,
                                         {"found_inf_at": 2})
        out[f"{kind}_main_decoupled_max"] = (kind, "main", "f32", 2_040, 0,
                                             [dict(b, weight_decay=0.25, decoupled_weight_decay=True, maximize=True)],
                                             False, False, {})
        out[f"{kind}_seg64_8groups_steps"] = (kind, "raw_bf16", "bf16", 2_048, 64, _groups8(kind), True, True,
                                              {"per_range": True, "found_inf_at": 4})
        out[f"{kind}_main_2groups"] = (kind, "main", "bf16", 2_048, 7, _groups8(kind)[3:5], True, False, {})
    return out


CASES = _cases()
STEPS = 8   # RAdam with beta2 = 0.999 takes its first rectified step at t = 6


@pytest.mark.parametrize("name", list(CASES))
def test_optim_family_step_matches_torch_float64(eng, name):
    L = _L()
    kind, src, lp, n_local, n_seg, groups, use_ranges, use_skip, ex = CASES[name]
    per_range = ex.get("per_range", False)
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
    hyp = (L.OptimHyper * ng)(*[_hyper(kind, h) for h in groups])
    ext = (L.OptimHyperExt * ng)(*[_ext(h) for h in groups])
    g32 = rng.standard_normal(n_local).astype(np.float32)
    w0 = torch.from_numpy(rng.standard_normal(n_local).astype(np.float32) * 1e-3)
    MB = Buf(n_local, F32, w0.cuda())
    MM = Buf(n_local, F32, torch.zeros(n_local).cuda())
    VV = Buf(n_local, F32, torch.zeros(n_local).cuda())
    LPB = None if lp is None else Buf(N, BF16 if lp == "bf16" else F32, torch.full((N,), -5.0))
    gdt = {"raw_bf16": BF16, "raw_f32": F32, "main": F32}[src]
    GB = Buf(N if src != "main" else n_local, gdt)
    nb = len(ends) if per_range else ng
    MU = Buf(nb, F32, torch.ones(nb).cuda())
    BC = Buf(nb * 4, F32)
    if use_ranges:
        rend = torch.tensor([e // 8 for e in ends], dtype=torch.int32).cuda()
        rgrp = torch.tensor([g | (0x80 if s else 0) for g, s in zip(rgroup, rskip)], dtype=torch.uint8).cuda()
    rsteps = torch.tensor([3 if j % 3 == 2 else 0 for j in range(len(ends))], dtype=torch.int32).cuda()
    sl = (C.c_size_t * (len(pieces) + 1))(*([p[0] for p in pieces] + [n_local]))
    sg = (C.c_size_t * len(pieces))(*[p[2] for p in pieces])
    lpp = L.ptr_array([LPB.ptr()]) if lp is not None else None
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0)
    # groups that own stepped local elements (the shuffled layout can leave a range without any)
    live = {rgroup[j] for j in range(len(ends)) if not rskip[j] and bool((elem_range == j).any())}
    muts = set(ofr.MUTATIONS[kind]) - ({"decoupled_as_l2"} if not any(
        groups[gi].get("decoupled_weight_decay") and groups[gi].get("weight_decay") for gi in live) else set())
    hit = set()

    for step in range(STEPS):
        g = torch.from_numpy(np.roll(g32, step * 37) * 1e-3).to(gdt)
        gfull = torch.zeros(GB.n, dtype=gdt)
        if src == "main":
            gfull[:] = g
        else:
            gfull[:] = torch.from_numpy(rng.standard_normal(GB.n).astype(np.float32)).to(gdt)
            gfull[torch.from_numpy(gidx)] = g
        GB.t.copy_(gfull.cuda())
        found_inf = ex.get("found_inf_at") == step
        eng.scaler_set(found_inf=int(found_inf))
        st0 = eng.scaler_get()
        w, m, v = MB.t.cpu().clone(), MM.t.cpu().clone(), VV.t.cpu().clone()
        mu_before = MU.t.cpu().clone()
        snap = {k: b.bits() for k, b in (("G", GB), ("M", MB), ("MM", MM), ("VV", VV), ("LP", LPB), ("MU", MU)) if b}
        steps_before = rsteps.cpu().clone()
        # prologue + step
        if per_range:
            eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, ext, ng, len(ends), rgrp.data_ptr(), rsteps.data_ptr(),
                                                       MU.ptr(), BC.ptr(), eng._stream()))
        else:
            eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, ext, ng, 0, None, None, MU.ptr(), BC.ptr(),
                                                       eng._stream()))
        a = L.OptimArgs()
        a.hyper, a.n_groups, a.hyper_ext = hyp, ng, ext
        a.master, a.exp_avg, a.exp_avg_sq = MB.ptr(), MM.ptr(), VV.ptr()
        a.grad, a.grad_dtype, a.grad_raw, a.grad_mul = GB.ptr(), _dt(gdt), int(src != "main"), 1.0
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
        got_w, got_m, got_v = MB.t.cpu(), MM.t.cpu(), VV.t.cpu()
        got_bc, got_mu = BC.t.cpu().view(nb, 4), MU.t.cpu()

        # ---- reference, per range ----
        skip_elem = torch.from_numpy(np.asarray(rskip)[elem_range]) | found_inf
        rw, rm, rv = w.double().clone(), m.double().clone(), v.double().clone()
        bw, bm, bv = (torch.zeros(n_local, dtype=torch.float64) for _ in range(3))
        mw = {mu: w.double().clone() for mu in muts}
        for j in range(len(ends)):
            s = torch.from_numpy(elem_range == j)
            gi = rgroup[j]
            h = groups[gi]
            done = int(steps_before[j]) if per_range else int(st0.opt_steps)
            slot = j if per_range else gi
            mu0 = float(mu_before[slot])
            # the prologue's scalars (1 fp32 ulp) and mu_product (bit for bit; unchanged when not stepped)
            want, want_mu = ofr.prologue_scalars(kind, h, done, mu0)
            for k in range(4):
                assert abs(float(got_bc[slot, k]) - want[k]) <= float(np.spacing(np.float32(abs(want[k])))), (step, j, k)
            stepped = not (rskip[j] or found_inf)
            if kind == "nadam":
                assert float(got_mu[slot]) == (want_mu if stepped else mu0), (step, j)
            if per_range:
                assert int(rsteps[j]) == done + (1 if stepped else 0)
            if not bool(s.any()) or not stepped:
                continue
            G = g[s].double() if src != "raw_bf16" else g[s].float().double()
            nw, nm, nv, _ = ofr.step_ref(kind, w[s], m[s], v[s], G, done, h, mu0)
            ew, em, ev = ofr.step_bound(kind, w[s], m[s], v[s], G, torch.zeros_like(G), done, h, nm, nv, mu0)
            rw[s], rm[s], rv[s], bw[s], bm[s], bv[s] = nw, nm, nv, ew, em, ev
            for mu in muts:
                if mu == "mu_not_advanced" and mu0 == 1.0:
                    continue
                mw[mu][s] = ofr.step_mutant(kind, w[s], m[s], v[s], G, done, h, mu, mu0)
        for what, got, ref, b in (("master", got_w, rw, bw), ("exp_avg", got_m, rm, bm), ("exp_avg_sq/exp_inf", got_v, rv, bv)):
            bad = (got.double() - ref).abs() > b
            assert not bool(bad.any()), f"step {step}: {what} off at {torch.nonzero(bad)[:5].flatten().tolist()}"
        for mu in muts:
            if bool(((got_w.double() - mw[mu]).abs() > bw).any()):
                hit.add(mu)
        # ---- where the kernel wrote ----
        frozen = skip_elem.clone()
        for j in range(len(ends)):
            if groups[rgroup[j]]["lr"] == 0.0 and not (groups[rgroup[j]].get("decoupled_weight_decay")):
                frozen |= torch.from_numpy(elem_range == j)
        MB.check_unchanged_except(snap["M"], ~frozen)
        MM.check_unchanged_except(snap["MM"], ~skip_elem)
        VV.check_unchanged_except(snap["VV"], ~skip_elem)
        assert torch.equal(got_w[frozen].view(torch.int32), w[frozen].view(torch.int32))
        if src != "main":
            seg = torch.zeros(GB.n, dtype=torch.bool)
            seg[torch.from_numpy(gidx)] = True
            GB.check_unchanged_except(snap["G"], seg)
            assert float(GB.t[torch.from_numpy(gidx).cuda()].float().abs().max()) == 0.0
        else:
            GB.check_unchanged_except(snap["G"], torch.zeros(GB.n, dtype=torch.bool))
        if LPB is not None:
            stepped_e = ~skip_elem
            mask = torch.zeros(LPB.n, dtype=torch.bool)
            mask[torch.from_numpy(gidx)[stepped_e]] = True
            LPB.check_unchanged_except(snap["LP"], mask)
            if bool(stepped_e.any()):
                glp = LPB.t[torch.from_numpy(gidx)[stepped_e].cuda()].cpu()
                assert torch.equal(glp.view(INT_VIEW[LPB.dtype]), got_w[stepped_e].to(LPB.dtype).view(INT_VIEW[LPB.dtype]))
        if found_inf:   # a skipped step: master, moments and mu_product bit-identical
            assert torch.equal(MB.bits(), snap["M"]) and torch.equal(MM.bits(), snap["MM"]) and torch.equal(VV.bits(), snap["VV"])
            assert torch.equal(MU.bits(), snap["MU"])
        MU.check_guards()
        BC.check_guards()
    assert hit == muts, f"negative controls that passed every step: {muts - hit}"


@pytest.mark.parametrize("kind", ofr.KINDS)
@pytest.mark.parametrize("src", ["raw_bf16", "main"])
def test_nan_gradient_without_scaler_follows_torch(eng, kind, src):
    """A NaN gradient element without a loss scaler: torch's fp32 step makes exactly that element's weight and state NaN
    (Adamax's exp_inf through the NaN-propagating torch.maximum); the kernel must give the same NaN pattern."""
    L = _L()
    n = 2_048
    h = KIND_BASE[kind]
    g = (torch.randn(n, generator=torch.Generator().manual_seed(5)) * 1e-3).to(BF16 if src == "raw_bf16" else F32)
    g[[3, 700, 2047]] = float("nan")
    w0 = torch.randn(n, generator=torch.Generator().manual_seed(6)) * 1e-3
    MB, MM, VV = Buf(n, F32, w0.cuda()), Buf(n, F32, torch.zeros(n).cuda()), Buf(n, F32, torch.zeros(n).cuda())
    GB = Buf(n, g.dtype, g.cuda())
    MU, BC = Buf(1, F32, torch.ones(1).cuda()), Buf(4, F32)
    hyp, ext = (L.OptimHyper * 1)(_hyper(kind, h)), (L.OptimHyperExt * 1)(_ext(h))
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0)
    eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, ext, 1, 0, None, None, MU.ptr(), BC.ptr(), eng._stream()))
    a = L.OptimArgs()
    a.hyper, a.n_groups, a.hyper_ext, a.group_bc = hyp, 1, ext, BC.ptr()
    a.master, a.exp_avg, a.exp_avg_sq = MB.ptr(), MM.ptr(), VV.ptr()
    a.grad, a.grad_dtype, a.grad_raw, a.grad_mul = GB.ptr(), _dt(g.dtype), int(src != "main"), 1.0
    a.n_local = n
    if src == "raw_bf16":   # the raw bf16 route writes the bf16 model copy
        LPB = Buf(n, BF16)
        lpp = L.ptr_array([LPB.ptr()])
        a.lp_ptrs, a.lp_world, a.lp_dtype = lpp, 1, L.BF16
    else:
        a.lp_ptrs, a.lp_world, a.lp_dtype = None, 0, L.F32
    eng.optim_step_ex(a)
    eng.step_epilogue()
    p = torch.nn.Parameter(w0.clone())
    opt = ofr.make_optimizer(kind, [p], h)
    p.grad = g.float()
    opt.step()
    st = opt.state[p]
    for got, want in ((MB.t.cpu(), p.detach()), (MM.t.cpu(), st["exp_avg"]), (VV.t.cpu(), st[ofr.second_key(kind)])):
        assert torch.equal(got.isnan(), want.isnan())
    assert int(MB.t.cpu().isnan().sum()) == 3


# ---- engine level ------------------------------------------------------------------------------------------------------------
from test_gpu_engine import OddNet, _inject, _oracle_flat, _rel  # noqa: E402

ENGINE_CASES = [
    (torch.optim.NAdam, {"lr": 2e-3}, torch.bfloat16, ("norm", 1.0, 2.0), 1),
    (torch.optim.NAdam, {"lr": 2e-3, "weight_decay": 0.05, "decoupled_weight_decay": True, "momentum_decay": 0.01},
     None, None, 2),
    (torch.optim.RAdam, {"lr": 1e-3, "weight_decay": 0.01}, torch.bfloat16, ("value", 0.3), 1),
    (torch.optim.RAdam, {"lr": 1e-3, "weight_decay": 0.05, "decoupled_weight_decay": True, "maximize": True}, None,
     ("norm", 0.5, 2.0), 1),
    (torch.optim.Adamax, {"lr": 2e-3, "weight_decay": 0.01}, torch.bfloat16, None, 1),
    (torch.optim.Adamax, {"lr": 2e-3, "betas": (0.8, 0.99)}, None, ("norm", 1.0, float("inf")), 2),
]


def _fused(net, cls, kw, lp, clip=None, accum=1, route=None):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import B200FusedOptimizer

    spec = None
    if clip is not None:
        spec = ClipSpec(_lib.CLIP_NORM, max_norm=clip[1], norm_type=clip[2]) if clip[0] == "norm" else \
            ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1])
    return B200FusedOptimizer(net, cls, kw, engine=get_engine(0), grad_accum=accum, clip=spec, lp_dtype=lp, route=route)


def _check_state(sd, oracle, cls):
    k_v = "exp_inf" if cls is torch.optim.Adamax else "exp_avg_sq"
    for i, p in enumerate(oracle.params):
        st = oracle.optimizer.state[p]
        assert _rel(sd["state"][i]["exp_avg"].cpu(), st["exp_avg"]) < TOL
        assert _rel(sd["state"][i][k_v].cpu(), st[k_v]) < TOL
        assert float(sd["state"][i]["step"]) == float(st["step"])
        assert sd["state"][i]["step"].dtype == torch.float32 and sd["state"][i]["step"].dim() == 0
        assert set(sd["state"][i]) == set(st), (set(sd["state"][i]), set(st))
        if cls is torch.optim.NAdam:
            got, want = sd["state"][i]["mu_product"], st["mu_product"]
            assert got.dtype == torch.float32 and got.dim() == 0
            assert abs(float(got) - float(want)) <= float(np.spacing(np.float32(float(want))))


@pytest.mark.parametrize("route", ["local", "main"])
@pytest.mark.parametrize("cls,kw,lp,clip,accum", ENGINE_CASES)
def test_gradient_injection_parity(cls, kw, lp, clip, accum, route):
    from engine_oracle import OracleEngine
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    net = OddNet().cuda()
    init = [p.detach().cpu().clone() for p in net.parameters()]
    opt = _fused(net, cls, kw, lp, clip, accum, route=route)
    assert isinstance(opt, B200FusedOptimizer) and opt.path.route == route
    path = opt.path
    oracle = OracleEngine(init, 1, cls, kw, grad_accum=accum, clip=clip)
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
    _check_state(opt.state_dict(), oracle, cls)
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


@pytest.mark.parametrize("cls", [torch.optim.NAdam, torch.optim.RAdam, torch.optim.Adamax])
def test_unused_parameter_and_stoke_facade(cls):
    """Through Stoke: the class builds a B200FusedOptimizer; head b is unused on some steps, so step counts (and NAdam's
    mu_product) go per parameter, as torch keeps them; every parameter, moment and count follows the oracle."""
    from engine_oracle import OracleEngine
    import stoke_b200 as sb
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    kw = {"lr": 1e-2, "weight_decay": 0.1}
    model = TwoHeads()
    init = [p.detach().clone() for p in model.parameters()]
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=cls, optimizer_kwargs=kw), loss=torch.nn.MSELoss(),
                 batch_size_per_device=8, gpu=True, verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    oracle = OracleEngine(init, 1, cls, kw)
    path = s.optimizer.path
    g = torch.Generator().manual_seed(0)
    for step in range(9):
        model.use_b = step % 3 != 1
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
    for a, b in zip(model.parameters(), oracle.weights()):
        assert _rel(a.detach().float().cpu().reshape(-1), b.reshape(-1)) < TOL
    sd = s.optimizer.state_dict()
    _check_state(sd, oracle, cls)
    assert [float(sd["state"][j]["step"]) for j in range(6)] == [9.0, 9.0, 9.0, 9.0, 6.0, 6.0]
    s.optimizer.close()


@pytest.mark.parametrize("cls,kw", [(torch.optim.NAdam, {"lr": 2e-3, "weight_decay": 0.01}),
                                    (torch.optim.RAdam, {"lr": 1e-3, "decoupled_weight_decay": True, "weight_decay": 0.1}),
                                    (torch.optim.Adamax, {"lr": 2e-3})])
def test_checkpoint_round_trip_with_plain_torch(cls, kw):
    """Engine -> torch: the engine's state_dict loaded into the plain CPU class continues to the same weights as the engine.
    torch -> engine: a plain torch state dict (no b200_* keys; the model weights loaded first) continues the same way."""
    torch.cuda.set_device(0)
    net = OddNet().cuda()
    opt = _fused(net, cls, kw, None)
    path = opt.path
    grads_of = lambda step: _inject(path, step, 0, torch.float32)   # noqa: E731 -- writes the engine's bucket too
    for step in range(4):
        grads_of(step)
        path.after_backward(sync=True, unscale=False)
        opt.step()
    sd = opt.state_dict()
    # engine -> torch
    cpu_params = [torch.nn.Parameter(w.cpu().clone()) for w in path.unflatten(path.gather_master())]
    topt = cls(cpu_params, **kw, foreach=False)
    topt.load_state_dict({k: v for k, v in sd.items() if not k.startswith("b200_")})
    for step in range(4, 8):
        for p, gr in zip(cpu_params, grads_of(step)):
            p.grad = gr.reshape(p.shape).clone()
        path.after_backward(sync=True, unscale=False)
        opt.step()
        topt.step()
    for a, b in zip(path.unflatten(path.gather_master().cpu()), cpu_params):
        assert _rel(a.reshape(-1), b.detach().reshape(-1)) < TOL
    # torch -> engine: a fresh engine optimizer from torch's state dict (reference format)
    net2 = OddNet().cuda()
    with torch.no_grad():
        for p, q in zip(net2.parameters(), cpu_params):
            p.copy_(q.detach())
    opt2 = _fused(net2, cls, kw, None)
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
        if cls is torch.optim.NAdam:
            assert abs(float(sd2["state"][i]["mu_product"]) - float(topt.state[p]["mu_product"])) <= \
                float(np.spacing(np.float32(float(topt.state[p]["mu_product"]))))
    opt.close()
    opt2.close()


@pytest.mark.multigpu
def test_sharded_matches_unsharded_w2(tmp_path):
    """fairscale_oss at W = 2: NAdam and RAdam sharded (ZeRO-1, in-kernel parameter all-gather) against the same classes
    replicated (all-reduce route): final weights and the gathered state_dict bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "optim_family_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29561", os.path.join(ROOT, "tests", "optim_family_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420,
                          env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    assert set(res) == {"nadam", "radam"}
    for name, r in res.items():
        assert r["sharded_route"] == "sharded" and r["replicated_route"] == "allreduce", (name, r)
        assert r["weights_identical"] and r["state_identical"], (name, r)
