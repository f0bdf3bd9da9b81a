"""Adadelta, Rprop and ASGD on the fused step (GPU).

Kernel level: stk_optim_step_prologue + stk_optim_step_ex called directly and compared element by element with the
references of tests/optim_elementwise_ref.py (Adadelta and ASGD within their fp32 bounds, Rprop bit for bit), restarted from
the kernel's own state every step, with the buffers between guard bands (see test_gpu_kernels.py).  Engine level:
gradient-injection parity of B200FusedOptimizer with the CPU oracle, unused parameters, the Stoke facade, checkpoints
exchanged with plain torch and a step without host synchronisation."""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import optim_elementwise_ref as oer
from test_gpu_kernels import BF16, F32, INT_VIEW, Buf, _dt, _layout

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-5
KIND_BASE = {"adadelta": {"lr": 0.5, "rho": 0.875, "eps": 1e-6},
             "rprop": {"lr": 2.0**-7, "etas": (0.5, 1.2), "step_sizes": (1e-6, 50.0)},
             "asgd": {"lr": 2.0**-4, "lambd": 1e-2, "alpha": 0.75, "t0": 1e6}}


def _L():
    from stoke_b200 import _lib

    return _lib


def _hyper(kind, h):
    L = _L()
    o = L.OptimHyper()
    o.kind = {"adadelta": L.OPT_ADADELTA, "rprop": L.OPT_RPROP, "asgd": L.OPT_ASGD}[kind]
    o.lr = h["lr"]
    o.eps = h.get("eps", 0.0)
    o.weight_decay = h.get("weight_decay", 0.0)
    o.maximize = int(h.get("maximize", False))
    o.clip_kind = L.CLIP_NONE
    return o


def _ext(h):
    x = _L().OptimHyperExt()
    x.rho = h.get("rho", 0.0)
    x.etaminus, x.etaplus = h.get("etas", (0.0, 0.0))
    x.step_size_min, x.step_size_max = h.get("step_sizes", (0.0, 0.0))
    x.lambd, x.alpha, x.t0 = h.get("lambd", 0.0), h.get("alpha", 0.0), h.get("t0", 0.0)
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
    if kind == "adadelta":
        return [b, dict(b, lr=1.0, rho=0.9), dict(b, weight_decay=0.25), dict(b, maximize=True), dict(b, eps=1e-4),
                dict(b, rho=0.5), dict(b, lr=0.0), dict(b, lr=0.25, weight_decay=0.5, maximize=True)]
    if kind == "rprop":
        return [b, dict(b, lr=2.0**-6), dict(b, etas=(1.0, 1.2)), dict(b, maximize=True), dict(b, etas=(1.2, 1.2)),
                dict(b, step_sizes=(2.0**-9, 2.0**-6)), dict(b, lr=0.0), dict(b, etas=(0.25, 2.0))]
    return [b, dict(b, lr=2.0**-5), dict(b, weight_decay=0.25), dict(b, maximize=True), dict(b, t0=2.0),
            dict(b, lambd=0.1, alpha=0.5), dict(b, lr=0.0), dict(b, t0=4.0, weight_decay=0.5)]


def _cases():
    out = {}
    for kind in oer.KINDS:
        b = KIND_BASE[kind]
        wd = {} if kind == "rprop" else {"weight_decay": 0.25}
        out[f"{kind}_raw_bf16"] = (kind, "raw_bf16", "bf16", 2_048, 0, [b], False, False, {})
        out[f"{kind}_raw_f32_wd_inf"] = (kind, "raw_f32", None, 2_056, 3, [dict(b, **wd)], False, False, {"found_inf_at": 2})
        out[f"{kind}_main_max"] = (kind, "main", "f32", 2_040, 0, [dict(b, maximize=True, **wd)], False, False, {})
        out[f"{kind}_seg64_8groups_steps"] = (kind, "raw_bf16", "bf16", 2_048, 64, _groups8(kind), True, True,
                                              {"per_range": True, "found_inf_at": 4})
        out[f"{kind}_main_2groups"] = (kind, "main", "bf16", 2_048, 7, _groups8(kind)[3:5], True, False, {})
    return out


CASES = _cases()
STEPS = 8


def _grad(kind, n, rng, step, g32):
    g = np.roll(g32, step * 37) * 1e-3
    if kind == "rprop":   # tiny gradients whose fp32 product with prev underflows to 0 (the sign is taken on the product)
        g[: n // 8] *= 1e-22
    if step % 3 == 2:
        g[n // 8: n // 8 + 64] = 0.0
    return g


@pytest.mark.parametrize("name", list(CASES))
def test_elementwise_step_matches_torch(eng, name):
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
    # Rprop's step_size buffer starts as NaN: its first step must seed it from lr without reading it
    VV = None if kind == "asgd" else Buf(n_local, F32, torch.full((n_local,), float("nan") if kind == "rprop" else 0.0).cuda())
    LPB = None if lp is None else Buf(N, BF16 if lp == "bf16" else F32, torch.full((N,), -5.0))
    gdt = {"raw_bf16": BF16, "raw_f32": F32, "main": F32}[src]
    GB = Buf(N if src != "main" else n_local, gdt)
    nb = len(ends) if per_range else ng
    width = 2 if kind == "asgd" else 1
    SC = Buf(nb * width, F32, torch.full((nb * width,), float("nan")).cuda())   # never read before the first step
    BC = Buf(nb * 4, F32)
    if use_ranges:
        rend = torch.tensor([e // 8 for e in ends], dtype=torch.int32).cuda()
        rgrp = torch.tensor([g | (0x80 if s else 0) for g, s in zip(rgroup, rskip)], dtype=torch.uint8).cuda()
    rsteps = torch.zeros(len(ends), dtype=torch.int32).cuda()
    sl = (C.c_size_t * (len(pieces) + 1))(*([p[0] for p in pieces] + [n_local]))
    sg = (C.c_size_t * len(pieces))(*[p[2] for p in pieces])
    lpp = L.ptr_array([LPB.ptr()]) if lp is not None else None
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0)
    live = {rgroup[j] for j in range(len(ends)) if not rskip[j] and bool((elem_range == j).any())}
    muts = set(oer.MUTATIONS[kind])
    if kind == "rprop":   # the mask quirk only shows with etaminus == 1 or etaplus == etaminus
        if not any(groups[gi]["etas"][0] in (1.0, groups[gi]["etas"][1]) for gi in live):
            muts.discard("no_mask_quirk")
    if kind == "asgd":
        muts.discard("never_average" if all(groups[gi]["t0"] > 100 for gi in live) else "always_average")
    hit = set()

    for step in range(STEPS):
        g = torch.from_numpy(_grad(kind, n_local, rng, step, g32).astype(np.float32)).to(gdt)
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
        w, m = MB.t.cpu().clone(), MM.t.cpu().clone()
        v = VV.t.cpu().clone() if VV else None
        sc_before = SC.t.cpu().clone().view(nb, width)
        snap = {k: b.bits() for k, b in (("G", GB), ("M", MB), ("MM", MM), ("VV", VV), ("LP", LPB), ("SC", SC)) if b}
        steps_before = rsteps.cpu().clone()
        if per_range:
            eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, ext, ng, len(ends), rgrp.data_ptr(), rsteps.data_ptr(),
                                                       SC.ptr(), BC.ptr(), eng._stream()))
        else:
            eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, ext, ng, 0, None, None, SC.ptr(), BC.ptr(),
                                                       eng._stream()))
        a = L.OptimArgs()
        a.hyper, a.n_groups, a.hyper_ext = hyp, ng, ext
        a.master, a.exp_avg, a.exp_avg_sq = MB.ptr(), MM.ptr(), (VV.ptr() if VV else None)
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
        got_w, got_m = MB.t.cpu(), MM.t.cpu()
        got_v = VV.t.cpu() if VV else None
        got_bc, got_sc = BC.t.cpu().view(nb, 4), SC.t.cpu().view(nb, width)

        skip_elem = torch.from_numpy(np.asarray(rskip)[elem_range]) | found_inf
        rw, rm = w.double().clone(), m.double().clone()
        rv = v.double().clone() if v is not None else None
        bw, bm = torch.zeros(n_local, dtype=torch.float64), torch.zeros(n_local, dtype=torch.float64)
        bv = torch.zeros(n_local, dtype=torch.float64)
        mres = {mu: None for mu in muts}
        mw = {mu: w.double().clone() for mu in muts}
        for j in range(len(ends)):
            s = torch.from_numpy(elem_range == j)
            gi = rgroup[j]
            h = groups[gi]
            done = int(steps_before[j]) if per_range else int(st0.opt_steps)
            slot = j if per_range else gi
            stepped = not (rskip[j] or found_inf)
            # the prologue's hand-off and scalar state
            if kind == "asgd":
                eta0, mu0 = (float(sc_before[slot, 0]), float(sc_before[slot, 1])) if done else (None, None)
                want = oer.asgd_handoff(h, done, eta0, mu0)
                assert tuple(float(x) for x in got_bc[slot]) == want, (step, j)
                if stepped:   # torch's fp32 eta / mu after the step, bit for bit
                    assert (float(got_sc[slot, 0]), float(got_sc[slot, 1])) == oer.asgd_next(h, done + 1), (step, j)
                elif done:
                    assert torch.equal(got_sc[slot].view(torch.int32), sc_before[slot].view(torch.int32))
            else:
                assert tuple(float(x) for x in got_bc[slot]) == (0.0, 0.0, 1.0 if done == 0 else 0.0, 0.0), (step, j)
            if per_range:
                assert int(rsteps[j]) == done + (1 if stepped else 0)
            if not bool(s.any()) or not stepped:
                continue
            G = g[s].float()
            eta, mu = (eta0, mu0) if kind == "asgd" else (None, None)
            if kind == "rprop":
                nw, nm, nv = oer.rprop_fp32(w[s], m[s], v[s], G, done, h)
                rw[s], rm[s], rv[s] = nw.double(), nm.double(), nv.double()
            else:
                nw, nm, nv, _, _ = oer.torch_step(kind, w[s], m[s], v[s] if v is not None else None, G, done, h, eta, mu)
                e_use, m_use = oer.asgd_used(h, done, eta, mu) if kind == "asgd" else (None, None)
                ew, em, ev = oer.step_bound(kind, w[s], m[s], v[s] if v is not None else None, G.double(),
                                            torch.zeros(int(s.sum()), dtype=torch.float64), h, nw, nm, nv, e_use, m_use)
                rw[s], rm[s], bw[s], bm[s] = nw, nm, ew, em
                if nv is not None:
                    rv[s], bv[s] = nv, ev
            for mu_ in muts:
                mwj, mmj, mvj = oer.step_mutant(kind, w[s], m[s], v[s] if v is not None else None, G, done, h, mu_, eta, mu)
                mw[mu_][s] = mwj.double()
                if kind == "rprop":
                    diff = not (torch.equal(mwj.view(torch.int32), got_w[s].view(torch.int32)) and
                                torch.equal(mmj.view(torch.int32), got_m[s].view(torch.int32)) and
                                torch.equal(mvj.view(torch.int32), got_v[s].view(torch.int32)))
                    if diff:
                        hit.add(mu_)
                elif bool(((got_m[s].double() - mmj).abs() > bm[s]).any()):
                    hit.add(mu_)
        if kind == "rprop":   # bit for bit
            for what, got, ref in (("master", got_w, rw), ("prev", got_m, rm), ("step_size", got_v, rv)):
                st = ~skip_elem
                assert torch.equal(got[st].view(torch.int32), ref[st].float().view(torch.int32)), f"step {step}: {what}"
        else:
            outs = [("master", got_w, rw, bw), ("state 1", got_m, rm, bm)] + ([("state 2", got_v, rv, bv)] if VV else [])
            for what, got, ref, b in outs:
                bad = (got.double() - ref).abs() > b
                assert not bool(bad.any()), f"step {step}: {what} off at {torch.nonzero(bad)[:5].flatten().tolist()}"
            for mu_ in muts:
                if bool(((got_w.double() - mw[mu_]).abs() > bw).any()):
                    hit.add(mu_)
        # ---- where the kernel wrote ----
        MB.check_unchanged_except(snap["M"], ~skip_elem)
        MM.check_unchanged_except(snap["MM"], ~skip_elem)
        if VV:
            VV.check_unchanged_except(snap["VV"], ~skip_elem)
        assert torch.equal(got_w[skip_elem].view(torch.int32), w[skip_elem].view(torch.int32))
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
        if found_inf:   # a skipped step: master, state and scalar state bit-identical
            assert torch.equal(MB.bits(), snap["M"]) and torch.equal(MM.bits(), snap["MM"])
            assert VV is None or torch.equal(VV.bits(), snap["VV"])
            assert torch.equal(SC.bits(), snap["SC"])
        SC.check_guards()
        BC.check_guards()
    assert hit == muts, f"negative controls that passed every step: {muts - hit}"


def test_rprop_seeds_step_size_with_lr_at_first_step(eng):
    """The lr passed at a parameter's first step (a scheduler may have changed it since construction) seeds step_size, the
    step_size buffer is not read then, and later steps keep the stored step_size whatever lr says."""
    L = _L()
    n = 2_048
    h = dict(KIND_BASE["rprop"], lr=0.125)
    MB, MM = Buf(n, F32, torch.zeros(n).cuda()), Buf(n, F32, torch.zeros(n).cuda())
    VV = Buf(n, F32, torch.full((n,), float("nan")).cuda())
    GB = Buf(n, F32)
    SC, BC = Buf(1, F32), Buf(4, F32)
    eng.scaler_set(opt_steps=0, skipped_steps=0, scale=1.0, enabled=0, found_inf=0)
    g = torch.randn(n, generator=torch.Generator().manual_seed(9))
    for step, lr in enumerate((0.125, 0.5)):
        h = dict(h, lr=lr)
        hyp, ext = (L.OptimHyper * 1)(_hyper("rprop", h)), (L.OptimHyperExt * 1)(_ext(h))
        GB.t.copy_(g.cuda())
        eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, ext, 1, 0, None, None, SC.ptr(), BC.ptr(), eng._stream()))
        a = L.OptimArgs()
        a.hyper, a.n_groups, a.hyper_ext, a.group_bc = hyp, 1, ext, BC.ptr()
        a.master, a.exp_avg, a.exp_avg_sq = MB.ptr(), MM.ptr(), VV.ptr()
        a.grad, a.grad_dtype, a.grad_raw, a.grad_mul = GB.ptr(), L.F32, 0, 1.0
        a.n_local = n
        a.lp_ptrs, a.lp_world, a.lp_dtype = None, 0, L.F32
        eng.optim_step_ex(a)
        eng.step_epilogue()
        if step == 0:
            assert torch.equal(VV.t.cpu(), torch.full((n,), 0.125))   # prev = 0: every factor is 1
        else:   # same-sign gradient twice: 0.125 * 1.2, not 0.5 * 1.2
            assert torch.equal(VV.t.cpu(), torch.full((n,), float(torch.tensor(0.125) * torch.tensor(1.2))))


# ---- engine level ------------------------------------------------------------------------------------------------------------
from test_gpu_engine import OddNet, _inject, _oracle_flat, _rel  # noqa: E402

ENGINE_CASES = [
    (torch.optim.Adadelta, {"lr": 0.5}, torch.bfloat16, ("norm", 1.0, 2.0), 1),
    (torch.optim.Adadelta, {"lr": 1.0, "rho": 0.8, "weight_decay": 0.01}, None, ("value", 0.3), 2),
    (torch.optim.Adadelta, {"lr": 0.5, "maximize": True}, None, None, 1),
    (torch.optim.Rprop, {"lr": 1e-3}, torch.bfloat16, ("norm", 1.0, 2.0), 1),
    (torch.optim.Rprop, {"lr": 2e-3, "etas": (0.4, 1.3), "step_sizes": (1e-5, 1e-2)}, None, ("value", 0.3), 1),
    (torch.optim.Rprop, {"lr": 1e-3, "maximize": True}, None, None, 2),
    (torch.optim.ASGD, {"lr": 1e-2}, torch.bfloat16, ("norm", 1.0, 2.0), 1),
    (torch.optim.ASGD, {"lr": 1e-2, "t0": 3.0, "lambd": 1e-2, "weight_decay": 0.01}, None, ("value", 0.3), 2),
    (torch.optim.ASGD, {"lr": 1e-2, "t0": 2.0, "maximize": True}, None, None, 1),
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


def _check_state(sd, oracle):
    for i, p in enumerate(oracle.params):
        st = oracle.optimizer.state.get(p, {})
        if not st:
            assert i not in sd["state"], i   # never stepped: no entry, as torch
            continue
        got = sd["state"][i]
        assert set(got) == set(st), (set(got), set(st))
        for k, want in st.items():
            if k == "step":
                assert float(got[k]) == float(want) and got[k].dtype == torch.float32 and got[k].dim() == 0
            elif k in ("eta", "mu"):   # ASGD: fp32 0-dim, bit-identical to torch's
                assert got[k].dtype == torch.float32 and got[k].dim() == 0 and float(got[k]) == float(want), (k, got[k], want)
            else:
                assert _rel(got[k].cpu(), want) < TOL, k


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
    oracle = OracleEngine(init, 1, cls, dict(kw, foreach=False), grad_accum=accum, clip=clip)
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


@pytest.mark.parametrize("cls,kw", [(torch.optim.Adadelta, {"lr": 0.5, "weight_decay": 0.1}),
                                    (torch.optim.Rprop, {"lr": 1e-3}),
                                    (torch.optim.ASGD, {"lr": 1e-2, "t0": 3.0, "weight_decay": 0.1})])
@pytest.mark.parametrize("clip", [None, ("norm", 1.0, 2.0), ("value", 0.2)])
def test_unused_parameter_and_stoke_facade(cls, kw, clip):
    """Through Stoke: the class builds a B200FusedOptimizer and the loss falls.  Head b receives no gradient on the first
    two steps and on some later ones, so step counts (and ASGD's eta / mu) go per parameter, as torch keeps them; a
    parameter not yet stepped has no state entry; every parameter and state tensor follows the oracle."""
    from engine_oracle import OracleEngine
    import stoke_b200 as sb
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec
    from stoke_b200.optim import B200FusedOptimizer

    torch.cuda.set_device(0)
    model = TwoHeads()
    init = [p.detach().clone() for p in model.parameters()]
    s = sb.Stoke(model=model, optimizer=sb.StokeOptimizer(optimizer=cls, optimizer_kwargs=kw), loss=torch.nn.MSELoss(),
                 batch_size_per_device=8, gpu=True, verbose=False)
    assert isinstance(s.optimizer, B200FusedOptimizer)
    path = s.optimizer.path
    if clip is not None:
        path.clip = ClipSpec(_lib.CLIP_NORM, max_norm=clip[1], norm_type=clip[2]) if clip[0] == "norm" else \
            ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1])
    oracle = OracleEngine(init, 1, cls, dict(kw, foreach=False), clip=clip)
    g = torch.Generator().manual_seed(0)
    x, y = torch.randn(8, 16, generator=g).cuda(), torch.randn(8, 1, generator=g).cuda()
    losses = []
    for step in range(12):
        model.use_b = step >= 2 and step % 4 != 1
        loss = s.loss(s.model(x), y)
        losses.append(float(loss.detach()))
        path.begin_backward(sync=True, unscale=False)
        loss.backward()
        grads = [gv.detach().float().cpu().clone() if path._touched[i] else None for i, gv in enumerate(path.grad_views)]
        oracle.micro_step([grads])
        s._grad_accum_counter += 1
        path.after_backward(sync=True, unscale=False)
        s._backward_steps += 1
        s.step()
        oracle.step()
        if step == 1:   # head b never stepped yet: no state entry
            sd = s.optimizer.state_dict()
            assert 4 not in sd["state"] and 5 not in sd["state"] and 0 in sd["state"]
    for a, b in zip(model.parameters(), oracle.weights()):
        assert _rel(a.detach().float().cpu().reshape(-1), b.reshape(-1)) < TOL
    sd = s.optimizer.state_dict()
    _check_state(sd, oracle)
    assert [float(sd["state"][j]["step"]) for j in range(6)] == [12.0] * 4 + [8.0, 8.0]
    assert losses[-1] < losses[2]   # both with head b in use
    s.optimizer.close()


@pytest.mark.parametrize("cls,kw", [(torch.optim.Adadelta, {"lr": 0.5, "weight_decay": 0.01}),
                                    (torch.optim.Rprop, {"lr": 1e-3, "etas": (0.4, 1.3)}),
                                    (torch.optim.ASGD, {"lr": 1e-2, "t0": 5.0, "lambd": 1e-2})])
def test_checkpoint_round_trip_with_plain_torch(cls, kw):
    """Engine -> torch: the engine's state_dict loaded into the plain CPU class continues to the same weights as the engine.
    torch -> engine: a plain torch state dict (no b200_* keys; the model weights loaded first) continues the same way."""
    torch.cuda.set_device(0)
    net = OddNet().cuda()
    opt = _fused(net, cls, kw, None)
    path = opt.path
    for step in range(4):
        _inject(path, step, 0, torch.float32)
        path.after_backward(sync=True, unscale=False)
        opt.step()
    sd = opt.state_dict()
    cpu_params = [torch.nn.Parameter(w.cpu().clone()) for w in path.unflatten(path.gather_master())]
    topt = cls(cpu_params, **kw, foreach=False)
    topt.load_state_dict({k: v for k, v in sd.items() if not k.startswith("b200_")})
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
        if cls is torch.optim.ASGD:
            assert float(sd2["state"][i]["eta"]) == float(topt.state[p]["eta"])
            assert float(sd2["state"][i]["mu"]) == float(topt.state[p]["mu"])
    opt.close()
    opt2.close()


def _continue_torch_checkpoint_with_unstepped_parameter(cls, kw):
    """A torch-written state where one parameter was never stepped (no entry) and the others took different numbers of
    steps: the fused optimizer goes per parameter, restarts the unstepped one at step 0 like torch, and continues exactly
    like torch, scalar state (ASGD's eta / mu, NAdam's mu_product) included."""
    torch.cuda.set_device(0)
    net = OddNet().cuda()
    cpu_params = [torch.nn.Parameter(p.detach().cpu().clone()) for p in net.parameters()]
    topt = cls(cpu_params, **kw, foreach=False)
    gen = torch.Generator().manual_seed(4)
    for step in range(5):
        for i, p in enumerate(cpu_params):
            p.grad = None if (i == 0 or (i == 1 and step < 3)) else torch.randn(p.shape, generator=gen) * 1e-2
        topt.step()
    assert cpu_params[0] not in topt.state
    with torch.no_grad():
        for p, q in zip(net.parameters(), cpu_params):
            p.copy_(q.detach())
    opt = _fused(net, cls, kw, None)
    opt.load_state_dict(topt.state_dict())
    assert opt.path._range_steps is not None
    for step in range(5, 9):
        grads = _inject(opt.path, step, 0, torch.float32)
        for p, gr in zip(cpu_params, grads):
            p.grad = gr.reshape(p.shape).clone()
        opt.path.after_backward(sync=True, unscale=False)
        opt.step()
        topt.step()
    for a, b in zip(opt.path.unflatten(opt.path.gather_master().cpu()), cpu_params):
        assert _rel(a.reshape(-1), b.detach().reshape(-1)) < TOL
    sd = opt.state_dict()
    for i, p in enumerate(cpu_params):
        assert float(sd["state"][i]["step"]) == float(topt.state[p]["step"])
        for k in ("eta", "mu", "mu_product"):
            if k in topt.state[p]:
                assert float(sd["state"][i][k]) == float(topt.state[p][k]), k
    opt.close()


def test_torch_checkpoint_with_unstepped_parameter_and_differing_asgd_scalars():
    """ASGD: the stepped parameters' eta / mu differ, and the unstepped one starts from torch's lazy initialisation."""
    _continue_torch_checkpoint_with_unstepped_parameter(torch.optim.ASGD, {"lr": 1e-2, "t0": 2.0, "lambd": 1e-2})


@pytest.mark.parametrize("cls", [torch.optim.Adam, torch.optim.NAdam])
def test_torch_checkpoint_with_unstepped_parameter_restarts_it_at_step_0(cls):
    """Adam and NAdam: the unstepped parameter's first bias correction (NAdam: with mu_product 1) is torch's step 1."""
    _continue_torch_checkpoint_with_unstepped_parameter(cls, {"lr": 1e-2})


def test_uniform_torch_checkpoint_replaces_per_parameter_counts():
    """Adam with per-parameter step counts already on (head b unused at the first step) loads a torch state whose counts
    are uniform: the loaded counts replace the old ones, and the step continues exactly like torch."""
    torch.cuda.set_device(0)
    kw = {"lr": 1e-2}
    model = TwoHeads().cuda()
    opt = _fused(model, torch.optim.Adam, kw, None)
    path = opt.path
    g = torch.Generator().manual_seed(0)
    x, y = torch.randn(8, 16, generator=g).cuda(), torch.randn(8, 1, generator=g).cuda()
    for step in range(3):
        model.use_b = step > 0
        path.begin_backward(sync=True, unscale=False)
        torch.nn.functional.mse_loss(model(x), y).backward()
        path.after_backward(sync=True, unscale=False)
        opt.step()
    assert path.param_steps() == [3, 3, 3, 3, 2, 2]
    cpu_params = [torch.nn.Parameter(p.detach().cpu().clone()) for p in model.parameters()]
    topt = torch.optim.Adam(cpu_params, **kw, foreach=False)
    for step in range(2):
        for p in cpu_params:
            p.grad = torch.randn(p.shape, generator=g) * 1e-2
        topt.step()
    with torch.no_grad():
        for p, q in zip(model.parameters(), cpu_params):
            p.copy_(q.detach())
    opt.load_state_dict(topt.state_dict())
    assert path.param_steps() == [2] * 6
    for step in range(4):
        grads = _inject(path, step, 0, torch.float32)
        for p, gr in zip(cpu_params, grads):
            p.grad = gr.reshape(p.shape).clone()
        path.after_backward(sync=True, unscale=False)
        opt.step()
        topt.step()
    for a, b in zip(path.unflatten(path.gather_master().cpu()), cpu_params):
        assert _rel(a.reshape(-1), b.detach().reshape(-1)) < TOL
    sd = opt.state_dict()
    assert [float(sd["state"][i]["step"]) for i in range(6)] == [6.0] * 6
    opt.close()


def test_torch_sgd_momentum_checkpoint_continues_the_buffer():
    """A torch-written SGD-momentum state (no `step`; parameter 0 never stepped, so it has no buffer): the loaded buffers
    continue as buf = momentum * buf + (1 - dampening) * g, parameter 0 starts with buf = g, as in torch."""
    torch.cuda.set_device(0)
    kw = {"lr": 1e-2, "momentum": 0.9, "dampening": 0.25}
    net = OddNet().cuda()
    cpu_params = [torch.nn.Parameter(p.detach().cpu().clone()) for p in net.parameters()]
    topt = torch.optim.SGD(cpu_params, **kw, foreach=False)
    gen = torch.Generator().manual_seed(6)
    for step in range(3):
        for i, p in enumerate(cpu_params):
            p.grad = None if i == 0 else torch.randn(p.shape, generator=gen) * 1e-2
        topt.step()
    with torch.no_grad():
        for p, q in zip(net.parameters(), cpu_params):
            p.copy_(q.detach())
    opt = _fused(net, torch.optim.SGD, kw, None)
    opt.load_state_dict(topt.state_dict())
    for step in range(3, 7):
        grads = _inject(opt.path, step, 0, torch.float32)
        for p, gr in zip(cpu_params, grads):
            p.grad = gr.reshape(p.shape).clone()
        opt.path.after_backward(sync=True, unscale=False)
        opt.step()
        topt.step()
    for a, b in zip(opt.path.unflatten(opt.path.gather_master().cpu()), cpu_params):
        assert _rel(a.reshape(-1), b.detach().reshape(-1)) < TOL
    sd = opt.state_dict()
    for i, p in enumerate(cpu_params):
        assert _rel(sd["state"][i]["momentum_buffer"].cpu().reshape(-1), topt.state[p]["momentum_buffer"].reshape(-1)) < TOL
    opt.close()


def test_asgd_step_makes_no_host_sync():
    """torch's single-tensor ASGD calls .item() three times per parameter; the fused step keeps eta and mu on the device."""
    net = OddNet().cuda()
    opt = _fused(net, torch.optim.ASGD, {"lr": 1e-2, "t0": 1.0}, torch.bfloat16, ("norm", 0.5, 2.0))
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
def test_sharded_matches_unsharded_w2(tmp_path):
    """fairscale_oss at W = 2: Adadelta, Rprop and ASGD sharded (ZeRO-1, in-kernel parameter all-gather) against the same
    classes replicated (all-reduce route): final weights and the gathered state_dict bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "optim_elementwise_w2.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29563", os.path.join(ROOT, "tests", "optim_elementwise_mgpu_worker.py"), str(out)]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=420,
                          env=dict(os.environ, STK_SPIN_TIMEOUT_S="30"))
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    import json

    res = json.loads(out.read_text())
    assert set(res) == {"adadelta", "rprop", "asgd"}
    for name, r in res.items():
        assert r["sharded_route"] == "sharded" and r["replicated_route"] == "allreduce", (name, r)
        assert r["weights_identical"] and r["state_identical"], (name, r)
