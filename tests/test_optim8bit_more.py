# -*- coding: utf-8 -*-
"""CPU: stoke_b200.Lion8bit and AdEMAMix8bit (block-wise 8-bit state on the quantizer of AdamW8bit) against an
independent numpy transcription of their updates (fp32 element ops, python-double scalars, codes by a full scan of the
map), plus argument validation, the state layout, step-count loading, checkpoints through the fused step's state
description, the load checks, routing, the ABI and AdEMAMix8bit's scalars against AdEMAMix's."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

import stoke_b200 as sb
from stoke_b200 import _lib
from stoke_b200.optim import (_GROUP_HYPER, _KINDS, _STATE_LAYOUT, AdEMAMix, AdEMAMix8bit, Lion8bit, ademamix8bit_scalars,
                              ademamix_schedule, check_8bit_entries, create_dynamic_map, export_state, fused_supported,
                              import_state, load_step_counts, state_buffers, state_dict_index)
from test_optim8bit import mem, np_deq, np_quant

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32

MIN = 128
SHAPES = [(127,), (128,), (129,), (300,), (16, 4, 3, 3), (40, 20), (7,), (3, 100)]
CHANNELS_LAST = 4
NO_GRAD = 6
Q1, Q2 = create_dynamic_map(True).numpy(), create_dynamic_map(False).numpy()


# ---- the numpy transcriptions ---------------------------------------------------------------------------------------------
def np_sign(c):
    return np.where(c > 0, f32(1), np.where(c < 0, f32(-1), f32(0))).astype(f32)   # NaN -> 0


def np_lion(w, g, st, hp, quant):
    b1, b2 = hp["betas"]
    lr, wd = hp["lr"], hp["weight_decay"]
    st["step"] += 1
    m = np_deq(st["state1"], Q1, st["absmax1"]) if quant else st["state1"]
    with np.errstate(invalid="ignore", over="ignore"):
        if wd != 0:
            w = (w * f32(1 - lr * wd)).astype(f32)
        c = ((m * f32(b1)).astype(f32) + (g * f32(1 - b1)).astype(f32)).astype(f32)
        w = (w - np_sign(c) * f32(lr)).astype(f32)
        m = ((m * f32(b2)).astype(f32) + (g * f32(1 - b2)).astype(f32)).astype(f32)
    if quant:
        st["state1"], st["absmax1"] = np_quant(m, Q1)
    else:
        st["state1"] = m
    return w


def np_schedule(hp, t):
    """alpha_t and beta3_t after apple/ml-ademamix's schedulers (linear alpha; beta3 linear in half-life)."""
    b1, _, b3 = hp["betas"]
    aw, bw = hp["alpha_warmup"], hp["beta3_warmup"]
    alpha_t = min(t * hp["alpha"] / aw, hp["alpha"]) if aw else hp["alpha"]
    if bw and t < bw:
        half = [math.log(0.5) / math.log(b + 1e-8) - 1 for b in (b1, b3)]
        beta3_t = 0.5 ** (1 / ((1 - t / bw) * half[0] + (t / bw) * half[1] + 1))
    else:
        beta3_t = b3
    return alpha_t, beta3_t


def np_ademamix(w, g, st, hp, quant):
    b1, b2, _ = hp["betas"]
    lr, eps, wd = hp["lr"], hp["eps"], hp["weight_decay"]
    st["step"] += 1
    t = float(st["step"])
    c1, c2 = 1 / (1 - b1 ** t), 1 / math.sqrt(1 - b2 ** t)
    alpha_t, beta3_t = np_schedule(hp, t)
    if quant:
        m1 = np_deq(st["state1"][0], Q1, st["absmax1"][0])
        m2 = np_deq(st["state1"][1], Q1, st["absmax1"][1])
        nu = np_deq(st["state2"], Q2, st["absmax2"])
    else:
        m1, m2, nu = st["state1"][0], st["state1"][1], st["state2"]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        m1 = ((m1 * f32(b1)).astype(f32) + (g * f32(1 - b1)).astype(f32)).astype(f32)
        m2 = ((m2 * f32(beta3_t)).astype(f32) + (g * f32(1 - beta3_t)).astype(f32)).astype(f32)
        nu = ((nu * f32(b2)).astype(f32) + ((g * g).astype(f32) * f32(1 - b2)).astype(f32)).astype(f32)
        den = ((np.sqrt(nu) * f32(c2)).astype(f32) + f32(eps)).astype(f32)
        u = (((m1 * f32(c1)).astype(f32) + (m2 * f32(alpha_t)).astype(f32)).astype(f32) / den).astype(f32)
        if wd != 0:
            u = (u + (w * f32(wd)).astype(f32)).astype(f32)
        w = (w - (u * f32(lr)).astype(f32)).astype(f32)
    if quant:
        (c_1, a_1), (c_2, a_2) = np_quant(m1, Q1), np_quant(m2, Q1)
        st["state1"], st["absmax1"] = np.stack([c_1, c_2]), np.stack([a_1, a_2])
        st["state2"], st["absmax2"] = np_quant(nu, Q2)
    else:
        st["state1"], st["state2"] = np.stack([m1, m2]), nu
    return w


# ---- the runs ---------------------------------------------------------------------------------------------------------------
def _params():
    g = torch.Generator().manual_seed(0)
    out = []
    for i, s in enumerate(SHAPES):
        p = torch.randn(*s, generator=g)
        if i == CHANNELS_LAST:
            p = p.to(memory_format=torch.channels_last)
        out.append(torch.nn.Parameter(p))
    return out


LION_GROUPS = [(slice(0, 4), dict(lr=1e-2, weight_decay=0.1)), (slice(4, 6), dict(betas=(0.8, 0.95))),
               (slice(6, 8), dict(lr=3e-3))]
ADEMAMIX_GROUPS = [(slice(0, 4), dict(lr=1e-2, weight_decay=0.1, alpha_warmup=4, beta3_warmup=3)),
                   (slice(4, 6), dict(betas=(0.8, 0.95, 0.99), alpha=5.0, eps=1e-6)),
                   (slice(6, 8), dict(lr=3e-3, beta3_warmup=9))]
CASES = {"lion8bit": (Lion8bit, LION_GROUPS, np_lion), "ademamix8bit": (AdEMAMix8bit, ADEMAMIX_GROUPS, np_ademamix)}


def _ref_state(p, name, quant):
    n, nb = p.numel(), -(-p.numel() // 256)
    two = name == "ademamix8bit"
    if quant:
        st = dict(state1=np.zeros((2, n) if two else n, np.uint8), absmax1=np.zeros((2, nb) if two else nb, f32))
        if two:
            st.update(state2=np.zeros(n, np.uint8), absmax2=np.zeros(nb, f32))
    else:
        st = dict(state1=np.zeros((2, n) if two else n, f32))
        if two:
            st["state2"] = np.zeros(n, f32)
    return dict(st, step=0)


def _run(name, steps, n_groups=3, nonfinite_at=None):
    cls, groups, np_step = CASES[name]
    params = _params()
    groups = groups[:n_groups - 1] + [(slice(groups[n_groups - 1][0].start, len(params)), groups[n_groups - 1][1])]
    opt = cls([dict(extra, params=params[sl]) for sl, extra in groups], min_8bit_size=MIN)
    group_of = [gi for gi, (sl, _) in enumerate(groups) for _ in params[sl]]
    ref_w, ref_st = [mem(p) for p in params], [None] * len(params)
    gen = torch.Generator().manual_seed(1)
    for k in range(steps):
        for i, p in enumerate(params):
            g = torch.randn(p.shape, generator=gen).to(memory_format=torch.channels_last if i == CHANNELS_LAST else
                                                       torch.contiguous_format)
            if nonfinite_at == k and i == 3:
                g.view(-1)[5] = float("nan")
                g.view(-1)[260] = float("inf")
            p.grad = None if i == NO_GRAD else g
        opt.step()
        for i, p in enumerate(params):
            if i == NO_GRAD:
                continue
            if ref_st[i] is None:
                ref_st[i] = _ref_state(p, name, p.numel() >= MIN)
            ref_w[i] = np_step(ref_w[i], mem(p.grad), ref_st[i], opt.param_groups[group_of[i]], p.numel() >= MIN)
    return params, opt, ref_w, ref_st


def _mem_state(t, stacked):
    return np.stack([mem(t[0]), mem(t[1])]) if stacked else mem(t)


def _assert_matches(name, params, opt, ref_w, ref_st):
    for i, p in enumerate(params):
        if i == NO_GRAD:
            assert not opt.state.get(p)
            continue
        st = opt.state[p]
        np.testing.assert_array_equal(mem(p), ref_w[i], err_msg=f"weights {i}")
        assert float(st["step"]) == ref_st[i]["step"]
        quant = p.numel() >= MIN
        for key in ("state1", "state2", "absmax1", "absmax2"):
            if key not in ref_st[i]:
                assert key not in st, (key, i)
                continue
            stacked = name == "ademamix8bit" and key.endswith("1")
            got = _mem_state(st[key], stacked) if key.startswith("state") else st[key].numpy()
            np.testing.assert_array_equal(got, ref_st[i][key], err_msg=f"{key} {i}")
            if key.startswith("state"):
                assert st[key].dtype == (torch.uint8 if quant else torch.float32)
                assert st[key].shape == ((2,) if stacked else ()) + p.shape
        assert ("qmap1" in st) == quant


@pytest.mark.parametrize("n_groups", [1, 2, 3])
@pytest.mark.parametrize("name", sorted(CASES))
def test_class_against_numpy_transcription(name, n_groups):
    params, opt, ref_w, ref_st = _run(name, 6, n_groups)
    _assert_matches(name, params, opt, ref_w, ref_st)
    want = ["step", "state1", "qmap1", "absmax1"] if name == "lion8bit" else \
        ["step", "state1", "qmap1", "state2", "qmap2", "absmax1", "absmax2"]
    assert list(opt.state[params[1]]) == want


@pytest.mark.parametrize("name", sorted(CASES))
def test_nonfinite_gradient(name):
    params, opt, ref_w, ref_st = _run(name, 3, nonfinite_at=1)
    _assert_matches(name, params, opt, ref_w, ref_st)


def test_ademamix8bit_scalars_are_ademamix_s():
    """At every step through both warm-ups (and after), the four scalars AdEMAMix8bit uses are the numbers AdEMAMix.step
    forms, and the transcription's."""
    for extra in (dict(alpha_warmup=5, beta3_warmup=7), dict(beta3_warmup=3), dict(betas=(0.5, 0.9, 0.999))):
        g = AdEMAMix8bit([torch.nn.Parameter(torch.zeros(1))], **extra).param_groups[0]
        b1, b2, _ = g["betas"]
        for t in range(1, 10):
            t = float(t)
            want = (1 / (1 - b1 ** t), 1 / math.sqrt(1 - b2 ** t)) + ademamix_schedule(g, t)
            assert ademamix8bit_scalars(g, t) == want
            assert ademamix8bit_scalars(g, t)[2:] == np_schedule(g, t)
    assert AdEMAMix([torch.nn.Parameter(torch.zeros(1))]).defaults.keys() <= AdEMAMix8bit(
        [torch.nn.Parameter(torch.zeros(1))]).defaults.keys()


@pytest.mark.parametrize("kw, name", [(dict(args=object()), "args"), (dict(percentile_clipping=5), "percentile_clipping"),
                                      (dict(block_wise=False), "block_wise"), (dict(is_paged=True), "is_paged")])
def test_lion8bit_refused_options(kw, name):
    with pytest.raises(ValueError, match=name):
        Lion8bit([torch.nn.Parameter(torch.zeros(4))], **kw)


def test_validation():
    p = [torch.nn.Parameter(torch.zeros(4))]
    for kw in (dict(lr=-1.0), dict(betas=(1.0, 0.9)), dict(weight_decay=-0.1)):
        with pytest.raises(ValueError):
            Lion8bit(p, **kw)
    for kw in (dict(lr=-1.0), dict(betas=(0.9, 0.99)), dict(betas=(0.9, 1.0, 0.9)), dict(eps=-1.0), dict(alpha=-1.0),
               dict(weight_decay=-1.0), dict(alpha_warmup=0), dict(beta3_warmup=2.5)):
        with pytest.raises(ValueError):
            AdEMAMix8bit(p, **kw)
    with pytest.raises(ValueError, match="betas"):
        AdEMAMix8bit(p, betas=(0.0, 0.9, 0.99))
    assert Lion8bit(p).defaults == dict(lr=1e-4, betas=(0.9, 0.99), weight_decay=0.0, min_8bit_size=4096)
    d = AdEMAMix8bit(p).defaults
    assert d == dict(lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=2.0, beta3_warmup=None, alpha_warmup=None, eps=1e-8,
                     weight_decay=0, min_8bit_size=4096)


def _views_of(name, params):
    """The fused step's views for these parameters, laid out like GradPath's (AdEMAMix's stacked state1 / absmax1
    strided over two halves of one buffer)."""
    lay = _STATE_LAYOUT[name]
    out = {t.key: [] for t in lay.tensors}
    three = name == "ademamix8bit"
    for p in params:
        quant = p.numel() >= MIN
        nb = -(-p.numel() // 256)
        dt = torch.uint8 if quant else torch.float32
        if three:
            buf = torch.zeros(2 * (p.numel() + 64), dtype=dt)
            d = dict(state1=buf.as_strided((2, *p.shape), (p.numel() + 64, *p.stride()), 16),
                     state2=torch.zeros_like(p, dtype=dt))
            if quant:
                d.update(absmax1=torch.zeros(2 * nb + 8).as_strided((2, nb), (nb + 4, 1), 2), absmax2=torch.zeros(nb),
                         qmap1=torch.from_numpy(Q1.copy()), qmap2=torch.from_numpy(Q2.copy()))
        else:
            d = dict(state1=torch.zeros_like(p, dtype=dt))
            if quant:
                d.update(absmax1=torch.zeros(nb), qmap1=torch.from_numpy(Q1.copy()))
        for k in out:
            out[k].append(d.get(k))
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_checkpoint_through_the_state_layout(name):
    """A class checkpoint imported into the fused step's views and exported again is the same checkpoint; loaded into a
    fresh class (python-int step) it continues bit for bit."""
    lay = _STATE_LAYOUT[name]
    assert state_buffers(lay, [{}]) == {"M": None, "V": None, "M2": None}
    assert all(t.buf == "q8" for t in lay.tensors) and lay.step and lay.unstepped == "omit"
    params, opt, _, _ = _run(name, 3)
    sd = opt.state_dict()
    group_of = [0] * 4 + [1] * 2 + [2] * 2
    sd_index = state_dict_index(group_of, 3)
    entries = [sd["state"].get(sd_index[i], {}) for i in range(len(params))]
    views = _views_of(name, params)
    import_state(lay, entries, views)
    steps = [0 if i == NO_GRAD else 3 for i in range(len(params))]
    state = export_state(lay, sd["param_groups"], group_of, sd_index, steps, None, views)
    assert set(state) == {sd_index[i] for i in range(len(params)) if i != NO_GRAD}
    for i in range(len(params)):
        if i != NO_GRAD:
            want, got = sd["state"][sd_index[i]], state[sd_index[i]]
            assert list(got) == list(want)
            for k in want:
                assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), (i, k)
    assert load_step_counts(name, entries, group_of, None, True) == (3, steps, None)
    # the exported (non-dense) state and an int step load into a fresh class, which continues like the original
    cls, groups, _ = CASES[name]
    fresh_params = [torch.nn.Parameter(p.detach().clone()) for p in params]
    fresh = cls([dict(extra, params=fresh_params[sl]) for sl, extra in groups], min_8bit_size=MIN)
    fresh.load_state_dict({"state": {k: dict(v, step=int(v["step"])) for k, v in state.items()},
                           "param_groups": sd["param_groups"]})
    for st, p in ((fresh.state[q], q) for q in fresh_params if q in fresh.state):
        assert torch.is_tensor(st["step"]) and st["step"].dtype == torch.float32 and float(st["step"]) == 3
        assert st["state1"].dtype == (torch.uint8 if p.numel() >= MIN else torch.float32)
        if st["state1"].dim() > p.dim():   # each stacked tensor laid out like the parameter again
            assert st["state1"][1].stride() == p.stride()
    gen = torch.Generator().manual_seed(9)
    for a, b in zip(params, fresh_params):
        if a.grad is not None:
            a.grad = b.grad = torch.randn(a.shape, generator=gen).to(memory_format=torch.preserve_format)
    opt.step()
    fresh.step()
    for a, b in zip(params, fresh_params):
        assert torch.equal(a.detach(), b.detach())


@pytest.mark.parametrize("name", sorted(CASES))
def test_load_checks(name):
    params, opt, _, _ = _run(name, 2)
    sd = opt.state_dict()
    keys = [t.key for t in _STATE_LAYOUT[name].tensors]
    states, maps = tuple(k for k in keys if k.startswith("state")), tuple(k for k in keys if k.startswith("qmap"))
    entries = [sd["state"].get(i, {}) for i in range(len(params))]
    quantized = [p.numel() >= MIN for p in params]
    assert len(check_8bit_entries(entries, quantized, states, maps, "X")) == len(maps)
    with pytest.raises(ValueError, match="state1"):   # fp32 state where 8-bit state belongs
        check_8bit_entries(entries, [True] * len(params), states, maps, "X")
    bad = [dict(e) for e in entries]
    bad[1]["qmap1"] = bad[1]["qmap1"].flip(0)
    with pytest.raises(ValueError, match="ascending"):
        check_8bit_entries(bad, quantized, states, maps, "X")
    bad = [dict(e) for e in entries]
    bad[1][maps[-1]] = bad[1][maps[-1]] * 0.5
    with pytest.raises(ValueError, match="differ"):
        check_8bit_entries(bad, quantized, states, maps, "X")
    bad = [dict(e) for e in entries]
    bad[1]["state1"] = bad[1]["state1"].float()
    cls = CASES[name][0]
    with pytest.raises(ValueError, match=f"{cls.__name__}: state1"):
        cls(_params(), min_8bit_size=MIN).load_state_dict(
            {"state": dict(enumerate(bad)), "param_groups": [dict(sd["param_groups"][0], params=list(range(8)))]})


def _model(n_groups):
    return torch.nn.Sequential(*[torch.nn.Linear(4, 4) for _ in range(n_groups)])


@pytest.mark.parametrize("cls", [Lion8bit, AdEMAMix8bit])
def test_routing_and_hypers(cls):
    for n, fused in ((8, True), (9, False)):
        m = _model(n)
        kw = dict(params=[dict(params=list(layer.parameters())) for layer in m], lr=1e-3)
        assert fused_supported(cls, kw, m) is fused
    assert getattr(sb, cls.__name__) is cls and cls.__name__ in sb.__all__
    kind = _KINDS[cls]
    g = cls([torch.nn.Parameter(torch.zeros(1))], lr=0.25, betas=(0.5, 0.75, 0.875)[:2 if cls is Lion8bit else 3],
            weight_decay=0.125).param_groups[0]
    h = _GROUP_HYPER[kind](g)
    if cls is AdEMAMix8bit:
        h, x = h
        assert (x.alpha, x.beta3, x.alpha_warmup, x.beta3_warmup) == (2.0, 0.875, 0, 0)
    assert (h.lr, h.beta1, h.beta2, h.weight_decay, h.eps) == (0.25, 0.5, 0.75, 0.125, 0.0 if cls is Lion8bit else 1e-8)


def test_abi():
    """The two entry points are declared beside stk_adam8bit_step and take its argument struct; AdEMAMix's also
    stk_ademamix_hyper_t (whose ctypes layout test_ademamix.py pins against the header) and two device pointers."""
    with open(os.path.join(ROOT, "include", "stoke_b200.h")) as f:
        header = re.sub(r"\s+", " ", f.read())
    assert "int stk_lion8bit_step(stk_ctx* ctx, const stk_adam8bit_args_t* args, void* stream);" in header
    assert ("int stk_ademamix8bit_step(stk_ctx* ctx, const stk_adam8bit_args_t* args, const stk_ademamix_hyper_t* "
            "ademamix, uint8_t* code3, float* absmax3, void* stream);") in header
    sig = _lib._SIGNATURES
    assert sig["stk_lion8bit_step"] == sig["stk_adam8bit_step"]
    assert sig["stk_ademamix8bit_step"][1][:2] == sig["stk_adam8bit_step"][1][:2]
    assert sig["stk_ademamix8bit_step"][1][2] is C.POINTER(_lib.AdemamixHyper) and len(sig["stk_ademamix8bit_step"][1]) == 6
    assert C.sizeof(_lib.AdemamixHyper) == 32 and C.sizeof(_lib.Adam8bitHyper) == 40
