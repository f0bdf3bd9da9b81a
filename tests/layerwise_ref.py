# -*- coding: utf-8 -*-
"""TEST INFRASTRUCTURE ONLY -- float64 reference of the fused LAMB / LARS steps, with per-element fp32 error bounds in
the conventions of oracle/kernel_ref.py (U, SLACK; every fp32 operation and every cast of a float64 scalar to fp32
contributes one u of its result, input errors are propagated to first order).

The values come from the classes' own ``step()`` (stoke_b200.optim.LAMB / LARS) on float64 tensors with the kernel's
pre-step state loaded.  Norms are sums of non-negative terms, so the relative error of any summation order of n terms is
at most (depth + 1) u, depth being the longest addition chain; every bound takes the larger of the kernel's depth (its
launch shapes: k2_layerwise.cu) and a depth that covers torch's fp32 CPU order (n / 16 + 16), so it holds for both."""
import math
from typing import Dict

import torch

from kernel_ref import SLACK, U

F64 = torch.float64
TILE = 8192   # k2_layerwise.cu: STK_LW_TILE

LAMB_DEFAULTS = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01, bias_correction=True, always_adapt=False)
LARS_DEFAULTS = dict(lr=1.0, momentum=0.9, dampening=0.0, weight_decay=0.0, nesterov=False, trust_coefficient=0.001,
                     eps=1e-8, always_adapt=False)


def hyper(kind: str, h: Dict) -> Dict:
    return dict(LAMB_DEFAULTS if kind == "lamb" else LARS_DEFAULTS, **h)


def make_optimizer(kind: str, params, h: Dict):
    from stoke_b200.optim import LAMB, LARS

    return (LAMB if kind == "lamb" else LARS)(params, **hyper(kind, h))


def state_keys(kind: str, h: Dict) -> tuple:
    if kind == "lamb":
        return ("exp_avg", "exp_avg_sq")
    return ("momentum_buffer",) if hyper(kind, h)["momentum"] != 0 else ()


def zero_state(kind: str, shape, h: Dict) -> Dict:
    """The state before a parameter's first step: LAMB's moments are zero; LARS has no buffer yet."""
    return {"exp_avg": torch.zeros(shape), "exp_avg_sq": torch.zeros(shape)} if kind == "lamb" else {}


def step_ref(kind: str, w, state: Dict, g, step: int, h: Dict, dtype=F64):
    """One step of the class in `dtype` (float64: the reference; float32: the class's own fp32 result) from the given
    state; `step` = steps already taken.  Returns (w, new state dict)."""
    p = torch.nn.Parameter(w.to(dtype).clone())
    opt = make_optimizer(kind, [p], h)
    if step > 0:
        st = {"step": torch.tensor(float(step))}
        st.update({k: v.to(dtype).clone() for k, v in state.items()})
        opt.state[p] = st
    p.grad = g.to(dtype).clone()
    opt.step()
    return p.detach(), {k: opt.state[p][k] for k in state_keys(kind, h)}


def depth_full(n: int) -> int:
    """||w||^2, ||r||^2, ||g||^2: kernel = 32 per thread + 8 (block tree) + ceil(tiles / 32) + 5 (warp fold); torch
    n / 16 + 16"""
    tiles = -(-n // TILE)
    return max(32 + 8 + -(-tiles // 32) + 5, -(-n // 16) + 16)


def _norm_rel(n: int) -> float:
    return (depth_full(n) + 1) * U / 2 + U   # the sum, then the square root


def _trust(a: float, b: float, value: float) -> float:
    return value if (a > 0 and b > 0) else 1.0


def step_bound(kind: str, w, state: Dict, G, step: int, h: Dict, ref_w, ref_state: Dict):
    """Per-element bounds of an fp32 step: (e_w, {key: e_state}).  w, state: the pre-step fp32 values (exact); G: the
    gradient the kernel sees (exact); ref_w / ref_state: the float64 reference's results.

    LAMB:  m' = lerp(m, G, 1 - b1):                 e_m = 3u (|m| + |G|)
           v' = v b2 + (1 - b2) G^2:                e_v = 6u v'                                   (non-negative terms)
           mh = m' / bc1, vh = v' / bc2:            e_mh = e_m / bc1 + 2u |mh|,  e_vh = e_v / bc2 + 2u vh
           den = sqrt(vh) + eps:                    e_den = min(e_vh / (2 sqrt vh), sqrt e_vh) + 2u den
           r = mh / den + wd w:                     e_r = e_mh / den + |q| e_den / den + u |q| + 2u |wd w| + u |r|
           trust = ||w|| / ||r||:                   rel_t = rel_n + e_rn / ||r|| + u,  e_rn = sum(|r| e_r) / ||r|| + rel_n ||r||
           w' = w - lr (trust r):                   e_w = lr (trust e_r + |trust r| (rel_t + 2u)) + u |w'|
    LARS:  trust = tc ||w|| / (||g|| + wd ||w|| + eps):   rel_t = 2 rel_n + 6u
           g2 = (G + wd w) trust:                   e_g2 = (2u |G + wd w| + u |wd w|) trust + |g2| (rel_t + u)
           buf' = g2 | buf mom + (1 - damp) g2:     e_b = e_g2 | (1 - damp) e_g2 + 4u (|buf mom| + |(1 - damp) g2|)
           d = g2 + mom buf' | buf':                e_d = e_g2 + mom e_b + 3u (|g2| + |mom buf'|) | e_b
           w' = w - lr d:                           e_w = lr e_d + 2u lr |d| + u |w'|
    A trust ratio that is 1 by its branch (a zero or NaN norm, or no adaptation) contributes no error."""
    h = hyper(kind, h)
    w, G, ref_w = w.to(F64), G.to(F64), ref_w.to(F64)
    st = {k: v.to(F64) for k, v in state.items()}
    n = w.numel()
    t = step + 1
    lr, wd, eps = h["lr"], h["weight_decay"], h["eps"]
    adapt = wd != 0 or h["always_adapt"]
    rel_n = _norm_rel(n)
    wn = float(w.norm())
    if kind == "lamb":
        b1, b2 = h["betas"]
        m = st["exp_avg"].lerp(G, 1 - b1)
        v = st["exp_avg_sq"] * b2 + (1 - b2) * G * G
        e_m = 3 * U * (st["exp_avg"].abs() + G.abs())
        e_v = 6 * U * v
        bc1, bc2 = (1 - b1**t, 1 - b2**t) if h["bias_correction"] else (1.0, 1.0)
        mh, vh = m / bc1, v / bc2
        e_mh = e_m / bc1 + 2 * U * mh.abs()
        e_vh = e_v / bc2 + 2 * U * vh
        s = vh.sqrt()
        e_s = torch.minimum(torch.where(s > 0, e_vh / (2 * s), torch.full_like(s, math.inf)), e_vh.sqrt())
        den = s + eps
        e_den = e_s + 2 * U * den
        q = mh / den
        r = q + wd * w
        e_r = e_mh / den + q.abs() * e_den / den + U * q.abs() + 2 * U * (wd * w).abs() + U * r.abs()
        rn = float(r.norm())
        trust, rel_t = 1.0, 0.0
        if adapt and wn > 0 and rn > 0:
            trust = wn / rn
            e_rn = float((r.abs() * e_r).sum()) / rn + rel_n * rn
            rel_t = rel_n + e_rn / rn + U
        e_w = lr * (trust * e_r + (trust * r).abs() * (rel_t + 2 * U)) + U * ref_w.abs()
        e_state = {"exp_avg": SLACK * e_m, "exp_avg_sq": SLACK * e_v}
        return SLACK * e_w, e_state
    mom, damp = h["momentum"], h["dampening"]
    g2, e_g2 = G, torch.zeros_like(G)
    if adapt:
        gn = float(G.norm())
        trust, rel_t = 1.0, 0.0
        if wn > 0 and gn > 0:
            trust = h["trust_coefficient"] * wn / (gn + wd * wn + eps)
            rel_t = 2 * rel_n + 6 * U
        x = G + wd * w
        g2 = x * trust
        e_g2 = (2 * U * x.abs() + U * (wd * w).abs()) * trust + g2.abs() * (rel_t + U)   # fp32(wd): u |wd w|
    d, e_d = g2, e_g2
    e_state = {}
    if mom != 0:
        if t == 1:
            buf, e_b = g2, e_g2
        else:
            old = st["momentum_buffer"]
            buf = old * mom + (1 - damp) * g2
            e_b = (1 - damp) * e_g2 + 4 * U * ((old * mom).abs() + ((1 - damp) * g2).abs())
        if h["nesterov"]:
            d = g2 + mom * buf
            e_d = e_g2 + mom * e_b + 3 * U * (g2.abs() + (mom * buf).abs())
        else:
            d, e_d = buf, e_b
        e_state = {"momentum_buffer": SLACK * e_b}
    e_w = lr * e_d + 2 * U * lr * d.abs() + U * ref_w.abs()
    return SLACK * e_w, e_state


# ---- deliberately wrong references (negative controls) ------------------------------------------------------------------
MUTATIONS = {"lamb": ("no_trust", "norm_after_update", "no_bias_correction"),
             "lars": ("no_trust", "norm_after_update", "norm_after_weight_decay", "momentum_zero_seed")}


def step_mutant(kind: str, w, state: Dict, g, step: int, h: Dict, mutation: str):
    """The weights after one float64 step (written out here, not the class's code) with one deliberate error:
    "no_trust": the trust ratio is not applied;  "norm_after_update": ||w|| of the weights after this step's (correct)
    update;  "no_bias_correction": LAMB without bias correction;  "norm_after_weight_decay": LARS's ||g|| of g + wd w;
    "momentum_zero_seed": LARS's buffer starts at zeros (buf = (1 - dampening) g at the first step)."""
    h = hyper(kind, h)
    w, g = w.to(F64), g.to(F64)
    st = {k: v.to(F64) for k, v in state.items()}
    t = step + 1
    lr, wd, eps = h["lr"], h["weight_decay"], h["eps"]
    adapt = wd != 0 or h["always_adapt"]
    wn = float(w.norm())
    if mutation == "norm_after_update":
        wn = float(step_ref(kind, w, state, g, step, h)[0].norm())
    if kind == "lamb":
        b1, b2 = h["betas"]
        m = st["exp_avg"].lerp(g, 1 - b1)
        v = st["exp_avg_sq"] * b2 + (1 - b2) * g * g
        bc = h["bias_correction"] and mutation != "no_bias_correction"
        bc1, bc2 = (1 - b1**t, 1 - b2**t) if bc else (1.0, 1.0)
        r = (m / bc1) / ((v / bc2).sqrt() + eps) + wd * w
        trust = _trust(wn, float(r.norm()), wn / max(float(r.norm()), 1e-300)) if adapt else 1.0
        if mutation == "no_trust":
            trust = 1.0
        return w - lr * (trust * r)
    mom, damp = h["momentum"], h["dampening"]
    if adapt:
        gn = float((g + wd * w).norm() if mutation == "norm_after_weight_decay" else g.norm())
        trust = _trust(wn, gn, h["trust_coefficient"] * wn / (gn + wd * wn + eps))
        if mutation == "no_trust":
            trust = 1.0
        g = (g + wd * w) * trust
    if mom != 0:
        if t == 1:
            buf = (1 - damp) * g if mutation == "momentum_zero_seed" else g.clone()
        else:
            buf = st["momentum_buffer"] * mom + (1 - damp) * g
        g = g + mom * buf if h["nesterov"] else buf
    return w - lr * g


def outside(got, ref, bound) -> torch.Tensor:
    """Elements where |got - ref| > bound; NaN on either side counts as outside unless both are NaN."""
    got, ref = got.to(F64), ref.to(F64)
    both_nan = got.isnan() & ref.isnan()
    return ~((got - ref).abs() <= bound) & ~both_nan
