# -*- coding: utf-8 -*-
"""TEST INFRASTRUCTURE ONLY -- float64 reference of one fused StableAdamW step, with per-element fp32 error bounds in the
conventions of oracle/kernel_ref.py (U, SLACK; every fp32 operation and every cast of a float64 scalar to fp32
contributes one u of its result, input errors are propagated to first order).

The values come from the class's own ``step()`` (stoke_b200.optim.StableAdamW) on float64 tensors with the kernel's
pre-step state loaded.  The RMS is the square root of a mean of non-negative terms, so any summation order of its n
terms has a relative error of at most (depth + 1) u, depth being the longest addition chain; the bound takes
layerwise_ref.depth_full(n), which covers both the kernel's launch shapes (k2_layerwise.cu) and torch's fp32 CPU order."""
import math
from typing import Dict

import torch

from kernel_ref import SLACK, U
from layerwise_ref import depth_full, outside  # noqa: F401  (outside: re-exported for the tests)

F64 = torch.float64
KEYS = ("exp_avg", "exp_avg_sq")
DEFAULTS = dict(lr=1e-3, betas=(0.9, 0.99), eps=1e-6, weight_decay=1e-2)


def hyper(h: Dict) -> Dict:
    return dict(DEFAULTS, **h)


def debiased(beta: float, t: int) -> float:
    """beta (1 - beta^(t-1)) / (1 - beta^t): the class's python double, 0 at t = 1."""
    t = float(t)
    return beta * (1 - beta ** (t - 1)) / (1 - beta ** t)


def zero_state(shape) -> Dict:
    return {"exp_avg": torch.zeros(shape), "exp_avg_sq": torch.zeros(shape)}


def step_ref(w, state: Dict, g, step: int, h: Dict, dtype=F64):
    """One step of the class in `dtype` (float64: the reference) from the given state; `step` = steps already taken.
    Returns (w, new state dict)."""
    from stoke_b200.optim import StableAdamW

    p = torch.nn.Parameter(w.to(dtype).clone())
    opt = StableAdamW([p], **hyper(h))
    if step > 0:
        st = {"step": torch.tensor(float(step))}
        st.update({k: v.to(dtype).clone() for k, v in state.items()})
        opt.state[p] = st
    p.grad = g.to(dtype).clone()
    opt.step()
    return p.detach(), {k: opt.state[p][k] for k in KEYS}


def rms_rel(n: int) -> float:
    """Relative error of the fp32 RMS: each term g^2 / max(v, eps^2) carries 9u (g * g, the division, v's 6u, the fp32
    eps^2), the sum (depth + 1) u, the mean 2u (fp32 n, the division); the square root halves that and adds u."""
    return (9 + depth_full(n) + 1 + 2) * U / 2 + U


def step_bound(w, state: Dict, G, step: int, h: Dict, ref_w, ref_state: Dict):
    """Per-element bounds of an fp32 step: (e_w, {key: e_state}).  w, state: the pre-step fp32 values (exact); G: the
    gradient the kernel sees (exact); ref_w / ref_state: the float64 reference's results.

        m' = lerp(m, G, 1 - b1):                e_m = 3u (|m| + |G|)          (either of torch's two lerp forms)
        v' = v b2 + (1 - b2) G^2:               e_v = 6u v'                   (non-negative terms)
        rms = sqrt(mean(G^2 / max(v', eps^2))): e_rms = rms_rel(n) rms
        c = max(rms, 1):                        e_c = e_rms                   (max is 1-Lipschitz)
        lr_t = (1 / c) lr:                      rel_l = e_c / c + 3u          (reciprocal, fp32 lr, product)
        f = 1 - lr_t wd:                        e_f = lr_t wd (rel_l + 2u) + u |f|
        w1 = w f (wd != 0):                     e_w1 = |w| e_f + u |w1|
        den = sqrt(v') + eps:                   e_den = 4u sqrt(v') + 2u den
        q = m' / den:                           e_q = e_m / den + |q| e_den / den + u |q|
        w' = w1 - lr_t q:                       e_w = e_w1 + lr_t e_q + lr_t |q| (rel_l + u) + u |w'|
    A NaN RMS makes the reference NaN everywhere (outside() accepts NaN against NaN)."""
    h = hyper(h)
    w, G, ref_w = w.to(F64), G.to(F64), ref_w.to(F64)
    m0, v0 = state["exp_avg"].to(F64), state["exp_avg_sq"].to(F64)
    t = step + 1
    lr, wd, eps = h["lr"], h["weight_decay"], h["eps"]
    b1, b2 = debiased(h["betas"][0], t), debiased(h["betas"][1], t)
    m = m0.lerp(G, 1 - b1)
    v = v0 * b2 + (1 - b2) * G * G
    e_m = 3 * U * (m0.abs() + G.abs())
    e_v = 6 * U * v
    rms = float((G * G / v.clamp(min=eps * eps)).mean().sqrt())
    c = max(rms, 1.0) if not math.isnan(rms) else rms
    lr_t = lr / c
    rel_l = rms_rel(w.numel()) * rms / c + 3 * U
    if wd != 0:
        f = 1 - lr_t * wd
        e_f = lr_t * wd * (rel_l + 2 * U) + U * abs(f)
        w1 = w * f
        e_w1 = w.abs() * e_f + U * w1.abs()
    else:
        w1, e_w1 = w, torch.zeros_like(w)
    s = v.sqrt()
    den = s + eps
    e_den = 4 * U * s + 2 * U * den
    q = m / den
    e_q = e_m / den + q.abs() * e_den / den + U * q.abs()
    e_w = e_w1 + lr_t * e_q + lr_t * q.abs() * (rel_l + U) + U * ref_w.abs()
    return SLACK * e_w, {"exp_avg": SLACK * e_m, "exp_avg_sq": SLACK * e_v}


def lr_t_of(state: Dict, G, step: int, h: Dict) -> float:
    """The float64 lr_t of one step (the factor the RMS leaves of lr)."""
    h = hyper(h)
    G = G.to(F64)
    b2 = debiased(h["betas"][1], step + 1)
    v = state["exp_avg_sq"].to(F64) * b2 + (1 - b2) * G * G
    rms = float((G * G / v.clamp(min=h["eps"] ** 2)).mean().sqrt())
    return h["lr"] / (rms if rms > 1 else 1.0) if not math.isnan(rms) else math.nan


# ---- deliberately wrong references (negative controls) ------------------------------------------------------------------
MUTATIONS = ("undebiased_betas", "fmax_clamp", "no_weight_decay")


def step_mutant(w, state: Dict, g, step: int, h: Dict, mutation: str):
    """The weights after one float64 step (written out here, not the class's code) with one deliberate error:
    "undebiased_betas": m, v with the plain betas (Adam's moments without any correction);  "fmax_clamp": max(rms, 1) as
    fmaxf takes it, a NaN RMS giving 1;  "no_weight_decay": the decoupled decay is left out.  Any other value (the tests
    use "none") gives the correct transcription, the positive control."""
    h = hyper(h)
    w, g = w.to(F64), g.to(F64)
    m0, v0 = state["exp_avg"].to(F64), state["exp_avg_sq"].to(F64)
    t = step + 1
    lr, wd, eps = h["lr"], h["weight_decay"], h["eps"]
    b1, b2 = h["betas"]
    if mutation != "undebiased_betas":
        b1, b2 = debiased(b1, t), debiased(b2, t)
    m = m0 + (1 - b1) * (g - m0)
    v = b2 * v0 + (1 - b2) * g * g
    rms = float((g * g / torch.clamp(v, min=eps * eps)).mean().sqrt())
    if mutation == "fmax_clamp":
        c = 1.0 if math.isnan(rms) else max(rms, 1.0)
    else:
        c = rms if (math.isnan(rms) or rms > 1) else 1.0
    lr_t = lr / c
    if wd != 0 and mutation != "no_weight_decay":
        w = w * (1 - lr_t * wd)
    return w - lr_t * (m / (v.sqrt() + eps))
