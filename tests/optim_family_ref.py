# -*- coding: utf-8 -*-
"""TEST INFRASTRUCTURE ONLY -- float64 reference of the fused step's NAdam, RAdam and Adamax kinds, with per-element fp32
error bounds, in the style of oracle/kernel_ref.py (same u, SLACK and conventions: every fp32 operation, and every cast of a
float64 scalar to fp32, contributes one u of its result; a fused multiply-add only removes roundings; input errors are
propagated to first order).

The values come from ``torch.optim.NAdam`` / ``RAdam`` / ``Adamax`` themselves, run on float64 tensors with the kernel's
pre-step state loaded (``step`` and, for NAdam, ``mu_product``), so the reference is torch's formula in higher precision.
Each bound covers both the kernel's order of operations and torch's own fp32 single-tensor order, where they differ (RAdam).
"""
import math
from typing import Dict, Optional

import torch

from kernel_ref import SLACK, U

F64 = torch.float64
KINDS = ("nadam", "radam", "adamax")


def _wd(h: Dict) -> float:
    return float(h.get("weight_decay", 0.0))


def _decoupled(kind: str, h: Dict) -> bool:
    return kind in ("nadam", "radam") and bool(h.get("decoupled_weight_decay", False)) and _wd(h) != 0.0


def make_optimizer(kind: str, params, h: Dict, dtype_state=None):
    """torch's single-tensor implementation (foreach=False) of `kind` with the hyper-parameters of `h`."""
    common = dict(lr=h["lr"], betas=(h["beta1"], h["beta2"]), eps=h["eps"], weight_decay=_wd(h),
                  maximize=bool(h.get("maximize", False)), foreach=False)
    if kind == "nadam":
        return torch.optim.NAdam(params, momentum_decay=h.get("momentum_decay", 4e-3),
                                 decoupled_weight_decay=bool(h.get("decoupled_weight_decay", False)), **common)
    if kind == "radam":
        return torch.optim.RAdam(params, decoupled_weight_decay=bool(h.get("decoupled_weight_decay", False)), **common)
    return torch.optim.Adamax(params, **common)


def second_key(kind: str) -> str:
    return "exp_inf" if kind == "adamax" else "exp_avg_sq"


def step_ref(kind: str, w, m, v, g, step: int, h: Dict, mu_product: Optional[float] = None):
    """One torch step in float64 from the given state; `step` = steps already taken, `mu_product` (NAdam) the product
    before the step.  Returns (w, m, v, mu_product after the step or None)."""
    p = torch.nn.Parameter(w.to(F64).clone())
    opt = make_optimizer(kind, [p], h)
    st = {"step": torch.tensor(float(step), dtype=F64), "exp_avg": m.to(F64).clone(), second_key(kind): v.to(F64).clone()}
    if kind == "nadam":
        st["mu_product"] = torch.tensor(float(mu_product), dtype=F64)
    opt.state[p] = st
    p.grad = g.to(F64).clone()
    opt.step()
    st = opt.state[p]
    return p.detach(), st["exp_avg"], st[second_key(kind)], (float(st["mu_product"]) if kind == "nadam" else None)


# ---- the per-step scalars (python floats in torch; stk_optim_step_prologue forms them in double) --------------------------
def nadam_mu(h: Dict, t: float) -> float:
    return h["beta1"] * (1.0 - 0.5 * (0.96 ** (t * h.get("momentum_decay", 4e-3))))


def mu_product_f32(mu_prev: float, h: Dict, t: int) -> float:
    """torch's ``mu_product *= mu`` on its fp32 tensor: fp32(mu_prev * fp32(mu))."""
    return float(torch.tensor(mu_prev, dtype=torch.float32) * torch.tensor(nadam_mu(h, float(t)), dtype=torch.float32))


def radam_rho(h: Dict, t: float) -> float:
    b2 = h["beta2"]
    rho_inf = 2 / (1 - b2) - 1
    return rho_inf - 2 * t * (b2**t) / (1 - b2**t)


def radam_rectified(h: Dict, t: int) -> bool:
    return t >= 1 and radam_rho(h, float(t)) > 5.0


def prologue_scalars(kind: str, h: Dict, done: int, mu_prev: float = 1.0):
    """The four floats stk_optim_step_prologue stores for step done + 1, in float64 (the kernel must be within 1 fp32 ulp
    of each), and NAdam's advanced fp32 mu_product."""
    t = float(done + 1)
    b1, b2, lr = h["beta1"], h["beta2"], h["lr"]
    bc1, bc2 = 1 - b1**t, 1 - b2**t
    if kind == "nadam":
        mu, mu_next = nadam_mu(h, t), nadam_mu(h, t + 1)
        prod = mu_product_f32(mu_prev, h, done + 1)
        return (-lr * (1 - mu) / (1 - prod), -lr * mu_next / (1 - prod * mu_next), bc2, 0.0), prod
    if kind == "radam":
        rho_inf, rho_t = 2 / (1 - b2) - 1, radam_rho(h, t)
        if rho_t > 5.0:
            rect = math.sqrt((rho_t - 4) * (rho_t - 2) * rho_inf / ((rho_inf - 4) * (rho_inf - 2) * rho_t))
            return (lr * rect * math.sqrt(bc2) / bc1, 1.0, 0.0, 0.0), None
        return (lr / bc1, 0.0, 0.0, 0.0), None
    return (lr / bc1, 0.0, 0.0, 0.0), None


# ---- bounds -------------------------------------------------------------------------------------------------------------
def step_bound(kind: str, w, m, v, G, e_g, step: int, h: Dict, ref_m, ref_v, mu_product: Optional[float] = None):
    """Per-element bounds (e_w, e_m, e_v) of an fp32 step of `kind`.  w, m, v: the pre-step fp32 state (exact); G: the
    reference gradient after clipping (float64; maximize is applied here), e_g its bound; ref_m, ref_v: the reference's
    new state; mu_product: NAdam's fp32 product before the step.  t = step + 1, bc1 = 1 - b1^t, bc2 = 1 - b2^t.

      L2 decay  Gd = G + wd w:                 e_d = e_g + u (2 |wd w| + |Gd|)          (NAdam / RAdam without decoupling,
                                                                                          Adamax)
      decoupled Wd = fp32(1 - lr wd) w:        e_Wd = 2u |Wd|                           (cast, product; else Wd = w exact)
      m' = lerp(m, Gd, 1 - b1):                e_m = (1-b1) e_d + 3u (1-b1) |Gd - m| + u |m'|     (as Adam)
      v' = b2 v + (1 - b2) Gd^2:               e_v = 2u b2 v + 2 (1-b2) |Gd| e_d + 3u (1-b2) Gd^2 + u v'   (as Adam)

    NAdam.  The kernel restarts from its own fp32 product P0, so the reference's P = P0 mu_t (float64) and the fp32
    P^ = fp32(P0 fp32(mu_t)) is off by e_P = 2u P (this is the fp32 rounding of the product the bound has to cover).
      c_g = -lr (1 - mu_t) / (1 - P):          relative error e_P / (1 - P) + u          (P enters the denominator; the cast)
      c_m = -lr mu' / (1 - P mu'):             relative error mu' e_P / (1 - P mu') + u
      q = v' / fp32(bc2):                      e_q = e_v / bc2 + 2u q                   (cast, division)
      s = sqrt(q), D = s + eps:                e_D = e_q / (2 s) + u s + u eps + u D
      r1 = Gd / D, r2 = m' / D:                e_ri = (e_num + |ri| e_D) / D + u |ri|
      w1 = Wd + c_g r1:                        e_w1 = e_Wd + |c_g| (e_r1 + rel_g |r1|) + 2u |c_g r1| + u |w1|
      w' = w1 + c_m r2:                        e_w = e_w1 + |c_m| (e_r2 + rel_m |r2|) + 2u |c_m r2| + u |w'|
    RAdam, rectified (rho_t > 5): upd = A m' / (sqrt(v') + eps), A = lr rect sqrt(bc2) / bc1.  The kernel rounds three
    times relative to upd (cast of A, division, product); torch's fp32 order (m' / bc1) * lr * (sqrt(bc2) / D) * rect rounds
    nine times (four casts, five operations), so k = 9:
      D = sqrt(v') + eps:                      e_D = e_v / (2 sqrt v') + u sqrt v' + u eps + u D
      upd:                                     e_upd = A (e_m + |m' / D| e_D) / D + 9u |upd|
    RAdam, unrectified: upd = (lr / bc1) m'.  Kernel: two roundings; torch (m' / bc1) * lr: four, so
      e_upd = (lr / bc1) e_m + 4u |upd|
    both:  w' = Wd - upd:                      e_w = e_Wd + e_upd + u |w'|
    Adamax.  u' = max(b2 u, |Gd| + eps): max is 1-Lipschitz, so its error is at most the larger of the two arguments':
      e_u = max(2u b2 u, e_d + u eps + u (|Gd| + eps))
      r = m' / u':                             e_r = (e_m + |r| e_u) / u' + u |r|
      w' = w - fp32(lr / bc1) r:               e_w = (lr / bc1) e_r + 2u |upd| + u |w'|
    """
    b1, b2, eps, lr = h["beta1"], h["beta2"], h["eps"], h["lr"]
    wd = _wd(h)
    w, m, v, G, e_g, ref_m, ref_v = (x.to(F64) for x in (w, m, v, G, e_g, ref_m, ref_v))
    if h.get("maximize", False):
        G = -G
    dec = _decoupled(kind, h)
    if wd != 0.0 and not dec:
        Gd = G + wd * w
        e_d = e_g + U * (2 * (wd * w).abs() + Gd.abs())
    else:
        Gd, e_d = G, e_g
    if dec:
        Wd = w * (1 - lr * wd)
        e_Wd = 2 * U * Wd.abs()
    else:
        Wd, e_Wd = w, torch.zeros_like(w)
    t = step + 1
    bc1, bc2 = 1 - b1**t, 1 - b2**t
    e_m = (1 - b1) * e_d + 3 * U * (1 - b1) * (Gd - m).abs() + U * ref_m.abs()
    if kind == "adamax":
        e_u = torch.maximum(2 * U * b2 * v, e_d + U * eps + U * (Gd.abs() + eps))
        r = ref_m / ref_v
        e_r = (e_m + r.abs() * e_u) / ref_v + U * r.abs()
        upd = (lr / bc1) * r
        w_new = w - upd
        e_w = (lr / bc1) * e_r + 2 * U * upd.abs() + U * w_new.abs()
        return SLACK * e_w, SLACK * e_m, SLACK * e_u
    e_v = 2 * U * b2 * v + 2 * (1 - b2) * Gd.abs() * e_d + 3 * U * (1 - b2) * Gd * Gd + U * ref_v
    if kind == "nadam":
        mu, mu_n = nadam_mu(h, float(t)), nadam_mu(h, float(t + 1))
        P = float(mu_product) * mu
        e_P = 2 * U * P
        c_g, c_m = -lr * (1 - mu) / (1 - P), -lr * mu_n / (1 - P * mu_n)
        rel_g, rel_m = e_P / (1 - P) + U, mu_n * e_P / (1 - P * mu_n) + U
        q = ref_v / bc2
        e_q = e_v / bc2 + 2 * U * q
        s = q.sqrt()
        D = s + eps
        e_s = torch.where(s > 0, e_q / (2 * s).clamp_min(1e-300), e_q.sqrt())
        e_D = e_s + U * s + U * eps + U * D
        r1, r2 = Gd / D, ref_m / D
        e_r1 = (e_d + r1.abs() * e_D) / D + U * r1.abs()
        e_r2 = (e_m + r2.abs() * e_D) / D + U * r2.abs()
        w1 = Wd + c_g * r1
        e_w1 = e_Wd + abs(c_g) * (e_r1 + rel_g * r1.abs()) + 2 * U * (c_g * r1).abs() + U * w1.abs()
        w_new = w1 + c_m * r2
        e_w = e_w1 + abs(c_m) * (e_r2 + rel_m * r2.abs()) + 2 * U * (c_m * r2).abs() + U * w_new.abs()
        return SLACK * e_w, SLACK * e_m, SLACK * e_v
    # RAdam
    if radam_rectified(h, t):
        rho_inf, rho_t = 2 / (1 - b2) - 1, radam_rho(h, float(t))
        rect = math.sqrt((rho_t - 4) * (rho_t - 2) * rho_inf / ((rho_inf - 4) * (rho_inf - 2) * rho_t))
        A = lr * rect * math.sqrt(bc2) / bc1
        sv = ref_v.sqrt()
        e_sv = torch.where(sv > 0, e_v / (2 * sv).clamp_min(1e-300), e_v.sqrt())
        D = sv + eps
        e_D = e_sv + U * sv + U * eps + U * D
        upd = A * ref_m / D
        e_upd = A * (e_m + (ref_m / D).abs() * e_D) / D + 9 * U * upd.abs()
    else:
        upd = (lr / bc1) * ref_m
        e_upd = (lr / bc1) * e_m + 4 * U * upd.abs()
    w_new = Wd - upd
    e_w = e_Wd + e_upd + U * w_new.abs()
    return SLACK * e_w, SLACK * e_m, SLACK * e_v


# ---- deliberately wrong references (negative controls) ------------------------------------------------------------------
MUTATIONS = {
    "nadam": ("mu_t_for_next", "mu_not_advanced", "decoupled_as_l2"),
    "radam": ("no_rect", "threshold_late", "threshold_early", "decoupled_as_l2"),
    "adamax": ("eps_after_max",),
}


def step_mutant(kind: str, w, m, v, g, step: int, h: Dict, mutation: str, mu_product: Optional[float] = None):
    """The master weights after one float64 step of `kind` with one deliberate error:
      NAdam  "mu_t_for_next":    mu_t where torch uses mu_{t+1} (in c_m)
             "mu_not_advanced":  the coefficients from the product before the step instead of after it
      RAdam  "no_rect":          the rectified update without its rect factor
             "threshold_late":   the rho_t > 5 test one step late (the first rectified step is taken unrectified)
             "threshold_early":  one step early (the last unrectified step is taken rectified)
      NAdam / RAdam "decoupled_as_l2": decoupled_weight_decay=True applied as L2 decay of the gradient
      Adamax "eps_after_max":    u = max(b2 u, |g|) + eps"""
    b1, b2, eps, lr = h["beta1"], h["beta2"], h["eps"], h["lr"]
    wd = _wd(h)
    w, m, v, g = (x.to(F64).clone() for x in (w, m, v, g))
    if h.get("maximize", False):
        g = -g
    dec = _decoupled(kind, h) and mutation != "decoupled_as_l2"
    if wd != 0.0:
        if dec:
            w = w * (1 - lr * wd)
        else:
            g = g + wd * w
    t = step + 1
    bc1, bc2 = 1 - b1**t, 1 - b2**t
    m = b1 * m + (1 - b1) * g
    if kind == "adamax":
        u = torch.maximum(b2 * v, g.abs()) + eps if mutation == "eps_after_max" else torch.maximum(b2 * v, g.abs() + eps)
        return w - (lr / bc1) * m / u
    v = b2 * v + (1 - b2) * g * g
    if kind == "nadam":
        mu, mu_n = nadam_mu(h, float(t)), nadam_mu(h, float(t + 1))
        P = float(mu_product) * (1.0 if mutation == "mu_not_advanced" else mu)
        if mutation == "mu_t_for_next":
            mu_n = mu
        D = (v / bc2).sqrt() + eps
        return w + (-lr * (1 - mu) / (1 - P)) * g / D + (-lr * mu_n / (1 - P * mu_n)) * m / D
    shift = {"threshold_late": -1, "threshold_early": 1}.get(mutation, 0)
    if radam_rectified(h, t + shift):
        rho_inf, rho_t = 2 / (1 - b2) - 1, radam_rho(h, float(t))
        rect = 1.0 if mutation == "no_rect" or rho_t <= 4 else \
            math.sqrt((rho_t - 4) * (rho_t - 2) * rho_inf / ((rho_inf - 4) * (rho_inf - 2) * rho_t))
        return w - lr * rect * math.sqrt(bc2) / bc1 * m / (v.sqrt() + eps)
    return w - (lr / bc1) * m
