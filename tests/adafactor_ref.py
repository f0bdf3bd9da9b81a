# -*- coding: utf-8 -*-
"""TEST INFRASTRUCTURE ONLY -- float64 reference of the fused Adafactor step, with per-element fp32 error bounds in the
conventions of oracle/kernel_ref.py (U, SLACK; every fp32 operation and every cast of a float64 scalar to fp32 contributes
one u of its result, input errors are propagated to first order).

The values come from ``torch.optim.Adafactor`` itself on float64 tensors with the kernel's pre-step state loaded.  eps1
"None" is resolved to the fp32 epsilon first: the engine steps fp32 masters, so that is what torch resolves it to there.

Sums of squares have non-negative terms, so the relative error of any summation order of n terms is at most (depth + 1) u,
depth being the length of the longest addition chain.  Every bound takes the larger of the kernel's depth (its launch
shapes: k2_adafactor.cu) and a depth that covers torch's fp32 CPU order: n for a row / column / mean reduction, n / 16 + 16
for a whole-tensor norm (16-lane vectorised accumulation), so each bound holds for both."""
import math
from typing import Dict, Optional

import torch

from kernel_ref import SLACK, U

F64 = torch.float64
EPS32 = float(torch.finfo(torch.float32).eps)
TILE, CHUNK = 8192, 32   # k2_adafactor.cu: kAfTile, kAfChunk


def eps1_of(h: Dict) -> float:
    e = h.get("eps", (None, 1e-3))[0]
    return EPS32 if e is None else float(e)


def make_optimizer(params, h: Dict, eps1: Optional[float] = None):
    """torch's single-tensor Adafactor (foreach=False) with the hyper-parameters of `h`."""
    eps = h.get("eps", (None, 1e-3))
    return torch.optim.Adafactor(params, lr=h.get("lr", 1e-2), beta2_decay=h.get("beta2_decay", -0.8),
                                 eps=(eps[0] if eps1 is None else eps1, eps[1]), d=h.get("d", 1.0),
                                 weight_decay=h.get("weight_decay", 0.0), maximize=bool(h.get("maximize", False)),
                                 foreach=False)


def state_keys(shape) -> tuple:
    return ("row_var", "col_var") if len(shape) >= 2 else ("variance",)


def step_ref(w, state: Dict, g, step: int, h: Dict, dtype=F64):
    """One torch step in `dtype` (float64: the reference; float32: torch's own fp32 result) from the given state
    (``state`` holds torch's tensors: row_var / col_var or variance); `step` = steps already taken.
    Returns (w, new state dict)."""
    p = torch.nn.Parameter(w.to(dtype).clone())
    opt = make_optimizer([p], h, eps1=eps1_of(h))
    st = {"step": torch.tensor(float(step))}
    st.update({k: v.to(dtype).clone() for k, v in state.items()})
    opt.state[p] = st
    p.grad = g.to(dtype).clone()
    opt.step()
    return p.detach(), {k: opt.state[p][k] for k in state}


def zero_state(shape) -> Dict:
    if len(shape) >= 2:
        r, c = list(shape), list(shape)
        r[-1], c[-2] = 1, 1
        return {"row_var": torch.zeros(r), "col_var": torch.zeros(c)}
    return {"variance": torch.zeros(shape)}


# ---- depths -------------------------------------------------------------------------------------------------------------
def depth_full(n: int) -> int:
    """||w||^2 and ||u||^2: kernel = 32 per thread + 8 (block tree) + ceil(tiles / 32) + 5 (warp fold); torch n / 16 + 16"""
    tiles = -(-n // TILE)
    return max(32 + 8 + -(-tiles // 32) + 5, -(-n // 16) + 16)


def depth_line(L: int) -> int:
    """row / column sums of g^2 over L terms: kernel chunks of 32 folded in order; torch up to L"""
    return max(L, min(CHUNK, L) + -(-L // CHUNK))


def depth_rowmean(R: int) -> int:
    return R + 5


# ---- bounds -------------------------------------------------------------------------------------------------------------
def step_bound(w, state: Dict, G, step: int, h: Dict, ref_w, ref_state: Dict):
    """Per-element bounds of an fp32 step: (e_w, {key: e_state}).  w, state: the pre-step fp32 values (exact); G: the
    gradient the kernel sees (exact; maximize is applied here); ref_w / ref_state: the float64 reference's results.

      alpha = max(eps2, ||w|| / sqrt n) rho:   rel_a = (D_full(n) + 1) u / 2 + u          (sum, sqrt; max is 1-Lipschitz)
      factored: m_row = mean_c G^2:            e = (D_line(C) + 4) u m_row                 (sum, torch's sqrt/square/div)
                row_var' = lerp(row_var, m_row, b2hat):  e_rv = b2hat e + 5u (|row_var| + m_row)   (same for columns)
                rm = clamp(mean_r row_var', eps1):        e_rm = mean_r e_rv + (D_rowmean(R) + 1) u mean_r |row_var'|
                v = row_var' col_var' / rm:               e_v = (e_rv |cv| + |rv| e_cv) / rm + |v| e_rm / rm + 2u |v|
      vector:   v = lerp(variance, G^2, b2hat):           e_v = b2hat u G^2 + 5u (|variance| + G^2)
      u = G / sqrt(clamp(v, eps1^2)):          e_u = |u| e_v / (2 vc) + 3u |u|
      N = ||u||:                               e_N = (sum 2 |u| e_u + (D_full(n) + 1) u N^2) / (2N) + u N
      coef = -alpha / max(1, N / (sqrt n d)):  rel_c = rel_a + e_N / (sqrt n d denom) [x > 1 side] + u
      w' = w fp32(1 - lr wd) + coef u:         e_w = 2u |w dec| [wd != 0] + |coef| e_u + |coef u| (rel_c + 2u) + u |w'|
    """
    w, G, ref_w = w.to(F64), G.to(F64), ref_w.to(F64)
    if h.get("maximize", False):
        G = -G
    st = {k: v.to(F64).reshape(v.shape) for k, v in state.items()}
    rs = {k: v.to(F64) for k, v in ref_state.items()}
    n = w.numel()
    lr, wd, d = h.get("lr", 1e-2), h.get("weight_decay", 0.0), h.get("d", 1.0)
    eps1, eps2 = eps1_of(h), h.get("eps", (None, 1e-3))[1]
    t = step + 1
    b2 = t ** h.get("beta2_decay", -0.8)
    rho = min(lr, 1 / t**0.5)
    rel_a = (depth_full(n) + 1) * U / 2 + U
    rms = float(w.norm()) / math.sqrt(n)
    alpha = max(eps2, rms) * rho
    e_state = {}
    if w.dim() >= 2:
        C_, R_ = w.shape[-1], w.shape[-2]
        m_row = (G * G).mean(dim=-1, keepdim=True)
        m_col = (G * G).mean(dim=-2, keepdim=True)
        e_row = b2 * (depth_line(C_) + 4) * U * m_row + 5 * U * (st["row_var"].abs() + m_row)
        e_col = b2 * (depth_line(R_) + 4) * U * m_col + 5 * U * (st["col_var"].abs() + m_col)
        rv, cv = rs["row_var"], rs["col_var"]
        rm_raw = rv.mean(dim=-2, keepdim=True)
        rm = rm_raw.clamp(min=eps1)
        e_rm = e_row.mean(dim=-2, keepdim=True) + (depth_rowmean(R_) + 1) * U * rv.abs().mean(dim=-2, keepdim=True)
        v = rv * cv / rm
        e_v = (e_row * cv.abs() + rv.abs() * e_col) / rm + v.abs() * e_rm / rm + 2 * U * v.abs()
        e_state = {"row_var": SLACK * e_row, "col_var": SLACK * e_col}
    else:
        v = rs["variance"]
        e_v = b2 * U * G * G + 5 * U * (st["variance"].abs() + G * G)
        e_state = {"variance": SLACK * e_v}
    vc = v.clamp(min=eps1 * eps1)
    u = G / vc.sqrt()
    e_u = u.abs() * e_v / (2 * vc) + 3 * U * u.abs()
    N = float(u.norm())
    e_N = (float((2 * u.abs() * e_u).sum()) + (depth_full(n) + 1) * U * N * N) / (2 * max(N, 1e-300)) + U * N
    x = N / (math.sqrt(n) * d)
    denom = max(1.0, x)
    rel_c = rel_a + (e_N / (math.sqrt(n) * d * denom) if x > 1.0 - e_N / (math.sqrt(n) * d) else 0.0) + U
    coef = -alpha / denom
    dec = 1 - lr * wd
    e_w = (2 * U * (w * dec).abs() if wd != 0 else 0.0) + abs(coef) * e_u + (coef * u).abs() * (rel_c + 2 * U) \
        + U * ref_w.abs()
    return SLACK * e_w, e_state


def update_ratio(state: Dict, g, step: int, h: Dict) -> float:
    """||u|| / (sqrt(numel) d) of one step in float64 (state: torch's row_var / col_var or variance before the step).
    torch divides the update by max(1, this): above 1 the update's RMS clip is active, below it is not."""
    g = g.to(F64)
    n = g.numel()
    eps1 = eps1_of(h)
    b2 = (step + 1) ** h.get("beta2_decay", -0.8)
    if g.dim() >= 2:
        rv = state["row_var"].to(F64).lerp((g * g).mean(dim=-1, keepdim=True), b2)
        cv = state["col_var"].to(F64).lerp((g * g).mean(dim=-2, keepdim=True), b2)
        v = rv * cv / rv.mean(dim=-2, keepdim=True).clamp(min=eps1)
    else:
        v = state["variance"].to(F64).lerp(g * g, b2)
    u = g / v.clamp(min=eps1 * eps1).sqrt()
    return float(u.norm()) / (math.sqrt(n) * h.get("d", 1.0))


# ---- deliberately wrong references (negative controls) ------------------------------------------------------------------
MUTATIONS = ("alpha_after_decay", "eps1_bf16", "rho_no_min", "sum_not_mean", "no_eps1sq_clamp", "denom_no_max1")


def step_mutant(w, state: Dict, g, step: int, h: Dict, mutation: str):
    """The master weights after one float64 Adafactor step (written out here, not torch's code) with one deliberate
    error:  "alpha_after_decay": the RMS of w after the weight decay;  "eps1_bf16": eps1 = bf16 epsilon (a bf16 model's
    parameter dtype) for None;  "rho_no_min": rho = 1 / sqrt(t) without min(lr, .);  "sum_not_mean": row / column sums of
    g^2 instead of means;  "no_eps1sq_clamp": v not clamped at eps1^2;  "denom_no_max1": denom = ||u|| / (sqrt n d)."""
    w, g = w.to(F64).clone(), g.to(F64)
    if h.get("maximize", False):
        g = -g
    n = w.numel()
    lr, wd, d = h.get("lr", 1e-2), h.get("weight_decay", 0.0), h.get("d", 1.0)
    eps_cfg = h.get("eps", (None, 1e-3))
    eps1 = (2.0**-7 if eps_cfg[0] is None else eps_cfg[0]) if mutation == "eps1_bf16" else eps1_of(h)
    eps2 = eps_cfg[1]
    t = step + 1
    b2 = t ** h.get("beta2_decay", -0.8)
    rho = 1 / t**0.5 if mutation == "rho_no_min" else min(lr, 1 / t**0.5)
    dec = 1 - lr * wd
    w_alpha = w * dec if mutation == "alpha_after_decay" else w
    alpha = max(eps2, float(w_alpha.norm()) / math.sqrt(n)) * rho
    if wd != 0:
        w = w * dec
    if w.dim() >= 2:
        red = (lambda x, dim: x.sum(dim=dim, keepdim=True)) if mutation == "sum_not_mean" else \
            (lambda x, dim: x.mean(dim=dim, keepdim=True))
        rv = state["row_var"].to(F64).lerp(red(g * g, -1), b2)
        cv = state["col_var"].to(F64).lerp(red(g * g, -2), b2)
        v = rv * cv / rv.mean(dim=-2, keepdim=True).clamp(min=eps1)
    else:
        v = state["variance"].to(F64).lerp(g * g, b2)
    if mutation != "no_eps1sq_clamp":
        v = v.clamp(min=eps1 * eps1)
    u = g / v.sqrt()
    x = float(u.norm()) / (math.sqrt(n) * d)
    denom = x if mutation == "denom_no_max1" else max(1.0, x)
    return w - (alpha / denom) * u


def outside(got, ref, bound) -> torch.Tensor:
    """Elements where |got - ref| > bound; NaN on either side counts as outside unless both are NaN."""
    got, ref = got.to(F64), ref.to(F64)
    both_nan = got.isnan() & ref.isnan()
    return ~((got - ref).abs() <= bound) & ~both_nan
