# -*- coding: utf-8 -*-
"""TEST INFRASTRUCTURE ONLY -- float64 reference of the single-GPU gradient kernels, with per-element error bounds.

The values come from torch's own ops run in float64 on the CPU (``torch.optim.Adam`` / ``AdamW`` / ``SGD`` with the
kernel's pre-step state loaded, ``clip_grad_norm_`` / ``clip_grads_with_norm_`` / ``clip_grad_value_``,
``torch.linalg.vector_norm``, ``torch._amp_update_scale_``), so the reference is torch's formula in higher precision, not a
restatement of the kernels.  What the kernels add on top of that formula is fp32 rounding; the ``*_bound`` functions bound
it element by element as

    |got - ref| <= k * u * S,     u = 2**-24 (fp32 unit round-off),

where S is built from the magnitudes of the terms of each formula and k counts the roundings those terms go through.  The
derivations below assume every fp32 operation rounds on its own (a product, a sum, and the cast of a float64
hyper-parameter to fp32 each contribute one u of their result); a fused multiply-add only removes roundings, so the same
bound covers the kernels (which use fma) and torch's fp32 CPU ops (which mostly do not).  Errors of the inputs of an
operation are propagated to first order; ``SLACK`` covers the second-order terms and the float64 reference's own rounding
(2**-53 relative), both below 1e-6 of the bound at these magnitudes.

Every step is compared against the reference restarted from the kernel's own state, so the bounds hold per step and
never have to absorb an accumulated drift.
"""
import math
from typing import Dict, Optional, Tuple

import torch

U = 2.0**-24
SLACK = 1.01
F64 = torch.float64


def f32_value(x: float) -> float:
    """The fp32 value the kernels use for a float64 scalar (hyper-parameters are cast once on the host or device)."""
    return float(torch.tensor(x, dtype=torch.float32))


def inv_scale_f32(scale: float) -> float:
    """1/loss_scale exactly as GradScaler computes it: float32(1 / float64(scale))."""
    return float(torch.tensor(float(scale), dtype=F64).reciprocal().float())


# ---- the gradient pipeline in front of the norm and the optimizer: x = ((g [+ acc]) * mul) * inv_scale -----------------
def scaled_grad(g: torch.Tensor, acc: Optional[torch.Tensor], mul: float, inv_scale: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """(x, e_x): the exact value in float64 of the unscaled gradient and the bound on the kernel's fp32 rounding of it.

    fp32 kernel: t = fl(g + acc) -> u|t| (only with an accumulator); t = fl(t * float(mul)) -> 2u|t| (cast of mul and the
    product; nothing when mul == 1); x = fl(t * inv_scale) -> u|x| (inv_scale is already the fp32 value GradScaler uses;
    nothing when it is 1).  So e_x = k_x * u * |x| with k_x = [acc] + 2 [mul != 1] + [inv_scale != 1] (first order)."""
    x = g.to(F64)
    k = 0
    if acc is not None:
        x = x + acc.to(F64)
        k += 1
    if mul != 1.0:
        x = x * mul
        k += 2
    if inv_scale != 1.0:
        x = x * inv_scale
        k += 1
    return x, k * U * x.abs()


def scaled_grad_f32(g: torch.Tensor, acc: Optional[torch.Tensor], mul: float, inv_scale: float) -> torch.Tensor:
    """The same pipeline as fp32 torch ops in the kernels' order: K1 must match it bit for bit (no sum is reordered)."""
    x = g.float()
    if acc is not None:
        x = x + acc.float()
    x = x * torch.tensor(mul, dtype=torch.float32)
    return x * torch.tensor(inv_scale, dtype=torch.float32)


# ---- norms --------------------------------------------------------------------------------------------------------------
def norm_ref(x: torch.Tensor, norm_type: float) -> float:
    """clip_grad_norm_'s total norm in float64 (NaN if any element is NaN, else inf if any is inf)."""
    x = x.to(F64).reshape(-1)
    if x.numel() == 0:
        return 0.0
    return float(torch.linalg.vector_norm(x, norm_type))


def depth_norm_pass(n: int, calls: int = 1) -> int:
    """Longest chain of fp32 additions an element goes through in stk_grad_norm (k_grad_norm + k_grad_norm_finish):
    64 in its thread (8 vectors of 8, fma into the running partial) + 10 in the block tree (5 shuffle levels in the warp,
    5 across the 8 warps' partials) + ceil(blocks / 1024) in the finisher's thread + 10 in the finisher's tree + one per
    call for the running total over calls."""
    blocks = max(1, -(-(n // 8) // 2048))
    return 64 + 10 + -(-blocks // 1024) + 10 + calls


def depth_reduce_w1(n: int, calls: int = 1) -> int:
    """The same for stk_grad_reduce at world 1 (k_grad_reduce<1> + k_grad_norm_finish): 16 in the thread (2 vectors of 8)
    + 10 in the block tree (5 shuffle levels in the warp, 5 across the 8 warps' partials) + ceil(blocks / 1024) in the
    finisher's thread + 10 in the finisher's tree + one per call for the running total over calls."""
    blocks = max(1, -(-(n // 8) // 512))
    return 16 + 10 + -(-blocks // 1024) + 10 + calls


def norm_bound(x: torch.Tensor, e_x: torch.Tensor, norm_type: float, depth: int) -> float:
    """Bound on |kernel norm - norm_ref(x)| for the fp32 inputs x (exact values, float64) with rounding e_x.

    L2: S = sum x^2.  Each x^2 carries 2 e_x |x| from its input; a sum over a tree whose longest chain is `depth` has
    |S^ - S| <= depth * u * sum|terms| = depth * u * S (terms >= 0; Higham, Accuracy and Stability, 4.2).  sqrtf halves the
    relative error and adds u:  |N^ - N| <= (sum 2 e_x |x| / S / 2 + depth * u / 2 + u) * N.
    inf: the max is exact, so |N^ - N| <= max e_x.
    p: each term |x|^p comes from __powf = exp2(p * log2|x|) with the hardware approximations: log2 has at most
    2**-22 * max(1, |log2 x|) absolute error, the product p * log2 one u of itself, exp2 2 ulp (2**-22) relative, so a term
    is off by delta = ln2 * p * (2**-22 * max(1, |log2 x|) + u |log2 x|) + 2**-22 relative (+ p e_x / |x| from its input).
    With the tree: |S^ - S| <= sum delta_i t_i + depth u S.  powf(S, float(1/p)) then gives (1/p) of S's relative
    error, |ln S| u / p from the rounding of 1/p, and 4 ulp (2**-21) of its own."""
    x = x.to(F64).reshape(-1)
    e_x = e_x.to(F64).reshape(-1)
    if x.numel() == 0:
        return 0.0
    a = x.abs()
    if math.isinf(norm_type):
        return SLACK * float(e_x.max())
    if norm_type == 2.0:
        S = float((a * a).sum())
        if S == 0.0:
            return 0.0
        N = math.sqrt(S)
        rel = float((2 * e_x * a).sum()) / S / 2 + depth * U / 2 + U
        return SLACK * rel * N
    p = float(norm_type)
    t = a**p
    S = float(t.sum())
    if S == 0.0:
        return 0.0
    nz = a > 0
    l2 = torch.zeros_like(a)
    l2[nz] = torch.log2(a[nz]).abs()
    delta = math.log(2) * p * (2.0**-22 * torch.clamp(l2, min=1.0) + U * l2) + 2.0**-22
    rel_in = torch.zeros_like(a)
    rel_in[nz] = p * e_x[nz] / a[nz]
    rel_S = (float(((delta + rel_in) * t).sum()) + depth * U * S) / S
    N = S ** (1.0 / p)
    rel = rel_S / p + abs(math.log(S)) * U / p + 2.0**-21
    return SLACK * rel * N


# ---- clipping -----------------------------------------------------------------------------------------------------------
def clip_coef(total_norm: float, max_norm: float) -> float:
    """clip_grad_norm_'s coefficient for a given total norm, from torch's own clip_grads_with_norm_ in float64."""
    one = torch.ones(1, dtype=F64, requires_grad=True)
    one.grad = torch.ones(1, dtype=F64)
    torch.nn.utils.clip_grads_with_norm_([one], max_norm, torch.tensor(total_norm, dtype=F64), foreach=False)
    return float(one.grad[0])


def clip_coef_bound(total_norm: float, max_norm: float) -> float:
    """fp32 kernel: c = min(fl(max_norm / fl(norm + 1e-6f)), 1) with max_norm an fp32 value: the sum rounds (u), 1e-6f
    differs from 1e-6 by |1e-6f - 1e-6|, the division rounds (u):  |c^ - c| <= c (2u + |1e-6f - 1e-6| / (norm + 1e-6)).
    The clamp at 1 does not increase the distance."""
    c = clip_coef(total_norm, max_norm)
    if not math.isfinite(c):
        return 0.0
    d = abs(f32_value(1e-6) - 1e-6) / (total_norm + 1e-6)
    return SLACK * c * (2 * U + d)


def clip_value_ref(g: torch.Tensor, clip_value: float) -> torch.Tensor:
    g = g.to(F64).clone()
    p = torch.zeros_like(g, requires_grad=True)
    p.grad = g
    torch.nn.utils.clip_grad_value_([p], clip_value, foreach=False)
    return p.grad


# ---- optimizer steps ----------------------------------------------------------------------------------------------------
def _optimizer(kind: str, w: torch.Tensor, hyper: Dict):
    p = torch.nn.Parameter(w.to(F64).clone())
    h = dict(hyper)
    if kind == "sgd":
        opt = torch.optim.SGD([p], lr=h["lr"], momentum=h.get("momentum", 0.0), dampening=h.get("dampening", 0.0),
                              weight_decay=h.get("weight_decay", 0.0), nesterov=h.get("nesterov", False),
                              maximize=h.get("maximize", False), foreach=False)
    else:
        cls = torch.optim.AdamW if kind == "adamw" else torch.optim.Adam
        opt = cls([p], lr=h["lr"], betas=(h["beta1"], h["beta2"]), eps=h["eps"],
                  weight_decay=h.get("weight_decay", 0.0 if kind == "adam" else 1e-2), maximize=h.get("maximize", False),
                  foreach=False)
    return p, opt


def adam_step(kind: str, w, m, v, g, step: int, hyper: Dict):
    """One torch.optim.Adam / AdamW step in float64 from the given state; `step` = steps already taken (torch's
    state["step"] before the call).  Returns (w, m, v)."""
    p, opt = _optimizer(kind, w, hyper)
    opt.state[p] = {"step": torch.tensor(float(step), dtype=F64), "exp_avg": m.to(F64).clone(),
                    "exp_avg_sq": v.to(F64).clone()}
    p.grad = g.to(F64).clone()
    opt.step()
    st = opt.state[p]
    return p.detach(), st["exp_avg"], st["exp_avg_sq"]


def sgd_step(w, buf: Optional[torch.Tensor], g, hyper: Dict):
    """One torch.optim.SGD step in float64.  buf = None: no momentum buffer yet (torch seeds it with the gradient).
    Returns (w, buf) (buf None without momentum)."""
    p, opt = _optimizer("sgd", w, hyper)
    if buf is not None and hyper.get("momentum", 0.0) != 0.0:
        opt.state[p] = {"momentum_buffer": buf.to(F64).clone()}
    p.grad = g.to(F64).clone()
    opt.step()
    nb = opt.state[p].get("momentum_buffer") if p in opt.state else None
    return p.detach(), nb


def adam_bound(kind: str, w, m, v, G, e_g, step: int, hyper: Dict, ref_m, ref_v):
    """Per-element bounds (e_w, e_m, e_v) of the kernel's fp32 Adam / AdamW step.  w, m, v: the pre-step fp32 state
    (exact); G: the reference gradient after clipping and maximize (float64), e_g its bound; ref_m, ref_v: the reference's
    new moments.  b1, b2, eps, lr, wd are the float64 hyper-parameters, t = step + 1.

      Adam weight decay  Gd = G + wd w:        e_d = e_g + u (2 |wd w| + |Gd|)         (cast of wd, product, sum)
      m' = b1 m + (1 - b1) Gd  (lerp):         e_m = (1-b1) e_d + 3u (1-b1) |Gd - m| + u |m'|
                                                  (difference, cast of 1-b1, product; the sum)
      v' = b2 v + (1 - b2) Gd^2:               e_v = 2u b2 v + 2 (1-b2) |Gd| e_d + 3u (1-b2) Gd^2 + u v'
      q = sqrt(v') / float(sqrt(1 - b2^t)):    e_q = (e_v / (2 sqrt v') + u sqrt v') / c2 + 2u q   (sqrt, cast, division)
      D = q + eps:                             e_D = e_q + u eps + u D
      r = m' / D:                              e_r = (e_m + |r| e_D) / D + u |r|
      upd = float(lr / (1 - b1^t)) r:          e_upd = s e_r + 2u |upd|                 (cast of the step size, product)
      Adam  w' = w - upd:                      e_w = e_upd + u |w'|
      AdamW w' = float(1 - lr wd) w - upd:     e_w = 2u |w (1 - lr wd)| + e_upd + u |w'|
    """
    b1, b2, eps, lr = hyper["beta1"], hyper["beta2"], hyper["eps"], hyper["lr"]
    wd = hyper.get("weight_decay", 0.0 if kind == "adam" else 1e-2)
    w, m, v, G, e_g = (t.to(F64) for t in (w, m, v, G, e_g))
    sign = -1.0 if hyper.get("maximize", False) else 1.0
    G = G * sign
    if kind == "adam" and wd != 0.0:
        Gd = G + wd * w
        e_d = e_g + U * (2 * (wd * w).abs() + Gd.abs())
    else:
        Gd, e_d = G, e_g
    t = step + 1
    e_m = (1 - b1) * e_d + 3 * U * (1 - b1) * (Gd - m).abs() + U * ref_m.abs()
    e_v = 2 * U * b2 * v + 2 * (1 - b2) * Gd.abs() * e_d + 3 * U * (1 - b2) * Gd * Gd + U * ref_v
    c2 = math.sqrt(1 - b2**t)
    sv = ref_v.sqrt()
    e_sqrt = torch.where(sv > 0, e_v / (2 * sv).clamp_min(1e-300), e_v.sqrt()) + U * sv
    q = sv / c2
    e_q = e_sqrt / c2 + 2 * U * q
    D = q + eps
    e_D = e_q + U * eps + U * D
    r = ref_m / D
    e_r = (e_m + r.abs() * e_D) / D + U * r.abs()
    s = lr / (1 - b1**t)
    e_upd = s * e_r + 2 * U * (s * r).abs()
    w_new_approx = w * (1 - lr * wd if kind == "adamw" else 1.0) - s * r
    e_w = e_upd + U * w_new_approx.abs()
    if kind == "adamw":
        e_w = e_w + 2 * U * (w * (1 - lr * wd)).abs()
    return SLACK * e_w, SLACK * e_m, SLACK * e_v


def sgd_bound(w, buf, G, e_g, hyper: Dict, ref_w, ref_buf):
    """Per-element bounds (e_w, e_buf) of the kernel's fp32 SGD step (torch/optim/sgd.py, _single_tensor_sgd).

      weight decay  Gd = G + wd w:                e_d = e_g + u (2 |wd w| + |Gd|)
      first step    B = Gd:                       e_B = e_d
      later         B = mom buf + (1-damp) Gd:    e_B = (1-damp) e_d + 2u (mom |buf| + (1-damp) |Gd|) + u |B|
      nesterov      Gn = Gd + mom B:              e_n = e_d + mom e_B + 2u mom |B| + u |Gn|      (else Gn = B, e_n = e_B)
      w' = w - lr Gn:                             e_w = lr e_n + 2u lr |Gn| + u |w'|
    Without momentum Gn = Gd, e_n = e_d."""
    lr, mom = hyper["lr"], hyper.get("momentum", 0.0)
    damp, wd = hyper.get("dampening", 0.0), hyper.get("weight_decay", 0.0)
    w, G, e_g = w.to(F64), G.to(F64), e_g.to(F64)
    if hyper.get("maximize", False):
        G = -G
    if wd != 0.0:
        Gd = G + wd * w
        e_d = e_g + U * (2 * (wd * w).abs() + Gd.abs())
    else:
        Gd, e_d = G, e_g
    e_B = None
    if mom != 0.0:
        B = ref_buf
        if buf is None:
            e_B = e_d
        else:
            e_B = (1 - damp) * e_d + 2 * U * (mom * buf.to(F64).abs() + (1 - damp) * Gd.abs()) + U * B.abs()
        if hyper.get("nesterov", False):
            Gn = Gd + mom * B
            e_n = e_d + mom * e_B + 2 * U * mom * B.abs() + U * Gn.abs()
        else:
            Gn, e_n = B, e_B
    else:
        Gn, e_n = Gd, e_d
    e_w = lr * e_n + 2 * U * lr * Gn.abs() + U * ref_w.abs()
    return SLACK * e_w, (None if e_B is None else SLACK * e_B)


# ---- per-range bookkeeping and the loss scaler ----------------------------------------------------------------------------
def bias_corrections(hyper: Dict, done: int) -> Tuple[float, float]:
    """(step_size, sqrt(bias_correction2)) of step done + 1 in float64, as torch/optim/adam.py forms them from python
    floats, then cast to fp32 (what stk_optim_step_prologue stores for Adam).  The kernel must be within 1 fp32 ulp."""
    t = float(done + 1)
    bc1 = 1.0 - hyper["beta1"] ** t
    bc2 = 1.0 - hyper["beta2"] ** t
    return f32_value(hyper["lr"] / bc1), f32_value(bc2**0.5)


def update_scale(scale: float, tracker: int, found_inf: bool, growth: float, backoff: float, interval: int):
    """GradScaler.update() through torch._amp_update_scale_ on CPU tensors: (new scale, new growth tracker)."""
    s = torch.tensor([scale], dtype=torch.float32)
    gt = torch.tensor([tracker], dtype=torch.int32)
    fi = torch.tensor([1.0 if found_inf else 0.0], dtype=torch.float32)
    torch._amp_update_scale_(s, gt, fi, growth, backoff, interval)
    return float(s[0]), int(gt[0])


# ---- deliberately wrong references (negative controls: the per-element checks must reject them) ---------------------------
def adam_step_mutant(kind: str, w, m, v, g, step: int, hyper: Dict, mutation: str):
    """Adam / AdamW in float64 with one deliberate error:
      "eps_in_sqrt":      denom = sqrt(v' / bc2 + eps)
      "bc2_not_sqrt":     denom = sqrt(v') / bc2 + eps
      "decay_after":      AdamW decay applied to the updated weight instead of before the update."""
    b1, b2, eps, lr = hyper["beta1"], hyper["beta2"], hyper["eps"], hyper["lr"]
    wd = hyper.get("weight_decay", 0.0 if kind == "adam" else 1e-2)
    w, m, v, g = (x.to(F64).clone() for x in (w, m, v, g))
    if hyper.get("maximize", False):
        g = -g
    if kind == "adam" and wd != 0.0:
        g = g + wd * w
    t = step + 1
    bc1, bc2 = 1 - b1**t, 1 - b2**t
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    if mutation == "eps_in_sqrt":
        denom = (v / bc2 + eps).sqrt()
    elif mutation == "bc2_not_sqrt":
        denom = v.sqrt() / bc2 + eps
    else:
        denom = v.sqrt() / math.sqrt(bc2) + eps
    upd = (lr / bc1) * m / denom
    if kind == "adamw" and mutation == "decay_after":
        w = (w - upd) * (1 - lr * wd)
    else:
        if kind == "adamw":
            w = w * (1 - lr * wd)
        w = w - upd
    return w, m, v


def sgd_step_mutant(w, buf, g, hyper: Dict, mutation: str):
    """SGD in float64 with one deliberate error: "no_dampening" (dampening ignored) or "no_nesterov" (Nesterov off)."""
    h = dict(hyper)
    if mutation == "no_dampening":
        h["dampening"] = 0.0
    elif mutation == "no_nesterov":
        h["nesterov"] = False
    return sgd_step(w, buf, g, h)


def clip_coef_mutant(total_norm: float, max_norm: float) -> float:
    """The clip coefficient without its +1e-6."""
    return min(max_norm / total_norm, 1.0)
