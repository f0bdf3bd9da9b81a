# -*- coding: utf-8 -*-
"""TEST INFRASTRUCTURE ONLY -- references of the fused step's Adadelta, Rprop and ASGD kinds.

Adadelta and ASGD: float64 values from ``torch.optim.Adadelta`` / ``ASGD`` themselves, run on float64 tensors with the
kernel's pre-step state loaded (``step`` and, for ASGD, the stored fp32 ``eta`` / ``mu``), and per-element fp32 error bounds
in the style of oracle/kernel_ref.py (same u, SLACK and conventions: every fp32 operation, and every cast of a float64
scalar to fp32, contributes one u of its result; a fused multiply-add only removes roundings; input errors are propagated to
first order).  Each bound covers both the kernel's order of operations and torch's own fp32 single-tensor order.

Rprop: torch's fp32 single-tensor Rprop itself.  Its update is a chain of sign decisions, a clamp and one subtraction, so
given the same fp32 gradient an fp32 implementation reproduces it exactly: the reference is bit-exact, not a bound.

ASGD's per-parameter scalars follow torch's python-double formulas, stored as fp32 (``asgd_next``).
"""
from typing import Dict, Optional, Tuple

import torch

from kernel_ref import SLACK, U

F64, F32 = torch.float64, torch.float32
KINDS = ("adadelta", "rprop", "asgd")
STATE_KEYS = {"adadelta": ("square_avg", "acc_delta"), "rprop": ("prev", "step_size"), "asgd": ("ax",)}


def _wd(h: Dict) -> float:
    return float(h.get("weight_decay", 0.0))


def make_optimizer(kind: str, params, h: Dict):
    """torch's single-tensor implementation (foreach=False) of `kind` with the hyper-parameters of `h`.  Rprop's etas are
    set on the group after construction, so that the values the constructor refuses (etaminus = 1, etaplus = etaminus) can
    be tested: torch's update itself takes them."""
    mx = bool(h.get("maximize", False))
    if kind == "adadelta":
        return torch.optim.Adadelta(params, lr=h["lr"], rho=h["rho"], eps=h["eps"], weight_decay=_wd(h), maximize=mx,
                                    foreach=False)
    if kind == "rprop":
        opt = torch.optim.Rprop(params, lr=h["lr"], step_sizes=tuple(h["step_sizes"]), maximize=mx, foreach=False)
        for g in opt.param_groups:
            g["etas"] = tuple(h["etas"])
        return opt
    return torch.optim.ASGD(params, lr=h["lr"], lambd=h["lambd"], alpha=h["alpha"], t0=h["t0"], weight_decay=_wd(h),
                            maximize=mx, foreach=False)


def _load(opt, p, kind: str, step: int, m, v, eta, mu, dtype):
    """The kernel's pre-step state as torch's; nothing at step 0 (torch initialises the state lazily at the first step)."""
    if step == 0:
        return
    st = {"step": torch.tensor(float(step), dtype=F32), STATE_KEYS[kind][0]: m.to(dtype).clone()}
    if kind != "asgd":
        st[STATE_KEYS[kind][1]] = v.to(dtype).clone()
    else:
        st["eta"] = torch.tensor(float(eta), dtype=dtype)
        st["mu"] = torch.tensor(float(mu), dtype=dtype)
    opt.state[p] = st


def torch_step(kind: str, w, m, v, g, step: int, h: Dict, eta: Optional[float] = None, mu: Optional[float] = None,
               dtype=F64):
    """One torch step in `dtype` from the given state; `step` = steps already taken.  Returns (w, m, v or None,
    eta or None, mu or None) after the step (ASGD's eta / mu as python floats of torch's tensors)."""
    p = torch.nn.Parameter(w.to(dtype).clone())
    opt = make_optimizer(kind, [p], h)
    _load(opt, p, kind, step, m, v, eta, mu, dtype)
    p.grad = g.to(dtype).clone()
    opt.step()
    st = opt.state[p]
    k = STATE_KEYS[kind]
    nv = st[k[1]] if len(k) > 1 else None
    if kind == "asgd":
        return p.detach(), st["ax"], None, float(st["eta"]), float(st["mu"])
    return p.detach(), st[k[0]], nv, None, None


# ---- ASGD's per-parameter scalars (python doubles in torch's single-tensor step, stored in fp32 tensors) ------------------
def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=F32))


def asgd_next(h: Dict, t: int) -> Tuple[float, float]:
    """(eta, mu) torch stores after step t: lr / (1 + lambd lr t)^alpha and 1 / max(1, t - t0), each as fp32."""
    lr = h["lr"]
    return _f32(lr / ((1 + h["lambd"] * lr * float(t)) ** h["alpha"])), _f32(1 / max(1, float(t) - h["t0"]))


def asgd_used(h: Dict, done: int, eta: Optional[float], mu: Optional[float]) -> Tuple[float, float]:
    """The (eta, mu) step done + 1 uses: the stored values, or torch's initial (fp32(lr), 1) at the first step."""
    return (_f32(h["lr"]), 1.0) if done == 0 else (float(eta), float(mu))


def asgd_handoff(h: Dict, done: int, eta: Optional[float], mu: Optional[float]) -> Tuple[float, float, float, float]:
    """The float4 stk_optim_step_prologue hands the ASGD step: {-eta, fp32(1 - lambd eta), mu, 0}."""
    eta, mu = asgd_used(h, done, eta, mu)
    return -eta, _f32(1.0 - h["lambd"] * eta), mu, 0.0


# ---- bounds (Adadelta, ASGD) ----------------------------------------------------------------------------------------------
def _decay(G, e_g, w, h):
    wd = _wd(h)
    if wd == 0.0:
        return G, e_g
    Gd = G + wd * w
    return Gd, e_g + U * (2 * (wd * w).abs() + Gd.abs())


def step_bound(kind: str, w, m, v, G, e_g, h: Dict, ref_w, ref_m, ref_v=None, eta: Optional[float] = None,
               mu: Optional[float] = None):
    """Per-element bounds (e_w, e_m, e_v or None) of an fp32 Adadelta / ASGD step.  w, m, v: the pre-step fp32 state
    (exact); G: the reference gradient after clipping (float64; maximize is applied here), e_g its bound; ref_*: the
    reference's new state; eta, mu: ASGD's stored fp32 scalars (the values the step uses).

    Adadelta (m = square_avg, v = acc_delta):
      L2 decay Gd = G + wd w:                  e_d = e_g + u (2 |wd w| + |Gd|)
      s' = rho s + (1 - rho) Gd^2:             e_s = 2u rho s + 2 (1-rho) |Gd| e_d + 3u (1-rho) Gd^2 + u s'     (as Adam's v)
      A = sqrt(a + eps):                       e_A = (u eps + u (a + eps)) / (2A) + u A          (cast of eps, sum, sqrt)
      S = sqrt(s' + eps):                      e_S = (e_s + u eps + u (s' + eps)) / (2S) + u S
      q = A / S, delta = q Gd:                 e_q = (e_A + q e_S) / S + u q;  e_delta = |Gd| e_q + q e_d + u |delta|
      a' = rho a + (1 - rho) delta^2:          e_a = 2u rho a + 2 (1-rho) |delta| e_delta + 3u (1-rho) delta^2 + u a'
      w' = w - lr delta:                       e_w = lr e_delta + 2u lr |delta| + u |w'|   (cast of lr or torch's product)
    ASGD (m = ax), c = fp32(1 - lambd eta):
      w1 = c w:                                e_w1 = 2u |w1|                                    (cast, product)
      w' = w1 - eta Gd:                        e_w = e_w1 + eta e_d + u eta |Gd| + u |w'|        (torch's product, sum)
      mu == 1: ax' = w' (a copy):              e_ax = e_w
      else ax' = ax + (w' - ax) mu:            e_ax = mu (e_w + u |w' - ax|) + u |(w' - ax) mu| + u |ax'|
    """
    w, m, G, e_g, ref_w, ref_m = (x.to(F64) for x in (w, m, G, e_g, ref_w, ref_m))
    if h.get("maximize", False):
        G = -G
    Gd, e_d = _decay(G, e_g, w, h)
    if kind == "adadelta":
        v, ref_v = v.to(F64), ref_v.to(F64)
        rho, eps, lr = h["rho"], h["eps"], h["lr"]
        e_s = 2 * U * rho * m + 2 * (1 - rho) * Gd.abs() * e_d + 3 * U * (1 - rho) * Gd * Gd + U * ref_m
        A = (v + eps).sqrt()
        e_A = (U * eps + U * (v + eps)) / (2 * A) + U * A
        S = (ref_m + eps).sqrt()
        e_S = (e_s + U * eps + U * (ref_m + eps)) / (2 * S) + U * S
        q = A / S
        e_q = (e_A + q * e_S) / S + U * q
        delta = q * Gd
        e_delta = Gd.abs() * e_q + q * e_d + U * delta.abs()
        e_a = 2 * U * rho * v + 2 * (1 - rho) * delta.abs() * e_delta + 3 * U * (1 - rho) * delta * delta + U * ref_v
        e_w = lr * e_delta + 2 * U * lr * delta.abs() + U * ref_w.abs()
        return SLACK * e_w, SLACK * e_s, SLACK * e_a
    # ASGD
    eta, mu = float(eta), float(mu)
    c = 1.0 - h["lambd"] * eta
    w1 = c * w
    e_w = 2 * U * w1.abs() + eta * e_d + U * eta * Gd.abs() + U * ref_w.abs()
    if mu == 1.0:
        e_ax = e_w
    else:
        d = ref_w - m
        e_ax = mu * (e_w + U * d.abs()) + U * (d * mu).abs() + U * ref_m.abs()
    return SLACK * e_w, SLACK * e_ax, None


# ---- Rprop, exact in fp32 ---------------------------------------------------------------------------------------------------
def rprop_fp32(w, prev, ss, g, step: int, h: Dict):
    """torch's fp32 single-tensor Rprop from the given state: (w, prev, step_size) after the step."""
    nw, nprev, nss, _, _ = torch_step("rprop", w, prev, ss, g, step, h, dtype=F32)
    return nw, nprev, nss


# ---- deliberately wrong references (negative controls) ---------------------------------------------------------------------
MUTATIONS = {
    "adadelta": ("eps_outside_sqrt",),
    "rprop": ("no_mask_quirk", "sign_per_factor"),
    "asgd": ("current_eta", "always_average", "never_average"),
}


def step_mutant(kind: str, w, m, v, g, step: int, h: Dict, mutation: str, eta: Optional[float] = None,
                mu: Optional[float] = None):
    """The state after one step of `kind` with one deliberate error: (w, m, v or None).
      Adadelta "eps_outside_sqrt": delta = (sqrt(a) + eps) / (sqrt(s') + eps) g
      Rprop    "no_mask_quirk":    the gradient zeroed where the product's sign is negative, not where the factor equals
                                   etaminus (misses the etaminus == 1 and etaplus == etaminus cases)
               "sign_per_factor":  sign(g) sign(prev) instead of the sign of the fp32 product (misses its underflow to 0)
      ASGD     "current_eta":      the update with this step's eta instead of the stored one
               "always_average":   ax averaged from the first step with mu = 1 / t, ignoring t0
               "never_average":    ax = w even when mu != 1
    Adadelta and ASGD in float64; Rprop in fp32 (compared bit for bit)."""
    if kind == "rprop":
        w, prev, ss, g = (x.to(F32).clone() for x in (w, m, v, g))
        if h.get("maximize", False):
            g = -g
        if step == 0:
            prev, ss = torch.zeros_like(w), torch.full_like(w, _f32(h["lr"]))
        etaminus, etaplus = (_f32(e) for e in h["etas"])
        s = g.sign() * prev.sign() if mutation == "sign_per_factor" else (g * prev).sign()
        f = torch.where(s > 0, torch.tensor(etaplus), torch.where(s < 0, torch.tensor(etaminus), torch.tensor(1.0)))
        ss = (ss * f).clamp(h["step_sizes"][0], h["step_sizes"][1])
        mask = s < 0 if mutation == "no_mask_quirk" else f == etaminus
        g = torch.where(mask, torch.zeros_like(g), g)
        return w - g.sign() * ss, g, ss
    w, m, g = (x.to(F64).clone() for x in (w, m, g))
    if h.get("maximize", False):
        g = -g
    wd = _wd(h)
    if wd != 0.0:
        g = g + wd * w
    if kind == "adadelta":
        v = v.to(F64).clone()
        rho, eps, lr = h["rho"], h["eps"], h["lr"]
        s = rho * m + (1 - rho) * g * g
        delta = (v.sqrt() + eps) / (s.sqrt() + eps) * g
        return w - lr * delta, s, rho * v + (1 - rho) * delta * delta
    t = step + 1
    eta, mu = asgd_used(h, step, eta, mu)
    e = asgd_next(h, t)[0] if mutation == "current_eta" else eta
    w = w * (1 - h["lambd"] * e) - e * g
    if mutation == "always_average":
        mu = 1.0 / t
    if mutation == "never_average" or mu == 1.0:
        ax = w.clone()
    else:
        ax = m + (w - m) * mu
    return w, ax, None
