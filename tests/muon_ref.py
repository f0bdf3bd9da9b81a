"""Float64 references for the Muon step (torch.optim.Muon, MuonWithAuxAdamW): an independent transcription of one step
in float64 (momentum as mu buf + (1 - mu) g, Newton-Schulz without bf16 rounding), the Newton-Schulz iteration alone
on a given input, the matrix view of a parameter, the descriptor table of the fused step and the algorithmic FLOPs."""
import math

import torch

COEFFS = (3.4445, -4.7750, 2.0315)


def ns64(x: torch.Tensor, coeffs=COEFFS, steps: int = 5) -> torch.Tensor:
    """``steps`` Newton-Schulz iterations in float64 on x (r x c, r <= c), as given: no normalisation, no rounding."""
    a, b, c = coeffs
    x = x.double()
    for _ in range(steps):
        gram = x @ x.T
        x = a * x + (b * gram + c * gram @ gram) @ x
    return x


def orthogonalize64(u: torch.Tensor, coeffs=COEFFS, steps: int = 5, eps: float = 1e-7) -> torch.Tensor:
    """Muon's orthogonalisation of an R x C matrix in float64: transposed when R > C, divided by max(||u||, eps), then
    ``ns64``, transposed back."""
    x = u.double()
    tall = x.shape[0] > x.shape[1]
    if tall:
        x = x.T
    x = x / max(float(x.norm()), eps)
    x = ns64(x, coeffs, steps)
    return x.T if tall else x


def lr_ratio(adjust_lr_fn, rows: int, cols: int) -> float:
    if adjust_lr_fn in (None, "original"):
        return max(1.0, rows / cols) ** 0.5
    return 0.2 * max(rows, cols) ** 0.5


def muon_step64(w, buf, g, group):
    """One Muon step of a parameter of 2 or more dims in float64: returns (w, buf) in the parameter's shape."""
    rows = w.shape[0]
    w2, g2, b2 = (t.double().reshape(rows, -1) for t in (w, g, buf))
    mu = group["momentum"]
    b2 = mu * b2 + (1 - mu) * g2
    u = mu * b2 + (1 - mu) * g2 if group["nesterov"] else b2
    x = orthogonalize64(u, group["ns_coefficients"], group["ns_steps"], group["eps"])
    lr = group["lr"]
    w2 = w2 * (1 - lr * group["weight_decay"]) - lr * lr_ratio(group["adjust_lr_fn"], *w2.shape) * x
    return w2.reshape(w.shape), b2.reshape(w.shape)


def adamw_step64(w, m, v, g, t, group):
    """One AdamW step in float64 at step count t (after the increment)."""
    b1, b2 = group["betas"]
    lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
    w, m, v, g = (x.double() for x in (w, m, v, g))
    w = w * (1 - lr * wd)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    w = w - lr / (1 - b1 ** t) * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + eps)
    return w, m, v


def plan(shapes):
    """The descriptor table of the fused step for these (rows, cols) matrices (None: not a Muon parameter), every
    parameter at a 16-element aligned offset: list of dicts with the keys of ``layout.muon_plan``."""
    out, off, x = [], 0, 0
    a = tiles = tri = full = 0
    for i, s in enumerate(shapes):
        if s is not None:
            r, c = sorted(s)
            t = math.ceil(r / 64)
            out.append(dict(param=i, offset=off, rows=r, cols=c, transposed=s[0] > s[1], x_offset=x, a_offset=a,
                            tile0=tiles, tri0=tri, full0=full))
            x += math.ceil(r * c / 8) * 8
            a += math.ceil(r * r / 8) * 8
            tiles += math.ceil(r * c / 8192)
            tri += sum(range(1, t + 1))
            full += t * math.ceil(c / 64)
        numel = 1 if s is None else s[0] * s[1]
        off += math.ceil(numel / 16) * 16
    return out


def ns_flops(rows: int, cols: int, steps: int) -> int:
    """Algorithmic FLOPs of Newton-Schulz on one matrix: per step X X^T (2 r^2 c), A A (2 r^3), B X (2 r^2 c)."""
    r, c = min(rows, cols), max(rows, cols)
    return steps * (4 * r * r * c + 2 * r ** 3)
