# -*- coding: utf-8 -*-
"""TEST INFRASTRUCTURE ONLY -- the quantizer of AdamW8bit at its edges: an independent nearest-code rule and crafted
gradient blocks that land on them.

``nearest_code`` is the documented rule written out by a full scan of the map, not by the class's ``searchsorted``: n is
clamped into [q[0], q[255]], every distance is one fp32 subtraction |n - q[i]|, and equal distances go to the lower
index.  ``nearest_code_upper`` breaks ties to the upper index instead; a kernel that agrees with ``nearest_code`` and not
with it on the tie elements below has been shown to apply the tie rule.

The crafted blocks each hold one element of exactly +-1.0, so their absmax is 1, 1 / absmax is 1 and n is the element
itself (for m at beta1 = 0) or its fp32 square (for v at beta2 = 0):

  qmap1_values   every entry of the signed map and its +-1 ulp neighbours, every fp32 point of a gap that is equally far
                 from both ends (an exact tie), with its +-1 and +-2 ulp neighbours, +-0, +-the smallest subnormal, -1
  qmap2_values   gradients whose fp32 squares are the unsigned map's entries, its exact ties and their +-1, +-2 ulp
                 neighbours

The subnormal-absmax blocks have absmax at or below 2 ** -128, where 1 / absmax overflows to +inf and every nonzero
element has n = +-inf (the clamp sends it to code 255 or 0), and one just above it, where 1 / absmax is finite."""
from typing import List, Tuple

import numpy as np

f32 = np.float32
BLOCK = 256
TWO_M128 = float(np.ldexp(f32(1), -128))                  # 1 / 2 ** -128 = 2 ** 128 overflows fp32
TWO_M149 = float(np.ldexp(f32(1), -149))                  # the smallest subnormal
ABOVE_M128 = float(np.ldexp(f32(1), -128) + TWO_M149)     # the next fp32 value: 1 / absmax is finite


def _as_f32(y) -> np.ndarray:
    y = np.asarray(y, dtype=np.float64)
    out = y.astype(f32)
    ok = np.isnan(y) | (out.astype(np.float64) == y)
    assert ok.all(), "nearest_code: the inputs must be fp32 values"
    return out


def _nearest(y, q, upper: bool, clamp: bool = True, chunk: int = 1 << 15) -> np.ndarray:
    q = _as_f32(q)
    assert q.size == BLOCK and (q[1:] > q[:-1]).all()
    y = _as_f32(y).ravel().copy()
    y[np.isnan(y)] = 0
    if clamp:
        y = np.clip(y, q[0], q[-1])
    out = np.empty(y.size, np.uint8)
    for s in range(0, y.size, chunk):
        with np.errstate(invalid="ignore", over="ignore"):
            d = np.abs(y[s: s + chunk, None] - q[None, :])   # fp32 subtractions
        if upper:
            out[s: s + chunk] = BLOCK - 1 - np.argmin(d[:, ::-1], axis=1)
        else:
            out[s: s + chunk] = np.argmin(d, axis=1)
    return out


def nearest_code(y, q, clamp: bool = True) -> np.ndarray:
    """The code of each n in y (float64 holding fp32 values; NaN takes the code of 0): clamp into [q[0], q[255]], then
    the map entry at the least fp32 distance, the lower index on a tie.  ``clamp=False`` is the same scan without it."""
    return _nearest(y, q, upper=False, clamp=clamp)


def nearest_code_upper(y, q) -> np.ndarray:
    """The negative control: ``nearest_code`` with ties broken to the upper index."""
    return _nearest(y, q, upper=True)


def _ulps(x: f32, k: int) -> f32:
    for _ in range(abs(k)):
        x = np.nextafter(x, f32(np.inf) if k > 0 else f32(-np.inf))
    return x


def tie_points(q) -> List[f32]:
    """Every fp32 y strictly inside a gap of q with |y - q[i]| == |y - q[i + 1]| in fp32 (near the gap's midpoint)."""
    q = _as_f32(q)
    out = []
    for a, b in zip(q[:-1], q[1:]):
        mid = f32((a + b) / f32(2))
        for k in range(-3, 4):
            y = _ulps(mid, k)
            if a < y < b and abs(f32(y - a)) == abs(f32(y - b)):
                out.append(y)
    return sorted(set(out))


def _near(points, ks) -> List[f32]:
    return [_ulps(f32(p), k) for p in points for k in ks]


def qmap1_values(q1) -> np.ndarray:
    """The signed map's crafted n values (all in [-1, 1]), sorted, without repeats."""
    q1 = _as_f32(q1)
    vals = _near(q1, (-1, 0, 1)) + _near(tie_points(q1), (-2, -1, 0, 1, 2))
    vals += [f32(TWO_M149), f32(-TWO_M149), f32(-1)]
    v = np.array(vals, f32)
    v = np.unique(v[(np.abs(v) <= 1) & (v != 0)])
    return np.concatenate([v, np.array([0.0, -0.0], f32)])   # np.unique would merge +0 and -0


def sqrt_preimage(t: f32):
    """An fp32 g >= 0 with fp32(g * g) == t, or None."""
    r = f32(np.sqrt(np.float64(t)))
    for g in (r, _ulps(r, -1), _ulps(r, 1)):
        if f32(g * g) == t:
            return g
    return None


def qmap2_values(q2) -> np.ndarray:
    """Gradients g in [0, 1] whose fp32 squares land on the unsigned map's entries, its exact ties and their +-1, +-2
    ulp neighbours."""
    q2 = _as_f32(q2)
    targets = list(q2) + _near(tie_points(q2), (-2, -1, 0, 1, 2))
    gs = [sqrt_preimage(t) for t in targets if 0 <= t <= 1]
    return np.unique(np.array([g for g in gs if g is not None], f32))


def blocks_with_unit_max(values: np.ndarray, rng: np.random.Generator, per_block: int = BLOCK - 1) -> np.ndarray:
    """values laid into whole 256-element blocks, each led by an element of exactly +1.0 or -1.0 (alternating) so its
    absmax is 1; the values' order and signs are shuffled by rng, the tail of the last block is filled with rng values in
    [-1, 1]."""
    v = np.asarray(values, f32)
    v = v[rng.permutation(v.size)]
    nb = -(-v.size // per_block)
    fill = (rng.random(nb * per_block - v.size) * 2 - 1).astype(f32)
    body = np.concatenate([v, fill]).reshape(nb, per_block)
    lead = np.where(np.arange(nb) % 2 == 0, f32(1), f32(-1)).astype(f32)[:, None]
    return np.concatenate([lead, body], axis=1).reshape(-1)


def signed_shuffle(values: np.ndarray, rng: np.random.Generator) -> np.ndarray:
    """Each value with a random sign (for gradients whose squares matter)."""
    v = np.asarray(values, f32)
    return (v * np.where(rng.random(v.size) < 0.5, f32(-1), f32(1))).astype(f32)


def subnormal_block(absmax: float) -> np.ndarray:
    """A short block whose absmax is exactly ``absmax``, with positive, negative and zero elements (a value that rounds
    to zero in fp32 is a zero element)."""
    a = f32(absmax)
    assert float(a) == absmax
    v = [a, -a, f32(0), f32(-0.0), f32(a / f32(2)), -f32(a / f32(4)), f32(a * f32(0.75)), -f32(a * f32(0.3))]
    return np.array(v, f32)


SUBNORMAL_ABSMAX = [("2^-128", TWO_M128), ("2^-128+2^-149", ABOVE_M128), ("1e-39", float(f32(1e-39))),
                    ("1e-43", float(f32(1e-43))), ("2^-149", TWO_M149)]


def v_subnormal_grads(scale: float) -> np.ndarray:
    """Gradients near ``scale`` (4e-20 at beta2 = 0, 1e-18 at the default beta2) whose v = (g * g) * (1 - beta2) is a
    nonzero subnormal at or below 2 ** -128, with zeros among them."""
    s = f32(scale)
    return np.array([s, -s, f32(0), f32(s * f32(0.5)), -f32(s * f32(0.7)), f32(s * f32(0.25)), f32(-0.0)], f32)


def overflows(absmax) -> np.ndarray:
    """Where fp32 1 / absmax (absmax > 0) is +inf."""
    a = np.asarray(absmax, f32)
    with np.errstate(divide="ignore", over="ignore"):
        return (a > 0) & np.isinf(f32(1) / a)


def n_of(x: np.ndarray, absmax: f32) -> np.ndarray:
    """n = x * (absmax == 0 ? 0 : fp32(1 / absmax)) for one block, NaN kept (``nearest_code`` maps it to 0)."""
    a = f32(absmax)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        inv = f32(0) if a == 0 else f32(f32(1) / a)
        return (np.asarray(x, f32) * inv).astype(f32)


def block_codes(x: np.ndarray, q) -> Tuple[np.ndarray, np.ndarray]:
    """(codes, absmax) of a 1-D fp32 array under ``nearest_code``: block-wise absmax (NaN if the block holds one)."""
    x = np.asarray(x, f32)
    nb = -(-x.size // BLOCK)
    codes, absmax = np.zeros(x.size, np.uint8), np.zeros(nb, f32)
    for b in range(nb):
        blk = x[BLOCK * b: BLOCK * (b + 1)]
        a = f32(np.nan) if np.isnan(blk).any() else f32(np.max(np.abs(blk)))
        absmax[b] = a
        codes[BLOCK * b: BLOCK * (b + 1)] = nearest_code(n_of(blk, a), q)
    return codes, absmax
