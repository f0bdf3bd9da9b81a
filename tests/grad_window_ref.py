# -*- coding: utf-8 -*-
"""TEST INFRASTRUCTURE ONLY -- gradient windows that every stage of the fused gradient pipeline forms exactly.

A window is the gradient of one optimizer step split over ``micro`` micro-batches.  Every micro value is k * 2^-e with an
integer k and a per-parameter exponent e, and |k| <= KMAX // micro, so every partial sum of a window has |sum k| <= KMAX =
256.  bf16 carries 8 significant bits, so every micro value, every partial sum and the window total are exact in bf16 (and
in fp32), and stay exact when multiplied by a power-of-two loss scale (all GradScaler ever produces).  Then
x = ((g [+ acc]) * mul) * 1/scale is exact at every stage, and a fused step cannot tell an accumulated, loss-scaled window
from one bucket that already holds the sum: the two runs must be bit-identical."""
from typing import List, Sequence

import numpy as np
import torch

KMAX = 256            # |sum of k| over any prefix of a window: the largest integer range exact in bf16's 8 bits
EXPS = (10, 14)       # per-parameter exponents e (inclusive): magnitudes differ between parameters


def window(numels: Sequence[int], micro: int, seed: int, exps=EXPS) -> List[List[torch.Tensor]]:
    """Per parameter, the ``micro`` fp32 micro-batch gradients (flat, logical element order) of one window."""
    rng = np.random.default_rng(seed)
    bound = KMAX // micro
    out = []
    for n in numels:
        e = int(rng.integers(exps[0], exps[1] + 1))
        ks = rng.integers(-bound, bound + 1, size=(micro, n))
        out.append([torch.from_numpy(k.astype(np.float32)) * 2.0**-e for k in ks])
    return out


def total(micros: Sequence[torch.Tensor]) -> torch.Tensor:
    """The window sum in fp32 (exact: the float64 sum rounds to itself)."""
    s = torch.zeros_like(micros[0], dtype=torch.float64)
    for m in micros:
        s += m.double()
    return s.float()


def exact_in(x: torch.Tensor, dtype: torch.dtype) -> bool:
    """x (any float dtype) round-trips through `dtype` unchanged."""
    return bool(torch.equal(x.double().to(dtype).double(), x.double()))
