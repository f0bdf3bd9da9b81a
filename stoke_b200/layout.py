# -*- coding: utf-8 -*-
"""Pure-Python planning of the flat-buffer layout (no CUDA, no torch): parameter offsets, gradient buckets in reverse
registration order (torch DDP's bucket order, torch/nn/parallel/distributed.py; size = DDPConfig.bucket_cap_mb,
/root/reference/stoke/configs.py:178-188), the per-bucket partition over the ranks and every rank's segment table (its
shard of each bucket, concatenated by ascending element offset = the layout of the sharded optimizer state).

Kept separate from ``engine.GradPath`` so that the partition logic -- which must be identical on every rank, or the block
barriers of the cross-rank kernels pair the wrong blocks -- is unit-tested on CPU (tests/test_layout.py)."""
from typing import Callable, List, Sequence, Tuple

ALIGN_ELEMS = 16   # every parameter starts on a 16-element boundary (32 B of bf16 / 64 B of fp32)
MAX_SEGMENTS = 64  # STK_MAX_SEGMENTS of the C ABI

Segment = Tuple[int, int, int, int]  # (global begin, global end, local begin, bucket index)


def shard_range(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Python twin of ``stk_shard_range`` (ctx.cu): shards are multiples of 16 elements; the last may be short or empty."""
    vecs = (n + 7) // 8
    per = (vecs + world - 1) // world
    per += per & 1
    b, e = per * rank * 8, per * (rank + 1) * 8
    return min(b, n), min(e, n)


def param_offsets(numels: Sequence[int]) -> Tuple[List[int], List[int], int]:
    """(offset per parameter, padded size per parameter, padded total)."""
    offsets, padded, off = [], [], 0
    for k in numels:
        offsets.append(off)
        pk = (k + ALIGN_ELEMS - 1) // ALIGN_ELEMS * ALIGN_ELEMS
        padded.append(pk)
        off += pk
    return offsets, padded, off


def plan_buckets(offsets: Sequence[int], n: int, cap_elems: int) -> List[Tuple[int, int]]:
    """Contiguous element ranges cut at parameter boundaries, in LAUNCH order: bucket 0 holds the last parameters (their
    gradients arrive first).  A bucket is closed as soon as it holds at least ``cap_elems`` elements."""
    buckets, hi = [], n
    for i in range(len(offsets) - 1, -1, -1):
        if hi - offsets[i] >= cap_elems or i == 0:
            buckets.append((offsets[i], hi))
            hi = offsets[i]
    if len(buckets) > MAX_SEGMENTS:  # keep the segment table bounded: merge the tail buckets
        keep = buckets[: MAX_SEGMENTS - 1]
        buckets = keep + [(0, keep[-1][0])]
    return buckets


def plan_segments(buckets: Sequence[Tuple[int, int]], world: int, sharded: bool,
                  shard_fn: Callable[[int, int, int], Tuple[int, int]] = shard_range):
    """(segments per rank, local element count per rank).  Unsharded: one segment covering everything on every rank."""
    if not sharded:
        n = max(b1 for _, b1 in buckets)
        return [[(0, n, 0, 0)] for _ in range(world)], [n] * world
    segs_by_rank, n_local = [], []
    order = sorted(range(len(buckets)), key=lambda k: buckets[k][0])
    for r in range(world):
        out, lo = [], 0
        for k in order:
            b0, b1 = buckets[k]
            sb, se = shard_fn(b1 - b0, world, r)
            if se > sb:
                out.append((b0 + sb, b0 + se, lo, k))
                lo += se - sb
        segs_by_rank.append(out)
        n_local.append(lo)
    return segs_by_rank, n_local


ADAFACTOR_MAX_DIM = 4  # stk_adafactor_param_t carries four logical dims; a larger parameter keeps the stock route


def adafactor_layout(shape: Sequence[int], stride: Sequence[int]) -> dict:
    """How the fused Adafactor step sees one parameter of logical ``shape`` laid out with element ``stride``:
    ``factored`` (dim >= 2: torch factors g^2 over the last two dims, leading dims are a batch), the sizes and strides
    left-padded with 1 to four dims (B0, B1, R, C), and ``state``, the fp32 elements of its state (row_var [..., R, 1] then
    col_var [..., 1, C]; or variance, one per element).  Raises ValueError for more than four dims or a layout that is not
    dense (overlapping or with holes)."""
    shape, stride = [int(s) for s in shape], [int(s) for s in stride]
    if len(shape) > ADAFACTOR_MAX_DIM:
        raise ValueError(f"Stoke -- fused Adafactor handles parameters of up to {ADAFACTOR_MAX_DIM} dims, got {len(shape)}")
    numel = 1
    for s in shape:
        numel *= s
    expect = 1
    for s, st in sorted(((s, st) for s, st in zip(shape, stride) if s != 1), key=lambda x: x[1]):
        if st != expect:
            raise ValueError("Stoke -- fused Adafactor needs dense parameters")
        expect *= s
    pad = ADAFACTOR_MAX_DIM - len(shape)
    size4 = [1] * pad + shape
    stride4 = [numel] * pad + stride
    factored = len(shape) >= 2
    B, R, C = size4[0] * size4[1], size4[2], size4[3]
    return {"factored": factored, "size": size4, "stride": stride4, "numel": numel, "B": B, "R": R, "C": C,
            "state": B * R + B * C if factored else numel}
