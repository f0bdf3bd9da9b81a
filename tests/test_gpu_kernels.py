"""The single-GPU gradient kernels, called directly through the C ABI and compared element by element with the float64
reference of oracle/kernel_ref.py (torch's own ops in float64, per-element fp32 error bounds derived there).

Every buffer sits inside a guard band of 0xFF bytes (a NaN in every float type) and is passed at a non-zero offset, so a
kernel that writes outside its range, or mixes global (flat-bucket) and local (shard) indices, fails here.  Each family
also carries a negative control: a deliberately wrong reference must fail the same per-element check, which shows the
check is sharp enough to catch that mistake in a kernel.
"""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch

import kernel_ref as kr

pytestmark = pytest.mark.gpu

GUARD = 4096  # bytes of 0xFF before and after every buffer
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
INT_VIEW = {F32: torch.int32, BF16: torch.int16, F16: torch.int16}


def _lib():
    from stoke_b200 import _lib

    return _lib


def _dt(dtype):
    L = _lib()
    return {F32: L.F32, BF16: L.BF16, F16: L.F16}[dtype]


def _norm_kind(p):
    L = _lib()
    if math.isinf(p):
        return L.NORM_INF
    return L.NORM_L2 if p == 2.0 else L.NORM_P


class Buf:
    """n elements of `dtype` inside GUARD bytes of 0xFF on each side."""

    def __init__(self, n, dtype, init=None):
        self.esz = torch.tensor([], dtype=dtype).element_size()
        self.n, self.dtype = n, dtype
        self.raw = torch.full((2 * GUARD + n * self.esz,), 0xFF, dtype=torch.uint8, device="cuda")
        self.t = self.raw[GUARD:GUARD + n * self.esz].view(dtype)
        if init is not None:
            self.t.copy_(init)

    def ptr(self, off=0):   # from the raw buffer: torch reports a null data_ptr for an empty view
        return self.raw.data_ptr() + GUARD + off * self.esz

    def bits(self):
        return self.t.view(INT_VIEW[self.dtype]).cpu()

    def check_guards(self):
        assert bool((self.raw[:GUARD] == 0xFF).all()) and bool((self.raw[-GUARD:] == 0xFF).all()), "guard band written"

    def check_unchanged_except(self, before_bits, changed):
        """Every element outside the boolean mask `changed` is bit-identical to `before_bits`; guards intact."""
        self.check_guards()
        keep = ~torch.as_tensor(changed, dtype=torch.bool)
        assert torch.equal(self.bits()[keep], before_bits[keep]), "an element outside the intended range changed"


def _rand(n, dtype, scale=1e-3, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g) * scale).to(dtype)


@pytest.fixture
def eng():
    from stoke_b200.engine import get_engine

    torch.cuda.set_device(0)
    e = get_engine(0)
    sid = e.state_create()
    e.state_select(sid)
    yield e
    torch.cuda.synchronize()
    e.state_destroy(sid)


# ---- 1. stk_grad_norm ----------------------------------------------------------------------------------------------------
NORM_CASES = [  # n, grad dtype, accumulator, mul, norm p, loss scale (None: no UNSCALE)
    (8, F32, False, 1.0, 2.0, None),
    (8, BF16, True, 0.5, math.inf, None),
    (16_376, BF16, False, 1.0, 2.0, 2.0**16),
    (16_376, F16, True, 1.0, 1.0, None),
    (16_384, F32, True, 0.25, 2.0, 2.0**-3),
    (16_384, BF16, False, 1.0, 1.5, None),
    (16_384, F16, False, 0.5, 2.0, 1.0),
    (16_392, BF16, True, 1.0, 3.0, 2.0**16),
    (16_392, F16, False, 1.0, math.inf, 2.0**-3),
    (16_392, F32, False, 1.0, 1.5, None),
    (16_777_224, BF16, False, 1.0, 2.0, None),          # 1025 blocks: the finisher's threads fold two partials
    (16_777_224, F32, True, 0.5, math.inf, 2.0**16),
]


@pytest.mark.parametrize("n,dtype,has_acc,mul,p,scale", NORM_CASES)
def test_grad_norm_matches_float64(eng, n, dtype, has_acc, mul, p, scale):
    L = _lib()
    off = 24
    g = _rand(n, dtype, scale=1e-3 * (scale or 1.0), seed=n)
    a = _rand(n, F32, scale=1e-3 * (scale or 1.0), seed=n + 1) if has_acc else None
    G = Buf(off + n + 40, dtype)
    G.t[off:off + n] = g.cuda()
    A = Buf(off + n + 40, F32) if has_acc else None
    if has_acc:
        A.t[off:off + n] = a.cuda()
    if scale is not None:
        eng.scaler_set(scale=scale, enabled=1)
    before = G.bits()
    flags = L.RF_FINAL | (L.RF_UNSCALE if scale is not None else 0)
    eng.grad_norm(G.ptr(off), dtype, A.ptr(off) if has_acc else None, n, mul, _norm_kind(p), p, flags)
    st = eng.scaler_get()
    x, e_x = kr.scaled_grad(g, a, mul, kr.inv_scale_f32(scale or 1.0))
    ref = kr.norm_ref(x, p)
    bound = kr.norm_bound(x, e_x, p, kr.depth_norm_pass(n))
    assert abs(st.grad_norm - ref) <= bound, (st.grad_norm, ref, bound)
    assert st.found_inf == 0
    G.check_unchanged_except(before, torch.zeros(G.n, dtype=torch.bool))
    if has_acc:
        A.check_guards()
    # negative control: the norm of the wrong kind (or of the input without the unscale) is outside the bound
    wrong = kr.norm_ref(x, 2.0 if p != 2.0 else math.inf)
    assert abs(st.grad_norm - wrong) > bound


def test_grad_norm_over_several_calls_and_empty(eng):
    """Three calls with FINAL only on the last give the norm of the whole buffer; n = 0 contributes nothing."""
    L = _lib()
    n = 3 * 16_392
    g = _rand(n, BF16, seed=7)
    G = Buf(n, BF16, g.cuda())
    for p in (2.0, math.inf, 3.0):
        cuts = [0, 16_392, 16_392, 2 * 16_392 + 8, n]
        for k in range(len(cuts) - 1):
            final = L.RF_FINAL if k == len(cuts) - 2 else 0
            eng.grad_norm(G.ptr(cuts[k]), BF16, None, cuts[k + 1] - cuts[k], 1.0, _norm_kind(p), p, final)
        st = eng.scaler_get()
        x, e_x = kr.scaled_grad(g, None, 1.0, 1.0)
        assert abs(st.grad_norm - kr.norm_ref(x, p)) <= kr.norm_bound(x, e_x, p, kr.depth_norm_pass(n, calls=4))
    eng.grad_norm(G.ptr(), BF16, None, 0, 1.0, L.NORM_L2, 2.0, L.RF_FINAL)
    st = eng.scaler_get()
    assert st.grad_norm == 0.0 and st.found_inf == 0


@pytest.mark.parametrize("p", [2.0, math.inf, 1.5])
@pytest.mark.parametrize("bad", ["nan", "inf"])
def test_grad_norm_nonfinite_follows_torch(eng, p, bad):
    """Without a loss scaler the total norm is what clip_grad_norm_ returns (NaN if any element is NaN, else inf) and
    found_inf stays 0 (no scaler, no skip); with UNSCALE found_inf is raised."""
    L = _lib()
    n = 3 * 16_384
    g = _rand(n, BF16, seed=3)
    g[40_000] = float(bad)
    G = Buf(n, BF16, g.cuda())
    eng.grad_norm(G.ptr(), BF16, None, n, 1.0, _norm_kind(p), p, L.RF_FINAL)
    st = eng.scaler_get()
    ref = kr.norm_ref(g, p)
    assert (math.isnan(st.grad_norm) and math.isnan(ref)) or st.grad_norm == ref == math.inf
    assert st.found_inf == 0
    eng.grad_norm(G.ptr(), BF16, None, n, 1.0, _norm_kind(p), p, L.RF_FINAL | L.RF_UNSCALE)
    assert eng.scaler_get().found_inf == 1


# ---- 2. stk_grad_reduce at world 1 (the main route) ----------------------------------------------------------------------
REDUCE_CASES = [  # n, in dtype, out dtype, accumulator, zero input, norm p, loss scale, buckets
    (4_088, F32, F32, False, True, 2.0, None, 1),
    (4_096, BF16, F32, True, True, math.inf, 2.0**16, 1),
    (4_104, F16, F32, False, False, 1.5, None, 1),
    (4_096, F32, BF16, True, False, 2.0, 2.0**-3, 1),
    (4_104, BF16, BF16, False, True, 3.0, None, 1),
    (262_136, BF16, F32, False, True, 2.0, None, 3),
    (262_152, F32, BF16, False, True, math.inf, None, 2),
    (262_152, F16, F32, True, True, 1.0, 2.0**16, 1),
    (25_557_040, BF16, F32, False, True, 2.0, None, 1),   # 6240 blocks: every finisher thread folds several partials
    (4_194_304, BF16, F32, False, True, 2.0, None, 1),    # 1024 blocks: one partial per finisher thread
    (4_194_312, BF16, F32, False, True, 2.0, None, 1),    # 1025 blocks: the finisher's thread 0 folds two partials
]


@pytest.mark.parametrize("n,din,dout,has_acc,zero_in,p,scale,buckets", REDUCE_CASES)
def test_grad_reduce_w1_matches_float32_ops(eng, n, din, dout, has_acc, zero_in, p, scale, buckets):
    """main = ((g [+ acc]) * mul) * inv_scale: bit-identical to the same fp32 ops in torch (a bf16 output is their RNE
    rounding); the norm within its float64 bound; the input zeroed exactly on its range when asked."""
    L = _lib()
    off = 16
    mul = 0.5
    g = _rand(n, din, scale=1e-3 * (scale or 1.0), seed=n)
    a = _rand(n, F32, scale=1e-3 * (scale or 1.0), seed=n + 5) if has_acc else None
    G = Buf(off + n + 32, din)
    G.t[off:off + n] = g.cuda()
    A = Buf(off + n + 32, F32) if has_acc else None
    if has_acc:
        A.t[off:off + n] = a.cuda()
    O = Buf(off + n + 32, dout, torch.full((off + n + 32,), 7.0, dtype=dout))
    if scale is not None:
        eng.scaler_set(scale=scale, enabled=1)
    bg, bo = G.bits(), O.bits()
    ba = A.bits() if has_acc else None
    cuts = [round(n * k / buckets / 8) * 8 for k in range(buckets)] + [n]
    flags0 = (L.RF_ZERO_INPUT if zero_in else 0) | (L.RF_UNSCALE if scale is not None else 0)
    for k in range(buckets):
        b0, b1 = cuts[k], cuts[k + 1]
        fl = flags0 | (L.RF_FINAL if k == buckets - 1 else 0)
        eng.grad_reduce(L.REDUCE_ALL, [G.ptr(off + b0)], din, [A.ptr(off + b0)] if has_acc else None, [O.ptr(off + b0)],
                        dout, b1 - b0, mul, _norm_kind(p), p, fl)
    inv = kr.inv_scale_f32(scale or 1.0)
    want = kr.scaled_grad_f32(g, a, mul, inv)
    got = O.t[off:off + n].cpu()
    assert torch.equal(got.view(INT_VIEW[dout]), want.to(dout).view(INT_VIEW[dout]))
    rng = torch.zeros(O.n, dtype=torch.bool)
    rng[off:off + n] = True
    O.check_unchanged_except(bo, rng)
    if zero_in:
        assert float(G.t[off:off + n].float().abs().max()) == 0.0
        G.check_unchanged_except(bg, rng)
    else:
        G.check_unchanged_except(bg, torch.zeros(G.n, dtype=torch.bool))
    if has_acc:   # the accumulator is left alone (the next first-micro-step accumulate overwrites it)
        A.check_unchanged_except(ba, torch.zeros(A.n, dtype=torch.bool))
    st = eng.scaler_get()
    x, e_x = kr.scaled_grad(g, a, mul, inv)
    bound = kr.norm_bound(x, e_x, p, kr.depth_reduce_w1(n // buckets + 8, calls=buckets) + buckets)
    assert abs(st.grad_norm - kr.norm_ref(x, p)) <= bound
    assert st.found_inf == 0
    # negative control: the output without the unscale / mul would not match
    assert not torch.equal(got.float(), kr.scaled_grad_f32(g, a, 1.0, 1.0).to(dout).float())


def test_grad_reduce_rejects_f16_to_bf16(eng):
    L = _lib()
    G, O = Buf(64, F16), Buf(64, BF16)
    with pytest.raises(Exception):
        eng.grad_reduce(L.REDUCE_ALL, [G.ptr()], F16, None, [O.ptr()], BF16, 64, 1.0, L.NORM_L2, 2.0, L.RF_FINAL)


# ---- 3. stk_grad_accumulate and stk_grad_scale ---------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 2_040, 2_048, 2_056])
@pytest.mark.parametrize("dtype", [F32, BF16, F16])
def test_grad_accumulate_bitwise(eng, n, dtype):
    off = 8
    g = _rand(n, dtype, seed=n + 11)
    a0 = _rand(n, F32, seed=n + 12)
    for first, zero in ((True, False), (False, True)):
        G = Buf(off + n + 8, dtype)
        G.t[off:off + n] = g.cuda()
        A = Buf(off + n + 8, F32)
        A.t[off:off + n] = a0.cuda()
        bg, ba = G.bits(), A.bits()
        eng.grad_accumulate(G.ptr(off), dtype, A.ptr(off), n, first, zero)
        want = g.float() if first else a0 + g.float()
        assert torch.equal(A.t[off:off + n].cpu().view(torch.int32), want.view(torch.int32))
        rng = torch.zeros(A.n, dtype=torch.bool)
        rng[off:off + n] = True
        A.check_unchanged_except(ba, rng)
        G.check_unchanged_except(bg, rng if zero else torch.zeros(G.n, dtype=torch.bool))
        if zero:
            assert n == 0 or float(G.t[off:off + n].float().abs().max()) == 0.0


@pytest.mark.parametrize("n", [2_040, 2_048, 2_056])
@pytest.mark.parametrize("clip", [("norm", 2.0**-7, 0.05), ("norm", 8.0, 0.05), ("value", 1.5e-3, None)])
def test_grad_scale_bitwise(eng, n, clip):
    """clip_grad_norm_'s scaling pass / clip_grad_value_ on fp32 grads: bit-identical to torch's fp32 ops."""
    L = _lib()
    off = 8
    g = _rand(n, F32, seed=n)
    g[5] = float("nan")                     # kept by both clamps, like torch.clamp
    G = Buf(off + n + 8, F32)
    G.t[off:off + n] = g.cuda()
    bg = G.bits()
    if clip[0] == "norm":
        eng.scaler_set(grad_norm=clip[2])
        eng.grad_scale(G.ptr(off), n, L.CLIP_NORM, clip[1], 0.0)
        norm = torch.tensor(clip[2], dtype=F32)
        coef = torch.clamp(torch.tensor(clip[1], dtype=F32) / (norm + 1e-6), max=1.0)
        want = g * coef
        bad = g * torch.clamp(torch.tensor(clip[1], dtype=F32) / norm, max=1.0)   # control: no +1e-6
    else:
        eng.grad_scale(G.ptr(off), n, L.CLIP_VALUE, 0.0, clip[1])
        want = torch.clamp(g, -clip[1], clip[1])
        bad = torch.clamp(torch.nan_to_num(g, nan=-clip[1]), -clip[1], clip[1])   # control: NaN turned into -clip
    got = G.t[off:off + n].cpu()
    nan = torch.isnan(want)   # a NaN's payload is not part of the result (the GPU returns the canonical NaN)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(got[~nan].view(torch.int32), want[~nan].view(torch.int32))
    if clip[0] == "value" or clip[1] < clip[2]:
        assert not torch.equal(got.view(torch.int32), bad.view(torch.int32))
    rng = torch.zeros(G.n, dtype=torch.bool)
    rng[off:off + n] = True
    G.check_unchanged_except(bg, rng)


# ---- 4. stk_optim_step_ex ------------------------------------------------------------------------------------------------
ADAM = {"lr": 2.0**-7, "beta1": 0.875, "beta2": 0.9921875, "eps": 2.0**-20}
SGD_M = {"lr": 2.0**-5, "momentum": 0.875, "dampening": 0.25}


def _hyper(kind, h, clip):
    L = _lib()
    o = L.OptimHyper()
    o.kind = {"adam": L.OPT_ADAM, "adamw": L.OPT_ADAMW, "sgd": L.OPT_SGD}[kind]
    o.lr = h["lr"]
    o.beta1, o.beta2, o.eps = h.get("beta1", 0.9), h.get("beta2", 0.999), h.get("eps", 1e-8)
    o.weight_decay = h.get("weight_decay", 0.0 if kind != "adamw" else 1e-2)
    o.momentum, o.dampening = h.get("momentum", 0.0), h.get("dampening", 0.0)
    o.nesterov, o.maximize = int(h.get("nesterov", False)), int(h.get("maximize", False))
    o.clip_kind = {None: L.CLIP_NONE, "norm": L.CLIP_NORM, "value": L.CLIP_VALUE}[clip[0] if clip else None]
    o.clip_max_norm = clip[1] if clip and clip[0] == "norm" else 0.0
    o.clip_value = clip[1] if clip and clip[0] == "value" else 0.0
    return o


def _layout(n_local, n_seg, rng, base):
    """Local pieces [l0, l1) placed at shuffled global offsets (16-element aligned, with gaps); returns (pieces, N)."""
    if n_seg == 0:
        return [(0, n_local, base)], base + n_local + 48
    nv = n_local // 8
    cuts = sorted(rng.choice(np.arange(1, nv), n_seg - 1, replace=False).tolist()) if n_seg > 1 else []
    bounds = [0] + cuts + [nv]
    pieces = [(bounds[k] * 8, bounds[k + 1] * 8) for k in range(n_seg)]
    pos, glob = base, [0] * n_seg
    for k in rng.permutation(n_seg):
        glob[k] = pos
        pos += -(-(pieces[k][1] - pieces[k][0]) // 16) * 16 + 16 * int(rng.integers(0, 3))
    return [(pieces[k][0], pieces[k][1], glob[k]) for k in range(n_seg)], pos + 48


OPT_CASES = {
    # name: kind, src, lp, n_local, n_seg, groups (list of hypers), ranges?, skip?, clip, extras
    "adam_raw_bf16": ("adam", "raw_bf16", "bf16", 2_048, 0, [ADAM], False, False, None, {}),
    "adam_raw_bf16_seg64_ranges": ("adam", "raw_bf16", "bf16", 2_048, 64,
                                   [ADAM, dict(ADAM, lr=2.0**-6, beta2=0.984375), dict(ADAM, weight_decay=0.25),
                                    dict(ADAM, maximize=True), dict(ADAM, beta1=0.0), dict(ADAM, eps=1e-8),
                                    dict(ADAM, lr=0.0), dict(ADAM, lr=2.0**-8, beta1=0.75)], True, True, None, {}),
    "adamw_raw_f32_acc": ("adamw", "raw_f32_acc", None, 2_056, 3, [dict(ADAM, weight_decay=0.25)], False, False,
                          ("norm", 2.0**-7), {"scale": 2.0**16, "mul": 0.5}),
    "adamw_main_lp_f32": ("adamw", "main", "f32", 2_040, 0, [dict(ADAM, weight_decay=0.25)], True, True,
                          ("value", 1.5e-3), {}),
    "adam_main_alias": ("adam", "main", "f32_alias", 2_048, 0, [dict(ADAM, weight_decay=2.0**-4)], False, False,
                        ("norm", "boundary"), {"steps0": 10**6}),
    "adam_main_eps_dominated": ("adam", "main", None, 2_056, 5, [dict(ADAM, eps=1e-8)], False, False, None,
                                {"g_scale": 1e-10, "found_inf_at": 2}),
    "adam_main_lp_bf16_ranges": ("adam", "main", "bf16", 2_048, 7, [ADAM, dict(ADAM, lr=0.0)], True, False, None, {}),
    "sgd_main_dampening": ("sgd", "main", "bf16", 2_048, 2, [SGD_M], False, False, ("norm", 2.0**-7), {}),
    "sgd_main_nesterov_wd": ("sgd", "main", None, 2_040, 0,
                             [{"lr": 2.0**-5, "momentum": 0.875, "nesterov": True, "weight_decay": 2.0**-4}],
                             False, False, None, {}),
    "sgd_main_nomom_wd_max": ("sgd", "main", "f32", 2_056, 4,
                              [{"lr": 2.0**-5, "weight_decay": 2.0**-4, "maximize": True}], False, False, None,
                              {"no_buf": True}),
    "sgd_raw_bf16_groups": ("sgd", "raw_bf16", "bf16", 2_040, 9,
                            [SGD_M, {"lr": 2.0**-6, "momentum": 0.5, "dampening": 0.0}], True, True, None,
                            {"found_inf_at": 3}),
    "adam_empty": ("adam", "main", None, 0, 0, [ADAM], False, False, None, {}),
}


@pytest.mark.parametrize("name", list(OPT_CASES))
def test_optim_step_matches_torch_float64(eng, name):
    """Five consecutive fused steps, each checked element by element against torch.optim in float64 restarted from the
    kernel's own state; the raw bucket is zeroed exactly on its segments' global ranges, the low-precision copy is
    written exactly at lp offset + global index, and nothing else in any buffer changes."""
    L = _lib()
    kind, src, lp, n_local, n_seg, groups, use_ranges, use_skip, clip, ex = OPT_CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    pieces, N = _layout(n_local, n_seg, rng, base=64)
    N = -(-N // 16) * 16
    gidx = np.concatenate([np.arange(g0, g0 + (l1 - l0)) for l0, l1, g0 in pieces]) if n_local else np.zeros(0, np.int64)
    # ranges over the global index space, cut on 16-element boundaries
    if use_ranges:
        nr = 12
        ends = sorted(rng.choice(np.arange(1, N // 16), nr - 1, replace=False).tolist()) + [N // 16]
        ends = [e * 16 for e in ends]
        rgroup = [j % len(groups) for j in range(nr)]
        rskip = [bool(use_skip and j % 4 == 1) for j in range(nr)]
    else:
        ends, rgroup, rskip = [N], [0], [False]
    starts = [0] + ends[:-1]
    elem_range = np.searchsorted(np.asarray(ends), gidx, side="right")
    mom = kind == "sgd" and not ex.get("no_buf")
    steps0 = ex.get("steps0", 0)
    scale, mul = ex.get("scale", 1.0), ex.get("mul", 1.0)
    inv = kr.inv_scale_f32(scale)
    hyp = (L.OptimHyper * len(groups))(*[_hyper(kind, h, clip if clip and clip[1] != "boundary" else
                                                ("norm", 0.0) if clip else None) for h in groups])
    g32 = rng.standard_normal(n_local).astype(np.float32)
    gsc = ex.get("g_scale", 1e-3)   # weights around 1e-3, lr around 1e-2: each update is far above ulp(w)
    w0 = torch.from_numpy(rng.standard_normal(n_local).astype(np.float32) * 1e-3)
    m0 = torch.from_numpy(rng.standard_normal(n_local).astype(np.float32) * gsc * 0.1)
    v0 = torch.from_numpy(rng.random(n_local).astype(np.float32) * gsc * gsc)
    # buffers
    alias = lp == "f32_alias"
    lp_off = pieces[0][2]
    if alias:
        LPB = Buf(N, F32, torch.full((N,), -3.0))
        LPB.t[lp_off:lp_off + n_local] = w0.cuda()
        master_ptr = LPB.ptr(lp_off)
        MB = None
    else:
        MB = Buf(n_local, F32, w0.cuda())
        master_ptr = MB.ptr()
        LPB = None if lp is None else Buf(N, BF16 if lp == "bf16" else F32, torch.full((N,), -5.0))
    MM = Buf(n_local, F32, m0.cuda()) if (kind != "sgd" or mom) else None
    VV = Buf(n_local, F32, v0.cuda()) if kind != "sgd" else None
    gdt = {"raw_bf16": BF16, "raw_f32_acc": F32, "main": F32}[src]
    GB = Buf(N if src != "main" else n_local, gdt)
    AB = Buf(N, F32) if src == "raw_f32_acc" else None
    if use_ranges:
        rend = torch.tensor([e // 8 for e in ends], dtype=torch.int32).cuda()
        rgrp = torch.tensor([g | (0x80 if s else 0) for g, s in zip(rgroup, rskip)], dtype=torch.uint8).cuda()
        rsteps = torch.tensor([steps0 + (3 if j % 3 == 2 else 0) for j in range(len(ends))], dtype=torch.int32).cuda()
        rbc = torch.zeros(len(ends), 4, dtype=torch.float32, device="cuda")
    sl = (C.c_size_t * (len(pieces) + 1))(*([p[0] for p in pieces] + [n_local]))
    sg = (C.c_size_t * len(pieces))(*[p[2] for p in pieces])
    lpp = _lib().ptr_array([LPB.ptr()]) if lp is not None else None
    eng.scaler_set(opt_steps=steps0, skipped_steps=0, scale=scale, enabled=0, found_inf=0)
    master_view = (lambda: LPB.t[lp_off:lp_off + n_local]) if alias else (lambda: MB.t)
    controls_hit = set()

    for step in range(5):
        # gradients: bf16 / fp32 values handed exactly to the reference
        gs = ex.get("g_scale", 1e-3) * scale
        g = torch.from_numpy(np.roll(g32, step * 37) * gs).to(gdt)
        gfull = torch.zeros(GB.n, dtype=gdt)
        if src == "main":
            gfull[:] = g
        else:
            gfull[:] = torch.from_numpy(rng.standard_normal(GB.n).astype(np.float32)).to(gdt)  # outside: must survive
            gfull[torch.from_numpy(gidx)] = g
        GB.t.copy_(gfull.cuda())
        acc = None
        if AB is not None:
            acc = torch.from_numpy((rng.standard_normal(n_local) * gs).astype(np.float32))
            afull = torch.from_numpy(rng.standard_normal(N).astype(np.float32))
            afull[torch.from_numpy(gidx)] = acc
            AB.t.copy_(afull.cuda())
        found_inf = ex.get("found_inf_at") == step
        gnorm = None
        if clip and clip[0] == "norm":
            gnorm = 0.05 if clip[1] != "boundary" else 0.25
            if clip[1] == "boundary":   # max_norm == norm + 1e-6 in fp32: the coefficient lands on 1 exactly
                for gi in range(len(groups)):
                    hyp[gi].clip_max_norm = kr.f32_value(kr.f32_value(gnorm) + kr.f32_value(1e-6))
            eng.scaler_set(grad_norm=gnorm)
        eng.scaler_set(found_inf=int(found_inf))
        st0 = eng.scaler_get()
        # pre-step state (the kernel's own)
        w, m = master_view().cpu().clone(), (MM.t.cpu().clone() if MM else None)
        v = VV.t.cpu().clone() if VV else None
        snap = {k: b.bits() for k, b in (("G", GB), ("A", AB), ("M", MB), ("MM", MM), ("VV", VV), ("LP", LPB)) if b}
        rsteps_before = rsteps.cpu().clone() if use_ranges else None
        # launch
        a = L.OptimArgs()
        a.hyper, a.n_groups = hyp, len(groups)
        a.master = master_ptr
        a.exp_avg = MM.ptr() if MM else None
        a.exp_avg_sq = VV.ptr() if VV else None
        a.grad, a.grad_dtype, a.grad_raw = GB.ptr(), _dt(gdt), int(src != "main")
        a.acc = AB.ptr() if AB else None
        a.grad_mul = mul
        a.n_local = n_local
        a.lp_ptrs, a.lp_world, a.lp_dtype = lpp, (1 if lp else 0), (L.BF16 if lp == "bf16" else L.F32)
        a.lp_offset = lp_off if n_seg == 0 else 0
        a.n_seg = n_seg
        a.seg_local, a.seg_global = (sl, sg) if n_seg else (None, None)
        if use_ranges:
            a.n_ranges, a.range_end_vec, a.range_group = len(ends), rend.data_ptr(), rgrp.data_ptr()
            eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, None, len(groups), len(ends), rgrp.data_ptr(),
                                                       rsteps.data_ptr(), None, rbc.data_ptr(), eng._stream()))
            a.range_bc = rbc.data_ptr()
        eng.optim_step_ex(a)
        eng.step_epilogue()
        st = eng.scaler_get()
        assert (st.opt_steps, st.skipped_steps) == (st0.opt_steps + (not found_inf), st0.skipped_steps + found_inf)
        assert st.found_inf == 0
        got_w = master_view().cpu()
        got_m = MM.t.cpu() if MM else None
        got_v = VV.t.cpu() if VV else None

        # ---- reference ----
        x, e_x = kr.scaled_grad(g.float() if src == "main" else g, acc, mul if src != "main" else 1.0,
                                inv if src != "main" else 1.0)
        if clip and clip[0] == "norm":
            mx = hyp[0].clip_max_norm
            c, e_c = kr.clip_coef(kr.f32_value(gnorm), mx), kr.clip_coef_bound(kr.f32_value(gnorm), mx)
            G = x * c
            e_g = c * e_x + x.abs() * e_c + kr.U * G.abs()
        elif clip:
            G = kr.clip_value_ref(x, clip[1])
            e_g = e_x + kr.U * clip[1]
        else:
            G, e_g = x, e_x
        skip_elem = torch.from_numpy(np.asarray(rskip)[elem_range]) | found_inf

        def reference(mut=None):
            rw, rm, rv = w.double().clone(), (m.double().clone() if m is not None else None), \
                (v.double().clone() if v is not None else None)
            bw, bm, bv = torch.zeros(n_local, dtype=torch.float64), torch.zeros(n_local, dtype=torch.float64), \
                torch.zeros(n_local, dtype=torch.float64)
            for j in range(len(ends)):
                sel = torch.from_numpy(elem_range == j)
                if mut == "neighbour_group" and j > 0:   # the first vector of the range takes the previous range's group
                    first = torch.from_numpy((elem_range == j) & (gidx < starts[j] + 8))
                    sel_sets = [(sel & ~first, rgroup[j]), (first, rgroup[j - 1])]
                else:
                    sel_sets = [(sel, rgroup[j])]
                for s, gi in sel_sets:
                    if not bool(s.any()):
                        continue
                    if bool(skip_elem[s].all()) and not (mut == "skip_stepped" and rskip[j] and not found_inf):
                        continue
                    h = groups[gi]
                    done = int(rsteps_before[j]) if use_ranges else int(st0.opt_steps)
                    if kind == "sgd":
                        buf = m[s] if (mom and done > 0) else None
                        hh = h
                        if mut == "no_dampening":
                            hh = dict(h, dampening=0.0)
                        elif mut == "no_nesterov":
                            hh = dict(h, nesterov=False)
                        nw, nb = kr.sgd_step(w[s], buf, G[s], hh)
                        ew, eb = kr.sgd_bound(w[s], buf, G[s], e_g[s], h, nw, nb)
                        rw[s], bw[s] = nw, ew
                        if nb is not None:
                            rm[s], bm[s] = nb, eb
                    else:
                        if mut in ("eps_in_sqrt", "bc2_not_sqrt", "decay_after"):
                            nw, nm, nv = kr.adam_step_mutant(kind, w[s], m[s], v[s], G[s], done, h, mut)
                        else:
                            nw, nm, nv = kr.adam_step(kind, w[s], m[s], v[s], G[s], done, h)
                        ew, em, ev = kr.adam_bound(kind, w[s], m[s], v[s], G[s], e_g[s], done, h, nm, nv)
                        rw[s], rm[s], rv[s], bw[s], bm[s], bv[s] = nw, nm, nv, ew, em, ev
            return rw, rm, rv, bw, bm, bv

        rw, rm, rv, bw, bm, bv = reference()
        ok_w = (got_w.double() - rw).abs() <= bw
        assert bool(ok_w.all()), f"step {step}: master off at {torch.nonzero(~ok_w)[:5].flatten().tolist()}"
        if got_m is not None and rm is not None:
            assert bool(((got_m.double() - rm).abs() <= bm).all()), f"step {step}: exp_avg / momentum"
        if got_v is not None:
            assert bool(((got_v.double() - rv).abs() <= bv).all()), f"step {step}: exp_avg_sq"
        # skipped elements (found_inf, skipped ranges) and lr = 0 groups: bit-identical master
        frozen = skip_elem.clone()
        for j in range(len(ends)):
            if groups[rgroup[j]]["lr"] == 0.0:
                frozen |= torch.from_numpy(elem_range == j)
        assert torch.equal(got_w[frozen].view(torch.int32), w[frozen].view(torch.int32))
        if got_m is not None:
            assert torch.equal(got_m[skip_elem].view(torch.int32), m[skip_elem].view(torch.int32))
        # negative controls
        muts = []
        if n_local and kind != "sgd" and not found_inf:
            # (after 10**6 steps bias_correction2 is 1, where its square root and itself coincide)
            muts += (["bc2_not_sqrt"] if steps0 < 1000 else []) + (["eps_in_sqrt"] if ex.get("g_scale") is None else []) + \
                (["decay_after"] if kind == "adamw" else [])
        if n_local and kind == "sgd" and not found_inf:
            h0 = groups[0]
            if h0.get("dampening") and step > 0:
                muts.append("no_dampening")
            if h0.get("nesterov"):
                muts.append("no_nesterov")
        if n_local and use_skip and not found_inf:
            muts.append("skip_stepped")
        if n_local and use_ranges and len(groups) > 1 and not found_inf:
            muts.append("neighbour_group")
        for mu in muts:
            mw = reference(mu)[0]
            if bool(((got_w.double() - mw).abs() > bw).any()):
                controls_hit.add(mu)
            else:
                pytest.fail(f"negative control {mu} passed the per-element check at step {step}")
        if muts and clip and clip[0] == "norm" and clip[1] != "boundary" and kind == "sgd":
            # the clip coefficient without its +1e-6 moves the update by more than the bound
            cm = kr.clip_coef_mutant(kr.f32_value(gnorm), hyp[0].clip_max_norm)
            h0 = groups[0]
            mw, _ = kr.sgd_step(w, m if (mom and st0.opt_steps > 0) else None, x * cm, h0)
            assert bool(((got_w.double() - mw).abs() > bw).any())
            controls_hit.add("clip_no_eps")

        # ---- where the kernel wrote ----
        none = lambda b: torch.zeros(b.n, dtype=torch.bool)
        loc_changed = ~frozen if not found_inf else torch.zeros(n_local, dtype=torch.bool)
        if MB is not None:
            MB.check_unchanged_except(snap["M"], loc_changed)
        if MM is not None:
            MM.check_unchanged_except(snap["MM"], ~skip_elem)
        if VV is not None:
            VV.check_unchanged_except(snap["VV"], ~skip_elem)
        if src != "main":   # raw bucket: zeroed exactly on the segments' global ranges, also on a skipped step
            seg_mask = none(GB)
            seg_mask[torch.from_numpy(gidx)] = True
            GB.check_unchanged_except(snap["G"], seg_mask)
            assert n_local == 0 or float(GB.t[torch.from_numpy(gidx).cuda()].float().abs().max()) == 0.0
        else:
            GB.check_unchanged_except(snap["G"], none(GB))
        if AB is not None:
            AB.check_unchanged_except(snap["A"], none(AB))
        if LPB is not None:
            stepped = ~skip_elem
            lp_mask = none(LPB)
            if alias:
                lp_mask[lp_off:lp_off + n_local] = loc_changed
            else:
                lp_mask[torch.from_numpy(gidx)[stepped]] = True
            LPB.check_unchanged_except(snap["LP"], lp_mask)
            if not alias and bool(stepped.any()):
                glp = LPB.t[torch.from_numpy(gidx)[stepped].cuda()].cpu()
                want = got_w[stepped].to(LPB.dtype)
                assert torch.equal(glp.view(INT_VIEW[LPB.dtype]), want.view(INT_VIEW[LPB.dtype]))
        if use_ranges:   # the prologue's per-range step counts: +1 unless skipped or found_inf
            inc = torch.tensor([0 if (s or found_inf) else 1 for s in rskip], dtype=torch.int32)
            assert torch.equal(rsteps.cpu(), rsteps_before + inc)
    if n_local:
        assert controls_hit or kind == "sgd" and not groups[0].get("momentum"), "no negative control ran"


# ---- 5. k_step_prologue and k_step_epilogue -------------------------------------------------------------------------------
def test_step_prologue_per_range_bias_corrections(eng):
    L = _lib()
    groups = [ADAM, {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-8}, dict(ADAM, beta1=0.0)]
    hyp = (L.OptimHyper * 3)(*[_hyper("adam", h, None) for h in groups])
    steps = [0, 1, 2, 9, 99, 10**6, 5, 0, 3, 7, 10**4, 1]
    nr = len(steps)
    rgrp_l = [(j % 3) | (0x80 if j % 5 == 4 else 0) for j in range(nr)]
    rgrp = torch.tensor(rgrp_l, dtype=torch.uint8).cuda()
    rs = torch.tensor(steps, dtype=torch.int32).cuda()
    rbc = torch.zeros(nr, 4, dtype=torch.float32, device="cuda")
    for found_inf in (0, 1):
        eng.scaler_set(found_inf=found_inf)
        before = rs.cpu().clone()
        eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, None, 3, nr, rgrp.data_ptr(), rs.data_ptr(), None,
                                                   rbc.data_ptr(), eng._stream()))
        got = rbc.cpu()
        for j in range(nr):
            ss, c2 = kr.bias_corrections(groups[rgrp_l[j] & 0x7F], int(before[j]))
            for g_, r_ in ((float(got[j, 0]), ss), (float(got[j, 1]), c2)):   # within 1 fp32 ulp
                assert abs(g_ - r_) <= float(np.spacing(np.float32(r_)))
            assert float(got[j, 2]) == (1.0 if int(before[j]) == 0 else 0.0)
            want = int(before[j]) + (0 if (rgrp_l[j] & 0x80 or found_inf) else 1)
            assert int(rs[j]) == want


@pytest.mark.parametrize("kind,h", [("adam", ADAM), ("adamw", dict(ADAM, weight_decay=0.25)), ("sgd", SGD_M)])
def test_group_bc_from_prologue_matches_in_kernel_scalars(eng, kind, h):
    """Adam / AdamW / SGD given the prologue's per-group scalars (group_bc) step bit for bit like the optimizer-wide step
    that forms them itself: master, moments and the bf16 copy, from the first step (SGD: buf = g) on."""
    L = _lib()
    n = 4096
    hyp = (L.OptimHyper * 1)(_hyper(kind, h, None))
    w0 = _rand(n, F32, seed=5).cuda()
    runs = []
    for use_bc in (False, True):
        M, MM, VV, GG = Buf(n, F32, w0), Buf(n, F32, torch.zeros(n)), Buf(n, F32, torch.zeros(n)), Buf(n, F32)
        LP = Buf(n, BF16, torch.zeros(n))
        bc = torch.zeros(1, 4, dtype=torch.float32, device="cuda")
        lpp = _lib().ptr_array([LP.ptr()])
        out = []
        for step in range(3):
            GG.t.copy_(_rand(n, F32, seed=10 + step).cuda())
            eng.scaler_set(opt_steps=step, skipped_steps=0, found_inf=0)
            a = L.OptimArgs()
            a.hyper, a.n_groups = hyp, 1
            a.master, a.exp_avg, a.exp_avg_sq = M.ptr(), MM.ptr(), (VV.ptr() if kind != "sgd" else None)
            a.grad, a.grad_dtype, a.grad_raw, a.n_local = GG.ptr(), L.F32, 0, n
            a.lp_ptrs, a.lp_world, a.lp_dtype = lpp, 1, L.BF16
            if use_bc:
                eng._check(eng.lib.stk_optim_step_prologue(eng.ctx, hyp, None, 1, 0, None, None, None, bc.data_ptr(),
                                                           eng._stream()))
                a.group_bc = bc.data_ptr()
            eng.optim_step_ex(a)
            out.append((M.bits(), MM.bits(), VV.bits(), LP.bits()))
        runs.append(out)
    for step, (a_, b_) in enumerate(zip(*runs)):
        for name, x, y in zip(("master", "exp_avg", "exp_avg_sq", "bf16"), a_, b_):
            assert torch.equal(x, y), (step, name)


def test_step_epilogue_follows_amp_update_scale(eng):
    """A scripted sequence of verdicts against torch._amp_update_scale_: back-off, growth at the interval, growth
    interval 1, and a growth that would overflow fp32 leaves the scale unchanged."""
    big = float(torch.finfo(torch.float32).max) / 1.5
    for scale0, interval, verdicts in ((2.0**16, 3, [0, 1, 0, 0, 0, 1, 0, 0, 0, 0]),
                                       (2.0**10, 1, [0, 0, 1, 0, 1, 1, 0]),
                                       (big, 1, [0, 0, 1, 0])):
        eng.scaler_set(scale=scale0, enabled=1, growth_interval=interval, growth_tracker=0, growth_factor=2.0,
                       backoff_factor=0.5, found_inf=0, opt_steps=0, skipped_steps=0)
        s, t = scale0, 0
        for k, bad in enumerate(verdicts):
            eng.scaler_set(found_inf=bad)
            eng.step_epilogue()
            s, t = kr.update_scale(s, t, bool(bad), 2.0, 0.5, interval)
            st = eng.scaler_get()
            assert (st.scale, st.growth_tracker) == (s, t), (scale0, k)
            assert st.found_inf == 0
        assert (st.opt_steps, st.skipped_steps) == (verdicts.count(0), verdicts.count(1))
    eng.scaler_set(enabled=0, scale=1.0)


# ---- 6. determinism --------------------------------------------------------------------------------------------------------
def test_repeated_calls_are_bitwise_identical(eng):
    L = _lib()
    n = 16_777_224
    G = Buf(n, BF16, _rand(n, BF16, seed=1).cuda())
    norms = []
    for _ in range(2):
        eng.grad_norm(G.ptr(), BF16, None, n, 1.0, L.NORM_L2, 2.0, L.RF_FINAL)
        norms.append(eng.scaler_get().grad_norm)
    assert norms[0] == norms[1]
    nl = 1 << 20
    w0, g = _rand(nl, F32, seed=2), _rand(nl, F32, seed=3)
    outs = []
    for _ in range(2):
        eng.scaler_set(opt_steps=3, found_inf=0, grad_norm=0.5)
        M, MM, VV, GG = Buf(nl, F32, w0.cuda()), Buf(nl, F32, (g * 0.1).cuda()), Buf(nl, F32, (g * g).cuda()), \
            Buf(nl, F32, g.cuda())
        hyp = (L.OptimHyper * 1)(_hyper("adamw", dict(ADAM, weight_decay=0.25), ("norm", 0.25)))
        eng.optim_step(hyp[0], M.ptr(), MM.ptr(), VV.ptr(), GG.ptr(), nl, None, F32, 0)
        outs.append((M.bits(), MM.bits(), VV.bits()))
    for a_, b_ in zip(*outs):
        assert torch.equal(a_, b_)
