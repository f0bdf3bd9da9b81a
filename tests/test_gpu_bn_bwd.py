"""stk_bn_act_backward (csrc/bn_act.cu) and BnAct's backward against the unfused torch backward
``threshold_backward`` + ``native_batch_norm_backward``, bit for bit, in bf16 channels-last.

The entry point's outputs (dx, dweight, dbias, dresidual) are written between 0xFF guard bands.  The shapes cover every
regime of torch's channels-last reduce launch (grid_y = 1, 8 <= grid_y < 128, grid_y = 128 with a partial last pass over
the rows, block_x < 32, channel counts that are not powers of two), with a channel whose ReLU masks every element, inf
and NaN in grad, x and out, and -0.0 gradients.  The module tests show that the backward runs the kernels (launch count)
when the gradient is bf16 channels-last, and torch's ops otherwise, with the same results."""
import pytest
import torch

from stoke_b200.engine import bn_backward_grid
from stoke_b200.fuse import BnAct

pytestmark = pytest.mark.gpu

GUARD = 4096
EPS = 1e-5
SHAPES = [
    (3, 8, 5, 5),        # grid_y 1, block_x 8
    (2, 24, 1, 3),       # grid_y 1, 6 rows, block_x 16
    (4, 200, 9, 9),      # grid_y 1, C not a power of two
    (16, 64, 14, 14),    # grid_y 13
    (16, 200, 20, 20),   # grid_y 25, C not a power of two
    (32, 16, 65, 63),    # grid_y 128, block_x 16, partial last pass
    (128, 128, 28, 28),  # grid_y 128, partial last pass (ResNet-50)
    (128, 1024, 14, 14), # grid_y 98 (ResNet-50)
    (128, 2048, 7, 7),   # grid_y 25 (ResNet-50)
]
SPECIAL = ["none", "masked", "infnan", "negzero"]


def test_shapes_cover_the_reduce_regimes():
    grids = {s: bn_backward_grid(s[0] * s[2] * s[3], s[1]) for s in SHAPES}
    assert any(g[1] == 1 for g in grids.values())
    assert any(8 <= g[1] < 128 for g in grids.values())
    assert any(g[1] == 128 and (s[0] * s[2] * s[3]) % (g[0] * g[1] * 4) for s, g in grids.items())
    assert bn_backward_grid(128 * 112 * 112, 64) == (16, 128, 196)
    assert bn_backward_grid(128 * 7 * 7, 2048) == (16, 25, 4)


def _bits(t):
    return t.contiguous().view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


def assert_same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert torch.equal(_bits(a), _bits(b)), f"{what}: {int((_bits(a) != _bits(b)).sum())} elements differ"


def _inputs(shape, special, seed):
    n, c, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(shape, device="cuda", generator=g) * 2 + 0.5).to(torch.bfloat16)
    r = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    gy = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    if special == "infnan":   # inf / NaN in x (one channel's statistics become NaN), the residual (out) and the gradient
        x[0, c - 1, 0, 0] = float("inf")
        x[n - 1, 0, h - 1, w - 1] = float("nan")
        for t, k in ((r, 0), (gy, 1)):
            flat = t.view(-1)
            flat[k::97] = float("nan")
            flat[k + 1::89] = float("inf")
            flat[k + 2::83] = float("-inf")
    if special == "negzero":  # -0.0 gradients: one whole channel and scattered elements
        gy[:, c // 2] = -0.0
        gy.view(-1)[::7] = -0.0
    cl = torch.channels_last
    return x.contiguous(memory_format=cl), r.contiguous(memory_format=cl), gy.contiguous(memory_format=cl)


def _bn(c, seed, special):
    g = torch.Generator().manual_seed(seed)
    bn = torch.nn.BatchNorm2d(c, eps=EPS)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.rand(c, generator=g) - 0.5)
        if special == "masked":   # every output of channel 0 is <= 0, so its gradient is all +0
            bn.bias[0] = -100.0
    return bn.to(device="cuda", dtype=torch.bfloat16)


@pytest.fixture
def eng():
    from stoke_b200.engine import get_engine

    torch.cuda.set_device(0)
    return get_engine(0)


def _guarded(numel, dtype, like=None):
    esz = torch.tensor([], dtype=dtype).element_size()
    raw = torch.full((2 * GUARD + esz * numel,), 0xFF, dtype=torch.uint8, device="cuda")
    t = raw[GUARD:GUARD + esz * numel].view(dtype)
    if like is not None:
        n, c, h, w = like.shape
        t = t.view(n, h, w, c).permute(0, 3, 1, 2)
    return raw, t


@pytest.mark.parametrize("special", SPECIAL)
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_entry_guarded(eng, shape, residual, special):
    c = shape[1]
    x, r, gy = _inputs(shape, special, seed=shape[1] + shape[2])
    bn = _bn(c, seed=c, special=special)
    mean, var = torch.batch_norm_update_stats(x, bn.running_mean.clone(), bn.running_var.clone(), 0.1)
    out = torch.empty_like(x)
    invstd = torch.empty_like(mean)
    eng.bn_act(x, r if residual else None, mean, var, bn.weight, bn.bias, EPS, out, invstd)
    if special == "masked":
        assert bool((out[:, 0] <= 0).all())
    if special == "infnan":
        assert bool(out.isnan().any()) and (not residual or bool(out.isinf().any()))

    g = torch.ops.aten.threshold_backward(gy, out, 0)
    ref_dx, ref_dw, ref_db = torch.ops.aten.native_batch_norm_backward(g, x, bn.weight, bn.running_mean, bn.running_var,
                                                                      mean, invstd, True, EPS, [True, True, True])
    bufs = [_guarded(x.numel(), torch.bfloat16, x), _guarded(c, torch.bfloat16), _guarded(c, torch.bfloat16)]
    if residual:
        bufs.append(_guarded(x.numel(), torch.bfloat16, x))
    (_, dx), (_, dw), (_, db) = bufs[:3]
    dr = bufs[3][1] if residual else None
    eng.bn_act_backward(gy, x, out if residual else None, mean, invstd, bn.weight, None if residual else bn.bias,
                        dx, dw, db, dr)
    torch.cuda.synchronize()
    for raw, _ in bufs:
        assert bool((raw[:GUARD] == 0xFF).all()) and bool((raw[-GUARD:] == 0xFF).all()), "guard band written"
    assert_same(dx, ref_dx, "dx")
    assert_same(dw, ref_dw, "dweight")
    assert_same(db, ref_db, "dbias")
    if residual:
        assert_same(dr, g, "dresidual")


MODULE_SHAPES = [(3, 24, 5, 5), (16, 200, 20, 20), (128, 256, 14, 14)]


@pytest.mark.parametrize("x_grad", [True, False])
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("shape", MODULE_SHAPES)
def test_module_runs_kernels(eng, shape, residual, x_grad):
    c = shape[1]
    ref_bn, my_bn = _bn(c, c + 1, "none"), _bn(c, c + 1, "none")
    relu = torch.nn.ReLU(inplace=True)
    fused = BnAct(my_bn, eng)
    x, r, gy = _inputs(shape, "none", seed=c)
    xa, ra = x.clone().requires_grad_(x_grad), r.clone().requires_grad_()
    xb, rb = x.clone().requires_grad_(x_grad), r.clone().requires_grad_()
    out = ref_bn(xa)
    if residual:
        out += ra
    a = relu(out)
    b = fused(xb, rb if residual else None)
    a.backward(gy)
    launches = eng.launches
    b.backward(gy)
    grid_y = bn_backward_grid(x.numel() // c, c)[1]
    assert eng.launches == launches + 1 + (grid_y > 1) + x_grad, "the backward did not run the kernels"
    if x_grad:
        assert_same(xb.grad, xa.grad, "dx")
    if residual:
        assert_same(rb.grad, ra.grad, "dresidual")
    assert_same(my_bn.weight.grad, ref_bn.weight.grad, "dweight")
    assert_same(my_bn.bias.grad, ref_bn.bias.grad, "dbias")


def _layout(gy, layout):
    if layout == "nchw":
        return gy.contiguous()
    if layout == "expanded":   # what the average pool's backward passes on: one value per (n, c), strides (C, 1, 0, 0)
        return gy[:, :, :1, :1].expand(gy.shape)
    n, c, h, w = gy.shape      # channels-last, but 2 bytes off the 16-byte alignment the kernels need
    buf = torch.empty(gy.numel() + 1, dtype=gy.dtype, device=gy.device)
    t = buf[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    t.copy_(gy)
    return t


@pytest.mark.parametrize("layout", ["nchw", "expanded", "misaligned"])
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("shape", MODULE_SHAPES)
def test_module_gradient_layouts(eng, shape, residual, layout):
    """threshold_backward lays g out like out (channels-last) whatever the incoming gradient's layout, so torch runs its
    channels-last BatchNorm backward and so do the kernels, after making the gradient channels-last; a misaligned
    gradient takes torch's ops."""
    c = shape[1]
    ref_bn, my_bn = _bn(c, c + 1, "none"), _bn(c, c + 1, "none")
    relu = torch.nn.ReLU(inplace=True)
    fused = BnAct(my_bn, eng)
    x, r, gy = _inputs(shape, "none", seed=c)
    gy = _layout(gy, layout)
    assert not (gy.is_contiguous(memory_format=torch.channels_last) and gy.data_ptr() % 16 == 0)
    xa, ra = x.clone().requires_grad_(), r.clone().requires_grad_()
    xb, rb = x.clone().requires_grad_(), r.clone().requires_grad_()
    out = ref_bn(xa)
    if residual:
        out += ra
    a = relu(out)
    b = fused(xb, rb if residual else None)
    a.backward(gy)
    launches = eng.launches
    b.backward(gy)
    kernels = 0 if layout == "misaligned" else 2 + (bn_backward_grid(x.numel() // c, c)[1] > 1)
    assert eng.launches == launches + kernels
    assert_same(xb.grad, xa.grad, "dx")
    if residual:
        assert_same(rb.grad, ra.grad, "dresidual")
    assert_same(my_bn.weight.grad, ref_bn.weight.grad, "dweight")
    assert_same(my_bn.bias.grad, ref_bn.bias.grad, "dbias")
