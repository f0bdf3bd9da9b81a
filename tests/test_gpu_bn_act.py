"""stk_bn_act (csrc/bn_act.cu) and the BnAct module of stoke_b200/fuse.py against the unfused torch sequence
``BatchNorm2d -> out += identity -> ReLU(inplace=True)`` in bf16 channels-last: bit for bit, at every BatchNorm shape of
ResNet-50 at B = 128 plus odd sizes, with and without the residual, with inf / NaN inputs and with outputs of -0.0, and with
``momentum`` 0.1 and None.

The kernel's own outputs (activation and save_invstd) are written between 0xFF guard bands, and save_mean / save_invstd
are compared with what torch's native_batch_norm returns.  The module comparison covers the output, the running statistics,
num_batches_tracked and every gradient (dx, dweight, dbias, dresidual) over two training steps."""
import pytest
import torch

from stoke_b200.fuse import BnAct

pytestmark = pytest.mark.gpu

GUARD = 4096
RESNET50_B128 = [(128, c, h, h) for c, h in [(64, 112), (64, 56), (128, 56), (256, 56), (128, 28), (256, 28), (512, 28),
                                              (256, 14), (512, 14), (1024, 14), (512, 7), (2048, 7)]]
ODD = [(3, 8, 5, 5), (3, 24, 5, 5), (2, 24, 1, 3), (5, 8, 7, 3)]
SHAPES = RESNET50_B128 + ODD
EPS = 1e-5


def _bits(t):
    return t.contiguous().view({torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int64: torch.int64}[t.dtype])


def assert_same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert torch.equal(_bits(a), _bits(b)), f"{what}: {int((_bits(a) != _bits(b)).sum())} elements differ"


def _inputs(shape, special, seed):
    n, c, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(shape, device="cuda", generator=g) * 2 + 0.5).to(torch.bfloat16)
    r = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    if special == "negzero":   # channel 0 all zero: mean 0, (x - mean) * weight = +0 * -1 = -0, + bias -0 (_bn), + residual -0
        x[:, 0] = 0.0
        r[:, 0] = -0.0
    if special == "infnan":   # inf / NaN in one channel of x (its statistics become NaN) and scattered through the residual
        x[0, c - 1, 0, 0] = float("inf")
        x[n - 1, 0, h - 1, w - 1] = float("nan")
        flat = r.view(-1)
        flat[::97] = float("nan")
        flat[1::89] = float("inf")
        flat[2::83] = float("-inf")
    x = x.contiguous(memory_format=torch.channels_last)
    r = r.contiguous(memory_format=torch.channels_last)
    return x, r


def _bn(c, seed, special="none", momentum=0.1):
    g = torch.Generator().manual_seed(seed)
    bn = torch.nn.BatchNorm2d(c, eps=EPS, momentum=momentum)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.rand(c, generator=g) - 0.5)
        if special == "negzero":
            bn.weight[0], bn.bias[0] = -1.0, -0.0
        bn.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn.to(device="cuda", dtype=torch.bfloat16)


@pytest.fixture
def eng():
    from stoke_b200.engine import get_engine

    torch.cuda.set_device(0)
    return get_engine(0)


SPECIAL = ["none", "infnan", "negzero"]


@pytest.mark.parametrize("special", SPECIAL)
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_kernel_guarded(eng, shape, residual, special):
    x, r = _inputs(shape, special, seed=shape[1] + shape[2])
    c = shape[1]
    bn = _bn(c, seed=c, special=special)
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    ref, ref_mean, ref_invstd = torch.ops.aten.native_batch_norm(x, bn.weight, bn.bias, rm, rv, True, 0.1, EPS)
    if residual:
        ref += r
    if special == "negzero":   # the ReLU sees -0.0 in channel 0
        assert bool((_bits(ref[:, 0]) == -32768).all())
    ref.relu_()

    mean, var = torch.batch_norm_update_stats(x, bn.running_mean.clone(), bn.running_var.clone(), 0.1)
    n = x.numel()
    out_raw = torch.full((2 * GUARD + 2 * n,), 0xFF, dtype=torch.uint8, device="cuda")
    inv_raw = torch.full((2 * GUARD + 4 * c,), 0xFF, dtype=torch.uint8, device="cuda")
    out = out_raw[GUARD:GUARD + 2 * n].view(torch.bfloat16).view(shape[0], shape[2], shape[3], c).permute(0, 3, 1, 2)
    invstd = inv_raw[GUARD:GUARD + 4 * c].view(torch.float32)
    eng.bn_act(x, r if residual else None, mean, var, bn.weight, bn.bias, EPS, out, invstd)
    torch.cuda.synchronize()
    for raw in (out_raw, inv_raw):
        assert bool((raw[:GUARD] == 0xFF).all()) and bool((raw[-GUARD:] == 0xFF).all()), "guard band written"
    assert_same(out, ref, "out")
    assert_same(mean, ref_mean, "save_mean")
    assert_same(invstd, ref_invstd, "save_invstd")


@pytest.mark.parametrize("momentum", [0.1, None])   # None: cumulative average from num_batches_tracked
@pytest.mark.parametrize("special", SPECIAL)
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_module_against_unfused(eng, shape, residual, special, momentum):
    c = shape[1]
    ref_bn, my_bn = _bn(c, c + 1, special, momentum), _bn(c, c + 1, special, momentum)
    relu = torch.nn.ReLU(inplace=True)
    fused = BnAct(my_bn, eng)
    for step in range(2):
        x, r = _inputs(shape, special, seed=step * 1000 + c)
        xa, ra = x.clone().requires_grad_(), r.clone().requires_grad_()
        xb, rb = x.clone().requires_grad_(), r.clone().requires_grad_()
        out = ref_bn(xa)
        if residual:
            out += ra
        a = relu(out)
        launches = eng.launches
        b = fused(xb, rb if residual else None)
        assert eng.launches == launches + 1, "the kernel did not run (BnAct took the unfused fallback)"
        assert_same(b, a, "out")
        gy = torch.randn(shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(step)).to(torch.bfloat16)
        gy = gy.contiguous(memory_format=torch.channels_last)
        a.backward(gy)
        b.backward(gy)
        assert_same(xb.grad, xa.grad, "dx")
        if residual:
            assert_same(rb.grad, ra.grad, "dresidual")
        assert_same(my_bn.weight.grad, ref_bn.weight.grad, "dweight")
        assert_same(my_bn.bias.grad, ref_bn.bias.grad, "dbias")
        assert_same(my_bn.running_mean, ref_bn.running_mean, "running_mean")
        assert_same(my_bn.running_var, ref_bn.running_var, "running_var")
        assert_same(my_bn.num_batches_tracked, ref_bn.num_batches_tracked, "num_batches_tracked")
