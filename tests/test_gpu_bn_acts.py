"""stk_bn_act_ex / stk_bn_act_backward_ex (csrc/bn_act.cu) with SiLU, Hardswish and ReLU6, and the BnAct module and the
fuse_bn_act rewrite that use them, against torch's unfused ops in bf16 channels-last, bit for bit.

* Exhaustive forward: an identity BatchNorm (mean 0, var 1, eps 0, weight 1, bias -0.0, so y = x, -0 included) over all
  65,536 bf16 bit patterns, against F.silu / F.hardswish / F.relu6 on the GPU.
* Exhaustive derivative: the same 65,536 activation inputs times 64 gradients (+-0, +-inf, NaNs, subnormals, random),
  through grad_pre, against silu_backward / hardswish_backward / hardtanh_backward(..., 0, 6).
* The entry points against the unfused chain at every fused BatchNorm shape of EfficientNet-B0, MobileNetV3-Large and
  MobileNetV2 at B = 128 (each model's eps and momentum) plus odd shapes, with inf / NaN and -0.0, outputs between
  0xFF guard bands.
* The BnAct module over two training steps, with incoming gradients in every layout, and whole EfficientNet-B0 and
  MobileNetV3-Small models rewritten against unrewritten."""
import copy

import pytest
import torch
import torch.nn.functional as F

from stoke_b200._lib import ACT_HARDSWISH, ACT_RELU, ACT_RELU6, ACT_SILU
from stoke_b200.engine import bn_backward_grid
from stoke_b200.fuse import BnAct, fuse_bn_act, site_shapes

pytestmark = pytest.mark.gpu

GUARD = 4096
ACTS = {ACT_SILU: F.silu, ACT_HARDSWISH: F.hardswish, ACT_RELU6: F.relu6, ACT_RELU: torch.relu}
ACT_BACKWARD = {
    ACT_SILU: lambda g, y: torch.ops.aten.silu_backward(g, y),
    ACT_HARDSWISH: lambda g, y: torch.ops.aten.hardswish_backward(g, y),
    ACT_RELU6: lambda g, y: torch.ops.aten.hardtanh_backward(g, y, 0, 6),
    ACT_RELU: lambda g, y: torch.ops.aten.threshold_backward(g, F.relu(y), 0),
}
ACT_MODULES = {ACT_SILU: torch.nn.SiLU, ACT_HARDSWISH: torch.nn.Hardswish, ACT_RELU6: torch.nn.ReLU6}
NEW_ACTS = [ACT_SILU, ACT_HARDSWISH, ACT_RELU6]


def _bits(t):
    return t.contiguous().view({torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int64: torch.int64}[t.dtype])


def assert_same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    diff = _bits(a) != _bits(b)
    if bool(diff.any()):
        i = diff.reshape(-1).nonzero()[:8].reshape(-1)
        got = _bits(a).reshape(-1)[i].tolist()
        want = _bits(b).reshape(-1)[i].tolist()
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ; first (index, got, want): "
                             f"{[(int(k), hex(u & 0xFFFFFFFF), hex(v & 0xFFFFFFFF)) for k, u, v in zip(i, got, want)]}")


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


def _check_guards(raws):
    for raw in raws:
        assert bool((raw[:GUARD] == 0xFF).all()) and bool((raw[-GUARD:] == 0xFF).all()), "guard band written"


# ---- exhaustive ------------------------------------------------------------------------------------------------------
def _all_bf16(repeat=1):
    """every bf16 bit pattern, `repeat` times, as a (8192 * repeat, 8, 1, 1) channels-last tensor"""
    bits = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).repeat(repeat)
    return bits.view(torch.bfloat16).view(-1, 8, 1, 1).contiguous(memory_format=torch.channels_last)


def _identity_bn():
    """mean 0, var 1, eps 0, weight 1, bias -0.0: y = fma(1 * (x - 0), 1, -0) = x, -0 kept (a +0 bias would make it +0)"""
    mean, var = torch.zeros(8, device="cuda"), torch.ones(8, device="cuda")
    w = torch.ones(8, device="cuda", dtype=torch.bfloat16)
    b = torch.full((8,), -0.0, device="cuda", dtype=torch.bfloat16)
    return mean, var, w, b


def _torch_y(x, mean, var, w, b):
    """torch's BatchNorm transform of x: x itself except that a NaN becomes the canonical NaN"""
    y = torch.batch_norm_elemt(x, w, b, mean, torch.rsqrt(var), 0.0)
    nan = x.isnan()
    assert torch.equal(_bits(y)[~nan], _bits(x)[~nan]) and bool(y[nan].isnan().all())
    return y


@pytest.mark.parametrize("act", NEW_ACTS)
def test_exhaustive_forward(eng, act):
    x = _all_bf16()
    mean, var, w, b = _identity_bn()
    y = _torch_y(x, mean, var, w, b)
    out_raw, out = _guarded(x.numel(), torch.bfloat16, x)
    inv_raw, invstd = _guarded(8, torch.float32)
    eng.bn_act(x, None, mean, var, w, b, 0.0, out, invstd, act)
    torch.cuda.synchronize()
    _check_guards([out_raw, inv_raw])
    assert bool((invstd == 1).all())
    assert_same(out, ACTS[act](y), "out")


def _gradients():
    """64 bf16 gradients: +-0, +-inf, NaNs with and without a payload and sign, subnormals, extremes, random values"""
    special = [0x0000, 0x8000, 0x7F80, 0xFF80, 0x7FC0, 0xFFC0, 0x7FC1, 0xFF81, 0x0001, 0x8001, 0x007F, 0x807F,
               0x0080, 0x8080, 0x7F7F, 0xFF7F, 0x3F80, 0xBF80, 0x3F00, 0x4040]
    g = torch.Generator().manual_seed(5)
    rnd = (torch.randn(44, generator=g) * torch.exp2(torch.randint(-20, 20, (44,), generator=g).float()))
    bits = torch.tensor(special, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    return torch.cat([bits, rnd.to(torch.bfloat16)]).cuda()


@pytest.mark.parametrize("act", NEW_ACTS)
def test_exhaustive_derivative(eng, act):
    grads = _gradients()
    k = grads.numel()
    x = _all_bf16(k)
    mean, var, w, b = _identity_bn()
    y = _torch_y(x, mean, var, w, b)
    gy = grads.repeat_interleave(65536).view(x.shape).contiguous(memory_format=torch.channels_last)
    ref = ACT_BACKWARD[act](gy, y)
    invstd = torch.ones(8, device="cuda")
    pre_raw, pre = _guarded(x.numel(), torch.bfloat16, x)
    dw, db = torch.empty_like(w), torch.empty_like(w)
    eng.bn_act_backward(gy, x, None, mean, invstd, w, b, None, dw, db, None, act, pre)
    torch.cuda.synchronize()
    _check_guards([pre_raw])
    assert_same(pre, ref, "grad_pre")


# ---- against the unfused chain ---------------------------------------------------------------------------------------
def _model_cases():
    """every fused site shape at B = 128, 224 x 224, found by running the rewritten models on the meta device (no
    arithmetic, so collection stays cheap), plus odd shapes"""
    import torchvision

    cases = set()
    for name in ("efficientnet_b0", "mobilenet_v3_large", "mobilenet_v2"):
        with torch.device("meta"):
            sites = site_shapes(fuse_bn_act(getattr(torchvision.models, name)(), None), torch.empty(2, 3, 224, 224))
        for (act, c, h, w, eps, momentum) in sites:
            cases.add((act, (128, c, h, w), eps, momentum))
    for act in NEW_ACTS:
        for shape in [(3, 8, 5, 5), (3, 24, 5, 5), (2, 24, 1, 3), (5, 8, 7, 3), (16, 200, 20, 20), (32, 16, 65, 63)]:
            cases.add((act, shape, 1e-5, 0.1))
    return sorted(cases)


CASES = _model_cases()
SPECIAL = ["none", "infnan", "negzero"]


def test_cases_cover_padded_reduce_rows():
    """the reduce pads a channel's rows to a multiple of block_y * grid_y * 4 with g = x = 0, which the overflow test
    below needs, both with one block per channel and with several"""
    grids = [bn_backward_grid(s[0] * s[2] * s[3], s[1])[1] for s in PADDED_SHAPES]
    assert all(_padded(s) for s in PADDED_SHAPES)
    assert any(g == 1 for g in grids) and any(g > 1 for g in grids)


def _inputs(shape, special, seed):
    n, c, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(shape, device="cuda", generator=g) * 2 + 0.5).to(torch.bfloat16)
    gy = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    if special == "negzero":   # channel 0 all zero: (x - mean) * weight = +0 * -1 = -0, + bias -0 (_bn); -0 gradients
        x[:, 0] = 0.0
        gy[:, c // 2] = -0.0
        gy.view(-1)[::7] = -0.0
    if special == "infnan":    # inf / NaN in x (those channels' statistics become NaN) and scattered through grad
        x[0, c - 1, 0, 0] = float("inf")
        x[n - 1, 0, h - 1, w - 1] = float("nan")
        flat = gy.view(-1)
        flat[1::97] = float("nan")
        flat[2::89] = float("inf")
        flat[3::83] = float("-inf")
    cl = torch.channels_last
    return x.contiguous(memory_format=cl), gy.contiguous(memory_format=cl)


def _bn(c, seed, special="none", eps=1e-5, momentum=0.1):
    g = torch.Generator().manual_seed(seed)
    bn = torch.nn.BatchNorm2d(c, eps=eps, momentum=momentum)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) * 2 + 0.5)
        bn.bias.copy_(torch.rand(c, generator=g) * 4 - 2)
        if special == "negzero":
            bn.weight[0], bn.bias[0] = -1.0, -0.0
        bn.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn.to(device="cuda", dtype=torch.bfloat16)


@pytest.mark.parametrize("special", SPECIAL)
@pytest.mark.parametrize("act,shape,eps,momentum", CASES)
def test_entry_points_against_unfused(eng, act, shape, eps, momentum, special):
    c = shape[1]
    x, gy = _inputs(shape, special, seed=c + shape[2])
    bn = _bn(c, seed=c, special=special, eps=eps, momentum=momentum)
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    y, ref_mean, ref_invstd = torch.ops.aten.native_batch_norm(x, bn.weight, bn.bias, rm, rv, True, momentum, eps)
    if special == "negzero":
        assert bool((_bits(y[:, 0]) == -32768).all())
    ref_out = ACTS[act](y)
    g = ACT_BACKWARD[act](gy, y)
    assert g.is_contiguous(memory_format=torch.channels_last)
    ref_dx, ref_dw, ref_db = torch.ops.aten.native_batch_norm_backward(g, x, bn.weight, rm, rv, ref_mean, ref_invstd,
                                                                      True, eps, [True, True, True])

    mean, var = torch.batch_norm_update_stats(x, bn.running_mean.clone(), bn.running_var.clone(), momentum)
    (out_raw, out), (inv_raw, invstd) = _guarded(x.numel(), torch.bfloat16, x), _guarded(c, torch.float32)
    eng.bn_act(x, None, mean, var, bn.weight, bn.bias, eps, out, invstd, act)
    bufs = [_guarded(x.numel(), torch.bfloat16, x), _guarded(c, torch.bfloat16), _guarded(c, torch.bfloat16)]
    (_, dx), (_, dw), (_, db) = bufs
    eng.bn_act_backward(gy, x, None, mean, invstd, bn.weight, bn.bias, dx, dw, db, None, act)
    torch.cuda.synchronize()
    _check_guards([out_raw, inv_raw] + [raw for raw, _ in bufs])
    assert_same(out, ref_out, "out")
    assert_same(mean, ref_mean, "save_mean")
    assert_same(invstd, ref_invstd, "save_invstd")
    assert_same(dx, ref_dx, "dx")
    assert_same(dw, ref_dw, "dweight")
    assert_same(db, ref_db, "dbias")


def _padded(shape):
    rows = shape[0] * shape[2] * shape[3]
    block_y, grid_y, _ = bn_backward_grid(rows, shape[1])
    return rows % (block_y * grid_y * 4) != 0


PADDED_SHAPES = sorted({s for _, s, _, _ in CASES if _padded(s)})


@pytest.mark.parametrize("shape", PADDED_SHAPES)
@pytest.mark.parametrize("act", NEW_ACTS + [ACT_RELU])
def test_padded_rows_where_the_activation_input_overflows(eng, act, shape):
    """A channel whose statistics are finite but whose BatchNorm maps x = 0 to +-inf: x held at 2^33 (mean 2^33, var 0)
    under a weight of 1e28, so every real y is the bias while bn_apply(0) = -1e28 * 2^33 * rsqrt(eps) overflows.  The
    reduce's padded rows must still add g = +0 (SiLU's backward of a zero gradient at y = -inf is NaN).  The statistics
    are given, not reduced, so the case does not depend on how exactly torch's reduction averages a constant; torch's
    backward takes the same mean and invstd."""
    n, c, h, w = shape
    eps = 1e-5
    x, gy = _inputs(shape, "none", seed=c + h)
    x[:, c - 1] = 2.0 ** 33
    bn = _bn(c, seed=c)
    with torch.no_grad():
        bn.weight[c - 1] = 1e28
    mean, var = torch.batch_norm_update_stats(x, bn.running_mean.clone(), bn.running_var.clone(), 0.1)
    mean[c - 1], var[c - 1] = 2.0 ** 33, 0.0
    (out_raw, out), (inv_raw, invstd) = _guarded(x.numel(), torch.bfloat16, x), _guarded(c, torch.float32)
    eng.bn_act(x, None, mean, var, bn.weight, bn.bias, eps, out, invstd, act)
    bufs = [_guarded(x.numel(), torch.bfloat16, x), _guarded(c, torch.bfloat16), _guarded(c, torch.bfloat16)]
    (_, dx), (_, dw), (_, db) = bufs
    eng.bn_act_backward(gy, x, None, mean, invstd, bn.weight, bn.bias, dx, dw, db, None, act)
    torch.cuda.synchronize()
    _check_guards([out_raw, inv_raw] + [raw for raw, _ in bufs])

    y = torch.batch_norm_elemt(x, bn.weight, bn.bias, mean, invstd, eps)
    k = c - 1
    pad = (bn.weight[k].float() * (0 - mean[k]) * invstd[k] + bn.bias[k].float()).to(torch.bfloat16)
    assert bool(pad.isinf()) and bool((y[:, k] == bn.bias[k]).all())
    g = ACT_BACKWARD[act](gy, y)
    ref_dx, ref_dw, ref_db = torch.ops.aten.native_batch_norm_backward(g, x, bn.weight, None, None, mean, invstd, True,
                                                                      eps, [True, True, True])
    assert bool(ref_db.isfinite().all()) and bool(ref_dw.isfinite().all())
    assert_same(out, ACTS[act](y), "out")
    assert_same(dx, ref_dx, "dx")
    assert_same(dw, ref_dw, "dweight")
    assert_same(db, ref_db, "dbias")


def test_residual_and_relu_grad_pre_are_rejected(eng):
    from stoke_b200._lib import StokeB200Error

    x, gy = _inputs((2, 8, 4, 4), "none", 0)
    bn = _bn(8, 0)
    mean, var = torch.batch_norm_update_stats(x, bn.running_mean.clone(), bn.running_var.clone(), 0.1)
    out, invstd = torch.empty_like(x), torch.empty_like(mean)
    with pytest.raises(StokeB200Error):
        eng.bn_act(x, x, mean, var, bn.weight, bn.bias, 1e-5, out, invstd, ACT_SILU)
    eng.bn_act(x, None, mean, var, bn.weight, bn.bias, 1e-5, out, invstd, ACT_SILU)
    dw, db = torch.empty_like(bn.weight), torch.empty_like(bn.weight)
    with pytest.raises(StokeB200Error):
        eng.bn_act_backward(gy, x, None, mean, invstd, bn.weight, bn.bias, None, dw, db, None, ACT_RELU,
                            torch.empty_like(x))
    with pytest.raises(StokeB200Error):
        eng.bn_act_backward(gy, x, None, mean, invstd, bn.weight, bn.bias, None, dw, db, None, 9)
    torch.cuda.synchronize()


# ---- the module ------------------------------------------------------------------------------------------------------
def _layout(gy, layout):
    if layout == "nchw":
        return gy.contiguous()
    if layout == "expanded":   # what the average pool's backward passes on: one value per (n, c), strides (C, 1, 0, 0)
        return gy[:, :, :1, :1].expand(gy.shape)
    if layout == "misaligned":  # channels-last, 2 bytes off the 16-byte alignment the kernels need
        n, c, h, w = gy.shape
        buf = torch.empty(gy.numel() + 1, dtype=gy.dtype, device=gy.device)
        t = buf[1:].view(n, h, w, c).permute(0, 3, 1, 2)
        t.copy_(gy)
        return t
    return gy


@pytest.mark.parametrize("layout", ["channels_last", "nchw", "expanded", "misaligned"])
@pytest.mark.parametrize("shape", [(3, 24, 5, 5), (16, 200, 20, 20), (128, 240, 14, 14)])
@pytest.mark.parametrize("act", NEW_ACTS)
def test_module_against_unfused(eng, act, shape, layout):
    c = shape[1]
    eps, momentum = (1e-3, 0.01) if act == ACT_HARDSWISH else (1e-5, 0.1)
    ref_bn, my_bn = _bn(c, c + 1, eps=eps, momentum=momentum), _bn(c, c + 1, eps=eps, momentum=momentum)
    ref_act = ACT_MODULES[act](inplace=True)
    fused = BnAct(my_bn, eng, act=act, act_fn=ACT_MODULES[act](inplace=True))
    for step in range(2):
        x, gy = _inputs(shape, "none", seed=step * 1000 + c)
        gy = _layout(gy, layout)
        xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
        a = ref_act(ref_bn(xa))
        launches = eng.launches
        b = fused(xb)
        assert eng.launches == launches + 1, "the kernel did not run (BnAct took the unfused fallback)"
        assert_same(b, a, "out")
        a.backward(gy)
        launches = eng.launches
        b.backward(gy)
        # torch's BatchNorm backward runs its channels-last kernels when the activation backward's output is
        # channels-last: all three backward ops keep an NCHW gradient's layout and make an expanded one channels-last
        cl_backward = layout in ("channels_last", "expanded")
        kernels = 2 + (bn_backward_grid(x.numel() // c, c)[1] > 1) if cl_backward else 0
        assert eng.launches == launches + kernels
        assert_same(xb.grad, xa.grad, "dx")
        assert_same(my_bn.weight.grad, ref_bn.weight.grad, "dweight")
        assert_same(my_bn.bias.grad, ref_bn.bias.grad, "dbias")
        assert_same(my_bn.running_mean, ref_bn.running_mean, "running_mean")
        assert_same(my_bn.running_var, ref_bn.running_var, "running_var")
        assert_same(my_bn.num_batches_tracked, ref_bn.num_batches_tracked, "num_batches_tracked")


# ---- whole models ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["efficientnet_b0", "mobilenet_v3_small"])
def test_whole_model_against_unrewritten(eng, name, monkeypatch):
    import torchvision

    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        torch.manual_seed(0)
        ref = getattr(torchvision.models, name)(num_classes=100)
        for m in ref.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                torch.nn.init.uniform_(m.weight, 0.5, 1.5)
                torch.nn.init.uniform_(m.bias, -0.5, 0.5)
        ref = ref.to(device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
        mine = copy.deepcopy(ref)
        fwd = fuse_bn_act(mine, eng)
        assert fwd is not None and fwd.fused_sites > 0
        lossf = torch.nn.CrossEntropyLoss()
        g = torch.Generator(device="cuda").manual_seed(1)
        for _ in range(2):
            x = torch.randn(32, 3, 160, 160, device="cuda", generator=g).to(torch.bfloat16)
            x = x.contiguous(memory_format=torch.channels_last)
            y = torch.randint(0, 100, (32,), device="cuda", generator=g)
            torch.manual_seed(7)   # dropout and stochastic depth draw the same masks in both models
            la = lossf(ref(x).float(), y)
            launches = eng.launches
            torch.manual_seed(7)
            lb = lossf(fwd(x).float(), y)
            assert eng.launches - launches == fwd.fused_sites
            la.backward()
            lb.backward()
            assert_same(lb.detach(), la.detach(), "loss")
            for (pname, p), q in zip(ref.named_parameters(), mine.parameters()):
                assert_same(q.grad, p.grad, pname)
            for (bname, u), v in zip(ref.named_buffers(), mine.buffers()):
                assert_same(v, u, bname)
    finally:
        torch.use_deterministic_algorithms(det)
