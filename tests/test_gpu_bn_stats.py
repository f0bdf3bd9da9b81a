"""stk_bn_stats_act (csrc/bn_act.cu): the BatchNorm forward with its batch statistics and running-statistics update in one
cooperative launch, against torch.batch_norm_update_stats followed by stk_bn_act_ex, and against native_batch_norm,
bit for bit.

* Every regime of torch's flexible_launch_configs(R, C, coop) (grid_y 1, 8 <= grid_y < 128, 128 with a partial last
  pass, block_x 8 and 16, C = 24 and 200), every fused ResNet-50 site shape at B = 128, and more than 2^24 rows (where
  the int -> float count conversion rounds).
* A constant channel, a channel at a 2^100 offset with a small spread, inf / NaN, an all-zero channel (-0 in x).
* momentum 0.1 and a cumulative average; fp32 and bf16 running statistics; all five kernel instantiations.
* BnAct: one launch per forward, bit-identical to the unfused module over two steps, and a whole ResNet-50 rewritten
  against unrewritten."""
import copy

import pytest
import torch

from stoke_b200._lib import ACT_HARDSWISH, ACT_RELU, ACT_RELU6, ACT_SILU
from stoke_b200.fuse import BnAct, fuse_bn_act

pytestmark = pytest.mark.gpu

GUARD = 4096
# the five instantiations: (act, residual)
KINDS = [(ACT_RELU, False), (ACT_RELU, True), (ACT_SILU, False), (ACT_HARDSWISH, False), (ACT_RELU6, False)]


def _bits(t):
    return t.contiguous().view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


def assert_same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    diff = _bits(a) != _bits(b)
    if bool(diff.any()):
        i = diff.reshape(-1).nonzero()[:8].reshape(-1)
        got, want = _bits(a).reshape(-1)[i].tolist(), _bits(b).reshape(-1)[i].tolist()
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


def _inputs(shape, special, seed, run_dtype):
    n, c, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, h, w, c, device="cuda", generator=g) * 2 + 0.5
    if special:
        x[..., 0] = 3.25                                                  # constant channel: var 0
        x[..., 1] = 2.0 ** 100 * (1 + x[..., 1] * 2.0 ** -6)              # huge offset, small spread
        x[..., 2] = -0.0                                                  # all -0
        x.view(-1, c)[::97, 3] = float("inf")
        x.view(-1, c)[5, 4] = float("nan")
        x.view(-1, c)[7, 5] = float("-inf")
    x = x.to(torch.bfloat16).permute(0, 3, 1, 2)
    r = (torch.randn(n, h, w, c, device="cuda", generator=g)).to(torch.bfloat16).permute(0, 3, 1, 2)
    w_ = (torch.rand(c, device="cuda", generator=g) + 0.5).to(torch.bfloat16)
    b_ = (torch.rand(c, device="cuda", generator=g) - 0.5).to(torch.bfloat16)
    rm = (torch.randn(c, device="cuda", generator=g) * 0.1).to(run_dtype)
    rv = (torch.rand(c, device="cuda", generator=g) + 0.5).to(run_dtype)
    return x, r, w_, b_, rm, rv


def _check(eng, shape, act, residual, run_dtype, momentum=0.1, special=False, eps=1e-5, seed=0, native=True):
    x, r, w, b, rm, rv = _inputs(shape, special, seed, run_dtype)
    r = r if residual else None
    c = shape[1]
    rm_ref, rv_ref = rm.clone(), rv.clone()
    mean_ref, var_ref = torch.batch_norm_update_stats(x, rm_ref, rv_ref, momentum)
    out_ref, inv_ref = torch.empty_like(x), torch.empty_like(mean_ref)
    eng.bn_act(x, r, mean_ref, var_ref, w, b, eps, out_ref, inv_ref, act)
    out_raw, out = _guarded(x.numel(), torch.bfloat16, x)
    mean_raw, mean = _guarded(c, torch.float32)
    inv_raw, inv = _guarded(c, torch.float32)
    launches = eng.launches
    eng.bn_stats_act(x, r, w, b, rm, rv, momentum, eps, out, mean, inv, act)
    assert eng.launches == launches + 1
    torch.cuda.synchronize()
    _check_guards([out_raw, mean_raw, inv_raw])
    assert_same(mean, mean_ref, "save_mean")
    assert_same(inv, inv_ref, "save_invstd")
    assert_same(rm, rm_ref, "running_mean")
    assert_same(rv, rv_ref, "running_var")
    assert_same(out, out_ref, "out")
    if native:
        # native_batch_norm wants its parameters and running statistics in one dtype
        _, nmean, ninv = torch.native_batch_norm(x, w, b, rm.to(w.dtype), rv.to(w.dtype), True, momentum, eps)
        assert_same(mean, nmean, "save_mean vs native_batch_norm")
        assert_same(inv, ninv, "save_invstd vs native_batch_norm")


REGIMES = [
    (2, 24, 5, 5),        # grid_y 1, block_x 16
    (16, 200, 20, 20),    # grid_y 25
    (37, 64, 29, 31),     # grid_y 128, partial last pass
    (64, 8, 17, 17),      # block_x 8, grid_y 19
    (32, 16, 30, 30),     # block_x 16, grid_y 57
    (3, 8, 1, 1),         # 3 rows
]


@pytest.mark.parametrize("run_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", REGIMES)
def test_regimes(eng, shape, kind, run_dtype):
    _check(eng, shape, *kind, run_dtype)


@pytest.mark.parametrize("run_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(2, 24, 5, 5), (16, 200, 20, 20), (37, 64, 29, 31)])
def test_special_values(eng, shape, run_dtype):
    _check(eng, shape, ACT_RELU, False, run_dtype, special=True, native=False)
    _check(eng, shape, ACT_SILU, False, run_dtype, special=True, momentum=1.0 / 3.0, native=False)


# every fused BatchNorm of ResNet-50 at B = 128 (the residual sites are the blocks' last BatchNorms)
RESNET50 = [(64, 112, False), (64, 56, False), (256, 56, True), (128, 56, False), (128, 28, False), (512, 28, True),
            (256, 28, False), (256, 14, False), (1024, 14, True), (512, 14, False), (512, 7, False), (2048, 7, True)]


@pytest.mark.parametrize("c,hw,residual", RESNET50)
def test_resnet50_sites(eng, c, hw, residual):
    _check(eng, (128, c, hw, hw), ACT_RELU, residual, torch.float32, seed=c + hw)


def test_count_rounding(eng):
    """R > 2^24: the counts of the cross-block merge no longer convert to float exactly"""
    shape = (256, 8, 256, 260)
    assert shape[0] * shape[2] * shape[3] > 2 ** 24
    _check(eng, shape, ACT_RELU, False, torch.float32, native=False)


def _bn(c, seed, momentum, run_dtype):
    torch.manual_seed(seed)
    bn = torch.nn.BatchNorm2d(c, momentum=momentum)
    torch.nn.init.uniform_(bn.weight, 0.5, 1.5)
    torch.nn.init.uniform_(bn.bias, -0.5, 0.5)
    bn = bn.to(device="cuda", dtype=torch.bfloat16)
    bn.running_mean = bn.running_mean.to(run_dtype)
    bn.running_var = bn.running_var.to(run_dtype)
    return bn


@pytest.mark.parametrize("run_dtype", [torch.bfloat16])
@pytest.mark.parametrize("momentum", [0.1, None])
@pytest.mark.parametrize("kind", KINDS)
def test_module_one_launch(eng, kind, momentum, run_dtype):
    act, residual = kind
    shape = (16, 200, 20, 20)
    ref_bn, my_bn = _bn(200, 3, momentum, run_dtype), _bn(200, 3, momentum, run_dtype)
    fused = BnAct(my_bn, eng, act=act)
    for step in range(2):
        x, r, *_ = _inputs(shape, False, step, run_dtype)
        r = r if residual else None
        gy = torch.randn(shape, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
        y = ref_bn(xa)
        a = BnAct(ref_bn, eng, act=act)._act_fn(y + r if residual else y)
        launches = eng.launches
        b = fused(xb, r)
        assert eng.launches == launches + 1, "the kernel did not run (BnAct took the unfused fallback)"
        assert_same(b, a, "out")
        a.backward(gy)
        b.backward(gy)
        assert_same(xb.grad, xa.grad, "dx")
        assert_same(my_bn.running_mean, ref_bn.running_mean, "running_mean")
        assert_same(my_bn.running_var, ref_bn.running_var, "running_var")
        assert torch.equal(my_bn.num_batches_tracked, ref_bn.num_batches_tracked), "num_batches_tracked"


def test_resnet50_against_unrewritten(eng, monkeypatch):
    from stoke_b200 import synthetic

    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        torch.manual_seed(0)
        ref = synthetic.resnet50().to(device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
        mine = copy.deepcopy(ref)
        fwd = fuse_bn_act(mine, eng)
        assert fwd is not None and fwd.fused_sites == 49
        lossf = torch.nn.CrossEntropyLoss()
        g = torch.Generator(device="cuda").manual_seed(1)
        for _ in range(2):
            x = torch.randn(32, 3, 224, 224, device="cuda", generator=g).to(torch.bfloat16)
            x = x.contiguous(memory_format=torch.channels_last)
            y = torch.randint(0, 1000, (32,), device="cuda", generator=g)
            la = lossf(ref(x).float(), y)
            launches = eng.launches
            lb = lossf(fwd(x).float(), y)
            assert eng.launches - launches == fwd.fused_sites
            la.backward()
            lb.backward()
            assert_same(lb.detach(), la.detach(), "loss")
            for (pname, p), q in zip(ref.named_parameters(), mine.parameters()):
                assert_same(q.grad, p.grad, pname)
            for (bname, u), v in zip(ref.named_buffers(), mine.buffers()):
                if v.dtype != torch.int64:
                    assert_same(v, u, bname)
    finally:
        torch.use_deterministic_algorithms(det)

