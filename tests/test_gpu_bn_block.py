"""The ResNet block boundary at the residual site (stoke_b200/fuse.py), bit for bit against the unfused torch modules.

The two-BatchNorm site (BnAct with ``residual_bn``): relu(bn(a) + bn_ds(b)) in one forward launch and the three backward
kernels, at the four ResNet-50 downsample shapes at B = 128 and odd shapes (grid_y 1 and > 1), fp32 and bf16 running
statistics, inf / NaN and -0.0, different eps / momentum on the two BatchNorms, and its fallback.

The forked residual site (BnAct with ``fork``): a block output with two users returns two tensors over one storage, and
the backward adds the users' two gradients inside k_bn_bwd_reduce as autograd's bf16 add would, against the unfused
module whose output autograd sums.

* The site at the ResNet-50 block-output shapes at B = 128 and odd shapes on both sides of grid_y = 1, with inf / NaN
  and -0.0 in the gradients.
* The aliasing: the two outputs share storage, and the backward runs the three k_bn_bwd kernels and nothing else (no
  copy, no add).
* The fallbacks: one gradient not channels-last, or one gradient absent.
* Whole ResNet-18 and ResNet-50, rewritten against unrewritten, over two steps."""
import copy

import pytest
import torch

from stoke_b200.engine import bn_backward_grid
from stoke_b200.fuse import BnAct, fuse_bn_act

from test_gpu_bn_bwd import _bn, _inputs, assert_same

pytestmark = pytest.mark.gpu

SHAPES = [
    (3, 8, 5, 5),         # grid_y 1
    (4, 200, 9, 9),       # grid_y 1, C not a power of two
    (16, 200, 20, 20),    # grid_y 25
    (128, 256, 56, 56),   # the ResNet-50 block outputs at B = 128
    (128, 512, 28, 28),
    (128, 1024, 14, 14),
    (128, 2048, 7, 7),
]


@pytest.fixture
def eng():
    from stoke_b200.engine import get_engine

    torch.cuda.set_device(0)
    return get_engine(0)


def _pair(shape, special):
    c = shape[1]
    x, r, g0 = _inputs(shape, special, seed=c + shape[2])
    _, _, g1 = _inputs(shape, special, seed=c + shape[2] + 1)
    if special == "negzero":   # -0 + -0 stays -0, -0 + +0 becomes +0
        g1[:, c // 2] = -0.0
        g1[:, c // 2 + 1] = 0.0
    return x, r, g0, g1


def _run(eng, shape, special, grads, fork=True):
    """(reference module, fused module, their inputs): the unfused site receives grads on its single output twice
    (autograd sums them), the forked one on its two outputs"""
    c = shape[1]
    ref_bn, my_bn = _bn(c, c + 1, "none"), _bn(c, c + 1, "none")
    x, r, _, _ = _pair(shape, special)
    xa, ra = x.clone().requires_grad_(), r.clone().requires_grad_()
    xb, rb = x.clone().requires_grad_(), r.clone().requires_grad_()
    out = ref_bn(xa)
    out += ra
    a = torch.relu_(out)
    fused = BnAct(my_bn, eng, fork=fork)
    b = fused(xb, rb)
    keep = [i for i, g in enumerate(grads) if g is not None]
    torch.autograd.backward([a] * len(keep), [grads[i] for i in keep])
    return (a, xa, ra, ref_bn), (b, xb, rb, my_bn), keep


def _check(ref, mine):
    (a, xa, ra, ref_bn), (b, xb, rb, my_bn) = ref, mine
    assert_same(b[0], a, "out")
    assert_same(xb.grad, xa.grad, "dx")
    assert_same(rb.grad, ra.grad, "dresidual")
    assert_same(my_bn.weight.grad, ref_bn.weight.grad, "dweight")
    assert_same(my_bn.bias.grad, ref_bn.bias.grad, "dbias")
    assert_same(my_bn.running_mean, ref_bn.running_mean, "running_mean")
    assert_same(my_bn.running_var, ref_bn.running_var, "running_var")


@pytest.mark.parametrize("special", ["none", "infnan", "negzero"])
@pytest.mark.parametrize("shape", SHAPES)
def test_forked_site(eng, shape, special):
    _, _, g0, g1 = _pair(shape, special)
    ref, mine, _ = _run(eng, shape, special, [g0, g1])
    b = mine[0]
    assert b[0].data_ptr() == b[1].data_ptr() and b[0].grad_fn is b[1].grad_fn
    launches = eng.launches
    torch.autograd.backward(list(b), [g0, g1])
    assert eng.launches == launches + 2 + (bn_backward_grid(g0.numel() // shape[1], shape[1])[1] > 1)
    _check(ref, mine)


def test_backward_runs_only_the_kernels(eng):
    """No copy of the aliased output and no add of the two gradients: the three k_bn_bwd kernels are all that run."""
    shape = (16, 200, 20, 20)
    _, _, g0, g1 = _pair(shape, "none")
    _, mine, _ = _run(eng, shape, "none", [g0, g1])
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch.autograd.backward(list(mine[0]), [g0, g1])
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
             and "memset" not in e.name.lower() and "memcpy" not in e.name.lower()]
    assert names and all("k_bn_bwd_" in n for n in names), names
    assert any("k_bn_bwd_reduce<0, true, true, false>" in n for n in names), names


@pytest.mark.parametrize("case", ["nchw", "none0", "none1"])
@pytest.mark.parametrize("shape", [(4, 200, 9, 9), (16, 200, 20, 20)])
def test_fallbacks(eng, shape, case):
    _, _, g0, g1 = _pair(shape, "none")
    grads = {"nchw": [g0, g1.contiguous()], "none0": [None, g1], "none1": [g0, None]}[case]
    ref, mine, keep = _run(eng, shape, "none", grads)
    b = mine[0]
    torch.autograd.backward([b[i] for i in keep], [grads[i] for i in keep])
    _check(ref, mine)


TWO_BN_SHAPES = [
    (3, 8, 5, 5),         # grid_y 1
    (16, 200, 20, 20),    # grid_y 25
    (128, 256, 56, 56),   # the four ResNet-50 downsample sites at B = 128
    (128, 512, 28, 28),
    (128, 1024, 14, 14),
    (128, 2048, 7, 7),
]


def _bn2(c, seed, run_dtype, eps, momentum):
    bn = _bn(c, seed, "none")
    bn.eps, bn.momentum = eps, momentum
    bn.running_mean = bn.running_mean.to(run_dtype)
    bn.running_var = bn.running_var.to(run_dtype)
    return bn


@pytest.mark.parametrize("run_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("special", ["none", "infnan", "negzero"])
@pytest.mark.parametrize("shape", TWO_BN_SHAPES)
def test_two_batchnorm_site(eng, shape, special, run_dtype):
    """relu(bn(a) + bn_ds(b)) in one launch (different eps / momentum on the two BatchNorms), forked and not, over two
    steps: out, both running statistics and num_batches_tracked, both inputs' gradients and all four parameter gradients"""
    if special != "none" and shape[0] == 128 and shape[1] != 2048:
        pytest.skip("special values at the smaller shapes and 2048 x 7^2")
    c = shape[1]
    mods = [(_bn2(c, c + 1, run_dtype, 1e-5, 0.1), _bn2(c, c + 2, run_dtype, 1e-3, None)) for _ in range(2)]
    (ref_bn, ref_ds), (my_bn, my_ds) = mods
    for step, fork in enumerate((False, True)):
        a, b, g0, g1 = _pair(shape, special)
        if step:
            a, b = b, a
        aa, ba = a.clone().requires_grad_(), b.clone().requires_grad_()
        ab, bb = a.clone().requires_grad_(), b.clone().requires_grad_()
        out = ref_bn(aa)
        out += ref_ds(ba)
        ref = torch.relu_(out)
        launches = eng.launches
        mine = BnAct(my_bn, eng, inplace=True, residual_bn=my_ds, fork=fork)(ab, bb)
        assert eng.launches == launches + 1, "the kernel did not run"
        outs = list(mine) if fork else [mine]
        assert_same(outs[0], ref, "out")
        torch.autograd.backward([ref, ref] if fork else [ref], [g0, g1] if fork else [g0])
        launches = eng.launches
        torch.autograd.backward(outs, [g0, g1] if fork else [g0])
        assert eng.launches == launches + 2 + (bn_backward_grid(a.numel() // c, c)[1] > 1), "the kernels did not run"
        assert_same(ab.grad, aa.grad, "da")
        assert_same(bb.grad, ba.grad, "db")
        for (mb, rb), what in (((my_bn, ref_bn), "bn"), ((my_ds, ref_ds), "downsample")):
            assert_same(mb.weight.grad, rb.weight.grad, f"{what} dweight")
            assert_same(mb.bias.grad, rb.bias.grad, f"{what} dbias")
            assert_same(mb.running_mean, rb.running_mean, f"{what} running_mean")
            assert_same(mb.running_var, rb.running_var, f"{what} running_var")
            assert torch.equal(mb.num_batches_tracked, rb.num_batches_tracked), what
            mb.weight.grad = mb.bias.grad = rb.weight.grad = rb.bias.grad = None


@pytest.mark.parametrize("shape", [(3, 8, 5, 5), (16, 200, 20, 20), (128, 2048, 7, 7)])
def test_two_batchnorm_save_statistics(eng, shape):
    """stk_bn_stats_act's save_mean / save_invstd for both BatchNorms against native_batch_norm's"""
    c = shape[1]
    a, b, _, _ = _pair(shape, "infnan")
    bn, ds = _bn2(c, 1, torch.float32, 1e-5, 0.1), _bn2(c, 2, torch.float32, 1e-3, 0.3)
    out = torch.empty_like(a)
    sm, si, sm2, si2 = (torch.empty(c, device="cuda") for _ in range(4))
    eng.bn_stats_act(a, b, bn.weight, bn.bias, bn.running_mean, bn.running_var, 0.1, 1e-5, out, sm, si,
                     residual_bn=(ds.weight, ds.bias, ds.running_mean, ds.running_var, 0.3, 1e-3, sm2, si2))
    for x, m, s, mean, invstd, eps in ((a, bn, "bn", sm, si, 1e-5), (b, ds, "downsample", sm2, si2, 1e-3)):
        _, rmean, rinv = torch.native_batch_norm(x, m.weight, m.bias, None, None, True, 0.1, eps)
        assert_same(mean, rmean, f"{s} save_mean")
        assert_same(invstd, rinv, f"{s} save_invstd")


@pytest.mark.parametrize("case", ["second_not_covered", "dtypes_differ"])
def test_two_batchnorm_fallback(eng, case):
    """only the first BatchNorm covered: the residual BatchNorm runs in torch, the site on its output"""
    shape = (16, 200, 20, 20)
    c = shape[1]
    run2 = torch.bfloat16 if case == "dtypes_differ" else torch.float32
    (ref_bn, ref_ds), (my_bn, my_ds) = [(_bn2(c, 1, torch.float32, 1e-5, 0.1), _bn2(c, 2, run2, 1e-3, 0.2))
                                        for _ in range(2)]
    if case == "second_not_covered":
        ref_ds.eval(), my_ds.eval()
    a, b, g0, _ = _pair(shape, "none")
    aa, ba, ab, bb = (t.clone().requires_grad_() for t in (a, b, a, b))
    out = ref_bn(aa)
    out += ref_ds(ba)
    ref = torch.relu_(out)
    mine = BnAct(my_bn, eng, inplace=True, residual_bn=my_ds)(ab, bb)
    assert_same(mine, ref, "out")
    ref.backward(g0)
    mine.backward(g0)
    assert_same(ab.grad, aa.grad, "da")
    assert_same(bb.grad, ba.grad, "db")
    for mb, rb in ((my_bn, ref_bn), (my_ds, ref_ds)):
        assert_same(mb.weight.grad, rb.weight.grad, "dweight")
        assert_same(mb.running_var, rb.running_var, "running_var")


@pytest.mark.parametrize("name,forks", [("resnet18", 7), ("resnet50", 15)])
def test_resnet_against_unrewritten(eng, monkeypatch, name, forks):
    import torchvision

    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        torch.manual_seed(0)
        ref = getattr(torchvision.models, name)()
        for m in ref.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                torch.nn.init.uniform_(m.weight, 0.5, 1.5)
                torch.nn.init.uniform_(m.bias, -0.5, 0.5)
        ref = ref.to(device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
        mine = copy.deepcopy(ref)
        fwd = fuse_bn_act(mine, eng)
        assert sum(isinstance(m, BnAct) and m.fork for m in fwd.graph_module.modules()) == forks
        lossf = torch.nn.CrossEntropyLoss()
        g = torch.Generator(device="cuda").manual_seed(1)
        for _ in range(2):
            x = torch.randn(32, 3, 224, 224, device="cuda", generator=g).to(torch.bfloat16)
            x = x.contiguous(memory_format=torch.channels_last)
            y = torch.randint(0, 1000, (32,), device="cuda", generator=g)
            la = lossf(ref(x).float(), y)
            lb = lossf(fwd(x).float(), y)
            la.backward()
            lb.backward()
            assert_same(lb.detach(), la.detach(), "loss")
            for (pname, p), q in zip(ref.named_parameters(), mine.parameters()):
                assert_same(q.grad, p.grad, pname)
            for (bname, u), v in zip(ref.named_buffers(), mine.buffers()):
                assert torch.equal(u, v), bname
    finally:
        torch.use_deterministic_algorithms(det)
