"""The gradient windows of tests/grad_window_ref.py are exact at every stage of the gradient pipeline (CPU).

The bit-identity tests of tests/test_gpu_grad_window.py rest on this: an accumulated, loss-scaled window and one bucket
holding its sum are the same fp32 values only if no stage rounds.  Checked here for the windows those tests use: every
micro value, partial sum and window total is exact in bf16; times a power-of-two scale too; and the fp32 pipeline
x = ((g + acc) * mul) * 1/scale (kernel_ref.scaled_grad_f32, the kernels' order) equals its float64 value
(kernel_ref.scaled_grad) bit for bit, which is the window total."""
import pytest
import torch

import grad_window_ref as gw
import kernel_ref as kr

NUMELS = [36864, 2048, 851, 385, 1000, 1, 16770]   # the parameter sizes of the GPU tests (+ odd ones)
SCALES = [1.0, 2.0**12, 2.0**13]


@pytest.mark.parametrize("micro", [1, 2, 3])
@pytest.mark.parametrize("seed", [0, 1, 7])
def test_window_partial_sums_exact_in_bf16(micro, seed):
    win = gw.window(NUMELS, micro, seed)
    for micros in win:
        assert len(micros) == micro
        run = torch.zeros_like(micros[0], dtype=torch.float64)
        for m in micros:
            assert m.dtype == torch.float32
            run += m.double()
            for s in SCALES:
                assert gw.exact_in(m * s, torch.bfloat16)
                assert gw.exact_in(run * s, torch.bfloat16)
        assert torch.equal(gw.total(micros).double(), run)
        assert gw.exact_in(gw.total(micros), torch.bfloat16)


@pytest.mark.parametrize("micro", [2, 3])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("scale", SCALES)
def test_scaled_pipeline_is_exact(micro, dtype, scale):
    """The last micro-batch in the model-dtype bucket, the earlier ones summed in the fp32 accumulator, both loss-scaled:
    the fp32 pipeline gives the float64 value, and that value is the unscaled window total."""
    inv = kr.inv_scale_f32(scale)
    assert inv * scale == 1.0   # a power of two: the unscale is exact
    for seed in range(3):
        for micros in gw.window(NUMELS, micro, seed):
            acc = torch.zeros_like(micros[0])
            for m in micros[:-1]:
                acc += m * scale   # the accumulate kernel's fp32 adds
            g = (micros[-1] * scale).to(dtype)
            x32 = kr.scaled_grad_f32(g, acc, 1.0, inv)
            x64, _ = kr.scaled_grad(g, acc, 1.0, inv)
            assert torch.equal(x32.double(), x64)
            assert torch.equal(x32.view(torch.int32), gw.total(micros).view(torch.int32))


def test_exponents_differ_between_parameters():
    win = gw.window([64] * 40, 2, 3)
    exps = {int(torch.frexp(m[0].abs().max())[1]) for m in win}
    assert len(exps) >= 3


def test_bound_is_tight():
    """One step past the window's range is no longer exact in bf16: the construction needs its bound."""
    for e in range(gw.EXPS[0], gw.EXPS[1] + 1):
        assert gw.exact_in(torch.tensor([gw.KMAX * 2.0**-e, -gw.KMAX * 2.0**-e]), torch.bfloat16)
        assert not gw.exact_in(torch.tensor([(gw.KMAX + 1) * 2.0**-e]), torch.bfloat16)
