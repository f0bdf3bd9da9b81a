"""Weight averaging (EMA / SWA) without a GPU: WeightAverageConfig validation, and the host schedule against
torch.optim.swa_utils.AveragedModel.update_parameters on CPU tensors.  Applying each due (copy | lerp, weight) to an fp32
tensor must reproduce AveragedModel over an fp32 copy of the weights bit for bit."""
import numpy as np
import pytest
import torch
from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn, get_swa_multi_avg_fn

import stoke_b200 as sb
from stoke_b200.status import StokeStatus
from stoke_b200.weight_average import COPY, LERP, due_update


def test_config_defaults_follow_torch():
    c = sb.WeightAverageConfig()
    assert (c.kind, c.decay, c.every, c.start_step, c.use_buffers) == ("ema", 0.999, 1, 0, False)
    assert "WeightAverageConfig" in StokeStatus._CONFIG_NAMES
    assert "WeightAverageConfig" in sb.__all__ and "WeightAverage" in sb.__all__


@pytest.mark.parametrize("kw", [dict(decay=-0.1), dict(decay=1.5), dict(every=0), dict(every=1.5), dict(start_step=-1),
                                dict(kind="polyak")])
def test_config_rejects_out_of_range(kw):
    with pytest.raises(ValueError):
        sb.WeightAverageConfig(**kw)


def test_config_accepts_edges():
    sb.WeightAverageConfig(decay=0.0)
    sb.WeightAverageConfig(decay=1.0, every=7, start_step=3, kind="swa", use_buffers=True)


def test_lerp_weights():
    assert due_update("ema", 0.999, 1, 0, 1, 0) == (COPY, 0.0)
    assert due_update("ema", 0.999, 1, 0, 2, 1) == (LERP, float(np.float32(1 - 0.999)))
    assert due_update("swa", 0.999, 1, 0, 5, 2) == (LERP, float(np.float32(1) / np.float32(3)))
    assert due_update("swa", 0.0, 1, 0, 5, 1) == (LERP, 0.5)
    assert due_update("ema", 0.5, 3, 2, 4, 0) is None
    assert due_update("ema", 0.5, 3, 2, 2, 0) is None
    assert due_update("ema", 0.5, 3, 2, 5, 0) == (COPY, 0.0)


@pytest.mark.parametrize("kind", ["ema", "swa"])
@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("start_step", [0, 2])
@pytest.mark.parametrize("grad_accum", [1, 3])
def test_schedule_matches_averaged_model(kind, every, start_step, grad_accum):
    """A training loop of 14 optimizer steps (grad_accum micro-steps each; only optimizer steps count), decay changed
    after step 6 and reset() after step 9: the averages after every step are bit-identical."""
    torch.manual_seed(0)
    master = torch.nn.Linear(41, 37).float()
    with torch.no_grad():
        master.weight.mul_(3.0)
    decay = 0.9 if kind == "ema" else 0.999
    fn = get_ema_multi_avg_fn(decay) if kind == "ema" else get_swa_multi_avg_fn()
    # on CUDA the default AveragedModel (no avg_fn) takes get_swa_multi_avg_fn(); on CPU it has to be asked for
    ref = AveragedModel(master, multi_avg_fn=fn)
    avg = [p.detach().clone() for p in master.parameters()]
    n_averaged, step, updates = 0, 0, []
    g = torch.Generator().manual_seed(1)
    for micro in range(14 * grad_accum):
        if (micro + 1) % grad_accum:
            continue   # accumulation micro-step: no optimizer step, no update
        step += 1
        with torch.no_grad():
            for p in master.parameters():
                p.add_(torch.randn(p.shape, generator=g) * (1e-3 * step))
        if step == 7 and kind == "ema":
            decay = 0.3   # the other lerp branch: fp32(1 - 0.3) >= 0.5
            ref.multi_avg_fn = get_ema_multi_avg_fn(decay)
        if step == 10:
            n_averaged = 0
            ref.n_averaged.zero_()
        due = due_update(kind, decay, every, start_step, step, n_averaged)
        due_ref = step > start_step and (step - start_step) % every == 0
        assert (due is not None) == due_ref
        if due is None:
            continue
        updates.append(step)
        ref.update_parameters(master)
        if due[0] == COPY:
            torch._foreach_copy_(avg, [p.detach() for p in master.parameters()])
        else:
            torch._foreach_lerp_(avg, [p.detach() for p in master.parameters()], due[1])
        n_averaged += 1
        assert n_averaged == int(ref.n_averaged)
        for a, r in zip(avg, ref.module.parameters()):
            assert torch.equal(a.view(torch.int32), r.detach().view(torch.int32)), (step, due)
    assert updates == [s for s in range(1, 15) if s > start_step and (s - start_step) % every == 0]
