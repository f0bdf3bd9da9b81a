"""CPU checks of the fused Adafactor step's reference, bounds, routing and parameter layouts (no GPU).

fp32 torch (the contract, _single_tensor_adafactor) lies inside the per-element bounds of tests/adafactor_ref.py around
float64 torch, over a run of steps and every layout the kernel distinguishes; deliberately wrong references lie outside
them somewhere; fused_supported routes Adafactor to the fused step; the layout helper gives torch's factorisation."""
import math
import zlib

import pytest
import torch

import adafactor_ref as ar

SHAPES = {
    "matrix": ((37, 23), False),
    "batched3d": ((5, 7, 11), False),
    "conv3x3_cl": ((8, 6, 3, 3), True),
    "conv1x1_cl": ((16, 8, 1, 1), True),
    "tall": ((300, 40), False),
    "vector": ((100,), False),
    "scalar": ((), False),
}
HYPERS = {
    "default": {"lr": 1e-2},
    "decay_max_d": {"lr": 3e-2, "weight_decay": 0.5, "maximize": True, "d": 2.0},
    "eps_given": {"lr": 1e-2, "eps": (1e-4, 1e-3), "beta2_decay": -0.5},
}


def _grad(shape, gen, step):
    g = torch.randn(shape, generator=gen) * 1e-3
    if len(shape) >= 1 and shape[0] > 2:
        g[1] = 0.0             # a zero row / element: v = 0 there, only the eps1^2 clamp keeps u finite
    return g


@pytest.mark.parametrize("hname", list(HYPERS))
@pytest.mark.parametrize("sname", list(SHAPES))
def test_fp32_torch_inside_bounds(sname, hname):
    shape, cl = SHAPES[sname]
    h = HYPERS[hname]
    gen = torch.Generator().manual_seed(zlib.crc32(f"{sname}{hname}".encode()))
    w = torch.randn(shape, generator=gen) * 0.1
    if cl:
        w = w.contiguous(memory_format=torch.channels_last)
    state = ar.zero_state(shape)
    for step in range(6):
        g = _grad(shape, gen, step)
        rw, rst = ar.step_ref(w, state, g, step, h)
        fw, fst = ar.step_ref(w, state, g, step, h, dtype=torch.float32)
        ew, est = ar.step_bound(w, state, g, step, h, rw, rst)
        assert not bool(ar.outside(fw, rw, ew).any()), (sname, hname, step)
        for k in rst:
            assert not bool(ar.outside(fst[k], rst[k], est[k]).any()), (sname, hname, step, k)
        # the bound is tight enough to say something: far below the update itself
        assert float(ew.max()) < 1e-3 * float((rw - w.double()).abs().max()) + 1e-6
        w, state = fw, {k: v.float() for k, v in fst.items()}


def test_reference_written_out_agrees_with_torch():
    """step_mutant without a mutation (the formula written out in float64) is torch's float64 step."""
    gen = torch.Generator().manual_seed(1)
    for shape in [(37, 23), (4, 3, 3, 3), (50,), ()]:
        for h in HYPERS.values():
            w = torch.randn(shape, generator=gen)
            st = {k: v + torch.rand(v.shape, generator=gen) * 1e-6 for k, v in ar.zero_state(shape).items()}
            g = torch.randn(shape, generator=gen) * 1e-3
            rw, _ = ar.step_ref(w, st, g, 3, h)
            assert torch.allclose(ar.step_mutant(w, st, g, 3, h, "none"), rw, rtol=1e-12, atol=1e-15)


def test_mutants_fall_outside_bounds():
    hit = set()
    gen = torch.Generator().manual_seed(7)
    cases = [((37, 23), {"lr": 1e-2, "weight_decay": 0.5}), ((5, 7, 11), {"lr": 1e-2}), ((100,), {"lr": 1e-2}),
             ((37, 23), {"lr": 1e-2, "d": 1.0})]
    for shape, h in cases:
        w = torch.randn(shape, generator=gen) * 0.1
        for step in (0, 4):
            # a prior state larger than g^2 makes ||u|| / sqrt(n) < 1, where max(1, .) matters
            st = {k: v + (4e-6 if step else 0.0) for k, v in ar.zero_state(shape).items()}
            g = _grad(shape, gen, step)
            rw, rst = ar.step_ref(w, st, g, step, h)
            ew, _ = ar.step_bound(w, st, g, step, h, rw, rst)
            for mu in ar.MUTATIONS:
                if bool(ar.outside(ar.step_mutant(w, st, g, step, h, mu), rw, ew).any()):
                    hit.add(mu)
    assert hit == set(ar.MUTATIONS), set(ar.MUTATIONS) - hit


def test_nan_follows_python_max_min():
    """A NaN gradient: ||u|| is NaN, python's max(1.0, nan) is 1.0; the reference keeps torch's NaN pattern."""
    w = torch.randn(50, generator=torch.Generator().manual_seed(3))
    g = torch.randn(50) * 1e-3
    g[7] = float("nan")
    rw, rst = ar.step_ref(w, ar.zero_state((50,)), g, 0, {"lr": 1e-2})
    fw, _ = ar.step_ref(w, ar.zero_state((50,)), g, 0, {"lr": 1e-2}, dtype=torch.float32)
    assert torch.equal(rw.isnan(), fw.isnan()) and int(rw.isnan().sum()) == 1


# ---- routing and layouts ----------------------------------------------------------------------------------------------------
class Net(torch.nn.Module):
    def __init__(self, extra_dim=False):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 4, 3)
        self.lin = torch.nn.Linear(4, 2)
        if extra_dim:
            self.big = torch.nn.Parameter(torch.zeros(2, 2, 2, 2, 2))


def test_routing():
    from stoke_b200.optim import fused_supported

    net = Net()
    assert fused_supported(torch.optim.Adafactor, {"lr": 1e-2}, net)
    assert fused_supported(torch.optim.Adafactor, {"lr": 1e-2, "foreach": True}, net)
    assert fused_supported(torch.optim.Adafactor, {"lr": 1e-2, "foreach": False}, net)
    ps = list(net.parameters())
    assert fused_supported(torch.optim.Adafactor, {"params": [{"params": [p]} for p in ps]}, net)
    many = [{"params": [p]} for p in ps] + [{"params": []} for _ in range(9 - len(ps))]
    assert not fused_supported(torch.optim.Adafactor, {"params": many}, net)
    assert not fused_supported(torch.optim.Adafactor, {"lr": 1e-2}, Net(extra_dim=True))   # 5-D parameter


@pytest.mark.parametrize("shape,cl,want", [
    ((1000, 2048), False, (True, 1, 1000, 2048, 1000 + 2048)),
    ((64, 64, 3, 3), True, (True, 64 * 64, 3, 3, 2 * 64 * 64 * 3)),
    ((256, 64, 1, 1), True, (True, 256 * 64, 1, 1, 2 * 256 * 64)),
    ((5, 7, 11), False, (True, 5, 7, 11, 5 * 7 + 5 * 11)),
    ((100,), False, (False, 1, 1, 100, 100)),
    ((), False, (False, 1, 1, 1, 1)),
])
def test_layout_helper(shape, cl, want):
    from stoke_b200 import layout

    t = torch.empty(shape)
    if cl:
        t = t.contiguous(memory_format=torch.channels_last)
    lay = layout.adafactor_layout(t.shape, t.stride())
    assert (lay["factored"], lay["B"], lay["R"], lay["C"], lay["state"]) == want
    assert lay["numel"] == t.numel() == math.prod(lay["size"])
    # the strides map every logical index to a distinct storage position in [0, numel)
    idx = torch.arange(t.numel()).view(lay["size"])
    pos = sum(torch.arange(s).view([-1 if k == j else 1 for k in range(4)]) * st
              for j, (s, st) in enumerate(zip(lay["size"], lay["stride"])))
    assert sorted((pos + 0 * idx).flatten().tolist()) == list(range(t.numel()))
    if cl and shape[-1] == 3:
        assert lay["stride"] == list(t.stride())


def test_layout_helper_rejects():
    from stoke_b200 import layout

    with pytest.raises(ValueError):
        layout.adafactor_layout((2, 2, 2, 2, 2), (16, 8, 4, 2, 1))
    with pytest.raises(ValueError):
        layout.adafactor_layout((4, 4), (8, 1))   # holes
