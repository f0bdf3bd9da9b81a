"""CPU checks of oracle/kernel_ref.py, the float64 reference the GPU kernel tests compare against.

1. The reference and its per-element bounds hold for the fp32 CPU oracle (torch's own fp32 ops): a bound that torch's fp32
   arithmetic can break is not a bound on fp32 rounding.
2. Every deliberately wrong reference differs from the true one by more than the bound on the inputs the GPU tests use,
   so those tests would notice each of these mistakes in a kernel.
"""
import math

import pytest
import torch

import kernel_ref as kr
from engine_oracle import OracleEngine

ADAM = {"lr": 2.0**-7, "beta1": 0.875, "beta2": 0.9921875, "eps": 2.0**-20}


def _inputs(n=640, seed=0, w_scale=1e-3, g_scale=1e-3):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(n, generator=g) * w_scale
    grads = [torch.randn(n, generator=g) * g_scale for _ in range(5)]
    return w, grads


def _torch_kwargs(kind, h):
    if kind == "sgd":
        return {k: h[k] for k in ("lr", "momentum", "dampening", "weight_decay", "nesterov", "maximize") if k in h}
    out = {"lr": h["lr"], "betas": (h["beta1"], h["beta2"]), "eps": h["eps"], "maximize": h.get("maximize", False)}
    if "weight_decay" in h:
        out["weight_decay"] = h["weight_decay"]
    return out


@pytest.mark.parametrize("kind,hyper", [
    ("adam", ADAM),
    ("adam", dict(ADAM, weight_decay=0.25, maximize=True)),
    ("adam", {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-8}),     # hyper-parameters not representable in fp32
    ("adam", dict(ADAM, beta1=0.0)),
    ("adamw", dict(ADAM, weight_decay=0.25)),
])
def test_adam_reference_bounds_fp32_oracle(kind, hyper):
    w, grads = _inputs()
    cls = torch.optim.AdamW if kind == "adamw" else torch.optim.Adam
    oracle = OracleEngine([w], 1, cls, _torch_kwargs(kind, hyper))
    p = oracle.params[0]
    m = torch.zeros_like(w)
    v = torch.zeros_like(w)
    for step, g in enumerate(grads):
        w0 = p.detach().clone()
        oracle.micro_step([[g]])
        oracle.step()
        st = oracle.optimizer.state[p]
        rw, rm, rv = kr.adam_step(kind, w0, m, v, g, step, hyper)
        bw, bm, bv = kr.adam_bound(kind, w0, m, v, g, torch.zeros_like(w), step, hyper, rm, rv)
        assert bool(((p.detach().double() - rw).abs() <= bw).all())
        assert bool(((st["exp_avg"].double() - rm).abs() <= bm).all())
        assert bool(((st["exp_avg_sq"].double() - rv).abs() <= bv).all())
        # the bound is tight enough to mean something: a small multiple of u relative to the update, not of the weight
        upd = (rw - w0.double()).abs()
        assert float((bw / upd.clamp_min(1e-30)).median()) < 1e-5
        m, v = st["exp_avg"].clone(), st["exp_avg_sq"].clone()


@pytest.mark.parametrize("hyper", [
    {"lr": 2.0**-5, "momentum": 0.875, "dampening": 0.25},
    {"lr": 2.0**-5, "momentum": 0.875, "nesterov": True, "weight_decay": 2.0**-4},
    {"lr": 2.0**-5, "momentum": 0.0, "weight_decay": 2.0**-4, "maximize": True},
    {"lr": 0.05, "momentum": 0.9, "dampening": 0.1},
])
def test_sgd_reference_bounds_fp32_oracle(hyper):
    w, grads = _inputs(seed=1)
    oracle = OracleEngine([w], 1, torch.optim.SGD, _torch_kwargs("sgd", hyper))
    p = oracle.params[0]
    buf = None
    for g in grads:
        w0 = p.detach().clone()
        oracle.micro_step([[g]])
        oracle.step()
        rw, rb = kr.sgd_step(w0, buf, g, hyper)
        bw, bb = kr.sgd_bound(w0, buf, g, torch.zeros_like(w), hyper, rw, rb)
        assert bool(((p.detach().double() - rw).abs() <= bw).all())
        if hyper["momentum"]:
            got = oracle.optimizer.state[p]["momentum_buffer"]
            assert bool(((got.double() - rb).abs() <= bb).all())
            buf = got.clone()


@pytest.mark.parametrize("norm_type", [2.0, math.inf, 1.0, 1.5, 3.0])
def test_norm_reference_bounds_fp32_torch(norm_type):
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(4096, generator=g) * 1e-3).float()
    ref = kr.norm_ref(x, norm_type)
    got = float(torch.linalg.vector_norm(x, norm_type))          # fp32 torch, its own summation order
    # any summation order has a longest chain of at most n - 1 additions
    assert abs(got - ref) <= kr.norm_bound(x, torch.zeros_like(x, dtype=torch.float64), norm_type, depth=x.numel())
    # the clip path as the oracle runs it (fp32 clip_grad_norm_) agrees with the float64 coefficient
    p = torch.nn.Parameter(torch.zeros_like(x))
    p.grad = x.clone()
    total = float(torch.nn.utils.clip_grad_norm_([p], 1e-3, norm_type))
    c = kr.clip_coef(total, 1e-3)
    assert abs(float((p.grad.double() / x.double())[0]) - c) <= 2 * kr.clip_coef_bound(total, 1e-3) + 2 * kr.U * c


def test_nan_and_inf_norms_follow_torch():
    x = torch.ones(16)
    x[3] = float("inf")
    assert kr.norm_ref(x, 2.0) == math.inf and kr.clip_coef(math.inf, 1.0) == 0.0
    x[5] = float("nan")
    for p in (2.0, math.inf, 1.5):
        assert math.isnan(kr.norm_ref(x, p))
    assert math.isnan(kr.clip_coef(math.nan, 1.0))
    y = kr.clip_value_ref(torch.tensor([float("nan"), 5.0, -5.0, float("inf")]), 1.0)
    assert math.isnan(float(y[0])) and y[1:].tolist() == [1.0, -1.0, 1.0]


def test_scaler_update_and_bias_corrections():
    assert kr.update_scale(8.0, 2, True, 2.0, 0.5, 3) == (4.0, 0)
    assert kr.update_scale(8.0, 2, False, 2.0, 0.5, 3) == (16.0, 0)
    assert kr.update_scale(8.0, 0, False, 2.0, 0.5, 3) == (8.0, 1)
    big = float(torch.finfo(torch.float32).max)
    assert kr.update_scale(big, 0, False, 2.0, 0.5, 1) == (big, 0)        # growth past fp32 max leaves the scale
    ss, c2 = kr.bias_corrections(ADAM, 0)
    assert ss == kr.f32_value(ADAM["lr"] / (1 - ADAM["beta1"])) and c2 == kr.f32_value(math.sqrt(1 - ADAM["beta2"]))
    assert kr.inv_scale_f32(3.0) == float(torch.tensor(1 / 3.0, dtype=torch.float32))


# ---- negative controls: each mistake is larger than the bound on the inputs the GPU tests use -----------------------------
def _exceeds(got, ref, bound):
    return bool(((got.double() - ref).abs() > bound).any())


@pytest.mark.parametrize("kind,mutation,hyper", [
    ("adam", "eps_in_sqrt", dict(ADAM, eps=1e-8)),
    ("adam", "bc2_not_sqrt", ADAM),
    ("adamw", "decay_after", dict(ADAM, weight_decay=0.25)),
])
def test_adam_mutants_exceed_bound(kind, mutation, hyper):
    w, grads = _inputs()
    m = torch.zeros_like(w)
    v = torch.zeros_like(w)
    for step, g in enumerate(grads[:3]):
        rw, rm, rv = kr.adam_step(kind, w, m, v, g, step, hyper)
        bw, bm, bv = kr.adam_bound(kind, w, m, v, g, torch.zeros_like(w), step, hyper, rm, rv)
        mw, _, _ = kr.adam_step_mutant(kind, w, m, v, g, step, hyper, mutation)
        assert _exceeds(mw, rw, bw), (mutation, step)
        # the true reference stays inside (sanity of the control itself)
        assert not _exceeds(rw, rw, bw)
        w, m, v = rw.float(), rm.float(), rv.float()


@pytest.mark.parametrize("mutation,hyper", [
    ("no_dampening", {"lr": 2.0**-5, "momentum": 0.875, "dampening": 0.25}),
    ("no_nesterov", {"lr": 2.0**-5, "momentum": 0.875, "nesterov": True, "weight_decay": 2.0**-4}),
])
def test_sgd_mutants_exceed_bound(mutation, hyper):
    w, grads = _inputs(seed=1)
    buf = None
    for g in grads[:3]:
        rw, rb = kr.sgd_step(w, buf, g, hyper)
        bw, _ = kr.sgd_bound(w, buf, g, torch.zeros_like(w), hyper, rw, rb)
        mw, _ = kr.sgd_step_mutant(w, buf, g, hyper, mutation)
        if buf is not None or mutation == "no_nesterov":    # dampening does not touch the first (seeding) step
            assert _exceeds(mw, rw, bw), mutation
        w, buf = rw.float(), rb.float()


def test_clip_mutant_exceeds_bound():
    # the norms the GPU tests set: the +1e-6 is many bounds wide there
    for norm in (0.02, 0.05, 0.125):
        c, b = kr.clip_coef(norm, 2.0**-7), kr.clip_coef_bound(norm, 2.0**-7)
        assert abs(kr.clip_coef_mutant(norm, 2.0**-7) - c) > 4 * b


def test_wrong_step_or_group_exceeds_bound():
    """The controls of the range table: a skipped range stepped anyway, or an element given its neighbour group's
    hyper-parameters, moves the weights by far more than the bound."""
    w, grads = _inputs()
    m = v = torch.zeros_like(w)
    rw, rm, rv = kr.adam_step("adam", w, m, v, grads[0], 0, ADAM)
    bw, _, _ = kr.adam_bound("adam", w, m, v, grads[0], torch.zeros_like(w), 0, ADAM, rm, rv)
    assert _exceeds(w, rw, bw)                                                 # stepped vs not stepped
    other = dict(ADAM, lr=ADAM["lr"] * 1.25, beta2=0.984375)
    ow, _, _ = kr.adam_step("adam", w, m, v, grads[0], 0, other)
    assert bool(((ow - rw).abs() > bw).all())                                  # every element would notice
