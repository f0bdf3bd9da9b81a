"""One gradient window, formed two ways: every fused optimizer step, bit for bit (GPU).

Every fused step forms its own gradient from the raw bucket, x = ((g [+ acc]) * mul) * 1/scale, then the clip, and
Adafactor, LAMB and LARS form it again in several of their passes.  The windows of tests/grad_window_ref.py are exact at
every stage (tests/test_grad_window_exact.py), so a step cannot tell an accumulated, loss-scaled window from one bucket
that already holds the sum.  Each case therefore runs the same three steps twice from the same weights:

  A  grad_accum = 1, no loss scaler, the bucket holds the window total (same model dtype and route);
  B  the window as training forms it: micro-batches accumulated (after_backward(sync=False)) into the fp32 accumulator,
     the last one in the model-dtype bucket, optionally loss-scaled by a DeviceGradScaler whose scale grows mid-run;

and requires B to be bit-identical to A after every step: master, every state tensor, the schedule-free group scalars,
the per-parameter step counts, the gradient norm, and the bf16 copy.  The float64 element suites check run A, so this
carries their guarantee over to the accumulated and loss-scaled paths of every kind.  Two negative controls show the
equality is not vacuous: A' (the window without its earlier micro-batches: a pass that ignores the accumulator) and A''
(the window times the loss scale: a pass that misses the unscale) must each differ from B.  The Adafactor cases also
assert that both regimes of the update's RMS clip occur (tests/adafactor_ref.py, float64)."""
import pytest
import torch

import adafactor_ref as ar
import grad_window_ref as gw

pytestmark = pytest.mark.gpu

STEPS = 3
# tests/test_gpu_adafactor.py's SMALL (a channels-last 3x3 and 1x1 conv, (37, 23), (5, 7, 11), 1000, a scalar) and one
# matrix over both tile sizes (STK_LW_TILE = kAfTile = 8192): three tiles, the last one partial
SHAPES = [((64, 64, 3, 3), True), ((64, 32, 1, 1), True), ((37, 23), False), ((5, 7, 11), False), ((1000,), False),
          ((), False), ((130, 129), False)]
GROUP1 = [1, 3, 5]   # the second parameter group; the others are in the first


def _kinds():
    from stoke_b200 import optim as so

    O = torch.optim
    return {
        # name: (class, first group's kwargs, second group's overrides)
        "adam": (O.Adam, {"lr": 1e-3, "betas": (0.9, 0.99), "weight_decay": 0.01}, {"lr": 2e-3, "weight_decay": 0.0,
                                                                                     "eps": 1e-6}),
        "adamw": (O.AdamW, {"lr": 1e-3, "weight_decay": 0.05}, {"lr": 3e-3, "betas": (0.8, 0.95), "weight_decay": 0.0}),
        "sgd_momentum": (O.SGD, {"lr": 0.05, "momentum": 0.9, "weight_decay": 1e-4}, {"lr": 0.1, "momentum": 0.5,
                                                                                    "dampening": 0.1}),
        "sgd_nesterov": (O.SGD, {"lr": 0.05, "momentum": 0.9, "nesterov": True}, {"lr": 0.02, "momentum": 0.8,
                                                                                "weight_decay": 1e-3}),
        "nadam": (O.NAdam, {"lr": 2e-3, "weight_decay": 0.01}, {"lr": 1e-3, "momentum_decay": 0.006,
                                                                "decoupled_weight_decay": True, "weight_decay": 0.02}),
        "radam": (O.RAdam, {"lr": 1e-3}, {"lr": 2e-3, "weight_decay": 0.01, "decoupled_weight_decay": True}),
        "adamax": (O.Adamax, {"lr": 2e-3}, {"lr": 1e-3, "weight_decay": 0.01, "betas": (0.8, 0.99)}),
        "adadelta": (O.Adadelta, {"lr": 1.0}, {"lr": 0.5, "rho": 0.8, "weight_decay": 0.01}),
        "rprop": (O.Rprop, {"lr": 1e-3}, {"lr": 2e-3, "etas": (0.4, 1.3), "step_sizes": (1e-6, 1.0)}),
        "asgd": (O.ASGD, {"lr": 1e-2, "t0": 1.0}, {"lr": 5e-3, "lambd": 1e-3, "alpha": 0.5, "weight_decay": 1e-3}),
        "lion": (so.Lion, {"lr": 1e-4, "weight_decay": 0.1}, {"lr": 3e-4, "betas": (0.95, 0.98)}),
        "sf_adamw": (so.AdamWScheduleFree, {"lr": 2.5e-3, "warmup_steps": 1, "weight_decay": 0.01},
                     {"lr": 1e-3, "betas": (0.8, 0.99), "r": 1.0}),
        "sf_sgd": (so.SGDScheduleFree, {"lr": 0.5, "momentum": 0.9}, {"lr": 0.2, "weight_decay": 1e-3,
                                                                      "warmup_steps": 2}),
        "ademamix": (so.AdEMAMix, {"lr": 1e-3, "alpha": 5.0, "beta3_warmup": 10, "alpha_warmup": 10},
                     {"betas": (0.0, 0.999, 0.999), "weight_decay": 0.01}),
        # d sets the threshold of the update's RMS clip: 2.0 keeps it off, 0.25 on (asserted below)
        "adafactor": (O.Adafactor, {"lr": 1e-2, "d": 2.0, "weight_decay": 0.01}, {"lr": 5e-3, "d": 0.25,
                                                                                   "eps": (1e-4, 1e-3)}),
        "lamb": (so.LAMB, {"lr": 1e-2, "weight_decay": 0.01}, {"lr": 5e-3, "weight_decay": 0.0, "betas": (0.8, 0.99),
                                                               "bias_correction": False}),
        "lars": (so.LARS, {"lr": 0.5, "weight_decay": 5e-4}, {"lr": 0.2, "weight_decay": 0.0, "always_adapt": True,
                                                              "momentum": 0.8, "nesterov": True}),
        # the 64x64x3x3 conv weight and the 130x129 matrix reach min_8bit_size (4096): 8-bit codes; the rest fp32
        "adamw8bit": (so.AdamW8bit, {"lr": 1e-3, "weight_decay": 0.01}, {"lr": 3e-3, "betas": (0.8, 0.95),
                                                                        "weight_decay": 0.0}),
    }


KINDS = ["adam", "adamw", "sgd_momentum", "sgd_nesterov", "nadam", "radam", "adamax", "adadelta", "rprop", "asgd", "lion",
         "sf_adamw", "sf_sgd", "ademamix", "adafactor", "lamb", "lars", "adamw8bit"]
# fused launches of one opt.step() (the step epilogue included): the stock route launches other kernels
LAUNCHES = dict({k: 2 for k in KINDS}, nadam=3, radam=3, adamax=3, adadelta=3, rprop=3, asgd=3, sf_adamw=3, sf_sgd=3,
                ademamix=3, adafactor=9, lamb=4, lars=4, adamw8bit=3)

# variant: (model dtype, route, grad_accum, loss scaler, clip)
VARIANTS = {
    "bf16_acc2": (torch.bfloat16, "local", 2, False, None),
    "bf16_acc3_clipnorm": (torch.bfloat16, "local", 3, False, ("norm", 1.0)),
    "f32_acc2_scaler_clipvalue": (None, "local", 2, True, ("value", 0.02)),
    "main_bf16_acc2_clipnorm": (torch.bfloat16, "main", 2, False, ("norm", 0.5)),
}
INIT_SCALE, GROWTH_INTERVAL = 2.0**12, 2   # the scale doubles after the second step


class Shapes(torch.nn.Module):
    def __init__(self, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        ps = []
        for s, cl in SHAPES:
            t = torch.randn(s, generator=g) * 0.1
            if cl:
                t = t.contiguous(memory_format=torch.channels_last)
            ps.append(torch.nn.Parameter(t))
        self.ps = torch.nn.ParameterList(ps)


def _hyper(kind, i):
    _, base, extra = _kinds()[kind]
    return dict(base, **extra) if i in GROUP1 else dict(base)


def _build(kind, lp, route, accum, clip):
    from stoke_b200 import _lib
    from stoke_b200.engine import ClipSpec, get_engine
    from stoke_b200.optim import B200FusedOptimizer

    cls, base, extra = _kinds()[kind]
    torch.cuda.set_device(0)
    net = Shapes().cuda()
    ps = list(net.parameters())
    kw = dict(base, params=[{"params": [p for i, p in enumerate(ps) if i not in GROUP1]},
                            dict(extra, params=[ps[i] for i in GROUP1])])
    spec = None
    if clip is not None:
        spec = ClipSpec(_lib.CLIP_NORM, max_norm=clip[1], norm_type=2.0) if clip[0] == "norm" else \
            ClipSpec(_lib.CLIP_VALUE, clip_value=clip[1])
    opt = B200FusedOptimizer(net, cls, kw, engine=get_engine(0), grad_accum=accum, clip=spec, lp_dtype=lp, route=route)
    assert opt.path.route == route
    if kind.startswith("sf_"):
        opt.train()
    return opt


def _windows(accum, seed):
    numels = [max(1, int(torch.Size(s).numel())) for s, _ in SHAPES]
    return [gw.window(numels, accum, 1000 * seed + step) for step in range(STEPS)]


def _put(path, flats):
    for gv, f in zip(path.grad_views, flats):
        gv.copy_(f.reshape(gv.shape))


def _snap(opt, launches):
    path = opt.path
    sd = opt.state_dict()
    state = {(i, k): (None if v is None else v.detach().cpu().clone()) for i, d in sd["state"].items()
             for k, v in d.items()}
    groups = [{k: g[k] for k in ("k", "lr_max", "weight_sum") if k in g} for g in sd["param_groups"]]
    st = path.engine.scaler_get(path.state_id)
    return {"master": path.gather_master().cpu().clone(), "state": state, "groups": groups, "steps": path.param_steps(),
            "norm": torch.tensor(st.grad_norm, dtype=torch.float32), "launches": launches}


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _state_same(sa, sb):
    if set(sa) != set(sb):
        return False
    return all((sa[k] is None and sb[k] is None) or (sa[k] is not None and sb[k] is not None and _same(sa[k], sb[k]))
               for k in sa)


def _run(kind, variant, mode, wins, scales=None, ratios=None):
    """mode "B": the window as training forms it; "A": one bucket with the total; "A_last": one bucket with only the last
    micro-batch; "A_scaled": one bucket with the total times the scale B had at that step.  Returns one snapshot per step
    (and, for B, the scale of every step)."""
    lp, route, accum, scaled, clip = VARIANTS[variant]
    opt = _build(kind, lp, route, accum if mode == "B" else 1, clip)
    path = opt.path
    scaler = None
    if mode == "B" and scaled:
        from stoke_b200.fp16 import DeviceGradScaler

        scaler = DeviceGradScaler(path.engine, init_scale=INIT_SCALE, growth_interval=GROWTH_INTERVAL,
                                  state_id=path.state_id)
    snaps, used = [], []
    try:
        for step, win in enumerate(wins):
            if mode == "B":
                S = scaler.get_scale() if scaler is not None else 1.0
                used.append(S)
                for mi in range(accum):
                    _put(path, [ms[mi] * S for ms in win])
                    path.after_backward(sync=(mi == accum - 1), unscale=scaler is not None)
            else:
                if mode == "A_last":
                    flats = [ms[-1] for ms in win]
                elif mode == "A_scaled":
                    flats = [gw.total(ms) * scales[step] for ms in win]
                else:
                    flats = [gw.total(ms) for ms in win]
                _put(path, flats)
                path.after_backward(sync=True, unscale=False)
            s0 = None
            if ratios is not None:
                s0 = [tuple(v.cpu().clone() for v in vs) for vs in path.adafactor_state_views()]
                steps0 = path.param_steps()
            l0 = path.engine.launches
            opt.step()
            snap = _snap(opt, path.engine.launches - l0)
            if lp is not None:
                assert torch.equal(path.p_flat.cpu(), path.gather_master().cpu().to(lp)), (kind, variant, mode, step)
            assert float(path.g_flat.float().abs().max()) == 0.0, (kind, variant, mode, step)
            if ratios is not None:
                coef = 1.0
                if clip is not None and clip[0] == "norm":
                    coef = torch.clamp(torch.tensor(clip[1], dtype=torch.float32) / (snap["norm"] + 1e-6), max=1.0)
                for i, p in enumerate(path.params):
                    G = gw.total(win[i]).reshape(p.shape)
                    if clip is not None:
                        G = G * coef if clip[0] == "norm" else G.clamp(-clip[1], clip[1])
                    state = dict(zip(ar.state_keys(p.shape), s0[i]))
                    ratios.append(ar.update_ratio(state, G, steps0[i], _hyper(kind, i)))
            snaps.append(snap)
    finally:
        opt.close()
    return snaps, used


CASES = [(k, v) for k in KINDS for v in VARIANTS]


@pytest.mark.parametrize("kind,variant", CASES, ids=[f"{k}-{v}" for k, v in CASES])
def test_accumulated_window_matches_single_bucket(kind, variant):
    lp, route, accum, scaled, clip = VARIANTS[variant]
    wins = _windows(accum, seed=KINDS.index(kind))
    ratios = [] if kind == "adafactor" else None
    b, scales = _run(kind, variant, "B", wins)
    a, _ = _run(kind, variant, "A", wins, ratios=ratios)
    for step, (sa, sb) in enumerate(zip(a, b)):
        tag = (kind, variant, step)
        assert sb["launches"] == sa["launches"] == LAUNCHES[kind], (tag, sa["launches"], sb["launches"])
        # the window's norm must not depend on how the window was accumulated
        assert _same(sa["norm"], sb["norm"]), (tag, float(sa["norm"]), float(sb["norm"]))
        assert sa["steps"] == sb["steps"] == [step + 1] * len(SHAPES), tag
        assert _same(sa["master"], sb["master"]), (tag, "master", int((_bits(sa["master"]) != _bits(sb["master"])).sum()))
        assert set(sa["state"]) == set(sb["state"]), tag
        for key, ta in sa["state"].items():
            tb = sb["state"][key]
            assert (ta is None and tb is None) or (ta is not None and tb is not None and _same(ta, tb)), (tag, key)
        assert sa["groups"] == sb["groups"], tag
    if scaled:
        assert scales == [INIT_SCALE, INIT_SCALE, 2 * INIT_SCALE], scales   # the scale changed during the run

    # negative controls: each must differ from B (master or state) at some step
    controls = {"A_last": accum > 1, "A_scaled": scaled}
    hit = set()
    for mode, applies in controls.items():
        if not applies:
            continue
        c, _ = _run(kind, variant, mode, wins, scales=scales)
        if any(not _same(sc["master"], sb["master"]) or not _state_same(sc["state"], sb["state"]) for sc, sb in zip(c, b)):
            hit.add(mode)
        else:
            pytest.fail(f"negative control {mode} is bit-identical to the accumulated run ({kind}, {variant})")
    assert hit == {m for m, applies in controls.items() if applies}
    if ratios is not None:
        # both regimes of Adafactor's max(1, ||u|| / (sqrt(n) d)), away from the boundary
        assert any(r > 1.01 for r in ratios) and any(r < 0.99 for r in ratios), ratios
