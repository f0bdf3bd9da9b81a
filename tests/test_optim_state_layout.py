# -*- coding: utf-8 -*-
"""CPU: every fused kind's row of ``optim._STATE_LAYOUT`` against the plain class.  Each class takes two steps on CPU
with two parameter groups that differ in the per-group conditions of its state (momentum or not, centered or not,
beta1 == 0 or not; a factored and an unfactored Adafactor parameter in each), one parameter never receiving a gradient.
The class's ``state_dict()`` then goes through ``import_state`` into flat buffers laid out by ``state_buffers`` and back
out through ``export_state``: the fused step's checkpoint format, without a GPU."""
import pytest
import torch

from stoke_b200 import _lib, layout
from stoke_b200.optim import (LAMB, LARS, AdamWScheduleFree, AdEMAMix, Lion, RMSpropTF, SGDScheduleFree, _STATE_LAYOUT,
                              export_state, import_state, state_buffers, state_dict_index)

# name -> (class, kind, per-group kwargs of the two groups)
CASES = {
    "sgd": (torch.optim.SGD, _lib.OPT_SGD, [dict(lr=0.1, momentum=0.9), dict(lr=0.1, momentum=0.0)]),
    "adam": (torch.optim.Adam, _lib.OPT_ADAM, [dict(lr=0.1), dict(lr=0.2)]),
    "adamw": (torch.optim.AdamW, _lib.OPT_ADAMW, [dict(lr=0.1), dict(lr=0.2)]),
    "nadam": (torch.optim.NAdam, _lib.OPT_NADAM, [dict(lr=0.1), dict(lr=0.2)]),
    "radam": (torch.optim.RAdam, _lib.OPT_RADAM, [dict(lr=0.1), dict(lr=0.2)]),
    "adamax": (torch.optim.Adamax, _lib.OPT_ADAMAX, [dict(lr=0.1), dict(lr=0.2)]),
    "adadelta": (torch.optim.Adadelta, _lib.OPT_ADADELTA, [dict(lr=0.1), dict(lr=0.2)]),
    "rprop": (torch.optim.Rprop, _lib.OPT_RPROP, [dict(lr=0.1), dict(lr=0.2)]),
    "asgd": (torch.optim.ASGD, _lib.OPT_ASGD, [dict(lr=0.1), dict(lr=0.2)]),
    "lion": (Lion, _lib.OPT_LION, [dict(lr=0.1), dict(lr=0.2)]),
    "sf_adamw": (AdamWScheduleFree, _lib.OPT_SF_ADAMW, [dict(lr=0.1), dict(lr=0.2)]),
    "sf_sgd": (SGDScheduleFree, _lib.OPT_SF_SGD, [dict(lr=0.1), dict(lr=0.2)]),
    "ademamix": (AdEMAMix, _lib.OPT_ADEMAMIX, [dict(lr=0.1), dict(lr=0.2, betas=(0.0, 0.999, 0.9999))]),
    "rmsprop_tf": (RMSpropTF, _lib.OPT_RMSPROP_TF, [dict(lr=0.1, momentum=0.9, centered=True), dict(lr=0.2)]),
    "lamb": (LAMB, "lamb", [dict(lr=0.1), dict(lr=0.2, weight_decay=0.0)]),
    "lars": (LARS, "lars", [dict(lr=0.1, weight_decay=0.01), dict(lr=0.2, momentum=0.0)]),
    "adafactor": (getattr(torch.optim, "Adafactor", None), "adafactor", [dict(lr=0.1), dict(lr=0.2)]),
}


def _params():
    g = torch.Generator().manual_seed(0)
    # a and c are factored for Adafactor, b and d are not; d never receives a gradient
    return [torch.nn.Parameter(torch.randn(*s, generator=g)) for s in ((4, 3), (3,), (2, 3), (5,))]


GROUP_OF = [1, 0, 0, 1]   # groups [b, c] and [a, d]: torch's state_dict numbering differs from the flat order
UNSTEPPED = 3


def _run_class(name):
    cls, _, kws = CASES[name]
    if cls is None:
        pytest.skip("torch.optim.Adafactor needs torch >= 2.5")
    params = _params()
    initial = [p.detach().clone() for p in params]
    opt = cls([dict(kws[gi], params=[p for p, g in zip(params, GROUP_OF) if g == gi]) for gi in (0, 1)])
    if isinstance(opt, (AdamWScheduleFree, SGDScheduleFree)):
        opt.train()
    g = torch.Generator().manual_seed(1)
    for _ in range(2):
        for i, p in enumerate(params):
            p.grad = None if i == UNSTEPPED else torch.randn(p.shape, generator=g)
        opt.step()
    return params, initial, opt.state_dict()


def _views(kind, params, initial, groups):
    """Per state key, every parameter's view of a full-length vector at the tensor's initial value (Adafactor: of
    torch-shaped zeros, row_var / col_var for a factored parameter, variance for the others)."""
    lay = _STATE_LAYOUT[kind]
    if kind == "adafactor":
        out = {t.key: [None] * len(params) for t in lay.tensors}
        for i, p in enumerate(params):
            if p.dim() >= 2:
                out["row_var"][i] = torch.zeros(*p.shape[:-1], 1)
                out["col_var"][i] = torch.zeros(*p.shape[:-2], 1, p.shape[-1])
            else:
                out["variance"][i] = torch.zeros(p.shape)
        return out
    offsets, _, n = layout.param_offsets([p.numel() for p in params])
    per_buf = {}
    for buf, init in state_buffers(lay, groups).items():
        if init is None:
            continue
        full = torch.zeros(n) if init == "master" else torch.full((n,), float(init))
        per_buf[buf] = [full[o: o + p.numel()].view(p.shape) for p, o in zip(params, offsets)]
        if init == "master":   # the schedule-free z: a copy of the parameter before its first step
            for view, x in zip(per_buf[buf], initial):
                view.copy_(x)
    return {t.key: per_buf[t.buf] for t in lay.tensors if t.buf in per_buf}


@pytest.mark.parametrize("name", list(CASES))
def test_export_import_against_the_class(name):
    _, kind, _ = CASES[name]
    lay = _STATE_LAYOUT[kind]
    params, initial, sd = _run_class(name)
    groups = sd["param_groups"]
    sd_index = state_dict_index(GROUP_OF, 2)
    entries = [sd["state"].get(sd_index[i], {}) for i in range(len(params))]
    steps = [0 if i == UNSTEPPED else 2 for i in range(len(params))]
    scalars = [[float(e[k]) if k in e else 1.0 for k in lay.scalars] for e in entries]
    views = _views(kind, params, initial, groups)
    import_state(lay, entries, views)
    state = export_state(lay, groups, GROUP_OF, sd_index, steps, scalars, views)

    for i in range(len(params)):
        j = sd_index[i]
        if i == UNSTEPPED:
            continue
        want, got = sd["state"].get(j), state[j]
        if kind == _lib.OPT_SGD and groups[GROUP_OF[i]]["momentum"] == 0:
            # torch keeps no state in a momentum-0 group; the export carries M's zeros there, M existing for the other
            assert list(got) == ["momentum_buffer"]
            assert torch.equal(got["momentum_buffer"], torch.zeros(params[i].shape))
            continue
        assert list(got) == list(want), (name, i)
        if "step" in want:
            assert float(want["step"]) == steps[i] and torch.equal(got["step"], torch.tensor(float(steps[i])))
        for key, w in want.items():
            if key == "step":
                continue
            if w is None:
                assert got[key] is None, (name, i, key)
            else:
                assert got[key].dtype == torch.float32 and torch.equal(got[key], w.float()), (name, i, key)

    j = sd_index[UNSTEPPED]
    if lay.unstepped == "omit":
        assert j not in state and not sd["state"].get(j)   # the schedule-free train() leaves an empty entry
    elif lay.unstepped == "none":
        assert state[j] == {t.key: None for t in lay.tensors}
    else:   # "same": the entry a parameter has at step 0, its state at the initial values
        assert list(state[j]) == ["step", *lay.scalars, *(t.key for t in lay.tensors)]
        assert torch.equal(state[j]["step"], torch.tensor(0.0))
        for k in lay.scalars:
            assert torch.equal(state[j][k], torch.tensor(1.0))
        for t in lay.tensors:
            assert torch.equal(state[j][t.key], torch.full(params[UNSTEPPED].shape, float(t.init)))


@pytest.mark.parametrize("name, groups, want", [
    ("sgd", [dict(momentum=0.9), dict(momentum=0.0)], (0.0, None, None)),
    ("sgd", [dict(momentum=0.0)], (None, None, None)),
    ("adam", [{}], (0.0, 0.0, None)),
    ("nadam", [{}], (0.0, 0.0, None)),
    ("adamax", [{}], (0.0, 0.0, None)),
    ("adadelta", [{}], (0.0, 0.0, None)),
    ("rprop", [{}], (0.0, 0.0, None)),
    ("asgd", [{}], (0.0, None, None)),
    ("lion", [{}], (0.0, None, None)),
    ("sf_adamw", [{}], ("master", 0.0, None)),
    ("sf_sgd", [{}], ("master", None, None)),
    ("ademamix", [dict(betas=(0.9, 0.999, 0.9999)), dict(betas=(0.0, 0.999, 0.9999))], (0.0, 0.0, 0.0)),
    ("ademamix", [dict(betas=(0.0, 0.999, 0.9999))], (None, 0.0, 0.0)),
    ("rmsprop_tf", [dict(momentum=0.9, centered=False), dict(momentum=0.0, centered=True)], (0.0, 1.0, 0.0)),
    ("rmsprop_tf", [dict(momentum=0.9, centered=False)], (0.0, 1.0, None)),
    ("rmsprop_tf", [dict(momentum=0.0, centered=True)], (None, 1.0, 0.0)),
    ("lamb", [{}], (0.0, 0.0, None)),
    ("lars", [dict(momentum=0.9), dict(momentum=0.0)], (0.0, None, None)),
    ("lars", [dict(momentum=0.0)], (None, None, None)),
    ("adafactor", [{}], (None, None, None)),
])
def test_buffers_to_allocate(name, groups, want):
    """``{"M", "V", "M2"} -> initial value`` for each group configuration (None: not allocated)."""
    assert state_buffers(_STATE_LAYOUT[CASES[name][1]], groups) == dict(zip(("M", "V", "M2"), want))
