"""The checkpoint-load decision of the fused optimizer (``stoke_b200.optim.load_step_counts``), on the CPU: which step
count and scalar state every parameter continues from, following torch's lazy state creation."""
import pytest
import torch

from stoke_b200 import _lib
from stoke_b200.optim import load_step_counts

ALL_KINDS = [_lib.OPT_ADAM, _lib.OPT_ADAMW, _lib.OPT_SGD, _lib.OPT_NADAM, _lib.OPT_RADAM, _lib.OPT_ADAMAX,
             _lib.OPT_ADADELTA, _lib.OPT_RPROP, _lib.OPT_ASGD]


def _entry(kind, step, **scalars):
    if kind == _lib.OPT_SGD:
        return {"momentum_buffer": torch.zeros(3)}
    e = {"step": torch.tensor(float(step))}
    e.update({k: torch.tensor(v, dtype=torch.float32) for k, v in scalars.items()})
    return e


def test_uniform_counts_replace_per_parameter_counts_already_on():
    """Per-parameter counts are on (some parameter was unused once); a uniform checkpoint still sets every count."""
    entries = [_entry(_lib.OPT_ADAM, 5)] * 3
    assert load_step_counts(_lib.OPT_ADAM, entries, [0, 0, 0], 5, per_param_on=True) == (5, [5, 5, 5], None)


def test_uniform_counts_stay_optimizer_wide():
    for opt_steps in (4, None):
        entries = [_entry(_lib.OPT_ADAM, 4)] * 3
        assert load_step_counts(_lib.OPT_ADAM, entries, [0, 1, 0], opt_steps, per_param_on=False) == (4, None, None)


@pytest.mark.parametrize("kind", ALL_KINDS + ["adafactor"])
def test_parameter_without_entry_has_taken_no_step(kind):
    """torch creates a parameter's state at its first step: no entry means step 0 and the initial scalar state."""
    scal = {_lib.OPT_NADAM: {"mu_product": 0.5}, _lib.OPT_ASGD: {"eta": 0.25, "mu": 1.0}}.get(kind, {})
    entries = [_entry(kind, 3, **scal), {}, _entry(kind, 3, **scal)]
    steps, per_param, scalars = load_step_counts(kind, entries, [0, 0, 0], None, False, momentum=[0.9])
    assert per_param[1] == 0 and per_param[0] == per_param[2] == steps > 0
    if scal:
        assert scalars[1] == [1.0] * len(scal) and scalars[0] == list(scal.values())
    else:
        assert scalars is None


def test_nadam_unstepped_parameter_starts_from_initial_mu_product():
    entries = [_entry(_lib.OPT_NADAM, 6, mu_product=0.5), {}]
    assert load_step_counts(_lib.OPT_NADAM, entries, [0, 0], 6, False) == (6, [6, 0], [[0.5], [1.0]])


def test_torch_sgd_momentum_continues_its_buffer():
    """torch's SGD has no `step`: a buffer means the parameter has been stepped, so the next step is not a first step."""
    buf = {"momentum_buffer": torch.ones(3)}
    assert load_step_counts(_lib.OPT_SGD, [buf, buf], [0, 0], None, False, momentum=[0.9]) == (1, None, None)
    assert load_step_counts(_lib.OPT_SGD, [buf, buf], [0, 0], 7, False, momentum=[0.9]) == (7, None, None)
    # a parameter without a buffer starts it at its own first step
    none = {"momentum_buffer": None}
    assert load_step_counts(_lib.OPT_SGD, [buf, none], [0, 0], 7, False, momentum=[0.9]) == (7, [7, 0], None)
    # without momentum torch keeps no state, and the count has no effect: it stays optimizer-wide
    assert load_step_counts(_lib.OPT_SGD, [{}, {}], [0, 1], 7, False, momentum=[0.9, 0.0]) == (7, [0, 7], None)
    assert load_step_counts(_lib.OPT_SGD, [{}, {}], [0, 0], 7, False, momentum=[0.0]) == (7, None, None)


@pytest.mark.parametrize("kind,a,b", [(_lib.OPT_NADAM, {"mu_product": 0.5}, {"mu_product": 0.25}),
                                      (_lib.OPT_ASGD, {"eta": 0.5, "mu": 1.0}, {"eta": 0.25, "mu": 0.5})])
def test_per_group_scalar_state(kind, a, b):
    """Scalars uniform within each group stay per group; scalars that differ within a group go per parameter."""
    entries = [_entry(kind, 2, **a), _entry(kind, 2, **b), _entry(kind, 2, **a)]
    assert load_step_counts(kind, entries, [0, 1, 0], 2, False) == (2, None, [list(a.values()), list(b.values())])
    got = load_step_counts(kind, entries, [0, 0, 0], 2, False)
    assert got == (2, [2, 2, 2], [list(a.values()), list(b.values()), list(a.values())])
