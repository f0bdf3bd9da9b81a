"""Which prologues and which entry point ``GradPath.optimizer_step`` calls for each K2 kind, and the struct type of
every array it hands them, with and without per-parameter step counts.  No GPU: the engine's library is a recording
stand-in and the path's tables are CPU tensors."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from stoke_b200 import _lib, optim
from stoke_b200.engine import ClipSpec, Engine, GradPath

_STEP_CALLS = ("stk_state_select", "stk_step_epilogue", "stk_comm_poll")


class _RecordingLib:
    """Stands in for libstoke_b200: records each stk_* call as its name, then per argument the element type of a ctypes
    array or the type of a struct passed by reference (``OptimArgs+OptimHyperExt`` when its hyper_ext is set)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            rec = [name]
            for a in args:
                if isinstance(a, C.Array):
                    rec.append(a._type_.__name__)
                elif type(a).__name__ == "CArgObject":
                    s = a._obj
                    rec.append(type(s).__name__ + ("+OptimHyperExt" if getattr(s, "hyper_ext", None) else ""))
            if name not in _STEP_CALLS:
                self.calls.append(tuple(rec))
            return 0
        return call


def _path(per_range: bool) -> GradPath:
    """A two-group, world-1 path on the local route: its range table is always given; the step counts are per
    parameter when ``per_range``."""
    e = Engine.__new__(Engine)
    e.lib, e.ctx, e.launches, e._cur_state, e.world = _RecordingLib(), C.c_void_p(1), 0, 0, 1
    e._stream = lambda stream=None: None
    p = GradPath.__new__(GradPath)
    buf = SimpleNamespace(ptr=0x1000)
    p.engine, p.state_id, p.clip, p.route, p.sharded, p.low_precision = e, 1, ClipSpec(), "local", False, False
    p.G = p.ACC = p.M = p.V = p.M2 = p.M3 = buf
    p.model_dtype, p.master_ptr, p.n_local, p.n_local_max, p._raw_has_acc = torch.float32, buf.ptr, 32, 32, False
    p.group_of, p.params = [0, 1], [None, None]
    p._touched, p._track_touched, p._range_skip_live = np.ones(2, dtype=bool), False, False
    p._range_end, p._range_group = torch.tensor([2, 4], dtype=torch.int32), torch.tensor([0, 1], dtype=torch.uint8)
    p._range_steps = torch.zeros(2, dtype=torch.int32) if per_range else None
    p._range_bc, p._group_bc = torch.zeros(2, 4), torch.zeros(2, 4)
    p._range_scal, p._group_scal = torch.ones(2, 2), torch.ones(2, 2)
    p._sf_state, p.avg_due = torch.zeros(2, 2, dtype=torch.float64), None
    return p


_OPT = ("stk_optim_step_prologue", "OptimHyper")
_EX = ("stk_optim_step_ex", "OptimArgs")
_EXT_KIND = [(_OPT[0], "OptimHyper", "OptimHyperExt"), ("stk_optim_step_ex", "OptimArgs+OptimHyperExt")]
# kind -> (calls with optimizer-wide step counts, calls with per-parameter counts)
_EXPECTED = {
    **{k: ([_EX], [_OPT, _EX]) for k in (_lib.OPT_ADAM, _lib.OPT_ADAMW, _lib.OPT_SGD, _lib.OPT_LION)},
    **{k: (_EXT_KIND, _EXT_KIND) for k in (_lib.OPT_NADAM, _lib.OPT_RADAM, _lib.OPT_ADAMAX, _lib.OPT_ADADELTA,
                                           _lib.OPT_RPROP, _lib.OPT_ASGD)},
    **{k: ([("stk_sf_step_prologue", "SfHyper"), _EX], [_OPT, ("stk_sf_step_prologue", "SfHyper"), _EX])
       for k in (_lib.OPT_SF_ADAMW, _lib.OPT_SF_SGD)},
    _lib.OPT_ADEMAMIX: ([("stk_ademamix_step_prologue", "OptimHyper", "AdemamixHyper"), _EX],) * 2,
    _lib.OPT_RMSPROP_TF: ([("stk_rmsprop_tf_step", "OptimArgs", "RmspropTfHyper")],
                          [_OPT, ("stk_rmsprop_tf_step", "OptimArgs", "RmspropTfHyper")]),
    _lib.OPT_ADAN: ([("stk_adan_step_prologue", "OptimHyper", "AdanHyper"),
                     ("stk_adan_step", "OptimArgs", "AdanHyper")],) * 2,
}


def test_every_k2_kind_is_pinned():
    assert set(_EXPECTED) == {k for k in optim._KINDS.values() if isinstance(k, int)}


@pytest.mark.parametrize("per_range", [False, True])
@pytest.mark.parametrize("kind", sorted(_EXPECTED))
def test_optimizer_step_calls(kind, per_range):
    cls = next(c for c, k in optim._KINDS.items() if k == kind)
    groups = [cls([torch.nn.Parameter(torch.zeros(1))]).param_groups[0] for _ in range(2)]
    build = optim._GROUP_HYPER.get(kind)
    path = _path(per_range)
    path.optimizer_step([_lib.OptimHyper(kind=kind) for _ in groups], [build(g) for g in groups] if build else None)
    assert path.engine.lib.calls == _EXPECTED[kind][per_range]
