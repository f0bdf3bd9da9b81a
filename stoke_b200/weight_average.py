# -*- coding: utf-8 -*-
"""``Stoke.weight_average``: an fp32 moving average of the weights (EMA / SWA) kept on the engine.

The average is ``torch.optim.swa_utils.AveragedModel`` applied to fp32 copies of the master weights after every optimizer
step, bit for bit.  Averaging the model's bf16 parameters instead (``AveragedModel(model)`` in ``fp16="bf16"``) stores
the average in bf16, where most updates at the decays of the usual recipes round away.  The schedule is host-side
(``due_update``); the update itself is one ``stk_weight_avg`` launch after the optimizer step, on every route.  Nothing
here synchronises the host with the device.
"""
from contextlib import contextmanager
from typing import Dict, List, Optional, Tuple

import attr
import numpy as np
import torch

from .configs import WeightAverageConfig

COPY, LERP = 1, 2   # the `mode` values of stk_weight_avg


def due_update(kind: str, decay: float, every: int, start_step: int, step: int,
               n_averaged: int) -> Optional[Tuple[int, float]]:
    """The update due after optimizer step ``step`` (1-based), as ``(COPY | LERP, weight)``, or None.

    The first update copies (AveragedModel with ``n_averaged == 0``).  Later ones lerp with torch's fp32 weight: EMA
    ``fp32(1 - decay)`` (the python scalar ``1 - decay`` that ``torch._foreach_lerp_`` takes as fp32); SWA the fp32
    quotient ``1 / (n_averaged + 1)`` that torch forms from its integer ``n_averaged`` tensor."""
    if step <= start_step or (step - start_step) % every != 0:
        return None
    if n_averaged == 0:
        return COPY, 0.0
    if kind == "ema":
        return LERP, float(np.float32(1.0 - float(decay)))
    return LERP, float(np.float32(1.0) / np.float32(n_averaged + 1))


def apply_update(avgs: List[torch.Tensor], srcs: List[torch.Tensor], due: Tuple[int, float]):
    """``due`` applied to fp32 tensors with the foreach ops AveragedModel uses (the buffers of ``use_buffers``); the
    sources are taken as fp32."""
    mode, w = due
    srcs = [s.float() for s in srcs]
    if mode == COPY:
        torch._foreach_copy_(avgs, srcs)
    else:
        torch._foreach_lerp_(avgs, srcs, w)


class WeightAverage:
    """The handle ``Stoke.weight_average`` returns when a ``WeightAverageConfig`` is given.

    ``n_averaged``: updates taken since the start or the last ``reset()``.  ``decay`` (EMA) is read by every update, so a
    warm-up schedule is the training loop setting it.  ``state_dict()`` / ``load_state_dict()`` use the model's own
    ``state_dict`` names and shapes; ``applied()`` puts the average into the model for evaluation.  At world > 1 on the
    sharded route ``state_dict()`` and ``applied()`` gather: every rank calls them."""

    def __init__(self, config: WeightAverageConfig, path, module: torch.nn.Module):
        self.config = config
        self._path = path
        self._module = module
        self._decay = float(config.decay)
        self.n_averaged = 0
        self.active = False
        path.enable_weight_average()
        path.avg_owner = self
        self._name_of = {id(p): name for name, p in module.named_parameters()}
        # fp32 copies of the floating buffers (use_buffers); non-floating buffers (num_batches_tracked) are the model's
        self._buffers: Dict[str, torch.Tensor] = {}
        if config.use_buffers:
            self._buffers = {n: b.detach().float().clone() for n, b in module.named_buffers() if b.is_floating_point()}

    @property
    def decay(self) -> float:
        return self._decay

    @decay.setter
    def decay(self, value: float):
        if not 0.0 <= float(value) <= 1.0:
            raise ValueError(f"Stoke -- weight average decay must be in [0, 1], got {value}")
        self._decay = float(value)

    def reset(self):
        """The next update copies the master (the average starts afresh)."""
        self.n_averaged = 0

    def _check_idle(self, what: str):
        if self.active:
            raise RuntimeError(f"Stoke -- {what} inside weight_average.applied(): the model holds the average")

    def _schedule(self, step: int):
        """Called by ``Stoke.step`` before the optimizer step ``step`` (1-based): hands a due update to the step."""
        c = self.config
        due = due_update(c.kind, self._decay, c.every, c.start_step, step, self.n_averaged)
        if due is None:
            return
        self._path.avg_due = due
        if self._buffers:
            cur = dict(self._module.named_buffers())
            apply_update(list(self._buffers.values()), [cur[n].detach() for n in self._buffers], due)
        self.n_averaged += 1

    # -- export --------------------------------------------------------------------------------------------------------
    def state_dict(self) -> Dict[str, torch.Tensor]:
        """``{name: tensor}`` in the layout of ``model.state_dict()``: trainable parameters from the fp32 average, frozen
        parameters at their current values (fp32), buffers from their fp32 averages (``use_buffers``) or current values;
        non-floating buffers as they are.  A plain fp32 copy of the model loads it with ``strict=True``."""
        path = self._path
        avg = {id(p): v for p, v in zip(path.params, path.unflatten(path.gather_avg()))}
        out = {}
        for name, t in self._module.state_dict(keep_vars=True).items():
            if id(t) in avg:
                out[name] = avg[id(t)]
            elif name in self._buffers:
                out[name] = self._buffers[name].clone()
            elif t.is_floating_point():
                out[name] = t.detach().float().clone()
            else:
                out[name] = t.detach().clone()
        return out

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], n_averaged: int = 1):
        """Sets the average from a ``state_dict()``-layout dict (trainable parameters and, with ``use_buffers``, the
        floating buffers) and the count of updates it stands for (0: the next update copies)."""
        path = self._path
        full = torch.zeros(path.n, dtype=torch.float32, device=path.avg_flat.device)
        for view, p in zip(path.unflatten(full), path.params):
            view.copy_(state_dict[self._name_of[id(p)]])
        path.scatter_local(full, path.avg_flat)
        for name, avg in self._buffers.items():
            avg.copy_(state_dict[name])
        self.n_averaged = int(n_averaged)

    def _checkpoint(self) -> dict:
        return {"state_dict": self.state_dict(), "n_averaged": self.n_averaged,
                "config": attr.asdict(attr.evolve(self.config, decay=self._decay))}

    def _load_checkpoint(self, entry: Optional[dict]):
        """``Stoke.load``: the checkpoint's average, its ``n_averaged`` and the ``decay`` in force when it was saved (a
        loop that sets ``decay`` itself sets it again at its next step), or, from a checkpoint without one, an average
        started afresh from the loaded weights.  ``kind``, ``every``, ``start_step`` and ``use_buffers`` are the
        configuration of the Stoke that loads."""
        if entry is not None:
            self.load_state_dict(entry["state_dict"], entry["n_averaged"])
            self.decay = entry["config"]["decay"]
            return
        path = self._path
        path.avg_flat.copy_(path.master_flat)
        cur = dict(self._module.named_buffers())
        for name, avg in self._buffers.items():
            avg.copy_(cur[name])
        self.n_averaged = 0

    # -- evaluation ----------------------------------------------------------------------------------------------------
    @contextmanager
    def applied(self):
        """Inside: the model's parameters hold the average cast to the model dtype (bf16: round to nearest even), its
        floating buffers the averaged buffers when ``use_buffers``.  On exit both are restored bit for bit.
        ``Stoke.backward`` and ``Stoke.step`` raise inside."""
        self._check_idle("applied()")
        path = self._path
        saved_p = path.params_from_average()
        saved_b = {}
        if self._buffers:
            cur = dict(self._module.named_buffers())
            with torch.no_grad():
                for name, avg in self._buffers.items():
                    saved_b[name] = cur[name].detach().clone()
                    cur[name].copy_(avg)
        self.active = True
        try:
            yield self._module
        finally:
            self.active = False
            path.params_restore(saved_p)
            if saved_b:
                cur = dict(self._module.named_buffers())
                with torch.no_grad():
                    for name, b in saved_b.items():
                        cur[name].copy_(b)
