"""Weight averaging with torch's interface (``torch.optim.swa_utils``) and a native, graph-capturable update.

``AveragedModel`` is torch's class with the same constructor, ``state_dict`` keys and ``n_averaged`` buffer.  Its
``update_parameters`` runs ``ops.average_update`` — one kernel launch per 48 tensors that reads ``n_averaged`` on the device
and advances it there — when the averaging function is one of this module's ``get_ema_multi_avg_fn`` / ``get_swa_multi_avg_fn``
(or the default, SWA) and every tensor is a contiguous CUDA tensor on one device, fp32 or int64 (``num_batches_tracked``).  The
result is torch's bit for bit.  Everything else takes torch's own update, which reads ``n_averaged`` on the host and so cannot be
captured in a CUDA graph: a custom ``avg_fn`` or ``multi_avg_fn``, torch's untagged functions, CPU tensors, other dtypes, and SWA
with ``use_buffers=True`` over integer buffers (torch's ``swa_update`` cannot average those and raises).

One difference in placement: built without ``device=``, torch's ``n_averaged`` lives on the CPU whatever the model's device;
here it is put on the device of the model's first tensor, so the native update never synchronises.
"""
from __future__ import annotations

import itertools
from typing import List, Optional, Tuple, Union

import torch
from torch.optim import swa_utils as _torch_swa
from torch.optim.swa_utils import SWALR, get_ema_avg_fn, get_swa_avg_fn, update_bn  # noqa: F401  (torch's, re-exported)

__all__ = ["AveragedModel", "SWALR", "get_ema_avg_fn", "get_ema_multi_avg_fn", "get_swa_avg_fn", "get_swa_multi_avg_fn", "update_bn"]


def get_ema_multi_avg_fn(decay: float = 0.999):
    """torch's EMA ``multi_avg_fn`` (same validation of ``decay``, same result when torch calls it), tagged so that
    ``AveragedModel`` runs it natively."""
    fn = _torch_swa.get_ema_multi_avg_fn(decay)
    fn._pdt_average = ("ema", float(decay))
    return fn


def get_swa_multi_avg_fn():
    """torch's SWA ``multi_avg_fn``, tagged so that ``AveragedModel`` runs it natively."""
    fn = _torch_swa.get_swa_multi_avg_fn()
    fn._pdt_average = ("swa", None)
    return fn


_Plan = Tuple[List[torch.Tensor], List[torch.Tensor], List[torch.Tensor], List[torch.Tensor], Optional[float]]


class AveragedModel(_torch_swa.AveragedModel):
    def __init__(self, model: torch.nn.Module, device=None, avg_fn=None, multi_avg_fn=None, use_buffers=False):
        super().__init__(model, device, avg_fn, multi_avg_fn, use_buffers)
        if device is None:
            first = next(itertools.chain(self.module.parameters(), self.module.buffers()), None)
            if first is not None and first.device != self.n_averaged.device:
                self.n_averaged = self.n_averaged.to(first.device)

    def native_plan(self, model: torch.nn.Module) -> Union[_Plan, str]:
        """``(averaged, current, copied, copied_from, decay)`` for ``ops.average_update`` (``decay`` None: SWA) when updating from
        ``model`` can run natively, else the reason it cannot."""
        if self.avg_fn is not None:
            return "a custom avg_fn"
        if self.multi_avg_fn is None:
            decay = None   # torch's default on a CUDA device: get_swa_multi_avg_fn()
        else:
            tag = getattr(self.multi_avg_fn, "_pdt_average", None)
            if tag is None:
                return "an untagged multi_avg_fn (use pdt.optim.swa_utils.get_ema_multi_avg_fn / get_swa_multi_avg_fn)"
            decay = tag[1]
        mine, theirs = list(self.module.parameters()), list(model.parameters())
        mine_b, theirs_b = list(self.module.buffers()), list(model.buffers())
        if len(mine) != len(theirs) or len(mine_b) != len(theirs_b):
            return "the averaged model and the model have different numbers of tensors"
        if self.use_buffers:
            averaged, current, copied, copied_from = mine + mine_b, theirs + theirs_b, [], []
        else:
            averaged, current, copied, copied_from = mine, theirs, mine_b, theirs_b
        dev = self.n_averaged.device
        if dev.type != "cuda":
            return "n_averaged is not on a CUDA device"
        for i, (a, c) in enumerate(zip(averaged + copied, current + copied_from)):
            if a.device != dev or c.device != dev:
                return "tensors on more than one device, or not on CUDA"
            if a.dtype != c.dtype or a.dtype not in (torch.float32, torch.int64) or a.shape != c.shape:
                return "a tensor that is neither float32 nor int64, or whose dtype or shape differs from the model's"
            if not (a.is_contiguous() and c.is_contiguous()):
                return "a non-contiguous tensor"
            if i < len(averaged) and a.dtype == torch.int64 and decay is None:
                return "SWA over an integer buffer (torch's swa_update cannot average it)"
        if not averaged and not copied:
            return "no tensors"
        return ([a.detach() for a in averaged], [c.detach() for c in current], [a.detach() for a in copied],
                [c.detach() for c in copied_from], decay)

    def update_parameters(self, model: torch.nn.Module) -> None:
        plan = self.native_plan(model)
        if isinstance(plan, str):
            return super().update_parameters(model)
        from .. import ops

        averaged, current, copied, copied_from, decay = plan
        ops.average_update(averaged, current, self.n_averaged, decay, copied, copied_from)
