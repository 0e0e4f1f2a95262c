"""What the native optimizers (``SGD``, ``Adam``, ``AdamW``) share: the device-resident learning rate that a captured CUDA
graph reads, and the checks that decide whether the update may ride on the reference ConvNet's last backward kernel."""
from __future__ import annotations

import math
import os
from typing import List, Optional

import torch


class RidingOptimizer(torch.optim.Optimizer):
    """Base of the optimizers with a native multi-tensor update.  Bookkeeping (param_groups / state_dict) comes from
    ``torch.optim.Optimizer``."""

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._lr_dev = {}           # group index -> (device scalar, last host value) when capturable
        self._rode = False

    # ---- device-resident learning rate (CUDA-graph friendly schedulers) ------------------------------
    def _lr_tensor(self, gi: int, group, device) -> Optional[torch.Tensor]:
        if not group.get("capturable") or device.type != "cuda":
            return None
        ent = self._lr_dev.get(gi)
        if ent is None:
            ent = [torch.full((1,), float(group["lr"]), dtype=torch.float32, device=device), float(group["lr"])]
            self._lr_dev[gi] = ent
        elif ent[1] != float(group["lr"]) and not torch.cuda.is_current_stream_capturing():
            ent[0].fill_(float(group["lr"]))
            ent[1] = float(group["lr"])
        return ent[0]

    def sync_lr(self) -> None:
        """Push ``param_groups[i]['lr']`` into the device scalars a captured step reads (call between
        graph replays after a scheduler step; a no-op when nothing changed)."""
        for gi, group in enumerate(self.param_groups):
            ent = self._lr_dev.get(gi)
            if ent is not None and ent[1] != float(group["lr"]):
                ent[0].fill_(float(group["lr"]))
                ent[1] = float(group["lr"])

    # ---- single GPU: the update rides on the model's last backward kernel ---------------------------------
    def _qualify_rider(self, model) -> Optional[List[torch.Tensor]]:
        """The reference ConvNet's ten parameters in the rider's order (conv1.w, conv1.b, bn1.w, bn1.b, conv2.w, conv2.b, fc.w, fc.b,
        bn2.w, bn2.b) when this optimizer may ride on its last backward kernel: one parameter group that holds exactly these
        parameters, all fp32, contiguous and on the GPU, and a world size of 1.  None otherwise.  ``PDT_SGD_RIDER=0`` turns riding
        off for every optimizer."""
        from .. import distributed as dist

        if os.environ.get("PDT_SGD_RIDER", "1") == "0":
            return None
        group_ = getattr(model, "process_group", None)
        world = group_.size() if group_ is not None else (dist.get_world_size() if dist.is_initialized() else 1)
        if world > 1:
            return None   # the gradients still have to be averaged first
        inner = getattr(model, "module", model)
        try:
            c1, b1, c2, b2, fc = inner.layer1[0], inner.layer1[1], inner.layer2[0], inner.layer2[1], inner.fc
            params = [c1.weight, c1.bias, b1.weight, b1.bias, c2.weight, c2.bias, fc.weight, fc.bias, b2.weight, b2.bias]
        except (AttributeError, IndexError, TypeError):
            return None
        if len(self.param_groups) != 1 or any(q is None for q in params):
            return None
        mine = self.param_groups[0]["params"]
        if len(mine) != len(params) or {id(q) for q in mine} != {id(q) for q in params}:
            return None
        if not all(q.is_cuda and q.dtype == torch.float32 and q.is_contiguous() for q in params):
            return None
        return params

    @staticmethod
    def _clip_qualifies(clip, params) -> bool:
        """``clip = (max_norm, norm_type, norm_out)`` can ride: norm type 2 or inf, ``norm_out`` one fp32 element on the
        parameters' device."""
        max_norm, norm_type, out = clip
        return (float(norm_type) in (2.0, math.inf) and isinstance(out, torch.Tensor) and out.numel() == 1
                and out.dtype == torch.float32 and out.device == params[0].device)

    def _arm_rider(self, kind: str, params, args, clip=None) -> None:
        from ..ops import functional as OF

        if clip is not None:
            # the rider tuple gains a trailing clip entry: the kernel clips the gradients to max_norm before the update and stores
            # the total norm in norm_out
            entry = (float(clip[0]), float(clip[1]), clip[2])
            plain = args

            def args(prev_grads):
                t = plain(prev_grads)
                return None if t is None else tuple(t) + (entry,)

        self._riding_params = params
        self._rode = False
        OF._sgd_rider = {"kind": kind, "params": params, "args": args, "owner": self, "clip": clip}

    def stop_riding(self) -> None:
        """Undo :meth:`ride_on_backward`."""
        from ..ops import functional as OF

        if OF._sgd_rider is not None and OF._sgd_rider.get("owner") is self:
            OF._sgd_rider = None
        self._rode = False
