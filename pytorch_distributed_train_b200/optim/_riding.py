"""What the native optimizers (``SGD``, ``Adam``, ``AdamW``, ``NAdam``, ``RAdam``, ``RMSprop``, ``Adagrad``, ``Adamax``, ``Adadelta``,
``ASGD``, ``Rprop``) share: the device-resident learning rate that a captured CUDA graph reads, the device-resident step counts (and
NAdam's ``mu_product``, ASGD's ``eta`` and ``mu``) that its kernels advance, and the checks that decide whether the update may ride on
the reference ConvNet's last backward kernel.

The learning rate lives in a device scalar per group when the group says ``capturable=True``, and for every group once
``engine.GraphedTrainStep`` has taken the optimizer: the captured kernels then read the scalar, and ``sync_lr()`` before each replay
pushes a scheduler's change into it.  Every other hyper-parameter is a kernel argument baked into the graph; a replay after one of
them changed is refused (``sync_lr``)."""
from __future__ import annotations

import math
import operator
import os
from dataclasses import dataclass
from typing import Callable, List, Optional, Tuple

import torch


@dataclass
class Rider:
    """An optimizer armed to ride on the reference ConvNet's last backward kernel (``ops.functional._sgd_rider``).  ``params``: its ten
    parameters in the kernel's order; ``clip``: ``(max_norm, norm_type, norm_out)`` or None; ``build(prev_grads)``: the rider
    description ``convnet_l1_bwd_wgrad`` takes, or None when the optimizer cannot ride this iteration."""
    owner: "RidingOptimizer"
    params: List[torch.Tensor]
    clip: Optional[Tuple[float, float, torch.Tensor]]
    build: Callable[[list], Optional[dict]]


class RidingOptimizer(torch.optim.Optimizer):
    """Base of the optimizers with a native multi-tensor update.  Bookkeeping (param_groups / state_dict) comes from
    ``torch.optim.Optimizer``."""

    # the group keys ``_hyper`` reads besides ``lr`` (at least two, so that ``itemgetter`` returns a tuple); a subclass names its own
    _FIXED_KEYS: Tuple[str, ...] = ()

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._lr_dev = {}           # group index -> (device scalar, last host value) when capturable
        self._rode = False
        # set by engine.GraphedTrainStep: every group's lr in a device scalar, whatever its ``capturable`` says (the group's
        # ``capturable`` is left alone: it is saved in state_dict)
        self._lr_on_device = False
        self._captured_hyper = None   # per group, the values of _FIXED_KEYS when GraphedTrainStep captured its step

    # ---- device-resident learning rate (CUDA-graph friendly schedulers) ------------------------------
    def _lr_tensor(self, gi: int, group, device) -> Optional[torch.Tensor]:
        if not (group.get("capturable") or self._lr_on_device) or device.type != "cuda":
            return None
        ent = self._lr_dev.get(gi)
        if ent is None:
            ent = [torch.full((1,), float(group["lr"]), dtype=torch.float32, device=device), float(group["lr"])]
            self._lr_dev[gi] = ent
        elif ent[1] != float(group["lr"]) and not torch.cuda.is_current_stream_capturing():
            ent[0].fill_(float(group["lr"]))
            ent[1] = float(group["lr"])
        return ent[0]

    def _record_captured_hyper(self) -> None:
        """Remember the hyper-parameters a captured step baked into its kernels (``sync_lr`` refuses a replay once they differ)."""
        self._fixed_of = operator.itemgetter(*self._FIXED_KEYS)
        self._captured_hyper = [self._fixed_of(g) for g in self.param_groups]

    def sync_lr(self) -> None:
        """Push ``param_groups[i]['lr']`` into the device scalars a captured step reads (call between
        graph replays after a scheduler step; a no-op when nothing changed).  After ``engine.GraphedTrainStep`` has captured
        a step, raises RuntimeError when any other hyper-parameter the update reads (momentum, betas, weight decay, …) has
        changed since: the graph would replay the captured value.  Runs before every replay, so the check is one tuple
        comparison per group."""
        captured = self._captured_hyper
        for gi, group in enumerate(self.param_groups):
            if captured is not None and gi < len(captured):
                now = self._fixed_of(group)
                if now != captured[gi]:
                    key, was, new = next((k, a, b) for k, a, b in zip(self._FIXED_KEYS, captured[gi], now) if a != b)
                    raise RuntimeError(
                        f"{type(self).__name__}: hyper-parameter '{key}' of param_groups[{gi}] changed from {was} to {new} after "
                        "the training step was captured in a CUDA graph, which would replay the captured value; only 'lr' can "
                        "change between replays (a scheduler that also cycles momentum or betas needs an eager loop)")
            ent = self._lr_dev.get(gi)
            if ent is not None and ent[1] != float(group["lr"]):
                ent[0].fill_(float(group["lr"]))
                ent[1] = float(group["lr"])

    def _steps_to_param_device(self) -> None:
        """Move every state's ``step`` (and NAdam's ``mu_product``, ASGD's ``eta`` and ``mu``) to its parameter's device as an fp32
        scalar, after ``load_state_dict``: torch keeps ``step`` on the CPU unless the saved group says ``capturable`` or ``fused``,
        casts the other scalars to the parameter's dtype, and the kernels read them where the parameter is, in fp32."""
        for group in self.param_groups:
            for p in group["params"]:
                st = self.state.get(p)
                for key in ("step", "mu_product", "eta", "mu"):
                    if st and key in st:
                        s = st[key]
                        s = s if isinstance(s, torch.Tensor) else torch.tensor(float(s))
                        st[key] = s.to(device=p.device, dtype=torch.float32).reshape(())

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

    def _arm_rider(self, params, build, clip=None) -> None:
        from ..ops import functional as OF

        self._rode = False
        OF._sgd_rider = Rider(self, params, None if clip is None else (float(clip[0]), float(clip[1]), clip[2]), build)

    def stop_riding(self) -> None:
        """Undo :meth:`ride_on_backward`."""
        from ..ops import functional as OF

        if OF._sgd_rider is not None and OF._sgd_rider.owner is self:
            OF._sgd_rider = None
        self._rode = False
