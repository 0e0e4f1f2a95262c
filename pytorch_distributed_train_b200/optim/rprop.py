"""Rprop with one fused multi-tensor kernel per step.

Constructor, defaults, errors and state keys (``step``, ``prev``, ``step_size``) are torch's, so a ``state_dict`` moves between this
class and ``torch.optim.Rprop`` in both directions.  Ours:

* the update of *all* fp32 contiguous CUDA parameters of a group is one sm_90a kernel launch (``ops.rprop_step``) with the
  arithmetic of torch's single-tensor Rprop, bit for bit; ``step`` lives on the parameter's device as an fp32 scalar and the kernel
  advances it;
* ``lr`` only sets the first ``step_size`` (``full_like(p, lr)``), as in torch, so it may change between graph replays and has no
  effect; the other hyper-parameters must not (``sync_lr``);
* on one GPU the update can ride on the reference ConvNet's last backward kernel (:meth:`Rprop.ride_on_backward`).

CPU parameters, other dtypes, complex parameters and ``differentiable=True`` take the reference math (torch's single-tensor
arithmetic).  ``foreach`` and ``capturable`` are kept in the group and saved; they do not change the native path.
"""
from __future__ import annotations

from typing import Iterable, Optional

import torch

from ._riding import RidingOptimizer


def _scalar(v):
    return v.item() if isinstance(v, torch.Tensor) else v


class Rprop(RidingOptimizer):
    def __init__(self, params: Iterable, lr: float = 1e-2, etas=(0.5, 1.2), step_sizes=(1e-6, 50), *, capturable: bool = False,
                 foreach: Optional[bool] = None, maximize: bool = False, differentiable: bool = False):
        # the checks and messages of torch.optim.Rprop
        if isinstance(lr, torch.Tensor) and lr.numel() != 1:
            raise ValueError("Tensor lr must be 1-element")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 < etas[0] < 1.0 < etas[1]:
            raise ValueError(f"Invalid eta values: {etas[0]}, {etas[1]}")
        # a tensor learning rate is read once here
        defaults = dict(lr=float(_scalar(lr)), etas=etas, step_sizes=step_sizes, foreach=foreach, maximize=maximize,
                        differentiable=differentiable, capturable=capturable)
        super().__init__(params, defaults)

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("foreach", None)
            group.setdefault("maximize", False)
            group.setdefault("differentiable", False)
            group.setdefault("capturable", False)

    # ---- state -----------------------------------------------------------------------------------------------
    def _state(self, p: torch.Tensor, group) -> dict:
        st = self.state[p]
        if len(st) == 0:
            # the step count lives on the parameter's device (torch's capturable layout): the kernel advances it
            st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
            st["prev"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            if p.dtype.is_complex:   # the real and imaginary parts step as two real numbers
                st["step_size"] = torch.full_like(p, complex(group["lr"], group["lr"]))
            else:
                st["step_size"] = torch.full_like(p, float(group["lr"]))
        return st

    def load_state_dict(self, state_dict) -> None:
        """Standard behaviour, plus: every ``step`` goes to its parameter's device as fp32 (the kernels read it there)."""
        super().load_state_dict(state_dict)
        self._steps_to_param_device()

    # ---- single GPU: the update rides on the model's last backward kernel ---------------------------------
    def ride_on_backward(self, model, clip=None) -> bool:
        """Let the reference ConvNet's last backward kernel apply this optimizer's update (csrc/cuda/fused_convnet.cu: RpropRider).
        Same contract, preconditions and ``clip = (max_norm, norm_type, norm_out)`` as :meth:`SGD.ride_on_backward`.
        ``differentiable=True`` does not ride.  Returns False (and changes nothing) when the model / optimizer combination does
        not qualify."""
        params = self._qualify_rider(model)
        if params is None or (clip is not None and not self._clip_qualifies(clip, params)):
            return False
        if self.param_groups[0]["differentiable"]:
            return False

        def build(prev_grads):
            group = self.param_groups[0]
            hyper = self._hyper(0, group, params[0].device)
            states = [self._state(q, group) for q in params]
            if not all(st[k].is_cuda and st[k].dtype == torch.float32 for st in states for k in ("step",)):
                return None   # leave this iteration to step()
            return dict(kind="rprop", params=params, prev_grads=list(prev_grads),
                        prev=[st["prev"] for st in states], step_size=[st["step_size"] for st in states],
                        step=[st["step"] for st in states], **hyper)

        self._arm_rider(params, build, clip)
        return True

    _FIXED_KEYS = ("etas", "step_sizes", "maximize")

    def _hyper(self, gi: int, group, device) -> dict:
        """The update's hyper-parameters, as ``ops.rprop_step`` and the rider description of the last backward kernel take them (the
        group keys ``_FIXED_KEYS``; ``lr`` is not one: it only sets the first step sizes)."""
        etaminus, etaplus = group["etas"]
        step_min, step_max = group["step_sizes"]
        return dict(etaminus=float(etaminus), etaplus=float(etaplus), step_size_min=float(step_min), step_size_max=float(step_max),
                    maximize=bool(group["maximize"]))

    # ---- the update ---------------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        from .. import ops

        if self._rode:
            self._rode = False   # the last backward kernel applied this step's update (ride_on_backward)
            return loss
        for gi, group in enumerate(self.param_groups):
            params, grads = [], []
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("Rprop does not support sparse gradients")
                params.append(p)
                grads.append(p.grad)
            if not params:
                continue
            states = [self._state(p, group) for p in params]
            native = not group["differentiable"] and params[0].is_cuda and ops.native_available() and all(
                p.dtype == torch.float32 and p.is_contiguous() and g.dtype == torch.float32 and g.is_contiguous() and p.device == params[0].device
                for p, g in zip(params, grads))
            if native:
                ops.rprop_step(params, grads, [st["prev"] for st in states], [st["step_size"] for st in states],
                               [st["step"] for st in states], **self._hyper(gi, group, params[0].device))
                continue
            self._reference_step(group, params, grads, states)
        return loss

    @staticmethod
    def _reference_step(group, params, grads, states) -> None:
        """torch's single-tensor Rprop (CPU parameters, other dtypes, complex parameters, ``differentiable=True``)."""
        from torch.optim.rprop import rprop

        etaminus, etaplus = group["etas"]
        step_min, step_max = group["step_sizes"]
        rprop(params, grads, [st["prev"] for st in states], [st["step_size"] for st in states], [st["step"] for st in states],
              foreach=False, capturable=False, maximize=group["maximize"], differentiable=group["differentiable"],
              has_complex=any(torch.is_complex(p) for p in params), step_size_min=step_min, step_size_max=step_max, etaminus=etaminus,
              etaplus=etaplus)
