"""Adagrad with one fused multi-tensor kernel per step.

Constructor, defaults, errors and state keys (``step``, ``sum``) are torch's, and the state is created in the constructor as
torch creates it, so a ``state_dict`` moves between this class and ``torch.optim.Adagrad`` in both directions, also before the
first step.  Ours:

* the update of *all* fp32 contiguous CUDA parameters of a group is one sm_90a kernel launch (``ops.adagrad_step``) with the
  arithmetic of torch's single-tensor Adagrad; ``step`` lives on the parameter's device as an fp32 scalar, and the kernel decays
  the learning rate from it and advances it, so a captured step decays ``lr`` from replay to replay (torch's class computes the
  decayed learning rate on the host, so a CUDA graph would replay the captured one);
* ``lr`` lives in a device scalar once ``engine.GraphedTrainStep`` has taken the optimizer, so schedulers work under CUDA graphs
  (the other hyper-parameters must not change between replays: ``sync_lr``);
* on one GPU the update can ride on the reference ConvNet's last backward kernel (:meth:`Adagrad.ride_on_backward`).

CPU parameters, other dtypes, complex parameters, sparse gradients and ``fused=False`` take the reference math (torch's
single-tensor arithmetic); ``fused=True`` with any of them raises.
"""
from __future__ import annotations

from typing import Iterable, Optional

import torch

from ._riding import RidingOptimizer


def _scalar(v):
    return v.item() if isinstance(v, torch.Tensor) else v


class Adagrad(RidingOptimizer):
    def __init__(self, params: Iterable, lr: float = 1e-2, lr_decay: float = 0, weight_decay: float = 0,
                 initial_accumulator_value: float = 0, eps: float = 1e-10, foreach: Optional[bool] = None, *,
                 maximize: bool = False, differentiable: bool = False, fused: Optional[bool] = None):
        # the checks and messages of torch.optim.Adagrad
        if isinstance(lr, torch.Tensor) and lr.numel() != 1:
            raise ValueError("Tensor lr must be 1-element")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= lr_decay:
            raise ValueError(f"Invalid lr_decay value: {lr_decay}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if not 0.0 <= initial_accumulator_value:
            raise ValueError(f"Invalid initial_accumulator_value value: {initial_accumulator_value}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        # the kernels take host scalars: a tensor learning rate is read once here
        defaults = dict(lr=float(_scalar(lr)), lr_decay=lr_decay, eps=eps, weight_decay=weight_decay,
                        initial_accumulator_value=initial_accumulator_value, foreach=foreach, maximize=maximize,
                        differentiable=differentiable, fused=fused)
        super().__init__(params, defaults)
        if fused:
            if differentiable:
                raise RuntimeError("`fused` does not support `differentiable`")
            if foreach:
                raise RuntimeError("`fused` and `foreach` cannot be `True` together.")
        for group in self.param_groups:
            for p in group["params"]:
                self._state(p, group)

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("foreach", None)
            group.setdefault("maximize", False)
            group.setdefault("differentiable", False)
            group.setdefault("fused", None)

    # ---- state -----------------------------------------------------------------------------------------------
    def _state(self, p: torch.Tensor, group) -> dict:
        st = self.state[p]
        if len(st) == 0:
            # the step count lives on the parameter's device: the kernel reads and advances it
            st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
            v = group["initial_accumulator_value"]
            st["sum"] = torch.full_like(p, complex(v, v) if torch.is_complex(p) else v, memory_format=torch.preserve_format)
        return st

    def load_state_dict(self, state_dict) -> None:
        """Standard behaviour, plus: every ``step`` goes to its parameter's device as fp32 (torch keeps it on the CPU; the kernels
        read it where the parameter is)."""
        super().load_state_dict(state_dict)
        self._steps_to_param_device()

    # ---- single GPU: the update rides on the model's last backward kernel ---------------------------------
    def ride_on_backward(self, model, clip=None) -> bool:
        """Let the reference ConvNet's last backward kernel apply this optimizer's update (csrc/cuda/fused_convnet.cu: AdagradRider).
        Same contract, preconditions and ``clip = (max_norm, norm_type, norm_out)`` as :meth:`SGD.ride_on_backward`.
        ``fused=False`` does not ride.  Returns False (and changes nothing) when the model / optimizer combination does not
        qualify."""
        params = self._qualify_rider(model)
        if params is None or (clip is not None and not self._clip_qualifies(clip, params)):
            return False
        if self.param_groups[0]["fused"] is False:
            return False

        def build(prev_grads):
            group = self.param_groups[0]
            states = [self._state(q, group) for q in params]
            if not all(st["step"].is_cuda and st["step"].dtype == torch.float32 for st in states):
                return None   # leave this iteration to step()
            return dict(kind="adagrad", params=params, prev_grads=list(prev_grads), sum=[st["sum"] for st in states],
                        step=[st["step"] for st in states], **self._hyper(0, group, params[0].device))

        self._arm_rider(params, build, clip)
        return True

    _FIXED_KEYS = ("lr_decay", "eps", "weight_decay", "maximize")

    def _hyper(self, gi: int, group, device) -> dict:
        """The update's hyper-parameters, as ``ops.adagrad_step`` and the rider description of the last backward kernel take them
        (``lr`` and the group keys ``_FIXED_KEYS``)."""
        return dict(lr=float(group["lr"]), lr_tensor=self._lr_tensor(gi, group, device), lr_decay=float(group["lr_decay"]),
                    eps=float(group["eps"]), weight_decay=float(group["weight_decay"]), maximize=bool(group["maximize"]))

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
                if p.grad is not None:
                    params.append(p)
                    grads.append(p.grad)
            if not params:
                continue
            states = [self._state(p, group) for p in params]
            native = group["fused"] is not False and params[0].is_cuda and ops.native_available() and all(
                p.dtype == torch.float32 and p.is_contiguous() and g.dtype == torch.float32 and not g.is_sparse and g.is_contiguous()
                and p.device == params[0].device for p, g in zip(params, grads))
            if native:
                ops.adagrad_step(params, grads, [st["sum"] for st in states], [st["step"] for st in states],
                                 **self._hyper(gi, group, params[0].device))
                continue
            if group["fused"]:
                raise RuntimeError("Adagrad(fused=True): the native kernel takes fp32 contiguous dense CUDA parameters on one device")
            self._reference_step(group, params, grads, states)
        return loss

    @staticmethod
    def _reference_step(group, params, grads, states) -> None:
        """torch's single-tensor Adagrad (CPU parameters, other dtypes, complex parameters, sparse gradients, ``fused=False``)."""
        from torch.optim.adagrad import adagrad

        adagrad(params, grads, [st["sum"] for st in states], [st["step"] for st in states], fused=False,
                has_sparse_grad=any(g.is_sparse for g in grads), foreach=False, differentiable=group["differentiable"],
                has_complex=any(torch.is_complex(p) for p in params), lr=group["lr"], weight_decay=group["weight_decay"],
                lr_decay=group["lr_decay"], eps=group["eps"], maximize=group["maximize"])
