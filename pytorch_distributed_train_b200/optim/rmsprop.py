"""RMSprop with one fused multi-tensor kernel per step.

Constructor, defaults, errors and state keys (``step``, ``square_avg``, plus ``momentum_buffer`` when ``momentum > 0`` and
``grad_avg`` when ``centered``) are torch's, so a ``state_dict`` moves between this class and ``torch.optim.RMSprop`` in both
directions.  Ours:

* the update of *all* fp32 contiguous CUDA parameters of a group is one sm_90a kernel launch (``ops.rmsprop_step``) with the
  arithmetic of torch's single-tensor RMSprop, momentum and centering included; it is graph-capturable because ``step`` lives on
  the parameter's device as an fp32 scalar and the kernel advances it itself;
* ``lr`` lives in a device scalar when ``capturable=True``, and always once ``engine.GraphedTrainStep`` has taken the optimizer,
  so schedulers work under CUDA graphs (the other hyper-parameters must not change between replays: ``sync_lr``);
* on one GPU the update can ride on the reference ConvNet's last backward kernel (:meth:`RMSprop.ride_on_backward`).

CPU parameters, other dtypes, complex parameters and ``differentiable=True`` take the reference math (torch's single-tensor
arithmetic).
"""
from __future__ import annotations

from typing import Iterable, Optional

import torch

from ._riding import RidingOptimizer


def _scalar(v):
    return v.item() if isinstance(v, torch.Tensor) else v


class RMSprop(RidingOptimizer):
    def __init__(self, params: Iterable, lr: float = 1e-2, alpha: float = 0.99, eps: float = 1e-8, weight_decay: float = 0,
                 momentum: float = 0, centered: bool = False, capturable: bool = False, foreach: Optional[bool] = None,
                 maximize: bool = False, differentiable: bool = False):
        # the checks and messages of torch.optim.RMSprop
        if isinstance(lr, torch.Tensor) and lr.numel() != 1:
            raise ValueError("Tensor lr must be 1-element")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= momentum:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if not 0.0 <= alpha:
            raise ValueError(f"Invalid alpha value: {alpha}")
        # the kernels take host scalars: a tensor learning rate is read once here
        defaults = dict(lr=float(_scalar(lr)), momentum=momentum, alpha=alpha, eps=eps, centered=centered, weight_decay=weight_decay,
                        capturable=capturable, foreach=foreach, maximize=maximize, differentiable=differentiable)
        super().__init__(params, defaults)

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("momentum", 0)
            group.setdefault("centered", False)
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
            st["square_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        if group["momentum"] > 0 and "momentum_buffer" not in st:
            st["momentum_buffer"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        if group["centered"] and "grad_avg" not in st:
            st["grad_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        return st

    def load_state_dict(self, state_dict) -> None:
        """Standard behaviour, plus: every ``step`` goes to its parameter's device as fp32 (the kernels read it there)."""
        super().load_state_dict(state_dict)
        self._steps_to_param_device()

    # ---- single GPU: the update rides on the model's last backward kernel ---------------------------------
    def ride_on_backward(self, model, clip=None) -> bool:
        """Let the reference ConvNet's last backward kernel apply this optimizer's update (csrc/cuda/fused_convnet.cu: RmspropRider).
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
            if not all(st["step"].is_cuda and st["step"].dtype == torch.float32 for st in states):
                return None   # leave this iteration to step()
            centered = hyper.pop("centered")
            return dict(kind="rmsprop", params=params, prev_grads=list(prev_grads), square_avg=[st["square_avg"] for st in states],
                        step=[st["step"] for st in states],
                        momentum_buffer=[st["momentum_buffer"] for st in states] if hyper["momentum"] > 0 else [],
                        grad_avg=[st["grad_avg"] for st in states] if centered else [], **hyper)

        self._arm_rider(params, build, clip)
        return True

    _FIXED_KEYS = ("alpha", "eps", "weight_decay", "momentum", "centered", "maximize")

    def _hyper(self, gi: int, group, device) -> dict:
        """The update's hyper-parameters, as ``ops.rmsprop_step`` and the rider description of the last backward kernel take them
        (``lr`` and the group keys ``_FIXED_KEYS``; the caller pops ``centered``, which decides whether ``grad_avg`` is passed)."""
        return dict(lr=float(group["lr"]), lr_tensor=self._lr_tensor(gi, group, device), alpha=float(group["alpha"]),
                    eps=float(group["eps"]), weight_decay=float(group["weight_decay"]), momentum=float(group["momentum"]),
                    maximize=bool(group["maximize"]), centered=bool(group["centered"]))

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
                    raise RuntimeError("RMSprop does not support sparse gradients")
                params.append(p)
                grads.append(p.grad)
            if not params:
                continue
            states = [self._state(p, group) for p in params]
            native = not group["differentiable"] and params[0].is_cuda and ops.native_available() and all(
                p.dtype == torch.float32 and p.is_contiguous() and g.dtype == torch.float32 and g.is_contiguous() and p.device == params[0].device
                for p, g in zip(params, grads))
            if native:
                hyper = self._hyper(gi, group, params[0].device)
                centered = hyper.pop("centered")
                ops.rmsprop_step(params, grads, [st["square_avg"] for st in states], [st["step"] for st in states], **hyper,
                                 momentum_buffers=[st["momentum_buffer"] for st in states] if hyper["momentum"] > 0 else None,
                                 grad_avgs=[st["grad_avg"] for st in states] if centered else None)
                continue
            self._reference_step(group, params, grads, states)
        return loss

    @staticmethod
    def _reference_step(group, params, grads, states) -> None:
        """torch's single-tensor RMSprop (CPU parameters, other dtypes, complex parameters, ``differentiable=True``)."""
        from torch.optim.rmsprop import rmsprop

        rmsprop(params, grads, [st["square_avg"] for st in states], [st["grad_avg"] for st in states] if group["centered"] else [],
                [st["momentum_buffer"] for st in states] if group["momentum"] > 0 else [], [st["step"] for st in states],
                foreach=False, maximize=group["maximize"], differentiable=group["differentiable"], capturable=False,
                has_complex=any(torch.is_complex(p) for p in params), lr=group["lr"], alpha=group["alpha"], eps=group["eps"],
                weight_decay=group["weight_decay"], momentum=group["momentum"], centered=group["centered"])
