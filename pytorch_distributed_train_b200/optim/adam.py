"""Adam and AdamW with one fused multi-tensor kernel per step.

Constructors, defaults, errors and state keys (``step``, ``exp_avg``, ``exp_avg_sq``, ``max_exp_avg_sq``) are torch's, so a
``state_dict`` moves between these classes and ``torch.optim.Adam`` / ``AdamW`` in both directions.  Ours:

* the update of *all* fp32 contiguous CUDA parameters of a group is one sm_90a kernel launch (``ops.adam_step``) with the
  arithmetic of torch's single-tensor Adam; it is graph-capturable because ``step`` lives on the parameter's device as an fp32
  scalar (as in torch's capturable mode) and the kernel advances it itself;
* ``lr`` lives in a device scalar when ``capturable=True``, and always once ``engine.GraphedTrainStep`` has taken the optimizer,
  so schedulers work under CUDA graphs (shared with ``SGD``; the betas and the other hyper-parameters must not change between
  replays: ``sync_lr``);
* ``amsgrad=True`` runs the same kernels with the running maximum ``max_exp_avg_sq`` as a fourth state tensor (``torch.maximum``'s
  NaN-keeping max, then the denominator from it);
* on one GPU the update can ride on the reference ConvNet's last backward kernel (:meth:`Adam.ride_on_backward`).

CPU parameters, other dtypes and ``fused=False`` take the reference math (torch's single-tensor arithmetic, op by op).
"""
from __future__ import annotations

from typing import Iterable, Optional

import torch

from ._riding import RidingOptimizer


def _scalar(v):
    return v.item() if isinstance(v, torch.Tensor) else v


class Adam(RidingOptimizer):
    def __init__(self, params: Iterable, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0,
                 amsgrad: bool = False, *, foreach: Optional[bool] = None, maximize: bool = False, capturable: bool = False,
                 differentiable: bool = False, fused: Optional[bool] = None, decoupled_weight_decay: bool = False):
        # the checks and messages of torch.optim.Adam
        if isinstance(lr, torch.Tensor):
            if foreach and not capturable:
                raise ValueError("lr as a Tensor is not supported for capturable=False and foreach=True")
            if lr.numel() != 1:
                raise ValueError("Tensor lr must be 1-element")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if not ((isinstance(betas[0], float) and isinstance(betas[1], float))
                or (isinstance(betas[0], torch.Tensor) and isinstance(betas[1], torch.Tensor))):
            raise ValueError("betas must be either both floats or both Tensors")
        for i, b in enumerate(betas):
            if isinstance(b, torch.Tensor):
                if not capturable and foreach:
                    raise ValueError(f"betas[{i}] as a Tensor is not supported for capturable=False and foreach=True")
                if b.numel() != 1:
                    raise ValueError(f"Tensor betas[{i}] must be 1-element")
        # the kernels take host scalars: a tensor learning rate or beta is read once here
        defaults = dict(lr=float(_scalar(lr)), betas=(float(_scalar(betas[0])), float(_scalar(betas[1]))), eps=eps,
                        weight_decay=weight_decay, amsgrad=amsgrad, maximize=maximize, foreach=foreach, capturable=capturable,
                        differentiable=differentiable, fused=fused, decoupled_weight_decay=decoupled_weight_decay)
        super().__init__(params, defaults)
        if fused:
            if differentiable:
                raise RuntimeError("`fused` does not support `differentiable`")
            if foreach:
                raise RuntimeError("`fused` and `foreach` cannot be `True` together.")

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("amsgrad", False)
            group.setdefault("maximize", False)
            group.setdefault("foreach", None)
            group.setdefault("capturable", False)
            group.setdefault("differentiable", False)
            group.setdefault("fused", None)
            group.setdefault("decoupled_weight_decay", False)

    # ---- state -----------------------------------------------------------------------------------------------
    def _state(self, p: torch.Tensor, amsgrad: bool) -> dict:
        st = self.state[p]
        if len(st) == 0:
            # the step count lives on the parameter's device (torch's capturable layout): the kernel reads and advances it
            st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
            st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        if amsgrad and "max_exp_avg_sq" not in st:
            st["max_exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        return st

    def load_state_dict(self, state_dict) -> None:
        """Standard behaviour, plus: every ``step`` goes to its parameter's device as fp32.  torch leaves it on the CPU unless
        the saved group says ``capturable`` or ``fused``; the kernels need it where the parameter is."""
        super().load_state_dict(state_dict)
        for group in self.param_groups:
            for p in group["params"]:
                st = self.state.get(p)
                if st and "step" in st:
                    s = st["step"]
                    s = s if isinstance(s, torch.Tensor) else torch.tensor(float(s))
                    st["step"] = s.to(device=p.device, dtype=torch.float32).reshape(())

    # ---- single GPU: the update rides on the model's last backward kernel ---------------------------------
    def ride_on_backward(self, model, clip=None) -> bool:
        """Let the reference ConvNet's last backward kernel apply this optimizer's update (csrc/cuda/fused_convnet.cu: AdamRider).
        Same contract, preconditions and ``clip = (max_norm, norm_type, norm_out)`` as :meth:`SGD.ride_on_backward`; with ``amsgrad``
        the kernel also keeps ``max_exp_avg_sq`` (AmsgradRider).  ``fused=False`` does not ride.  Returns False (and changes nothing)
        when the model / optimizer combination does not qualify."""
        params = self._qualify_rider(model)
        if params is None or (clip is not None and not self._clip_qualifies(clip, params)):
            return False
        if self.param_groups[0]["fused"] is False:
            return False

        def build(prev_grads):
            hyper = self._hyper(0, self.param_groups[0], params[0].device)
            amsgrad = hyper.pop("amsgrad")
            states = [self._state(q, amsgrad) for q in params]
            if not all(st["step"].is_cuda and st["step"].dtype == torch.float32 for st in states):
                return None   # leave this iteration to step()
            if amsgrad:
                hyper["max_exp_avg_sq"] = [st["max_exp_avg_sq"] for st in states]
            return dict(kind="adam", params=params, prev_grads=list(prev_grads), exp_avg=[st["exp_avg"] for st in states],
                        exp_avg_sq=[st["exp_avg_sq"] for st in states], step=[st["step"] for st in states], **hyper)

        self._arm_rider(params, build, clip)
        return True

    _FIXED_KEYS = ("betas", "eps", "weight_decay", "decoupled_weight_decay", "maximize", "amsgrad")

    def _hyper(self, gi: int, group, device) -> dict:
        """The update's hyper-parameters, as ``ops.adam_step`` and the rider description of the last backward kernel take them
        (``lr`` and the group keys ``_FIXED_KEYS``; the caller pops ``amsgrad``, which decides whether ``max_exp_avg_sq`` is passed)."""
        beta1, beta2 = group["betas"]
        return dict(lr=float(group["lr"]), lr_tensor=self._lr_tensor(gi, group, device), beta1=float(beta1), beta2=float(beta2),
                    eps=float(group["eps"]), weight_decay=float(group["weight_decay"]), decoupled=bool(group["decoupled_weight_decay"]),
                    maximize=bool(group["maximize"]), amsgrad=bool(group["amsgrad"]))

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
                    raise RuntimeError("Adam does not support sparse gradients, please consider SparseAdam instead")
                params.append(p)
                grads.append(p.grad)
            if not params:
                continue
            amsgrad = group["amsgrad"]
            states = [self._state(p, amsgrad) for p in params]
            native = group["fused"] is not False and params[0].is_cuda and ops.native_available() and all(
                p.dtype == torch.float32 and p.is_contiguous() and g.dtype == torch.float32 and g.is_contiguous() and p.device == params[0].device
                for p, g in zip(params, grads))
            if native:
                hyper = self._hyper(gi, group, params[0].device)
                vmax = [st["max_exp_avg_sq"] for st in states] if hyper.pop("amsgrad") else None
                ops.adam_step(params, grads, [st["exp_avg"] for st in states], [st["exp_avg_sq"] for st in states],
                              [st["step"] for st in states], **hyper, max_exp_avg_sqs=vmax)
                continue
            if group["fused"]:
                raise RuntimeError("Adam(fused=True): the native kernel takes fp32 contiguous CUDA parameters on one device")
            self._reference_step(group, params, grads, states)
        return loss

    @staticmethod
    def _reference_step(group, params, grads, states) -> None:
        """torch's single-tensor Adam, op by op (CPU parameters, other dtypes, ``fused=False``)."""
        lr, (beta1, beta2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
        for p, g, st in zip(params, grads, states):
            g = -g if group["maximize"] else g
            st["step"] += 1
            if wd != 0:
                if group["decoupled_weight_decay"]:
                    p.mul_(1 - lr * wd)
                else:
                    g = g.add(p, alpha=wd)
            st["exp_avg"].lerp_(g, 1 - beta1)
            st["exp_avg_sq"].mul_(beta2).addcmul_(g, g, value=1 - beta2)
            step = st["step"].item()
            step_size = lr / (1 - beta1 ** step)
            bc2_sqrt = (1 - beta2 ** step) ** 0.5
            if group["amsgrad"]:
                torch.maximum(st["max_exp_avg_sq"], st["exp_avg_sq"], out=st["max_exp_avg_sq"])
                denom = (st["max_exp_avg_sq"].sqrt() / bc2_sqrt).add_(eps)
            else:
                denom = (st["exp_avg_sq"].sqrt() / bc2_sqrt).add_(eps)
            p.addcdiv_(st["exp_avg"], denom, value=-step_size)


class AdamW(Adam):
    """Adam with decoupled weight decay (``p *= 1 - lr·weight_decay``), torch's defaults (``weight_decay=1e-2``)."""

    def __init__(self, params: Iterable, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 amsgrad: bool = False, *, maximize: bool = False, foreach: Optional[bool] = None, capturable: bool = False,
                 differentiable: bool = False, fused: Optional[bool] = None):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, foreach=foreach, maximize=maximize, capturable=capturable,
                         differentiable=differentiable, fused=fused, decoupled_weight_decay=True)

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group["decoupled_weight_decay"] = True
