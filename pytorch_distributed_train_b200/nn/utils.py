"""``clip_grad_norm_`` with torch's signature and behaviour, on native kernels where it can.

fp32 contiguous CUDA gradients that are all on one device, with ``norm_type`` 2 or inf, take two sm_90a launches per 48 tensors
(``ops.grad_norm_clip``: the norm, then the scale), graph-capturable and bit-reproducible from run to run.  Everything else —
CPU tensors, other dtypes, other norm types, several devices — goes to ``torch.nn.utils.clip_grad_norm_`` unchanged.
"""
from __future__ import annotations

import math
from typing import Iterable, Optional, Union

import torch

__all__ = ["clip_grad_norm_"]


def _native(grads, norm_type: float) -> bool:
    from .. import ops

    if not grads or (norm_type != 2.0 and norm_type != math.inf) or not ops.native_available():
        return False
    if norm_type == math.inf and any(g.numel() == 0 for g in grads):
        return False   # torch refuses the inf-norm of an empty tensor: its path raises that error
    dev = grads[0].device
    return all(g.is_cuda and g.device == dev and g.dtype == torch.float32 and not g.is_sparse and g.is_contiguous()
               and g.numel() < 2 ** 31 for g in grads)


@torch.no_grad()
def clip_grad_norm_(parameters: Union[torch.Tensor, Iterable[torch.Tensor]], max_norm: float, norm_type: float = 2.0,
                    error_if_nonfinite: bool = False, foreach: Optional[bool] = None) -> torch.Tensor:
    """Clip the gradient norm of ``parameters`` in place and return the total norm, as ``torch.nn.utils.clip_grad_norm_`` does:
    the norm over all gradients viewed as one vector, every gradient multiplied by ``min(max_norm / (norm + 1e-6), 1)``.
    Parameters without a gradient are skipped; ``foreach`` only matters on the torch path."""
    if isinstance(parameters, torch.Tensor):
        parameters = [parameters]
    else:
        parameters = list(parameters)
    grads = [p.grad for p in parameters if p.grad is not None]
    norm_type = float(norm_type)
    if not _native(grads, norm_type):
        return torch.nn.utils.clip_grad_norm_(parameters, max_norm, norm_type, error_if_nonfinite, foreach)
    from .. import ops

    if not error_if_nonfinite:
        return ops.grad_norm_clip(grads, max_norm, norm_type, scale=True)
    # torch checks the norm on the host before anything is scaled
    norm = ops.grad_norm_clip(grads, max_norm, norm_type, scale=False)
    if torch.logical_or(norm.isnan(), norm.isinf()):
        raise RuntimeError(
            f"The total norm of order {norm_type} for gradients from "
            "`parameters` is non-finite, so it cannot be clipped. To disable "
            "this error and scale the gradients by the non-finite norm anyway, "
            "set `error_if_nonfinite=False`"
        )
    ops.grad_scale(grads, norm)
    return norm
