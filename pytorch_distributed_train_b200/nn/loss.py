"""Cross-entropy loss (ref: ddp_example.py:61,87 ``nn.CrossEntropyLoss().cuda(gpu)``).

On CUDA, float32 ``[B, C]`` logits (C ≤ 1024) with class-index targets run as one fused sm_90a kernel (log-softmax + NLL +
reduction, saving the softmax so backward is a single pass) instead of the reference stack's ``_log_softmax`` +
``nll_loss_forward`` pair and their two backward kernels.  torch's options are native too: class ``weight`` (fp32, contiguous,
``[C]``, on the logits' device), any ``ignore_index``, ``reduction`` 'mean' or 'sum', and ``label_smoothing`` in [0, 1].  As in
torch, rows whose target is ``ignore_index`` add nothing and get a zero gradient, and a mean over no counted rows is NaN; a target
outside [0, C) counts as ignored too.

Class-probability targets (MixUp, distillation, averaged labels) run on a kernel of their own when they are fp32, contiguous,
shaped like the logits and on their device, with ``ignore_index`` left at -100: as in torch, a row adds Σ_c w_c·q'_c·(lse − x_c)
with q' = q·(1 − ε) + ε/C, the mean divides by the batch size whatever the weights, and the entries are not validated.
``reduction='none'`` and everything else (fp64 or fp16 probabilities, a non-contiguous or misshapen target, another
``ignore_index``) defer to the standard functional, which keeps torch's results and errors."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F


def native_ok(input: torch.Tensor, target: torch.Tensor, weight, reduction: str, label_smoothing: float,
              ignore_index: int = -100) -> bool:
    """Whether a cross-entropy of ``input`` and ``target`` (class indices, or class probabilities) with these options runs on the
    native kernels."""
    from .. import ops

    if not (input.is_cuda and ops.native_available() and input.dim() == 2 and input.dtype == torch.float32):
        return False   # unbatched [C] input among others: torch's functional
    soft = (target.dtype == torch.float32 and target.shape == input.shape and target.is_contiguous() and target.device == input.device
            and ignore_index == -100 and input.shape[1] >= 1)
    return ((target.dtype == torch.int64 or soft) and reduction in ("mean", "sum") and 0.0 <= label_smoothing <= 1.0
            and input.shape[1] <= 1024
            and (weight is None or (weight.dtype == torch.float32 and weight.is_contiguous() and weight.shape == (input.shape[1],)
                                    and weight.device == input.device)))


class CrossEntropyLoss(nn.Module):
    def __init__(self, weight=None, ignore_index: int = -100, reduction: str = "mean", label_smoothing: float = 0.0):
        super().__init__()
        self.register_buffer("weight", weight)
        self.ignore_index, self.reduction, self.label_smoothing = ignore_index, reduction, label_smoothing

    def native_ok(self, input: torch.Tensor, target: torch.Tensor) -> bool:
        """Whether ``forward(input, target)`` runs on the native kernels."""
        return native_ok(input, target, self.weight, self.reduction, self.label_smoothing, self.ignore_index)

    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        from .. import ops

        if self.native_ok(input, target):
            return ops.cross_entropy(input, target, self.weight, self.ignore_index, self.reduction, self.label_smoothing)
        return F.cross_entropy(input, target, self.weight, ignore_index=self.ignore_index,
                               reduction=self.reduction, label_smoothing=self.label_smoothing)
