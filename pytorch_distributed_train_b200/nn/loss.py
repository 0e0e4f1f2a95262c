"""Cross-entropy loss (ref: ddp_example.py:61,87 ``nn.CrossEntropyLoss().cuda(gpu)``).

On CUDA, float32 ``[B, C]`` logits (C ≤ 1024) with class-index targets run as one fused sm_90a kernel (log-softmax + NLL +
reduction, saving the softmax so backward is a single pass) instead of the reference stack's ``_log_softmax`` +
``nll_loss_forward`` pair and their two backward kernels.  torch's options are native too: class ``weight`` (fp32, contiguous,
``[C]``, on the logits' device), any ``ignore_index``, ``reduction`` 'mean' or 'sum', and ``label_smoothing`` in [0, 1].  As in
torch, rows whose target is ``ignore_index`` add nothing and get a zero gradient, and a mean over no counted rows is NaN; a target
outside [0, C) counts as ignored too.  ``reduction='none'``, probability targets and everything else defer to the standard
functional."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F


class CrossEntropyLoss(nn.Module):
    def __init__(self, weight=None, ignore_index: int = -100, reduction: str = "mean", label_smoothing: float = 0.0):
        super().__init__()
        self.register_buffer("weight", weight)
        self.ignore_index, self.reduction, self.label_smoothing = ignore_index, reduction, label_smoothing

    def native_ok(self, input: torch.Tensor, target: torch.Tensor) -> bool:
        """Whether ``forward(input, target)`` runs on the native kernels."""
        from .. import ops

        w = self.weight
        return (input.is_cuda and ops.native_available() and input.dim() == 2 and input.dtype == torch.float32
                and target.dtype == torch.int64 and self.reduction in ("mean", "sum") and 0.0 <= self.label_smoothing <= 1.0
                and input.shape[1] <= 1024
                and (w is None or (w.dtype == torch.float32 and w.is_contiguous() and w.shape == (input.shape[1],)
                                   and w.device == input.device)))

    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        from .. import ops

        if self.native_ok(input, target):
            return ops.cross_entropy(input, target, self.weight, self.ignore_index, self.reduction, self.label_smoothing)
        return F.cross_entropy(input, target, self.weight, ignore_index=self.ignore_index,
                               reduction=self.reduction, label_smoothing=self.label_smoothing)
