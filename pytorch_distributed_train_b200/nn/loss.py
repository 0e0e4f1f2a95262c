"""Cross-entropy loss (ref: ddp_example.py:61,87 ``nn.CrossEntropyLoss().cuda(gpu)``).

On CUDA, float32 ``[B, C]`` logits with class-index targets and ``reduction='mean'`` run as one
fused sm_90a kernel (log-softmax + NLL + mean, saving the softmax so backward is a single
``(softmax − onehot)/B`` pass) instead of the reference stack's ``_log_softmax`` +
``nll_loss_forward`` pair and their two backward kernels.  Everything else defers to the
standard functional."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F


class CrossEntropyLoss(nn.Module):
    def __init__(self, weight=None, ignore_index: int = -100, reduction: str = "mean", label_smoothing: float = 0.0):
        super().__init__()
        self.register_buffer("weight", weight)
        self.ignore_index, self.reduction, self.label_smoothing = ignore_index, reduction, label_smoothing

    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        from .. import ops

        if (input.is_cuda and ops.native_available() and input.dim() == 2 and input.dtype == torch.float32
                and target.dtype == torch.int64 and self.weight is None and self.reduction == "mean"
                and self.label_smoothing == 0.0 and self.ignore_index == -100 and input.shape[1] <= 1024):
            return ops.cross_entropy(input, target)
        return F.cross_entropy(input, target, self.weight, ignore_index=self.ignore_index,
                               reduction=self.reduction, label_smoothing=self.label_smoothing)
