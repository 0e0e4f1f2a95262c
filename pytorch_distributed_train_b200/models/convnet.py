"""The reference's model: 2×[Conv5×5(pad 2) → BatchNorm → ReLU → MaxPool2×2] → Linear(1568→10)
(ref: ddp_example.py:22-41).  Module tree and ``state_dict`` keys are identical
(``layer1.0.weight`` … ``fc.bias``) so checkpoints interchange and
``SyncBatchNorm.convert_sync_batchnorm`` finds the BatchNorm layers where it expects them.

On an H100 the forward does not walk the ``nn.Sequential``s.  In training the whole forward is TWO cooperative
sm_90a kernels with one CTA per image (``csrc/cuda/fused_convnet.cu``): conv1+BN1+ReLU+pool1, and
conv2 (wgmma, register accumulators, haloed image in shared memory) +BN2+ReLU+pool2+classifier — the BatchNorm batch
statistics cross a device-side grid barrier inside the kernel instead of a kernel boundary; backward is one such
kernel per layer plus the tensor-core weight gradient.  Shapes the fused kernels do not cover (eval mode,
SyncBatchNorm, batch > #SMs) run each ``layerN`` as two per-op kernels (implicit-GEMM conv with the BN statistics in
its epilogue, then BN-apply+ReLU+MaxPool) and the classifier as one linear kernel.  The same modules fall back to
the stock layers on CPU (plumbing tests) or when ``fused=False``.
"""
from __future__ import annotations

import torch
import torch.nn as nn


class ConvNet(nn.Module):
    def __init__(self, num_classes: int = 10, fused=None):
        super().__init__()
        self.layer1 = nn.Sequential(
            nn.Conv2d(1, 16, kernel_size=5, stride=1, padding=2),
            nn.BatchNorm2d(16),
            nn.ReLU(),
            nn.MaxPool2d(kernel_size=2, stride=2))
        self.layer2 = nn.Sequential(
            nn.Conv2d(16, 32, kernel_size=5, stride=1, padding=2),
            nn.BatchNorm2d(32),
            nn.ReLU(),
            nn.MaxPool2d(kernel_size=2, stride=2))
        self.fc = nn.Linear(7 * 7 * 32, num_classes)
        self.fused = fused  # None = auto (CUDA + native runtime present)

    def _use_fused(self, x: torch.Tensor) -> bool:
        if self.fused is False:
            return False
        from .. import ops

        ok = x.is_cuda and x.dtype == torch.float32 and ops.native_available()
        if self.fused is True and not ok:
            raise RuntimeError("ConvNet(fused=True) needs float32 CUDA input and the native sm_90a runtime")
        return ok

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self._use_fused(x):
            from .. import ops
            from ..ops import functional as OF

            if torch.is_grad_enabled() and OF.fused_convnet_ok(x, self):
                # one cooperative kernel per layer (conv + BN statistics barrier + BN/ReLU/pool [+ classifier])
                return OF.fused_convnet_forward(x, self)
            out = ops.conv_bn_relu_pool(x, self.layer1[0], self.layer1[1])
            out = ops.conv_bn_relu_pool(out, self.layer2[0], self.layer2[1])
            out = out.reshape(out.size(0), -1)
            return ops.linear(out, self.fc.weight, self.fc.bias)
        out = self.layer1(x)
        out = self.layer2(out)
        out = out.reshape(out.size(0), -1)
        return self.fc(out)
