"""The reference's model: 2×[Conv5×5(pad 2) → BatchNorm → ReLU → MaxPool2×2] → Linear(1568→10)
(ref: ddp_example.py:22-41).  Module tree and ``state_dict`` keys are identical
(``layer1.0.weight`` … ``fc.bias``) so checkpoints interchange and
``SyncBatchNorm.convert_sync_batchnorm`` finds the BatchNorm layers where it expects them.

On an H100 the forward does not walk the ``nn.Sequential``s.  In training the whole forward is ONE cooperative
sm_90a kernel with one CTA per image (``csrc/cuda/fused_convnet.cu``): conv1+BN1+ReLU+pool1 → conv2 (wgmma, register
accumulators, haloed image in shared memory) +BN2+ReLU+pool2+classifier — the BatchNorm batch statistics cross a
device-side grid barrier inside the kernel instead of a kernel boundary; backward is one such kernel per layer, with the
classifier's backward and conv2's weight gradient riding along.  What the fused kernels do not cover (eval mode,
SyncBatchNorm, batch > #SMs, a partially frozen model, an input that requires grad) runs each ``layerN`` as two per-op kernels (implicit-GEMM conv with the
BN statistics in its epilogue, then BN-apply+ReLU+MaxPool) and the classifier as one linear kernel.  The same modules fall back
to the stock layers on CPU (plumbing tests) or when ``fused=False``.  Other layer configurations (another padding mode,
dilation or stride, a swapped activation, pool or norm layer, an extra module in a ``Sequential``, module hooks, weight norm)
run torch's layers, since neither kernel route computes them.
"""
from __future__ import annotations

import torch
import torch.nn as nn
from torch.nn.modules import module as _torch_module

from ..parallel.sync_batchnorm import SyncBatchNorm


def _unhooked(m) -> bool:
    return not (m._forward_hooks or m._forward_pre_hooks or m._backward_hooks or m._backward_pre_hooks)


def _native_layer(layer) -> bool:
    """Exactly Conv2d(5×5, stride 1, pad 2) → BatchNorm2d / pdt.SyncBatchNorm → ReLU → MaxPool2d(2, 2), none of them hooked."""
    if type(layer) is not nn.Sequential or len(layer._modules) != 4 or not _unhooked(layer):
        return False
    conv, bn, act, pool = layer._modules.values()
    return (type(conv) is nn.Conv2d and conv.kernel_size == (5, 5) and conv.stride == (1, 1) and conv.padding in ((2, 2), "same")
            and conv.dilation == (1, 1) and conv.groups == 1 and conv.padding_mode == "zeros"
            and type(bn) in (nn.BatchNorm2d, SyncBatchNorm) and type(act) is nn.ReLU
            and type(pool) is nn.MaxPool2d and pool.kernel_size in (2, (2, 2)) and pool.stride in (2, (2, 2))
            and pool.padding in (0, (0, 0)) and pool.dilation in (1, (1, 1)) and not pool.ceil_mode
            and _unhooked(conv) and _unhooked(bn) and _unhooked(act) and _unhooked(pool))


def _native_layers(model) -> bool:
    """Whether ``model``'s layers are the ones the native kernels compute: the stock layer stack, with no hooks on the modules
    ``forward`` uses and no global module hooks (the native routes never call the submodules, so their hooks would not run).  The
    model's own hooks do not matter: ``__call__`` runs them.  Pure host logic on module attributes: it reads no device tensor and
    never synchronises."""
    mods = model._modules
    fc = mods.get("fc")
    return (type(fc) is nn.Linear and _unhooked(fc) and _native_layer(mods.get("layer1")) and _native_layer(mods.get("layer2"))
            and not (_torch_module._global_forward_hooks or _torch_module._global_forward_pre_hooks
                     or _torch_module._global_backward_hooks or _torch_module._global_backward_pre_hooks))


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
        if _native_layers(self) and self._use_fused(x):
            from .. import ops
            from ..ops import functional as OF

            if torch.is_grad_enabled() and OF.fused_convnet_ok(x, self):
                # one cooperative kernel for the forward (conv + BN statistics barrier + BN/ReLU/pool, per layer, + classifier)
                return OF.fused_convnet_forward(x, self)
            out = ops.conv_bn_relu_pool(x, self.layer1[0], self.layer1[1])
            out = ops.conv_bn_relu_pool(out, self.layer2[0], self.layer2[1])
            out = out.reshape(out.size(0), -1)
            return ops.linear(out, self.fc.weight, self.fc.bias)
        out = self.layer1(x)
        out = self.layer2(out)
        out = out.reshape(out.size(0), -1)
        return self.fc(out)
