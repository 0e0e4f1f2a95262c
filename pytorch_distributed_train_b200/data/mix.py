"""Batch-level MixUp (Zhang et al., 2018) and CutMix (Yun et al., 2019) with torchvision's ``transforms.v2.MixUp`` / ``CutMix``
definitions.  On a CUDA batch λ and the box are drawn on the device and the batch is mixed in one launch (``ops.mix_batch``), so the
transform can run inside a captured training step (``engine.GraphedTrainStep(mix=...)``); a CPU batch makes torchvision's own draws
with torch ops."""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F

from .mixup import draw_lambda, mix_rows_


class _MixBase:
    _cutmix = False

    def __init__(self, *, alpha: float = 1.0, num_classes: Optional[int] = None, generator: Optional[torch.Generator] = None,
                 record_params: bool = False):
        if not float(alpha) > 0:
            raise ValueError(f"{type(self).__name__}: alpha must be positive (got {alpha})")
        self.alpha = float(alpha)
        self.num_classes = num_classes
        self.generator = generator
        self.record_params = bool(record_params)
        self.last_params: Optional[torch.Tensor] = None

    def __repr__(self) -> str:
        return f"{type(self).__name__}(alpha={self.alpha}, num_classes={self.num_classes})"

    def _check(self, images, labels):
        # torchvision's checks and messages (_BaseMixUpCutMix.forward, _check_image_or_video), then the dtypes this implementation takes
        if not isinstance(labels, torch.Tensor):
            raise ValueError(f"The labels must be a tensor, but got {type(labels)} instead.")
        if labels.ndim not in (1, 2):
            raise ValueError(f"labels should be index based with shape (batch_size,) or probability based with shape (batch_size, "
                             f"num_classes), but got a tensor of shape {labels.shape} instead.")
        if labels.ndim == 2 and self.num_classes is not None and labels.shape[-1] != self.num_classes:
            raise ValueError(f"When passing 2D labels, the number of elements in last dimension must match num_classes: "
                             f"{labels.shape[-1]} != {self.num_classes}. You can Leave num_classes to None.")
        if labels.ndim == 1 and self.num_classes is None:
            raise ValueError("num_classes must be passed if the labels are index-based (1D)")
        if images.ndim != 4:
            raise ValueError(f"Expected a batched input with 4 dims, but got {images.ndim} dimensions instead.")
        if images.shape[0] != labels.shape[0]:
            raise ValueError(f"The batch size of the image or video does not match the batch size of the labels: "
                             f"{images.shape[0]} != {labels.shape[0]}.")
        name = type(self).__name__
        if images.dtype != torch.float32:
            raise TypeError(f"{name}: images must be float32 (got {images.dtype})")
        want = torch.int64 if labels.ndim == 1 else torch.float32
        if labels.dtype != want:
            raise TypeError(f"{name}: {'index' if labels.ndim == 1 else 'probability'} labels must be {want} (got {labels.dtype})")
        if labels.device != images.device:
            raise ValueError(f"{name}: the labels are on {labels.device}, the images on {images.device}")

    def __call__(self, images: torch.Tensor, labels: torch.Tensor):
        """(images [B, C, H, W], labels) → (mixed images, fp32 targets [B, num_classes])."""
        self._check(images, labels)
        if images.is_cuda:
            from .. import ops

            out, targets, params = ops.mix_batch(images.contiguous(), labels.contiguous(), self.num_classes, self.alpha, self._cutmix,
                                                 generator=self.generator, record_params=self.record_params)
        else:
            out, targets, params = self._cpu(images, labels)
        if self.record_params:
            self.last_params = params
        return out, targets

    def _targets(self, labels, lam):
        t = F.one_hot(labels, self.num_classes).to(torch.float32) if labels.ndim == 1 else labels.clone()
        return mix_rows_(t, lam)


class MixUp(_MixBase):
    """torchvision's ``transforms.v2.MixUp`` on a batch: every image mixed with the one before it (the first with the last),

        images ← λ·images + (1 − λ)·images.roll(1, 0),   targets = λ·onehot(labels) + (1 − λ)·onehot(labels).roll(1, 0)

    with one λ ~ Beta(α, α) for the batch, rounded as torchvision's tensor ops round.  Called as ``t(images, labels)`` on fp32
    ``[B, C, H, W]`` images and int64 class indices ``[B]`` (``num_classes`` required) or fp32 probabilities ``[B, K]``; returns a
    new image tensor and fp32 targets ``[B, K]``.  Arguments, checks and messages are torchvision's (``labels_getter`` is not
    supported); other dtypes raise ``TypeError``.

    * A CUDA batch takes the native kernel: one launch, λ drawn on the device from ``generator`` (a CUDA generator on the batch's
      device; the default one when None), nothing on the host, capturable in a CUDA graph where every replay draws anew.  An index
      label outside [0, num_classes) adds no mass to its row (torch's ``one_hot`` would raise; the kernel cannot, inside a graph).
    * A CPU batch draws λ as torchvision does, from ``generator`` (a CPU generator; torch's default one when None), so under the
      same seed it equals torchvision's output bit for bit; an index label outside [0, num_classes) raises there, as it does in
      torchvision.

    ``record_params=True`` keeps the last call's λ in ``last_params``: fp64 ``[1]`` on the batch's device (inside a CUDA graph the
    graph's static tensor, holding the last replay's draw)."""

    def _cpu(self, images, labels):
        lam = draw_lambda(self.alpha, self.generator)
        return mix_rows_(images.clone(), lam), self._targets(labels, lam), torch.tensor([lam], dtype=torch.float64)


class CutMix(_MixBase):
    """torchvision's ``transforms.v2.CutMix`` on a batch: with λ ~ Beta(α, α), r_x uniform in {0..W−1} and r_y in {0..H−1}, torchvision's
    box r = ½·√(1 − λ), (x1, y1, x2, y2) = (max(r_x − ⌊r·W⌋, 0), max(r_y − ⌊r·H⌋, 0), min(r_x + ⌊r·W⌋, W), min(r_y + ⌊r·H⌋, H)) is
    pasted into every image from the one before it (the first from the last), on every channel, and the targets are mixed with
    λ_adj = 1 − (x2 − x1)(y2 − y1)/(W·H) as ``MixUp`` mixes them with λ.  Calling convention, checks, the CUDA and CPU paths and the
    out-of-range labels are ``MixUp``'s.

    ``record_params=True`` keeps the last call's parameters in ``last_params``: fp64 ``[8]`` (λ, r_x, r_y, x1, y1, x2, y2, λ_adj) on
    the batch's device."""

    _cutmix = True

    def _cpu(self, images, labels):
        """torchvision's CutMix.make_params and transform, drawing from the transform's generator."""
        lam = draw_lambda(self.alpha, self.generator)
        H, W = images.shape[-2:]
        r_x = int(torch.randint(W, size=(1,), generator=self.generator))
        r_y = int(torch.randint(H, size=(1,), generator=self.generator))
        r = 0.5 * math.sqrt(1.0 - lam)
        r_w_half, r_h_half = int(r * W), int(r * H)
        x1, y1 = max(r_x - r_w_half, 0), max(r_y - r_h_half, 0)
        x2, y2 = min(r_x + r_w_half, W), min(r_y + r_h_half, H)
        lam_adj = float(1.0 - (x2 - x1) * (y2 - y1) / (W * H))
        out = images.clone()
        out[..., y1:y2, x1:x2] = images.roll(1, 0)[..., y1:y2, x1:x2]
        record = torch.tensor([lam, r_x, r_y, x1, y1, x2, y2, lam_adj], dtype=torch.float64)
        return out, self._targets(labels, lam_adj), record
