"""MixUp (Zhang et al., 2018) on one batch, with torchvision's ``transforms.v2.MixUp`` definition."""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F


def mixup(images: torch.Tensor, labels: torch.Tensor, num_classes: int, alpha: float,
          generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """Mix every image of the batch with the one before it (the first with the last) and return the matching class-probability
    targets.  λ ~ Beta(α, α) is drawn once for the batch, on the host from ``generator`` (a CPU generator; torch's default one when
    None), and then

        images ← λ·images + (1 − λ)·images.roll(1, 0)             in place
        targets = λ·onehot(labels) + (1 − λ)·onehot(labels).roll(1, 0)    fp32 [B, num_classes]

    rounded as torchvision computes them.  ``labels`` are int64 class indices in [0, num_classes).  The arithmetic runs on the
    tensors' own device and nothing waits for it: in place, pinned host images stay pinned."""
    if not alpha > 0:
        raise ValueError(f"mixup: alpha must be positive (got {alpha})")
    lam = draw_lambda(alpha, generator)
    mix_rows_(images, lam)
    return mix_rows_(F.one_hot(labels, num_classes).to(torch.float32), lam)


def draw_lambda(alpha: float, generator: Optional[torch.Generator] = None) -> float:
    """λ ~ Beta(α, α) on the host: what torch.distributions.Beta(α, α).sample() draws (torchvision's λ), here from the caller's
    generator.  torch.distributions takes no generator, so the private sampler Beta.sample calls is called directly
    (test_mixup_cli.py pins the equivalence)."""
    return float(torch._sample_dirichlet(torch.tensor([alpha, alpha]), generator=generator)[0])


def mix_rows_(t: torch.Tensor, lam: float) -> torch.Tensor:
    """t ← λ·t + (1 − λ)·t.roll(1, 0) in place, rounded as torchvision's MixUp: fl(fl(t·fp32(λ)) + fl(t.roll(1, 0)·fp32(1 − λ))), with
    1 − λ formed in double.  Returns t."""
    rolled = t.roll(1, 0)
    return t.mul_(lam).add_(rolled.mul_(1.0 - lam))
