"""Test-set evaluation: the loss and top-1 accuracy of a model over a whole split, exact across ranks.

The model's forward runs as it runs in eval mode (for the ConvNet, the per-op kernels); the metrics are counted on the device by
the cross-entropy kernel (``ops.cross_entropy_accumulate``), which adds each batch's loss terms, the mean's divisor, top-1 hits
and counted rows to one float64 ``[4]`` accumulator.  Nothing is read back per batch: the host sees the four totals once, after
one all-reduce across the ranks.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn

from .. import distributed as dist
from .. import ops
from ..data.sampler import DistributedSampler
from ..nn.loss import CrossEntropyLoss
from ..parallel.ddp import DistributedDataParallel


def _criterion_spec(criterion) -> tuple:
    """(weight, ignore_index, reduction, label_smoothing) of a cross-entropy criterion with a reduction the totals can express."""
    if not isinstance(criterion, (CrossEntropyLoss, nn.CrossEntropyLoss)):
        raise ValueError(f"evaluate: criterion must be a pdt.nn.CrossEntropyLoss or torch.nn.CrossEntropyLoss, got {type(criterion).__name__}")
    if criterion.reduction not in ("mean", "sum"):
        raise ValueError(f"evaluate: the criterion's reduction must be 'mean' or 'sum', got {criterion.reduction!r}")
    return (criterion.weight, criterion.ignore_index, criterion.reduction, criterion.label_smoothing)


def _rank_samples(sampler) -> Optional[int]:
    """How many of this rank's samples are real images when ``sampler`` pads the split, else None.  Sample i of rank r sits at
    position r + i·W of the padded global order, and the padding is whatever lies at positions ≥ len(dataset)."""
    if not isinstance(sampler, DistributedSampler) or sampler.drop_last:
        return None
    return max(0, math.ceil((len(sampler.dataset) - sampler.rank) / sampler.num_replicas))


def evaluate(model: nn.Module, loader, criterion=None) -> dict:
    """The ``criterion``'s loss on the whole split ``loader`` yields, and the model's top-1 accuracy on it.

    Returns ``{"loss", "accuracy", "correct", "count"}``: ``loss`` is what ``criterion`` (default ``pdt.nn.CrossEntropyLoss()``;
    a pdt or torch ``CrossEntropyLoss`` with reduction 'mean' or 'sum') returns on the split's concatenated logits, ``count`` the
    rows it counts (targets in [0, C) other than ``ignore_index``) and ``correct`` those whose argmax is the target.

    The model runs in eval mode under ``torch.no_grad()`` and its previous mode is restored; a ``DistributedDataParallel`` is
    evaluated through its ``.module``, so the forward starts no collective.  With a process group of two or more ranks, each
    rank evaluates its own shard and the totals are summed by one all-reduce; a ``DistributedSampler`` without ``drop_last``
    pads the shards with repeated images, and those are left out, so every image counts exactly once."""
    spec = _criterion_spec(CrossEntropyLoss() if criterion is None else criterion)
    net = model.module if isinstance(model, DistributedDataParallel) else model
    first = next(iter(net.parameters()), None)
    device = first.device if first is not None else torch.device("cpu")
    real = _rank_samples(getattr(loader, "sampler", None))
    acc = torch.zeros(4, dtype=torch.float64, device=device)
    was_training = net.training
    net.eval()
    try:
        with torch.no_grad():
            seen = 0
            for images, labels in loader:
                images = images.to(device, non_blocking=True)
                labels = labels.to(device, non_blocking=True)
                n = labels.shape[0]
                rows = n if real is None else min(n, max(0, real - seen))
                seen += n
                ops.cross_entropy_accumulate(net(images), labels, acc, rows, spec)
    finally:
        net.train(was_training)
    if dist.is_initialized() and dist.get_world_size() >= 2:
        dist.all_reduce(acc)
    total, divisor, correct, count = acc.tolist()
    loss = total if spec[2] == "sum" else (total / divisor if divisor != 0 else math.nan)
    return {"loss": loss, "accuracy": correct / count if count else math.nan, "correct": int(correct), "count": int(count)}
