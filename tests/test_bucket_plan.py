"""Bucket planner vs torch's _compute_bucket_assignment_by_size (oracle)."""
import sys

import torch
import torch.distributed as tdist

from pytorch_distributed_train_b200 import _C, models


def _plan(params, limits, order=()):
    nbytes = [p.numel() * p.element_size() for p in params]
    keys = [hash(str(p.dtype)) & 0xFFFF for p in params]
    return _C.plan_buckets(nbytes, keys, limits, list(order))


def test_convnet_single_bucket():
    ps = list(models.ConvNet().parameters())
    b, lim = _plan(ps, [sys.maxsize])
    assert b == [list(range(10))]
    assert sum(p.numel() * 4 for p in ps) == 116136


def test_matches_torch_on_resnet18_forward_and_rebuilt_order():
    ps = list(models.resnet18().parameters())
    assert len(ps) == 62 and sum(p.numel() for p in ps) == 11689512
    limits = [1024 * 1024, 25 * 1024 * 1024]
    ours, _ = _plan(ps, limits)
    ref, _ = tdist._compute_bucket_assignment_by_size(ps, limits)
    assert ours == ref
    order = list(reversed(range(len(ps))))
    ours_r, _ = _plan(ps, limits, order)
    ref_r, _ = tdist._compute_bucket_assignment_by_size([ps[i] for i in order], limits, [False] * len(ps), order)
    assert ours_r == ref_r
    sizes = [sum(ps[i].numel() * 4 for i in b) for b in ours_r]
    assert [len(b) for b in ours_r] == [2, 12, 48]
    assert sizes == [2052000, 28852224, 15853824]  # torch DDP's plan for ResNet-18


def test_mixed_dtypes_split():
    ps = [torch.zeros(10), torch.zeros(10, dtype=torch.float64), torch.zeros(10)]
    b, _ = _plan(ps, [sys.maxsize])
    assert sorted(map(tuple, b)) == [(0, 2), (1,)]
