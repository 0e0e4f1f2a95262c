"""Cross-replica BatchNorm.

Replaces ``nn.SyncBatchNorm.convert_sync_batchnorm(model)`` (ref: ddp_example.py:53-54; module
semantics torch/nn/modules/batchnorm.py:615-905, function torch/nn/modules/_functions.py:7-209).

Same statistics, different wire protocol.  The reference stack all-gathers ``(mean, invstd,
count)`` per rank and then host-syncs on a mask; we all-*reduce* ``(Σx, Σx², n)`` — mathematically
equivalent, still count-weighted so uneven per-rank batches (and empty ranks) stay correct, but it
is one small SUM over a fixed-layout buffer: on the NVLink backend that is a single fused
peer-memory kernel with no host synchronisation, so the whole step stays CUDA-graph capturable.
Backward all-reduces ``(Σdy, Σdy·(x-μ))`` exactly like the reference; ``dγ``/``dβ`` are left to
DDP's bucket reduce.

On CUDA the per-channel reductions and the elementwise passes run as our sm_90a kernels
(``ops.bn_*``); on CPU the same math runs through torch ops so the logic is testable without a
GPU (torch's own SyncBatchNorm refuses CPU tensors).
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import distributed as dist


def _allreduce_now(group, t: torch.Tensor) -> None:
    """SUM-allreduce whose result the very next kernel consumes: on the NVLink backend this is one
    fused peer-memory kernel on the *current* stream (no stream hop, no host sync)."""
    comm = group.comm
    if hasattr(comm, "allreduce_inline"):
        comm.allreduce_inline(t, dist.ReduceOp.SUM, 1.0)
    else:
        comm.allreduce(t, dist.ReduceOp.SUM, 1.0).wait()


def _reduce_dims(x: torch.Tensor):
    return [0] + list(range(2, x.dim()))


def _bshape(x: torch.Tensor):
    return [1, -1] + [1] * (x.dim() - 2)


class _SyncBatchNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, eps, momentum, group):
        from .. import ops

        C = x.shape[1]
        count = x.numel() // C if x.numel() else 0
        native = x.is_cuda and ops.native_available() and x.dtype == torch.float32
        # debugging aid: PDT_SYNCBN_KERNELS is a bit mask of the native kernels to use
        # (1 = local stats, 2 = normalise, 4 = backward reduce, 8 = backward elementwise — default 15 = all four;
        #  16 = fused statistics finalisation, experimental)
        mask = int(os.environ.get("PDT_SYNCBN_KERNELS", "15")) if native else 0
        fused = bool(mask & 2)
        xc = x.contiguous()
        # local (Σx, Σx², n) in one *float64* vector of 2C+1: var = E[x²] − μ² magnifies the rounding of
        # the sums by μ²/σ², so they are accumulated, exchanged and combined in fp64 (torch gets the
        # same robustness from Welford + count-weighted merging, _functions.py:39-124)
        if mask & 1:
            stats = ops.bn_local_stats(xc)  # [2C+2] float64: Σx, Σx², count, one zero pad (16-byte multiple)
        else:
            xf = xc.double()
            dims = _reduce_dims(xf)
            stats = torch.cat([xf.sum(dims), (xf * xf).sum(dims), xf.new_full((1,), float(count)), xf.new_zeros(1)])
        _allreduce_now(group, stats)
        if mask & 16 and stats.is_cuda:
            # one kernel: mean, invstd, count and the running-statistics update (experimental: bit 16 is not in the default mask)
            mean, invstd, total = ops.bn_finalize(stats, C, eps, momentum, running_mean, running_var)
            total = total[0]
        else:
            total64 = stats[2 * C]
            # every rank holding zero samples is legal as long as somebody has data
            n = total64.clamp_min(1.0)
            mean64 = stats[:C] / n
            var64 = (stats[C:2 * C] / n - mean64 * mean64).clamp_min_(0.0)
            mean, invstd, total = mean64.float(), torch.rsqrt(var64 + eps).float(), total64.float()
            if running_mean is not None:
                with torch.no_grad():
                    unbiased = var64 * (n / (n - 1.0).clamp_min(1.0))
                    running_mean.mul_(1 - momentum).add_(mean.to(running_mean.dtype), alpha=momentum)
                    running_var.mul_(1 - momentum).add_(unbiased.to(running_var.dtype), alpha=momentum)
        if fused:
            out = ops.bn_apply(xc, mean, invstd, weight, bias)
        else:
            shp = _bshape(xc)
            out = (xc.float() - mean.view(shp)) * invstd.view(shp)
            if weight is not None:
                out = out * weight.float().view(shp)
            if bias is not None:
                out = out + bias.float().view(shp)
            out = out.to(x.dtype)
        ctx.save_for_backward(xc, weight, mean, invstd, total)
        ctx.group = group
        ctx.mask = mask
        ctx.has_bias = bias is not None
        return out

    @staticmethod
    def backward(ctx, dy):
        from .. import ops

        x, weight, mean, invstd, total = ctx.saved_tensors
        C = x.shape[1]
        dy = dy.contiguous()
        if ctx.mask & 4:
            red = ops.bn_backward_reduce(dy, x, mean, invstd)  # [4C]: Σdy, Σdy·(x-μ), dγ, dβ
        else:
            dims = _reduce_dims(x)
            shp = _bshape(x)
            dyf, xmu = dy.float(), x.float() - mean.view(shp)
            sum_dy = dyf.sum(dims)
            sum_dy_xmu = (dyf * xmu).sum(dims)
            red = torch.cat([sum_dy, sum_dy_xmu, sum_dy_xmu * invstd, sum_dy])
        grad_weight = red[2 * C:3 * C].clone() if weight is not None and ctx.needs_input_grad[1] else None
        grad_bias = red[3 * C:4 * C].clone() if ctx.has_bias and ctx.needs_input_grad[2] else None
        dx = None
        if ctx.needs_input_grad[0]:
            sums = red[:2 * C].contiguous()
            _allreduce_now(ctx.group, sums)
            n = total.clamp_min(1.0)
            mean_dy = sums[:C] / n
            mean_dy_xmu = sums[C:] / n
            if ctx.mask & 8:
                dx = ops.bn_backward_apply(dy, x, mean, invstd, weight, mean_dy, mean_dy_xmu)
            else:
                shp = _bshape(x)
                w = weight.float().view(shp) if weight is not None else 1.0
                xmu = x.float() - mean.view(shp)
                dx = (dy.float() - mean_dy.view(shp) - xmu * (invstd * invstd * mean_dy_xmu).view(shp)) * invstd.view(shp) * w
                dx = dx.to(x.dtype)
        return dx, grad_weight, grad_bias, None, None, None, None, None


class SyncBatchNorm(nn.modules.batchnorm._BatchNorm):
    """BatchNorm whose batch statistics are computed over the whole process group."""

    def __init__(self, num_features: int, eps: float = 1e-5, momentum: Optional[float] = 0.1, affine: bool = True,
                 track_running_stats: bool = True, process_group=None, device=None, dtype=None):
        super().__init__(num_features, eps, momentum, affine, track_running_stats, device=device, dtype=dtype)
        self.process_group = process_group

    def _check_input_dim(self, input):
        if input.dim() < 2:
            raise ValueError(f"expected at least 2D input (got {input.dim()}D input)")

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        self._check_input_dim(input)
        if self.momentum is None:
            eaf = 0.0
        else:
            eaf = self.momentum
        if self.training and self.track_running_stats and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
            if self.momentum is None:
                eaf = 1.0 / float(self.num_batches_tracked)
        bn_training = self.training or (self.running_mean is None and self.running_var is None)
        need_sync = bn_training and self.training and dist.is_initialized()
        group = None
        if need_sync:
            group = self.process_group or dist.get_default_group()
            need_sync = group.size() > 1
        if not need_sync:
            # world of one, or eval: plain batch norm (batchnorm.py:818-828)
            return F.batch_norm(input, self.running_mean if not self.training or self.track_running_stats else None,
                                self.running_var if not self.training or self.track_running_stats else None,
                                self.weight, self.bias, bn_training, eaf, self.eps)
        if group.is_cuda != input.is_cuda:
            raise ValueError("SyncBatchNorm: input device does not match the process group's backend")
        return _SyncBatchNormFn.apply(input, self.weight, self.bias,
                                      self.running_mean if self.track_running_stats else None,
                                      self.running_var if self.track_running_stats else None,
                                      self.eps, eaf, group)

    @classmethod
    def convert_sync_batchnorm(cls, module: nn.Module, process_group=None) -> nn.Module:
        """Recursively swap every ``_BatchNorm`` for ``SyncBatchNorm``, *sharing* the affine
        parameters and running statistics (batchnorm.py:844-905)."""
        out = module
        if isinstance(module, nn.modules.batchnorm._BatchNorm) and not isinstance(module, cls):
            out = cls(module.num_features, module.eps, module.momentum, module.affine, module.track_running_stats,
                      process_group)
            if module.affine:
                with torch.no_grad():
                    out.weight = module.weight
                    out.bias = module.bias
            out.running_mean = module.running_mean
            out.running_var = module.running_var
            out.num_batches_tracked = module.num_batches_tracked
            out.training = module.training
            if hasattr(module, "qconfig"):
                out.qconfig = module.qconfig
        for name, child in module.named_children():
            out.add_module(name, cls.convert_sync_batchnorm(child, process_group))
        del module
        return out
