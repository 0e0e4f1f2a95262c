"""Autograd bindings for the sm_90a kernels in ``_C`` (csrc/cuda/ops_simt.cu, conv_wgmma.cu).

Layout convention: activations between fused layers are NHWC in memory and are handed to PyTorch
as ``channels_last`` tensors (logical NCHW shape), so module hooks / user code see ordinary tensors.

Gradient placement: when a parameter's ``.grad`` is ``None`` at backward time (the reference's
``optimizer.zero_grad()`` default, ref: ddp_example.py:90) and DDP has published a bucket view for it
(``param._pdt_grad_view``), the weight-gradient kernels write **directly into the DDP bucket** and
return an alias of that view; autograd adopts it as ``.grad`` and the reducer finds the gradient
already in place — no per-parameter copy or scale kernels (the reference path spends ~20 tiny kernels
per step there).
"""
from __future__ import annotations

import os
from typing import Optional

import torch

from .. import _C
from .. import distributed as dist


_claim_epoch = 0   # bumped by DistributedDataParallel.forward: one direct write per parameter per iteration


def begin_iteration() -> None:
    """Called by DDP at every training forward: bucket slots may be claimed (once each) by the coming backward."""
    global _claim_epoch
    _claim_epoch += 1


def _grad_dst(param: Optional[torch.Tensor], like: torch.Tensor) -> torch.Tensor:
    """Where a parameter gradient should be written: the DDP bucket slot when that is safe.

    Safe = ``.grad`` is None, DDP has published a view for this parameter, and the slot has not been handed out
    yet in this iteration.  A parameter used twice in one forward (tied weights, siamese towers, recurrent use) gets
    the slot for its first backward call only; later calls write a temporary that autograd *adds* into the slot,
    so the result is dW1 + dW2 rather than two aliases of one buffer.  The same guard makes ``torch.autograd.grad``
    / a backward outside ``DDP.forward`` fall back to temporaries instead of clobbering live bucket memory."""
    view = getattr(param, "_pdt_grad_view", None) if param is not None else None
    if (view is not None and param.grad is None and view.shape == like.shape and view.is_contiguous()
            and getattr(param, "_pdt_grad_claim", -1) != _claim_epoch):
        param._pdt_grad_claim = _claim_epoch
        return view.detach().view(like.shape)  # fresh alias: autograd may adopt it without copying
    return torch.empty_like(like, memory_format=torch.contiguous_format)


def _inline_allreduce(group, t: torch.Tensor) -> None:
    comm = group.comm
    if hasattr(comm, "allreduce_inline"):
        comm.allreduce_inline(t, dist.ReduceOp.SUM, 1.0)   # our kernel, on the current stream
    else:
        comm.allreduce(t, dist.ReduceOp.SUM, 1.0).wait()   # NCCL baseline: stream hop + wait


def _padded_stats(stats: torch.Tensor) -> torch.Tensor:
    """conv5x5_fwd hands back the first 2C+1 entries of a zeroed [2C+4] vector; all-reduce the whole padded
    vector (a 16-byte multiple takes the vectorised kernel, an odd length would bounce through a temporary)."""
    n = (stats.numel() + 3) // 4 * 4
    if stats.dim() == 1 and stats.is_contiguous() and stats.untyped_storage().nbytes() >= (stats.storage_offset() + n) * stats.element_size():
        return stats.as_strided((n,), (1,), stats.storage_offset())
    return stats


def _to_nhwc(x: torch.Tensor) -> torch.Tensor:
    """[B,C,H,W] (any strides) → contiguous [B,H,W,C] without a copy when already channels_last."""
    if x.shape[1] == 1:
        return x.contiguous().view(x.shape[0], x.shape[2], x.shape[3], 1)
    return x.permute(0, 2, 3, 1).contiguous()


class _ConvBnReluPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps, training, group, out_nchw, impl):
        xh = _to_nhwc(x)
        C = w.shape[0]
        if training:
            y, stats = _C.conv5x5_fwd(xh, w, b, True, impl, group is not None)
            if group is not None:
                _inline_allreduce(group, _padded_stats(stats))   # Σy, Σy², n across the group: SyncBatchNorm
            out, saved = _C.bn_relu_pool_fwd(y, stats, gamma, beta, running_mean, running_var, nbt, momentum, eps, out_nchw)
            count = stats[2 * C:2 * C + 1]
        else:
            y, _ = _C.conv5x5_fwd(xh, w, b, False, impl)
            stats = torch.cat([running_mean, running_var + running_mean * running_mean, running_mean.new_ones(1)])
            out, saved = _C.bn_relu_pool_fwd(y, stats, gamma, beta, None, None, None, 0.0, eps, out_nchw)
            count = stats[2 * C:2 * C + 1]
        ctx.save_for_backward(xh, w, y, saved, gamma, beta, count)
        ctx.group, ctx.out_nchw, ctx.impl, ctx.training = group, out_nchw, impl, training
        ctx.params = (w, b, gamma, beta)
        ctx.x_is_image = x.shape[1] == 1
        ctx.x_shape = x.shape
        return out if out_nchw else out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dout):
        xh, w, y, saved, gamma, beta, count = ctx.saved_tensors
        w_p, b_p, g_p, be_p = ctx.params
        if not ctx.training:
            raise RuntimeError("conv_bn_relu_pool: backward through eval-mode BatchNorm is not supported by the fused op")
        d = dout.contiguous() if ctx.out_nchw else dout.permute(0, 2, 3, 1).contiguous()
        gview = _grad_dst(g_p, gamma) if g_p is not None else None
        bview = _grad_dst(be_p, beta) if be_p is not None else None
        sums, dgamma, dbeta = _C.bn_relu_pool_bwd_reduce(d, y, saved, gamma, beta, ctx.out_nchw, gview, bview)
        if ctx.group is not None:
            _inline_allreduce(ctx.group, sums)     # Σdz, Σdz·x̂ across the group
        dy = _C.bn_relu_pool_bwd_apply(d, y, saved, gamma, beta, sums, count, ctx.out_nchw)
        dw = _grad_dst(w_p, w)
        db = _grad_dst(b_p, w.new_empty(w.shape[0])) if b_p is not None else None
        _C.conv5x5_wgrad(dy, xh, dw, db, ctx.impl)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = _C.conv5x5_dgrad(dy, w, ctx.impl).permute(0, 3, 1, 2)
        return dx, dw, db, (dgamma if g_p is not None else None), (dbeta if be_p is not None else None), None, None, None, None, None, None, None, None, None


# =====================================================================================================
# Cooperative fused layers of the reference ConvNet (csrc/cuda/fused_convnet.cu): one kernel per layer and direction
# =====================================================================================================
def fused_convnet_ok(x: torch.Tensor, model) -> bool:
    """The per-image cooperative kernels cover exactly the reference architecture (ref: ddp_example.py:22-41) in
    training mode with local BatchNorm statistics; everything else takes the per-op kernels."""
    if os.environ.get("PDT_FUSED_LAYERS", "1") == "0" or not hasattr(_C, "convnet_l1_fwd"):
        return False
    c1, b1, c2, b2, fc = model.layer1[0], model.layer1[1], model.layer2[0], model.layer2[1], model.fc
    if not (x.dim() == 4 and x.shape[1:] == (1, 28, 28) and x.is_contiguous() and _C.fused_convnet_supported(x.shape[0])):
        return False
    if x.requires_grad and torch.is_grad_enabled():
        return False   # the fused layer-1 backward produces parameter gradients only (the reference never asks for d/d(image))
    if not (c1.weight.shape == (16, 1, 5, 5) and c2.weight.shape == (32, 16, 5, 5) and fc.weight.shape[1] == 1568 and fc.weight.shape[0] <= 64):
        return False
    for bn in (b1, b2):
        if not bn.training or type(bn).__name__ == "SyncBatchNorm" or not bn.track_running_stats or bn.momentum is None or not bn.affine:
            return False
    return all(p.is_contiguous() for p in (c1.weight, c2.weight, fc.weight))


# Targets of the batch whose forward pass is about to run (engine.GraphedTrainStep knows them before it calls the model): the
# whole-forward kernel then also produces the mean cross-entropy and its gradient, and `cross_entropy(logits, target)` picks
# them up instead of launching a kernel.  A plain `loss = criterion(model(x), y)` loop never sets this and is unaffected.
_upcoming_target: Optional[torch.Tensor] = None


_loss_read_after_backward = False


class upcoming_targets:
    """``loss_read_after_backward=True`` (a captured step: nobody looks at the loss before the whole step has run) lets the
    batch mean of the per-image loss terms be folded by the first backward kernel instead of by the forward kernel's tail."""

    def __init__(self, target: Optional[torch.Tensor], loss_read_after_backward: bool = False):
        self.target, self.late = target, loss_read_after_backward

    def __enter__(self):
        global _upcoming_target, _loss_read_after_backward
        self.prev = (_upcoming_target, _loss_read_after_backward)
        _upcoming_target, _loss_read_after_backward = self.target, self.late
        return self

    def __exit__(self, *exc):
        global _upcoming_target, _loss_read_after_backward
        _upcoming_target, _loss_read_after_backward = self.prev
        return False


# The optimizer whose update rides on the last backward kernel (optim.SGD / optim.Adam .ride_on_backward, armed by
# engine.GraphedTrainStep when the gradient reduction does not already carry it, i.e. on one GPU):
# {"kind": "sgd" | "adam", "params": [...10 parameters...], "args": callable -> the rider tuple of convnet_l1_bwd_wgrad, "owner": optimizer}
_sgd_rider: Optional[dict] = None
_sgd_rider_enabled = False


class sgd_rider_enabled:
    """The armed optimizer may ride on backward passes started inside this context only (engine.GraphedTrainStep wraps its step in it):
    a backward pass anywhere else — gradient inspection, clipping experiments, an eager loop — never updates parameters behind the
    caller's back.  Inside it the parameters are already updated when backward returns, so a clip call of the user's own between
    backward and step sees the updated model; clipping is expressible through ``GraphedTrainStep(max_grad_norm=…)``, which lets the
    rider clip the gradients before it applies the update."""

    def __enter__(self):
        global _sgd_rider_enabled
        self.prev, _sgd_rider_enabled = _sgd_rider_enabled, True
        return self

    def __exit__(self, *exc):
        global _sgd_rider_enabled
        _sgd_rider_enabled = self.prev
        return False


def _wgrad_rides_on_layer1() -> bool:
    """conv2's weight gradient runs on the tensor cores *inside* the layer-1 backward kernel (two extra warps per CTA)
    instead of as a kernel of its own between the two layer kernels.  PDT_WGRAD_MERGED=0 restores the separate launch."""
    return os.environ.get("PDT_WGRAD_MERGED", "1") != "0" and hasattr(_C, "convnet_l1_bwd_wgrad")


class _FusedLayer1(torch.autograd.Function):
    """conv1 + BN1 + ReLU + pool1 forward, and its whole backward, as one cooperative kernel each.

    ``w2`` / ``b2`` (conv2's parameters) are inputs of this node on purpose: when conv2's weight gradient rides on the
    layer-1 backward kernel, *this* node returns it, so autograd (and DDP's reducer hooks behind it) sees the gradient
    only after the kernel that produces it has been launched."""

    @staticmethod
    def forward(ctx, x, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps, w2=None, b2=None, whole=None, link=None):
        if whole is not None:
            # ONE launch for the whole forward pass (csrc/cuda/fused_convnet.cu: convnet_fwd_kernel): layer 2 and the
            # classifier of an image run in the same CTA; their results are handed to the next autograd nodes through `whole`
            c2, bn2, fc = whole["conv2"], whole["bn2"], whole["fc"]
            defer = bool(whole.get("defer_loss_mean", False))
            out, y, saved, p2, y2, saved2, logits, loss, dlogits, loss_parts = _C.convnet_fwd(
                x, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps, c2.weight, c2.bias, bn2.weight, bn2.bias,
                bn2.running_mean, bn2.running_var, bn2.num_batches_tracked, float(bn2.momentum), float(bn2.eps), fc.weight, fc.bias,
                whole.get("target"), defer)
            whole["layer2"] = (p2, y2, saved2, logits)
            whole["ce"] = (loss, dlogits)
            whole["ce_deferred"] = (loss_parts, loss) if defer else None
        else:
            out, y, saved = _C.convnet_l1_fwd(x, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps)
        ctx.save_for_backward(x, y, saved, gamma, beta)
        ctx.params = (w, b, gamma, beta, w2, b2)
        ctx.link = link
        return out  # [B,18,18,16]: zero-haloed NHWC frame

    @staticmethod
    def backward(ctx, dp):
        x, y, saved, gamma, beta = ctx.saved_tensors
        w_p, b_p, g_p, be_p, w2_p, b2_p = ctx.params
        dw = _grad_dst(w_p, w_p)
        db = _grad_dst(b_p, b_p) if b_p is not None else None
        dg = _grad_dst(g_p, gamma)
        dbe = _grad_dst(be_p, beta)
        fresh = all(q is None or q.grad is None for q in (w_p, b_p, g_p, be_p, w2_p, b2_p))
        pending = ctx.link.pop("wgrad", None) if ctx.link is not None else None
        dw2 = db2 = None
        if pending is not None:
            dy2, p1, dysum2 = pending
            dw2 = _grad_dst(w2_p, w2_p)
            db2 = _grad_dst(b2_p, b2_p) if b2_p is not None else None
            sgd = None
            prev = ctx.link.pop("prev", None)
            rider = _sgd_rider if _sgd_rider_enabled else None
            if rider is not None and prev is not None and prev[4] and fresh:
                mine = [w_p, b_p, g_p, be_p, w2_p, b2_p] + [q for q, _ in prev[:4]]
                if len(mine) == len(rider["params"]) and all(a is b for a, b in zip(mine, rider["params"])):
                    # autograd has accumulated layer 2's gradients by now (AccumulateGrad runs as soon as its input is ready): they
                    # must be exactly the tensors layer 2's kernel wrote
                    grads = [q.grad if q is not None else None for q, _ in prev[:4]]
                    if all((g is None and ptr == 0) or (g is not None and g.data_ptr() == ptr) for g, (_, ptr) in zip(grads, prev[:4])):
                        sgd = rider["args"](grads)   # None when the optimizer cannot ride this iteration
            _C.convnet_l1_bwd_wgrad(dp.contiguous(), y, x, saved, gamma, beta, dg, dbe, dw, db, dy2, p1, dysum2, dw2, db2, sgd)
        else:
            _C.convnet_l1_bwd(dp.contiguous(), y, x, saved, gamma, beta, dg, dbe, dw, db)
        return None, dw, db, dg, dbe, None, None, None, None, None, dw2, db2, None, None


class _FusedLayer2(torch.autograd.Function):
    """conv2 (wgmma) + BN2 + ReLU + pool2 (+ the classifier's logits, which ride on the pooled activations while they
    are still in shared memory) forward; pool/ReLU/BN backward + conv2 data gradient as one kernel backward.  The
    tensor-core weight gradient follows as its own kernel, or — the default — rides on layer 1's backward kernel."""

    @staticmethod
    def forward(ctx, p1, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps, fcw, fcb, whole=None, link=None, fc_rides=False):
        if whole is not None and "layer2" in whole:
            out, y, saved, logits = whole.pop("layer2")   # produced by the whole-forward launch of layer 1's node
        else:
            out, y, saved, logits = _C.convnet_l2_fwd(p1, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps, fcw, fcb)
        ctx.params = (w, b, gamma, beta, fcw, fcb)
        ctx.link = link
        ctx.fc_rides = fc_rides
        ctx.ce_deferred = whole.get("ce_deferred") if (whole is not None and fc_rides) else None
        if fc_rides:
            # the classifier's backward runs inside this node's backward kernel: the logits are this node's differentiable output
            ctx.save_for_backward(p1, y, saved, gamma, beta, w, out, fcw)
            ctx.set_materialize_grads(False)
        else:
            ctx.save_for_backward(p1, y, saved, gamma, beta, w)
            ctx.mark_non_differentiable(logits)
        return out, logits  # [B,32,7,7] NCHW, [B,classes]

    @staticmethod
    def backward(ctx, dout, dlogits):
        w_p, b_p, g_p, be_p, fcw_p, fcb_p = ctx.params
        dg = _grad_dst(g_p, ctx.saved_tensors[3])
        dbe = _grad_dst(be_p, ctx.saved_tensors[4])
        dfcw = dfcb = None
        if ctx.link is not None:   # do the gradients written here become `.grad` as they are (nothing to accumulate into)?
            ctx.link["prev_fresh"] = ctx.fc_rides and all(q is None or q.grad is None for q in (fcw_p, fcb_p, g_p, be_p))
        if ctx.fc_rides:
            p1, y, saved, gamma, beta, w, out, fcw = ctx.saved_tensors
            if dout is not None:
                raise RuntimeError("fused ConvNet: the pooled activations of the fused classifier path must not be used outside the model")
            dfcw = _grad_dst(fcw_p, fcw)
            dfcb = _grad_dst(fcb_p, fcb_p) if fcb_p is not None else None
            lp, lo = ctx.ce_deferred if ctx.ce_deferred is not None else (None, None)
            dy, dp1, dysum = _C.convnet_l2_bwd_fc(dlogits.contiguous(), fcw, out, dfcw, dfcb, y, saved, gamma, beta, w, dg, dbe, lp, lo)
        else:
            p1, y, saved, gamma, beta, w = ctx.saved_tensors
            dy, dp1, dysum = _C.convnet_l2_bwd(dout.contiguous(), y, saved, gamma, beta, w, dg, dbe)
        if ctx.link is not None and ctx.needs_input_grad[0]:
            # layer 1's backward kernel computes (and layer 1's node returns) conv2's weight / bias gradient
            ctx.link["wgrad"] = (dy, p1, dysum)
            # for the optimizer rider of layer 1's kernel: WHERE these gradients were written — addresses, not tensors (an extra
            # reference would make autograd's AccumulateGrad clone the gradient instead of adopting the bucket view)
            ctx.link["prev"] = ((fcw_p, dfcw.data_ptr() if dfcw is not None else 0), (fcb_p, dfcb.data_ptr() if dfcb is not None else 0),
                                (g_p, dg.data_ptr()), (be_p, dbe.data_ptr()), ctx.link.pop("prev_fresh", False))
            return dp1, None, None, dg, dbe, None, None, None, None, None, dfcw, dfcb, None, None, None
        dw = _grad_dst(w_p, w)
        db = _grad_dst(b_p, b_p) if b_p is not None else None
        # dy and p1 are zero-haloed frames: every operand of the tensor-core weight gradient arrives by TMA
        _C.conv5x5_wgrad_win(dy, p1, dysum, dw, db)
        return dp1, dw, db, dg, dbe, None, None, None, None, None, dfcw, dfcb, None, None, None


class _FusedClassifier(torch.autograd.Function):
    """Autograd node of the classifier whose forward value was already produced by the layer-2 kernel."""

    @staticmethod
    def forward(ctx, feat, w, b, logits):
        ctx.save_for_backward(feat, w)
        ctx.params = (w, b)
        return logits.view_as(logits)

    @staticmethod
    def backward(ctx, dout):
        feat, w = ctx.saved_tensors
        w_p, b_p = ctx.params
        dw = _grad_dst(w_p, w)
        db = _grad_dst(b_p, b_p) if b_p is not None else None
        dx = _C.linear_bwd(dout.contiguous(), feat.reshape(feat.shape[0], -1), w, True, dw, db)
        return dx.view_as(feat), dw, db, None


def fused_convnet_forward(x: torch.Tensor, model) -> torch.Tensor:
    """The reference ConvNet's training forward as ONE kernel (two with PDT_FUSED_WHOLE_FWD=0) (ref: ddp_example.py:36-41)."""
    c1, b1, c2, b2_bn, fc = model.layer1[0], model.layer1[1], model.layer2[0], model.layer2[1], model.fc
    # the classifier's backward rides on layer 2's backward kernel (PDT_FC_MERGED=0: separate linear_bwd launch)
    fc_rides = (os.environ.get("PDT_FC_MERGED", "1") != "0" and hasattr(_C, "convnet_l2_bwd_fc") and fc.weight.shape[0] <= 16
                and fc.weight.requires_grad and c2.weight.requires_grad and fc.weight.data_ptr() % 16 == 0)
    whole = None
    if os.environ.get("PDT_FUSED_WHOLE_FWD", "1") != "0" and fc.weight.shape[0] <= 16 and hasattr(_C, "convnet_fwd"):
        whole = {"conv2": c2, "bn2": b2_bn, "fc": fc}
        t = _upcoming_target
        if (t is not None and os.environ.get("PDT_FUSED_CE", "1") != "0" and t.is_cuda and t.dtype == torch.int64 and t.dim() == 1
                and t.shape[0] == x.shape[0] and t.is_contiguous() and torch.is_grad_enabled()):
            whole["target"] = t
            whole["defer_loss_mean"] = bool(_loss_read_after_backward and fc_rides)
    # conv2's weight gradient is produced by layer 1's backward kernel: layer 1's node owns (w2, b2) for autograd, `link` carries
    # the operands from layer 2's backward to it.  Only when conv1's parameters need gradients (layer 1's backward runs at all).
    link = {} if (_wgrad_rides_on_layer1() and c1.weight.requires_grad and c2.weight.requires_grad) else None
    w2, b2 = (c2.weight, c2.bias) if link is not None else (None, None)
    p1 = _FusedLayer1.apply(x, c1.weight, c1.bias, b1.weight, b1.bias, b1.running_mean, b1.running_var, b1.num_batches_tracked,
                            float(b1.momentum), float(b1.eps), w2, b2, whole, link)
    p2, logits = _FusedLayer2.apply(p1, c2.weight, c2.bias, b2_bn.weight, b2_bn.bias, b2_bn.running_mean, b2_bn.running_var,
                                    b2_bn.num_batches_tracked, float(b2_bn.momentum), float(b2_bn.eps), fc.weight, fc.bias, whole, link, fc_rides)
    if whole is not None and whole.get("target") is not None:
        logits = logits if fc_rides else _FusedClassifier.apply(p2, fc.weight, fc.bias, logits)
        logits._pdt_ce = (whole["target"],) + whole["ce"]   # (target, loss, dlogits) for ops.cross_entropy
        return logits
    if fc_rides:
        return logits
    return _FusedClassifier.apply(p2, fc.weight, fc.bias, logits)


def conv_bn_relu_pool(x: torch.Tensor, conv: torch.nn.Conv2d, bn: torch.nn.Module, out_nchw: Optional[bool] = None,
                      impl: str = "auto") -> torch.Tensor:
    """Conv5×5(pad 2) → BatchNorm (batch stats, optionally synchronised) → ReLU → MaxPool2×2 as two
    kernels forward / four backward (ref layers: ddp_example.py:25-33)."""
    if conv.kernel_size != (5, 5) or conv.stride != (1, 1) or conv.padding != (2, 2) or conv.groups != 1:
        raise ValueError("conv_bn_relu_pool: only 5x5 / stride 1 / pad 2 convolutions are fused")
    if impl == "auto":
        impl = os.environ.get("PDT_CONV_IMPL", "auto")  # auto = tensor cores where implemented, SIMT elsewhere
    group = None
    training = bn.training
    if training and type(bn).__name__ == "SyncBatchNorm" and dist.is_initialized():
        g = getattr(bn, "process_group", None) or dist.get_default_group()
        if g.size() > 1:
            group = g
    if out_nchw is None:
        out_nchw = conv.out_channels >= 32  # last fused layer feeds the flatten: plain NCHW keeps it a view
    momentum = 0.0 if bn.momentum is None else bn.momentum
    if training and bn.momentum is None and bn.num_batches_tracked is not None:
        momentum = 1.0 / float(bn.num_batches_tracked + 1)
    track = bn.track_running_stats
    return _ConvBnReluPool.apply(x, conv.weight, conv.bias, bn.weight, bn.bias, bn.running_mean if track else None,
                                 bn.running_var if track else None, bn.num_batches_tracked if (track and training) else None,
                                 momentum, bn.eps, training or not track, group, out_nchw, impl)


class _Conv5x5(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, impl):
        xh = _to_nhwc(x)
        y, _ = _C.conv5x5_fwd(xh, w, b, False, impl)
        ctx.save_for_backward(xh, w)
        ctx.params, ctx.impl = (w, b), impl
        return y.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dout):
        xh, w = ctx.saved_tensors
        w_p, b_p = ctx.params
        dy = dout.permute(0, 2, 3, 1).contiguous()
        dw = _grad_dst(w_p, w)
        db = _grad_dst(b_p, w.new_empty(w.shape[0])) if b_p is not None else None
        _C.conv5x5_wgrad(dy, xh, dw, db, ctx.impl)
        dx = _C.conv5x5_dgrad(dy, w, ctx.impl).permute(0, 3, 1, 2) if ctx.needs_input_grad[0] else None
        return dx, dw, db, None


def conv2d(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, impl: str = "auto") -> torch.Tensor:
    """5×5 / stride 1 / pad 2 convolution on our kernels (tensor cores for 16→32 channels); returns a
    channels_last tensor."""
    return _Conv5x5.apply(x, weight, bias, impl)


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        xc = x.contiguous()
        ctx.save_for_backward(xc, w)
        ctx.params = (w, b)
        return _C.linear_fwd(xc, w, b)

    @staticmethod
    def backward(ctx, dout):
        x, w = ctx.saved_tensors
        w_p, b_p = ctx.params
        dw = _grad_dst(w_p, w)
        db = _grad_dst(b_p, w.new_empty(w.shape[0])) if b_p is not None else None
        dx = _C.linear_bwd(dout.contiguous(), x, w, ctx.needs_input_grad[0], dw, db)
        return (dx if ctx.needs_input_grad[0] else None), dw, db


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Classifier head ``x·Wᵀ + b`` for narrow outputs (N ≤ 16) (ref: ddp_example.py:34,40)."""
    if weight.shape[0] > 16:
        return torch.nn.functional.linear(x, weight, bias)
    return _Linear.apply(x, weight, bias)


class _CrossEntropy(torch.autograd.Function):
    """Mean cross-entropy whose forward launch also produces the gradient w.r.t. the logits for a unit incoming
    gradient, (softmax − onehot)/B.  Backward is then free when the incoming gradient is known to be one
    (``engine.GraphedTrainStep`` seeds backward with a tensor tagged ``_pdt_unit_seed``) and one scaling kernel otherwise."""

    @staticmethod
    def forward(ctx, logits, target):
        loss, grad0 = _C.cross_entropy_fwd(logits.contiguous(), target.contiguous(), True)
        ctx.save_for_backward(grad0)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        (grad0,) = ctx.saved_tensors
        if getattr(dloss, "_pdt_unit_seed", False):
            return grad0, None
        return grad0 * dloss, None


class _CrossEntropyPrecomputed(torch.autograd.Function):
    """Autograd node of a mean cross-entropy whose value and unit-gradient were produced by the model's forward kernel."""

    @staticmethod
    def forward(ctx, logits, loss, grad0):
        ctx.save_for_backward(grad0)
        return loss.view_as(loss)

    @staticmethod
    def backward(ctx, dloss):
        (grad0,) = ctx.saved_tensors
        if getattr(dloss, "_pdt_unit_seed", False):
            return grad0, None, None
        return grad0 * dloss, None, None


def cross_entropy(logits: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """Mean cross-entropy over the batch: fused log-softmax + NLL (ref: ddp_example.py:61,87)."""
    pre = getattr(logits, "_pdt_ce", None)
    if pre is not None and pre[0] is target:
        return _CrossEntropyPrecomputed.apply(logits, pre[1], pre[2])
    return _CrossEntropy.apply(logits, target)


def sgd_step(params, grads, momentum_bufs, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False,
             maximize=False, first_step=False, lr_tensor=None) -> None:
    _C.sgd_multi(list(params), list(grads), list(momentum_bufs) if momentum_bufs else [], float(lr), lr_tensor, float(momentum),
                 float(dampening), float(weight_decay), bool(nesterov), bool(maximize), bool(first_step))


def adam_step(params, grads, exp_avgs, exp_avg_sqs, steps, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0,
              decoupled=False, maximize=False, lr_tensor=None) -> None:
    """One Adam (``decoupled=False``) or AdamW update of every tensor, one kernel launch per 48 tensors.  ``steps`` are the fp32
    step counts on the device: the launch uses step + 1 for the bias corrections and stores it, so a replayed graph advances it."""
    _C.adam_multi(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), list(steps), float(lr), lr_tensor, float(beta1),
                  float(beta2), float(eps), float(weight_decay), bool(decoupled), bool(maximize))


def grad_norm_clip(grads, max_norm, norm_type=2.0, scale=True) -> torch.Tensor:
    """The total ``norm_type`` norm (2 or inf) of fp32 contiguous gradients on one device, and — with ``scale`` — every gradient
    multiplied by torch's clip coefficient ``min(max_norm / (norm + 1e-6), 1)``: two launches per 48 tensors, graph-capturable,
    the norm the same bit for bit from run to run.  Returns the norm as a 0-d device tensor; ``scale=False`` stops after the
    norm, and ``grad_scale(grads, norm)`` applies the coefficient later."""
    return _C.grad_norm_clip(list(grads), float(max_norm), float(norm_type), bool(scale))


def grad_scale(grads, norm: torch.Tensor) -> None:
    """Multiply every gradient by the clip coefficient of ``norm``, a tensor returned by :func:`grad_norm_clip`."""
    _C.grad_scale(list(grads), norm)


# ---- generic (NCHW) BatchNorm pieces used by parallel.SyncBatchNorm ------------------------------------------
def bn_local_stats(x: torch.Tensor) -> torch.Tensor:
    """float64 [2C+2] = per-channel Σx, Σx² (accumulated in fp64), the per-channel element count, one zero pad."""
    return _C.bn_stats_nchw_f64(x)


def bn_finalize(stats, C, eps, momentum, running_mean, running_var):
    """All-reduced float64 statistics → (mean, invstd, count) in fp32, running statistics updated in place: one kernel."""
    return _C.bn_finalize(stats, int(C), float(eps), float(momentum), running_mean, running_var)


def bn_apply(x, mean, invstd, weight, bias):
    return _C.bn_apply_nchw(x, mean.contiguous(), invstd.contiguous(), weight, bias)


def bn_backward_reduce(dy, x, mean, invstd):
    """[4C] = Σdy, Σdy·(x−μ), dγ, dβ (local batch)."""
    return _C.bn_bwd_reduce_nchw(dy, x, mean.contiguous(), invstd.contiguous())


def bn_backward_apply(dy, x, mean, invstd, weight, mean_dy, mean_dy_xmu):
    return _C.bn_bwd_apply_nchw(dy, x, mean.contiguous(), invstd.contiguous(), weight, mean_dy.contiguous(), mean_dy_xmu.contiguous())
