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


def _to_nhwc(x: torch.Tensor) -> torch.Tensor:
    """[B,C,H,W] (any strides) → contiguous [B,H,W,C] without a copy when already channels_last."""
    if x.shape[1] == 1:
        return x.contiguous().view(x.shape[0], x.shape[2], x.shape[3], 1)
    return x.permute(0, 2, 3, 1).contiguous()


def _refuse_double_backward(op: str) -> None:
    """Called first in every native backward.  Autograd runs a backward in grad mode only under ``create_graph=True`` (gradient
    penalties, Hessian-vector products); the kernels' gradients carry no graph, so a loss built from them would silently train
    without its gradient term.  Refuse instead."""
    if torch.is_grad_enabled():
        raise RuntimeError(f"{op}: the native kernels have no double backward (create_graph=True); torch's layers have one: "
                           "ConvNet(fused=False), torch.nn.CrossEntropyLoss")


class _ConvBnReluPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps, training, group, out_nchw):
        xh = _to_nhwc(x)
        C = w.shape[0]
        if training and group is None:
            # one GPU: [mean, M2, n], no cancellation when |mean| ≫ std
            y, stats = _C.conv5x5_fwd(xh, w, b, True, centred=True)
            out, saved = _C.bn_relu_pool_fwd(y, stats, gamma, beta, running_mean, running_var, nbt, momentum, eps, out_nchw,
                                             centred=True)
            count = stats[2 * C:2 * C + 1]
        elif training:
            # SyncBatchNorm: fp64 [Σy = n·mean, Σy² = M2 + n·mean², n, 0] from this rank's centred fold, summed across the group;
            # the group's mean and variance are then taken in fp64, where Σy²/N − mean² keeps the variance's digits
            y, stats = _C.conv5x5_fwd(xh, w, b, True, fp64_sums=True)
            _inline_allreduce(group, stats)
            out, saved = _C.bn_relu_pool_fwd(y, stats, gamma, beta, running_mean, running_var, nbt, momentum, eps, out_nchw,
                                             fp64_sums=True)
            count = saved[2 * C:]   # the group's count, which bn_relu_pool_fwd leaves behind the mean and invstd
        else:
            y, _ = _C.conv5x5_fwd(xh, w, b, False)
            # the running mean and variance as they are: no round trip through sums, which would cancel the variance's digits
            out, saved = _C.bn_relu_pool_fwd(y, torch.cat([running_mean, running_var]), gamma, beta, None, None, None, 0.0, eps, out_nchw,
                                             mean_var=True)
            count = None   # the running statistics are constants: backward has no batch-mean terms
        ctx.save_for_backward(xh, w, y, saved, gamma, beta, count)
        ctx.group, ctx.out_nchw, ctx.training = group, out_nchw, training
        ctx.params = (w, b, gamma, beta)
        ctx.x_is_image = x.shape[1] == 1
        ctx.x_shape = x.shape
        return out if out_nchw else out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dout):
        _refuse_double_backward("conv_bn_relu_pool")
        xh, w, y, saved, gamma, beta, count = ctx.saved_tensors
        w_p, b_p, g_p, be_p = ctx.params
        d = dout.contiguous() if ctx.out_nchw else dout.permute(0, 2, 3, 1).contiguous()
        gview = _grad_dst(g_p, gamma) if g_p is not None else None
        bview = _grad_dst(be_p, beta) if be_p is not None else None
        # dγ = Σdz·x̂ and dβ = Σdz in either mode: `saved` holds the mean and invstd the forward normalised with
        sums, dgamma, dbeta = _C.bn_relu_pool_bwd_reduce(d, y, saved, gamma, beta, ctx.out_nchw, gview, bview)
        if not ctx.training:
            dy = _C.bn_relu_pool_bwd_apply(d, y, saved, gamma, beta, None, None, ctx.out_nchw, mean_var=True)
        else:
            if ctx.group is not None:
                _inline_allreduce(ctx.group, sums)     # Σdz, Σdz·x̂ across the group
            dy = _C.bn_relu_pool_bwd_apply(d, y, saved, gamma, beta, sums, count, ctx.out_nchw)
        dw = _grad_dst(w_p, w)
        db = _grad_dst(b_p, w.new_empty(w.shape[0])) if b_p is not None else None
        _C.conv5x5_wgrad(dy, xh, dw, db)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = _C.conv5x5_dgrad(dy, w).permute(0, 3, 1, 2)
        return dx, dw, db, (dgamma if g_p is not None else None), (dbeta if be_p is not None else None), None, None, None, None, None, None, None, None


# =====================================================================================================
# Cooperative fused layers of the reference ConvNet (csrc/cuda/fused_convnet.cu): one kernel per layer and direction
# =====================================================================================================
def fused_convnet_ok(x: torch.Tensor, model) -> bool:
    """The per-image cooperative kernels cover exactly the reference architecture (ref: ddp_example.py:22-41) in
    training mode with local BatchNorm statistics, a classifier of at most 16 classes (the width of the fused classifier
    and its backward) and every parameter trainable (the two fused backward kernels write all ten gradients); everything
    else, a partially frozen model included, takes the per-op kernels."""
    if os.environ.get("PDT_FUSED_LAYERS", "1") == "0" or not hasattr(_C, "convnet_fwd"):
        return False
    c1, b1, c2, b2, fc = model.layer1[0], model.layer1[1], model.layer2[0], model.layer2[1], model.fc
    if not (x.dim() == 4 and x.shape[1:] == (1, 28, 28) and x.is_contiguous() and _C.fused_convnet_supported(x.shape[0])):
        return False
    if x.requires_grad and torch.is_grad_enabled():
        return False   # the fused layer-1 backward produces parameter gradients only (the reference never asks for d/d(image))
    if not (c1.weight.shape == (16, 1, 5, 5) and c2.weight.shape == (32, 16, 5, 5) and fc.weight.shape[1] == 1568 and fc.weight.shape[0] <= 16):
        return False
    for bn in (b1, b2):
        if not bn.training or type(bn).__name__ == "SyncBatchNorm" or not bn.track_running_stats or bn.momentum is None or not bn.affine:
            return False
    params = (c1.weight, c1.bias, b1.weight, b1.bias, c2.weight, c2.bias, b2.weight, b2.bias, fc.weight, fc.bias)
    if not all(p is None or p.requires_grad for p in params):
        return False
    if fc.weight.data_ptr() % 16 != 0:
        return False   # layer 2's backward kernel stages the classifier weights in 16-byte copies
    return all(p.is_contiguous() for p in (c1.weight, c2.weight, fc.weight))


# Targets of the batch whose forward pass is about to run (engine.GraphedTrainStep knows them before it calls the model): the
# whole-forward kernel then also produces the mean cross-entropy and its gradient, and `cross_entropy(logits, target)` picks
# them up instead of launching a kernel.  A plain `loss = criterion(model(x), y)` loop never sets this and is unaffected.
_upcoming_target: Optional[torch.Tensor] = None


_loss_read_after_backward = False
_upcoming_grad_scale = 1.0

# torch's cross-entropy options as (weight, ignore_index, reduction, label_smoothing); the default is the plain mean
DEFAULT_CE_SPEC = (None, -100, "mean", 0.0)
_upcoming_spec = DEFAULT_CE_SPEC


def ce_spec_of(criterion) -> tuple:
    """The options of a ``pdt.nn.CrossEntropyLoss`` criterion as a spec for ``upcoming_targets``; the default spec for any other."""
    from ..nn.loss import CrossEntropyLoss

    if isinstance(criterion, CrossEntropyLoss):
        return (criterion.weight, criterion.ignore_index, criterion.reduction, criterion.label_smoothing)
    return DEFAULT_CE_SPEC


def _same_spec(a: tuple, b: tuple) -> bool:
    """The same weight tensor (or none) and equal scalars."""
    return a[0] is b[0] and a[1] == b[1] and a[2] == b[2] and a[3] == b[3]


class upcoming_targets:
    """``loss_read_after_backward=True`` (a captured step: nobody looks at the loss before the whole step has run) lets the
    batch mean of the per-image loss terms be folded by the first backward kernel instead of by the forward kernel's tail.

    ``grad_scale`` (gradient accumulation over k micro-batches: 1/k) makes the forward kernel produce ``grad_scale · loss`` and its
    gradient, so backward seeded with one yields torch's ``(loss / k).backward()`` with no scaling kernel.  That is right only when
    the criterion's result IS the cross-entropy ``cross_entropy`` returned (its ``_pdt_loss_scale`` says by how much it is scaled):
    a criterion that computes anything from it (``ce * w``, ``ce + reg``) would see the scaled value.  ``fused_ce_consumed`` lists
    every fused cross-entropy handed out since ``reset_fused_ce_consumed``, so the caller can check that before it scales.

    ``spec`` = (weight, ignore_index, reduction, label_smoothing): the options of the criterion that will consume the loss
    (``ce_spec_of``); the forward kernel computes that loss, and ``cross_entropy`` uses it only when called with the same options."""

    def __init__(self, target: Optional[torch.Tensor], loss_read_after_backward: bool = False, grad_scale: float = 1.0,
                 spec: tuple = DEFAULT_CE_SPEC):
        if not float(grad_scale) > 0:
            raise ValueError(f"grad_scale must be positive, got {grad_scale}")
        self.target, self.late, self.scale, self.spec = target, loss_read_after_backward, float(grad_scale), tuple(spec)

    def __enter__(self):
        global _upcoming_target, _loss_read_after_backward, _upcoming_grad_scale, _upcoming_spec
        self.prev = (_upcoming_target, _loss_read_after_backward, _upcoming_grad_scale, _upcoming_spec)
        _upcoming_target, _loss_read_after_backward, _upcoming_grad_scale, _upcoming_spec = self.target, self.late, self.scale, self.spec
        return self

    def __exit__(self, *exc):
        global _upcoming_target, _loss_read_after_backward, _upcoming_grad_scale, _upcoming_spec
        _upcoming_target, _loss_read_after_backward, _upcoming_grad_scale, _upcoming_spec = self.prev
        return False


# Gradient accumulation inside the two fused backward kernels (engine.GraphedTrainStep(accumulation_steps=k)).  On micro-batches 2..k
# the engine sets every .grad to None and hands the buffers micro-batch 1 left back through `accumulate_into`: the fused nodes take
# them as their destinations, launch their kernels in accumulate mode (g = g_old + v) and return them, and autograd adopts the sums
# as fresh gradients — no AccumulateGrad add, and the optimizer rider's fresh-gradient checks hold on the last micro-batch.  A writer
# that overwrites (the per-op kernels) never consults this, so the engine arms it only when `fused_backward_params` shows that the
# fused kernels wrote every gradient of micro-batch 1.
_accumulate: Optional[dict] = None     # {"grads": {id(param): buffer}, "loss": tensor the loss fold adds to, or None}
_fused_backward_params: Optional[list] = None


class accumulate_into:
    """Inside this context the fused backward kernels add into ``grads`` ({parameter: buffer}) instead of writing fresh gradients,
    and the deferred loss fold adds into ``loss``.  ``leftover()`` lists the parameters whose buffer no kernel took."""

    def __init__(self, grads: dict, loss: Optional[torch.Tensor] = None):
        self.state = {"grads": {id(p): g for p, g in grads.items()}, "loss": loss}
        self.params = {id(p): p for p in grads}

    def __enter__(self):
        global _accumulate
        self.prev, _accumulate = _accumulate, self.state
        return self

    def __exit__(self, *exc):
        global _accumulate
        _accumulate = self.prev
        return False

    def leftover(self) -> list:
        return [self.params[i] for i in self.state["grads"]]


def fused_backward_params() -> Optional[list]:
    """The parameters whose gradients the last backward pass wrote through the two fused ConvNet backward kernels — all ten, the
    classifier's and conv2's included — or None when that pass did not run them.  Reset with ``reset_fused_backward_params``."""
    return _fused_backward_params


def reset_fused_backward_params() -> None:
    global _fused_backward_params
    _fused_backward_params = None


def _take_accumulated(params) -> Optional[list]:
    """Under ``accumulate_into``: the kept buffers of ``params`` (None entries stay None) as fresh aliases autograd may adopt, when
    every one of them has one; None otherwise (nothing is taken)."""
    acc = _accumulate
    if acc is None or not all(p is None or id(p) in acc["grads"] for p in params):
        return None
    return [None if p is None else acc["grads"].pop(id(p)).detach().view(p.shape) for p in params]


# The optimizer whose update rides on the last backward kernel (optim.SGD / optim.Adam .ride_on_backward, armed by
# engine.GraphedTrainStep when the gradient reduction does not already carry it, i.e. on one GPU): an optim._riding.Rider
_sgd_rider = None
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


class _FusedLayer1(torch.autograd.Function):
    """conv1 + BN1 + ReLU + pool1 forward — the node of the whole-forward launch — and its whole backward as one cooperative kernel.

    ``w2`` / ``b2`` (conv2's parameters) are inputs of this node on purpose: conv2's weight gradient rides on the layer-1
    backward kernel, so *this* node returns it, and autograd (and DDP's reducer hooks behind it) sees the gradient only after
    the kernel that produces it has been launched."""

    @staticmethod
    def forward(ctx, x, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps, w2, b2, whole, link):
        # ONE launch for the whole forward pass (csrc/cuda/fused_convnet.cu: convnet_fwd_kernel): layer 2 and the
        # classifier of an image run in the same CTA; their results are handed to the next autograd nodes through `whole`
        c2, bn2, fc = whole["conv2"], whole["bn2"], whole["fc"]
        defer = bool(whole.get("defer_loss_mean", False))
        cw, ignore_index, reduction, smoothing = whole.get("spec", DEFAULT_CE_SPEC)
        out, _, saved, p2, y2, saved2, logits, loss, dlogits, loss_parts = _C.convnet_fwd(
            x, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps, c2.weight, c2.bias, bn2.weight, bn2.bias,
            bn2.running_mean, bn2.running_var, bn2.num_batches_tracked, float(bn2.momentum), float(bn2.eps), fc.weight, fc.bias,
            whole.get("target"), defer, float(whole.get("grad_scale", 1.0)), cw, int(ignore_index), float(smoothing), reduction,
            keep_y1=False)
        whole["layer2"] = (p2, y2, saved2, logits)
        whole["ce"] = (loss, dlogits)
        whole["ce_deferred"] = (loss_parts, loss) if defer else None
        # conv1's output is not kept: the backward kernel recomputes it from x, w and b, bit for bit.  w and b are saved tensors, so an
        # in-place change to them before backward fails autograd's version check instead of recomputing from other weights.
        ctx.save_for_backward(x, w, b, saved, gamma, beta)
        ctx.params = (w, b, gamma, beta, w2, b2)
        ctx.link = link
        return out  # [B,18,18,16]: zero-haloed NHWC frame

    @staticmethod
    def backward(ctx, dp):
        global _fused_backward_params
        _refuse_double_backward("fused ConvNet layer 1")
        x, w, b, saved, gamma, beta = ctx.saved_tensors
        params = ctx.params   # w, b, gamma, beta, w2, b2
        # gradient accumulation (accumulate_into): the buffers of the earlier micro-batches, added to by the kernel
        # (only when layer 2's kernel accumulated too)
        acc = _take_accumulated(params) if ctx.link.get("accumulated") else None
        if acc is not None:
            dw, db, dg, dbe, dw2, db2 = acc
        else:
            w_p, b_p, g_p, be_p, w2_p, b2_p = params
            dw = _grad_dst(w_p, w_p)
            db = _grad_dst(b_p, b_p) if b_p is not None else None
            dg = _grad_dst(g_p, gamma)
            dbe = _grad_dst(be_p, beta)
            dw2 = _grad_dst(w2_p, w2_p)
            db2 = _grad_dst(b2_p, b2_p) if b2_p is not None else None
        fresh = all(q is None or q.grad is None for q in params)
        # layer 2's kernel left conv2's per-image weight-gradient partials; this kernel folds them with its Σdy rows
        dysum2 = ctx.link.pop("dysum")
        prev = ctx.link.pop("prev")
        desc = None
        rider = _sgd_rider if _sgd_rider_enabled else None
        if rider is not None and prev[4] and fresh:
            mine = list(params) + [q for q, _ in prev[:4]]
            if len(mine) == len(rider.params) and all(a is b for a, b in zip(mine, rider.params)):
                # autograd has accumulated layer 2's gradients by now (AccumulateGrad runs as soon as its input is ready): they
                # must be exactly the tensors layer 2's kernel wrote
                grads = [q.grad if q is not None else None for q, _ in prev[:4]]
                if all((g is None and ptr == 0) or (g is not None and g.data_ptr() == ptr) for g, (_, ptr) in zip(grads, prev[:4])):
                    desc = rider.build(grads)   # None when the optimizer cannot ride this iteration
        _C.convnet_l1_bwd_wgrad(dp.contiguous(), None, x, saved, gamma, beta, dg, dbe, dw, db, None, None, dysum2, dw2, db2, desc,
                                clip=rider.clip if desc is not None else None, accumulate=acc is not None, w1=w, b1=b)
        if desc is not None:
            rider.owner._rode = True
        _fused_backward_params = list(params) + [q for q, _ in prev[:4]]
        return None, dw, db, dg, dbe, None, None, None, None, None, dw2, db2, None, None


class _FusedLayer2(torch.autograd.Function):
    """conv2 (wgmma) + BN2 + ReLU + pool2 + the classifier's logits, forward (produced by the whole-forward launch of layer 1's
    node); the classifier's backward + pool/ReLU/BN backward + conv2 data gradient + the per-image partials of conv2's weight
    gradient as one kernel backward.  Layer 1's backward kernel folds those partials."""

    @staticmethod
    def forward(ctx, p1, w, b, gamma, beta, running_mean, running_var, nbt, momentum, eps, fcw, fcb, whole, link):
        out, y, saved, logits = whole.pop("layer2")
        ctx.params = (w, b, gamma, beta, fcw, fcb)
        ctx.link = link
        ctx.ce_deferred = whole.get("ce_deferred")
        # the classifier's backward runs inside this node's backward kernel: the logits are this node's differentiable output
        ctx.save_for_backward(p1, y, saved, gamma, beta, w, out, fcw)
        ctx.set_materialize_grads(False)
        return out, logits  # [B,32,7,7] NCHW, [B,classes]

    @staticmethod
    def backward(ctx, dout, dlogits):
        _refuse_double_backward("fused ConvNet layer 2")
        w_p, b_p, g_p, be_p, fcw_p, fcb_p = ctx.params
        p1, y, saved, gamma, beta, w, out, fcw = ctx.saved_tensors
        if dout is not None:
            raise RuntimeError("fused ConvNet: the pooled activations of the fused classifier path must not be used outside the model")
        # do the gradients written here become `.grad` as they are (nothing to accumulate into)?
        fresh = all(q is None or q.grad is None for q in (fcw_p, fcb_p, g_p, be_p))
        # gradient accumulation (accumulate_into): this kernel and layer 1's add into the earlier micro-batches' buffers
        acc = _take_accumulated((g_p, be_p, fcw_p, fcb_p))
        ctx.link["accumulated"] = acc is not None
        lp, lo = ctx.ce_deferred if ctx.ce_deferred is not None else (None, None)
        if acc is not None:
            dg, dbe, dfcw, dfcb = acc
            if lp is not None:   # the step's loss adds up over the micro-batches too
                lo = _accumulate["loss"]
                if lo is None:
                    raise RuntimeError("gradient accumulation: the deferred loss of this micro-batch has no buffer to add into")
        else:
            dg = _grad_dst(g_p, gamma)
            dbe = _grad_dst(be_p, beta)
            dfcw = _grad_dst(fcw_p, fcw)
            dfcb = _grad_dst(fcb_p, fcb_p) if fcb_p is not None else None
        # given p1, the kernel computes conv2's per-image weight-gradient partials for layer 1's kernel to fold
        _, dp1, dysum = _C.convnet_l2_bwd_fc(dlogits.contiguous(), fcw, out, dfcw, dfcb, y, saved, gamma, beta, w, dg, dbe, lp, lo, p1,
                                             accumulate=acc is not None)
        ctx.link["dysum"] = dysum
        # for the optimizer rider of layer 1's kernel: WHERE these gradients were written — addresses, not tensors (an extra
        # reference would make autograd's AccumulateGrad clone the gradient instead of adopting the bucket view)
        ctx.link["prev"] = ((fcw_p, dfcw.data_ptr()), (fcb_p, dfcb.data_ptr() if dfcb is not None else 0),
                            (g_p, dg.data_ptr()), (be_p, dbe.data_ptr()), fresh)
        return dp1, None, None, dg, dbe, None, None, None, None, None, dfcw, dfcb, None, None


def fused_convnet_forward(x: torch.Tensor, model) -> torch.Tensor:
    """The reference ConvNet's training forward as ONE kernel (ref: ddp_example.py:36-41)."""
    c1, b1, c2, b2_bn, fc = model.layer1[0], model.layer1[1], model.layer2[0], model.layer2[1], model.fc
    whole = {"conv2": c2, "bn2": b2_bn, "fc": fc}
    t = _upcoming_target
    spec = _upcoming_spec
    # class indices [B], or class probabilities [B, ncls] (fp32, as pdt.nn.CrossEntropyLoss runs them natively)
    index = t is not None and t.dtype == torch.int64 and t.dim() == 1 and t.shape[0] == x.shape[0]
    soft = t is not None and t.dtype == torch.float32 and t.shape == (x.shape[0], fc.weight.shape[0])
    if ((index or soft) and t.is_cuda and t.is_contiguous() and torch.is_grad_enabled()
            and _rider_spec_ok(spec, fc.weight, soft)):
        whole["target"] = t
        whole["defer_loss_mean"] = bool(_loss_read_after_backward)
        whole["grad_scale"] = _upcoming_grad_scale
        whole["spec"] = spec
    # conv2's weight gradient is produced by layer 1's backward kernel: layer 1's node owns (w2, b2) for autograd, `link` carries
    # the operands from layer 2's backward to it
    link = {}
    p1 = _FusedLayer1.apply(x, c1.weight, c1.bias, b1.weight, b1.bias, b1.running_mean, b1.running_var, b1.num_batches_tracked,
                            float(b1.momentum), float(b1.eps), c2.weight, c2.bias, whole, link)
    _, logits = _FusedLayer2.apply(p1, c2.weight, c2.bias, b2_bn.weight, b2_bn.bias, b2_bn.running_mean, b2_bn.running_var,
                                   b2_bn.num_batches_tracked, float(b2_bn.momentum), float(b2_bn.eps), fc.weight, fc.bias, whole, link)
    if whole.get("target") is not None:
        # (target, loss, dlogits, scale of loss and gradient, loss folded by layer 2's backward kernel, spec) for ops.cross_entropy
        logits._pdt_ce = (whole["target"],) + whole["ce"] + (float(whole.get("grad_scale", 1.0)), whole["ce_deferred"] is not None,
                                                             whole["spec"])
    return logits


def _rider_spec_ok(spec: tuple, fcw: torch.Tensor, soft: bool = False) -> bool:
    """Whether the forward kernel's cross-entropy can take these options (what pdt.nn.CrossEntropyLoss runs natively); a criterion
    with others computes its loss itself, so the rider is left off.  ``soft``: class-probability targets, which torch takes with
    the default ``ignore_index`` only."""
    w, ignore_index, reduction, smoothing = spec
    return (reduction in ("mean", "sum") and 0.0 <= float(smoothing) <= 1.0 and isinstance(ignore_index, int)
            and (not soft or ignore_index == -100)
            and (w is None or (w.dtype == torch.float32 and w.is_contiguous() and w.shape == (fcw.shape[0],) and w.device == fcw.device)))


def conv_bn_relu_pool(x: torch.Tensor, conv: torch.nn.Conv2d, bn: torch.nn.Module, out_nchw: Optional[bool] = None) -> torch.Tensor:
    """Conv5×5(pad 2) → BatchNorm (batch stats, optionally synchronised) → ReLU → MaxPool2×2 as two
    kernels forward / four backward (ref layers: ddp_example.py:25-33).  ``padding="same"`` is pad 2 for a 5×5 kernel."""
    if (conv.kernel_size != (5, 5) or conv.stride != (1, 1) or conv.padding not in ((2, 2), "same") or conv.dilation != (1, 1)
            or conv.groups != 1 or conv.padding_mode != "zeros"):
        raise ValueError("conv_bn_relu_pool: only 5x5 / stride 1 / pad 2 / undilated / zero-padded convolutions are fused")
    # A PDT_CONV_IMPL that names another conv2 kernel (as bench.py --conv-impl does) is refused rather than ignored, so that no
    # run reports TMA-im2col numbers under another kernel's name.
    conv_impl = os.environ.get("PDT_CONV_IMPL", "auto")
    if conv_impl not in ("auto", "tma"):
        raise ValueError(f"PDT_CONV_IMPL={conv_impl!r}: the per-op conv2 always runs the TMA-im2col kernels now; "
                         "unset PDT_CONV_IMPL or set it to 'auto' or 'tma'")
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
                                 momentum, bn.eps, training or not track, group, out_nchw)


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        xc = x.contiguous()
        ctx.save_for_backward(xc, w)
        ctx.params = (w, b)
        return _C.linear_fwd(xc, w, b)

    @staticmethod
    def backward(ctx, dout):
        _refuse_double_backward("linear")
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
    (``engine.GraphedTrainStep`` seeds backward with a tensor tagged ``_pdt_unit_seed``) and one scaling kernel otherwise.
    ``spec`` (weight, ignore_index, reduction, label_smoothing): torch's options, in the same launch."""

    @staticmethod
    def forward(ctx, logits, target, spec=DEFAULT_CE_SPEC):
        w, ignore_index, reduction, smoothing = spec
        loss, grad0 = _C.cross_entropy_fwd(logits.contiguous(), target.contiguous(), True, w, int(ignore_index), float(smoothing),
                                           reduction)
        ctx.save_for_backward(grad0)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        _refuse_double_backward("cross_entropy")
        (grad0,) = ctx.saved_tensors
        if getattr(dloss, "_pdt_unit_seed", False):
            return grad0, None, None
        return grad0 * dloss, None, None


class _CrossEntropyPrecomputed(torch.autograd.Function):
    """Autograd node of a mean cross-entropy whose value and unit-gradient were produced by the model's forward kernel."""

    @staticmethod
    def forward(ctx, logits, loss, grad0):
        ctx.save_for_backward(grad0)
        return loss.view_as(loss)

    @staticmethod
    def backward(ctx, dloss):
        _refuse_double_backward("cross_entropy (computed by the fused forward)")
        (grad0,) = ctx.saved_tensors
        if getattr(dloss, "_pdt_unit_seed", False):
            return grad0, None, None
        return grad0 * dloss, None, None


_fused_ce_consumed: list = []   # the losses cross_entropy built from the forward kernel's cross-entropy (as id, scale)


def reset_fused_ce_consumed() -> None:
    _fused_ce_consumed.clear()


def fused_ce_consumed() -> list:
    """``(id(loss), scale)`` of every loss ``cross_entropy`` built from the forward kernel's cross-entropy since the last
    ``reset_fused_ce_consumed``: a caller that wants the loss pre-scaled (``upcoming_targets(grad_scale=…)``) checks that its
    criterion returned exactly one of them, unchanged."""
    return list(_fused_ce_consumed)


def cross_entropy(logits: torch.Tensor, target: torch.Tensor, weight: Optional[torch.Tensor] = None, ignore_index: int = -100,
                  reduction: str = "mean", label_smoothing: float = 0.0) -> torch.Tensor:
    """Cross-entropy over the batch, mean or sum, with torch's class weights, ignore_index and label smoothing: fused log-softmax +
    NLL (ref: ddp_example.py:61,87).  ``target``: int64 class indices [B], or fp32 class probabilities [B, C].  The value the
    model's forward kernel computed is used when it was computed for this target tensor with the same options (the same weight
    tensor, equal scalars)."""
    spec = (weight, ignore_index, reduction, label_smoothing)
    pre = getattr(logits, "_pdt_ce", None)
    if pre is not None and pre[0] is target and _same_spec(pre[5], spec):
        loss = _CrossEntropyPrecomputed.apply(logits, pre[1], pre[2])
        loss._pdt_loss_scale = pre[3]   # upcoming_targets(grad_scale=…): the value and its gradient are grad_scale · the mean
        loss._pdt_loss_deferred = pre[4]
        _fused_ce_consumed.append((id(loss), pre[3]))
        return loss
    return _CrossEntropy.apply(logits, target, spec)


def cross_entropy_accumulate(logits: torch.Tensor, target: torch.Tensor, acc: torch.Tensor, rows: int,
                             spec: tuple = DEFAULT_CE_SPEC) -> None:
    """Add the evaluation metrics of ``logits[:rows]`` against ``target[:rows]`` to ``acc``, a float64 ``[4]`` tensor on the logits'
    device: Σ of the loss terms, Σ of the counted rows' target weights (the mean's divisor, whatever the reduction), the counted
    rows whose ``argmax`` is the target, and the counted rows.  A row counts when its target lies in [0, C) and is not
    ``ignore_index``.  ``spec`` = (weight, ignore_index, reduction, label_smoothing), the criterion's options.

    One launch of the native cross-entropy kernel where ``nn.loss.native_ok`` holds, torch ops otherwise; neither synchronises
    with the host."""
    from ..nn.loss import native_ok

    weight, ignore_index, reduction, smoothing = spec
    if target.dtype == torch.int64 and native_ok(logits, target, weight, reduction, smoothing):
        _C.cross_entropy_eval(logits.contiguous(), target.contiguous(), acc, int(rows), weight, int(ignore_index), float(smoothing))
        return
    logits, target = logits[:rows], target[:rows]
    counted = (target >= 0) & (target < logits.shape[1]) & (target != ignore_index)
    safe = torch.where(counted, target, 0)   # torch's cross-entropy rejects a target outside [0, C) that is not ignore_index
    terms = torch.nn.functional.cross_entropy(logits, safe, weight, reduction="none", label_smoothing=smoothing)
    w_t = weight.index_select(0, safe) if weight is not None else torch.ones_like(terms)
    hits = counted & (logits.argmax(1) == target)
    zero = terms.new_zeros(())
    acc += torch.stack([torch.where(counted, terms, zero).sum(dtype=torch.float64), torch.where(counted, w_t, zero).sum(dtype=torch.float64),
                        hits.sum().to(torch.float64), counted.sum().to(torch.float64)])


def sgd_step(params, grads, momentum_bufs, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False,
             maximize=False, first_step=False, lr_tensor=None) -> None:
    _C.sgd_multi(list(params), list(grads), list(momentum_bufs) if momentum_bufs else [], float(lr), lr_tensor, float(momentum),
                 float(dampening), float(weight_decay), bool(nesterov), bool(maximize), bool(first_step))


def adam_step(params, grads, exp_avgs, exp_avg_sqs, steps, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0,
              decoupled=False, maximize=False, lr_tensor=None, max_exp_avg_sqs=None) -> None:
    """One Adam (``decoupled=False``) or AdamW update of every tensor, one kernel launch per 48 tensors.  ``steps`` are the fp32
    step counts on the device: the launch uses step + 1 for the bias corrections and stores it, so a replayed graph advances it.
    ``max_exp_avg_sqs``: AMSGrad — each becomes ``torch.maximum(max_exp_avg_sq, exp_avg_sq)`` (a NaN stays) and the denominator
    is formed from it."""
    _C.adam_multi(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), list(steps), float(lr), lr_tensor, float(beta1),
                  float(beta2), float(eps), float(weight_decay), bool(decoupled), bool(maximize),
                  None if max_exp_avg_sqs is None else list(max_exp_avg_sqs))


def rmsprop_step(params, grads, square_avgs, steps, lr, alpha=0.99, eps=1e-8, weight_decay=0.0, momentum=0.0, maximize=False,
                 momentum_buffers=None, grad_avgs=None, lr_tensor=None) -> None:
    """One RMSprop update of every tensor (torch's single-tensor arithmetic), one kernel launch per 48 tensors.  ``momentum_buffers``
    are required when ``momentum > 0``; ``grad_avgs`` make it centered.  ``steps`` (fp32 scalars on the device) do not enter the
    update; the launch advances them, as torch's step does."""
    _C.rmsprop_multi(list(params), list(grads), list(square_avgs), list(momentum_buffers) if momentum_buffers else [],
                     list(grad_avgs) if grad_avgs else [], list(steps), float(lr), lr_tensor, float(alpha), float(eps),
                     float(weight_decay), float(momentum), bool(maximize))


def adagrad_step(params, grads, sums, steps, lr, lr_decay=0.0, eps=1e-10, weight_decay=0.0, maximize=False, lr_tensor=None) -> None:
    """One Adagrad update of every tensor (torch's single-tensor arithmetic), one kernel launch per 48 tensors.  ``steps`` are the
    fp32 step counts s on the device: the launch decays the learning rate to lr / (1 + s·lr_decay) and stores s + 1, so a replayed
    graph advances it."""
    _C.adagrad_multi(list(params), list(grads), list(sums), list(steps), float(lr), lr_tensor, float(lr_decay), float(eps),
                     float(weight_decay), bool(maximize))


def nadam_step(params, grads, exp_avgs, exp_avg_sqs, mu_products, steps, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0,
               momentum_decay=4e-3, decoupled=False, maximize=False, lr_tensor=None) -> None:
    """One NAdam update of every tensor (torch's single-tensor arithmetic), one kernel launch per 48 tensors.  ``steps`` and
    ``mu_products`` are fp32 scalars on the device: the launch forms the momentum schedule of step + 1 from them and stores step + 1
    and the advanced product, so a replayed graph advances both.  ``decoupled``: the weight decay scales the parameter
    (``decoupled_weight_decay=True``) instead of adding to the gradient."""
    _C.nadam_multi(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), list(steps), list(mu_products), float(lr), lr_tensor,
                   float(beta1), float(beta2), float(eps), float(weight_decay), bool(decoupled), bool(maximize), float(momentum_decay))


def radam_step(params, grads, exp_avgs, exp_avg_sqs, steps, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, decoupled=False,
               maximize=False, lr_tensor=None) -> None:
    """One RAdam update of every tensor (torch's single-tensor arithmetic), one kernel launch per 48 tensors.  ``steps`` are the fp32
    step counts on the device: the launch decides from step + 1 whether the update is rectified (ρ_t > 5) and stores it, so a
    replayed graph crosses into the rectified update when torch's step would."""
    _C.radam_multi(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), list(steps), float(lr), lr_tensor, float(beta1),
                   float(beta2), float(eps), float(weight_decay), bool(decoupled), bool(maximize))


def adamax_step(params, grads, exp_avgs, exp_infs, steps, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, maximize=False,
                lr_tensor=None) -> None:
    """One Adamax update of every tensor (torch's single-tensor arithmetic), one kernel launch per 48 tensors.  ``steps`` are the fp32
    step counts on the device: the launch forms the bias correction of step + 1 from them and stores step + 1."""
    _C.adamax_multi(list(params), list(grads), list(exp_avgs), list(exp_infs), list(steps), float(lr), lr_tensor, float(beta1),
                    float(beta2), float(eps), float(weight_decay), bool(maximize))


def adadelta_step(params, grads, square_avgs, acc_deltas, steps, lr, rho=0.9, eps=1e-6, weight_decay=0.0, maximize=False,
                  lr_tensor=None) -> None:
    """One Adadelta update of every tensor (torch's single-tensor arithmetic), one kernel launch per 48 tensors; ``steps`` (fp32 on the
    device) are advanced as torch advances them."""
    _C.adadelta_multi(list(params), list(grads), list(square_avgs), list(acc_deltas), list(steps), float(lr), lr_tensor, float(rho),
                      float(eps), float(weight_decay), bool(maximize))


def asgd_step(params, grads, axs, steps, etas, mus, lr, lambd=1e-4, alpha=0.75, t0=1e6, weight_decay=0.0, maximize=False,
              lr_tensor=None) -> None:
    """One ASGD update of every tensor (torch's single-tensor, non-capturable arithmetic), one kernel launch per 48 tensors.
    ``steps``, ``etas`` and ``mus`` are fp32 scalars on the device: the launch updates with eta and mu and stores step + 1 and the
    eta and mu of that count (from ``lr``, or ``lr_tensor`` when given), so a replayed graph follows torch's schedules."""
    _C.asgd_multi(list(params), list(grads), list(axs), list(steps), list(etas), list(mus), float(lr), lr_tensor, float(lambd),
                  float(alpha), float(t0), float(weight_decay), bool(maximize))


def rprop_step(params, grads, prevs, step_sizes, steps, etaminus=0.5, etaplus=1.2, step_size_min=1e-6, step_size_max=50.0,
               maximize=False) -> None:
    """One Rprop update of every tensor (torch's single-tensor arithmetic, bit for bit), one kernel launch per 48 tensors; ``steps``
    (fp32 on the device) are advanced as torch advances them."""
    _C.rprop_multi(list(params), list(grads), list(prevs), list(step_sizes), list(steps), float(etaminus), float(etaplus),
                   float(step_size_min), float(step_size_max), bool(maximize))


def grad_norm_clip(grads, max_norm, norm_type=2.0, scale=True) -> torch.Tensor:
    """The total ``norm_type`` norm (2 or inf) of fp32 contiguous gradients on one device, and — with ``scale`` — every gradient
    multiplied by torch's clip coefficient ``min(max_norm / (norm + 1e-6), 1)``: two launches per 48 tensors, graph-capturable,
    the norm the same bit for bit from run to run.  Returns the norm as a 0-d device tensor; ``scale=False`` stops after the
    norm, and ``grad_scale(grads, norm)`` applies the coefficient later."""
    return _C.grad_norm_clip(list(grads), float(max_norm), float(norm_type), bool(scale))


def grad_scale(grads, norm: torch.Tensor) -> None:
    """Multiply every gradient by the clip coefficient of ``norm``, a tensor returned by :func:`grad_norm_clip`."""
    _C.grad_scale(list(grads), norm)


def average_update(averaged, current, n_averaged: torch.Tensor, decay: Optional[float] = None, copied=(), copied_from=()) -> None:
    """One ``AveragedModel.update_parameters`` with torch's EMA (``decay``) or SWA (``decay=None``) ``multi_avg_fn``: every
    ``averaged`` tensor (fp32, or int64 under EMA) takes its ``current`` partner's value when ``n_averaged`` (an int64 device
    scalar) is 0 and is averaged with it otherwise; every ``copied`` tensor takes its ``copied_from`` partner's value; then
    ``n_averaged`` advances by one.  One launch per 48 pairs, no host synchronisation, graph-capturable."""
    _C.avg_multi(list(averaged), list(current), n_averaged, -1.0 if decay is None else float(decay), list(copied), list(copied_from))


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
