"""Whole-step CUDA graph: forward + loss + backward + bucket allreduce + optimizer update
captured once and replayed with a single ``cudaGraphLaunch``.  With ``fuse_optimizer=True`` (default)
and a single-bucket model on the NVLink backend, the bucket allreduce and the SGD update are one
kernel (``optim.SGD.fuse_with_ddp``).

Why this exists: one ConvNet step is a few µs of arithmetic behind 60-80 kernel launches in the
reference stack, so the step is launch/host bound.  The reference's DDP
cannot be graph-captured as a whole because its gradient reduction is a host-side NCCL call per
bucket; ours is a plain kernel launched from the autograd hook on the comm stream, so the reducer,
the per-step buffer sync and the fused optimizer all land inside the graph.

Cross-GPU safety of replay: the reduce kernels use monotonically increasing epoch counters kept
in *device* memory (not kernel arguments), so replaying the same graph on every rank advances all
ranks in lockstep.  The staged collectives double-buffer their peer-visible staging area and the
half they use is a *launch argument* (baked into the graph): if a step issues an odd number of
them, replaying one graph would use the same half twice in a row across the step boundary and a
fast rank could overwrite a slot a slow rank is still reading.  Two things prevent that: (a) a step
that also contains an independent barrier-synchronised collective (DDP's per-forward buffer
broadcast: every rank must have finished step k before anyone leaves the broadcast of step k+1) is
safe as is — this is the ConvNet/ResNet case; (b) otherwise the step is captured twice (the second
capture starts on the other half) and replays alternate between the two graphs, which reproduces
exactly the eager alternation.

Learning-rate schedules: with a native optimizer (``pdt.optim.SGD``, ``Adam``, ``AdamW``) every group's lr lives in a device scalar
that the captured kernels read, whatever the group's ``capturable`` says, and each replay first copies ``param_groups[i]['lr']``
into it (``sync_lr``), so a ``torch.optim.lr_scheduler`` stepped between replays takes effect on the next one.  The other
hyper-parameters are baked into the graph: a replay after one of them changed (``OneCycleLR(cycle_momentum=True)``) raises.

Gradient-norm clipping (``max_grad_norm``, as ``torch.nn.utils.clip_grad_norm_`` between backward and ``optimizer.step()``):
on one GPU, when the update rides on the last backward kernel, that kernel clips before it updates (still three launches);
otherwise the native clip runs between backward and ``step()`` inside the graph (two launches).  With clipping the optimizer
is not fused into the gradient reduction: the reducer averages, the step clips, then ``step()`` runs.  The averaged gradients
are bitwise identical on every rank and the norm is reproducible bit for bit, so every rank derives the same coefficient
without a collective.

Gradient accumulation (``accumulation_steps=k``): the step's inputs carry k micro-batches of b rows each (micro-batch i is rows
[i·b, (i+1)·b)); one captured step runs k forward/backward passes and one update on the summed gradient of ``loss / k`` (torch's
convention; BatchNorm uses per-micro-batch statistics and updates its running statistics k times).  On the reference ConvNet
whose ten gradients all come from the two fused backward kernels, with a criterion that returns the fused cross-entropy
unchanged, the forward kernel emits the gradient of ``loss / k``, the backward kernels of micro-batches 2..k add into the
gradients of micro-batch 1 (accumulate mode, ops.functional.accumulate_into) and the update — with the clipping — rides on the
last micro-batch's backward: 3k launches, no AccumulateGrad add, no separate optimizer or clip kernel.  Any other model,
criterion or configuration accumulates through autograd.  One GPU only for now: for a model whose gradients are reduced across
ranks the micro-batches 1..k−1 would have to skip the reduction (``no_sync``) inside the captured step.

Weight averaging (``averaged_model``, a ``pdt.optim.swa_utils.AveragedModel``): every replay ends with
``averaged_model.update_parameters(model)`` after the optimizer step, as a training loop calls it after ``optimizer.step()``;
with accumulation, once per replay, after the last micro-batch.  The native update (``ops.average_update``) is one more launch
inside the graph, on one GPU too: it reads and advances ``n_averaged`` on the device.  (An averaging rider of the last backward
kernel was measured slower than this launch: DESIGN.md §7.)  torch's own update reads ``n_averaged`` on the host and
cannot be captured, so an averaged model that would take it is refused.  The warm-up steps the constructor runs are not
averaged.
"""
from __future__ import annotations

from typing import Optional, Sequence

import contextlib
import os

import torch


class GraphedTrainStep:
    # private switch for comparisons (tools/accum_step_bench.py): False accumulates through autograd even where the fused backward
    # kernels could add in place
    _accumulate_in_kernel = True

    def __init__(self, model, criterion, optimizer, example_inputs: Sequence[torch.Tensor], warmup: int = 3,
                 zero_grad_set_to_none: bool = True, fuse_optimizer: bool = True, double_buffer_inputs: bool = True,
                 max_grad_norm: Optional[float] = None, norm_type: float = 2.0, accumulation_steps: int = 1, averaged_model=None):
        if not torch.cuda.is_available():
            raise RuntimeError("GraphedTrainStep needs CUDA")
        self.averaged_model = averaged_model
        self._averaged_source = getattr(model, "module", model)   # the averaged model was copied from the bare model
        if averaged_model is not None:
            plan = averaged_model.native_plan(self._averaged_source) if hasattr(averaged_model, "native_plan") else (
                "it is not a pdt.optim.swa_utils.AveragedModel")
            if isinstance(plan, str):
                raise ValueError(f"GraphedTrainStep(averaged_model=...): the averaged model has no native update ({plan}); torch's "
                                 "AveragedModel.update_parameters reads n_averaged on the host and cannot be captured in a CUDA graph")
        self._averaging = False   # True while a graph is captured: the warm-up steps are not averaged
        k = int(accumulation_steps)
        if k != accumulation_steps or k < 1:
            raise ValueError(f"accumulation_steps must be a positive integer, got {accumulation_steps}")
        if k > 1:
            rows = {int(t.shape[0]) for t in example_inputs}
            if len(rows) != 1 or next(iter(rows)) % k != 0:
                raise ValueError(f"accumulation_steps={k}: every input must have the same number of rows, a multiple of {k} "
                                 f"(got {sorted(rows)})")
            # a model that reduces its gradients across ranks (DistributedDataParallel) would need the reduction skipped on all but the
            # last micro-batch; an unwrapped model accumulates locally whatever the default group's size
            group_ = getattr(model, "process_group", None)
            if group_ is not None and group_.size() > 1:
                raise NotImplementedError("GraphedTrainStep(accumulation_steps > 1) runs on one GPU only: at world size >= 2 the "
                                          "micro-batches before the last would have to skip the gradient reduction (no_sync) inside "
                                          "the captured step")
        self.accumulation_steps = k
        # ``step`` of the last eager or captured step: whether micro-batches 2..k accumulated inside the fused backward kernels
        self.accumulates_in_kernel = False
        # whether the forward kernel may emit the cross-entropy already scaled by 1/k: decided by the first (unscaled) eager step, True
        # when the criterion returned the fused cross-entropy itself on every micro-batch (None: not decided yet)
        self._prescale: Optional[bool] = None
        self.model, self.criterion, self.optimizer = model, criterion, optimizer
        if hasattr(optimizer, "_lr_on_device"):
            # a native optimizer's kernels read every group's lr from a device scalar from the warm-up steps on, so that sync_lr()
            # before a replay carries a scheduler's change into the graph (a captured host lr would be replayed forever)
            optimizer._lr_on_device = True
        self.static_inputs = [t.clone() for t in example_inputs]
        # two input buffers, one captured graph each: the next batch's copy into the step's static inputs (host→device from pinned
        # memory, or device→device) runs on a copy stream while the current replay computes, instead of in front of it
        # (PDT_DOUBLE_BUFFER_INPUTS=0: one buffer, copies on the compute stream)
        self.double_buffer = bool(double_buffer_inputs) and os.environ.get("PDT_DOUBLE_BUFFER_INPUTS", "1") != "0"
        self.input_sets = [self.static_inputs] + ([[t.clone() for t in example_inputs]] if self.double_buffer else [])
        self.set_to_none = zero_grad_set_to_none
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.static_loss: Optional[torch.Tensor] = None
        self.replays = 0
        self._last = 0
        self._seed: Optional[torch.Tensor] = None   # d(loss)/d(loss) = 1, allocated once (autograd would fill a new one per step)
        self.fused_optimizer = False
        # gradient-norm clipping: the total norm of the last replay's gradients (a device scalar per captured graph, alternating
        # with them as static_loss does)
        if max_grad_norm is not None and not float(max_grad_norm) > 0:
            raise ValueError(f"max_grad_norm must be positive, got {max_grad_norm}")
        self.max_grad_norm = None if max_grad_norm is None else float(max_grad_norm)
        self.norm_type = float(norm_type)
        self.grad_norm: Optional[torch.Tensor] = None
        self._clip_params = [p for g in optimizer.param_groups for p in g["params"]]
        self._rider_norms = [torch.zeros((), device=self.static_inputs[0].device) for _ in range(2)] if self.max_grad_norm is not None else []
        self._riding = False
        if fuse_optimizer and self.max_grad_norm is None and hasattr(optimizer, "fuse_with_ddp") and hasattr(model, "enable_optimizer_fusion"):
            optimizer.fuse_with_ddp(model)
            warmup = max(warmup, 4)  # bucket rebuild after step 1, fusion switches on after step 2
        if fuse_optimizer and hasattr(optimizer, "ride_on_backward"):
            # one GPU: the update (and the clipping) rides on the model's last backward kernel (no-op when it cannot)
            self._riding = bool(self._ride(0))
        self._capture(warmup)
        self.fused_optimizer = bool(getattr(optimizer, "_fused_active", False))

    def _ride(self, k: int) -> bool:
        """(Re-)arm the riding update; with clipping, the rider stores the norm in the device scalar of graph k."""
        if self.max_grad_norm is None:
            return self.optimizer.ride_on_backward(self.model)
        self._rider_norm = self._rider_norms[k]
        return self.optimizer.ride_on_backward(self.model, clip=(self.max_grad_norm, self.norm_type, self._rider_norm))

    def _eager_step(self, inputs=None):
        inputs = self.static_inputs if inputs is None else inputs
        from ..ops import functional as OF

        if self.accumulation_steps > 1:
            return self._finish_step(self._accumulate(inputs))

        # the step owns the targets before the model runs: a model whose forward kernel can fold the loss in does so
        # (ops.functional.upcoming_targets); the criterion then finds value and gradient ready
        with OF.upcoming_targets(inputs[1] if len(inputs) == 2 else None, loss_read_after_backward=True,
                                 spec=OF.ce_spec_of(self.criterion)):
            out = self.model(inputs[0])
        loss = self.criterion(out, *inputs[1:])
        self.optimizer.zero_grad(set_to_none=self.set_to_none)
        with OF.sgd_rider_enabled():   # an optimizer armed with ride_on_backward may apply its update inside this backward pass
            loss.backward(self._unit_seed(loss))
        return self._finish_step(loss)

    def _unit_seed(self, loss):
        if self._seed is None or self._seed.shape != loss.shape or self._seed.dtype != loss.dtype:
            self._seed = torch.ones_like(loss)
            self._seed._pdt_unit_seed = True   # lets ops that pre-compute their unit-gradient backward skip the scaling kernel
        return self._seed

    def _accumulate(self, inputs):
        """Forward and backward of the k micro-batches; returns the mean of their losses.  Micro-batches 2..k add into the gradient
        buffers micro-batch 1 left — inside the fused backward kernels when micro-batch 1 showed that they wrote every gradient and
        the loss is the fused cross-entropy's (scaled by 1/k in the forward kernel, its mean folded by a backward kernel), through
        autograd's accumulation otherwise.  The riding update is enabled for the last micro-batch's backward only.

        The forward kernel scales the cross-entropy, and a backward kernel folds its mean, only for a criterion that returns it
        unchanged (pdt.nn.CrossEntropyLoss): a criterion that computes anything from it (``ce * w``, ``ce + reg``) would see — and
        scale once more — the scaled value, and would read the loss before backward has folded it.  The first eager step therefore
        runs unscaled with the mean folded by the forward kernel and backpropagates ``loss / k``; it records whether the criterion's
        result was the fused cross-entropy itself, and only then do later steps let the kernels scale and fold.  A criterion that
        changes its mind later is an error, not a silently doubled scale."""
        from ..ops import functional as OF

        k = self.accumulation_steps
        b = inputs[0].shape[0] // k
        scale = 1.0 / k
        grad_scale = scale if self._prescale else 1.0
        returns_ce = True
        params = [p for p in self.model.parameters() if p.requires_grad]
        self.optimizer.zero_grad(set_to_none=self.set_to_none)
        kept = None     # (gradient buffers of micro-batch 1, its loss buffer): the in-kernel accumulation's destinations
        total = None
        for i in range(k):
            micro = [t[i * b:(i + 1) * b] for t in inputs]
            OF.reset_fused_ce_consumed()
            with OF.upcoming_targets(micro[1] if len(micro) == 2 else None, loss_read_after_backward=bool(self._prescale),
                                     grad_scale=grad_scale, spec=OF.ce_spec_of(self.criterion)):
                out = self.model(micro[0])
            loss = self.criterion(out, *micro[1:])
            consumed = OF.fused_ce_consumed()
            # the criterion's result is the one fused cross-entropy of this forward, as cross_entropy returned it
            is_ce = (len(consumed) == 1 and consumed[0] == (id(loss), grad_scale)
                     and getattr(loss, "_pdt_loss_scale", None) == grad_scale)
            returns_ce = returns_ce and is_ce
            if grad_scale != 1.0 and not is_ce:
                raise RuntimeError("gradient accumulation: the forward kernel scaled the cross-entropy by 1/k because the criterion "
                                   "returned it unchanged in the first step, but this time the criterion computed something else from "
                                   "it; the scale would be applied twice")
            prescaled = grad_scale != 1.0
            fused_loss = prescaled and getattr(loss, "_pdt_loss_deferred", False)
            part = loss if prescaled else loss / k
            into = None
            if kept is not None and fused_loss:
                for p in params:
                    p.grad = None   # the kernels add into the kept buffers and hand them back as fresh gradients
                into = OF.accumulate_into(kept[0], kept[1])
            OF.reset_fused_backward_params()
            riding = OF.sgd_rider_enabled() if i == k - 1 else contextlib.nullcontext()
            with (into if into is not None else contextlib.nullcontext()), riding:
                part.backward(self._unit_seed(part))
            if into is not None:
                lost = into.leftover() + [p for p in kept[0] if p.grad is None]
                if lost:
                    raise RuntimeError(f"gradient accumulation: {len(lost)} gradient(s) of micro-batch {i + 1} were not added in the fused "
                                       "backward kernels")
                # the sums, where .grad holds them now (a DDP reducer that has just rebuilt its buckets copies them into the new ones)
                kept = ({p: p.grad for p in kept[0]}, kept[1])
            if i == 0:
                wrote = OF.fused_backward_params()
                grads = {p: p.grad for p in params if p.grad is not None}
                if (self._accumulate_in_kernel and fused_loss and wrote is not None and {id(p) for p in wrote if p is not None} == {id(p) for p in grads}
                        and all(g.is_contiguous() for g in grads.values())):
                    kept = (grads, part.detach())
            self.accumulates_in_kernel = kept is not None
            if into is None or total is None:
                total = part if total is None else total + part.detach()
        if self._prescale is None:
            self._prescale = returns_ce
        return total   # in-kernel: micro-batch 1's loss buffer, to which the later folds added

    def _finish_step(self, loss):
        """Clipping (unless the riding update did it) and the optimizer step after the backward pass(es)."""
        norm = None
        if self.max_grad_norm is not None:
            if getattr(self.optimizer, "_rode", False):
                norm = self._rider_norm   # the backward kernel clipped and updated
            else:
                from ..nn.utils import clip_grad_norm_

                norm = clip_grad_norm_(self._clip_params, self.max_grad_norm, self.norm_type)
        self.optimizer.step()
        if self._averaging:
            self.averaged_model.update_parameters(self._averaged_source)
        return loss, norm

    def _capture(self, warmup: int):
        dev = self.static_inputs[0].device
        from .. import _C

        side = torch.cuda.Stream(device=dev)
        self.capture_stream = side
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            # AccumulateGrad nodes run on the stream they were created on: give the reducer (which
            # pins them) a fresh start on the stream that will be captured
            if hasattr(self.model, "_reset_reducer"):
                self.model._reset_reducer()
            for _ in range(max(warmup, 2)):  # ≥2: the reducer rebuilds its buckets after iteration 1
                self._eager_step()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        comm = getattr(self.model, "comm", None)
        parity = (lambda: list(comm.parity_state())) if hasattr(comm, "parity_state") else (lambda: [])
        self.graphs, self.losses, self.norms = [], [], []
        p0 = parity()
        for k in range(2):
            if self._riding and self.max_grad_norm is not None:
                self._ride(k)   # each graph's rider stores the norm in its own scalar
            g = torch.cuda.CUDAGraph()
            before = _C.kernel_launch_count()
            self._averaging = self.averaged_model is not None
            with torch.cuda.graph(g, stream=side):
                loss, norm = self._eager_step(self.input_sets[k % len(self.input_sets)])
            self._averaging = False
            # how many of *our* kernels one replay runs (ATen glue kernels are not counted)
            self.kernels_per_replay = int(_C.kernel_launch_count() - before)
            self.graphs.append(g)
            self.losses.append(loss)
            self.norms.append(norm)
            torch.cuda.synchronize(dev)
            ordered = getattr(self.model, "syncs_buffers_every_step", None)
            if not self.double_buffer and (parity() == p0 or (ordered is not None and ordered())):
                break  # even number of staged collectives per step, or case (a): one graph replays safely
        self.graph, self.static_loss = self.graphs[0], self.losses[0]
        self.grad_norm = None
        if hasattr(self.optimizer, "_record_captured_hyper"):
            self.optimizer._record_captured_hyper()   # sync_lr() refuses a replay once any of them has changed
        # the host side of a replay (input staging on a copy stream, ordering against the replays that use the buffers, losses to pinned
        # memory on a side stream) is native: csrc/engine/step_pipeline.cpp
        self._io = _C.StepPipeline(dev.index if dev.index is not None else torch.cuda.current_device(), len(self.graphs), self.static_loss)

    def __call__(self, *inputs: torch.Tensor, inputs_ready: bool = False) -> torch.Tensor:
        """One training step on ``inputs`` (pinned host tensors or device tensors).  ``inputs_ready=True``: the caller guarantees
        that device-resident inputs are complete already (a GPU-resident dataset, a batch produced on another stream and
        synchronised) — their copy into the step's buffers then overlaps the previous step instead of queueing behind it."""
        if hasattr(self.optimizer, "sync_lr"):
            # scheduler changes of lr reach the captured step through a device scalar; a change of any other hyper-parameter is
            # refused here, before anything of this step is enqueued
            self.optimizer.sync_lr()
        i = self.replays % len(self.graphs)
        self._io.stage_inputs(i, self.input_sets[i % len(self.input_sets)], list(inputs), inputs_ready, self.double_buffer)
        self.graphs[i].replay()
        self._io.replayed(i)
        self.replays += 1
        self._last = i
        self.static_loss = self.losses[i]
        self.grad_norm = self.norms[i]
        return self.static_loss

    def loss_to_host(self) -> "HostLoss":
        """Start an asynchronous device→host copy of the last step's loss on a side stream (pinned ring of 16 slots) and return a
        handle; ``handle.item()`` blocks until that copy has landed.  Nothing is queued on the compute stream, so the next
        replay is not held up by the copy — call it every step and read the handles you want to log whenever convenient
        (reading a handle *after* the next step has been enqueued keeps the device busy while the host waits)."""
        return HostLoss(self._io, self._io.loss_to_host(self._last, self.static_loss))


class HostLoss:
    """Handle of one loss value on its way to pinned host memory (``GraphedTrainStep.loss_to_host``); valid for 15 further steps."""

    __slots__ = ("_io", "_gen", "_value")

    def __init__(self, io, gen):
        self._io, self._gen, self._value = io, gen, None

    def item(self) -> float:
        if self._value is None:
            self._value = float(self._io.loss_value(self._gen))
        return self._value
