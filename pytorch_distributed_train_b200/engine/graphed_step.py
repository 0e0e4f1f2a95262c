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

Gradient-norm clipping (``max_grad_norm``, as ``torch.nn.utils.clip_grad_norm_`` between backward and ``optimizer.step()``):
on one GPU, when the update rides on the last backward kernel, that kernel clips before it updates (still three launches);
otherwise the native clip runs between backward and ``step()`` inside the graph (two launches).  With clipping the optimizer
is not fused into the gradient reduction: the reducer averages, the step clips, then ``step()`` runs.  The averaged gradients
are bitwise identical on every rank and the norm is reproducible bit for bit, so every rank derives the same coefficient
without a collective.
"""
from __future__ import annotations

from typing import Optional, Sequence

import os

import torch


class GraphedTrainStep:
    def __init__(self, model, criterion, optimizer, example_inputs: Sequence[torch.Tensor], warmup: int = 3,
                 zero_grad_set_to_none: bool = True, fuse_optimizer: bool = True, double_buffer_inputs: bool = True,
                 max_grad_norm: Optional[float] = None, norm_type: float = 2.0):
        if not torch.cuda.is_available():
            raise RuntimeError("GraphedTrainStep needs CUDA")
        self.model, self.criterion, self.optimizer = model, criterion, optimizer
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
        return self.optimizer.ride_on_backward(self.model, clip=(self.max_grad_norm, self.norm_type, self._rider_norms[k]))

    def _eager_step(self, inputs=None):
        inputs = self.static_inputs if inputs is None else inputs
        from ..ops import functional as OF

        # the step owns the targets before the model runs: a model whose forward kernel can fold the loss in does so
        # (ops.functional.upcoming_targets); the criterion then finds value and gradient ready
        with OF.upcoming_targets(inputs[1] if len(inputs) == 2 else None, loss_read_after_backward=True):
            out = self.model(inputs[0])
        loss = self.criterion(out, *inputs[1:])
        self.optimizer.zero_grad(set_to_none=self.set_to_none)
        if self._seed is None or self._seed.shape != loss.shape or self._seed.dtype != loss.dtype:
            self._seed = torch.ones_like(loss)
            self._seed._pdt_unit_seed = True   # lets ops that pre-compute their unit-gradient backward skip the scaling kernel
        with OF.sgd_rider_enabled():   # an optimizer armed with ride_on_backward may apply its update inside this backward pass
            loss.backward(self._seed)
        norm = None
        if self.max_grad_norm is not None:
            if getattr(self.optimizer, "_rode", False):
                norm = OF._sgd_rider["clip"][2]   # the backward kernel clipped and updated
            else:
                from ..nn.utils import clip_grad_norm_

                norm = clip_grad_norm_(self._clip_params, self.max_grad_norm, self.norm_type)
        self.optimizer.step()
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
            with torch.cuda.graph(g, stream=side):
                loss, norm = self._eager_step(self.input_sets[k % len(self.input_sets)])
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
        # the host side of a replay (input staging on a copy stream, ordering against the replays that use the buffers, losses to pinned
        # memory on a side stream) is native: csrc/engine/step_pipeline.cpp
        self._io = _C.StepPipeline(dev.index if dev.index is not None else torch.cuda.current_device(), len(self.graphs), self.static_loss)

    def __call__(self, *inputs: torch.Tensor, inputs_ready: bool = False) -> torch.Tensor:
        """One training step on ``inputs`` (pinned host tensors or device tensors).  ``inputs_ready=True``: the caller guarantees
        that device-resident inputs are complete already (a GPU-resident dataset, a batch produced on another stream and
        synchronised) — their copy into the step's buffers then overlaps the previous step instead of queueing behind it."""
        i = self.replays % len(self.graphs)
        self._io.stage_inputs(i, self.input_sets[i % len(self.input_sets)], list(inputs), inputs_ready, self.double_buffer)
        if hasattr(self.optimizer, "sync_lr"):
            self.optimizer.sync_lr()  # scheduler changes reach the captured step through a device scalar
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
