"""SGD with one fused multi-tensor kernel per step.

The reference uses ``torch.optim.SGD(model.parameters(), 1e-4)`` (ref: ddp_example.py:62,90,92),
i.e. ``p -= lr·g`` through a foreach kernel, with ``zero_grad()`` dropping the gradients so
autograd re-allocates them every backward.  Ours:

* the update for *all* parameters is one sm_90a kernel launch (``ops.sgd_step``) over a pointer
  table — momentum, dampening, Nesterov and weight decay included — so it is graph-capturable
  and launch-count-free as the model grows;
* ``lr`` lives in a device scalar when ``capturable=True``, and always once ``engine.GraphedTrainStep`` has taken the optimizer,
  so schedulers work under CUDA graphs (the other hyper-parameters must not change between replays: ``sync_lr``);
* ``zero_grad(set_to_none=False)`` keeps gradients as views of the DDP bucket (no re-allocation,
  no copy into the bucket next step). ``set_to_none=True`` (the reference's default behaviour)
  still works — the reducer re-homes gradients on the next backward.

Bookkeeping (param_groups / state_dict) comes from ``torch.optim.Optimizer``; the device-resident learning rate and the
riding checks are shared with ``Adam`` (``_riding.RidingOptimizer``).
"""
from __future__ import annotations

from typing import Iterable, Optional

import torch

from ._riding import RidingOptimizer


class SGD(RidingOptimizer):
    def __init__(self, params: Iterable, lr: float = 1e-3, momentum: float = 0.0, dampening: float = 0.0,
                 weight_decay: float = 0.0, nesterov: bool = False, maximize: bool = False,
                 capturable: bool = False, fused: Optional[bool] = None):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay,
                        nesterov=nesterov, maximize=maximize, capturable=capturable, fused=fused)
        super().__init__(params, defaults)
        self._ddp = None            # set by fuse_with_ddp()
        self._fused_active = False
        self._flat_momentum = None

    # ---- single GPU: the update rides on the model's last backward kernel ---------------------------------
    def ride_on_backward(self, model, clip=None) -> bool:
        """Let the reference ConvNet's last backward kernel apply this optimizer's update (csrc/cuda/fused_convnet.cu: SgdRider): the
        thread that writes a folded gradient element updates the parameter with the value still in its register; the parameters whose
        gradients are complete earlier are updated in the shadow of that kernel's first grid barrier.  ``step()`` then has only
        bookkeeping left.  Used by ``engine.GraphedTrainStep`` when the gradient reduction does not already carry the update (one GPU).

        ``clip = (max_norm, norm_type, norm_out)``: the kernel clips the gradient norm first, as ``clip_grad_norm_`` would
        (ClipRider: one more grid barrier, then every gradient is scaled and updated in one pass; ``.grad`` reads the clipped
        gradient and ``norm_out``, one fp32 element on the device, the total norm).  ``norm_type`` must be 2 or inf.

        Same contract as :meth:`fuse_with_ddp`: between ``backward()`` and ``step()`` the parameters are already updated.  Returns
        False (and changes nothing) when the model / optimizer combination does not qualify."""
        params = self._qualify_rider(model)
        if params is None or (clip is not None and not self._clip_qualifies(clip, params)):
            return False

        def build(prev_grads):
            if getattr(self, "_fused_active", False):   # the reduce kernels carry the update (N >= 2)
                return None
            g = self.param_groups[0]
            bufs = []
            first = False
            if g["momentum"] != 0:
                states = [self.state[q] for q in params]
                have = [st.get("momentum_buffer") is not None for st in states]
                if any(have) and not all(have):
                    return None   # mixed first-step state: leave this iteration to step()
                first = not any(have)
                for q, st in zip(params, states):
                    if st.get("momentum_buffer") is None:
                        st["momentum_buffer"] = torch.zeros_like(q, memory_format=torch.contiguous_format)
                    bufs.append(st["momentum_buffer"])
            return dict(kind="sgd", params=params, prev_grads=list(prev_grads), momentum_buffer=bufs, first_step=first,
                        **self._hyper(0, g, params[0].device))

        self._arm_rider(params, build, clip)
        return True

    _FIXED_KEYS = ("momentum", "dampening", "weight_decay", "nesterov", "maximize")

    def _hyper(self, gi: int, group, device) -> dict:
        """The update's hyper-parameters, as ``ops.sgd_step`` and the rider description of the last backward kernel take them
        (``lr`` and the group keys ``_FIXED_KEYS``)."""
        return dict(lr=float(group["lr"]), lr_tensor=self._lr_tensor(gi, group, device), momentum=float(group["momentum"]),
                    dampening=float(group["dampening"]), weight_decay=float(group["weight_decay"]), nesterov=bool(group["nesterov"]),
                    maximize=bool(group["maximize"]))

    # ---- DDP fusion: the update rides on the gradient reduction ----------------------------------------
    def fuse_with_ddp(self, ddp) -> "SGD":
        """Fuse this optimizer into DDP's gradient reduction.

        The reference's step is ``backward`` (→ NCCL allreduce of the bucket, launched after the last gradient)
        followed by a foreach SGD kernel (ddp_example.py:89-92).  Fused, every *reduce chunk* the reducer launches
        from the autograd hook — a contiguous piece of the bucket in grad-ready order — is ONE kernel on the comm
        stream that pushes the chunk into the peers' staging slots, crosses one device-side barrier, folds the
        ``world`` slots in rank order and applies the SGD update to the parameters the chunk belongs to
        (``Comm.allreduce_sgd``), so the reduction *and* the update of the late layers overlap the backward pass
        of the early ones.  The last chunk also carries DDP's per-step BatchNorm-buffer broadcast.
        ``step()`` then only has bookkeeping left; ``.grad`` reads as the averaged gradient, as in the reference.

        Contract: between ``backward()`` and ``step()`` the parameters are already updated — a clip call of the user's own
        there sees an already-updated model, and a skipped ``step()`` is not expressible in this mode.  Clipping is expressible
        through ``engine.GraphedTrainStep(max_grad_norm=…)``, which does not fuse the optimizer into the reduction then.  Takes
        effect on the first ``step()`` after the reducer has settled its bucket layout; until then (and whenever the
        preconditions fail) the ordinary path runs.

        The update of a backward uses the hyper-parameters in ``param_groups`` when DDP's forward starts: a scheduler stepped
        (or a value set) before the forward takes effect in that iteration, as on the unfused path; a change made between the
        forward and ``backward()`` is not picked up until the next forward."""
        self._ddp = ddp
        return self

    def _maybe_activate_fusion(self) -> None:
        ddp = self._ddp
        if self._fused_active or ddp is None or len(self.param_groups) != 1:
            return
        group = self.param_groups[0]
        if group["maximize"] or ddp.process_group.size() == 1:
            return
        mine = [p for p in group["params"]]
        if len(mine) != len(ddp._params) or {id(p) for p in mine} != {id(p) for p in ddp._params}:
            return
        if any(p.dtype != torch.float32 for p in mine):
            return
        if group["momentum"] != 0:
            missing = [self.state[p].get("momentum_buffer") is None for p in ddp._params]
            if any(missing) and not all(missing) and group["dampening"] != 0:
                return  # "first step" is a per-parameter rule; wait until every parameter has its buffer
        if not ddp.enable_optimizer_fusion():
            return
        if group["momentum"] != 0:
            flat = torch.zeros_like(ddp.param_arena)
            for p, off in zip(ddp._params, ddp._param_offsets):
                view = flat[off:off + p.numel()].view(p.shape)
                st = self.state[p]
                if st.get("momentum_buffer") is not None:
                    view.copy_(st["momentum_buffer"])
                    st["momentum_buffer"] = view
            self._flat_momentum = flat
        self._fused_active = True
        ddp._rearm_fused_optimizer = self._arm_fused
        self._arm_fused()

    def _arm_fused(self, changed_only: bool = False) -> None:
        """(Re-)install the update the reducer applies with every reduce chunk of the *next* backward.  DDP calls this when its
        forward starts with ``changed_only=True``: the reducer is re-armed only when a hyper-parameter or the first-step flag
        differs from what it holds (a device-resident lr is refreshed here either way)."""
        ddp, group = self._ddp, self.param_groups[0]
        first = False
        if group["momentum"] != 0:
            # zero buffer + "not first" is exact when dampening == 0 (b = μ·0 + g); a uniform first step sets the flag
            first = all(self.state[p].get("momentum_buffer") is None for p in ddp._params)
        h = self._hyper(0, group, ddp.param_arena.device)
        armed = (h["lr"], h["lr_tensor"] is not None, h["momentum"], h["dampening"], h["weight_decay"], h["nesterov"], first)
        if changed_only and armed == self._armed:
            return
        self._armed = armed
        ddp.reducer.set_fused_sgd(ddp.param_arena, self._flat_momentum, lr=h["lr"], lr_tensor=h["lr_tensor"], momentum=h["momentum"],
                                  dampening=h["dampening"], weight_decay=h["weight_decay"], nesterov=h["nesterov"], first_step=first,
                                  bcast=ddp.tail_broadcast_buffer(), bcast_root=0)

    def _fused_step(self) -> bool:
        ddp = self._ddp
        if not (self._fused_active and ddp.reducer.fused_sgd):
            return False
        if not ddp.require_backward_grad_sync:
            return True   # no_sync(): gradients accumulate locally; the next synchronised backward reduces and applies them
        group = self.param_groups[0]
        # the reduction of this iteration's backward has already applied the update (see fuse_with_ddp)
        if group["momentum"] != 0:
            for p, off in zip(ddp._params, ddp._param_offsets):
                if self.state[p].get("momentum_buffer") is None:
                    self.state[p]["momentum_buffer"] = self._flat_momentum[off:off + p.numel()].view(p.shape)
        # the first-step flag drops, and changed hyper-parameters are picked up, when DDP's next forward starts (_arm_fused)
        return True

    def load_state_dict(self, state_dict) -> None:
        """Standard behaviour, plus: when the step is fused with DDP the momentum lives in ONE flat buffer that
        mirrors the bucket — restored values are copied into it instead of replacing its views."""
        super().load_state_dict(state_dict)
        if self._flat_momentum is not None and self._ddp is not None:
            for p, off in zip(self._ddp._params, self._ddp._param_offsets):
                st = self.state.get(p)
                if st is None or st.get("momentum_buffer") is None:
                    continue
                view = self._flat_momentum[off:off + p.numel()].view(p.shape)
                if st["momentum_buffer"].data_ptr() != view.data_ptr():
                    view.copy_(st["momentum_buffer"])
                    st["momentum_buffer"] = view

    def zero_grad(self, set_to_none: bool = True) -> None:
        if set_to_none:
            return super().zero_grad(set_to_none=True)
        grads = [p.grad for g in self.param_groups for p in g["params"] if p.grad is not None]
        if grads:
            torch._foreach_zero_(grads)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        from .. import ops

        if getattr(self, "_rode", False):
            self._rode = False   # the last backward kernel applied this step's update (ride_on_backward)
            return loss
        if self._ddp is not None:
            if self._fused_step():
                return loss
            self._maybe_activate_fusion()  # takes effect from the next backward on
        for gi, group in enumerate(self.param_groups):
            params, grads, bufs = [], [], []
            momentum = group["momentum"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("SGD does not support sparse gradients")
                params.append(p)
                grads.append(p.grad)
                if momentum != 0:
                    st = self.state[p]
                    if "momentum_buffer" not in st:
                        st["momentum_buffer"] = None
                    bufs.append(st)
            if not params:
                continue
            use_fused = group["fused"]
            if use_fused is None:
                use_fused = params[0].is_cuda and ops.native_available() and all(
                    p.dtype == torch.float32 and p.is_contiguous() and g.is_contiguous() and g.dtype == torch.float32
                    for p, g in zip(params, grads))
            if use_fused:
                if momentum == 0:
                    ops.sgd_step(params, grads, None, first_step=False, **self._hyper(gi, group, params[0].device))
                    continue
                # "first step" (buf = g, no dampening) is a per-parameter decision, as in torch: parameters that see
                # their first gradient now go through one launch with first_step=True, the rest through another
                fresh = [st["momentum_buffer"] is None for st in bufs]   # decided before any buffer is created below
                for want_first in (True, False):
                    sel = [i for i, f in enumerate(fresh) if f == want_first]
                    if not sel:
                        continue
                    ps, gs_ = [params[i] for i in sel], [grads[i] for i in sel]
                    if want_first:
                        for i in sel:
                            bufs[i]["momentum_buffer"] = torch.zeros_like(params[i], memory_format=torch.contiguous_format)
                    ops.sgd_step(ps, gs_, [bufs[i]["momentum_buffer"] for i in sel], first_step=want_first,
                                 **self._hyper(gi, group, params[0].device))
                continue
            # reference math through foreach ops (CPU / exotic dtypes)
            gs = [(-g if group["maximize"] else g) for g in grads] if group["maximize"] else list(grads)
            if group["weight_decay"] != 0:
                gs = torch._foreach_add(gs, params, alpha=group["weight_decay"])
            if momentum != 0:
                new = []
                for st, g in zip(bufs, gs):
                    if st["momentum_buffer"] is None:
                        st["momentum_buffer"] = torch.clone(g).detach()
                    else:
                        st["momentum_buffer"].mul_(momentum).add_(g, alpha=1 - group["dampening"])
                    new.append(st["momentum_buffer"])
                gs = torch._foreach_add(gs, new, alpha=momentum) if group["nesterov"] else new
            torch._foreach_add_(params, gs, alpha=-group["lr"])
        return loss
