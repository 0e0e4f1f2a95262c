"""DistributedDataParallel — the data-parallel strategy of the framework.

Drop-in for the call the reference makes, ``nn.parallel.DistributedDataParallel(model,
device_ids=[gpu])`` (ref: ddp_example.py:64; behaviour per torch/nn/parallel/distributed.py
:655-972 ctor, :1553-1691 forward, c10d reducer.hpp).  Same observable contract:

* an ``nn.Module`` that stores the wrapped network as ``self.module`` (state_dict keys gain the
  ``module.`` prefix), forward passthrough;
* construction verifies parameter shapes across ranks and broadcasts rank 0's parameters and
  buffers to everyone;
* gradients are **averaged** over the group, bucket by bucket, overlapped with backward;
* module buffers (BatchNorm running stats) follow rank 0 before every training forward;
* ``no_sync()``, ``register_comm_hook``, ``join()``, ``find_unused_parameters``, ``static_graph``,
  ``gradient_as_bucket_view``, ``bucket_cap_mb``, ``broadcast_buffers`` are supported.

What is different (H100-first):

* the reducer is our own C++ (``_C.Reducer``); gradients live inside the bucket
  (``gradient_as_bucket_view=True`` by default) and on the NVLink backend the bucket is peer-mapped
  symmetric memory that the fused allreduce kernel reads from every GPU directly — no flatten
  copies, no per-parameter ``1/N`` kernels, no NCCL call;
* parameters and buffers can be re-homed into flat symmetric arenas (``flatten_parameters``) so the
  init broadcast and the per-step buffer sync are one kernel each and the optimizer can run as a
  single fused kernel. ``Parameter`` objects are never replaced, so an optimizer built *before*
  wrapping (as the reference does, ref: ddp_example.py:62-64) keeps working.
"""
from __future__ import annotations

import sys
import time
from contextlib import contextmanager
from typing import Callable, List, Optional

import torch
import torch.nn as nn

from .. import _C
from .. import distributed as dist
from ..ops.functional import begin_iteration as _begin_iteration

_DEFAULT_FIRST_BUCKET_BYTES = 1024 * 1024
_BROADCAST_BUCKET_BYTES = 250 * 1024 * 1024


def _group_key(t: torch.Tensor) -> int:
    dev = 0 if t.device.index is None else t.device.index + 1
    return (hash(str(t.dtype)) & 0xFFFF) << 20 | (1 if t.is_cuda else 0) << 12 | dev


def _to_device(obj, device, non_blocking=True):
    if isinstance(obj, torch.Tensor):
        return obj.to(device, non_blocking=non_blocking) if obj.device != device else obj
    if isinstance(obj, tuple) and hasattr(obj, "_fields"):
        return type(obj)(*(_to_device(o, device) for o in obj))
    if isinstance(obj, (tuple, list)):
        return type(obj)(_to_device(o, device) for o in obj)
    if isinstance(obj, dict):
        return {k: _to_device(v, device) for k, v in obj.items()}
    return obj


def _flatten_outputs(out) -> List[torch.Tensor]:
    if isinstance(out, torch.Tensor):
        return [out]
    if isinstance(out, (tuple, list)):
        r = []
        for o in out:
            r += _flatten_outputs(o)
        return r
    if isinstance(out, dict):
        r = []
        for o in out.values():
            r += _flatten_outputs(o)
        return r
    return []


def broadcast_coalesced(comm, tensors: List[torch.Tensor], src: int = 0,
                        buffer_size: int = _BROADCAST_BUCKET_BYTES) -> None:
    """Broadcast many tensors from ``src`` in few collectives: group by dtype, pack chunks of at
    most ``buffer_size`` bytes, broadcast, unpack in place (contract: c10d comm.hpp:13-17)."""
    by_dtype = {}
    for t in tensors:
        by_dtype.setdefault((t.dtype, t.device), []).append(t)
    for (_dtype, _dev), group in by_dtype.items():
        chunk, nbytes = [], 0
        chunks = []
        for t in group:
            sz = t.numel() * t.element_size()
            if chunk and nbytes + sz > buffer_size:
                chunks.append(chunk)
                chunk, nbytes = [], 0
            chunk.append(t)
            nbytes += sz
        if chunk:
            chunks.append(chunk)
        for chunk in chunks:
            if len(chunk) == 1 and chunk[0].is_contiguous():
                comm.broadcast(chunk[0].detach(), src).wait()
                continue
            flat = torch.cat([t.detach().reshape(-1) for t in chunk])
            comm.broadcast(flat, src).wait()
            if comm.rank != src:
                off = 0
                for t in chunk:
                    n = t.numel()
                    t.detach().copy_(flat[off:off + n].view_as(t))
                    off += n


class DistributedDataParallel(nn.Module):
    def __init__(self, module: nn.Module, device_ids=None, output_device=None, dim: int = 0,
                 broadcast_buffers: bool = True, init_sync: bool = True, process_group=None,
                 bucket_cap_mb: Optional[float] = None, find_unused_parameters: bool = False,
                 check_reduction: bool = False, gradient_as_bucket_view: bool = True,
                 static_graph: bool = False, first_bucket_cap_mb: Optional[float] = None,
                 flatten_parameters: Optional[bool] = None):
        super().__init__()
        if not dist.is_initialized() and process_group is None:
            raise RuntimeError("Default process group has not been initialized, please make sure to call init_process_group.")
        self.process_group = process_group or dist.get_default_group()
        self.comm = self.process_group.comm
        self.module = module
        self.dim = dim
        self.broadcast_buffers = broadcast_buffers
        self.find_unused_parameters = find_unused_parameters
        self.static_graph = static_graph
        self.gradient_as_bucket_view = gradient_as_bucket_view
        self.require_backward_grad_sync = True
        self.require_forward_param_sync = True
        self._join_active = False
        self._comm_hook_registered = False

        params_all = list(module.parameters())
        if not any(p.requires_grad for p in params_all):
            raise RuntimeError("DistributedDataParallel is not needed when a module doesn't have any parameter that requires a gradient.")
        devices = {p.device for p in params_all}
        if len(devices) != 1:
            raise ValueError(f"DistributedDataParallel requires all parameters on one device, found {sorted(map(str, devices))}")
        self.device = next(iter(devices))
        if device_ids is not None:
            if len(device_ids) != 1:
                raise ValueError("device_ids must hold exactly one device (one process per GPU)")
            d = device_ids[0]
            d = torch.device("cuda", d) if isinstance(d, int) else torch.device(d)
            if d.type == "cuda" and self.device.type == "cuda" and d.index is not None and d.index != self.device.index:
                raise ValueError(f"device_ids={device_ids} but the module lives on {self.device}")
        self.device_ids = [self.device.index] if self.device.type == "cuda" else None
        self.output_device = output_device if output_device is not None else (self.device_ids[0] if self.device_ids else None)
        if self.comm.is_cuda != (self.device.type == "cuda"):
            raise ValueError(f"process group backend {self.process_group.backend!r} cannot reduce gradients living on {self.device}")

        # parameters that take part in reduction, deduplicated, in registration order
        seen = set()
        self._param_names: List[str] = []
        self._params: List[nn.Parameter] = []
        for name, p in module.named_parameters():
            if p.requires_grad and id(p) not in seen:
                seen.add(id(p))
                self._params.append(p)
                self._param_names.append(name)
        self._buffers_to_sync = [b for b in module.buffers()]
        self._has_sync_bn = any(type(m).__name__ == "SyncBatchNorm" for m in module.modules())
        # (torch refuses SyncBatchNorm on CPU modules, distributed.py:2259-2266; ours runs on both)

        self.bucket_bytes_cap = int((25 if bucket_cap_mb is None else bucket_cap_mb) * 1024 * 1024)
        self.first_bucket_bytes_cap = int(_DEFAULT_FIRST_BUCKET_BYTES if first_bucket_cap_mb is None
                                          else first_bucket_cap_mb * 1024 * 1024)
        self._custom_caps = bucket_cap_mb is not None or first_bucket_cap_mb is not None

        self._verify_params_across_processes()
        if flatten_parameters is None:
            flatten_parameters = self.device.type == "cuda" and getattr(self.process_group, "comm_kind", "") == "nvlink"
        self.param_arena = None
        self.buffer_arenas = {}
        self.buffer_arena = None
        if flatten_parameters:
            self._flatten_into_arenas()
        if init_sync:
            self._sync_module_states()
        self._build_reducer()
        self._construction_time = time.time()

    # ---- construction helpers ----------------------------------------------------------------
    def _verify_params_across_processes(self):
        """All ranks must wrap the same architecture (c10d reducer.hpp:602-605). Mismatch raises
        on *every* rank with the offending parameter named."""
        g = self.process_group
        if g.size() == 1:
            return
        sig = [(n, tuple(p.shape), str(p.dtype)) for n, p in zip(self._param_names, self._params)]
        all_sigs = dist.all_gather_object(sig, g)
        ref = all_sigs[0]
        for r, s in enumerate(all_sigs):
            if len(s) != len(ref):
                raise RuntimeError(f"DDP expects same model across all ranks, but rank {r} has {len(s)} params, "
                                   f"while rank 0 has {len(ref)} params.")
            for a, b in zip(ref, s):
                if a[1:] != b[1:]:
                    raise RuntimeError(f"[rank{g.rank()}] params not equal across ranks: rank 0 has {a[0]} "
                                       f"{a[1]} {a[2]} but rank {r} has {b[0]} {b[1]} {b[2]}")

    def _flatten_into_arenas(self):
        """Re-home parameters (and buffers, per dtype) into flat arenas from the backend allocator.
        ``p.data`` is swapped for a view; the Parameter objects and their values are preserved."""
        align = 4
        by_dtype = {}
        for p in self._params:
            by_dtype.setdefault(p.dtype, []).append(p)
        if len(by_dtype) == 1:
            (dtype, ps), = by_dtype.items()
            total, offs = 0, []
            for p in ps:
                total = (total + align - 1) // align * align
                offs.append(total)
                total += p.numel()
            total = (total + align - 1) // align * align
            arena = self.comm.alloc_flat(total, dtype, self.device)
            with torch.no_grad():
                for p, off in zip(ps, offs):
                    view = arena[off:off + p.numel()].view(p.shape)
                    view.copy_(p.data)
                    p.data = view
            self.param_arena = arena
            self._param_offsets = offs
        # buffers of every dtype share ONE byte arena, so the per-step buffer sync is one broadcast kernel
        bufs = {}
        for b in self._buffers_to_sync:
            bufs.setdefault(b.dtype, []).append(b)
        regions, total_bytes = [], 0
        for dtype, bs in bufs.items():
            esize = max(1, bs[0].element_size())
            a = max(1, 16 // esize)
            total, offs = 0, []
            for b in bs:
                total = (total + a - 1) // a * a
                offs.append(total)
                total += b.numel()
            total = (total + a - 1) // a * a
            regions.append((dtype, bs, offs, total_bytes, total))
            total_bytes += total * esize
        if total_bytes:
            self.buffer_arena = self.comm.alloc_flat(total_bytes, torch.uint8, self.device)
            with torch.no_grad():
                for dtype, bs, offs, start, total in regions:
                    region = self.buffer_arena[start:start + total * bs[0].element_size()].view(dtype)
                    for b, off in zip(bs, offs):
                        view = region[off:off + b.numel()].view(b.shape)
                        view.copy_(b.data)
                        b.data = view
                    self.buffer_arenas[dtype] = region

    def enable_optimizer_fusion(self) -> bool:
        """Prepare for an optimizer fused into the gradient reduction (``optim.SGD.fuse_with_ddp``): once the
        reducer has settled on a single bucket, re-home the parameters into an arena that mirrors the bucket
        element for element, so that every reduce chunk launched from the autograd hook can also apply the update
        to "its" parameters (``Reducer.set_fused_sgd``).  Returns False (and changes nothing) when the
        preconditions do not hold."""
        if getattr(self, "_fused_optimizer", False):
            return True
        st = self.reducer.stats()
        if (not st["has_rebuilt_buckets"] or len(st["bucket_indices"]) != 1 or self._comm_hook_registered
                or self.find_unused_parameters or not self.gradient_as_bucket_view or self._join_active):
            return False
        flat = self.reducer.bucket_buffers()[0]
        views = self.reducer.grad_views()
        if flat.dtype != torch.float32 or any(not v.is_contiguous() for v in views):
            return False
        offs = [(v.data_ptr() - flat.data_ptr()) // 4 for v in views]
        arena = self.comm.alloc_flat(flat.numel(), torch.float32, self.device)
        with torch.no_grad():
            arena.zero_()
            for p, off in zip(self._params, offs):
                view = arena[off:off + p.numel()].view(p.shape)
                view.copy_(p.data)
                p.data = view
        self.param_arena, self._param_offsets = arena, offs
        self._fused_optimizer = True
        # the last reduce chunk of every step carries rank 0's module buffers to everybody (C4 riding on C5): the
        # separate barrier-synchronised broadcast kernel in front of every forward is no longer needed
        self._tail_broadcast = bool(self.broadcast_buffers and self.buffer_arena is not None and self.process_group.size() > 1)
        return True

    def tail_broadcast_buffer(self):
        """The byte arena the fused last chunk broadcasts from rank 0 (None: buffers are synced before forward)."""
        return self.buffer_arena if getattr(self, "_tail_broadcast", False) else None

    def _sync_module_states(self):
        if self.process_group.size() == 1:
            return
        if self.param_arena is not None:
            self.comm.broadcast(self.param_arena, 0).wait()
            rest = [p for p in self.module.parameters() if not p.requires_grad]
            if rest:
                broadcast_coalesced(self.comm, rest, 0)
        else:
            broadcast_coalesced(self.comm, [p for p in self.module.parameters()], 0)
        self._sync_buffers()

    def syncs_buffers_every_step(self) -> bool:
        """True when every training forward runs a barrier-synchronised buffer broadcast (C4) — which
        also orders consecutive steps across ranks (engine.GraphedTrainStep relies on it)."""
        if self._buffers_ride_on_reduce():
            return False
        return bool(self.broadcast_buffers and self._buffers_to_sync and self.process_group.size() > 1)

    def _buffers_ride_on_reduce(self) -> bool:
        return bool(getattr(self, "_tail_broadcast", False) and self.reducer.fused_sgd and self.require_backward_grad_sync)

    def _sync_buffers(self):
        if not self._buffers_to_sync or self.process_group.size() == 1:
            return
        if self.buffer_arena is not None:
            if hasattr(self.comm, "broadcast_inline"):
                self.comm.broadcast_inline(self.buffer_arena, 0)  # our kernel, on the compute stream
            else:
                self.comm.broadcast(self.buffer_arena, 0).wait()
        else:
            broadcast_coalesced(self.comm, self._buffers_to_sync, 0)

    def _build_reducer(self):
        nbytes = [p.numel() * p.element_size() for p in self._params]
        keys = [_group_key(p) for p in self._params]
        if self.static_graph or self.find_unused_parameters or self._custom_caps:
            limits = [self.first_bucket_bytes_cap, self.bucket_bytes_cap]
        else:
            # one bucket now; the real layout is rebuilt from the observed grad-ready order after
            # the first backward (same policy as the reference's substrate, distributed.py:1224-1244)
            limits = [sys.maxsize]
        buckets, _ = _C.plan_buckets(nbytes, keys, limits)
        buckets = list(reversed(buckets))  # last layers produce gradients first
        self.reducer = _C.Reducer([p for p in self._params], buckets, self.comm, self.bucket_bytes_cap,
                                  self.first_bucket_bytes_cap, self.find_unused_parameters,
                                  self.gradient_as_bucket_view, self.static_graph)
        self._rebuild_checked = False
        self._publish_grad_views()

    def _reset_reducer(self):
        """Re-create the native reducer (and with it the parameters' AccumulateGrad nodes) under the
        *current* CUDA stream.  Autograd runs an AccumulateGrad node on the stream it was created
        on; a whole-step CUDA graph is captured on a side stream, so the nodes must be born there
        (the reference's DDP has the same constraint: "DDP must be constructed on the capture stream")."""
        st = self.reducer.stats()
        layout, rebuilt = st["bucket_indices"], st["has_rebuilt_buckets"]
        for p in self._params:
            p.grad = None
            if hasattr(p, "_pdt_grad_view"):
                del p._pdt_grad_view
        del self.reducer
        import gc

        gc.collect()  # drop dead autograd graphs that may still pin the old AccumulateGrad nodes
        self.reducer = _C.Reducer([p for p in self._params], layout, self.comm, self.bucket_bytes_cap,
                                  self.first_bucket_bytes_cap, self.find_unused_parameters,
                                  self.gradient_as_bucket_view, self.static_graph)
        if rebuilt:
            self.reducer.apply_rebuild(layout)
            self._rebuild_checked = True
        self._publish_grad_views()
        rearm = getattr(self, "_rearm_fused_optimizer", None)
        if rearm is not None:
            rearm()  # the optimizer re-installs its fused update on the new reducer

    def _publish_grad_views(self):
        """Let our backward kernels write weight gradients straight into the bucket (ops.functional._grad_dst)."""
        if not self.gradient_as_bucket_view:
            return
        for p, v in zip(self._params, self.reducer.grad_views()):
            p._pdt_grad_view = v

    # ---- forward -----------------------------------------------------------------------------
    def _maybe_rebuild_buckets(self):
        if self._rebuild_checked or not self.reducer.should_rebuild():
            return
        self._rebuild_checked = True
        g = self.process_group
        proposal = self.reducer.propose_rebuild() if g.rank() == 0 else None  # group rank 0 proposes
        layout = dist.broadcast_object(proposal, g.ranks[0], g) if g.size() > 1 else proposal  # C6: agree on rank 0's layout
        self.reducer.apply_rebuild(layout)
        self._publish_grad_views()

    def _pre_forward(self, inputs, kwargs):
        sync = torch.is_grad_enabled() and self.require_backward_grad_sync
        if sync:
            self.reducer.prepare_for_forward()
            self._maybe_rebuild_buckets()
            rearm = getattr(self, "_rearm_fused_optimizer", None)
            if rearm is not None:
                rearm(changed_only=True)   # this iteration's update uses the hyper-parameters set before its forward
        if self._join_active:
            self._join_notify_active()
        if self.broadcast_buffers and self.require_forward_param_sync and self.module.training and not self._buffers_ride_on_reduce():
            self._sync_buffers()
        if self.device_ids:
            inputs = _to_device(inputs, self.device)
            kwargs = _to_device(kwargs, self.device)
        return inputs, kwargs

    def forward(self, *inputs, **kwargs):
        inputs, kwargs = self._pre_forward(inputs, kwargs)
        out = self.module(*inputs, **kwargs)
        if torch.is_grad_enabled():
            _begin_iteration()  # bucket slots may be written directly, once per parameter, by this iteration's backward
            self.reducer.set_require_sync(self.require_backward_grad_sync)
            self.reducer.prepare_for_backward(_flatten_outputs(out) if self.find_unused_parameters else [])
        return out

    # ---- user surface ------------------------------------------------------------------------
    @contextmanager
    def no_sync(self):
        """Accumulate gradients locally; the first forward/backward outside the block reduces the sum."""
        old = self.require_backward_grad_sync
        self.require_backward_grad_sync = False
        try:
            yield
        finally:
            self.require_backward_grad_sync = old

    def register_comm_hook(self, state, hook: Callable):
        if self._comm_hook_registered:
            raise RuntimeError("register_comm_hook can only be called once")
        self._comm_hook_registered = True
        self.reducer.register_comm_hook(lambda bucket: hook(state, bucket))

    def _get_ddp_logging_data(self) -> dict:
        s = self.reducer.stats()
        g = self.process_group
        s.update({
            "world_size": g.size(), "rank": g.rank(), "backend_name": g.backend,
            "comm_kind": getattr(g, "comm_kind", g.backend), "module_name": type(self.module).__name__,
            "broadcast_buffers": self.broadcast_buffers, "has_sync_bn": self._has_sync_bn,
            "num_parameter_tensors": len(self._params), "device_ids": self.device_ids,
            "bucket_cap_bytes": self.bucket_bytes_cap, "static_graph": self.static_graph,
            "params_flattened": self.param_arena is not None,
            "fused_optimizer": bool(self.reducer.fused_sgd),
            "buffers_ride_on_reduce": bool(getattr(self, "_tail_broadcast", False) and self.reducer.fused_sgd),
        })
        return s

    # ---- uneven inputs -----------------------------------------------------------------------
    def _join_notify_active(self):
        self._join_iters += 1
        flag = torch.ones(1, dtype=torch.int32, device=self.device)
        self.comm.allreduce(flag, dist.ReduceOp.SUM, 1.0).wait()

    @contextmanager
    def join(self, divide_by_initial_world_size: bool = True):
        """Train with uneven inputs: a rank that exhausts its data keeps shadowing the collectives
        of the ranks that still have batches (contract of ``DistributedDataParallel.join``,
        distributed.py:1798).  Gradients are divided by the full world size."""
        if not divide_by_initial_world_size:
            raise NotImplementedError("join(divide_by_initial_world_size=False) is not supported")
        if getattr(self, "_fused_optimizer", False):
            # a joined rank shadows plain bucket allreduces; the fused chunks also update parameters and carry buffers
            raise RuntimeError("join() cannot be combined with the optimizer fused into the reduction (optim.SGD.fuse_with_ddp)")
        self._join_active = True
        self._join_iters = 0
        # A rank that runs out of data cannot take part in the one-time bucket rebuild agreement (C6) of the ranks that
        # keep training — worse, rank 0 (the proposer) may be the one that stopped.  Every rank enters join() before its
        # loop, so all of them freeze the bucket layout here and the shadowed allreduces keep matching sizes.
        self._rebuild_checked = True
        try:
            yield
            # this rank is out of data: mirror the others until everybody is done
            while True:
                flag = torch.zeros(1, dtype=torch.int32, device=self.device)
                self.comm.allreduce(flag, dist.ReduceOp.SUM, 1.0).wait()
                if int(flag.item()) == 0:
                    break
                if self.broadcast_buffers and self.module.training:
                    self._sync_buffers()
                for buf in self.reducer.bucket_buffers():
                    z = torch.zeros_like(buf)
                    self.comm.allreduce(z, dist.ReduceOp.SUM, 1.0 / self.process_group.size()).wait()
            # everybody has joined: adopt the model of the rank that trained longest
            # (torch: _DDPJoinHook.post_hook → _sync_final_model)
            g = self.process_group
            counts = torch.zeros(g.size(), dtype=torch.int64, device=self.device)
            mine = torch.tensor([self._join_iters], dtype=torch.int64, device=self.device)
            self.comm.allgather(counts, mine).wait()
            src = int(torch.argmax(counts).item())
            broadcast_coalesced(self.comm, [p for p in self.module.parameters()] + self._buffers_to_sync, src)
        finally:
            self._join_active = False

    # pickling support: drop the native objects, rebuild on load (distributed.py:1306-1336)
    def __getstate__(self):
        d = self.__dict__.copy()
        for k in ("reducer", "comm", "process_group"):
            d.pop(k, None)
        return d

    def __setstate__(self, state):
        self.__dict__.update(state)
        self.process_group = dist.get_default_group()
        self.comm = self.process_group.comm
        self._build_reducer()
