"""Process-group API (``init_process_group`` and friends) on our own native runtime.

This is the surface the reference touches with ``dist.init_process_group(backend=,
init_method=, world_size=, rank=)`` (ref: ddp_example.py:50) plus the calls a DDP user
expects next to it.  Nothing here imports ``torch.distributed``: stores, rendezvous, the CPU
mesh backend, the NVLink symmetric-memory backend and the NCCL baseline binding all live in
``pytorch_distributed_train_b200._C``.

Backends
--------
``"nccl"``  (the reference's default flag value, ref: ddp_example.py:105)
    GPU group. ``comm="fused"`` (default): collectives are our sm_90a kernels over NVLink peer /
    multicast memory (``SymmComm``). ``comm="nccl"``: the thin libnccl binding, kept as the measured
    baseline and oracle. Also selectable via ``PDT_COMM``.
``"gloo"`` / ``"cpu"``
    CPU tensors over a TCP mesh (``CpuComm``).
"""
from __future__ import annotations

import os
import sys
import threading
import time
from typing import List, Optional, Sequence

import torch

from .. import _C
from .rendezvous import RendezvousError, rendezvous

ReduceOp = _C.ReduceOp
Work = _C.Work
Store = _C.Store
TCPStore = _C.TCPStore
HashStore = _C.HashStore
FileStore = _C.FileStore
PrefixStore = _C.PrefixStore

DEFAULT_TIMEOUT_NCCL = 600.0    # seconds; same defaults the reference inherits
DEFAULT_TIMEOUT_OTHER = 1800.0  # (torch distributed_c10d.py:777-790)

_GPU_BACKENDS = ("nccl", "nvlink", "symm", "nccl-lib")
_CPU_BACKENDS = ("gloo", "cpu")


class ProcessGroup:
    """A communicator over a fixed set of ranks."""

    def __init__(self, comm, store, rank: int, size: int, backend: str, ranks: Sequence[int], name: str,
                 timeout: float):
        self.comm = comm
        self.store = store
        self._rank = rank
        self._size = size
        self.backend = backend
        self.ranks = list(ranks)          # global ranks, group order
        self.name = name
        self.timeout = timeout
        self._seq = 0

    def rank(self) -> int:
        return self._rank

    def size(self) -> int:
        return self._size

    @property
    def is_cuda(self) -> bool:
        return self.comm.is_cuda

    def __repr__(self):
        return f"ProcessGroup(name={self.name!r}, backend={self.backend!r}, rank={self._rank}, size={self._size})"


class _World:
    def __init__(self):
        self.default: Optional[ProcessGroup] = None
        self.store = None
        self.groups: List[ProcessGroup] = []
        self.group_count = 0
        self.prev_excepthook = None
        self.lock = threading.Lock()


_world = _World()


def _install_excepthook(rank: int):
    """Prefix uncaught exceptions with ``[rankN]:`` (parity: distributed_c10d.py:1860-1877)."""
    prev = sys.excepthook
    _world.prev_excepthook = prev

    def hook(tp, val, tb):
        import io
        import traceback

        buf = io.StringIO()
        traceback.print_exception(tp, val, tb, file=buf)
        sys.stderr.write("".join(f"[rank{rank}]: {line}\n" for line in buf.getvalue().rstrip("\n").split("\n")))

    sys.excepthook = hook


def is_available() -> bool:
    return True


def is_initialized() -> bool:
    return _world.default is not None


def is_nccl_available() -> bool:
    return hasattr(_C, "NcclComm") and _C.nccl_available()


def is_gloo_available() -> bool:
    return True


def _make_comm(backend: str, comm_kind: str, store, rank: int, size: int, timeout: float, device_id):
    if backend in _CPU_BACKENDS:
        host = os.environ.get("PDT_BIND_HOST", "127.0.0.1")
        return _C.CpuComm(store, rank, size, timeout, host), "cpu"
    if backend in _GPU_BACKENDS:
        if not torch.cuda.is_available():
            raise RuntimeError(
                f"backend {backend!r} needs a CUDA device; on a CPU-only host use backend='gloo' "
                "(the reference script has the same constraint, ref: ddp_example.py:57-58)")
        if not hasattr(_C, "SymmComm"):
            raise RuntimeError("the native CUDA runtime is missing from _C.so; rebuild with pytorch_distributed_train_b200._build")
        if device_id is None:
            device_id = torch.cuda.current_device()
        elif isinstance(device_id, torch.device):
            device_id = device_id.index if device_id.index is not None else torch.cuda.current_device()
        if backend == "nccl-lib":
            comm_kind = "nccl"
        if backend in ("nvlink", "symm"):
            comm_kind = "fused"
        if comm_kind == "nccl":
            return _C.NcclComm(store, rank, size, int(device_id), timeout), "nccl-lib"
        heap_mb = int(os.environ.get("PDT_SYMM_HEAP_MB", "1024"))
        return _C.SymmComm(store, rank, size, int(device_id), timeout, heap_mb << 20), "nvlink"
    raise ValueError(f"unknown backend {backend!r}; expected one of {_GPU_BACKENDS + _CPU_BACKENDS}")


def init_process_group(backend: Optional[str] = None, init_method: Optional[str] = None,
                       timeout: Optional[float] = None, world_size: int = -1, rank: int = -1,
                       store=None, group_name: str = "", device_id=None, comm: Optional[str] = None) -> None:
    """Initialise the default process group.

    Mirrors the call at ref: ddp_example.py:50.  ``init_method`` XOR ``store``; default
    ``env://``; double initialisation is an error; rank 0 hosts the TCP store.
    ``timeout`` may be seconds or a ``datetime.timedelta``.
    """
    if _world.default is not None:
        raise RuntimeError("trying to initialize the default process group twice!")
    if store is not None and init_method is not None:
        raise ValueError("Cannot specify both init_method and store.")
    if backend is None:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
    backend = backend.lower()
    if hasattr(timeout, "total_seconds"):
        timeout = timeout.total_seconds()
    if timeout is None:
        timeout = DEFAULT_TIMEOUT_NCCL if backend in _GPU_BACKENDS else DEFAULT_TIMEOUT_OTHER
    comm_kind = (comm or os.environ.get("PDT_COMM", "fused")).lower()
    if comm_kind not in ("fused", "nccl"):
        raise ValueError(f"comm must be 'fused' or 'nccl', got {comm_kind!r}")

    if store is None:
        store, rank, world_size = rendezvous(init_method, rank, world_size, min(timeout, 300.0))
    else:
        if rank < 0 or world_size <= 0:
            raise ValueError("rank and world_size are required when a store is passed")
    if not (0 <= rank < world_size):
        raise ValueError(f"rank {rank} out of range for world_size {world_size}")
    store.set_timeout(timeout)
    _world.store = store
    pg_store = PrefixStore("default_pg", store)
    comm_obj, resolved = _make_comm(backend, comm_kind, PrefixStore("comm0", pg_store), rank, world_size, timeout, device_id)
    pg = ProcessGroup(comm_obj, pg_store, rank, world_size, backend, list(range(world_size)),
                      group_name or "default", timeout)
    pg.comm_kind = resolved
    _world.default = pg
    _world.groups = [pg]
    _world.group_count = 1
    _install_excepthook(rank)
    if os.environ.get("PDT_DIST_INIT_BARRIER", "0") == "1":
        _C.store_barrier(pg_store, "init", rank, world_size, timeout)


def destroy_process_group(group: Optional[ProcessGroup] = None) -> None:
    """Tear down (the reference never calls this, ref: ddp_example.py:96-97; we provide it)."""
    if _world.default is None:
        return
    targets = list(_world.groups) if group is None or group is _world.default else [group]
    if group is None or group is _world.default:
        # Rank 0 hosts the store: it must outlive every peer that may still be inside a store
        # call, so it leaves last (bounded wait — a dead peer must not wedge shutdown).
        d = _world.default
        try:
            d.store.add("__destroy__/count", 1)
            if d.rank() == 0 and d.size() > 1:
                deadline = time.time() + float(os.environ.get("PDT_DESTROY_WAIT", "10"))
                while d.store.add("__destroy__/count", 0) < d.size() and time.time() < deadline:
                    time.sleep(0.002)
        except Exception:
            pass
    for g in targets:
        try:
            g.comm.shutdown()
        except Exception:
            pass
        if g in _world.groups:
            _world.groups.remove(g)
    if group is None or group is _world.default:
        _world.default = None
        _world.store = None
        _world.groups = []
        if _world.prev_excepthook is not None:
            sys.excepthook = _world.prev_excepthook
            _world.prev_excepthook = None


def _group(group: Optional[ProcessGroup]) -> ProcessGroup:
    if group is not None:
        return group
    if _world.default is None:
        raise RuntimeError("Default process group has not been initialized, please make sure to call init_process_group.")
    return _world.default


def get_default_group() -> ProcessGroup:
    return _group(None)


def get_rank(group: Optional[ProcessGroup] = None) -> int:
    return _group(group).rank()


def get_world_size(group: Optional[ProcessGroup] = None) -> int:
    return _group(group).size()


def get_backend(group: Optional[ProcessGroup] = None) -> str:
    return _group(group).backend


def get_store():
    return _world.store


def new_group(ranks: Optional[Sequence[int]] = None, backend: Optional[str] = None,
              timeout: Optional[float] = None, comm: Optional[str] = None) -> Optional[ProcessGroup]:
    """Collective over the default group: every rank must call it with the same ``ranks``."""
    world = _group(None)
    ranks = list(range(world.size())) if ranks is None else sorted(ranks)
    with _world.lock:
        gid = _world.group_count
        _world.group_count += 1
    backend = (backend or world.backend).lower()
    timeout = timeout or world.timeout
    if world.rank() not in ranks:
        return None
    sub_rank = ranks.index(world.rank())
    store = PrefixStore(f"group{gid}", world.store)
    comm_kind = (comm or ("nccl" if getattr(world, "comm_kind", "") == "nccl-lib" else "fused"))
    dev = torch.cuda.current_device() if backend in _GPU_BACKENDS else None
    comm_obj, resolved = _make_comm(backend, comm_kind, PrefixStore("comm0", store), sub_rank, len(ranks), timeout, dev)
    pg = ProcessGroup(comm_obj, store, sub_rank, len(ranks), backend, ranks, f"group{gid}", timeout)
    pg.comm_kind = resolved
    _world.groups.append(pg)
    return pg


# ---- collectives ---------------------------------------------------------------------------
def _debug_level() -> str:
    return (os.environ.get("PDT_DISTRIBUTED_DEBUG") or os.environ.get("TORCH_DISTRIBUTED_DEBUG") or "OFF").upper()


def _precheck(g: ProcessGroup, op: str, tensors: Sequence[torch.Tensor], extra: str = "") -> None:
    """Debug layer (the reference stack's counterpart is ProcessGroupWrapper under
    TORCH_DISTRIBUTED_DEBUG=DETAIL, torch distributed_c10d.py:5121-5137, and TORCH_NCCL_NAN_CHECK).

    ``PDT_DISTRIBUTED_DEBUG=DETAIL``: before a collective runs, every rank publishes a fingerprint
    (sequence number, op, shapes, dtypes, root/op argument) through the group's store and compares it
    with every peer's, so "rank 3 called broadcast while the rest called all_reduce" is an exception
    naming the ranks instead of a hang or silent corruption.  ``PDT_NAN_CHECK=1``: refuse to
    communicate non-finite floating-point payloads."""
    nan_check = os.environ.get("PDT_NAN_CHECK", "0") == "1"
    detail = _debug_level() == "DETAIL"
    if not (nan_check or detail):
        return
    if nan_check:
        for t in tensors:
            if t.is_floating_point() and t.numel() and not bool(torch.isfinite(t).all()):
                raise RuntimeError(f"[rank{g.rank()}] {op}: non-finite values in a tensor handed to a collective "
                                   f"(shape {tuple(t.shape)}, dtype {t.dtype}) — PDT_NAN_CHECK=1")
    if detail and g.size() > 1:
        g._dbg_seq = getattr(g, "_dbg_seq", 0) + 1
        seq = g._dbg_seq
        fp = f"{op}|{extra}|" + ";".join(f"{tuple(t.shape)}:{t.dtype}" for t in tensors)
        base = f"dbg/{g.name}/{seq}"
        g.store.set(f"{base}/{g.rank()}", fp.encode())
        bad = []
        for r in range(g.size()):
            if r == g.rank():
                continue
            other = bytes(g.store.get(f"{base}/{r}")).decode()
            if other != fp:
                bad.append((r, other))
        if seq > 2:
            try:
                g.store.delete_key(f"dbg/{g.name}/{seq - 2}/{g.rank()}")
            except Exception:
                pass
        if bad:
            lines = "\n".join(f"  rank {r}: {o}" for r, o in bad)
            raise RuntimeError(f"[rank{g.rank()}] collective mismatch at sequence number {seq} in group {g.name!r}:\n"
                               f"  rank {g.rank()}: {fp}\n{lines}")


def _finish(work, async_op: bool):
    if async_op:
        return work
    work.wait()
    return None


def _contig(t: torch.Tensor, what: str) -> torch.Tensor:
    if not t.is_contiguous():
        raise ValueError(f"{what}: tensor must be contiguous")
    return t


def all_reduce(tensor: torch.Tensor, op=ReduceOp.SUM, group: Optional[ProcessGroup] = None, async_op: bool = False):
    g = _group(group)
    _precheck(g, "all_reduce", [tensor], str(op))
    if op == ReduceOp.AVG and g.is_cuda:
        return _finish(g.comm.allreduce(_contig(tensor, "all_reduce"), ReduceOp.SUM, 1.0 / g.size()), async_op)
    return _finish(g.comm.allreduce(_contig(tensor, "all_reduce"), op, 1.0), async_op)


def _group_rank(g: ProcessGroup, global_rank: int, what: str) -> int:
    """torch's API takes *global* ranks for src / dst in every rooted and point-to-point op, also on subgroups;
    the communicators index by rank inside the group."""
    ranks = list(g.ranks)
    if global_rank not in ranks:
        raise ValueError(f"{what}: global rank {global_rank} is not part of the group (ranks {ranks})")
    return ranks.index(global_rank)


def broadcast(tensor: torch.Tensor, src: int, group: Optional[ProcessGroup] = None, async_op: bool = False):
    g = _group(group)
    root = _group_rank(g, src, "broadcast")
    _precheck(g, "broadcast", [tensor], f"root={root}")
    return _finish(g.comm.broadcast(_contig(tensor, "broadcast"), root), async_op)


def all_gather_into_tensor(output_tensor: torch.Tensor, input_tensor: torch.Tensor,
                           group: Optional[ProcessGroup] = None, async_op: bool = False):
    g = _group(group)
    _precheck(g, "all_gather_into_tensor", [input_tensor])
    return _finish(g.comm.allgather(_contig(output_tensor, "all_gather output"), _contig(input_tensor, "all_gather input")), async_op)


def all_gather(tensor_list: List[torch.Tensor], tensor: torch.Tensor, group: Optional[ProcessGroup] = None,
               async_op: bool = False):
    g = _group(group)
    if len(tensor_list) != g.size():
        raise ValueError("all_gather: tensor_list must have world_size entries")
    flat = torch.empty((g.size(),) + tuple(tensor.shape), dtype=tensor.dtype, device=tensor.device)
    work = g.comm.allgather(flat.view(-1), _contig(tensor, "all_gather input").view(-1))

    class _Scatter:
        def wait(self_inner):
            work.wait()
            for i, t in enumerate(tensor_list):
                t.copy_(flat[i])
            return True

        def is_completed(self_inner):
            return work.is_completed()

    w = _Scatter()
    if async_op:
        return w
    w.wait()
    return None


def reduce(tensor: torch.Tensor, dst: int, op=ReduceOp.SUM, group: Optional[ProcessGroup] = None, async_op: bool = False):
    g = _group(group)
    root = _group_rank(g, dst, "reduce")
    _precheck(g, "reduce", [tensor], f"{op},dst={root}")
    return _finish(g.comm.reduce(_contig(tensor, "reduce"), op, root), async_op)


def reduce_scatter_tensor(output: torch.Tensor, input: torch.Tensor, op=ReduceOp.SUM,
                          group: Optional[ProcessGroup] = None, async_op: bool = False):
    g = _group(group)
    _precheck(g, "reduce_scatter_tensor", [input], str(op))
    return _finish(g.comm.reduce_scatter(_contig(output, "reduce_scatter output"), _contig(input, "reduce_scatter input"), op), async_op)


def gather(tensor: torch.Tensor, gather_list: Optional[List[torch.Tensor]] = None, dst: int = 0,
           group: Optional[ProcessGroup] = None):
    g = _group(group)
    dst = _group_rank(g, dst, "gather")
    out = torch.empty((g.size(),) + tuple(tensor.shape), dtype=tensor.dtype, device=tensor.device) if g.rank() == dst else tensor.new_empty(0)
    g.comm.gather(out.view(-1), _contig(tensor, "gather").view(-1), dst).wait()
    if g.rank() == dst and gather_list is not None:
        for i, t in enumerate(gather_list):
            t.copy_(out[i])


def scatter(tensor: torch.Tensor, scatter_list: Optional[List[torch.Tensor]] = None, src: int = 0,
            group: Optional[ProcessGroup] = None):
    g = _group(group)
    src = _group_rank(g, src, "scatter")
    inp = torch.stack(list(scatter_list)).contiguous().view(-1) if g.rank() == src else tensor.new_empty(0)
    g.comm.scatter(_contig(tensor, "scatter").view(-1), inp, src).wait()


def all_to_all_single(output: torch.Tensor, input: torch.Tensor, group: Optional[ProcessGroup] = None, async_op: bool = False):
    g = _group(group)
    _precheck(g, "all_to_all_single", [input])
    return _finish(g.comm.alltoall(_contig(output, "all_to_all output").view(-1), _contig(input, "all_to_all input").view(-1)), async_op)


def all_to_all(output_tensor_list: List[torch.Tensor], input_tensor_list: List[torch.Tensor], group: Optional[ProcessGroup] = None,
               async_op: bool = False):
    """List form of the all-to-all (equal-sized chunks): ``input_tensor_list[j]`` goes to rank j, ``output_tensor_list[i]`` comes from
    rank i (parity: distributed_c10d.py ``all_to_all``).  One flat exchange underneath."""
    g = _group(group)
    if len(output_tensor_list) != g.size() or len(input_tensor_list) != g.size():
        raise ValueError("all_to_all: one input and one output tensor per rank expected")
    shapes = {tuple(t.shape) for t in input_tensor_list} | {tuple(t.shape) for t in output_tensor_list}
    if len(shapes) != 1:
        raise ValueError("all_to_all: only equal-sized chunks are supported")
    inp = torch.stack([_contig(t, "all_to_all input") for t in input_tensor_list]).view(-1)
    out = torch.empty_like(inp)
    work = all_to_all_single(out, inp, group=g, async_op=True)

    def finish():
        work.wait()
        for i, t in enumerate(output_tensor_list):
            t.copy_(out.view(g.size(), *t.shape)[i])

    if async_op:
        return _Deferred(finish)
    finish()
    return None


def reduce_scatter(output: torch.Tensor, input_list: List[torch.Tensor], op=ReduceOp.SUM, group: Optional[ProcessGroup] = None,
                   async_op: bool = False):
    """List form of reduce-scatter: rank i receives the reduction of every rank's ``input_list[i]``."""
    g = _group(group)
    if len(input_list) != g.size():
        raise ValueError("reduce_scatter: one input tensor per rank expected")
    flat = torch.stack([_contig(t, "reduce_scatter input") for t in input_list]).view(-1)
    return reduce_scatter_tensor(output, flat, op=op, group=g, async_op=async_op)


class _Deferred:
    """Work-like handle of an operation with a host-side epilogue (copy-out of a staged result)."""

    def __init__(self, finish):
        self._finish, self._done = finish, False

    def wait(self, timeout=None):
        if not self._done:
            self._finish()
            self._done = True
        return True

    def is_completed(self):
        return self._done


def get_process_group_ranks(group: Optional[ProcessGroup] = None) -> List[int]:
    """Global ranks of the group, in group order (parity: distributed_c10d.py ``get_process_group_ranks``)."""
    return list(_group(group).ranks)


def get_global_rank(group: Optional[ProcessGroup], group_rank: int) -> int:
    ranks = _group(group).ranks
    if not 0 <= group_rank < len(ranks):
        raise ValueError(f"get_global_rank: group rank {group_rank} out of range (group size {len(ranks)})")
    return ranks[group_rank]


def get_group_rank(group: Optional[ProcessGroup], global_rank: int) -> int:
    return _group_rank(_group(group), global_rank, "get_group_rank")


class P2POp:
    """One point-to-point operation of a batch (parity: distributed_c10d.py ``P2POp``): ``op`` is ``isend`` or ``irecv``."""

    def __init__(self, op, tensor: torch.Tensor, peer: int, group: Optional[ProcessGroup] = None, tag: int = 0):
        if op not in (isend, irecv):
            raise ValueError("P2POp: op must be distributed.isend or distributed.irecv")
        self.op, self.tensor, self.peer, self.group, self.tag = op, tensor, peer, group, tag


def batch_isend_irecv(p2p_op_list: List[P2POp]) -> list:
    """Issue a list of sends / receives and return their work handles (in list order).  Both backends execute a rank's point-to-point
    operations in issue order (one worker thread / one comm stream) with an eager protocol for messages up to the staging size: a send
    completes without its receiver, a receive waits for its sender.  Sends are therefore issued first — a ring in which every rank
    posted its receive first would wait on itself."""
    if not p2p_op_list or not all(isinstance(o, P2POp) for o in p2p_op_list):
        raise ValueError("batch_isend_irecv: a non-empty list of P2POp expected")
    order = sorted(range(len(p2p_op_list)), key=lambda i: 0 if p2p_op_list[i].op is isend else 1)
    works = [None] * len(p2p_op_list)
    for i in order:
        o = p2p_op_list[i]
        works[i] = o.op(o.tensor, o.peer, o.group)
    return works


def send(tensor: torch.Tensor, dst: int, group: Optional[ProcessGroup] = None):
    g = _group(group)
    g.comm.send(_contig(tensor, "send"), _group_rank(g, dst, "send")).wait()


def recv(tensor: torch.Tensor, src: int, group: Optional[ProcessGroup] = None):
    g = _group(group)
    g.comm.recv(_contig(tensor, "recv"), _group_rank(g, src, "recv")).wait()


def isend(tensor: torch.Tensor, dst: int, group: Optional[ProcessGroup] = None):
    g = _group(group)
    return g.comm.send(_contig(tensor, "isend"), _group_rank(g, dst, "isend"))


def irecv(tensor: torch.Tensor, src: int, group: Optional[ProcessGroup] = None):
    g = _group(group)
    return g.comm.recv(_contig(tensor, "irecv"), _group_rank(g, src, "irecv"))


def barrier(group: Optional[ProcessGroup] = None, async_op: bool = False):
    g = _group(group)
    w = g.comm.barrier()
    if async_op:
        return w
    w.wait()
    if g.is_cuda:
        w.synchronize()
    return None


def monitored_barrier(group: Optional[ProcessGroup] = None, timeout: Optional[float] = None):
    """Store-based barrier that names the ranks that failed to arrive (debug aid)."""
    g = _group(group)
    timeout = timeout or g.timeout
    g._seq += 1
    key = f"monitored/{g._seq}"
    g.store.set(f"{key}/{g.rank()}", "1")
    deadline = time.time() + timeout
    missing = list(range(g.size()))
    while missing and time.time() < deadline:
        missing = [r for r in missing if not g.store.check([f"{key}/{r}"])]
        if missing:
            time.sleep(0.005)
    if missing:
        raise RuntimeError(f"[rank{g.rank()}] monitored_barrier: ranks {missing} did not arrive within {timeout}s")


def all_gather_object(obj, group: Optional[ProcessGroup] = None) -> list:
    """Gather picklable objects through the store (host side channel; used for one-off metadata)."""
    import pickle

    g = _group(group)
    g._seq += 1
    key = f"ago/{g._seq}"
    g.store.set(f"{key}/{g.rank()}", pickle.dumps(obj))
    out = [pickle.loads(b) for b in g.store.multi_get([f"{key}/{r}" for r in range(g.size())])]
    # last reader cleans up
    if g.store.add(f"{key}/done", 1) == g.size():
        for r in range(g.size()):
            g.store.delete_key(f"{key}/{r}")
        g.store.delete_key(f"{key}/done")
    return out


def _object_key(g: ProcessGroup, tag: str) -> str:
    g._seq += 1
    return f"{tag}/{g._seq}"


def _last_one_cleans(g: ProcessGroup, key: str, keys) -> None:
    """Every participant checks out; the last one deletes the exchange's keys so the store does not grow."""
    if g.store.add(f"{key}/done", 1) == g.size():
        for k in keys:
            g.store.delete_key(k)
        g.store.delete_key(f"{key}/done")


def broadcast_object(obj, src: int = 0, group: Optional[ProcessGroup] = None):
    """Returns ``src``'s object on every rank (control-plane traffic through the store, like the substrate's
    object collectives which pickle into byte tensors)."""
    import pickle

    g = _group(group)
    src = _group_rank(g, src, "broadcast_object")
    key = _object_key(g, "bco")
    if g.rank() == src:
        g.store.set(key, pickle.dumps(obj))
        out = obj
    else:
        out = pickle.loads(g.store.get(key))
    _last_one_cleans(g, key, [key])
    return out


def broadcast_object_list(object_list: list, src: int = 0, group: Optional[ProcessGroup] = None) -> None:
    """torch signature: ``object_list`` is overwritten in place with ``src``'s list (same length on every rank)."""
    g0 = _group(group)
    got = broadcast_object(list(object_list) if g0.rank() == _group_rank(g0, src, "broadcast_object_list") else None, src, group)
    if len(got) != len(object_list):
        raise ValueError(f"broadcast_object_list: rank {_group(group).rank()} passed {len(object_list)} slots, src sent {len(got)}")
    object_list[:] = got


def gather_object(obj, object_gather_list: Optional[list] = None, dst: int = 0, group: Optional[ProcessGroup] = None) -> None:
    g = _group(group)
    dst = _group_rank(g, dst, "gather_object")
    if g.rank() == dst and (object_gather_list is None or len(object_gather_list) != g.size()):
        raise ValueError("gather_object: the destination rank must pass a list with world_size slots")
    allobjs = all_gather_object(obj, g)
    if g.rank() == dst:
        object_gather_list[:] = allobjs


def scatter_object_list(scatter_object_output_list: list, scatter_object_input_list: Optional[list] = None, src: int = 0,
                        group: Optional[ProcessGroup] = None) -> None:
    """Rank r receives ``scatter_object_input_list[r]`` of ``src`` into ``scatter_object_output_list[0]``."""
    import pickle

    g = _group(group)
    if not scatter_object_output_list:
        raise ValueError("scatter_object_list: the output list needs at least one slot")
    src = _group_rank(g, src, "scatter_object_list")
    key = _object_key(g, "sco")
    keys = [f"{key}/{r}" for r in range(g.size())]
    if g.rank() == src:
        if scatter_object_input_list is None or len(scatter_object_input_list) != g.size():
            raise ValueError("scatter_object_list: src must pass world_size objects")
        g.store.multi_set(keys, [pickle.dumps(o) for o in scatter_object_input_list])
    scatter_object_output_list[0] = pickle.loads(g.store.get(keys[g.rank()]))
    _last_one_cleans(g, key, keys)


__all__ = [
    "ReduceOp", "Work", "Store", "TCPStore", "HashStore", "FileStore", "PrefixStore", "ProcessGroup",
    "RendezvousError", "rendezvous", "init_process_group", "destroy_process_group", "is_initialized",
    "is_available", "is_nccl_available", "is_gloo_available", "get_rank", "get_world_size", "get_backend",
    "get_default_group", "get_store", "new_group", "all_reduce", "broadcast", "all_gather",
    "all_gather_into_tensor", "reduce", "reduce_scatter_tensor", "gather", "scatter", "all_to_all_single",
    "send", "recv", "isend", "irecv", "barrier", "monitored_barrier", "all_gather_object", "broadcast_object",
    "broadcast_object_list", "gather_object", "scatter_object_list",
]
