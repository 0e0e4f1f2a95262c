"""Device-side timing helpers: CUDA events on the launching stream, max over ranks
(the metric contract of BASELINE.json: "device-timed, max over ranks")."""
from __future__ import annotations

import time
from typing import Optional

import torch


class DeviceTimer:
    """``with DeviceTimer() as t: ...; t.ms`` — CUDA events when a GPU is present, else wall clock."""

    def __init__(self, stream: Optional["torch.cuda.Stream"] = None, sync: bool = True):
        self.cuda = torch.cuda.is_available()
        self.stream = stream
        self.sync = sync
        self.ms = float("nan")

    def __enter__(self):
        if self.cuda:
            if self.sync:
                torch.cuda.synchronize()
            self._a = torch.cuda.Event(enable_timing=True)
            self._b = torch.cuda.Event(enable_timing=True)
            self._a.record(self.stream)
        else:
            self._t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        if self.cuda:
            self._b.record(self.stream)
            self._b.synchronize()
            self.ms = self._a.elapsed_time(self._b)
        else:
            self.ms = (time.perf_counter() - self._t0) * 1e3
        return False


def max_over_ranks(value: float, group=None) -> float:
    """MAX-allreduce a host scalar through our own process group (1 rank: identity)."""
    from .. import distributed as dist

    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return float(value)
    g = group or dist.get_default_group()
    dev = torch.device("cuda", torch.cuda.current_device()) if g.is_cuda else torch.device("cpu")
    t = torch.tensor([float(value)], dtype=torch.float32, device=dev)
    dist.all_reduce(t, dist.ReduceOp.MAX, g)
    return float(t.item())


_FLUSH = {}


def l2_flush(device=None, nbytes: int = 256 << 20) -> None:
    """Evict L2 (50 MB on H100) by overwriting a buffer larger than it."""
    if not torch.cuda.is_available():
        return
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    buf = _FLUSH.get(dev)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _FLUSH[dev] = buf
    buf.zero_()
