"""Checkpoint / resume.

The reference saves nothing — the trained model is discarded at process exit (ref: ddp_example.py:96-97) —
but a user switching from torch's DDP expects the usual surface to work: ``state_dict()`` keys carry the
``module.`` prefix of the wrapper, rank 0 writes, everybody waits, any rank can load.  These helpers add
exactly that on top of ``state_dict`` / ``load_state_dict``:

* ``save_checkpoint`` — rank 0 serialises model (+ optimizer, sampler epoch, user extras) to CPU tensors,
  writes ``path`` atomically (temp file + rename) and the whole group passes a barrier, so no rank can
  run ahead and a crash never leaves a half-written file;
* ``load_checkpoint`` — every rank reads the file and restores in place: parameters stay where DDP put them
  (flat symmetric arenas, bucket-mirroring layout of the fused optimizer step), momentum buffers are copied into
  the optimizer's existing flat buffer, so a resumed run is bit-identical to an uninterrupted one.
"""
from __future__ import annotations

import os
import tempfile
from typing import Any, Dict, Optional

import torch


def _to_cpu(obj):
    if isinstance(obj, torch.Tensor):
        return obj.detach().to("cpu", copy=True)
    if isinstance(obj, dict):
        return {k: _to_cpu(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_to_cpu(v) for v in obj)
    return obj


def save_checkpoint(path: str, model: torch.nn.Module, optimizer: Optional[torch.optim.Optimizer] = None, *, epoch: int = 0,
                    step: int = 0, sampler=None, extra: Optional[Dict[str, Any]] = None, group=None) -> None:
    from .. import distributed as dist

    initialized = dist.is_initialized()
    rank = dist.get_rank(group) if initialized else 0
    if rank == 0:
        payload = {"format": 1, "epoch": int(epoch), "step": int(step), "model": _to_cpu(model.state_dict()),
                   "optimizer": _to_cpu(optimizer.state_dict()) if optimizer is not None else None,
                   "sampler_epoch": getattr(sampler, "epoch", None), "extra": extra or {}}
        d = os.path.dirname(os.path.abspath(path))
        os.makedirs(d, exist_ok=True)
        fd, tmp = tempfile.mkstemp(prefix=".ckpt-", dir=d)
        try:
            with os.fdopen(fd, "wb") as f:
                torch.save(payload, f)
                f.flush()
                os.fsync(f.fileno())
            os.replace(tmp, path)  # atomic on POSIX: readers see the old or the new file, never a partial one
        except BaseException:
            if os.path.exists(tmp):
                os.unlink(tmp)
            raise
    if initialized and dist.get_world_size(group) > 1:
        dist.barrier(group)


def load_checkpoint(path: str, model: torch.nn.Module, optimizer: Optional[torch.optim.Optimizer] = None, *, sampler=None,
                    strict: bool = True) -> Dict[str, Any]:
    """Restores in place and returns ``{"epoch", "step", "extra"}``.  Accepts checkpoints written from the wrapped
    (``module.``-prefixed) or the bare model and loads them into either."""
    payload = torch.load(path, map_location="cpu", weights_only=False)
    sd = payload["model"]
    want_prefix = any(k.startswith("module.") for k in model.state_dict().keys())
    have_prefix = any(k.startswith("module.") for k in sd.keys())
    if want_prefix and not have_prefix:
        sd = {"module." + k: v for k, v in sd.items()}
    elif have_prefix and not want_prefix:
        sd = {k[len("module."):]: v for k, v in sd.items()}
    model.load_state_dict(sd, strict=strict)
    if optimizer is not None and payload.get("optimizer") is not None:
        optimizer.load_state_dict(payload["optimizer"])
    if sampler is not None and payload.get("sampler_epoch") is not None and hasattr(sampler, "set_epoch"):
        sampler.set_epoch(payload["sampler_epoch"])
    return {"epoch": payload.get("epoch", 0), "step": payload.get("step", 0), "extra": payload.get("extra", {})}
