"""pytorch_distributed_train_b200 — a H100-native distributed data-parallel training engine.

Same capabilities and entry points as the tutorial repo it replaces (spawn launcher,
``init_process_group``, ``DistributedDataParallel``, ``DistributedSampler``, ``SyncBatchNorm``,
MNIST ConvNet training CLI), rebuilt H100-first: own C++ store / process groups / reducer, and
sm_90a CUDA kernels for the gradient allreduce over NVLink peer memory and for the model's hot
ops.  PyTorch is the tensor + autograd substrate only.
"""
from __future__ import annotations

import importlib
import os as _os

__version__ = "0.1.0"


def _load_native():
    try:
        return importlib.import_module(__name__ + "._C")
    except ImportError as first:
        if _os.environ.get("PDT_NO_AUTOBUILD") == "1":
            raise
        # first use in a fresh checkout: build in-tree (sources → _C.so next to this file)
        from . import _build

        _build.build(verbose=bool(_os.environ.get("PDT_BUILD_VERBOSE")))
        try:
            return importlib.import_module(__name__ + "._C")
        except ImportError as second:
            raise ImportError(f"could not load the native runtime: {second} (first attempt: {first})") from second


import torch as _torch  # noqa: E402  (libtorch must be loaded before _C.so)

_C = _load_native()
if hasattr(_C, "_mark_exiting"):
    import atexit as _atexit

    _atexit.register(_C._mark_exiting)

from . import data, distributed, engine, launcher, models, nn, ops, optim, parallel, utils  # noqa: E402
from .data import DataLoader, DistributedSampler  # noqa: E402
from .distributed import (destroy_process_group, get_rank, get_world_size, init_process_group,  # noqa: E402
                          is_initialized)
from .launcher import spawn  # noqa: E402
from .parallel import DataParallel, DistributedDataParallel, SyncBatchNorm  # noqa: E402

__all__ = [
    "data", "distributed", "engine", "launcher", "models", "nn", "ops", "optim", "parallel", "utils",
    "DataLoader", "DistributedSampler", "DistributedDataParallel", "DataParallel", "SyncBatchNorm",
    "init_process_group", "destroy_process_group", "get_rank", "get_world_size", "is_initialized", "spawn",
]
