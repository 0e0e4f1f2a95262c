"""sm_90a operator library (Python face).  Every function here launches hand-written CUDA
kernels from ``_C`` (csrc/cuda/*.cu); there is no eager fallback on a GPU: if the native runtime
is missing on a CUDA machine the ops raise instead of silently running ATen kernels."""
from __future__ import annotations

import torch

from .. import _C

_HAS_NATIVE = hasattr(_C, "ops_ready")


def native_available() -> bool:
    """True when the compiled sm_90a kernels are present *and* a CUDA device is usable."""
    return _HAS_NATIVE and torch.cuda.is_available()


def require_native(what: str) -> None:
    if not _HAS_NATIVE:
        raise RuntimeError(f"{what}: the native sm_90a runtime (_C.so with CUDA kernels) is missing; "
                           "run `python -m pytorch_distributed_train_b200._build`")
    if not torch.cuda.is_available():
        raise RuntimeError(f"{what}: no CUDA device available")


if _HAS_NATIVE:
    from .functional import (adadelta_step, adagrad_step, adam_step, adamax_step, asgd_step, average_update, bn_apply,  # noqa: F401
                             bn_backward_apply, bn_backward_reduce, bn_finalize, bn_local_stats, conv_bn_relu_pool, cross_entropy,
                             grad_norm_clip, grad_scale, linear, nadam_step, radam_step, rmsprop_step, rprop_step, sgd_step)
else:  # CPU-only build of the extension: keep the names importable, fail loudly on use
    def _missing(name):
        def f(*a, **k):
            require_native(name)
        f.__name__ = name
        return f

    for _n in ("adadelta_step", "adagrad_step", "adam_step", "adamax_step", "asgd_step", "average_update", "bn_apply", "bn_backward_apply",
               "bn_backward_reduce", "bn_finalize", "bn_local_stats", "conv_bn_relu_pool", "cross_entropy", "grad_norm_clip", "grad_scale",
               "linear", "nadam_step", "radam_step", "rmsprop_step", "rprop_step", "sgd_step"):
        globals()[_n] = _missing(_n)

# evaluation metrics: the native kernel where it applies, torch ops elsewhere (CPU, gloo, other dtypes), so importable in any build
from .functional import cross_entropy_accumulate  # noqa: E402,F401
