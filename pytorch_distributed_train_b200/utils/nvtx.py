"""NVTX ranges (no-ops without CUDA) so phases show up in ncu/nsys timelines."""
from __future__ import annotations

from contextlib import contextmanager

import torch


@contextmanager
def nvtx_range(name: str):
    on = torch.cuda.is_available()
    if on:
        torch.cuda.nvtx.range_push(name)
    try:
        yield
    finally:
        if on:
            torch.cuda.nvtx.range_pop()
