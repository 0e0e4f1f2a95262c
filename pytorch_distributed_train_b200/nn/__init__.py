"""Layers whose CUDA path is our own kernels."""
from . import utils
from .loss import CrossEntropyLoss

__all__ = ["CrossEntropyLoss", "utils"]
