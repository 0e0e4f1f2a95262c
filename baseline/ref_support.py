"""Harness-only helpers for ``bench.py --impl reference``.

Standalone on purpose: the reference arm must not import (or memory-map) anything from
``pytorch_distributed_train_b200`` — no model, kernel, engine or ``_C.so`` of ours may sit in the
reference process.  Everything here is plain Python + numpy + NVML:

* :func:`write_synthetic_mnist` writes idx files of MNIST's shape where ``torchvision.datasets.MNIST``
  expects them (the reference calls it with ``download=True``, ref: ddp_example.py:66-69; with the raw
  files present torchvision skips the download);
* :class:`Clocks` samples SM clock / throttle reasons during the timed region.
"""
from __future__ import annotations

import os
import statistics
import struct
import threading
import time

import numpy as np

_FILES = {True: ("train-images-idx3-ubyte", "train-labels-idx1-ubyte", 60000),
          False: ("t10k-images-idx3-ubyte", "t10k-labels-idx1-ubyte", 10000)}


def _write_idx(path: str, arr: np.ndarray) -> None:
    os.makedirs(os.path.dirname(path), exist_ok=True)
    tmp = path + f".tmp{os.getpid()}"
    with open(tmp, "wb") as f:
        f.write(struct.pack(">HBB", 0, 0x08, arr.ndim))
        f.write(struct.pack(">" + "I" * arr.ndim, *arr.shape))
        f.write(np.ascontiguousarray(arr, dtype=np.uint8).tobytes())
    os.replace(tmp, path)


def write_synthetic_mnist(root: str, seed: int = 0) -> None:
    """Deterministic MNIST-shaped idx files (train + test): class-specific blobs plus noise."""
    for train in (True, False):
        img_name, lbl_name, n = _FILES[train]
        rng = np.random.default_rng(seed + (0 if train else 1))
        labels = rng.integers(0, 10, size=n)
        protos = np.zeros((10, 28, 28), dtype=np.float32)
        prng = np.random.default_rng(1234)
        for c in range(10):
            for (y, x) in prng.integers(4, 24, size=(6, 2)):
                protos[c, y - 2:y + 3, x - 2:x + 3] += 1.0
        protos /= protos.max(axis=(1, 2), keepdims=True)
        imgs = np.clip(protos[labels] * 0.85 + rng.random((n, 28, 28), dtype=np.float32) * 0.25, 0, 1)
        raw = os.path.join(root, "MNIST", "raw")
        _write_idx(os.path.join(raw, img_name), (imgs * 255).astype(np.uint8))
        _write_idx(os.path.join(raw, lbl_name), labels.astype(np.uint8))


class Clocks:
    """NVML poller (2 ms period) around a timed region; ``summary()`` is the bench JSON block."""

    def __init__(self, gpu_index: int = 0, period_ms: float = 2.0):
        self.gpu_index, self.period = gpu_index, period_ms / 1e3
        self.rows = []
        self._stop = threading.Event()
        self._th = None

    def _handle(self):
        import pynvml as nv

        nv.nvmlInit()
        try:
            import torch

            uuid = str(torch.cuda.get_device_properties(self.gpu_index).uuid)
            uuid = uuid if uuid.startswith("GPU-") else "GPU-" + uuid
            return nv, nv.nvmlDeviceGetHandleByUUID(uuid.encode())
        except Exception:  # noqa: BLE001
            return nv, nv.nvmlDeviceGetHandleByIndex(self.gpu_index)

    def __enter__(self):
        try:
            nv, h = self._handle()
        except Exception:  # noqa: BLE001 - no NVML: the block says so
            return self
        get = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or nv.nvmlDeviceGetCurrentClocksThrottleReasons

        def loop():
            while not self._stop.is_set():
                try:
                    self.rows.append((nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM), nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM),
                                      nv.nvmlDeviceGetPowerUsage(h) / 1000.0, int(get(h))))
                except Exception:  # noqa: BLE001
                    pass
                time.sleep(self.period)

        self._th = threading.Thread(target=loop, daemon=True)
        self._th.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        if self._th is not None:
            self._th.join(1.0)
        return False

    def summary(self) -> dict:
        if not self.rows:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        sm = sorted(r[0] for r in self.rows)
        load = sm[len(sm) // 2:]  # the upper half = samples taken under load
        bits = 0
        for r in self.rows:
            bits |= r[3]
        names = {0x4: "sw_power_cap", 0x8: "hw_slowdown", 0x20: "sw_thermal_slowdown", 0x40: "hw_thermal_slowdown"}
        return {"sm_mhz": statistics.median(load), "sm_max_mhz": max(r[1] for r in self.rows),
                "reasons": [n for b, n in names.items() if bits & b], "power_w_max": max(r[2] for r in self.rows),
                "samples": len(self.rows)}
