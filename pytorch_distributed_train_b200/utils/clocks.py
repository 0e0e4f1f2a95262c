"""Sample SM clocks / throttle reasons *during* a timed region.

Primary source: NVML in-process (``pynvml``), polled every couple of milliseconds by a background
thread — a 200-step timed region of the ConvNet lasts tens of milliseconds, far less than one ``nvidia-smi -lms``
period plus its start-up time.  Fallback: one long-lived ``nvidia-smi -lms`` process.
``summary()`` gives the JSON block bench.py prints."""
from __future__ import annotations

import shutil
import statistics
import subprocess
import threading
import time
from typing import List, Optional

_Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
      "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
      "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")


class ClockSampler:
    def __init__(self, gpu_index: Optional[int] = None, period_ms: int = 100, nvml_period_ms: float = 2.0):
        self.gpu_index = gpu_index
        self.period_ms = period_ms
        self.nvml_period_ms = nvml_period_ms
        self.rows: List[List[str]] = []
        self.proc = None
        self.thread = None
        self.source = None
        self._stop = threading.Event()

    # ---- NVML path --------------------------------------------------------------------------------------
    def _nvml_handle(self):
        import pynvml

        pynvml.nvmlInit()
        idx = 0 if self.gpu_index is None else self.gpu_index
        try:  # CUDA ordinals follow CUDA_VISIBLE_DEVICES, NVML's do not: go through the UUID when torch has it
            import torch

            uuid = str(torch.cuda.get_device_properties(idx).uuid)
            return pynvml, pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid).encode() if not uuid.startswith("GPU-") else uuid.encode())
        except Exception:  # noqa: BLE001
            return pynvml, pynvml.nvmlDeviceGetHandleByIndex(idx)

    def _nvml_sample(self, nv, h):
        sm = nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)
        mx = nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)
        try:
            pw = nv.nvmlDeviceGetPowerUsage(h) / 1000.0
        except Exception:  # noqa: BLE001
            pw = 0.0
        get = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or nv.nvmlDeviceGetCurrentClocksThrottleReasons
        bits = int(get(h))
        flag = lambda b: "Active" if bits & b else "Not Active"  # noqa: E731
        # NVML reason bits: SwPowerCap 0x4, HwSlowdown 0x8, SwThermalSlowdown 0x20, HwThermalSlowdown 0x40
        self.rows.append([str(self.gpu_index), str(sm), str(mx), f"{pw:.2f}", hex(bits), flag(0x8), flag(0x40), flag(0x20), flag(0x4)])

    def _start_nvml(self) -> bool:
        try:
            nv, h = self._nvml_handle()
            self._nvml_sample(nv, h)  # fail here rather than in the thread
            self.rows.clear()
        except Exception:  # noqa: BLE001
            return False

        def poll():
            while not self._stop.is_set():
                try:
                    self._nvml_sample(nv, h)
                except Exception:  # noqa: BLE001
                    break
                time.sleep(self.nvml_period_ms / 1e3)

        self.source = "nvml"
        self.thread = threading.Thread(target=poll, name="pdt-clocks", daemon=True)
        self.thread.start()
        return True

    def start(self):
        if self._start_nvml():
            return self
        self.source = "nvidia-smi"
        exe = shutil.which("nvidia-smi")
        if exe is None:
            return self
        cmd = [exe, f"--query-gpu={_Q}", "--format=csv,noheader,nounits", "-lms", str(self.period_ms)]
        if self.gpu_index is not None:
            cmd += ["-i", str(self.gpu_index)]
        try:
            self.proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self.proc = None
            return self

        def pump():
            for line in self.proc.stdout:
                parts = [p.strip() for p in line.split(",")]
                if len(parts) >= 9:
                    self.rows.append(parts)

        self.thread = threading.Thread(target=pump, daemon=True)
        self.thread.start()
        return self

    def stop(self):
        self._stop.set()
        if self.proc is None and self.thread is not None:
            self.thread.join(1)
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(2)
            except subprocess.TimeoutExpired:
                self.proc.kill()
            if self.thread is not None:
                self.thread.join(1)
        return self

    def __enter__(self):
        return self.start()

    def __exit__(self, *exc):
        self.stop()
        return False

    def summary(self) -> dict:
        sm, mx, pw, reasons = [], [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[1]))
                mx.append(float(r[2]))
                pw.append(float(r[3]))
            except ValueError:
                continue
            for name, val in zip(names, r[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "power_w_max": max(pw),
                "reasons": sorted(reasons), "samples": len(sm), "source": self.source}
