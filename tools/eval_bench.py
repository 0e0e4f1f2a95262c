#!/usr/bin/env python
"""Wall time to evaluate the MNIST ConvNet on a 10,000-image test split at batch 100 on one GPU, three ways:

* ``evaluate``: ``pdt.engine.evaluate``, the metrics counted on the device by the cross-entropy kernel, one read at the end;
* ``item_loop``: the tutorial loop, ``loss.item()`` and ``(out.argmax(1) == y).sum().item()`` after every batch;
* ``device_loop``: the same torch ops accumulated into device tensors, read once at the end.

Every arm runs the same eval forward (the per-op kernels) over the same pinned batches, and every timing ends in a device
synchronise.  The arms alternate over the repeats; the card's name and power limit are read in the same run.  One JSON line.
Usage: python tools/eval_bench.py [--repeats 7]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_distributed_train_b200 as pdt  # noqa: E402


def item_loop(model, loader, criterion, dev):
    model.eval()
    total, correct, count = 0.0, 0, 0
    with torch.no_grad():
        for x, y in loader:
            x, y = x.to(dev, non_blocking=True), y.to(dev, non_blocking=True)
            out = model(x)
            total += criterion(out, y).item() * y.shape[0]
            correct += (out.argmax(1) == y).sum().item()
            count += y.shape[0]
    model.train()
    return {"loss": total / count, "correct": correct, "count": count}


def device_loop(model, loader, criterion, dev):
    model.eval()
    total = torch.zeros((), dtype=torch.float64, device=dev)
    correct = torch.zeros((), dtype=torch.int64, device=dev)
    count = 0
    with torch.no_grad():
        for x, y in loader:
            x, y = x.to(dev, non_blocking=True), y.to(dev, non_blocking=True)
            out = model(x)
            total += F.cross_entropy(out, y, reduction="sum")
            correct += (out.argmax(1) == y).sum()
            count += y.shape[0]
    model.train()
    return {"loss": total.item() / count, "correct": int(correct.item()), "count": count}


def evaluate(model, loader, criterion, dev):
    return pdt.engine.evaluate(model, loader, criterion)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    model = pdt.models.ConvNet().to(dev)
    criterion = pdt.nn.CrossEntropyLoss()
    loader = pdt.DataLoader(pdt.data.SyntheticMNIST(10000, seed=1), batch_size=100, pin_memory=True)
    arms = {"evaluate": evaluate, "item_loop": item_loop, "device_loop": device_loop}
    times = {k: [] for k in arms}
    results = {}
    for k, fn in arms.items():   # warm-up: module loads, allocator, pinned pool
        results[k] = fn(model, loader, criterion, dev)
    for _ in range(args.repeats):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn(model, loader, criterion, dev)
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    out = {"card": card(), "images": 10000, "batch": 100, "repeats": args.repeats,
           "ms_median": {k: round(sorted(v)[len(v) // 2], 3) for k, v in times.items()},
           "ms_min": {k: round(min(v), 3) for k, v in times.items()},
           "correct": {k: r["correct"] for k, r in results.items()},
           "loss": {k: r["loss"] for k, r in results.items()}}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
