#!/usr/bin/env python
"""Device time of one graphed training step of the reference ConvNet with the cross-entropy's options (one GPU, batch 100, pdt SGD
lr 1e-4):

  pdt_plain            pdt.nn.CrossEntropyLoss()
  pdt_smooth           pdt.nn.CrossEntropyLoss(label_smoothing=0.1)
  pdt_smooth_weighted  the same with class weights
  torch_smooth         torch.nn.CrossEntropyLoss(label_smoothing=0.1): the loss and its backward are ATen kernels in the graph
  k2_pdt_plain, k2_pdt_smooth   the first two with accumulation_steps=2 (two micro-batches of 100 per step)
  pdt_soft             pdt.nn.CrossEntropyLoss() on class-probability targets with two non-zeros per row, as MixUp makes them
  pdt_soft_smooth_weighted      the same with label smoothing 0.1 and class weights
  torch_soft           torch.nn.CrossEntropyLoss() on the same targets
  k2_pdt_soft          pdt_soft with accumulation_steps=2

The pdt criteria take their loss from the forward kernel's cross-entropy rider; torch's criterion computes its own, next to the
rider's unused one.  Every arm gets its own model (same initial weights) and its own GraphedTrainStep.  Inputs rotate through a
device-resident pool larger than L2, as in bench.py; the steps are timed with CUDA events, in rounds that alternate between the arms,
and the median round is reported, in ms per optimizer step.  Prints the card, its power limit and one JSON line.

Usage: python tools/loss_step_bench.py [--steps 500] [--warmup 50] [--rounds 7]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from optim_step_bench import power_limit_w  # noqa: E402

MICRO, IMG, POOL_IMAGES = 100, (1, 28, 28), 51200   # 51,200 x 784 x 4 B = 160.6 MB of images > 50 MB L2 (as bench.py)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500, help="timed optimizer steps per arm and round")
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()

    import pytorch_distributed_train_b200 as pdt
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(1234)
    xs = torch.rand((POOL_IMAGES,) + IMG, generator=g).to(dev)
    ys = torch.randint(0, 10, (POOL_IMAGES,), generator=g).to(dev)
    w = (torch.rand(10, generator=g) + 0.5).to(dev)
    # MixUp-like probability targets: λ·onehot(y) + (1 − λ)·onehot(y of the previous image), λ drawn per image
    lam = torch.rand(POOL_IMAGES, 1, generator=g).to(dev)
    onehot = torch.nn.functional.one_hot(ys, 10).float()
    qs = (lam * onehot + (1 - lam) * onehot.roll(1, 0)).contiguous()
    torch.manual_seed(0)
    init = pdt.models.ConvNet().to(dev).state_dict()
    criteria = {   # name: (criterion factory, accumulation steps, targets)
        "pdt_plain": (lambda: pdt.nn.CrossEntropyLoss(), 1, ys),
        "pdt_smooth": (lambda: pdt.nn.CrossEntropyLoss(label_smoothing=0.1), 1, ys),
        "pdt_smooth_weighted": (lambda: pdt.nn.CrossEntropyLoss(label_smoothing=0.1, weight=w), 1, ys),
        "torch_smooth": (lambda: torch.nn.CrossEntropyLoss(label_smoothing=0.1), 1, ys),
        "k2_pdt_plain": (lambda: pdt.nn.CrossEntropyLoss(), 2, ys),
        "k2_pdt_smooth": (lambda: pdt.nn.CrossEntropyLoss(label_smoothing=0.1), 2, ys),
        "pdt_soft": (lambda: pdt.nn.CrossEntropyLoss(), 1, qs),
        "pdt_soft_smooth_weighted": (lambda: pdt.nn.CrossEntropyLoss(label_smoothing=0.1, weight=w), 1, qs),
        "torch_soft": (lambda: torch.nn.CrossEntropyLoss(), 1, qs),
        "k2_pdt_soft": (lambda: pdt.nn.CrossEntropyLoss(), 2, qs),
    }
    arms = {}
    for name, (make, k, ts) in criteria.items():
        model = pdt.models.ConvNet().to(dev)
        model.load_state_dict(init)
        opt = pdt.optim.SGD(list(model.parameters()), 1e-4)
        step = GraphedTrainStep(model, make(), opt, (xs[:k * MICRO], ts[:k * MICRO]), warmup=3, accumulation_steps=k)
        if hasattr(opt, "stop_riding"):
            opt.stop_riding()   # the captured graph keeps the rider; disarm it so that the next model captures on its own
        arms[name] = (step, k, ts)

    def run(name, n, base):
        step, k, ts = arms[name]
        rows = k * MICRO
        for i in range(n):
            j = ((base + i) * rows) % (POOL_IMAGES - rows + 1)
            step(xs[j:j + rows], ts[j:j + rows], inputs_ready=True)

    per = {name: [] for name in arms}
    for r in range(args.rounds):
        for name in arms:
            step = arms[name][0]
            run(name, args.warmup, 0)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(name, args.steps, args.warmup)
            e1.record()
            torch.cuda.synchronize()
            per[name].append(e0.elapsed_time(e1) / args.steps)
            loss = float(step.static_loss.detach())
            assert loss == loss, f"{name}: loss is NaN"
    med = {name: statistics.median(v) for name, v in per.items()}
    result = {
        "card": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(),
        "micro_batch": MICRO,
        "steps_per_round": args.steps,
        "rounds": args.rounds,
        "kernels_per_replay": {name: arms[name][0].kernels_per_replay for name in arms},
        "accumulates_in_kernel": {name: arms[name][0].accumulates_in_kernel for name in arms if arms[name][1] > 1},
        "us_per_step_median": {name: round(v * 1e3, 2) for name, v in med.items()},
        "us_per_step_min": {name: round(min(v) * 1e3, 2) for name, v in per.items()},
    }
    print(f"{result['card']}, power limit {result['power_limit_w']} W")
    for name in arms:
        print(f"  {name:24s} {result['us_per_step_median'][name]:8.2f} us/step (median of {args.rounds} rounds, min "
              f"{result['us_per_step_min'][name]:.2f})  {result['kernels_per_replay'][name]} own kernels per replay")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
