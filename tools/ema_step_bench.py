#!/usr/bin/env python
"""Time of one graphed training step of the reference ConvNet (batch 100, one GPU, pdt SGD riding on the last backward kernel)
with and without an EMA of the weights and buffers (``AveragedModel(model, get_ema_multi_avg_fn(0.999), use_buffers=True)``):

  none          no averaging
  native        GraphedTrainStep(averaged_model=...): the native update is one more launch inside the graph
  torch_after   torch's AveragedModel.update_parameters(model) after every replay, outside the graph

The first two are timed with CUDA events.  torch's update reads ``n_averaged`` on the host, so that arm synchronises on every
step anyway; it is timed on the host clock around the steps and a final synchronise, and so is the ``none`` arm again
(``none_host``) for a like-for-like comparison.  Inputs rotate through a device-resident pool larger than L2, as in bench.py; the
arms alternate within every round so that clock drift hits all of them alike.  Prints the card, its power limit and one JSON line.

Usage: python tools/ema_step_bench.py [--steps 500] [--warmup 50] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BATCH, IMG, POOL_BATCHES = 100, (1, 28, 28), 512   # 512 x 100 x 784 x 4 B = 160.6 MB of images > 50 MB L2 (as bench.py)
DECAY = 0.999


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500, help="timed steps per arm and round")
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import pytorch_distributed_train_b200 as pdt
    from pytorch_distributed_train_b200.engine import GraphedTrainStep
    from pytorch_distributed_train_b200.optim import swa_utils

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(1234)
    xs = torch.rand((POOL_BATCHES, BATCH) + IMG, generator=g).to(dev)
    ys = torch.randint(0, 10, (POOL_BATCHES, BATCH), generator=g).to(dev)
    torch.manual_seed(0)
    init = pdt.models.ConvNet().to(dev).state_dict()
    crit = pdt.nn.CrossEntropyLoss()

    arms = {}   # name -> (GraphedTrainStep, torch AveragedModel updated after each replay or None)
    for name in ("none", "native", "torch_after"):
        model = pdt.models.ConvNet().to(dev)
        model.load_state_dict(init)
        opt = pdt.optim.SGD(model.parameters(), 1e-3)
        ours = swa_utils.AveragedModel(model, multi_avg_fn=swa_utils.get_ema_multi_avg_fn(DECAY), use_buffers=True) if name == "native" else None
        after = (torch.optim.swa_utils.AveragedModel(model, device=dev, multi_avg_fn=torch.optim.swa_utils.get_ema_multi_avg_fn(DECAY),
                                                     use_buffers=True) if name == "torch_after" else None)
        step = GraphedTrainStep(model, crit, opt, (xs[0], ys[0]), warmup=3, averaged_model=ours)
        opt.stop_riding()   # the captured graph keeps the rider; disarm it so that the next model captures on its own
        arms[name] = (step, after, model)

    def run(name, n, base):
        step, after, model = arms[name]
        for i in range(n):
            j = (base + i) % POOL_BATCHES
            step(xs[j], ys[j], inputs_ready=True)
            if after is not None:
                after.update_parameters(model)

    def device_time(name):
        run(name, args.warmup, 0)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(name, args.steps, args.warmup)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    def host_time(name):
        run(name, args.warmup, 0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(name, args.steps, args.warmup)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / args.steps

    timed = {"none": device_time, "native": device_time, "none_host": lambda _: host_time("none"), "torch_after": host_time}
    per = {name: [] for name in timed}
    for _ in range(args.rounds):
        for name, fn in timed.items():
            per[name].append(fn(name))
    for name, (step, _, _) in arms.items():
        loss = float(step.static_loss)
        assert loss == loss, f"{name}: loss is NaN"
    result = {
        "card": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(),
        "batch": BATCH,
        "decay": DECAY,
        "steps_per_round": args.steps,
        "rounds": args.rounds,
        "kernels_per_replay": {name: arms[name][0].kernels_per_replay for name in arms},
        "ms_per_step_median": {name: round(statistics.median(v), 5) for name, v in per.items()},
        "ms_per_step_min": {name: round(min(v), 5) for name, v in per.items()},
        "clock": {"none": "device", "native": "device", "none_host": "host", "torch_after": "host"},
    }
    print(f"{result['card']}, power limit {result['power_limit_w']} W")
    for name in timed:
        print(f"  {name:12s} {result['ms_per_step_median'][name]:.4f} ms/step (median of {args.rounds} rounds, {result['clock'][name]} clock)")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
