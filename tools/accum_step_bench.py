#!/usr/bin/env python
"""Device time of one graphed training step of the reference ConvNet with gradient accumulation (one GPU, micro-batches of 100):

  k in {1, 2, 4}  x  pdt SGD, pdt AdamW  x  in-kernel accumulation, autograd accumulation

"in_kernel" is GraphedTrainStep(accumulation_steps=k) as it is: micro-batches 2..k add into the gradients inside the fused backward
kernels and the update rides on the last one (3k launches).  "autograd" runs the same kernels but lets autograd add each micro-batch's
temporaries (AccumulateGrad) and runs the optimizer after the last backward (the engine's private switch
GraphedTrainStep._accumulate_in_kernel = False).  At k = 1 the two are the same step.

Every arm gets its own model (same initial weights) and its own GraphedTrainStep.  Inputs rotate through a device-resident pool larger
than L2, as in bench.py; the steps are timed with CUDA events, in rounds that alternate between the arms.  Reports ms per optimizer step
and images per second.  Prints the card, its power limit and one JSON line.

Usage: python tools/accum_step_bench.py [--steps 200] [--warmup 20] [--rounds 5]
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
    ap.add_argument("--steps", type=int, default=200, help="timed optimizer steps per arm and round")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import pytorch_distributed_train_b200 as pdt
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(1234)
    xs = torch.rand((POOL_IMAGES,) + IMG, generator=g).to(dev)
    ys = torch.randint(0, 10, (POOL_IMAGES,), generator=g).to(dev)
    torch.manual_seed(0)
    init = pdt.models.ConvNet().to(dev).state_dict()
    lr = 1e-3
    makers = {"sgd": lambda ps: pdt.optim.SGD(ps, lr), "adamw": lambda ps: pdt.optim.AdamW(ps, lr)}
    crit = pdt.nn.CrossEntropyLoss()
    arms = {}
    for k in (1, 2, 4):
        for opt_name, make in makers.items():
            for mode in (("in_kernel",) if k == 1 else ("in_kernel", "autograd")):
                model = pdt.models.ConvNet().to(dev)
                model.load_state_dict(init)
                opt = make(list(model.parameters()))
                GraphedTrainStep._accumulate_in_kernel = mode == "in_kernel"
                try:
                    step = GraphedTrainStep(model, crit, opt, (xs[:k * MICRO], ys[:k * MICRO]), warmup=3, accumulation_steps=k)
                finally:
                    GraphedTrainStep._accumulate_in_kernel = True
                if hasattr(opt, "stop_riding"):
                    opt.stop_riding()   # the captured graph keeps the rider; disarm it so that the next model captures on its own
                if k > 1:
                    assert step.accumulates_in_kernel == (mode == "in_kernel"), (k, opt_name, mode)
                arms[f"k{k}_{opt_name}_{mode}"] = (step, k)

    def run(name, n, base):
        step, k = arms[name]
        rows = k * MICRO
        for i in range(n):
            j = ((base + i) * rows) % (POOL_IMAGES - rows + 1)
            step(xs[j:j + rows], ys[j:j + rows], inputs_ready=True)

    per = {name: [] for name in arms}
    for r in range(args.rounds):
        for name in arms:
            step, _ = arms[name]
            run(name, args.warmup, 0)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(name, args.steps, args.warmup)
            e1.record()
            torch.cuda.synchronize()
            per[name].append(e0.elapsed_time(e1) / args.steps)
            loss = float(step.static_loss)
            assert loss == loss, f"{name}: loss is NaN"
    med = {name: statistics.median(v) for name, v in per.items()}
    result = {
        "card": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(),
        "micro_batch": MICRO,
        "steps_per_round": args.steps,
        "rounds": args.rounds,
        "kernels_per_replay": {name: arms[name][0].kernels_per_replay for name in arms},
        "ms_per_step_median": {name: round(v, 5) for name, v in med.items()},
        "ms_per_step_min": {name: round(min(v), 5) for name, v in per.items()},
        "images_per_s": {name: round(arms[name][1] * MICRO / (v * 1e-3)) for name, v in med.items()},
    }
    print(f"{result['card']}, power limit {result['power_limit_w']} W")
    for name in arms:
        print(f"  {name:22s} {result['ms_per_step_median'][name]:.4f} ms/step (median of {args.rounds} rounds)  "
              f"{result['images_per_s'][name]:>9d} images/s  {result['kernels_per_replay'][name]} own kernels per replay")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
