#!/usr/bin/env python
"""Device time of one graphed training step of the reference ConvNet (batch 100, one GPU) with seven optimizers:

  pdt SGD, pdt Adam, pdt AdamW               (native update; on one GPU it rides on the last backward kernel)
  pdt AdamW(amsgrad=True)                    (the same with the running maximum max_exp_avg_sq: AmsgradRider)
  torch AdamW(capturable=True, foreach=True) (torch's multi-tensor kernels, replayed inside the same graph)
  torch AdamW(capturable=True, fused=True)   (torch's fused kernel, replayed inside the same graph)
  torch AdamW(amsgrad=True, capturable=True, fused=True)

With ``--max-grad-norm X`` four more arms clip the global gradient norm to X in the same rounds:

  pdt SGD / pdt AdamW with clipping, riding   (the last backward kernel clips, then updates: still 3 launches)
  pdt AdamW with clipping, not riding          (GraphedTrainStep(fuse_optimizer=False): native clip + Adam kernel after backward)
  torch clip_grad_norm_(foreach=True) + AdamW(capturable=True, fused=True) in the same graph

Every optimizer gets its own model (same initial weights) and its own ``engine.GraphedTrainStep``.  Inputs rotate through a
device-resident pool larger than L2, as in bench.py; the steps are timed with CUDA events, in rounds that alternate between the
optimizers so that clock drift hits all of them alike.  Prints the card, its power limit and one JSON line.

Usage: python tools/optim_step_bench.py [--steps 200] [--warmup 20] [--rounds 5] [--max-grad-norm 1.0]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BATCH, IMG, POOL_BATCHES = 100, (1, 28, 28), 512   # 512 x 100 x 784 x 4 B = 160.6 MB of images > 50 MB L2 (as bench.py)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


class _TorchClip:
    """torch.optim optimizer whose step() first runs torch.nn.utils.clip_grad_norm_(foreach=True): the torch arm of the clipped
    step, captured in the same graph as ours."""

    def __init__(self, opt, params, max_norm):
        self.opt, self.params, self.max_norm = opt, params, max_norm
        self.param_groups = opt.param_groups

    def zero_grad(self, set_to_none=True):
        self.opt.zero_grad(set_to_none=set_to_none)

    def step(self):
        torch.nn.utils.clip_grad_norm_(self.params, self.max_norm, foreach=True)
        self.opt.step()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="timed steps per optimizer and round")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--max-grad-norm", type=float, default=None, help="also time the arms that clip the gradient norm to this value")
    args = ap.parse_args()

    import pytorch_distributed_train_b200 as pdt
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(1234)
    xs = torch.rand((POOL_BATCHES, BATCH) + IMG, generator=g).to(dev)
    ys = torch.randint(0, 10, (POOL_BATCHES, BATCH), generator=g).to(dev)
    torch.manual_seed(0)
    init = pdt.models.ConvNet().to(dev).state_dict()
    lr = 1e-3
    makers = {
        "pdt_sgd": lambda ps: pdt.optim.SGD(ps, lr),
        "pdt_adam": lambda ps: pdt.optim.Adam(ps, lr),
        "pdt_adamw": lambda ps: pdt.optim.AdamW(ps, lr),
        "pdt_adamw_amsgrad": lambda ps: pdt.optim.AdamW(ps, lr, amsgrad=True),
        "torch_adamw_foreach": lambda ps: torch.optim.AdamW(ps, lr, capturable=True, foreach=True),
        "torch_adamw_fused": lambda ps: torch.optim.AdamW(ps, lr, capturable=True, fused=True),
        "torch_adamw_amsgrad_fused": lambda ps: torch.optim.AdamW(ps, lr, amsgrad=True, capturable=True, fused=True),
    }
    # name -> GraphedTrainStep keyword arguments of the arm
    kwargs = {name: {} for name in makers}
    if args.max_grad_norm is not None:
        mg = args.max_grad_norm
        makers.update({
            "pdt_sgd_clip": lambda ps: pdt.optim.SGD(ps, lr),
            "pdt_adamw_clip": lambda ps: pdt.optim.AdamW(ps, lr),
            "pdt_adamw_clip_unfused": lambda ps: pdt.optim.AdamW(ps, lr),
            "torch_clip_adamw_fused": lambda ps: _TorchClip(torch.optim.AdamW(ps, lr, capturable=True, fused=True), ps, mg),
        })
        kwargs.update({"pdt_sgd_clip": {"max_grad_norm": mg}, "pdt_adamw_clip": {"max_grad_norm": mg},
                       "pdt_adamw_clip_unfused": {"max_grad_norm": mg, "fuse_optimizer": False}, "torch_clip_adamw_fused": {}})
    crit = pdt.nn.CrossEntropyLoss()
    steps = {}
    for name, make in makers.items():
        model = pdt.models.ConvNet().to(dev)
        model.load_state_dict(init)
        opt = make(list(model.parameters()))
        steps[name] = (GraphedTrainStep(model, crit, opt, (xs[0], ys[0]), warmup=3, **kwargs[name]), opt)
        if hasattr(opt, "stop_riding"):
            opt.stop_riding()   # the captured graph keeps the rider; disarm it so that the next model captures on its own

    def run(name, n, base):
        step = steps[name][0]
        for i in range(n):
            j = (base + i) % POOL_BATCHES
            step(xs[j], ys[j], inputs_ready=True)

    per = {name: [] for name in makers}
    for r in range(args.rounds):
        for name in makers:
            step, opt = steps[name]
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
    result = {
        "card": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(),
        "batch": BATCH,
        "steps_per_round": args.steps,
        "rounds": args.rounds,
        "kernels_per_replay": {name: steps[name][0].kernels_per_replay for name in makers},
        "ms_per_step_median": {name: round(statistics.median(v), 5) for name, v in per.items()},
        "ms_per_step_min": {name: round(min(v), 5) for name, v in per.items()},
        "max_grad_norm": args.max_grad_norm,
    }
    print(f"{result['card']}, power limit {result['power_limit_w']} W")
    for name in makers:
        print(f"  {name:26s} {result['ms_per_step_median'][name]:.4f} ms/step (median of {args.rounds} rounds)  "
              f"{result['kernels_per_replay'][name]} own kernels per replay")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
