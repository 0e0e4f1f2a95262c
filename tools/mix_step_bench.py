#!/usr/bin/env python
"""Cost of batch-level CutMix and MixUp in the graphed training step of the reference ConvNet (batch 100, one GPU, pdt SGD riding
on the last backward kernel), α = 1:

  none            no mixing
  cutmix          GraphedTrainStep(mix=pdt.data.CutMix(...)): one more launch inside the graph
  mixup           GraphedTrainStep(mix=pdt.data.MixUp(...)): likewise
  affine_cutmix   RandomAffine(15, (0.1, 0.1), (0.9, 1.1)) then CutMix, both native: two more launches
  torch_ops       CutMix as torch ops captured in the same graph: λ from torch._sample_dirichlet and r_x, r_y from torch.randint on
                  the device, a box mask, roll and one_hot
  torchvision     host clock: torchvision.transforms.v2.CutMix applied eagerly to the device batch before each step (it draws on the
                  host and reads the box back), then the graphed step on its fp32 targets (only when torchvision is importable)

The first five are device times from CUDA events; inputs rotate through a device-resident pool larger than L2, as in bench.py,
and the arms alternate within every round so that clock drift hits all of them alike.  Prints the card, its power limit and one
JSON line with the medians over the rounds.

Usage: python tools/mix_step_bench.py [--steps 500] [--warmup 50] [--rounds 5]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BATCH, IMG, POOL_BATCHES, CLASSES, ALPHA = 100, (1, 28, 28), 512, 10, 1.0   # 512 x 100 x 784 x 4 B = 160.6 MB of images > 50 MB L2


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


class TorchOpsCutMix:
    """CutMix(α) as torch ops, capturable: the comparison arm."""

    def __init__(self, device):
        self.conc = torch.full((2,), ALPHA, device=device)

    def __call__(self, x, y):
        B, C, H, W = x.shape
        lam = torch._sample_dirichlet(self.conc)[0].double()
        rx = torch.randint(W, (1,), device=x.device)
        ry = torch.randint(H, (1,), device=x.device)
        r = 0.5 * torch.sqrt(1.0 - lam)
        rw, rh = (r * W).long(), (r * H).long()
        x1, y1 = (rx - rw).clamp(min=0), (ry - rh).clamp(min=0)
        x2, y2 = (rx + rw).clamp(max=W), (ry + rh).clamp(max=H)
        cols, rows = torch.arange(W, device=x.device), torch.arange(H, device=x.device)
        mask = ((rows >= y1) & (rows < y2)).view(H, 1) & ((cols >= x1) & (cols < x2)).view(1, W)
        out = torch.where(mask, x.roll(1, 0), x)
        lam_adj = 1.0 - ((x2 - x1) * (y2 - y1)).double() / (W * H)
        onehot = F.one_hot(y, CLASSES).float()
        return out, onehot.roll(1, 0) * (1.0 - lam_adj).float() + onehot * lam_adj.float()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500, help="timed steps per arm and round")
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import pytorch_distributed_train_b200 as pdt
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(1234)
    xs = torch.rand((POOL_BATCHES, BATCH) + IMG, generator=g).to(dev)
    ys = torch.randint(0, CLASSES, (POOL_BATCHES, BATCH), generator=g).to(dev)
    torch.manual_seed(0)
    init = pdt.models.ConvNet().to(dev).state_dict()
    crit = pdt.nn.CrossEntropyLoss()

    def affine():
        return pdt.data.RandomAffine(15.0, (0.1, 0.1), (0.9, 1.1))

    configs = {
        "none": dict(),
        "cutmix": dict(mix=pdt.data.CutMix(alpha=ALPHA, num_classes=CLASSES)),
        "mixup": dict(mix=pdt.data.MixUp(alpha=ALPHA, num_classes=CLASSES)),
        "affine_cutmix": dict(augment=affine(), mix=pdt.data.CutMix(alpha=ALPHA, num_classes=CLASSES)),
        "torch_ops": dict(mix=TorchOpsCutMix(dev)),
    }

    def make_step(example_targets, **kw):
        model = pdt.models.ConvNet().to(dev)
        model.load_state_dict(init)
        opt = pdt.optim.SGD(model.parameters(), 1e-3)
        step = GraphedTrainStep(model, crit, opt, (xs[0], example_targets), warmup=3, **kw)
        opt.stop_riding()   # the captured graph keeps the rider; disarm it so that the next model captures on its own
        return step

    arms, failed = {}, {}
    for name, kw in configs.items():
        try:
            arms[name] = make_step(ys[0], **kw)
        except Exception as e:   # noqa: BLE001  (an arm that cannot be captured is reported, not fatal)
            failed[name] = f"{type(e).__name__}: {e}"[:300]

    def run(name, n, base):
        step = arms[name]
        for i in range(n):
            j = (base + i) % POOL_BATCHES
            step(xs[j], ys[j], inputs_ready=True)

    def device_time(name):
        run(name, args.warmup, 0)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(name, args.steps, args.warmup)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / args.steps

    tv_step = tv = None
    try:
        from torchvision.transforms import v2

        tv = v2.CutMix(alpha=ALPHA, num_classes=CLASSES)
        tv_step = make_step(torch.zeros(BATCH, CLASSES, device=dev))
    except Exception:   # noqa: BLE001  (torchvision is optional)
        tv = None

    def torchvision_time():
        def go(n, base):
            for i in range(n):
                j = (base + i) % POOL_BATCHES
                tv_step(*tv(xs[j], ys[j]))
        go(args.warmup, 0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        go(args.steps, args.warmup)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e6 / args.steps

    per = {name: [] for name in arms}
    host = []
    for _ in range(args.rounds):
        for name in arms:
            per[name].append(device_time(name))
        if tv is not None:
            host.append(torchvision_time())
    for name, step in arms.items():
        loss = float(step.static_loss.detach())
        assert math.isfinite(loss), f"{name}: loss {loss}"
    result = {
        "card": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(),
        "batch": BATCH,
        "alpha": ALPHA,
        "steps_per_round": args.steps,
        "rounds": args.rounds,
        "kernels_per_replay": {name: step.kernels_per_replay for name, step in arms.items()},
        "us_per_step_median": {name: round(statistics.median(v), 2) for name, v in per.items()},
        "us_per_step_min": {name: round(min(v), 2) for name, v in per.items()},
        "torchvision_eager_us_per_step_host_median": round(statistics.median(host), 2) if host else None,
        "failed_arms": failed,
    }
    print(f"{result['card']}, power limit {result['power_limit_w']} W")
    for name in arms:
        print(f"  {name:14s} {result['us_per_step_median'][name]:8.2f} us/step (median of {args.rounds} rounds, device clock)")
    if host:
        print(f"  torchvision v2.CutMix eagerly + graphed step: {result['torchvision_eager_us_per_step_host_median']:.2f} us/step (host clock)")
    for name, why in failed.items():
        print(f"  {name}: not measured ({why})")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
