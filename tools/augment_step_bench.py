#!/usr/bin/env python
"""Cost of per-image random affine augmentation in the graphed training step of the reference ConvNet (batch 100, one GPU, pdt
SGD riding on the last backward kernel), with torchvision's RandomAffine(15, (0.1, 0.1), (0.9, 1.1)) definition:

  none        no augmentation
  native      GraphedTrainStep(augment=pdt.data.RandomAffine(...)): one more launch inside the graph
  torch_ops   the same augmentation as torch ops inside the same graph: device draws (torch.rand), the per-image theta,
              F.affine_grid + F.grid_sample on the images with a ones channel appended, and the fill where the mask is < 0.5
  torchvision host images/s of torchvision.transforms.v2.RandomAffine as a per-sample transform= of pdt.data.MNIST through
              pdt.DataLoader (no GPU work; only when torchvision is importable)

The first three are device times from CUDA events; inputs rotate through a device-resident pool larger than L2, as in bench.py,
and the arms alternate within every round so that clock drift hits all of them alike.  Prints the card, its power limit and one
JSON line with the medians over the rounds.

Usage: python tools/augment_step_bench.py [--steps 500] [--warmup 50] [--rounds 5] [--host-images 2000]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BATCH, IMG, POOL_BATCHES = 100, (1, 28, 28), 512   # 512 x 100 x 784 x 4 B = 160.6 MB of images > 50 MB L2 (as bench.py)
DEGREES, TRANSLATE, SCALE = 15.0, (0.1, 0.1), (0.9, 1.1)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


class TorchOpsAffine:
    """RandomAffine(15, (0.1, 0.1), (0.9, 1.1)) with nearest sampling and fill 0 as torch ops, capturable: the comparison arm."""

    def __call__(self, x):
        B, C, H, W = x.shape
        r = torch.rand(B, 4, device=x.device)
        angle = (r[:, 0] * 2 - 1) * DEGREES
        tx = torch.round((r[:, 1] * 2 - 1) * (TRANSLATE[0] * W))
        ty = torch.round((r[:, 2] * 2 - 1) * (TRANSLATE[1] * H))
        s = SCALE[0] + r[:, 3] * (SCALE[1] - SCALE[0])
        rot = angle * (math.pi / 180)
        cos, sin = torch.cos(rot) / s, torch.sin(rot) / s
        # torchvision's inverse matrix without shear, in pixels about the centre, then normalised for affine_grid(align_corners=False)
        m2 = -(cos * tx + sin * ty)
        m5 = -(-sin * tx + cos * ty)
        theta = torch.stack([torch.stack([cos, sin * (H / W), m2 * (2 / W)], 1),
                             torch.stack([-sin * (W / H), cos, m5 * (2 / H)], 1)], 1)
        grid = F.affine_grid(theta, [B, C + 1, H, W], align_corners=False)
        out = F.grid_sample(torch.cat([x, torch.ones_like(x[:, :1])], 1), grid, mode="nearest", padding_mode="zeros", align_corners=False)
        img, mask = out[:, :C], out[:, C:]
        return torch.where(mask < 0.5, torch.zeros((), device=x.device), img)


def torchvision_images_per_s(n):
    try:
        from torchvision.transforms import v2
    except Exception:   # noqa: BLE001
        return None
    import pytorch_distributed_train_b200 as pdt

    with tempfile.TemporaryDirectory() as root:
        ds = pdt.data.MNIST(root=root, train=False, synthetic_fallback=True, transform=v2.RandomAffine(DEGREES, TRANSLATE, SCALE))
        loader = pdt.data.DataLoader(ds, batch_size=BATCH, shuffle=False)
        seen, t0 = 0, time.perf_counter()
        for images, _ in loader:
            seen += images.shape[0]
            if seen >= n:
                break
        return seen / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500, help="timed steps per arm and round")
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-images", type=int, default=2000, help="images through torchvision's per-sample transform")
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
    crit = pdt.nn.CrossEntropyLoss()

    augments = {"none": None, "native": pdt.data.RandomAffine(DEGREES, TRANSLATE, SCALE), "torch_ops": TorchOpsAffine()}
    arms = {}
    for name, aug in augments.items():
        model = pdt.models.ConvNet().to(dev)
        model.load_state_dict(init)
        opt = pdt.optim.SGD(model.parameters(), 1e-3)
        arms[name] = GraphedTrainStep(model, crit, opt, (xs[0], ys[0]), warmup=3, augment=aug)
        opt.stop_riding()   # the captured graph keeps the rider; disarm it so that the next model captures on its own

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

    per = {name: [] for name in arms}
    for _ in range(args.rounds):
        for name in arms:
            per[name].append(device_time(name))
    for name, step in arms.items():
        loss = float(step.static_loss.detach())
        assert math.isfinite(loss), f"{name}: loss {loss}"
    host = torchvision_images_per_s(args.host_images)
    result = {
        "card": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(),
        "batch": BATCH,
        "augment": f"RandomAffine({DEGREES}, {TRANSLATE}, {SCALE}), nearest, fill 0",
        "steps_per_round": args.steps,
        "rounds": args.rounds,
        "kernels_per_replay": {name: step.kernels_per_replay for name, step in arms.items()},
        "us_per_step_median": {name: round(statistics.median(v), 2) for name, v in per.items()},
        "us_per_step_min": {name: round(min(v), 2) for name, v in per.items()},
        "torchvision_per_sample_images_per_s": None if host is None else round(host, 1),
    }
    print(f"{result['card']}, power limit {result['power_limit_w']} W")
    for name in arms:
        print(f"  {name:10s} {result['us_per_step_median'][name]:8.2f} us/step (median of {args.rounds} rounds, device clock)")
    if host is not None:
        print(f"  torchvision per-sample RandomAffine through pdt.DataLoader: {host:.0f} images/s (host clock)")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
