#!/usr/bin/env python
"""Cost of per-image random affine and elastic augmentation in the graphed training step of the reference ConvNet (batch 100, one
GPU, pdt SGD riding on the last backward kernel), with torchvision's RandomAffine(15, (0.1, 0.1), (0.9, 1.1)) and
ElasticTransform(alpha=50, sigma=5) (its defaults: bilinear, fill 0) definitions:

  none               no augmentation
  native             GraphedTrainStep(augment=pdt.data.RandomAffine(...)): one more launch inside the graph
  torch_ops          the same augmentation as torch ops inside the same graph: device draws (torch.rand), the per-image theta,
                     F.affine_grid + F.grid_sample on the images with a ones channel appended, and the fill where the mask is < 0.5
  elastic            GraphedTrainStep(augment=pdt.data.ElasticTransform()): one more launch inside the graph
  affine_elastic     GraphedTrainStep(augment=[RandomAffine(...), ElasticTransform()]): two more launches
  elastic_torch_ops  the elastic transform as torch ops inside the same graph: torch.rand, a reflect pad, a depthwise 41x41
                     F.conv2d, the identity grid plus the displacement, and F.grid_sample with a mask channel
  torchvision        host images/s of torchvision.transforms.v2.RandomAffine and of v2.ElasticTransform as a per-sample transform=
                     of pdt.data.MNIST through pdt.DataLoader (no GPU work; only when torchvision is importable)

The device arms are device times from CUDA events; inputs rotate through a device-resident pool larger than L2, as in bench.py,
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
ELASTIC_ALPHA, ELASTIC_SIGMA = 50.0, 5.0


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


class TorchOpsElastic:
    """ElasticTransform(50, 5) with bilinear sampling and fill 0 as torch ops, capturable: the comparison arm."""

    def __init__(self, device, H=28, W=28):
        from pytorch_distributed_train_b200.data.elastic import _gaussian_kernel1d

        self.k = int(8 * ELASTIC_SIGMA + 1) | 1
        w = _gaussian_kernel1d(self.k, ELASTIC_SIGMA)
        self.kernel = (w.unsqueeze(-1) * w).expand(2, 1, self.k, self.k).contiguous().to(device)
        self.scale = torch.tensor([ELASTIC_ALPHA / W, ELASTIC_ALPHA / H], device=device).view(1, 2, 1, 1)
        xs = torch.linspace((-W + 1) / W, (W - 1) / W, W, device=device)
        ys = torch.linspace((-H + 1) / H, (H - 1) / H, H, device=device)
        self.identity = torch.stack([xs.view(1, W).expand(H, W), ys.view(H, 1).expand(H, W)], -1).unsqueeze(0)

    def __call__(self, x):
        B, C, H, W = x.shape
        d = torch.rand(B, 2, H, W, device=x.device) * 2 - 1
        d = F.conv2d(F.pad(d, [self.k // 2] * 4, mode="reflect"), self.kernel, groups=2) * self.scale
        grid = self.identity + d.permute(0, 2, 3, 1)
        out = F.grid_sample(torch.cat([x, torch.ones_like(x[:, :1])], 1), grid, mode="bilinear", padding_mode="zeros", align_corners=False)
        return out[:, :C] * out[:, C:]   # torchvision's (img − fill)·mask + fill at fill 0


def torchvision_images_per_s(n, transform):
    import pytorch_distributed_train_b200 as pdt

    with tempfile.TemporaryDirectory() as root:
        ds = pdt.data.MNIST(root=root, train=False, synthetic_fallback=True, transform=transform)
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

    augments = {"none": None, "native": pdt.data.RandomAffine(DEGREES, TRANSLATE, SCALE), "torch_ops": TorchOpsAffine(),
                "elastic": pdt.data.ElasticTransform(ELASTIC_ALPHA, ELASTIC_SIGMA),
                "affine_elastic": [pdt.data.RandomAffine(DEGREES, TRANSLATE, SCALE), pdt.data.ElasticTransform(ELASTIC_ALPHA, ELASTIC_SIGMA)],
                "elastic_torch_ops": TorchOpsElastic(dev)}
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
    try:
        from torchvision.transforms import v2
        host = {"RandomAffine": torchvision_images_per_s(args.host_images, v2.RandomAffine(DEGREES, TRANSLATE, SCALE)),
                "ElasticTransform": torchvision_images_per_s(args.host_images, v2.ElasticTransform(ELASTIC_ALPHA, ELASTIC_SIGMA))}
    except ImportError:
        host = None
    result = {
        "card": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(),
        "batch": BATCH,
        "augment": f"RandomAffine({DEGREES}, {TRANSLATE}, {SCALE}), nearest, fill 0; ElasticTransform({ELASTIC_ALPHA}, {ELASTIC_SIGMA}), "
                   "bilinear, fill 0",
        "steps_per_round": args.steps,
        "rounds": args.rounds,
        "kernels_per_replay": {name: step.kernels_per_replay for name, step in arms.items()},
        "us_per_step_median": {name: round(statistics.median(v), 2) for name, v in per.items()},
        "us_per_step_min": {name: round(min(v), 2) for name, v in per.items()},
        "torchvision_per_sample_images_per_s": None if host is None else {name: round(v, 1) for name, v in host.items()},
    }
    print(f"{result['card']}, power limit {result['power_limit_w']} W")
    for name in arms:
        print(f"  {name:18s} {result['us_per_step_median'][name]:8.2f} us/step (median of {args.rounds} rounds, device clock)")
    for name, v in (host or {}).items():
        print(f"  torchvision per-sample {name} through pdt.DataLoader: {v:.0f} images/s (host clock)")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
