#!/usr/bin/env python
"""Device time of one graphed training step of the reference ConvNet (batch 100, one GPU) with twenty-nine optimizers:

  pdt SGD, pdt Adam, pdt AdamW               (native update; on one GPU it rides on the last backward kernel)
  pdt AdamW(amsgrad=True)                    (the same with the running maximum max_exp_avg_sq: AmsgradRider)
  pdt RMSprop, pdt RMSprop(momentum=0.9, centered=True), pdt Adagrad   (RmspropRider, AdagradRider)
  pdt NAdam, pdt RAdam                       (NadamRider, RadamRider)
  pdt NAdam, pdt RAdam, not riding           (GraphedTrainStep(fuse_optimizer=False): the multi-tensor kernel after backward)
  pdt Adamax, Adadelta, ASGD, Rprop          (AdamaxRider, AdadeltaRider, AsgdRider, RpropRider)
  pdt Adamax, Adadelta, ASGD, Rprop, not riding
  torch AdamW(capturable=True, foreach=True) (torch's multi-tensor kernels, replayed inside the same graph)
  torch AdamW(capturable=True, fused=True)   (torch's fused kernel, replayed inside the same graph)
  torch AdamW(amsgrad=True, capturable=True, fused=True)
  torch RMSprop(capturable=True, foreach=True)
  torch NAdam(capturable=True, foreach=True), torch RAdam(capturable=True, foreach=True)
  torch Adamax / Adadelta / ASGD / Rprop(capturable=True, foreach=True)

torch's Adagrad has no arm: it computes its decayed learning rate on the host from a CPU step count, so a captured step would
replay the captured rate.

With ``--max-grad-norm X`` ten more arms clip the global gradient norm to X in the same rounds:

  pdt SGD / AdamW / NAdam / RAdam / Adamax / Adadelta / ASGD / Rprop with clipping, riding   (the last backward kernel clips, then
                                                                                            updates: still 3 launches)
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
        "pdt_rmsprop": lambda ps: pdt.optim.RMSprop(ps, lr),
        "pdt_rmsprop_centered_momentum": lambda ps: pdt.optim.RMSprop(ps, lr, momentum=0.9, centered=True),
        "pdt_adagrad": lambda ps: pdt.optim.Adagrad(ps, lr),
        "pdt_nadam": lambda ps: pdt.optim.NAdam(ps, lr),
        "pdt_radam": lambda ps: pdt.optim.RAdam(ps, lr),
        "pdt_nadam_unfused": lambda ps: pdt.optim.NAdam(ps, lr),
        "pdt_radam_unfused": lambda ps: pdt.optim.RAdam(ps, lr),
        "pdt_adamax": lambda ps: pdt.optim.Adamax(ps, lr),
        "pdt_adadelta": lambda ps: pdt.optim.Adadelta(ps, lr),
        "pdt_asgd": lambda ps: pdt.optim.ASGD(ps, lr),
        "pdt_rprop": lambda ps: pdt.optim.Rprop(ps, lr),
        "pdt_adamax_unfused": lambda ps: pdt.optim.Adamax(ps, lr),
        "pdt_adadelta_unfused": lambda ps: pdt.optim.Adadelta(ps, lr),
        "pdt_asgd_unfused": lambda ps: pdt.optim.ASGD(ps, lr),
        "pdt_rprop_unfused": lambda ps: pdt.optim.Rprop(ps, lr),
        "torch_adamw_foreach": lambda ps: torch.optim.AdamW(ps, lr, capturable=True, foreach=True),
        "torch_adamw_fused": lambda ps: torch.optim.AdamW(ps, lr, capturable=True, fused=True),
        "torch_adamw_amsgrad_fused": lambda ps: torch.optim.AdamW(ps, lr, amsgrad=True, capturable=True, fused=True),
        "torch_rmsprop_foreach": lambda ps: torch.optim.RMSprop(ps, lr, capturable=True, foreach=True),
        "torch_nadam_foreach": lambda ps: torch.optim.NAdam(ps, lr, capturable=True, foreach=True),
        "torch_radam_foreach": lambda ps: torch.optim.RAdam(ps, lr, capturable=True, foreach=True),
        "torch_adamax_foreach": lambda ps: torch.optim.Adamax(ps, lr, capturable=True, foreach=True),
        "torch_adadelta_foreach": lambda ps: torch.optim.Adadelta(ps, lr, capturable=True, foreach=True),
        "torch_asgd_foreach": lambda ps: torch.optim.ASGD(ps, lr, capturable=True, foreach=True),
        "torch_rprop_foreach": lambda ps: torch.optim.Rprop(ps, lr, capturable=True, foreach=True),
    }
    # name -> GraphedTrainStep keyword arguments of the arm
    kwargs = {name: {} for name in makers}
    kwargs.update({name: {"fuse_optimizer": False} for name in makers if name.endswith("_unfused")})
    if args.max_grad_norm is not None:
        mg = args.max_grad_norm
        makers.update({
            "pdt_sgd_clip": lambda ps: pdt.optim.SGD(ps, lr),
            "pdt_adamw_clip": lambda ps: pdt.optim.AdamW(ps, lr),
            "pdt_nadam_clip": lambda ps: pdt.optim.NAdam(ps, lr),
            "pdt_radam_clip": lambda ps: pdt.optim.RAdam(ps, lr),
            "pdt_adamax_clip": lambda ps: pdt.optim.Adamax(ps, lr),
            "pdt_adadelta_clip": lambda ps: pdt.optim.Adadelta(ps, lr),
            "pdt_asgd_clip": lambda ps: pdt.optim.ASGD(ps, lr),
            "pdt_rprop_clip": lambda ps: pdt.optim.Rprop(ps, lr),
            "pdt_adamw_clip_unfused": lambda ps: pdt.optim.AdamW(ps, lr),
            "torch_clip_adamw_fused": lambda ps: _TorchClip(torch.optim.AdamW(ps, lr, capturable=True, fused=True), ps, mg),
        })
        kwargs.update({"pdt_sgd_clip": {"max_grad_norm": mg}, "pdt_adamw_clip": {"max_grad_norm": mg},
                       "pdt_nadam_clip": {"max_grad_norm": mg}, "pdt_radam_clip": {"max_grad_norm": mg},
                       "pdt_adamax_clip": {"max_grad_norm": mg}, "pdt_adadelta_clip": {"max_grad_norm": mg},
                       "pdt_asgd_clip": {"max_grad_norm": mg}, "pdt_rprop_clip": {"max_grad_norm": mg},
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
        print(f"  {name:30s} {result['ms_per_step_median'][name]:.4f} ms/step (median of {args.rounds} rounds)  "
              f"{result['kernels_per_replay'][name]} own kernels per replay")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
