"""Training entry point — the framework's equivalent of the reference script
(ref: ddp_example.py:47-115).  Same four flags with the same names and defaults
(``-g/--gpus``, ``--epochs``, ``--backend``, ``--syncbn``; ref: ddp_example.py:103-106), same
stdout lines (``Rank id:``, ``Use SyncBN in training``, ``Epoch [e/E], Step [i/N], Loss: x``,
``Training complete in:``; ref: ddp_example.py:49,56,94,97), same flow: spawn one process per
GPU → init_process_group over TCP → seed → model → optional SyncBN → DDP → sampler/loader → loop.

Extra flags cover what the reference hard-codes: ``--init-method`` (its LAN address
``tcp://10.9.1.2:34567`` only works on the author's network, ref: ddp_example.py:110; we default
to loopback with a free port), ``--data synthetic|mnist``, ``--model``, ``--comm fused|nccl``, ``--algo``,
``--steps``, ``--graph`` (whole-step CUDA graph), ``--batch-size``, ``--optimizer`` (sgd | adam | adamw | nadam | radam | rmsprop |
adagrad | adamax | adadelta | asgd | rprop), ``--lr``, ``--momentum``, ``--amsgrad``, ``--weight-decay``, ``--clip-grad-norm``, ``--accumulation-steps``, ``--label-smoothing``, ``--mixup``,
``--ema-decay``, ``--checkpoint`` / ``--resume``, ``--eval`` (test loss and accuracy after every epoch).
"""
from __future__ import annotations

import argparse
import contextlib
import socket
import sys
from datetime import datetime

import torch


def _free_port() -> int:
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="H100-native DDP training (MNIST ConvNet / ResNet-18)")
    p.add_argument("-g", "--gpus", default=1, type=int, help="number of gpus per node")
    p.add_argument("--epochs", default=2, type=int, metavar="N", help="number of total epochs to run")
    p.add_argument("--backend", default="nccl", type=str, help="backend used for distributed train (nccl | gloo)")
    p.add_argument("--syncbn", default=False, action="store_true", help="whether to use syncbn while training")
    p.add_argument("--init-method", default=None, type=str, help="rendezvous URL (default: tcp://127.0.0.1:<free port>)")
    p.add_argument("--comm", default="fused", choices=["fused", "nccl"],
                   help="GPU collectives: our fused NVLink kernels (default) or the libnccl baseline")
    p.add_argument("--algo", default="auto", choices=["auto", "oneshot", "oneshot_mc", "twoshot", "nvls"],
                   help="allreduce algorithm of the fused backend (auto: by message size and world size; sets PDT_AR_ALGO)")
    p.add_argument("--data", default="synthetic", choices=["synthetic", "mnist"], help="dataset (no network: synthetic default)")
    p.add_argument("--data-root", default="./data", type=str)
    p.add_argument("--model", default="convnet", choices=["convnet", "resnet18"])
    p.add_argument("--batch-size", default=100, type=int, help="per-GPU batch size (reference: 100)")
    p.add_argument("--optimizer", default="sgd",
                   choices=["sgd", "adam", "adamw", "nadam", "radam", "rmsprop", "adagrad", "adamax", "adadelta", "asgd", "rprop"],
                   help="optimizer: SGD (the reference's), Adam, AdamW, NAdam, RAdam, RMSprop, Adagrad, Adamax, Adadelta, ASGD or Rprop, "
                        "each a native multi-tensor kernel with torch's defaults")
    p.add_argument("--lr", default=1e-4, type=float, help="learning rate (reference: 1e-4)")
    p.add_argument("--momentum", default=None, type=float, help="SGD momentum (default 0; not accepted with the other optimizers)")
    p.add_argument("--amsgrad", default=False, action="store_true",
                   help="Adam / AdamW with AMSGrad: the running maximum of exp_avg_sq in the denominator (not accepted with the other "
                        "optimizers)")
    p.add_argument("--weight-decay", default=None, type=float,
                   help="weight decay (default: 0 for SGD, Adam, NAdam, RAdam, RMSprop, Adagrad, Adamax, Adadelta and ASGD, 1e-2 for "
                        "AdamW, torch's defaults; NAdam, RAdam, Adamax, Adadelta and ASGD take it as L2 decay added to the gradient; not "
                        "accepted with Rprop, which has none)")
    p.add_argument("--clip-grad-norm", default=None, type=float, metavar="MAX",
                   help="clip the global gradient norm (L2) to MAX before every optimizer step (default: off)")
    p.add_argument("--accumulation-steps", default=1, type=int, metavar="K",
                   help="gradient accumulation: K micro-batches of --batch-size images per optimizer step, each backward of loss / K "
                        "(default 1)")
    p.add_argument("--label-smoothing", default=0.0, type=float, metavar="EPS",
                   help="label smoothing of the cross-entropy loss, in [0, 1] (default 0)")
    p.add_argument("--mixup", default=None, type=float, metavar="ALPHA",
                   help="MixUp every training batch with lambda ~ Beta(ALPHA, ALPHA), ALPHA > 0, and train on the mixed class "
                        "probabilities (default: off)")
    p.add_argument("--ema-decay", default=None, type=float, metavar="D",
                   help="keep an exponential moving average of the weights and buffers with decay D in [0, 1], updated after every "
                        "optimizer step and saved with --checkpoint (default: off)")
    p.add_argument("--steps", default=0, type=int, help="stop each epoch after this many (optimizer) steps (0 = full epoch)")
    p.add_argument("--samples", default=60000, type=int, help="synthetic dataset size")
    p.add_argument("--graph", default=False, action="store_true", help="capture the whole training step in a CUDA graph")
    p.add_argument("--log-interval", default=10, type=int)
    p.add_argument("--checkpoint", default=None, type=str, help="write a checkpoint here at the end of every epoch (rank 0, atomic)")
    p.add_argument("--resume", default=None, type=str, help="restore model/optimizer/epoch from this checkpoint before training")
    p.add_argument("--eval", default=False, action="store_true",
                   help="after every epoch, print the loss and top-1 accuracy on the test split (and of the --ema-decay average)")
    p.add_argument("--set-epoch", default=False, action="store_true",
                   help="call sampler.set_epoch(e) each epoch (the reference does not)")
    return p


def make_optimizer(args, params):
    """The optimizer ``--optimizer`` / ``--lr`` / ``--momentum`` / ``--amsgrad`` / ``--weight-decay`` describe."""
    import pytorch_distributed_train_b200 as pdt

    kw = {} if args.weight_decay is None else {"weight_decay": args.weight_decay}
    if args.optimizer == "sgd":
        return pdt.optim.SGD(params, args.lr, momentum=args.momentum or 0.0, **kw)
    if args.optimizer == "rmsprop":
        return pdt.optim.RMSprop(params, args.lr, **kw)
    if args.optimizer == "adagrad":
        return pdt.optim.Adagrad(params, args.lr, **kw)
    if args.optimizer == "nadam":
        return pdt.optim.NAdam(params, args.lr, **kw)
    if args.optimizer == "radam":
        return pdt.optim.RAdam(params, args.lr, **kw)
    if args.optimizer == "adamax":
        return pdt.optim.Adamax(params, args.lr, **kw)
    if args.optimizer == "adadelta":
        return pdt.optim.Adadelta(params, args.lr, **kw)
    if args.optimizer == "asgd":
        return pdt.optim.ASGD(params, args.lr, **kw)
    if args.optimizer == "rprop":
        return pdt.optim.Rprop(params, args.lr)
    cls = pdt.optim.Adam if args.optimizer == "adam" else pdt.optim.AdamW
    return cls(params, args.lr, amsgrad=getattr(args, "amsgrad", False), **kw)


def check_args(p: argparse.ArgumentParser, args) -> None:
    if args.optimizer != "sgd" and args.momentum is not None:
        why = {"rmsprop": "RMSprop's momentum is a library option (pdt.optim.RMSprop(..., momentum=...))",
               "adagrad": "Adagrad has no momentum", "adadelta": "Adadelta has no momentum", "asgd": "ASGD has no momentum",
               "rprop": "Rprop has no momentum"}.get(args.optimizer, f"{args.optimizer} takes its moments from its betas")
        p.error(f"--momentum applies to SGD only; {why}")
    if args.optimizer not in ("adam", "adamw") and getattr(args, "amsgrad", False):
        p.error("--amsgrad applies to Adam and AdamW only (--optimizer adam | adamw)")
    if args.optimizer == "rprop" and args.weight_decay is not None:
        p.error("--weight-decay does not apply to Rprop, which has no weight decay")
    if args.clip_grad_norm is not None and not args.clip_grad_norm > 0:
        p.error(f"--clip-grad-norm must be positive (got {args.clip_grad_norm})")
    if args.accumulation_steps < 1:
        p.error(f"--accumulation-steps must be at least 1 (got {args.accumulation_steps})")
    if not 0.0 <= args.label_smoothing <= 1.0:
        p.error(f"--label-smoothing must lie in [0, 1] (got {args.label_smoothing})")
    if args.mixup is not None and not args.mixup > 0:
        p.error(f"--mixup must be positive (got {args.mixup})")
    if args.ema_decay is not None and not 0.0 <= args.ema_decay <= 1.0:
        p.error(f"--ema-decay must lie in [0, 1] (got {args.ema_decay})")
    if args.graph and args.gpus >= 2 and args.accumulation_steps > 1:
        p.error("--graph with --accumulation-steps > 1 runs on one GPU only (-g 1)")


def dist_train(gpu: int, args) -> None:
    """Per-process body: ``fn(i, *args)`` target of the launcher."""
    import pytorch_distributed_train_b200 as pdt
    from pytorch_distributed_train_b200 import data as pdata

    rank = gpu  # single node: spawn index is both global rank and device ordinal (ref: ddp_example.py:48)
    print("Rank id: ", rank)
    use_cuda = args.backend not in ("gloo", "cpu")
    if use_cuda:
        torch.cuda.set_device(gpu)
    if getattr(args, "algo", "auto") != "auto":
        import os

        os.environ["PDT_AR_ALGO"] = args.algo   # read by the fused backend when the process group is created
    pdt.init_process_group(backend=args.backend, init_method=args.init_method, world_size=args.world_size,
                           rank=rank, comm=args.comm)
    torch.manual_seed(0)
    if args.model == "convnet":
        model = pdt.models.ConvNet()
        shape, num_classes = (1, 28, 28), 10
    else:
        model = pdt.models.resnet18(num_classes=1000)
        shape, num_classes = (3, 224, 224), 1000
    if args.syncbn:
        model = pdt.SyncBatchNorm.convert_sync_batchnorm(model)
        if gpu == 0:
            print("Use SyncBN in training")
    device = torch.device("cuda", gpu) if use_cuda else torch.device("cpu")
    model.to(device)
    batch_size = args.batch_size
    accum = args.accumulation_steps
    criterion = pdt.nn.CrossEntropyLoss(label_smoothing=args.label_smoothing).to(device)
    optimizer = make_optimizer(args, model.parameters())
    ema = None
    if args.ema_decay is not None:
        from pytorch_distributed_train_b200.optim import swa_utils

        ema = swa_utils.AveragedModel(model, multi_avg_fn=swa_utils.get_ema_multi_avg_fn(args.ema_decay), use_buffers=True)
    bare = model
    model = pdt.DistributedDataParallel(model, device_ids=[gpu] if use_cuda else None)

    if args.data == "mnist" and args.model == "convnet":
        train_dataset = pdata.MNIST(root=args.data_root, train=True, download=True, synthetic_fallback=True)
    else:
        n = args.samples if args.model == "convnet" else min(args.samples, 4096)
        train_dataset = pdata.SyntheticMNIST(n, seed=0, num_classes=num_classes, image_shape=shape)
    train_sampler = pdt.DistributedSampler(train_dataset, num_replicas=args.world_size, rank=rank)
    # one loader batch = one optimizer step: `accum` micro-batches of batch_size images
    train_loader = pdt.DataLoader(dataset=train_dataset, batch_size=accum * batch_size, shuffle=False, num_workers=0,
                                  pin_memory=use_cuda, sampler=train_sampler)

    if args.eval:
        # the test split: every image counted once across the ranks (engine.evaluate leaves out the sampler's padding)
        if args.data == "mnist" and args.model == "convnet":
            test_dataset = pdata.MNIST(root=args.data_root, train=False, synthetic_fallback=True)
        else:
            test_dataset = pdata.SyntheticMNIST(10000 if args.model == "convnet" else 4096, seed=1, num_classes=num_classes,
                                                image_shape=shape)
        test_loader = pdt.DataLoader(dataset=test_dataset, batch_size=batch_size, shuffle=False, pin_memory=use_cuda,
                                     sampler=pdt.DistributedSampler(test_dataset, num_replicas=args.world_size, rank=rank, shuffle=False))

    mix_gen = None
    if args.mixup is not None:
        # MixUp on the host, before the batch's copy to the device: one λ per loader batch, each rank drawing its own (seeded per
        # epoch below)
        mix_gen = torch.Generator()

    step_fn = None
    if args.graph and use_cuda:
        from pytorch_distributed_train_b200.engine import GraphedTrainStep

        rows = accum * batch_size
        example_targets = (torch.zeros(rows, dtype=torch.int64, device=device) if mix_gen is None else
                           torch.zeros(rows, num_classes, device=device))
        step_fn = GraphedTrainStep(model, criterion, optimizer, example_inputs=(torch.zeros((rows,) + shape, device=device), example_targets),
                                   max_grad_norm=args.clip_grad_norm, accumulation_steps=accum, averaged_model=ema)

    first_epoch = 0
    if args.resume:
        info = pdt.utils.load_checkpoint(args.resume, model, optimizer, sampler=train_sampler, averaged_model=ema)
        first_epoch = info["epoch"]
        if gpu == 0:
            print(f"Resumed from {args.resume} at epoch {first_epoch}")

    start = datetime.now()
    total_step = len(train_loader)
    for epoch in range(first_epoch, args.epochs):
        if args.set_epoch:
            train_sampler.set_epoch(epoch)
        if mix_gen is not None:
            # from (epoch, rank): a run resumed from an epoch's checkpoint draws the λ sequence of an uninterrupted run
            mix_gen.manual_seed(epoch * args.world_size + rank)
        pending = None   # (step index, loss handle) of a log line whose value is still on its way to the host
        fmt = "Epoch [{}/{}], Step [{}/{}], Loss: {:.4f}"
        for i, (images, labels) in enumerate(train_loader):
            if args.steps and i >= args.steps:
                break
            if mix_gen is not None:
                # the images are mixed in place and stay pinned; the targets are pinned too, so their copy stays asynchronous
                labels = pdata.mixup(images, labels, num_classes, args.mixup, mix_gen)
                if use_cuda:
                    labels = labels.pin_memory()
            graphed = step_fn is not None and images.shape[0] == accum * batch_size
            if graphed:
                # the (pinned) host batch goes straight into the captured step's input buffers; the copy overlaps the previous step
                step_fn(images, labels)
                handle = step_fn.loss_to_host()
            else:
                images = images.to(device, non_blocking=True)
                labels = labels.to(device, non_blocking=True)
                optimizer.zero_grad()
                if accum == 1:
                    outputs = model(images)
                    loss = criterion(outputs, labels)
                    loss.backward()
                else:
                    # micro-batches of batch_size rows (a short last batch gives fewer); the gradient reduction runs on the last one
                    micro = list(zip(images.split(batch_size), labels.split(batch_size)))
                    loss = 0.0
                    for j, (x, t) in enumerate(micro):
                        with model.no_sync() if j + 1 < len(micro) else contextlib.nullcontext():
                            part = criterion(model(x), t) / len(micro)
                            part.backward()
                        loss = loss + part.detach()
                if args.clip_grad_norm is not None:
                    pdt.nn.utils.clip_grad_norm_(model.parameters(), args.clip_grad_norm)
                optimizer.step()
                if ema is not None:
                    ema.update_parameters(bare)
                handle = loss
            if pending is not None and gpu == 0:
                # the log line of the previous step, printed once this step has been queued: the GPU keeps working while the host waits
                print(fmt.format(epoch + 1, args.epochs, pending[0], total_step, pending[1].item()))
                pending = None
            if (i + 1) % args.log_interval == 0 and gpu == 0:
                if graphed:
                    pending = (i + 1, handle)
                else:
                    print(fmt.format(epoch + 1, args.epochs, i + 1, total_step, handle.item()))
        if pending is not None and gpu == 0:
            print(fmt.format(epoch + 1, args.epochs, pending[0], total_step, pending[1].item()))
        if args.checkpoint:
            pdt.utils.save_checkpoint(args.checkpoint, model, optimizer, epoch=epoch + 1, sampler=train_sampler, averaged_model=ema)
        if args.eval:
            for tag, evaluated in [("", model)] + ([("EMA ", ema)] if ema is not None else []):
                r = pdt.engine.evaluate(evaluated, test_loader, criterion)
                if gpu == 0:
                    print(f"Epoch [{epoch + 1}/{args.epochs}], {tag}Test Loss: {r['loss']:.4f}, Accuracy: {100 * r['accuracy']:.2f}% "
                          f"({r['count']} images)")
    if use_cuda:
        torch.cuda.synchronize()
    if gpu == 0:
        print("Training complete in: " + str(datetime.now() - start))
    pdt.destroy_process_group()


def main(argv=None) -> None:
    p = build_parser()
    args = p.parse_args(argv)
    check_args(p, args)
    args.world_size = args.gpus  # one process per GPU (ref: ddp_example.py:109)
    if args.init_method is None:
        args.init_method = f"tcp://127.0.0.1:{_free_port()}"
    from pytorch_distributed_train_b200.launcher import spawn

    spawn(dist_train, nprocs=args.gpus, args=(args,))


if __name__ == "__main__":
    main(sys.argv[1:])
