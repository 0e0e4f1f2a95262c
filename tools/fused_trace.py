"""Phase timeline of the cooperative fused ConvNet kernels (globaltimer stamps written by thread 0 of every CTA).
    python tools/fused_trace.py            # one eager training step at batch 100, prints per-phase medians in µs
Then the same inside the replayed CUDA graph of GraphedTrainStep, and the gap between two replays.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C
from pytorch_distributed_train_b200.ops import functional as OF

B = int(os.environ.get("B", "100"))
dev = torch.device("cuda", 0)
torch.manual_seed(0)
net = pdt.models.ConvNet().to(dev)
crit = pdt.nn.CrossEntropyLoss()
x = torch.rand(B, 1, 28, 28, device=dev)
y = torch.randint(0, 10, (B,), device=dev)
for _ in range(3):
    for p in net.parameters():
        p.grad = None
    crit(net(x), y).backward()
torch.cuda.synchronize()
_C.fused_convnet_trace_enable(True)
for p in net.parameters():
    p.grad = None
with OF.upcoming_targets(y):
    out = net(x)
crit(out, y).backward()
t = _C.fused_convnet_trace_read()[:, :B, :].double()
_C.fused_convnet_trace_enable(False)
names = {0: ("forward (whole)", ["start", "conv1 done", "stats partial written", "barrier 1 passed", "pooled patch in smem",
                                 "conv2 done (ys + stats 2 in smem)", "stats 2 partial written", "barrier 2 passed", "pooled 2 in smem",
                                 "logits written", "end (incl. loss)", "prologue done (halo zeroed, weights requested)"]),
         1: ("l1_bwd (+conv2 wgrad fold)", ["start", "partial written", "barrier passed", "folded", "conv1 wgrad partial written", "barrier 2 passed",
                                            "end", "dW2 folded", "y recomputed (conv1)"]),
         3: ("l2_bwd (+conv2 wgrad partials)", ["start", "B built", "partial written", "barrier passed", "folded", "dy written", "end",
                                                "dW2 atoms done (warp 0)", "dx written (warp 4)"])}
def report(t, title):
    print(f"######## {title}")
    spans = {}
    for k, (name, phases) in names.items():
        tk = t[k]
        if tk[:, 0].max() == 0:
            continue   # kernel did not run in this configuration
        t0 = tk[:, 0].min()
        spans[name] = (t0.item(), tk.max().item())
        print(f"== {name}: kernel span {(tk.max() - t0) / 1e3:.2f} us (first CTA start -> last CTA end)")
        order = sorted(range(len(phases)), key=lambda i: tk[:, i].median().item())
        for i in order:
            if tk[:, i].max() == 0:
                continue
            col = (tk[:, i] - t0) / 1e3
            print(f"   {phases[i]:30s} min {col.min():7.2f}  median {col.median():7.2f}  max {col.max():7.2f}")
    seq = sorted(spans.items(), key=lambda kv: kv[1][0])
    for (a, (_, ea)), (b, (sb, _)) in zip(seq, seq[1:]):
        print(f"-- gap {a} -> {b}: {(sb - ea) / 1e3:.2f} us (last CTA end -> first CTA start)")
    if seq:
        print(f"-- first kernel start -> last kernel end: {(seq[-1][1][1] - seq[0][1][0]) / 1e3:.2f} us")


report(t, "eager launches")

# the same step inside the captured graph the benchmark replays (one-rank process group, DDP, fused SGD)
import socket

with socket.socket() as s_:
    s_.bind(("127.0.0.1", 0))
    port = s_.getsockname()[1]
pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", world_size=1, rank=0)
try:
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    net2 = pdt.models.ConvNet().to(dev)
    opt = pdt.optim.SGD(net2.parameters(), 1e-4)
    ddp = pdt.DistributedDataParallel(net2, device_ids=[0])
    step = GraphedTrainStep(ddp, crit, opt, (x, y))
    for _ in range(5):
        step(x, y)
    torch.cuda.synchronize()
    _C.fused_convnet_trace_enable(True)
    step(x, y)
    step(x, y)   # the stamps are those of the second replay, which starts behind the first one's last kernel
    t2 = _C.fused_convnet_trace_read()[:, :B, :].double()
    _C.fused_convnet_trace_enable(False)
    report(t2, f"inside the replayed CUDA graph ({step.kernels_per_replay} launches)")

    # The launch cost left between two replays.  The stamps of one replay overwrite the other's, so the gap from the layer-1 backward's
    # end to the next forward's start is the replay period less the stamped span above.  The period is timed with device events around
    # back-to-back launches of the captured graphs, without the host work of step() (input staging), so that the host stays ahead.
    span = (t2[1].max() - t2[0][:, 0].min()).item() / 1e3
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 2000
    with torch.cuda.stream(step.capture_stream):
        ev0.record()
        for r in range(reps):
            step.graphs[r % len(step.graphs)].replay()
        ev1.record()
    torch.cuda.synchronize()
    period = ev0.elapsed_time(ev1) * 1e3 / reps
    print(f"-- replay period {period:.2f} us over {reps} replays; gap l1_bwd -> next replay's forward: {period - span:.2f} us "
          f"(period - first kernel start -> last kernel end)")
finally:
    pdt.destroy_process_group()
