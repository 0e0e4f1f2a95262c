#!/usr/bin/env python
"""Per-kernel device times of the ConvNet step, ours next to the library kernels the reference stack runs for the
same work (cuDNN convolution fwd/dgrad/wgrad, ATen batch-norm / ReLU / max-pool and their backward ops, cuBLAS addmm,
log-softmax + NLL, foreach SGD) — same box, same shapes (batch 100), same method:

* every row is timed as a CUDA graph of REPS back-to-back launches (CUDA events around the replay, ÷ REPS), i.e. what
  the op costs inside a captured step, launch gap included, host overhead excluded — for both arms;
* "cold" rows additionally overwrite a 256 MB buffer (> 50 MB L2) before a single eager launch.

Writes tool_out/op_bench.json and prints a table.
"""
import json
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorch_distributed_train_b200 import _C  # noqa: E402
from pytorch_distributed_train_b200.utils import l2_flush  # noqa: E402

dev = torch.device("cuda", 0)
B = 100
REPS = 20


def graph_time(fn, reps=REPS, iters=20):
    """µs per launch of `fn` inside a CUDA graph holding `reps` copies of it."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for _ in range(reps):
            fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / reps)
    ts.sort()
    return ts[len(ts) // 2]


def cold_time(fn, iters=15):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        l2_flush(dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = True          # the reference's default: TF32 allowed in cuDNN convolutions
    torch.backends.cudnn.benchmark = True            # let cuDNN pick its fastest engine for these shapes
    x = torch.rand(B, 1, 28, 28, device=dev)
    tgt = torch.randint(0, 10, (B,), device=dev)
    c1, bn1 = nn.Conv2d(1, 16, 5, 1, 2).to(dev), nn.BatchNorm2d(16).to(dev)
    c2, bn2 = nn.Conv2d(16, 32, 5, 1, 2).to(dev), nn.BatchNorm2d(32).to(dev)
    fc = nn.Linear(1568, 10).to(dev)
    w1, b1, g1, be1 = c1.weight.detach(), c1.bias.detach(), bn1.weight.detach(), bn1.bias.detach()
    w2, b2, g2, be2 = c2.weight.detach(), c2.bias.detach(), bn2.weight.detach(), bn2.bias.detach()
    wf, bf = fc.weight.detach(), fc.bias.detach()

    # ---- ours: the cooperative fused kernels a captured step launches (4 per step), plus the stand-alone variants ----------
    rm1, rv1, nb1 = bn1.running_mean, bn1.running_var, bn1.num_batches_tracked
    rm2, rv2, nb2 = bn2.running_mean, bn2.running_var, bn2.num_batches_tracked

    def fwd_whole():
        return _C.convnet_fwd(x, w1, b1, g1, be1, rm1, rv1, nb1, 0.1, 1e-5, w2, b2, g2, be2, rm2, rv2, nb2, 0.1, 1e-5, wf, bf, tgt, True)

    p1, y1, sv1, p2, y2, sv2, logits, loss, dlog, lparts = fwd_whole()
    dwf, dbf = torch.empty_like(wf), torch.empty_like(bf)
    dg2, dbe2 = torch.empty(32, device=dev), torch.empty(32, device=dev)

    def l2_bwd_fc():
        return _C.convnet_l2_bwd_fc(dlog, wf, p2, dwf, dbf, y2, sv2, g2, be2, w2, dg2, dbe2, lparts, loss)

    dy2, dp1, dysum = l2_bwd_fc()
    dw2, db2 = torch.empty_like(w2), torch.empty_like(b2)
    dg1, dbe1, dw1, db1 = torch.empty(16, device=dev), torch.empty(16, device=dev), torch.empty_like(w1), torch.empty_like(b1)
    params = [w1, b1, g1, be1, w2, b2, g2, be2, wf, bf]
    grads = [torch.randn_like(p) for p in params]
    dflat = torch.randn(B, 32, 7, 7, device=dev)
    ours = [
        ("forward: conv1+BN+ReLU+pool + conv2(wgmma)+BN+ReLU+pool + fc + cross-entropy (1 kernel)", fwd_whole),
        ("backward A: classifier bwd + pool/ReLU/BN2 bwd + conv2 dgrad(wgmma) (1 kernel)", l2_bwd_fc),
        ("backward B: pool/ReLU/BN1 bwd + conv1 wgrad(mma.sync) + conv2 wgrad(mma.sync, window) (1 kernel)",
         lambda: _C.convnet_l1_bwd_wgrad(dp1, y1, x, sv1, g1, be1, dg1, dbe1, dw1, db1, dy2, p1, dysum, dw2, db2)),
        ("SGD, 10 tensors (1 kernel)", lambda: _C.sgd_multi(params, grads, [], 1e-4, None, 0.0, 0.0, 0.0, False, False, False)),
        ("(variant) cross-entropy fwd (+dlogits) as its own kernel", lambda: _C.cross_entropy_fwd(logits, tgt, True)),
        ("(variant) fc bwd as its own kernel", lambda: _C.linear_bwd(dlog, p2.reshape(B, -1), wf, True, dwf, dbf)),
        ("(variant) layer-2 bwd without the classifier rider", lambda: _C.convnet_l2_bwd(dflat, y2, sv2, g2, be2, w2, dg2, dbe2)),
        ("(variant) conv2 wgrad as its own kernel (TMA-materialised tap pairs + in-kernel fold)", lambda: _C.conv5x5_wgrad_win(dy2, p1, dysum, dw2, db2)),
        ("(variant) layer-1 bwd without the wgrad rider", lambda: _C.convnet_l1_bwd(dp1, y1, x, sv1, g1, be1, dg1, dbe1, dw1, db1)),
    ]

    # ---- library: the ATen / cuDNN / cuBLAS ops the reference's modules dispatch to, same shapes -----------------------
    def lib_l1_fwd():
        return F.max_pool2d(F.relu(F.batch_norm(F.conv2d(x, w1, b1, padding=2), None, None, g1, be1, True, 0.1, 1e-5)), 2, 2)

    a1 = lib_l1_fwd()

    def lib_l2_fwd():
        return F.max_pool2d(F.relu(F.batch_norm(F.conv2d(a1, w2, b2, padding=2), None, None, g2, be2, True, 0.1, 1e-5)), 2, 2)

    a2 = lib_l2_fwd()
    flat = a2.reshape(B, -1)
    lg = torch.addmm(bf, flat, wf.t())

    def lib_fwd_bwd(make_out, inputs, grad_out):
        ins = [t.detach().requires_grad_(True) for t in inputs]
        out = make_out(*ins)
        return torch.autograd.grad(out, ins, grad_out)

    go1, go2 = torch.randn_like(a1), torch.randn_like(a2)
    lib = [
        ("layer1 fwd: cudnn conv + batch_norm + relu + max_pool2d", lib_l1_fwd),
        ("layer2 fwd: cudnn conv + batch_norm + relu + max_pool2d", lib_l2_fwd),
        ("fc fwd: addmm", lambda: torch.addmm(bf, flat, wf.t())),
        ("cross-entropy fwd: log_softmax + nll_loss", lambda: F.cross_entropy(lg, tgt)),
        ("cross-entropy fwd+bwd", lambda: lib_fwd_bwd(lambda l: F.cross_entropy(l, tgt), [lg], torch.ones((), device=dev))),
        ("fc fwd+bwd: addmm, mm, mm, sum", lambda: lib_fwd_bwd(lambda f_, w_, b_: torch.addmm(b_, f_, w_.t()), [flat, wf, bf], torch.randn(B, 10, device=dev))),
        ("layer2 fwd+bwd: + pool/relu/bn backward + cudnn dgrad + wgrad",
         lambda: lib_fwd_bwd(lambda a_, w_, b_, g_, e_: F.max_pool2d(F.relu(F.batch_norm(F.conv2d(a_, w_, b_, padding=2), None, None, g_, e_, True, 0.1, 1e-5)), 2, 2),
                             [a1, w2, b2, g2, be2], go2)),
        ("layer1 fwd+bwd: + pool/relu/bn backward + cudnn wgrad",
         lambda: lib_fwd_bwd(lambda w_, b_, g_, e_: F.max_pool2d(F.relu(F.batch_norm(F.conv2d(x, w_, b_, padding=2), None, None, g_, e_, True, 0.1, 1e-5)), 2, 2),
                             [w1, b1, g1, be1], go1)),
        ("conv2 cudnn fwd only", lambda: F.conv2d(a1, w2, b2, padding=2)),
        ("conv2 cudnn dgrad only", lambda: torch.ops.aten.convolution_backward(go_c2, a1, w2, [32], [1, 1], [2, 2], [1, 1], False, [0, 0], 1, [True, False, False])),
        ("conv2 cudnn wgrad(+bias) only", lambda: torch.ops.aten.convolution_backward(go_c2, a1, w2, [32], [1, 1], [2, 2], [1, 1], False, [0, 0], 1, [False, True, True])),
        ("conv1 cudnn fwd only", lambda: F.conv2d(x, w1, b1, padding=2)),
        ("conv1 cudnn wgrad(+bias) only", lambda: torch.ops.aten.convolution_backward(go_c1, x, w1, [16], [1, 1], [2, 2], [1, 1], False, [0, 0], 1, [False, True, True])),
        ("SGD: _foreach_add_ over 10 tensors", lambda: torch._foreach_add_(params, grads, alpha=-1e-4)),
    ]
    go_c2 = torch.randn(B, 32, 14, 14, device=dev)
    go_c1 = torch.randn(B, 16, 28, 28, device=dev)

    rows = []
    for arm, ops in (("ours", ours), ("library", lib)):
        for name, fn in ops:
            try:
                r = {"arm": arm, "op": name, "us_in_graph": graph_time(fn), "us_cold_eager": cold_time(fn)}
            except Exception as e:  # noqa: BLE001 - an op that cannot be captured still gets its eager number
                r = {"arm": arm, "op": name, "us_in_graph": None, "us_cold_eager": cold_time(fn), "note": f"{type(e).__name__}: {e}"[:120]}
            rows.append(r)
            g = f"{r['us_in_graph']:8.2f}" if r["us_in_graph"] is not None else "     n/a"
            print(f"{arm:8s} {g} us in-graph   {r['us_cold_eager']:8.2f} us cold eager   {name}", flush=True)
    floor = {"arm": "floor", "op": "empty launch (zero_ on 1 element)", "us_in_graph": graph_time(lambda: go_c1[0, 0, 0, :1].zero_()),
             "us_cold_eager": cold_time(lambda: go_c1[0, 0, 0, :1].zero_())}
    rows.append(floor)
    print(f"floor    {floor['us_in_graph']:8.2f} us in-graph   {floor['us_cold_eager']:8.2f} us cold eager   {floor['op']}")
    t_ours = sum(r["us_in_graph"] for r in rows if r["arm"] == "ours" and r["us_in_graph"] and not r["op"].startswith("(variant)"))
    print(f"ours, sum of the step's kernels in-graph: {t_ours:.1f} us")
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tool_out", "op_bench.json"), "w") as f:
        json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
