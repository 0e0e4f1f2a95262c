"""Single-GPU numerics of every sm_90a kernel against a plain PyTorch fp32 reference of the same op
(tolerance policy: TF32 level for the tensor-core convolution, fp32 level for everything else)."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C, ops

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_reference():
    # the oracle must be true fp32: no TF32 inside cuDNN/cuBLAS
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def dev():
    return torch.device("cuda", 0)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def test_native_cuda_runtime_is_loaded():
    assert ops.native_available() and hasattr(_C, "SymmComm") and hasattr(_C, "convnet_fwd")
    assert torch.cuda.get_device_capability(0) == (9, 0), "these kernels are built for sm_90a only"


# the shape picks the kernel: conv1 (1→16) runs on SIMT, conv2 (16→32) on the TMA-im2col wgmma kernel (TF32 operands)
@pytest.mark.parametrize("cin,cout,H,kernel", [(1, 16, 28, "simt"), (16, 32, 14, "wgmma")])
@pytest.mark.parametrize("B", [100, 3])
def test_conv5x5_forward_and_stats(cin, cout, H, kernel, B):
    x = torch.randn(B, cin, H, H, device=dev())
    w = torch.randn(cout, cin, 5, 5, device=dev()) * 0.1
    b = torch.randn(cout, device=dev())
    y, stats = _C.conv5x5_fwd(nhwc(x), w, b, True)
    # float64 oracle: cuDNN's fp32 algorithms are not all IEEE-accurate at this size
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=2).float()
    tol = 2e-2 if kernel == "wgmma" else 1e-4
    assert torch.allclose(y.permute(0, 3, 1, 2), ref, atol=tol, rtol=tol), (y.permute(0, 3, 1, 2) - ref).abs().max()
    yn = y.double()
    assert torch.allclose(stats[:cout].double(), yn.sum((0, 1, 2)), rtol=1e-4, atol=1e-2)
    assert torch.allclose(stats[cout:2 * cout].double(), (yn * yn).sum((0, 1, 2)), rtol=1e-4, atol=1e-2)
    assert stats[2 * cout].item() == B * H * H
    # deterministic: bitwise identical on a second run
    y2, stats2 = _C.conv5x5_fwd(nhwc(x), w, b, True)
    assert torch.equal(y, y2) and torch.equal(stats, stats2)


@pytest.mark.parametrize("B", [1, 5, 100, 2048])   # 2 tiles of 128 pixels, …, 3136 tiles: more than the grid
def test_conv_tma_im2col_exact(B):
    """conv2's per-op kernels on TF32-representable integers, so every product and sum is exact: the TMA-im2col forward
    (SWIZZLE_64B rows, bias, Σy) and data gradient (SWIZZLE_128B rows), and the mma.sync weight gradient (MN-major operands)
    with the bias gradient from its im2col column of ones."""
    x = torch.randint(-3, 4, (B, 16, 14, 14), device=dev()).float()
    w = torch.randint(-2, 3, (32, 16, 5, 5), device=dev()).float()
    b = torch.randint(-2, 3, (32,), device=dev()).float()
    y, stats = _C.conv5x5_fwd(nhwc(x), w, b, True)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=2)
    assert torch.equal(y.permute(0, 3, 1, 2).double(), ref)
    assert torch.equal(stats[:32].double(), ref.sum((0, 2, 3))) and stats[64].item() == B * 196
    dy = torch.randint(-3, 4, (B, 32, 14, 14), device=dev()).float()
    dx = _C.conv5x5_dgrad(nhwc(dy), w)
    xd = x.double().requires_grad_()
    gx = torch.autograd.grad(F.conv2d(xd, w.double(), padding=2), xd, dy.double())[0]
    assert torch.equal(dx.permute(0, 3, 1, 2).double(), gx)
    wd = w.double().requires_grad_()
    bd = torch.zeros(32, dtype=torch.float64, device=dev(), requires_grad=True)
    gw, gb = torch.autograd.grad(F.conv2d(x.double(), wd, bd, padding=2), (wd, bd), dy.double())
    dw, db = torch.empty_like(w), torch.empty(32, device=dev())
    _C.conv5x5_wgrad(nhwc(dy), nhwc(x), dw, db)
    assert torch.equal(dw.double(), gw) and torch.equal(db.double(), gb)


def test_conv5x5_backward():
    B = 100
    x = torch.randn(B, 16, 14, 14, device=dev(), requires_grad=True)
    w = (torch.randn(32, 16, 5, 5, device=dev()) * 0.1).requires_grad_()
    b = torch.randn(32, device=dev(), requires_grad=True)
    dy = torch.randn(B, 32, 14, 14, device=dev())
    xd, wd, bd = (t.detach().double().requires_grad_() for t in (x, w, b))
    gx, gw, gb = (g.float() for g in torch.autograd.grad(F.conv2d(xd, wd, bd, padding=2), (xd, wd, bd), dy.double()))
    dx = _C.conv5x5_dgrad(nhwc(dy), w.detach())
    assert torch.allclose(dx.permute(0, 3, 1, 2), gx, atol=3e-2, rtol=3e-2)
    dw, db = torch.empty_like(w), torch.empty_like(b)
    _C.conv5x5_wgrad(nhwc(dy), nhwc(x.detach()), dw, db)
    # TF32 operands: ~1e-3 relative per product, random-walk over 19,600 pixels
    assert torch.allclose(dw, gw, atol=1.0, rtol=5e-3), (dw - gw).abs().max()
    assert torch.allclose(db, gb, atol=1.0, rtol=5e-3), (db - gb).abs().max()
    # conv1 weight gradient (its data gradient: test_convnet_input_grads.py)
    x1 = torch.randn(B, 1, 28, 28, device=dev())
    w1 = torch.randn(16, 1, 5, 5, device=dev(), requires_grad=True)
    b1 = torch.randn(16, device=dev(), requires_grad=True)
    dy1 = torch.randn(B, 16, 28, 28, device=dev())
    w1d, b1d = w1.detach().double().requires_grad_(), b1.detach().double().requires_grad_()
    gw1, gb1 = (g.float() for g in torch.autograd.grad(F.conv2d(x1.double(), w1d, b1d, padding=2), (w1d, b1d), dy1.double()))
    dw1, db1 = torch.empty_like(w1), torch.empty_like(b1)
    _C.conv5x5_wgrad(nhwc(dy1), nhwc(x1), dw1, db1)
    assert torch.allclose(dw1, gw1, atol=5e-3, rtol=1e-3) and torch.allclose(db1, gb1, atol=5e-3, rtol=1e-4)


@pytest.mark.parametrize("C,H,out_nchw", [(16, 28, False), (32, 14, True)])
def test_bn_relu_pool_forward_backward(C, H, out_nchw):
    B = 100
    y = torch.randn(B, C, H, H, device=dev()) * 2 + 0.5
    gamma = torch.rand(C, device=dev()) + 0.5
    beta = torch.randn(C, device=dev()) * 0.1
    bn = nn.BatchNorm2d(C).to(dev())
    with torch.no_grad():
        bn.weight.copy_(gamma)
        bn.bias.copy_(beta)
    yr = y.clone().requires_grad_()
    ref = F.max_pool2d(F.relu(bn(yr)), 2, 2)
    yh = nhwc(y)
    stats = torch.cat([yh.sum((0, 1, 2)), (yh * yh).sum((0, 1, 2)), yh.new_full((1,), B * H * H)])
    rm, rv, nbt = torch.zeros(C, device=dev()), torch.ones(C, device=dev()), torch.zeros((), dtype=torch.int64, device=dev())
    out, saved = _C.bn_relu_pool_fwd(yh, stats, gamma, beta, rm, rv, nbt, 0.1, 1e-5, out_nchw)
    got = out if out_nchw else out.permute(0, 3, 1, 2)
    assert torch.allclose(got, ref, atol=2e-4, rtol=1e-4), (got - ref).abs().max()
    assert torch.allclose(rm, bn.running_mean, atol=1e-5) and torch.allclose(rv, bn.running_var, atol=1e-4) and int(nbt) == 1
    dout = torch.randn_like(ref)
    ref.backward(dout)
    d = dout.contiguous() if out_nchw else nhwc(dout)
    sums, dgamma, dbeta = _C.bn_relu_pool_bwd_reduce(d, yh, saved, gamma, beta, out_nchw)
    assert torch.allclose(dgamma, bn.weight.grad, atol=2e-2, rtol=1e-3) and torch.allclose(dbeta, bn.bias.grad, atol=2e-2, rtol=1e-3)
    dy = _C.bn_relu_pool_bwd_apply(d, yh, saved, gamma, beta, sums, stats[2 * C:], out_nchw)
    assert torch.allclose(dy.permute(0, 3, 1, 2), yr.grad, atol=2e-4, rtol=1e-3), (dy.permute(0, 3, 1, 2) - yr.grad).abs().max()


def test_linear_and_cross_entropy():
    B, K, N = 100, 1568, 10
    x = torch.randn(B, K, device=dev(), requires_grad=True)
    lin = nn.Linear(K, N).to(dev())
    t = torch.randint(0, N, (B,), device=dev())
    ref_loss = F.cross_entropy(lin(x), t)
    gx, gw, gb = torch.autograd.grad(ref_loss, (x, lin.weight, lin.bias))
    x2 = x.detach().clone().requires_grad_()
    w2, b2 = lin.weight.detach().clone().requires_grad_(), lin.bias.detach().clone().requires_grad_()
    loss = ops.cross_entropy(ops.linear(x2, w2, b2), t)
    assert torch.allclose(loss, ref_loss, atol=1e-5)
    loss.backward()
    assert torch.allclose(x2.grad, gx, atol=1e-6, rtol=1e-4)
    assert torch.allclose(w2.grad, gw, atol=1e-5, rtol=1e-4) and torch.allclose(b2.grad, gb, atol=1e-6, rtol=1e-4)
    crit = pdt.nn.CrossEntropyLoss()
    assert torch.allclose(crit(lin(x).detach(), t), ref_loss.detach(), atol=1e-5)


@pytest.mark.parametrize("momentum,nesterov,wd", [(0.0, False, 0.0), (0.9, False, 1e-3), (0.9, True, 0.0)])
def test_fused_sgd_matches_torch(momentum, nesterov, wd):
    shapes = [(16, 1, 5, 5), (16,), (32, 16, 5, 5), (10, 1568), (10,)]
    ps = [torch.randn(s, device=dev()) for s in shapes]
    ours = [p.clone().requires_grad_() for p in ps]
    ref = [p.clone().requires_grad_() for p in ps]
    o1 = pdt.optim.SGD(ours, lr=0.05, momentum=momentum, nesterov=nesterov, weight_decay=wd)
    o2 = torch.optim.SGD(ref, lr=0.05, momentum=momentum, nesterov=nesterov, weight_decay=wd)
    for step in range(3):
        for a, b in zip(ours, ref):
            g = torch.randn_like(a)
            a.grad, b.grad = g.clone(), g.clone()
        o1.step()
        o2.step()
    for a, b in zip(ours, ref):
        assert torch.allclose(a, b, atol=1e-6, rtol=1e-5)


@pytest.mark.parametrize("syncbn_module", [False, True])
def test_convnet_fused_matches_unfused(syncbn_module):
    torch.manual_seed(1)
    ref = pdt.models.ConvNet(fused=False).to(dev())
    net = pdt.models.ConvNet(fused=True).to(dev())
    net.load_state_dict(ref.state_dict())
    if syncbn_module:  # world of one: SyncBatchNorm must degrade to local statistics
        net = pdt.SyncBatchNorm.convert_sync_batchnorm(net)
    ref = ref.double()  # float64 oracle (cuDNN fp32 paths are not all IEEE-accurate)
    x = torch.rand(100, 1, 28, 28, device=dev())
    t = torch.randint(0, 10, (100,), device=dev())
    l_ref = F.cross_entropy(ref(x.double()), t)
    l_ref.backward()
    l = pdt.nn.CrossEntropyLoss()(net(x), t)
    l.backward()
    assert abs(l.item() - l_ref.item()) < 2e-3, (l.item(), l_ref.item())
    for (n1, p1), (_, p2) in zip(net.named_parameters(), ref.named_parameters()):
        scale = p2.grad.abs().max().item() + 1e-6
        # conv2 runs in TF32 (10-bit mantissa) forward and in dgrad: ~1e-3 relative per product
        assert (p1.grad.double() - p2.grad).abs().max().item() <= 5e-2 * scale + 1e-4, n1
    for (n1, b1), (_, b2) in zip(net.named_buffers(), ref.named_buffers()):
        assert torch.allclose(b1.double(), b2.double(), atol=2e-3, rtol=1e-3), n1
    net.eval(), ref.eval()
    assert torch.allclose(net(x).double(), ref(x.double()), atol=3e-2, rtol=1e-2)


@pytest.mark.parametrize("B", [100, 3, "sms"])   # "sms": one image per SM, i.e. one CTA on every SM of the device
def test_cooperative_fused_layers_match_per_op_kernels(B, monkeypatch):
    """csrc/cuda/fused_convnet.cu (one cooperative kernel for the forward and one per layer for the backward, grid barriers
    for the batch statistics) against the per-op kernels on the same weights and data: same TF32 convolution, same fp32
    rest — only summation orders differ."""
    if B == "sms":
        B = torch.cuda.get_device_properties(0).multi_processor_count
    torch.manual_seed(2)
    a = pdt.models.ConvNet(fused=True).to(dev())
    b = pdt.models.ConvNet(fused=True).to(dev())
    b.load_state_dict(a.state_dict())
    x = torch.rand(B, 1, 28, 28, device=dev())
    t = torch.randint(0, 10, (B,), device=dev())
    crit = pdt.nn.CrossEntropyLoss()
    before = _C.kernel_launch_count()
    la = crit(a(x), t)
    la.backward()
    fused_launches = _C.kernel_launch_count() - before
    monkeypatch.setenv("PDT_FUSED_LAYERS", "0")
    before = _C.kernel_launch_count()
    lb = crit(b(x), t)
    lb.backward()
    per_op_launches = _C.kernel_launch_count() - before
    monkeypatch.delenv("PDT_FUSED_LAYERS")
    assert fused_launches < per_op_launches, (fused_launches, per_op_launches)
    assert abs(la.item() - lb.item()) < 1e-4, (la.item(), lb.item())
    for (n1, p1), (_, p2) in zip(a.named_parameters(), b.named_parameters()):
        scale = p2.grad.abs().max().item() + 1e-6
        # TF32 operand rounding of slightly different dy; conv biases in front of a BatchNorm have a true gradient of zero (noise level)
        assert (p1.grad - p2.grad).abs().max().item() <= 2e-2 * scale + 5e-4, (n1, (p1.grad - p2.grad).abs().max().item(), scale)
    for (n1, b1), (_, b2) in zip(a.named_buffers(), b.named_buffers()):
        assert torch.allclose(b1.float(), b2.float(), atol=1e-5, rtol=1e-5), n1


def test_cooperative_layer2_exact_on_small_integers():
    """Integer-valued inputs/weights are exact in TF32 and in fp32 accumulation: the fused conv2 forward (window
    descriptors over the haloed image) and data gradient must reproduce a float64 convolution bit for bit."""
    B = 5
    # layer 1 with BN1's gamma = 0: the pooled frame p1 is relu(beta) = beta inside an exact zero halo, a distinct small integer
    # per channel, so that the border rows of both output tiles and every 16-byte swizzle chunk of a patch row carry distinct values
    x1 = torch.rand(B, 1, 28, 28, device=dev())
    w1, b1 = torch.randn(16, 1, 5, 5, device=dev()) * 0.2, torch.randn(16, device=dev()) * 0.1
    be1 = (torch.randperm(16, device=dev()) + 1).float()
    w = torch.randint(-2, 3, (32, 16, 5, 5), device=dev()).float()
    bias = torch.randint(-2, 3, (32,), device=dev()).float()
    gamma, beta = torch.ones(32, device=dev()), torch.zeros(32, device=dev())
    fcw, fcb = torch.randn(10, 1568, device=dev()) * 0.02, torch.randn(10, device=dev()) * 0.1
    p1, y1, sv1, out, y, saved, logits, *_ = _C.convnet_fwd(x1, w1, b1, torch.zeros(16, device=dev()), be1, None, None, None, 0.1, 1e-5,
                                                            w, bias, gamma, beta, None, None, None, 0.1, 1e-5, fcw, fcb)
    frame = torch.zeros(B, 18, 18, 16, device=dev())
    frame[:, 2:16, 2:16, :] = be1
    assert torch.equal(p1, frame)
    ref = F.conv2d(p1[:, 2:16, 2:16, :].permute(0, 3, 1, 2).double(), w.double(), bias.double(), padding=2)
    assert torch.equal(y.permute(0, 3, 1, 2).double(), ref)
    mean = ref.mean((0, 2, 3))
    assert torch.allclose(saved[:32].double(), mean, atol=1e-4, rtol=1e-5)
    # data gradient: feed a gradient that passes the classifier and pool/ReLU/BN backward, compare the conv part through dy (the
    # form without p1 writes the dy frame)
    dlogits = torch.randn(B, 10, device=dev())
    dfcw, dfcb = torch.empty_like(fcw), torch.empty_like(fcb)
    dg, db = torch.empty(32, device=dev()), torch.empty(32, device=dev())
    dy, dx, dysum = _C.convnet_l2_bwd_fc(dlogits, fcw, out, dfcw, dfcb, y, saved, gamma, beta, w, dg, db)
    dyi = dy[:, 2:16, 2:16, :]
    halo = dy.clone()
    halo[:, 2:16, 2:16, :] = 0
    assert halo.abs().max().item() == 0.0, "halo of the dy frame must be zero"
    ref_dx = torch.nn.grad.conv2d_input((B, 16, 14, 14), w.double(), dyi.permute(0, 3, 1, 2).double(), padding=2)
    err = (dx[:, 2:16, 2:16, :].permute(0, 3, 1, 2).double() - ref_dx).abs().max().item()
    assert err <= 2e-3 * ref_dx.abs().max().item() + 1e-5, err   # dy is not integer valued: TF32 operand rounding
    assert torch.allclose(dysum.sum(0).double(), dyi.double().sum((0, 1, 2)), atol=1e-4)
    # weight gradient on integer-valued frames, as the layer-1 backward kernel folds it from the per-image partials of the K-major
    # operand copies (written here from the frames, as the layer-2 backward kernel writes them from its registers): exact
    xq = torch.zeros(B, 18, 18, 16, device=dev())   # zero-haloed frame
    xq[:, 2:16, 2:16, :] = torch.randint(-3, 4, (B, 14, 14, 16), device=dev()).float()
    dyq = torch.zeros(B, 18, 18, 32, device=dev())
    dyq[:, 2:16, 2:16, :] = torch.randint(-2, 3, (B, 14, 14, 32), device=dev()).float()
    ref_dw = torch.nn.grad.conv2d_weight(xq[:, 2:16, 2:16, :].permute(0, 3, 1, 2).double(), (32, 16, 5, 5),
                                         dyq[:, 2:16, 2:16, :].permute(0, 3, 1, 2).double(), padding=2)
    dp1 = torch.zeros(B, 18, 18, 16, device=dev())
    dp1[:, 2:16, 2:16, :] = torch.randn(B, 14, 14, 16, device=dev())
    g1 = torch.rand(16, device=dev()) + 0.5
    l1_out = [torch.full((16,), 7.0, device=dev()), torch.full((16,), 7.0, device=dev()), torch.full((16, 1, 5, 5), 7.0, device=dev()),
              torch.full((16,), 7.0, device=dev())]
    dw_m, db_m = torch.full((32, 16, 5, 5), 7.0, device=dev()), torch.full((32,), 7.0, device=dev())
    _C.convnet_l1_bwd_wgrad(dp1, y1, x1, sv1, g1, be1, *l1_out, dyq, xq, dyq[:, 2:16, 2:16, :].sum((1, 2)).contiguous(), dw_m, db_m)
    assert torch.equal(dw_m.double(), ref_dw), (dw_m.double() - ref_dw).abs().max()
    assert torch.equal(db_m.double(), dyq.double().sum((0, 1, 2)))


def test_generic_bn_kernels_match_torch():
    x = torch.randn(8, 12, 9, 7, device=dev()) * 3 + 1
    st = ops.bn_local_stats(x)
    assert st.dtype == torch.float64 and st.numel() == 26 and st[24].item() == 8 * 63 and st[25].item() == 0
    assert torch.allclose(st[:12], x.double().sum((0, 2, 3)), rtol=1e-9) and torch.allclose(st[12:24], (x.double() ** 2).sum((0, 2, 3)), rtol=1e-9)
    mean = x.mean((0, 2, 3))
    invstd = (x.var((0, 2, 3), unbiased=False) + 1e-5).rsqrt()
    w, b = torch.rand(12, device=dev()) + 0.5, torch.randn(12, device=dev())
    xr = x.clone().requires_grad_()
    ref = F.batch_norm(xr, None, None, w, b, True, 0.0, 1e-5)
    assert torch.allclose(ops.bn_apply(x, mean, invstd, w, b), ref, atol=1e-4, rtol=1e-4)
    dy = torch.randn_like(x)
    ref.backward(dy)
    red = ops.bn_backward_reduce(dy, x, mean, invstd)
    n = 8 * 63
    dx = ops.bn_backward_apply(dy, x, mean, invstd, w, red[:12] / n, red[12:24] / n)
    assert torch.allclose(dx, xr.grad, atol=1e-4, rtol=1e-3)


def _one_rank_group():
    from mp_helpers import free_port

    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)


def test_single_gpu_ddp_and_graphed_step():
    """One process, one GPU: the whole product path (SymmComm heap, reducer, fused ops, CUDA graph)."""
    torch.cuda.set_device(0)
    _one_rank_group()
    try:
        g = pdt.distributed.get_default_group()
        assert g.comm.backend_name == "nvlink" and "SymmComm" in g.comm.describe()
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(dev())
        opt = pdt.optim.SGD(model.parameters(), 1e-2)
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        assert ddp.param_arena is not None and g.comm.is_symmetric(ddp.param_arena)
        crit = pdt.nn.CrossEntropyLoss()
        x = torch.rand(100, 1, 28, 28, device=dev())
        t = torch.randint(0, 10, (100,), device=dev())
        eager = []
        for _ in range(3):
            loss = crit(ddp(x), t)
            opt.zero_grad()
            loss.backward()
            opt.step()
            eager.append(loss.item())
        assert eager[2] < eager[0]
        info = ddp._get_ddp_logging_data()
        assert info["copies_into_bucket"] == 0, "gradients must be produced in place inside the bucket"
        assert ddp.reducer.grads_are_views()
        from pytorch_distributed_train_b200.engine import GraphedTrainStep

        # the old loss keeps last iteration's autograd graph — and with it AccumulateGrad nodes that
        # were created on the default stream — alive; drop it before capturing on a side stream
        del loss
        step = GraphedTrainStep(ddp, crit, opt, (x, t))
        l0 = step(x, t).item()
        l1 = step(x, t).item()
        assert l1 < l0 < eager[2] + 1e-3
        # pinned host batches, double-buffered inputs, losses delivered through the side-stream ring: same trajectory as device batches
        xp, tp = x.cpu().pin_memory(), t.cpu().pin_memory()
        handles = []
        for _ in range(20):
            step(xp, tp)
            handles.append(step.loss_to_host())
        vals = [h.item() for h in handles[-16:]]
        assert all(a > b for a, b in zip(vals, vals[1:])) and vals[0] < l1, (l1, vals)
        assert abs(vals[-1] - step.static_loss.item()) < 1e-7
        with pytest.raises(RuntimeError, match="read too late"):
            handles[0].item()
    finally:
        pdt.destroy_process_group()


def test_parameter_used_twice_sums_both_gradients():
    """ADVICE r1 (medium): a weight used twice in one forward must get dW1 + dW2, not two aliases of one bucket slot."""
    torch.cuda.set_device(0)
    _one_rank_group()
    try:
        class Tied(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.fc = torch.nn.Linear(64, 64)

            def forward(self, x):
                return ops.linear(torch.relu(ops.linear(x, self.fc.weight, self.fc.bias)), self.fc.weight, self.fc.bias)

        torch.manual_seed(0)
        model = Tied().to(dev())
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        x = torch.randn(32, 64, device=dev())
        ddp(x).square().mean().backward()
        w, b = model.fc.weight.detach().clone().requires_grad_(), model.fc.bias.detach().clone().requires_grad_()
        F.linear(torch.relu(F.linear(x, w, b)), w, b).square().mean().backward()
        assert torch.allclose(model.fc.weight.grad, w.grad, atol=1e-5, rtol=1e-4)
        assert torch.allclose(model.fc.bias.grad, b.grad, atol=1e-5, rtol=1e-4)
    finally:
        pdt.destroy_process_group()


@pytest.mark.parametrize("late", [False, True])
@pytest.mark.parametrize("B", [100, 7])
def test_cross_entropy_folded_into_the_forward_kernel(B, late):
    """engine.GraphedTrainStep announces the targets before it calls the model (ops.functional.upcoming_targets): the whole-forward
    kernel then also produces the mean cross-entropy and d(loss)/d(logits); `criterion(logits, target)` launches nothing."""
    from pytorch_distributed_train_b200.ops import functional as OF

    torch.manual_seed(3)
    a = pdt.models.ConvNet(fused=True).to(dev())
    b = pdt.models.ConvNet(fused=True).to(dev())
    b.load_state_dict(a.state_dict())
    x = torch.rand(B, 1, 28, 28, device=dev())
    t = torch.randint(0, 10, (B,), device=dev())
    crit = pdt.nn.CrossEntropyLoss()
    before = _C.kernel_launch_count()
    with OF.upcoming_targets(t, loss_read_after_backward=late):   # late: the batch mean is folded by the first backward kernel
        out = a(x)
    assert getattr(out, "_pdt_ce", None) is not None and out._pdt_ce[0] is t
    la = crit(out, t)
    la.backward()
    folded = _C.kernel_launch_count() - before
    before = _C.kernel_launch_count()
    lb = crit(b(x), t)
    lb.backward()
    separate = _C.kernel_launch_count() - before
    assert folded == separate - 1, (folded, separate)
    ref = F.cross_entropy(out.detach().double(), t).item()
    assert abs(la.item() - ref) < 1e-5 and abs(la.item() - lb.item()) < 1e-5, (la.item(), lb.item(), ref)
    for (n1, p1), (_, p2) in zip(a.named_parameters(), b.named_parameters()):
        # softmax rounding differs in the last bit between the two kernels; the BatchNorm backward amplifies it
        scale = p2.grad.abs().max().item() + 1e-6
        assert (p1.grad - p2.grad).abs().max().item() <= 2e-3 * scale + 1e-5, (n1, (p1.grad - p2.grad).abs().max().item(), scale)
    # a different target tensor at the criterion: the precomputed loss must not be used
    t2 = torch.randint(0, 10, (B,), device=dev())
    with OF.upcoming_targets(t):
        out = a(x)
    assert abs(crit(out, t2).item() - F.cross_entropy(out.detach().double(), t2).item()) < 1e-5


@pytest.mark.parametrize("momentum,nesterov,wd", [(0.0, False, 0.0), (0.9, True, 1e-3)])
def test_optimizer_rides_on_the_last_backward_kernel(momentum, nesterov, wd):
    """optim.SGD.ride_on_backward: the layer-1 backward kernel applies the update of all ten parameters (fused_convnet.cu: SgdRider);
    parameters and momentum buffers must follow the separate multi-tensor SGD kernel."""
    torch.manual_seed(4)
    a = pdt.models.ConvNet(fused=True).to(dev())
    b = pdt.models.ConvNet(fused=True).to(dev())
    b.load_state_dict(a.state_dict())
    oa = pdt.optim.SGD(a.parameters(), 0.05, momentum=momentum, nesterov=nesterov, weight_decay=wd)
    ob = pdt.optim.SGD(b.parameters(), 0.05, momentum=momentum, nesterov=nesterov, weight_decay=wd)
    crit = pdt.nn.CrossEntropyLoss()
    assert oa.ride_on_backward(a)
    try:
        for s in range(4):
            x = torch.rand(100, 1, 28, 28, device=dev(), generator=torch.Generator(device=dev()).manual_seed(s))
            t = torch.randint(0, 10, (100,), device=dev(), generator=torch.Generator(device=dev()).manual_seed(50 + s))
            before = _C.kernel_launch_count()
            oa.zero_grad()
            la = crit(a(x), t)
            if s == 0:   # outside the engine's context an armed optimizer must not touch the parameters
                la.backward(retain_graph=False)
                assert not oa._rode
                oa.zero_grad()
                before = _C.kernel_launch_count()
                la = crit(a(x), t)
            from pytorch_distributed_train_b200.ops import functional as OF
            with OF.sgd_rider_enabled():
                la.backward()
            assert oa._rode, "the backward kernel should have applied the update"
            oa.step()
            riding = _C.kernel_launch_count() - before
            before = _C.kernel_launch_count()
            ob.zero_grad()
            crit(b(x), t).backward()
            ob.step()
            separate = _C.kernel_launch_count() - before
            assert riding < separate, (riding, separate)
            for (n1, p1), (_, p2) in zip(a.named_parameters(), b.named_parameters()):
                assert torch.allclose(p1, p2, atol=1e-6, rtol=1e-5), (s, n1, (p1 - p2).abs().max().item())
        if momentum:
            for p1, p2 in zip(a.parameters(), b.parameters()):
                assert torch.allclose(oa.state[p1]["momentum_buffer"], ob.state[p2]["momentum_buffer"], atol=1e-6, rtol=1e-5)
    finally:
        oa.stop_riding()
