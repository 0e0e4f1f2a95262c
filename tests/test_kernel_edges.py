"""The ConvNet kernels against float64 beyond the reference configuration: batches far above one CTA per SM (per-op grid folds of
more than 512 groups), class counts other than 10, targets equal to ``ignore_index``, every channel count the BatchNorm + ReLU +
pool kernels accept, and eval-mode BatchNorm with large running means.  Tolerance policy: TF32 level where conv2 runs on the
tensor cores, fp32 level for everything else."""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C, ops
from pytorch_distributed_train_b200.ops import functional as OF

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


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cooperative_step(B=100, steps=8):
    """Fused ConvNet forwards and backwards: afterwards the grid barrier's epoch word is well above 16, as in any process that
    has trained a few steps (a fold-group ticket that shared the word would then never see its last arrival)."""
    net = pdt.models.ConvNet(fused=True).to(dev())
    x = torch.rand(B, 1, 28, 28, device=dev())
    t = torch.randint(0, 10, (B,), device=dev())
    assert OF.fused_convnet_ok(x, net)
    for _ in range(steps):
        pdt.nn.CrossEntropyLoss()(net(x), t).backward()
    torch.cuda.synchronize()


def _assert_fused_matches_per_op(B=100):
    """The cooperative kernels against the per-op kernels on the same weights and data (test_gpu_kernels.py:
    test_cooperative_fused_layers_match_per_op_kernels): after the wide folds, both paths must still be right."""
    torch.manual_seed(2)
    a = pdt.models.ConvNet(fused=True).to(dev())
    b = pdt.models.ConvNet(fused=True).to(dev())
    b.load_state_dict(a.state_dict())
    x = torch.rand(B, 1, 28, 28, device=dev())
    t = torch.randint(0, 10, (B,), device=dev())
    crit = pdt.nn.CrossEntropyLoss()
    assert OF.fused_convnet_ok(x, a)
    la = crit(a(x), t)
    la.backward()
    mp = pytest.MonkeyPatch()
    mp.setenv("PDT_FUSED_LAYERS", "0")
    try:
        lb = crit(b(x), t)
        lb.backward()
    finally:
        mp.undo()
    assert abs(la.item() - lb.item()) < 1e-4, (la.item(), lb.item())
    for (n1, p1), (_, p2) in zip(a.named_parameters(), b.named_parameters()):
        scale = p2.grad.abs().max().item() + 1e-6
        # TF32 operand rounding of slightly different dy; conv biases in front of a BatchNorm have a true gradient of zero (noise level)
        assert (p1.grad - p2.grad).abs().max().item() <= 2e-2 * scale + 5e-4, (n1, (p1.grad - p2.grad).abs().max().item(), scale)
    for (n1, b1), (_, b2) in zip(a.named_buffers(), b.named_buffers()):
        assert torch.allclose(b1.float(), b2.float(), atol=1e-5, rtol=1e-5), n1


# ---- 1. per-op grid folds of more than 512 groups -------------------------------------------------------------------------------
def _assert_sums(got, terms, dims, what):
    """fp32 sums of up to 2 M terms in a tree a few dozen additions deep: 2e-5 of the sum of magnitudes."""
    ref, mag = terms.sum(dims), terms.abs().sum(dims)
    err = (got.double() - ref).abs()
    assert bool((err <= 2e-5 * mag + 1e-6).all()), (what, (err / (mag + 1e-30)).max().item())


@pytest.mark.parametrize("B", [2044, 2048, 2520])   # 4·B CTAs: 511, 512 and 630 fold groups
def test_conv1_statistics_fold_beyond_512_groups(B):
    _cooperative_step()
    x = torch.rand(B, 1, 28, 28, device=dev())
    w = torch.randn(16, 1, 5, 5, device=dev()) * 0.2
    b = torch.randn(16, device=dev()) * 0.1
    y, stats = _C.conv5x5_fwd(nhwc(x), w, b, True)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=2)
    assert torch.allclose(y.permute(0, 3, 1, 2).double(), ref, atol=1e-5, rtol=1e-5), (y.permute(0, 3, 1, 2).double() - ref).abs().max()
    yd = y.double()
    _assert_sums(stats[:16], yd, (0, 1, 2), "Σy")
    _assert_sums(stats[16:32], yd * yd, (0, 1, 2), "Σy²")
    assert stats[32].item() == B * 784
    y2, stats2 = _C.conv5x5_fwd(nhwc(x), w, b, True)
    assert torch.equal(y, y2) and torch.equal(stats, stats2)
    _assert_fused_matches_per_op()


def test_bn_relu_pool_backward_fold_beyond_512_groups():
    B, C, H = 2700, 16, 28   # 2700·14·14·4 threads: 8269 CTAs, 517 fold groups
    _cooperative_step()
    y = torch.rand(B, H, H, C, device=dev())            # x̂ within ±1.8 ...
    gamma = torch.rand(C, device=dev()) + 0.5
    beta = torch.full((C,), 3.0, device=dev())          # ... so every BN output is positive: ReLU routes by the arg-max only
    yd = y.double()
    mean = yd.mean((0, 1, 2))
    invstd = (yd.var((0, 1, 2), unbiased=False) + 1e-5).rsqrt()
    saved = torch.cat([mean, invstd]).float()
    dout = torch.randn(B, H // 2, H // 2, C, device=dev())
    sums, dgamma, dbeta = _C.bn_relu_pool_bwd_reduce(dout, y, saved, gamma, beta, False)
    # float64: x̂ at each window's arg-max (γ > 0: the arg-max of y), weighted by the pooled gradient
    yn = yd.permute(0, 3, 1, 2)
    _, idx = F.max_pool2d(yn, 2, 2, return_indices=True)
    sm, si = saved.double()[:C], saved.double()[C:]
    xhat = ((yn.flatten(2).gather(2, idx.flatten(2)) - sm[None, :, None]) * si[None, :, None])
    d = dout.double().permute(0, 3, 1, 2).flatten(2)
    _assert_sums(sums[:C], d.permute(0, 2, 1), (0, 1), "Σdz")
    _assert_sums(sums[C:], (d * xhat).permute(0, 2, 1), (0, 1), "Σdz·x̂")
    assert torch.equal(dbeta, sums[:C]) and torch.equal(dgamma, sums[C:])
    sums2, _, _ = _C.bn_relu_pool_bwd_reduce(dout, y, saved, gamma, beta, False)
    assert torch.equal(sums, sums2)
    _assert_fused_matches_per_op()


# ---- 2. the ConvNet beyond one CTA per SM ---------------------------------------------------------------------------------------
def _float64_twin(net):
    ref = pdt.models.ConvNet(num_classes=net.fc.out_features, fused=False).to(dev())
    ref.load_state_dict(net.state_dict())
    return ref.double()


def _assert_matches_float64(net, ref, loss, ref_loss):
    if math.isnan(ref_loss.item()):
        assert math.isnan(loss.item()), loss.item()
    else:
        # conv2 runs in TF32 (10-bit mantissa) forward and in dgrad: ~1e-3 relative per product
        assert abs(loss.item() - ref_loss.item()) < 2e-3, (loss.item(), ref_loss.item())
    for (n1, p1), (_, p2) in zip(net.named_parameters(), ref.named_parameters()):
        # TF32 as above, measured over the whole tensor: a few large elements of a small gradient (few counted targets, B = 1)
        # carry ~5 % TF32 noise; conv biases in front of a BatchNorm have a true gradient of zero (noise level)
        err, norm = (p1.grad.double() - p2.grad).norm().item(), p2.grad.norm().item()
        assert err <= 3e-2 * norm + 1e-4 * p2.numel() ** 0.5, (n1, err, norm)


@pytest.mark.parametrize("B", ["sms+1", 2048])
def test_convnet_beyond_one_cta_per_sm_matches_float64(B):
    B = sms() + 1 if B == "sms+1" else B
    _cooperative_step()
    torch.manual_seed(1)
    net = pdt.models.ConvNet(fused=True).to(dev())
    ref = _float64_twin(net)
    x = torch.rand(B, 1, 28, 28, device=dev())
    t = torch.randint(0, 10, (B,), device=dev())
    assert not OF.fused_convnet_ok(x, net)   # the per-op kernels
    loss = pdt.nn.CrossEntropyLoss()(net(x), t)
    loss.backward()
    ref_loss = F.cross_entropy(ref(x.double()), t)
    ref_loss.backward()
    _assert_matches_float64(net, ref, loss, ref_loss)
    for (n1, b1), (_, b2) in zip(net.named_buffers(), ref.named_buffers()):
        if n1.endswith("num_batches_tracked"):
            assert int(b1) == int(b2) == 1, n1
        else:
            # batch statistics of the TF32 conv2 output
            assert torch.allclose(b1.double(), b2.double(), atol=2e-3, rtol=1e-3), (n1, (b1.double() - b2.double()).abs().max().item())


# ---- 3. class counts (and ignored targets through the fused cross-entropy) ------------------------------------------------------
def _targets(kind, B, ncls, gen):
    t = torch.randint(0, ncls, (B,), device=dev(), generator=gen)
    if kind == "some_ignored":
        t[::3] = -100
    elif kind == "all_ignored":
        t[:] = -100
    return t


@pytest.mark.parametrize("targets", ["valid", "some_ignored", "all_ignored"])
@pytest.mark.parametrize("mode", ["plain", "upcoming", "upcoming_late"])
@pytest.mark.parametrize("B", [1, 100])
@pytest.mark.parametrize("ncls", [1, 2, 10, 16, 17, 64, 65])
def test_convnet_class_counts_match_float64(ncls, B, mode, targets):
    gen = torch.Generator(device=dev()).manual_seed(7)
    torch.manual_seed(3)
    net = pdt.models.ConvNet(num_classes=ncls, fused=True).to(dev())
    ref = _float64_twin(net)
    x = torch.rand(B, 1, 28, 28, device=dev(), generator=gen)
    t = _targets(targets, B, ncls, gen)
    crit = pdt.nn.CrossEntropyLoss()
    if mode == "plain":
        logits = net(x)
    else:
        with OF.upcoming_targets(t, loss_read_after_backward=mode == "upcoming_late"):
            logits = net(x)
        if ncls <= 16:   # the whole-forward kernel computed the loss
            assert getattr(logits, "_pdt_ce", None) is not None
    assert logits.shape == (B, ncls)
    loss = crit(logits, t)
    loss.backward()
    ref_loss = F.cross_entropy(ref(x.double()), t)
    ref_loss.backward()
    _assert_matches_float64(net, ref, loss, ref_loss)


# ---- 4. cross-entropy -----------------------------------------------------------------------------------------------------------
def _logits(kind, B, C, t):
    x = torch.randn(B, C, device=dev())
    if kind == "scaled":
        x = x * 1e3
    elif kind == "neg_inf":   # one -inf entry per row, never at the target
        col = torch.where(t >= 0, t + 1, torch.zeros_like(t)) % C
        x[torch.arange(B, device=dev()), col] = -math.inf
    elif kind == "equal":     # every other row constant
        x[::2] = 7.0
    return x


def _ce_reference(x, t, scale):
    xd = x.double().requires_grad_()
    loss = F.cross_entropy(xd, t)
    (g,) = torch.autograd.grad(loss * scale, xd)
    return loss.detach(), g


def _assert_ce_grad(got, ref, n):
    if n == 0:
        assert torch.equal(got, torch.zeros_like(got))
        return
    # __expf / __logf: a few ulp of the softmax
    assert torch.allclose(got.double(), ref, rtol=1e-5, atol=1e-6 / n), (got.double() - ref).abs().max().item()


def _assert_ce_loss(got, ref):
    if math.isnan(ref.item()):
        assert math.isnan(got.item()), got.item()
    else:
        # fp32 block reduction over up to 1000 rows, __logf of the row sums
        assert abs(got.item() - ref.item()) <= 1e-5 * abs(ref.item()) + 1e-6, (got.item(), ref.item())


@pytest.mark.parametrize("targets", ["valid", "some_ignored", "all_ignored"])
@pytest.mark.parametrize("kind", ["plain", "scaled", "neg_inf", "equal"])
@pytest.mark.parametrize("C", [1, 2, 10, 1024])
@pytest.mark.parametrize("B", [1, 7, 256, 1000])
def test_cross_entropy_matches_float64(B, C, kind, targets):
    if kind == "neg_inf" and C == 1:
        pytest.skip("a single class with a -inf logit has no finite loss")
    t = torch.randint(0, C, (B,), device=dev())
    if targets == "some_ignored":
        t[1::2] = -100
    elif targets == "all_ignored":
        t[:] = -100
    n = int((t >= 0).sum())
    x = _logits(kind, B, C, t)
    crit = pdt.nn.CrossEntropyLoss()
    for scale in (1.0, 3.0):
        ref_loss, ref_g = _ce_reference(x, t, scale)
        xs = x.clone().requires_grad_()
        loss = crit(xs, t)
        if scale == 1.0:
            loss.backward()
        else:
            (loss * scale).backward()
        _assert_ce_loss(loss, ref_loss)
        _assert_ce_grad(xs.grad, ref_g, n)
    # the separate backward kernel, from the saved softmax
    loss, probs = _C.cross_entropy_fwd(x, t, False)
    _assert_ce_loss(loss, ref_loss)
    assert torch.allclose(probs.double(), torch.softmax(x.double(), 1), rtol=1e-5, atol=1e-7)
    g = _C.cross_entropy_bwd(probs, t, torch.tensor(3.0, device=dev()))
    _assert_ce_grad(g, ref_g, n)


# ---- 5. linear head -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("N", [1, 7, 16])
@pytest.mark.parametrize("K", [1, 31, 33, 1568])
@pytest.mark.parametrize("B", [1, 3, 129, 1000])   # 129 and 1000 cross the 128-row staging chunk of linear_bwd_kernel
def test_linear_matches_float64(B, K, N, bias):
    x = torch.randn(B, K, device=dev(), requires_grad=True)
    w = torch.randn(N, K, device=dev(), requires_grad=True)
    b = torch.randn(N, device=dev(), requires_grad=True) if bias else None
    out = ops.linear(x, w, b)
    dout = torch.randn(B, N, device=dev())
    out.backward(dout)
    xd, wd, dd = x.detach().double(), w.detach().double(), dout.double()

    def close(got, ref, mag, what):
        # fp32 dot products: 1e-5 of the sum of the terms' magnitudes
        err = (got.double() - ref).abs()
        assert bool((err <= 1e-5 * mag + 1e-30).all()), (what, (err / (mag + 1e-30)).max().item())

    close(out, xd @ wd.t() + (b.detach().double() if bias else 0), xd.abs() @ wd.abs().t() + (b.detach().double().abs() if bias else 0), "out")
    close(x.grad, dd @ wd, dd.abs() @ wd.abs(), "dx")
    close(w.grad, dd.t() @ xd, dd.abs().t() @ xd.abs(), "dw")
    if bias:
        close(b.grad, dd.sum(0), dd.abs().sum(0), "db")


# ---- 6. BatchNorm + ReLU + max-pool ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_nchw", [False, True])
@pytest.mark.parametrize("C", [4, 8, 64])
def test_bn_relu_pool_channel_counts_match_float64(C, out_nchw):
    B, H = 24, 12
    # multiples of 1/256: distinct values of a pooling window stay apart after the fp32 BN affine, so the kernel and the
    # float64 oracle route every window's gradient to the same position (exact ties go to the first in both)
    y = torch.round(torch.randn(B, C, H, H, device=dev()) * 512) / 256 + 0.5
    gamma = torch.rand(C, device=dev()) + 0.5
    beta = torch.randn(C, device=dev()) * 0.1
    bn = nn.BatchNorm2d(C).to(dev()).double()
    with torch.no_grad():
        bn.weight.copy_(gamma)
        bn.bias.copy_(beta)
    yr = y.double().requires_grad_()
    ref = F.max_pool2d(F.relu(bn(yr)), 2, 2)
    yh = nhwc(y)
    yhd = yh.double()
    stats = torch.cat([yhd.sum((0, 1, 2)), (yhd * yhd).sum((0, 1, 2)), yhd.new_full((1,), B * H * H)]).float()
    rm, rv, nbt = torch.zeros(C, device=dev()), torch.ones(C, device=dev()), torch.zeros((), dtype=torch.int64, device=dev())
    out, saved = _C.bn_relu_pool_fwd(yh, stats, gamma, beta, rm, rv, nbt, 0.1, 1e-5, out_nchw)
    got = out if out_nchw else out.permute(0, 3, 1, 2)
    # fp32 statistics (var = E[y²] − mean²) and the BN affine in fp32
    assert torch.allclose(got.double(), ref, atol=1e-4, rtol=1e-4), (got.double() - ref).abs().max().item()
    assert torch.allclose(rm.double(), bn.running_mean, atol=1e-6, rtol=1e-5)
    assert torch.allclose(rv.double(), bn.running_var, atol=1e-6, rtol=1e-5) and int(nbt) == 1
    dout = torch.randn_like(ref)
    ref.backward(dout)
    d = dout.float().contiguous() if out_nchw else nhwc(dout.float())
    sums, dgamma, dbeta = _C.bn_relu_pool_bwd_reduce(d, yh, saved, gamma, beta, out_nchw)
    mag = (dout.abs().sum((0, 2, 3)) * 2).clamp_min(1.0)
    # fp32 sums over B·H·W/4 windows, as above
    assert bool(((dbeta.double() - bn.bias.grad).abs() <= 1e-5 * mag).all()), (dbeta.double() - bn.bias.grad).abs().max().item()
    assert bool(((dgamma.double() - bn.weight.grad).abs() <= 1e-4 * mag).all()), (dgamma.double() - bn.weight.grad).abs().max().item()
    dy = _C.bn_relu_pool_bwd_apply(d, yh, saved, gamma, beta, sums, stats[2 * C:], out_nchw)
    # fp32 statistics as above, amplified by the BatchNorm backward
    assert torch.allclose(dy.permute(0, 3, 1, 2).double(), yr.grad, atol=1e-4, rtol=1e-3), (dy.permute(0, 3, 1, 2).double() - yr.grad).abs().max().item()


@pytest.mark.parametrize("C,H", [(12, 12), (48, 12), (16, 13)])
def test_bn_relu_pool_rejects_shapes_it_cannot_index(C, H):
    B = 4
    y = torch.randn(B, H, H, C, device=dev())
    gamma, beta = torch.ones(C, device=dev()), torch.zeros(C, device=dev())
    stats = torch.cat([y.sum((0, 1, 2)), (y * y).sum((0, 1, 2)), y.new_full((1,), B * H * H)])
    saved = torch.cat([torch.zeros(C, device=dev()), torch.ones(C, device=dev())])
    dout = torch.randn(B, H // 2, H // 2, C, device=dev())
    with pytest.raises((RuntimeError, ValueError), match="bn_relu_pool"):
        _C.bn_relu_pool_fwd(y, stats, gamma, beta, None, None, None, 0.1, 1e-5, False)
    with pytest.raises((RuntimeError, ValueError), match="bn_relu_pool"):
        _C.bn_relu_pool_bwd_reduce(dout, y, saved, gamma, beta, False)
    with pytest.raises((RuntimeError, ValueError), match="bn_relu_pool"):
        _C.bn_relu_pool_bwd_apply(dout, y, saved, gamma, beta, torch.zeros(2 * C, device=dev()), stats[2 * C:], False)
    torch.cuda.synchronize()


def test_eval_batchnorm_with_large_running_mean_matches_float64():
    """Running means of 30 and variances of 0.01: the per-op eval path must normalise with the running variance as it is."""
    B = 32
    conv = nn.Conv2d(1, 16, 5, padding=2).to(dev())
    bn = nn.BatchNorm2d(16).to(dev()).eval()
    with torch.no_grad():
        conv.weight.mul_(0.1)
        conv.bias.copy_(30 + torch.linspace(0.0, 1.5, 16, device=dev()))
        bn.running_mean.copy_(30 + torch.linspace(0.0, 1.5, 16, device=dev()) - 0.3)   # x̂ ≈ 3: positive after BN, kept by ReLU
        bn.running_var.fill_(0.01)
        bn.weight.copy_(torch.rand(16, device=dev()) + 0.5)
        bn.bias.copy_(torch.randn(16, device=dev()) * 0.1)
    x = torch.rand(B, 1, 28, 28, device=dev())
    with torch.no_grad():
        out = ops.conv_bn_relu_pool(x, conv, bn)
        yd = F.conv2d(x.double(), conv.weight.double(), conv.bias.double(), padding=2)
        ref = F.max_pool2d(F.relu(F.batch_norm(yd, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(),
                                               bn.bias.double(), False, 0.0, bn.eps)), 2, 2)
    assert out.shape == ref.shape
    # y ≈ 30 in fp32 (ulp 1.9e-6) is magnified tenfold by 1/std, and the fp32 BN affine cancels terms of ≈300 down to O(1)
    assert torch.allclose(out.double(), ref, atol=5e-4, rtol=1e-4), (out.double() - ref).abs().max().item()


# ---- 7. bn_finalize -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 130, 1000])
def test_bn_finalize_matches_float64_and_batchnorm(C):
    N, H = 6, 5
    x = torch.randn(N, C, H, H, device=dev()) * 2 + 3
    stats = ops.bn_local_stats(x)
    rm, rv = torch.randn(C, device=dev()) * 0.1, torch.rand(C, device=dev()) + 0.5
    bn = nn.BatchNorm2d(C, momentum=0.1, eps=1e-5).to(dev()).train()
    with torch.no_grad():
        bn.running_mean.copy_(rm)
        bn.running_var.copy_(rv)
        bn(x)
    rm0, rv0 = rm.double(), rv.double()
    mean, invstd, count = ops.bn_finalize(stats, C, 1e-5, 0.1, rm, rv)
    xd = x.double()
    n = N * H * H
    m_ref = xd.mean((0, 2, 3))
    var_ref = xd.var((0, 2, 3), unbiased=False)
    assert count.item() == n
    assert torch.allclose(mean.double(), m_ref, rtol=1e-6, atol=1e-7)
    assert torch.allclose(invstd.double(), (var_ref + 1e-5).rsqrt(), rtol=1e-6)
    rm_ref = 0.9 * rm0 + 0.1 * m_ref
    rv_ref = 0.9 * rv0 + 0.1 * var_ref * n / (n - 1)
    # fp32 running-statistics update
    assert torch.allclose(rm.double(), rm_ref, rtol=1e-6, atol=1e-6) and torch.allclose(rv.double(), rv_ref, rtol=1e-6, atol=1e-6)
    assert torch.allclose(rm, bn.running_mean, rtol=1e-5, atol=1e-6) and torch.allclose(rv, bn.running_var, rtol=1e-5, atol=1e-6)
