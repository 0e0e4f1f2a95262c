"""The ConvNet's input gradients, eval-mode backward and double backward against float64.

Three common uses of a trained classifier beyond the training step run on the native kernels: gradients with respect to the image
(adversarial examples, adversarial training, saliency maps), backward through a model in ``eval()`` (fine-tuning with frozen
BatchNorm, attacking an eval model), and double backward (``create_graph=True``: gradient penalties, Hessian-vector products).  The
first two take the per-op kernels: conv1's data gradient (a SIMT kernel, 16→1) and the eval form of the BatchNorm + ReLU + max-pool
backward (the running statistics are constants, so there are no batch-mean terms).  The third is refused: the kernels' gradients
carry no graph, so every native backward raises under ``create_graph=True`` instead of returning a gradient that a penalty term
would silently drop out of.

Oracle: test_convnet_module_options.py's ``fused=False`` float64 twin, loaded from the same ``state_dict``, with perturbed affines
and no TF32 inside cuDNN or cuBLAS.  Tolerance policy (test_kernel_edges.py): TF32 level wherever conv2 takes part, fp32 level
elsewhere."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C, ops
from pytorch_distributed_train_b200.ops import functional as OF
from test_convnet_module_options import NATIVE, _assert_buffers_match, _assert_matches_float64, _models

pytestmark = pytest.mark.gpu

EPS = 1e-5


@pytest.fixture(autouse=True)
def _fp32_reference():
    # the oracle must be true fp32 / fp64: no TF32 inside cuDNN/cuBLAS
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def dev():
    return torch.device("cuda", 0)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _batch_size(B):
    return {"sms": sms(), "sms+1": sms() + 1}.get(B, B)


# ---- 1. conv1's data gradient ----------------------------------------------------------------------------------------------------
def _dgrad64(dy, w):
    """float64 d/dx of conv2d(x, w, padding=2) against the NHWC gradient dy [B,H,W,Cout], as NCHW [B,Cin,H,W]."""
    x = torch.zeros(dy.shape[0], w.shape[1], dy.shape[1], dy.shape[2], dtype=torch.float64, device=dev(), requires_grad=True)
    return torch.autograd.grad(F.conv2d(x, w.double(), padding=2), x, dy.double().permute(0, 3, 1, 2))[0]


@pytest.mark.parametrize("B", [1, 3, 100, 2048])
def test_conv1_data_gradient_matches_float64(B):
    gen = torch.Generator(device=dev()).manual_seed(B)
    # integers: every product and partial sum is exact in fp32, so the kernel must match exactly, the pad-2 borders included
    dy = torch.randint(-3, 4, (B, 28, 28, 16), device=dev(), generator=gen).float()
    w = torch.randint(-2, 3, (16, 1, 5, 5), device=dev(), generator=gen).float()
    dx = _C.conv5x5_dgrad(dy, w)
    assert dx.shape == (B, 28, 28, 1)
    assert torch.equal(dx.permute(0, 3, 1, 2).double(), _dgrad64(dy, w))
    # random data: a pixel is one chain of 400 fmaf, so |error| ≤ γ₄₀₀·Σ|terms| with γₙ = n·2⁻²⁴ / (1 − n·2⁻²⁴) < 2.4e-5
    dy = torch.randn(B, 28, 28, 16, device=dev(), generator=gen)
    w = torch.randn(16, 1, 5, 5, device=dev(), generator=gen) * 0.2
    dx = _C.conv5x5_dgrad(dy, w)
    ref, mag = _dgrad64(dy, w), _dgrad64(dy.abs(), w.abs())
    err = (dx.permute(0, 3, 1, 2).double() - ref).abs()
    assert bool((err <= 2.4e-5 * mag).all()), (err / mag).max().item()
    assert torch.equal(dx, _C.conv5x5_dgrad(dy, w))


@pytest.mark.parametrize("cin,cout", [(16, 16), (1, 32), (32, 16)])
def test_conv_data_gradient_refuses_shapes_no_kernel_computes(cin, cout):
    dy = torch.randn(2, 28, 28, cout, device=dev())
    w = torch.randn(cout, cin, 5, 5, device=dev())
    torch.cuda.synchronize()
    launches = _C.kernel_launch_count()
    with pytest.raises(ValueError, match="conv5x5_dgrad"):
        _C.conv5x5_dgrad(dy, w)
    assert _C.kernel_launch_count() == launches   # refused on the host, before any launch


# ---- 2. BatchNorm + ReLU + max-pool backward in eval mode -------------------------------------------------------------------------
def _eval_frame(B, C, H, affine, gen):
    """y, running mean / variance, γ, β where every channel's y lies on a grid of std/16 about a running mean of up to 3000 std.

    Standard deviations are powers of two and means whole multiples of them, so y, the mean and the variance are exact in fp32 and
    y − mean is exact too.  Values sit half a grid step off the grid's zero and β is a multiple of γ/16, so no BatchNorm output lies
    within |γ|/32 of the ReLU threshold, and distinct values of a window stay |γ|/16 apart: fp32 and float64 route every window
    alike, and exact ties (γ = 0, repeated values) go to the first position in both."""
    std = torch.tensor([0.125, 1.0, 8.0], device=dev()).repeat(C)[:C]
    r = torch.linspace(-3000, 3000, C, device=dev()).round()
    r[C // 2] = 0
    mean, var = std * r, std * std
    k = torch.randint(-48, 48, (B, C, H, H), device=dev(), generator=gen).float()
    y = std[None, :, None, None] * (r[None, :, None, None] + (k + 0.5) / 16)
    if not affine:
        return y, mean, var, None, None
    gamma = torch.rand(C, device=dev(), generator=gen) + 0.5
    gamma[::3] *= -1
    gamma[1] = 0.0
    beta = gamma * torch.randint(-8, 9, (C,), device=dev(), generator=gen).float() / 16
    beta[1] = 0.25   # γ = 0: every window ties at β > 0 and routes to its first position
    return y, mean, var, gamma, beta


@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("out_nchw", [False, True])
@pytest.mark.parametrize("C,H", [(16, 28), (32, 14)])
def test_bn_relu_pool_eval_backward_matches_float64(C, H, out_nchw, affine):
    B = 20
    y, mean, var, gamma, beta = _eval_frame(B, C, H, affine, torch.Generator(device=dev()).manual_seed(C + out_nchw))
    yh = nhwc(y)
    out, saved = _C.bn_relu_pool_fwd(yh, torch.cat([mean, var]), gamma, beta, None, None, None, 0.0, EPS, out_nchw, mean_var=True)
    yr = y.double().requires_grad_()
    g64 = gamma.double().requires_grad_() if affine else None
    b64 = beta.double().requires_grad_() if affine else None
    ref = F.max_pool2d(F.relu(F.batch_norm(yr, mean.double(), var.double(), g64, b64, False, 0.0, EPS)), 2, 2)
    got = out if out_nchw else out.permute(0, 3, 1, 2)
    # the fp32 affine γ·invstd·y + (β − mean·γ·invstd) cancels terms of up to 3000·|γ| down to O(1): a few ulp of those
    assert torch.allclose(got.double(), ref, atol=1e-6 * 3000 * 1.5 + 1e-5, rtol=1e-5), (got.double() - ref).abs().max().item()
    dout = torch.randn(ref.shape, device=dev())
    ref.backward(dout.double())
    d = dout.contiguous() if out_nchw else nhwc(dout)
    _, dgamma, dbeta = _C.bn_relu_pool_bwd_reduce(d, yh, saved, gamma, beta, out_nchw)
    dy = _C.bn_relu_pool_bwd_apply(d, yh, saved, gamma, beta, None, None, out_nchw, mean_var=True)
    # dy = γ·invstd·dz at the arg-max, 0 elsewhere: a few ulp of the product (rsqrtf, two roundings); misrouting moves O(1)
    assert torch.allclose(dy.permute(0, 3, 1, 2).double(), yr.grad, rtol=1e-6, atol=0), (dy.permute(0, 3, 1, 2).double() - yr.grad).abs().max().item()
    if affine:
        # fp32 sums over B·H·W/4 windows of dz and dz·x̂ (|x̂| ≤ 3.1, exact to a few ulp)
        mag = dout.double().abs().sum((0, 2, 3))
        assert bool(((dbeta.double() - b64.grad).abs() <= 1e-5 * mag).all()), (dbeta.double() - b64.grad).abs().max().item()
        assert bool(((dgamma.double() - g64.grad).abs() <= 4e-5 * mag).all()), (dgamma.double() - g64.grad).abs().max().item()
    # the statistics' form is explicit: batch statistics need the sums and the count, the running ones take neither
    with pytest.raises(RuntimeError, match="bn_relu_pool_bwd_apply"):
        _C.bn_relu_pool_bwd_apply(d, yh, saved, gamma, beta, None, None, out_nchw)
    with pytest.raises(RuntimeError, match="bn_relu_pool_bwd_apply"):
        _C.bn_relu_pool_bwd_apply(d, yh, saved, gamma, beta, torch.zeros(2 * C, device=dev()), torch.ones(1, device=dev()), out_nchw,
                                  mean_var=True)


# ---- 3. the ConvNet: input gradients in training mode --------------------------------------------------------------------------
def _stock(net):
    pass


def _batch(B, seed):
    gen = torch.Generator(device=dev()).manual_seed(seed)
    return torch.rand(B, 1, 28, 28, device=dev(), generator=gen), torch.randint(0, 10, (B,), device=dev(), generator=gen)


def _assert_input_grad_matches(got, ref, rel):
    """TF32 level over the whole [B, 1, 28, 28] tensor: the gradient reaches the image through conv2's data gradient."""
    err, norm = (got.double() - ref).norm().item(), ref.norm().item()
    assert err <= rel * norm, (err, norm)


def _rel(B):
    # one image: as test_convnet_module_options.py's measured bound for the parameters
    return 2.5e-1 if B == 1 else 3e-2


@pytest.mark.parametrize("frozen", [False, True])
@pytest.mark.parametrize("B", [1, 3, 100, "sms", "sms+1"])
def test_training_input_gradient_matches_float64(B, frozen):
    B = _batch_size(B)
    net, ref, _, _ = _models(_stock)
    if frozen:   # an attack loop: the model's parameters fixed, the gradient taken with respect to the image only
        for p in (*net.parameters(), *ref.parameters()):
            p.requires_grad_(False)
    x, t = _batch(B, B)
    x.requires_grad_()
    assert not OF.fused_convnet_ok(x, net)   # the per-op kernels compute d/d(image)
    loss = pdt.nn.CrossEntropyLoss()(net(x), t)
    xr = x.detach().double().requires_grad_()
    ref_loss = F.cross_entropy(ref(xr), t)
    if frozen:
        (gx,) = torch.autograd.grad(loss, x)
        (gr,) = torch.autograd.grad(ref_loss, xr)
        assert abs(loss.item() - ref_loss.item()) < 2e-3, (loss.item(), ref_loss.item())
        assert all(p.grad is None for p in net.parameters())
    else:
        loss.backward()
        ref_loss.backward()
        gx, gr = x.grad, xr.grad
        _assert_matches_float64(net, ref, loss, ref_loss, rel=_rel(B))
    assert gx.shape == x.shape
    _assert_input_grad_matches(gx, gr, _rel(B))
    _assert_buffers_match(net, ref, 1)


# ---- 4. the ConvNet: backward in eval mode ---------------------------------------------------------------------------------------
def _eval_models(name):
    """The model and its twin after three training forwards of the model (the native kernels set the running statistics), in eval."""
    if name == "sync_batchnorm":
        net, ref, _, _ = _models(_stock)
        net = pdt.SyncBatchNorm.convert_sync_batchnorm(net)   # eval takes the per-op path and needs no process group
    else:
        net, ref, _, _ = _models(NATIVE[name][0] if name != "stock" else _stock)
    with torch.no_grad():
        for i in range(3):
            net(_batch(100, 100 + i)[0])
    ref.load_state_dict(net.state_dict())
    return net.eval(), ref.eval()


@pytest.mark.parametrize("name", ["stock", *NATIVE, "sync_batchnorm"])
def test_eval_backward_matches_float64(name):
    B = 100
    net, ref = _eval_models(name)
    buffers = {n: b.clone() for n, b in net.named_buffers()}
    x, t = _batch(B, 7)
    x.requires_grad_()
    loss = pdt.nn.CrossEntropyLoss()(net(x), t)
    loss.backward()
    xr = x.detach().double().requires_grad_()
    ref_loss = F.cross_entropy(ref(xr), t)
    ref_loss.backward()
    _assert_matches_float64(net, ref, loss, ref_loss)
    # Three passes at momentum 0.1 leave running statistics far from the batch's: BatchNorm's outputs then vary little within a
    # pooling window, and TF32 rounding of conv2 moves the arg-max of more windows.  Measured on an H100 against float64 on this file's
    # data: the native kernels up to 4.1 % of the norm (stock 4.1 %, bn_options 3.6 %, momentum_none 1.8 %), torch's own TF32 layers
    # (cuDNN) 2.9 %, 3.6 % and 2.6 % on the same models.
    _assert_input_grad_matches(x.grad, xr.grad, 6e-2)
    # eval reads the running statistics and never writes them
    for n, b in net.named_buffers():
        assert torch.equal(b, buffers[n]), n


# ---- 5. double backward is refused on every native route --------------------------------------------------------------------------
# (route, criterion): "pdt" refuses in the cross-entropy node, "torch" lets torch's cross-entropy run and refuses in the model's first
# native node; "pdt_upcoming" takes the cross-entropy the fused forward kernel computed
DOUBLE = [("fused_train", "pdt"), ("fused_train", "pdt_upcoming"), ("fused_train", "torch"), ("per_op_train", "pdt"),
          ("per_op_train", "torch"), ("per_op_eval", "pdt"), ("per_op_eval", "torch")]
REFUSED_BY = {"pdt": "cross_entropy", "pdt_upcoming": r"cross_entropy \(computed by the fused forward\)",
              ("fused_train", "torch"): "fused ConvNet layer 2", ("per_op_train", "torch"): "linear", ("per_op_eval", "torch"): "linear"}


@pytest.mark.parametrize("route,criterion", DOUBLE)
def test_double_backward_is_refused(route, criterion):
    B = 100
    if route == "per_op_eval":
        net, ref = _eval_models("stock")
    else:
        net, ref, _, _ = _models(_stock)
    x, t = _batch(B, 11)
    xr = x.double()
    if route != "fused_train":
        x.requires_grad_()
        xr.requires_grad_()
    assert OF.fused_convnet_ok(x, net) == (route == "fused_train")
    if criterion == "pdt_upcoming":
        with OF.upcoming_targets(t):
            logits = net(x)
        assert getattr(logits, "_pdt_ce", None) is not None
    else:
        logits = net(x)
    loss = pdt.nn.CrossEntropyLoss()(logits, t) if criterion.startswith("pdt") else F.cross_entropy(logits, t)
    wrt = list(net.parameters()) + ([x] if x.requires_grad else [])
    ref_wrt = list(ref.parameters()) + ([xr] if xr.requires_grad else [])
    with pytest.raises(RuntimeError, match=REFUSED_BY.get(criterion) or REFUSED_BY[(route, criterion)]):
        torch.autograd.grad(loss, wrt, create_graph=True)
    # the refusal leaves the graph as it was: without create_graph the same call returns the gradients
    ref_loss = F.cross_entropy(ref(xr), t)
    grads = torch.autograd.grad(loss, wrt)
    ref_grads = torch.autograd.grad(ref_loss, ref_wrt)
    assert abs(loss.item() - ref_loss.item()) < 2e-3, (loss.item(), ref_loss.item())
    names = [n for n, _ in net.named_parameters()] + (["x"] if x.requires_grad else [])
    for n, g, r in zip(names, grads, ref_grads, strict=True):
        # test_convnet_module_options.py's bounds
        err, norm = (g.double() - r).norm().item(), r.norm().item()
        assert err <= 3e-2 * norm + (0 if n == "x" else 1e-4 * r.numel() ** 0.5), (n, err, norm)


@pytest.mark.parametrize("training", [True, False])
def test_conv_bn_relu_pool_refuses_double_backward(training):
    conv = nn.Conv2d(1, 16, 5, padding=2).to(dev())
    bn = nn.BatchNorm2d(16).to(dev()).train(training)
    with torch.no_grad():
        bn.running_mean.normal_(0.0, 0.1)
        bn.running_var.uniform_(0.5, 1.5)
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0.0, 0.2)
    rm, rv = bn.running_mean.double(), bn.running_var.double()
    x = torch.rand(8, 1, 28, 28, device=dev(), requires_grad=True)
    c = torch.randn(8, 16, 14, 14, device=dev())
    loss = (ops.conv_bn_relu_pool(x, conv, bn) * c).sum()
    with pytest.raises(RuntimeError, match="conv_bn_relu_pool"):
        torch.autograd.grad(loss, x, create_graph=True)
    (gx,) = torch.autograd.grad(loss, x)
    xr = x.detach().double().requires_grad_()
    y = F.conv2d(xr, conv.weight.double(), conv.bias.double(), padding=2)
    z = F.batch_norm(y, rm, rv, bn.weight.double(), bn.bias.double(), training, 0.0, bn.eps)
    (gr,) = torch.autograd.grad((F.max_pool2d(F.relu(z), 2, 2) * c.double()).sum(), xr)
    # fp32 kernels throughout (conv1 forward and data gradient, BatchNorm)
    err, norm = (gx.double() - gr).norm().item(), gr.norm().item()
    assert err <= 1e-4 * norm, (err, norm)


def test_cross_entropy_refuses_double_backward():
    B = 64
    logits = torch.randn(B, 10, device=dev(), requires_grad=True)
    t = torch.randint(0, 10, (B,), device=dev())
    loss = pdt.nn.CrossEntropyLoss()(logits, t)
    with pytest.raises(RuntimeError, match="cross_entropy"):
        torch.autograd.grad(loss, logits, create_graph=True)
    (g,) = torch.autograd.grad(loss, logits)
    xd = logits.detach().double().requires_grad_()
    ref = F.cross_entropy(xd, t)
    (gr,) = torch.autograd.grad(ref, xd)
    # test_kernel_edges.py's bounds: fp32 reduction and __logf for the loss, a few ulp of the softmax for the gradient
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item()) + 1e-6, (loss.item(), ref.item())
    assert torch.allclose(g.double(), gr, rtol=1e-5, atol=1e-6 / B), (g.double() - gr).abs().max().item()


def test_linear_refuses_double_backward():
    x = torch.randn(33, 1568, device=dev(), requires_grad=True)
    w = torch.randn(10, 1568, device=dev(), requires_grad=True)
    b = torch.randn(10, device=dev(), requires_grad=True)
    c = torch.randn(33, 10, device=dev())
    loss = (ops.linear(x, w, b) * c).sum()   # the gradient at the output is c, exactly
    with pytest.raises(RuntimeError, match="linear"):
        torch.autograd.grad(loss, (x, w, b), create_graph=True)
    gx, gw, gb = torch.autograd.grad(loss, (x, w, b))
    xd, wd, cd = x.detach().double(), w.detach().double(), c.double()
    # fp32 dot products: 1e-5 of the sum of the terms' magnitudes (test_kernel_edges.py)
    for got, ref, mag in ((gx, cd @ wd, cd.abs() @ wd.abs()), (gw, cd.t() @ xd, cd.abs().t() @ xd.abs()), (gb, cd.sum(0), cd.abs().sum(0))):
        assert bool(((got.double() - ref).abs() <= 1e-5 * mag).all()), ((got.double() - ref).abs() / mag).max().item()
