"""Training-mode BatchNorm statistics where a channel's mean dwarfs its spread, against float64.

A conv bias in front of a BatchNorm has no true gradient, so it stays wherever it was initialised or loaded; inputs with an
offset and β₁ ≫ γ₁ do the same to layer 1's or layer 2's outputs.  The batch variance must then not come from Σy²/n − mean²
in fp32, which loses digits in proportion to mean²/var.  Here the conv biases are set to r times the spread of each channel's
conv output, for mean/spread ratios r up to 3000, and the statistics the native paths normalise with (the saved mean and
invstd) and the running statistics they update are compared with float64 statistics of the kernels' own conv outputs, so that
TF32 rounding in conv2 stays out of the comparison.  Covered: the cooperative forward kernel (convnet_fwd), the per-op
conv5x5_fwd → bn_relu_pool_fwd pair for both convolutions, a whole training step of the ConvNet on both routes against a
float64 twin followed by an eval forward with the updated running statistics, and that every path repeats bit for bit."""
import pytest
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C
from pytorch_distributed_train_b200.ops import functional as OF

pytestmark = pytest.mark.gpu

EPS, MOM = 1e-5, 0.1
RATIOS = [1, 30, 300, 3000]


@pytest.fixture(autouse=True)
def _fp32_reference():
    # the float64 twin's layers must not pick up TF32 either
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def dev():
    return torch.device("cuda", 0)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _spread(y_nchw):
    """Per-channel standard deviation (float64) of a conv output without its bias."""
    return y_nchw.double().std((0, 2, 3))


def _check_layer(y, saved, rm, rv, rm0, rv0, C, what):
    """saved = (mean, invstd) and the running statistics updated from (rm0, rv0), against float64 statistics of y (NHWC).

    Tolerances: 1e-5 of the spread for the mean and 2e-5 relative for the variance, as for ordinary data, plus what fp32 itself
    costs at a large mean: an fp32 mean is good to an ulp or two (2⁻²²·|mean|), and each CTA's fp32 sum of its n elements, from
    which its share of the between-CTA deviations comes, is rounded to 2⁻²⁴ of n·|mean| — worth up to 2⁻²⁴·|mean|/spread of
    the variance.  Σy²/n − mean² in fp32 misses that by orders of magnitude from |mean|/spread ≈ 30 on."""
    v = y.double().reshape(-1, C)
    cnt = v.shape[0]
    mean, var = v.mean(0), v.var(0, unbiased=False)
    spread = var.sqrt()
    k_mean, k_invstd = saved[:C].double(), saved[C:2 * C].double()
    err = ((k_mean - mean).abs() / (1e-5 * spread + 2.0 ** -22 * mean.abs())).max().item()
    assert err <= 1, (what, "mean (share of the tolerance)", err)
    var_tol = 2e-5 + 2.0 ** -24 * mean.abs() / spread
    k_var = 1.0 / k_invstd ** 2 - EPS   # the variance the kernel normalised with
    err = ((k_var - var).abs() / var / var_tol).max().item()
    assert err <= 1, (what, "var (share of the tolerance)", err)
    ref_rm = (1 - MOM) * rm0 + MOM * mean
    err = ((rm.double() - ref_rm).abs() / (1e-5 * spread + 2.0 ** -22 * (ref_rm.abs() + mean.abs()))).max().item()
    assert err <= 1, (what, "running mean (share of the tolerance)", err)
    ref_rv = (1 - MOM) * rv0 + MOM * var * cnt / max(cnt - 1, 1)
    err = ((rv.double() - ref_rv).abs() / ref_rv / var_tol).max().item()
    assert err <= 1, (what, "running var (share of the tolerance)", err)


def _running(C, m0, v0):
    return (torch.full((C,), m0, device=dev()), torch.full((C,), v0, device=dev()), torch.zeros((), dtype=torch.long, device=dev()))


# ---- a. the cooperative forward kernel --------------------------------------------------------------------------------------
def _fused_inputs(B, r, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(dev())
    x = torch.rand(B, 1, 28, 28, generator=g).to(dev())
    w1 = rnd(16, 1, 5, 5, scale=0.2)
    g1, be1 = 1.0 + rnd(16, scale=0.1), rnd(16, scale=0.1)
    w2 = rnd(32, 16, 5, 5, scale=0.05)
    g2, be2 = 1.0 + rnd(32, scale=0.1), rnd(32, scale=0.1)
    fcw, fcb = rnd(10, 1568, scale=0.02), rnd(10, scale=0.1)
    t = torch.randint(0, 10, (B,), generator=g).to(dev())
    b1 = (r * _spread(F.conv2d(x.double(), w1.double(), padding=2))).float()
    args = [x, w1, b1, g1, be1, w2, torch.zeros(32, device=dev()), g2, be2, fcw, fcb, t]
    # layer 2's spread from the kernel's own conv2 output without a bias (its input depends on layer 1 only)
    (_, _, _, _, y2, *_), _ = _fused_run(args)
    args[6] = (r * _spread(y2.permute(0, 3, 1, 2))).float()
    return args


def _fused_run(args):
    x, w1, b1, g1, be1, w2, b2, g2, be2, fcw, fcb, t = args
    rm1, rv1, nbt1 = _running(16, 0.25, 2.0)
    rm2, rv2, nbt2 = _running(32, -0.5, 3.0)
    outs = _C.convnet_fwd(x, w1, b1, g1, be1, rm1, rv1, nbt1, MOM, EPS, w2, b2, g2, be2, rm2, rv2, nbt2, MOM, EPS, fcw, fcb, t)
    torch.cuda.synchronize()
    return outs, (rm1, rv1, nbt1, rm2, rv2, nbt2)


@pytest.mark.parametrize("r", RATIOS)
@pytest.mark.parametrize("B", [1, 3, 100, "sms"])
def test_fused_forward_statistics_with_large_means(B, r):
    B = sms() if B == "sms" else B
    args = _fused_inputs(B, r, 17 + B)
    first, state = _fused_run(args)
    _, y1, saved1, _, y2, saved2, *_ = first
    rm1, rv1, nbt1, rm2, rv2, nbt2 = state
    _check_layer(y1, saved1, rm1, rv1, 0.25, 2.0, 16, "layer 1")
    _check_layer(y2, saved2, rm2, rv2, -0.5, 3.0, 32, "layer 2")
    assert nbt1.item() == 1 and nbt2.item() == 1
    second, state2 = _fused_run(args)
    names = ["p1", "y1", "saved1", "out", "y2", "saved2", "logits", "loss", "dlogits", "loss_parts"]
    for name, a, b in zip(names, first, second):
        assert torch.equal(a, b), name
    for a, b in zip(state, state2):
        assert torch.equal(a, b)


# ---- b. the per-op kernels: conv5x5_fwd's statistics through bn_relu_pool_fwd ---------------------------------------------------
def _per_op_layer(xh, w, b, gamma, beta, C):
    rm, rv, nbt = _running(C, 0.25, 2.0)
    y, stats = _C.conv5x5_fwd(xh, w, b, True, centred=True)
    out, saved = _C.bn_relu_pool_fwd(y, stats, gamma, beta, rm, rv, nbt, MOM, EPS, False, centred=True)
    torch.cuda.synchronize()
    return (y, out, saved), (rm, rv, nbt)


@pytest.mark.parametrize("r", RATIOS)
@pytest.mark.parametrize("layer,B", [(1, 3), (1, 2048), (2, 3), (2, 100), (2, 2048)])
def test_per_op_statistics_with_large_means(layer, B, r):
    g = torch.Generator(device="cpu").manual_seed(5 + B)
    cin, C, H = (1, 16, 28) if layer == 1 else (16, 32, 14)
    x = torch.rand(B, cin, H, H, generator=g).to(dev())
    w = (torch.randn(C, cin, 5, 5, generator=g) * (0.2 if layer == 1 else 0.05)).to(dev())
    b = (r * _spread(F.conv2d(x.double(), w.double(), padding=2))).float()
    gamma, beta = (1.0 + torch.randn(C, generator=g) * 0.1).to(dev()), (torch.randn(C, generator=g) * 0.1).to(dev())
    first, state = _per_op_layer(nhwc(x), w, b, gamma, beta, C)
    y, _, saved = first
    rm, rv, nbt = state
    _check_layer(y, saved, rm, rv, 0.25, 2.0, C, f"conv{layer}")
    assert nbt.item() == 1
    second, state2 = _per_op_layer(nhwc(x), w, b, gamma, beta, C)
    for a, c in zip(first + state, second + state2):
        assert torch.equal(a, c)


# ---- c. one training step of the ConvNet against a float64 twin, then an eval forward -----------------------------------------
def _offset_biases(net, x, r):
    """Both conv biases at r times their channel's spread (layer 2's measured on layer 1's float64 output)."""
    with torch.no_grad():
        c1, bn1, c2 = net.layer1[0], net.layer1[1], net.layer2[0]
        y1 = F.conv2d(x.double(), c1.weight.double(), padding=2)
        c1.bias.copy_((r * _spread(y1)).float())
        h = F.max_pool2d(F.relu(F.batch_norm(y1, None, None, bn1.weight.double(), bn1.bias.double(), True, 0.0, bn1.eps)), 2, 2)
        c2.bias.copy_((r * _spread(F.conv2d(h, c2.weight.double(), padding=2))).float())


def _float64_twin(net):
    ref = pdt.models.ConvNet(num_classes=net.fc.out_features, fused=False).to(dev())
    ref.load_state_dict(net.state_dict())
    for a, b in zip((net.layer1[1], net.layer2[1]), (ref.layer1[1], ref.layer2[1])):
        b.momentum = a.momentum
    return ref.double()


def _assert_matches_float64(net, ref, loss, ref_loss):
    # conv2 runs in TF32 (10-bit mantissa) forward and in dgrad: ~1e-3 relative per product
    assert abs(loss.item() - ref_loss.item()) < 2e-3, (loss.item(), ref_loss.item())
    for (n1, p1), (_, p2) in zip(net.named_parameters(), ref.named_parameters()):
        # TF32 as above, over the whole tensor; conv biases in front of a BatchNorm have a true gradient of zero (noise level)
        err, norm = (p1.grad.double() - p2.grad).norm().item(), p2.grad.norm().item()
        assert err <= 3e-2 * norm + 1e-4 * p2.numel() ** 0.5, (n1, err, norm)


@pytest.mark.parametrize("route", ["fused", "per_op"])
def test_training_step_with_large_means_matches_float64(route):
    # |mean|/spread = 300: Σy²/n − mean² in fp32 is 2 % off there; at 3000 the fp32 y itself (ulp 2⁻²³·3000 of the spread) costs
    # the conv1 weight gradient about the TF32 tolerance below
    r = 300
    B = 100 if route == "fused" else sms() + 1
    torch.manual_seed(1)
    x = torch.rand(B, 1, 28, 28, device=dev())
    t = torch.randint(0, 10, (B,), device=dev())

    def make():
        torch.manual_seed(1)
        net = pdt.models.ConvNet(fused=True).to(dev())
        _offset_biases(net, x, r)
        # momentum 1: the running statistics are this batch's, so that the eval forward below normalises to O(1) values and
        # depends on every digit of the running variance
        net.layer1[1].momentum = net.layer2[1].momentum = 1.0
        return net

    ref = _float64_twin(make())
    nets = []
    for _ in range(2):   # the second net repeats the step: bit for bit
        net = make()
        assert OF.fused_convnet_ok(x, net) == (route == "fused")
        loss = pdt.nn.CrossEntropyLoss()(net(x), t)
        loss.backward()
        nets.append((net, loss))
    (net, loss), (net_b, loss_b) = nets
    assert torch.equal(loss, loss_b)
    for (n1, p1), (_, p2) in zip(net.named_parameters(), net_b.named_parameters()):
        assert torch.equal(p1.grad, p2.grad), n1
    for (n1, b1), (_, b2) in zip(net.named_buffers(), net_b.named_buffers()):
        assert torch.equal(b1, b2), n1
    ref_loss = F.cross_entropy(ref(x.double()), t)
    ref_loss.backward()
    _assert_matches_float64(net, ref, loss, ref_loss)
    for (n1, b1), (_, b2) in zip(net.named_buffers(), ref.named_buffers()):
        if n1.endswith("num_batches_tracked"):
            assert int(b1) == int(b2) == 1, n1
        else:
            # batch statistics of the TF32 conv2 output
            assert torch.allclose(b1.double(), b2.double(), atol=2e-3, rtol=1e-3), (n1, (b1.double() - b2.double()).abs().max().item())
    net.eval()
    ref.eval()
    with torch.no_grad():
        out, ref_out = net(x), ref(x.double())
    # TF32 in conv2, and y ≈ r·spread in fp32 (ulp 2⁻²³·r of the spread) magnified by 1/spread in both layers
    err = (out.double() - ref_out).abs().max().item()
    assert err <= 1e-2 * ref_out.abs().max().item(), (err, ref_out.abs().max().item())
