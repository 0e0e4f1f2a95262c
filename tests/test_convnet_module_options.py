"""The ConvNet's layer options against float64.

Options the native kernels implement (per-layer BatchNorm eps and momentum, missing biases, an in-place ReLU, ``momentum=None``,
``affine=False``, ``track_running_stats=False``) are trained for three passes on the fused route (B ≤ SM count) and the per-op route
(B = SM count + 1), then evaluated.  Configurations the kernels do not compute (other padding modes, dilation, stride,
``padding="same"``, swapped activation, pool or norm layers, an added module, module hooks, weight norm) must run torch's layers and
give the same model as ``fused=False``.  The CPU tests check the predicate that tells the two apart, and ``conv_bn_relu_pool``'s
refusals.  Tolerance policy: TF32 level where conv2 runs on the tensor cores, fp32 level elsewhere."""
import math
import warnings

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import ops
from pytorch_distributed_train_b200.models.convnet import _native_layers


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


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- cases: each changes a fresh ConvNet in place; a hook case returns the list its hook appends to ------------------------------
def _bn_options(net):
    net.layer1[1].eps, net.layer1[1].momentum = 1e-3, 0.01
    net.layer2[1].eps, net.layer2[1].momentum = 0.25, 0.7


def _no_bias(*names):
    def case(net):
        mods = {"conv1": net.layer1[0], "conv2": net.layer2[0], "fc": net.fc}
        for n in names:
            mods[n].bias = None
    return case


def _relu_inplace(net):
    net.layer1[2], net.layer2[2] = nn.ReLU(inplace=True), nn.ReLU(inplace=True)


def _momentum_none(net):
    net.layer1[1].momentum = net.layer2[1].momentum = None


def _batchnorms(**kw):
    def case(net):
        net.layer1[1], net.layer2[1] = nn.BatchNorm2d(16, **kw), nn.BatchNorm2d(32, **kw)
    return case


# fused route at B ≤ SM count?
NATIVE = {
    "bn_options": (_bn_options, True),
    "no_conv1_bias": (_no_bias("conv1"), True),
    "no_conv2_bias": (_no_bias("conv2"), True),
    "no_fc_bias": (_no_bias("fc"), True),
    "no_biases": (_no_bias("conv1", "conv2", "fc"), True),
    "relu_inplace": (_relu_inplace, True),
    "momentum_none": (_momentum_none, False),
    "affine_false": (_batchnorms(affine=False), False),
    "no_running_stats": (_batchnorms(track_running_stats=False), False),
}


def _conv(layer, **kw):
    def case(net):
        seq = getattr(net, layer)
        seq[0] = nn.Conv2d(seq[0].in_channels, seq[0].out_channels, 5, **{"padding": 2, **kw})
    return case


def _both_convs(**kw):
    def case(net):
        _conv("layer1", **kw)(net)
        _conv("layer2", **kw)(net)
    return case


def _stride2_conv1(net):
    net.layer1[0].stride = (2, 2)      # 28 → 14 → pool 7 → 7 → pool 3
    net.fc = nn.Linear(32 * 3 * 3, 10)


def _swap(index, make):
    def case(net):
        net.layer1[index], net.layer2[index] = make(), make()
    return case


def _dropout(net):
    net.layer1.append(nn.Dropout(p=0.0))


def _pre_hook_layer2(net):
    calls = []

    def hook(module, args):
        calls.append(1)
        return (args[0] * 0.5,)
    net.layer2.register_forward_pre_hook(hook)
    return calls


def _hook_conv1(net):
    calls = []

    def hook(module, args, out):
        calls.append(1)
        return out + 1
    net.layer1[0].register_forward_hook(hook)
    return calls


def _weight_norm_conv2(net):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)   # torch.nn.utils.weight_norm is deprecated in favour of parametrizations
        torch.nn.utils.weight_norm(net.layer2[0])


def _group_norm(net):
    net.layer1[1] = nn.GroupNorm(4, 16)


NOT_NATIVE = {
    "conv1_reflect": _conv("layer1", padding_mode="reflect"),
    "conv1_circular": _conv("layer1", padding_mode="circular"),
    "conv2_reflect": _conv("layer2", padding_mode="reflect"),
    "conv2_circular": _conv("layer2", padding_mode="circular"),
    "dilation2": _both_convs(dilation=2, padding=4),
    "stride2_conv1": _stride2_conv1,
    "padding_same": _both_convs(padding="same"),
    "leaky_relu": _swap(2, lambda: nn.LeakyReLU(0.1)),
    "avg_pool": _swap(3, lambda: nn.AvgPool2d(2)),
    "max_pool_3_2_1": _swap(3, lambda: nn.MaxPool2d(kernel_size=3, stride=2, padding=1)),
    "dropout_appended": _dropout,
    "pre_hook_layer2": _pre_hook_layer2,
    "hook_conv1": _hook_conv1,
    "weight_norm_conv2": _weight_norm_conv2,
    "group_norm": _group_norm,
}


# ---- the float64 twin --------------------------------------------------------------------------------------------------------
def _perturb(net):
    """Normalisation affines away from (1, 0) and a classifier bias that moves the loss: a kernel that dropped one would show."""
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, (nn.BatchNorm2d, nn.GroupNorm)) and m.weight is not None:
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0.0, 0.2)
        if net.fc.bias is not None:
            net.fc.bias.normal_(0.0, 0.5)


def _models(case):
    """(model on the default route, its float64 fused=False twin, the hook calls of each or None)."""
    net = pdt.models.ConvNet()
    calls = case(net)
    _perturb(net)
    net = net.to(dev())
    ref = pdt.models.ConvNet(fused=False)
    ref_calls = case(ref)
    ref.load_state_dict(net.state_dict())   # not copy.deepcopy: a weight-normed conv's weight is not a graph leaf
    return net, ref.to(dev()).double(), calls, ref_calls


def _batch(B, gen):
    return torch.rand(B, 1, 28, 28, device=dev(), generator=gen), torch.randint(0, 10, (B,), device=dev(), generator=gen)


def _assert_matches_float64(net, ref, loss, ref_loss, rel=3e-2):
    """test_kernel_edges.py's bounds (``rel``: the gradients' TF32 share of their norm)."""
    if math.isnan(ref_loss.item()):
        assert math.isnan(loss.item()), loss.item()
    else:
        # conv2 runs in TF32 (10-bit mantissa) forward and in dgrad: ~1e-3 relative per product
        assert abs(loss.item() - ref_loss.item()) < 2e-3, (loss.item(), ref_loss.item())
    for (n1, p1), (n2, p2) in zip(net.named_parameters(), ref.named_parameters(), strict=True):
        assert n1 == n2
        # TF32 as above, measured over the whole tensor; conv biases in front of a BatchNorm have a true gradient of zero (noise level)
        err, norm = (p1.grad.double() - p2.grad).norm().item(), p2.grad.norm().item()
        assert err <= rel * norm + 1e-4 * p2.numel() ** 0.5, (n1, err, norm)


def _assert_buffers_match(net, ref, passes):
    for (n1, b1), (n2, b2) in zip(net.named_buffers(), ref.named_buffers(), strict=True):
        assert n1 == n2
        if n1.endswith("num_batches_tracked"):
            assert int(b1) == int(b2) == passes, (n1, int(b1), int(b2))
        else:
            # batch statistics of the TF32 conv2 output
            assert torch.allclose(b1.double(), b2, atol=2e-3, rtol=1e-3), (n1, (b1.double() - b2).abs().max().item())


def _assert_logits_match(out, ref_out):
    # TF32 as for the gradients, over the whole [B, 10] tensor
    err, norm = (out.double() - ref_out).norm().item(), ref_out.norm().item()
    assert err <= 3e-2 * norm + 1e-4 * ref_out.numel() ** 0.5, (err, norm)


def _train_and_eval(net, ref, B, passes=3):
    """`passes` forward+backward passes on the same weights (no update: the BatchNorm buffers compound), then eval logits."""
    gen = torch.Generator(device=dev()).manual_seed(B)
    crit = pdt.nn.CrossEntropyLoss()
    for _ in range(passes):
        x, t = _batch(B, gen)
        net.zero_grad()
        ref.zero_grad()
        loss = crit(net(x), t)
        loss.backward()
        ref_loss = F.cross_entropy(ref(x.double()), t)
        ref_loss.backward()
    torch.cuda.synchronize()
    # one image: BatchNorm's backward takes out its mean and x̂-projection over that image alone, and TF32 rounding of conv2 (forward
    # masks, data gradient) is left at up to ~10 % of the BatchNorm and layer-1 gradients.  Measured on an H100 against float64 on
    # this file's B = 1 data: torch's own TF32 layers (cuDNN) up to 9.5 %, the native kernels up to 13 %.
    _assert_matches_float64(net, ref, loss, ref_loss, rel=2.5e-1 if B == 1 else 3e-2)
    _assert_buffers_match(net, ref, passes)
    _assert_eval_matches(net, ref, B, gen)


def _assert_eval_matches(net, ref, B, gen):
    net.eval()
    ref.eval()
    x, _ = _batch(B, gen)
    with torch.no_grad():
        out = net(x)
        ref_out = ref(x.double())
    assert out.shape == ref_out.shape
    _assert_logits_match(out, ref_out)


# ---- A1. options the native kernels implement ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3, 100, "sms", "sms+1"])
@pytest.mark.parametrize("name", list(NATIVE))
def test_native_options_match_float64(name, B):
    case, fused = NATIVE[name]
    B = {"sms": sms(), "sms+1": sms() + 1}.get(B, B)
    net, ref, _, _ = _models(case)
    x = torch.rand(B, 1, 28, 28, device=dev())
    assert _native_layers(net)
    # the route: without this, a case meant for the fused kernels could test the per-op kernels twice
    assert ops.functional.fused_convnet_ok(x, net) == (fused and B <= sms()), (name, B)
    _train_and_eval(net, ref, B)


# ---- A2. per-layer eps and momentum baked into a captured step -----------------------------------------------------------------
@pytest.mark.gpu
def test_graphed_step_with_per_layer_batchnorm_options_matches_eager_loop():
    from mp_helpers import free_port

    from pytorch_distributed_train_b200.engine import GraphedTrainStep
    from pytorch_distributed_train_b200.ops import functional as OF

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        model = pdt.models.ConvNet()
        _bn_options(model)
        model = model.to(dev())
        eager = pdt.models.ConvNet()
        _bn_options(eager)
        eager = eager.to(dev())
        eager.load_state_dict(model.state_dict())
        hyper = dict(lr=0.05, momentum=0.9, weight_decay=1e-3)
        opt = pdt.optim.SGD(model.parameters(), **hyper)
        eopt = pdt.optim.SGD(eager.parameters(), **hyper)
        crit = pdt.nn.CrossEntropyLoss()
        g = torch.Generator(device=dev()).manual_seed(9)
        xs = torch.rand(4, 100, 1, 28, 28, device=dev(), generator=g)
        ts = torch.randint(0, 10, (4, 100), device=dev(), generator=g)
        step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), crit, opt, (xs[0], ts[0]), warmup=3)
        # the engine's eager warm-up steps trained the model on the example batch (capturing runs nothing): the eager loop takes them too
        warm = int(model.layer1[1].num_batches_tracked)
        assert warm >= 3

        def eager_step(x, t):
            eopt.zero_grad()
            with OF.upcoming_targets(t):   # the forward kernel's cross-entropy, as in the captured step
                loss = crit(eager(x), t)
            loss.backward()
            eopt.step()

        for _ in range(warm):
            eager_step(xs[0], ts[0])
        for i in range(5):
            step(xs[i % 4], ts[i % 4], inputs_ready=True)
            eager_step(xs[i % 4], ts[i % 4])
        torch.cuda.synchronize()
        for (n, p), q in zip(model.named_parameters(), eager.parameters(), strict=True):
            assert torch.allclose(p, q, atol=1e-6, rtol=1e-5), (n, (p - q).abs().max().item())
        for (n, b), c in zip(model.named_buffers(), eager.buffers(), strict=True):
            if n.endswith("num_batches_tracked"):
                assert int(b) == int(c) == warm + 5, n
            else:
                assert torch.allclose(b, c, atol=1e-6, rtol=1e-5), (n, (b - c).abs().max().item())
    finally:
        pdt.destroy_process_group()


# ---- A3. configurations the kernels do not compute -----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["train_100", "train_sms+1", "eval_100"])
@pytest.mark.parametrize("name", list(NOT_NATIVE))
def test_other_layer_configurations_match_float64(name, mode):
    net, ref, calls, ref_calls = _models(NOT_NATIVE[name])
    if mode == "eval_100":
        _assert_eval_matches(net, ref, 100, torch.Generator(device=dev()).manual_seed(5))
        forwards = 1
    else:
        _train_and_eval(net, ref, 100 if mode == "train_100" else sms() + 1)
        forwards = 4
    if calls is not None:
        assert len(calls) == len(ref_calls) == forwards, (len(calls), len(ref_calls), forwards)


# ---- C. the predicate and conv_bn_relu_pool's refusals, on CPU modules ----------------------------------------------------------
def _cpu_net(case=None):
    net = pdt.models.ConvNet()
    if case is not None:
        case(net)
    return net


def test_default_convnet_is_native():
    assert _native_layers(pdt.models.ConvNet())
    assert _native_layers(pdt.models.ConvNet(num_classes=16))


@pytest.mark.parametrize("name", list(NATIVE))
def test_native_options_keep_the_native_layers(name):
    assert _native_layers(_cpu_net(NATIVE[name][0]))


def test_padding_same_on_a_5x5_kernel_is_native():
    # "same" is pad 2 for a 5×5 kernel: both routes compute it
    net = _cpu_net(NOT_NATIVE["padding_same"])
    assert net.layer1[0].padding == net.layer2[0].padding == "same"
    assert _native_layers(net)


def test_pdt_syncbatchnorm_is_native_torch_syncbatchnorm_is_not():
    assert _native_layers(pdt.SyncBatchNorm.convert_sync_batchnorm(_cpu_net()))
    net = _cpu_net()
    net.layer1[1] = nn.SyncBatchNorm(16)
    assert not _native_layers(net)


@pytest.mark.parametrize("name", [n for n in NOT_NATIVE if n != "padding_same"])   # "same" is pad 2 here: native
def test_other_layer_configurations_are_not_native(name):
    assert not _native_layers(_cpu_net(NOT_NATIVE[name]))


@pytest.mark.parametrize("what", ["subclass_bn", "subclass_conv", "extra_layer_module", "backward_hook", "fc_swapped"])
def test_near_misses_are_not_native(what):
    net = _cpu_net()
    if what == "subclass_bn":
        class MyBN(nn.BatchNorm2d):
            pass
        net.layer2[1] = MyBN(32)
    elif what == "subclass_conv":
        class MyConv(nn.Conv2d):
            pass
        net.layer1[0] = MyConv(1, 16, 5, padding=2)
    elif what == "extra_layer_module":
        net.layer2.append(nn.Identity())
    elif what == "backward_hook":
        net.fc.register_full_backward_hook(lambda m, gi, go: None)
    else:
        net.fc = nn.Sequential(nn.Linear(1568, 10))
    assert not _native_layers(net)


def test_hooks_on_the_convnet_itself_keep_it_native_global_hooks_do_not():
    net = _cpu_net()
    h = net.register_forward_hook(lambda m, a, out: out)
    try:
        assert _native_layers(net)   # ConvNet.__call__ runs them whatever route forward takes
    finally:
        h.remove()
    for register in (nn.modules.module.register_module_forward_hook, nn.modules.module.register_module_forward_pre_hook):
        h = register(lambda *args: None)
        try:
            assert not _native_layers(net)
        finally:
            h.remove()
    assert _native_layers(net)


@pytest.mark.parametrize("kw", [dict(dilation=2, padding=4), dict(padding_mode="reflect"), dict(padding_mode="circular"),
                                dict(stride=2), dict(padding=1)])
def test_conv_bn_relu_pool_refuses_convolutions_it_does_not_compute(kw):
    conv = nn.Conv2d(1, 16, 5, **{"padding": 2, **kw})
    with pytest.raises(ValueError, match="conv_bn_relu_pool"):
        ops.conv_bn_relu_pool(torch.rand(2, 1, 28, 28), conv, nn.BatchNorm2d(16))
