"""The BatchNorm statistics of the cooperative forward kernel (convnet_fwd) against float64 statistics of its own conv outputs.

Layer 1's sums are reduced from the two pixels each thread owns, layer 2's straight from the wgmma accumulators of conv2's
epilogue; both are folded over the CTAs in a fixed order.  Checked here: the saved (mean, invstd) pairs and the running-statistics
updates of both layers against float64 over the kernel's y1 / y2, and that two identical calls agree bit for bit."""
import pytest
import torch

from pytorch_distributed_train_b200 import _C

pytestmark = pytest.mark.gpu

EPS, MOM = 1e-5, 0.1


def dev():
    return torch.device("cuda", 0)


def _batches():
    return [1, 3, 100, "sms"]   # "sms": one image per SM, i.e. one CTA on every SM of the device


def _inputs(B, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(dev())
    x = torch.rand(B, 1, 28, 28, generator=g).to(dev())
    w1, b1 = r(16, 1, 5, 5, scale=0.2), r(16, scale=0.1)
    g1, be1 = 1.0 + r(16, scale=0.1), r(16, scale=0.1)
    w2, b2 = r(32, 16, 5, 5, scale=0.05), r(32, scale=0.1)
    g2, be2 = 1.0 + r(32, scale=0.1), r(32, scale=0.1)
    fcw, fcb = r(10, 1568, scale=0.02), r(10, scale=0.1)
    t = torch.randint(0, 10, (B,), generator=g).to(dev())
    return x, w1, b1, g1, be1, w2, b2, g2, be2, fcw, fcb, t


def _run(args):
    x, w1, b1, g1, be1, w2, b2, g2, be2, fcw, fcb, t = args
    rm1, rv1, nbt1 = torch.full((16,), 0.25, device=dev()), torch.full((16,), 2.0, device=dev()), torch.zeros((), dtype=torch.long, device=dev())
    rm2, rv2, nbt2 = torch.full((32,), -0.5, device=dev()), torch.full((32,), 3.0, device=dev()), torch.zeros((), dtype=torch.long, device=dev())
    outs = _C.convnet_fwd(x, w1, b1, g1, be1, rm1, rv1, nbt1, MOM, EPS, w2, b2, g2, be2, rm2, rv2, nbt2, MOM, EPS, fcw, fcb, t)
    torch.cuda.synchronize()
    return outs, (rm1, rv1, nbt1, rm2, rv2, nbt2)


def _check_layer(y, saved, rm, rv, rm0, rv0, C, what):
    v = y.double().reshape(-1, C)   # NHWC: channels innermost
    cnt = v.shape[0]
    mean, var = v.mean(0), v.var(0, unbiased=False)
    spread = var.sqrt()
    k_mean, k_invstd = saved[:C].double(), saved[C:2 * C].double()
    err = ((k_mean - mean).abs() / spread).max().item()
    assert err < 1e-5, (what, "mean", err)
    k_var = 1.0 / k_invstd ** 2 - EPS   # the variance the kernel normalised with
    err = ((k_var - var).abs() / var).max().item()
    assert err < 2e-5, (what, "var", err)
    unbiased = var * cnt / max(cnt - 1, 1)
    err = ((rm.double() - ((1 - MOM) * rm0 + MOM * mean)).abs() / spread).max().item()
    assert err < 1e-5, (what, "running mean", err)
    ref_rv = (1 - MOM) * rv0 + MOM * unbiased
    err = ((rv.double() - ref_rv).abs() / ref_rv).max().item()
    assert err < 2e-5, (what, "running var", err)


@pytest.mark.parametrize("B", _batches())
def test_forward_statistics_match_float64_of_its_own_outputs(B):
    if B == "sms":
        B = torch.cuda.get_device_properties(0).multi_processor_count
    (p1, y1, saved1, out, y2, saved2, *_), (rm1, rv1, nbt1, rm2, rv2, nbt2) = _run(_inputs(B, 11 + B))
    _check_layer(y1, saved1, rm1, rv1, 0.25, 2.0, 16, "layer 1")
    _check_layer(y2, saved2, rm2, rv2, -0.5, 3.0, 32, "layer 2")
    assert nbt1.item() == 1 and nbt2.item() == 1


@pytest.mark.parametrize("B", _batches())
def test_forward_is_bitwise_deterministic(B):
    if B == "sms":
        B = torch.cuda.get_device_properties(0).multi_processor_count
    args = _inputs(B, 5)
    first, state_a = _run(args)
    second, state_b = _run(args)
    names = ["p1", "y1", "saved1", "out", "y2", "saved2", "logits", "loss", "dlogits", "loss_parts"]
    for name, a, b in zip(names, first, second):
        assert torch.equal(a, b), name
    for a, b in zip(state_a, state_b):
        assert torch.equal(a, b)
