"""The layer-1 backward kernel recomputes conv1's output y1 from the image and conv1's weights instead of loading a copy the forward
kernel stored.  Both accumulate every pixel in the same order (conv1_pixels in fused_convnet.cu), so the recompute is y1 bit for
bit, and so is everything computed from it: the kernel given the stored y1 is the reference, and every comparison is exact."""
import pytest
import torch

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda", 0)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _forward(B, bias, seed):
    """Random layer parameters and images through convnet_fwd, which keeps y1 by default."""
    g = torch.Generator(device=dev()).manual_seed(seed)
    r = lambda *s: torch.randn(*s, device=dev(), generator=g)   # noqa: E731
    x = torch.rand(B, 1, 28, 28, device=dev(), generator=g)
    w1, b1 = r(16, 1, 5, 5) * 0.2, (r(16) * 0.1 if bias else None)
    g1, be1 = torch.rand(16, device=dev(), generator=g) + 0.5, r(16) * 0.1
    w2, b2, g2, be2 = r(32, 16, 5, 5) * 0.05, r(32) * 0.1, torch.rand(32, device=dev(), generator=g) + 0.5, r(32) * 0.1
    fcw, fcb = r(10, 1568) * 0.02, r(10) * 0.1
    p1, y1, saved1, *_ = _C.convnet_fwd(x, w1, b1, g1, be1, None, None, None, 0.1, 1e-5, w2, b2, g2, be2, None, None, None, 0.1, 1e-5,
                                        fcw, fcb)
    dp = r(B, 18, 18, 16)
    frames = (r(B, 18, 18, 32), p1)   # conv2's weight-gradient partials from given frames: no layer-2 backward needed
    return dict(x=x, w1=w1, b1=b1, g1=g1, be1=be1, y1=y1, saved1=saved1, dp=dp, frames=frames, dysum2=r(B, 32), g=g)


def _l1_bwd(d, y, init, accumulate, **kw):
    out = [t.clone() for t in init]   # dgamma, dbeta, dw, db, dw2, db2
    dg, dbe, dw, db, dw2, db2 = out
    _C.convnet_l1_bwd_wgrad(d["dp"], y, d["x"], d["saved1"], d["g1"], d["be1"], dg, dbe, dw, db, *d["frames"], d["dysum2"], dw2, db2,
                            accumulate=accumulate, **kw)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("B", [1, 7, 100, "sms"])
def test_recompute_matches_stored_y1_bit_for_bit(B, bias, accumulate):
    B = sms() if B == "sms" else B
    d = _forward(B, bias, seed=B + 2 * bias)
    g = d["g"]
    shapes = [(16,), (16,), (16, 1, 5, 5), (16,), (32, 16, 5, 5), (32,)]
    # accumulate mode adds to what the buffers hold (earlier micro-batches); otherwise they are overwritten
    init = [torch.randn(*s, device=dev(), generator=g) if accumulate else torch.full(s, float("nan"), device=dev()) for s in shapes]
    stored = _l1_bwd(d, d["y1"], init, accumulate)
    recomputed = _l1_bwd(d, None, init, accumulate, w1=d["w1"], b1=d["b1"])
    for name, a, b in zip(["dgamma", "dbeta", "dw", "db", "dw2", "db2"], stored, recomputed):
        assert torch.equal(a, b), (name, (a - b).abs().max().item())


def test_recompute_needs_conv1_weights():
    d = _forward(3, True, seed=0)
    init = [torch.zeros(*s, device=dev()) for s in [(16,), (16,), (16, 1, 5, 5), (16,), (32, 16, 5, 5), (32,)]]
    with pytest.raises(RuntimeError, match="w1"):
        _l1_bwd(d, None, init, False)
    with pytest.raises(RuntimeError, match="w1"):
        _l1_bwd(d, None, init, False, b1=d["b1"])


class _StoredY1:
    """The extension module with the forward kernel storing y1 and the layer-1 backward kernel given it: the model's path before the
    recompute, for the training step to be compared against."""

    def __init__(self, C):
        self._C, self.y1 = C, None

    def __getattr__(self, name):
        return getattr(self._C, name)

    def convnet_fwd(self, *args, **kwargs):
        kwargs["keep_y1"] = True
        out = self._C.convnet_fwd(*args, **kwargs)
        self.y1 = out[1]
        return out

    def convnet_l1_bwd_wgrad(self, dp, y, *args, w1=None, b1=None, **kwargs):
        assert y is None and w1 is not None
        return self._C.convnet_l1_bwd_wgrad(dp, self.y1, *args, **kwargs)


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_riding_update_is_the_same_bits_with_stored_y1(opt, monkeypatch):
    """Three training steps with the optimizer riding on the layer-1 backward kernel, once recomputing y1 and once with y1 stored by
    the forward kernel: the same parameters, optimizer state and BatchNorm buffers, bit for bit."""
    from pytorch_distributed_train_b200.ops import functional as OF

    torch.manual_seed(3)
    a = pdt.models.ConvNet(fused=True).to(dev())
    b = pdt.models.ConvNet(fused=True).to(dev())
    b.load_state_dict(a.state_dict())
    make = (lambda m: pdt.optim.SGD(m.parameters(), 1e-2, momentum=0.9, weight_decay=1e-4)) if opt == "sgd" else \
        (lambda m: pdt.optim.Adam(m.parameters(), 1e-3, weight_decay=1e-2))
    crit = pdt.nn.CrossEntropyLoss()
    for model, stored in ((a, False), (b, True)):
        o = make(model)
        with monkeypatch.context() as mp:
            if stored:
                mp.setattr(OF, "_C", _StoredY1(_C))
            assert o.ride_on_backward(model)
            try:
                for s in range(3):
                    x = torch.rand(100, 1, 28, 28, device=dev(), generator=torch.Generator(device=dev()).manual_seed(s))
                    t = torch.randint(0, 10, (100,), device=dev(), generator=torch.Generator(device=dev()).manual_seed(50 + s))
                    o.zero_grad()
                    loss = crit(model(x), t)
                    with OF.sgd_rider_enabled():
                        loss.backward()
                    assert o._rode
                    o.step()
            finally:
                o.stop_riding()
        model.opt = o
    torch.cuda.synchronize()
    for (n, p), q in zip(a.named_parameters(), b.parameters()):
        assert torch.equal(p, q), (n, (p - q).abs().max().item())
        assert torch.equal(p.grad, q.grad), n
        for k, v in a.opt.state[p].items():
            assert torch.equal(v, b.opt.state[q][k]), (n, k)
    for (n, u), v in zip(a.named_buffers(), b.buffers()):
        assert torch.equal(u, v), n


def test_inplace_change_of_conv1_weight_before_backward_raises():
    """conv1's weight and bias are saved for the recompute: changing them in place between forward and backward is refused by
    autograd's version check, not recomputed from the new values."""
    torch.manual_seed(0)
    model = pdt.models.ConvNet(fused=True).to(dev())
    x = torch.rand(8, 1, 28, 28, device=dev())
    t = torch.randint(0, 10, (8,), device=dev())
    loss = pdt.nn.CrossEntropyLoss()(model(x), t)
    w1 = model.layer1[0].weight
    with torch.no_grad():
        w1.mul_(0.5)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        loss.backward()
