"""conv2's weight gradient split over the two backward kernels: the layer-2 backward kernel computes the per-image partials
(given conv2's input frame p1), the layer-1 backward kernel folds them.  Checked against the stand-alone form of the layer-1
binding fed the dy frame the layer-2 kernel writes without p1 (bit for bit), against float64, and in a graphed training step against
the same step without the optimizer riding on the backward kernels."""
import pytest
import torch

import pytorch_distributed_train_b200 as pdt
from pytorch_distributed_train_b200 import _C

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda", 0)


def tf32_rna(t):
    """cvt.rna.tf32.f32: round to 10 mantissa bits, ties away from zero (finite values)."""
    bits = t.contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


def _layer_inputs(B, ncls, seed):
    g = torch.Generator(device=dev()).manual_seed(seed)
    r = lambda *s: torch.randn(*s, device=dev(), generator=g)   # noqa: E731
    x1 = torch.rand(B, 1, 28, 28, device=dev(), generator=g)
    w1, b1, g1, be1 = r(16, 1, 5, 5) * 0.2, r(16) * 0.1, torch.rand(16, device=dev(), generator=g) + 0.5, r(16) * 0.1
    w2, b2, g2, be2 = r(32, 16, 5, 5) * 0.05, r(32) * 0.1, torch.rand(32, device=dev(), generator=g) + 0.5, r(32) * 0.1
    fcw, fcb = r(ncls, 1568) * 0.02, r(ncls) * 0.1
    p1, y1, sv1, out, y2, sv2, *_ = _C.convnet_fwd(x1, w1, b1, g1, be1, None, None, None, 0.1, 1e-5, w2, b2, g2, be2, None, None, None,
                                                   0.1, 1e-5, fcw, fcb)
    dlogits = r(B, ncls) / B
    dp1 = torch.zeros(B, 18, 18, 16, device=dev())
    dp1[:, 2:16, 2:16, :] = r(B, 14, 14, 16)
    return dict(x1=x1, g1=g1, be1=be1, p1=p1, y1=y1, sv1=sv1, w2=w2, g2=g2, be2=be2, fcw=fcw, out=out, y2=y2, sv2=sv2,
                dlogits=dlogits, dp1=dp1)


def _layer2_bwd(d, p1=None):
    """(dy or None, dx, dysum, [dg, dbe, dfcw, dfcb]) of the layer-2 backward kernel."""
    grads = [torch.full((32,), 7.0, device=dev()), torch.full((32,), 7.0, device=dev()), torch.full_like(d["fcw"], 7.0),
             torch.full((d["fcw"].shape[0],), 7.0, device=dev())]
    res = _C.convnet_l2_bwd_fc(d["dlogits"], d["fcw"], d["out"], grads[2], grads[3], d["y2"], d["sv2"], d["g2"], d["be2"], d["w2"],
                               grads[0], grads[1], p1=p1)
    return (*res, grads)


def _l1_outputs():
    return [torch.full((16,), 7.0, device=dev()), torch.full((16,), 7.0, device=dev()), torch.full((16, 1, 5, 5), 7.0, device=dev()),
            torch.full((16,), 7.0, device=dev())]


@pytest.mark.parametrize("ncls", [10, 16])
@pytest.mark.parametrize("B", [1, 3, 100, "sms"])
def test_layer2_partials_folded_by_layer1_match_the_standalone_path(B, ncls):
    if B == "sms":
        B = torch.cuda.get_device_properties(0).multi_processor_count
    d = _layer_inputs(B, ncls, seed=B * 31 + ncls + 7)
    dy, dx, dysum, grads = _layer2_bwd(d)
    none, dx_r, dysum_r, grads_r = _layer2_bwd(d, p1=d["p1"])
    assert none is None, "with p1 the layer-2 kernel does not write the dy frame"
    # everything else the layer-2 kernel produces is unchanged
    assert torch.equal(dx_r[:, 2:16, 2:16, :], dx[:, 2:16, 2:16, :]) and torch.equal(dysum_r, dysum)
    for got, want in zip(grads_r, grads):
        assert torch.equal(got, want)

    common = (d["dp1"], d["y1"], d["x1"], d["sv1"], d["g1"], d["be1"])
    ref, chain = _l1_outputs(), _l1_outputs()
    dw_ref, db_ref = torch.full((32, 16, 5, 5), 7.0, device=dev()), torch.full((32,), 7.0, device=dev())
    dw_c, db_c = torch.full_like(dw_ref, 7.0), torch.full_like(db_ref, 7.0)
    # the stand-alone form (per-image kernel on the given frames, then layer 1), fed the dy frame of the form without p1
    _C.convnet_l1_bwd_wgrad(*common, *ref, dy, d["p1"], dysum, dw_ref, db_ref)
    # the chain: layer 2 (p1 given) left the partials, layer 1 folds them.  Layer 2 runs again so that its partials are the pending ones.
    _layer2_bwd(d, p1=d["p1"])
    _C.convnet_l1_bwd_wgrad(*common, *chain, None, None, dysum_r, dw_c, db_c)
    assert torch.equal(dw_c, dw_ref), (dw_c - dw_ref).abs().max().item()
    assert torch.equal(db_c, db_ref)
    for got, want in zip(chain, ref):
        assert torch.equal(got, want)

    # float64 conv2d_weight on the TF32-rounded (rna) operands; the kernel accumulates in fp32 (256 positions per image, then B rows)
    xi = tf32_rna(d["p1"][:, 2:16, 2:16, :]).permute(0, 3, 1, 2).double()
    dyi = tf32_rna(dy[:, 2:16, 2:16, :]).permute(0, 3, 1, 2).double()
    want = torch.nn.grad.conv2d_weight(xi, (32, 16, 5, 5), dyi, padding=2)
    scale = torch.nn.grad.conv2d_weight(xi.abs(), (32, 16, 5, 5), dyi.abs(), padding=2)
    err = (dw_c.double() - want).abs()
    assert bool((err <= (256 + B) * 2.0 ** -23 * scale + 1e-30).all()), err.max().item()
    want_b = dy.double()[:, 2:16, 2:16, :].sum((0, 1, 2))
    assert torch.allclose(db_c.double(), want_b, atol=1e-5 * dy.abs().sum().item() / 32 + 1e-7, rtol=0)


def test_layer1_without_frames_needs_pending_partials():
    d = _layer_inputs(3, 10, seed=5)
    common = (d["dp1"], d["y1"], d["x1"], d["sv1"], d["g1"], d["be1"])
    dw2, db2 = torch.empty(32, 16, 5, 5, device=dev()), torch.empty(32, device=dev())
    _layer2_bwd(d, p1=d["p1"])
    _C.convnet_l1_bwd_wgrad(*common, *_l1_outputs(), None, None, torch.zeros(3, 32, device=dev()), dw2, db2)
    with pytest.raises(RuntimeError, match="none are pending"):   # consumed by the call above
        _C.convnet_l1_bwd_wgrad(*common, *_l1_outputs(), None, None, torch.zeros(3, 32, device=dev()), dw2, db2)


def _graphed_run(opt_kind, clip, riding, monkeypatch):
    from mp_helpers import free_port

    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    monkeypatch.setenv("PDT_SGD_RIDER", "1" if riding else "0")
    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        torch.manual_seed(0)
        model = pdt.models.ConvNet().to(dev())
        if opt_kind == "sgd":
            opt = pdt.optim.SGD(model.parameters(), 0.05, momentum=0.9, weight_decay=1e-3)
        else:
            opt = pdt.optim.AdamW(model.parameters(), 1e-3, weight_decay=1e-2)
        ddp = pdt.DistributedDataParallel(model, device_ids=[0])
        crit = pdt.nn.CrossEntropyLoss()
        g = torch.Generator(device=dev()).manual_seed(9)
        xs = torch.rand(4, 100, 1, 28, 28, device=dev(), generator=g)
        ts = torch.randint(0, 10, (4, 100), device=dev(), generator=g)
        step = GraphedTrainStep(ddp, crit, opt, (xs[0], ts[0]), warmup=3, max_grad_norm=0.5 if clip else None)
        kernels = step.kernels_per_replay
        norms = []
        for i in range(4):
            step(xs[i % 4], ts[i % 4], inputs_ready=True)
            if clip:
                norms.append(step.grad_norm.item())
        torch.cuda.synchronize()
        return kernels, {n: p.detach().clone() for n, p in model.named_parameters()}, norms
    finally:
        pdt.destroy_process_group()


@pytest.mark.parametrize("opt_kind,clip", [("sgd", False), ("adamw", False), ("sgd", True), ("adamw", True)])
def test_graphed_step_matches_the_step_without_the_rider(opt_kind, clip, monkeypatch):
    k_ride, ride, n_ride = _graphed_run(opt_kind, clip, True, monkeypatch)
    k_plain, plain, n_plain = _graphed_run(opt_kind, clip, False, monkeypatch)
    assert k_ride == 3 and k_plain > k_ride, (k_ride, k_plain)
    # the conv biases feed a BatchNorm: their gradient is rounding noise, which Adam scales up to full-size steps
    skip = ("layer1.0.bias", "layer2.0.bias") if opt_kind == "adamw" else ()
    keep = [n for n in ride if n not in skip]
    if not clip:
        # the same gradients and the same update arithmetic: only the launch that applies it differs
        for n in keep:
            assert torch.allclose(ride[n], plain[n], atol=1e-6, rtol=1e-5), (n, (ride[n] - plain[n]).abs().max().item())
        return
    # the rider and the stand-alone clip kernel fold the norm in different orders: the coefficients differ in the last bits, and
    # through the BatchNorms the steps that follow amplify that (the tolerances of test_clip_grad.py's graphed-step tests)
    assert abs(n_ride[0] - n_plain[0]) <= 1e-4 * n_plain[0], (n_ride, n_plain)
    assert all(abs(a - b) <= 2e-2 * b for a, b in zip(n_ride, n_plain)), (n_ride, n_plain)
    flat_r = torch.cat([ride[n].reshape(-1) for n in keep])
    flat_p = torch.cat([plain[n].reshape(-1) for n in keep])
    assert (flat_r - flat_p).abs().max().item() <= 2e-2 * flat_p.abs().max().item()
