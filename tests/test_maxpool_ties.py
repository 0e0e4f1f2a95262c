"""Max-pool gradient routing against float64 where pooling windows tie.

No backward kernel of the ConvNet stores max-pool indices: each recomputes the arg-max of every 2×2 window from the saved conv
output and the BatchNorm statistics, routes the pooled gradient to the *first* maximum in row-major order (torch's max_pool2d) and
masks it with the ReLU (torch passes gradient only where the ReLU output is > 0).  Three implementations do this: ``route()`` of the
per-op kernels (ops_simt.cu), the four-lane bitmask of the fused layer-1 backward and the ``z > best`` scan of the fused layer-2
backward (fused_convnet.cu).  Continuous data never ties, but MNIST does (four in five pixels are exactly 0, so conv outputs over
blank regions are equal), and so does every window of a channel whose BatchNorm weight γ is 0: there dγ = Σ dout·x̂ at the first
position, and routing anywhere else changes it by O(1).

The frames here tie by construction (``tied_frames``): every window gets one of the 15 non-empty subsets of its four slots as its
set of tied maxima, cycled over window position, channel and image so that every pattern meets every window position (image
borders, both sides of every warp boundary of the kernels' thread maps) and every channel kind (γ > 0, γ < 0, γ = 0 < β, γ = β = 0,
and β low enough that the ReLU blocks some tied maxima).  Values lie on a 1/16 grid, so ties are exact in every precision and
distinct values stay ≥ |γ|·invstd/16 apart after the BatchNorm affine; the ReLU threshold sits half a grid step from every value.

Tolerance policy: fp32 level for the per-op kernels and layer 1's BatchNorm sums, TF32 level where an operand passes through the
tensor cores (conv1's weight gradient, conv2).  A misrouted window moves an O(1) gradient (dγ of a γ = 0 channel, one element of
the dy frame, a different 5×5 image neighbourhood in dW1), far above those levels.  NaN propagation through the pool is not covered.
"""
import contextlib
import math

import pytest
import torch
import torch.nn.functional as F

import pytorch_distributed_train_b200 as pdt

GRID = 16
EPS = 1e-5
# channel kinds: the BatchNorm weight's sign, and where the ReLU threshold lies
KINDS = ("pos", "neg", "zero", "zero_zero", "relu", "neg_relu")
# the ReLU threshold in units of the designed value u (z > 0 ⇔ u > threshold): half a grid step from every grid value
THRESH_U = {"pos": -0.5 / GRID, "neg": -0.5 / GRID, "relu": 7.5 / GRID, "neg_relu": 7.5 / GRID}


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


def kinds(C):
    return [KINDS[c % len(KINDS)] for c in range(C)]


def _negated(C):
    return torch.tensor([k in ("neg", "neg_relu") for k in kinds(C)])


# ---- 1. frames with ties by construction ----------------------------------------------------------------------------------------
def tied_frames(B, H, C, seed=0):
    """Conv outputs y [B, H, H, C] (NHWC, fp32) and the tie pattern of every window [B, H/2, H/2, C] (bitmask of the tied maxima of
    slots d = 2·row + column).  Window (n, ph, pw) of channel c has pattern (ph·H/2 + pw + c + 7n) mod 15 + 1: with C ≥ 15 every
    window position meets every pattern, and every channel kind meets every pattern over the windows of one image.  The tied slots
    hold the window's top value T/16 (T = 1..16: 16 is a saturated pixel), the others a grid value below it (0 = a blank pixel).  For
    γ < 0 channels y = 1 − u: the arg-max of the BatchNorm output is then the arg-min of y, tied in the same slots."""
    g = torch.Generator().manual_seed(seed)
    PH = H // 2
    n = torch.arange(B).view(B, 1, 1, 1)
    win = torch.arange(PH * PH).view(1, PH, PH, 1)
    c = torch.arange(C).view(1, 1, 1, C)
    pat = (win + c + 7 * n) % 15 + 1
    top = torch.randint(1, GRID + 1, (B, PH, PH, C), generator=g)
    low = torch.randint(0, GRID, (B, PH, PH, C, 4), generator=g) % top[..., None]
    bits = ((pat[..., None] >> torch.arange(4)) & 1).bool()
    u = torch.where(bits, top[..., None], low).double() / GRID              # [B, ph, pw, C, slot]
    u = torch.where(_negated(C).view(1, 1, 1, C, 1), 1.0 - u, u)
    y = u.view(B, PH, PH, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(B, H, H, C)
    return y.float().contiguous(), pat


def bn_params(y, to_y=lambda t: 1.0 - t):
    """γ, β per channel kind for frames y [B, H, W, C], with the ReLU threshold half a grid step from every value: β = −γ·(y_t −
    mean)·invstd puts z = 0 at y_t = the threshold in y (to_y maps a designed value u of a γ < 0 channel to y).  Also returns the
    float64 batch mean and invstd."""
    yd = y.double()
    C = y.shape[-1]
    mean = yd.mean((0, 1, 2))
    invstd = (yd.var((0, 1, 2), unbiased=False) + EPS).rsqrt()
    gamma, beta = torch.zeros(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64)
    for ch, k in enumerate(kinds(C)):
        if k == "zero":
            beta[ch] = 0.75
        elif k != "zero_zero":
            neg = k in ("neg", "neg_relu")
            gamma[ch] = (-1.0 if neg else 1.0) * (0.5 + 0.25 * (ch % 3))
            t = to_y(THRESH_U[k]) if neg else THRESH_U[k]
            beta[ch] = -gamma[ch] * (t - mean[ch].item()) * invstd[ch].item()
    return gamma.float(), beta.float(), mean, invstd


def _windows(t):
    """[B, C, H, W] → [B, C, H/2, W/2, 4] in slot order d = 2·row + column."""
    B, C, H, W = t.shape
    return t.view(B, C, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, H // 2, W // 2, 4)


def test_tied_frames_builder():
    """The builder makes what the GPU tests rely on: every pattern at every window position and in every channel kind, tied values
    bit-equal in fp32 and ≥ 1/16 above the rest (after the fp32 BatchNorm affine: ≥ |γ|·invstd/16 apart), the ReLU threshold half a
    grid step from every value, and torch's float64 max_pool2d picking the first tied slot."""
    for B, H, C in ((4, 28, 16), (4, 14, 32), (2, 28, 16), (6, 14, 32)):
        y, pat = tied_frames(B, H, C)
        PH = H // 2
        u = _windows(y.permute(0, 3, 1, 2))                                # [B, C, ph, pw, 4]
        neg = _negated(C).view(1, C, 1, 1, 1)
        u = torch.where(neg, 1.0 - u, u)
        assert bool(((u * GRID).round() == u * GRID).all()) and u.min() >= 0 and u.max() <= 1
        assert bool((u == 0).any()) and bool((u == 1).any()), "blank and saturated pixels"
        patc = pat.permute(0, 3, 1, 2)                                     # [B, C, ph, pw]
        for p in range(1, 16):
            at = patc == p
            assert bool(at.any((0, 1)).all()), ("pattern", p, "misses a window position")
            for k in KINDS:
                chans = [ch for ch, kk in enumerate(kinds(C)) if kk == k]
                assert bool(at[:, chans].any()), ("pattern", p, "misses kind", k)
        bits = ((patc[..., None] >> torch.arange(4)) & 1).bool()
        top = u.amax(-1, keepdim=True)
        assert torch.equal(u == top, bits), "exactly the pattern's slots hold the window maximum"
        gap = torch.where(bits, torch.full_like(u, 9.0), top - u).amin(-1)
        assert gap.min().item() >= 1.0 / GRID
        # the fp32 BatchNorm affine the kernels apply (scale = γ·invstd, shift = β − mean·scale, one fma)
        gamma, beta, mean, invstd = bn_params(y)
        sv = torch.cat([mean, invstd]).float()
        scale = gamma * sv[C:]
        shift = beta - sv[:C] * scale
        z = torch.addcmul(shift.view(1, C, 1, 1).expand(B, C, H, H), y.permute(0, 3, 1, 2), scale.view(1, C, 1, 1))
        zw = _windows(z)
        zt = torch.where(bits, zw, torch.full_like(zw, -math.inf)).amax(-1, keepdim=True)
        assert bool(torch.where(bits, zw == zt, torch.ones_like(bits)).all()), "ties stay bit-equal in fp32"
        zgap = torch.where(bits, torch.full_like(zw, math.inf), zt - zw).amin(-1)
        bound = (scale.abs().double() / GRID).view(1, C, 1, 1)
        assert bool((zgap.double() >= 0.999 * bound).all()), "distinct values stay |γ|·invstd/16 apart"
        margin = zw.double().abs().amin(-1)
        nonzero = (scale != 0).view(1, C, 1, 1)
        assert bool((margin >= 0.499 * bound)[nonzero.expand_as(margin)].all()), "no value within half a step of the ReLU threshold"
        # some tied maxima pass the ReLU and some are blocked, in the ReLU channels of both signs
        for k in ("relu", "neg_relu"):
            chans = [ch for ch, kk in enumerate(kinds(C)) if kk == k]
            zmax = zt[:, chans].squeeze(-1)
            assert bool((zmax > 0).any()) and bool((zmax < 0).any()), k
        # torch's float64 BN → ReLU → max_pool2d routes to the first tied slot wherever the maximum is positive
        zd = F.batch_norm(y.permute(0, 3, 1, 2).double(), None, None, gamma.double(), beta.double(), True, 0.0, EPS)
        _, idx = F.max_pool2d(F.relu(zd), 2, 2, return_indices=True)
        first = bits.int().argmax(-1)                                      # lowest set bit: the first tied slot
        first = torch.where((gamma == 0).view(1, C, 1, 1), 0, first)       # γ = 0: all four slots tie at β
        ph, pw = torch.arange(PH).view(1, 1, PH, 1), torch.arange(PH).view(1, 1, 1, PH)
        want = (2 * ph + first // 2) * H + 2 * pw + first % 2
        live = zd.new_tensor(0).lt(_windows(zd).amax(-1))
        assert torch.equal(idx[live], want[live])
        assert bool(live.any()) and bool((~live).any())


# ---- 2. kernel-level probes ---------------------------------------------------------------------------------------------------
def _oracle(y, gamma, beta, dout):
    """float64 BN (batch statistics) → ReLU → max_pool2d of NHWC frames y, backward of dout [B, C, H/2, W/2]: pooled output,
    dy [B, C, H, W], dγ, dβ, and the gradient at the BatchNorm output gz (nonzero only where a window routed)."""
    yd = y.double().permute(0, 3, 1, 2).contiguous().requires_grad_()
    g, b = gamma.double().requires_grad_(), beta.double().requires_grad_()
    z = F.batch_norm(yd, None, None, g, b, True, 0.0, EPS)
    z.retain_grad()
    out = F.max_pool2d(F.relu(z), 2, 2)
    out.backward(dout.double())
    return out.detach(), yd.grad, g.grad, b.grad, z.grad


def _xhat(y, mean, invstd):
    return (y.double().permute(0, 3, 1, 2) - mean.view(1, -1, 1, 1)) * invstd.view(1, -1, 1, 1)


def _assert_bn_sums(dgamma, dbeta, ref_dg, ref_db, gz, xh, what):
    """fp32 sums over the windows: 1e-5 of the sum of the terms' magnitudes."""
    mag_b = gz.abs().sum((0, 2, 3))
    mag_g = (gz * xh).abs().sum((0, 2, 3))
    eb = (dbeta.double().cpu() - ref_db.cpu()).abs()
    eg = (dgamma.double().cpu() - ref_dg.cpu()).abs()
    assert bool((eb <= 1e-5 * mag_b.cpu() + 1e-6).all()), (what, "dβ", eb.max().item())
    assert bool((eg <= 1e-5 * mag_g.cpu() + 1e-6).all()), (what, "dγ", eg.max().item(), (eg - 1e-5 * mag_g.cpu()).argmax().item())


def _assert_dy(dy_nchw, ref, gamma, invstd, gmax, what):
    """dy = γ·invstd·(dz − mean(dz) − x̂·mean(dz·x̂)) in fp32: 1e-5 of γ·invstd·(max |dz| + 1) per channel (a misrouted window
    moves γ·invstd·dz between two elements; γ = 0 channels must be exactly 0)."""
    C = ref.shape[1]
    tol = (1e-5 * (gamma.double().abs() * invstd.to(gamma.device)).view(1, C, 1, 1) * (gmax + 1.0)).cpu()
    err = (dy_nchw.double().cpu() - ref.cpu()).abs()
    assert bool((err <= tol).all()), (what, "dy", err.max().item(), (err - tol).max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("out_nchw", [False, True])
@pytest.mark.parametrize("C,H", [(16, 28), (32, 14)])
def test_per_op_route_matches_float64_on_ties(C, H, out_nchw):
    """bn_relu_pool_fwd / _bwd_reduce / _bwd_apply (the per-op path: SyncBatchNorm, batches above the SM count, partly frozen
    models) on tied windows: forward elementwise, dγ and dβ per channel, dy elementwise."""
    from pytorch_distributed_train_b200 import _C

    B = 4
    y, _ = tied_frames(B, H, C, seed=C + H)
    gamma, beta, mean, invstd = bn_params(y)
    y, gamma, beta = y.to(dev()), gamma.to(dev()), beta.to(dev())
    mean, invstd = mean.to(dev()), invstd.to(dev())
    dout = torch.randn(B, C, H // 2, H // 2, device=dev(), dtype=torch.float64)
    ref_out, ref_dy, ref_dg, ref_db, gz = _oracle(y, gamma, beta, dout)
    var = (y.double().var((0, 1, 2), unbiased=False))
    out, saved_fwd = _C.bn_relu_pool_fwd(y, torch.cat([mean, var]).float(), gamma, beta, None, None, None, 0.1, EPS, out_nchw,
                                         mean_var=True)
    got = out if out_nchw else out.permute(0, 3, 1, 2)
    # the fp32 affine of values ≤ 1 around a mean ≤ 1, scaled by invstd ≤ 4: a few ulp of ~10
    assert torch.allclose(got.double(), ref_out, atol=1e-5, rtol=1e-5), (got.double() - ref_out).abs().max().item()
    saved = torch.cat([mean, invstd]).float()
    assert torch.allclose(saved_fwd, saved, rtol=1e-6, atol=0)
    d = dout.float().contiguous() if out_nchw else dout.float().permute(0, 2, 3, 1).contiguous()
    sums, dgamma, dbeta = _C.bn_relu_pool_bwd_reduce(d, y, saved, gamma, beta, out_nchw)
    xh = _xhat(y, mean, invstd)
    _assert_bn_sums(dgamma, dbeta, ref_dg, ref_db, gz, xh, "per-op")
    count = torch.full((1,), float(B * H * H), device=dev())
    dy = _C.bn_relu_pool_bwd_apply(d, y, saved, gamma, beta, sums, count, out_nchw)
    _assert_dy(dy.permute(0, 3, 1, 2), ref_dy, gamma, invstd, dout.abs().max().item(), "per-op")


@pytest.mark.gpu
def test_fused_layer2_backward_routes_ties_like_float64():
    """convnet_l2_bwd_fc (the z > best scan, windows g + 8k of warp g) on a tied conv2 output: dγ2, dβ2 and the dy frame against
    float64 BN → ReLU → pool → classifier backward, and the classifier gradients it computes alongside."""
    from pytorch_distributed_train_b200 import _C

    B, ncls = 6, 10
    y, _ = tied_frames(B, 14, 32, seed=3)
    gamma, beta, mean, invstd = bn_params(y)
    y, gamma, beta, mean, invstd = (t.to(dev()) for t in (y, gamma, beta, mean, invstd))
    fcw = torch.randn(ncls, 1568, device=dev()) * 0.05
    fcb = torch.randn(ncls, device=dev()) * 0.1
    dlogits = torch.randn(B, ncls, device=dev())
    # the classifier's backward in float64 gives the pooled gradient the oracle routes
    pooled = F.max_pool2d(F.relu(F.batch_norm(y.double().permute(0, 3, 1, 2), None, None, gamma.double(), beta.double(), True, 0.0,
                                              EPS)), 2, 2)
    dpool = (dlogits.double() @ fcw.double()).view(B, 32, 7, 7)
    ref_out, ref_dy, ref_dg, ref_db, gz = _oracle(y, gamma, beta, dpool)
    assert torch.equal(ref_out, pooled)
    out = ref_out.float().contiguous()
    w2 = torch.randn(32, 16, 5, 5, device=dev()) * 0.1
    dfcw, dfcb = torch.empty_like(fcw), torch.empty_like(fcb)
    dg, db = torch.empty(32, device=dev()), torch.empty(32, device=dev())
    saved = torch.cat([mean, invstd]).float()
    dy, _, _ = _C.convnet_l2_bwd_fc(dlogits, fcw, out, dfcw, dfcb, y, saved, gamma, beta, w2, dg, db)
    torch.cuda.synchronize()
    xh = _xhat(y, mean, invstd)
    _assert_bn_sums(dg, db, ref_dg, ref_db, gz, xh, "layer 2")
    assert float(dy[:, :2].abs().max()) == 0.0 and float(dy[:, 16:].abs().max()) == 0.0
    assert float(dy[:, :, :2].abs().max()) == 0.0 and float(dy[:, :, 16:].abs().max()) == 0.0
    _assert_dy(dy[:, 2:16, 2:16, :].permute(0, 3, 1, 2), ref_dy, gamma, invstd, dpool.abs().max().item(), "layer 2")
    # the classifier: dW = dlogitsᵀ·pooled, db = Σ dlogits, fp32 sums over B images
    od, dd = out.double().view(B, -1), dlogits.double()
    ref_dfcw, mag = dd.t() @ od, dd.abs().t() @ od.abs()
    assert bool(((dfcw.double() - ref_dfcw).abs() <= 1e-5 * mag + 1e-7).all()), (dfcw.double() - ref_dfcw).abs().max().item()
    assert torch.allclose(dfcb.double(), dd.sum(0), atol=1e-6, rtol=1e-5)


@pytest.mark.gpu
def test_fused_layer1_backward_routes_ties_like_float64():
    """convnet_l1_bwd_wgrad (the four-lane bitmask over L1Map's 784 threads) on a tied conv1 output with a random pooled gradient
    and random images: dγ1, dβ1 (fp32) and dW1, db1 (TF32: conv1's weight gradient runs on mma.sync).  A window routed to another
    tied pixel multiplies another 5×5 image neighbourhood into dW1."""
    from pytorch_distributed_train_b200 import _C

    B = 2
    y, _ = tied_frames(B, 28, 16, seed=5)
    gamma, beta, mean, invstd = bn_params(y)
    y, gamma, beta, mean, invstd = (t.to(dev()) for t in (y, gamma, beta, mean, invstd))
    x = torch.randint(0, GRID + 1, (B, 1, 28, 28), device=dev()).float() / GRID   # exact in TF32
    dp = torch.zeros(B, 18, 18, 16, device=dev())
    dp[:, 2:16, 2:16, :] = torch.randn(B, 14, 14, 16, device=dev())
    dpool = dp[:, 2:16, 2:16, :].permute(0, 3, 1, 2).double()
    _, ref_dy, ref_dg, ref_db, gz = _oracle(y, gamma, beta, dpool)
    xd = x.double()
    ref_dw = torch.nn.grad.conv2d_weight(xd, (16, 1, 5, 5), ref_dy, padding=2)
    mag_dw = torch.nn.grad.conv2d_weight(xd.abs(), (16, 1, 5, 5), ref_dy.abs(), padding=2)
    saved = torch.cat([mean, invstd]).float()
    dg, dbe = torch.empty(16, device=dev()), torch.empty(16, device=dev())
    dw, db = torch.empty(16, 1, 5, 5, device=dev()), torch.empty(16, device=dev())
    dw2, db2 = torch.empty(32, 16, 5, 5, device=dev()), torch.empty(32, device=dev())
    _C.convnet_l1_bwd_wgrad(dp, y, x, saved, gamma, beta, dg, dbe, dw, db, torch.zeros(B, 18, 18, 32, device=dev()),
                            torch.zeros(B, 18, 18, 16, device=dev()), torch.zeros(B, 32, device=dev()), dw2, db2)
    torch.cuda.synchronize()
    _assert_bn_sums(dg, dbe, ref_dg, ref_db, gz, _xhat(y, mean, invstd), "layer 1")
    # dy rounded to TF32 (2⁻¹¹ relative) times exact x, fp32 accumulation over B·784 products
    err = (dw.double() - ref_dw).abs()
    assert bool((err <= 1e-3 * mag_dw + 1e-6).all()), ("dW1", err.max().item(), (err / mag_dw.clamp_min(1e-30)).max().item())
    mag_db = ref_dy.abs().sum((0, 2, 3))
    assert bool(((db.double() - ref_dy.sum((0, 2, 3))).abs() <= 1e-3 * mag_db + 1e-6).all()), "db1"


@pytest.mark.gpu
def test_fused_forward_pools_ties_like_float64():
    """convnet_fwd on images whose conv1 outputs tie: a centre-tap conv1 filter of ±1 without bias makes y1 = ±x exactly, and a
    centre-tap conv2 filter of ±1 makes y2 = ±p1 (TF32-rounded).  The pooled frame p1 (fp32) and layer 2's pooled output (TF32)
    against float64, over 15 images so that every tie pattern meets every window of both thread mappings (win, win + 98)."""
    from pytorch_distributed_train_b200 import _C

    B = 15
    u, _ = tied_frames(B, 28, 1, seed=7)
    x = u.permute(0, 3, 1, 2).contiguous().to(dev())                      # [B, 1, 28, 28] on the 1/16 grid
    sign1 = torch.where(_negated(16), -1.0, 1.0)
    w1 = torch.zeros(16, 1, 5, 5)
    w1[:, 0, 2, 2] = sign1
    y1_ref = (x.cpu().double() * sign1.double().view(1, 16, 1, 1)).permute(0, 2, 3, 1).float()
    g1, be1, _, _ = bn_params(y1_ref, to_y=lambda t: -t)
    # layer 2: y2[co] = ±p1[co mod 16]; its BatchNorm kinds with fixed β (the pooled value is continuous in z)
    sign2 = torch.where(torch.arange(32) % 3 == 1, -1.0, 1.0)
    w2 = torch.zeros(32, 16, 5, 5)
    w2[torch.arange(32), torch.arange(32) % 16, 2, 2] = sign2
    k2 = kinds(32)
    g2 = torch.tensor([0.0 if k.startswith("zero") else (-1.0 if k.startswith("neg") else 1.0) * (0.6 + 0.2 * (c % 3))
                       for c, k in enumerate(k2)])
    be2 = torch.tensor([{"zero": 0.75, "zero_zero": 0.0, "relu": -0.5, "neg_relu": -0.5}.get(k, 0.1) for k in k2])
    fcw, fcb = torch.randn(10, 1568) * 0.02, torch.zeros(10)
    w1, g1, be1, w2, g2, be2, fcw, fcb = (t.to(dev()) for t in (w1, g1, be1, w2, g2, be2, fcw, fcb))
    p1, y1, sv1, out, y2, sv2, *_ = _C.convnet_fwd(x, w1, None, g1, be1, None, None, None, 0.1, EPS, w2, None, g2, be2, None, None,
                                                   None, 0.1, EPS, fcw, fcb)
    torch.cuda.synchronize()
    assert torch.equal(y1.cpu(), y1_ref)
    z1 = F.batch_norm(y1_ref.double().permute(0, 3, 1, 2), None, None, g1.double().cpu(), be1.double().cpu(), True, 0.0, EPS)
    ref_p1 = F.max_pool2d(F.relu(z1), 2, 2)
    got_p1 = p1[:, 2:16, 2:16, :].permute(0, 3, 1, 2).double().cpu()
    # fp32 batch statistics and affine: a few ulp of values up to ~5
    assert torch.allclose(got_p1, ref_p1, atol=2e-5, rtol=1e-5), (got_p1 - ref_p1).abs().max().item()
    assert float(_windows(z1).amax(-1).lt(0).sum()) > 0 and float(_windows(z1).amax(-1).gt(0).sum()) > 0
    z2 = F.batch_norm(F.conv2d(ref_p1, w2.double().cpu(), None, padding=2), None, None, g2.double().cpu(), be2.double().cpu(), True,
                      0.0, EPS)
    ref_out = F.max_pool2d(F.relu(z2), 2, 2)
    # y2 is p1 rounded to TF32 (2⁻¹¹ relative), normalised by batch statistics of the rounded values
    err = (out.double().cpu() - ref_out).abs().max().item()
    assert err <= 2e-3 * ref_out.abs().max().item(), err


# ---- 3. the ConvNet on MNIST-like images --------------------------------------------------------------------------------------
def mnist_like(B, seed):
    """Digit-like images: an exactly-zero background, strokes of three segments in the central 14×14 with cores saturated at 1.0
    and edges in k/255 steps (the blank border keeps conv outputs tied in both layers)."""
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(B, 3, 2, 2, generator=g) * 10 + 9                       # segment endpoints in [9, 19)
    a, b = p[:, :, 0], p[:, :, 1]
    rr, cc = torch.meshgrid(torch.arange(28.0), torch.arange(28.0), indexing="ij")
    q = torch.stack([rr, cc], -1).view(1, 1, 28, 28, 2)
    ab = (b - a).view(B, 3, 1, 1, 2)
    t = (((q - a.view(B, 3, 1, 1, 2)) * ab).sum(-1) / (ab * ab).sum(-1).clamp_min(1e-6)).clamp(0, 1)
    d = (q - a.view(B, 3, 1, 1, 2) - t[..., None] * ab).norm(dim=-1).amin(1)   # distance to the nearest segment
    v = ((2.2 - d) / 1.2).clamp(0, 1)                                      # core radius 1, edge 1.2 wide
    return (torch.round(v * 255) / 255).view(B, 1, 28, 28)


def _set_batchnorm(net):
    """γ = 0 on a few BatchNorm channels (one of them with β = 0 too), γ < 0 on one, small random β elsewhere."""
    with torch.no_grad():
        for bn, zero, neg in ((net.layer1[1], [3, 7, 12], 10), (net.layer2[1], [5, 17, 29], 20)):
            bn.bias.copy_(torch.randn(bn.bias.shape) * 0.1)
            bn.weight[zero] = 0.0
            bn.bias[zero[:2]] = 0.3
            bn.bias[zero[2]] = 0.0
            bn.weight[neg] = -0.8


def _float64_twin(net):
    ref = pdt.models.ConvNet(num_classes=net.fc.out_features, fused=False).to(dev())
    ref.load_state_dict(net.state_dict())
    return ref.double()


def _tied_windows(ref, x):
    """Windows of the float64 oracle whose maximum is positive and tied, per layer: (all channels, channels with γ ≠ 0)."""
    def count(z, gamma):
        w = _windows(z)
        m = w.amax(-1, keepdim=True)
        tied = ((w == m).sum(-1) >= 2) & (m.squeeze(-1) > 0)
        return int(tied.sum()), int(tied[:, gamma != 0].sum())

    with torch.no_grad():
        l1, l2 = ref.layer1, ref.layer2
        z1 = F.batch_norm(l1[0](x), None, None, l1[1].weight, l1[1].bias, True, 0.0, l1[1].eps)
        z2 = F.batch_norm(l2[0](F.max_pool2d(F.relu(z1), 2, 2)), None, None, l2[1].weight, l2[1].bias, True, 0.0, l2[1].eps)
        return count(z1, l1[1].weight), count(z2, l2[1].weight)


def _assert_grads(net, ref):
    for (n1, p1), (_, p2) in zip(net.named_parameters(), ref.named_parameters()):
        # conv2 runs in TF32 forward and in dgrad; conv biases in front of a BatchNorm have a true gradient of zero (noise level)
        err, norm = (p1.grad.double() - p2.grad).norm().item(), p2.grad.norm().item()
        assert err <= 3e-2 * norm + 1e-4 * p2.numel() ** 0.5, (n1, err, norm)


def _assert_buffers(net, ref):
    for (n1, b1), (_, b2) in zip(net.named_buffers(), ref.named_buffers()):
        if n1.endswith("num_batches_tracked"):
            assert int(b1) == int(b2), n1
        else:
            # batch statistics of the TF32 conv2 output
            assert torch.allclose(b1.double(), b2.double(), atol=2e-3, rtol=1e-3), (n1, (b1.double() - b2.double()).abs().max().item())


def _run_model(B, per_op, seed):
    from pytorch_distributed_train_b200.ops import functional as OF

    torch.manual_seed(seed)
    net = pdt.models.ConvNet(fused=True).to(dev())
    _set_batchnorm(net)
    ref = _float64_twin(net)
    x = mnist_like(B, seed).to(dev())
    t = torch.randint(0, 10, (B,), device=dev())
    (t1, t1g), (t2, t2g) = _tied_windows(ref, x.double())
    assert t1g > 0 and t2 > 0, ("the batch must tie windows with a positive maximum in both layers", t1, t1g, t2, t2g)
    with (pytest.MonkeyPatch.context() if per_op else contextlib.nullcontext()) as mp:
        if per_op:
            mp.setenv("PDT_FUSED_LAYERS", "0")
        assert OF.fused_convnet_ok(x, net) == (not per_op)
        loss = pdt.nn.CrossEntropyLoss()(net(x), t)
        loss.backward()
    ref_loss = F.cross_entropy(ref(x.double()), t)
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) < 2e-3, (loss.item(), ref_loss.item())
    _assert_grads(net, ref)
    _assert_buffers(net, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 100, "sms"])
def test_fused_convnet_on_mnist_like_ties_matches_float64(B):
    B = sms() if B == "sms" else B
    _run_model(B, per_op=False, seed=11)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [100, "sms+1"])
def test_per_op_convnet_on_mnist_like_ties_matches_float64(B):
    B = sms() + 1 if B == "sms+1" else B
    _run_model(B, per_op=True, seed=12)


@pytest.mark.gpu
def test_graphed_sgd_step_on_mnist_like_ties_matches_float64():
    """One replay of the graphed step (forward, both backward kernels, SGD riding on the last): gradients, running statistics and
    updated parameters against the float64 twin of the model as the replay found it."""
    from mp_helpers import free_port
    from pytorch_distributed_train_b200.engine import GraphedTrainStep

    torch.cuda.set_device(0)
    pdt.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{free_port()}", world_size=1, rank=0)
    try:
        torch.manual_seed(13)
        model = pdt.models.ConvNet(fused=True).to(dev())
        opt = pdt.optim.SGD(model.parameters(), lr=0.05)
        crit = pdt.nn.CrossEntropyLoss()
        x = mnist_like(100, 13).to(dev())
        t = torch.randint(0, 10, (100,), device=dev())
        step = GraphedTrainStep(pdt.DistributedDataParallel(model, device_ids=[0]), crit, opt, (x, t), warmup=2,
                                double_buffer_inputs=False)
        assert step._riding
        _set_batchnorm(model)   # the warm-up steps moved γ off 0: set it again in place, where the graph reads it
        ref = _float64_twin(model)
        p0 = [p.detach().double().clone() for p in model.parameters()]
        (t1, t1g), (t2, t2g) = _tied_windows(ref, x.double())
        assert t1g > 0 and t2 > 0, (t1, t1g, t2, t2g)
        step(x, t, inputs_ready=True)
        torch.cuda.synchronize()
        F.cross_entropy(ref(x.double()), t).backward()
        _assert_grads(model, ref)
        _assert_buffers(model, ref)
        lr = torch.tensor(0.05, dtype=torch.float32).item()
        for (n1, p), q, r0 in zip(model.named_parameters(), ref.parameters(), p0):
            # the rider's p − lr·g in fp32, from the gradient it stored
            own = r0 - lr * p.grad.double()
            assert bool(((p.double() - own).abs() <= 2 * 2.0 ** -24 * (r0.abs() + lr * p.grad.double().abs()) + 1e-30).all()), n1
            err = (p.double() - (r0 - lr * q.grad)).norm().item()
            assert err <= lr * (3e-2 * q.grad.norm().item() + 1e-4 * q.numel() ** 0.5) + 1e-6, (n1, err)
        opt.stop_riding()
    finally:
        pdt.destroy_process_group()
