"""CPU emulation of the shared-memory operands of conv2's weight gradient on wgmma (no GPU): what the descriptors address, not how
fast.

The layer-2 backward kernel and conv2_wgrad_partials_kernel (csrc/cuda/fused_convnet.cu, Conv2Wg) write K-major copies of x and dy
in the no-swizzle canonical layout — a core matrix is 8 rows × 4 positions, 128 contiguous bytes — and issue 10 tiles × 32 K-steps
of wgmma m64n32k8 over them.  This builds both byte images with the kernels' index arithmetic (memory nobody writes holds NaN),
walks every tile's descriptors (start address, LBO, SBO, K-step) the way the tensor core reads them, and checks the implied GEMM
against torch.nn.grad.conv2d_weight in float64: real rows exact, pad rows (kh > 4) and the slack positions past the frame included,
every read inside the allocation.
"""
import numpy as np
import torch

FRAME, FIRST = 18 * 18, 2 * 18 + 2
X_BLOCKS = 83
X_COPY = (2 * (X_BLOCKS - 1) + 9 + 1) * 128
LBO_A, SBO_A = 256, 1152
LBO_B, SBO_B = 512, 128
X_REACH = 3 * X_COPY + 2 * 4 * 128 + 7 * SBO_A + 31 * 512 + LBO_A + 128
X_BYTES = (X_REACH + 1023) // 1024 * 1024
DYT_BYTES = 64 * 512
# layer-2 backward kernel, FC form: the x copies go over the fc weights, dyᵀ behind them; the kernel's smem size and the opt-in limit
PATCH_ALLOC, DGRAD_B, MISC, FC_W = 43008, 25 * 16 * 128, 4096, 16 * 1568 * 4


def dyt_off(co, p):
    return (p >> 2) * 512 + (co >> 3) * 128 + (co & 7) * 16 + (p & 3) * 4


def build_x(frame):
    """Conv2WgX (load, store): frame [324, 16] → the byte image of the four residue copies, as float64 words (unwritten: NaN)."""
    img = np.full(X_BYTES // 4, np.nan)
    for ci in range(16):
        for q in range(X_BLOCKS):
            v = [frame[4 * q + k, ci] if 4 * q + k < FRAME else 0.0 for k in range(7)]
            dst = (2 * q + 9 * (ci >> 3)) * 128 + (ci & 7) * 16
            for r in range(4):
                for i in range(4):
                    w = (dst + r * X_COPY) // 4 + i
                    assert np.isnan(img[w]), "two blocks overlap"
                    img[w] = v[r + i]
    return img


def build_dyt_layer2(frame):
    """The layer-2 backward kernel's dyᵀ: interior values from the dy registers, zeros at the 60 halo positions of the window."""
    img = np.full(DYT_BYTES // 4, np.nan)
    for oh in range(14):
        for ow in range(14):
            P = (oh + 2) * 18 + ow + 2
            for c in range(32):
                img[dyt_off(c, P - FIRST) // 4] = frame[P, c]
    for h in range(64):
        if h < 60:
            P = 18 * (2 + (h >> 2)) + 16 + (h & 3) if h < 52 else 286 + h - 52
            for c in range(32):
                img[dyt_off(c, P - FIRST) // 4] = 0.0
    return img


def build_dyt_standalone(frame):
    """conv2_wgrad_partials_kernel's dyᵀ: task (co, kc) writes positions 4kc .. 4kc + 3 of channel co from the frame."""
    img = np.full(DYT_BYTES // 4, np.nan)
    for co in range(32):
        for kc in range(64):
            for i in range(4):
                img[(dyt_off(co, 4 * kc) + 4 * i) // 4] = frame[FIRST + 4 * kc + i, co]
    return img


def core_kmajor(start, lbo, sbo, rows):
    """Word index of element (row, k) of a K-major no-swizzle operand of `rows` rows and K = 8 (one wgmma K-step)."""
    m = np.arange(rows)[:, None]
    k = np.arange(8)[None, :]
    return (start + (m >> 3) * sbo + (k >> 2) * lbo + (m & 7) * 16 + (k & 3) * 4) // 4


def partial_from_images(ximg, dyimg):
    """conv2_wgrad_wgmma on the byte images: the per-image partial [400][32] and the largest byte offset read from the x copies."""
    part = np.full((400, 32), np.nan)
    reach = 0
    for kw in range(5):
        for par in range(2):
            off = 18 * par + kw
            astart = (off & 3) * X_COPY + (off >> 2) * 256
            acc = np.zeros((64, 32))
            for s in range(32):
                ai = core_kmajor(astart + s * 512, LBO_A, SBO_A, 64)
                bi = core_kmajor(s * 1024, LBO_B, SBO_B, 32)
                reach = max(reach, 4 * int(ai.max()) + 4)
                with np.errstate(invalid="ignore"):
                    acc += ximg[ai] @ dyimg[bi].T
            for row in range(64):
                g = row >> 3
                kh = par + 2 * (g >> 1)
                if kh < 5:
                    part[(kh * 5 + kw) * 16 + 8 * (g & 1) + (row & 7)] = acc[row]
                else:
                    assert kh in (5, 6, 7)   # pad rows: computed, not stored
    return part, reach


def _frames(B, C, gen):
    f = torch.zeros(B, 18, 18, C, dtype=torch.float64)
    f[:, 2:16, 2:16, :] = torch.randn(B, 14, 14, C, dtype=torch.float64, generator=gen)
    return f


def test_kmajor_operands_and_descriptors_match_conv2d_weight():
    g = torch.Generator().manual_seed(0)
    B = 2
    x, dy = _frames(B, 16, g), _frames(B, 32, g)
    want = torch.nn.grad.conv2d_weight(x[:, 2:16, 2:16, :].permute(0, 3, 1, 2), (32, 16, 5, 5), dy[:, 2:16, 2:16, :].permute(0, 3, 1, 2),
                                       padding=2).numpy()
    got = np.zeros((32, 16, 5, 5))
    for n in range(B):
        xf, dyf = x[n].reshape(FRAME, 16).numpy(), dy[n].reshape(FRAME, 32).numpy()
        ximg = build_x(xf)
        dy2, dys = build_dyt_layer2(dyf), build_dyt_standalone(dyf)
        # both kernels write every word of dyᵀ, and the same values
        assert not np.isnan(dy2).any() and np.array_equal(dy2, dys)
        part, reach = partial_from_images(ximg, dy2)
        assert np.isfinite(part).all(), "a real row met memory nobody wrote"
        assert reach == X_REACH <= X_BYTES
        for kh in range(5):
            for kw in range(5):
                for ci in range(16):
                    got[:, ci, kh, kw] += part[(kh * 5 + kw) * 16 + ci]
    assert np.abs(got - want).max() < 1e-10


def test_shared_memory_placement():
    x_t = PATCH_ALLOC + DGRAD_B + MISC
    dy_t = x_t + X_BYTES
    total = 1024 + dy_t + DYT_BYTES
    assert X_BYTES <= FC_W and total <= 227 * 1024
    assert x_t % 1024 == 0 and dy_t % 1024 == 0 and X_COPY % 16 == 0
