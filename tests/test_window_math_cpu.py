"""CPU emulation of the index arithmetic of the tensor-core "window" kernels (no GPU): what the descriptors address, not how fast.

* forward / data gradient (K-major patch, 25 row-shifted descriptors): tools/emulate_window_conv.py, run here as a test;
* weight gradient riding on layer-1 backward (csrc/cuda/fused_convnet.cu, L1WgCfg): ONE overlapping-row view of the zero-haloed
  x frame (row r = positions r and r+1 × 16 channels = a 32-wide MN-major atom), four M = 128 tiles whose four atoms sit at a
  uniform row stride (the descriptor's LBO) — tiles 0-2 stack kh = 0..3 at 18 rows for kw/2 = 0,1,2; tile 3 stacks kw/2 = 0..3 at
  2 rows for kh = 4 — K = 256 positions from the first interior one in 32 steps of 8, and the fold's accumulator-row → (kh, kw, ci)
  mapping.  Checked against torch.nn.grad.conv2d_weight in float64.
"""
import importlib.util
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PW, FRAME, FIRST = 18, 18 * 18, 2 * 18 + 2


def _frames(B, C, gen):
    f = torch.zeros(B, 18, 18, C, dtype=torch.float64)
    f[:, 2:16, 2:16, :] = torch.randn(B, 14, 14, C, dtype=torch.float64, generator=gen)
    return f


def window_wgrad(x_frames: torch.Tensor, dy_frames: torch.Tensor) -> torch.Tensor:
    """x_frames [B,18,18,16], dy_frames [B,18,18,32] (zero halos) → dW [32,16,5,5] through the kernel's addressing."""
    B = x_frames.shape[0]
    xf = x_frames.reshape(B * FRAME, 16)
    dyf = dy_frames.reshape(B * FRAME, 32)
    # overlapping-row view of the whole batch: row r = [x[r], x[r+1]]; rows past the tensor read as zero (TMA out-of-bounds fill)
    xpad = torch.cat([xf, torch.zeros(512, 16, dtype=xf.dtype)])
    view = torch.cat([xpad[:-1], xpad[1:]], dim=1)                     # [rows, 32]
    dw = torch.zeros(32, 16, 5, 5, dtype=xf.dtype)
    for n in range(B):
        frame0 = n * FRAME
        window = view[frame0:frame0 + 6 * 64]                          # six 64-row TMA boxes = the A window in smem
        btile = torch.cat([dyf, torch.zeros(512, 32, dtype=dyf.dtype)])[frame0 + FIRST:frame0 + FIRST + 256]   # two 128-row boxes
        acc = torch.zeros(4, 128, 32, dtype=xf.dtype)                  # four accumulators [M = 128][N = 32]
        for mt in range(4):
            shift0 = (0 - 2) * 18 + 2 * mt - 2 if mt < 3 else 2 * 18 - 2
            lbo_rows = 18 if mt < 3 else 2
            for kc in range(32):                                       # K = 8 positions per MMA
                a = torch.zeros(8, 128, dtype=xf.dtype)                # A[k][m], MN-major
                for atom in range(4):
                    row = FIRST + 8 * kc + shift0 + atom * lbo_rows
                    a[:, atom * 32:(atom + 1) * 32] = window[row:row + 8]
                acc[mt] += a.t() @ btile[8 * kc:8 * kc + 8]
        for kh in range(5):
            for kw in range(5):
                for ci in range(16):
                    mrow = ((kw >> 1) * 128 + kh * 32 if kh < 4 else 384 + (kw >> 1) * 32) + (kw & 1) * 16 + ci
                    dw[:, ci, kh, kw] += acc[mrow // 128, mrow % 128]
    return dw


def test_window_weight_gradient_addressing_matches_conv2d_weight():
    g = torch.Generator().manual_seed(0)
    for B in (1, 3):
        x, dy = _frames(B, 16, g), _frames(B, 32, g)
        ref = torch.nn.grad.conv2d_weight(x[:, 2:16, 2:16, :].permute(0, 3, 1, 2), (32, 16, 5, 5), dy[:, 2:16, 2:16, :].permute(0, 3, 1, 2), padding=2)
        got = window_wgrad(x, dy)
        assert (got - ref).abs().max().item() < 1e-10
    # the window never reaches outside its six boxes, and the dummy fourth atom of tile 3 (kw/2 = 3) is the only garbage column block
    assert FIRST + 8 * 31 + (2 * 18 - 2) + 3 * 2 + 7 < 6 * 64 and FIRST + (0 - 2) * 18 - 2 == 0


def test_window_forward_and_dgrad_addressing():
    spec = importlib.util.spec_from_file_location("emulate_window_conv", os.path.join(ROOT, "tools", "emulate_window_conv.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.main() == 0
