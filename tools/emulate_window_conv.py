#!/usr/bin/env python
"""CPU emulation of the index math of the planned "window" conv2 kernel (conv_tcgen05.cu).

The kernel will load, per tile, ONE zero-haloed patch of the NHWC input in padded-width coordinates
(PW = W + 4 positions per padded image row) and feed the tensor core 25 row-shifted views of that single
buffer: for tap (kh, kw) the A operand is buffer rows [off + kh·PW + kw, … + M).  Output row m of the tile is
padded position q = q0 + m → (oh, ow') = divmod(q, PW); it is a real output iff ow' < W.  This script checks
that mapping against F.conv2d for forward and data-gradient, including the tile → TMA-box arithmetic
(box = full padded rows [ih0, ih0 + box_h) × [-2, W + 2), zero fill outside the image).

    python tools/emulate_window_conv.py        # exits non-zero on mismatch
"""
import sys

import torch
import torch.nn.functional as F


def window_conv(x_nhwc: torch.Tensor, w_taps: torch.Tensor, rows_per_tile: int):
    """x_nhwc [B,H,W,C]; w_taps [25][C][N] (tap-major GEMM B operand); returns y [B,H,W,N]."""
    B, H, W, C = x_nhwc.shape
    N = w_taps.shape[2]
    PW = W + 4
    M = rows_per_tile * PW                      # MMA rows per tile (126 for 7 output rows of a 14-wide image)
    assert H % rows_per_tile == 0 and M <= 128
    box_h = rows_per_tile + 4                   # padded input rows the tile needs
    y = torch.zeros(B, H, W, N, dtype=x_nhwc.dtype)
    for n in range(B):
        for t in range(H // rows_per_tile):
            oh0 = t * rows_per_tile
            # --- what the TMA box delivers: padded rows ih' = oh0 .. oh0+box_h-1 (input rows oh0-2 ...), all PW columns
            buf = torch.zeros(box_h * PW + 4, C, dtype=x_nhwc.dtype)   # +4: the last tap of the last row reads 4 past
            for r in range(box_h):
                ih = oh0 + r - 2
                if 0 <= ih < H:
                    buf[r * PW + 2:r * PW + 2 + W] = x_nhwc[n, ih]      # columns -2,-1 and W,W+1 stay zero (OOB fill)
            acc = torch.zeros(M, N, dtype=x_nhwc.dtype)
            for kh in range(5):
                for kw in range(5):
                    start = kh * PW + kw                                  # descriptor row shift of this tap
                    acc += buf[start:start + M] @ w_taps[kh * 5 + kw]
            for m in range(M):
                r, owp = divmod(m, PW)
                if owp < W:                                               # the other 4 of every 18 rows are padding
                    y[n, oh0 + r, owp] = acc[m]
    return y


def main() -> int:
    torch.manual_seed(0)
    ok = True
    for (B, H, C, N, rows) in [(3, 14, 16, 32, 7), (2, 14, 32, 16, 7), (2, 28, 4, 8, 4)]:
        x = torch.randn(B, C, H, H, dtype=torch.float64)
        w = torch.randn(N, C, 5, 5, dtype=torch.float64)
        ref = F.conv2d(x, w, padding=2).permute(0, 2, 3, 1)
        w_taps = w.permute(2, 3, 1, 0).reshape(25, C, N)                  # [tap][ci][co]
        got = window_conv(x.permute(0, 2, 3, 1).contiguous(), w_taps, rows)
        e = (got - ref).abs().max().item()
        print(f"forward  B={B} H={H} C={C} N={N}: max err {e:.2e}")
        ok &= e < 1e-10
        # data gradient = the same kernel on dy with flipped, transposed weights
        dy = torch.randn(B, N, H, H, dtype=torch.float64)
        xr = x.clone().requires_grad_()
        F.conv2d(xr, w, padding=2).backward(dy)
        wT = w.flip(2, 3).permute(2, 3, 0, 1).reshape(25, N, C)           # [tap][co][ci], tap order reversed
        gx = window_conv(dy.permute(0, 2, 3, 1).contiguous(), wT, rows)
        e = (gx - xr.grad.permute(0, 2, 3, 1)).abs().max().item()
        print(f"dgrad    B={B} H={H} C={C} N={N}: max err {e:.2e}")
        ok &= e < 1e-10
    print("window-conv index math:", "OK" if ok else "MISMATCH")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
