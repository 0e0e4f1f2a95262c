#!/usr/bin/env python
"""Hardware check of the experimental window conv kernels (impl="win") against the SIMT oracle.

    PDT_WIN_BASE_OFFSET=0 python tools/check_conv_win.py     # base offset 0: address-based swizzle (default, correct)
    PDT_WIN_BASE_OFFSET=1 python tools/check_conv_win.py     # descriptor base offset = (start >> 7) & 7  (wrong on Hopper)

Small-integer inputs make TF32 exact, so "max err" must be 0 for a correct kernel.  Also times both variants.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch

    import pytorch_distributed_train_b200 as pdt

    C = pdt._C
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    for B in (3, 100):
        x = torch.randint(-3, 4, (B, 14, 14, 16), device=dev, generator=g).float()
        w = torch.randint(-2, 3, (32, 16, 5, 5), device=dev, generator=g).float()
        b = torch.randint(-2, 3, (32,), device=dev, generator=g).float()
        dy = torch.randint(-3, 4, (B, 14, 14, 32), device=dev, generator=g).float()
        y0, s0 = C.conv5x5_fwd(x, w, b, True, "simt")
        y1, s1 = C.conv5x5_fwd(x, w, b, True, "win")
        d0 = C.conv5x5_dgrad(dy, w, "simt")
        d1 = C.conv5x5_dgrad(dy, w, "win")
        torch.cuda.synchronize()
        print(f"B={B}: fwd max err {(y0 - y1).abs().max().item():.3g}  stats max err {(s0 - s1).abs().max().item():.3g}  "
              f"dgrad max err {(d0 - d1).abs().max().item():.3g}", flush=True)

    def t(fn, n=50):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        e.record()
        torch.cuda.synchronize()
        return a.elapsed_time(e) / n * 1e3

    for impl in ("tma", "win"):
        print(f"{impl}: fwd {t(lambda: C.conv5x5_fwd(x, w, b, True, impl)):.1f} us   dgrad {t(lambda: C.conv5x5_dgrad(dy, w, impl)):.1f} us "
              "(back-to-back launches, incl. weight repack)", flush=True)


if __name__ == "__main__":
    main()
