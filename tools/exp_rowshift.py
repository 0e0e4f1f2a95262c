#!/usr/bin/env python
"""Hardware check of the descriptor convention the window convolutions rely on (filter taps read as row-shifted descriptors).

Question: with a K-major SWIZZLE_64B / SWIZZLE_128B operand in shared memory, may the wgmma
descriptor start at an arbitrary ROW of a larger TMA-loaded buffer (that is what turns 25 im2col
gathers per pixel into one tiled load of the haloed patch)?  For every shift in 0..40 and for
descriptor base-offset = 0 (mode 0) or (start >> 7) & 7 (mode 1) the kernel computes
D = A[shift:shift+128] · Bᵀ on small integers (exact in TF32) and we compare with the exact result.

    python tools/exp_rowshift.py          # prints one line per (row bytes, mode): which shifts are exact
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch

    import pytorch_distributed_train_b200 as pdt

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    for kf in (32, 16):
        a = torch.randint(-4, 5, (256, kf), device=dev, generator=g).float()
        b = torch.randint(-4, 5, (32, kf), device=dev, generator=g).float()
        for mode in (0, 1):
            ok, bad = [], []
            for shift in range(0, 41):
                d = pdt._C.umma_rowshift_probe(a, b, shift, mode)
                torch.cuda.synchronize()
                exact = a[shift:shift + 128].double() @ b.double().t()
                (ok if torch.equal(d.double(), exact) else bad).append(shift)
            print(f"row bytes {kf * 4:3d}  base_offset mode {mode}:  exact for shifts {ok}   WRONG for {bad}", flush=True)


if __name__ == "__main__":
    main()
