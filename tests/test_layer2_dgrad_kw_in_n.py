"""CPU emulation of conv2's data gradient in the layer-2 backward kernel (no GPU): what the descriptors address and what the epilogue
adds, not how fast.

convnet_l2_bwd_kernel (csrc/cuda/fused_convnet.cu) puts the filter column kw into N: warps 4..7 issue 80 wgmma m64n80k8 that compute
D'[q][16·kw + ci] = Σ_{kh, co} dy[q + 18·kh][co] · Bd[5·kh + kw][ci][co] over patch rows q = 0..255, the A descriptor of row kh being
the swizzled dy patch 18·kh rows further in and the B descriptor the 80 rows (kw, ci) of the flipped weight tiles at kh·10240 bytes.
l2_dgrad_epilogue then forms dx[p][ci] = Σ_kw D'[p + kw][16·kw + ci] from the accumulator fragments: shuffles inside a warp's 16 rows,
the first four rows of the next range through the edge buffer (l2_dgrad_edge_store, l2_dgrad_edge_slot).  This builds the patch and
the weight tiles as byte images with the kernel's index arithmetic (memory nobody writes holds NaN), reads them through the
SWIZZLE_128B descriptors the way the tensor core does, replays the epilogue lane by lane, and checks dx against
torch.nn.grad.conv2d_input in float64, every read inside its region.
"""
import numpy as np
import torch

KPW = 18
PATCH_ALLOC = 43008                      # kPatchAlloc: the dy patch and its slack rows
DGRAD_B = 25 * 16 * 128                  # L2BwdSmem::kB: Bd[tap][16 ci][128 B = 32 co], 2048 B per tap
SMEM_WORDS = (PATCH_ALLOC + DGRAD_B) // 4
EDGE_SLOTS, EDGE_SLOT = 9, 10 * 16       # L2BwdSmem::kDxEdgeBytes = 9 slots × [10][16] floats


def sw128(addr):
    """SWIZZLE_128B: the 16-byte chunk index (address bits 4..6) XORed with the 128-byte row index mod 8 (bits 7..9)."""
    return addr ^ (((addr >> 7) & 7) << 4)


def sw128_off(row, chunk16):
    return row * 128 + ((chunk16 ^ (row & 7)) << 4)


def build_smem(dy, w):
    """The kernel's writes: the patch zeroed whole, then dy[oh][ow][c] at row (oh + 2)·18 + ow + 2; Bd[tap][ci][co] = w[co][ci][24 − tap]
    behind it."""
    img = np.full(SMEM_WORDS, np.nan)
    img[:PATCH_ALLOC // 4] = 0.0
    for oh in range(14):
        for ow in range(14):
            P = (oh + 2) * KPW + ow + 2
            for c in range(32):
                img[(sw128_off(P, c >> 2) + (c & 3) * 4) // 4] = dy[oh, ow, c]
    wf = w.reshape(32, 16, 25)
    for co in range(32):
        for ci in range(16):
            dst = PATCH_ALLOC + sw128_off(ci, co >> 2) + (co & 3) * 4
            for tap in range(25):
                img[(dst + (24 - tap) * 2048) // 4] = wf[co, ci, tap]
    return img


def kmajor_sw128(start, rows):
    """Word index of element (row, k) of a K-major SWIZZLE_128B operand (SBO = 1024: 128-byte rows) and one K = 8 step."""
    m = np.arange(rows)[:, None]
    k = np.arange(8)[None, :]
    return sw128(start + m * 128 + k * 4) // 4


def dprime_tile(img, tile, reach):
    """The 20 wgmma m64n80k8 of M tile `tile` (patch rows 64·tile ..): D' rows [64][80], with the byte ranges read recorded."""
    acc = np.zeros((64, 80))
    for kh in range(5):
        for k in range(4):
            ai = kmajor_sw128((64 * tile + KPW * kh) * 128 + k * 32, 64)
            bi = kmajor_sw128(PATCH_ALLOC + kh * 10240 + k * 32, 80)
            reach["a"] = max(reach["a"], 4 * int(ai.max()) + 4)
            reach["b_lo"] = min(reach["b_lo"], 4 * int(bi.min()))
            reach["b_hi"] = max(reach["b_hi"], 4 * int(bi.max()) + 4)
            acc += img[ai] @ img[bi].T
    return acc


def frag(acc, wq, lane):
    """The 40 accumulator elements of lane `lane` of warp wq: element e is D[16·wq + lane/4 + 8·((e >> 1) & 1)][8·(e >> 2) + 2·(lane % 4) + (e & 1)]."""
    g, t4 = lane >> 2, lane & 3
    return [acc[16 * wq + g + 8 * ((e >> 1) & 1), 8 * (e >> 2) + 2 * t4 + (e & 1)] for e in range(40)]


def edge_slot(r):
    return (r + 1) % 9


def edge_store(a, edge, r, lane):
    s, t4 = lane >> 2, lane & 3
    if s >= 4:
        return
    for kw in range(1, 5):
        if kw > s:
            for cg in range(2):
                e = 4 * (2 * kw + cg)
                base = edge_slot(r) * EDGE_SLOT + (kw * (kw - 1) // 2 + s) * 16 + 8 * cg + 2 * t4
                edge[base], edge[base + 1] = a[e], a[e + 1]


def epilogue(frags, edge, dx, written, r):
    """l2_dgrad_epilogue for the 32 lanes of range r (frags[lane] = that lane's 40 elements), shuffles as reads of the source lane."""
    for lane in range(32):
        g, t4 = lane >> 2, lane & 3
        a = frags[lane]
        o = [[[a[4 * cg + 2 * hh + b] for b in range(2)] for cg in range(2)] for hh in range(2)]
        for kw in range(1, 5):
            src = 4 * ((g + kw) & 7) + t4
            sa = frags[src]
            send_upper = (src >> 2) < kw
            take_next = g + kw >= 8
            for cg in range(2):
                for b in range(2):
                    e = 4 * (2 * kw + cg) + b
                    lo = sa[e + 2] if send_upper else sa[e]
                    hi = sa[e + 2]
                    o[0][cg][b] += lo
                    if not take_next:
                        o[1][cg][b] += hi
                    elif r < 15:
                        o[1][cg][b] += edge[edge_slot(r + 1) * EDGE_SLOT + (kw * (kw - 1) // 2 + g + kw - 8) * 16 + 8 * cg + 2 * t4 + b]
        for hh in range(2):
            p = 16 * r + g + 8 * hh
            oh, ow = divmod(p, KPW)
            if oh < 14 and ow < 14:
                for cg in range(2):
                    for b in range(2):
                        ci = 8 * cg + 2 * t4 + b
                        assert not written[oh, ow, ci], "two lanes store one dx element"
                        written[oh, ow, ci] = True
                        dx[oh, ow, ci] = o[hh][cg][b]


def dgrad_image(dy, w):
    img = build_smem(dy, w)
    reach = {"a": 0, "b_lo": 1 << 30, "b_hi": 0}
    edge = np.full(EDGE_SLOTS * EDGE_SLOT, np.nan)
    dx = np.full((14, 14, 16), np.nan)
    written = np.zeros((14, 14, 16), dtype=bool)
    for t0 in (2, 0):   # the kernel's two passes: tiles 2, 3, then 0, 1
        accs = {t0 + h: dprime_tile(img, t0 + h, reach) for h in range(2)}
        frags = {4 * t + wq: [frag(accs[t], wq, lane) for lane in range(32)] for t in accs for wq in range(4)}
        for r, fr in frags.items():
            for lane in range(32):
                edge_store(fr[lane], edge, r, lane)
        for r, fr in frags.items():
            epilogue(fr, edge, dx, written, r)
    return dx, written, reach


def test_dgrad_descriptors_and_epilogue_match_conv2d_input():
    g = torch.Generator().manual_seed(0)
    B = 2
    dy = torch.randn(B, 14, 14, 32, dtype=torch.float64, generator=g)
    w = torch.randn(32, 16, 5, 5, dtype=torch.float64, generator=g)
    want = torch.nn.grad.conv2d_input((B, 16, 14, 14), w, dy.permute(0, 3, 1, 2), padding=2).permute(0, 2, 3, 1).numpy()
    for n in range(B):
        dx, written, reach = dgrad_image(dy[n].numpy(), w.numpy())
        assert written.all(), "a dx element was never stored"
        assert np.isfinite(dx).all(), "an output met memory nobody wrote"
        # A reads rows up to 255 + 4·18 = 327 of the patch; B stays in the weight tiles
        assert reach["a"] == (255 + 4 * KPW) * 128 + 128 <= PATCH_ALLOC
        assert PATCH_ALLOC <= reach["b_lo"] and reach["b_hi"] <= PATCH_ALLOC + DGRAD_B
        assert np.abs(dx - want[n]).max() < 1e-10


def test_edge_slots():
    """The second pass overwrites only slots the first has finished reading, and range 7 still finds range 8's rows."""
    first_written = {edge_slot(r) for r in range(8, 16)}
    first_read = {edge_slot(r + 1) for r in range(8, 15)}
    second_written = {edge_slot(r) for r in range(0, 8)}
    assert first_written == set(range(0, 8)) and second_written == set(range(1, 9))
    assert edge_slot(8) in first_written and edge_slot(8) not in second_written
    assert first_read <= first_written and max(first_written | second_written) < EDGE_SLOTS


def test_shared_memory_placement():
    # L2BwdSmem: the FC form's end, the WG form's operands, the edge buffer behind dyᵀ
    x_t = PATCH_ALLOC + DGRAD_B + 4096
    x_bytes, dyt_bytes = 92160, 64 * 512
    total_fc = 1024 + PATCH_ALLOC + DGRAD_B + 4096 + 16 * 1568 * 4 + 2 * 160 * 16 * 4
    dx_edge = x_t + x_bytes + dyt_bytes
    total = 1024 + dx_edge + EDGE_SLOTS * EDGE_SLOT * 4
    assert dx_edge >= total_fc - 1024 and total == 230016 <= 227 * 1024
