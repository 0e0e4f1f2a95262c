"""The NVLink collective kernels (symm_kernels.cu) against float64 on one GPU, with the other ranks emulated.

``SymmComm`` skips the kernels in a world of one, so ``_C._SymmEmu`` launches them directly as rank r of a world of W: the W
"heaps" are plain device buffers laid out like the symmetric heap (flag pads, then data) and the kernel's ``peer[q]`` points at
heap q.  Before every launch the test stages, in rank r's heap, what the other ranks would have put there (their data, and in
rank r's flag rows an epoch 64 ahead of rank r's, so that no barrier can wait); one kernel runs at a time, on one stream.  Rank
r's result is then checked against "every other rank exact", and so is everything it wrote into the other heaps.

From the flag rows of the other heaps each launch also yields the grid size and the number of barriers per block.  Both must be
the same for every rank of a world (a rank with another grid or barrier count would deadlock a real run), and rank r's
``epochs[b]`` must advance by exactly that count.

Tolerances are first-order rounding bounds, with u = 2⁻²⁴ (fp32) or 2⁻⁵³ (fp64) for the accumulator type.  Floating-point
reductions must also equal, bit for bit, a CPU replay of the kernel's arithmetic: the accumulator type, rank order 0…W−1, then
× the scale converted once to the accumulator type, then one rounding to the element type."""
import pytest
import torch

import pytorch_distributed_train_b200 as pdt

pytestmark = pytest.mark.gpu

C = pdt._C
MAXB = C._symm_max_blocks
MAXW = C._symm_max_world
PAD = C._symm_flag_pad_bytes        # the flag pads of every channel; the data region follows
P2P_BLOCKS = C._symm_p2p_blocks
P2P_ACK_ROW = 80                    # kP2PAckRow (symm_kernels.cu): the rows of the p2p acknowledgements
CHANNEL = 2                         # kChanAux
TIMEOUT_NS = 3_000_000_000          # a kernel that waits anyway traps after 3 s and leaves its code in the status word
AHEAD = 64                          # the other ranks' flags are this far ahead of rank r's epoch
WORLDS = (2, 3, 5, 8)

EPS = 2.0 ** -24
U64 = 2.0 ** -53

SD = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 3, torch.int8: 4, torch.uint8: 5, torch.int32: 6,
      torch.int64: 7, torch.bool: 8, torch.int16: 9}
SUM, AVG, PROD, MIN, MAX, BAND, BOR, BXOR = range(8)
OPNAME = {SUM: "sum", AVG: "avg", PROD: "prod", MIN: "min", MAX: "max", BAND: "band", BOR: "bor", BXOR: "bxor"}
FLOATS = (torch.float32, torch.float64, torch.float16, torch.bfloat16)
ACC = {torch.float16: torch.float32, torch.bfloat16: torch.float32}
UNIT = {torch.float32: EPS, torch.float64: U64}
# op_supported (symm_kernels.cu): SUM for every type, PROD/MIN/MAX for the 32/64-bit ones, the bitwise ops for i32, i64 and u8
GRID = ([(dt, SUM) for dt in (torch.float32, torch.float64, torch.float16, torch.bfloat16, torch.int8, torch.uint8, torch.int16,
                              torch.int32, torch.int64)] +
        [(dt, op) for op in (PROD, MIN, MAX) for dt in (torch.float32, torch.float64, torch.int32, torch.int64)] +
        [(dt, op) for op in (BAND, BOR, BXOR) for dt in (torch.int32, torch.int64, torch.uint8)])
# bool: SUM and MAX are logical OR, PRODUCT and MIN logical AND (what torch's NCCL backend does), BXOR is XOR
BOOL_OPS = (SUM, PROD, MIN, MAX, BAND, BOR, BXOR)


def dev():
    return torch.device("cuda", 0)


def _id(v):
    return str(v).replace("torch.", "") if isinstance(v, torch.dtype) else OPNAME.get(v, str(v))


def _wrap32(t):
    """int64 → the int32 with the same low 32 bits."""
    return ((t + 2 ** 31) % 2 ** 32 - 2 ** 31).to(torch.int32)


def _diff32(a, b):
    """(a − b) mod 2³² of two int32 tensors, as int64."""
    return (a.long() - b.long()) % 2 ** 32


# ---- the emulated world ---------------------------------------------------------------------------------------------------------
class World:
    """W heaps (flag pads + `data_bytes`), each emulated rank's epochs, one status word."""

    def __init__(self, W, data_bytes, epoch0=0):
        self.W = W
        self.heaps = [torch.zeros(PAD + data_bytes, dtype=torch.uint8, device=dev()) for _ in range(W)]
        self.epochs = [_wrap32(torch.full((MAXB,), epoch0, dtype=torch.int64, device=dev())) for _ in range(W)]
        self.status = torch.zeros(1, dtype=torch.int32, device=dev())
        self.shapes = []     # (grid, barriers per block) of every launch

    def flags(self, q):
        """Heap q's flag rows of the channel: [block, writer rank]."""
        off = CHANNEL * MAXB * MAXW * 4
        return self.heaps[q][off:off + MAXB * MAXW * 4].view(torch.int32).view(MAXB, MAXW)

    def bytes(self, q, off, n):
        return self.heaps[q][PAD + off:PAD + off + n]

    def typed(self, q, off, dtype, n):
        es = torch.empty(0, dtype=dtype).element_size()
        return self.bytes(q, off, n * es).view(dtype)

    def launch(self, r, call):
        """Run `call(emu)` as rank r with every barrier pre-satisfied; return (grid, barriers per block) read back from the flag
        rows rank r wrote into the other heaps, after checking them against rank r's epochs."""
        base = self.epochs[r].clone()
        ahead = _wrap32(base.long() + AHEAD)
        for q in range(self.W):
            if q != r:
                self.flags(r)[:, q] = ahead    # rank q has passed every barrier rank r may meet
                self.flags(q)[:, r] = base     # rank r's signals to q: still the old epoch
        emu = C._SymmEmu(self.heaps, r, CHANNEL, TIMEOUT_NS, self.epochs[r], self.status)
        call(emu)
        torch.cuda.synchronize()
        assert int(self.status.item()) == 0, f"status word {int(self.status.item()):#x}"
        sig = [_diff32(self.flags(q)[:, r], base) for q in range(self.W) if q != r]
        for s in sig[1:]:
            assert torch.equal(s, sig[0]), "rank r signalled its peers unevenly"
        s = sig[0].cpu()
        grid = int((s > 0).sum())
        assert grid >= 1 and bool((s[:grid] > 0).all()) and bool((s[grid:] == 0).all()), s[:grid + 2].tolist()
        n = int(s[0])
        assert bool((s[:grid] == n).all()), ("blocks ran different barrier counts", s[:grid].tolist())
        adv = _diff32(self.epochs[r], base).cpu()
        assert bool((adv[:grid] == n).all()) and bool((adv[grid:] == 0).all()), ("epochs advanced unevenly", adv[:grid + 2].tolist(), n)
        self.shapes.append((grid, n))
        return grid, n


def _same_shape(shapes, what):
    assert len(set(shapes)) == 1, (what, "grid / barrier count differs across ranks", shapes)
    return shapes[0]


# ---- inputs and the replay of the kernel's arithmetic ---------------------------------------------------------------------------
def _inputs(dtype, op, W, n, gen, nan_rank=None):
    xs = []
    for q in range(W):
        if dtype == torch.bool:
            x = torch.randint(0, 2, (n,), generator=gen).bool()
            if n:
                x[0] = q != 0         # a mix of all-true, all-false and mixed columns at every length
        elif dtype in FLOATS:
            if op == PROD:            # |x| in [0.5, 2): eight factors stay far from overflow and underflow
                x = (torch.rand(n, generator=gen, dtype=torch.float64) * 1.5 + 0.5) * (torch.randint(0, 2, (n,), generator=gen) * 2 - 1)
            else:
                x = torch.randn(n, generator=gen, dtype=torch.float64) * 3
            x = x.to(dtype)
            if nan_rank == q:
                x[::3] = float("nan")
        else:
            info = torch.iinfo(dtype)
            lo, hi = (info.min, info.max) if dtype != torch.int64 else (-2 ** 62, 2 ** 62)
            if op == PROD:
                lo, hi = max(lo, -2 ** 12), min(hi, 2 ** 12)
            x = torch.randint(lo, hi, (n,), generator=gen, dtype=torch.int64).to(dtype)   # sums of eight wrap around
        xs.append(x)
    return xs


def _combine(a, b, op):
    if op in (SUM, AVG):
        return a + b
    if op == PROD:
        return a * b
    if op == MIN:
        return torch.minimum(a, b)
    if op == MAX:
        return torch.maximum(a, b)
    if op == BAND:
        return a & b
    if op == BOR:
        return a | b
    return a ^ b


def _replay(xs, dtype, op, scale):
    """The kernel's arithmetic on the CPU: accumulator type, rank order, × fl_acc(scale), one rounding."""
    if dtype == torch.bool:
        bop = {SUM: BOR, MAX: BOR, BOR: BOR, PROD: BAND, MIN: BAND, BAND: BAND, BXOR: BXOR}[op]
        a = xs[0].clone()
        for x in xs[1:]:
            a = _combine(a, x, bop)
        return a
    acc = ACC.get(dtype, dtype)
    a = xs[0].to(acc)
    for x in xs[1:]:
        a = _combine(a, x.to(acc), op)
    if dtype in FLOATS:
        a = a * torch.tensor(scale, dtype=acc)
    return a.to(dtype)


def _bits(t):
    """A tensor's bytes, so that equality is bitwise (−0, bool bytes other than 0 and 1).  Every NaN becomes the same NaN first:
    torch's CPU minimum / maximum return their own NaN, the kernels the input's."""
    if t.is_floating_point():
        t = torch.where(torch.isnan(t), torch.full_like(t, float("nan")), t)
    return t.contiguous().view(torch.uint8)


def _check_float64(got, xs, dtype, op, scale, W, what):
    """fp32 / fp64 SUM and PROD within the first-order bound of the float64 result.  SUM: each of the W−1 additions rounds
    relative to a partial sum ≤ Σ|x|, fl_acc(scale) is off by ≤ u·|s| and the product rounds once, so |err| ≤ (W+1)·u·|s|·Σ|x|.
    PROD: W−1 products, the scale and the final product round, each relative to the result: (W+1)·u·|s·Πx|.  The float64
    reference carries its own ≤ W·u₆₄ of the same magnitudes."""
    if dtype not in UNIT or op not in (SUM, PROD):
        return
    x64 = torch.stack([x.double() for x in xs])
    if op == SUM:
        ref, mag = x64.sum(0) * scale, x64.abs().sum(0) * abs(scale)
    else:
        ref = x64.prod(0) * scale
        mag = ref.abs()
    tol = ((W + 1) * UNIT[dtype] + W * U64) * mag
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)
    assert not bool(bad.any()), (what, int(bad.sum()), (err / tol.clamp_min(1e-300)).max().item())


def _scales(dtype, W):
    return (1.0, 1.0 / W, 0.37) if dtype in FLOATS else (1.0,)


def _es(dtype):
    return torch.empty(0, dtype=dtype).element_size()


# ---- one-shot push allreduce ----------------------------------------------------------------------------------------------------
def _oneshot_world(W, dtype, op, nvec, scales, seed, blocks=0, threads=0, inplace=True, nan_rank=None, epoch0=0):
    """Every rank r of a world of W: stage the other ranks' slots in heap r, push + reduce, check the output, the slot r of every
    heap, and that all ranks agree bit for bit and on the launch shape."""
    es = _es(dtype)
    count = nvec * 16 // es
    slot = nvec * 16
    w = World(W, W * slot, epoch0)
    gen = torch.Generator().manual_seed(seed)
    for scale in scales:
        xs = _inputs(dtype, op, W, count, gen, nan_rank)
        exp = _replay(xs, dtype, op, scale)
        xg = [x.to(dev()) for x in xs]
        outs, shapes = [], []
        for r in range(W):
            for q in range(W):
                w.bytes(q, r * slot, slot).fill_(0xA5)                        # rank r's slot everywhere: poisoned
                if q != r:
                    w.typed(r, q * slot, dtype, count).copy_(xg[q])           # rank q's push into rank r's staging
            inp = xg[r].clone()
            out = inp if inplace else torch.full_like(inp, 7) if dtype != torch.bool else torch.ones_like(inp)
            shapes.append(w.launch(r, lambda e: e.oneshot(inp.data_ptr(), out.data_ptr(), PAD, count, SD[dtype], op, scale, blocks, threads)))
            for q in range(W):
                assert torch.equal(w.bytes(q, r * slot, slot), _bits(xg[r])), (r, q, "rank r's vector is not in slot r of heap q")
            if not inplace:
                assert torch.equal(inp, xg[r]), "the input was modified"
            outs.append(out.cpu())
        what = (W, _id(dtype), _id(op), scale, nvec)
        assert torch.equal(_bits(outs[0]), _bits(exp)), (what, "differs from the replay of the kernel's arithmetic")
        for r in range(1, W):
            assert torch.equal(_bits(outs[r]), _bits(outs[0])), (what, r, "ranks disagree")
        _check_float64(outs[0], xs, dtype, op, scale, W, what)
        _same_shape(shapes, what)
    return w


@pytest.mark.parametrize("dtype,op", GRID, ids=[f"{_id(d)}-{_id(o)}" for d, o in GRID])
@pytest.mark.parametrize("W", WORLDS)
def test_oneshot_dtype_op(W, dtype, op):
    _oneshot_world(W, dtype, op, 45, _scales(dtype, W), seed=W * 100 + SD[dtype] * 10 + op)


@pytest.mark.parametrize("op", BOOL_OPS, ids=[_id(o) for o in BOOL_OPS])
@pytest.mark.parametrize("W", WORLDS)
def test_oneshot_bool_is_logical(W, op):
    """bool results are 0 or 1: SUM/MAX are OR and PRODUCT/MIN are AND, never a byte count of the true ranks."""
    _oneshot_world(W, torch.bool, op, 3, (1.0,), seed=W)


@pytest.mark.parametrize("dtype", (torch.float32, torch.float64), ids=_id)
@pytest.mark.parametrize("op", (MIN, MAX), ids=_id)
@pytest.mark.parametrize("W", WORLDS)
def test_oneshot_nan_propagates_from_any_rank(W, op, dtype):
    """torch.minimum / torch.maximum semantics: a NaN at any rank gives NaN, so permuting inputs across ranks changes nothing."""
    for q in range(W):
        _oneshot_world(W, dtype, op, 6, (1.0,), seed=q, nan_rank=q)


@pytest.mark.parametrize("dtype", (torch.int32, torch.int64, torch.uint8, torch.bool), ids=_id)
def test_integer_scale_and_bool_avg_are_rejected(dtype):
    """A scale ≠ 1 (AVG's 1/W) has no integer result; no launcher may silently return the sum.  AVG on bool has none either."""
    w = World(2, 4096)
    buf = torch.zeros(64, dtype=dtype, device=dev())
    n = 64
    calls = [("scale", lambda e: e.oneshot(buf.data_ptr(), buf.data_ptr(), PAD, n, SD[dtype], SUM, 0.5)),
             ("scale", lambda e: e.twoshot(PAD, n, SD[dtype], SUM, 0.5)),
             ("scale", lambda e: e.reduce_pull(PAD, 0, 1, 2, buf.data_ptr(), SD[dtype], SUM, 0.5))]
    if dtype == torch.bool:
        calls.append(("bool", lambda e: e.oneshot(buf.data_ptr(), buf.data_ptr(), PAD, n, SD[dtype], AVG, 1.0)))
    for match, call in calls:
        with pytest.raises(ValueError, match=match):
            w.launch(0, call)        # staged like every launch, so that a launcher that does not refuse cannot make a kernel wait
    torch.cuda.synchronize()
    assert int(w.status.item()) == 0 and torch.equal(w.epochs[0], torch.zeros_like(w.epochs[0]))   # nothing was launched


# sizes around the auto grid: one-shot runs 256 threads, 2·256 vectors per block, at most 64 blocks (auto_blocks)
ONESHOT_NVEC = (1, 2, 3, 7, 511, 512, 513, 64 * 512 - 1, 64 * 512 + 1)
CFGS = ((0, 0), (1, 0), (160, 0), (200, 0), (0, 32), (0, 64), (0, 512))


@pytest.mark.parametrize("blocks,threads", CFGS, ids=[f"b{b}t{t}" for b, t in CFGS])
@pytest.mark.parametrize("nvec", ONESHOT_NVEC)
@pytest.mark.parametrize("W", WORLDS)
def test_oneshot_sizes_and_launch_shapes(W, nvec, blocks, threads):
    w = _oneshot_world(W, torch.float32, SUM, nvec, (1.0 / W,), seed=nvec, blocks=blocks, threads=threads, inplace=nvec % 2 == 0)
    grid, n = w.shapes[0]
    assert n == 1
    t = threads or 256
    want = min(blocks, MAXB) if blocks else max(1, min(-(-nvec // (2 * t)), 64))
    assert grid == want, (grid, want)


@pytest.mark.parametrize("W", WORLDS)
def test_oneshot_4mb(W):
    _oneshot_world(W, torch.float32, SUM, (4 << 20) // 16, (1.0 / W,), seed=W)


# ---- two-shot allreduce, in place -----------------------------------------------------------------------------------------------
def _twoshot_world(W, dtype, op, nvec, scales, seed, blocks=0, threads=0, epoch0=0, w=None):
    """Heap q ≠ r holds rank q's input, except that slice q already holds the reduced result (rank q's first phase); rank r must
    reduce its own slice out of every heap and gather the others, leaving the whole reduced vector in heap r."""
    es = _es(dtype)
    count = nvec * 16 // es
    per = -(-nvec // W) * 16 // es      # elements per slice
    w = w or World(W, nvec * 16, epoch0)
    gen = torch.Generator().manual_seed(seed)
    for scale in scales:
        xs = _inputs(dtype, op, W, count, gen)
        exp = _replay(xs, dtype, op, scale)
        xg, eg = [x.to(dev()) for x in xs], exp.to(dev())
        outs, shapes = [], []
        for r in range(W):
            for q in range(W):
                buf = w.typed(q, 0, dtype, count)
                buf.copy_(xg[q])
                if q != r:
                    buf[per * q:per * (q + 1)] = eg[per * q:per * (q + 1)]
            shapes.append(w.launch(r, lambda e: e.twoshot(PAD, count, SD[dtype], op, scale, blocks, threads)))
            outs.append(w.typed(r, 0, dtype, count).cpu())
        what = (W, _id(dtype), _id(op), scale, nvec)
        for r in range(W):
            assert torch.equal(_bits(outs[r]), _bits(exp)), (what, r, "differs from the replay of the kernel's arithmetic")
            sl = slice(per * r, per * (r + 1))
            _check_float64(outs[r][sl], [x[sl] for x in xs], dtype, op, scale, W, what)
        _same_shape(shapes, what)
    return w


@pytest.mark.parametrize("dtype,op", GRID + [(torch.bool, SUM), (torch.bool, PROD)],
                         ids=[f"{_id(d)}-{_id(o)}" for d, o in GRID + [(torch.bool, SUM), (torch.bool, PROD)]])
@pytest.mark.parametrize("W", WORLDS)
def test_twoshot_dtype_op(W, dtype, op):
    # nvec not divisible by W, and nvec < W (the last ranks own empty slices)
    for nvec in (3 * W + 1, W - 1):
        _twoshot_world(W, dtype, op, nvec, _scales(dtype, W), seed=W * 100 + SD[dtype] * 10 + op + nvec)


@pytest.mark.parametrize("blocks,threads", CFGS, ids=[f"b{b}t{t}" for b, t in CFGS])
@pytest.mark.parametrize("W", WORLDS)
def test_twoshot_sizes_and_launch_shapes(W, blocks, threads):
    for nvec in (1, 7, 2 * 512 * W - 1, 2 * 512 * W + 1, 5000):
        w = _twoshot_world(W, torch.float32, SUM, nvec, (1.0 / W,), seed=nvec, blocks=blocks, threads=threads)
        assert w.shapes[0][1] == 3
        if blocks:
            assert w.shapes[0][0] == min(blocks, MAXB)


# ---- reduce-scatter / rooted reduce ---------------------------------------------------------------------------------------------
RP_CASES = ((torch.float32, SUM), (torch.float64, SUM), (torch.bfloat16, SUM), (torch.int32, MAX), (torch.int64, BXOR),
            (torch.float32, MIN), (torch.bool, SUM))


@pytest.mark.parametrize("dtype,op", RP_CASES, ids=[f"{_id(d)}-{_id(o)}" for d, o in RP_CASES])
@pytest.mark.parametrize("W", WORLDS)
def test_reduce_pull(W, dtype, op):
    es = _es(dtype)
    for pvec, blocks, threads in ((5, 0, 0), (1, 0, 0), (300, 0, 64), (300, 3, 0)):
        total = pvec * W
        count = total * 16 // es
        w = World(W, total * 16)
        gen = torch.Generator().manual_seed(W * 7 + pvec)
        for scale in _scales(dtype, W):
            xs = _inputs(dtype, op, W, count, gen)
            exp = _replay(xs, dtype, op, scale)
            for q in range(W):
                w.typed(q, 0, dtype, count).copy_(xs[q].to(dev()))
            what = (W, _id(dtype), _id(op), scale, pvec)
            # reduce_scatter: rank r reduces slice r
            per = pvec * 16 // es
            shapes = []
            for r in range(W):
                out = torch.zeros(per, dtype=dtype, device=dev())
                shapes.append(w.launch(r, lambda e: e.reduce_pull(PAD, r * pvec, pvec, total, out.data_ptr(), SD[dtype], op, scale, blocks, threads)))
                assert torch.equal(_bits(out.cpu()), _bits(exp[per * r:per * (r + 1)])), (what, r, "reduce_scatter")
                _check_float64(out.cpu(), [x[per * r:per * (r + 1)] for x in xs], dtype, op, scale, W, what)
            _same_shape(shapes, what + ("reduce_scatter",))
            # reduce to every root: the root takes the whole vector, the others attend with count 0 and write nothing
            for root in range(W):
                shapes = []
                for r in range(W):
                    out = torch.full((count * es,), 0x5A, dtype=torch.uint8, device=dev()).view(dtype)
                    before = _bits(out).clone()
                    n = total if r == root else 0
                    shapes.append(w.launch(r, lambda e: e.reduce_pull(PAD, 0, n, total, out.data_ptr(), SD[dtype], op, scale, blocks, threads)))
                    if r == root:
                        assert torch.equal(_bits(out.cpu()), _bits(exp)), (what, root, "reduce")
                    else:
                        assert torch.equal(_bits(out), before), (what, root, r, "a non-root wrote its output")
                _same_shape(shapes, what + ("reduce", root))


# ---- pull kernel: broadcast / allgather / alltoall ------------------------------------------------------------------------------
# (nbytes, source offset, destination offset): 16-byte vectors with a 1–15 byte tail, 4-byte words at misaligned offsets,
# single bytes
PULL_SIZES = ((16, 0, 0), (1, 0, 0), (15, 0, 0), (16 * 5 + 1, 0, 0), (16 * 700 + 15, 0, 0), (16 * 9000 + 7, 0, 0),
              (20, 4, 0), (4 * 1001, 0, 8), (4 * 3, 12, 4), (13, 3, 0), (1001, 0, 1), (16 * 40, 1, 1), (7, 16, 5))


def _pull_world(W, nbytes, stride):
    w = World(W, W * stride + 64)
    gen = torch.Generator().manual_seed(nbytes)
    src = [torch.randint(0, 256, (W * stride + 64,), generator=gen, dtype=torch.uint8).to(dev()) for _ in range(W)]
    for q in range(W):
        w.bytes(q, 0, W * stride + 64).copy_(src[q])
    return w, src


@pytest.mark.parametrize("nbytes,soff,doff", PULL_SIZES)
@pytest.mark.parametrize("W", WORLDS)
def test_broadcast_pull(W, nbytes, soff, doff):
    w, src = _pull_world(W, nbytes, nbytes + soff)
    for exit_barrier in (True, False):
        for root in range(W):
            shapes = []
            for r in range(W):
                dst = torch.full((nbytes + doff + 32,), 0xEE, dtype=torch.uint8, device=dev())
                if r == root and doff == soff:   # in place at the root: the source is the destination, nothing moves
                    ptr = w.heaps[root].data_ptr() + PAD + soff
                else:
                    ptr = dst.data_ptr() + doff
                shapes.append(w.launch(r, lambda e: e.broadcast(PAD + soff, ptr, nbytes, root, exit_barrier, 0, 64 if nbytes < 64 else 0)))
                if ptr == dst.data_ptr() + doff:
                    assert torch.equal(dst[doff:doff + nbytes], src[root][soff:soff + nbytes]), (W, root, r, nbytes, soff, doff)
                    assert bool((dst[:doff] == 0xEE).all()) and bool((dst[doff + nbytes:] == 0xEE).all()), "wrote outside dst"
                assert torch.equal(w.bytes(root, 0, src[root].numel()), src[root]), "the root's source changed"
            _same_shape(shapes, (W, nbytes, root, exit_barrier))
            assert shapes[0][1] == (2 if exit_barrier else 1)


@pytest.mark.parametrize("nbytes,soff,doff", PULL_SIZES)
@pytest.mark.parametrize("W", WORLDS)
def test_allgather_and_gather_pull(W, nbytes, soff, doff):
    """allgather into a dst_stride layout; a gather, where only the root pulls and the others attend with dst = nullptr."""
    for dst_stride in (nbytes, nbytes + 3):
        w, src = _pull_world(W, nbytes, nbytes + soff)
        for root in (None,) + tuple(range(W)):
            for exit_barrier in (True, False):
                shapes = []
                for r in range(W):
                    pulls = root is None or r == root
                    dst = torch.full((W * dst_stride + doff + 32,), 0xEE, dtype=torch.uint8, device=dev())
                    ptr = dst.data_ptr() + doff if pulls else 0
                    shapes.append(w.launch(r, lambda e: e.allgather(PAD + soff, ptr, nbytes, dst_stride, exit_barrier)))
                    if pulls:
                        for q in range(W):
                            got = dst[doff + q * dst_stride:doff + q * dst_stride + nbytes]
                            assert torch.equal(got, src[q][soff:soff + nbytes]), (W, root, r, q, nbytes, soff, doff, dst_stride)
                        assert bool((dst[:doff] == 0xEE).all()) and bool((dst[doff + (W - 1) * dst_stride + nbytes:] == 0xEE).all())
                    else:
                        assert bool((dst == 0xEE).all())
                _same_shape(shapes, (W, nbytes, root, exit_barrier))
                assert shapes[0][1] == (2 if exit_barrier else 1)


@pytest.mark.parametrize("nbytes,soff,doff", PULL_SIZES)
@pytest.mark.parametrize("W", WORLDS)
def test_alltoall_pull(W, nbytes, soff, doff):
    for stride in (nbytes, nbytes + 5):
        w, src = _pull_world(W, nbytes, stride + soff)
        shapes = []
        for r in range(W):
            dst = torch.full((W * stride + doff + 32,), 0xEE, dtype=torch.uint8, device=dev())
            shapes.append(w.launch(r, lambda e: e.alltoall(PAD + soff, dst.data_ptr() + doff, nbytes, stride, False)))
            for q in range(W):
                got = dst[doff + q * stride:doff + q * stride + nbytes]
                assert torch.equal(got, src[q][soff + r * stride:soff + r * stride + nbytes]), (W, r, q, nbytes, soff, doff, stride)
        _same_shape(shapes, (W, nbytes, stride))


@pytest.mark.parametrize("blocks,threads", CFGS, ids=[f"b{b}t{t}" for b, t in CFGS])
def test_pull_launch_shapes(blocks, threads):
    W = 3
    for nbytes in (1, 16 * 1023 + 9, 16 * 300000 + 5):
        w, src = _pull_world(W, nbytes, nbytes)
        shapes = []
        for r in range(W):
            dst = torch.zeros(nbytes, dtype=torch.uint8, device=dev())
            shapes.append(w.launch(r, lambda e: e.broadcast(PAD, dst.data_ptr(), nbytes, 1, True, blocks, threads)))
            assert torch.equal(dst, src[1][:nbytes])
        grid, _ = _same_shape(shapes, (nbytes, blocks, threads))
        if blocks:
            assert grid == min(blocks, MAXB)


# ---- fused allreduce + SGD (+ broadcast rider) ----------------------------------------------------------------------------------
def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _sgd64(g, p, b, lr, mom, damp, wd, nesterov, first, absval=False):
    """torch.optim.SGD's step in float64 on the averaged gradient g.  absval: the same chain on magnitudes (every term added),
    which bounds each intermediate's magnitude for the rounding bound."""
    f = (lambda t: t.abs()) if absval else (lambda t: t)
    sgn = 1.0 if absval else -1.0
    k = abs(1.0 - damp) if absval else 1.0 - damp
    g, p = f(g), f(p)
    if wd:
        g = g + wd * p
    if mom:
        b = g if first else mom * f(b) + k * g
        g = g + mom * b if nesterov else b
    return p + sgn * lr * g, b


SGD_CASES = [
    dict(momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, first_step=False),
    dict(momentum=0.0, dampening=0.0, weight_decay=1e-2, nesterov=False, first_step=False),
    dict(momentum=0.9, dampening=0.0, weight_decay=0.0, nesterov=False, first_step=True),
    dict(momentum=0.9, dampening=0.5, weight_decay=0.0, nesterov=False, first_step=True),
    dict(momentum=0.9, dampening=0.5, weight_decay=5e-4, nesterov=False, first_step=False),
    dict(momentum=0.9, dampening=0.0, weight_decay=1e-2, nesterov=True, first_step=False),
    dict(momentum=0.8, dampening=0.0, weight_decay=0.0, nesterov=True, first_step=True),
]


@pytest.mark.parametrize("lr_on_device", (False, True), ids=("lr_host", "lr_dev"))
@pytest.mark.parametrize("case", range(len(SGD_CASES)))
@pytest.mark.parametrize("W", WORLDS)
def test_allreduce_sgd(W, case, lr_on_device):
    h = {k: (_f32(v) if isinstance(v, float) else v) for k, v in SGD_CASES[case].items()}
    lr = _f32(0.05)
    scale = _f32(1.0 / W)          # what SymmComm passes: 1.0f / world
    for nvec, blocks, bc_vec in ((300, 0, 0), (3, 0, 5), (1100, 1, 2), (2049, 0, 0)):
        count = 4 * nvec
        slot = count * 4
        w = World(W, W * slot + bc_vec * 16)
        gen = torch.Generator().manual_seed(W * 1000 + case * 10 + nvec)
        gs = [torch.randn(count, generator=gen) for _ in range(W)]
        p0 = torch.randn(count, generator=gen)
        b0 = torch.randn(count, generator=gen)
        payload = [torch.randint(0, 256, (bc_vec * 16,), generator=gen, dtype=torch.uint8) for _ in range(W)]
        bc_root = (case + nvec) % W
        g64 = torch.stack([g.double() for g in gs]).sum(0) * scale
        gmag = torch.stack([g.double().abs() for g in gs]).sum(0) * scale
        hyper = (lr, h["momentum"], h["dampening"], h["weight_decay"], h["nesterov"], h["first_step"])
        p_ref, b_ref = _sgd64(g64, p0.double(), b0.double(), *hyper)
        p_mag, b_mag = _sgd64(gmag, p0.double(), b0.double(), *hyper, absval=True)
        # W−1 additions and the scale round the averaged gradient (≤ W·ε of its magnitude); weight decay, the momentum update
        # (with fl(1 − dampening)), nesterov and the parameter update add at most 9 roundings, each ≤ ε of an intermediate whose
        # magnitude, carried to the output, is bounded by the magnitude chain: |err| ≤ (W + 9)·ε·magnitude
        k = (W + 9) * EPS
        lr_t = torch.tensor([lr], device=dev())
        shapes = []
        for r in range(W):
            for q in range(W):
                w.bytes(q, r * slot, slot).fill_(0xA5)
                if q != r:
                    w.typed(r, q * slot, torch.float32, count).copy_(gs[q].to(dev()))
            if bc_vec:
                w.bytes(r, W * slot, bc_vec * 16).copy_(payload[bc_root].to(dev()) if r != bc_root else torch.zeros(bc_vec * 16, dtype=torch.uint8, device=dev()))
            grad, param, mbuf = gs[r].to(dev()), p0.to(dev()), b0.to(dev())
            bc = payload[r].to(dev())
            mom_ptr = mbuf.data_ptr() if h["momentum"] else 0
            shapes.append(w.launch(r, lambda e: e.allreduce_sgd(
                grad.data_ptr(), param.data_ptr(), mom_ptr, PAD, count, scale, lr_t.data_ptr() if lr_on_device else 0,
                -1.0 if lr_on_device else lr, h["momentum"], h["dampening"], h["weight_decay"], h["nesterov"], h["first_step"],
                bc.data_ptr() if bc_vec else 0, bc_vec * 16, bc_root, blocks, 0)))
            what = (W, case, r, nvec)
            err = (grad.double().cpu() - g64).abs()
            assert bool((err <= W * EPS * gmag).all()), (what, "grad is not the averaged gradient")
            err = (param.double().cpu() - p_ref).abs()
            assert bool((err <= k * p_mag).all()), (what, "param", (err / (k * p_mag).clamp_min(1e-300)).max().item())
            if h["momentum"]:
                err = (mbuf.double().cpu() - b_ref).abs()
                assert bool((err <= k * b_mag).all()), (what, "momentum buffer", (err / (k * b_mag).clamp_min(1e-300)).max().item())
            else:
                assert torch.equal(mbuf.cpu(), b0)
            for q in range(W):
                assert torch.equal(w.typed(q, r * slot, torch.float32, count).cpu(), gs[r]), (what, q, "pushed gradient")
            if bc_vec:
                assert torch.equal(bc.cpu(), payload[bc_root]), (what, "broadcast rider")
                if r == bc_root:
                    for q in range(W):
                        assert torch.equal(w.bytes(q, W * slot, bc_vec * 16).cpu(), payload[bc_root]), (what, q, "rider not pushed")
        _same_shape(shapes, (W, case, nvec))
        assert shapes[0][1] == 1


# ---- point-to-point -------------------------------------------------------------------------------------------------------------
P2P_SIZES = ((1, 0), (15, 0), (16, 0), (16 * 7 + 9, 0), (16 * 513 + 3, 0), (16 * 100, 1), (16 * 33 + 5, 4), (1000, 3))


@pytest.mark.parametrize("seq", (1, 0x80000005))
@pytest.mark.parametrize("nbytes,mis", P2P_SIZES)
@pytest.mark.parametrize("W", (2, 5))
def test_p2p_send_recv(W, nbytes, mis, seq):
    slot = (nbytes + 16 + 255) // 256 * 256
    w = World(W, W * slot)
    gen = torch.Generator().manual_seed(nbytes)
    payload = torch.randint(0, 256, (nbytes,), generator=gen, dtype=torch.uint8).to(dev())
    before = _wrap32(torch.tensor(seq - 1, dtype=torch.int64)).item()
    for r in range(W):
        for peer in range(W):
            if peer == r:
                continue
            # send r → peer: the previous chunk has been acknowledged; the message lands in slot r of peer's heap, ready = seq
            src = torch.zeros(nbytes + 16, dtype=torch.uint8, device=dev())
            src[mis:mis + nbytes] = payload
            w.flags(r)[P2P_ACK_ROW:P2P_ACK_ROW + P2P_BLOCKS, peer] = before
            w.flags(peer)[:P2P_BLOCKS, r] = before
            w.bytes(peer, r * slot, slot).fill_(0xEE)
            emu = C._SymmEmu(w.heaps, r, CHANNEL, TIMEOUT_NS, w.epochs[r], w.status)
            emu.p2p_send(src.data_ptr() + mis, nbytes, peer, PAD + r * slot, seq)
            torch.cuda.synchronize()
            assert int(w.status.item()) == 0
            assert torch.equal(w.bytes(peer, r * slot, nbytes), payload), (W, r, peer, nbytes, mis, "send payload")
            assert bool((w.bytes(peer, r * slot + nbytes, slot - nbytes) == 0xEE).all()), "send wrote past the message"
            assert bool((w.flags(peer)[:P2P_BLOCKS, r] == _wrap32(torch.tensor(seq))).all()), "ready flags"
            # recv peer → r: the chunk is in slot peer of r's heap with ready = seq; r copies it out and acknowledges with ack = seq
            w.flags(r)[:P2P_BLOCKS, peer] = _wrap32(torch.tensor(seq))
            w.flags(peer)[P2P_ACK_ROW:P2P_ACK_ROW + P2P_BLOCKS, r] = before
            w.bytes(r, peer * slot, nbytes).copy_(payload)
            dst = torch.full((nbytes + 32,), 0xEE, dtype=torch.uint8, device=dev())
            emu.p2p_recv(dst.data_ptr() + mis, nbytes, peer, PAD + peer * slot, seq)
            torch.cuda.synchronize()
            assert int(w.status.item()) == 0
            assert torch.equal(dst[mis:mis + nbytes], payload), (W, r, peer, nbytes, mis, "recv payload")
            assert bool((dst[:mis] == 0xEE).all()) and bool((dst[mis + nbytes:] == 0xEE).all()), "recv wrote outside dst"
            assert bool((w.flags(peer)[P2P_ACK_ROW:P2P_ACK_ROW + P2P_BLOCKS, r] == _wrap32(torch.tensor(seq))).all()), "ack flags"
    assert all(bool((e == 0).all()) for e in w.epochs), "p2p kernels do not touch the barrier epochs"


# ---- barrier, and epochs that wrap past 2³² -------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", WORLDS)
def test_barrier(W):
    w = World(W, 16)
    shapes = [w.launch(r, lambda e: e.barrier()) for r in range(W)]
    assert _same_shape(shapes, W) == (1, 1)


@pytest.mark.parametrize("W", WORLDS)
def test_epochs_wrap_past_2_32(W):
    """Start every block at epoch 0xFFFFFFF0: after a few launches the epochs (and the flags) wrap, and the signed comparison
    must keep every barrier satisfied."""
    w = _twoshot_world(W, torch.float32, SUM, 4 * W + 3, (1.0, 1.0 / W, 0.37), seed=W, epoch0=0xFFFFFFF0)
    for _ in range(3):
        _twoshot_world(W, torch.float32, SUM, 4 * W + 3, (1.0 / W,), seed=W, w=w)
    assert all(bool((e[:w.shapes[0][0]] >= 0).all()) for e in w.epochs), "the epochs did not wrap"
