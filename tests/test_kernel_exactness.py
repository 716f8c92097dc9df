"""Exactness of the masked-convolution, bias-gradient and BatchNorm kernels at training extents, against float64.

Operands are chosen so that the exact result is known and a bf16 / fp32 kernel must reproduce it bit for bit:
activations and output gradients are integers (x, dy in {-1, 0, 1}; integers in [-64, 64] for the rounding cases) and
masked weights are in {-1, 0, 1} * 2^e.  Every product is then exact, and every fp32 partial sum of an output element is
an exact multiple of its quantum in any summation order, split-K partition or tensor-core accumulation that keeps 24
significand bits, as long as S = sum |a| * |b| over that element's terms stays below 2^24 quanta.  Each check asserts
S <= 2^22 quanta for every element first (S is the same convolution of the absolute operands, in float64).

The reference is torch's convolution and its two gradients in float64 on the GPU, from the same operands, rounded to
the quantum: that is the exact value.  bf16 outputs must equal it rounded to nearest-even, fp32 weight and bias
gradients must equal it, masked weights get exactly zero.  Values are compared as numbers (the sign of a zero is not
compared).  A mismatch is a bug, not a tolerance question: the failure lists S and the difference at the first elements.

Every case asserts the kernel path it exists for (wgrad split count, split lanes of the finalize, K blocks per split,
length of the last split, fprop items per CTA), computed by a mirror of the host code, so that no case silently
degrades to a one-block or one-split walk.  The BatchNorm statistics and the fused BatchNorm-backward epilogue are
checked the same way where the arithmetic is exact, and against stated bars where it is not (see each test)."""
import ctypes
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from test_fwd_pingpong import _fprop_items, _sms

H100_SMS = 132              # the wgrad plans in the case tables are the ones a 132-SM H100 runs
EXACT = 2.0 ** 22           # largest S (in quanta) an exactness check accepts


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: the gpu-marked tests need an H100")
    from turboprune_b200 import _cabi
    _cabi.load()
    return torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _release_memory():
    """Every case frees its tensors before the next one (the GPU is shared; the largest case needs a few GB)."""
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


# ---------------------------------------------------------------- mirror of the wgrad host code ------------------------
def wgrad_plan(npix, kcols, cout, sms):
    """wgrad_geom, pick_wgrad_splits and the split fix-up and split-lane choice of tp_conv_wgrad (tp_igemm.cu) for a
    GEMM that contracts ``npix`` pixels into a [cout, kcols] weight gradient (kcols = R*S*Cin of the descriptor)."""
    chunks = (kcols + 63) // 64
    nb = min(chunks, 4)
    tiles = ((cout + 127) // 128) * ((chunks + nb - 1) // nb)
    kblocks = (npix + 63) // 64
    smax = max(1, min(kblocks, 2 * sms // tiles))
    c_kb, c_part, c_fin = 0.30, 0.33 * nb, 0.013 * nb
    best, best_cost = 1, 1e30
    for s in range(1, smax + 1):
        kb = (kblocks + s - 1) // s
        s_eff = (kblocks + kb - 1) // kb
        items = tiles * s_eff
        waves = (items + sms - 1) // sms
        cost = waves * (kb * c_kb + c_part) + items * c_fin
        if cost < best_cost - 1e-9:
            best_cost, best = cost, s_eff
    kbps = (kblocks + best - 1) // best
    splits = (kblocks + kbps - 1) // kbps
    sl = 8 if splits >= 64 else (4 if splits >= 32 else (2 if splits >= 16 else 1))
    return SimpleNamespace(nb=nb, tiles=tiles, kblocks=kblocks, smax=smax, splits=splits, kbps=kbps,
                           last=kblocks - (splits - 1) * kbps, sl=sl,
                           ws_bytes=tiles * smax * 128 * nb * 64 * 4 + 1024)


def _assert_plan(plan, want, sms):
    """``want`` = (splits, sl, K blocks per split, K blocks of the last split) on a 132-SM H100; elsewhere the case must
    still reach the same finalize path (split lanes) and the same raggedness of the last split."""
    got = (plan.splits, plan.sl, plan.kbps, plan.last)
    if sms == H100_SMS:
        assert got == want, (got, want)
    else:
        assert plan.sl == want[1] and (plan.last < plan.kbps) == (want[3] < want[2]), (sms, got, want)


# ---------------------------------------------------------------- operands and comparisons ------------------------------
def _ints(g, shape, lo, hi, dev):
    """bf16 tensor of integers in [lo, hi] (exact in bf16 for |v| <= 256)."""
    return torch.randint(lo, hi + 1, shape, generator=g, device=dev, dtype=torch.int16).to(torch.bfloat16)


def _signs(g, shape, dev):
    return (torch.randint(0, 2, shape, generator=g, device=dev, dtype=torch.int16) * 2 - 1).float()


def _exact(t, quantum):
    """Round a float64 result to its quantum: the float64 convolution algorithms may leave tiny errors, the exact value
    is a multiple of the quantum."""
    return torch.round(t / quantum) * quantum


def _bounded(S, quantum, what):
    s = float(S.max()) / quantum
    assert s <= EXACT, f"{what}: S = {s:.0f} quanta > 2^22, the operands do not keep every fp32 partial sum exact"


def _same(got, want, S, what):
    """got (bf16 / fp32 kernel output) == want (float64 exact reference, already rounded to got's dtype), as values."""
    bad = got.float() != want.float()
    nbad = int(bad.sum())
    if nbad:
        lines = []
        for i in bad.nonzero()[:8].tolist():
            i = tuple(i)
            a, b = float(got[i]), float(want[i])
            lines.append(f"  at {i}: kernel {a!r}, exact {b!r}, difference {a - b!r}, S {float(S[i]) if S is not None else '-'}")
        pytest.fail(f"{what}: {nbad} of {bad.numel()} elements differ from the exact result\n" + "\n".join(lines))


def _per_batch(n, elems_per_image, budget=1 << 25):
    """Batch slices whose float64 tensors stay around ``budget`` elements."""
    per = max(1, budget // max(1, elems_per_image))
    return [slice(i, min(n, i + per)) for i in range(0, n, per)]


def _nchw64(t):
    return t.permute(0, 3, 1, 2).double().contiguous()


def _check_row_stats(y, stats, what):
    """Per-32-row statistics of the conv epilogue ([rows, 2, C]: per 32 consecutive output pixels the sum and the sum
    of squares of the stored bf16 outputs) equal float64 sums of the stored y, bit for bit.  Rows past the last output
    pixel (the rest of the last 128-pixel tile) are zero.  Precondition: every sum of squares is below 2^24."""
    C = y.shape[-1]
    yf = y.reshape(-1, C)
    M, rows = yf.shape[0], stats.shape[0]
    assert rows * 32 >= M and rows % 4 == 0
    step = max(4, (1 << 19) // C)
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        seg = torch.zeros((r1 - r0) * 32, C, dtype=torch.float64, device=y.device)
        p0, p1 = r0 * 32, min(M, r1 * 32)
        if p1 > p0:
            seg[:p1 - p0] = yf[p0:p1].double()
        seg = seg.view(-1, 32, C)
        s1, s2 = seg.sum(1), (seg * seg).sum(1)
        assert float(s2.max()) < 2.0 ** 24, f"{what}: a 32-row sum of squares is not exact in fp32"
        _same(stats[r0:r1, 0], s1, None, f"{what}: per-row sum")
        _same(stats[r0:r1, 1], s2, None, f"{what}: per-row sum of squares")


def _kblock_walks(dead):
    """K-block skipping on and off when the mask has empty 64x64 blocks; otherwise both walks are the dense one."""
    return (True, False) if dead else (True,)


def _kill_blocks(m, dead):
    """Structured zeros in the mask.  'blocks': some 64x64 weight blocks of the fprop and dgrad operands are empty, every
    wgrad output tile keeps live entries.  'tile': additionally a whole 128 x 256 wgrad output tile is empty (its
    work items are skipped, the finalize writes zeros without reading partials)."""
    cout, cin = m.shape[:2]
    if dead == "blocks":
        m[:64, :64, 0, 0] = 0                       # fprop: output group 0 loses K block 0; dgrad: input group 0 loses a tap
        m[64:128, :, -1, -1] = 0                    # output group 1 loses the last tap (every channel block of it)
    elif dead == "tile":
        m[:, 64:128] = 0                            # fprop K block 1 empty; dgrad rows 64..127 have no block at all
        m[:, 256:] = 0                              # wgrad N tile 1 (K columns 256..511) empty for every output channel


# ---------------------------------------------------------------- masked convolutions ----------------------------------
# (id, n, hw, cin, cout, k, stride, pad, magnitude of x / dy, weight exponent e, bias, dgrad addend, structured zeros,
#  ops checked (f = fprop + epilogue statistics, d = dgrad, w = wgrad + bias gradient), wgrad plan on 132 SMs)
CONV_CASES = [
    # ResNet-50 layer 1 at a per-GPU batch of 64: one wgrad tile, 131 splits, sl = 8, last split 16 of 24 blocks
    ("l1.1x1.64-64.b64", 64, 56, 64, 64, 1, 1, 0, 1, 0, True, True, None, "fdw", (131, 8, 24, 16)),
    ("l1.1x1.256-64.b64", 64, 56, 256, 64, 1, 1, 0, 1, 0, False, False, None, "fdw", (131, 8, 24, 16)),
    # occupancy mask under sl = 8: fprop / dgrad skip blocks, one of the two wgrad tiles is skipped whole
    ("l1.1x1.512-64.b64.empty-tile", 64, 56, 512, 64, 1, 1, 0, 1, 0, False, True, "tile", "fdw", (66, 8, 48, 16)),
    ("l1.3x3.64.b64", 64, 56, 64, 64, 3, 1, 1, 1, 0, True, False, "blocks", "fdw", (44, 4, 72, 40)),
    ("l2.3x3.128.b64", 64, 28, 128, 128, 3, 1, 1, 1, 0, False, True, None, "fdw", (26, 2, 31, 9)),
    # strided: im2col walk with stride 2 (fprop, wgrad), four parity classes (dgrad)
    ("l2.3x3.128.s2.b64", 64, 56, 128, 128, 3, 2, 1, 1, 0, True, True, None, "fdw", (26, 2, 31, 9)),
    # the train step's own extent: 25 088 K blocks, 571 per split; fprop ~95 work items per CTA
    ("l1.3x3.64.b512", 512, 56, 64, 64, 3, 1, 1, 1, 0, False, False, None, "fw", (44, 4, 571, 535)),
    # P*Q = 49 < 64: K blocks cross images, 1813 pixels = 28 blocks + a 21-pixel tail, one split of 29 blocks
    ("l4.3x3.512.n37", 37, 7, 512, 512, 3, 1, 1, 1, 0, True, True, None, "fdw", (1, 1, 29, 29)),
    # the two remaining k_igemm_wgrad instantiations (2 and 3 column chunks per tile; 1 and 4 are above)
    ("nb2.1x1.128-64", 16, 28, 128, 64, 1, 1, 0, 1, 0, True, False, None, "fdw", (49, 4, 4, 4)),
    ("nb3.1x1.192-64", 16, 28, 192, 64, 1, 1, 0, 1, 0, False, True, None, "fdw", (40, 4, 5, 1)),
    # rounding: |outputs| up to thousands in quanta of 1/4, so bf16 round-to-nearest-even and exact ties are exercised
    ("round.3x3.64", 8, 56, 64, 64, 3, 1, 1, 64, -2, True, True, "blocks", "fd", (28, 2, 14, 14)),
    ("round.1x1.128-256.s2", 8, 28, 128, 256, 1, 2, 0, 64, -2, True, True, None, "fd", (13, 1, 2, 1)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_masked_conv_exact(dev, case):
    """fprop (+ bias, + the epilogue's per-row BatchNorm statistics), dgrad (+ the fused addend) and wgrad (+ the bias
    gradient) of one masked convolution equal the exact result bit for bit, with K-block skipping on and off.  The
    split-K workspace is filled with NaN before every wgrad call, so a partial tile that is read without having been
    written shows up."""
    from turboprune_b200 import ops
    lib = ops._cabi.load()
    name, n, hw, cin, cout, k, st, pad, mag, e, has_bias, has_add, dead, which, want_plan = case
    sms = _sms()
    desc = ops.make_desc(n, hw, hw, cin, cout, k, k, (st, st), (pad, pad))
    plan = wgrad_plan(n * desc.p * desc.q, k * k * cin, cout, sms)
    assert lib.tp_conv_workspace_bytes(ctypes.byref(desc), 2) == plan.ws_bytes
    _assert_plan(plan, want_plan, sms)
    assert plan.kblocks == (n * desc.p * desc.q + 63) // 64
    if n == 512:
        items, _ = _fprop_items(n, hw, cout, k, k, st, pad)
        assert 95 * sms <= items < 96 * sms, (items, sms)

    g = torch.Generator(device=dev).manual_seed(sum(case[1:8]) + mag)
    x = _ints(g, (n, hw, hw, cin), -mag, mag, dev)
    w = _signs(g, (cout, cin, k, k), dev) * 2.0 ** e
    m = (torch.rand(cout, cin, k, k, generator=g, device=dev) < 0.5).float()
    _kill_blocks(m, dead)
    bias = torch.randint(-8, 9, (cout,), generator=g, device=dev).float() if has_bias else None
    dy = _ints(g, (n, desc.p, desc.q, cout), -mag, mag, dev)
    add = _ints(g, (n, hw, hw, cin), -8, 8, dev) if has_add else None
    quantum = 2.0 ** min(e, 0)

    outs = {}
    for skip in _kblock_walks(dead):
        ops.set_kblock_skip(skip)
        try:
            wf, wd = ops.stage_weights(w, m, cin, "d" in which, cout)
            if dead and skip:
                assert ops.kblock_occupancy(wf.kmask, wf.shape[1])[0] > 0
                assert wd is None or ops.kblock_occupancy(wd.kmask, wd.shape[1])[0] > 0
            o = {}
            if "f" in which:
                o["y"], o["stats"] = ops.conv_fprop(desc, x, wf, bias, want_stats=True)
            if "d" in which:
                o["dx"] = ops.conv_dgrad(desc, dy, wd, addend=add)
            if "w" in which:
                wsb = ops._workspace(lib.tp_conv_workspace_bytes(ctypes.byref(desc), 2), dev, "wgrad")
                wsb[: wsb.numel() // 4 * 4].view(torch.float32).fill_(float("nan"))
                o["dw"], o["db"] = ops.conv_wgrad(desc, x, dy, m, cin, want_db=has_bias, kmask=wf.kmask if skip else None)
            outs[skip] = o
            del wf, wd
        finally:
            ops.set_kblock_skip(True)

    wm = (w * m).double()
    dw_ref = torch.zeros(cout, cin, k, k, dtype=torch.float64, device=dev)
    dw_s = torch.zeros_like(dw_ref)
    db_ref = torch.zeros(cout, dtype=torch.float64, device=dev)
    for sl in _per_batch(n, hw * hw * max(cin, cout)):
        x64 = _nchw64(x[sl])
        dy64 = _nchw64(dy[sl])
        if "f" in which:
            S = F.conv2d(x64.abs(), wm.abs(), None, st, pad)
            _bounded(S, quantum, "fprop")
            ref = _exact(F.conv2d(x64, wm, None, st, pad), quantum)
            if has_bias:
                ref += bias.double().view(1, -1, 1, 1)
            ref = ref.permute(0, 2, 3, 1).to(torch.bfloat16)
            S = S.permute(0, 2, 3, 1)
            for skip, o in outs.items():
                _same(o["y"][sl], ref, S, f"{name} fprop (K-block skipping {skip})")
            del S, ref
        if "d" in which:
            S = conv2d_input(x64.shape, wm.abs(), dy64.abs(), st, pad)
            _bounded(S, quantum, "dgrad")
            ref = _exact(conv2d_input(x64.shape, wm, dy64, st, pad), quantum)
            if has_add:
                ref += _nchw64(add[sl])
            ref = ref.permute(0, 2, 3, 1).to(torch.bfloat16)
            S = S.permute(0, 2, 3, 1)
            for skip, o in outs.items():
                _same(o["dx"][sl], ref, S, f"{name} dgrad (K-block skipping {skip})")
            del S, ref
        if "w" in which:
            dw_ref += conv2d_weight(x64, w.shape, dy64, st, pad)
            dw_s += conv2d_weight(x64.abs(), w.shape, dy64.abs(), st, pad)
            db_ref += dy64.sum(dim=(0, 2, 3))
        del x64, dy64
    if "w" in which:
        _bounded(dw_s, 1.0, "wgrad")
        dw_ref = _exact(dw_ref, 1.0) * m.double()
        db_s = dy.abs().double().sum(dim=(0, 1, 2))
        _bounded(db_s, 1.0, "bias gradient")
        for skip, o in outs.items():
            _same(o["dw"], dw_ref, dw_s, f"{name} wgrad (K-block skipping {skip})")
            if has_bias:
                _same(o["db"], db_ref, db_s, f"{name} bias gradient")
    if "f" in which and mag == 1 and e == 0:
        for skip, o in outs.items():
            _check_row_stats(o["y"], o["stats"], f"{name} epilogue statistics (K-block skipping {skip})")


# ---------------------------------------------------------------- stems and linear layers through autograd --------------
# (id, layer kind, batch, input extent, cin, cout, k, stride, pad, bias, wgrad plan on 132 SMs, chunks of the wgrad GEMM)
LAYER_CASES = [
    # ImageNet stem: explicit im2col (K = 147 padded to 152 columns = 3 chunks, the last one partial), plain-GEMM wgrad
    ("stem.7x7.s2.224", "stem", 16, 224, 3, 64, 7, 2, 3, False, (131, 8, 24, 16), 3),
    # CIFAR stem: K = 27 padded to 32 columns, one partial chunk
    ("stem.3x3.32", "stem", 64, 32, 3, 64, 3, 1, 1, True, (128, 8, 8, 8), 1),
    # ResNet-50 fc (Conv1dMask): 1000 outputs = 7 full 128-row tiles + 104 rows, 8 K blocks in one split
    ("fc.2048-1000.b512", "conv1d", 512, None, 2048, 1000, 1, 1, 0, True, (1, 1, 8, 8), 32),
    # DeiT-S qkv (LinearMask) over 8 x 197 tokens: 1576 rows = 12 full M tiles + 40 rows, 25 K blocks in 3 splits
    ("deit.qkv.384-1152", "linear", 8 * 197, None, 384, 1152, 1, 1, 0, True, (3, 1, 9, 7), 6),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LAYER_CASES, ids=[c[0] for c in LAYER_CASES])
def test_masked_layer_exact(dev, case):
    """The stems and the linear layers through the layers' own autograd path (ops.masked_conv2d / masked_linear): the
    output, the input gradient (not computed for a stem), the weight gradient and the bias gradient equal the exact
    result bit for bit."""
    from turboprune_b200 import ops
    from turboprune_b200.utils.mask_layers import Conv1dMask, LinearMask
    name, kind, n, hw, cin, cout, k, st, pad, has_bias, want_plan, want_chunks = case
    sms = _sms()
    g = torch.Generator(device=dev).manual_seed(cin + cout + n)
    if kind == "stem":
        p = (hw + 2 * pad - k) // st + 1
        kcols = ops.stem_geometry(cin, k, k)[1]
        npix = n * p * p
    else:
        kcols, npix = cin, n
    plan = wgrad_plan(npix, kcols, cout, sms)
    assert (kcols + 63) // 64 == want_chunks
    _assert_plan(plan, want_plan, sms)

    w = _signs(g, (cout, cin, k, k), dev)
    m = (torch.rand(cout, cin, k, k, generator=g, device=dev) < 0.5).float()
    b = torch.randint(-8, 9, (cout,), generator=g, device=dev).float() if has_bias else None
    if kind == "stem":
        x = _ints(g, (n, cin, hw, hw), -1, 1, dev).float()          # fp32 input: the stem converts while gathering
        wp = w.clone().requires_grad_(True)
        bp = b.clone().requires_grad_(True) if has_bias else None
        y = ops.masked_conv2d(x, wp, m, bp, (st, st), (pad, pad))
        dy = _ints(g, tuple(y.shape), -1, 1, dev).contiguous(memory_format=torch.channels_last)
        y.backward(dy)
        gw, gb, gx = wp.grad, (bp.grad if has_bias else None), None
        x64, dy64, wm = x.double(), dy.double(), (w * m).double()
        S = F.conv2d(x64.abs(), wm.abs(), None, st, pad)
        y_ref = _exact(F.conv2d(x64, wm, None, st, pad), 1.0)
        dw64 = conv2d_weight(x64, w.shape, dy64, st, pad)
        dw_s = conv2d_weight(x64.abs(), w.shape, dy64.abs(), st, pad)
        dx_ref = dx_s = None
    else:
        layer = (Conv1dMask(cin, cout, bias=has_bias) if kind == "conv1d" else LinearMask(in_features=cin, out_features=cout,
                                                                                          bias=has_bias)).to(dev)
        with torch.no_grad():
            layer.weight.copy_(w.view(layer.weight.shape))
            if has_bias:
                layer.bias.copy_(b)
        layer.mask = m.view(layer.weight.shape).clone()
        shape = (8, 197, cin) if kind == "linear" else (n, cin)
        x = _ints(g, shape, -1, 1, dev).requires_grad_(True)
        y = layer(x)
        dy = _ints(g, tuple(y.shape), -1, 1, dev)
        y.backward(dy)
        gw, gb, gx = layer.weight.grad.view(cout, cin, 1, 1), (layer.bias.grad if has_bias else None), x.grad
        x64, dy64 = x.detach().reshape(-1, cin).double(), dy.reshape(-1, cout).double()
        wm = (w * m).double().view(cout, cin)
        S = x64.abs() @ wm.abs().t()
        y_ref = _exact(x64 @ wm.t(), 1.0)
        dx_ref, dx_s = _exact(dy64 @ wm, 1.0), dy64.abs() @ wm.abs()
        dw64 = (dy64.t() @ x64).view(cout, cin, 1, 1)
        dw_s = (dy64.abs().t() @ x64.abs()).view(cout, cin, 1, 1)
        y, gx = y.reshape(-1, cout), gx.reshape(-1, cin)
    if has_bias:
        y_ref += b.double().view(1, -1, *([1, 1] if kind == "stem" else []))
    _bounded(S, 1.0, "fprop")
    _same(y.detach(), y_ref.to(torch.bfloat16), S, f"{name} output")
    if dx_ref is not None:
        _bounded(dx_s, 1.0, "dgrad")
        _same(gx, dx_ref.to(torch.bfloat16), dx_s, f"{name} input gradient")
    _bounded(dw_s, 1.0, "wgrad")
    _same(gw, _exact(dw64, 1.0) * m.double(), dw_s, f"{name} weight gradient")
    assert float(gw[m == 0].abs().max()) == 0.0
    if has_bias:
        dims = (0, 2, 3) if kind == "stem" else (0,)
        db_s = dy64.abs().sum(dim=dims)
        _bounded(db_s, 1.0, "bias gradient")
        _same(gb, dy64.sum(dim=dims), db_s, f"{name} bias gradient")


def test_wgrad_plan_mirror_on_h100():
    """The mirror of the wgrad host code gives every case above the plan it is meant to reach on a 132-SM H100 (the GPU
    tests check the mirror against the library's own workspace size on the device they run on)."""
    for c in CONV_CASES:
        _, n, hw, cin, cout, k, st, pad = c[:8]
        pq = (hw + 2 * pad - k) // st + 1
        plan = wgrad_plan(n * pq * pq, k * k * cin, cout, H100_SMS)
        assert (plan.splits, plan.sl, plan.kbps, plan.last) == c[-1], c[0]
    for c in LAYER_CASES:
        name, kind, n, hw, cin, cout, k, st, pad = c[:9]
        if kind == "stem":
            pq = (hw + 2 * pad - k) // st + 1
            plan = wgrad_plan(n * pq * pq, (k * k * cin + 7) // 8 * 8, cout, H100_SMS)
        else:
            plan = wgrad_plan(n, cin, cout, H100_SMS)
        assert (plan.splits, plan.sl, plan.kbps, plan.last) == c[-2], name
    # the paths the tables claim: every split-lane count of the finalize, ragged last splits, every chunk count
    plans = [c[-1] for c in CONV_CASES] + [c[-2] for c in LAYER_CASES]
    assert {p[1] for p in plans} == {1, 2, 4, 8}
    assert any(p[1] == 8 and p[3] < p[2] for p in plans)
    assert {min(4, (c[5] * c[5] * c[3] + 63) // 64) for c in CONV_CASES} == {1, 2, 3, 4}


# ---------------------------------------------------------------- BatchNorm statistics at training M ---------------------
def _bf16_ulp(v):
    """Spacing of bf16 numbers at |v| (float64 tensor): 2^(exponent - 8) with |v| = mantissa * 2^exponent, mantissa in [0.5, 1)."""
    _, ex = torch.frexp(v.abs())
    return torch.ldexp(torch.ones_like(v), ex - 8)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


@pytest.mark.gpu
def test_batchnorm_statistics_at_training_extent(dev):
    """conv (3x3, 64 -> 64, batch 512 at 56 x 56, integer operands and an integer bias per channel that puts |mean| / std
    between 0 and about 30) with the epilogue statistics, then BatchNorm folded from those rows (tp_bn_forward_ext) and
    BatchNorm with its own two-pass statistics (tp_bn_forward) of the same stored y.

    - Every per-row entry equals the float64 sums of the stored bf16 y bit for bit (each sum of squares < 2^24).
    - Against float64 statistics of the stored y, per channel: |mean error| <= 1e-5 (|mean| + std); relative error of
      invstd <= 1e-4 where |mean| / std <= 8 and <= 1e-3 up to 32; every z = relu(y * scale + shift) within one bf16 ulp
      of the float64 result (the BatchNorm shift is 8, so |z| >= 0.5 and an ulp is a relative bar)."""
    from turboprune_b200 import ops
    lib = ops._cabi.load()
    n, hw, c, k = 512, 56, 64, 3
    g = torch.Generator(device=dev).manual_seed(512)
    desc = ops.make_desc(n, hw, hw, c, c, k, k, (1, 1), (1, 1))
    x = _ints(g, (n, hw, hw, c), -1, 1, dev)
    w = _signs(g, (c, c, k, k), dev)
    m = (torch.rand(c, c, k, k, generator=g, device=dev) < 0.5).float()
    std_est = (k * k * c * (2 / 3) * 0.5) ** 0.5
    bias = torch.round(torch.linspace(0, 30, c, device=dev) * std_est * torch.where(torch.arange(c, device=dev) % 2 == 0, 1.0, -1.0))
    wf, _ = ops.stage_weights(w, m, c, False, c)
    y, stats = ops.conv_fprop(desc, x, wf, bias, want_stats=True)
    del x, wf
    _check_row_stats(y, stats, "epilogue statistics")

    M = n * hw * hw
    yf = y.view(M, c)
    s1 = torch.zeros(c, dtype=torch.float64, device=dev)
    for r in range(0, M, 1 << 18):
        s1 += yf[r:r + (1 << 18)].double().sum(0)
    mean = s1 / M
    var = torch.zeros_like(mean)
    for r in range(0, M, 1 << 18):
        var += ((yf[r:r + (1 << 18)].double() - mean) ** 2).sum(0)
    var /= M
    std = var.sqrt()
    ratio = mean.abs() / std
    assert float(ratio.min()) < 1 and 25 < float(ratio.max()) <= 32, ratio
    eps = float(torch.tensor(1e-5, dtype=torch.float32))
    invstd = 1.0 / torch.sqrt(var + eps)
    bn_w = torch.ones(c, device=dev)
    bn_b = torch.full((c,), 8.0, device=dev)
    ws = torch.empty(int(lib.tp_bn_workspace_bytes(M, c)), dtype=torch.uint8, device=dev)
    worst = {}
    for path in ("epilogue rows", "two-pass"):
        z = torch.empty_like(y)
        save_mean, save_invstd = torch.empty(c, device=dev), torch.empty(c, device=dev)
        rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        with torch.cuda.device(dev):
            if path == "epilogue rows":
                rc = lib.tp_bn_forward_ext(_ptr(y), None, _ptr(z), M, c, _ptr(bn_w), _ptr(bn_b), _ptr(rm), _ptr(rv), None, 0.1, 1e-5,
                                           1, 1, _ptr(save_mean), _ptr(save_invstd), _ptr(stats), stats.shape[0], _ptr(ws),
                                           ws.numel(), ops._cabi.stream_ptr(dev))
            else:
                rc = lib.tp_bn_forward(_ptr(y), None, _ptr(z), M, c, _ptr(bn_w), _ptr(bn_b), _ptr(rm), _ptr(rv), None, 0.1, 1e-5,
                                       1, 1, _ptr(save_mean), _ptr(save_invstd), _ptr(ws), ws.numel(), ops._cabi.stream_ptr(dev))
        ops._cabi.check(rc, path)
        dmean = (save_mean.double() - mean).abs() / (mean.abs() + std)
        dinv = (save_invstd.double() - invstd).abs() / invstd
        zerr = torch.zeros((), dtype=torch.float64, device=dev)
        zf = z.view(M, c)
        for r in range(0, M, 1 << 18):
            z64 = (yf[r:r + (1 << 18)].double() - mean) * invstd + 8.0
            assert float(z64.min()) >= 0.5
            zerr = torch.maximum(zerr, ((zf[r:r + (1 << 18)].double() - z64).abs() / _bf16_ulp(z64)).max())
        worst[path] = (float(dmean.max()), float(dinv[ratio <= 8].max()), float(dinv.max()), float(zerr))
        print(f"[batchnorm statistics, {path}] worst |dmean|/(|mean|+std) {worst[path][0]:.3g}, invstd rel. error "
              f"{worst[path][1]:.3g} (|mean|/std <= 8), {worst[path][2]:.3g} (all, max |mean|/std {float(ratio.max()):.1f}), "
              f"z {worst[path][3]:.3g} ulp")
    for path, (dm, di8, di, dz) in worst.items():
        assert dm <= 1e-5, (path, dm)
        assert di8 <= 1e-4 and di <= 1e-3, (path, di8, di)
        assert dz <= 1.0, (path, dz)


# ---------------------------------------------------------------- fused BatchNorm-backward dgrad epilogue ------------------
BNB_CASES = [("l1.1x1.256-64", 256, 56, 256, 64, 1), ("l1.3x3.64", 256, 56, 64, 64, 3), ("l3.3x3.256", 256, 14, 256, 256, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", BNB_CASES, ids=[c[0] for c in BNB_CASES])
def test_bn_backward_dgrad_epilogue_exact(dev, case):
    """ops.conv_dgrad_bnrelu: dgrad of a convolution whose input is a BatchNorm+ReLU output, with the BatchNorm backward
    reduction in its epilogue.  BatchNorm weight, bias, mean and invstd are small dyadic numbers (means on a 1/4 grid,
    so y == mean ties occur; invstd a power of two), which makes the ReLU gate fma(y, scale, shift) > 0 and
    g * (y - mean) * invstd exact in fp32.

    - g = dx * [gate] and every per-32-row partial (sum g, sum g * xhat) equal the float64 reference bit for bit.
    - tp_bn_backward_ext from those partials: dgamma and dbeta within 1e-5 relative of the float64 sums (relative to
      sum |g * xhat| and sum |g| of the channel; with dy >= 0, positive weights and a zero BatchNorm bias every term of a
      channel has one sign, and there the bar is relative to the value itself); the BatchNorm input gradient dy within
      2^-8 |reference| plus one bf16 ulp of the largest of its three terms k0 g, k1 y, k2, per element."""
    bnb_dgrad_check(dev, case)


def bnb_dgrad_check(dev, case):
    """The checks of test_bn_backward_dgrad_epilogue_exact for one (id, n, hw, cin, cout, k) case."""
    from turboprune_b200 import ops
    lib = ops._cabi.load()
    name, n, hw, cin, cout, k = case
    g_ = torch.Generator(device=dev).manual_seed(cin * k + hw)
    desc = ops.make_desc(n, hw, hw, cin, cout, k, k, (1, 1), (k // 2, k // 2))
    M = n * hw * hw
    dy = (torch.rand(n, hw, hw, cout, generator=g_, device=dev) < 0.25).to(torch.bfloat16)
    w = torch.ones(cout, cin, k, k, device=dev)
    m = (torch.rand(cout, cin, k, k, generator=g_, device=dev) < 0.5).float()
    _, wd = ops.stage_weights(w, m, cin, True, cout)
    y = _ints(g_, (n, hw, hw, cin), -8, 8, dev)
    pick = lambda vals: torch.tensor(vals, device=dev)[torch.randint(0, len(vals), (cin,), generator=g_, device=dev)]
    bn_w = pick([-1.0, 0.5, 1.0, 1.5, 2.0])
    bn_b = pick([0.0, 0.0, 0.125, -0.25])
    bn_mean = torch.randint(-8, 9, (cin,), generator=g_, device=dev).float() / 4
    bn_inv = pick([0.125, 0.25, 0.5])
    out = ops.conv_dgrad_bnrelu(desc, dy, wd, (y, bn_w, bn_b, bn_mean, bn_inv))
    assert out is not None, "the fused path must exist for this shape"
    g, partial = out
    rows = partial.shape[0]
    assert rows * 32 >= M

    sc = bn_w.double() * bn_inv.double()
    sf = bn_b.double() - bn_mean.double() * sc
    assert torch.equal(sc.float().double(), sc) and torch.equal(sf.float().double(), sf)       # scale, shift exact in fp32
    wm = (w * m).double()
    g_ref = torch.empty_like(g)
    for sl in _per_batch(n, hw * hw * max(cin, cout)):
        dy64 = _nchw64(dy[sl])
        shape = (dy64.shape[0], cin, hw, hw)
        dx_s = conv2d_input(shape, wm.abs(), dy64.abs(), 1, k // 2)
        _bounded(dx_s, 1.0, "dgrad")
        dx = _exact(conv2d_input(shape, wm, dy64, 1, k // 2), 1.0).permute(0, 2, 3, 1).to(torch.bfloat16)
        y64 = y[sl].double()
        g_ref[sl] = torch.where(y64 * sc + sf > 0, dx.double(), 0.0).to(torch.bfloat16)
        _same(g[sl], g_ref[sl], dx_s.permute(0, 2, 3, 1), f"{name} gated gradient g")
        del dy64, dx_s, dx, y64

    gf, yf = g_ref.view(M, cin), y.view(M, cin)
    mean64, inv64 = bn_mean.double(), bn_inv.double()
    sums = torch.zeros(4, cin, dtype=torch.float64, device=dev)        # sum g, sum g*xhat, sum |g|, sum |g*xhat|
    step = max(1, (1 << 19) // cin)
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        p0, p1 = r0 * 32, min(M, r1 * 32)
        gg = torch.zeros((r1 - r0) * 32, cin, dtype=torch.float64, device=dev)
        xh = torch.zeros_like(gg)
        if p1 > p0:
            gg[:p1 - p0] = gf[p0:p1].double()
            xh[:p1 - p0] = (yf[p0:p1].double() - mean64) * inv64
        gx = gg * xh
        s_row = gx.abs().view(-1, 32, cin).sum(1)
        _bounded(s_row, 2.0 ** -5, "sum g * xhat per 32 rows")         # xhat is a multiple of 1/32
        _same(partial[r0:r1, 0], gg.view(-1, 32, cin).sum(1), None, f"{name} partial sum g")
        _same(partial[r0:r1, 1], gx.view(-1, 32, cin).sum(1), s_row, f"{name} partial sum g * xhat")
        sums += torch.stack([gg.sum(0), gx.sum(0), gg.abs().sum(0), gx.abs().sum(0)])
        del gg, xh, gx

    dyb = torch.empty_like(y)
    dgamma, dbeta = torch.empty(cin, device=dev), torch.empty(cin, device=dev)
    ws = torch.empty(int(lib.tp_bn_workspace_bytes(M, cin)), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = lib.tp_bn_backward_ext(_ptr(g), _ptr(y), M, cin, _ptr(bn_w), _ptr(bn_b), _ptr(bn_mean), _ptr(bn_inv), _ptr(partial),
                                    rows, _ptr(dyb), _ptr(dgamma), _ptr(dbeta), _ptr(ws), ws.numel(), ops._cabi.stream_ptr(dev))
    ops._cabi.check(rc, "tp_bn_backward_ext")
    sg, sgx, sga, sgxa = sums
    assert float(((dbeta.double() - sg).abs() / sga.clamp_min(1e-30)).max()) <= 1e-5
    assert float(((dgamma.double() - sgx).abs() / sgxa.clamp_min(1e-30)).max()) <= 1e-5
    k0 = bn_w.double() * inv64
    k1 = -k0 * inv64 * (sgx / M)
    k2 = -k0 * (sg / M) - k1 * mean64
    worst, step = 0.0, (1 << 24) // cin
    for p0 in range(0, M, step):
        gg, yy = gf[p0:p0 + step].double(), yf[p0:p0 + step].double()
        ref = k0 * (gg - sg / M - (yy - mean64) * inv64 * (sgx / M))
        terms = torch.maximum(torch.maximum((k0 * gg).abs(), (k1 * yy).abs()), k2.abs().expand_as(gg))
        err = (dyb.view(M, cin)[p0:p0 + step].double() - ref).abs() / (2.0 ** -8 * ref.abs() + _bf16_ulp(terms))
        worst = max(worst, float(err.max()))
    assert worst <= 1.0, worst
